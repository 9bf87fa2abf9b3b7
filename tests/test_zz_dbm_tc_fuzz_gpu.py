"""Random ragged configurations of the tensor-core DBM engine on the GPU against the bf16 emulation oracle: the checker of
tools/fuzz_dbm_tc_hostsim.py (training steps, queries, AIS), run on the kernels themselves instead of their CPU
interpretation."""
import numpy as np
import pytest

from tools.fuzz_dbm_tc_hostsim import draw, one

pytestmark = pytest.mark.gpu

SEEDS = range(40)


def test_random_tc_dbm_models_on_the_gpu():
    """No seed may fail.  'mf-count' (a mean-field sweep count one apart: a change within bf16 rounding of mf_tol) and
    'sample-flip' (a uniform within rounding of its probability) end a seed early without a verdict; at most a quarter of
    the seeds may end so."""
    outcomes, failures = {}, []
    for seed in SEEDS:
        cfg, run = draw(np.random.RandomState(seed))
        try:
            r = one(cfg, run, seed)
        except Exception as e:             # noqa: BLE001 -- collect every failing seed, then fail once
            r = 'FAIL'
            failures.append('seed {0}: {1}'.format(seed, ' '.join(str(e).split())[:300]))
        outcomes[r] = outcomes.get(r, 0) + 1
    print('\n[dbm-tc-fuzz] outcomes of {0} seeds: {1}'.format(len(SEEDS), outcomes))
    assert not failures, '\n'.join(failures)
    assert outcomes.get('mf-count', 0) + outcomes.get('sample-flip', 0) <= len(SEEDS) // 4, outcomes
