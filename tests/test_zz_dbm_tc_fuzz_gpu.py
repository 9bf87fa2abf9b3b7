"""Random ragged configurations of the tensor-core DBM engine on the GPU against the bf16 emulation oracle: the checker of
tools/fuzz_dbm_tc_hostsim.py (training steps, queries, AIS; every combination of the engine's switches), run on the kernels
themselves instead of their CPU interpretation."""
import os

import numpy as np
import pytest

from tools.fuzz_dbm_tc_hostsim import draw, one

pytestmark = pytest.mark.gpu

SEEDS = range(40)
SWITCHES = ('BM_DBM_TC_MIXED', 'BM_DBM_AIS_FUSED', 'BM_DBM_MF_CHUNK', 'BM_DBM_PCD_PROGRAM', 'BM_DBM_AIS_EPILOGUE')


def test_dbm_tc_fuzz_on_the_gpu():
    """No seed may fail.  'mf-count' (a mean-field sweep count one apart: a change within bf16 rounding of mf_tol) and
    'sample-flip' (a uniform within rounding of its probability) end a seed early without a verdict; at most a quarter of
    the seeds may end so."""
    saved = {k: os.environ.get(k) for k in SWITCHES}
    outcomes, failures = {}, []
    try:
        for seed in SEEDS:
            cfg, env, run = draw(np.random.RandomState(seed))
            try:
                r = one(cfg, env, run, seed)
            except Exception as e:             # noqa: BLE001 -- collect every failing seed, then fail once
                r = 'FAIL'
                failures.append('seed {0}: {1}'.format(seed, ' '.join(str(e).split())[:300]))
            outcomes[r] = outcomes.get(r, 0) + 1
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    print('\n[dbm-tc-fuzz] outcomes of {0} seeds: {1}'.format(len(SEEDS), outcomes))
    assert not failures, '\n'.join(failures)
    assert outcomes.get('mf-count', 0) + outcomes.get('sample-flip', 0) <= len(SEEDS) // 4, outcomes
