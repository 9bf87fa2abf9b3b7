"""Pins the oracle's RNG against the reference's own known-answer test
(the reference's boltzmann_machines/rbm/tests/test_rbm.py:52-67)."""
import numpy as np
from numpy.testing import assert_almost_equal

from oracle import philox as P


def test_philox_block_vector():
    # counter (0,0,1337,0), key (87654321,0): the block behind the reference KAT
    w = P.philox4x32_10(0, 0, 1337, 0, 87654321, 0)
    assert [int(x) for x in w] == [0x371b9c90, 0xb9746224, 0xcd9caac4, 0x59978421]


def test_reference_init_kat_float32_and_float64():
    W32 = P.tf_random_normal((12, 8), 0.01, 1337, 'float32')
    W64 = P.tf_random_normal((12, 8), 0.01, 1337, 'float64')
    assert W32.dtype == np.float32 and W64.dtype == np.float64
    assert_almost_equal(W32[0][0], -0.0094548017)        # test_rbm.py:65
    assert_almost_equal(W64[0][0], -0.0077341544416)     # test_rbm.py:67


def test_c_accelerator_matches_numpy():
    a = P.site_words(37, 1021, 0x123456789abc, 3, 5, 9, row0=11, use_c=False)
    b = P.site_words(37, 1021, 0x123456789abc, 3, 5, 9, row0=11, use_c=True)
    assert (a == b).all()


def test_uniform_range_and_rows_independent_of_shape():
    u = P.uniform_at(64, 100, 7, P.SITE_H, 2, 5)
    assert u.dtype == np.float32 and u.min() >= 0 and u.max() < 1
    # a sub-block drawn with a row offset equals the slice of the big draw
    v = P.uniform_at(16, 40, 7, P.SITE_H, 2, 5, row0=8)
    assert (v == u[8:24, :40]).all()
    assert abs(u.mean() - 0.5) < 0.02


def test_normals_moments():
    z = P.normal_at(256, 512, 99, P.SITE_V, 1, 0)
    assert abs(z.mean()) < 0.01 and abs(z.std() - 1) < 0.01
