"""CPU tests of the NumPy restatement of the Wide & Deep wide part (tests/_wide_ref.py): the crossed-column hash pinned by a
table and by an independent Python-integer restatement, the cross enumeration, and TF's dense ApplyFtrl on hand-checked
cases."""
import math

import numpy as np
import pytest

import _wide_ref as R

M64 = (1 << 64) - 1

# (vocabulary ids of the keys, num_buckets, bucket).  Computed from the FingerprintCat64 chain of SURVEY A.11; a TensorFlow
# run of sparse_cross_hashed on the same int64 ids would confirm them.
PINNED = (
    ((0, 0), 100000, 71304),
    ((1, 2), 100000, 1357),
    ((2, 1), 100000, 9716),
    ((-1, 5), 100000, 49399),
    ((5, -1), 100000, 84240),
    ((123456, 7), 100000, 33806),
    ((0, 0, 0), 100000, 48447),
    ((3, 1, 4, 1), 100000, 86697),
    ((7, 9), 10000000, 7365746),
    ((-1, -1), 2, 1),
    ((42, 17), 2147483647, 753125615),
)


def _py_bucket(ids, num_buckets, hash_key=R.HASH_KEY):
    """The same chain on Python integers (masking every product to 64 bits)."""
    kmul = 0xc6a4a7935bd1e995
    mix = lambda x: x ^ (x >> 47)
    h = hash_key
    for v in ids:
        r = h ^ kmul
        r ^= (mix((v & M64) * kmul & M64) * kmul) & M64
        r = (r * kmul) & M64
        r = (mix(r) * kmul) & M64
        h = mix(r)
    return h % num_buckets


@pytest.mark.parametrize("ids,num_buckets,bucket", PINNED)
def test_cross_hash_pinned(ids, num_buckets, bucket):
    assert int(R.cross_bucket(np.array([ids]), num_buckets)[0]) == bucket
    assert _py_bucket(ids, num_buckets) == bucket


def test_cross_hash_matches_python_integers_on_random_ids():
    rng = np.random.default_rng(0)
    for K in (2, 3, 4):
        ids = rng.integers(-1, 1 << 40, (200, K))
        nb = int(rng.integers(2, 1 << 31))
        got = R.cross_bucket(ids, nb)
        assert got.tolist() == [_py_bucket(row.tolist(), nb) for row in ids]
    assert R.cross_bucket(np.array([[1, 2]]), 100, hash_key=7)[0] == _py_bucket([1, 2], 100, 7)


def test_cross_enumeration_order_and_empty_keys():
    """Cartesian product in key order, last key fastest; a sample with an empty key has no crosses; duplicates stay."""
    # key 0: s0 = [10, 11], s1 = [], s2 = [30];  key 1: s0 = [20, 21, 21], s1 = [40], s2 = []
    offsets = np.array([[0, 2, 2, 3], [3, 6, 7, 7]], np.int64)
    values = np.array([10, 11, 30, 20, 21, 21, 40], np.int64)
    nb = 1000
    got = R.crossed_ids(values, offsets, nb)
    want0 = [R.cross_bucket(np.array([[a, b]]), nb)[0] for a in (10, 11) for b in (20, 21, 21)]
    assert got[0].tolist() == want0 and len(got[1]) == 0 and len(got[2]) == 0
    hist = R.histogram(got, nb)
    assert hist.sum() == 6 and hist[want0[1]] >= 2
    k = np.arange(nb, dtype=np.float64)
    assert R.wide_fwd(got, k, 0.5).ravel().tolist() == [0.5 + sum(want0), 0.5, 0.5]
    dk, db = R.wide_bwd(got, [2.0, 3.0, 4.0], nb)
    assert db == 9.0 and np.array_equal(dk, 2.0 * hist)


def test_ftrl_hand_checked_step():
    """One element at TF's defaults (lr_power -0.5, accum 0.1, linear 0, l1 = l2 = 0), worked by hand."""
    lr, w, g = 0.005, 0.3, 0.2
    na = 0.1 + g * g
    lin = g - (math.sqrt(na) - math.sqrt(0.1)) / lr * w
    want = -lin / (math.sqrt(na) / lr)
    v, a, l = R.ftrl(np.array([w]), np.array([0.1]), np.array([0.0]), np.array([g]), lr)
    assert a[0] == pytest.approx(na, rel=1e-15) and l[0] == pytest.approx(lin, rel=1e-15) and v[0] == pytest.approx(want, rel=1e-15)


def test_ftrl_untouched_rows_become_zero_at_step_one():
    """With g = 0 and linear = 0 the new linear is exactly 0, so |linear| > l1 fails and var becomes 0 whatever it was."""
    var = np.array([0.0071, -0.0069, 0.0001, 0.0])
    v, a, l = R.ftrl(var, np.full(4, 0.1), np.zeros(4), np.zeros(4), 0.005)
    assert np.array_equal(v, np.zeros(4)) and np.array_equal(l, np.zeros(4)) and np.array_equal(a, np.full(4, 0.1))


def test_ftrl_l1_l2_and_power():
    """l1 shrinks |linear| by l1 and zeroes it inside [-l1, l1]; l2 adds 2*l2 to the denominator; a general power uses
    new_accum^-p."""
    lr, p = 0.1, -0.3
    var, acc, lin, g = np.array([0.5, 0.5]), np.array([0.2, 0.2]), np.array([0.0, 0.0]), np.array([0.4, 0.01])
    na = acc + g * g
    l_new = lin + g - (na ** 0.3 - acc ** 0.3) / lr * var
    l1, l2 = 0.05, 0.25
    v, a, l = R.ftrl(var, acc, lin, g, lr, p, l1, l2)
    assert np.allclose(l, l_new, rtol=1e-15)
    y = na ** 0.3 / lr + 2 * l2
    want = np.where(np.abs(l_new) > l1, (l1 * np.sign(l_new) - l_new) / y, 0.0)
    assert np.allclose(v, want, rtol=1e-15) and abs(l_new[1]) < l1 < abs(l_new[0]) and v[1] == 0.0 and v[0] != 0.0
