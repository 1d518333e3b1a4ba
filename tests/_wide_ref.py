"""NumPy restatement of the Wide & Deep wide part (WideAndDeep/wide_and_deep.py:121-122,208-210,254-257), independent of the
kernels: TF's crossed-column hash on vocabulary ids in uint64 arithmetic (SURVEY A.11), the wide logit and its dense kernel
gradient in float64 through an explicit list of crossed ids, and TF's dense ApplyFtrl in float64 (SURVEY A.12)."""
import itertools

import numpy as np

HASH_KEY = 0xDECAFCAFFE
_MUL = np.uint64(0xc6a4a7935bd1e995)


def _shift_mix(x):
    return x ^ (x >> np.uint64(47))


def fingerprint_cat64(a, b):
    """TF's FingerprintCat64, elementwise on uint64 arrays (wrapping multiplication)."""
    a, b = np.asarray(a, np.uint64), np.asarray(b, np.uint64)
    with np.errstate(over="ignore"):
        r = a ^ _MUL
        r = r ^ (_shift_mix(b * _MUL) * _MUL)
        r = r * _MUL
        r = _shift_mix(r) * _MUL
        return _shift_mix(r)


def cross_bucket(ids, num_buckets, hash_key=HASH_KEY):
    """Bucket of crosses: ids (..., K) int64 vocabulary ids (OOV -1 hashes as 2^64 - 1)."""
    ids = np.asarray(ids, np.int64)
    h = np.full(ids.shape[:-1], hash_key, np.uint64)
    for k in range(ids.shape[-1]):
        h = fingerprint_cat64(h, ids[..., k].astype(np.uint64))
    return (h % np.uint64(num_buckets)).astype(np.int64)


def crossed_ids(values, offsets, num_buckets, hash_key=HASH_KEY):
    """Per sample, the bucket of every cross: the Cartesian product of the keys' values, last key fastest (none when a key is
    empty).  values (nnz,), offsets (K, B+1) as ctr_crossed_indicator_fwd takes them.  Returns a list of int64 arrays."""
    values, offsets = np.asarray(values, np.int64), np.asarray(offsets, np.int64)
    K, B = offsets.shape[0], offsets.shape[1] - 1
    out = []
    for b in range(B):
        keys = [values[offsets[k, b]:offsets[k, b + 1]] for k in range(K)]
        prod = np.array(list(itertools.product(*keys)), np.int64).reshape(-1, K)
        out.append(cross_bucket(prod, num_buckets, hash_key) if len(prod) else np.zeros((0,), np.int64))
    return out


def wide_fwd(crosses, kernel, bias):
    """wide_logit[b] = bias + sum over b's crosses of kernel[id] (the multi-hot counts duplicates), float64, (B, 1)."""
    kernel = np.asarray(kernel, np.float64).reshape(-1)
    return np.array([[float(bias) + kernel[c].sum()] for c in crosses], np.float64).reshape(-1, 1)


def wide_bwd(crosses, d_logit, num_buckets):
    """Dense gradient multi_hot^T d_logit (num_buckets,) and d_bias = sum d_logit, float64."""
    d_logit = np.asarray(d_logit, np.float64).reshape(-1)
    dk = np.zeros(num_buckets, np.float64)
    for c, g in zip(crosses, d_logit):
        np.add.at(dk, c, g)
    return dk, float(d_logit.sum())


def histogram(crosses, num_buckets):
    """Number of crosses per bucket over the batch."""
    cat = np.concatenate(crosses) if crosses else np.zeros((0,), np.int64)
    return np.bincount(cat, minlength=num_buckets)


def ftrl(var, accum, linear, grad, lr, lr_power=-0.5, l1=0.0, l2=0.0):
    """TF's dense ApplyFtrl in float64; returns new (var, accum, linear)."""
    var, accum, linear, grad = (np.asarray(a, np.float64) for a in (var, accum, linear, grad))
    new_accum = accum + grad * grad
    p = -lr_power
    linear = linear + grad - (new_accum ** p - accum ** p) / lr * var
    y = new_accum ** p / lr + 2.0 * l2
    var = np.where(np.abs(linear) > l1, (l1 * np.sign(linear) - linear) / y, 0.0)
    return var, new_accum, linear


def fixture_kernel(num_buckets, seed):
    """The dense(1) kernel injected into a fixture run (tools/make_golden_wide.py), regenerated rather than stored: entry i is
    an integer in [-256, 256] over 4096 (exact in float32), drawn by the splitmix64 finaliser of seed + i * 0x9E3779B97F4A7C15
    in plain uint64 arithmetic."""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + np.arange(num_buckets, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return ((z % np.uint64(513)).astype(np.int64) - 256).astype(np.float32) / np.float32(4096)
