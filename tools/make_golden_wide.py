"""Generate tests/golden/wide/*.npz by executing the Wide & Deep wide part (WideAndDeep/wide_and_deep.py:121-122 and
:208-210) over the TF1 shim.

    python tools/make_golden_wide.py /path/to/RecAlgorithm/algorithm      (or set RECALG_REFERENCE)

The cited lines are read from the reference checkout at generation time and exec()'d eagerly: lines 121-122 build
`cross_userid_manualtag_indicator` from the categorical columns `userid` and `manual_tag_list`, and lines 208-210 run
`fc.input_layer` over it and `tf.layers.dense(wide_input, 1, name="wide_part_variables")` under
`tf.variable_scope("wide_part", reuse=tf.AUTO_REUSE)`.  The shared shim (oracle/tf1_shim) provides variable_scope (reuse
accepted), AUTO_REUSE and layers.dense.  It has no feature columns, so the `fc` those lines call is defined here, for this
run only, with TF 1.14 semantics (SURVEY A.11):
- categorical columns map each string through their vocabulary (id = line number, -1 out of vocabulary);
- crossed_column takes the keys, hash_bucket_size and hash_key (None or 0 -> 0xDECAFCAFFE), and is named by the sorted key
  names joined by "_X_"; indicator_column appends "_indicator";
- input_layer builds the (B, hash_bucket_size) multi-hot LITERALLY: for every sample, every element of the Cartesian product
  of the keys' ids (last key fastest; none if a key is empty) is hashed by the FingerprintCat64 chain on Python integers and
  counts +1 in its bucket.
The kernel is injected (tests/_wide_ref.fixture_kernel, regenerated from a per-fixture seed rather than stored) with a
non-zero bias; the block runs in float32 and float64 and must create exactly wide_part/wide_part_variables/kernel
(100000, 1) and .../bias (1,).  The backward of dense(1) is the multi-hot transposed times an upstream gradient g, taken
from the same literal multi-hot in float64.  A fixture stores the two vocabularies, each key's strings per sample (flat +
offsets), the column name, hash_bucket_size, the kernel seed and the SHA-256 of the kernel, bias, g, the logits and
d_kernel.  tests/golden/wide/reference_digests.json holds the SHA-256 of every array (tests/test_wide_golden.py checks
them, and re-runs this script when RECALG_REFERENCE is set).
"""
from __future__ import annotations

import hashlib
import itertools
import json
import os
import sys
import textwrap

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "wide")
REF = os.environ.get("RECALG_REFERENCE", "")
M64 = (1 << 64) - 1

sys.path.insert(0, os.path.join(ROOT, "oracle", "tf1_shim"))
import tensorflow as tf  # noqa: E402  (the shim)

assert "tf1_shim" in tf.__file__, "the TF shim must shadow any real tensorflow"
sys.path.insert(0, os.path.join(ROOT, "tests"))
from _wide_ref import fixture_kernel  # noqa: E402

# (name, B, tags per sample (max), userid vocabulary size, tag vocabulary size, seed, tags parse empty)
CASES = (("wide_B16", 16, 5, 10, 12, 1, False), ("wide_B64", 64, 12, 40, 30, 2, False),
         ("wide_B8_no_tags", 8, 0, 10, 12, 3, True))


def _fingerprint_cat64(a, b):
    kmul = 0xc6a4a7935bd1e995
    mix = lambda x: x ^ (x >> 47)
    r = a ^ kmul
    r ^= (mix((b * kmul) & M64) * kmul) & M64
    r = (r * kmul) & M64
    r = (mix(r) * kmul) & M64
    return mix(r)


class _Categorical:
    def __init__(self, key, tokens):
        self.key, self.name = key, key
        self.table = {t: i for i, t in reversed(list(enumerate(tokens)))}

    def ids(self, strings):
        return [self.table.get(s, -1) for s in strings]


class _Crossed:
    def __init__(self, keys, hash_bucket_size, hash_key=None):
        if not hash_bucket_size or hash_bucket_size < 1:
            raise ValueError("hash_bucket_size must be > 1")
        if len(keys) < 2:
            raise ValueError("keys must be a list with length > 1")
        self.keys, self.hash_bucket_size = list(keys), int(hash_bucket_size)
        self.hash_key = hash_key if hash_key else 0xDECAFCAFFE
        self.name = "_X_".join(sorted(k.name for k in self.keys))


class _Indicator:
    def __init__(self, col):
        self.categorical_column, self.name = col, col.name + "_indicator"


class _WideFC:
    """tf.feature_column as lines 121-122 and 208-210 use it (indicator columns of crossed columns only)."""
    crossed_column = _Crossed
    indicator_column = _Indicator

    @staticmethod
    def input_layer(features, feature_columns):
        blocks = []
        for col in sorted(feature_columns, key=lambda c: c.name):
            cross = col.categorical_column
            per_key = [features[k.key] for k in cross.keys]
            B = len(per_key[0])
            hot = np.zeros((B, cross.hash_bucket_size), tf._STATE.dtype)
            for b in range(B):
                for combo in itertools.product(*(k.ids(rows[b]) for k, rows in zip(cross.keys, per_key))):
                    h = cross.hash_key
                    for v in combo:
                        h = _fingerprint_cat64(h, v & M64)
                    hot[b, h % cross.hash_bucket_size] += 1
            blocks.append(hot)
        return tf.Tensor(np.concatenate(blocks, axis=1))


def _ref_lines(first, last, must):
    with open(os.path.join(REF, "WideAndDeep", "wide_and_deep.py"), encoding="utf-8") as fh:
        lines = fh.read().split("\n")[first - 1:last]
    assert must[0] in lines[0] and must[1] in lines[-1], (lines[0], lines[-1])
    return compile(textwrap.dedent("\n".join(lines)), f"WideAndDeep/wide_and_deep.py:{first}-{last}", "exec")


def run_wide(features, userid, manual_tag_list, variables, dtype):
    tf.reset(dtype=dtype, variables=variables)
    ns = {"fc": _WideFC, "tf": tf, "userid": userid, "manual_tag_list": manual_tag_list}
    exec(_ref_lines(121, 122, ("crossed_column([userid, manual_tag_list]", "indicator_column(cross_userid_manualtag)")), ns)
    col = ns["cross_userid_manualtag_indicator"]
    ns.update({"features": features, "params": {"wide_part_feature_columns": [col]}})
    exec(_ref_lines(208, 210, ('variable_scope("wide_part"', 'name="wide_part_variables"')), ns)
    return np.asarray(tf._arr(ns["wide_input"])), np.asarray(tf._arr(ns["wide_logit"])), col, tf.created_variables()


def digest(a):
    return f"{a.dtype.str}:{'x'.join(map(str, a.shape))}:{hashlib.sha256(a.tobytes()).hexdigest()}"


def _ragged(rows):
    flat = np.array([s for r in rows for s in r], dtype="S16").reshape(-1)
    return flat, np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)


def gen_wide(out_dir=OUT):
    os.makedirs(out_dir, exist_ok=True)
    digests = {}
    for name, B, max_tags, n_uid, n_tag, seed, no_tags in CASES:
        rng = np.random.default_rng(1000 + seed)
        uid_vocab = [b"userid_%d" % i for i in range(n_uid)]
        tag_vocab = [b"tag_%d" % i for i in range(n_tag)]
        # strings drawn from a slightly larger range than the vocabularies: some are out of vocabulary (id -1)
        uid = [[b"userid_%d" % int(rng.integers(0, n_uid + 3))] for _ in range(B)]
        tags = [[] if no_tags else [b"tag_%d" % int(t) for t in rng.integers(0, n_tag + 3, int(rng.integers(0, max_tags + 1)))]
                for _ in range(B)]
        userid, manual_tag_list = _Categorical("userid", uid_vocab), _Categorical("manual_tag_list", tag_vocab)
        nb = 100000
        kernel = fixture_kernel(nb, seed).reshape(nb, 1)
        bias = np.array([0.375], np.float32)
        g = (rng.integers(-64, 65, B) / 64).astype(np.float32)
        variables = {"wide_part/wide_part_variables/kernel": kernel, "wide_part/wide_part_variables/bias": bias}
        arrays = {"hash_bucket_size": np.array(nb, np.int64), "kernel_seed": np.array(seed, np.int64), "bias": bias, "g": g}
        features = {"userid": uid, "manual_tag_list": tags}
        for tag, dt in (("f32", np.float32), ("f64", np.float64)):
            hot, logit, col, created = run_wide(features, userid, manual_tag_list, variables, dt)
            assert created == {"wide_part/wide_part_variables/kernel": (nb, 1), "wide_part/wide_part_variables/bias": (1,)}, created
            assert col.categorical_column.hash_bucket_size == nb and hot.shape == (B, nb) and logit.shape == (B, 1)
            arrays["wide_logit_" + tag] = logit.astype(dt)
        arrays["d_kernel_f64"] = hot.astype(np.float64).T @ g.astype(np.float64)
        arrays["column_name"] = np.array(col.name)
        arrays["kernel_sha256"] = np.array(hashlib.sha256(kernel.tobytes()).hexdigest())
        arrays["userid_vocab"], arrays["manual_tag_list_vocab"] = np.array(uid_vocab, "S16"), np.array(tag_vocab, "S16")
        arrays["userid_values"], arrays["userid_offsets"] = _ragged(uid)
        arrays["manual_tag_list_values"], arrays["manual_tag_list_offsets"] = _ragged(tags)
        arrays["source"] = np.array("reference-executed:WideAndDeep/wide_and_deep.py:121-122,208-210")
        path = os.path.join(out_dir, name + ".npz")
        np.savez_compressed(path, **arrays)
        z = np.load(path, allow_pickle=False)
        digests[name + ".npz"] = {k: digest(z[k]) for k in z.files}
        print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB, {int((hot > 0).sum())} buckets hit")
    return digests


if __name__ == "__main__":
    if len(sys.argv) > 1:
        REF = sys.argv[1]
    assert os.path.isdir(REF), "usage: make_golden_wide.py <reference checkout>/algorithm (or set RECALG_REFERENCE)"
    d = gen_wide()
    with open(os.path.join(OUT, "reference_digests.json"), "w") as fh:
        json.dump(d, fh, indent=1, sort_keys=True)
        fh.write("\n")
