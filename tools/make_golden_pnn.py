"""Generate tests/golden/pnn/*.npz by executing the reference's PNN product layer (PNN/pnn.py:126-181) over the TF1 shim.

    python tools/make_golden_pnn.py /path/to/RecAlgorithm/algorithm      (or set RECALG_REFERENCE)

The cited lines are read from the reference checkout at generation time and exec()'d eagerly, with `fc.input_layer` returning
the injected per-column embeddings and a FLAGS stand-in for `embedding_dim`.  The block needs four TensorFlow 1.14 primitives
the shared shim (oracle/tf1_shim) does not provide; they are added to it here, for this run only:
  tf.matrix_band_part, tf.contrib.layers.l2_regularizer, get_variable(..., regularizer=) and a list `axis` in reduce_sum.
Each fixture stores the seeded inputs, the injected weights (TF names), the reference outputs in float32 and float64, and
the REGULARIZATION_LOSSES sum of a run at weight_regularizer = 0.01.  tests/golden/pnn/reference_digests.json holds the
SHA-256 of every array (tests/test_pnn_oracle.py checks them, and re-runs this script when RECALG_REFERENCE is set).
"""
from __future__ import annotations

import hashlib
import json
import os
import sys
import textwrap
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "pnn")
REF = os.environ.get("RECALG_REFERENCE", "")
CASES = ((8, 8, 128, 16), (5, 4, 24, 9))          # (F, K, output_dimension, batch)

sys.path.insert(0, os.path.join(ROOT, "oracle", "tf1_shim"))
import tensorflow as tf  # noqa: E402  (the shim)

assert "tf1_shim" in tf.__file__, "the TF shim must shadow any real tensorflow"

# ---- the four primitives PNN/pnn.py:126-181 needs on top of the shim (TF 1.14 semantics) ----
_REG_LOSSES = []


def matrix_band_part(a, num_lower, num_upper):
    """tf.matrix_band_part: keeps x[.., i, j] where (num_lower < 0 or i - j <= num_lower) and (num_upper < 0 or j - i <= num_upper)."""
    x = tf._arr(a)
    i = np.arange(x.shape[-2])[:, None]
    j = np.arange(x.shape[-1])[None, :]
    keep = ((num_lower < 0) | (i - j <= num_lower)) & ((num_upper < 0) | (j - i <= num_upper))
    return tf.Tensor(np.where(keep, x, 0).astype(x.dtype))


def l2_regularizer(scale, scope=None):
    """tf.contrib.layers.l2_regularizer: scale 0.0 -> a function returning None (no loss); else scale * sum(w**2) / 2."""
    if scale == 0.0:
        return lambda _: None
    return lambda w: tf.Tensor(tf._arr(w).dtype.type(scale) * np.sum(np.square(tf._arr(w))) / 2)


_get_variable = tf.get_variable


def get_variable(name, shape=None, dtype=None, initializer=None, regularizer=None):
    """get_variable(..., regularizer=): the regularizer's loss (if not None) goes to REGULARIZATION_LOSSES."""
    v = _get_variable(name, shape=shape, dtype=dtype, initializer=initializer)
    if regularizer is not None:
        loss = regularizer(v)
        if loss is not None:
            _REG_LOSSES.append(loss)
    return v


_reduce_sum = tf.reduce_sum


def reduce_sum(a, axis=None, keepdims=False):
    """tf.reduce_sum with a list of axes (numpy wants a tuple)."""
    return _reduce_sum(a, axis=tuple(axis) if isinstance(axis, list) else axis, keepdims=keepdims)


tf.matrix_band_part = matrix_band_part
tf.contrib.layers.l2_regularizer = staticmethod(l2_regularizer)
tf.get_variable = get_variable
tf.reduce_sum = reduce_sum


class _FakeFC:
    """`fc.input_layer(features, [col])` returns the (B, K) embedding injected for that column."""
    @staticmethod
    def input_layer(features, columns):
        return tf.concat([tf.Tensor(features[c]) for c in columns], axis=1)


def run_block(e, variables, dtype, product_method, output_dimension, weight_regularizer=0.0):
    B, F, K = e.shape
    cols = [f"c{f:02d}" for f in range(F)]
    tf.reset(dtype=dtype, variables=variables)
    _REG_LOSSES.clear()
    ns = {"tf": tf, "fc": _FakeFC, "FLAGS": types.SimpleNamespace(embedding_dim=K),
          "features": {c: e[:, f, :].astype(dtype) for f, c in enumerate(cols)},
          "params": {"category_feature_columns": cols, "output_dimension": output_dimension,
                     "product_method": product_method, "weight_regularizer": weight_regularizer}}
    with open(os.path.join(REF, "PNN", "pnn.py"), encoding="utf-8") as fh:
        lines = fh.read().split("\n")[125:181]                   # lines 126-181
    assert "fields_embeddings = []" in lines[0] and "product_final = tf.nn.relu" in lines[-1], (lines[0], lines[-1])
    exec(compile(textwrap.dedent("\n".join(lines)), "PNN/pnn.py:126-181", "exec"), ns)
    reg = float(sum(float(tf._arr(x)) for x in _REG_LOSSES))
    return ns, tf.created_variables(), reg


def glorot(rng, shape, fan_in, fan_out):
    lim = (6.0 / (fan_in + fan_out)) ** 0.5
    return rng.uniform(-lim, lim, size=shape).astype(np.float32)


def digest(a):
    return f"{a.dtype.str}:{'x'.join(map(str, a.shape))}:{hashlib.sha256(a.tobytes()).hexdigest()}"


def gen_pnn(out_dir=OUT):
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(9753)
    digests = {}
    for F, K, N, B in CASES:
        e = (np.clip(rng.standard_normal((B, F, K)), -2, 2) / np.sqrt(K)).astype(np.float32)
        for method in ("IPNN", "OPNN"):
            wshape = (N, F) if method == "IPNN" else (N, K, K)
            wname = "product_part/inner_product_w" if method == "IPNN" else "product_part/outer_product_w"
            fans = (N, F) if method == "IPNN" else (N * K, N * K)
            variables = {"linear_part/linear_w": glorot(rng, (F * K, N), F * K, N), wname: glorot(rng, wshape, *fans),
                         "bias": glorot(rng, (N,), N, N)}
            outs = {}
            for tag, dt in (("f32", np.float32), ("f64", np.float64)):
                ns, created, _ = run_block(e, variables, dt, method, N)
                outs[tag] = np.asarray(tf._arr(ns["product_final"]))
            assert created == {"linear_part/linear_w": (F * K, N), wname: wshape, "bias": (N,)}, created
            _, _, reg = run_block(e, variables, np.float64, method, N, weight_regularizer=0.01)
            arrays = dict(e=e, linear_w=variables["linear_part/linear_w"], product_w=variables[wname], bias=variables["bias"],
                          out_f32=outs["f32"], out_f64=outs["f64"], reg_loss_scale_0_01=np.float64(reg),
                          source=np.array("reference-executed:PNN/pnn.py:126-181"))
            name = f"pnn_{method.lower()}_F{F}_K{K}_N{N}"
            path = os.path.join(out_dir, name + ".npz")
            np.savez_compressed(path, **arrays)
            z = np.load(path, allow_pickle=False)
            digests[name + ".npz"] = {k: digest(z[k]) for k in z.files}
            print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB")
    # quirk: any product_method other than the exact string "IPNN" takes the OPNN branch (:146,160)
    _, created, _ = run_block(np.zeros((1, 2, 3), np.float32), {}, np.float64, "ipnn", 4)
    assert "product_part/outer_product_w" in created and "product_part/inner_product_w" not in created
    return digests


if __name__ == "__main__":
    if len(sys.argv) > 1:
        REF = sys.argv[1]
    assert os.path.isdir(REF), "usage: make_golden_pnn.py <reference checkout>/algorithm (or set RECALG_REFERENCE)"
    d = gen_pnn()
    with open(os.path.join(OUT, "reference_digests.json"), "w") as fh:
        json.dump(d, fh, indent=1, sort_keys=True)
        fh.write("\n")
