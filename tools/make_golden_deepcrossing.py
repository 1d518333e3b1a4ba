"""Generate tests/golden/deepcrossing/*.npz by executing DeepCrossing's residual module (DeepCrossing/deepcrossing.py:154-157)
over the TF1 shim, with the reference's residual_unit imported verbatim from DeepCrossing/residual_unit.py.

    python tools/make_golden_deepcrossing.py /path/to/RecAlgorithm/algorithm      (or set RECALG_REFERENCE)

residual_unit.py only uses tf.layers.dense, tf.nn.relu and get_shape(), which the shared shim (oracle/tf1_shim) provides with
TensorFlow 1.x semantics (dense variables <name>/kernel and <name>/bias, bias initialised to zeros).  Each case injects seeded
weights under the reference's variable names, runs the loop in float32 and float64, and checks that the loop created exactly
the variables residual_unit's signature implies.  tests/golden/deepcrossing/reference_digests.json holds the SHA-256 of every
array (tests/test_deepcrossing_oracle.py checks them, and re-runs this script when RECALG_REFERENCE is set).
"""
from __future__ import annotations

import hashlib
import importlib.util
import json
import os
import sys
import textwrap

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "deepcrossing")
REF = os.environ.get("RECALG_REFERENCE", "")
CASES = ((82, 256, 2, 16), (82, 128, 1, 16), (5, 3, 3, 9))     # (d, H, units, B): the best result.md row first

sys.path.insert(0, os.path.join(ROOT, "oracle", "tf1_shim"))
import tensorflow as tf  # noqa: E402  (the shim)

assert "tf1_shim" in tf.__file__, "the TF shim must shadow any real tensorflow"


def _load_residual_unit():
    spec = importlib.util.spec_from_file_location("deepcrossing_residual_unit",
                                                  os.path.join(REF, "DeepCrossing", "residual_unit.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.residual_unit


def run_module(residual_unit, x, variables, dtype, H, units):
    tf.reset(dtype=dtype, variables=variables)
    ns = {"tf": tf, "residual_unit": residual_unit, "concat_all": tf.Tensor(x.astype(dtype)),
          "params": {"residual_network_num": units, "residual_internal_dim": H}}
    with open(os.path.join(REF, "DeepCrossing", "deepcrossing.py"), encoding="utf-8") as fh:
        lines = fh.read().split("\n")[153:157]                    # lines 154-157
    assert 'tf.variable_scope("residual_module")' in lines[0] and "residual_unit(net" in lines[-1], (lines[0], lines[-1])
    exec(compile(textwrap.dedent("\n".join(lines)), "DeepCrossing/deepcrossing.py:154-157", "exec"), ns)
    return np.asarray(tf._arr(ns["net"])), tf.created_variables()


def names(i):
    return (("w0", f"residual_module/dense_{i}_0/kernel"), ("b0", f"residual_module/dense_{i}_0/bias"),
            ("w1", f"residual_module/dense_{i}_1/kernel"), ("b1", f"residual_module/dense_{i}_1/bias"))


def digest(a):
    return f"{a.dtype.str}:{'x'.join(map(str, a.shape))}:{hashlib.sha256(a.tobytes()).hexdigest()}"


def gen_deepcrossing(out_dir=OUT):
    residual_unit = _load_residual_unit()
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(9186)
    digests = {}
    for d, H, units, B in CASES:
        x = (rng.standard_normal((B, d)) * 0.7).astype(np.float32)
        arrays, variables = {"x": x}, {}
        for i in range(units):
            w = {"w0": rng.uniform(-1, 1, (d, H)) * (6.0 / (d + H)) ** 0.5, "b0": rng.uniform(-0.1, 0.1, H),
                 "w1": rng.uniform(-1, 1, (H, d)) * (6.0 / (d + H)) ** 0.5, "b1": rng.uniform(-0.1, 0.1, d)}
            for k, n in names(i):
                arrays[f"{k}_{i}"] = w[k].astype(np.float32)
                variables[n] = arrays[f"{k}_{i}"]
        for tag, dt in (("f32", np.float32), ("f64", np.float64)):
            out, created = run_module(residual_unit, x, variables, dt, H, units)
            arrays["out_" + tag] = out.astype(dt)
            assert created == {n: variables[n].shape for i in range(units) for _, n in names(i)}, created
        arrays["source"] = np.array("reference-executed:DeepCrossing/deepcrossing.py:154-157 + DeepCrossing/residual_unit.py")
        name = f"deepcrossing_d{d}_H{H}_units{units}_B{B}"
        path = os.path.join(out_dir, name + ".npz")
        np.savez_compressed(path, **arrays)
        z = np.load(path, allow_pickle=False)
        digests[name + ".npz"] = {k: digest(z[k]) for k in z.files}
        print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB")
    # quirk: index=None names the variables dense_None_{0,1} (an f-string of None)
    tf.reset(dtype=np.float64)
    residual_unit(tf.Tensor(np.ones((2, 4))), 3, index=None)
    assert tf.created_variables() == {"dense_None_0/kernel": (4, 3), "dense_None_0/bias": (3,), "dense_None_1/kernel": (3, 4),
                                      "dense_None_1/bias": (4,)}, tf.created_variables()
    return digests


if __name__ == "__main__":
    if len(sys.argv) > 1:
        REF = sys.argv[1]
    assert os.path.isdir(REF), "usage: make_golden_deepcrossing.py <reference checkout>/algorithm (or set RECALG_REFERENCE)"
    d = gen_deepcrossing()
    with open(os.path.join(OUT, "reference_digests.json"), "w") as fh:
        json.dump(d, fh, indent=1, sort_keys=True)
        fh.write("\n")
