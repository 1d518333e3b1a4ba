"""Generate tests/golden/mmoe/*.npz by executing MMoE's experts, gates and tower sums (MMOE/mmoe.py:207-236) over the TF1 shim.

    python tools/make_golden_mmoe.py /path/to/RecAlgorithm/algorithm      (or set RECALG_REFERENCE)

The cited lines are read from the reference checkout at generation time and exec()'d eagerly on `concat_all_input` and a
`params` dict.  They use tf.layers.dense (relu experts, softmax gates without bias), tf.concat, tf.expand_dims, tf.matmul
(transpose_a) and tf.squeeze, which the shared shim (oracle/tf1_shim) provides with TensorFlow 1.x semantics, and
`tf.newaxis`, which it does not: it is added here, for this run only, as TF defines it (None, numpy's new axis).
Each case injects seeded weights under the reference's variable names, runs the block in float32 and float64, and checks
that the block created exactly the expected variables.  The weights are small multiples of powers of two (exact in float32,
and compact in the archive).  A fixture stores x, the weights packed as the C ABI takes them -- w_experts (E,d,H),
b_experts (E,H), w_gates (T,d,E) -- and the reference's towers (T,B,H) and gates (T,B,E) in both precisions.
tests/golden/mmoe/reference_digests.json holds the SHA-256 of every array (tests/test_mmoe_oracle.py checks them, and re-runs
this script when RECALG_REFERENCE is set).
"""
from __future__ import annotations

import hashlib
import json
import os
import sys
import textwrap

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "mmoe")
REF = os.environ.get("RECALG_REFERENCE", "")
# (d, E, H, T, B): the reference default (mmoe.py:39-41), the widest result.md row, and E = 1 with ragged shapes
CASES = ((82, 3, 512, 3, 16), (82, 6, 1024, 3, 8), (5, 1, 7, 2, 9))

sys.path.insert(0, os.path.join(ROOT, "oracle", "tf1_shim"))
import tensorflow as tf  # noqa: E402  (the shim)

assert "tf1_shim" in tf.__file__, "the TF shim must shadow any real tensorflow"

tf.newaxis = None                    # tf.newaxis (TF 1.14: None), the one name MMOE/mmoe.py:207-236 needs on top of the shim


def run_block(x, variables, dtype, E, H, T):
    tf.reset(dtype=dtype, variables=variables)
    ns = {"tf": tf, "concat_all_input": tf.Tensor(x.astype(dtype)),
          "params": {"num_experts": E, "expert_hidden_units": H, "num_tasks": T}}
    with open(os.path.join(REF, "MMOE", "mmoe.py"), encoding="utf-8") as fh:
        lines = fh.read().split("\n")[206:236]                    # lines 207-236
    assert "# experts" in lines[0] and "towers.append(tower)" in lines[-1], (lines[0], lines[-1])
    exec(compile(textwrap.dedent("\n".join(lines)), "MMOE/mmoe.py:207-236", "exec"), ns)
    towers = np.stack([np.asarray(tf._arr(t)) for t in ns["towers"]])
    gates = np.stack([np.asarray(tf._arr(g)) for g in ns["gates"]])
    return towers, gates, tf.created_variables()


def names(E, T):
    return ([f"experts/expert_{i}/kernel" for i in range(E)], [f"experts/expert_{i}/bias" for i in range(E)],
            [f"gates/gate_{t}/kernel" for t in range(T)])


def digest(a):
    return f"{a.dtype.str}:{'x'.join(map(str, a.shape))}:{hashlib.sha256(a.tobytes()).hexdigest()}"


def gen_mmoe(out_dir=OUT):
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(2071)
    digests = {}
    for d, E, H, T, B in CASES:
        x = (rng.standard_normal((B, d)) * 0.7).astype(np.float32)
        we = (rng.integers(-26, 27, (E, d, H)) / 256).astype(np.float32)         # ~ glorot-uniform scale at d = 82, H = 512
        be = (rng.integers(-25, 26, (E, H)) / 256).astype(np.float32)
        wg = (rng.integers(-64, 65, (T, d, E)) / 128).astype(np.float32)          # gates far from uniform
        kn, bn, gn = names(E, T)
        variables = {**{n: we[i] for i, n in enumerate(kn)}, **{n: be[i] for i, n in enumerate(bn)},
                     **{n: wg[t] for t, n in enumerate(gn)}}
        arrays = {"x": x, "w_experts": we, "b_experts": be, "w_gates": wg}
        for tag, dt in (("f32", np.float32), ("f64", np.float64)):
            towers, gates, created = run_block(x, variables, dt, E, H, T)
            assert towers.shape == (T, B, H) and gates.shape == (T, B, E), (towers.shape, gates.shape)
            arrays["towers_" + tag] = towers.astype(dt)
            arrays["gates_" + tag] = gates.astype(dt)
            want = {**{n: (d, H) for n in kn}, **{n: (H,) for n in bn}, **{n: (d, E) for n in gn}}
            assert created == want, created
        arrays["source"] = np.array("reference-executed:MMOE/mmoe.py:207-236")
        name = f"mmoe_d{d}_E{E}_H{H}_T{T}_B{B}"
        path = os.path.join(out_dir, name + ".npz")
        np.savez_compressed(path, **arrays)
        z = np.load(path, allow_pickle=False)
        digests[name + ".npz"] = {k: digest(z[k]) for k in z.files}
        print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB")
    return digests


if __name__ == "__main__":
    if len(sys.argv) > 1:
        REF = sys.argv[1]
    assert os.path.isdir(REF), "usage: make_golden_mmoe.py <reference checkout>/algorithm (or set RECALG_REFERENCE)"
    d = gen_mmoe()
    with open(os.path.join(OUT, "reference_digests.json"), "w") as fh:
        json.dump(d, fh, indent=1, sort_keys=True)
        fh.write("\n")
