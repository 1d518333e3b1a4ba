"""Generate tests/golden/ple/*.npz by executing PLE's extraction network (PLE/extraction_network.py) and final experts and
gates (PLE/ple.py:185-226) over the TF1 shim.

    python tools/make_golden_ple.py /path/to/RecAlgorithm/algorithm      (or set RECALG_REFERENCE)

At generation time the extraction network is imported from the reference checkout, and the cited lines of ple.py are read
and exec()'d eagerly on `input` and a `params` dict.  They use tf.layers.dense (relu experts, softmax gates without bias),
tf.variable_scope, tf.concat, tf.expand_dims, tf.matmul (transpose_a), tf.squeeze and tf.add_n, which the shared shim
(oracle/tf1_shim) provides with TensorFlow 1.x semantics, and `tf.newaxis`, which it does not: it is added here, for this
run only, as TF defines it (None, numpy's new axis).
Each case injects seeded weights under the reference's variable names, runs the block in float32 and float64, and records
the names of the variables the block created, in creation order.  The weights are integer multiples of a power of two
(exact in float32) drawn from a counter-based hash of a per-fixture seed (tests/_ple_ref.py's fixture_weights), so a
fixture stores the seed instead of the weights, which keeps the archives small.  tests/_ple_ref.py's fixture() rebuilds
them in the packed layout the C ABI takes: w_experts (E,d,H) and b_experts (E,H) in [task 0 .. task T-1, shared] order, and
w_gates (d,GC), the gate kernels concatenated by columns.  A fixture also stores the SHA-256 of those weights, so that a
change to the hash is caught.
tests/golden/ple/reference_digests.json holds the SHA-256 of every array (tests/test_ple_oracle.py checks them).
"""
from __future__ import annotations

import hashlib
import json
import os
import sys
import textwrap

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "ple")
REF = os.environ.get("RECALG_REFERENCE", "")
TASKS = ("read_comment", "like", "click_avatar")
# (mode, d, n, S, H, B): the default result.md row (1 extraction network at the input width, then the final layer at
# d = H), the widest row's final layer, and a ragged small case in both modes
CASES = (("extraction", 82, (5, 5, 5), 10, 256, 8), ("final", 256, (5, 5, 5), 10, 256, 8),
         ("final", 256, (10, 10, 10), 20, 256, 4),
         ("extraction", 5, (2, 1), 1, 7, 9), ("final", 5, (2, 1), 1, 7, 9))

sys.path.insert(0, os.path.join(ROOT, "tests"))
from _ple_ref import fixture_weights  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "oracle", "tf1_shim"))
import tensorflow as tf  # noqa: E402  (the shim)

assert "tf1_shim" in tf.__file__, "the TF shim must shadow any real tensorflow"

tf.newaxis = None                    # tf.newaxis (TF 1.14: None), the one name the PLE blocks need on top of the shim


def names(mode, n, S, tasks):
    """(expert kernel/bias name prefixes in packed order, gate kernel names in column order)."""
    if mode == "extraction":
        p = "extract_network_0/"
        experts = [f"{p}task_specific_expert_{t}_{i}" for t, nt in zip(tasks, n) for i in range(nt)]
        experts += [f"{p}shared_expert_{i}" for i in range(S)]
        gates = [f"{p}gate_{t}/kernel" for t in tasks] + [f"{p}all_gate/kernel"]
    else:
        experts = [f"task_specific_experts_final/task_specific_expert_final_{t}_{i}" for t, nt in zip(tasks, n)
                   for i in range(nt)]
        experts += [f"shared_experts_final/shared_expert_final_{i}" for i in range(S)]
        gates = [f"task_specific_experts_final/task_gate_final/gate_final_{t}/kernel" for t in tasks]
    return experts, gates


def run_block(mode, x, variables, dtype, n, S, H, tasks):
    tf.reset(dtype=dtype, variables=variables)
    if mode == "extraction":
        sys.path.insert(0, os.path.join(REF, "PLE"))
        try:
            import extraction_network as xn
        finally:
            sys.path.pop(0)
        out = xn.extraction_network(input=tf.Tensor(x.astype(dtype)), task_names=list(tasks), num_experts_per_task=list(n),
                                    num_experts_in_shared=S, expert_hidden_units=H, name="extract_network_0")
        out = np.asarray(tf._arr(out))
    else:
        ns = {"tf": tf, "input": tf.Tensor(x.astype(dtype)), "task_tower_inputs": [],
              "params": {"task_names": list(tasks), "num_experts_per_task": list(n), "num_experts_in_shared": S,
                         "expert_hidden_units": H}}
        with open(os.path.join(REF, "PLE", "ple.py"), encoding="utf-8") as fh:
            lines = fh.read().split("\n")[184:226]                # lines 185-226
        assert "shared_experts_final" in lines[0] and "task_tower_inputs.append" in lines[-1], (lines[0], lines[-1])
        exec(compile(textwrap.dedent("\n".join(lines)), "PLE/ple.py:185-226", "exec"), ns)
        out = np.stack([np.asarray(tf._arr(t)) for t in ns["task_tower_inputs"]])
    return out, list(tf.created_variables().items())


def digest(a):
    return f"{a.dtype.str}:{'x'.join(map(str, a.shape))}:{hashlib.sha256(a.tobytes()).hexdigest()}"


def weights_digest(we, be, wg):
    return hashlib.sha256(b"".join(np.ascontiguousarray(a, np.float64).tobytes() for a in (we, be, wg))).hexdigest()


def gen_ple(out_dir=OUT):
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(2077)
    digests = {}
    for case, (mode, d, n, S, H, B) in enumerate(CASES):
        tasks = TASKS[:len(n)]
        E = sum(n) + S
        widths = [nt + S for nt in n] + ([E] if mode == "extraction" else [])
        x = (rng.standard_normal((B, d)) * 0.7).astype(np.float32)
        seed = 1000 * (case + 1)
        w64 = fixture_weights(seed, E, d, H, sum(widths))
        we, be, wg = (a.astype(np.float32) for a in w64)
        experts, gate_names = names(mode, n, S, tasks)
        variables = {**{f"{p}/kernel": we[e] for e, p in enumerate(experts)},
                     **{f"{p}/bias": be[e] for e, p in enumerate(experts)}}
        cols = np.cumsum([0] + widths)
        variables.update({nm: wg[:, cols[g]:cols[g + 1]] for g, nm in enumerate(gate_names)})
        arrays = {"x": x, "weight_seed": np.array(seed, np.int64), "weights_sha256": np.array(weights_digest(*w64)),
                  "experts_per_task": np.array(n, np.int64),
                  "num_experts_in_shared": np.array(S, np.int64), "extraction": np.array(mode == "extraction")}
        for tag, dt in (("f32", np.float32), ("f64", np.float64)):
            out, created = run_block(mode, x, variables, dt, n, S, H, tasks)
            want_shape = (B, H) if mode == "extraction" else (len(n), B, H)
            assert out.shape == want_shape, out.shape
            arrays["out_" + tag] = out.astype(dt)
            assert {k for k, _ in created} == set(variables), {k for k, _ in created} ^ set(variables)
            arrays["variables"] = np.array([k for k, _ in created])
            arrays["variable_shapes"] = np.array([list(s) + [0] * (2 - len(s)) for _, s in created], np.int64)
        arrays["source"] = np.array("reference-executed:" + ("PLE/extraction_network.py:4-85" if mode == "extraction"
                                                             else "PLE/ple.py:185-226"))
        name = f"ple_{mode}_d{d}_n{'-'.join(map(str, n))}_S{S}_H{H}_B{B}"
        path = os.path.join(out_dir, name + ".npz")
        np.savez_compressed(path, **arrays)
        z = np.load(path, allow_pickle=False)
        digests[name + ".npz"] = {k: digest(z[k]) for k in z.files}
        print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB")
    return digests


if __name__ == "__main__":
    if len(sys.argv) > 1:
        REF = sys.argv[1]
    assert os.path.isdir(REF), "usage: make_golden_ple.py <reference checkout>/algorithm (or set RECALG_REFERENCE)"
    d = gen_ple()
    with open(os.path.join(OUT, "reference_digests.json"), "w") as fh:
        json.dump(d, fh, indent=1, sort_keys=True)
        fh.write("\n")
