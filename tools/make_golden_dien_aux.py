"""Generate tests/golden/dien_aux/*.npz by executing DIEN's seq_encoder block (DIEN/dien.py:199-229) and then its auxiliary
loss (DIEN/dien.py:266-300) over the TF1 shim, with the shim modules, the restated dynamic_rnn / GRUCell and the reference's
verbatim AGRUCell / AUGRUCell taken from tools/make_golden_dien.py.

    python tools/make_golden_dien_aux.py /path/to/RecAlgorithm/algorithm      (or set RECALG_REFERENCE)

Three restatements, all recorded in every fixture:
  - line 265 reads ``pos_sequnence_input = sequnence_length[:, 1:, :]``, a slice of the (B,) length vector; the intent is the
    next behaviours ``sequnence_input[:, 1:, :]``, which is what the generator binds before executing :266-300;
  - line 283 reshapes neg_part (B, T-1, T_neg) back to (B, (T-1)*T_neg), after which :294 multiplies it by the
    (B, T-1, T_neg) mask (a broadcast TF rejects) and :298 sums it over axes [1, 2]; both later lines want the 3-D tensor,
    so line 283 is left out;
  - :266-300 run inside ``tf.variable_scope("aux_loss")`` (line 264), so the projection is ``aux_loss/aux_project_matrix``.
For this run only the shim gains tf.log, tf.sigmoid and a list ``axis`` in tf.reduce_sum.  The fixtures record the
reference's aux_loss as executed (its sign: a sum of log-likelihoods); the kernels compute its negative.  The inputs keep
every log term of the reference finite, at every position (a masked -inf would turn into NaN through -inf * 0).
tests/golden/dien_aux/reference_digests.json holds the SHA-256 of every array (tests/test_dien_aux_oracle.py checks them, and
re-runs this script when RECALG_REFERENCE is set).
"""
from __future__ import annotations

import json
import os
import sys
import textwrap

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden_dien as MG  # noqa: E402  (installs the shim path)

tf = MG.tf
ROOT = MG.ROOT
OUT = os.path.join(ROOT, "tests", "golden", "dien_aux")
CASES = ((16, 8, 50, 3, 16), (5, 3, 7, 2, 9))      # (na, nh, T, T_neg, B)
SLICE = "pos_sequnence_input = sequnence_input[:, 1:, :]"
RESHAPE = "neg_part = tf.reshape(neg_part, shape=(-1, (T-1)*T_neg))"

_reduce_sum = tf.reduce_sum


def reduce_sum(a, axis=None, keepdims=False):
    """tf.reduce_sum with a list of axes (numpy wants a tuple)."""
    return _reduce_sum(a, axis=tuple(axis) if isinstance(axis, list) else axis, keepdims=keepdims)


tf.reduce_sum = reduce_sum
tf.log = lambda x: tf.Tensor(np.log(tf._arr(x)))
tf.sigmoid = lambda x: tf.Tensor(1 / (1 + np.exp(-tf._arr(x))))


def run_aux(cells, seq, seq_len, tgt, neg, variables, dtype, custom_gru_type, nh, T_neg):
    """dien.py:199-229 (make_golden_dien.run_block), then :266-300 in the same namespace."""
    ns, _, _ = MG.run_block(cells, seq, seq_len, tgt, variables, dtype, custom_gru_type, nh)
    with open(os.path.join(MG.REF, "DIEN", "dien.py"), encoding="utf-8") as fh:
        src = fh.read().split("\n")
    assert 'tf.variable_scope("aux_loss")' in src[263] and "sequnence_length[:, 1:, :]" in src[264], (src[263], src[264])
    assert RESHAPE in src[282], src[282]
    lines = src[265:282] + src[283:300]                                 # lines 266-300 without 283
    assert "h_ = h[:, :-1, :]" in lines[0] and "aux_loss = tf.reduce_mean(pos_part+neg_part)" in lines[-1], (lines[0], lines[-1])
    ns["params"]["negative_sample_number"] = T_neg
    ns["neg_sequnence_input"] = tf.Tensor(neg.astype(dtype))
    ns["pos_sequnence_input"] = tf.Tensor(seq.astype(dtype)[:, 1:, :])  # the restated line 265
    with tf.variable_scope("aux_loss"):
        exec(compile(textwrap.dedent("\n".join(lines)), "DIEN/dien.py:266-300", "exec"), ns)
    return ns, tf.created_variables()


def gen_dien_aux(out_dir=OUT):
    cells = MG._load_cells()
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(5151)
    digests = {}
    for na, nh, T, T_neg, B in CASES:
        L = np.concatenate([[-1, 0, 1, 2, T, T + 3], rng.integers(0, T + 1, B - 6)]).astype(np.int64)
        seq = (rng.standard_normal((B, T, na)) * 0.7).astype(np.float32)
        seq[np.arange(T)[None, :] >= np.clip(L, 0, T)[:, None]] = 0          # sequence_input_layer pads with zeros
        neg = (rng.standard_normal((B, (T - 1) * T_neg, na)) * 0.7).astype(np.float32)
        tgt = (rng.standard_normal((B, na)) * 0.7).astype(np.float32)
        w = {"gk": MG.glorot(rng, (na + nh, 2 * nh)), "ck": MG.glorot(rng, (na + nh, nh)), "att": MG.glorot(rng, (nh, na)),
             "egk": MG.glorot(rng, (2 * nh, 2 * nh)), "eck": MG.glorot(rng, (2 * nh, nh))}
        for k, n in (("gb", 2 * nh), ("cb", nh), ("egb", 2 * nh), ("ecb", nh)):
            w[k] = rng.uniform(-0.5, 0.5, n).astype(np.float32) + (1.0 if k in ("gb", "egb") else 0.0)
        w_aux = (MG.glorot(rng, (na, nh)) * 3.0).astype(np.float32)           # logits of order 1
        variables = {n: w[k] for k, n in MG.NAMES}
        variables["aux_loss/aux_project_matrix"] = w_aux
        for gru in ("AGRU", "AUGRU"):
            outs = {}
            for tag, dt in (("f32", np.float32), ("f64", np.float64)):
                ns, created = run_aux(cells, seq, L, tgt, neg, variables, dt, gru, nh, T_neg)
                aux = np.asarray(tf._arr(ns["aux_loss"]))
                assert np.isfinite(aux), (gru, tag, aux)
                outs["aux_loss_ref_" + tag] = aux
                outs["final_state_" + tag] = np.asarray(tf._arr(ns["final_state"]))
                h = np.asarray(tf._arr(ns["h"]))
                z = np.concatenate([np.einsum("bti,ij,btj->bt", seq[:, 1:], w_aux, h[:, :-1]).ravel(),
                                    np.einsum("btni,ij,btj->btn", neg.reshape(B, T - 1, T_neg, na), w_aux, h[:, :-1]).ravel()])
                assert np.abs(z).max() < 30, np.abs(z).max()                 # every log term of the reference is finite
            want = {n: w[k].shape for k, n in MG.NAMES}
            want["aux_loss/aux_project_matrix"] = (na, nh)
            assert created == want, created
            arrays = dict(seq=seq, seq_len=L, tgt=tgt, neg=neg, T_neg=np.int64(T_neg), **w, w_aux=w_aux, **outs,
                          slice_restated=np.array("DIEN/dien.py:265 -> " + SLICE),
                          reshape_skipped=np.array("DIEN/dien.py:283 not executed: " + RESHAPE),
                          source=np.array("reference-executed:DIEN/dien.py:199-229+266-300 + DIEN/custom_grucell.py"))
            name = f"dien_aux_{gru.lower()}_na{na}_nh{nh}_T{T}_Tneg{T_neg}_B{B}"
            path = os.path.join(out_dir, name + ".npz")
            np.savez_compressed(path, **arrays)
            z = np.load(path, allow_pickle=False)
            digests[name + ".npz"] = {k: MG.digest(z[k]) for k in z.files}
            print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB")
    return digests


if __name__ == "__main__":
    if len(sys.argv) > 1:
        MG.REF = sys.argv[1]
    assert os.path.isdir(MG.REF), "usage: make_golden_dien_aux.py <reference checkout>/algorithm (or set RECALG_REFERENCE)"
    d = gen_dien_aux()
    with open(os.path.join(OUT, "reference_digests.json"), "w") as fh:
        json.dump(d, fh, indent=1, sort_keys=True)
        fh.write("\n")
