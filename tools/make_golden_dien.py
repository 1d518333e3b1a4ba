"""Generate tests/golden/dien/*.npz by executing DIEN's seq_encoder block (DIEN/dien.py:198-229) over the TF1 shim, with the
reference's own AGRUCell / AUGRUCell imported verbatim from DIEN/custom_grucell.py.

    python tools/make_golden_dien.py /path/to/RecAlgorithm/algorithm      (or set RECALG_REFERENCE)

custom_grucell.py is imported unchanged from the reference checkout.  For this run only, the modules it imports are provided
over the shared shim (oracle/tf1_shim), with TensorFlow 1.14 semantics:
  tensorflow.python.ops.rnn_cell (RNNCell, LayerRNNCell), tensorflow.contrib.rnn.python.ops.core_rnn_cell._Linear (concat on
  axis 1, variables `kernel` / `bias` in the current scope, default bias zeros), math_ops.sigmoid / tanh,
  init_ops.constant_initializer, array_ops.split, variable_scope.
Two pieces are restated, because the reference takes them from TensorFlow itself: `dynamic_rnn` (DIEN/rnn.py:737-798, the
time loop with att_scores[:, t, :] passed to the cell, plus _rnn_step with skip_conditionals=True, rnn.py:201-217: past
sequence_length the output is zero and the state is copied through) and tf.nn.rnn_cell.GRUCell (TF 1.14: gates in scope
gru_cell/gates with bias ones, candidate in gru_cell/candidate with bias zeros, h' = u*h + (1-u)*c).  The generator pins the
GRUCell restatement against the verbatim AUGRUCell at att_score = 0 and records the difference (exactly 0) in each fixture.
Each fixture stores the seeded inputs, the injected weights, and the reference's final_state and attention scores in float32
and float64.  tests/golden/dien/reference_digests.json holds the SHA-256 of every array (tests/test_dien_oracle.py checks
them, and re-runs this script when RECALG_REFERENCE is set).
"""
from __future__ import annotations

import contextlib
import hashlib
import importlib.util
import json
import os
import sys
import textwrap
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "dien")
REF = os.environ.get("RECALG_REFERENCE", "")
CASES = ((16, 8, 50, 16), (5, 3, 7, 9))           # (na, nh, T, B)

sys.path.insert(0, os.path.join(ROOT, "oracle", "tf1_shim"))
import tensorflow as tf  # noqa: E402  (the shim)

assert "tf1_shim" in tf.__file__, "the TF shim must shadow any real tensorflow"

_INITS = {}                                        # full variable name -> initializer the reference asked for


class _Const:
    """init_ops.constant_initializer(value)."""
    def __init__(self, value=0, dtype=None):
        self.value = value


class RNNCell:
    """tensorflow.python.ops.rnn_cell.RNNCell: only the constructor the custom cells call."""
    def __init__(self, _reuse=None, name=None, dtype=None):
        self._reuse = _reuse


class _Linear:
    """TF 1.14 core_rnn_cell._Linear: kernel (sum of arg widths, output_size) and bias (output_size) in the current scope;
    __call__ = concat(args, axis=1) . kernel + bias.  bias_initializer None -> zeros."""
    def __init__(self, args, output_size, build_bias, bias_initializer=None, kernel_initializer=None):
        width = sum(int(tf._arr(a).shape[1]) for a in args)
        self._kernel = tf.get_variable("kernel", shape=(width, output_size))
        _INITS[tf._full_name("kernel")] = kernel_initializer
        self._bias = None
        if build_bias:
            self._bias = tf.get_variable("bias", shape=(output_size,))
            _INITS[tf._full_name("bias")] = bias_initializer if bias_initializer is not None else _Const(0.0)

    def __call__(self, args):
        out = tf.matmul(tf.concat(args, 1), self._kernel)
        return out + self._bias if self._bias is not None else out


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def _install_shim_modules():
    sigmoid = lambda x: tf.Tensor(1 / (1 + np.exp(-tf._arr(x))))
    tanh = lambda x: tf.Tensor(np.tanh(tf._arr(x)))
    split = lambda value, num_or_size_splits, axis: [tf.Tensor(a) for a in np.split(tf._arr(value), num_or_size_splits, axis)]
    _module("tensorflow.python")
    _module("tensorflow.python.ops")
    _module("tensorflow.python.ops.rnn_cell", RNNCell=RNNCell, LayerRNNCell=RNNCell)
    _module("tensorflow.python.ops.math_ops", sigmoid=sigmoid, tanh=tanh)
    _module("tensorflow.python.ops.init_ops", constant_initializer=_Const)
    _module("tensorflow.python.ops.array_ops", split=split)
    _module("tensorflow.python.ops.variable_scope", variable_scope=tf.variable_scope)
    for n in ("tensorflow.contrib", "tensorflow.contrib.rnn", "tensorflow.contrib.rnn.python", "tensorflow.contrib.rnn.python.ops"):
        _module(n)
    _module("tensorflow.contrib.rnn.python.ops.core_rnn_cell", _Linear=_Linear)


class GRUCell:
    """tf.nn.rnn_cell.GRUCell (TF 1.14), restated: variables gru_cell/gates/{kernel,bias} (bias ones) and
    gru_cell/candidate/{kernel,bias} (bias zeros); [r, u] = sigmoid([x, h] . Wg + bg), c = tanh([x, r*h] . Wc + bc),
    h' = u*h + (1-u)*c."""
    def __init__(self, num_units):
        self._n = num_units
        self._built = False

    def __call__(self, inputs, state):
        with tf.variable_scope("gru_cell"):
            if not self._built:
                with tf.variable_scope("gates"):
                    self._gates = _Linear([inputs, state], 2 * self._n, True, bias_initializer=_Const(1.0))
                with tf.variable_scope("candidate"):
                    self._cand = _Linear([inputs, state], self._n, True)
                self._built = True
            value = sys.modules["tensorflow.python.ops.math_ops"].sigmoid(self._gates([inputs, state]))
            r, u = sys.modules["tensorflow.python.ops.array_ops"].split(value=value, num_or_size_splits=2, axis=1)
            c = sys.modules["tensorflow.python.ops.math_ops"].tanh(self._cand([inputs, r * state]))
            new_h = u * state + (1 - u) * c
        return new_h, new_h


def dynamic_rnn(cell, inputs, att_scores=None, sequence_length=None, initial_state=None, dtype=None, scope=None):
    """DIEN/rnn.py:443 dynamic_rnn as its loop (rnn.py:737-798) computes it, eagerly: zero initial state, cell called per step
    with att_scores[:, t, :] when given; with sequence_length, _rnn_step(skip_conditionals=True) (rnn.py:201-217) zeroes the
    output and copies the state through for t >= sequence_length."""
    x = tf._arr(inputs)
    B, T = x.shape[0], x.shape[1]
    n = cell._num_units if hasattr(cell, "_num_units") else cell._n
    state = tf.Tensor(np.zeros((B, n), x.dtype))
    outs = []
    with tf.variable_scope(scope or "rnn"):
        for t in range(T):
            inp = tf.Tensor(x[:, t])
            if att_scores is not None:
                out, new_state = cell(inp, state, tf.Tensor(tf._arr(att_scores)[:, t, :]))
            else:
                out, new_state = cell(inp, state)
            if sequence_length is not None:
                copy = (t >= np.asarray(tf._arr(sequence_length)))[:, None]
                out = tf.Tensor(np.where(copy, np.zeros_like(tf._arr(out)), tf._arr(out)))
                new_state = tf.Tensor(np.where(copy, tf._arr(state), tf._arr(new_state)))
            outs.append(tf._arr(out))
            state = new_state
    return tf.Tensor(np.stack(outs, 1)), state


def _load_cells():
    _install_shim_modules()
    spec = importlib.util.spec_from_file_location("dien_custom_grucell", os.path.join(REF, "DIEN", "custom_grucell.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def run_block(cells, seq, seq_len, tgt, variables, dtype, custom_gru_type, nh):
    tf.reset(dtype=dtype, variables=variables)
    _INITS.clear()
    tf.nn.rnn_cell = types.SimpleNamespace(GRUCell=GRUCell)
    ns = {"tf": tf, "dynamic_rnn": dynamic_rnn, "AGRUCell": cells.AGRUCell, "AUGRUCell": cells.AUGRUCell,
          "params": {"gru_output_units": nh, "custom_gru_type": custom_gru_type},
          "sequnence_input": tf.Tensor(seq.astype(dtype)), "sequnence_length": tf.Tensor(seq_len),
          "target_input": tf.Tensor(tgt.astype(dtype))}
    with open(os.path.join(REF, "DIEN", "dien.py"), encoding="utf-8") as fh:
        lines = fh.read().split("\n")[197:229]                   # lines 198-229
    assert 'tf.variable_scope("seq_encoder")' in lines[1] and "dtype=tf.float32)" in lines[-1], (lines[1], lines[-1])
    exec(compile(textwrap.dedent("\n".join(lines)), "DIEN/dien.py:198-229", "exec"), ns)
    return ns, tf.created_variables(), dict(_INITS)


def glorot(rng, shape):
    lim = (6.0 / (shape[0] + shape[1])) ** 0.5
    return rng.uniform(-lim, lim, size=shape).astype(np.float32)


def digest(a):
    return f"{a.dtype.str}:{'x'.join(map(str, a.shape))}:{hashlib.sha256(a.tobytes()).hexdigest()}"


NAMES = (("gk", "seq_encoder/rnn/gru_cell/gates/kernel"), ("gb", "seq_encoder/rnn/gru_cell/gates/bias"),
         ("ck", "seq_encoder/rnn/gru_cell/candidate/kernel"), ("cb", "seq_encoder/rnn/gru_cell/candidate/bias"),
         ("att", "seq_encoder/attention_project_matrix"), ("egk", "seq_encoder/rnn/gates/kernel"),
         ("egb", "seq_encoder/rnn/gates/bias"), ("eck", "seq_encoder/rnn/candidate/kernel"),
         ("ecb", "seq_encoder/rnn/candidate/bias"))


def _grucell_vs_augru(cells, rng, na, nh, w):
    """max |GRUCell restatement - verbatim AUGRUCell at att_score = 0| on random inputs with the same weights (float64)."""
    x = tf.Tensor(rng.standard_normal((7, na))); h = tf.Tensor(rng.standard_normal((7, nh)))
    tf.reset(dtype=np.float64, variables={"gru_cell/gates/kernel": w["gk"], "gru_cell/gates/bias": w["gb"],
                                          "gru_cell/candidate/kernel": w["ck"], "gru_cell/candidate/bias": w["cb"],
                                          "gates/kernel": w["gk"], "gates/bias": w["gb"], "candidate/kernel": w["ck"],
                                          "candidate/bias": w["cb"]})
    a = tf._arr(GRUCell(nh)(x, h)[0])
    b = tf._arr(cells.AUGRUCell(nh)(x, h, tf.Tensor(np.zeros((7, 1))))[0])
    return float(np.abs(a - b).max())


def gen_dien(out_dir=OUT):
    cells = _load_cells()
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(4242)
    digests = {}
    for na, nh, T, B in CASES:
        L = np.concatenate([[0, 1, T, T + 3], rng.integers(0, T + 1, B - 4)]).astype(np.int64)
        seq = (rng.standard_normal((B, T, na)) * 0.7).astype(np.float32)
        seq[np.arange(T)[None, :] >= np.minimum(L, T)[:, None]] = 0          # sequence_input_layer pads with zeros
        tgt = (rng.standard_normal((B, na)) * 0.7).astype(np.float32)
        w = {"gk": glorot(rng, (na + nh, 2 * nh)), "ck": glorot(rng, (na + nh, nh)), "att": glorot(rng, (nh, na)),
             "egk": glorot(rng, (2 * nh, 2 * nh)), "eck": glorot(rng, (2 * nh, nh))}
        for k, n in (("gb", 2 * nh), ("cb", nh), ("egb", 2 * nh), ("ecb", nh)):      # away from the initial ones / zeros
            w[k] = rng.uniform(-0.5, 0.5, n).astype(np.float32) + (1.0 if k in ("gb", "egb") else 0.0)
        pin = _grucell_vs_augru(cells, rng, na, nh, {k: v.astype(np.float64) for k, v in w.items()})
        assert pin == 0.0, pin
        for gru in ("AGRU", "AUGRU"):
            outs = {}
            for tag, dt in (("f32", np.float32), ("f64", np.float64)):
                ns, created, inits = run_block(cells, seq, L, tgt, {n: w[k] for k, n in NAMES}, dt, gru, nh)
                outs["final_state_" + tag] = np.asarray(tf._arr(ns["final_state"]))
                outs["att_" + tag] = np.asarray(tf._arr(ns["attention_scores"]))
            assert created == {n: w[k].shape for k, n in NAMES}, created
            # initialisers: gate biases ones, candidate biases zeros, kernels the default (glorot-uniform)
            for k, n in NAMES:
                if k in ("gb", "egb", "cb", "ecb"):
                    assert inits[n].value == (1.0 if k in ("gb", "egb") else 0.0), (n, inits[n].value)
                elif k != "att":
                    assert inits[n] is None, n
            arrays = dict(seq=seq, seq_len=L, tgt=tgt, **w, **outs, grucell_vs_augru_at_a0_maxabs=np.float64(pin),
                          source=np.array("reference-executed:DIEN/dien.py:198-229 + DIEN/custom_grucell.py"))
            name = f"dien_{gru.lower()}_na{na}_nh{nh}_T{T}_B{B}"
            path = os.path.join(out_dir, name + ".npz")
            np.savez_compressed(path, **arrays)
            z = np.load(path, allow_pickle=False)
            digests[name + ".npz"] = {k: digest(z[k]) for k in z.files}
            print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB")
    # quirk: any custom_gru_type other than the exact string "AUGRU" takes the AGRU branch (dien.py:220-223)
    na, nh, T, B = 3, 2, 4, 2
    args = (np.ones((B, T, na), np.float32), np.array([2, 4]), np.ones((B, na), np.float32))
    outs = [tf._arr(run_block(cells, *args, {}, np.float64, g, nh)[0]["final_state"]) for g in ("AGRU", "augru", "GRU", "AUGRU")]
    assert np.array_equal(outs[0], outs[1]) and np.array_equal(outs[0], outs[2]) and not np.array_equal(outs[0], outs[3])
    return digests


if __name__ == "__main__":
    if len(sys.argv) > 1:
        REF = sys.argv[1]
    assert os.path.isdir(REF), "usage: make_golden_dien.py <reference checkout>/algorithm (or set RECALG_REFERENCE)"
    d = gen_dien()
    with open(os.path.join(OUT, "reference_digests.json"), "w") as fh:
        json.dump(d, fh, indent=1, sort_keys=True)
        fh.write("\n")
