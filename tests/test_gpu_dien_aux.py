"""GPU parity: DIEN's auxiliary loss (csrc/dien.cu, dien_aux_*_kernel and dien_bwd_aux_kernel) against the reference-executed
fixtures (tests/golden/dien_aux, sign flipped) and the float64 restatement with its analytic backward (tests/_dien_aux_ref.py),
over the shape table of test_gpu_dien; bit-identity of ctr_dien_bwd_aux at g_aux = 0 with ctr_dien_bwd; exact zeros where a
position does not count; extreme logits; the bounds; a launch trace; and one training step of dien_logit with the loss."""
import glob
import os
import sys

import numpy as np
import pytest
import torch

import _dien_aux_ref as X
import _dien_ref as R
from _util import GOLDEN, TOL, assert_close, dev
from test_gpu_dien import SHAPES, _err, _inputs, _lens, _nhp, _packed, _resident_batch
from test_gpu_layer_variants import check_reduced, chunked_reference

pytestmark = pytest.mark.gpu

FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "dien_aux", "*.npz")))
PNAMES = ("gk", "gb", "ck", "cb", "att", "egk", "egb", "eck", "ecb")


def _f64(a):
    return np.asarray(a, np.float64)


def _aux_inputs(B, T, na, nh, T_neg, seed):
    rng = np.random.default_rng(seed + 7)
    neg = (rng.standard_normal((B, (T - 1) * T_neg, na)) * 0.7).astype(np.float32)
    w = (rng.uniform(-1, 1, (na, nh)) * np.sqrt(6.0 / (na + nh)) * 2).astype(np.float32)
    return neg, w


def _run(seq, L, tgt, neg, params, w, g, g_aux, nh, cell, T_neg):
    from recalgorithm_b200 import ops
    a = (dev(seq), dev(L), dev(tgt), dev(neg), _packed(params), dev(w))
    fs, att, aux, ws = ops.dien_fwd_aux(*a, nh, cell, T_neg)
    grads = ops.dien_bwd_aux(*a, dev(g), torch.tensor(g_aux, dtype=torch.float32, device="cuda"), nh, cell, T_neg, ws)
    return fs, att, aux, grads


@pytest.mark.parametrize("name", FIXTURES)
def test_dien_aux_fixture_through_ops_and_layers(name):
    """aux_loss == -(the reference's aux_loss) at TOL, and final_state is bit-identical to ctr_dien_fwd's."""
    from recalgorithm_b200 import layers as L, ops
    z = np.load(os.path.join(GOLDEN, "dien_aux", name + ".npz"), allow_pickle=False)
    cell = 1 if "_augru_" in name else 0
    seq, lens, tgt, neg, w = z["seq"], z["seq_len"], z["tgt"], z["neg"], z["w_aux"]
    nh, T_neg = z["att"].shape[0], int(z["T_neg"])
    a = (dev(seq), dev(lens), dev(tgt))
    fs, att, aux, _ = ops.dien_fwd_aux(*a, dev(neg), _packed([z[k] for k in PNAMES]), dev(w), nh, cell, T_neg)
    want = -float(z["aux_loss_ref_f64"])
    assert abs(float(aux) - want) <= TOL * abs(want), (float(aux), want)
    assert_close(fs, z["final_state_f64"], TOL, f"{name} final_state vs reference (float64)")
    fs0, att0, _ = ops.dien_fwd(*a, _packed([z[k] for k in PNAMES]), nh, cell)
    assert torch.equal(fs, fs0) and torch.equal(att, att0)
    store = L.set_default_store(L.VariableStore(device="cuda", seed=0))
    gru = "AUGRU" if cell else "AGRU"
    with L.variable_scope("seq_encoder"):
        L.dien_interest_evolution_aux(*a, dev(neg), dev(w), str(nh), gru, str(T_neg))
    store.assign({"seq_encoder/" + n: z[k] for n, k in zip(ops.DIEN_PARAM_ORDER, PNAMES)})
    with L.variable_scope("seq_encoder"):
        fs2, att2, aux2 = L.dien_interest_evolution_aux(*a, dev(neg), dev(w), str(nh), gru, str(T_neg),
                                                        return_attention_scores=True)
    assert torch.equal(fs2, fs) and torch.equal(att2[..., 0], att) and torch.equal(aux2, aux)


# T_neg cycles over 1, 2, 3 along the table, so that every class meets each of them
TABLE = [(B, T, na, nh, 1 + i % 3) for i, (B, T, na, nh) in enumerate(SHAPES)]


def test_table_covers_every_class_with_every_t_neg():
    for nhp in (8, 16, 32, 64):
        assert {tn for _, _, _, nh, tn in TABLE if _nhp(nh) == nhp} == {1, 2, 3}, nhp


@pytest.mark.parametrize("cell", [0, 1])
@pytest.mark.parametrize("B,T,na,nh,T_neg", TABLE)
def test_dien_aux_fwd_bwd_against_float64(B, T, na, nh, T_neg, cell):
    """aux_loss and every output of ctr_dien_bwd_aux (random g_final and g_aux) against float64.  Per-sample outputs (d_seq,
    d_neg, d_tgt) are held to TOL element-wise; the batch-reduced ones (the nine and d_w_aux, shared-memory then global
    atomics) to check_reduced over 64-sample chunks, as test_gpu_dien holds the nine.  At T >= 64 d_seq and d_tgt may use
    3x the worst error of the float32 restatement, as in test_gpu_dien, for the same reason (the extractor's BPTT over 128
    steps in float32); both errors are printed.  aux_loss (a float64 sum of float32 terms) is held to TOL relative."""
    if B == "resident":
        B = _resident_batch(nh)
    seed = B + T + na + nh + cell
    seq, L, tgt, params, g = _inputs(B, T, na, nh, seed=seed, lens=_lens(T))
    neg, w = _aux_inputs(B, T, na, nh, T_neg, seed)
    g_aux = float(np.random.default_rng(seed).uniform(0.5, 2.0))
    p64 = [_f64(p) for p in params]
    fs, att, aux, (d_seq, d_neg, d_tgt, d_p, d_w) = _run(seq, L, tgt, neg, params, w, g, g_aux, nh, cell, T_neg)
    r_fs, _, r_aux = X.dien_aux_fwd(_f64(seq), L, _f64(tgt), _f64(neg), p64, _f64(w), cell, T_neg)

    def part(lo, hi):                                        # the chunk's share of the 1/B scale: g_aux (hi - lo) / B
        r_seq, r_neg, r_tgt, r_p, r_w = X.dien_aux_bwd(_f64(seq[lo:hi]), L[lo:hi], _f64(tgt[lo:hi]), _f64(neg[lo:hi]), p64,
                                                        _f64(w), cell, T_neg, _f64(g[lo:hi]), g_aux * (hi - lo) / B)
        return {"d_seq": r_seq, "d_neg": r_neg, "d_tgt": r_tgt}, dict(zip(PNAMES + ("w_aux",), r_p + [r_w]))
    per, red = chunked_reference(B, part)

    bars = {"final_state": TOL, "d_seq": TOL, "d_neg": TOL, "d_tgt": TOL}
    restated = {}
    if T >= 64:
        s_seq, _, s_tgt, _, _ = X.dien_aux_bwd(seq, L, tgt, neg, params, w, cell, T_neg, g, np.float32(g_aux))
        for name, s in (("d_seq", s_seq), ("d_tgt", s_tgt)):
            restated[name] = _err(s, per[name])
            bars[name] = max(TOL, 3 * restated[name])
    errs = {"final_state": _err(fs, r_fs), "d_seq": _err(d_seq, per["d_seq"]), "d_neg": _err(d_neg, per["d_neg"]),
            "d_tgt": _err(d_tgt, per["d_tgt"])}
    case = f"B={B} T={T} na={na} nh={nh} T_neg={T_neg} NHP={_nhp(nh)} cell={cell}"
    aux_err = abs(float(aux) - r_aux) / max(abs(r_aux), 1e-30)
    print(f"{case}: aux_loss {aux_err / TOL:.3f} TOL, " + ", ".join(f"{k} {v / TOL:.3f} TOL" for k, v in errs.items()) +
          "".join(f"; {k}: kernel {errs[k]:.2e}, float32 restatement {v:.2e}, bar {bars[k]:.2e}" for k, v in restated.items()))
    assert aux_err <= TOL or (r_aux == 0 and float(aux) == 0), f"{case}: aux_loss {float(aux)} vs {r_aux}"
    for name, e in errs.items():
        assert e <= bars[name], f"{case}: {name} error {e:.3e} > bar {bars[name]:.3e}"
    from recalgorithm_b200 import ops
    worst = max(check_reduced(got, red[n], f"{case}: d {n}")
                for n, got in zip(PNAMES + ("w_aux",), ops.dien_unpack_params(d_p, na, nh) + [d_w]))
    print(f"{case}: d_params, d_w_aux {worst:.3f} of the reduced bar")

    # exact zeros where a position does not count
    Lc = np.clip(L, 0, T)
    pad = np.arange(T)[None, :] >= Lc[:, None]
    assert torch.count_nonzero(d_seq[dev(pad)]) == 0, "padded positions of d_seq get exactly 0"
    cnt = X.counted(L, T)
    assert torch.count_nonzero(d_neg.reshape(B, T - 1, T_neg, na)[dev(~cnt)]) == 0, "d_neg is exactly 0 at t >= L - 1"
    fs2, _, aux2, _ = _run(seq, L, tgt, neg, params, w, g, g_aux, nh, cell, T_neg)
    assert torch.equal(aux2, aux) and torch.equal(fs2, fs), "deterministic aux_loss and forward"


@pytest.mark.parametrize("cell", [0, 1])
@pytest.mark.parametrize("B,T,na,nh,T_neg", [(333, 7, 16, 8, 3), (257, 50, 4, 16, 2), (64, 13, 33, 17, 1),
                                             (30, 4, 64, 50, 2), ("resident", 3, 31, 17, 3)])
def test_bwd_aux_at_zero_aux_gradient_is_the_plain_backward(B, T, na, nh, T_neg, cell):
    """With g_aux = 0, ctr_dien_bwd_aux gives exactly the bits of ctr_dien_bwd for d_seq, d_target and the nine (the extra
    terms are signed zeros added to values that are never -0), and exact zeros for d_neg and d_w_aux."""
    from recalgorithm_b200 import ops
    if B == "resident":
        B = _resident_batch(nh)
    seq, L, tgt, params, g = _inputs(B, T, na, nh, seed=B + nh, lens=_lens(T))
    neg, w = _aux_inputs(B, T, na, nh, T_neg, B)
    a = (dev(seq), dev(L), dev(tgt))
    _, _, _, (d_seq, d_neg, d_tgt, d_p, d_w) = _run(seq, L, tgt, neg, params, w, g, 0.0, nh, cell, T_neg)
    ws = ops.dien_fwd(*a, _packed(params), nh, cell)[2]
    p_seq, p_tgt, p_p = ops.dien_bwd(*a, _packed(params), dev(g), nh, cell, ws)
    bits = lambda t: t.view(torch.int32)
    assert torch.equal(bits(d_seq), bits(p_seq)) and torch.equal(bits(d_tgt), bits(p_tgt))
    assert torch.count_nonzero(d_neg) == 0 and torch.count_nonzero(d_w) == 0
    # Every per-sample term of the nine is bit-identical too, but they are summed with float atomics (shared memory, then
    # global), whose order differs between runs of ctr_dien_bwd itself.  So d_params must equal one of two plain runs bit
    # for bit, or differ from the first by no more than the plain runs differ from each other plus one float32 ulp of the
    # largest element per summand order (2^-22 relative).
    p_p2 = ops.dien_bwd(*a, _packed(params), dev(g), nh, cell, ws)[2]
    same = torch.equal(bits(d_p), bits(p_p)) or torch.equal(bits(d_p), bits(p_p2))
    spread = float((p_p2 - p_p).abs().max())
    print(f"B={B} nh={nh} cell={cell}: d_params bit-identical to a plain run: {same}; plain run-to-run spread {spread:.2e}")
    assert same or float((d_p - p_p).abs().max()) <= 2 * spread + float(p_p.abs().max()) * 2.0 ** -22


def test_extreme_logits_are_finite_and_match_float64():
    """Logits near +-100: the reference's tf.log(tf.sigmoid(.)) gives -inf there; the kernels' softplus form gives the float64
    stable value, and finite gradients."""
    from recalgorithm_b200 import ops
    B, T, na, nh, T_neg, cell = 64, 9, 16, 8, 3, 1
    seq, L, tgt, params, g = _inputs(B, T, na, nh, seed=11, lens=_lens(T))
    neg, w = _aux_inputs(B, T, na, nh, T_neg, 11)
    _, _, cc = R.dien_fwd(_f64(seq), L, _f64(tgt), [_f64(p) for p in params], cell, return_cache=True)
    _, zp, zn = X.logits(cc["H"], _f64(seq), _f64(neg), _f64(w), T_neg)
    cnt = X.counted(L, T)
    scale = 100.0 / np.median(np.abs(np.concatenate([zp[cnt], zn[cnt].ravel()])))
    w = (w * scale).astype(np.float32)
    _, zp, zn = X.logits(cc["H"], _f64(seq), _f64(neg), _f64(w), T_neg)
    assert (zp[cnt] > 50).any() and (zp[cnt] < -50).any() and (zn[cnt] > 50).any() and (zn[cnt] < -50).any()
    assert not np.isfinite(X.reference_form(cc["H"], _f64(seq), L, _f64(neg), _f64(w), T_neg))
    fs, att, aux, (d_seq, d_neg, d_tgt, d_p, d_w) = _run(seq, L, tgt, neg, params, w, g, 1.0, nh, cell, T_neg)
    r_aux = X.dien_aux_fwd(_f64(seq), L, _f64(tgt), _f64(neg), [_f64(p) for p in params], _f64(w), cell, T_neg)[2]
    assert np.isfinite(float(aux)) and abs(float(aux) - r_aux) <= TOL * abs(r_aux), (float(aux), r_aux)
    for t in (d_seq, d_neg, d_tgt, d_p, d_w):
        assert torch.isfinite(t).all()


def test_zero_batch_and_single_step():
    """B = 0: aux_loss and d_w_aux are 0.  T = 1: nothing counts."""
    from recalgorithm_b200 import ops
    for B, T in ((0, 5), (9, 1)):
        seq, L, tgt, params, g = _inputs(B, T, 16, 8, seed=3)
        neg, w = _aux_inputs(B, T, 16, 8, 2, 3)
        _, _, aux, (d_seq, d_neg, d_tgt, d_p, d_w) = _run(seq, L, tgt, neg, params, w, g, 1.0, 8, 0, 2)
        assert float(aux) == 0.0 and torch.count_nonzero(d_w) == 0 and d_neg.numel() == 0


@pytest.mark.parametrize("entry", ["ctr_dien_aux_workspace_bytes", "ctr_dien_aux_fwd", "ctr_dien_bwd_aux"])
@pytest.mark.parametrize("B,T,na,nh,T_neg", [(4, 129, 16, 8, 3), (4, 10, 65, 8, 3), (4, 10, 16, 65, 3),
                                             (4, 10, 16, 8, 1 << 31), (1 << 20, 17, 16, 8, 8)])
def test_aux_entries_reject_out_of_range_shapes(entry, B, T, na, nh, T_neg):
    """Every new entry refuses shapes past its bounds (T, na, nh, T_neg and B*(T-1)*T_neg*na < 2^31) with
    CTR_ERR_UNSUPPORTED before touching any argument; T_neg = 0 is an invalid argument."""
    import ctypes
    from recalgorithm_b200 import _lib
    h = _lib.lib()
    buf = torch.zeros(1 << 16, device="cuda")
    lens = torch.zeros(8, dtype=torch.int64, device="cuda")
    p, ln, nb = buf.data_ptr(), lens.data_ptr(), buf.numel() * 4

    def call(tn):
        if entry == "ctr_dien_aux_workspace_bytes":
            return h.ctr_dien_aux_workspace_bytes(B, T, na, nh, tn, ctypes.byref(ctypes.c_int64(0)))
        if entry == "ctr_dien_aux_fwd":
            return h.ctr_dien_aux_fwd(p, p, ln, p, B, T, na, nh, tn, p, p, nb, None)
        return h.ctr_dien_bwd_aux(p, p, ln, p, p, p, p, p, B, T, na, nh, tn, 1, p, p, p, p, p, p, nb, None)
    assert call(T_neg) == _lib.CTR_ERR_UNSUPPORTED
    assert h.ctr_last_error().decode().startswith(entry)
    assert call(0) in (_lib.CTR_ERR_INVALID_ARG, _lib.CTR_ERR_UNSUPPORTED)
    torch.cuda.synchronize()


_PROFILE = """
import json, sys
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, "tests")
from _util import dev
from test_gpu_dien import _inputs, _lens, _packed
from recalgorithm_b200 import ops
out = []
for nh in (8, 16, 32, 64):
    for cell in (0, 1):
        B, T, na, T_neg = 70, 6, 16, 2
        seq, L, tgt, params, g = _inputs(B, T, na, nh, seed=0, lens=_lens(T))
        neg = dev(np.ones((B, (T - 1) * T_neg, na), np.float32)); w = dev(np.full((na, nh), 0.01, np.float32))
        a = (dev(seq), dev(L), dev(tgt), neg, _packed(params), w)
        run = lambda: ops.dien_bwd_aux(*a, dev(g), torch.ones((), device="cuda"), nh, cell, T_neg, ops.dien_fwd_aux(*a, nh, cell, T_neg)[3])
        run()                                                            # first launches (module load) outside the trace
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run()
            torch.cuda.synchronize()
        out.append([nh, cell, [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]])
print(json.dumps(out))
"""


def test_aux_path_launches_its_kernels():
    """The aux path (forward, aux forward, aux backward) launches, per class and cell, dien_fwd_kernel, the two aux-loss
    kernels of the forward (per-sample terms, fixed-order sum), dien_aux_bwd_kernel and dien_bwd_aux_kernel of its class --
    never the plain dien_bwd_kernel -- and reaches all 8 dien_bwd_aux_kernel instantiations.  Traced in a process of its
    own, like test_gpu_dien's trace."""
    import json
    import re
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    run = subprocess.run([sys.executable, "-c", _PROFILE], cwd=root, capture_output=True, text=True, timeout=900)
    assert run.returncode == 0, run.stderr[-3000:]
    seen = set()
    for nh, cell, names in json.loads(run.stdout.strip().splitlines()[-1]):
        got = {m.group(1) for n in names for m in [re.search(r"(dien_\w+_kernel)\b", n)] if m}
        assert got == {"dien_fwd_kernel", "dien_aux_fwd_kernel", "dien_aux_sum_kernel", "dien_aux_bwd_kernel",
                       "dien_bwd_aux_kernel"}, (nh, cell, names)
        cls = {(int(m[1]), int(m[2])) for n in names for m in [re.search(r"dien_bwd_aux_kernel<(\d+), (\d+)>", n)] if m}
        assert cls == {(_nhp(nh), cell)}, (nh, cell, names)
        seen |= cls
    assert len(seen) == 8


@pytest.mark.parametrize("gru", ["AGRU", "AUGRU"])
def test_dien_logit_trains_with_the_auxiliary_loss(gru):
    """One step of ce + aux_loss (dien.py:316-317) with the history, the target and the negatives looked up in the shared feedid
    table: a finite loss, three IndexedSlices on the table, and a gradient on aux_loss/aux_project_matrix."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import model_bodies as M
    from recalgorithm_b200 import autograd, layers as L
    B, T, H, rows, T_neg = 96, 12, 16, 80, 3
    store = L.set_default_store(L.VariableStore(device="cuda", seed=2))
    gen = torch.Generator(device="cuda").manual_seed(2)
    item = autograd.EmbeddingTables([rows], H, device="cuda")
    lens = torch.randint(0, T + 1, (B,), device="cuda", generator=gen)
    hist = torch.randint(0, rows, (B, T), device="cuda", generator=gen)
    hist[torch.arange(T, device="cuda")[None, :] >= lens[:, None]] = -1
    negs = torch.randint(0, rows, (B, (T - 1) * T_neg), device="cuda", generator=gen)
    tgt = torch.randint(0, rows, (B, 1), device="cuda", generator=gen)
    seq = autograd.lookup(item, hist.reshape(B * T, 1)).reshape(B, T, H)
    neg = autograd.lookup(item, negs.reshape(-1, 1)).reshape(B, (T - 1) * T_neg, H)
    target = autograd.lookup(item, tgt).reshape(B, H)
    dense_input = torch.randn(B, 3, device="cuda", generator=gen)
    cat = torch.randn(B, 8, device="cuda", generator=gen)
    y = (torch.rand((B, 1), device="cuda", generator=gen) < 0.3).float()
    logit, att, aux = M.dien_logit(dense_input, cat, target, seq, lens, gru_output_units="8", custom_gru_type=gru,
                                   use_auxiliary_loss=True, neg_sequnence_input=neg, negative_sample_number="3")
    loss = torch.nn.functional.binary_cross_entropy_with_logits(logit, y) + aux
    assert torch.isfinite(loss) and float(aux) > 0
    loss.backward()
    assert len(item.grad_slices) == 3 and all(float(s.values.abs().max()) > 0 for s in item.grad_slices)
    w = store.vars["aux_loss/aux_project_matrix"]
    assert tuple(w.shape) == (H, 8) and float(w.grad.abs().max()) > 0
    for n, v in store.vars.items():
        assert v.grad is not None and torch.isfinite(v.grad).all(), n
