"""GPU parity: DIEN's interest extractor + attention + interest evolution (csrc/dien.cu) against the reference-executed
fixtures (tests/golden/dien) and the float64 restatement with its analytic backward (tests/_dien_ref.py)."""
import glob
import os
import sys

import numpy as np
import pytest
import torch

import _dien_ref as R
from _util import GOLDEN, TOL, assert_close, dev

pytestmark = pytest.mark.gpu

FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "dien", "*.npz")))
PNAMES = ("gk", "gb", "ck", "cb", "att", "egk", "egb", "eck", "ecb")


def _packed(params):
    return dev(np.concatenate([np.asarray(p, np.float32).reshape(-1) for p in params]))


def _inputs(B, T, na, nh, seed, lens=None):
    rng = np.random.default_rng(seed)
    L = rng.integers(0, T + 1, B) if lens is None else np.resize(np.asarray(lens, np.int64), B)
    seq = (rng.standard_normal((B, T, na)) * 0.7).astype(np.float32)
    seq[np.arange(T)[None, :] >= np.clip(L, 0, T)[:, None]] = 0
    tgt = (rng.standard_normal((B, na)) * 0.7).astype(np.float32)
    params = R.init_params(rng, na, nh, np.float32, bias_scale=0.5)
    g = rng.standard_normal((B, nh)).astype(np.float32)
    return seq, L.astype(np.int64), tgt, params, g


def _f64(a):
    return np.asarray(a, np.float64)


@pytest.mark.parametrize("name", FIXTURES)
def test_dien_fixture_through_ops_and_layers(name):
    from recalgorithm_b200 import layers as L, ops
    z = np.load(os.path.join(GOLDEN, "dien", name + ".npz"), allow_pickle=False)
    cell = 1 if "_augru_" in name else 0
    seq, lens, tgt = z["seq"], z["seq_len"], z["tgt"]
    nh = z["att"].shape[0]
    fs, att, _ = ops.dien_fwd(dev(seq), dev(lens), dev(tgt), _packed([z[k] for k in PNAMES]), nh, cell)
    assert_close(fs, z["final_state_f64"], TOL, f"{name} final_state vs reference (float64)")
    assert_close(att, z["att_f64"][..., 0], TOL, f"{name} attention vs reference (float64)")
    store = L.set_default_store(L.VariableStore(device="cuda", seed=0))
    with L.variable_scope("seq_encoder"):
        L.dien_interest_evolution(dev(seq), dev(lens), dev(tgt), str(nh), "AUGRU" if cell else "AGRU")
    from recalgorithm_b200.ops import DIEN_PARAM_ORDER
    store.assign({"seq_encoder/" + n: z[k] for n, k in zip(DIEN_PARAM_ORDER, PNAMES)})
    with L.variable_scope("seq_encoder"):
        fs2, att2 = L.dien_interest_evolution(dev(seq), dev(lens), dev(tgt), str(nh), "AUGRU" if cell else "AGRU",
                                              return_attention_scores=True)
    assert torch.equal(fs2, fs) and torch.equal(att2[..., 0], att)
    assert sorted(store.vars) == sorted("seq_encoder/" + n for n in DIEN_PARAM_ORDER)


# (B, T, na, nh): one sample, ragged B, the reference shape, wide nh, the largest na and nh, and odd widths
SHAPES = [(1, 1, 16, 8), (333, 7, 16, 8), (1024, 50, 16, 8), (257, 50, 4, 16), (128, 20, 64, 64), (64, 13, 3, 5)]


@pytest.mark.parametrize("cell", [0, 1])
@pytest.mark.parametrize("B,T,na,nh", SHAPES)
def test_dien_fwd_bwd_against_float64(B, T, na, nh, cell):
    from recalgorithm_b200 import ops
    lens = [0, 1, T, T + 3] + list(range(T + 1))                              # 0, 1, T and > T, then every length
    seq, L, tgt, params, g = _inputs(B, T, na, nh, seed=B + T + na + nh + cell, lens=lens)
    p64 = [_f64(p) for p in params]
    fs, att, ws = ops.dien_fwd(dev(seq), dev(L), dev(tgt), _packed(params), nh, cell)
    r_fs, r_att = R.dien_fwd(_f64(seq), L, _f64(tgt), p64, cell)
    assert_close(fs, r_fs, TOL, "final_state")
    assert_close(att, r_att, TOL, "attention scores")
    d_seq, d_tgt, d_p = ops.dien_bwd(dev(seq), dev(L), dev(tgt), _packed(params), dev(g), nh, cell, ws)
    r_seq, r_tgt, r_p = R.dien_bwd(_f64(seq), L, _f64(tgt), p64, cell, _f64(g))
    assert_close(d_seq, r_seq, TOL, "d_sequnence_input")
    assert_close(d_tgt, r_tgt, TOL, "d_target_input")
    for name, got, want in zip(ops.DIEN_PARAM_ORDER, ops.dien_unpack_params(d_p, na, nh), r_p):
        assert_close(got, want, TOL, f"d {name}")
    pad = np.arange(T)[None, :] >= np.clip(L, 0, T)[:, None]
    assert torch.count_nonzero(d_seq[torch.from_numpy(pad).cuda()]) == 0, "padded positions get exactly 0"
    if cell == 0:
        dp = ops.dien_unpack_params(d_p, na, nh)
        assert torch.count_nonzero(dp[5][:, nh:]) == 0 and torch.count_nonzero(dp[6][nh:]) == 0, "AGRU: u half gets exactly 0"
    again = ops.dien_fwd(dev(seq), dev(L), dev(tgt), _packed(params), nh, cell)[0]
    assert torch.equal(again, fs), "deterministic forward"


@pytest.mark.parametrize("cell", [0, 1])
def test_dien_all_zero_lengths(cell):
    from recalgorithm_b200 import ops
    B, T, na, nh = 70, 9, 16, 8
    seq, L, tgt, params, g = _inputs(B, T, na, nh, seed=5, lens=[0])
    fs, att, ws = ops.dien_fwd(dev(seq), dev(L), dev(tgt), _packed(params), nh, cell)
    assert torch.count_nonzero(fs) == 0
    assert torch.all(att == torch.tensor(1.0 / T, device="cuda"))
    d_seq, d_tgt, d_p = ops.dien_bwd(dev(seq), dev(L), dev(tgt), _packed(params), dev(g), nh, cell, ws)
    for t in (d_seq, d_tgt, d_p):
        assert torch.count_nonzero(t) == 0


def test_dien_rejects_out_of_range_shapes():
    from recalgorithm_b200 import _lib, ops
    for B, T, na, nh in ((4, 129, 16, 8), (4, 10, 65, 8), (4, 10, 16, 65)):
        seq, L, tgt, params, g = _inputs(B, T, na, nh, seed=1)
        with pytest.raises(_lib.CtrInvalidArgument) as e:
            ops.dien_fwd(dev(seq), dev(L), dev(tgt), _packed(params), nh, 0)
        assert e.value.code == _lib.CTR_ERR_UNSUPPORTED and "ctr_dien_workspace_bytes" in str(e.value)


@pytest.mark.parametrize("entry", ["ctr_dien_fwd", "ctr_dien_bwd"])
@pytest.mark.parametrize("B,T,na,nh", [(4, 129, 16, 8), (4, 10, 65, 8), (4, 10, 16, 65), (700000, 128, 16, 8)])
def test_dien_entries_reject_out_of_range_shapes(entry, B, T, na, nh):
    """Both compute entries refuse shapes past their bounds themselves (T, na, nh, and B*T*(3nh+2) < 2^31), before touching
    any argument: called through the C ABI with small real buffers and a dummy workspace."""
    from recalgorithm_b200 import _lib
    h = _lib.lib()
    buf = torch.zeros(1 << 16, device="cuda")
    lens = torch.zeros(8, dtype=torch.int64, device="cuda")
    p, ln = buf.data_ptr(), lens.data_ptr()
    if entry == "ctr_dien_fwd":
        rc = h.ctr_dien_fwd(p, ln, p, p, B, T, na, nh, 0, p, p, p, buf.numel() * 4, None)
    else:
        rc = h.ctr_dien_bwd(p, ln, p, p, p, B, T, na, nh, 1, p, p, p, p, buf.numel() * 4, None)
    assert rc == _lib.CTR_ERR_UNSUPPORTED
    msg = h.ctr_last_error().decode()
    assert msg.startswith(entry) and ("unsupported" in msg or "too large" in msg), msg
    torch.cuda.synchronize()


@pytest.mark.parametrize("gru", ["AGRU", "AUGRU", "GRU"])
def test_dien_logit_body(gru):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import model_bodies as M
    from recalgorithm_b200 import autograd, layers as L
    B, T, H, rows = 96, 12, 16, 80
    store = L.set_default_store(L.VariableStore(device="cuda", seed=2))
    gen = torch.Generator(device="cuda").manual_seed(2)
    item = autograd.EmbeddingTables([rows], H, device="cuda")                 # the shared feedid table
    lens = torch.randint(0, T + 1, (B,), device="cuda", generator=gen)
    hist = torch.randint(0, rows, (B, T), device="cuda", generator=gen)
    hist[torch.arange(T, device="cuda")[None, :] >= lens[:, None]] = -1
    tgt = torch.randint(0, rows, (B, 1), device="cuda", generator=gen)
    seq = autograd.lookup(item, hist.reshape(B * T, 1)).reshape(B, T, H)
    target = autograd.lookup(item, tgt).reshape(B, H)
    dense_input = torch.randn(B, 3, device="cuda", generator=gen)
    cat = torch.randn(B, 8, device="cuda", generator=gen)
    y = (torch.rand((B, 1), device="cuda", generator=gen) < 0.3).float()
    logit, att = M.dien_logit(dense_input, cat, target, seq, lens, gru_output_units="8", custom_gru_type=gru)
    assert logit.shape == (B, 1) and att.shape == (B, T, 1) and torch.isfinite(logit).all()
    torch.nn.functional.binary_cross_entropy_with_logits(logit, y).backward()
    assert len(item.grad_slices) == 2 and all(float(s.values.abs().max()) > 0 for s in item.grad_slices)
    names = {"seq_encoder/" + n for n in ("rnn/gru_cell/gates/kernel", "attention_project_matrix", "rnn/gates/kernel",
                                          "rnn/candidate/bias", "fcn/dense/kernel", "fcn/dense_2/kernel")}
    assert names <= set(store.vars)
    for n, v in store.vars.items():
        assert v.grad is not None and torch.isfinite(v.grad).all(), n
    u_half = store.vars["seq_encoder/rnn/gates/kernel"].grad[:, 8:]
    assert (torch.count_nonzero(u_half) == 0) == (gru != "AUGRU")
