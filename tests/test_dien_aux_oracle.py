"""CPU tests of DIEN's auxiliary loss (DIEN/dien.py:256-300): the float64 restatement (tests/_dien_aux_ref.py) against the
fixtures produced by executing the reference's lines (tools/make_golden_dien_aux.py) -- with the sign flipped, since the
kernels compute the paper's loss -- its analytic backward through the whole seq_encoder against torch.autograd, the stable
log form against the reference's form, and the fixture digests."""
import glob
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _dien_aux_ref as X
import _dien_ref as R

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dien_aux")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(G, "*.npz")))
PNAMES = ("gk", "gb", "ck", "cb", "att", "egk", "egb", "eck", "ecb")


def rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-30)


def test_fixtures_present():
    assert NAMES == ["dien_aux_agru_na16_nh8_T50_Tneg3_B16", "dien_aux_agru_na5_nh3_T7_Tneg2_B9",
                     "dien_aux_augru_na16_nh8_T50_Tneg3_B16", "dien_aux_augru_na5_nh3_T7_Tneg2_B9"]


@pytest.mark.parametrize("name", NAMES)
def test_restatement_matches_reference_executed(name):
    """Parity notes 1-3 (DESIGN §2, DIEN auxiliary loss): the restatement is the negative of the reference's aux_loss, executed with line 265 restated
    (and line 283 left out); final_state is the seq_encoder's."""
    z = np.load(os.path.join(G, name + ".npz"), allow_pickle=False)
    assert str(z["source"]).startswith("reference-executed:DIEN/dien.py:199-229+266-300")
    assert str(z["slice_restated"]) == "DIEN/dien.py:265 -> pos_sequnence_input = sequnence_input[:, 1:, :]"
    assert str(z["reshape_skipped"]).startswith("DIEN/dien.py:283 not executed")
    cell = 1 if "_augru_" in name else 0
    L, T, T_neg = z["seq_len"], z["seq"].shape[1], int(z["T_neg"])
    assert {-1, 0, 1, 2, T, T + 3} <= set(L.tolist())
    for dt, sfx, tol in ((np.float32, "f32", 2e-6), (np.float64, "f64", 1e-13)):
        params = [z[k].astype(dt) for k in PNAMES]
        fs, _, aux = X.dien_aux_fwd(z["seq"].astype(dt), L, z["tgt"].astype(dt), z["neg"].astype(dt), params,
                                    z["w_aux"].astype(dt), cell, T_neg)
        ref = float(z["aux_loss_ref_" + sfx])
        assert ref < 0 < aux                                               # a sum of log-likelihoods; ours its negative
        assert abs(aux - (-ref)) <= tol * abs(ref), (sfx, aux, ref)
        assert rel(fs, z["final_state_" + sfx]) <= tol, sfx


def _torch_forward(seq, L, tgt, neg, params, W, cell, T_neg):
    """The reference form in torch float64 (every extractor position, masked softmax, copy-through past len), plus the
    auxiliary loss with the paper's sign computed at every position and masked."""
    gk, gb, ck, cb, Wa, egk, egb, eck, ecb = params
    B, T, na = seq.shape
    nh = Wa.shape[0]

    def gru(x, h, gk, gb, ck, cb):
        v = torch.sigmoid(torch.cat([x, h], 1) @ gk + gb)
        r, u = v[:, :nh], v[:, nh:]
        c = torch.tanh(torch.cat([x, r * h], 1) @ ck + cb)
        return r, u, c

    h = seq.new_zeros(B, nh)
    hs = []
    for t in range(T):
        r, u, c = gru(seq[:, t], h, gk, gb, ck, cb)
        h = u * h + (1 - u) * c
        hs.append(h)
    Hs = torch.stack(hs, 1)
    Lt = torch.as_tensor(np.clip(L, 0, T))
    mask = (torch.arange(T)[None, :] < Lt[:, None])[:, :, None]
    sc = Hs @ (Wa @ tgt[:, :, None])
    att = torch.softmax(torch.where(mask, sc, torch.full_like(sc, R.PAD)), dim=1)
    s = seq.new_zeros(B, nh)
    for t in range(T):
        a = att[:, t]
        r, u, c = gru(Hs[:, t], s, egk, egb, eck, ecb)
        sn = ((1 - a) * u) * s + (1 - (1 - a) * u) * c if cell == 1 else (1 - a) * s + a * c
        s = torch.where(mask[:, t], sn, s)
    q = Hs[:, :-1] @ W.T
    zp = (q * seq[:, 1:]).sum(-1)
    zn = torch.einsum("bti,btni->btn", q, neg.reshape(B, T - 1, T_neg, na))
    m = (torch.arange(T - 1)[None, :] < (Lt - 1)[:, None]).to(seq.dtype)
    aux = -(torch.nn.functional.logsigmoid(zp) * m).sum() - (torch.nn.functional.logsigmoid(-zn) * m[..., None]).sum()
    return s, aux / B


@pytest.mark.parametrize("cell", [0, 1])
@pytest.mark.parametrize("B,T,na,nh,T_neg", [(7, 7, 5, 3, 2), (6, 4, 3, 8, 1), (6, 5, 4, 4, 3)])
def test_analytic_backward_matches_autograd(B, T, na, nh, T_neg, cell):
    """d seq, d neg, d target, the nine and d W of g_final . final_state + g_aux * aux_loss."""
    rng = np.random.default_rng(B * 100 + T * 10 + T_neg + cell)
    L = np.array([-1, 0, 1, 2, T, T + 3] + [T - 1] * (B - 6), np.int64)
    seq = rng.standard_normal((B, T, na)) * 0.7
    seq[np.arange(T)[None, :] >= np.clip(L, 0, T)[:, None]] = 0
    neg = rng.standard_normal((B, (T - 1) * T_neg, na)) * 0.7
    tgt = rng.standard_normal((B, na)) * 0.7
    params = R.init_params(rng, na, nh, np.float64, bias_scale=0.5)
    W = rng.uniform(-1, 1, (na, nh)) * np.sqrt(6.0 / (na + nh)) * 2
    g, g_aux = rng.standard_normal((B, nh)), 1.7
    ts = [torch.tensor(x, requires_grad=True) for x in [seq, tgt, neg, W] + params]
    s, aux = _torch_forward(ts[0], L, ts[1], ts[2], ts[4:], ts[3], cell, T_neg)
    fs, _, aux_r = X.dien_aux_fwd(seq, L, tgt, neg, params, W, cell, T_neg)
    assert rel(fs, s.detach().numpy()) < 1e-13 and abs(aux_r - float(aux.detach())) <= 1e-13 * abs(float(aux.detach()))
    (s * torch.tensor(g)).sum().add(g_aux * aux).backward()
    d_seq, d_neg, d_tgt, dp, dW = X.dien_aux_bwd(seq, L, tgt, neg, params, W, cell, T_neg, g, g_aux)
    assert rel(d_seq, ts[0].grad.numpy()) < 1e-12
    assert rel(d_tgt, ts[1].grad.numpy()) < 1e-12
    assert rel(d_neg, ts[2].grad.numpy()) < 1e-12
    assert rel(dW, ts[3].grad.numpy()) < 1e-12
    for n, got, t in zip(PNAMES, dp, ts[4:]):
        assert rel(got, t.grad.numpy()) < 1e-12, n
    # exact zeros where a position does not count
    cnt = X.counted(L, T)
    assert np.all(d_neg.reshape(B, T - 1, T_neg, na)[~cnt] == 0)
    a_seq = X.aux_bwd(R.dien_fwd(seq, L, tgt, params, cell, return_cache=True)[2]["H"], seq, L, neg, W, T_neg, g_aux)[0]
    assert np.all(a_seq[:, 0] == 0)
    assert np.all(a_seq[np.arange(T)[None, :] >= np.clip(L, 0, T)[:, None]] == 0)


def test_stable_form_equals_reference_form_where_finite():
    """Parity note 5 (DESIGN §2, DIEN auxiliary loss): where tf.log(tf.sigmoid(.)) is finite the two forms agree to fp32; at extreme logits the reference
    gives inf (or NaN through -inf * 0 at a masked position) and the stable form stays finite."""
    rng = np.random.default_rng(3)
    B, T, na, nh, T_neg = 5, 6, 4, 3, 2
    L = np.array([0, 1, 3, 6, 9])
    seq = (rng.standard_normal((B, T, na)) * 0.7).astype(np.float32)
    neg = (rng.standard_normal((B, (T - 1) * T_neg, na)) * 0.7).astype(np.float32)
    H = rng.standard_normal((B, T, nh)).astype(np.float32)
    W = (rng.standard_normal((na, nh)) * 0.5).astype(np.float32)
    ours = X.aux_fwd(H, seq, L, neg, W, T_neg)
    ref = X.reference_form(H, seq, L, neg, W, T_neg)
    assert np.isfinite(ref) and abs(ours - ref) <= 2e-6 * abs(ref)
    big = W * 400                                                          # logits of order +-100 and beyond
    assert not np.isfinite(X.reference_form(H, seq, L, neg, big, T_neg))
    ours64 = X.aux_fwd(H.astype(np.float64), seq.astype(np.float64), L, neg.astype(np.float64), big.astype(np.float64), T_neg)
    ours32 = X.aux_fwd(H, seq, L, neg, big, T_neg)
    assert np.isfinite(ours64) and np.isfinite(ours32) and abs(ours32 - ours64) <= 1e-5 * abs(ours64)


def _digest(a):
    return f"{a.dtype.str}:{'x'.join(map(str, a.shape))}:{hashlib.sha256(a.tobytes()).hexdigest()}"


def test_fixtures_match_reference_digests(tmp_path):
    """Every array of every fixture is bit-identical to the recorded run over the reference.  With RECALG_REFERENCE set to a
    reference checkout's algorithm/ directory, tools/make_golden_dien_aux.py is run again into a scratch directory and held
    to the same digests."""
    want = json.load(open(os.path.join(G, "reference_digests.json")))
    assert sorted(want) == [n + ".npz" for n in NAMES]

    def check(directory):
        for name in want:
            z = np.load(os.path.join(directory, name), allow_pickle=False)
            assert {k: _digest(z[k]) for k in z.files} == want[name], name

    check(G)
    ref = os.environ.get("RECALG_REFERENCE")
    if not ref:
        return
    code = ("import importlib.util as u, sys; sys.argv=['make_golden_dien_aux'];"
            f"sys.path.insert(0, r'{ROOT}/tools');"
            f"s=u.spec_from_file_location('mga', r'{ROOT}/tools/make_golden_dien_aux.py'); m=u.module_from_spec(s);"
            f"s.loader.exec_module(m); m.gen_dien_aux(r'{tmp_path}')")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT,
                         env={**os.environ, "RECALG_REFERENCE": ref})
    assert out.returncode == 0, out.stderr[-2000:]
    check(str(tmp_path))
