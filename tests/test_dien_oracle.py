"""CPU tests of DIEN's seq_encoder block (DIEN/dien.py:198-229): the float64 restatement (tests/_dien_ref.py) against the
fixtures produced by executing the reference's lines and its verbatim cells (tools/make_golden_dien.py), its analytic
backward against torch.autograd, the exactness of skipping the positions t >= len, and the fixture digests."""
import glob
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _dien_ref as R

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dien")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(G, "*.npz")))
PNAMES = ("gk", "gb", "ck", "cb", "att", "egk", "egb", "eck", "ecb")


def rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def _case(rng, B, T, na, nh, lens=None, dtype=np.float64, bias_scale=0.5):
    seq = rng.standard_normal((B, T, na)) * 0.7
    L = rng.integers(0, T + 4, B) if lens is None else np.asarray(lens)
    seq[np.arange(T)[None, :] >= np.clip(L, 0, T)[:, None]] = 0          # sequence_input_layer pads with zeros
    tgt = rng.standard_normal((B, na)) * 0.7
    params = R.init_params(rng, na, nh, dtype, bias_scale=bias_scale)
    return seq.astype(dtype), L.astype(np.int64), tgt.astype(dtype), params


def test_fixtures_present():
    assert NAMES == ["dien_agru_na16_nh8_T50_B16", "dien_agru_na5_nh3_T7_B9", "dien_augru_na16_nh8_T50_B16",
                     "dien_augru_na5_nh3_T7_B9"]


@pytest.mark.parametrize("name", NAMES)
def test_restatement_matches_reference_executed(name):
    z = np.load(os.path.join(G, name + ".npz"), allow_pickle=False)
    assert str(z["source"]).startswith("reference-executed:DIEN/dien.py:198-229")
    cell = 1 if "_augru_" in name else 0
    L = z["seq_len"]
    T = z["seq"].shape[1]
    assert {0, 1, T, T + 3} <= set(L.tolist())
    for dt, sfx, tol in ((np.float32, "f32", 2e-6), (np.float64, "f64", 1e-13)):
        params = [z[k].astype(dt) for k in PNAMES]
        fs, att = R.dien_fwd(z["seq"].astype(dt), L, z["tgt"].astype(dt), params, cell)
        assert rel(fs, z["final_state_" + sfx]) <= tol, sfx
        assert rel(att, z["att_" + sfx][..., 0]) <= tol, sfx
    att = z["att_f64"][..., 0]
    assert np.all(att[L == 0] == 1.0 / T)                                  # len = 0: uniform 1/T
    assert np.all(z["final_state_f64"][L == 0] == 0)                       # ... and a zero final state
    for b in np.nonzero(L >= 1)[0]:
        assert np.all(att[b, min(L[b], T):] == 0)                          # masked weights are exactly 0


def test_restated_grucell_is_the_reference_augru_at_zero_attention():
    """Pinned by the generator (GRUCell restatement == verbatim AUGRUCell at att_score = 0); recorded in every fixture."""
    for name in NAMES:
        z = np.load(os.path.join(G, name + ".npz"), allow_pickle=False)
        assert float(z["grucell_vs_augru_at_a0_maxabs"]) == 0.0


def _torch_forward(seq, L, tgt, params, cell):
    """The reference form in torch float64: every extractor position, masked softmax, copy-through past len."""
    gk, gb, ck, cb, W, egk, egb, eck, ecb = params
    B, T, na = seq.shape
    nh = W.shape[0]

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
    sc = Hs @ (W @ tgt[:, :, None])
    mask = (torch.arange(T)[None, :] < torch.as_tensor(L)[:, None])[:, :, None]
    att = torch.softmax(torch.where(mask, sc, torch.full_like(sc, R.PAD)), dim=1)
    s = seq.new_zeros(B, nh)
    for t in range(T):
        a = att[:, t]
        r, u, c = gru(Hs[:, t], s, egk, egb, eck, ecb)
        sn = ((1 - a) * u) * s + (1 - (1 - a) * u) * c if cell == 1 else (1 - a) * s + a * c
        s = torch.where(mask[:, t], sn, s)
    return s, att[..., 0]


@pytest.mark.parametrize("cell", [0, 1])
@pytest.mark.parametrize("B,T,na,nh", [(6, 7, 5, 3), (5, 4, 3, 8)])
def test_analytic_backward_matches_autograd(B, T, na, nh, cell):
    rng = np.random.default_rng(B * 10 + T + cell)
    seq, L, tgt, params = _case(rng, B, T, na, nh, lens=[0, 1, T, T + 3] + [2] * (B - 4))
    g = rng.standard_normal((B, nh))
    ts = [torch.tensor(x, requires_grad=True) for x in [seq, tgt] + params]
    s, att = _torch_forward(ts[0], np.clip(L, 0, T), ts[1], ts[2:], cell)
    fs, A = R.dien_fwd(seq, L, tgt, params, cell)
    assert rel(fs, s.detach().numpy()) < 1e-13 and rel(A, att.detach().numpy()) < 1e-13
    s.backward(torch.tensor(g))
    d_seq, d_tgt, dp = R.dien_bwd(seq, L, tgt, params, cell, g)
    assert rel(d_seq, ts[0].grad.numpy()) < 1e-12
    assert rel(d_tgt, ts[1].grad.numpy()) < 1e-12
    for n, got, t in zip(PNAMES, dp, ts[2:]):
        assert rel(got, t.grad.numpy()) < 1e-12, n
    if cell == 0:                                                          # AGRU never uses u
        assert np.all(dp[5][:, nh:] == 0) and np.all(dp[6][nh:] == 0)
        assert np.all(ts[7].grad.numpy()[:, nh:] == 0) and np.all(ts[8].grad.numpy()[nh:] == 0)
    pad = np.arange(T)[None, :] >= np.clip(L, 0, T)[:, None]
    assert np.all(d_seq[pad] == 0) and np.all(ts[0].grad.numpy()[pad] == 0)


@pytest.mark.parametrize("cell", [0, 1])
def test_skipping_padded_positions_is_exact(cell):
    """Computing only t < len (what the kernels do) gives bit-identical outputs and gradients in float64."""
    rng = np.random.default_rng(77 + cell)
    B, T, na, nh = 9, 11, 6, 5
    seq, L, tgt, params = _case(rng, B, T, na, nh, lens=[0, 1, T, T + 3, 5, 7, 2, 10, 3])
    g = rng.standard_normal((B, nh))
    full = R.dien_fwd(seq, L, tgt, params, cell, skip=False)
    skip = R.dien_fwd(seq, L, tgt, params, cell, skip=True)
    for a, b in zip(full, skip):
        assert np.array_equal(a, b)
    gf = R.dien_bwd(seq, L, tgt, params, cell, g, skip=False)
    gs = R.dien_bwd(seq, L, tgt, params, cell, g, skip=True)
    assert np.array_equal(gf[0], gs[0]) and np.array_equal(gf[1], gs[1])
    for a, b in zip(gf[2], gs[2]):
        assert np.array_equal(a, b)
    A = full[1]
    for b in range(B):
        if 1 <= L[b] < T:
            assert np.all(A[b, L[b]:] == 0)                                # exp(-2^32 - max) underflows to exactly 0
    # the same in fp32: a masked weight is exactly 0
    A32 = R.dien_fwd(seq.astype(np.float32), L, tgt.astype(np.float32), [p.astype(np.float32) for p in params], cell)[1]
    assert all(np.all(A32[b, L[b]:] == 0) for b in range(B) if 1 <= L[b] < T)


def _digest(a):
    return f"{a.dtype.str}:{'x'.join(map(str, a.shape))}:{hashlib.sha256(a.tobytes()).hexdigest()}"


def test_fixtures_match_reference_digests(tmp_path):
    """Every array of every fixture is bit-identical to the recorded run over the reference.  With RECALG_REFERENCE set to a
    reference checkout's algorithm/ directory, tools/make_golden_dien.py is run again into a scratch directory and held to
    the same digests."""
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
    code = ("import importlib.util as u, sys; sys.argv=['make_golden_dien'];"
            f"s=u.spec_from_file_location('mg', r'{ROOT}/tools/make_golden_dien.py'); m=u.module_from_spec(s); s.loader.exec_module(m);"
            f"m.gen_dien(r'{tmp_path}')")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT,
                         env={**os.environ, "RECALG_REFERENCE": ref})
    assert out.returncode == 0, out.stderr[-2000:]
    check(str(tmp_path))
