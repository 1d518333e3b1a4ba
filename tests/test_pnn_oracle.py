"""CPU tests of the PNN product layer (PNN/pnn.py:125-181): the restatement (tests/_pnn_ref.py) against the fixtures produced by
executing the reference's lines (tools/make_golden_pnn.py), its analytic backward against torch.autograd, the single-GEMM
feature-row form the kernels compute against the direct form, the fixture digests, and the host layer's variables."""
import glob
import hashlib
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _pnn_ref as R

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pnn")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(G, "*.npz")))


def rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def test_fixtures_present():
    assert NAMES == ["pnn_ipnn_F5_K4_N24", "pnn_ipnn_F8_K8_N128", "pnn_opnn_F5_K4_N24", "pnn_opnn_F8_K8_N128"]


@pytest.mark.parametrize("name", NAMES)
def test_restatement_matches_reference_executed(name):
    z = np.load(os.path.join(G, name + ".npz"), allow_pickle=False)
    assert str(z["source"]).startswith("reference-executed:PNN/pnn.py")
    method = 0 if "_ipnn_" in name else 1
    for dt, key, tol in ((np.float32, "out_f32", 2e-6), (np.float64, "out_f64", 1e-13)):
        out = R.pnn_fwd(*(z[k].astype(dt) for k in ("e", "linear_w", "product_w", "bias")), method)
        assert rel(out, z[key]) <= tol, key
    assert 0.2 < (z["out_f64"] > 0).mean() < 0.9                       # the relu is exercised on both sides
    # weight_regularizer (quirk 4): l2_regularizer(0.01) adds 0.01 * sum(w**2) / 2 for linear_w and the product weight only
    want = 0.01 * 0.5 * sum(float(np.sum(z[k].astype(np.float64) ** 2)) for k in ("linear_w", "product_w"))
    assert abs(float(z["reg_loss_scale_0_01"]) - want) <= 1e-12 * want


@pytest.mark.parametrize("method", [0, 1])
def test_analytic_backward_matches_autograd(method):
    rng = np.random.default_rng(5 + method)
    B, F, K, N = 6, 5, 4, 9
    e, wl, b, g = rng.standard_normal((B, F, K)), rng.standard_normal((F * K, N)), rng.standard_normal(N), rng.standard_normal((B, N))
    wp = rng.standard_normal((N, F) if method == 0 else (N, K, K))
    et, wlt, wpt, bt = (torch.tensor(x, requires_grad=True) for x in (e, wl, wp, b))
    lz = et.reshape(B, -1) @ wlt
    if method == 0:
        delta = torch.einsum("bfk,nf->bnk", et, wpt)
        lp = (delta * delta).sum(-1)
    else:
        s = et.sum(1)
        up = torch.triu(wpt)
        lp = torch.einsum("bkl,nkl->bn", s[:, :, None] * s[:, None, :],
                          up + up.transpose(1, 2) - torch.diag_embed(torch.diagonal(wpt, dim1=1, dim2=2)))
    out = torch.relu(lz + lp + bt)
    assert rel(R.pnn_fwd(e, wl, wp, b, method), out.detach().numpy()) < 1e-13
    out.backward(torch.tensor(g))
    for got, t in zip(R.pnn_bwd(e, wl, wp, b, method, g), (et, wlt, wpt, bt)):
        assert rel(got, t.grad.numpy()) < 1e-12
    if method == 1:                                                      # quirk 3: the lower triangle is never read
        low = np.tril(np.ones((K, K), bool), -1)
        assert np.all(wpt.grad.numpy()[:, low] == 0)
        d = R.pnn_bwd(e, wl, wp, b, method, g)[2]
        assert np.all(d[:, low] == 0)


@pytest.mark.parametrize("method", [0, 1])
@pytest.mark.parametrize("F,K,N", [(8, 8, 64), (1, 5, 7), (6, 1, 9), (30, 16, 12)])
def test_feature_row_form_equals_direct_form(F, K, N, method):
    """out = relu(xt . Wm): xt = [e_flat | upper-triangle pair features | 1], Wm = [linear_w ; c-weighted products ; bias]."""
    rng = np.random.default_rng(F * 100 + K * 10 + method)
    B = 7
    e, wl, b = rng.standard_normal((B, F, K)), rng.standard_normal((F * K, N)), rng.standard_normal(N)
    wp = rng.standard_normal((N, F) if method == 0 else (N, K, K))
    xt, wm = R.feature_rows(e, method), R.feature_weights(wl, wp, b, method)
    Q = F * (F + 1) // 2 if method == 0 else K * (K + 1) // 2
    assert xt.shape == (B, F * K + Q + 1) and wm.shape == (F * K + Q + 1, N)
    _, lz, lp = R.pnn_fwd(e, wl, wp, b, method, return_parts=True)
    pre = xt @ wm
    assert np.abs(pre - (lz + lp + b)).max() <= 1e-12 * np.abs(lz + lp + b).max()
    if method == 1:                                                      # changing the lower triangle changes nothing
        wp2 = wp + np.tril(rng.standard_normal(wp.shape), -1)
        assert np.array_equal(R.feature_weights(wl, wp2, b, method), wm)


def _digest(a):
    return f"{a.dtype.str}:{'x'.join(map(str, a.shape))}:{hashlib.sha256(a.tobytes()).hexdigest()}"


def test_fixtures_match_reference_digests(tmp_path):
    """Every array of every fixture is bit-identical to the recorded run over the reference.  With RECALG_REFERENCE set to a
    reference checkout's algorithm/ directory, tools/make_golden_pnn.py is run again into a scratch directory and held to
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
    code = ("import importlib.util as u, sys; sys.argv=['make_golden_pnn'];"
            f"s=u.spec_from_file_location('mg', r'{ROOT}/tools/make_golden_pnn.py'); m=u.module_from_spec(s); s.loader.exec_module(m);"
            f"m.gen_pnn(r'{tmp_path}')")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT,
                         env={**os.environ, "RECALG_REFERENCE": ref})
    assert out.returncode == 0, out.stderr[-2000:]
    check(str(tmp_path))


# ---------------------------------------------------------------- host layer: variables, shapes, initialisers (launch stubbed)
@pytest.fixture()
def store(monkeypatch):
    from recalgorithm_b200 import autograd, layers as L
    calls = []

    def fake_pnn(e, wlin, wprod, bias, method):
        calls.append((e, wlin, wprod, bias, method))
        return torch.zeros(e.shape[0], wlin.shape[1])
    monkeypatch.setattr(autograd, "pnn", fake_pnn)
    st = L.set_default_store(L.VariableStore(device="cpu", seed=0))
    st.calls = calls
    yield st
    L.set_default_store(L.VariableStore(device="cpu"))


@pytest.mark.parametrize("product_method,method", [("IPNN", 0), ("OPNN", 1), ("ipnn", 1), ("anything", 1)])
def test_pnn_product_layer_variables(store, product_method, method):
    """Quirk 1: only the exact string "IPNN" builds inner_product_w; any other product_method takes the OPNN branch.
    Quirk 2: bias is a plain get_variable -- glorot-uniform, not zero."""
    from recalgorithm_b200 import layers as L
    F, K, N, B = 8, 8, 1024, 3
    out = L.pnn_product_layer(torch.randn(B, F * K), F, K, N, product_method=product_method)
    assert out.shape == (B, N)
    wname = "product_part/inner_product_w" if method == 0 else "product_part/outer_product_w"
    wshape = (N, F) if method == 0 else (N, K, K)
    assert {k: tuple(v.shape) for k, v in store.vars.items()} == {"linear_part/linear_w": (F * K, N), wname: wshape, "bias": (N,)}
    fans = {"linear_part/linear_w": (F * K, N), wname: (N, F) if method == 0 else (N * K, N * K), "bias": (N, N)}
    for name, (fi, fo) in fans.items():
        v = store.vars[name].detach()
        lim = math.sqrt(6.0 / (fi + fo))
        assert float(v.abs().max()) <= lim and float(v.abs().max()) > 0.9 * lim, name      # glorot-uniform, bias included
    e, wlin, wprod, bias, m = store.calls[-1]
    assert m == method and tuple(e.shape) == (B, F, K) and wprod is store.vars[wname] and bias is store.vars["bias"]
