"""CPU tests of the float64 DCN-V2 restatement (tests/_dcnv2_ref.py) that the GPU tests compare against: its analytic
backward against torch.autograd, its anchor to row CROSS (DCN v1, pinned by the cross fixtures), and the identity between
the low-rank layer at r = d, u = I and the full-rank layer."""
import numpy as np
import pytest
import torch

from _dcnv2_ref import cross_v2_bwd, cross_v2_fwd
from _util import golden
from oracle import layers_np as O


def _torch_fwd(x0, w, u, b, xl):
    x = x0 if xl is None else xl
    for l in range(w.shape[0]):
        z = (x @ w[l] if u is None else (x @ w[l]) @ u[l]) + b[l]
        x = x0 * z + x
    return x


@pytest.mark.parametrize("rank", [0, 1, 3, 7])
@pytest.mark.parametrize("with_xl", [False, True])
@pytest.mark.parametrize("L", [1, 3])
def test_analytic_backward_equals_autograd(rank, with_xl, L):
    rng = np.random.default_rng(rank * 10 + L + with_xl)
    B, d = 6, 9
    x0 = rng.standard_normal((B, d))
    xl = rng.standard_normal((B, d)) if with_xl else None
    w = rng.standard_normal((L, d, rank or d)) * 0.3
    u = rng.standard_normal((L, rank, d)) * 0.3 if rank else None
    b = rng.standard_normal((L, d))
    g = rng.standard_normal((B, d))
    out, cache = cross_v2_fwd(x0, w, u, b, xl)
    got = cross_v2_bwd(cache, w, u, g)
    ts = {k: torch.tensor(v, requires_grad=True) for k, v in (("x0", x0), ("xl", xl), ("w", w), ("u", u), ("b", b))
          if v is not None}
    ref_out = _torch_fwd(ts["x0"], ts["w"], ts.get("u"), ts["b"], ts.get("xl"))
    np.testing.assert_allclose(out, ref_out.detach().numpy(), rtol=1e-12, atol=1e-12)
    ref_out.backward(torch.tensor(g))
    for name, val in zip(("x0", "xl", "w", "u", "b"), got):
        if name in ts:
            np.testing.assert_allclose(val, ts[name].grad.numpy(), rtol=1e-11, atol=1e-11, err_msg=name)
        else:
            assert val is None, name


@pytest.mark.parametrize("fixture", ["cross_d82_L3", "cross_d480_L3"])
def test_anchor_to_row_cross(fixture):
    """With b = 0, the rank-1 layer w[l] = ws[l] as a column, u[l] = a row of ones, and the full-rank layer whose every
    column is ws[l], are both DCN v1's x0 (x_l . ws[l]) + x_l: out, dx0 and dw match oracle.layers_np.cross_stack_* (v1 with
    zero bias; its forward is pinned by the fixture)."""
    z = golden(fixture)
    x0, ws = z["x0"].astype(np.float64), z["ws"].astype(np.float64)
    L, d = ws.shape
    zero_b = np.zeros((L, d))
    np.testing.assert_allclose(O.cross_stack_fwd(x0, ws, z["bs"].astype(np.float64))[-1], z["out_f64"], rtol=1e-12, atol=1e-12)
    v1_out = O.cross_stack_fwd(x0, ws, zero_b)[-1]
    g = np.random.default_rng(0).standard_normal(x0.shape)
    v1_dx0, v1_dw, _ = O.cross_stack_bwd(x0, ws, zero_b, g)

    w1, u1 = ws[:, :, None], np.ones((L, 1, d))
    out, cache = cross_v2_fwd(x0, w1, u1, zero_b)
    dx0, _, dw, du, _ = cross_v2_bwd(cache, w1, u1, g)
    np.testing.assert_allclose(out, v1_out, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(dx0, v1_dx0, rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(dw[:, :, 0], v1_dw, rtol=1e-11, atol=1e-11)

    wf = np.repeat(ws[:, :, None], d, axis=2)                  # every column of W_l is ws[l]
    out, cache = cross_v2_fwd(x0, wf, None, zero_b)
    dx0, _, dw, _, _ = cross_v2_bwd(cache, wf, None, g)
    np.testing.assert_allclose(out, v1_out, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(dx0, v1_dx0, rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(dw.sum(axis=2), v1_dw, rtol=1e-11, atol=1e-11)   # dW_l[:, j] summed over j is v1's dw


def test_rank_d_with_identity_u_is_the_full_rank_layer():
    rng = np.random.default_rng(3)
    B, d, L = 5, 7, 3
    x0, xl = rng.standard_normal((B, d)), rng.standard_normal((B, d))
    w, b = rng.standard_normal((L, d, d)) * 0.3, rng.standard_normal((L, d))
    g = rng.standard_normal((B, d))
    u = np.repeat(np.eye(d)[None], L, axis=0)
    full_out, full_cache = cross_v2_fwd(x0, w, None, b, xl)
    low_out, low_cache = cross_v2_fwd(x0, w, u, b, xl)
    np.testing.assert_allclose(low_out, full_out, rtol=1e-12, atol=1e-12)
    full = cross_v2_bwd(full_cache, w, None, g)
    low = cross_v2_bwd(low_cache, w, u, g)
    for name, a, c in zip(("dx0", "dxl", "dw", "db"), low[:3] + low[4:], full[:3] + full[4:]):
        np.testing.assert_allclose(a, c, rtol=1e-11, atol=1e-11, err_msg=name)
