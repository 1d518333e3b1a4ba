"""CPU tests of the float64 DCN-Mix restatement (tests/_dcnmix_ref.py) that the GPU tests compare against: its analytic
backward against torch.autograd, the paper's per-expert form against the collapsed form the kernels compute, and its
anchor to the DCN-V2 low-rank layer (tests/_dcnv2_ref.py) and, through it, to row CROSS (DCN v1, pinned by the cross
fixtures)."""
import numpy as np
import pytest
import torch

from _dcnmix_ref import cross_mix_bwd, cross_mix_fwd, cross_mix_fwd_collapsed
from _dcnv2_ref import cross_v2_bwd, cross_v2_fwd
from _util import golden
from oracle import layers_np as O


def _weights(rng, L, K, d, r, scale=0.4):
    v = rng.standard_normal((L, K, d, r)) * scale
    c = rng.standard_normal((L, K, r, r)) * scale
    u = rng.standard_normal((L, K, r, d)) * scale
    b = rng.standard_normal((L, d))
    gate = rng.standard_normal((d, K))
    return v, c, u, b, gate


def _torch_fwd(x0, v, c, u, b, gate, act):
    g = torch.tanh if act else (lambda t: t)
    x = x0
    for l in range(v.shape[0]):
        p = torch.softmax(x @ gate, dim=1)
        x = sum(p[:, i:i + 1] * (x0 * (g(g(x @ v[l, i]) @ c[l, i]) @ u[l, i] + b[l])) for i in range(v.shape[1])) + x
    return x


@pytest.mark.parametrize("act", [0, 1])
@pytest.mark.parametrize("L", [1, 3])
@pytest.mark.parametrize("K,r", [(1, 1), (3, 2), (4, 5)])
def test_analytic_backward_equals_autograd(act, L, K, r):
    rng = np.random.default_rng(act * 100 + L * 10 + K + r)
    B, d = 6, 9
    x0 = rng.standard_normal((B, d))
    w = _weights(rng, L, K, d, r)
    g = rng.standard_normal((B, d))
    out, cache = cross_mix_fwd(x0, *w, act)
    got = cross_mix_bwd(cache, w[0], w[1], w[2], w[4], g)
    ts = [torch.tensor(a, requires_grad=True) for a in (x0, *w)]
    ref_out = _torch_fwd(*ts, act)
    np.testing.assert_allclose(out, ref_out.detach().numpy(), rtol=1e-12, atol=1e-12)
    ref_out.backward(torch.tensor(g))
    for name, val, t in zip(("dx0", "dv", "dc", "du", "db", "dgate"), got, ts):
        np.testing.assert_allclose(val, t.grad.numpy(), rtol=1e-11, atol=1e-11, err_msg=name)


@pytest.mark.parametrize("act", [0, 1])
def test_per_expert_form_equals_the_collapsed_form(act):
    rng = np.random.default_rng(20 + act)
    B, d, L, K, r = 7, 11, 3, 4, 3
    x0 = rng.standard_normal((B, d))
    w = _weights(rng, L, K, d, r)
    np.testing.assert_allclose(cross_mix_fwd_collapsed(x0, *w, act), cross_mix_fwd(x0, *w, act)[0], rtol=1e-13, atol=1e-13)


def test_one_expert_with_identity_and_c_equal_to_i_is_the_dcn_v2_low_rank_layer():
    rng = np.random.default_rng(4)
    B, d, L, r = 6, 10, 3, 4
    x0 = rng.standard_normal((B, d))
    v, _, u, b, gate = _weights(rng, L, 1, d, r)
    c = np.broadcast_to(np.eye(r), (L, 1, r, r))
    g = rng.standard_normal((B, d))
    out, cache = cross_mix_fwd(x0, v, c, u, b, gate, 0)
    dx0, dv, dc, du, db, dgate = cross_mix_bwd(cache, v, c, u, gate, g)
    v2_out, v2_cache = cross_v2_fwd(x0, v[:, 0], u[:, 0], b)
    v2_dx0, _, v2_dw, v2_du, v2_db = cross_v2_bwd(v2_cache, v[:, 0], u[:, 0], g)
    np.testing.assert_allclose(out, v2_out, rtol=1e-13, atol=1e-13)
    for name, a, e in (("dx0", dx0, v2_dx0), ("dv", dv[:, 0], v2_dw), ("du", du[:, 0], v2_du), ("db", db, v2_db)):
        np.testing.assert_allclose(a, e, rtol=1e-13, atol=1e-13, err_msg=name)
    assert not dgate.any()                                  # one expert: p = 1 whatever the gate


@pytest.mark.parametrize("act", [0, 1])
def test_rank_one_expert_with_zero_bias_is_row_cross(act):
    """r = 1, K = 1, c = 1, b = 0, v[l] = ws[l] as a column and u[l] a row of ones: DCN v1 with zero bias, whose forward
    the fixture pins (oracle.layers_np.cross_stack_fwd/bwd).  Only the identity makes it so; tanh is checked to differ."""
    z = golden("cross_d82_L3")
    x0, ws = z["x0"].astype(np.float64), z["ws"].astype(np.float64)
    L, d = ws.shape
    zero_b = np.zeros((L, d))
    np.testing.assert_allclose(O.cross_stack_fwd(x0, ws, z["bs"].astype(np.float64))[-1], z["out_f64"], rtol=1e-12, atol=1e-12)
    v1_out = O.cross_stack_fwd(x0, ws, zero_b)[-1]
    g = np.random.default_rng(0).standard_normal(x0.shape)
    v1_dx0, v1_dw, _ = O.cross_stack_bwd(x0, ws, zero_b, g)
    v, c, u = ws[:, None, :, None], np.ones((L, 1, 1, 1)), np.ones((L, 1, 1, d))
    gate = np.random.default_rng(1).standard_normal((d, 1))
    out, cache = cross_mix_fwd(x0, v, c, u, zero_b, gate, act)
    if not act:
        dx0, dv, _, _, _, _ = cross_mix_bwd(cache, v, c, u, gate, g)
        np.testing.assert_allclose(out, v1_out, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(dx0, v1_dx0, rtol=1e-11, atol=1e-11)
        np.testing.assert_allclose(dv[:, 0, :, 0], v1_dw, rtol=1e-11, atol=1e-11)
    else:
        assert np.abs(out - v1_out).max() > 1e-3
