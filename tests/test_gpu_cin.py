"""GPU parity: xDeepFM CIN layer (row CIN) -- wgmma tensor-core path and the CUDA-core path -- vs golden vectors
(reference source executed) and the oracle."""
import numpy as np
import pytest
import torch

from _util import TOL, assert_close, dev, golden, relerr, trunc_normal
from oracle import layers_np as O

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["cin_m8_D8_50x50x50", "cin_m10_D16_128x128", "cin_m8_D16_17"])
def test_cin_golden(name):
    from recalgorithm_b200 import ops
    g = golden(name)
    x0 = dev(g["x0"])
    xk, pools = x0, []
    for i in range(int(g["n_layers"])):
        xk, pooled = ops.cin_fwd(x0, xk, dev(g[f"filter_{i + 1}"]), want_pooled=True)
        assert_close(xk, g[f"x{i + 1}_f64"], TOL, f"layer {i + 1} vs reference(float64)")
        assert_close(xk, g[f"x{i + 1}_f32"], TOL, f"layer {i + 1} vs reference(float32)")
        pools.append(pooled)
    assert_close(torch.cat(pools, dim=-1), g["p_plus_f64"], TOL, "p_plus")


CASES = [(3, 5, 4, 8, 7), (16, 30, 30, 16, 128), (16, 30, 128, 16, 128), (33, 8, 50, 8, 50), (5, 30, 100, 16, 100),
         (40, 6, 6, 32, 16), (2, 32, 3, 4, 128), (9, 1, 1, 16, 1), (130, 10, 20, 16, 64)]


@pytest.mark.parametrize("B,m,hk,D,H", CASES)
def test_cin_fwd_tensor_path(B, m, hk, D, H):
    from recalgorithm_b200 import ops
    rng = np.random.default_rng(B + m + hk + D + H)
    x0 = trunc_normal(rng, (B, m, D), 0.5); xk = trunc_normal(rng, (B, hk, D), 0.5)
    w = trunc_normal(rng, (hk * m, H), 0.2)
    ref = O.cin_layer_fwd(x0.astype(np.float64), xk.astype(np.float64), w.astype(np.float64))
    out, pooled = ops.cin_fwd(dev(x0), dev(xk), dev(w), want_pooled=True)
    assert_close(out, ref, TOL, "3xTF32 tensor-core forward")
    assert_close(pooled, ref.sum(-1), TOL, "pooled")
    fast = ops.cin_fwd(dev(x0), dev(xk), dev(w), precision=1)
    e = relerr(fast, ref)
    assert e < 5e-3, f"single-pass TF32 error {e}"
    assert torch.equal(ops.cin_fwd(dev(x0), dev(xk), dev(w)), out), "deterministic"


@pytest.mark.parametrize("B,m,hk,D,H", [(3, 40, 5, 8, 9), (4, 6, 7, 12, 10), (2, 5, 6, 64, 8), (3, 4, 4, 8, 130)])
def test_cin_fwd_cuda_core_path(B, m, hk, D, H):
    """Shapes outside the tensor path (m > 32, D not a power of two, D > 32, H > 128)."""
    from recalgorithm_b200 import ops
    rng = np.random.default_rng(B + m + hk + D + H)
    x0 = trunc_normal(rng, (B, m, D), 0.5); xk = trunc_normal(rng, (B, hk, D), 0.5)
    w = trunc_normal(rng, (hk * m, H), 0.2)
    ref = O.cin_layer_fwd(x0.astype(np.float64), xk.astype(np.float64), w.astype(np.float64))
    out, pooled = ops.cin_fwd(dev(x0), dev(xk), dev(w), want_pooled=True)
    assert_close(out, ref, TOL, "fwd"); assert_close(pooled, ref.sum(-1), TOL, "pooled")


@pytest.mark.parametrize("B,m,hk,D,H", [(3, 5, 4, 8, 7), (8, 30, 30, 16, 128), (4, 30, 128, 16, 128), (33, 8, 50, 8, 50),
                                        (70, 30, 100, 16, 100), (9, 32, 13, 32, 48), (1, 1, 1, 16, 1), (300, 6, 9, 16, 20),
                                        (5, 7, 6, 4, 9), (3, 40, 5, 8, 9)])
def test_cin_bwd(B, m, hk, D, H):
    from recalgorithm_b200 import ops
    rng = np.random.default_rng(B + m + hk + D + H + 1)
    x0 = trunc_normal(rng, (B, m, D), 0.5); xk = trunc_normal(rng, (B, hk, D), 0.5)
    w = trunc_normal(rng, (hk * m, H), 0.2); g = trunc_normal(rng, (B, H, D), 1.0)
    d = lambda a: a.astype(np.float64)
    dx0, dxk, dw = ops.cin_bwd(dev(x0), dev(xk), dev(w), dev(g))
    ex0, exk, ew = O.cin_layer_bwd(d(x0), d(xk), d(w), d(g))
    assert_close(dx0, ex0, TOL, "dx0"); assert_close(dxk, exk, TOL, "dxk"); assert_close(dw, ew, TOL, "dfilter")


def test_cin_config3_properties():
    """BASELINE config 3 (B=8192, m=30, D=16, maps [128,128]): linearity in the filter and agreement with a float64
    einsum on a batch subsample."""
    from recalgorithm_b200 import ops
    B, m, D, H = 8192, 30, 16, 128
    gen = torch.Generator(device="cuda").manual_seed(3)
    x0 = torch.randn((B, m, D), device="cuda", generator=gen) * 0.25
    w1 = torch.randn((m * m, H), device="cuda", generator=gen) * 0.05
    w2 = torch.randn((H * m, H), device="cuda", generator=gen) * 0.05
    x1 = ops.cin_fwd(x0, x0, w1)
    x2, p2 = ops.cin_fwd(x0, x1, w2, want_pooled=True)
    sub = slice(0, B, 257)
    r1 = torch.einsum("bid,bjd,ijn->bnd", x0[sub].double(), x0[sub].double(), w1.double().reshape(m, m, H))
    r2 = torch.einsum("bid,bjd,ijn->bnd", r1, x0[sub].double(), w2.double().reshape(H, m, H))
    assert_close(x1[sub], r1, TOL, "layer 1"); assert_close(x2[sub], r2, TOL, "layer 2")
    assert_close(p2[sub], r2.sum(-1), TOL, "pooled")
    # linearity in the filter: cin(w_a + w_b) == cin(w_a) + cin(w_b)
    wb = torch.randn((H * m, H), device="cuda", generator=gen) * 0.05
    lhs = ops.cin_fwd(x0, x1, w2 + wb)
    rhs = ops.cin_fwd(x0, x1, w2) + ops.cin_fwd(x0, x1, wb)
    assert_close(lhs, rhs.double(), 2e-5, "linearity")


@pytest.mark.parametrize("D", [16, 32])
def test_cin_config3_backward(D):
    """Backward at BASELINE config-3 size (B=8192, m=30, hk=128, H=128; D=16 as in the config, D=32 for the dW kernel's
    128-byte swizzled gradient tiles: several rounds of the persistent dX schedule incl. its tail, 32 (i,j)-groups x 4 batch
    slices of the dW kernel): dx0 / dxk against a float64 einsum on a batch subsample (a sample's input gradients only depend
    on that sample), dfilter against the float64 contraction over the WHOLE batch (chunked)."""
    from recalgorithm_b200 import ops
    B, m, hk, H = 8192, 30, 128, 128
    gen = torch.Generator(device="cuda").manual_seed(5)
    x0 = torch.randn((B, m, D), device="cuda", generator=gen) * 0.25
    xk = torch.randn((B, hk, D), device="cuda", generator=gen) * 0.25
    w = torch.randn((hk * m, H), device="cuda", generator=gen) * 0.05
    g = torch.randn((B, H, D), device="cuda", generator=gen)
    dx0, dxk, dw = ops.cin_bwd(x0, xk, w, g)
    torch.cuda.synchronize()
    sub = torch.arange(0, B, 131, device="cuda")                       # 63 samples spread over the tiles (incl. tile boundaries)
    sub = torch.cat([sub, torch.tensor([7, 8, 15, 16, B - 1], device="cuda")])
    w3 = w.double().reshape(hk, m, H)
    dz = torch.einsum("bnd,ijn->bijd", g[sub].double(), w3)            # dL/d(outer[b,i,j,d])
    assert_close(dxk[sub], torch.einsum("bijd,bjd->bid", dz, x0[sub].double()), TOL, "dxk (config-3 size)")
    assert_close(dx0[sub], torch.einsum("bijd,bid->bjd", dz, xk[sub].double()), TOL, "dx0 (config-3 size)")
    ref = torch.zeros((hk, m, H), dtype=torch.float64, device="cuda")
    for b0 in range(0, B, 512):
        sl = slice(b0, b0 + 512)
        z = torch.einsum("bid,bjd->bdij", xk[sl].double(), x0[sl].double()).reshape(-1, hk * m)       # (b*d, i*m+j)
        ref += (z.t() @ g[sl].double().permute(0, 2, 1).reshape(-1, H)).reshape(hk, m, H)
    assert_close(dw, ref.reshape(hk * m, H), TOL, "dfilter (config-3 size, whole batch)")
