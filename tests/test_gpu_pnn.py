"""GPU parity: the PNN product layer (IPNN / OPNN) -- wgmma tensor-core kernels and the CUDA-core path -- against the
reference-executed fixtures (tests/golden/pnn) and the float64 restatement (tests/_pnn_ref.py)."""
import glob
import os

import numpy as np
import pytest
import torch

from _pnn_ref import pnn_bwd as ref_bwd, pnn_fwd as ref_fwd
from _util import GOLDEN, TOL, assert_close, dev

pytestmark = pytest.mark.gpu

FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "pnn", "*.npz")))


def _fixture(name):
    return np.load(os.path.join(GOLDEN, "pnn", name + ".npz"), allow_pickle=False)


def _inputs(B, F, K, N, method, seed):
    rng = np.random.default_rng(seed)
    u = lambda shape, lim: rng.uniform(-lim, lim, size=shape).astype(np.float32)
    e = (np.clip(rng.standard_normal((B, F, K)), -2, 2) / np.sqrt(K)).astype(np.float32)
    wlin = u((F * K, N), np.sqrt(6.0 / (F * K + N)))
    wprod = u((N, F), np.sqrt(6.0 / (N + F))) if method == 0 else u((N, K, K), np.sqrt(6.0 / (2 * N * K)))
    bias = u((N,), np.sqrt(3.0 / N))
    g = rng.standard_normal((B, N)).astype(np.float32)
    return e, wlin, wprod, bias, g


@pytest.mark.parametrize("name", FIXTURES)
def test_pnn_fixture_through_ops_and_layers(name):
    from recalgorithm_b200 import layers as L, ops
    z = _fixture(name)
    method = 0 if "_ipnn_" in name else 1
    e = z["e"]
    B, F, K = e.shape
    N = z["bias"].shape[0]
    out = ops.pnn_fwd(dev(e), dev(z["linear_w"]), dev(z["product_w"]), dev(z["bias"]), method)
    assert_close(out, z["out_f64"], TOL, f"{name} vs reference (float64)")
    assert_close(out, z["out_f32"], TOL, f"{name} vs reference (float32)")
    store = L.set_default_store(L.VariableStore(device="cuda", seed=0))
    wname = "product_part/inner_product_w" if method == 0 else "product_part/outer_product_w"
    L.pnn_product_layer(dev(e).reshape(B, F * K), F, K, N, product_method="IPNN" if method == 0 else "OPNN")
    store.assign({"linear_part/linear_w": z["linear_w"], wname: z["product_w"], "bias": z["bias"]})
    out2 = L.pnn_product_layer(dev(e).reshape(B, F * K), F, K, N, product_method="IPNN" if method == 0 else "OPNN")
    assert torch.equal(out2, out)
    assert sorted(store.vars) == sorted(["linear_part/linear_w", wname, "bias"])


# (B, F, K, N): the reference default, ragged B and N, F = 1, K = 1, a mid shape, and shapes on the CUDA-core path
# (F*K + Q + 1 > 128, or N % 4 != 0)
SHAPES = [(1024, 8, 8, 1024), (1000, 8, 8, 1000), (333, 1, 16, 200), (129, 20, 1, 128), (257, 6, 16, 256), (64, 40, 32, 256),
          (50, 8, 8, 30)]


@pytest.mark.parametrize("method", [0, 1])
@pytest.mark.parametrize("B,F,K,N", SHAPES)
def test_pnn_fwd_bwd_against_float64(B, F, K, N, method):
    from recalgorithm_b200 import ops
    e, wlin, wprod, bias, g = _inputs(B, F, K, N, method, seed=B + 7 * F + 13 * K + N + method)
    d = lambda a: a.astype(np.float64)
    out = ops.pnn_fwd(dev(e), dev(wlin), dev(wprod), dev(bias), method)
    ref = ref_fwd(d(e), d(wlin), d(wprod), d(bias), method)
    assert_close(out, ref, TOL, "forward")
    d_e, d_wlin, d_wprod, d_bias = ops.pnn_bwd(dev(e), dev(wlin), dev(wprod), out, dev(g), method)
    # the mask is the kernel's own forward output: elements with |pre-activation| ~ 1e-7 could fall on either side of 0 in
    # the float64 reference, so the reference gradient is taken with the kernel's mask
    mask = out.cpu().numpy() > 0
    ge = np.where(mask, d(g), 0.0)
    r_e, r_wlin, r_wprod, r_bias = ref_bwd(d(e), d(wlin), d(wprod), d(bias) + 1e6 * (2 * mask - 1), method, ge)
    assert_close(d_e, r_e, TOL, "d_e")
    assert_close(d_wlin, r_wlin, TOL, "d_linear_w")
    assert_close(d_wprod, r_wprod, TOL, "d_product_w")
    assert_close(d_bias, r_bias, TOL, "d_bias")
    if method == 1:
        low = np.tril(np.ones((K, K), bool), -1)
        assert np.all(d_wprod.cpu().numpy()[:, low] == 0), "OPNN: the strictly lower triangle gets exactly zero"
    again = ops.pnn_fwd(dev(e), dev(wlin), dev(wprod), dev(bias), method)
    assert torch.equal(again, out), "deterministic"


def _torch_ref(e, wlin, wprod, bias, method, g, mask, chunk=4096):
    """float64 direct form on the GPU, chunked over the batch: (out, d_wlin, d_wprod, d_bias); the relu mask is given."""
    B, F, K = e.shape
    e, wlin, wprod, bias, g = (t.double() for t in (e, wlin, wprod, bias, g))
    if method == 1:
        up = torch.triu(wprod)
        wsym = up + up.transpose(1, 2) - torch.diag_embed(torch.diagonal(wprod, dim1=1, dim2=2))
    outs, d_wlin, d_wprod, d_bias = [], torch.zeros_like(wlin), torch.zeros_like(wprod), torch.zeros_like(bias)
    for b0 in range(0, B, chunk):
        x = e[b0:b0 + chunk]
        lz = x.reshape(x.shape[0], -1) @ wlin
        if method == 0:
            delta = torch.einsum("bfk,nf->bnk", x, wprod)
            lp = (delta * delta).sum(-1)
        else:
            s = x.sum(1)
            p = s[:, :, None] * s[:, None, :]
            lp = torch.einsum("bkl,nkl->bn", p, wsym)
        out = torch.relu(lz + lp + bias)
        G = g[b0:b0 + chunk] * mask[b0:b0 + chunk]
        outs.append(out)
        d_wlin += x.reshape(x.shape[0], -1).t() @ G
        d_bias += G.sum(0)
        if method == 0:
            d_wprod += torch.einsum("bnk,bfk->nf", 2 * G[:, :, None] * delta, x)
        else:
            dsym = torch.einsum("bn,bkl->nkl", G, p)
            d_wprod += torch.triu(dsym) + torch.triu(dsym.transpose(1, 2)) - torch.diag_embed(torch.diagonal(dsym, dim1=1, dim2=2))
    return torch.cat(outs), d_wlin, d_wprod, d_bias


@pytest.mark.parametrize("method", [0, 1])
def test_pnn_large_batch_weight_gradients(method):
    """B = 65 536 at the reference F, K, N: the batch-reduced weight gradients (a dW kernel with many batch slices and many
    96-MMA accumulation chains per CTA) against the float64 contraction over the whole batch."""
    from recalgorithm_b200 import ops
    B, F, K, N = 65536, 8, 8, 1024
    gen = torch.Generator(device="cuda").manual_seed(11 + method)
    e = torch.randn((B, F, K), device="cuda", generator=gen) / K ** 0.5
    wlin = (torch.rand((F * K, N), device="cuda", generator=gen) * 2 - 1) * (6.0 / (F * K + N)) ** 0.5
    wshape = (N, F) if method == 0 else (N, K, K)
    wprod = (torch.rand(wshape, device="cuda", generator=gen) * 2 - 1) * 0.1
    bias = (torch.rand((N,), device="cuda", generator=gen) * 2 - 1) * 0.05
    g = torch.randn((B, N), device="cuda", generator=gen)
    out = ops.pnn_fwd(e, wlin, wprod, bias, method)
    d_e, d_wlin, d_wprod, d_bias = ops.pnn_bwd(e, wlin, wprod, out, g, method)
    ref_out, r_wlin, r_wprod, r_bias = _torch_ref(e, wlin, wprod, bias, method, g, out > 0)
    assert_close(out, ref_out, TOL, "forward (B = 65536)")
    assert_close(d_wlin, r_wlin, TOL, "d_linear_w (B = 65536)")
    assert_close(d_wprod, r_wprod, TOL, "d_product_w (B = 65536)")
    assert_close(d_bias, r_bias, TOL, "d_bias (B = 65536)")


@pytest.mark.parametrize("method", [0, 1])
def test_pnn_dead_relu_gives_exact_zeros(method):
    from recalgorithm_b200 import ops
    B, F, K, N = 300, 8, 8, 256
    e, wlin, wprod, _, g = _inputs(B, F, K, N, method, seed=3)
    bias = np.full((N,), -1e3, np.float32)
    out = ops.pnn_fwd(dev(e), dev(wlin), dev(wprod), dev(bias), method)
    assert torch.count_nonzero(out) == 0
    grads = ops.pnn_bwd(dev(e), dev(wlin), dev(wprod), out, dev(g), method)
    for t in grads:
        assert torch.count_nonzero(t) == 0


def test_pnn_refuses_cpu_tensors():
    from recalgorithm_b200 import ops
    e, wlin, wprod, bias, _ = (torch.from_numpy(a) for a in _inputs(4, 3, 2, 8, 0, seed=0))
    with pytest.raises(RuntimeError):
        ops.pnn_fwd(e, wlin, wprod, bias, 0)


@pytest.mark.parametrize("method", ["IPNN", "OPNN"])
def test_pnn_logit_body(method):
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import model_bodies as M
    from recalgorithm_b200 import autograd, layers as L
    F, K, B, rows = 8, 8, 128, 50
    store = L.set_default_store(L.VariableStore(device="cuda", seed=1))
    gen = torch.Generator(device="cuda").manual_seed(1)
    tables = autograd.EmbeddingTables([rows] * F, K, device="cuda")
    ids = torch.randint(-1, rows, (B, F), device="cuda", generator=gen)
    y = (torch.rand((B, 1), device="cuda", generator=gen) < 0.3).float()
    fields = autograd.lookup(tables, ids).reshape(B, F * K)
    logit, reg = M.pnn_logit(fields, F, K, output_dimension=256, product_method=method, weight_regularizer=0.01)
    assert logit.shape == (B, 1) and torch.isfinite(logit).all() and float(reg) > 0
    (torch.nn.functional.binary_cross_entropy_with_logits(logit, y) + reg).backward()
    assert tables.grad_slices and any(float(s.values.abs().max()) > 0 for s in tables.grad_slices)
    wname = "product_part/inner_product_w" if method == "IPNN" else "product_part/outer_product_w"
    assert {"linear_part/linear_w", wname, "bias", "fcn/dense/kernel", "fcn/dense_2/kernel"} <= set(store.vars)
    for n, v in store.vars.items():
        assert v.grad is not None and torch.isfinite(v.grad).all(), n
