"""CPU checks of the float64 AutoInt restatement (tests/_autoint_ref.py): its analytic backward against torch.autograd,
its attention core against torch's scaled_dot_product_attention, and the identities the paper's equations imply."""
import numpy as np
import pytest
import torch

from _autoint_ref import attention_core, interacting_bwd, interacting_fwd


def _draw(rng, B, F, d, H, dk):
    x = rng.standard_normal((B, F, d))
    ws = [rng.standard_normal((d, H * dk)) / np.sqrt(d) for _ in range(4)]
    return x, ws


def _torch_layer(x, ws, H, dk):
    B, F, d = x.shape
    heads = lambda t: t.reshape(B, F, H, dk).transpose(1, 2)
    q, k, v = (heads(x @ w) for w in ws[:3])
    a = torch.softmax(q @ k.transpose(-1, -2), dim=-1)
    o = (a @ v).transpose(1, 2).reshape(B, F, H * dk)
    return torch.relu(o + x @ ws[3])


@pytest.mark.parametrize("B,F,d,H,dk", [(3, 7, 5, 3, 5), (2, 1, 4, 2, 3), (4, 10, 16, 2, 8), (2, 39, 32, 2, 32)])
def test_analytic_backward_equals_autograd(B, F, d, H, dk):
    rng = np.random.default_rng(B * 100 + F)
    x, ws = _draw(rng, B, F, d, H, dk)
    g = rng.standard_normal((B, F, H * dk))
    out, cache = interacting_fwd(x, *ws, H, dk)
    grads = interacting_bwd(cache, *ws, g, H, dk)
    xt = torch.tensor(x, requires_grad=True)
    wt = [torch.tensor(w, requires_grad=True) for w in ws]
    ot = _torch_layer(xt, wt, H, dk)
    ot.backward(torch.tensor(g))
    np.testing.assert_allclose(out, ot.detach().numpy(), rtol=1e-12, atol=1e-12)
    for mine, theirs in zip(grads, [xt.grad] + [w.grad for w in wt]):
        np.testing.assert_allclose(mine, theirs.numpy(), rtol=1e-10, atol=1e-11)


@pytest.mark.parametrize("F,dk", [(1, 4), (7, 3), (40, 32)])
def test_attention_core_equals_sdpa(F, dk):
    """An independent implementation: torch's own attention operator at scale 1 (the paper's unscaled scores)."""
    rng = np.random.default_rng(F)
    q, k, v = (rng.standard_normal((3, 2, F, dk)) for _ in range(3))
    o, _ = attention_core(q, k, v)
    ref = torch.nn.functional.scaled_dot_product_attention(torch.tensor(q), torch.tensor(k), torch.tensor(v), scale=1.0)
    assert np.abs(o - ref.numpy()).max() <= 1e-13


def test_single_field_is_value_plus_residual():
    """F = 1: the one attention weight is 1, so out = relu(x wv + x wr), and the query / key weights get exactly zero."""
    rng = np.random.default_rng(1)
    x, ws = _draw(rng, 4, 1, 6, 2, 3)
    out, cache = interacting_fwd(x, *ws, 2, 3)
    np.testing.assert_allclose(out, np.maximum(x @ ws[2] + x @ ws[3], 0), rtol=1e-13, atol=1e-14)
    grads = interacting_bwd(cache, *ws, rng.standard_normal(out.shape), 2, 3)
    assert np.all(grads[1] == 0) and np.all(grads[2] == 0)


def test_zero_query_gives_uniform_attention():
    """w_query = 0: every score is 0, the attention is 1/F, and d_w_key is exactly 0."""
    rng = np.random.default_rng(2)
    x, ws = _draw(rng, 3, 5, 4, 2, 3)
    ws[0] = np.zeros_like(ws[0])
    out, cache = interacting_fwd(x, *ws, 2, 3)
    assert np.all(cache[4] == 1.0 / 5)
    grads = interacting_bwd(cache, *ws, rng.standard_normal(out.shape), 2, 3)
    assert np.all(grads[2] == 0)


def test_field_permutation_permutes_output():
    rng = np.random.default_rng(3)
    x, ws = _draw(rng, 2, 6, 5, 2, 4)
    perm = rng.permutation(6)
    out, _ = interacting_fwd(x, *ws, 2, 4)
    outp, _ = interacting_fwd(x[:, perm], *ws, 2, 4)
    np.testing.assert_allclose(outp, out[:, perm], rtol=1e-13, atol=1e-14)
