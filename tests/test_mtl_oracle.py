"""CPU: the float64 restatement of the multi-task balancing methods (tests/_mtl_ref.py) against torch.autograd and against
the papers' vector forms."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _mtl_ref as R  # noqa: E402


def _inputs(T, B, seed):
    rng = np.random.default_rng(seed)
    x = torch.tensor(rng.normal(0, 3, (T, B)), dtype=torch.float64, requires_grad=True)
    z = torch.tensor(rng.random((T, B)), dtype=torch.float64)
    return x, z, rng


@pytest.mark.parametrize("T", [1, 3, 8])
def test_uncertainty_gradients_match_autograd(T):
    """d total / d s_t = -exp(-s_t) L_t + 1/2 and d total / d logit[t,b] = exp(-s_t) (sigmoid(x) - z) / B."""
    x, z, rng = _inputs(T, 37, T)
    s = torch.tensor(rng.normal(0, 0.7, T), dtype=torch.float64, requires_grad=True)
    tot = R.total(R.sigmoid_ce(x, z), "uncertainty", s)
    tot.backward()
    L, want_total, d, d_s = R.loss_outputs(x.detach().numpy(), z.numpy(), "uncertainty", s.detach().numpy())
    np.testing.assert_allclose(tot.item(), want_total, rtol=1e-13)
    np.testing.assert_allclose(s.grad.numpy(), d_s, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(x.grad.numpy(), np.exp(-s.detach().numpy())[:, None] * d, rtol=1e-12, atol=1e-16)


def test_gradnorm_weight_gradient_matches_autograd():
    """dL_grad / dw_t = sign(G_t - Gbar r_t^alpha) n_t with the target detached; the Gram form of the step agrees."""
    rng = np.random.default_rng(1)
    T, P, alpha = 4, 50, 1.5
    g = torch.tensor(rng.normal(0, 1, (T, P)) * rng.uniform(0.2, 3, (T, 1)), dtype=torch.float64)
    L = torch.tensor(rng.uniform(0.3, 1.0, T), dtype=torch.float64)
    L0 = torch.tensor(rng.uniform(0.5, 1.2, T), dtype=torch.float64)
    w = torch.tensor(rng.uniform(0.5, 1.5, T), dtype=torch.float64, requires_grad=True)
    loss = R.gradnorm_loss(g, L, L0, w, alpha)
    loss.backward()
    w_new, L_grad, d_w = R.gradnorm_step((g @ g.T).numpy(), L.numpy(), L0.numpy(), w.detach().numpy(), alpha, lr=0.1)
    np.testing.assert_allclose(d_w, w.grad.numpy(), rtol=1e-12)
    np.testing.assert_allclose(L_grad, loss.item(), rtol=1e-12)
    w1 = w.detach().numpy() - 0.1 * w.grad.numpy()
    np.testing.assert_allclose(w_new, T * w1 / w1.sum(), rtol=1e-12)
    assert abs(w_new.sum() - T) < 1e-12


def test_gradnorm_sign_zero_keeps_the_weights():
    """Identical tasks sit on the target: sign(0) = 0, no gradient, weights unchanged."""
    g = np.tile(np.arange(1.0, 6.0), (2, 1))
    w, L_grad, d_w = R.gradnorm_step(g @ g.T, [0.7, 0.7], [0.9, 0.9], [1.0, 1.0], 1.5, 0.5)
    assert L_grad == 0 and np.all(d_w == 0) and np.all(w == 1.0)


def _conflicting(T, P, rng):
    """Rows sharing a direction with random signs (conflicts in every draw), plus noise and per-row scales."""
    u = rng.normal(0, 1, P)
    return (rng.choice([-1.0, 1.0], (T, 1)) * rng.uniform(0.5, 2, (T, 1)) * u + rng.normal(0, 0.7, (T, P)))


@pytest.mark.parametrize("seed", range(24))
def test_pcgrad_coefficient_form_equals_vector_form(seed):
    rng = np.random.default_rng(100 + seed)
    T = int(rng.integers(1, 9))
    g = _conflicting(T, int(rng.integers(1, 300)), rng)
    order = rng.permutation(T)
    want, _ = R.pcgrad_vector(g, order)
    c = R.pcgrad_coef(g @ g.T, order)
    got = c @ g
    assert np.abs(got - want).max() <= 1e-12 * max(np.abs(want).max(), np.abs(g).max())


def test_pcgrad_two_conflicting_tasks_become_orthogonal():
    rng = np.random.default_rng(7)
    g = np.stack([rng.normal(0, 1, 40), rng.normal(0, 1, 40)])
    g[1] -= 2 * (g[0] @ g[1] + 5) / (g[0] @ g[0]) * g[0]             # force g_1 . g_2 < 0
    assert g[0] @ g[1] < 0
    out, (g1, g2) = R.pcgrad_vector(g, [0, 1])
    assert abs(g1 @ g[1]) <= 1e-12 * np.abs(g).max() ** 2 * 40
    assert abs(g2 @ g[0]) <= 1e-12 * np.abs(g).max() ** 2 * 40
    np.testing.assert_allclose(R.pcgrad_coef(g @ g.T, [0, 1]) @ g, out, rtol=0, atol=1e-12)


def test_pcgrad_without_conflict_is_the_plain_sum():
    rng = np.random.default_rng(8)
    g = np.abs(rng.normal(0, 1, (5, 30)))                            # all dot products positive
    for order in ([0, 1, 2, 3, 4], [4, 2, 0, 3, 1]):
        out, _ = R.pcgrad_vector(g, order)
        np.testing.assert_array_equal(out, g.sum(axis=0))
        np.testing.assert_array_equal(R.pcgrad_coef(g @ g.T, order), np.ones(5))


def test_pcgrad_antiparallel_pair_gives_zero_and_zero_rows_give_no_nan():
    g = np.stack([np.linspace(-1, 2, 17), -2 * np.linspace(-1, 2, 17)])
    out, _ = R.pcgrad_vector(g, [1, 0])
    c = R.pcgrad_coef(g @ g.T, [1, 0])
    assert np.all(out == 0) and np.all(c @ g == 0)
    z = np.stack([np.zeros(9), np.arange(9.0), -np.arange(9.0) + 1])
    for order in ([0, 1, 2], [2, 0, 1]):
        out, _ = R.pcgrad_vector(z, order)
        c = R.pcgrad_coef(z @ z.T, order)
        assert np.all(np.isfinite(out)) and np.all(np.isfinite(c))
        np.testing.assert_allclose(c @ z, out, rtol=0, atol=1e-12)
