"""CPU checks of the float64 FwBI restatement (tests/_flen_ref.py): its analytic backward against torch.autograd, its forward
against explicit loops over the field pairs, the NFM and FwFM fixtures through the two degenerate groupings, and the
identities of the definition."""
import itertools

import numpy as np
import pytest
import torch

from _flen_ref import fwbi_bwd, fwbi_fwd, pairs
from _util import golden


def _draw(rng, B, F, D, M):
    e = rng.standard_normal((B, F, D))
    group = list(rng.integers(0, M, F))
    kmf = rng.standard_normal(M * (M - 1) // 2)
    kfm = rng.standard_normal(M)
    bmf, bfm = rng.standard_normal(D), rng.standard_normal(D)
    return e, group, kmf, kfm, bmf, bfm


def _torch_fwbi(e, group, M, kmf, kfm, bmf, bfm):
    oh = torch.zeros(len(group), M, dtype=e.dtype)
    oh[torch.arange(len(group)), torch.tensor(group)] = 1.0
    p = torch.einsum("bfd,fm->bmd", e, oh)
    q = torch.einsum("bfd,fm->bmd", e * e, oh)
    h = bmf + bfm + torch.einsum("m,bmd->bd", kfm, p * p - q)
    for k, (i, j) in enumerate(pairs(M)):
        h = h + kmf[k] * p[:, i] * p[:, j]
    return h


@pytest.mark.parametrize("B,F,D,M", [(3, 7, 4, 3), (2, 1, 8, 1), (4, 12, 5, 8), (2, 40, 32, 3), (3, 9, 4, 2)])
def test_analytic_backward_equals_autograd(B, F, D, M):
    rng = np.random.default_rng(B * 100 + F + M)
    e, group, kmf, kfm, bmf, bfm = _draw(rng, B, F, D, M)
    g, dt = rng.standard_normal((B, D)), rng.standard_normal((B, F, D))
    ts = [torch.tensor(x, requires_grad=True) for x in (e, kmf, kfm, bmf, bfm)]
    h = _torch_fwbi(ts[0], group, M, *ts[1:])
    (h * torch.tensor(g)).sum().add((ts[0] * torch.tensor(dt)).sum()).backward()
    np.testing.assert_allclose(fwbi_fwd(e, group, M, kmf, kfm, bmf, bfm), h.detach().numpy(), rtol=1e-12, atol=1e-12)
    for mine, t in zip(fwbi_bwd(e, group, M, kmf, kfm, g, dt), ts):
        theirs = t.grad.numpy() if t.grad is not None else np.zeros(t.shape)   # M = 1: kernel_mf is empty
        np.testing.assert_allclose(mine, theirs, rtol=1e-11, atol=1e-11)


def _brute(e, group, M, kmf, kfm, bmf, bfm):
    """Explicit loops: inter-group products of every field pair in different groups, intra-group products of every field
    pair inside one group (p_m^2 - q_m = 2 sum_{i<j in m} e_i e_j)."""
    B, F, D = e.shape
    h = np.tile(np.asarray(bmf) + np.asarray(bfm), (B, 1)).astype(np.float64)
    pidx = {pr: k for k, pr in enumerate(pairs(M))}
    for fi, fj in itertools.combinations(range(F), 2):
        gi, gj = group[fi], group[fj]
        w = 2.0 * kfm[gi] if gi == gj else kmf[pidx[(min(gi, gj), max(gi, gj))]]
        h += w * e[:, fi] * e[:, fj]
    return h


@pytest.mark.parametrize("B,F,D,M", [(3, 7, 4, 3), (2, 13, 8, 8), (4, 5, 4, 1), (2, 30, 16, 4)])
def test_forward_equals_brute_force_pair_loops(B, F, D, M):
    rng = np.random.default_rng(7 * F + M)
    e, group, kmf, kfm, bmf, bfm = _draw(rng, B, F, D, M)
    ref = _brute(e, group, M, kmf, kfm, bmf, bfm)
    got = fwbi_fwd(e, group, M, kmf, kfm, bmf, bfm)
    assert np.abs(got - ref).max() <= 1e-13 * np.abs(ref).max()


@pytest.mark.parametrize("name", ["nfm_bi_F6_D8", "nfm_bi_F40_D32"])
def test_one_group_is_nfm_bi_interaction(name):
    z = golden(name)
    e = z["e"].astype(np.float64)
    F, D = e.shape[1:]
    h = fwbi_fwd(e, [0] * F, 1, [], [0.5], np.zeros(D), np.zeros(D))
    assert np.abs(h - z["out_f64"]).max() <= 1e-13 * np.abs(z["out_f64"]).max()


@pytest.mark.parametrize("name", ["fwfm_F6_D8", "fwfm_F30_D16"])
def test_singleton_groups_are_fwfm(name):
    z = golden(name)
    e = z["e"].astype(np.float64)
    F, D = e.shape[1:]
    e2, group, kmf, kfm, bmf, bfm = _draw(np.random.default_rng(F), 1, F, D, F)
    h = fwbi_fwd(e, list(range(F)), F, z["r"].astype(np.float64), kfm, np.zeros(D), np.zeros(D))
    assert np.abs(h.sum(-1, keepdims=True) - z["out_f64"]).max() <= 1e-13 * np.abs(z["out_f64"]).max()
    p_fm = fwbi_fwd(e, list(range(F)), F, np.zeros(F * (F - 1) // 2), kfm, np.zeros(D), np.zeros(D))
    assert np.array_equal(p_fm, np.zeros_like(p_fm))                  # h_fm of singleton groups: exactly 0


def test_invariant_under_permuting_fields_within_a_group():
    rng = np.random.default_rng(3)
    B, F, D, M = 4, 11, 8, 3
    e, group, kmf, kfm, bmf, bfm = _draw(rng, B, F, D, M)
    perm = np.arange(F)
    members = [f for f in range(F) if group[f] == group[0]]
    perm[members] = rng.permutation(members)
    h0 = fwbi_fwd(e, group, M, kmf, kfm, bmf, bfm)
    h1 = fwbi_fwd(e[:, perm], group, M, kmf, kfm, bmf, bfm)
    np.testing.assert_allclose(h1, h0, rtol=1e-12, atol=1e-12)


def test_one_group_has_no_field_pair_term():
    rng = np.random.default_rng(5)
    e, group, kmf, kfm, bmf, bfm = _draw(rng, 3, 6, 4, 1)
    h_mf = fwbi_fwd(e, [0] * 6, 1, [], [0.0], bmf, np.zeros(4))
    assert np.array_equal(h_mf, np.tile(bmf, (3, 1)))


def test_singleton_group_gives_zero_fm_gradient():
    rng = np.random.default_rng(9)
    B, F, D, M = 3, 5, 4, 3
    e, _, kmf, kfm, bmf, bfm = _draw(rng, B, F, D, M)
    group = [0, 1, 1, 2, 2]                                             # group 0 is the singleton field 0
    g = rng.standard_normal((B, D))
    rg, d_kmf, d_kfm, _, _ = fwbi_bwd(e, group, M, np.zeros_like(kmf), kfm, g)
    assert d_kfm[0] == 0.0 and np.array_equal(rg[:, 0], np.zeros((B, D)))
