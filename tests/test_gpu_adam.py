"""GPU: Adam on IndexedSlices table gradients (SURVEY 8f.3) -- reference-faithful dense variant and LazyAdam -- vs oracle."""
import numpy as np
import pytest
import torch

from _util import assert_close, dev, trunc_normal
from oracle import layers_np as O

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("lazy", [False, True])
@pytest.mark.parametrize("D", [4, 16, 32])
def test_table_adam_matches_oracle(lazy, D):
    from recalgorithm_b200 import autograd, optim
    rng = np.random.default_rng(D + int(lazy))
    F, B, rows = 5, 64, 37
    tables = autograd.EmbeddingTables([rows] * F, D, device="cuda")
    opt = optim.TableAdam(tables, lr=0.01, lazy=lazy)
    var = tables.weight.cpu().double().numpy()
    m = np.zeros_like(var); v = np.zeros_like(var)
    off = tables.field_row_offset.cpu().numpy()
    for t in range(1, 5):
        ids = rng.integers(-1, rows + 1, size=(B, F)).astype(np.int64)        # duplicates, OOV and out-of-range ids
        d_tile = trunc_normal(rng, (B, F, D), 1.0); g = trunc_normal(rng, (B,), 1.0)
        tile, fm2 = autograd.lookup_fm2(tables, dev(ids))
        (tile * dev(d_tile)).sum().add((fm2[:, 0] * dev(g)).sum()).backward()
        sl = tables.grad_slices[0]
        valid = (ids >= 0) & (ids < rows)
        grows = (ids + off[:-1][None, :])[valid]
        gvals = sl.values.cpu().double().numpy()[valid]
        opt.step()
        assert opt.last_unique_rows() == len(np.unique(grows)) and not tables.grad_slices
        assert bool((opt._slot == -1).all()), "slot table must be idle (-1) between steps"
        var, m, v = O.adam_sparse_apply(var, m, v, grows, gvals, t, 0.01, lazy=lazy)
        assert_close(tables.weight, var, 2e-6, f"var step {t}")
        assert_close(opt.m, m, 1e-5, f"m step {t}"); assert_close(opt.v, v, 1e-5, f"v step {t}")
    if not lazy:      # a step without any gradient still moves every row (dense semantics)
        before = tables.weight.clone()
        opt.step()
        assert not torch.equal(before, tables.weight)


@pytest.mark.parametrize("lazy", [False, True])
def test_table_adam_heavy_duplicates_and_two_backward_passes(lazy):
    """3 rows per field shared by 512 samples (every row has ~170 duplicates) and two backward passes before one step:
    TF sums every IndexedSlices entry of a row before the moment update."""
    from recalgorithm_b200 import autograd, optim
    rng = np.random.default_rng(7 + int(lazy))
    F, B, rows, D = 3, 512, 3, 8
    tables = autograd.EmbeddingTables([rows] * F, D, device="cuda")
    opt = optim.TableAdam(tables, lr=0.05, lazy=lazy)
    var = tables.weight.cpu().double().numpy(); m = np.zeros_like(var); v = np.zeros_like(var)
    off = tables.field_row_offset.cpu().numpy()
    for t in range(1, 4):
        grows, gvals = [], []
        for _ in range(2):
            ids = rng.integers(0, rows, size=(B, F)).astype(np.int64)
            d_tile = trunc_normal(rng, (B, F, D), 1.0)
            tile, _ = autograd.lookup_fm2(tables, dev(ids))
            (tile * dev(d_tile)).sum().backward()
            grows.append((ids + off[:-1][None, :]).reshape(-1)); gvals.append(d_tile.reshape(-1, D).astype(np.float64))
        opt.step()
        assert opt.last_unique_rows() == rows * F
        var, m, v = O.adam_sparse_apply(var, m, v, np.concatenate(grows), np.concatenate(gvals), t, 0.05, lazy=lazy)
        assert_close(tables.weight, var, 2e-6, f"var step {t}")
        assert_close(opt.m, m, 1e-5, f"m step {t}"); assert_close(opt.v, v, 1e-5, f"v step {t}")


def test_full_size_adam_properties():
    """BASELINE config 5 shape (B=65536, F=40, D=32, 100 M rows; 38 GB with m and v), ids with heavy duplication in one
    field -- size-independent properties of the fused IndexedSlices step."""
    from recalgorithm_b200 import autograd, optim
    B, F, D, rows = 65536, 40, 32, 2_500_000
    gen = torch.Generator(device="cuda").manual_seed(99)
    tables = autograd.EmbeddingTables([rows] * F, D, device="cuda", init=None)
    tables.weight.normal_(0, D ** -0.5, generator=gen)
    ids = torch.randint(0, rows, (B, F), device="cuda", generator=gen)
    ids[:, 0] = torch.randint(0, 50, (B,), device="cuda", generator=gen)            # ~1300 duplicates per row in field 0
    ids[torch.rand((B, F), device="cuda", generator=gen) < 0.03] = -1
    vals = torch.randn((B, F, D), device="cuda", generator=gen)
    flat = (ids + tables.field_row_offset[:-1][None, :])[ids >= 0]
    uniq = torch.unique(flat)
    opt = optim.TableAdam(tables, lr=0.01, lazy=True)
    w0 = tables.weight[uniq].clone()
    probe = torch.randint(0, rows * F, (1 << 20,), device="cuda", generator=gen)      # random rows, mostly untouched
    untouched = probe[~torch.isin(probe, uniq)]
    u0 = tables.weight[untouched].clone()
    tables.grad_slices.append(autograd.IndexedSlices(vals.clone(), ids, tables.field_row_offset))
    opt.step()
    # (1) distinct rows counted exactly, scratch back to idle
    assert opt.last_unique_rows() == int(uniq.numel()) and bool((opt._slot == -1).all())
    # (2) untouched rows are bit-identical under LazyAdam, moments stay zero
    assert torch.equal(tables.weight[untouched], u0) and float(opt.m[untouched].abs().max()) == 0.0
    # (3) first step from zero state: m = (1-b1) g, v = (1-b2) g^2 with g the SUM over duplicates  =>  |dw| = lr * |g| / (|g| + eps')
    g = torch.zeros((uniq.numel(), D), device="cuda", dtype=torch.float64)
    g.index_add_(0, torch.searchsorted(uniq, flat), vals[ids >= 0].double())
    # rows of field 0 sum ~1300 duplicates through fp32 atomics: |sum| ~ 36 against sum|terms| ~ 1000, so the per-element
    # criterion (relative to |result|) does not apply to them; max-norm over the 2.5 M rows does
    assert_close(opt.m[uniq], (1.0 - float(np.float32(0.9))) * g, 1e-5, "m = (1-b1) * summed gradient", elementwise=False)
    dw = (tables.weight[uniq] - w0).double()
    assert float((dw.abs() - _half_ulp(w0)).max()) <= 0.01 * (1 + 1e-5)
    big = g.abs() > 1e-2
    assert_close(dw[big], -0.01 * torch.sign(g[big]), 1e-4, "first Adam step is -lr * sign(g) where |g| >> eps")



def _half_ulp(w):
    """Half a float32 ulp of each updated weight: storing w - lr*m/(sqrt(v)+eps) in float32 rounds by up to this much, so a
    step of exactly lr can read back that much larger (1.2e-5 lr at |w| ~ 1)."""
    w = w.float().abs()
    return (torch.nextafter(w, torch.full_like(w, float("inf"))) - w).double() / 2

@pytest.mark.parametrize("lazy", [False, True])
@pytest.mark.parametrize("B,F,D,rows", [(64, 5, 16, 37), (512, 3, 8, 3), (300, 40, 32, 1000), (129, 33, 4, 11), (40, 12, 128, 50)])
def test_backward_fused_with_adam_equals_unfused(lazy, B, F, D, rows):
    """ctr_embed_fm2_bwd_adam (backward + row update in one pass, duplicates finished through the parked list) against
    ctr_embed_fm2_bwd + ctr_adam_indexed_slices and the float64 oracle, three steps, duplicates / OOV / out-of-range ids."""
    from recalgorithm_b200 import autograd, optim
    rng = np.random.default_rng(B + F + D + int(lazy))
    tf = autograd.EmbeddingTables([rows] * F, D, device="cuda")
    tu = autograd.EmbeddingTables([rows] * F, D, device="cuda", init=None)
    tu.weight.copy_(tf.weight)
    of = optim.TableAdam(tf, lr=0.01, lazy=lazy, fused_backward=True)
    ou = optim.TableAdam(tu, lr=0.01, lazy=lazy)
    var = tf.weight.cpu().double().numpy(); m = np.zeros_like(var); v = np.zeros_like(var)
    off = tf.field_row_offset.cpu().numpy()
    for t in range(1, 4):
        ids = rng.integers(-1, rows + 1, size=(B, F)).astype(np.int64)
        d_tile = trunc_normal(rng, (B, F, D), 1.0); g = trunc_normal(rng, (B,), 1.0)
        for tb in (tf, tu):
            tile, fm2 = autograd.lookup_fm2(tb, dev(ids))
            (tile * dev(d_tile)).sum().add((fm2[:, 0] * dev(g)).sum()).backward()
        assert not tf.grad_slices, "the fused backward must not materialise IndexedSlices"
        valid = (ids >= 0) & (ids < rows)
        grows = (ids + off[:-1][None, :])[valid]
        gvals = tu.grad_slices[0].values.cpu().double().numpy()[valid]
        of.step(); ou.step()
        assert of.last_unique_rows() == ou.last_unique_rows() == len(np.unique(grows))
        assert bool((of._slot == -1).all()), "slot table must be idle (-1) between steps"
        var, m, v = O.adam_sparse_apply(var, m, v, grows, gvals, t, 0.01, lazy=lazy)
        assert_close(tf.weight, var, 2e-6, f"fused var step {t}")
        assert_close(of.m, m, 1e-5, f"fused m step {t}"); assert_close(of.v, v, 1e-5, f"fused v step {t}")
        assert_close(tf.weight, tu.weight.double(), 2e-6, f"fused vs unfused var step {t}")


def test_backward_fused_with_adam_full_size():
    """Config-5 shape with ~1300 duplicates per row in one field: same first-step properties as the unfused test."""
    from recalgorithm_b200 import autograd, optim, ops
    B, F, D, rows = 65536, 40, 32, 2_500_000
    gen = torch.Generator(device="cuda").manual_seed(199)
    tables = autograd.EmbeddingTables([rows] * F, D, device="cuda", init=None)
    tables.weight.normal_(0, D ** -0.5, generator=gen)
    ids = torch.randint(0, rows, (B, F), device="cuda", generator=gen)
    ids[:, 0] = torch.randint(0, 50, (B,), device="cuda", generator=gen)
    ids[torch.rand((B, F), device="cuda", generator=gen) < 0.03] = -1
    d_tile = torch.randn((B, F, D), device="cuda", generator=gen)
    d_fm2 = torch.randn((B,), device="cuda", generator=gen)
    tile, _ = ops.embed_fm2_fwd(tables.weight, tables.field_row_offset, ids)
    vals = ops.embed_fm2_bwd(tile, d_tile, d_fm2)
    flat = (ids + tables.field_row_offset[:-1][None, :])[ids >= 0]
    uniq = torch.unique(flat)
    opt = optim.TableAdam(tables, lr=0.01, lazy=True, fused_backward=True)
    w0 = tables.weight[uniq].clone()
    probe = torch.randint(0, rows * F, (1 << 20,), device="cuda", generator=gen)
    untouched = probe[~torch.isin(probe, uniq)]
    u0 = tables.weight[untouched].clone()
    opt.apply_fused(tile, d_tile, d_fm2, ids)
    opt.step()
    assert opt.last_unique_rows() == int(uniq.numel()) and bool((opt._slot == -1).all())
    assert torch.equal(tables.weight[untouched], u0) and float(opt.m[untouched].abs().max()) == 0.0
    g = torch.zeros((uniq.numel(), D), device="cuda", dtype=torch.float64)
    g.index_add_(0, torch.searchsorted(uniq, flat), vals[ids >= 0].double())
    # rows of field 0 sum ~1300 duplicates through fp32 atomics: |sum| ~ 36 against sum|terms| ~ 1000, so the per-element
    # criterion (relative to |result|) does not apply to them; max-norm over the 2.5 M rows does
    assert_close(opt.m[uniq], (1.0 - float(np.float32(0.9))) * g, 1e-5, "m = (1-b1) * summed gradient", elementwise=False)
    dw = (tables.weight[uniq] - w0).double()
    assert float((dw.abs() - _half_ulp(w0)).max()) <= 0.01 * (1 + 1e-5)
