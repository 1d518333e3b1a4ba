"""GPU parity: fused lookup + FM2 (rows L, FM2 of SURVEY 8a) through the C ABI vs the oracle."""
import numpy as np
import pytest
import torch

from _util import TOL, assert_close, dev, golden, relerr, trunc_normal
from oracle import layers_np as O

pytestmark = pytest.mark.gpu


def make_case(rng, B, F, D, rows, p_oov=0.15, p_range=0.02):
    rows = np.asarray(rows, dtype=np.int64)
    off = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
    table = trunc_normal(rng, (int(off[-1]), D), 1.0 / np.sqrt(D))
    ids = np.stack([rng.integers(0, rows[f], size=B) for f in range(F)], axis=1).astype(np.int64)
    ids[rng.random((B, F)) < p_oov] = -1                      # OOV / '' -> -1
    hi = rng.random((B, F)) < p_range                         # out of range -> zero vector as well
    ids[hi] = (np.broadcast_to(rows[None, :], (B, F)) + 3)[hi]
    return table, off, ids


def oracle_lookup(table, off, ids):
    rows = np.diff(off)
    clean = np.where(ids >= rows[None, :], -1, ids)
    return O.embedding_lookup(table, clean, off)


@pytest.mark.parametrize("B,F,D", [(1, 1, 4), (7, 6, 8), (33, 30, 16), (64, 40, 32), (19, 33, 32), (5, 70, 64),
                                   (9, 3, 128), (130, 8, 4), (257, 65, 16), (20, 24, 32)])
def test_fwd_bwd_parity(B, F, D):
    from recalgorithm_b200 import ops
    rng = np.random.default_rng(B * 1000 + F * 10 + D)
    table, off, ids = make_case(rng, B, F, D, rng.integers(1, 50, size=F))
    tile, fm2 = ops.embed_fm2_fwd(dev(table), dev(off), dev(ids))
    e = oracle_lookup(table, off, ids)
    assert np.array_equal(tile.cpu().numpy(), e), "gathered rows must be bit-exact copies"
    assert_close(fm2, O.fm2_fwd(e.astype(np.float64)), TOL, "fm2")
    # forward variants: lookup only / fm2 only
    t2, none = ops.embed_fm2_fwd(dev(table), dev(off), dev(ids), want_fm2=False)
    assert none is None and torch.equal(t2, tile)
    none, f2 = ops.embed_fm2_fwd(dev(table), dev(off), dev(ids), want_tile=False)
    assert none is None and torch.equal(f2, fm2)
    # backward
    d_tile = trunc_normal(rng, (B, F, D), 0.5)
    g = trunc_normal(rng, (B,), 1.0)
    want = d_tile.astype(np.float64) + O.fm2_bwd(e.astype(np.float64), g.astype(np.float64))
    assert_close(ops.embed_fm2_bwd(tile, dev(d_tile), dev(g)), want, TOL, "row_grads")
    assert_close(ops.embed_fm2_bwd(tile, None, dev(g)), O.fm2_bwd(e.astype(np.float64), g.astype(np.float64)), TOL, "fm2-only grads")
    assert torch.equal(ops.embed_fm2_bwd(tile, dev(d_tile), None), dev(d_tile))
    d_bi = trunc_normal(rng, (B, D), 1.0)
    e64 = e.astype(np.float64)
    want_bi = d_tile.astype(np.float64) + d_bi.astype(np.float64)[:, None, :] * (e64.sum(1, keepdims=True) - e64)
    assert_close(ops.embed_bi_bwd(tile, dev(d_tile), dev(d_bi)), want_bi, TOL, "bi row_grads")
    # IndexedSlices densified (duplicates summed, invalid ids dropped)
    rg = ops.embed_fm2_bwd(tile, dev(d_tile), dev(g))
    dense = torch.zeros_like(dev(table))
    ops.embed_scatter_add(dense, dev(off), dev(ids), rg)
    rows = np.diff(off)
    clean = np.where(ids >= rows[None, :], -1, ids)
    assert_close(dense, O.embedding_lookup_bwd_dense(table.shape[0], clean, off, rg.cpu().numpy()), TOL, "dense grad")


@pytest.mark.parametrize("name", ["fm2_F6_D8", "fm2_F40_D32"])
def test_fm2_golden(name):
    """FM2 fixtures: feed the embeddings through an identity lookup (table = e, ids = arange)."""
    from recalgorithm_b200 import ops
    g = golden(name)
    e = g["e"]
    B, F, D = e.shape
    table = np.ascontiguousarray(e.transpose(1, 0, 2).reshape(F * B, D))       # field f owns rows f*B..f*B+B
    off = (np.arange(F + 1) * B).astype(np.int64)
    ids = np.tile(np.arange(B, dtype=np.int64)[:, None], (1, F))
    tile, fm2 = ops.embed_fm2_fwd(dev(table), dev(off), dev(ids))
    assert np.array_equal(tile.cpu().numpy(), e)
    assert_close(fm2, g["out_f64"], TOL, "fm2 vs float64 reference")
    assert_close(fm2, g["out_f32"], TOL, "fm2 vs float32 reference")
    assert_close(fm2, g["pairwise_f64"], TOL, "fm2 vs pairwise identity")


def test_lookup_golden_edges():
    from recalgorithm_b200 import ops
    g = golden("lookup_edge")
    table = np.ascontiguousarray(g["table"])
    off = np.concatenate([g["field_row_offset"], [table.shape[0]]]).astype(np.int64)     # fixture stores the F starts
    tile, _ = ops.embed_fm2_fwd(dev(table), dev(off), dev(g["ids"]), want_fm2=False)
    assert np.array_equal(tile.cpu().numpy(), g["out"])
    out = ops.bag_lookup_fwd(dev(table), dev(g["bag_ids"]), dev(g["bag_offsets"]))
    assert np.array_equal(out.cpu().numpy(), g["bag_out"]), "mean combiner must match bit for bit (same op order)"


@pytest.mark.parametrize("D", [2, 4, 16, 33, 100, 256])
def test_bag_lookup(D):
    from recalgorithm_b200 import ops
    rng = np.random.default_rng(D)
    V, B = 57, 41
    table = trunc_normal(rng, (V, D), 1.0)
    lens = rng.integers(0, 6, size=B)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ids = rng.integers(-1, V + 2, size=int(offsets[-1])).astype(np.int64)      # includes -1 and >= V
    clean = np.where(ids >= V, -1, ids)
    want = O.bag_lookup_mean(table, clean, offsets)
    buf = torch.full((B, D + 5), 7.0, device="cuda")
    ops.bag_lookup_fwd(dev(table), dev(ids), dev(offsets), out=buf, out_col=3)
    assert np.array_equal(buf[:, 3:3 + D].cpu().numpy(), want)
    assert torch.all(buf[:, :3] == 7.0) and torch.all(buf[:, 3 + D:] == 7.0)
    # backward vs autograd of the same mean in torch (float64, CPU)
    d_out = trunc_normal(rng, (B, D + 5), 1.0)
    rg = ops.bag_lookup_bwd(dev(d_out), 3, V, D, dev(ids), dev(offsets)).cpu().numpy()
    for b in range(B):
        sl = slice(offsets[b], offsets[b + 1])
        valid = clean[sl] >= 0
        n = valid.sum()
        exp = np.where(valid[:, None], d_out[b, 3:3 + D][None, :] / max(n, 1), 0).astype(np.float32)
        assert np.allclose(rg[sl], exp, rtol=1e-6, atol=0)


def test_argument_errors():
    from recalgorithm_b200 import _lib, ops
    t = torch.zeros((4, 6), device="cuda")
    off = torch.tensor([0, 4], device="cuda")
    ids = torch.zeros((2, 1), dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):                      # D = 6 is not a 128-bit power-of-two width
        ops.embed_fm2_fwd(t, off, ids)
    with pytest.raises(RuntimeError):                    # CPU tensors are refused: no CPU path
        ops.embed_fm2_fwd(t.cpu(), off.cpu(), ids.cpu())
    assert _lib.kernel_launches() >= 0


def test_full_size_properties():
    """BASELINE config 5 shape (B=65536, F=40, D=32, 100 M rows) -- size-independent properties."""
    from recalgorithm_b200 import ops
    B, F, D, rows = 65536, 40, 32, 2_500_000
    gen = torch.Generator(device="cuda").manual_seed(1234)
    table = torch.empty((rows * F, D), device="cuda")
    table.normal_(0, D ** -0.5, generator=gen)
    off = (torch.arange(F + 1, device="cuda") * rows)
    ids = torch.randint(0, rows, (B, F), device="cuda", generator=gen)
    ids[torch.rand((B, F), device="cuda", generator=gen) < 0.05] = -1
    tile, fm2 = ops.embed_fm2_fwd(table, off, ids)
    # (1) gather is an exact copy (checked against torch indexing on a 1/16 sample of the batch)
    sub = slice(0, B, 16)
    gidx = (ids[sub] + off[:-1][None, :]).clamp_min(0)
    want = table[gidx.reshape(-1)].reshape(-1, F, D) * (ids[sub] >= 0)[..., None]
    assert torch.equal(tile[sub], want)
    # (2) fm2 vs float64 evaluation of the pairwise-equivalent closed form
    e64 = tile.double()
    ref = 0.5 * (e64.sum(1).pow(2) - e64.pow(2).sum(1)).sum(1, keepdim=True)
    assert_close(fm2, ref, TOL, "fm2 @ full size")
    # (3) backward: linearity in (d_tile, d_fm2) and the sum-over-fields identity
    d_tile = torch.randn((B, F, D), device="cuda", generator=gen)
    g = torch.randn((B,), device="cuda", generator=gen)
    r1 = ops.embed_fm2_bwd(tile, d_tile, g)
    r2 = ops.embed_fm2_bwd(tile, None, g)
    assert_close(r1 - r2, d_tile, 1e-5, "bwd linearity")
    # sum_f g*(S - e_f) = g*(F-1)*S
    S = e64.sum(1)
    assert_close(r2.double().sum(1), g.double()[:, None] * (F - 1) * S, TOL, "bwd field-sum identity")
    # (4) idempotence / determinism
    tile2, fm2b = ops.embed_fm2_fwd(table, off, ids)
    assert torch.equal(tile, tile2) and torch.equal(fm2, fm2b)


@pytest.mark.parametrize("B,F,D", [(7, 6, 8), (64, 40, 32), (19, 33, 32), (130, 8, 4), (257, 65, 16), (9, 3, 128),
                                   (50, 24, 32), (8192, 40, 32)])
def test_int32_ids_and_fused_linear_head(B, F, D):
    """int32 ids (half the PCIe bytes) give the identical tile and a widened int64 copy; the fused dense(1) head equals the
    unfused chain tile.reshape(B, F*D) @ w and its backward equals ctr_embed_fm2_bwd fed with the rank-1 d_tile."""
    from recalgorithm_b200 import autograd, ops
    rng = np.random.default_rng(7 * B + F + D)
    table, off, ids = make_case(rng, B, F, D, rng.integers(1, 50, size=F))
    tile, fm2 = ops.embed_fm2_fwd(dev(table), dev(off), dev(ids))
    ids64 = torch.empty((B, F), dtype=torch.int64, device="cuda")
    t32, f32 = ops.embed_fm2_fwd(dev(table), dev(off), dev(ids).int(), ids64_out=ids64)
    assert torch.equal(t32, tile) and torch.equal(f32, fm2) and torch.equal(ids64, dev(ids))
    w = trunc_normal(rng, (F * D, 1), 0.3)
    for id_t in (dev(ids), dev(ids).int()):
        tl, fl, lin = ops.embed_fm2_lin_fwd(dev(table), dev(off), id_t, dev(w))
        assert torch.equal(tl, tile) and torch.equal(fl, fm2)
        e64 = tile.double().cpu().numpy().reshape(B, F * D)
        assert_close(lin, e64 @ w.astype(np.float64), TOL, "fused dense(1) head")
    g = trunc_normal(rng, (B,), 1.0)
    gl = trunc_normal(rng, (B,), 1.0)
    rg, dw = ops.embed_fm2_lin_bwd(tile, dev(w), dev(g), dev(gl))
    d_tile = (gl.astype(np.float64)[:, None] * w.astype(np.float64).reshape(1, F * D)).reshape(B, F, D)
    e = tile.double().cpu().numpy()
    assert_close(rg, d_tile + O.fm2_bwd(e, g.astype(np.float64)), TOL, "row_grads (rank-1 d_tile)")
    assert_close(dw, (gl.astype(np.float64)[:, None] * e.reshape(B, F * D)).sum(0), TOL, "d_wlin")
    # autograd wrapper: same numbers as the unfused public API with a torch matmul head
    tables = autograd.EmbeddingTables(np.diff(off).tolist(), D, device="cuda", init=None)
    tables.weight.copy_(dev(table))
    w_a = dev(w).clone().requires_grad_()
    f_a, l_a = autograd.lookup_fm2_linear(tables, dev(ids).int(), w_a)
    ((f_a.reshape(-1) * dev(g)).sum() + (l_a.reshape(-1) * dev(gl)).sum()).backward()
    assert torch.equal(tables.grad_slices[0].values, rg) and torch.equal(tables.grad_slices[0].ids, dev(ids))
    assert_close(w_a.grad.reshape(-1), dw, TOL, "autograd d_wlin")


@pytest.mark.parametrize("B,T,D", [(1, 1, 4), (33, 50, 16), (257, 7, 8), (64, 70, 32), (5, 3, 128)])
def test_sequence_lookup(B, T, D):
    """ctr_embed_seq_fwd: a (B,T) id matrix over ONE table == the F = 1 lookup of every id, zero rows for -1 / out of range."""
    from recalgorithm_b200 import ops
    rng = np.random.default_rng(B + T + D)
    V = 91
    table = trunc_normal(rng, (V + 10, D), 0.5)
    ids = rng.integers(-1, V + 2, size=(B, T)).astype(np.int64)
    rr = torch.tensor([5, 5 + V], device="cuda")
    out = ops.embed_seq_fwd(dev(table), dev(ids), rr)
    valid = (ids >= 0) & (ids < V)
    want = table[5 + np.clip(ids, 0, V - 1)] * valid[..., None]
    assert np.array_equal(out.cpu().numpy(), want), "sequence lookup must copy rows bit-exactly"
    off = torch.tensor([5, 5 + V], device="cuda")
    flat, _ = ops.embed_fm2_fwd(dev(table), off, dev(ids.reshape(-1, 1)), want_fm2=False)
    assert torch.equal(flat.reshape(B, T, D), out)
