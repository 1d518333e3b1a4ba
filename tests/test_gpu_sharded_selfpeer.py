"""GPU (ONE device is enough): the row-sharded kernels -- peer-pull lookup (`embed_fm2_fwd_kernel<.., SH=true>`), the queue
plan, the fused backward+push, the plain push and the owner-side Adam -- with all G "ranks" resident on cuda:0.  Every shard,
receive queue and count vector is an ordinary cuda:0 buffer, so the peer pointers the kernels dereference are local ones; the
arithmetic, slot assignment, queue layout and owner-side consumption are exactly what runs across NVLink (tests/mp_sharded_gpu.py
repeats this under torchrun when >= 2 GPUs are present)."""
import ctypes

import numpy as np
import pytest
import torch

from _util import assert_close

pytestmark = pytest.mark.gpu


def _ptrs(ts):
    return (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


class LocalShardGroup:
    """G ranks' worth of shards and receive queues on one device (test harness; mirrors sharded.ShardedEmbeddingTables)."""

    def __init__(self, rows_per_field, D, G, batch, slack=3.0, seed=0):
        from recalgorithm_b200 import sharded as S
        self.S, self.G, self.D = S, G, D
        dev = torch.device("cuda", 0)
        rows = torch.as_tensor(rows_per_field, dtype=torch.int64)
        off = torch.zeros(rows.numel() + 1, dtype=torch.int64)
        off[1:] = torch.cumsum(rows, 0)
        self.F, self.num_rows = int(rows.numel()), int(off[-1])
        self.off = off.to(dev)
        g = torch.Generator(device=dev).manual_seed(seed)
        self.full = torch.randn((self.num_rows, D), device=dev, generator=g)
        self.local_rows = S.shard_rows(self.num_rows, G)
        self.shards = [S.full_to_shard(self.full, r, G) for r in range(G)]
        self.capacity = S.receive_capacity(batch, self.F, G, slack)
        self.vals = [torch.zeros((G, self.capacity, D), device=dev) for _ in range(G)]
        self.rows = [torch.full((G, self.capacity), -7, dtype=torch.int64, device=dev) for _ in range(G)]
        self.counts = [torch.zeros((G,), dtype=torch.int64, device=dev) for _ in range(G)]
        self.counters = torch.zeros((9,), dtype=torch.int64, device=dev)
        self.overflow = torch.zeros((1,), dtype=torch.int32, device=dev)
        self.w_ptrs, self.v_ptrs, self.r_ptrs, self.c_ptrs = _ptrs(self.shards), _ptrs(self.vals), _ptrs(self.rows), _ptrs(self.counts)

    def lookup(self, ids):
        from recalgorithm_b200 import _lib, ops
        B, F = ids.shape
        tile = torch.empty((B, F, self.D), device=ids.device)
        fm2 = torch.empty((B, 1), device=ids.device)
        L = _lib.lib()
        if ids.dtype == torch.int32:
            ids64 = torch.empty((B, F), dtype=torch.int64, device=ids.device)
            _lib.check(L.ctr_embed_fm2_fwd_sharded_ids32(self.w_ptrs, self.G, self.off.data_ptr(), ops._ptr(ids), B, F, self.D,
                                                         ops._ptr(tile), ops._ptr(fm2), ops._ptr(ids64), ops._stream()))
            return tile, fm2, ids64
        _lib.check(L.ctr_embed_fm2_fwd_sharded(self.w_ptrs, self.G, self.off.data_ptr(), ops._ptr(ids), B, F, self.D, ops._ptr(tile),
                                               ops._ptr(fm2), ops._stream()))
        return tile, fm2, ids

    def plan(self, rank, ids):
        from recalgorithm_b200 import _lib, ops
        B, F = ids.shape
        plan = torch.empty((B, F), dtype=torch.int32, device=ids.device)
        _lib.check(_lib.lib().ctr_sharded_plan(self.off.data_ptr(), ops._ptr(ids), int(ids.dtype == torch.int32), B, F, self.G, rank, self.r_ptrs, self.c_ptrs,
                                               self.capacity, self.counters.data_ptr(), self.overflow.data_ptr(), ops._ptr(plan),
                                               ops._stream()))
        return plan

    def bwd_push(self, rank, tile, d_tile, d_fm2, plan, row_grads=None):
        from recalgorithm_b200 import _lib, ops
        B, F, D = tile.shape
        _lib.check(_lib.lib().ctr_embed_fm2_bwd_push(ops._ptr(tile), ops._ptr(d_tile), ops._ptr(d_fm2), ops._ptr(plan), B, F, D,
                                                     self.G, rank, self.v_ptrs, self.capacity, ops._ptr(row_grads), ops._stream()))

    def push(self, rank, row_grads, plan):
        from recalgorithm_b200 import _lib, ops
        B, F, D = row_grads.shape
        _lib.check(_lib.lib().ctr_sharded_grad_push(ops._ptr(row_grads), ops._ptr(plan), B, F, D, self.G, rank, self.v_ptrs,
                                                    self.capacity, ops._stream()))

    def received_dense(self, owner):
        from recalgorithm_b200 import _lib, ops
        dense = torch.zeros((self.local_rows, self.D), device=self.off.device)
        for src in range(self.G):
            _lib.check(_lib.lib().ctr_rows_scatter_add(dense.data_ptr(), self.local_rows, self.D, self.rows[owner][src].data_ptr(),
                                                       self.vals[owner][src].data_ptr(), self.counts[owner][src:].data_ptr(),
                                                       self.capacity, ops._stream()))
        return dense


def _ids(gen, B, rows_t, dev):
    # includes -1 (OOV) and ids >= the field's row count (both -> zero vector / no gradient)
    return (torch.rand((B, rows_t.numel()), device=dev, generator=gen) * (rows_t[None, :] + 3)).long() - 1


def _reference_dense(grp, ids_per_rank, rg_per_rank):
    """float64 dense gradient of the FULL table from every rank's IndexedSlices, then split by owner."""
    full = torch.zeros((grp.num_rows, grp.D), dtype=torch.float64, device=grp.off.device)
    rows_t = grp.off[1:] - grp.off[:-1]
    for ids, rg in zip(ids_per_rank, rg_per_rank):
        valid = ((ids >= 0) & (ids < rows_t[None, :])).reshape(-1)
        gr = (ids + grp.off[:-1][None, :]).reshape(-1)[valid]
        full.index_add_(0, gr, rg.reshape(-1, grp.D)[valid].double())
    return [grp.S.full_to_shard(full, r, grp.G) for r in range(grp.G)]


@pytest.mark.parametrize("G", [2, 4, 8])
@pytest.mark.parametrize("B,F,D,rows_each", [(257, 40, 32, 5000), (64, 6, 8, 300), (1000, 33, 16, 1), (513, 100, 4, 50),
                                              (40, 20, 128, 30)])
def test_selfpeer_lookup_plan_push(G, B, F, D, rows_each):
    from recalgorithm_b200 import ops
    dev = torch.device("cuda", 0)
    rows = [rows_each + 3 * f for f in range(F)]
    grp = LocalShardGroup(rows, D, G, B)
    rows_t = torch.tensor(rows, device=dev)
    gen = torch.Generator(device=dev).manual_seed(100 + G)
    ids_all, rg_all = [], []
    for rank in range(G):
        ids = _ids(gen, B, rows_t, dev)
        tile, fm2, _ = grp.lookup(ids)
        valid = (ids >= 0) & (ids < rows_t[None, :])
        want = grp.full[(ids + grp.off[:-1][None, :]).clamp(0, grp.num_rows - 1)] * valid[..., None]
        assert torch.equal(tile, want), "peer-pull lookup must be an exact copy"
        e = want.double()
        assert_close(fm2, 0.5 * (e.sum(1).pow(2) - e.pow(2).sum(1)).sum(1, keepdim=True), what="fm2")
        tile32, fm232, ids64 = grp.lookup(ids.int())                      # int32 ids: same rows, widened copy returned
        assert torch.equal(tile32, tile) and torch.equal(fm232, fm2) and torch.equal(ids64, ids)
        d_tile = torch.randn((B, F, D), device=dev, generator=gen)
        d_fm2 = torch.randn((B,), device=dev, generator=gen)
        row_grads = ops.embed_fm2_bwd(tile, d_tile, d_fm2)
        plan = grp.plan(rank, ids)
        assert torch.equal((grp.plan(rank, ids.int()) >> 28), (plan >> 28)), "int32 ids plan to the same owners"
        plan = grp.plan(rank, ids)
        # plan words: valid ids have owner = global row % G and a slot below the published count; invalid ids are -1
        gr = ids + grp.off[:-1][None, :]
        assert torch.equal(plan < 0, ~valid)
        assert torch.equal((plan >> 28)[valid].long(), (gr % G)[valid])
        assert int(grp.overflow.item()) == 0
        for d in range(G):
            n_d = int(((gr % G == d) & valid).sum())
            assert int(grp.counts[d][rank]) == n_d
            slots = (plan & ((1 << 28) - 1))[valid & (gr % G == d)].long()
            assert slots.numel() == n_d and torch.equal(torch.sort(slots).values, torch.arange(n_d, device=dev)), "slots must be a permutation of 0..n-1"
            # the queue's row index at each slot is the entry's local row
            lrow = (gr // G)[valid & (gr % G == d)]
            assert torch.equal(grp.rows[d][rank][slots], lrow)
        # fused backward + push (row_grads also kept locally, must equal the unfused backward bit for bit)
        rg2 = torch.empty_like(row_grads)
        grp.bwd_push(rank, tile, d_tile, d_fm2, plan, row_grads=rg2)
        assert torch.equal(rg2, row_grads)
        ids_all.append(ids); rg_all.append(row_grads)
    want_shards = _reference_dense(grp, ids_all, rg_all)
    for d in range(G):
        assert_close(grp.received_dense(d), want_shards[d], what=f"fused push, owner {d}")
    # the plain push of existing row gradients fills the same queues (zero them first); row_grads = NULL in the fused form
    for v in grp.vals:
        v.zero_()
    for rank in range(G):
        plan = grp.plan(rank, ids_all[rank])
        if rank % 2 == 0:
            grp.push(rank, rg_all[rank], plan)
        else:
            tile, _, _ = grp.lookup(ids_all[rank])
            # reconstruct the same values through the fused kernel without the local copy: d_tile = row_grads, d_fm2 = 0
            grp.bwd_push(rank, tile, rg_all[rank], None, plan, row_grads=None)
    for d in range(G):
        assert_close(grp.received_dense(d), want_shards[d], what=f"plain push / NULL row_grads, owner {d}")


def test_selfpeer_overflow_is_flagged_and_counts_clamped():
    dev = torch.device("cuda", 0)
    G, B, F, D = 2, 512, 8, 8
    grp = LocalShardGroup([4] * F, D, G, B, slack=0.0)           # capacity = 1024 < entries sent to one owner? force it:
    grp.capacity = 100
    ids = torch.zeros((B, F), dtype=torch.int64, device=dev)      # every id 0 -> global rows 0,4,8,... -> all owner 0
    plan = grp.plan(0, ids)
    assert int(grp.overflow.item()) == 1
    assert int(grp.counts[0][0]) == 100 and int(grp.counts[1][0]) == 0
    assert int((plan >= 0).sum()) == 100
    ids[:] = -1
    plan = grp.plan(0, ids)                                        # the flag and the counts are reset by every plan
    assert int(grp.overflow.item()) == 0 and int(grp.counts[0][0]) == 0 and bool((plan == -1).all())


@pytest.mark.parametrize("lazy", [True, False])
def test_selfpeer_owner_adam(lazy):
    """Owner-side Adam straight from the receive queues (ctr_adam_rows_dedup) vs the float64 reference, heavy duplicates."""
    from oracle import sharded_ref as R                      # checker only
    from recalgorithm_b200 import _lib, ops
    dev = torch.device("cuda", 0)
    G, B, F, D = 4, 300, 12, 16
    rows = [40 + f for f in range(F)]
    grp = LocalShardGroup(rows, D, G, B)
    rows_t = torch.tensor(rows, device=dev)
    gen = torch.Generator(device=dev).manual_seed(5)
    V = grp.local_rows
    mv = [torch.zeros((V, 2, D), device=dev) for _ in range(G)]          # interleaved moments (state_stride = 2*D)
    m = [x[:, 0, :] for x in mv]
    v = [x[:, 1, :] for x in mv]
    dup_list = torch.empty((G * grp.capacity + 1,), dtype=torch.int32, device=dev)
    slot = [torch.full((V,), -1, dtype=torch.int32, device=dev) for _ in range(G)]
    ref = [(grp.shards[d].double().clone(), torch.zeros((V, D), dtype=torch.float64, device=dev),
            torch.zeros((V, D), dtype=torch.float64, device=dev)) for d in range(G)]
    lr = 0.01
    L = _lib.lib()
    for step in (1, 2):
        ids_all, rg_all = [], []
        for rank in range(G):
            ids = _ids(gen, B, rows_t, dev)
            rg = torch.randn((B, F, D), device=dev, generator=gen)
            grp.push(rank, rg, grp.plan(rank, ids))
            ids_all.append(ids); rg_all.append(rg)
        gd = _reference_dense(grp, ids_all, rg_all)
        lr_t = lr * (1.0 - 0.999 ** step) ** 0.5 / (1.0 - 0.9 ** step)
        for d in range(G):
            touched = torch.zeros((V,), dtype=torch.bool, device=dev)
            for src in range(G):
                touched[grp.rows[d][src, : int(grp.counts[d][src])]] = True
            bitmap = None if lazy else torch.zeros(((V + 31) // 32,), dtype=torch.int32, device=dev)
            n_unique = torch.zeros((1,), dtype=torch.int64, device=dev)
            _lib.check(L.ctr_adam_rows_dedup(grp.shards[d].data_ptr(), m[d].data_ptr(), v[d].data_ptr(), 2 * D, V, D, grp.rows[d].data_ptr(),
                                             grp.vals[d].data_ptr(), grp.counts[d].data_ptr(), G, grp.capacity, slot[d].data_ptr(),
                                             (dup_list.data_ptr() if d % 2 == 0 else None),       # both merge forms
                                             lr_t, 0.9, 0.999, 1e-8, ops._ptr(bitmap), n_unique.data_ptr(), ops._stream()))
            if not lazy:
                _lib.check(L.ctr_adam_dense_rest(grp.shards[d].data_ptr(), m[d].data_ptr(), v[d].data_ptr(), 2 * D, V, D, lr_t, 0.9,
                                                 0.999, 1e-8, ops._ptr(bitmap), ops._stream()))
            assert int(n_unique.item()) == int(touched.sum()) and bool((slot[d] == -1).all())
            ref[d] = R.adam_reference(*ref[d], gd[d], touched, step, lr, lazy)
            for name, a, b_ in (("var", grp.shards[d], ref[d][0]), ("m", m[d], ref[d][1]), ("v", v[d], ref[d][2])):
                assert_close(a, b_, what=f"owner adam lazy={lazy} step {step} owner {d} {name}")


@pytest.mark.parametrize("B,F,D,G", [(300, 40, 32, 2), (300, 40, 32, 8), (300, 16, 32, 2), (300, 24, 32, 8), (8192, 40, 32, 2)])
def test_selfpeer_fused_linear_head(B, F, D, G):
    """Sharded lookup + FM2 + fused dense(1) head and its backward+push equal the unsharded fused kernels / the plain chain."""
    from recalgorithm_b200 import _lib, ops
    dev = torch.device("cuda", 0)
    rows = [500 + 3 * f for f in range(F)]
    grp = LocalShardGroup(rows, D, G, B)
    rows_t = torch.tensor(rows, device=dev)
    gen = torch.Generator(device=dev).manual_seed(17 + G)
    wlin = torch.randn((F * D,), device=dev, generator=gen) * 0.3
    L = _lib.lib()
    ids_all, rg_all = [], []
    dw_sum = torch.zeros((F * D,), dtype=torch.float64, device=dev)
    for rank in range(G):
        ids = _ids(gen, B, rows_t, dev)
        id_in = ids.int() if rank % 2 else ids
        tile = torch.empty((B, F, D), device=dev); fm2 = torch.empty((B, 1), device=dev); lin = torch.empty((B, 1), device=dev)
        ids64 = torch.empty((B, F), dtype=torch.int64, device=dev)
        _lib.check(L.ctr_embed_fm2_lin_fwd_sharded(grp.w_ptrs, G, grp.off.data_ptr(), ops._ptr(id_in), int(rank % 2), B, F, D, ops._ptr(wlin),
                                                   ops._ptr(tile), ops._ptr(fm2), ops._ptr(lin), ops._ptr(ids64), ops._stream()))
        t_ref, f_ref, _ = grp.lookup(ids)
        assert torch.equal(tile, t_ref) and torch.equal(fm2, f_ref)
        if rank % 2:
            assert torch.equal(ids64, ids)
        assert_close(lin, tile.double().reshape(B, F * D) @ wlin.double()[:, None], what="fused head")
        d_fm2 = torch.randn((B,), device=dev, generator=gen); d_lin = torch.randn((B,), device=dev, generator=gen)
        rg_ref, dw_ref = ops.embed_fm2_lin_bwd(tile, wlin, d_fm2, d_lin)
        plan = grp.plan(rank, ids)
        rg = torch.empty_like(tile); dw = torch.empty((F * D,), device=dev)
        _lib.check(L.ctr_embed_fm2_lin_bwd_push(ops._ptr(tile), ops._ptr(wlin), ops._ptr(d_fm2), ops._ptr(d_lin), ops._ptr(plan), B, F, D, G,
                                                rank, grp.v_ptrs, grp.capacity, ops._ptr(rg), ops._ptr(dw), ops._stream()))
        assert torch.equal(rg, rg_ref), "row_grads (fused head + push vs fused head)"             # one kernel body
        assert_close(dw, dw_ref.double(), what="d_wlin")
        ids_all.append(ids); rg_all.append(rg_ref)
    want = _reference_dense(grp, ids_all, rg_all)
    for d in range(G):
        assert_close(grp.received_dense(d), want[d], what=f"fused-head push, owner {d}")
