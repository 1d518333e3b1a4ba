"""GPU parity: the FLEN field-wise bi-interaction (csrc/flen.cu) against the float64 restatement (tests/_flen_ref.py) --
both forward forms, the backward, the NFM and FwFM fixtures through the two degenerate groupings, exact cases, refusals,
graph capture, the launches autograd makes, and the model body."""
import itertools
import os
import sys

import numpy as np
import pytest
import torch

from _flen_ref import fwbi_bwd, fwbi_fwd, pairs
from _util import TOL, assert_close, dev, golden

pytestmark = pytest.mark.gpu

ROWS = 50          # rows per field; ids are drawn from [-2, ROWS + 5): negative and out-of-range ids give zero rows


def _inputs(B, F, D, M, seed):
    rng = np.random.default_rng(seed)
    table = (rng.standard_normal((F * ROWS, D)) * 0.5).astype(np.float32)
    off = np.arange(F + 1, dtype=np.int64) * ROWS
    ids = rng.integers(-2, ROWS + 5, (B, F)).astype(np.int64)
    group = [int(g) for g in rng.integers(0, M, F)]
    kmf = rng.standard_normal(M * (M - 1) // 2).astype(np.float32)
    kfm = rng.standard_normal(M).astype(np.float32)
    bmf, bfm = (rng.standard_normal(D).astype(np.float32) for _ in range(2))
    g = rng.standard_normal((B, D)).astype(np.float32)
    dt = rng.standard_normal((B, F, D)).astype(np.float32)
    return table, off, ids, group, (kmf, kfm, bmf, bfm), g, dt


def _gather(table, off, ids):
    ok = (ids >= 0) & (ids < np.diff(off)[None, :])
    rows = np.where(ok, off[:-1][None, :] + ids, 0)
    return np.where(ok[..., None], table[rows], np.float32(0))


def _check(B, F, D, M, seed):
    from recalgorithm_b200 import ops
    table, off, ids, group, w, g, dt = _inputs(B, F, D, M, seed)
    e = _gather(table, off, ids)
    wd = [dev(t) for t in w]
    h_ref = fwbi_fwd(e, group, M, *w)
    # fused forward: int64 ids with the tile, int32 ids without it (widened ids written)
    tile, h = ops.embed_fwbi_fwd(dev(table), dev(off), dev(ids), group, *wd)
    assert np.array_equal(tile.cpu().numpy(), e), "the tile must be the table rows, bit for bit"
    assert_close(h, h_ref, TOL, f"h B={B} F={F} D={D} M={M}")
    ids64 = torch.empty((B, F), dtype=torch.int64, device="cuda")
    none, h32 = ops.embed_fwbi_fwd(dev(table), dev(off), dev(ids, torch.int32), group, *wd, want_tile=False, ids64_out=ids64)
    assert none is None and torch.equal(h32, h) and np.array_equal(ids64.cpu().numpy(), ids)
    assert torch.equal(ops.fwbi_fwd(tile, group, *wd), h)                      # tile-input form: same sums, same order
    for d_tile in (dt, None):
        got = ops.fwbi_bwd(tile, None if d_tile is None else dev(d_tile), dev(g), group, wd[0], wd[1])
        ref = fwbi_bwd(e, group, M, w[0], w[1], g, d_tile)
        assert_close(got[0], ref[0], TOL, f"row_grads d_tile={d_tile is not None} B={B} F={F} D={D} M={M}")
        for name, a, b in zip(("d_kernel_mf", "d_kernel_fm", "d_bias_mf", "d_bias_fm"), got[1:], ref[1:]):
            # batch-reduced sums over B*D terms of both signs: the float32 error follows sum|terms|, not |result|
            assert_close(a, b, TOL, f"{name} B={B} F={F} D={D} M={M}", elementwise=2.0)


GRID = list(itertools.product((1, 2, 7, 32, 33, 40, 64, 256), (4, 8, 32, 128), (1, 2, 3, 8)))


@pytest.mark.parametrize("F,D,M", GRID)
def test_fwbi_against_float64(F, D, M):
    """Every HOLD class (F*D <= 512, 1024, 1536) and the two-pass backward (F*D > 1536); B cycles through 1, 9, 1031."""
    B = (1, 9, 1031)[GRID.index((F, D, M)) % 3]
    _check(B, F, D, M, seed=F * 1000 + D * 10 + M)


@pytest.mark.parametrize("F,D", [(40, 32), (64, 32)])
@pytest.mark.parametrize("M", [4, 5])
def test_slot_count_boundary(F, D, M):
    """M = 4 is the largest group count of the 4-slot kernels, M = 5 the smallest of the 8-slot ones."""
    _check(1031, F, D, M, seed=F + 10 * M)


def test_biases_need_only_float_alignment():
    """bias_mf and bias_fm at a 4-byte offset (slices of one flat parameter buffer) give the same h as aligned copies."""
    from recalgorithm_b200 import ops
    table, off, ids, group, w, g, dt = _inputs(9, 7, 32, 3, seed=12)
    flat = torch.zeros(1 + 2 * 32, device="cuda")
    flat[1:33], flat[33:] = dev(w[2]), dev(w[3])
    bmf, bfm = flat[1:33], flat[33:]
    assert bmf.data_ptr() % 16 == 4 and bfm.data_ptr() % 16 == 4
    kmf, kfm = dev(w[0]), dev(w[1])
    tile, h = ops.embed_fwbi_fwd(dev(table), dev(off), dev(ids), group, *(dev(t) for t in w))
    assert torch.equal(ops.embed_fwbi_fwd(dev(table), dev(off), dev(ids), group, kmf, kfm, bmf, bfm)[1], h)
    assert torch.equal(ops.fwbi_fwd(tile, group, kmf, kfm, bmf, bfm), h)


def test_full_batch():
    _check(65536, 40, 32, 3, seed=11)


@pytest.mark.parametrize("name", ["nfm_bi_F6_D8", "nfm_bi_F40_D32"])
def test_one_group_reproduces_nfm_fixture(name):
    from recalgorithm_b200 import ops
    z = golden(name)
    B, F, D = z["e"].shape
    zeros = torch.zeros(D, device="cuda")
    h = ops.fwbi_fwd(dev(z["e"]), [0] * F, torch.zeros(0, device="cuda"), dev(np.float32([0.5])), zeros, zeros)
    assert_close(h, z["out_f64"], TOL, name)


def test_singleton_groups_reproduce_fwfm_fixture():
    from recalgorithm_b200 import ops
    z = golden("fwfm_F6_D8")
    B, F, D = z["e"].shape
    zeros = torch.zeros(D, device="cuda")
    h = ops.fwbi_fwd(dev(z["e"]), list(range(F)), dev(z["r"]), dev(np.full(F, 0.37, np.float32)), zeros, zeros)
    assert_close(h.sum(-1, keepdim=True), z["out_f64"], TOL, "fwfm_F6_D8")


@pytest.mark.parametrize("F,D", [(1, 4), (5, 32), (8, 128)])
def test_singleton_groups_give_exact_zeros(F, D):
    from recalgorithm_b200 import ops
    table, off, ids, _, _, g, _ = _inputs(33, F, D, F, seed=F)
    zeros = torch.zeros(D, device="cuda")
    kmf, kfm = torch.zeros(F * (F - 1) // 2, device="cuda"), dev(np.linspace(-1, 1, F, dtype=np.float32))
    tile, h = ops.embed_fwbi_fwd(dev(table), dev(off), dev(ids), list(range(F)), kmf, kfm, zeros, zeros)
    rg, _, d_kfm, _, _ = ops.fwbi_bwd(tile, None, dev(g), list(range(F)), kmf, kfm)
    assert not h.any() and not rg.any() and not d_kfm.any()


def test_empty_batch_launches_nothing_and_zeroes_weight_gradients():
    from recalgorithm_b200 import _lib, ops
    table, off, ids, group, w, g, dt = _inputs(0, 7, 8, 3, seed=3)
    wd = [dev(t) for t in w]
    n0 = _lib.kernel_launches()
    tile, h = ops.embed_fwbi_fwd(dev(table), dev(off), dev(ids), group, *wd)
    assert ops.fwbi_fwd(tile, group, *wd).shape == (0, 8)
    out = ops.fwbi_bwd(tile, None, torch.zeros((0, 8), device="cuda"), group, wd[0], wd[1])
    torch.cuda.synchronize()
    assert _lib.kernel_launches() == n0 and h.shape == (0, 8) and out[0].shape == (0, 7, 8)
    assert all(t.numel() > 0 and not t.any() for t in out[1:])


def test_batch_permutation_and_repeat_are_bitwise():
    from recalgorithm_b200 import ops
    table, off, ids, group, w, g, dt = _inputs(1031, 40, 32, 3, seed=4)
    wd = [dev(t) for t in w]
    perm = np.random.default_rng(0).permutation(1031)

    def run(i, gg, d):
        tile, h = ops.embed_fwbi_fwd(dev(table), dev(off), dev(i), group, *wd)
        return h, ops.fwbi_bwd(tile, dev(d), dev(gg), group, wd[0], wd[1])
    h0, b0 = run(ids, g, dt)
    h1, b1 = run(ids, g, dt)
    hp, bp = run(ids[perm], g[perm], dt[perm])
    assert torch.equal(h0, h1) and torch.equal(b0[0], b1[0])
    assert torch.equal(hp, h0[perm]) and torch.equal(bp[0], b0[0][perm])
    for a, b in zip(b0[1:], bp[1:]):                                    # atomics: the weight gradients to tolerance only
        assert_close(a, b.double(), TOL, "weight gradient under permutation", elementwise=2.0)


def test_cuda_graph_replay_matches_eager():
    from recalgorithm_b200 import ops
    table, off, ids, group, w, g, dt = _inputs(1031, 33, 32, 8, seed=5)
    args = [dev(table), dev(off), dev(ids)]
    wd = [dev(t) for t in w]
    gd, dtd = dev(g), dev(dt)

    def step():
        tile, h = ops.embed_fwbi_fwd(*args, group, *wd)
        return (h, *ops.fwbi_bwd(tile, dtd, gd, group, wd[0], wd[1]))
    eager = step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()                                                          # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured[0], eager[0]) and torch.equal(captured[1], eager[1])
    for a, b in zip(captured[2:], eager[2:]):
        assert_close(a, b.double(), TOL, "graph weight gradient", elementwise=2.0)


def test_refusals():
    from recalgorithm_b200 import _lib, ops
    x = torch.randn(4, 8, 32, device="cuda")
    z32 = torch.zeros(32, device="cuda")
    kw = lambda M: (torch.ones(M * (M - 1) // 2, device="cuda"), torch.ones(M, device="cuda"), z32, z32)

    def refused(code, match, fn, *a):
        with pytest.raises(_lib.CtrInvalidArgument, match=match) as err:
            fn(*a)
        assert err.value.code == code
    U, I = _lib.CTR_ERR_UNSUPPORTED, _lib.CTR_ERR_INVALID_ARG
    refused(U, "F <= 256", ops.fwbi_fwd, torch.randn(2, 257, 32, device="cuda"), [0] * 257, *kw(1))
    refused(U, "1 <= M <= 8", ops.fwbi_fwd, x, [0] * 8, *kw(9))
    refused(U, "1 <= M <= 8", ops.fwbi_fwd, x, [0] * 8, *kw(0))
    refused(U, "power of two", ops.fwbi_fwd, torch.randn(4, 8, 12, device="cuda"), [0] * 8, torch.ones(0, device="cuda"),
            torch.ones(1, device="cuda"), torch.zeros(12, device="cuda"), torch.zeros(12, device="cuda"))
    refused(I, r"field_group\[3\]=2 outside \[0, M=2\)", ops.fwbi_fwd, x, [0, 1, 0, 2, 0, 0, 0, 0], *kw(2))
    refused(I, r"field_group\[0\]=-1", ops.fwbi_bwd, x, None, torch.randn(4, 32, device="cuda"), [-1] + [0] * 7, *kw(2)[:2])
    flat = torch.zeros(4 * 8 * 32 + 1, device="cuda")
    refused(I, "16-byte aligned", ops.fwbi_fwd, flat[1:].view(4, 8, 32), [0] * 8, *kw(2))
    refused(I, "16-byte aligned", ops.fwbi_bwd, x, flat[1:].view(4, 8, 32), torch.randn(4, 32, device="cuda"), [0] * 8,
            *kw(2)[:2])
    table = torch.randn(8 * 10, 32, device="cuda")
    off = torch.arange(9, dtype=torch.int64, device="cuda") * 10
    refused(I, "16-byte aligned", ops.embed_fwbi_fwd, torch.zeros(80 * 32 + 1, device="cuda")[1:].view(80, 32), off,
            torch.zeros(4, 8, dtype=torch.int64, device="cuda"), [0] * 8, *kw(2))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.fwbi_fwd(x.cpu(), [0] * 8, *kw(2))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.embed_fwbi_fwd(table, off, torch.zeros(4, 8, dtype=torch.int64), [0] * 8, *kw(2))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.fwbi_bwd(x, None, torch.randn(4, 32), [0] * 8, *kw(2)[:2])


_PROFILE = """
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, "tests")
from _util import dev
from test_gpu_flen import _inputs
from recalgorithm_b200 import autograd
table, off, ids, group, w, g, dt = _inputs(512, 40, 32, 3, seed=6)
tables = autograd.EmbeddingTables([50] * 40, 32, device="cuda", init=None)
tables.weight.copy_(dev(table))
wt = [dev(t).requires_grad_(True) for t in w]
idt, gd, dtd = dev(ids), dev(g), dev(dt)
def step():
    tile, h = autograd.lookup_fwbi(tables, idt, group, *wt)
    torch.autograd.backward([tile, h], [dtd, gd])
step()                                                          # first launches (module load) outside the trace
torch.cuda.synchronize()
for t in wt:
    t.grad = None                                               # a second backward would accumulate into .grad with adds
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    step()
    torch.cuda.synchronize()
print(json.dumps([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]))
"""


def test_profiler_sees_only_the_new_kernels():
    """One autograd step (fused forward, backward) launches the two FwBI kernels and nothing else (memsets aside).  The trace
    is taken in a process of its own, so that this profiler session leaves the test process's profiler as it was."""
    import json
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    run = subprocess.run([sys.executable, "-c", _PROFILE], cwd=root, capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr[-3000:]
    kernels = [n for n in json.loads(run.stdout.strip().splitlines()[-1]) if not n.startswith("Memset")]
    assert sum("fwbi_fwd_kernel" in n for n in kernels) == 1, kernels
    assert sum("fwbi_bwd_kernel" in n for n in kernels) == 1, kernels
    assert len(kernels) == 2, kernels


def _torch_body(table, off, ids, group, M, fo, v, hidden):
    """flen_logit in float64 torch: gather, FwBI, DNN, dense(concat([h, dnn]), 1) + first-order logit."""
    ok = (ids >= 0) & (ids < torch.diff(off)[None, :])
    rows = torch.where(ok, off[:-1][None, :] + ids, torch.zeros_like(ids))
    e = table[rows] * ok[..., None]
    oh = torch.zeros(len(group), M, dtype=torch.float64)
    oh[torch.arange(len(group)), torch.tensor(group)] = 1.0
    p, q = torch.einsum("bfd,fm->bmd", e, oh), torch.einsum("bfd,fm->bmd", e * e, oh)
    s = "field_wise_bi_interaction/"
    h = v[s + "bias_mf"] + v[s + "bias_fm"] + torch.einsum("m,bmd->bd", v[s + "kernel_fm"], p * p - q)
    for k, (i, j) in enumerate(pairs(M)):
        h = h + v[s + "kernel_mf"][k] * p[:, i] * p[:, j]
    net = e.reshape(e.shape[0], -1)
    for i in range(hidden):
        net = torch.relu(net @ v[f"dnn_part/dense_{i}/kernel"] + v[f"dnn_part/dense_{i}/bias"])
    return torch.cat([h, net], -1) @ v["output_part/dense/kernel"] + v["output_part/dense/bias"] + fo


def test_model_body_and_one_adam_step_match_float64():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import model_bodies as MB
    from recalgorithm_b200 import autograd, layers as L
    B, F, D = 64, 10, 16
    table, off, ids, _, _, _, _ = _inputs(B, F, D, 3, seed=8)
    keys = ["user", "user", "item", "item", "item", "context", "user", "context", "item", "user"]
    group, M = [0, 0, 1, 1, 1, 2, 0, 2, 1, 0], 3
    fo = np.random.default_rng(9).standard_normal((B, 1)).astype(np.float32)
    tables = autograd.EmbeddingTables([ROWS] * F, D, device="cuda", init=None)
    tables.weight.copy_(dev(table))
    fo_t = dev(fo).requires_grad_(True)
    store = L.set_default_store(L.VariableStore(device="cuda", seed=5))
    try:
        logit = MB.flen_logit(tables, dev(ids), keys, fo_t, hidden_units=(64, 32))
        names = sorted(store.vars)
        tv = {n: torch.tensor(store.vars[n].detach().cpu().numpy().astype(np.float64), requires_grad=True) for n in names}
        t64 = torch.tensor(table.astype(np.float64), requires_grad=True)
        fo64 = torch.tensor(fo.astype(np.float64), requires_grad=True)
        ref = _torch_body(t64, torch.tensor(off), torch.tensor(ids), group, M, fo64, tv, 2)
        assert_close(logit, ref.detach().numpy(), TOL, "flen_logit")
        logit.sum().backward()
        ref.sum().backward()
        assert len(tables.grad_slices) == 1
        assert_close(tables.grad_slices[0].to_dense(tables.num_rows), t64.grad.numpy(), TOL, "table gradient (IndexedSlices)")
        assert_close(fo_t.grad, fo64.grad.numpy(), TOL, "first-order logit gradient")
        for n in names:
            # batch-reduced weight gradients (sums over B samples whose terms cancel): doubled element-wise bound
            assert_close(store.vars[n].grad, tv[n].grad.numpy(), TOL, f"gradient {n}", elementwise=2.0)
        torch.optim.Adam(list(store.vars.values()), lr=1e-2).step()
        torch.optim.Adam([tv[n] for n in names], lr=1e-2).step()
        for n in names:
            assert_close(store.vars[n], tv[n].detach().numpy(), TOL, f"Adam step {n}")
    finally:
        L.set_default_store(L.VariableStore(device="cpu"))
