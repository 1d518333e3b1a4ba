"""GPU parity: the DCN-V2 cross network (csrc/cross_v2.cu) against the float64 restatement of the paper's equations
(tests/_dcnv2_ref.py) -- forward and every gradient at the width, rank, depth and tile edges, the anchor to row CROSS,
the zero batch, per-sample bitwise rows, refusals, graph capture, the launches autograd makes, and the host layers and
model body."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest
import torch

from _dcnv2_ref import cross_v2_bwd, cross_v2_fwd
from _util import TOL, assert_close, dev

pytestmark = pytest.mark.gpu

# the weight gradients run tc_ptx.cuh's shared kernel; its cross_v2:: Rows type marks this layer's instantiations
DW_KERNEL = r"weight_grad_wgmma_kernel<[^,]+, ctr::cross_v2::"
KERNELS = ("cross_v2_prep_kernel", "cross_v2_rows_wgmma_kernel", DW_KERNEL)


def _inputs(B, d, L, rank, seed, with_xl):
    """x0, xl and g standard normal; weights scaled so that z_l has about half the spread of x_l at every width and rank,
    and biases of that order, so that x_l grows by about 1.25x in variance per layer."""
    rng = np.random.default_rng(seed)
    x0 = rng.standard_normal((B, d)).astype(np.float32)
    xl = rng.standard_normal((B, d)).astype(np.float32) if with_xl else None
    if rank:
        w = (rng.uniform(-1, 1, (L, d, rank)) * np.sqrt(3.0 / d)).astype(np.float32)
        u = (rng.uniform(-1, 1, (L, rank, d)) * 0.5 * np.sqrt(3.0 / rank)).astype(np.float32)
    else:
        w, u = (rng.uniform(-1, 1, (L, d, d)) * 0.5 * np.sqrt(3.0 / d)).astype(np.float32), None
    b = (rng.standard_normal((L, d)) * 0.3).astype(np.float32)
    g = rng.standard_normal((B, d)).astype(np.float32)
    return x0, xl, w, u, b, g


def _run(x0, xl, w, u, b, g, rank):
    from recalgorithm_b200 import ops
    args = [None if t is None else dev(t) for t in (x0, w, u, b)]
    xlt = None if xl is None else dev(xl)
    out, saved = ops.cross_v2_fwd(*args, rank, xl_in=xlt)
    grads = ops.cross_v2_bwd(*args, rank, saved, dev(g), xl_in=xlt)
    torch.cuda.synchronize()
    return out, grads


def _check(x0, xl, w, u, b, g, out, grads, what):
    ref_out, cache = cross_v2_fwd(x0, w, u, b, xl)
    ref = cross_v2_bwd(cache, w, u, g)
    assert_close(out, ref_out, TOL, f"{what}: out")
    for name, got, want in zip(("dx0", "dxl_in"), grads[:2], ref[:2]):
        if want is None:
            assert got is None, name
        else:
            assert_close(got, want, TOL, f"{what}: {name}")
    # the weight gradients are batch reductions over B samples whose terms cancel: doubled element-wise bound
    for name, got, want in zip(("dw", "du", "db"), grads[2:], ref[2:]):
        if want is None:
            assert got is None, name
        else:
            assert_close(got, want, TOL, f"{what}: {name}", elementwise=2.0)


DS = (1, 5, 31, 32, 33, 82, 127, 128, 129, 480, 511, 512)
RANKS = (0, 1, 7, 32, 64, 120, 128)
LS = (1, 3, 8)
BS = (1, 63, 64, 65, 127, 128, 129)
SHAPES = ([(BS[(i + j) % len(BS)], d, LS[(i + 2 * j) % len(LS)], rank, (i + j) % 2 == 1)
           for i, d in enumerate(DS) for j, rank in enumerate(RANKS)] +
          [(4096, 480, 3, rank, xl) for rank in (0, 120, 64) for xl in (False, True)] +
          [(4096, 82, 3, rank, False) for rank in (0, 16)])


@pytest.mark.parametrize("B,d,L,rank,with_xl", SHAPES)
def test_cross_v2_against_float64(B, d, L, rank, with_xl):
    inputs = _inputs(B, d, L, rank, B * 7 + d * 131 + L * 17 + rank * 5 + with_xl, with_xl)
    out, grads = _run(*inputs, rank)
    _check(*inputs, out, grads, f"B={B} d={d} L={L} rank={rank} xl={with_xl}")


@pytest.mark.parametrize("rank", [0, 120])
def test_full_batch_runs_many_weight_gradient_slices(rank):
    """B = 65536 at DCN config 2's width: the weight-gradient kernel splits the batch over many CTAs per weight row."""
    inputs = _inputs(65536, 480, 2, rank, 11 + rank, False)
    out, grads = _run(*inputs, rank)
    _check(*inputs, out, grads, f"B=65536 d=480 rank={rank}")


def test_rank_one_matches_row_cross():
    """With u = a row of ones and b = 0, the rank-1 layer is DCN v1 with zero bias: ctr_cross_fwd/bwd on the same inputs."""
    from recalgorithm_b200 import ops
    B, d, L = 300, 82, 3
    rng = np.random.default_rng(12)
    x0 = dev(rng.standard_normal((B, d)).astype(np.float32))
    ws = dev((rng.uniform(-1, 1, (L, d)) * np.sqrt(3.0 / d)).astype(np.float32))
    g = dev(rng.standard_normal((B, d)).astype(np.float32))
    zero = torch.zeros((L, d), device="cuda")
    v1_out = ops.cross_fwd(x0, ws, zero)
    v1_dx0, _, v1_dw, _ = ops.cross_bwd(x0, ws, zero, g)
    w, u = ws[:, :, None].contiguous(), torch.ones((L, 1, d), device="cuda")
    out, saved = ops.cross_v2_fwd(x0, w, u, zero, 1)
    dx0, _, dw, _, _ = ops.cross_v2_bwd(x0, w, u, zero, 1, saved, g)
    assert_close(out, v1_out.double(), TOL, "out against row CROSS")
    assert_close(dx0, v1_dx0.double(), TOL, "dx0 against row CROSS")
    assert_close(dw[:, :, 0], v1_dw.double(), TOL, "dw against row CROSS", elementwise=2.0)


@pytest.mark.parametrize("rank", [0, 5])
def test_empty_batch_launches_nothing_and_zeroes_the_weight_gradients(rank):
    from recalgorithm_b200 import _lib
    x0, xl, w, u, b, g = _inputs(0, 33, 3, rank, 1, True)
    w_ = dev(w)
    _run(x0, xl, w, u, b, g, rank)                      # module load outside the count
    n0 = _lib.kernel_launches()
    out, grads = _run(x0, xl, w, u, b, g, rank)
    assert _lib.kernel_launches() == n0
    assert out.shape == (0, 33) and grads[0].shape == (0, 33) and grads[1].shape == (0, 33)
    for t in grads[2:]:
        if t is not None:
            assert t.numel() > 0 and torch.count_nonzero(t) == 0
    assert grads[2].shape == w_.shape


@pytest.mark.parametrize("d,rank", [(82, 0), (480, 0), (480, 64)])
def test_per_sample_rows_are_bitwise_under_permutation_and_repetition(d, rank):
    B, L = 200, 3
    x0, xl, w, u, b, g = _inputs(B, d, L, rank, 5, True)
    out, grads = _run(x0, xl, w, u, b, g, rank)
    out2, grads2 = _run(x0, xl, w, u, b, g, rank)
    assert torch.equal(out, out2) and torch.equal(grads[0], grads2[0]) and torch.equal(grads[1], grads2[1])
    perm = np.random.default_rng(6).permutation(B)
    outp, gradsp = _run(x0[perm], xl[perm], w, u, b, g[perm], rank)
    inv = torch.from_numpy(np.argsort(perm)).cuda()
    assert torch.equal(outp[inv], out) and torch.equal(gradsp[0][inv], grads[0]) and torch.equal(gradsp[1][inv], grads[1])
    rep = lambda a: np.concatenate([a, a, a[:7]])
    outr, gradsr = _run(rep(x0), rep(xl), w, u, b, rep(g), rank)
    for k in (0, B):
        assert torch.equal(outr[k:k + B], out)
        assert torch.equal(gradsr[0][k:k + B], grads[0]) and torch.equal(gradsr[1][k:k + B], grads[1])


def test_forward_without_saved_equals_the_forward_with_it():
    """A forward-only call (saved = NULL) runs the layers in place in `out`: the same bits as the saving forward."""
    from recalgorithm_b200 import ops
    for rank in (0, 24):
        x0, _, w, u, b, _ = _inputs(1000, 480, 4, rank, 9, False)
        args = [None if t is None else dev(t) for t in (x0, w, u, b)]
        a, saved = ops.cross_v2_fwd(*args, rank)
        c, none = ops.cross_v2_fwd(*args, rank, want_saved=False)
        assert none is None and torch.equal(a, c), rank


BOUNDS = ((513, 1, 0, "d <= 512"), (0, 1, 0, "d <= 512"), (16, 9, 0, "L <= 8"), (16, 0, 0, "L <= 8"),
          (16, 2, 129, "rank <= 128"))


@pytest.mark.parametrize("d,L,rank,bound", BOUNDS)
def test_entries_refuse_shapes_past_the_bounds(d, L, rank, bound):
    from recalgorithm_b200 import _lib
    h = _lib.lib()
    buf = torch.zeros(1 << 16, device="cuda")
    P = buf.data_ptr()
    n, s = ctypes.c_int64(0), ctypes.c_int64(0)
    calls = {"ctr_cross_v2_workspace_bytes": lambda: h.ctr_cross_v2_workspace_bytes(4, d, L, rank, ctypes.byref(n),
                                                                                    ctypes.byref(s)),
             "ctr_cross_v2_fwd": lambda: h.ctr_cross_v2_fwd(P, None, P, P, P, 4, d, L, rank, P, P, P, buf.numel() * 4, None),
             "ctr_cross_v2_bwd": lambda: h.ctr_cross_v2_bwd(P, None, P, P, P, P, P, 4, d, L, rank, P, None, P, P, P, P,
                                                            buf.numel() * 4, None)}
    for entry, call in calls.items():
        assert call() == _lib.CTR_ERR_UNSUPPORTED, entry
        msg = h.ctr_last_error().decode()
        assert msg.startswith(entry) and bound in msg, msg
    torch.cuda.synchronize()


def test_short_workspace_short_saved_and_cpu_tensors_are_refused():
    from recalgorithm_b200 import _lib, ops
    h = _lib.lib()
    n, s = ctypes.c_int64(0), ctypes.c_int64(0)
    assert h.ctr_cross_v2_workspace_bytes(4, 33, 2, 5, ctypes.byref(n), ctypes.byref(s)) == 0
    assert s.value == 4 * ((2 * 2 - 1) * 33 + 2 * 5) * 4
    buf = torch.zeros(int(n.value) // 4 + 64, device="cuda")
    P = buf.data_ptr()
    assert h.ctr_cross_v2_bwd(P, None, P, P, P, P, P, 4, 33, 2, 5, P, None, P, P, P, P, int(n.value) - 128, None) == \
        _lib.CTR_ERR_INVALID_ARG
    assert "workspace" in h.ctr_last_error().decode()
    assert h.ctr_cross_v2_workspace_bytes(0, 33, 2, 5, ctypes.byref(n), ctypes.byref(s)) == 0
    assert h.ctr_cross_v2_fwd(P, None, P, P, P, 4, 33, 2, 5, P, P, P, int(n.value) - 128, None) == _lib.CTR_ERR_INVALID_ARG
    assert "workspace" in h.ctr_last_error().decode()
    x0, xl, w, u, b, g = _inputs(4, 33, 2, 5, 2, False)
    args = [dev(t) for t in (x0, w, u, b)]
    out, saved = ops.cross_v2_fwd(*args, 5)
    with pytest.raises(ValueError, match="saved"):
        ops.cross_v2_bwd(*args, 5, saved[:-4], dev(g))
    with pytest.raises(ValueError, match="saved"):
        ops.cross_v2_fwd(*args, 5, saved=saved[:-4])
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.cross_v2_fwd(*(torch.from_numpy(t) for t in (x0, w, u, b)), 5)
    torch.cuda.synchronize()


@pytest.mark.parametrize("rank", [0, 32])
def test_forward_and_backward_replay_in_a_cuda_graph(rank):
    from recalgorithm_b200 import ops
    x0, xl, w, u, b, g = _inputs(1000, 82, 3, rank, 13, True)
    args = [None if t is None else dev(t) for t in (x0, w, u, b)]
    xlt, gt = dev(xl), dev(g)

    def step():
        out, saved = ops.cross_v2_fwd(*args, rank, xl_in=xlt)
        return (out, *ops.cross_v2_bwd(*args, rank, saved, gt, xl_in=xlt))
    eager = step()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize()
    for k in range(3):                        # out, dx0, dxl_in: per-sample rows, bitwise
        assert torch.equal(captured[k], eager[k]), k
    for a, c in zip(captured[3:], eager[3:]):
        if c is not None:                     # fp32 atomics across CTAs: the weight gradients' order of adds may differ
            assert_close(a, c.double(), TOL, "graph weight gradient", elementwise=2.0)


_PROFILE = """
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, "tests")
from _util import dev
from test_gpu_dcnv2 import _inputs
from recalgorithm_b200 import autograd
for rank in (0, 16):
    x0, xl, w, u, b, g = _inputs(512, 480, 3, rank, 4, True)
    ts = [None if t is None else dev(t).requires_grad_(True) for t in (x0, xl, w, u, b)]
    gd = dev(g)
    autograd.cross_v2(ts[0], ts[2], ts[3], ts[4], rank, xl=ts[1]).backward(gd)   # first launches outside the trace
    torch.cuda.synchronize()
    for t in ts:
        if t is not None:
            t.grad = None
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        autograd.cross_v2(ts[0], ts[2], ts[3], ts[4], rank, xl=ts[1]).backward(gd)
        torch.cuda.synchronize()
    print(json.dumps([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]))
"""


def test_profiler_sees_only_the_new_kernels():
    """The autograd forward and backward launch the cross-V2 kernels and nothing else (memsets aside), at both ranks.  The
    trace is taken in a process of its own, so that this profiler session leaves the test process's profiler as it was."""
    import json
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    run = subprocess.run([sys.executable, "-c", _PROFILE], cwd=root, capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr[-3000:]
    for line in run.stdout.strip().splitlines()[-2:]:
        kernels = [n for n in json.loads(line) if not n.startswith("Memset")]
        assert kernels and all(any(re.search(k, n) for k in KERNELS) for n in kernels), sorted(set(kernels))
        for k in KERNELS:
            assert any(re.search(k, n) for n in kernels), k


@pytest.mark.parametrize("projection_dim", [None, 24])
def test_three_layer_stack_through_layers_matches_float64(projection_dim):
    from recalgorithm_b200 import layers as L
    B, d = 300, 82
    x = np.random.default_rng(7).standard_normal((B, d)).astype(np.float32)
    outs = {}
    store = L.set_default_store(L.VariableStore(device="cuda", seed=3))
    try:
        x0 = dev(x)
        with L.variable_scope("net"):
            outs["network"] = L.cross_network_v2(x0, 3, projection_dim)
        with L.variable_scope("net"):                 # the same variables, one layer per call
            net = x0
            for i in range(3):
                net = L.cross_layer_v2(x0, net, i, projection_dim)
            outs["loop"] = net
        v = {k: t.detach().cpu().numpy() for k, t in store.vars.items()}
    finally:
        L.set_default_store(L.VariableStore(device="cpu"))
    names = ("kernel",) if projection_dim is None else ("kernel_v", "kernel_u")
    w = np.stack([v[f"net/cross_v2_{i}/{names[0]}"] for i in range(3)])
    u = None if projection_dim is None else np.stack([v[f"net/cross_v2_{i}/kernel_u"] for i in range(3)])
    b = np.stack([v[f"net/cross_v2_{i}/bias"] for i in range(3)])
    ref, _ = cross_v2_fwd(x, w, u, b)
    for k, got in outs.items():
        assert_close(got, ref, TOL, f"three cross-V2 layers ({k})")


@pytest.mark.parametrize("structure", ["stacked", "parallel"])
@pytest.mark.parametrize("projection_dim", [None, 16])
def test_model_body_reaches_the_tables_and_every_variable(structure, projection_dim):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import model_bodies as M
    from recalgorithm_b200 import autograd, layers as L
    B, F, D, rows, n_dense = 64, 5, 16, 100, 2
    rng = np.random.default_rng(9)
    store = L.set_default_store(L.VariableStore(device="cuda", seed=5))
    try:
        tables = autograd.EmbeddingTables([rows] * F, D, device="cuda")
        ids = torch.from_numpy(rng.integers(0, rows, (B, F))).cuda()
        cat = autograd.lookup(tables, ids).reshape(B, F * D)
        dense_in = dev(rng.standard_normal((B, n_dense)).astype(np.float32))
        logit = M.dcn_v2_logit(dense_in, cat, num_cross_layer=3, projection_dim=projection_dim, structure=structure)
        assert logit.shape == (B, 1)
        logit.sum().backward()
        assert tables.grad_slices and all(torch.isfinite(gs.values).all() for gs in tables.grad_slices)
        assert any(torch.count_nonzero(gs.values) > 0 for gs in tables.grad_slices)
        want = {f"cross_part/cross_v2_{i}/{n}" for i in range(3)
                for n in (("kernel",) if projection_dim is None else ("kernel_v", "kernel_u")) + ("bias",)}
        assert want <= set(store.vars)
        for name, v in store.vars.items():
            assert v.grad is not None and torch.isfinite(v.grad).all() and torch.count_nonzero(v.grad) > 0, name
    finally:
        L.set_default_store(L.VariableStore(device="cpu"))
