"""GPU parity: the DCN-Mix cross network (csrc/cross_mix.cu) against the float64 restatement of the paper's equations
(tests/_dcnmix_ref.py) -- forward and every gradient at the width, expert, rank, depth and tile edges, the anchor to row
CROSS-V2, the gate's edge cases, the zero batch, per-sample bitwise rows, refusals, graph capture, the launches autograd
makes, and the host layer and model body."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest
import torch

from _dcnmix_ref import cross_mix_bwd, cross_mix_fwd
from _util import TOL, assert_close, dev

pytestmark = pytest.mark.gpu

# the weight gradients run tc_ptx.cuh's shared kernel; its cross_mix:: Rows type marks this layer's instantiations
DW_KERNEL = r"weight_grad_wgmma_kernel<[^,]+, ctr::cross_mix::"
KERNELS = ("cross_mix_prep_kernel", "cross_mix_rows_wgmma_kernel", "cross_mix_fold_kernel", DW_KERNEL)
NAMES = ("dx0", "dv", "dc", "du", "db", "dgate")


def _inputs(B, d, L, K, r, seed, gate_scale=1.0, act=1):
    """x0 and g standard normal; v and gate scaled so that q and the gate logits have about unit spread, c so that m has
    about the spread of t, u so that z_l has about half the spread of x_l; biases of that order.  The identity does not
    saturate, so x_{l+1} grows with x0 * x_l; for it u is halved, which keeps eight layers well conditioned enough for
    plain fp32 arithmetic to meet the 1e-5 bars (at d = 1, L = 8 it does not without)."""
    rng = np.random.default_rng(seed)
    x0 = rng.standard_normal((B, d)).astype(np.float32)
    v = (rng.uniform(-1, 1, (L, K, d, r)) * np.sqrt(3.0 / d)).astype(np.float32)
    c = (rng.uniform(-1, 1, (L, K, r, r)) * np.sqrt(3.0 / r)).astype(np.float32)
    u = (rng.uniform(-1, 1, (L, K, r, d)) * (0.5 if act else 0.25) * np.sqrt(3.0 / r)).astype(np.float32)
    b = (rng.standard_normal((L, d)) * 0.3).astype(np.float32)
    gate = (rng.uniform(-1, 1, (d, K)) * gate_scale * np.sqrt(3.0 / d)).astype(np.float32)
    g = rng.standard_normal((B, d)).astype(np.float32)
    return x0, v, c, u, b, gate, g


def _run(x0, v, c, u, b, gate, g, act):
    from recalgorithm_b200 import ops
    args = [dev(t) for t in (x0, v, c, u, b, gate)]
    out, saved = ops.cross_mix_fwd(*args, act)
    grads = ops.cross_mix_bwd(*args, saved, dev(g), act)
    torch.cuda.synchronize()
    return out, grads, saved


def _check(x0, v, c, u, b, gate, g, act, out, grads, what):
    ref_out, cache = cross_mix_fwd(x0, v, c, u, b, gate, act)
    ref = cross_mix_bwd(cache, v, c, u, gate, g)
    assert_close(out, ref_out, TOL, f"{what}: out")
    assert_close(grads[0], ref[0], TOL, f"{what}: dx0")
    # the weight gradients are batch reductions over B samples whose terms cancel: doubled element-wise bound
    for name, got, want in zip(NAMES[1:], grads[1:], ref[1:]):
        assert_close(got, want, TOL, f"{what}: {name}", elementwise=2.0)


DS = (1, 5, 82, 128, 129, 480, 512)
KRS = ((1, 1), (1, 128), (3, 7), (4, 32), (8, 16), (16, 8))
LS = (1, 3, 8)
BS = (1, 63, 64, 65, 1000)
SHAPES = [(BS[(i + j) % len(BS)], d, LS[(i + 2 * j) % len(LS)], K, r, (i + j) % 2)
          for i, d in enumerate(DS) for j, (K, r) in enumerate(KRS)]


@pytest.mark.parametrize("B,d,L,K,r,act", SHAPES)
def test_cross_mix_against_float64(B, d, L, K, r, act):
    inputs = _inputs(B, d, L, K, r, B * 7 + d * 131 + L * 17 + K * 5 + r, act=act)
    out, grads, _ = _run(*inputs, act)
    _check(*inputs, act, out, grads, f"B={B} d={d} L={L} K={K} r={r} act={act}")


@pytest.mark.parametrize("K,r", [(4, 32), (8, 16)])
def test_full_batch_runs_many_weight_gradient_slices(K, r):
    """B = 65536 at DCN config 2's width: the weight-gradient kernel splits the batch over many CTAs per weight row."""
    inputs = _inputs(65536, 480, 2, K, r, 11 + K)
    out, grads, _ = _run(*inputs, 1)
    _check(*inputs, 1, out, grads, f"B=65536 d=480 K={K} r={r}")


def test_one_expert_with_identity_and_c_equal_to_i_is_row_cross_v2():
    """K = 1, the identity and c = I make each layer CROSS-V2's low-rank layer with w = v[:,0], u = u[:,0]: the same
    inputs through ctr_cross_v2_fwd/bwd."""
    from recalgorithm_b200 import ops
    B, d, L, r = 300, 82, 3, 24
    x0, v, _, u, b, gate, g = _inputs(B, d, L, 1, r, 12)
    c = np.broadcast_to(np.eye(r, dtype=np.float32), (L, 1, r, r)).copy()
    out, grads, _ = _run(x0, v, c, u, b, gate, g, 0)
    w2, u2 = dev(v[:, 0]), dev(u[:, 0])
    v2_out, saved = ops.cross_v2_fwd(dev(x0), w2, u2, dev(b), r)
    v2 = ops.cross_v2_bwd(dev(x0), w2, u2, dev(b), r, saved, dev(g))
    assert_close(out, v2_out.double(), TOL, "out against CROSS-V2")
    assert_close(grads[0], v2[0].double(), TOL, "dx0 against CROSS-V2")
    for name, got, want in (("dv", grads[1][:, 0], v2[2]), ("du", grads[3][:, 0], v2[3]), ("db", grads[4], v2[4])):
        assert_close(got, want.double(), TOL, f"{name} against CROSS-V2", elementwise=2.0)


def test_one_expert_gates_with_exactly_one_and_gets_no_gate_gradient():
    B, d, L, K, r = 200, 82, 3, 1, 16
    x0, v, c, u, b, gate, g = _inputs(B, d, L, K, r, 3, gate_scale=5.0)
    out, grads, saved = _run(x0, v, c, u, b, gate, g, 1)
    p = saved.view(torch.float32)[-L * B * K:]          # saved ends with p (L, B, K)
    assert torch.equal(p, torch.ones_like(p))
    assert torch.count_nonzero(grads[5]) == 0


def test_identical_experts_equal_one_expert_for_any_gate():
    B, d, L, r = 257, 82, 3, 16
    x0, v, c, u, b, _, g = _inputs(B, d, L, 1, r, 4)
    K = 4
    rep = lambda a: np.repeat(a, K, axis=1)
    gate = (np.random.default_rng(5).standard_normal((d, K)) * 0.5).astype(np.float32)
    one_out, one, _ = _run(x0, v, c, u, b, np.zeros((d, 1), np.float32), g, 1)
    out, grads, _ = _run(x0, rep(v), rep(c), rep(u), b, gate, g, 1)
    assert_close(out, one_out.double(), TOL, "out")
    assert_close(grads[0], one[0].double(), TOL, "dx0")
    for k, name in ((1, "dv"), (2, "dc"), (3, "du")):        # the expert gradients sum to the single expert's
        assert_close(grads[k].sum(1), one[k][:, 0].double(), TOL, name, elementwise=2.0)
    assert_close(grads[4], one[4].double(), TOL, "db", elementwise=2.0)


def test_gate_logits_near_80_stay_finite():
    """Logits of magnitude ~80 (exp would overflow without the max subtracted) give finite outputs and gradients that
    still follow float64."""
    B, d, L, K, r = 300, 82, 2, 4, 8
    inputs = list(_inputs(B, d, L, K, r, 6))
    rng = np.random.default_rng(7)
    inputs[5] = (80.0 * np.sign(rng.standard_normal((d, K))) / d).astype(np.float32)
    inputs[0] = np.abs(inputs[0]) * np.sign(inputs[5][:, :1].T)          # x0 . gate[:, 0] ~ +80, others ~ +-80 / ..
    out, grads, saved = _run(*inputs, 1)
    logits = inputs[0].astype(np.float64) @ inputs[5].astype(np.float64)
    assert np.abs(logits).max() > 60
    for t in (out, *grads):
        assert torch.isfinite(t).all()
    p = saved.view(torch.float32)[-L * B * K:].reshape(L, B, K)
    assert torch.allclose(p.sum(-1), torch.ones_like(p[..., 0]), atol=1e-6)
    ref_out, _ = cross_mix_fwd(*inputs[:6], 1)
    assert_close(out, ref_out, 1e-4, "out at large logits")


def test_empty_batch_launches_nothing_and_zeroes_the_weight_gradients():
    from recalgorithm_b200 import _lib
    inputs = _inputs(0, 33, 3, 4, 5, 1)
    _run(*inputs, 1)                                     # module load outside the count
    n0 = _lib.kernel_launches()
    out, grads, _ = _run(*inputs, 1)
    assert _lib.kernel_launches() == n0
    assert out.shape == (0, 33) and grads[0].shape == (0, 33)
    for t, ref in zip(grads[1:], inputs[1:6]):
        assert t.shape == ref.shape and torch.count_nonzero(t) == 0


@pytest.mark.parametrize("d,K,r", [(82, 4, 32), (480, 8, 16)])
def test_per_sample_rows_are_bitwise_under_permutation_and_repetition(d, K, r):
    B, L = 200, 3
    x0, v, c, u, b, gate, g = _inputs(B, d, L, K, r, 5)
    w = (v, c, u, b, gate)
    out, grads, _ = _run(x0, *w, g, 1)
    out2, grads2, _ = _run(x0, *w, g, 1)
    assert torch.equal(out, out2) and torch.equal(grads[0], grads2[0])
    perm = np.random.default_rng(6).permutation(B)
    outp, gradsp, _ = _run(x0[perm], *w, g[perm], 1)
    inv = torch.from_numpy(np.argsort(perm)).cuda()
    assert torch.equal(outp[inv], out) and torch.equal(gradsp[0][inv], grads[0])
    rep = lambda a: np.concatenate([a, a, a[:7]])
    outr, gradsr, _ = _run(rep(x0), *w, rep(g), 1)
    for k in (0, B):
        assert torch.equal(outr[k:k + B], out) and torch.equal(gradsr[0][k:k + B], grads[0])


def test_forward_without_saved_equals_the_forward_with_it():
    """A forward-only call (saved = NULL) runs the layers in place in `out`: the same bits as the saving forward."""
    from recalgorithm_b200 import ops
    for act in (0, 1):
        x0, v, c, u, b, gate, _ = _inputs(1000, 480, 4, 4, 32, 9)
        args = [dev(t) for t in (x0, v, c, u, b, gate)]
        a, saved = ops.cross_mix_fwd(*args, act)
        o, none = ops.cross_mix_fwd(*args, act, want_saved=False)
        assert none is None and torch.equal(a, o), act


BOUNDS = ((513, 1, 1, 4, "d <= 512"), (0, 1, 1, 4, "d <= 512"), (16, 9, 1, 4, "L <= 8"), (16, 0, 1, 4, "L <= 8"),
          (16, 2, 17, 4, "K <= 16"), (16, 2, 0, 4, "K <= 16"), (16, 2, 4, 0, "r >= 1"), (16, 2, 4, 33, "K*r <= 128"),
          (16, 2, 1, 129, "K*r <= 128"))


@pytest.mark.parametrize("d,L,K,r,bound", BOUNDS)
def test_entries_refuse_shapes_past_the_bounds(d, L, K, r, bound):
    from recalgorithm_b200 import _lib
    h = _lib.lib()
    buf = torch.zeros(1 << 16, device="cuda")
    P = buf.data_ptr()
    n, s = ctypes.c_int64(0), ctypes.c_int64(0)
    calls = {"ctr_cross_mix_workspace_bytes": lambda: h.ctr_cross_mix_workspace_bytes(4, d, L, K, r, ctypes.byref(n),
                                                                                      ctypes.byref(s)),
             "ctr_cross_mix_fwd": lambda: h.ctr_cross_mix_fwd(P, P, P, P, P, P, 4, d, L, K, r, 1, P, P, P,
                                                              buf.numel() * 4, None),
             "ctr_cross_mix_bwd": lambda: h.ctr_cross_mix_bwd(P, P, P, P, P, P, P, P, 4, d, L, K, r, 1, P, P, P, P, P, P,
                                                              P, buf.numel() * 4, None)}
    for entry, call in calls.items():
        assert call() == _lib.CTR_ERR_UNSUPPORTED, entry
        msg = h.ctr_last_error().decode()
        assert msg.startswith(entry) and bound in msg, msg
    torch.cuda.synchronize()


def test_short_workspace_short_saved_and_cpu_tensors_are_refused():
    from recalgorithm_b200 import _lib, ops
    h = _lib.lib()
    n, s = ctypes.c_int64(0), ctypes.c_int64(0)
    B, d, L, K, r = 4, 33, 2, 3, 5
    assert h.ctr_cross_mix_workspace_bytes(B, d, L, K, r, ctypes.byref(n), ctypes.byref(s)) == 0
    assert s.value == B * ((2 * L - 1) * d + L * (2 * K * r + K)) * 4
    buf = torch.zeros(int(n.value) // 4 + 64, device="cuda")
    P = buf.data_ptr()
    assert h.ctr_cross_mix_bwd(P, P, P, P, P, P, P, P, B, d, L, K, r, 1, P, P, P, P, P, P, P, int(n.value) - 128,
                               None) == _lib.CTR_ERR_INVALID_ARG
    assert "workspace" in h.ctr_last_error().decode()
    assert h.ctr_cross_mix_workspace_bytes(0, d, L, K, r, ctypes.byref(n), ctypes.byref(s)) == 0
    assert h.ctr_cross_mix_fwd(P, P, P, P, P, P, B, d, L, K, r, 1, P, P, P, int(n.value) - 128, None) == \
        _lib.CTR_ERR_INVALID_ARG
    assert "workspace" in h.ctr_last_error().decode()
    assert h.ctr_cross_mix_fwd(P, P, P, P, P, P, B, d, L, K, r, 2, P, P, P, buf.numel() * 4, None) == \
        _lib.CTR_ERR_INVALID_ARG
    assert "activation" in h.ctr_last_error().decode()
    x0, v, c, u, b, gate, g = _inputs(B, d, L, K, r, 2)
    args = [dev(t) for t in (x0, v, c, u, b, gate)]
    out, saved = ops.cross_mix_fwd(*args)
    with pytest.raises(ValueError, match="saved"):
        ops.cross_mix_bwd(*args, saved[:-4], dev(g))
    with pytest.raises(ValueError, match="saved"):
        ops.cross_mix_fwd(*args, saved=saved[:-4])
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.cross_mix_fwd(*(torch.from_numpy(t) for t in (x0, v, c, u, b, gate)))
    torch.cuda.synchronize()


def test_forward_and_backward_replay_in_a_cuda_graph():
    from recalgorithm_b200 import ops
    x0, v, c, u, b, gate, g = _inputs(1000, 82, 3, 4, 32, 13)
    args = [dev(t) for t in (x0, v, c, u, b, gate)]
    gt = dev(g)

    def step():
        out, saved = ops.cross_mix_fwd(*args)
        return (out, *ops.cross_mix_bwd(*args, saved, gt))
    eager = step()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize()
    for k in range(2):                        # out, dx0: per-sample rows, bitwise
        assert torch.equal(captured[k], eager[k]), k
    for a, c_ in zip(captured[2:], eager[2:]):  # fp32 atomics across CTAs: the weight gradients' order of adds may differ
        assert_close(a, c_.double(), TOL, "graph weight gradient", elementwise=2.0)


_PROFILE = """
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, "tests")
from _util import dev
from test_gpu_dcnmix import _inputs
from recalgorithm_b200 import autograd
for act in ("tanh", "identity"):
    x0, v, c, u, b, gate, g = _inputs(512, 480, 3, 4, 32, 4)
    ts = [dev(t).requires_grad_(True) for t in (x0, v, c, u, b, gate)]
    gd = dev(g)
    autograd.cross_mix(*ts, act).backward(gd)          # first launches outside the trace
    torch.cuda.synchronize()
    for t in ts:
        t.grad = None
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        autograd.cross_mix(*ts, act).backward(gd)
        torch.cuda.synchronize()
    print(json.dumps([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]))
"""


def test_profiler_sees_only_the_new_kernels():
    """The autograd forward and backward launch the DCN-Mix kernels and nothing else (memsets aside), for both
    activations.  The trace is taken in a process of its own, so that this profiler session leaves the test process's
    profiler as it was."""
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


def test_three_layer_network_through_layers_matches_float64():
    from recalgorithm_b200 import layers as L
    B, d, K, r = 300, 82, 4, 16
    x = np.random.default_rng(7).standard_normal((B, d)).astype(np.float32)
    store = L.set_default_store(L.VariableStore(device="cuda", seed=3))
    try:
        with L.variable_scope("net"):
            out = L.cross_network_mix(dev(x), 3, num_experts=K, low_rank=r)
        vs = {k: t.detach().cpu().numpy() for k, t in store.vars.items()}
    finally:
        L.set_default_store(L.VariableStore(device="cpu"))
    st = lambda n: np.stack([np.stack([vs[f"net/cross_mix_{l}/expert_{i}/{n}"] for i in range(K)]) for l in range(3)])
    b = np.stack([vs[f"net/cross_mix_{l}/bias"] for l in range(3)])
    ref, _ = cross_mix_fwd(x, st("kernel_v"), st("kernel_c"), st("kernel_u"), b, vs["net/cross_mix_gates/kernel"], 1)
    assert_close(out, ref, TOL, "three DCN-Mix layers")


@pytest.mark.parametrize("structure", ["stacked", "parallel"])
def test_model_body_reaches_the_tables_and_every_variable(structure):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import model_bodies as M
    from recalgorithm_b200 import autograd, layers as L
    B, F, D, rows, n_dense, K = 64, 5, 16, 100, 2, 3
    rng = np.random.default_rng(9)
    store = L.set_default_store(L.VariableStore(device="cuda", seed=5))
    try:
        tables = autograd.EmbeddingTables([rows] * F, D, device="cuda")
        ids = torch.from_numpy(rng.integers(0, rows, (B, F))).cuda()
        cat = autograd.lookup(tables, ids).reshape(B, F * D)
        dense_in = dev(rng.standard_normal((B, n_dense)).astype(np.float32))
        logit = M.dcn_v2_logit(dense_in, cat, num_cross_layer=3, projection_dim=8, structure=structure, num_experts=K)
        assert logit.shape == (B, 1)
        logit.sum().backward()
        assert tables.grad_slices and all(torch.isfinite(gs.values).all() for gs in tables.grad_slices)
        assert any(torch.count_nonzero(gs.values) > 0 for gs in tables.grad_slices)
        want = {f"cross_part/cross_mix_{l}/expert_{i}/{n}" for l in range(3) for i in range(K)
                for n in ("kernel_v", "kernel_c", "kernel_u")}
        want |= {f"cross_part/cross_mix_{l}/bias" for l in range(3)} | {"cross_part/cross_mix_gates/kernel"}
        assert want <= set(store.vars)
        for name, v in store.vars.items():
            assert v.grad is not None and torch.isfinite(v.grad).all() and torch.count_nonzero(v.grad) > 0, name
    finally:
        L.set_default_store(L.VariableStore(device="cpu"))
