"""GPU parity: the AutoInt interacting layer (csrc/autoint.cu) against the float64 restatement of the paper's equations
(tests/_autoint_ref.py) -- forward, every gradient, exact cases, refusals, the launches autograd makes, and the host layer
and model body."""
import os
import re
import sys

import numpy as np
import pytest
import torch

from _autoint_ref import interacting_bwd, interacting_fwd, model_logit
from _util import TOL, assert_close, dev

pytestmark = pytest.mark.gpu

# the weight gradients run tc_ptx.cuh's shared kernel; its autoint:: Rows type marks this layer's instantiations
DW_KERNEL = r"weight_grad_wgmma_kernel<[^,]+, ctr::autoint::"
KERNELS = ("autoint_prep_kernel", "autoint_fwd_wgmma_kernel", "autoint_bwd_attn_wgmma_kernel", "autoint_bwd_dx_wgmma_kernel",
           DW_KERNEL)


def _inputs(B, F, d, H, dk, seed, scale=1.0):
    """x, weights and g_out in float32; samples whose pre-activations come within a small margin of the relu edge are
    redrawn, since float32 may take the other side of the relu there, which is not a kernel error.  w_query and w_key are
    drawn dk**-0.25 smaller than w_value and w_res, so that the unscaled scores have unit spread at every dk: a score of
    magnitude s carries about s * 1e-7 of rounding from the float32 Q and K alone, and exp turns that into a relative error
    of the attention weights, so scores in the tens would measure float32 itself rather than the kernels against 1e-5."""
    rng = np.random.default_rng(seed)
    ws = [(rng.uniform(-1, 1, (d, H * dk)) * scale * np.sqrt(3.0 / d) * (dk ** -0.25 if i < 2 else 1.0)).astype(np.float32)
          for i in range(4)]
    x = rng.standard_normal((B, F, d)).astype(np.float32)
    rows = np.arange(B)                                  # the samples still to check: all, then only the redrawn ones
    scale = None
    for _ in range(50):
        if rows.size == 0:
            break
        pre = interacting_fwd(x[rows], *ws, H, dk)[1][5]
        scale = np.abs(pre).max(initial=1e-30) if scale is None else scale
        rows = rows[(np.abs(pre) < 1e-5 * scale).any(axis=(1, 2))]
        x[rows] = rng.standard_normal((rows.size, F, d)).astype(np.float32)
    else:
        raise AssertionError("could not draw inputs away from the relu edges")
    g = rng.standard_normal((B, F, H * dk)).astype(np.float32)
    return x, ws, g


def _run(x, ws, g, H, dk):
    from recalgorithm_b200 import ops
    args = [dev(t) for t in (x, *ws)]
    out = ops.autoint_fwd(*args, H, dk)
    grads = ops.autoint_bwd(*args, out, dev(g), H, dk)
    torch.cuda.synchronize()
    return out, grads


def _check(x, ws, g, H, dk, out, grads, what):
    ref_out, cache = interacting_fwd(x, *ws, H, dk)
    ref = interacting_bwd(cache, *ws, g.astype(np.float64), H, dk)
    assert_close(out, ref_out, TOL, f"{what}: out")
    # d_x sums the 4 H dk projection gradients of a row times the weights, and those terms cancel: its float32 error follows
    # the sum of the terms' magnitudes rather than |d_x|.  At d = 128 it reaches 1.36x the element-wise bound on the H100
    # (B=63 F=40 d=128 H=2 dk=32 and B=1000 F=64 d=128 H=1 dk=64), so that bound is doubled; the max-norm bar is unchanged.
    assert_close(grads[0], ref[0], TOL, f"{what}: d_x", elementwise=2.0)
    # the weight gradients are batch reductions over B F rows whose terms cancel: doubled element-wise bound
    for name, got, want in zip(("d_w_query", "d_w_key", "d_w_value", "d_w_res"), grads[1:], ref[1:]):
        assert_close(got, want, TOL, f"{what}: {name}", elementwise=2.0)


FS = (1, 2, 7, 39, 40, 64)
DS = (1, 5, 16, 32, 64, 82, 128)
HDK = ((1, 1), (3, 5), (2, 8), (2, 32), (1, 64), (8, 16), (4, 32))
SHAPES = ([(65, F, DS[(i + j) % len(DS)], H, dk) for i, F in enumerate(FS) for j, (H, dk) in enumerate(HDK)] +
          [(63, 40, d, 2, 32) for d in DS] + [(64, 39, d, 3, 5) for d in DS] +
          [(B, 40, 16, 2, 32) for B in (1, 63, 64, 65, 1000)] + [(1000, 39, 32, 2, 8), (1000, 64, 128, 1, 64)])


@pytest.mark.parametrize("B,F,d,H,dk", SHAPES)
def test_autoint_against_float64(B, F, d, H, dk):
    x, ws, g = _inputs(B, F, d, H, dk, seed=B * 7 + F * 131 + d * 17 + H * 5 + dk)
    out, grads = _run(x, ws, g, H, dk)
    _check(x, ws, g, H, dk, out, grads, f"B={B} F={F} d={d} H={H} dk={dk}")


def test_paper_shape_at_full_batch():
    B, F, d, H, dk = 65536, 40, 16, 2, 32
    x, ws, g = _inputs(B, F, d, H, dk, seed=11)
    out, grads = _run(x, ws, g, H, dk)
    _check(x, ws, g, H, dk, out, grads, "paper shape B=65536")


def test_empty_batch_gives_zero_weight_gradients():
    x, ws, g = _inputs(3, 7, 5, 3, 5, seed=1)
    out, grads = _run(x[:0], ws, g[:0], 3, 5)
    assert out.shape == (0, 7, 15) and grads[0].shape == (0, 7, 5)
    for t in grads[1:]:
        assert t.numel() > 0 and torch.count_nonzero(t) == 0


def test_single_field_gives_exact_zero_query_and_key_gradients():
    x, ws, g = _inputs(300, 1, 16, 2, 8, seed=2)
    out, grads = _run(x, ws, g, 2, 8)
    assert torch.count_nonzero(grads[1]) == 0 and torch.count_nonzero(grads[2]) == 0
    _check(x, ws, g, 2, 8, out, grads, "F=1")


def test_all_negative_preactivations_give_exact_zero_gradients():
    B, F, d, H, dk = 64, 10, 8, 2, 4
    rng = np.random.default_rng(3)
    x = np.abs(rng.standard_normal((B, F, d))).astype(np.float32)
    ws = [np.zeros((d, H * dk), np.float32) for _ in range(3)] + [-np.abs(rng.standard_normal((d, H * dk))).astype(np.float32)]
    g = rng.standard_normal((B, F, H * dk)).astype(np.float32)
    out, grads = _run(x, ws, g, H, dk)
    assert torch.count_nonzero(out) == 0
    for t in grads:
        assert torch.count_nonzero(t) == 0


def test_large_scores_stay_finite():
    """Scores near +-80: the row max is subtracted before exp, so nothing overflows."""
    B, F, d, H, dk = 32, 12, 4, 1, 4
    rng = np.random.default_rng(4)
    x = rng.choice([-1.0, 1.0], (B, F, d)).astype(np.float32)
    wq = np.full((d, dk), 2.0, np.float32); wk = np.full((d, dk), 1.25, np.float32)   # |score| up to 4*4*2*1.25*... = 80
    ws = [wq / 2, wk / 2 * 2, rng.standard_normal((d, dk)).astype(np.float32), rng.standard_normal((d, dk)).astype(np.float32)]
    g = rng.standard_normal((B, F, dk)).astype(np.float32)
    _, cache = interacting_fwd(x, *ws, H, dk)
    s = np.einsum("bhik,bhjk->bhij", cache[1], cache[2])
    assert np.abs(s).max() >= 70
    out, grads = _run(x, ws, g, H, dk)
    for t in (out, *grads):
        assert torch.isfinite(t).all()


def test_batch_permutation_and_repeat_are_bitwise():
    B, F, d, H, dk = 200, 39, 16, 2, 32
    x, ws, g = _inputs(B, F, d, H, dk, seed=5)
    out, grads = _run(x, ws, g, H, dk)
    out2, grads2 = _run(x, ws, g, H, dk)
    assert torch.equal(out, out2) and torch.equal(grads[0], grads2[0])
    perm = np.random.default_rng(6).permutation(B)
    outp, gradsp = _run(x[perm], ws, g[perm], H, dk)
    inv = torch.from_numpy(np.argsort(perm)).cuda()
    assert torch.equal(outp[inv], out) and torch.equal(gradsp[0][inv], grads[0])


BOUNDS = ((65, 8, 2, 8, "F <= 64"), (8, 129, 2, 8, "d <= 128"), (8, 8, 1, 65, "dk <= 64"), (8, 8, 9, 8, "H <= 8"),
          (8, 8, 5, 26, "H*dk <= 128"))


@pytest.mark.parametrize("F,d,H,dk,bound", BOUNDS)
def test_entries_refuse_shapes_past_the_bounds(F, d, H, dk, bound):
    import ctypes
    from recalgorithm_b200 import _lib
    h = _lib.lib()
    buf = torch.zeros(1 << 16, device="cuda")
    P = buf.data_ptr()
    n = ctypes.c_int64(0)
    calls = {"ctr_autoint_workspace_bytes": lambda: h.ctr_autoint_workspace_bytes(4, F, d, H, dk, ctypes.byref(n)),
             "ctr_autoint_fwd": lambda: h.ctr_autoint_fwd(P, P, P, P, P, 4, F, d, H, dk, P, P, buf.numel() * 4, None),
             "ctr_autoint_bwd": lambda: h.ctr_autoint_bwd(P, P, P, P, P, P, P, 4, F, d, H, dk, P, P, P, P, P, P,
                                                          buf.numel() * 4, None)}
    for entry, call in calls.items():
        assert call() == _lib.CTR_ERR_UNSUPPORTED, entry
        msg = h.ctr_last_error().decode()
        assert msg.startswith(entry) and bound in msg, msg
    torch.cuda.synchronize()


def test_small_workspace_and_cpu_tensors_are_refused():
    import ctypes
    from recalgorithm_b200 import _lib, ops
    h = _lib.lib()
    n = ctypes.c_int64(0)
    assert h.ctr_autoint_workspace_bytes(4, 7, 5, 3, 5, ctypes.byref(n)) == 0
    buf = torch.zeros(int(n.value) // 4 + 64, device="cuda")
    P = buf.data_ptr()
    assert h.ctr_autoint_bwd(P, P, P, P, P, P, P, 4, 7, 5, 3, 5, P, P, P, P, P, P, int(n.value) - 128, None) == \
        _lib.CTR_ERR_INVALID_ARG
    assert "workspace" in h.ctr_last_error().decode()
    x, ws, g = _inputs(4, 7, 5, 3, 5, seed=2)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.autoint_fwd(*(torch.from_numpy(t) for t in (x, *ws)), 3, 5)


_PROFILE = """
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, "tests")
from _util import dev
from test_gpu_autoint import _inputs
from recalgorithm_b200 import autograd
x, ws, g = _inputs(512, 40, 16, 2, 32, seed=4)
xt = dev(x).requires_grad_(True)
wt = [dev(w).requires_grad_(True) for w in ws]
gd = dev(g)
autograd.autoint_interacting(xt, *wt, 2, 32).backward(gd)      # first launches (module load) outside the trace
torch.cuda.synchronize()
for t in (xt, *wt):
    t.grad = None
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    autograd.autoint_interacting(xt, *wt, 2, 32).backward(gd)
    torch.cuda.synchronize()
print(json.dumps([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]))
"""


def test_profiler_sees_only_the_new_kernels():
    """The autograd forward and backward launch the AutoInt kernels and nothing else (memsets aside).  The trace is taken in
    a process of its own, so that this profiler session leaves the test process's profiler as it was."""
    import json
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    run = subprocess.run([sys.executable, "-c", _PROFILE], cwd=root, capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr[-3000:]
    names = json.loads(run.stdout.strip().splitlines()[-1])
    kernels = [n for n in names if not n.startswith("Memset")]
    assert kernels and all(any(re.search(k, n) for k in KERNELS) for n in kernels), sorted(set(kernels))
    for k in KERNELS:
        assert any(re.search(k, n) for n in kernels), k
    assert sum("autoint_fwd_wgmma_kernel" in n for n in kernels) == 1


def test_three_layer_stack_through_layers_matches_float64():
    from recalgorithm_b200 import layers as L
    B, F, d, H, dk = 96, 39, 32, 2, 8
    rng = np.random.default_rng(7)
    x = rng.standard_normal((B, F, d)).astype(np.float32)
    store = L.set_default_store(L.VariableStore(device="cuda", seed=3))
    try:
        with L.variable_scope("autoint"):
            net = dev(x)
            for i in range(3):
                net = L.interacting_layer(net, dk, H, index=i)
        layers = [[store.vars[f"autoint/interacting_layer_{i}/{n}"].detach().cpu().numpy() for n in
                   ("query", "key", "value", "res")] for i in range(3)]
    finally:
        L.set_default_store(L.VariableStore(device="cpu"))
    ref = x.astype(np.float64)
    for w in layers:
        ref, _ = interacting_fwd(ref, *w, H, dk)
    # each layer's float32 output is the next layer's input, so three layers' roundings compound: the stack reaches 1.30x
    # the element-wise bound on the H100, so that bound is doubled; the max-norm bar is unchanged
    assert_close(net, ref, TOL, "three interacting layers", elementwise=2.0)


def test_model_body_and_one_adam_step_match_float64():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import model_bodies as M
    from recalgorithm_b200 import layers as L
    B, n_dense, F_cat, D = 64, 3, 10, 16
    rng = np.random.default_rng(8)
    dense = rng.standard_normal((B, n_dense)).astype(np.float32)
    fields = rng.standard_normal((B, F_cat, D)).astype(np.float32)
    store = L.set_default_store(L.VariableStore(device="cuda", seed=5))
    try:
        logit = M.autoint_logit(dev(dense), dev(fields), att_layer_num=3, att_head_num=2, att_embedding_size=8)
        names = sorted(store.vars)
        vals = {n: store.vars[n].detach().cpu().numpy().astype(np.float64) for n in names}

        def ref_logit(v):
            layers = [[v[f"interacting_layer_{i}/{n}"] for n in ("query", "key", "value", "res")] for i in range(3)]
            dn = [n for n in names if "interacting_layer" not in n and n not in ("dense/kernel", "dense/bias")]
            return model_logit(dense, fields, v[dn[0]], layers, v["dense/kernel"], v["dense/bias"], 2, 8)
        assert_close(logit, ref_logit(vals), TOL, "autoint_logit")
        # the gradients of sum(logit) against float64 autograd of the same body, then one Adam step from them
        params = [store.vars[n] for n in names]
        logit.sum().backward()
        tv = {n: torch.tensor(vals[n], requires_grad=True) for n in names}
        _torch_logit(dense, fields, tv, names).sum().backward()
        for n in names:
            # batch-reduced weight gradients (sums over B F rows whose terms cancel): doubled element-wise bound
            assert_close(store.vars[n].grad, tv[n].grad.numpy(), TOL, f"gradient {n}", elementwise=2.0)
        opt = torch.optim.Adam(params, lr=1e-2)
        opt.step()
        ref_opt = torch.optim.Adam(list(tv.values()), lr=1e-2)
        ref_opt.step()
        for n in names:
            assert_close(store.vars[n], tv[n].detach().numpy(), TOL, f"Adam step {n}")
    finally:
        L.set_default_store(L.VariableStore(device="cpu"))


def _torch_logit(dense, fields, tv, names):
    dn = [n for n in names if "interacting_layer" not in n and n not in ("dense/kernel", "dense/bias")][0]
    net = torch.cat([torch.tensor(dense, dtype=torch.float64)[:, :, None] * tv[dn][None],
                     torch.tensor(fields, dtype=torch.float64)], dim=1)
    B, F, _ = net.shape
    for i in range(3):
        wq, wk, wv, wr = (tv[f"interacting_layer_{i}/{n}"] for n in ("query", "key", "value", "res"))
        heads = lambda t: t.reshape(B, F, 2, 8).transpose(1, 2)
        a = torch.softmax(heads(net @ wq) @ heads(net @ wk).transpose(-1, -2), dim=-1)
        net = torch.relu((a @ heads(net @ wv)).transpose(1, 2).reshape(B, F, 16) + net @ wr)
    return net.reshape(B, -1) @ tv["dense/kernel"] + tv["dense/bias"]
