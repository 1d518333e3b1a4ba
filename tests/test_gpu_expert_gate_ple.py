"""GPU parity: PLE's extraction network and final experts and gates (csrc/ple.cu) against the reference-executed fixtures
(tests/golden/ple) and the float64 restatement with its analytic backward (tests/_ple_ref.py).

The file name sorts before test_gpu_layer_variants.py for the reason test_gpu_expert_gate_mmoe.py gives: the launch-order
checks there trace with torch.profiler in the test process and lose kernels once enough idle time has passed since the
process's first profiler session.  This file's own trace is taken in a subprocess."""
import glob
import os
import sys

import numpy as np
import pytest
import torch

import _ple_ref as R
from _util import GOLDEN, TOL, assert_close, dev
from test_gpu_layer_variants import CHUNK, check_reduced

pytestmark = pytest.mark.gpu

FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "ple", "*.npz")))
KERNELS = ("ple_prep_kernel", "ple_fwd_wgmma_kernel", "ple_bwd_dz_wgmma_kernel", "ple_bwd_dx_wgmma_kernel",
           "ple_bwd_dw_wgmma_kernel")
TASKS = ("read_comment", "like", "click_avatar", "forward")


def _gc(n, S, extraction):
    return sum(n) + len(n) * S + ((sum(n) + S) if extraction else 0)


def _inputs(B, d, H, n, S, extraction, seed, gate_scale=1.0):
    """x (B,d), (w_experts, b_experts, w_gates) and g (shaped as out) in float32.  Samples whose expert pre-activation lies
    within 1e-6 of 0, relative to the sum of the magnitudes of its terms, are redrawn: float32 may take the other side of
    the relu there, which is not a kernel error."""
    rng = np.random.default_rng(seed)
    E = sum(n) + S
    we = (rng.uniform(-1, 1, (E, d, H)) * (6.0 / (d + H)) ** 0.5).astype(np.float32)
    be = rng.uniform(-0.1, 0.1, (E, H)).astype(np.float32)
    GC = _gc(n, S, extraction)
    wg = (rng.uniform(-1, 1, (d, GC)) * (6.0 / (d + GC)) ** 0.5 * gate_scale).astype(np.float32)
    x = (rng.standard_normal((B, d)) * 0.7).astype(np.float32)
    we64, be64 = dev(we, torch.float64), dev(be, torch.float64)
    rows = np.arange(B)
    for _ in range(100):
        x64 = dev(x[rows], torch.float64)
        a = x64 @ we64 + be64[:, None, :]
        scale = x64.abs() @ we64.abs() + be64.abs()[:, None, :]
        rows = rows[(a.abs() <= 1e-6 * scale).any(dim=2).any(dim=0).cpu().numpy()]
        if rows.size == 0:
            break
        x[rows] = (rng.standard_normal((rows.size, d)) * 0.7).astype(np.float32)
    else:
        raise AssertionError("could not draw inputs away from the relu edges")
    g = rng.standard_normal((B, H) if extraction else (len(n), B, H)).astype(np.float32)
    return x, (we, be, wg), g


def _run(x, p, g, n, S, extraction):
    from recalgorithm_b200 import ops
    args = [dev(t) for t in (x, *p)]
    out, gates = ops.ple_fwd(*args, n, S, extraction)
    grads = ops.ple_bwd(*args, gates, dev(g), n, S, extraction)
    return out, gates, grads


def _reduced(x, dz, dlogit, group=128):
    """Each batch-reduced gradient as (sum over the batch, sum over CHUNK-sample chunks of |chunk sum|): the bar of
    test_gpu_layer_variants.check_reduced (the batch is zero padded to whole chunks; a padded sample adds nothing)."""
    B, d = x.shape
    nc = max(1, -(-B // CHUNK))
    pad = nc * CHUNK - B
    xc = torch.nn.functional.pad(x, (0, 0, 0, pad)).view(nc, CHUNK, d)
    dzc = torch.nn.functional.pad(dz, (0, 0, 0, pad)).view(dz.shape[0], nc, CHUNK, -1)
    dlc = torch.nn.functional.pad(dlogit, (0, 0, 0, pad)).view(nc, CHUNK, -1)
    red = {k: [0.0, 0.0] for k in ("dwe", "dbe", "dwg")}
    for c0 in range(0, nc, group):
        sl = slice(c0, min(nc, c0 + group))
        parts = {"dwe": torch.einsum("cbd,ecbh->cedh", xc[sl], dzc[:, sl]), "dbe": dzc[:, sl].sum(2).transpose(0, 1),
                 "dwg": torch.einsum("cbd,cbg->cdg", xc[sl], dlc[sl])}
        for k, v in parts.items():
            red[k][0] = red[k][0] + v.sum(0)
            red[k][1] = red[k][1] + v.abs().sum(0)
    return {k: (v[0].cpu().numpy(), v[1].cpu().numpy()) for k, v in red.items()}


def _check(x, p, g, n, S, extraction, out, gates, grads):
    what = f"B={x.shape[0]} d={x.shape[1]} H={p[0].shape[2]} n={tuple(n)} S={S} extraction={extraction}"
    ts = [dev(t, torch.float64) for t in (x, *p, g)]
    r_out, r_gates, _ = R.fwd(*ts[:4], n, S, extraction)
    assert_close(out, r_out.cpu().numpy(), TOL, f"out {what}")
    assert_close(gates, r_gates.cpu().numpy(), TOL, f"gates {what}")
    d_x, _, _, _, dz, dlogit = R.bwd(*ts, n, S, extraction)
    assert_close(grads[0], d_x.cpu().numpy(), TOL, f"d_x {what}")
    red = _reduced(ts[0], dz, dlogit)
    for name, got in zip(("dwe", "dbe", "dwg"), grads[1:]):
        check_reduced(got, red[name], f"{name} {what}")


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_through_ops_and_layers(name):
    """Forward and backward through ops against float64 and the reference's own float64 run, then the block through layers
    with the fixture's weights assigned under the reference's names."""
    from recalgorithm_b200 import layers as L
    z = np.load(os.path.join(GOLDEN, "ple", name + ".npz"), allow_pickle=False)
    arrays, (n, S, extraction) = R.fixture(z)
    x = arrays[0].float().numpy()
    p = [a.float().numpy() for a in arrays[1:]]
    H = p[0].shape[2]
    g = np.random.default_rng(7).standard_normal(z["out_f64"].shape).astype(np.float32)
    out, gates, grads = _run(x, p, g, n, S, extraction)
    _check(x, p, g, n, S, extraction, out, gates, grads)
    assert_close(out, z["out_f64"], TOL, f"{name}: out vs reference (float64)")

    store = L.set_default_store(L.VariableStore(device="cuda", seed=0))
    xt = dev(x).requires_grad_(True)
    tasks = TASKS[:len(n)]
    layer = ((lambda: [L.extraction_network(xt, tasks, n, S, H, "extract_network_0")]) if extraction else
             (lambda: L.ple_final_experts_gates(xt, tasks, n, S, H)))
    layer()
    names = [str(v) for v in z["variables"]]
    assert list(store.vars) == names
    kernels = [v for v in names if v.endswith("kernel")]
    experts = [v[:-len("/kernel")] for v in kernels if "gate" not in v]
    order = [e for e in experts if "task_specific" in e] + [e for e in experts if "shared" in e]
    gate_names = [v for v in kernels if "gate" in v]
    gate_names = [v for v in gate_names if "all_gate" not in v] + [v for v in gate_names if "all_gate" in v]
    widths = [len(e) for e in R.gate_experts(n, S, extraction)]
    cols = np.cumsum([0] + widths)
    store.assign({**{f"{e}/kernel": p[0][i] for i, e in enumerate(order)},
                  **{f"{e}/bias": p[1][i] for i, e in enumerate(order)},
                  **{nm: p[2][:, cols[k]:cols[k + 1]] for k, nm in enumerate(gate_names)}})
    outs = layer()
    want = z["out_f64"] if not extraction else z["out_f64"][None]
    assert all(o.is_contiguous() and o.shape == want.shape[1:] for o in outs)
    for t, o in enumerate(outs):
        assert_close(o, want[t], TOL, f"{name}: layers out {t}")
    gl = g if not extraction else g[None]
    sum((o * dev(gl[t])).sum() for t, o in enumerate(outs)).backward()
    r = R.bwd(*(dev(t, torch.float64) for t in (x, *p, g)), n, S, extraction)
    assert_close(xt.grad, r[0].cpu().numpy(), TOL, f"{name}: layers d_x")
    for i, e in enumerate(order):
        assert_close(store.vars[f"{e}/kernel"].grad, r[1][i].cpu().numpy(), TOL, f"{name}: d {e}", elementwise=False)
        assert_close(store.vars[f"{e}/bias"].grad, r[2][i].cpu().numpy(), TOL, f"{name}: d {e} bias", elementwise=False)
    for k, nm in enumerate(gate_names):
        assert_close(store.vars[nm].grad, r[3][:, cols[k]:cols[k + 1]].cpu().numpy(), TOL, f"{name}: d {nm}",
                     elementwise=False)


# (n, S) sets: one task with one expert each, the reference row, and sets at the bounds (E = 64 for the final layer,
# GC = 160 for the extraction network)
SETS = {False: (((1,), 1), ((5, 5, 5), 10), ((12, 12, 12, 12), 16)),
        True: (((1,), 1), ((5, 5, 5), 10), ((10, 10, 10, 10), 16))}
DS = (1, 31, 32, 33, 82, 127, 128, 129, 255, 256, 257, 511, 512)
HS = (1, 63, 64, 65, 512)
SHAPES = ([(129, d, H, n, S, ext) for ext in (True, False) for d in DS for H in HS for n, S in SETS[ext]] +
          [(B, 82, 256, (5, 5, 5), 10, True) for B in (0, 1, 63, 64, 65, 127, 128, 129, 1000)] +
          [(B, 256, 256, (5, 5, 5), 10, False) for B in (0, 1, 63, 64, 65, 127, 128, 129, 1000)] +
          [(65536, 82, 256, (5, 5, 5), 10, True), (65536, 256, 256, (5, 5, 5), 10, False)])


@pytest.mark.parametrize("B,d,H,n,S,extraction", SHAPES)
def test_ple_against_float64(B, d, H, n, S, extraction):
    x, p, g = _inputs(B, d, H, n, S, extraction, seed=B * 7 + d * 131 + H * 3 + sum(n) * 17 + S + extraction)
    out, gates, grads = _run(x, p, g, n, S, extraction)
    _check(x, p, g, n, S, extraction, out, gates, grads)


@pytest.mark.parametrize("extraction", [True, False])
def test_saturated_gates_do_not_overflow(extraction):
    """Gate logits near +-80 (expf would overflow float32 past 88 without the max subtracted): the gates stay finite, each
    gate sums to 1, and the forward matches float64."""
    B, d, H, n, S = 300, 82, 128, (2, 3), 2
    x, p, g = _inputs(B, d, H, n, S, extraction, seed=12)
    logits = x.astype(np.float64) @ p[2].astype(np.float64)
    p = (p[0], p[1], (p[2] * (80.0 / np.abs(logits).max())).astype(np.float32))
    out, gates, _ = _run(x, p, g, list(n), S, extraction)
    assert np.abs(x.astype(np.float64) @ p[2].astype(np.float64)).max() > 70
    assert torch.isfinite(gates).all() and torch.isfinite(out).all()
    widths = [len(e) for e in R.gate_experts(n, S, extraction)]
    for s in torch.split(gates, widths, dim=1):
        assert float((s.sum(1) - 1).abs().max()) < 1e-6
    r_out, r_gates, _ = R.fwd(*(dev(t, torch.float64) for t in (x, *p)), list(n), S, extraction)
    assert_close(out, r_out.cpu().numpy(), TOL, "saturated out")
    assert_close(gates, r_gates.cpu().numpy(), TOL, "saturated gates")


@pytest.mark.parametrize("extraction", [True, False])
def test_empty_batch_gives_zero_weight_gradients(extraction):
    from recalgorithm_b200 import ops
    n, S = [2, 1], 2
    x, p, g = _inputs(4, 82, 128, n, S, extraction, seed=1)
    args = [dev(t) for t in p]
    out, gates = ops.ple_fwd(dev(x[:0]), *args, n, S, extraction)
    g0 = g[:0] if extraction else g[:, :0]
    grads = ops.ple_bwd(dev(x[:0]), *args, gates, dev(g0), n, S, extraction)
    assert out.shape == ((0, 128) if extraction else (2, 0, 128)) and gates.shape == (0, _gc(n, S, extraction))
    assert grads[0].shape == (0, 82)
    for t in grads[1:]:
        assert t.numel() > 0 and torch.count_nonzero(t) == 0


def _abi_calls(h, P, nbytes, B, d, H, n, S, extraction):
    import ctypes
    arr = (ctypes.c_int64 * len(n))(*n)
    T = len(n)
    w = ctypes.c_int64(0)
    return {"ctr_ple_workspace_bytes": lambda: h.ctr_ple_workspace_bytes(B, d, H, T, arr, S, extraction, ctypes.byref(w)),
            "ctr_ple_fwd": lambda: h.ctr_ple_fwd(P, P, P, P, B, d, H, T, arr, S, extraction, P, P, P, nbytes, None),
            "ctr_ple_bwd": lambda: h.ctr_ple_bwd(P, P, P, P, P, P, B, d, H, T, arr, S, extraction, P, P, P, P, P, nbytes,
                                                 None)}


@pytest.mark.parametrize("d,H,n,S,extraction,bound", [
    (513, 256, (5, 5, 5), 10, 1, "d <= 512"), (82, 513, (5, 5, 5), 10, 1, "H <= 512"),
    (82, 256, (1, 1, 1, 1, 1), 1, 0, "T <= 4"), (82, 256, (20, 20, 20), 5, 0, "E <= 64"),
    (82, 256, (65,), 1, 0, "E <= 64"), (82, 256, (10, 10, 10), 26, 1, "GC <= 160")])
def test_entries_refuse_shapes_past_the_bounds(d, H, n, S, extraction, bound):
    """All three entries refuse larger shapes with CTR_ERR_UNSUPPORTED and a message naming the bound, called through the C
    ABI with small real buffers."""
    from recalgorithm_b200 import _lib
    h = _lib.lib()
    buf = torch.zeros(1 << 16, device="cuda")
    for entry, call in _abi_calls(h, buf.data_ptr(), buf.numel() * 4, 4, d, H, n, S, extraction).items():
        assert call() == _lib.CTR_ERR_UNSUPPORTED, entry
        msg = h.ctr_last_error().decode()
        assert msg.startswith(entry) and bound in msg, msg
    torch.cuda.synchronize()


def test_bad_counts_are_refused():
    from recalgorithm_b200 import _lib
    h = _lib.lib()
    buf = torch.zeros(1 << 16, device="cuda")
    for n, S, ext in (((5, 0, 5), 10, 0), ((5, 5, 5), 0, 1), ((5, 5, 5), 10, 2)):
        for entry, call in _abi_calls(h, buf.data_ptr(), buf.numel() * 4, 4, 82, 256, n, S, ext).items():
            assert call() == _lib.CTR_ERR_INVALID_ARG, entry
            assert h.ctr_last_error().decode().startswith(entry)


def test_too_small_workspace_is_refused():
    from recalgorithm_b200 import _lib, ops
    h = _lib.lib()
    B, d, H, n, S = 64, 82, 256, (5, 5, 5), 10
    need_fwd = ops.ple_workspace(0, d, H, n, S, True, "cuda").numel()
    need_bwd = ops.ple_workspace(B, d, H, n, S, True, "cuda").numel()
    assert need_bwd > need_fwd
    buf = torch.zeros(need_bwd // 4 + 64, device="cuda")
    calls = _abi_calls(h, buf.data_ptr(), 1024, B, d, H, n, S, 1)
    assert calls["ctr_ple_fwd"]() == _lib.CTR_ERR_INVALID_ARG
    assert h.ctr_last_error().decode().startswith("ctr_ple_fwd: workspace")
    calls = _abi_calls(h, buf.data_ptr(), need_bwd - 128, B, d, H, n, S, 1)
    assert calls["ctr_ple_bwd"]() == _lib.CTR_ERR_INVALID_ARG
    assert h.ctr_last_error().decode().startswith("ctr_ple_bwd: workspace")
    torch.cuda.synchronize()


def test_cpu_tensors_are_refused():
    from recalgorithm_b200 import ops
    x, p, g = _inputs(4, 8, 16, [1, 1], 1, True, seed=2)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.ple_fwd(*(torch.from_numpy(t) for t in (x, *p)), [1, 1], 1, True)


_PROFILE = """
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile
from recalgorithm_b200 import ops
gen = torch.Generator(device="cuda").manual_seed(4)
n, S = (5, 5, 5), 10
runs = []
for d, ext, gc in ((82, True, 70), (256, False, 45)):
    args = [torch.randn(s, device="cuda", generator=gen) * 0.1 for s in ((1024, d), (25, d, 256), (25, 256), (d, gc))]
    gd = torch.randn((1024, 256) if ext else (3, 1024, 256), device="cuda", generator=gen)
    ops.ple_bwd(*args, ops.ple_fwd(*args, n, S, ext)[1], gd, n, S, ext)     # first launches (module load) outside the trace
    runs.append((args, gd, ext))
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for args, gd, ext in runs:
        out, gates = ops.ple_fwd(*args, n, S, ext)
        ops.ple_bwd(*args, gates, gd, n, S, ext)
    torch.cuda.synchronize()
print(json.dumps([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]))
"""


def test_profiler_sees_only_the_new_kernels():
    """Forward and backward of both blocks launch the PLE kernels and nothing else: no torch kernel touches the expert
    tensor.  The trace is taken in a process of its own, so that this profiler session leaves the test process's profiler
    as it was."""
    import json
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    run = subprocess.run([sys.executable, "-c", _PROFILE], cwd=root, capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr[-3000:]
    names = json.loads(run.stdout.strip().splitlines()[-1])
    kernels = [n for n in names if not n.startswith("Memset")]
    assert kernels and all(any(k in n for k in KERNELS) for n in kernels), sorted(set(kernels))
    for k in KERNELS:
        assert any(k in n for n in kernels), k
    for k in KERNELS[1:]:
        assert sum(k in n for n in kernels) == 2, k
    assert sum("ple_prep_kernel" in n for n in kernels) == 4


def test_ple_logits_training_step():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import model_bodies as M
    from recalgorithm_b200 import layers as L
    B, tasks = 256, TASKS[:3]
    store = L.set_default_store(L.VariableStore(device="cuda", seed=5))
    gen = torch.Generator(device="cuda").manual_seed(5)
    dense_input = torch.randn(B, 16, device="cuda", generator=gen).requires_grad_(True)
    cat = torch.randn(B, 66, device="cuda", generator=gen).requires_grad_(True)
    labels = {t: (torch.rand((B, 1), device="cuda", generator=gen) < 0.3).float() for t in tasks}
    kw = dict(num_extract_network=1, num_experts_per_task=(2, 2, 2), num_experts_in_shared=3, expert_hidden_units=64,
              hidden_units=(64, 32))
    logits, loss = M.ple_logits(dense_input, cat, labels, tasks, **kw)
    assert len(logits) == 3 and all(lg.shape == (B, 1) for lg in logits) and torch.isfinite(loss)
    opt = torch.optim.SGD(store.parameters(), lr=0.1)
    opt.zero_grad()
    loss.backward()
    assert any(v.startswith("extract_network_0/all_gate") for v in store.vars)
    assert any(v.startswith("task_specific_experts_final/task_gate_final/gate_final_like") for v in store.vars)
    assert any(v.startswith("tower/tower_click_avatar_logit") for v in store.vars)
    for n, v in store.vars.items():
        assert v.grad is not None and torch.isfinite(v.grad).all() and torch.count_nonzero(v.grad) > 0, n
    assert float(dense_input.grad.abs().max()) > 0 and float(cat.grad.abs().max()) > 0
    opt.step()
    with torch.no_grad():
        loss2 = M.ple_logits(dense_input, cat, labels, tasks, **kw)[1]
    assert torch.isfinite(loss2) and float(loss2) < float(loss.detach())
