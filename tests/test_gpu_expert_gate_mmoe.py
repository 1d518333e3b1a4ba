"""GPU parity: MMoE's expert-gate layer (csrc/mmoe.cu) against the reference-executed fixtures (tests/golden/mmoe) and the
float64 restatement with its analytic backward (tests/_mmoe_ref.py).

The file name sorts before test_gpu_layer_variants.py on purpose.  The launch-order checks of test_gpu_layer_variants.py and
test_gpu_tc_variants.py trace with torch.profiler inside the test process, and the later ones lose the first kernels of
their trace once enough time has passed since the process's first profiler session: an idle 28 s pause between the two
files makes 45 of them fail, with no MMoE test in the run.  These tests take about that long, so they run before the
first session, where the time they add does not matter."""
import glob
import os
import re
import sys

import numpy as np
import pytest
import torch

import _mmoe_ref as R
from _util import GOLDEN, TOL, assert_close, dev
from test_gpu_layer_variants import CHUNK, check_reduced

pytestmark = pytest.mark.gpu

FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "mmoe", "*.npz")))
# the weight gradients run tc_ptx.cuh's shared kernel; its mmoe:: Rows type marks this layer's instantiations
DW_KERNEL = r"weight_grad_wgmma_kernel<[^,]+, ctr::mmoe::"
KERNELS = ("mmoe_prep_kernel", "mmoe_fwd_wgmma_kernel", "mmoe_bwd_dx_wgmma_kernel", DW_KERNEL)


def _f32(*arrays):
    return [np.asarray(a, np.float32) for a in arrays]


def _weights(rng, d, E, H, T, gate_scale=1.0):
    we = rng.uniform(-1, 1, (E, d, H)) * (6.0 / (d + H)) ** 0.5
    be = rng.uniform(-0.1, 0.1, (E, H))
    wg = rng.uniform(-1, 1, (T, d, E)) * (6.0 / (d + E)) ** 0.5 * gate_scale
    return _f32(we, be, wg)


def _inputs(B, d, E, H, T, seed, weights=None):
    """x (B,d), weights and g (T,B,H) in float32.  Samples whose expert pre-activation lies within 1e-6 of 0, relative to the
    sum of the magnitudes of its terms, are redrawn: float32 may take the other side of the relu there, which is not a kernel
    error."""
    rng = np.random.default_rng(seed)
    p = weights if weights is not None else _weights(rng, d, E, H, T)
    we64, be64 = np.asarray(p[0], np.float64), np.asarray(p[1], np.float64)
    x = _f32(rng.standard_normal((B, d)) * 0.7)[0]
    we64, be64 = dev(we64), dev(be64)
    rows = np.arange(B)                                  # the samples still to check: all, then only the redrawn ones
    for _ in range(100):
        x64 = dev(x[rows], torch.float64)                # float64 on the GPU: NumPy takes seconds at 65 536 samples
        a = x64 @ we64 + be64[:, None, :]
        scale = x64.abs() @ we64.abs() + be64.abs()[:, None, :]
        rows = rows[(a.abs() <= 1e-6 * scale).any(dim=2).any(dim=0).cpu().numpy()]
        if rows.size == 0:
            break
        x[rows] = _f32(rng.standard_normal((rows.size, d)) * 0.7)[0]
    else:
        raise AssertionError("could not draw inputs away from the relu edges")
    g = _f32(rng.standard_normal((T, B, H)))[0]
    return x, p, g


def _run(x, p, g):
    from recalgorithm_b200 import ops
    args = [dev(t) for t in (x, *p)]
    towers, gates = ops.mmoe_fwd(*args)
    grads = ops.mmoe_bwd(*args, gates, dev(g))
    return towers, gates, grads


def _check(x, p, g, towers, gates, grads):
    B, d = x.shape
    E, _, H = p[0].shape
    T = p[2].shape[0]
    what = f"B={B} d={d} E={E} H={H} T={T}"
    per, red = R.chunked_torch(*(dev(t, torch.float64) for t in (x, *p, g)), chunk=CHUNK)
    assert_close(towers, per["towers"], TOL, f"towers {what}")
    assert_close(gates, per["gates"], TOL, f"gates {what}")
    assert_close(grads[0], per["dx"], TOL, f"d_x {what}")
    for name, got in zip(("dwe", "dbe", "dwg"), grads[1:]):
        check_reduced(got, red[name], f"{name} {what}")


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_through_ops_and_layers(name):
    """Forward and backward through ops against float64 and the reference's own float64 run, then the block through layers
    with the fixture's weights assigned under the reference's names."""
    from recalgorithm_b200 import layers as L
    z = np.load(os.path.join(GOLDEN, "mmoe", name + ".npz"), allow_pickle=False)
    x = np.asarray(z["x"], np.float32)
    p = _f32(z["w_experts"], z["b_experts"], z["w_gates"])
    E, d, H = p[0].shape
    T, B = p[2].shape[0], x.shape[0]
    g = np.random.default_rng(7).standard_normal((T, B, H)).astype(np.float32)
    towers, gates, grads = _run(x, p, g)
    _check(x, p, g, towers, gates, grads)
    assert_close(towers, z["towers_f64"], TOL, f"{name}: towers vs reference (float64)")
    assert_close(gates, z["gates_f64"], TOL, f"{name}: gates vs reference (float64)")

    store = L.set_default_store(L.VariableStore(device="cuda", seed=0))
    xt = dev(x).requires_grad_(True)
    L.mmoe_experts_gates(xt, E, H, T)
    store.assign({**{f"experts/expert_{i}/kernel": z["w_experts"][i] for i in range(E)},
                  **{f"experts/expert_{i}/bias": z["b_experts"][i] for i in range(E)},
                  **{f"gates/gate_{t}/kernel": z["w_gates"][t] for t in range(T)}})
    tw, gl = L.mmoe_experts_gates(xt, str(E), float(H), T, return_gates=True)
    assert len(tw) == T and len(gl) == T and all(t.is_contiguous() and t.shape == (B, H) for t in tw)
    for t in range(T):
        assert_close(tw[t], z["towers_f64"][t], TOL, f"{name}: layers tower {t}")
        assert_close(gl[t], z["gates_f64"][t], TOL, f"{name}: layers gate {t}")
    sum((tw[t] * dev(g[t])).sum() for t in range(T)).backward()
    r = R.bwd(np.asarray(x, np.float64), *R.fixture(z)[1:], g.astype(np.float64))
    assert_close(xt.grad, r[0], TOL, f"{name}: layers d_x")
    for i in range(E):
        assert_close(store.vars[f"experts/expert_{i}/kernel"].grad, r[1][i], TOL, f"{name}: d expert_{i}", elementwise=False)
        assert_close(store.vars[f"experts/expert_{i}/bias"].grad, r[2][i], TOL, f"{name}: d bias_{i}", elementwise=False)
    for t in range(T):
        want = r[3][t]
        got = store.vars[f"gates/gate_{t}/kernel"].grad
        if E == 1:
            assert torch.count_nonzero(got) == 0
        else:
            assert_close(got, want, TOL, f"{name}: d gate_{t}", elementwise=False)


ET = ((1, 1), (3, 3), (8, 4))                      # (E, T): one each, the reference values, the bounds
SHAPES = ([(129, d, E, H, T) for d in (1, 31, 32, 33, 82, 96, 128) for H in (1, 31, 32, 33, 512, 1000, 1024)
           for E, T in ET] +
          [(B, 82, 3, 512, 3) for B in (0, 1, 63, 64, 65, 127, 128, 129, 1000)] +
          [(65536, 82, 3, 512, 3)])


@pytest.mark.parametrize("B,d,E,H,T", SHAPES)
def test_mmoe_against_float64(B, d, E, H, T):
    x, p, g = _inputs(B, d, E, H, T, seed=B * 7 + d * 131 + H * 3 + E * 17 + T)
    towers, gates, grads = _run(x, p, g)
    _check(x, p, g, towers, gates, grads)


def test_single_expert_gates_are_exactly_one():
    """E = 1: the softmax is exactly 1, every tower is the single expert bit for bit, and d_w_gates is exactly 0."""
    x, p, g = _inputs(200, 82, 1, 256, 3, seed=11)
    towers, gates, grads = _run(x, p, g)
    assert torch.equal(gates, torch.ones_like(gates))
    for t in range(1, 3):
        assert torch.equal(towers[t], towers[0])
    assert torch.count_nonzero(grads[3]) == 0
    _check(x, p, g, towers, gates, grads)


def test_saturated_gates_do_not_overflow():
    """Gate logits near +-80 (expf would overflow float32 past 88 without the max subtracted): the gates stay finite, sum to
    1 and match float64."""
    B, d, E, H, T = 300, 82, 4, 128, 3
    rng = np.random.default_rng(12)
    p = _weights(rng, d, E, H, T)
    x, _, g = _inputs(B, d, E, H, T, seed=12, weights=p)
    logits = np.einsum("bd,tde->tbe", x.astype(np.float64), p[2].astype(np.float64))
    p[2] = (p[2] * (80.0 / np.abs(logits).max())).astype(np.float32)
    towers, gates, grads = _run(x, p, g)
    lg = np.einsum("bd,tde->tbe", x.astype(np.float64), p[2].astype(np.float64))
    assert np.abs(lg).max() > 70
    assert torch.isfinite(gates).all() and torch.isfinite(towers).all()
    assert float((gates.sum(-1) - 1).abs().max()) < 1e-6
    assert float(gates.max()) > 0.999
    x64, p64, g64 = np.asarray(x, np.float64), [np.asarray(t, np.float64) for t in p], np.asarray(g, np.float64)
    r_towers, r_gates, a = R.fwd(x64, *p64)
    assert_close(towers, r_towers, TOL, "saturated towers")
    assert_close(gates, r_gates, TOL, "saturated gates")
    d_x, d_we, d_be, d_wg = R.bwd(x64, *p64, g64)
    check_reduced(grads[1], (d_we, np.einsum("bd,ebh->edh", np.abs(x64), np.abs(_dz(r_gates, a, g64)))), "saturated dwe")
    check_reduced(grads[2], (d_be, np.abs(_dz(r_gates, a, g64)).sum(1)), "saturated dbe")
    # dlogit = p (dp - sum_e p dp) cancels to far below its terms when one gate is ~1, and the gate kernels are large here:
    # d_x and d_w_gates are held to TOL times the magnitude of their terms, which float32 inputs cannot beat
    dl_mag = _dlogit_mag(r_gates, a, g64)
    dx_mag = np.einsum("ebh,edh->bd", np.abs(_dz(r_gates, a, g64)), np.abs(p64[0])) + np.einsum("tbe,tde->bd", dl_mag, np.abs(p64[2]))
    err = np.abs(grads[0].cpu().double().numpy() - d_x)
    assert (err <= TOL * (dx_mag + np.sqrt(np.mean(d_x ** 2)))).all(), float((err / (dx_mag + 1e-30)).max())
    check_reduced(grads[3], (d_wg, np.einsum("bd,tbe->tde", np.abs(x64), dl_mag)), "saturated dwg")


def _dz(p, a, g):
    return np.einsum("tbe,tbh->ebh", p, g) * (a > 0)


def _dlogit_mag(p, a, g):
    """p (|dp| + sum_e p |dp|) with |dp| = sum_h |g h|: the magnitude of the terms of dlogit."""
    dpm = np.einsum("tbh,ebh->tbe", np.abs(g), np.maximum(a, 0))
    return p * (dpm + (p * dpm).sum(-1, keepdims=True))


def test_empty_batch_gives_zero_weight_gradients():
    from recalgorithm_b200 import ops
    x, p, g = _inputs(4, 82, 3, 128, 3, seed=1)
    args = [dev(t) for t in p]
    towers, gates = ops.mmoe_fwd(dev(x[:0]), *args)
    grads = ops.mmoe_bwd(dev(x[:0]), *args, gates, dev(g[:, :0]))
    assert towers.shape == (3, 0, 128) and gates.shape == (3, 0, 3) and grads[0].shape == (0, 82)
    for t in grads[1:]:
        assert t.numel() > 0 and torch.count_nonzero(t) == 0


def _abi_calls(h, P, nbytes, B, d, E, H, T):
    import ctypes
    n = ctypes.c_int64(0)
    return {"ctr_mmoe_workspace_bytes": lambda: h.ctr_mmoe_workspace_bytes(B, d, E, H, T, ctypes.byref(n)),
            "ctr_mmoe_fwd": lambda: h.ctr_mmoe_fwd(P, P, P, P, B, d, E, H, T, P, P, P, nbytes, None),
            "ctr_mmoe_bwd": lambda: h.ctr_mmoe_bwd(P, P, P, P, P, P, B, d, E, H, T, P, P, P, P, P, nbytes, None)}


@pytest.mark.parametrize("d,E,H,T,bound", [(129, 3, 512, 3, "d <= 128"), (82, 9, 512, 3, "E <= 8"),
                                           (82, 3, 1025, 3, "H <= 1024"), (82, 3, 512, 5, "T <= 4")])
def test_entries_refuse_shapes_past_the_bounds(d, E, H, T, bound):
    """All three entries refuse larger shapes with CTR_ERR_UNSUPPORTED and a message naming the bound, called through the C
    ABI with small real buffers."""
    from recalgorithm_b200 import _lib
    h = _lib.lib()
    buf = torch.zeros(1 << 16, device="cuda")
    for entry, call in _abi_calls(h, buf.data_ptr(), buf.numel() * 4, 4, d, E, H, T).items():
        assert call() == _lib.CTR_ERR_UNSUPPORTED, entry
        msg = h.ctr_last_error().decode()
        assert msg.startswith(entry) and bound in msg, msg
    torch.cuda.synchronize()


def test_too_small_workspace_is_refused():
    from recalgorithm_b200 import _lib, ops
    h = _lib.lib()
    B, d, E, H, T = 64, 82, 3, 512, 3
    need_fwd = ops.mmoe_workspace(0, d, E, H, T, "cuda").numel()
    need_bwd = ops.mmoe_workspace(B, d, E, H, T, "cuda").numel()
    assert need_bwd > need_fwd
    buf = torch.zeros(need_bwd // 4 + 64, device="cuda")
    calls = _abi_calls(h, buf.data_ptr(), 1024, B, d, E, H, T)          # the forward needs at most need_fwd bytes
    assert calls["ctr_mmoe_fwd"]() == _lib.CTR_ERR_INVALID_ARG
    assert h.ctr_last_error().decode().startswith("ctr_mmoe_fwd: workspace")
    calls = _abi_calls(h, buf.data_ptr(), need_bwd - 128, B, d, E, H, T)
    assert calls["ctr_mmoe_bwd"]() == _lib.CTR_ERR_INVALID_ARG
    assert h.ctr_last_error().decode().startswith("ctr_mmoe_bwd: workspace")
    torch.cuda.synchronize()


def test_cpu_tensors_are_refused():
    from recalgorithm_b200 import ops
    x, p, g = _inputs(4, 8, 2, 16, 2, seed=2)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.mmoe_fwd(*(torch.from_numpy(t) for t in (x, *p)))


_PROFILE = """
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile
from recalgorithm_b200 import ops
gen = torch.Generator(device="cuda").manual_seed(4)
args = [torch.randn(s, device="cuda", generator=gen) * 0.1 for s in ((1024, 82), (3, 82, 512), (3, 512), (3, 82, 3))]
gd = torch.randn((3, 1024, 512), device="cuda", generator=gen)
ops.mmoe_bwd(*args, ops.mmoe_fwd(*args)[1], gd)        # first launches (module load) outside the trace
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    towers, gates = ops.mmoe_fwd(*args)
    ops.mmoe_bwd(*args, gates, gd)
    torch.cuda.synchronize()
print(json.dumps([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]))
"""


def test_profiler_sees_only_the_new_kernels():
    """Forward and backward launch the MMoE kernels and nothing else: no torch kernel touches the expert tensor.  The trace
    is taken in a process of its own, so that this profiler session leaves the test process's profiler as it was."""
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
    assert sum("mmoe_fwd_wgmma_kernel" in n for n in kernels) == 1
    assert sum(bool(re.search(DW_KERNEL, n)) for n in kernels) == 1


def test_mmoe_logits_training_step():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import model_bodies as M
    from recalgorithm_b200 import layers as L
    B, tasks = 256, ("read_comment", "like", "click_avatar")
    store = L.set_default_store(L.VariableStore(device="cuda", seed=5))
    gen = torch.Generator(device="cuda").manual_seed(5)
    dense_input = torch.randn(B, 16, device="cuda", generator=gen).requires_grad_(True)
    cat = torch.randn(B, 66, device="cuda", generator=gen).requires_grad_(True)
    labels = {t: (torch.rand((B, 1), device="cuda", generator=gen) < 0.3).float() for t in tasks}
    logits, loss = M.mmoe_logits(dense_input, cat, labels, tasks, num_experts=3, expert_hidden_units=512,
                                 hidden_units=(64, 32))
    assert len(logits) == 3 and all(lg.shape == (B, 1) for lg in logits) and torch.isfinite(loss)
    opt = torch.optim.SGD(store.parameters(), lr=0.1)
    opt.zero_grad()
    loss.backward()
    want = ({f"experts/expert_{i}/{v}" for i in range(3) for v in ("kernel", "bias")} |
            {f"gates/gate_{t}/kernel" for t in range(3)} |
            {f"tower/{n}/{v}" for n in ("dense", *(f"dense_{i}" for i in range(1, 6))) for v in ("kernel", "bias")} |
            {f"tower/tower_{t}_logit/{v}" for t in tasks for v in ("kernel", "bias")})
    assert set(store.vars) == want, set(store.vars) ^ want
    for n, v in store.vars.items():
        assert v.grad is not None and torch.isfinite(v.grad).all() and torch.count_nonzero(v.grad) > 0, n
    assert float(dense_input.grad.abs().max()) > 0 and float(cat.grad.abs().max()) > 0
    opt.step()
    with torch.no_grad():
        loss2 = M.mmoe_logits(dense_input, cat, labels, tasks, num_experts=3, expert_hidden_units=512,
                              hidden_units=(64, 32))[1]
    assert torch.isfinite(loss2) and float(loss2) < float(loss.detach())
