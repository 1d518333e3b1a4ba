"""GPU parity: DeepCrossing's residual unit (csrc/residual_unit.cu) against the reference-executed fixtures
(tests/golden/deepcrossing) and the float64 restatement with its analytic backward (tests/_deepcrossing_ref.py)."""
import glob
import os
import sys

import numpy as np
import pytest
import torch

import _deepcrossing_ref as R
from _util import GOLDEN, TOL, assert_close, dev
from test_gpu_layer_variants import check_reduced, chunked_reference

pytestmark = pytest.mark.gpu

FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "deepcrossing", "*.npz")))
KERNELS = ("resunit_prep_kernel", "resunit_fwd_wgmma_kernel", "resunit_bwd_dx_wgmma_kernel", "resunit_bwd_dw_wgmma_kernel")


def _f32(*arrays):
    return [np.asarray(a, np.float32) for a in arrays]


def _inputs(B, d, H, seed, b0=None, b1=None):
    """x (B,d), weights and g in float32.  Samples whose hidden or output pre-activation lies within 1e-6 of 0, relative to the
    sum of the magnitudes of its terms, are redrawn: float32 may take the other side of the relu there, which is not a kernel
    error (a 65 536-sample draw had an output at 3.8e-7 of its terms' scale, which the kernel rounded to the other side)."""
    rng = np.random.default_rng(seed)
    w0 = rng.uniform(-1, 1, (d, H)) * (6.0 / (d + H)) ** 0.5
    w1 = rng.uniform(-1, 1, (H, d)) * (6.0 / (d + H)) ** 0.5
    b0 = rng.uniform(-0.1, 0.1, H) if b0 is None else b0
    b1 = rng.uniform(-0.1, 0.1, d) if b1 is None else b1
    p = [np.asarray(t, np.float64) for t in _f32(w0, b0, w1, b1)]
    x = _f32(rng.standard_normal((B, d)) * 0.7)[0]
    for _ in range(100):
        x64 = x.astype(np.float64)
        _, a, z = R.unit_fwd(x64, *p)
        scale_a = np.abs(x64) @ np.abs(p[0]) + np.abs(p[1])
        scale_z = np.abs(x64) + np.maximum(a, 0) @ np.abs(p[2]) + np.abs(p[3])
        bad = (np.abs(a) <= 1e-6 * scale_a).any(1) | (np.abs(z) <= 1e-6 * scale_z).any(1)
        if not bad.any():
            break
        x[bad] = _f32(rng.standard_normal((int(bad.sum()), d)) * 0.7)[0]
    else:
        raise AssertionError("could not draw inputs away from the relu edges")
    g = _f32(rng.standard_normal((B, d)))[0]
    return x, _f32(*p), g


def _run(x, p, g):
    from recalgorithm_b200 import ops
    args = [dev(t) for t in (x, *p)]
    out = ops.residual_unit_fwd(*args)
    grads = ops.residual_unit_bwd(*args, out, dev(g))
    return out, grads


def _check(B, d, H, x, p, g, out, grads):
    x64, p64, g64 = np.asarray(x, np.float64), [np.asarray(t, np.float64) for t in p], np.asarray(g, np.float64)

    def part(lo, hi):
        dx, dw0, db0, dw1, db1 = R.unit_bwd(x64[lo:hi], *p64, g64[lo:hi])
        return {"out": R.unit_fwd(x64[lo:hi], *p64)[0], "dx": dx}, {"dw0": dw0, "db0": db0, "dw1": dw1, "db1": db1}
    per, red = chunked_reference(B, part)
    if B == 0:
        per = {"out": np.zeros((0, d)), "dx": np.zeros((0, d))}
    assert_close(out, per["out"], TOL, f"out B={B} d={d} H={H}")
    assert_close(grads[0], per["dx"], TOL, f"d_x B={B} d={d} H={H}")
    for name, got in zip(("dw0", "db0", "dw1", "db1"), grads[1:]):
        check_reduced(got, red[name], f"{name} B={B} d={d} H={H}")


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_through_ops_and_layers(name):
    """Each unit through ops (forward and backward against float64), then the whole residual_module loop through layers with
    the fixture's weights assigned under the reference's names."""
    from recalgorithm_b200 import layers as L
    z = np.load(os.path.join(GOLDEN, "deepcrossing", name + ".npz"), allow_pickle=False)
    units = R.fixture_units(z)
    B, d = z["x"].shape
    H = units[0][0].shape[1]
    g = np.random.default_rng(7).standard_normal((B, d)).astype(np.float32)
    xi = np.asarray(z["x"], np.float32)
    for p in units:
        p32 = _f32(*p)
        out, grads = _run(xi, p32, g)
        _check(B, d, H, xi, p32, g, out, grads)
        xi = out.cpu().numpy()
    assert_close(out, z["out_f64"], TOL, f"{name}: out vs reference (float64)")

    store = L.set_default_store(L.VariableStore(device="cuda", seed=0))
    x = dev(z["x"]).requires_grad_(True)

    def module():
        with L.variable_scope("residual_module"):
            net = x
            for i in range(len(units)):
                net = L.residual_unit(net, str(H), index=i)
        return net
    module()
    store.assign({f"residual_module/dense_{i}_{k}": z[f"{w}_{i}"] for i in range(len(units))
                  for k, w in (("0/kernel", "w0"), ("0/bias", "b0"), ("1/kernel", "w1"), ("1/bias", "b1"))})
    net = module()
    assert_close(net, z["out_f64"], TOL, f"{name}: layers vs reference (float64)")
    net.backward(dev(g))
    r_dx, r_units = R.module_bwd(np.asarray(z["x"], np.float64), units, g.astype(np.float64))
    assert_close(x.grad, r_dx, TOL, f"{name}: layers d_x")
    for i, rg in enumerate(r_units):
        for k, want in zip(("0/kernel", "0/bias", "1/kernel", "1/bias"), rg):
            got = store.vars[f"residual_module/dense_{i}_{k}"].grad
            assert_close(got, want, TOL, f"{name}: layers d dense_{i}_{k}", elementwise=False)


SHAPES = ([(129, d, H) for d in (1, 31, 32, 33, 82, 96, 127, 128) for H in (1, 63, 64, 65, 128, 256, 1000, 1024)] +
          [(B, d, H) for B in (0, 1, 127, 128, 129, 1024) for d, H in ((82, 256), (82, 128), (128, 1024), (33, 65))] +
          [(65536, 82, 256)])


@pytest.mark.parametrize("B,d,H", SHAPES)
def test_residual_unit_against_float64(B, d, H):
    x, p, g = _inputs(B, d, H, seed=B * 7 + d * 131 + H)
    out, grads = _run(x, p, g)
    _check(B, d, H, x, p, g, out, grads)


def test_dead_hidden_unit_and_dead_output_give_exact_zeros():
    B, d, H = 300, 82, 256
    rng = np.random.default_rng(3)
    b0 = rng.uniform(-0.1, 0.1, H); b0[[5, 200]] = -1e3          # hidden units 5 and 200 never fire
    b1 = rng.uniform(-0.1, 0.1, d); b1[[0, 40]] = -1e3           # outputs 0 and 40 are always 0
    x, p, g = _inputs(B, d, H, seed=3, b0=b0, b1=b1)
    out, (dx, dw0, db0, dw1, db1) = _run(x, p, g)
    assert torch.count_nonzero(out[:, [0, 40]]) == 0
    assert torch.count_nonzero(db0[[5, 200]]) == 0 and torch.count_nonzero(dw0[:, [5, 200]]) == 0
    assert torch.count_nonzero(dw1[[5, 200], :]) == 0
    assert torch.count_nonzero(db1[[0, 40]]) == 0 and torch.count_nonzero(dw1[:, [0, 40]]) == 0
    _check(B, d, H, x, p, g, out, (dx, dw0, db0, dw1, db1))


def test_empty_batch_gives_zero_weight_gradients():
    from recalgorithm_b200 import ops
    x, p, g = _inputs(4, 82, 128, seed=1)
    args = [dev(t) for t in p]
    out = ops.residual_unit_fwd(dev(x[:0]), *args)
    grads = ops.residual_unit_bwd(dev(x[:0]), *args, out, dev(g[:0]))
    assert out.shape == (0, 82) and grads[0].shape == (0, 82)
    for t in grads[1:]:
        assert t.numel() > 0 and torch.count_nonzero(t) == 0


@pytest.mark.parametrize("d,H", [(129, 64), (82, 1025)])
def test_entries_refuse_shapes_past_the_tensor_core_bounds(d, H):
    """d <= 128 and H <= 1024: all three entries refuse larger shapes with CTR_ERR_UNSUPPORTED and a message naming the bound,
    called through the C ABI with small real buffers."""
    import ctypes
    from recalgorithm_b200 import _lib
    h = _lib.lib()
    buf = torch.zeros(1 << 16, device="cuda")
    P = buf.data_ptr()
    n = ctypes.c_int64(0)
    calls = {"ctr_residual_unit_workspace_bytes": lambda: h.ctr_residual_unit_workspace_bytes(4, d, H, ctypes.byref(n)),
             "ctr_residual_unit_fwd": lambda: h.ctr_residual_unit_fwd(P, P, P, P, P, 4, d, H, P, P, buf.numel() * 4, None),
             "ctr_residual_unit_bwd": lambda: h.ctr_residual_unit_bwd(P, P, P, P, P, P, P, 4, d, H, P, P, P, P, P, P,
                                                                      buf.numel() * 4, None)}
    for entry, call in calls.items():
        assert call() == _lib.CTR_ERR_UNSUPPORTED, entry
        msg = h.ctr_last_error().decode()
        assert msg.startswith(entry) and ("d <= 128" if d > 128 else "H <= 1024") in msg, msg
    torch.cuda.synchronize()


def test_cpu_tensors_are_refused():
    from recalgorithm_b200 import ops
    x, p, g = _inputs(4, 8, 16, seed=2)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.residual_unit_fwd(*(torch.from_numpy(t) for t in (x, *p)))


_PROFILE = """
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, "tests")
from _util import dev
from test_gpu_deepcrossing import _inputs
from recalgorithm_b200 import ops
x, p, g = _inputs(1024, 82, 256, seed=4)
args, gd = [dev(t) for t in (x, *p)], dev(g)
ops.residual_unit_bwd(*args, ops.residual_unit_fwd(*args), gd)        # first launches (module load) outside the trace
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    out = ops.residual_unit_fwd(*args)
    ops.residual_unit_bwd(*args, out, gd)
    torch.cuda.synchronize()
print(json.dumps([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]))
"""


def test_profiler_sees_only_the_new_kernels():
    """Forward and backward launch the residual-unit kernels and nothing else: no torch kernel touches the hidden tensor.
    The trace is taken in a process of its own, so that this profiler session leaves the test process's profiler as it was."""
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
    assert sum("resunit_fwd_wgmma_kernel" in n for n in kernels) == 1
    assert sum("resunit_bwd_dw_wgmma_kernel" in n for n in kernels) == 2


def test_deepcrossing_logit_body():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import model_bodies as M
    from recalgorithm_b200 import layers as L
    B = 256
    store = L.set_default_store(L.VariableStore(device="cuda", seed=5))
    gen = torch.Generator(device="cuda").manual_seed(5)
    dense_input = torch.randn(B, 16, device="cuda", generator=gen).requires_grad_(True)
    cat = torch.randn(B, 66, device="cuda", generator=gen).requires_grad_(True)
    y = (torch.rand((B, 1), device="cuda", generator=gen) < 0.3).float()
    logit = M.deepcrossing_logit(dense_input, cat, residual_internal_dim=256, residual_network_num=2)
    assert logit.shape == (B, 1) and torch.isfinite(logit).all()
    torch.nn.functional.binary_cross_entropy_with_logits(logit, y).backward()
    want = {f"residual_module/dense_{i}_{k}/{v}" for i in range(2) for k in (0, 1) for v in ("kernel", "bias")}
    assert set(store.vars) == want | {"dense/kernel", "dense/bias"}
    for n, v in store.vars.items():
        assert v.grad is not None and torch.isfinite(v.grad).all() and torch.count_nonzero(v.grad) > 0, n
    assert float(dense_input.grad.abs().max()) > 0 and float(cat.grad.abs().max()) > 0
