"""Float64 restatement of DeepCrossing's residual unit (DeepCrossing/residual_unit.py:4-21) with its analytic backward; the
GPU tests compare the kernels against it, and tests/test_deepcrossing_oracle.py pins it to the reference-executed fixtures."""
import numpy as np


def unit_fwd(x, w0, b0, w1, b1):
    """out = relu(x + relu(x . w0 + b0) . w1 + b1); also returns the hidden pre-activation a and the output pre-activation."""
    a = x @ w0 + b0
    z = x + (np.maximum(a, 0) @ w1 + b1)
    return np.maximum(z, 0), a, z


def unit_bwd(x, w0, b0, w1, b1, g):
    """(d_x, d_w0, d_b0, d_w1, d_b1) for upstream gradient g."""
    out, a, _ = unit_fwd(x, w0, b0, w1, b1)
    h = np.maximum(a, 0)
    gy = g * (out > 0)
    gh = (gy @ w1.T) * (a > 0)
    return gy + gh @ w0.T, x.T @ gh, gh.sum(0), h.T @ gy, gy.sum(0)


def module_fwd(x, units):
    """The loop of DeepCrossing/deepcrossing.py:154-157 over units [(w0, b0, w1, b1), ...]."""
    for p in units:
        x = unit_fwd(x, *p)[0]
    return x


def fixture_units(z):
    """[(w0, b0, w1, b1) per unit] of a tests/golden/deepcrossing fixture, in float64."""
    n = len([k for k in z.files if k.startswith("w0_")])
    return [tuple(np.asarray(z[f"{k}_{i}"], np.float64) for k in ("w0", "b0", "w1", "b1")) for i in range(n)]


def module_bwd(x, units, g):
    """Backward of module_fwd: (d_x, [(d_w0, d_b0, d_w1, d_b1) per unit])."""
    xs = [x]
    for p in units:
        xs.append(unit_fwd(xs[-1], *p)[0])
    grads = []
    for xi, p in zip(reversed(xs[:-1]), reversed(units)):
        g, *dp = unit_bwd(xi, *p, g)
        grads.append(tuple(dp))
    return g, grads[::-1]
