"""CPU tests of the DeepCrossing oracle: the float64 restatement (tests/_deepcrossing_ref.py) against the reference-executed
fixtures (tests/golden/deepcrossing), its analytic backward against torch autograd, and the fixture digests."""
import glob
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _deepcrossing_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden", "deepcrossing")
FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(G, "*.npz")))


def test_fixtures_present():
    assert FIXTURES == ["deepcrossing_d5_H3_units3_B9", "deepcrossing_d82_H128_units1_B16", "deepcrossing_d82_H256_units2_B16"]


@pytest.mark.parametrize("name", FIXTURES)
def test_restatement_equals_reference_run(name):
    z = np.load(os.path.join(G, name + ".npz"), allow_pickle=False)
    units = R.fixture_units(z)
    x = np.asarray(z["x"], np.float64)
    out64 = R.module_fwd(x, units)
    assert np.abs(out64 - z["out_f64"]).max() <= 1e-13 * max(1.0, np.abs(z["out_f64"]).max())
    out32 = np.asarray(z["x"], np.float32)
    for p in units:
        out32 = R.unit_fwd(out32, *(np.asarray(t, np.float32) for t in p))[0]
    assert np.abs(out32 - z["out_f32"]).max() <= 2e-6 * max(1.0, np.abs(z["out_f32"]).max())
    assert np.abs(z["out_f32"] - z["out_f64"]).max() <= 1e-5 * np.abs(z["out_f64"]).max()


@pytest.mark.parametrize("B,d,H", [(9, 5, 3), (16, 82, 256), (7, 33, 65)])
def test_analytic_backward_equals_autograd(B, d, H):
    rng = np.random.default_rng(B + d + H)
    x = rng.standard_normal((B, d))
    p = (rng.standard_normal((d, H)) / d ** 0.5, rng.standard_normal(H) * 0.1, rng.standard_normal((H, d)) / H ** 0.5,
         rng.standard_normal(d) * 0.1)
    g = rng.standard_normal((B, d))
    ts = [torch.tensor(t, dtype=torch.float64, requires_grad=True) for t in (x,) + p]
    xt, w0, b0, w1, b1 = ts
    out = torch.relu(xt + torch.relu(xt @ w0 + b0) @ w1 + b1)
    out.backward(torch.tensor(g))
    assert np.allclose(out.detach().numpy(), R.unit_fwd(x, *p)[0], rtol=0, atol=1e-13)
    for got, t in zip(R.unit_bwd(x, *p, g), ts):
        assert np.allclose(got, t.grad.numpy(), rtol=1e-12, atol=1e-12)


def _digest(a):
    return f"{a.dtype.str}:{'x'.join(map(str, a.shape))}:{hashlib.sha256(a.tobytes()).hexdigest()}"


def test_fixtures_match_reference_digests(tmp_path):
    """Every array of every fixture is bit-identical to the recorded run over the reference.  With RECALG_REFERENCE set to a
    reference checkout (the `algorithm` directory), the generator re-runs into a temporary directory and must reproduce
    the same digests."""
    want = json.load(open(os.path.join(G, "reference_digests.json")))
    assert sorted(want) == sorted(n + ".npz" for n in FIXTURES)
    for name in want:
        with np.load(os.path.join(G, name), allow_pickle=False) as z:
            assert {k: _digest(z[k]) for k in z.files} == want[name], name
    ref = os.environ.get("RECALG_REFERENCE")
    if not ref:
        return
    code = ("import sys, json; sys.path.insert(0, 'tools'); import make_golden_deepcrossing as m; "
            f"print(json.dumps(m.gen_deepcrossing({str(tmp_path)!r})))")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True,
                         env={**os.environ, "RECALG_REFERENCE": ref})
    assert out.returncode == 0, out.stderr
    assert json.loads(out.stdout.strip().splitlines()[-1]) == want
