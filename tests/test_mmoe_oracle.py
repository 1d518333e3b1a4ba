"""CPU tests of the MMoE oracle: the float64 restatement (tests/_mmoe_ref.py) against the reference-executed fixtures
(tests/golden/mmoe), its analytic backward against torch autograd, the fixture digests, and the E = 1 quirk."""
import glob
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _mmoe_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden", "mmoe")
FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(G, "*.npz")))


def test_fixtures_present():
    assert FIXTURES == ["mmoe_d5_E1_H7_T2_B9", "mmoe_d82_E3_H512_T3_B16", "mmoe_d82_E6_H1024_T3_B8"]


@pytest.mark.parametrize("name", FIXTURES)
def test_restatement_equals_reference_run(name):
    z = np.load(os.path.join(G, name + ".npz"), allow_pickle=False)
    towers, gates, _ = R.fwd(*R.fixture(z))
    for got, key in ((towers, "towers_f64"), (gates, "gates_f64")):
        assert np.abs(got - z[key]).max() <= 1e-13 * max(1.0, np.abs(z[key]).max()), key
    towers32, gates32, _ = R.fwd(*(np.asarray(z[k], np.float32) for k in ("x", "w_experts", "b_experts", "w_gates")))
    for got, key in ((towers32, "towers_f32"), (gates32, "gates_f32")):
        assert got.dtype == np.float32
        assert np.abs(got - z[key]).max() <= 2e-6 * max(1.0, np.abs(z[key]).max()), key
    assert np.abs(z["towers_f32"] - z["towers_f64"]).max() <= 1e-5 * np.abs(z["towers_f64"]).max()


@pytest.mark.parametrize("B,d,E,H,T", [(9, 5, 1, 7, 2), (16, 82, 3, 64, 3), (7, 33, 6, 65, 4)])
def test_analytic_backward_equals_autograd(B, d, E, H, T):
    rng = np.random.default_rng(B + d + H + E + T)
    x = rng.standard_normal((B, d))
    p = (rng.standard_normal((E, d, H)) / d ** 0.5, rng.standard_normal((E, H)) * 0.1, rng.standard_normal((T, d, E)))
    g = rng.standard_normal((T, B, H))
    ts = [torch.tensor(t, dtype=torch.float64, requires_grad=True) for t in (x,) + p]
    xt, we, be, wg = ts
    h = torch.relu(torch.einsum("bd,edh->ebh", xt, we) + be[:, None, :])
    gates = torch.softmax(torch.einsum("bd,tde->tbe", xt, wg), dim=-1)
    towers = torch.einsum("tbe,ebh->tbh", gates, h)
    towers.backward(torch.tensor(g))
    r_towers, r_gates, _ = R.fwd(x, *p)
    assert np.allclose(towers.detach().numpy(), r_towers, rtol=0, atol=1e-13)
    assert np.allclose(gates.detach().numpy(), r_gates, rtol=0, atol=1e-13)
    for got, t in zip(R.bwd(x, *p, g), ts):
        assert np.allclose(got, t.grad.numpy(), rtol=1e-12, atol=1e-12)


def test_single_expert_softmax_is_exactly_one():
    """E = 1 (the ragged fixture): the reference's gates are exactly 1, every tower is the expert itself, and the gate
    kernels get exactly zero gradient."""
    z = np.load(os.path.join(G, "mmoe_d5_E1_H7_T2_B9.npz"), allow_pickle=False)
    for tag in ("f32", "f64"):
        assert np.all(z["gates_" + tag] == 1.0)
        expert = np.maximum(np.asarray(z["x"], z["towers_" + tag].dtype) @ z["w_experts"][0].astype(z["towers_" + tag].dtype)
                            + z["b_experts"][0], 0)
        for t in range(z["towers_" + tag].shape[0]):
            assert np.array_equal(z["towers_" + tag][t], z["towers_" + tag][0])
        assert np.allclose(z["towers_" + tag][0], expert, rtol=0, atol=1e-6)
    x, we, be, wg = R.fixture(z)
    g = np.random.default_rng(0).standard_normal((wg.shape[0], x.shape[0], we.shape[2]))
    assert np.all(R.bwd(x, we, be, wg, g)[3] == 0)


def test_large_logits_do_not_overflow():
    """The softmax runs over the experts axis with the max subtracted: logits near +-80 give finite gates."""
    z = np.array([[[80.0, -80.0, 79.0]]])
    p = R.softmax(z)
    assert np.isfinite(p).all() and abs(p.sum() - 1) < 1e-15 and p[0, 0, 1] < 1e-60


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
    code = ("import sys, json; sys.path.insert(0, 'tools'); import make_golden_mmoe as m; "
            f"print(json.dumps(m.gen_mmoe({str(tmp_path)!r})))")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True,
                         env={**os.environ, "RECALG_REFERENCE": ref})
    assert out.returncode == 0, out.stderr
    assert json.loads(out.stdout.strip().splitlines()[-1]) == want


@pytest.mark.parametrize("B", [0, 1, 64, 150])
def test_chunked_torch_equals_restatement(B):
    """The float64 torch form the GPU tests use equals the NumPy restatement, and its magnitudes are the sums of |chunk sums|."""
    rng = np.random.default_rng(B)
    d, E, H, T = 9, 3, 20, 2
    x, g = rng.standard_normal((B, d)), rng.standard_normal((T, B, H))
    p = (rng.standard_normal((E, d, H)) / 3, rng.standard_normal((E, H)) * 0.1, rng.standard_normal((T, d, E)))
    per, red = R.chunked_torch(*(torch.tensor(t) for t in (x, *p, g)), chunk=64, group=1)
    towers, gates, _ = R.fwd(x, *p)
    d_x, *w = R.bwd(x, *p, g)
    for got, want in ((per["towers"], towers), (per["gates"], gates), (per["dx"], d_x)):
        assert np.allclose(got, want, rtol=0, atol=1e-12)
    mags = [0.0, 0.0, 0.0]
    for lo in range(0, max(B, 1), 64):
        for i, v in enumerate(R.bwd(x[lo:lo + 64], *p, g[:, lo:lo + 64])[1:]):
            mags[i] = mags[i] + np.abs(v)
    for k, want, mag in zip(("dwe", "dbe", "dwg"), w, mags):
        assert np.allclose(red[k][0], want, rtol=0, atol=1e-12) and np.allclose(red[k][1], mag, rtol=0, atol=1e-12), k
