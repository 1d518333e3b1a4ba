"""CPU tests of the PLE oracle: the float64 restatement (tests/_ple_ref.py) against the reference-executed fixtures
(tests/golden/ple), its analytic backward against torch autograd, the fixture digests, and the variables each reference
run created."""
import glob
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import _ple_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden", "ple")
FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(G, "*.npz")))


def test_fixtures_present():
    assert FIXTURES == ["ple_extraction_d5_n2-1_S1_H7_B9", "ple_extraction_d82_n5-5-5_S10_H256_B8",
                        "ple_final_d256_n10-10-10_S20_H256_B4", "ple_final_d256_n5-5-5_S10_H256_B8",
                        "ple_final_d5_n2-1_S1_H7_B9"]


@pytest.mark.parametrize("name", FIXTURES)
def test_restatement_equals_reference_run(name):
    z = np.load(os.path.join(G, name + ".npz"), allow_pickle=False)
    arrays, counts = R.fixture(z)
    out, gates, _ = R.fwd(*arrays, *counts)
    ref = z["out_f64"]
    assert out.shape == ref.shape
    assert np.abs(out.numpy() - ref).max() <= 1e-13 * max(1.0, np.abs(ref).max())
    assert np.abs(z["out_f32"] - ref).max() <= 1e-5 * np.abs(ref).max()
    # every gate is a distribution over its own columns
    widths = [len(e) for e in R.gate_experts(*counts)]
    assert gates.shape == (ref.shape[-2], sum(widths))
    for s in torch.split(gates, widths, dim=1):
        assert torch.allclose(s.sum(1), torch.ones(s.shape[0], dtype=torch.float64), atol=1e-14)


@pytest.mark.parametrize("name", FIXTURES)
def test_reference_creates_the_variables_the_layers_create(name):
    """The names and shapes, in creation order, that the reference run recorded are those recalgorithm_b200.layers
    creates for the same block (with the launch stubbed)."""
    from recalgorithm_b200 import autograd
    from recalgorithm_b200 import layers as L
    z = np.load(os.path.join(G, name + ".npz"), allow_pickle=False)
    (x, we, be, wg), (n, S, extraction) = R.fixture(z)
    tasks = ("read_comment", "like", "click_avatar")[:len(n)]
    store = L.set_default_store(L.VariableStore(device="cpu", seed=0))
    real = autograd.ple
    autograd.ple = lambda x, *a: (torch.zeros((x.shape[0], 1)), None) if a[-1] else (torch.zeros((len(n), x.shape[0], 1)),
                                                                                     torch.zeros((x.shape[0], 1)))
    try:
        xt = x.float()
        if extraction:
            L.extraction_network(xt, tasks, n, S, we.shape[2], "extract_network_0")
        else:
            L.ple_final_experts_gates(xt, tasks, n, S, we.shape[2])
    finally:
        autograd.ple = real
    shapes = [tuple(int(v) for v in s if v) for s in z["variable_shapes"]]
    assert list(store.vars) == [str(v) for v in z["variables"]]
    assert [tuple(v.shape) for v in store.vars.values()] == shapes


@pytest.mark.parametrize("B,d,n,S,H,extraction", [(9, 5, (2, 1), 1, 7, True), (9, 5, (2, 1), 1, 7, False),
                                                  (16, 33, (3, 1, 2), 2, 40, True), (7, 20, (1, 2, 1, 3), 4, 17, False)])
def test_analytic_backward_equals_autograd(B, d, n, S, H, extraction):
    rng = np.random.default_rng(B + d + H + S + sum(n))
    E, GC = sum(n) + S, sum(n) + len(n) * S + ((sum(n) + S) if extraction else 0)
    x = rng.standard_normal((B, d))
    p = (rng.standard_normal((E, d, H)) / d ** 0.5, rng.standard_normal((E, H)) * 0.1, rng.standard_normal((d, GC)))
    ts = [torch.tensor(t, dtype=torch.float64, requires_grad=True) for t in (x,) + p]
    out, gates, _ = R.fwd(*ts, list(n), S, extraction)
    g = torch.tensor(rng.standard_normal(tuple(out.shape)))
    out.backward(g)
    with torch.no_grad():
        got = R.bwd(*(t.detach() for t in ts), g, list(n), S, extraction)
    for a, t in zip(got[:4], ts):
        assert torch.allclose(a, t.grad, rtol=1e-12, atol=1e-12)


def test_extraction_output_is_the_sum_of_the_gated_outputs():
    """The extraction network's output equals the final-layer form of its task gates summed, plus the all-gate output."""
    rng = np.random.default_rng(3)
    n, S, B, d, H = [2, 3], 2, 6, 11, 9
    E = sum(n) + S
    x, we, be = (torch.tensor(rng.standard_normal(s)) for s in ((B, d), (E, d, H), (E, H)))
    wg = torch.tensor(rng.standard_normal((d, sum(n) + len(n) * S + E)))
    out, gates, a = R.fwd(x, we, be, wg, n, S, True)
    tasks, _, _ = R.fwd(x, we, be, wg[:, :sum(n) + len(n) * S], n, S, False)
    p_all = gates[:, sum(n) + len(n) * S:]
    assert torch.allclose(out, tasks.sum(0) + torch.einsum("be,ebh->bh", p_all, torch.relu(a)), atol=1e-12)


@pytest.mark.parametrize("name", FIXTURES)
def test_regenerated_weights_are_those_the_reference_ran(name):
    """The weights fixture() rebuilds from the stored seed hash to the digest recorded when the reference ran on them."""
    z = np.load(os.path.join(G, name + ".npz"), allow_pickle=False)
    (_, we, be, wg), _ = R.fixture(z)
    got = hashlib.sha256(b"".join(np.ascontiguousarray(t.numpy(), np.float64).tobytes() for t in (we, be, wg))).hexdigest()
    assert got == str(z["weights_sha256"])
    assert float(we.abs().max()) <= 26 / 256 and float(be.abs().max()) <= 25 / 256 and float(wg.abs().max()) <= 0.25


def test_digests_match():
    with open(os.path.join(G, "reference_digests.json")) as fh:
        want = json.load(fh)
    assert sorted(want) == [f + ".npz" for f in FIXTURES]
    for fname, arrays in want.items():
        z = np.load(os.path.join(G, fname), allow_pickle=False)
        assert sorted(z.files) == sorted(arrays), fname
        for k, dig in arrays.items():
            a = z[k]
            assert dig == f"{a.dtype.str}:{'x'.join(map(str, a.shape))}:{hashlib.sha256(a.tobytes()).hexdigest()}", (fname, k)
