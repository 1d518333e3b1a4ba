"""CPU tests of the AutoInt host layer (layers.interacting_layer) with the kernel launch stubbed: variable names, shapes and
initialisers for a three-layer stack in a caller's scope, reuse under the same index, and string widths."""
import math

import pytest
import torch


@pytest.fixture()
def store(monkeypatch):
    from recalgorithm_b200 import autograd, layers as L
    calls = []

    def fake_autoint(x, wq, wk, wv, wr, heads, dk):
        calls.append((x, wq, wk, wv, wr, heads, dk))
        return torch.zeros(x.shape[0], x.shape[1], heads * dk)
    monkeypatch.setattr(autograd, "autoint_interacting", fake_autoint)
    st = L.set_default_store(L.VariableStore(device="cpu", seed=0))
    st.calls = calls
    yield st
    L.set_default_store(L.VariableStore(device="cpu"))


def test_three_layer_stack_variables_and_initialisers(store):
    from recalgorithm_b200 import layers as L
    B, F, d, H, dk = 4, 40, 16, 2, 32
    with L.variable_scope("autoint"):
        net = torch.randn(B, F, d)
        for i in range(3):
            net = L.interacting_layer(net, dk, H, index=i)
    assert net.shape == (B, F, H * dk)
    want = {}
    for i in range(3):
        width = d if i == 0 else H * dk
        want.update({f"autoint/interacting_layer_{i}/{n}": (width, H * dk) for n in ("query", "key", "value", "res")})
    assert {k: tuple(v.shape) for k, v in store.vars.items()} == want
    for name, v in store.vars.items():
        limit = math.sqrt(6.0 / sum(v.shape))
        v = v.detach()
        assert float(v.abs().max()) <= limit and float(v.std()) > 0.3 * limit, name
    assert [c[5:] for c in store.calls] == [(H, dk)] * 3


def test_reuses_variables_under_the_same_index(store):
    from recalgorithm_b200 import layers as L
    x = torch.randn(2, 5, 8)
    L.interacting_layer(x, 4, 2, index=0)
    n = len(store.vars)
    L.interacting_layer(x, 4, 2, index=0)
    assert len(store.vars) == n
    assert all(a is b for a, b in zip(store.calls[0][1:5], store.calls[1][1:5]))


def test_string_widths_and_none(store):
    from recalgorithm_b200 import layers as L
    out = L.interacting_layer(torch.randn(3, 5, 8), "4", "2", index=7)
    assert out.shape == (3, 5, 8)
    assert tuple(store.vars["interacting_layer_7/query"].shape) == (8, 8)
    with pytest.raises(TypeError):
        L.interacting_layer(torch.randn(3, 5, 8), None, 2, index=1)
