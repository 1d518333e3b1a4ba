"""CPU tests of the DCN-Mix host layer (layers.cross_network_mix) with the kernel call recorded: variable names, shapes and
initialisers, one gate matrix for every layer, reuse and shape conflicts, string arguments, bad values and zero layers."""
import math

import pytest
import torch


@pytest.fixture()
def store(monkeypatch):
    from recalgorithm_b200 import autograd, layers as L
    calls = []

    def fake_cross_mix(x0, v, c, u, b, gate, activation="tanh"):
        calls.append((x0, v, c, u, b, gate, activation))
        return torch.zeros_like(x0)
    monkeypatch.setattr(autograd, "cross_mix", fake_cross_mix)
    st = L.set_default_store(L.VariableStore(device="cpu", seed=0))
    st.calls = calls
    yield st
    L.set_default_store(L.VariableStore(device="cpu"))


def _check_glorot(v, name):
    limit = math.sqrt(6.0 / sum(v.shape))
    v = v.detach()
    assert float(v.abs().max()) <= limit and float(v.std()) > 0.3 * limit, name


def test_variables_shapes_and_initialisers(store):
    from recalgorithm_b200 import layers as L
    B, d, K, r = 4, 82, 3, 16
    x0 = torch.randn(B, d)
    with L.variable_scope("cross_part"):
        L.cross_network_mix(x0, 2, num_experts=K, low_rank=r)
    want = {"cross_part/cross_mix_gates/kernel": (d, K)}
    for l in range(2):
        for i in range(K):
            want[f"cross_part/cross_mix_{l}/expert_{i}/kernel_v"] = (d, r)
            want[f"cross_part/cross_mix_{l}/expert_{i}/kernel_c"] = (r, r)
            want[f"cross_part/cross_mix_{l}/expert_{i}/kernel_u"] = (r, d)
        want[f"cross_part/cross_mix_{l}/bias"] = (d,)
    assert {k: tuple(v.shape) for k, v in store.vars.items()} == want
    for name, v in store.vars.items():
        if name.endswith("bias"):
            assert torch.count_nonzero(v) == 0
        else:
            _check_glorot(v, name)
    (call,) = store.calls
    x, v, c, u, b, gate, act = call
    assert x is x0 and act == "tanh"
    assert v.shape == (2, K, d, r) and c.shape == (2, K, r, r) and u.shape == (2, K, r, d) and b.shape == (2, d)
    assert torch.equal(v[1, 2], store.vars["cross_part/cross_mix_1/expert_2/kernel_v"])
    assert torch.equal(c[0, 1], store.vars["cross_part/cross_mix_0/expert_1/kernel_c"])
    assert torch.equal(u[1, 0], store.vars["cross_part/cross_mix_1/expert_0/kernel_u"])
    assert torch.equal(b[1], store.vars["cross_part/cross_mix_1/bias"])
    assert gate is store.vars["cross_part/cross_mix_gates/kernel"]


def test_defaults_and_the_gate_is_created_once_for_every_layer(store):
    from recalgorithm_b200 import layers as L
    x = torch.randn(2, 40)
    L.cross_network_mix(x, 3)
    gates = [k for k in store.vars if "gates" in k]
    assert gates == ["cross_mix_gates/kernel"] and tuple(store.vars[gates[0]].shape) == (40, 4)
    assert tuple(store.vars["cross_mix_2/expert_3/kernel_v"].shape) == (40, 32)
    assert store.calls[-1][1].shape == (3, 4, 40, 32)


def test_reuse_and_shape_conflict(store):
    from recalgorithm_b200 import layers as L
    x = torch.randn(2, 10)
    L.cross_network_mix(x, 2, 2, 4)
    n = len(store.vars)
    L.cross_network_mix(x, 2, 2, 4)
    assert len(store.vars) == n
    assert torch.equal(store.calls[0][1], store.calls[1][1]) and store.calls[0][5] is store.calls[1][5]
    with pytest.raises(ValueError, match="cross_mix_0/expert_0/kernel_v"):
        L.cross_network_mix(torch.randn(2, 12), 2, 2, 4)
    with pytest.raises(ValueError, match="cross_mix_0/expert_0/kernel_v"):
        L.cross_network_mix(x, 2, 2, 5)


def test_string_arguments_and_activation(store):
    from recalgorithm_b200 import layers as L
    x = torch.randn(3, 8)
    L.cross_network_mix(x, "2", num_experts="3", low_rank="5", activation="identity")
    assert tuple(store.vars["cross_mix_1/expert_2/kernel_c"].shape) == (5, 5)
    assert store.calls[-1][6] == "identity"


@pytest.mark.parametrize("kwargs", [dict(activation="relu"), dict(activation=None), dict(num_experts=0),
                                    dict(low_rank=0), dict(num_experts=5, low_rank=26), dict(num_experts=17, low_rank=1),
                                    dict(num_cross_layer=-1)])
def test_bad_values_raise(store, kwargs):
    from recalgorithm_b200 import layers as L
    args = dict(num_cross_layer=2)
    args.update(kwargs)
    with pytest.raises(ValueError):
        L.cross_network_mix(torch.randn(3, 8), **args)
    assert store.vars == {} and store.calls == []


def test_largest_mixture_is_accepted(store):
    from recalgorithm_b200 import layers as L
    with L.variable_scope("a"):
        L.cross_network_mix(torch.randn(3, 8), 1, num_experts=16, low_rank=8)
    with L.variable_scope("b"):
        L.cross_network_mix(torch.randn(3, 8), 1, num_experts=1, low_rank=128)
    assert len(store.calls) == 2


def test_zero_layers_returns_x0_without_a_variable_or_a_call(store):
    from recalgorithm_b200 import layers as L
    x = torch.randn(3, 8)
    assert L.cross_network_mix(x, 0) is x
    assert L.cross_network_mix(x, "0", num_experts=2, low_rank=3) is x
    assert store.vars == {} and store.calls == []
