"""CPU tests of the MMoE host layer (layers.mmoe_experts_gates) with the kernel launch stubbed: variable names, shapes and
initialisers, the packed layout handed to the kernels, int() on the sizes, and the returned views."""
import math

import pytest
import torch


@pytest.fixture()
def store(monkeypatch):
    from recalgorithm_b200 import autograd, layers as L
    calls = []

    def fake_mmoe(x, w_experts, b_experts, w_gates):
        calls.append((x, w_experts, b_experts, w_gates))
        T, E, H = w_gates.shape[0], w_experts.shape[0], w_experts.shape[2]
        towers = torch.arange(T, dtype=torch.float32).reshape(T, 1, 1).expand(T, x.shape[0], H).contiguous()
        return towers, torch.full((T, x.shape[0], E), 1.0 / E)
    monkeypatch.setattr(autograd, "mmoe", fake_mmoe)
    st = L.set_default_store(L.VariableStore(device="cpu", seed=0))
    st.calls = calls
    yield st
    L.set_default_store(L.VariableStore(device="cpu"))


def test_mmoe_variables_and_initialisers(store):
    """mmoe.py:207-224 at the reference default: expert kernels glorot-uniform, expert biases zero, gate kernels glorot-uniform
    and no gate bias; gates are named by task index."""
    from recalgorithm_b200 import layers as L
    B, d, E, H, T = 5, 82, 3, 512, 3
    x = torch.randn(B, d)
    towers = L.mmoe_experts_gates(x, E, H, T)
    want = {**{f"experts/expert_{i}/kernel": (d, H) for i in range(E)}, **{f"experts/expert_{i}/bias": (H,) for i in range(E)},
            **{f"gates/gate_{t}/kernel": (d, E) for t in range(T)}}
    assert {k: tuple(v.shape) for k, v in store.vars.items()} == want
    for name, v in store.vars.items():
        if name.endswith("bias"):
            assert torch.count_nonzero(v) == 0, name
        else:
            lim = math.sqrt(6.0 / sum(v.shape))
            assert 0.85 * lim < float(v.detach().abs().max()) <= lim, name
    x0, we, be, wg = store.calls[0]
    assert x0 is x and we.shape == (E, d, H) and be.shape == (E, H) and wg.shape == (T, d, E)
    for i in range(E):
        assert torch.equal(we[i], store.vars[f"experts/expert_{i}/kernel"])
        assert torch.equal(be[i], store.vars[f"experts/expert_{i}/bias"])
    for t in range(T):
        assert torch.equal(wg[t], store.vars[f"gates/gate_{t}/kernel"])
    assert len(towers) == T
    for t, tw in enumerate(towers):
        assert tw.shape == (B, H) and tw.is_contiguous() and torch.all(tw == t)


def test_mmoe_sizes_go_through_int_and_gates_on_request(store):
    from recalgorithm_b200 import layers as L
    towers, gates = L.mmoe_experts_gates(torch.randn(4, 6), "2", 7.0, "3", return_gates=True)
    assert len(towers) == 3 and len(gates) == 3 and gates[0].shape == (4, 2) and towers[0].shape == (4, 7)
    assert set(store.vars) == {"experts/expert_0/kernel", "experts/expert_0/bias", "experts/expert_1/kernel",
                               "experts/expert_1/bias", "gates/gate_0/kernel", "gates/gate_1/kernel", "gates/gate_2/kernel"}
    with pytest.raises(TypeError):
        L.mmoe_experts_gates(torch.randn(4, 6), None, 7, 3)


def test_mmoe_scope_and_reuse(store):
    """The variables live in the caller's scope; a second call reuses them."""
    from recalgorithm_b200 import layers as L
    x = torch.randn(2, 5)
    with L.variable_scope("outer"):
        L.mmoe_experts_gates(x, 2, 3, 2)
        first = dict(store.vars)
        L.mmoe_experts_gates(x, 2, 3, 2)
    assert store.vars == first and len(first) == 6 and all(k.startswith("outer/") for k in first)


def test_mmoe_gradients_reach_every_variable(monkeypatch, store):
    """torch.stack routes the packed gradients back to each variable."""
    from recalgorithm_b200 import autograd, layers as L

    def torch_mmoe(x, we, be, wg):
        h = torch.relu(torch.einsum("bd,edh->ebh", x, we) + be[:, None, :])
        p = torch.softmax(torch.einsum("bd,tde->tbe", x, wg), dim=-1)
        return torch.einsum("tbe,ebh->tbh", p, h), p.detach()
    monkeypatch.setattr(autograd, "mmoe", torch_mmoe)
    towers = L.mmoe_experts_gates(torch.randn(6, 5), 2, 4, 3)
    sum(t.square().sum() for t in towers).backward()
    for name, v in store.vars.items():
        assert v.grad is not None and v.grad.shape == v.shape, name
