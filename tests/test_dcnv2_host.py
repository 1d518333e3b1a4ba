"""CPU tests of the DCN-V2 host layers (layers.cross_layer_v2, layers.cross_network_v2) with the kernel call recorded:
variable names, shapes and initialisers, reuse and shape conflicts, string projection_dim, and num_cross_layer = 0."""
import math

import pytest
import torch


@pytest.fixture()
def store(monkeypatch):
    from recalgorithm_b200 import autograd, layers as L
    calls = []

    def fake_cross_v2(x0, w, u, b, rank, xl=None):
        calls.append((x0, w, u, b, rank, xl))
        return torch.zeros_like(x0)
    monkeypatch.setattr(autograd, "cross_v2", fake_cross_v2)
    st = L.set_default_store(L.VariableStore(device="cpu", seed=0))
    st.calls = calls
    yield st
    L.set_default_store(L.VariableStore(device="cpu"))


def _check_glorot(v, name):
    limit = math.sqrt(6.0 / sum(v.shape))
    v = v.detach()
    assert float(v.abs().max()) <= limit and float(v.std()) > 0.3 * limit, name


@pytest.mark.parametrize("projection_dim", [None, 16])
def test_layer_loop_variables_and_initialisers(store, projection_dim):
    from recalgorithm_b200 import layers as L
    B, d = 4, 82
    x0 = torch.randn(B, d)
    with L.variable_scope("cross_part"):
        x = x0
        for i in range(3):
            x = L.cross_layer_v2(x0, x, i, projection_dim=projection_dim)
    want = {}
    for i in range(3):
        if projection_dim is None:
            want[f"cross_part/cross_v2_{i}/kernel"] = (d, d)
        else:
            want[f"cross_part/cross_v2_{i}/kernel_v"] = (d, projection_dim)
            want[f"cross_part/cross_v2_{i}/kernel_u"] = (projection_dim, d)
        want[f"cross_part/cross_v2_{i}/bias"] = (d,)
    assert {k: tuple(v.shape) for k, v in store.vars.items()} == want
    for name, v in store.vars.items():
        if name.endswith("bias"):
            assert torch.count_nonzero(v) == 0
        else:
            _check_glorot(v, name)
    assert len(store.calls) == 3
    assert store.calls[0][5] is None and all(c[5] is not None for c in store.calls[1:])   # layer 0 starts at x0
    for c in store.calls:
        assert c[4] == (projection_dim or 0)
        assert c[1].shape == ((1, d, d) if projection_dim is None else (1, d, projection_dim))
        assert (c[2] is None) == (projection_dim is None)


@pytest.mark.parametrize("projection_dim", [None, 8])
def test_network_creates_what_the_loop_creates_in_one_call(store, projection_dim):
    from recalgorithm_b200 import layers as L
    x0 = torch.randn(3, 20)
    with L.variable_scope("loop"):
        x = x0
        for i in range(3):
            x = L.cross_layer_v2(x0, x, i, projection_dim)
    loop = {k[len("loop/"):]: tuple(v.shape) for k, v in store.vars.items()}
    store.calls.clear()
    with L.variable_scope("net"):
        L.cross_network_v2(x0, 3, projection_dim)
    net = {k[len("net/"):]: tuple(v.shape) for k, v in store.vars.items() if k.startswith("net/")}
    assert net == loop
    (call,) = store.calls
    x, w, u, b, rank, xl = call
    assert x is x0 and xl is None and rank == (projection_dim or 0)
    assert w.shape == ((3, 20, 20) if projection_dim is None else (3, 20, 8)) and b.shape == (3, 20)
    assert torch.equal(w[1], store.vars["net/cross_v2_1/kernel" if projection_dim is None else "net/cross_v2_1/kernel_v"])
    if projection_dim:
        assert u.shape == (3, 8, 20) and torch.equal(u[2], store.vars["net/cross_v2_2/kernel_u"])


def test_reuse_and_shape_conflict(store):
    from recalgorithm_b200 import layers as L
    x = torch.randn(2, 10)
    L.cross_layer_v2(x, x, 0)
    n = len(store.vars)
    L.cross_layer_v2(x, x, 0)
    assert len(store.vars) == n
    assert store.calls[0][1].data_ptr() == store.calls[1][1].data_ptr()        # views of the same variable
    with pytest.raises(ValueError, match="cross_v2_0/kernel"):
        L.cross_layer_v2(torch.randn(2, 12), torch.randn(2, 12), 0)
    L.cross_layer_v2(x, x, 1, projection_dim=4)
    with pytest.raises(ValueError, match="cross_v2_1/kernel_v"):
        L.cross_layer_v2(x, x, 1, projection_dim=5)


def test_string_projection_dim_and_bad_values(store):
    from recalgorithm_b200 import layers as L
    x = torch.randn(3, 8)
    L.cross_layer_v2(x, x, 7, projection_dim="4")
    assert tuple(store.vars["cross_v2_7/kernel_v"].shape) == (8, 4) and store.calls[-1][4] == 4
    L.cross_network_v2(x, "2", projection_dim="3")
    assert tuple(store.vars["cross_v2_1/kernel_u"].shape) == (3, 8)
    with pytest.raises(ValueError, match="projection_dim"):
        L.cross_layer_v2(x, x, 8, projection_dim=0)
    with pytest.raises(ValueError):
        L.cross_layer_v2(x, x, 8, projection_dim="two")


def test_zero_layers_returns_x0_without_a_variable_or_a_call(store):
    from recalgorithm_b200 import layers as L
    x = torch.randn(3, 8)
    assert L.cross_network_v2(x, 0) is x
    assert L.cross_network_v2(x, 0, projection_dim=4) is x
    assert store.vars == {} and store.calls == []
