"""CPU tests of the DeepCrossing host layer (layers.residual_unit) with the kernel launch stubbed: variable names, shapes and
initialisers, index=None, and a string internal_dim."""
import math

import pytest
import torch


@pytest.fixture()
def store(monkeypatch):
    from recalgorithm_b200 import autograd, layers as L
    calls = []

    def fake_residual_unit(x, w0, b0, w1, b1):
        calls.append((x, w0, b0, w1, b1))
        return torch.zeros_like(x)
    monkeypatch.setattr(autograd, "residual_unit", fake_residual_unit)
    st = L.set_default_store(L.VariableStore(device="cpu", seed=0))
    st.calls = calls
    yield st
    L.set_default_store(L.VariableStore(device="cpu"))


def test_residual_unit_variables_and_initialisers(store):
    """Two units in residual_module (deepcrossing.py:154-157): kernels glorot-uniform, both tf.layers.dense biases zero."""
    from recalgorithm_b200 import layers as L
    B, d, H = 5, 82, 256
    x = torch.randn(B, d)
    with L.variable_scope("residual_module"):
        net = x
        for i in range(2):
            net = L.residual_unit(net, H, index=i)
    assert net.shape == (B, d)
    want = {}
    for i in range(2):
        want.update({f"residual_module/dense_{i}_0/kernel": (d, H), f"residual_module/dense_{i}_0/bias": (H,),
                     f"residual_module/dense_{i}_1/kernel": (H, d), f"residual_module/dense_{i}_1/bias": (d,)})
    assert {k: tuple(v.shape) for k, v in store.vars.items()} == want
    for name, v in store.vars.items():
        if name.endswith("bias"):
            assert torch.count_nonzero(v) == 0, name
        else:
            lim = math.sqrt(6.0 / sum(v.shape))
            assert 0.9 * lim < float(v.abs().max()) <= lim, name
    x0, w0, b0, w1, b1 = store.calls[0]
    assert x0 is x and w0 is store.vars["residual_module/dense_0_0/kernel"] and b1 is store.vars["residual_module/dense_0_1/bias"]
    assert store.calls[1][0] is not x


def test_residual_unit_index_none_and_string_width(store):
    """index=None names the variables dense_None_0 / dense_None_1 (an f-string of None); internal_dim goes through int()."""
    from recalgorithm_b200 import layers as L
    L.residual_unit(torch.randn(3, 4), "7")
    assert {k: tuple(v.shape) for k, v in store.vars.items()} == {
        "dense_None_0/kernel": (4, 7), "dense_None_0/bias": (7,), "dense_None_1/kernel": (7, 4), "dense_None_1/bias": (4,)}
    with pytest.raises(TypeError):
        L.residual_unit(torch.randn(3, 4), None, index=1)


def test_residual_unit_reuses_variables(store):
    from recalgorithm_b200 import layers as L
    x = torch.randn(2, 6)
    L.residual_unit(x, 3, index=0)
    first = dict(store.vars)
    L.residual_unit(x, 3, index=0)
    assert store.vars == first and len(first) == 4
