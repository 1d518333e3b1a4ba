"""CPU tests of the DIEN host layer (layers.dien_interest_evolution) with the kernel launch stubbed: variable names, shapes and
initialisers, the cell-type selection, and the packing the C ABI expects."""
import math

import pytest
import torch


@pytest.fixture()
def store(monkeypatch):
    from recalgorithm_b200 import autograd, layers as L
    calls = []

    def fake_dien(seq, seq_len, target, params, nh, cell):
        calls.append((seq, seq_len, target, params, nh, cell))
        B, T = seq.shape[:2]
        return torch.zeros(B, nh), torch.full((B, T), 1.0 / T)
    monkeypatch.setattr(autograd, "dien", fake_dien)
    st = L.set_default_store(L.VariableStore(device="cpu", seed=0))
    st.calls = calls
    yield st
    L.set_default_store(L.VariableStore(device="cpu"))


@pytest.mark.parametrize("gru_type,cell", [("AGRU", 0), ("AUGRU", 1), ("augru", 0), ("GRU", 0), ("", 0)])
def test_dien_layer_variables_and_cell_selection(store, gru_type, cell):
    """custom_gru_type == "AUGRU" selects AUGRU, any other value AGRU (dien.py:220-223); gru_output_units may be a string."""
    from recalgorithm_b200 import layers as L, ops
    B, T, na, nh = 3, 5, 16, 8
    with L.variable_scope("seq_encoder"):
        out, att = L.dien_interest_evolution(torch.randn(B, T, na), torch.tensor([0, 2, 9]), torch.randn(B, na), str(nh),
                                             custom_gru_type=gru_type, return_attention_scores=True)
    assert out.shape == (B, nh) and att.shape == (B, T, 1)
    want = {"seq_encoder/" + n: s for n, s in zip(ops.DIEN_PARAM_ORDER, ops.dien_param_shapes(na, nh))}
    assert {k: tuple(v.shape) for k, v in store.vars.items()} == want
    assert want["seq_encoder/rnn/gru_cell/gates/kernel"] == (na + nh, 2 * nh)
    assert want["seq_encoder/rnn/gates/kernel"] == (2 * nh, 2 * nh)
    v = {k[len("seq_encoder/"):]: t.detach() for k, t in store.vars.items()}
    for name in ("rnn/gru_cell/gates/bias", "rnn/gates/bias"):                       # gate biases start at ones
        assert torch.equal(v[name], torch.ones_like(v[name])), name
    for name in ("rnn/gru_cell/candidate/bias", "rnn/candidate/bias"):               # candidate biases at zeros
        assert torch.equal(v[name], torch.zeros_like(v[name])), name
    for name in ("rnn/gru_cell/gates/kernel", "rnn/gru_cell/candidate/kernel", "attention_project_matrix", "rnn/gates/kernel",
                 "rnn/candidate/kernel"):                                             # glorot-uniform kernels
        fi, fo = v[name].shape
        lim = math.sqrt(6.0 / (fi + fo))
        assert 0.8 * lim < float(v[name].abs().max()) <= lim, name
    seq, seq_len, target, params, got_nh, got_cell = store.calls[-1]
    assert got_cell == cell and got_nh == nh and seq_len.dtype == torch.int64
    assert all(p is store.vars["seq_encoder/" + n] for p, n in zip(params, ops.DIEN_PARAM_ORDER))


def test_dien_layer_reuses_variables(store):
    from recalgorithm_b200 import layers as L
    x, n, e = torch.randn(2, 4, 6), torch.tensor([1, 4]), torch.randn(2, 6)
    L.dien_interest_evolution(x, n, e, 5)
    first = dict(store.vars)
    L.dien_interest_evolution(x, n, e, 5, custom_gru_type="AUGRU")
    assert store.vars == first and len(first) == 9


def test_dien_param_packing_round_trip():
    from recalgorithm_b200 import ops
    na, nh = 5, 3
    params = [torch.randn(s) for s in ops.dien_param_shapes(na, nh)]
    packed = ops.dien_pack_params(params, na, nh)
    assert packed.numel() == 3 * nh * (na + nh) + 3 * nh + nh * na + 6 * nh * nh + 3 * nh
    for a, b in zip(ops.dien_unpack_params(packed, na, nh), params):
        assert torch.equal(a, b)
    with pytest.raises(ValueError):
        ops.dien_pack_params(params[::-1], na, nh)
