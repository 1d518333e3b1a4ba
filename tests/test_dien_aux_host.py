"""CPU tests of the DIEN auxiliary-loss host layer (layers.dien_interest_evolution_aux, model_bodies.dien_logit with
use_auxiliary_loss) with the kernel launch stubbed: the projection variable, the string negative_sample_number, the
negative-row shape check, and that the nine seq_encoder variables are the ones dien_interest_evolution creates."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))


@pytest.fixture()
def store(monkeypatch):
    from recalgorithm_b200 import autograd, layers as L
    calls = []

    def fake_dien(seq, seq_len, target, params, nh, cell):
        B, T = seq.shape[:2]
        return torch.zeros(B, nh), torch.full((B, T), 1.0 / T)

    def fake_dien_aux(seq, seq_len, target, neg_seq, w_aux, params, nh, cell, T_neg):
        calls.append((seq, seq_len, target, neg_seq, w_aux, params, nh, cell, T_neg))
        B, T = seq.shape[:2]
        return torch.zeros(B, nh), torch.full((B, T), 1.0 / T), torch.zeros(())
    monkeypatch.setattr(autograd, "dien", fake_dien)
    monkeypatch.setattr(autograd, "dien_aux", fake_dien_aux)
    st = L.set_default_store(L.VariableStore(device="cpu", seed=0))
    st.calls = calls
    yield st
    L.set_default_store(L.VariableStore(device="cpu"))


def _inputs(B=3, T=5, na=16, T_neg=3):
    return torch.randn(B, T, na), torch.tensor([0, 2, 9]), torch.randn(B, na), torch.randn(B, (T - 1) * T_neg, na)


@pytest.mark.parametrize("gru_type,cell", [("AGRU", 0), ("AUGRU", 1), ("GRU", 0)])
def test_aux_layer_creates_the_same_nine_variables(store, gru_type, cell):
    """The nine seq_encoder variables are the very objects dien_interest_evolution creates (and reuses) in that scope."""
    from recalgorithm_b200 import layers as L, ops
    na, nh = 16, 8
    seq, n, e, neg = _inputs(na=na)
    w = torch.randn(na, nh)
    with L.variable_scope("seq_encoder"):
        out, att, aux = L.dien_interest_evolution_aux(seq, n, e, neg, w, str(nh), custom_gru_type=gru_type,
                                                      return_attention_scores=True)
    assert out.shape == (3, nh) and att.shape == (3, 5, 1) and aux.shape == ()
    created = dict(store.vars)
    assert list(created) == ["seq_encoder/" + k for k in ops.DIEN_PARAM_ORDER]
    *_, params, got_nh, got_cell, T_neg = store.calls[-1]
    assert got_cell == cell and got_nh == nh and T_neg == 3
    assert all(p is created["seq_encoder/" + k] for p, k in zip(params, ops.DIEN_PARAM_ORDER))
    with L.variable_scope("seq_encoder"):
        L.dien_interest_evolution(seq, n, e, nh, custom_gru_type=gru_type)
    assert store.vars == created                                          # same names, same objects, nothing new

    fresh = L.set_default_store(L.VariableStore(device="cpu", seed=0))    # same seed, the plain layer first
    with L.variable_scope("seq_encoder"):
        L.dien_interest_evolution(seq, n, e, nh)
    assert list(fresh.vars) == list(created)
    for k in created:
        assert torch.equal(fresh.vars[k], created[k]), k


def test_negative_sample_number_may_be_a_string(store):
    from recalgorithm_b200 import layers as L
    seq, n, e, neg = _inputs(T_neg=2)
    final, aux = L.dien_interest_evolution_aux(seq, n, e, neg, torch.randn(16, 8), 8, negative_sample_number="2")
    assert final.shape == (3, 8) and store.calls[-1][-1] == 2 and isinstance(store.calls[-1][-1], int)


@pytest.mark.parametrize("T_neg,rows", [(3, 4 * 2), (3, 5 * 3), (2, 4 * 3)])
def test_negative_rows_shape_is_checked(store, T_neg, rows):
    from recalgorithm_b200 import layers as L
    seq, n, e, _ = _inputs()
    with pytest.raises(ValueError, match="neg_sequnence_input"):
        L.dien_interest_evolution_aux(seq, n, e, torch.randn(3, rows, 16), torch.randn(16, 8), 8, negative_sample_number=T_neg)
    with pytest.raises(ValueError, match="aux_project_matrix"):
        L.dien_interest_evolution_aux(seq, n, e, torch.randn(3, 4 * 3, 16), torch.randn(8, 16), 8)


def test_dien_logit_creates_the_aux_projection_at_the_top_scope(store):
    """aux_loss/aux_project_matrix (na, nh), glorot-uniform, outside seq_encoder (dien.py:264, 268); the flag off creates
    nothing of the kind and returns two values."""
    import model_bodies as MB
    from recalgorithm_b200 import layers as L
    na, nh = 16, 8
    seq, n, e, neg = _inputs(na=na)
    dense_in, cat_in = torch.randn(3, 4), torch.randn(3, 6)
    out = MB.dien_logit(dense_in, cat_in, e, seq, n, gru_output_units=nh, use_auxiliary_loss=True, neg_sequnence_input=neg,
                        negative_sample_number="3")
    assert len(out) == 3 and out[0].shape == (3, 1) and out[2].shape == ()
    w = store.vars["aux_loss/aux_project_matrix"]
    assert tuple(w.shape) == (na, nh)
    lim = math.sqrt(6.0 / (na + nh))
    assert 0.8 * lim < float(w.detach().abs().max()) <= lim
    assert store.calls[-1][4] is w
    L.set_default_store(L.VariableStore(device="cpu", seed=0))
    out = MB.dien_logit(dense_in, cat_in, e, seq, n, gru_output_units=nh)
    assert len(out) == 2
    assert not any(k.startswith("aux_loss") for k in L.default_store().vars)
