"""CPU tests of the FLEN host layers (layers.field_wise_bi_interaction and its fused-lookup form) with the kernel launches
stubbed: variable names, shapes and initialisers in the caller's scope, group numbering by first appearance, reuse, and the
argument errors."""
import pytest
import torch


@pytest.fixture()
def store(monkeypatch):
    from recalgorithm_b200 import autograd, layers as L
    calls = []

    def fake_fwbi(tile, groups, kmf, kfm, bmf, bfm):
        calls.append((groups, kmf, kfm, bmf, bfm))
        return torch.zeros(tile.shape[0], tile.shape[2])

    def fake_lookup(tables, ids, groups, kmf, kfm, bmf, bfm):
        calls.append((groups, kmf, kfm, bmf, bfm))
        return torch.zeros(ids.shape[0], ids.shape[1], tables.dim), torch.zeros(ids.shape[0], tables.dim)
    monkeypatch.setattr(autograd, "fwbi", fake_fwbi)
    monkeypatch.setattr(autograd, "lookup_fwbi", fake_lookup)
    st = L.set_default_store(L.VariableStore(device="cpu", seed=0))
    st.calls = calls
    yield st
    L.set_default_store(L.VariableStore(device="cpu"))


def test_variables_initialisers_and_group_numbering(store):
    from recalgorithm_b200 import layers as L
    B, F, D = 4, 6, 8
    with L.variable_scope("flen"):
        h = L.field_wise_bi_interaction(torch.randn(B, F, D), ["item", "user", "item", "context", "user", "user"])
    assert h.shape == (B, D)
    shapes = {k: tuple(v.shape) for k, v in store.vars.items()}
    assert shapes == {"flen/field_wise_bi_interaction/kernel_mf": (3,), "flen/field_wise_bi_interaction/kernel_fm": (3,),
                      "flen/field_wise_bi_interaction/bias_mf": (D,), "flen/field_wise_bi_interaction/bias_fm": (D,)}
    v = {k.split("/")[-1]: t.detach() for k, t in store.vars.items()}
    assert torch.equal(v["kernel_mf"], torch.ones(3)) and torch.equal(v["kernel_fm"], torch.full((3,), 0.5))
    assert torch.equal(v["bias_mf"], torch.zeros(D)) and torch.equal(v["bias_fm"], torch.zeros(D))
    assert store.calls[0][0] == (0, 1, 0, 2, 1, 1)                    # first appearance: item, user, context


def test_lookup_form_shares_the_variables(store):
    from recalgorithm_b200 import autograd, layers as L
    tables = autograd.EmbeddingTables([5, 5, 5], 4, device="cpu")
    tile, h = L.field_wise_bi_interaction_lookup(tables, torch.zeros(2, 3, dtype=torch.int64), (7, 7, 7))
    assert tile.shape == (2, 3, 4) and h.shape == (2, 4)
    assert {k: tuple(t.shape) for k, t in store.vars.items()} == {
        "field_wise_bi_interaction/kernel_mf": (0,), "field_wise_bi_interaction/kernel_fm": (1,),
        "field_wise_bi_interaction/bias_mf": (4,), "field_wise_bi_interaction/bias_fm": (4,)}
    n = len(store.vars)
    L.field_wise_bi_interaction(torch.randn(2, 3, 4), ["a", "a", "a"])
    assert len(store.vars) == n and all(a is b for a, b in zip(store.calls[0][1:], store.calls[1][1:]))
    assert store.calls[0][0] == (0, 0, 0)


def test_argument_errors(store):
    from recalgorithm_b200 import layers as L
    with pytest.raises(ValueError, match="3 entries but there are 4 fields"):
        L.field_wise_bi_interaction(torch.randn(2, 4, 4), ["a", "b", "c"])
    with pytest.raises(ValueError, match="at most 8"):
        L.field_wise_bi_interaction(torch.randn(2, 9, 4), list(range(9)))
    assert store.calls == [] and store.vars == {}
    L.field_wise_bi_interaction(torch.randn(2, 9, 4), list(range(8)) + [0])     # 8 groups is the bound, not past it
