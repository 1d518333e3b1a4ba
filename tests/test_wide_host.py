"""CPU tests of the Wide & Deep wide part's host layer with the kernel launches stubbed: crossed_column and its names, the
parse spec, indicator_dense over crossed columns (variables, blocks, the ragged key block handed to the kernel, the gradient
contract) and every ValueError of crossed_column, indicator_dense and optim.Ftrl."""
import math

import numpy as np
import pytest
import torch

import _wide_ref as R


def _cols():
    from recalgorithm_b200 import feature_column as fc
    userid = fc.categorical_column_with_vocabulary_file("userid", [b"u0", b"u1", b"u2"])
    tags = fc.categorical_column_with_vocabulary_file("manual_tag_list", [b"t0", b"t1", b"t2", b"t3"])
    return fc, userid, tags


@pytest.fixture()
def store(monkeypatch):
    """Stubs the two kernel wrappers with the NumPy restatement (float64 on the host) and records their arguments."""
    from recalgorithm_b200 import layers as L, ops
    calls = []

    def fake_fwd(values, offsets, nb, kernel, bias, hash_key=ops.CROSS_HASH_KEY):
        calls.append(("fwd", values, offsets, nb, hash_key))
        cr = R.crossed_ids(values.numpy(), offsets.numpy(), nb, hash_key)
        return torch.from_numpy(R.wide_fwd(cr, kernel.numpy(), 0.0)).float() + bias.reshape(1, 1)

    def fake_bwd(values, offsets, nb, d_logit, hash_key=ops.CROSS_HASH_KEY, want_bias=True):
        calls.append(("bwd", values, offsets, nb, hash_key))
        dk, db = R.wide_bwd(R.crossed_ids(values.numpy(), offsets.numpy(), nb, hash_key), d_logit.numpy(), nb)
        return torch.from_numpy(dk).float(), torch.tensor([db], dtype=torch.float32) if want_bias else None
    monkeypatch.setattr(ops, "crossed_indicator_fwd", fake_fwd)
    monkeypatch.setattr(ops, "crossed_indicator_bwd", fake_bwd)
    st = L.set_default_store(L.VariableStore(device="cpu", seed=0))
    st.calls = calls
    yield st
    L.set_default_store(L.VariableStore(device="cpu"))


def _features():
    # userid single-valued (b2 out of vocabulary), tags multi-valued (b1 empty, b3 holds a duplicate)
    return {"userid": ([b"u1", b"u0", b"zz", b"u2"], np.array([0, 1, 2, 3, 4])),
            "manual_tag_list": ([b"t0", b"t3", b"t1", b"t2", b"t2"], np.array([0, 2, 2, 3, 5]))}


def test_crossed_column_names_and_parse_spec():
    fc, userid, tags = _cols()
    cross = fc.crossed_column([userid, tags], hash_bucket_size=100000)
    assert cross.name == "manual_tag_list_X_userid" and cross.num_buckets == 100000 and cross.hash_key == 0xDECAFCAFFE
    ind = fc.indicator_column(cross)
    assert ind.name == "manual_tag_list_X_userid_indicator"
    spec = fc.make_parse_example_spec([ind, fc.indicator_column(userid), fc.numeric_column("x")])
    assert sorted(spec) == ["manual_tag_list", "userid", "x"]
    assert fc.crossed_column([userid, tags], 7, hash_key=5).hash_key == 5


def test_crossed_column_errors():
    fc, userid, tags = _cols()
    with pytest.raises(ValueError, match="hash_bucket_size"):
        fc.crossed_column([userid, tags], 1)
    with pytest.raises(ValueError, match="hash_bucket_size"):
        fc.crossed_column([userid, tags], 0)
    with pytest.raises(ValueError, match="length > 1"):
        fc.crossed_column([userid], 10)
    with pytest.raises(ValueError, match="string keys"):
        fc.crossed_column(["userid", tags], 10)
    with pytest.raises(ValueError, match="string keys"):
        fc.crossed_column([fc.embedding_column(userid, 4), tags], 10)
    with pytest.raises(ValueError, match="at most 4"):
        fc.crossed_column([userid, tags, userid, tags, userid], 10)
    with pytest.raises(ValueError, match="2\\*\\*31"):
        fc.crossed_column([userid, tags], 2 ** 31)


def test_crossed_indicator_dense_variables_and_values(store):
    """wide_and_deep.py:208-210: kernel (100000, 1) glorot-uniform with limit sqrt(6/100001), bias (1,) zeros, under
    wide_part/wide_part_variables; the keys reach the kernel as one ragged block of vocabulary ids (OOV -1 kept)."""
    from recalgorithm_b200 import layers as L
    fc, userid, tags = _cols()
    ind = fc.indicator_column(fc.crossed_column([userid, tags], hash_bucket_size=100000))
    with L.variable_scope("wide_part", reuse=L.AUTO_REUSE):
        logit = fc.indicator_dense(_features(), [ind], units=1, name="wide_part_variables", device="cpu")
    assert {k: tuple(v.shape) for k, v in store.vars.items()} == {"wide_part/wide_part_variables/kernel": (100000, 1),
                                                                  "wide_part/wide_part_variables/bias": (1,)}
    k = store.vars["wide_part/wide_part_variables/kernel"]
    lim = math.sqrt(6.0 / 100001)
    assert 0.99 * lim < float(k.detach().abs().max()) <= lim
    assert torch.count_nonzero(store.vars["wide_part/wide_part_variables/bias"]) == 0
    _, values, offsets, nb, hk = store.calls[0]
    assert nb == 100000 and hk == 0xDECAFCAFFE
    assert values.tolist() == [1, 0, -1, 2, 0, 3, 1, 2, 2]
    assert offsets.tolist() == [[0, 1, 2, 3, 4], [4, 6, 6, 7, 9]]
    cr = R.crossed_ids(values.numpy(), offsets.numpy(), nb)
    assert [len(c) for c in cr] == [2, 0, 1, 2]
    assert torch.allclose(logit.detach().double(), torch.from_numpy(R.wide_fwd(cr, k.detach().double().numpy(), 0.0)), rtol=1e-6)
    assert logit.shape == (4, 1)


def test_crossed_indicator_dense_gradients_and_blocks(store):
    """Two crossed columns: blocks of one (sum buckets, 1) kernel in name order; .grad of the kernel is the dense gradient of
    every block and .grad of the bias the sum of d_logit."""
    fc, userid, tags = _cols()
    a = fc.indicator_column(fc.crossed_column([userid, tags], hash_bucket_size=50))      # manual_tag_list_X_userid
    b = fc.indicator_column(fc.crossed_column([tags, userid, tags], hash_bucket_size=30))  # manual_tag_list_X_manual_tag_list_X_userid
    logit = fc.indicator_dense(_features(), [a, b], units=1, name="wide", device="cpu")
    kernel, bias = store.vars["wide/kernel"], store.vars["wide/bias"]
    assert kernel.shape == (80, 1)
    assert [c[3] for c in store.calls] == [30, 50]                  # name order: the 3-key cross sorts first
    g = torch.tensor([[1.0], [2.0], [-0.5], [3.0]])
    logit.backward(g)
    fb = _features()
    want = []
    for col, nb in ((b, 30), (a, 50)):
        vals, offs = fc.crossed_ragged_ids(fb, col.categorical_column)
        want.append(R.wide_bwd(R.crossed_ids(vals, offs, nb), g.numpy(), nb)[0])
    assert np.allclose(kernel.grad.numpy().ravel(), np.concatenate(want))
    assert float(bias.grad) == pytest.approx(5.5)


def test_indicator_dense_refuses_mixed_lists(store):
    fc, userid, tags = _cols()
    cross = fc.indicator_column(fc.crossed_column([userid, tags], hash_bucket_size=10))
    with pytest.raises(ValueError, match="mixes crossed and plain"):
        fc.indicator_dense(_features(), [cross, fc.indicator_column(userid)], device="cpu")
    with pytest.raises(ValueError, match="units=1"):
        fc.indicator_dense(_features(), [cross], units=2, device="cpu")


def test_ftrl_constructor_errors_and_slots():
    from recalgorithm_b200 import optim
    v = torch.nn.Parameter(torch.zeros(8))
    with pytest.raises(ValueError, match="initial_accumulator_value"):
        optim.Ftrl([v], 0.1, initial_accumulator_value=-0.1)
    with pytest.raises(ValueError, match="learning_rate_power"):
        optim.Ftrl([v], 0.1, learning_rate_power=0.5)
    with pytest.raises(ValueError, match="l1_regularization_strength"):
        optim.Ftrl([v], 0.1, l1_regularization_strength=-1.0)
    with pytest.raises(ValueError, match="l2_regularization_strength"):
        optim.Ftrl([v], 0.1, l2_regularization_strength=-1.0)
    with pytest.raises(ValueError, match="shrinkage"):
        optim.Ftrl([v], 0.1, l2_shrinkage_regularization_strength=0.1)
    opt = optim.Ftrl([v], 0.005)
    assert torch.equal(opt.get_slot(v, "accum"), torch.full((8,), 0.1)) and torch.equal(opt.get_slot(v, "linear"), torch.zeros(8))
    with pytest.raises(ValueError, match="No gradients"):
        opt.step()


def test_ftrl_step_skips_variables_without_gradient(monkeypatch):
    from recalgorithm_b200 import ops, optim
    seen = []
    monkeypatch.setattr(ops, "ftrl_apply", lambda var, acc, lin, g, lr, p, l1, l2: seen.append((var, acc, lin, g, lr, p, l1, l2)))
    a, b = torch.nn.Parameter(torch.zeros(4)), torch.nn.Parameter(torch.zeros(2))
    opt = optim.Ftrl([a, b], 0.2, learning_rate_power=-0.3, l1_regularization_strength=0.01, l2_regularization_strength=0.02)
    b.grad = torch.ones(2)
    opt.step()
    assert len(seen) == 1 and seen[0][0].data_ptr() == b.data_ptr() and torch.equal(seen[0][3], b.grad)
    assert seen[0][1] is opt.get_slot(b, "accum") and seen[0][2] is opt.get_slot(b, "linear") and seen[0][4:] == (0.2, -0.3, 0.01, 0.02)
    opt.zero_grad()
    assert a.grad is None and b.grad is None
