"""GPU parity: the Wide & Deep wide part (csrc/wide.cu) against the NumPy restatement (tests/_wide_ref.py).

The hash is checked bit-exactly through the public entries alone: with kernel[h] = h and bias 0 the forward returns the
bucket id of a single cross exactly (ids < 2^24 are exact in float32) and otherwise the exact integer sum, and the backward
with d_logit = 1 returns the exact per-bucket histogram.  Forward and backward are also checked against float64 on random
weights, three FTRL steps on the wide layer against the float64 dense ApplyFtrl, and the Wide & Deep model body.

The file name sorts after test_gpu_tc_variants.py: see the docstring of test_gpu_expert_gate_mmoe.py for why the tests that
run before the profiler-tracing files must stay short."""
import os
import sys

import numpy as np
import pytest
import torch

import _wide_ref as R
from _util import TOL, assert_close, dev, elementwise_excess

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ragged(rng, B, K, max_len, vocab, empty_frac=0.0, oov_frac=0.1):
    """K keys of B samples: key 0 single-valued (userid-like), the others 1..max_len values (tags), with OOV -1 ids,
    duplicates (small vocabularies) and, when asked, empty keys."""
    vals, offs, base = [], [], 0
    for k in range(K):
        lens = np.ones(B, np.int64) if k == 0 else rng.integers(1, max_len + 1, B)
        lens[rng.random(B) < empty_frac] = 0
        v = rng.integers(0, vocab, int(lens.sum()))
        v[rng.random(v.size) < oov_frac] = -1
        vals.append(v)
        offs.append(np.concatenate([[0], np.cumsum(lens)]) + base)
        base += v.size
    return np.concatenate(vals).astype(np.int64), np.stack(offs).astype(np.int64)


def _run(values, offsets, nb, kernel, bias, d_logit):
    from recalgorithm_b200 import ops
    v, o = dev(values), dev(offsets)
    out = ops.crossed_indicator_fwd(v, o, nb, dev(kernel), dev(np.array([bias], np.float32)))
    dk, db = ops.crossed_indicator_bwd(v, o, nb, dev(d_logit))
    torch.cuda.synchronize()
    return out.cpu().numpy(), dk.cpu().numpy(), float(db.cpu()[0])


CASES = [  # (B, K, max tags, vocab, num_buckets, empty fraction)
    (1, 2, 1, 5, 100000, 0.0), (7, 2, 12, 3, 100000, 0.2), (300, 3, 4, 4, 1000, 0.1), (257, 4, 3, 6, 10 ** 7, 0.1),
    (65536, 2, 12, 1000, 100000, 0.05),
]


@pytest.mark.parametrize("B,K,L,vocab,nb,empty", CASES)
def test_hash_bit_exact(B, K, L, vocab, nb, empty):
    rng = np.random.default_rng(B * 10 + K)
    values, offsets = _ragged(rng, B, K, L, vocab, empty)
    cr = R.crossed_ids(values, offsets, nb)
    ones = np.ones(B, np.float32)
    out, dk, db = _run(values, offsets, nb, np.arange(nb, dtype=np.float32), 0.0, ones)
    assert np.array_equal(dk, R.histogram(cr, nb).astype(np.float32)), "histogram"
    assert db == float(B)
    want = np.array([float(c.sum()) for c in cr])
    exact = want < 2 ** 24                       # every partial sum of non-negative integers below 2^24 is exact in float32
    assert np.array_equal(out.ravel()[exact].astype(np.float64), want[exact])
    single = np.array([len(c) == 1 for c in cr])
    assert np.array_equal(out.ravel()[single].astype(np.int64), np.array([c[0] for c, s in zip(cr, single) if s], np.int64))


def test_hash_single_valued_keys_return_the_bucket():
    """With one value per key and kernel[h] = h, the logit is the bucket id itself, for every sample of a 65 536 batch."""
    rng = np.random.default_rng(5)
    B, nb = 65536, 100000
    for K in (2, 3, 4):
        values = rng.integers(-1, 1 << 20, B * K).astype(np.int64)
        offsets = (np.arange(B + 1)[None, :] + (np.arange(K) * B)[:, None]).astype(np.int64)
        out, _, _ = _run(values, offsets, nb, np.arange(nb, dtype=np.float32), 0.0, np.ones(B, np.float32))
        want = R.cross_bucket(values.reshape(K, B).T, nb)
        assert np.array_equal(out.ravel().astype(np.int64), want), K


def test_empty_batches():
    """An all-empty batch gives the bias and a zero gradient; B = 0 gives an empty logit and a zero kernel gradient."""
    from recalgorithm_b200 import ops
    nb = 1000
    kernel = np.random.default_rng(0).standard_normal(nb).astype(np.float32)
    values = np.array([3, 4], np.int64)
    offsets = np.array([[0, 1, 2, 2], [2, 2, 2, 2]], np.int64)           # key 1 is empty for every sample
    out, dk, db = _run(values, offsets, nb, kernel, 0.25, np.array([1.0, 2.0, 3.0], np.float32))
    assert np.array_equal(out.ravel(), np.full(3, 0.25, np.float32)) and not dk.any() and db == 6.0
    v0, o0 = dev(np.zeros(0, np.int64)), dev(np.zeros((2, 1), np.int64))
    out = ops.crossed_indicator_fwd(v0, o0, nb, dev(kernel), dev(np.array([0.5], np.float32)))
    dk0, db0 = ops.crossed_indicator_bwd(v0, o0, nb, dev(np.zeros(0, np.float32)))
    assert out.shape == (0, 1) and not dk0.any() and float(db0) == 0.0


@pytest.mark.parametrize("seed", range(4))
def test_fwd_bwd_against_float64(seed):
    rng = np.random.default_rng(100 + seed)
    B, K = int(rng.integers(1, 3000)), int(rng.integers(2, 5))
    nb = int(rng.choice([97, 100000, 10 ** 7]))
    values, offsets = _ragged(rng, B, K, int(rng.integers(1, 13)), int(rng.integers(2, 500)), 0.05)
    kernel = rng.uniform(-1, 1, nb).astype(np.float32)
    g = rng.standard_normal(B).astype(np.float32)
    out, dk, db = _run(values, offsets, nb, kernel, 0.1, g)
    cr = R.crossed_ids(values, offsets, nb)
    assert_close(out, R.wide_fwd(cr, kernel, np.float32(0.1)), TOL, "wide logit")
    want_dk, want_db = R.wide_bwd(cr, g, nb)
    assert_close(dk, want_dk, TOL, "d_kernel")
    assert abs(db - want_db) <= TOL * np.abs(g).sum()


def test_refusals():
    from recalgorithm_b200 import _lib, ops
    v, o = dev(np.zeros(2, np.int64)), dev(np.array([[0, 1], [1, 2]], np.int64))
    k, b = dev(np.zeros(10, np.float32)), dev(np.zeros(1, np.float32))
    o5 = dev(np.zeros((5, 2), np.int64))
    with pytest.raises(_lib.CtrInvalidArgument, match="K=5"):
        ops.crossed_indicator_fwd(v, o5, 10, k, b)
    with pytest.raises(_lib.CtrInvalidArgument, match="num_buckets=1"):
        ops.crossed_indicator_fwd(v, o, 1, k[:1], b)
    x = dev(np.zeros(8, np.float32))
    for kw in ({"lr": 0.0}, {"lr": 0.1, "lr_power": 0.5}, {"lr": 0.1, "l1": -1.0}, {"lr": 0.1, "l2": -1.0}):
        with pytest.raises(_lib.CtrInvalidArgument, match="ctr_ftrl_apply"):
            ops.ftrl_apply(x, x.clone(), x.clone(), x.clone(), **kw)


def _draw_ftrl_case(seed, B, nb, lr, p, l1, l2, steps=3):
    """Inputs, upstream gradients and the float64 trajectory; redrawn while any |linear| lies within 1e-5 relative of l1
    (float32 may take the other side of TF's select there, which is not a kernel error)."""
    for attempt in range(20):
        rng = np.random.default_rng(seed * 100 + attempt)
        values, offsets = _ragged(rng, B, 2, 12, 50, 0.05)
        kernel0 = rng.uniform(-1, 1, nb) * np.sqrt(6.0 / (nb + 1))
        kernel0 = kernel0.astype(np.float32)
        gs = [rng.standard_normal(B).astype(np.float32) for _ in range(steps)]
        cr = R.crossed_ids(values, offsets, nb)
        var, acc, lin = kernel0.astype(np.float64), np.full(nb, 0.1), np.zeros(nb)
        bvar, bacc, blin = 0.0, 0.1, 0.0
        traj, ok = [], True
        for g in gs:
            dk, db = R.wide_bwd(cr, g, nb)
            var, acc, lin = R.ftrl(var, acc, lin, dk, lr, p, l1, l2)
            bvar, bacc, blin = (float(x) for x in R.ftrl(bvar, bacc, blin, db, lr, p, l1, l2))
            if l1 > 0 and (np.any(np.abs(np.abs(lin) - l1) <= 1e-5 * l1) or abs(abs(blin) - l1) <= 1e-5 * l1):
                ok = False
                break
            traj.append((var.copy(), acc.copy(), lin.copy(), bvar, bacc, blin))
        if ok:
            return values, offsets, kernel0, gs, traj
    raise AssertionError("no draw keeps |linear| away from l1")


@pytest.mark.parametrize("p", [-0.5, -0.3])
@pytest.mark.parametrize("l1,l2", [(0.0, 0.0), (0.01, 0.0), (0.0, 0.5), (0.01, 0.5)])
def test_ftrl_three_steps_on_the_wide_layer(p, l1, l2):
    """indicator_dense over a crossed column, backward, Ftrl.step(): every row of var, accum and linear of the kernel and of
    the bias against the float64 dense ApplyFtrl after each of three steps.  After step 1, rows no cross touched are exactly 0."""
    from recalgorithm_b200 import feature_column as fc, layers as L, optim
    B, nb, lr = 512, 5000, 0.05
    values, offsets, kernel0, gs, traj = _draw_ftrl_case(int(-p * 10) + int(l1 * 100) + int(l2 * 10), B, nb, lr, p, l1, l2)
    userid = fc.categorical_column_with_vocabulary_file("userid", [b"x"])
    tags = fc.categorical_column_with_vocabulary_file("manual_tag_list", [b"y"])
    col = fc.indicator_column(fc.crossed_column([userid, tags], hash_bucket_size=nb))
    n0 = offsets[0, -1] - offsets[0, 0]
    feats = {"userid": (values[:n0], offsets[0] - offsets[0, 0]), "manual_tag_list": (values[n0:], offsets[1] - offsets[1, 0])}
    st = L.set_default_store(L.VariableStore(device="cuda", seed=0))
    try:
        with L.variable_scope("wide_part"):
            fc.indicator_dense(feats, [col], name="wide_part_variables")
        kernel, bias = st.vars["wide_part/wide_part_variables/kernel"], st.vars["wide_part/wide_part_variables/bias"]
        kernel.data.copy_(dev(kernel0).reshape(nb, 1))
        opt = optim.Ftrl([kernel, bias], lr, learning_rate_power=p, l1_regularization_strength=l1, l2_regularization_strength=l2)
        touched = R.histogram(R.crossed_ids(values, offsets, nb), nb) > 0
        for step, (g, (var, acc, lin, bvar, bacc, blin)) in enumerate(zip(gs, traj)):
            opt.zero_grad()
            with L.variable_scope("wide_part"):
                logit = fc.indicator_dense(feats, [col], name="wide_part_variables")
            logit.backward(dev(g).reshape(B, 1))
            opt.step()
            torch.cuda.synchronize()
            what = f"step {step + 1} p={p} l1={l1} l2={l2}"
            assert_close(kernel.detach().reshape(-1), var, TOL, what + " var")
            assert_close(opt.get_slot(kernel, "accum").reshape(-1), acc, TOL, what + " accum")
            assert_close(opt.get_slot(kernel, "linear").reshape(-1), lin, TOL, what + " linear")
            for got, want, name in ((bias, bvar, "bias"), (opt.get_slot(bias, "accum"), bacc, "bias accum"),
                                    (opt.get_slot(bias, "linear"), blin, "bias linear")):
                assert elementwise_excess(got.detach().reshape(1), np.array([want])) <= 1.0, (what, name)
            if step == 0:
                assert not kernel.detach().reshape(-1).cpu().numpy()[~touched].any(), "untouched rows must be exactly 0 after step 1"
                assert touched.sum() < nb
    finally:
        L.set_default_store(L.VariableStore())


def _wechat_records(rng, B, tag_vocab):
    """tf.train.SequenceExample records shaped like the reference ETL's: userid in the context, manual_tag_list in the
    feature_lists (one tag per step)."""
    from recalgorithm_b200 import io as cio
    recs = []
    for i in range(B):
        tags = [("bytes", [tag_vocab[int(t)]]) for t in rng.integers(0, len(tag_vocab), int(rng.integers(1, 5)))]
        ctx = {"userid": ("bytes", [b"u%d" % int(rng.integers(0, 40))]), "feedid": ("bytes", [b"f%d" % int(rng.integers(0, 30))]),
               "videoplayseconds": ("float", [float(rng.integers(0, 60))]), "read_comment": ("float", [float(rng.random() < 0.3)])}
        recs.append(cio.encode_sequence_example(ctx, {"manual_tag_list": tags}))
    return recs


@pytest.mark.parametrize("read_fl", [False, True])
def test_model_body_train_step(tmp_path, read_fl):
    """examples/model_bodies.wide_and_deep_logit over records parsed natively: forward, backward, one Ftrl step on the wide
    variables and one torch Adam step on the deep ones.  Without feature_lists (parity note 8) manual_tag_list parses empty:
    every sample has no crosses, the logit's wide part is the bias, and the first FTRL step zeroes the whole kernel."""
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import model_bodies as MB
    from recalgorithm_b200 import feature_column as fc, io as cio, layers as L, optim
    from recalgorithm_b200.io import native
    rng = np.random.default_rng(7)
    B = 256
    tag_vocab = [b"t%d" % i for i in range(20)]
    path = str(tmp_path / "w.tfrecord")
    cio.write_records(path, _wechat_records(rng, B, tag_vocab))
    userid = fc.categorical_column_with_vocabulary_file("userid", [b"u%d" % i for i in range(40)])
    feedid = fc.categorical_column_with_vocabulary_file("feedid", [b"f%d" % i for i in range(30)])
    tags = fc.categorical_column_with_vocabulary_file("manual_tag_list", tag_vocab)
    wide_cols = [fc.indicator_column(fc.crossed_column([userid, tags], hash_bucket_size=100000))]
    deep_cols = [fc.numeric_column("videoplayseconds"), fc.embedding_column(userid, 16), fc.embedding_column(feedid, 16),
                 fc.embedding_column(tags, 4)]
    label = fc.numeric_column("read_comment")
    buf, off, ln = native.read_tfrecord_file(path)
    feats = fc.parse_example_native(buf, off, ln, wide_cols + deep_cols + [label], read_feature_lists=read_fl)
    assert (feats["manual_tag_list"][1][-1] > 0) == read_fl
    st = L.set_default_store(L.VariableStore(device="cuda", seed=1))
    try:
        ctx = fc.LookupContext()
        logit = MB.wide_and_deep_logit(feats, wide_cols, deep_cols, hidden_units=(64, 32), ctx=ctx)
        assert logit.shape == (B, 1)
        wide_vars = [st.vars["wide_part/wide_part_variables/kernel"], st.vars["wide_part/wide_part_variables/bias"]]
        deep_vars = [v for k, v in st.vars.items() if k.startswith("deep_part/")]
        assert len(deep_vars) == 3 + 2 * 3 and len(st.vars) == len(deep_vars) + 2
        with L.variable_scope("wide_part"):
            wide_only = fc.indicator_dense(feats, wide_cols, name="wide_part_variables")
        if not read_fl:
            assert torch.equal(wide_only, wide_vars[1].detach().expand(B, 1))
        y = torch.from_numpy(np.asarray(feats["read_comment"], np.float32).reshape(B, 1)).cuda()
        loss = torch.nn.functional.binary_cross_entropy_with_logits(logit, y)
        loss.backward()
        for t, g in ctx.to_dense().items():
            next(v for v in deep_vars if id(v) == t).grad = g
        assert all(v.grad is not None for v in wide_vars + deep_vars)
        before = [v.detach().clone() for v in wide_vars + deep_vars]
        ftrl = optim.Ftrl(wide_vars, 0.005)
        adam = torch.optim.Adam(deep_vars, lr=0.001)
        ftrl.step()
        adam.step()
        torch.cuda.synchronize()
        # every wide variable moves; a deep variable moves when its gradient is not all zero (without feature_lists the tag
        # embedding table has no looked-up row)
        assert all(not torch.equal(b, v.detach()) for b, v in zip(before, wide_vars))
        assert all(not torch.equal(b, v.detach()) for b, v in zip(before[2:], deep_vars) if v.grad.any())
        kern = wide_vars[0].detach()
        if not read_fl:
            assert not kern.any(), "no crosses: the first FTRL step zeroes the whole kernel"
        else:
            assert kern.any() and (kern == 0).sum() > 0.9 * kern.numel()
    finally:
        L.set_default_store(L.VariableStore())
