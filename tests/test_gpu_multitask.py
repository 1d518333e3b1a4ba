"""GPU: the multi-task balancing kernels (csrc/mtl.cu) against the float64 restatement (tests/_mtl_ref.py) at the 1e-5 bars
of tests/_util.py, their bitwise repeatability, and one MMoE / PLE training step with each balancer."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "examples"))
import _mtl_ref as R  # noqa: E402
from _util import TOL, assert_close, dev  # noqa: E402

METHODS = {"sum": 0, "gradnorm": 1, "uncertainty": 2}


def _loss_inputs(T, B, seed):
    """Logits: mostly N(0, 4), one in eight at +-80.  Labels: hard 0 / 1 or soft in [0.05, 0.95], so that a single
    element's loss is never a float32 cancellation of two numbers near 80."""
    rng = np.random.default_rng(seed)
    x = rng.normal(0, 4, (T, B))
    far = rng.random((T, B)) < 0.125
    x[far] = rng.choice([-80.0, 80.0], int(far.sum())) * rng.uniform(0.9, 1.0, int(far.sum()))
    z = np.where(rng.random((T, B)) < 0.5, rng.integers(0, 2, (T, B)), rng.uniform(0.05, 0.95, (T, B)))
    return x.astype(np.float32), z.astype(np.float32), rng


@pytest.mark.parametrize("method", list(METHODS))
@pytest.mark.parametrize("T", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("B", [0, 1, 9, 1031, 65536])
def test_multitask_loss_against_float64(method, T, B):
    from recalgorithm_b200 import ops
    x, z, rng = _loss_inputs(T, B, 1000 * T + B)
    p = None
    if method == "gradnorm":
        p = rng.uniform(0.5, 1.5, T).astype(np.float32)
    elif method == "uncertainty":
        p = rng.uniform(0.0, 1.0, T).astype(np.float32)
    args = (dev(x).reshape(T, B), dev(z).reshape(T, B), METHODS[method], None if p is None else dev(p))
    tl, tot, d, dp = ops.multitask_sigmoid_ce(*args)
    L, want_tot, want_d, want_dp = R.loss_outputs(x, z, method, p)
    assert_close(tl, L, TOL, f"task_loss {method} T={T} B={B}")
    assert_close(tot, np.array([want_tot]), TOL, f"total {method} T={T} B={B}")
    assert_close(d, want_d, TOL, f"d_logits {method} T={T} B={B}")
    if method == "sum":
        assert dp is None
    elif method == "gradnorm":
        assert_close(dp, want_dp, TOL, f"d_w T={T} B={B}")
    else:                                   # -exp(-s) L + 1/2 may cancel: its scale is exp(-s) L + 1/2
        scale = np.exp(-p.astype(np.float64)) * L + 0.5
        err = np.abs(dp.cpu().double().numpy() - want_dp) / scale
        assert err.max() <= TOL, f"d_s T={T} B={B}: {err.max():.3e}"
    if B == 0:
        assert torch.all(tl == 0)
    again = ops.multitask_sigmoid_ce(*args)
    for a, b in zip((tl, tot, d, dp), again):
        assert (a is None and b is None) or torch.equal(a, b), "two calls must give identical bits"


def _rows(T, P, seed, ld=None):
    """T gradient rows of P floats at row pitch ld = P + 1 (a column slice of a (T, P+1) buffer)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.randn((T, (P + 1) if ld is None else ld), device="cuda", generator=g)
    buf *= torch.rand((T, 1), device="cuda", generator=g) * 2 + 0.25
    return buf[:, :P]


@pytest.mark.parametrize("T", [1, 2, 3, 8])
@pytest.mark.parametrize("P", [0, 1, 5, 4097, 127488, 657920, (1 << 24) + 3])
def test_gram_against_float64(T, P):
    """P: 127 488 floats are MMoE's reference experts (3 x (82 x 512 + 512)), 657 920 PLE's default final shared experts
    (10 x (256 x 256 + 256)); 2^24 + 3 crosses the CTA cap of the first pass."""
    from recalgorithm_b200 import ops
    g = _rows(T, P, T * 7 + P)
    gram = ops.multitask_gram(g)
    g64 = g.double()
    want = g64 @ g64.T
    assert_close(gram, want, TOL, f"gram T={T} P={P}")
    assert torch.equal(gram, gram.T)
    assert torch.equal(ops.multitask_gram(g), gram), "two calls must give identical bits"


def _conflicting(T, P, seed):
    rng = np.random.default_rng(seed)
    u = rng.normal(0, 1, P)
    g = rng.choice([-1.0, 1.0], (T, 1)) * rng.uniform(0.5, 2, (T, 1)) * u + rng.normal(0, 0.7, (T, P))
    return g.astype(np.float32), rng


@pytest.mark.parametrize("T", [2, 3, 5, 8])
@pytest.mark.parametrize("P", [1, 4097, 127488])
def test_pcgrad_combine_against_float64(T, P):
    from recalgorithm_b200 import ops
    g, rng = _conflicting(T, P, 10 * T + P)
    buf = np.zeros((T, P + 1), np.float32)
    buf[:, :P] = g
    rows = dev(buf)[:, :P]
    gram = ops.multitask_gram(rows)
    for _ in range(3):
        order = rng.permutation(T)
        out, coef = ops.pcgrad_combine(rows, gram, dev(order.astype(np.int32)), want_coef=True)
        want, _ = R.pcgrad_vector(g, order)
        assert_close(coef, R.pcgrad_coef(gram.cpu().numpy(), order), 1e-12, f"coef T={T} P={P}")
        # out is a float64 sum of terms c_k g_k that may cancel to 0 (at P = 1 every conflict does): the element-wise bar
        # gets a floor of 1e-12 of the terms' magnitude
        err = np.abs(out.cpu().double().numpy() - want)
        mag = np.abs(coef.cpu().numpy()) @ np.abs(g.astype(np.float64))
        bound = TOL * (np.abs(want) + np.sqrt(np.mean(want * want))) + 1e-12 * mag
        assert np.all(err <= bound), f"pcgrad T={T} P={P} order={order.tolist()}: {(err / bound).max():.2f}x the bound"
        out2, _ = ops.pcgrad_combine(rows, gram, dev(order.astype(np.int32)))
        assert torch.equal(out, out2)


def test_pcgrad_combine_edges():
    """T = 1 is the row bit for bit (negative zeros included); an antiparallel pair gives exactly 0; a zero row triggers
    no projection and no NaN; P = 0 still writes coef."""
    from recalgorithm_b200 import ops
    one = _rows(1, 4099, 3)
    one[0, :7] = -0.0
    out, coef = ops.pcgrad_combine(one, ops.multitask_gram(one), dev(np.zeros(1, np.int32)), want_coef=True)
    assert torch.equal(out.view(torch.int32), one[0].contiguous().view(torch.int32)) and float(coef) == 1.0
    base = torch.linspace(-1, 2, 1000, device="cuda")
    anti = torch.stack([base, -2 * base])
    out, coef = ops.pcgrad_combine(anti, ops.multitask_gram(anti), dev(np.array([1, 0], np.int32)), want_coef=True)
    assert torch.all(out == 0), float(out.abs().max())
    zero = torch.stack([torch.zeros(1000, device="cuda"), base, 1 - base])
    for order in ([0, 1, 2], [2, 0, 1], [1, 2, 0]):
        out, _ = ops.pcgrad_combine(zero, ops.multitask_gram(zero), dev(np.array(order, np.int32)))
        want, _ = R.pcgrad_vector(zero.cpu().numpy(), order)
        assert torch.isfinite(out).all()
        assert_close(out, want, TOL, f"zero row, order {order}")
    empty = torch.zeros((3, 0), device="cuda")
    out, coef = ops.pcgrad_combine(empty, ops.multitask_gram(empty), dev(np.array([2, 1, 0], np.int32)), want_coef=True)
    assert out.numel() == 0 and torch.equal(coef.cpu(), torch.ones(3, dtype=torch.float64))


@pytest.mark.parametrize("T", [2, 3, 8])
def test_gradnorm_update_against_float64(T):
    from recalgorithm_b200 import ops
    rng = np.random.default_rng(T)
    L0 = rng.uniform(0.5, 1.0, T).astype(np.float32)
    w = torch.ones(T, device="cuda")
    w_ref = np.ones(T)
    for step in range(3):
        g = _rows(T, 5000, 50 + step + T)
        gram = ops.multitask_gram(g)
        L = (L0 * rng.uniform(0.6, 1.0, T)).astype(np.float32) if step else L0
        grad_loss, d_w = ops.gradnorm_update(gram, dev(L), dev(L0), w, 1.5, 0.05, want_d_weights=True)
        w_ref, lg, dw = R.gradnorm_step(gram.cpu().numpy(), L, L0, w_ref, 1.5, 0.05)
        assert_close(w, w_ref, TOL, f"weights after {step + 1} updates")
        assert_close(grad_loss, np.array([lg]), TOL, f"L_grad step {step + 1}")
        assert_close(d_w, dw, TOL, f"d_w step {step + 1}")
        assert abs(float(w.sum()) - T) <= TOL * T


def test_gradnorm_update_sign_zero():
    """On the target (T = 1, or two identical tasks) sign(0) = 0: no weight gradient, weights unchanged."""
    from recalgorithm_b200 import ops
    for T in (1, 2):
        g = _rows(1, 777, 9).expand(T, 777).contiguous()
        L = dev(np.full(T, 0.6, np.float32))
        w = torch.ones(T, device="cuda")
        grad_loss, d_w = ops.gradnorm_update(ops.multitask_gram(g), L, dev(np.full(T, 0.8, np.float32)), w, 1.5, 0.3,
                                             want_d_weights=True)
        assert torch.all(d_w == 0) and float(grad_loss) == 0 and torch.all(w == 1), (T, d_w, w)


def test_gradnorm_update_leaves_the_weights_when_every_loss_is_zero():
    """All current losses 0 (B = 0, or a batch fitted exactly): r_t is 0/0, so the step leaves w unchanged and writes a
    zero L_grad and d_w instead of NaN."""
    from recalgorithm_b200 import ops
    g = _rows(3, 500, 4)
    w = dev(np.array([1.2, 0.5, 1.3], np.float32))
    before = w.clone()
    grad_loss, d_w = ops.gradnorm_update(ops.multitask_gram(g), torch.zeros(3, device="cuda"),
                                         dev(np.full(3, 0.7, np.float32)), w, 1.5, 0.1, want_d_weights=True)
    assert torch.equal(w, before) and torch.all(d_w == 0) and float(grad_loss) == 0


def test_balancing_kernels_replay_in_a_cuda_graph():
    """The Gram, the PCGrad combination and the GradNorm update (with their workspace and output allocations) are
    captured in one CUDA graph; a replay on new gradients gives the bits of the eager calls."""
    from recalgorithm_b200 import ops
    T, P = 3, 40001
    g = _rows(T, P, 21).contiguous()
    L = dev(np.array([0.6, 0.5, 0.9], np.float32))
    L0 = dev(np.array([0.7, 0.8, 0.9], np.float32))
    order = dev(np.array([2, 0, 1], np.int32))
    w = torch.ones(T, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                               # warm-up outside the capture, as torch recommends
        ops.pcgrad_combine(g, ops.multitask_gram(g), order)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gram = ops.multitask_gram(g)
        out, _ = ops.pcgrad_combine(g, gram, order)
        grad_loss, _ = ops.gradnorm_update(gram, L, L0, w, 1.5, 0.05)
    g.copy_(_rows(T, P, 22))
    w.fill_(1.0)
    graph.replay()
    torch.cuda.synchronize()
    w_eager = torch.ones(T, device="cuda")
    gram_e = ops.multitask_gram(g)
    out_e, _ = ops.pcgrad_combine(g, gram_e, order)
    grad_loss_e, _ = ops.gradnorm_update(gram_e, L, L0, w_eager, 1.5, 0.05)
    assert torch.equal(gram, gram_e) and torch.equal(out, out_e)
    assert torch.equal(w, w_eager) and torch.equal(grad_loss, grad_loss_e)


# ------------------------------------------------------------------------------------------------------------ end to end
def _model(kind, B=2048, seed=0):
    """mmoe_logits at the reference shape (d = 82, E = 3, H = 512, T = 3) or ple_logits at its defaults, over a lookup of
    10 fields x 8 and 2 dense features (d = 82)."""
    import model_bodies as M
    from recalgorithm_b200 import autograd, layers as L
    store = L.set_default_store(L.VariableStore(device="cuda", seed=seed))
    gen = torch.Generator(device="cuda").manual_seed(seed)
    tables = autograd.EmbeddingTables([100] * 10, 8, device="cuda", generator=gen)
    ids = torch.randint(-1, 100, (B, 10), device="cuda", generator=gen)
    dense = torch.randn((B, 2), device="cuda", generator=gen)
    names = ("read_comment", "like", "click_avatar")
    labels = {n: (torch.rand((B, 1), device="cuda", generator=gen) < 0.3).float() for n in names}
    cat = autograd.lookup(tables, ids).reshape(B, -1)
    if kind == "mmoe":
        logits, _ = M.mmoe_logits(dense, cat, labels, task_names=names, num_experts=3, expert_hidden_units=512)
    else:
        logits, _ = M.ple_logits(dense, cat, labels, task_names=names)
    return store, tables, logits, [labels[n] for n in names]


def _shared(kind, store):
    from recalgorithm_b200 import multitask as MT
    return MT.mmoe_shared_parameters(store) if kind == "mmoe" else MT.ple_shared_parameters(store)


def _plain_step(kind):
    from recalgorithm_b200 import multitask as MT
    store, tables, logits, labels = _model(kind)
    total, _ = MT.multitask_sigmoid_ce(logits, labels, "sum")
    total.backward()
    return ({n: v.grad.clone() for n, v in store.vars.items()}, tables.grad_slices[0].values.clone())


@pytest.mark.parametrize("kind", ["mmoe", "ple"])
@pytest.mark.parametrize("balancer", ["uncertainty", "gradnorm", "pcgrad"])
def test_one_balanced_step(kind, balancer):
    from recalgorithm_b200 import multitask as MT
    plain, plain_slices = _plain_step(kind)
    store, tables, logits, labels = _model(kind)
    shared = _shared(kind, store)
    shared_ids = {id(p) for p in shared}
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        if balancer == "uncertainty":
            uw = MT.UncertaintyWeighting(3)
            total, task_losses = MT.multitask_sigmoid_ce(logits, labels, "uncertainty", uw.log_vars)
        elif balancer == "gradnorm":
            gn = MT.GradNorm(3, shared, lr=0.025)
            total = gn.loss(logits, labels)
            task_losses = gn._task_losses
        else:
            pc = MT.PCGrad(3, shared, seed=11)
            total, task_losses = MT.multitask_sigmoid_ce(logits, labels, "sum")
    finally:
        torch.cuda.set_sync_debug_mode(0)
    # the per-task gradients the restatement is applied to (autograd.grad does not touch .grad or the lookup)
    per_task = torch.stack([torch.cat([g.reshape(-1) for g in torch.autograd.grad(l, shared, retain_graph=True)])
                            for l in task_losses]).double().cpu().numpy()
    L = torch.stack([l.detach() for l in task_losses]).double().cpu().numpy()
    torch.cuda.set_sync_debug_mode("error")
    try:
        if balancer == "pcgrad":
            pc.backward(task_losses)
        else:
            total.backward(retain_graph=balancer == "gradnorm")
            if balancer == "gradnorm":
                gn.update()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    got = torch.cat([p.grad.reshape(-1) for p in shared]).double().cpu().numpy()
    if balancer == "pcgrad":
        want, _ = R.pcgrad_vector(per_task, pc.order.cpu().tolist())
        assert_close(got, want, TOL, f"{kind} PCGrad shared gradient")
    else:
        # one backward of the summed towers against the sum of T per-task backwards of the expert layer: both batch-reduced
        # by the layer's weight-gradient kernel, so held to the max-norm bar (as in test_gpu_expert_gate_*.py)
        assert_close(got, per_task.sum(axis=0), TOL, f"{kind} {balancer} shared gradient", elementwise=False)
    if balancer == "uncertainty":
        assert_close(uw.log_vars.grad, -L + 0.5, TOL, f"{kind} d log_vars")
    if balancer == "gradnorm":
        gram = per_task @ per_task.T
        w, _, _ = R.gradnorm_step(gram, L, L, np.ones(3), 1.5, 0.025)
        assert_close(gn.weights, w, TOL, f"{kind} GradNorm weights")
        assert abs(float(gn.weights.sum()) - 3) <= 3 * TOL
    assert len(tables.grad_slices) == 1
    # At s = 0 and w = 1 every balancer trains the rest of the network on the plain sum.  The towers and the lookup's
    # gradient come out bit for bit; the expert-gate layer's gates and task experts are summed through atomics in its
    # weight-gradient kernel, whose order differs between runs, so they are held to the 1e-5 bars instead.
    assert torch.equal(tables.grad_slices[0].values, plain_slices)
    for n, v in store.vars.items():
        if id(v) in shared_ids:
            continue
        if n.startswith("tower/"):
            assert torch.equal(v.grad, plain[n]), n
        else:
            assert_close(v.grad, plain[n], TOL, n, elementwise=False)


@pytest.mark.parametrize("kind", ["mmoe", "ple"])
@pytest.mark.parametrize("balancer", ["uncertainty", "gradnorm"])
def test_weighted_step_away_from_one(kind, balancer):
    """One step at s != 0 / w != 1, where the weights change what the network trains on: each logit's gradient is
    c_t (sigmoid(x) - z) / B with c_t = exp(-s_t) or w_t, and the shared gradient is sum_t c_t d L_t / d W."""
    from recalgorithm_b200 import multitask as MT
    store, tables, logits, labels = _model(kind)
    shared = _shared(kind, store)
    for l in logits:
        l.retain_grad()
    if balancer == "uncertainty":
        uw = MT.UncertaintyWeighting(3)
        with torch.no_grad():
            uw.log_vars.copy_(torch.tensor([0.8, -0.5, 0.3]))
        total, task_losses = MT.multitask_sigmoid_ce(logits, labels, "uncertainty", uw.log_vars)
        c = np.exp(-np.array([0.8, -0.5, 0.3], np.float32).astype(np.float64))
    else:
        gn = MT.GradNorm(3, shared, lr=0.025)
        gn.weights.copy_(torch.tensor([1.6, 0.3, 1.1]))
        total = gn.loss(logits, labels)
        task_losses = gn._task_losses
        c = np.array([1.6, 0.3, 1.1], np.float32).astype(np.float64)
    per_task = torch.stack([torch.cat([g.reshape(-1) for g in torch.autograd.grad(l, shared, retain_graph=True)])
                            for l in task_losses]).double().cpu().numpy()
    for l in logits:
        l.grad = None                                           # the per-task passes above reach the logits too
    total.backward()
    B = logits[0].shape[0]
    for t, (l, y) in enumerate(zip(logits, labels)):
        x64, z64 = l.detach().double().cpu().numpy(), y.double().cpu().numpy()
        assert_close(l.grad, c[t] * (1 / (1 + np.exp(-x64)) - z64) / B, TOL, f"{kind} {balancer} d logit {t}")
    got = torch.cat([p.grad.reshape(-1) for p in shared]).double().cpu().numpy()
    assert_close(got, c @ per_task, TOL, f"{kind} {balancer} shared gradient", elementwise=False)
