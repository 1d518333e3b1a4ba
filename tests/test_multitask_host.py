"""CPU tests of the multi-task balancing host layer (recalgorithm_b200.multitask) with the kernel launches replaced by
recorders that compute the float64 restatement (tests/_mtl_ref.py): argument checks, the default shared parameters of MMoE
and PLE, the gradient routing of each balancer, and L(0) recorded once."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _mtl_ref as R  # noqa: E402

from recalgorithm_b200 import autograd, layers as L, multitask as MT, ops  # noqa: E402

METHOD_NAMES = {0: "sum", 1: "gradnorm", 2: "uncertainty"}


@pytest.fixture()
def calls(monkeypatch):
    rec = []

    def loss(x, z, method, task_param=None, want_grad=True):
        rec.append(("loss", method))
        p = None if task_param is None else task_param.detach().double().numpy()
        tl, tot, d, dp = R.loss_outputs(x.detach().double().numpy(), z.double().numpy(), METHOD_NAMES[method], p)
        f = lambda a: None if a is None else torch.tensor(np.asarray(a), dtype=torch.float32)
        return f(tl), f([tot]), f(d), f(dp)

    def gram(grads, gram=None):
        rec.append(("gram", grads))
        return grads.double() @ grads.double().T

    def combine(grads, gram, order, out=None, want_coef=False):
        rec.append(("combine", order.clone()))
        c = R.pcgrad_coef(gram.numpy(), order.tolist())
        res = torch.tensor(c @ grads.double().numpy(), dtype=torch.float32)
        if out is None:
            return res, None
        out.copy_(res)
        return out, None

    def update(gram, task_loss, initial_loss, weights, alpha, lr, want_d_weights=False):
        rec.append(("update", initial_loss))
        w, lg, _ = R.gradnorm_step(gram.numpy(), task_loss.numpy(), initial_loss.numpy(), weights.numpy(), alpha, lr)
        weights.copy_(torch.tensor(w, dtype=torch.float32))
        return torch.tensor([lg], dtype=torch.float32), None

    monkeypatch.setattr(ops, "multitask_sigmoid_ce", loss)
    monkeypatch.setattr(ops, "multitask_gram", gram)
    monkeypatch.setattr(ops, "pcgrad_combine", combine)
    monkeypatch.setattr(ops, "gradnorm_update", update)
    return rec


def _model(seed=0, T=3, B=6, P_shared=(4, 3)):
    """A tiny two-layer model: shared W (4,3) + b (3,), one head per task; returns (params, logits, labels)."""
    g = torch.Generator().manual_seed(seed)
    W = torch.nn.Parameter(torch.randn(P_shared, generator=g))
    b = torch.nn.Parameter(torch.randn(P_shared[1], generator=g))
    heads = [torch.nn.Parameter(torch.randn(P_shared[1], 1, generator=g)) for _ in range(T)]
    x = torch.randn(B, P_shared[0], generator=g)
    h = torch.tanh(x @ W + b)
    logits = [h @ v for v in heads]
    labels = [torch.rand(B, 1, generator=g) for _ in range(T)]
    return (W, b), heads, logits, labels


def test_method_strings_task_counts_and_list_lengths(calls):
    _, _, logits, labels = _model()
    for bad in ("Sum", "pcgrad", "", None):
        with pytest.raises(ValueError, match="method must be one of"):
            MT.multitask_sigmoid_ce(logits, labels, bad)
    with pytest.raises(ValueError, match="2 labels"):
        MT.multitask_sigmoid_ce(logits, labels[:2], "sum")
    with pytest.raises(ValueError, match="1 to 8"):
        MT.multitask_sigmoid_ce(logits * 3, labels * 3, "sum")
    with pytest.raises(ValueError, match="needs task_param"):
        MT.multitask_sigmoid_ce(logits, labels, "uncertainty")
    with pytest.raises(ValueError, match="needs task_param"):
        MT.multitask_sigmoid_ce(logits, labels, "gradnorm", torch.ones(2))
    shared = [torch.nn.Parameter(torch.ones(3))]
    for make in (lambda: MT.GradNorm(9, shared, lr=0.1), lambda: MT.PCGrad(9, shared, seed=0),
                 lambda: MT.UncertaintyWeighting(9, device="cpu"), lambda: MT.PCGrad(0, shared, seed=0)):
        with pytest.raises(ValueError, match="1 to 8"):
            make()
    with pytest.raises(ValueError, match="task losses"):
        MT.PCGrad(2, shared, seed=0).backward([torch.zeros(())] * 3)
    assert calls == []                                                  # every check happens before a launch


def test_task_losses_route_only_their_own_gradient(calls):
    """Each L_t is its own output: differentiating one leaves the other towers untouched (None), and the total's
    gradient is d_logits scaled by 1, w_t or exp(-s_t)."""
    _, heads, logits, labels = _model()
    s = torch.nn.Parameter(torch.tensor([0.3, -0.2, 0.1]))
    total, task_losses = MT.multitask_sigmoid_ce(logits, labels, "uncertainty", s)
    assert total.shape == () and len(task_losses) == 3 and all(t.shape == () for t in task_losses)
    g = torch.autograd.grad(task_losses[1], logits, retain_graph=True, allow_unused=True)
    assert g[0] is None and g[2] is None and g[1].shape == (6, 1)
    x = torch.stack([l.detach().reshape(-1) for l in logits]).double()
    z = torch.stack([y.reshape(-1) for y in labels]).double()
    _, _, d, d_s = R.loss_outputs(x.numpy(), z.numpy(), "uncertainty", s.detach().double().numpy())
    np.testing.assert_allclose(g[1].reshape(-1).numpy(), d[1], rtol=1e-6)
    total.backward()
    np.testing.assert_allclose(s.grad.numpy(), d_s, rtol=1e-6)
    for t, h in enumerate(heads):
        assert h.grad is not None and torch.isfinite(h.grad).all(), t


def test_default_shared_parameters_by_variable_name(monkeypatch):
    """MMoE: experts/expert_*/{kernel,bias}; PLE: the final layer's shared experts only (not the extraction network's, not
    the task-specific ones), in creation order."""
    monkeypatch.setattr(autograd, "mmoe", lambda x, we, be, wg: (torch.zeros(wg.shape[0], x.shape[0], we.shape[2]),
                                                                  torch.zeros(wg.shape[0], x.shape[0], we.shape[0])))
    monkeypatch.setattr(autograd, "ple", lambda x, we, be, wg, n, S, ext: (
        torch.zeros(x.shape[0], we.shape[2]) if ext else torch.zeros(len(n), x.shape[0], we.shape[2]),
        torch.zeros(x.shape[0], wg.shape[1])))
    try:
        st = L.set_default_store(L.VariableStore(device="cpu", seed=0))
        with L.variable_scope("mmoe"):
            L.mmoe_experts_gates(torch.zeros(2, 6), 3, 5, 2)
        got = MT.mmoe_shared_parameters()
        want = [f"mmoe/experts/expert_{i}/{k}" for i in range(3) for k in ("kernel", "bias")]
        assert [id(p) for p in got] == [id(st.vars[n]) for n in want]

        st = L.set_default_store(L.VariableStore(device="cpu", seed=0))
        net = L.extraction_network(torch.zeros(2, 6), ["a", "b"], [2, 1], 3, 4, "extract_network_0")
        L.ple_final_experts_gates(net, ["a", "b"], [2, 1], 3, 4)
        got = MT.ple_shared_parameters(st)
        want = [f"shared_experts_final/shared_expert_final_{i}/{k}" for i in range(3) for k in ("kernel", "bias")]
        assert [id(p) for p in got] == [id(st.vars[n]) for n in want]
        with pytest.raises(ValueError, match="no variable"):
            MT.mmoe_shared_parameters(st)
    finally:
        L.set_default_store(L.VariableStore(device="cpu"))


def _plain_grads(seed):
    shared, heads, logits, labels = _model(seed)
    total, _ = MT.multitask_sigmoid_ce(logits, labels, "sum")
    total.backward()
    return [p.grad.clone() for p in shared], [h.grad.clone() for h in heads]


def _per_task(shared, task_losses):
    return np.stack([torch.cat([g.reshape(-1) for g in torch.autograd.grad(l, shared, retain_graph=True)]).double().numpy()
                     for l in task_losses])


def test_pcgrad_writes_the_combination_into_the_shared_grads(calls):
    plain_shared, plain_heads = _plain_grads(0)
    shared, heads, logits, labels = _model(0)
    _, task_losses = MT.multitask_sigmoid_ce(logits, labels, "sum")
    g = _per_task(shared, task_losses)
    pc = MT.PCGrad(3, shared, seed=5)
    pc.backward(task_losses)
    order = [c for c in calls if c[0] == "combine"][-1][1].tolist()
    assert sorted(order) == [0, 1, 2]
    want, _ = R.pcgrad_vector(g, order)
    got = torch.cat([p.grad.reshape(-1) for p in shared]).double().numpy()
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-7)
    assert all(p.grad.untyped_storage().data_ptr() == pc.out.untyped_storage().data_ptr() for p in shared)  # views
    for h, want_h in zip(heads, plain_heads):
        assert torch.equal(h.grad, want_h)                              # non-shared: the plain-sum backward
    again = MT.PCGrad(3, shared, seed=5)                                # the same seed draws the same order
    _, _, logits, labels = _model(0)
    again.backward(MT.multitask_sigmoid_ce(logits, labels, "sum")[1])
    assert [c for c in calls if c[0] == "combine"][-1][1].tolist() == order


def test_gradnorm_records_initial_losses_once(calls):
    shared, heads, logits, labels = _model(1)
    gn = MT.GradNorm(3, shared, lr=0.05)
    with pytest.raises(RuntimeError, match="needs a loss"):
        gn.update()
    for step in range(3):
        if step:
            _, _, logits, labels = _model(1 + step)
        total = gn.loss(logits, labels)
        total.backward(retain_graph=True)
        gn.update()
    inits = [c[1] for c in calls if c[0] == "update"]
    assert len(inits) == 3 and all(i is inits[0] for i in inits)       # one device copy, made at the first update
    x = torch.stack([l.detach().reshape(-1) for l in _model(1)[2]]).double().numpy()
    z = torch.stack([y.reshape(-1) for y in _model(1)[3]]).double().numpy()
    np.testing.assert_allclose(gn.initial_loss.numpy(), R.loss_outputs(x, z, "sum")[0], rtol=1e-6)
    assert abs(float(gn.weights.sum()) - 3) < 1e-5


def _f64_logit_grads(logits, labels, method, param):
    """torch.autograd of the float64 restatement: d total / d logit[t] for every task."""
    x = torch.stack([l.detach().reshape(-1) for l in logits]).double().requires_grad_(True)
    z = torch.stack([y.reshape(-1) for y in labels]).double()
    p = None if param is None else param.detach().double()
    R.total(R.sigmoid_ce(x, z), method, p).backward()
    return x.grad.numpy()


@pytest.mark.parametrize("method", ["sum", "uncertainty", "gradnorm"])
def test_weighted_total_routes_its_weights_to_the_logits(calls, method):
    """The logit gradient of the total is d_logits scaled by 1, exp(-s_t) or w_t: against torch.autograd of the float64
    restatement at weights away from 1 (s = 0 and w = 1 would hide a wrong scale)."""
    _, _, logits, labels = _model(3)
    for l in logits:
        l.retain_grad()
    param = {"sum": None, "uncertainty": torch.nn.Parameter(torch.tensor([0.9, -0.6, 0.25])),
             "gradnorm": torch.tensor([1.7, 0.4, 0.9])}[method]
    total, _ = MT.multitask_sigmoid_ce(logits, labels, method, param)
    total.backward()
    got = np.stack([l.grad.reshape(-1).double().numpy() for l in logits])
    np.testing.assert_allclose(got, _f64_logit_grads(logits, labels, method, param), rtol=1e-6, atol=1e-9)


def test_gradnorm_trains_on_the_weights_from_before_each_update(calls):
    """Over three steps on one model, the logits' gradient of each step is w_t (d_logits) with the w that step's loss()
    saw, although update() changes w in place after the backward."""
    shared, heads, logits, labels = _model(4)
    gn = MT.GradNorm(3, shared, lr=0.3)
    for step in range(3):
        if step:
            W, b = shared
            h = torch.tanh(torch.randn(6, 4, generator=torch.Generator().manual_seed(step)) @ W + b)
            logits = [h @ v for v in heads]
        for l in logits:
            l.retain_grad()
        w_before = gn.weights.clone()
        gn.loss(logits, labels).backward(retain_graph=True)
        got = np.stack([l.grad.reshape(-1).double().numpy() for l in logits])   # before update()'s per-task passes
        gn.update()
        np.testing.assert_allclose(got, _f64_logit_grads(logits, labels, "gradnorm", w_before), rtol=1e-6, atol=1e-9)
        if step:
            assert not torch.equal(w_before, torch.ones(3))                  # the weights have moved away from 1
        assert not torch.equal(gn.weights, w_before)


def test_pcgrad_accumulates_like_an_ordinary_backward(calls):
    """Two backward() calls without zeroing: every .grad is the sum of the two steps' gradients, the shared ones the sum of
    the two PCGrad combinations (the first step's result is not overwritten by the second)."""
    shared, heads, _, labels = _model(5)
    pc = MT.PCGrad(3, shared, seed=1)
    W, b = shared
    want_shared, want_heads = 0, [0, 0, 0]
    for step in range(2):
        h = torch.tanh(torch.randn(6, 4, generator=torch.Generator().manual_seed(10 + step)) @ W + b)
        logits = [h @ v for v in heads]
        _, task_losses = MT.multitask_sigmoid_ce(logits, labels, "sum")
        g = _per_task(shared, task_losses)
        head_g = [torch.autograd.grad(sum(task_losses), v, retain_graph=True)[0] for v in heads]
        pc.backward(task_losses)
        order = [c for c in calls if c[0] == "combine"][-1][1].tolist()
        want_shared = want_shared + R.pcgrad_vector(g, order)[0]
        want_heads = [a + b_ for a, b_ in zip(want_heads, head_g)]
    got = torch.cat([p.grad.reshape(-1) for p in shared]).double().numpy()
    np.testing.assert_allclose(got, want_shared, rtol=1e-6, atol=1e-7)
    for h, want_h in zip(heads, want_heads):
        torch.testing.assert_close(h.grad, want_h, rtol=1e-6, atol=1e-7)
