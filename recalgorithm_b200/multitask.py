"""Multi-task loss balancing for MMoE and PLE: uncertainty weighting, GradNorm and PCGrad (Row MTL).

The reference sums its per-task losses (MMOE/mmoe.py:261-263, PLE/ple.py:251-254: ``tf.add_n``) and lists these three
methods as a to-do; the definitions are in include/ctr_b200.h ("Row MTL") and DESIGN §2.  Every computation is one launch of
a ``csrc/mtl.cu`` kernel through ``ops``; torch only stacks, slices and scales by per-task scalars.

Per-task gradients over the shared parameters come from ``torch.autograd.grad(L_t, shared, retain_graph=True)``, once per
task after the ordinary backward.  Those passes run only the nodes between the task losses and the shared parameters: the
task's own tower and the expert layer's backward, never the embedding lookup's backward, so ``EmbeddingTables.grad_slices``
still gets exactly one entry per step.  Embedding tables are never shared parameters here (their gradients are
IndexedSlices with duplicate rows).

Typical use, with ``logits`` from ``examples/model_bodies.mmoe_logits`` and ``labels`` the matching list of (B, 1) tensors:

    balancer = PCGrad(len(logits), mmoe_shared_parameters(), seed=0)
    total, task_losses = multitask_sigmoid_ce(logits, labels, "sum")
    balancer.backward(task_losses)          # every .grad set; the shared ones hold the PCGrad combination
"""
from __future__ import annotations

import re
from typing import List, Optional, Sequence

import torch

from . import layers as L
from . import ops

MAX_TASKS = ops.MTL_MAX_TASKS


def _check_lists(logits, labels):
    logits, labels = list(logits), list(labels)
    if len(logits) != len(labels):
        raise ValueError(f"{len(logits)} logits but {len(labels)} labels: one (B, 1) pair per task")
    if not 1 <= len(logits) <= MAX_TASKS:
        raise ValueError(f"{len(logits)} tasks: multi-task balancing supports 1 to {MAX_TASKS}")
    return logits, labels


class _MultitaskSigmoidCE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, method, task_param, labels, *logits):
        ctx.set_materialize_grads(False)
        T, B = len(logits), logits[0].shape[0]
        x = torch.stack([l.reshape(B) for l in logits])
        z = torch.stack([y.reshape(B) for y in labels]).to(x.dtype)
        task_loss, total, d_logits, d_param = ops.multitask_sigmoid_ce(x, z, method, task_param)
        if method == 0:
            scale = torch.ones((T,), dtype=x.dtype, device=x.device)
        elif method == 1:
            scale = task_param.detach().clone()                     # GradNorm updates w in place after the backward
        else:
            scale = torch.exp(-task_param.detach())
        ctx.save_for_backward(d_logits, d_param, scale)
        ctx.shape = (T, B, logits[0].shape)
        return (total.reshape(()),) + tuple(task_loss.unbind(0))

    @staticmethod
    def backward(ctx, grad_total, *grad_task_losses):
        d_logits, d_param, scale = ctx.saved_tensors
        T, B, shape = ctx.shape
        live = [grad_total is not None or g is not None for g in grad_task_losses]
        s = None                                                    # (T,): grad_total * c_t + grad_task_losses[t]
        if grad_total is not None:
            s = grad_total * scale
        if any(g is not None for g in grad_task_losses):
            zero = d_logits.new_zeros(())
            g = torch.stack([g if g is not None else zero for g in grad_task_losses])
            s = g if s is None else s + g
        d_x = d_logits * s.reshape(T, 1) if s is not None else None
        d_task_param = grad_total * d_param if grad_total is not None and d_param is not None else None
        return (None, d_task_param, None) + tuple(d_x[t].reshape(shape) if live[t] else None for t in range(T))


def multitask_sigmoid_ce(logits: Sequence[torch.Tensor], labels: Sequence[torch.Tensor], method: str,
                         task_param: Optional[torch.Tensor] = None):
    """Per-task mean sigmoid cross-entropies of T lists of (B, 1) logits and labels, and their balanced total, in one
    kernel launch.  Returns (total, task_losses): total is a scalar, task_losses a tuple of T scalars (separate outputs, so
    that differentiating one L_t runs only that task's tower).

    method: "sum" (total = sum_t L_t, the reference's add_n; task_param unused), "gradnorm" (sum_t w_t L_t with task_param =
    w) or "uncertainty" (sum_t exp(-s_t) L_t + s_t / 2 with task_param = s = log sigma^2).  Gradients reach the logits and,
    for "uncertainty", task_param; gradients arriving through task_losses are served too."""
    if method not in ops.MTL_METHODS:
        raise ValueError(f"method must be one of {sorted(ops.MTL_METHODS)}, got {method!r}")
    logits, labels = _check_lists(logits, labels)
    code = ops.MTL_METHODS[method]
    if code != 0:
        if task_param is None or tuple(task_param.shape) != (len(logits),):
            raise ValueError(f"method {method!r} needs task_param of shape ({len(logits)},)")
    out = _MultitaskSigmoidCE.apply(code, task_param if code != 0 else None, labels, *logits)
    return out[0], tuple(out[1:])


# ---------------------------------------------------------------------------------------------- shared parameters
MMOE_SHARED = r"(^|/)experts/expert_\d+/(kernel|bias)$"
PLE_SHARED = r"(^|/)shared_experts_final/shared_expert_final_\d+/(kernel|bias)$"


def _select(pattern: str, store: Optional[L.VariableStore]) -> List[torch.nn.Parameter]:
    store = store or L.default_store()
    params = [v for name, v in store.vars.items() if re.search(pattern, name)]
    if not params:
        raise ValueError(f"no variable of the store matches {pattern!r}: build the model before the balancer")
    return params


def mmoe_shared_parameters(store: Optional[L.VariableStore] = None) -> List[torch.nn.Parameter]:
    """The default shared parameters of an MMoE model, the last shared layer as in GradNorm's paper: every
    ``experts/expert_{i}/{kernel,bias}`` of the store, in creation order."""
    return _select(MMOE_SHARED, store)


def ple_shared_parameters(store: Optional[L.VariableStore] = None) -> List[torch.nn.Parameter]:
    """The default shared parameters of a PLE model: the final layer's shared experts
    ``shared_experts_final/shared_expert_final_{i}/{kernel,bias}``, in creation order.  Callers may add the extraction
    networks' variables."""
    return _select(PLE_SHARED, store)


class _SharedGradients:
    """The shared parameters flattened in list order into P floats, and one preallocated (T, P) buffer of per-task
    gradients."""

    def __init__(self, num_tasks: int, shared_parameters):
        if not 1 <= int(num_tasks) <= MAX_TASKS:
            raise ValueError(f"{num_tasks} tasks: multi-task balancing supports 1 to {MAX_TASKS}")
        self.num_tasks = int(num_tasks)
        self.params = list(shared_parameters)
        if not self.params:
            raise ValueError("shared_parameters is empty")
        self.sizes = [p.numel() for p in self.params]
        self.P = sum(self.sizes)
        dev = self.params[0].device
        self.grads = torch.empty((self.num_tasks, self.P), dtype=torch.float32, device=dev)

    def _views(self, flat: torch.Tensor):
        return [v.view_as(p) for v, p in zip(flat.split(self.sizes), self.params)]

    def per_task(self, task_losses) -> torch.Tensor:
        """Fills row t with d L_t / d shared; the last pass frees the graph."""
        task_losses = list(task_losses)
        if len(task_losses) != self.num_tasks:
            raise ValueError(f"{len(task_losses)} task losses for a balancer of {self.num_tasks} tasks")
        for t, loss in enumerate(task_losses):
            gs = torch.autograd.grad(loss, self.params, retain_graph=t + 1 < len(task_losses), allow_unused=True)
            for dst, g in zip(self._views(self.grads[t]), gs):
                if g is None:
                    dst.zero_()
                else:
                    dst.copy_(g)
        return self.grads


class UncertaintyWeighting(torch.nn.Module):
    """Kendall et al. (CVPR 2018) eq. 10: total = sum_t exp(-s_t) L_t + s_t / 2 with the learnable s = log sigma^2
    (``log_vars``, (T,), starts at 0); hand ``log_vars`` to the optimizer with the network's parameters."""

    def __init__(self, num_tasks: int, device="cuda"):
        super().__init__()
        if not 1 <= int(num_tasks) <= MAX_TASKS:
            raise ValueError(f"{num_tasks} tasks: multi-task balancing supports 1 to {MAX_TASKS}")
        self.log_vars = torch.nn.Parameter(torch.zeros(int(num_tasks), device=device))

    def forward(self, logits, labels) -> torch.Tensor:
        return multitask_sigmoid_ce(logits, labels, "uncertainty", self.log_vars)[0]


class GradNorm:
    """Chen et al. (ICML 2018) Algorithm 1.  The network trains on sum_t w_t L_t (``loss``); after its backward,
    ``update()`` takes the per-task gradients over the shared parameters, their Gram matrix and one GradNorm step on w
    (plain gradient descent at ``lr``, then renormalised to sum T; no clamp).  The first update records the task losses
    L(0).  The ordinary backward must keep the graph for the per-task passes: ``total.backward(retain_graph=True)``.
    ``update()`` never reads back to the host: the weights, L(0) and L_grad stay on the device."""

    def __init__(self, num_tasks: int, shared_parameters, lr: float, alpha: float = 1.5):
        self._shared = _SharedGradients(num_tasks, shared_parameters)
        dev = self._shared.grads.device
        self.lr, self.alpha = float(lr), float(alpha)
        self.weights = torch.ones(self._shared.num_tasks, dtype=torch.float32, device=dev)
        self.initial_loss: Optional[torch.Tensor] = None
        self.grad_loss: Optional[torch.Tensor] = None
        self._task_losses = None

    def loss(self, logits, labels) -> torch.Tensor:
        total, self._task_losses = multitask_sigmoid_ce(logits, labels, "gradnorm", self.weights)
        return total

    def update(self) -> torch.Tensor:
        """One GradNorm step on ``weights`` after the network's backward; returns L_grad (1,)."""
        if self._task_losses is None:
            raise RuntimeError("GradNorm.update() needs a loss() and its backward first")
        task_losses, self._task_losses = self._task_losses, None
        task_loss = torch.stack([l.detach() for l in task_losses])
        if self.initial_loss is None:
            self.initial_loss = task_loss.clone()
        gram = ops.multitask_gram(self._shared.per_task(task_losses))
        self.grad_loss, _ = ops.gradnorm_update(gram, task_loss, self.initial_loss, self.weights, self.alpha, self.lr)
        return self.grad_loss


class PCGrad:
    """Yu et al. (NeurIPS 2020) Algorithm 1 over the shared parameters, summed like add_n.  ``backward(task_losses)`` runs
    the ordinary backward of sum_t L_t (every parameter's .grad), the per-task gradients, their Gram matrix and the
    combination.  Like an ordinary backward it accumulates: each shared parameter's .grad becomes what it held before the
    call plus its slice of the combination (a view of this step's flat result when it held nothing).  The projection order
    is one permutation per step, drawn on the device from a ``torch.Generator`` seeded with ``seed``, so runs are
    reproducible."""

    def __init__(self, num_tasks: int, shared_parameters, seed: int):
        self._shared = _SharedGradients(num_tasks, shared_parameters)
        dev = self._shared.grads.device
        self.generator = torch.Generator(device=dev)
        self.generator.manual_seed(int(seed))
        self.out: Optional[torch.Tensor] = None
        self.order: Optional[torch.Tensor] = None

    def backward(self, task_losses) -> None:
        task_losses = list(task_losses)
        if len(task_losses) != self._shared.num_tasks:
            raise ValueError(f"{len(task_losses)} task losses for a balancer of {self._shared.num_tasks} tasks")
        params = self._shared.params
        prior = [p.grad for p in params]                 # the shared sum of this backward is replaced, not accumulated
        for p in params:
            p.grad = None
        torch.autograd.backward(task_losses, retain_graph=True)
        grads = self._shared.per_task(task_losses)
        T = self._shared.num_tasks
        keys = torch.rand((T,), generator=self.generator, device=grads.device)
        self.order = torch.argsort(keys).to(torch.int32)
        # a fresh buffer per step: a .grad left as a view of the previous step's result is never overwritten
        self.out, _ = ops.pcgrad_combine(grads, ops.multitask_gram(grads), self.order)
        for p, v, g0 in zip(params, self._shared._views(self.out), prior):
            p.grad = v if g0 is None else g0.add_(v)
