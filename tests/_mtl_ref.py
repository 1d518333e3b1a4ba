"""Float64 restatement of the multi-task balancing definitions (include/ctr_b200.h, Row MTL; DESIGN §2): the per-task
sigmoid cross-entropies and the three totals, GradNorm's step (Chen et al. 2018, Algorithm 1), and PCGrad (Yu et al. 2020,
Algorithm 1) both in the paper's vector form and in the coefficient form the kernel solves.  numpy float64 throughout;
the functions marked "torch" take float64 tensors so that the CPU tests can differentiate them."""
import numpy as np
import torch


def sigmoid_ce(x, z):
    """torch: per-task mean of TF's stable sigmoid cross-entropy over (T,B): L (T,)."""
    return (torch.clamp(x, min=0) - x * z + torch.log1p(torch.exp(-x.abs()))).mean(dim=1)


def total(L, method, param=None):
    """torch: "sum" sum_t L_t; "gradnorm" sum_t w_t L_t; "uncertainty" sum_t exp(-s_t) L_t + s_t / 2."""
    if method == "sum":
        return L.sum()
    if method == "gradnorm":
        return (param * L).sum()
    return (torch.exp(-param) * L + 0.5 * param).sum()


def loss_outputs(x, z, method, param=None):
    """numpy float64 (task_loss (T,), total, d_logits (T,B) unweighted, d_task_param (T,) | None) of the loss kernel."""
    x, z = np.asarray(x, np.float64), np.asarray(z, np.float64)
    T, B = x.shape
    L = (np.maximum(x, 0) - x * z + np.log1p(np.exp(-np.abs(x)))).mean(axis=1) if B else np.zeros(T)
    d = (1 / (1 + np.exp(-x)) - z) / max(B, 1)
    if method == "sum":
        return L, L.sum(), d, None
    p = np.asarray(param, np.float64)
    if method == "gradnorm":
        return L, (p * L).sum(), d, L
    e = np.exp(-p)
    return L, (e * L + 0.5 * p).sum(), d, -e * L + 0.5


def gradnorm_step(gram, L, L0, w, alpha, lr):
    """numpy: one GradNorm step from the Gram matrix of the unweighted per-task gradients: (w_new, L_grad, d_w)."""
    gram, L, L0, w = (np.asarray(a, np.float64) for a in (gram, L, L0, w))
    n = np.sqrt(np.diag(gram))
    G = w * n
    q = L / L0
    if not q.mean() > 0:                                             # every loss 0: r undefined, w unchanged
        return w.copy(), 0.0, np.zeros_like(w)
    r = q / q.mean()
    diff = G - G.mean() * r ** alpha
    d_w = np.sign(diff) * n
    w1 = w - lr * d_w
    return len(w) * w1 / w1.sum(), np.abs(diff).sum(), d_w


def gradnorm_loss(grads, L, L0, w, alpha):
    """torch: L_grad = sum_t |G_t - Gbar r_t^alpha| with G_t = w_t |g_t| and the target detached (as in the paper)."""
    G = w * grads.norm(dim=1)
    q = L / L0
    target = (G.mean() * (q / q.mean()) ** alpha).detach()
    return (G - target).abs().sum()


def pcgrad_vector(g, order):
    """numpy: the paper's vector form over rows g (T,P): (sum_i g_i', [g_i'])."""
    g = np.asarray(g, np.float64)
    out = []
    for i in range(len(g)):
        gi = g[i].copy()
        for j in order:
            if j == i:
                continue
            dot = gi @ g[j]
            nn = g[j] @ g[j]
            if dot < 0 and nn > 0:
                gi -= dot / nn * g[j]
        out.append(gi)
    return np.sum(out, axis=0), out


def pcgrad_coef(gram, order):
    """numpy: the coefficient form from the Gram matrix: c (T,) with sum_i g_i' = sum_k c_k g_k."""
    gram = np.asarray(gram, np.float64)
    T = len(gram)
    C = np.eye(T)
    for i in range(T):
        for j in order:
            if j == i:
                continue
            dot = C[i] @ gram[:, j]
            if dot < 0 and gram[j, j] > 0:
                C[i, j] -= dot / gram[j, j]
    return C.sum(axis=0)
