"""Float64 restatement of the DCN-Mix cross network (Wang et al., WWW 2021, arXiv:2008.13535, eq. 3-4) and its analytic
backward, in the row-vector form of include/ctr_b200.h's Row CROSS-MIX.  The forward is the paper's per-expert form,

    x_{l+1} = sum_i p_i E_i(x_l) + x_l,   E_i(x_l) = x0 * (g(g(x_l . v[l,i]) . c[l,i]) . u[l,i] + b[l]),
    p = softmax_i(x_l . gate),

and `cross_mix_fwd_collapsed` is the form the kernels compute, x_{l+1} = x0 * (sum_i p_i c~_i . u[l,i] + b[l]) + x_l.
g is tanh (activation 1) or the identity (0)."""
import numpy as np


def _f64(a):
    return np.asarray(a, dtype=np.float64)


def _g(x, act):
    return np.tanh(x) if act else x


def _softmax(s):
    e = np.exp(s - s.max(axis=1, keepdims=True))
    return e / e.sum(axis=1, keepdims=True)


def cross_mix_fwd(x0, v, c, u, b, gate, act=1):
    """-> (out (B,d), cache).  v (L,K,d,r), c (L,K,r,r), u (L,K,r,d), b (L,d), gate (d,K)."""
    x0, v, c, u, b, gate = (_f64(a) for a in (x0, v, c, u, b, gate))
    L, K = v.shape[:2]
    x = x0
    xs, zs, ts, cts, ps = [], [], [], [], []
    for l in range(L):
        p = _softmax(x @ gate)
        t = [_g(x @ v[l, i], act) for i in range(K)]
        ct = [_g(t[i] @ c[l, i], act) for i in range(K)]
        experts = [x0 * (ct[i] @ u[l, i] + b[l]) for i in range(K)]
        xs.append(x); ts.append(t); cts.append(ct); ps.append(p)
        zs.append(sum(p[:, i:i + 1] * (ct[i] @ u[l, i]) for i in range(K)) + b[l])
        x = sum(p[:, i:i + 1] * experts[i] for i in range(K)) + x
    return x, (x0, xs, zs, ts, cts, ps, act)


def cross_mix_fwd_collapsed(x0, v, c, u, b, gate, act=1):
    """The kernels' form: one product of [p_1 c~_1 | .. | p_K c~_K] with the stacked u per layer."""
    x0, v, c, u, b, gate = (_f64(a) for a in (x0, v, c, u, b, gate))
    L, K, d, r = v.shape
    x = x0
    for l in range(L):
        p = _softmax(x @ gate)
        t = _g(x @ v[l].transpose(1, 0, 2).reshape(d, K * r), act)
        bd = np.zeros((K * r, K * r))
        for i in range(K):
            bd[i * r:(i + 1) * r, i * r:(i + 1) * r] = c[l, i]
        a = np.repeat(p, r, axis=1) * _g(t @ bd, act)
        x = x0 * (a @ u[l].reshape(K * r, d) + b[l]) + x
    return x


def cross_mix_bwd(cache, v, c, u, gate, g_out):
    """-> (dx0, dv, dc, du, db, dgate) given dL/dout."""
    x0, xs, zs, ts, cts, ps, act = cache
    v, c, u, gate, G = (_f64(a) for a in (v, c, u, gate, g_out))
    L, K = v.shape[:2]
    dx0 = np.zeros_like(x0)
    dv, dc, du = np.zeros_like(v), np.zeros_like(c), np.zeros_like(u)
    db, dgate = np.zeros((L, x0.shape[1])), np.zeros_like(gate)
    for l in range(L - 1, -1, -1):
        x, t, ct, p = xs[l], ts[l], cts[l], ps[l]
        dz = G * x0
        dx0 += G * zs[l]
        db[l] = dz.sum(0)
        e = [dz @ u[l, i].T for i in range(K)]
        dp = np.stack([(ct[i] * e[i]).sum(1) for i in range(K)], axis=1)
        ds = p * (dp - (p * dp).sum(1, keepdims=True))
        G = G + ds @ gate.T
        dgate += x.T @ ds
        for i in range(K):
            pi = p[:, i:i + 1]
            dm = pi * e[i] * ((1 - ct[i] ** 2) if act else 1.0)
            dq = (dm @ c[l, i].T) * ((1 - t[i] ** 2) if act else 1.0)
            du[l, i] = (pi * ct[i]).T @ dz
            dc[l, i] = t[i].T @ dm
            dv[l, i] = x.T @ dq
            G = G + dq @ v[l, i].T
    return dx0 + G, dv, dc, du, db, dgate
