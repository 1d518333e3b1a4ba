"""Float64 restatement of the AutoInt interacting layer (Song et al., CIKM 2019, arXiv:1810.11921, eq. 5-8) and its analytic
backward.  The reference tree has no AutoInt code, so this restatement of the paper is the parity target of
csrc/autoint.cu; tests/test_autoint_oracle.py checks it against torch.autograd and torch's own attention operator."""
import numpy as np


def attention_core(q, k, v):
    """softmax_j(q_i . k_j) v over the last two axes, no 1/sqrt(dk) scaling; row max subtracted.  Returns (o, a)."""
    s = q @ np.swapaxes(k, -1, -2)
    s = s - s.max(axis=-1, keepdims=True)
    e = np.exp(s)
    a = e / e.sum(axis=-1, keepdims=True)
    return a @ v, a


def _heads(t, H, dk):
    B, F, _ = t.shape
    return t.reshape(B, F, H, dk).transpose(0, 2, 1, 3)        # (B, H, F, dk)


def _merge(t):
    B, H, F, dk = t.shape
    return t.transpose(0, 2, 1, 3).reshape(B, F, H * dk)


def interacting_fwd(x, wq, wk, wv, wr, H, dk):
    """x (B,F,d), each w (d, H*dk) -> out (B,F,H*dk) = relu(concat_h softmax(Q_h K_h^T) V_h + x wr), and the cache."""
    x = np.asarray(x, np.float64)
    wq, wk, wv, wr = (np.asarray(w, np.float64) for w in (wq, wk, wv, wr))
    Q, K, V = (_heads(x @ w, H, dk) for w in (wq, wk, wv))
    o, a = attention_core(Q, K, V)
    pre = _merge(o) + x @ wr
    return np.maximum(pre, 0.0), (x, Q, K, V, a, pre)


def interacting_bwd(cache, wq, wk, wv, wr, g_out, H, dk):
    """Analytic gradients: (d_x, d_wq, d_wk, d_wv, d_wr)."""
    x, Q, K, V, a, pre = cache
    wq, wk, wv, wr = (np.asarray(w, np.float64) for w in (wq, wk, wv, wr))
    G = np.asarray(g_out, np.float64) * (pre > 0)
    dO = _heads(G, H, dk)
    dA = dO @ np.swapaxes(V, -1, -2)
    dV = np.swapaxes(a, -1, -2) @ dO
    dS = a * (dA - (a * dA).sum(axis=-1, keepdims=True))
    dQ = dS @ K
    dK = np.swapaxes(dS, -1, -2) @ Q
    dQ, dK, dV = _merge(dQ), _merge(dK), _merge(dV)
    d = x.shape[-1]
    xf = x.reshape(-1, d)
    grads_w = [xf.T @ t.reshape(xf.shape[0], -1) for t in (dQ, dK, dV, G)]
    d_x = dQ @ wq.T + dK @ wk.T + dV @ wv.T + G @ wr.T
    return (d_x, *grads_w)


def model_logit(dense_input, fields_embeddings, v_dense, layers, w_out, b_out, H, dk):
    """examples/model_bodies.autoint_logit in float64: dense features embedded as x_m v_m, concatenated with the field
    embeddings, `layers` interacting layers [(wq, wk, wv, wr), ...], flatten, dense(1)."""
    dense_input = np.asarray(dense_input, np.float64)
    emb = dense_input[:, :, None] * np.asarray(v_dense, np.float64)[None]
    net = np.concatenate([emb, np.asarray(fields_embeddings, np.float64)], axis=1)
    for (wq, wk, wv, wr) in layers:
        net, _ = interacting_fwd(net, wq, wk, wv, wr, H, dk)
    flat = net.reshape(net.shape[0], -1)
    return flat @ np.asarray(w_out, np.float64) + np.asarray(b_out, np.float64)
