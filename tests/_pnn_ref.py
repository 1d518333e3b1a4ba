"""NumPy restatement of the PNN product layer (PNN/pnn.py:125-181) for the PNN tests.

`pnn_fwd` / `pnn_bwd` follow the reference's direct form (Delta and p, then the per-output reductions); `feature_rows` and
`feature_weights` restate the single-GEMM form the kernels compute (csrc/pnn.cu), so the CPU tests pin that algebra to the
direct form before any GPU run."""
import numpy as np


def _sym_upper(w):
    """W'_n = triu(W_n) + triu(W_n)^T - diag(W_n)   (pnn.py:169-170): W'[k,l] = W[min(k,l), max(k,l)]."""
    up = np.triu(w)
    return up + np.swapaxes(up, -1, -2) - np.einsum("nkk->nk", w)[:, :, None] * np.eye(w.shape[-1])


def pnn_fwd(e, wlin, wprod, bias, method, return_parts=False):
    """e (B,F,K); wlin (F*K,N); wprod theta (N,F) (method 0, IPNN) | W (N,K,K) (method 1, OPNN); bias (N,) -> (B,N)."""
    B, F, K = e.shape
    lz = e.reshape(B, F * K) @ wlin                                              # :133-139
    if method == 0:
        delta = np.einsum("bfk,nf->bnk", e, wprod)                              # :152-153
        lp = np.sum(delta * delta, axis=-1)                                       # :154
    else:
        s = e.sum(1)                                                              # :166
        p = s[:, :, None] * s[:, None, :]                                         # :167
        lp = np.einsum("bkl,nkl->bn", p, _sym_upper(wprod))                      # :168-172
    out = np.maximum(lz + lp + bias, 0)                                           # :178-181
    return (out, lz, lp) if return_parts else out


def pnn_bwd(e, wlin, wprod, bias, method, g):
    """Analytic gradients of pnn_fwd: (d_e, d_wlin, d_wprod, d_bias).  The relu passes where out > 0."""
    B, F, K = e.shape
    out = pnn_fwd(e, wlin, wprod, bias, method)
    G = g * (out > 0)
    d_wlin = e.reshape(B, F * K).T @ G
    d_bias = G.sum(0)
    d_e = (G @ wlin.T).reshape(B, F, K)
    if method == 0:
        delta = np.einsum("bfk,nf->bnk", e, wprod)
        d_delta = 2 * G[:, :, None] * delta
        d_e = d_e + np.einsum("bnk,nf->bfk", d_delta, wprod)
        d_wprod = np.einsum("bnk,bfk->nf", d_delta, e)
    else:
        s = e.sum(1)
        p = s[:, :, None] * s[:, None, :]
        d_sym = np.einsum("bn,bkl->nkl", G, p)                                    # dL/dW'
        d_wprod = np.triu(d_sym) + np.triu(np.swapaxes(d_sym, -1, -2)) - np.einsum("nkk->nk", d_sym)[:, :, None] * np.eye(K)
        d_p = np.einsum("bn,nkl->bkl", G, _sym_upper(wprod))
        ds = np.einsum("bkl,bl->bk", d_p + np.swapaxes(d_p, -1, -2), s)
        d_e = d_e + ds[:, None, :]
    return d_e, d_wlin, d_wprod, d_bias


def pairs(n):
    return [(i, j) for i in range(n) for j in range(i, n)]


def feature_rows(e, method):
    """xt (B, F*K + Q + 1) = [e_flat | upper-triangle pair features | 1]: <e_i, e_j> (IPNN) or s_k s_l (OPNN)."""
    B, F, K = e.shape
    if method == 0:
        gram = np.einsum("bik,bjk->bij", e, e)
        q = np.stack([gram[:, i, j] for i, j in pairs(F)], 1)
    else:
        s = e.sum(1)
        q = np.stack([s[:, k] * s[:, l] for k, l in pairs(K)], 1)
    return np.concatenate([e.reshape(B, F * K), q, np.ones((B, 1), e.dtype)], 1)


def feature_weights(wlin, wprod, bias, method):
    """Wm (F*K + Q + 1, N) = [linear_w ; c theta_i theta_j (IPNN) | c W[k,l] (OPNN) ; bias], c = 1 on the diagonal, 2 off."""
    if method == 0:
        rows = [(1.0 if i == j else 2.0) * wprod[:, i] * wprod[:, j] for i, j in pairs(wprod.shape[1])]
    else:
        rows = [(1.0 if k == l else 2.0) * wprod[:, k, l] for k, l in pairs(wprod.shape[1])]
    return np.concatenate([wlin, np.stack(rows, 0), bias[None, :]], 0)
