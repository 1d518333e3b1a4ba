"""NumPy restatement of the reference hot path (TEST INFRASTRUCTURE -- see oracle/__init__.py).

Every function follows the reference file:line it cites (paths relative to
the reference's algorithm/ directory).  Arithmetic runs in the dtype of the inputs: float32 mirrors
the reference's TF1 CPU graph, float64 is the high-precision anchor the fp32 results are
themselves checked against.  Forward functions mirror the reference op-for-op (including
its quirks); backward functions are the analytic gradients of those forwards and are
cross-checked against torch.autograd(float64) in tests/test_oracle.py.

Weights are always explicit arguments: the reference never seeds its initialisers, so
parity is defined on injected weights (SURVEY.md section 7, step 1).
"""
from __future__ import annotations

import itertools
from typing import List, Sequence, Tuple

import numpy as np

# --------------------------------------------------------------------------------------
# Row L -- embedding lookup  (fc.input_layer over embedding columns)
# --------------------------------------------------------------------------------------


def vocab_ids(keys: Sequence[bytes], vocab: Sequence[bytes]) -> np.ndarray:
    """String key -> vocabulary line index, OOV (and b'') -> -1.

    ``fc.categorical_column_with_vocabulary_file(key, file)`` with the defaults the
    reference uses (DeepFM/deepfm.py:56-64): ``num_oov_buckets=0, default_value=None`` =>
    id = 0-based line number, out-of-vocabulary => -1  [TF-internal, SURVEY A.4].
    Vocabulary files hold one token per line (dataset/wechat_algo_data1/DataGenerator.py:206-210).
    """
    table = {}
    for i, tok in enumerate(vocab):
        table.setdefault(tok, i)  # first occurrence wins, like a hash-table init from file
    return np.asarray([table.get(k, -1) for k in keys], dtype=np.int64)


def embedding_lookup(table: np.ndarray, ids: np.ndarray, field_row_offset: np.ndarray) -> np.ndarray:
    """Single-valued per-field lookup -> (B, F, D).

    ``fc.input_layer(features, [embedding_column(col, D)])`` for one id per row
    (DeepFM/deepfm.py:187-190, xDeepFM/xdeepfm.py:158,167):
    ``safe_embedding_lookup_sparse(combiner='mean')`` on a one-element bag is the row itself
    (bit-exact copy); id < 0 is pruned => empty bag => **zero vector**  [TF-internal, SURVEY A.5].

    ``table`` is the concatenation of the F per-field tables, field f owning rows
    ``field_row_offset[f] : field_row_offset[f+1]``; ``ids`` are per-field local ids (B, F).
    """
    B, F = ids.shape
    D = table.shape[1]
    out = np.zeros((B, F, D), dtype=table.dtype)
    for f in range(F):
        valid = ids[:, f] >= 0
        out[valid, f, :] = table[field_row_offset[f] + ids[valid, f]]
    return out


def bag_lookup_mean(table: np.ndarray, ids: np.ndarray, offsets: np.ndarray) -> np.ndarray:
    """Multi-valued lookup with combiner='mean' -> (B, D).

    ``embedding_column(col, D, combiner='mean')`` over a VarLen feature, e.g.
    ``manual_tag_list`` (DCN/dcn.py:98,103; xDeepFM/xdeepfm.py:103,108).
    [TF-internal, SURVEY A.5]: (1) drop ids < 0; (2) sum the remaining rows in bag order and
    divide by their count; (3) a bag with no valid id yields zeros.
    ``ids`` is the flat CSR value array, bag b = ids[offsets[b]:offsets[b+1]].
    """
    B = offsets.shape[0] - 1
    D = table.shape[1]
    out = np.zeros((B, D), dtype=table.dtype)
    for b in range(B):
        acc = np.zeros((D,), dtype=table.dtype)
        n = 0
        for i in ids[offsets[b]:offsets[b + 1]]:
            if i >= 0:
                acc = acc + table[i]
                n += 1
        if n:
            out[b] = acc / table.dtype.type(n)
    return out


def embedding_lookup_bwd_dense(V: int, ids: np.ndarray, field_row_offset: np.ndarray,
                               row_grads: np.ndarray) -> np.ndarray:
    """Densify the IndexedSlices gradient of ``embedding_lookup`` (duplicates summed, ids<0 dropped).

    TF's gradient of the gather is ``IndexedSlices(values=(B*F, D), indices)``; the optimizer
    sums duplicate indices before applying [TF-internal, SURVEY A.8].  float64 accumulate.
    """
    B, F = ids.shape
    D = row_grads.shape[-1]
    g = np.zeros((V, D), dtype=np.float64)
    for f in range(F):
        valid = ids[:, f] >= 0
        np.add.at(g, field_row_offset[f] + ids[valid, f], row_grads[valid, f, :].astype(np.float64))
    return g


# --------------------------------------------------------------------------------------
# Row FM2 -- DeepFM second-order term (inline in deepfm_model_fn)
# --------------------------------------------------------------------------------------


def fm2_fwd(e: np.ndarray) -> np.ndarray:
    """FM second-order logit (B, 1) from the F field embeddings e: (B, F, K).

    DeepFM/deepfm.py:184-200: ``square(add_n(e_f))``, ``add_n(square(e_f))``,
    ``reduce_sum(0.5 * (a - b), axis=1, keepdims=True)``; add_n accumulates in list order.
    """
    F = e.shape[1]
    s = e[:, 0, :].copy()
    q = np.square(e[:, 0, :])
    for f in range(1, F):
        s = s + e[:, f, :]
        q = q + np.square(e[:, f, :])
    half = e.dtype.type(0.5)
    return np.sum(half * (np.square(s) - q), axis=1, keepdims=True)


def fm2_bwd(e: np.ndarray, g: np.ndarray) -> np.ndarray:
    """d(fm2)/d(e) * g : ``de[b,f,:] = g[b] * (S[b,:] - e[b,f,:])`` with S = sum_f e."""
    s = e.sum(axis=1, keepdims=True)
    return g.reshape(-1, 1, 1) * (s - e)


def fm2_pairwise(e: np.ndarray) -> np.ndarray:
    """Identity check: FM2 == sum_{i<j} <e_i, e_j> (float64)."""
    e = e.astype(np.float64)
    F = e.shape[1]
    out = np.zeros((e.shape[0], 1))
    for i, j in itertools.combinations(range(F), 2):
        out[:, 0] += np.sum(e[:, i, :] * e[:, j, :], axis=1)
    return out

# ---- SURVEY 8f.4: siblings of FM2 (NFM bi-interaction, FwFM, AFM) ---------------------------------------------------------

def bi_interaction_fwd(e: np.ndarray) -> np.ndarray:
    """NFM bi-interaction pooling (B, K): FM2 without the sum over K.  NFM/nfm.py:155-168:
    ``0.5 * (square(add_n(e_f)) - add_n(square(e_f)))`` (the BN/dropout after it are outside the path)."""
    F = e.shape[1]
    s = e[:, 0, :].copy()
    q = np.square(e[:, 0, :])
    for f in range(1, F):
        s = s + e[:, f, :]
        q = q + np.square(e[:, f, :])
    return e.dtype.type(0.5) * (np.square(s) - q)


def bi_interaction_bwd(e: np.ndarray, g: np.ndarray) -> np.ndarray:
    """g: (B, K) -> de[b,f,:] = g[b,:] * (S[b,:] - e[b,f,:])."""
    return g[:, None, :] * (e.sum(axis=1, keepdims=True) - e)


def pair_index(i: int, j: int, n: int) -> int:
    """Flat index of (i, j), i < j, in the row-major strict upper triangle of an n x n matrix
    (utils.py:67-82: sum_{k<i}(n-1-k) + j-i-1)."""
    return i * (n - 1) - i * (i - 1) // 2 + (j - i - 1)


def fwfm_fwd(e: np.ndarray, r: np.ndarray) -> np.ndarray:
    """FwFM second-order logit (B, 1): sum_{i<j} r[pair_index(i,j,F)] * <e_i, e_j>, pairs accumulated in the reference's
    loop order (FwFM/fwfm.py:152-158: ``+= scalar_mul(r[index], batch_dot(e_i, e_j, axes=1))``)."""
    B, F, _ = e.shape
    out = np.zeros((B, 1), dtype=e.dtype)
    for i in range(F - 1):
        for j in range(i + 1, F):
            out = out + r[pair_index(i, j, F)] * np.sum(e[:, i, :] * e[:, j, :], axis=1, keepdims=True)
    return out


def fwfm_bwd(e: np.ndarray, r: np.ndarray, g: np.ndarray):
    """g: (B,) or (B,1).  Returns (de (B,F,K), dr (P,))."""
    B, F, _ = e.shape
    g = g.reshape(B, 1)
    de = np.zeros_like(e)
    dr = np.zeros_like(r)
    for i in range(F - 1):
        for j in range(i + 1, F):
            p = pair_index(i, j, F)
            de[:, i, :] += g * r[p] * e[:, j, :]
            de[:, j, :] += g * r[p] * e[:, i, :]
            dr[p] = np.sum(g[:, 0] * np.sum(e[:, i, :] * e[:, j, :], axis=1))
    return de, dr


def afm_pairs(F: int):
    return [(i, j) for i in range(F) for j in range(i + 1, F)]        # AFM/afm.py:162-164


def afm_fwd(e: np.ndarray, w: np.ndarray, b: np.ndarray, h: np.ndarray, return_all: bool = False):
    """AFM attention pooling (B, K).  AFM/afm.py:152-186: pair_hadamard (B,P,K) = e_i * e_j for i<j;
    attention = relu(pair @ w + b) @ h -> (B,P,1); softmax over the PAIR axis; sum_p score * pair."""
    pairs = afm_pairs(e.shape[1])
    had = np.stack([e[:, i, :] * e[:, j, :] for i, j in pairs], axis=1)                  # (B,P,K)
    pre = np.matmul(had, w) + b                                                            # (B,P,t)
    act = np.maximum(pre, 0)
    att = np.matmul(act, h)                                                                # (B,P,1)
    att = att - att.max(axis=1, keepdims=True)
    ex = np.exp(att)
    score = ex / ex.sum(axis=1, keepdims=True)
    out = np.sum(had * score, axis=1)
    return (out, had, pre, act, score) if return_all else out


def afm_bwd(e, w, b, h, g):
    """g: (B,K) gradient of the pooled vector.  Returns (de, dw, db, dh)."""
    e, w, b, h, g = (np.asarray(x, dtype=np.float64) for x in (e, w, b, h, g))
    out, had, pre, act, score = afm_fwd(e, w, b, h, return_all=True)
    pairs = afm_pairs(e.shape[1])
    dscore = np.sum(had * g[:, None, :], axis=2, keepdims=True)                            # (B,P,1)
    datt = score * (dscore - np.sum(score * dscore, axis=1, keepdims=True))
    dh = np.einsum("bpt,bpo->to", act, datt)
    dact = datt * h[:, 0][None, None, :]
    dpre = dact * (pre > 0)
    dw = np.einsum("bpk,bpt->kt", had, dpre)
    db = dpre.sum(axis=(0, 1))
    dhad = g[:, None, :] * score + np.matmul(dpre, w.T)
    de = np.zeros_like(e)
    for p, (i, j) in enumerate(pairs):
        de[:, i, :] += dhad[:, p, :] * e[:, j, :]
        de[:, j, :] += dhad[:, p, :] * e[:, i, :]
    return de, dw, db, dh


# --------------------------------------------------------------------------------------
# Row CROSS -- DCN cross layer
# --------------------------------------------------------------------------------------


def cross_layer_fwd(x0: np.ndarray, xl: np.ndarray, wl: np.ndarray, bl: np.ndarray) -> np.ndarray:
    """One cross layer.  DCN/cross_layer.py:21-24; wl, bl have shape (d, 1) (:18-19)."""
    xl_wl = xl @ wl                      # (B, 1)
    x0_xl_wl = x0 * xl_wl                # (B, d)
    out = x0_xl_wl + bl.T                # + (1, d)
    return out + xl


def cross_stack_fwd(x0: np.ndarray, ws: np.ndarray, bs: np.ndarray) -> List[np.ndarray]:
    """The stack loop of DCN/dcn.py:157-160.  ws, bs: (L, d).  Returns [x_0, x_1, ..., x_L]."""
    xs = [x0]
    for l in range(ws.shape[0]):
        xs.append(cross_layer_fwd(x0, xs[-1], ws[l][:, None], bs[l][:, None]))
    return xs


def cross_stack_bwd(x0: np.ndarray, ws: np.ndarray, bs: np.ndarray, g_out: np.ndarray
                    ) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Gradient of the stack w.r.t. (x0, ws, bs) given dL/dx_L.  Returns (dx0, dws, dbs)."""
    xs = cross_stack_fwd(x0, ws, bs)
    L = ws.shape[0]
    g = g_out.copy()
    dx0 = np.zeros_like(x0)
    dws = np.zeros_like(ws)
    dbs = np.zeros_like(bs)
    for l in range(L - 1, -1, -1):
        xl = xs[l]
        s = xl @ ws[l]                                   # (B,)
        t = np.sum(g * x0, axis=1)                       # (B,)
        dx0 += g * s[:, None]
        dws[l] = xl.T @ t
        dbs[l] = g.sum(axis=0)
        g = g + t[:, None] * ws[l][None, :]
    return dx0 + g, dws, dbs


# --------------------------------------------------------------------------------------
# Row CIN -- xDeepFM compressed interaction network layer
# --------------------------------------------------------------------------------------


def cin_layer_fwd(x0: np.ndarray, xk: np.ndarray, filt: np.ndarray) -> np.ndarray:
    """One CIN layer.  xDeepFM/cin_layer.py:17-28.

    x0 (B, m, D), xk (B, hk, D), filt (hk*m, hk_1) == the conv1d filter (1, hk*m, hk_1)[0].
    outer[b,d,i,j] = xk[b,i,d] * x0[b,j,d] (:21), flattened with index i*m+j (:22),
    conv1d(width 1, VALID) == matmul over the last axis (:25-27), transposed to (B, hk_1, D) (:28).
    The outer tensor is materialised exactly like the reference does.
    """
    B, m, D = x0.shape
    hk = xk.shape[1]
    outer = np.einsum('bik,bjk->bkij', xk, x0).reshape(B, D, hk * m)
    xk_1 = outer @ filt                                   # (B, D, hk_1)
    return np.transpose(xk_1, (0, 2, 1))


def cin_layer_bwd(x0: np.ndarray, xk: np.ndarray, filt: np.ndarray, g: np.ndarray
                  ) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Gradients (dx0, dxk, dfilt) of ``cin_layer_fwd`` given g = dL/d(out) (B, hk_1, D)."""
    B, m, D = x0.shape
    hk = xk.shape[1]
    gt = np.transpose(g, (0, 2, 1))                       # (B, D, hk_1)
    outer = np.einsum('bik,bjk->bkij', xk, x0).reshape(B, D, hk * m)
    dfilt = np.einsum('bdz,bdn->zn', outer, gt)
    dz = (gt @ filt.T).reshape(B, D, hk, m)               # (B, D, hk, m)
    dxk = np.einsum('bdij,bjd->bid', dz, x0)
    dx0 = np.einsum('bdij,bid->bjd', dz, xk)
    return dx0, dxk, dfilt


def cin_stack_fwd(x0: np.ndarray, filters: Sequence[np.ndarray]) -> Tuple[List[np.ndarray], np.ndarray]:
    """xDeepFM/xdeepfm.py:166-174: every layer's full output feeds the next layer and the pooled sum.

    Returns ([X^1, X^2, ...], p_plus (B, sum_k h_k)).
    """
    xs, xk = [], x0
    for filt in filters:
        xk = cin_layer_fwd(x0, xk, filt)
        xs.append(xk)
    p_plus = np.concatenate([x.sum(axis=-1) for x in xs], axis=-1)
    return xs, p_plus


# --------------------------------------------------------------------------------------
# Row DIN-ATT -- DIN attention unit
# --------------------------------------------------------------------------------------

DIN_PAD = -2 ** 32 + 1   # DIN/din_attention.py:31 -- Python precedence: -(2**32) + 1


def din_attention_fwd(query: np.ndarray, keys: np.ndarray, keys_length: np.ndarray,
                      w1, b1, w2, b2, w3, b3, is_softmax: bool = False, return_cache: bool = False):
    """DIN/din_attention.py:17-43.

    query (B,H); keys (B,T,H); keys_length (B,); dense f1_att (4H->64, relu), f2_att (64->32, relu),
    f3_att (32->1).  Non-softmax (default): weights * mask (:37-38).  Softmax: masked scores are
    filled with -2**32+1, THEN divided by sqrt(H), then softmax over T (:31-35).
    """
    dt = query.dtype
    B, T, H = keys.shape
    q = np.broadcast_to(query[:, None, :], (B, T, H))                    # tile + reshape (:18-19)
    cross = np.concatenate([q, keys, q - keys, q * keys], axis=-1)       # (:20)
    h1 = np.maximum(cross @ w1 + b1, 0)                                  # (:21)
    h2 = np.maximum(h1 @ w2 + b2, 0)                                     # (:22)
    s = h2 @ w3 + b3                                                     # (B,T,1) (:23)
    mask = (np.arange(T)[None, :] < keys_length[:, None])[..., None]     # (:27-28)
    if is_softmax:
        pad = np.ones_like(s) * dt.type(DIN_PAD)
        s2 = np.where(mask, s, pad)
        s2 = s2 / dt.type(H ** 0.5)
        s2 = s2 - s2.max(axis=1, keepdims=True)
        ex = np.exp(s2)
        w = ex / ex.sum(axis=1, keepdims=True)
    else:
        w = s * mask.astype(dt)
    out = np.matmul(np.transpose(w, (0, 2, 1)), keys)[:, 0, :]           # (:40-41)
    if return_cache:
        return out, dict(cross=cross, h1=h1, h2=h2, w=w, mask=mask)
    return out


def din_attention_bwd(query, keys, keys_length, w1, b1, w2, b2, w3, b3, g_out, is_softmax=False):
    """Gradients of ``din_attention_fwd`` given g_out (B,H).

    Returns dict(query, keys, w1, b1, w2, b2, w3, b3).
    """
    dt = query.dtype
    B, T, H = keys.shape
    _, c = din_attention_fwd(query, keys, keys_length, w1, b1, w2, b2, w3, b3, is_softmax, True)
    cross, h1, h2, w, mask = c['cross'], c['h1'], c['h2'], c['w'], c['mask']
    dw = np.einsum('bh,bth->bt', g_out, keys)[..., None]                  # (B,T,1)
    dkeys = w * g_out[:, None, :]
    if is_softmax:
        ds2 = w * (dw - np.sum(w * dw, axis=1, keepdims=True))
        ds = np.where(mask, ds2 / dt.type(H ** 0.5), 0).astype(dt)
    else:
        ds = dw * mask.astype(dt)
    dw3 = np.einsum('btk,bto->ko', h2, ds)
    db3 = ds.sum(axis=(0, 1))
    dh2 = (ds @ w3.T) * (h2 > 0)
    dw2 = np.einsum('btk,bto->ko', h1, dh2)
    db2 = dh2.sum(axis=(0, 1))
    dh1 = (dh2 @ w2.T) * (h1 > 0)
    dw1 = np.einsum('btk,bto->ko', cross, dh1)
    db1 = dh1.sum(axis=(0, 1))
    dcross = dh1 @ w1.T                                                   # (B,T,4H)
    dq_a, dk_a, dqmk, dqk = np.split(dcross, 4, axis=-1)
    q = query[:, None, :]
    dquery = (dq_a + dqmk + dqk * keys).sum(axis=1)
    dkeys = dkeys + dk_a - dqmk + dqk * q
    return dict(query=dquery, keys=dkeys, w1=dw1, b1=db1, w2=dw2, b2=db2, w3=dw3, b3=db3)


# --------------------------------------------------------------------------------------
# Row SENET / BILINEAR -- FiBiNET
# --------------------------------------------------------------------------------------


def senet_fwd(x: np.ndarray, w1: np.ndarray, w2: np.ndarray) -> np.ndarray:
    """FiBiNET/senet.py:26-34.  x (B,F,K); w1 (F,r); w2 (r,F); no bias.

    NB ``r = embedding_dim // reduction_ratio`` (:18) -- reduced from K, not F (reference quirk).
    """
    z = x.mean(axis=-1)
    a = np.maximum(z @ w1, 0)
    a = np.maximum(a @ w2, 0)
    return x * a[..., None]


def senet_bwd(x, w1, w2, g):
    """Gradients (dx, dw1, dw2) of ``senet_fwd``."""
    K = x.shape[-1]
    z = x.mean(axis=-1)
    a1 = np.maximum(z @ w1, 0)
    a2 = np.maximum(a1 @ w2, 0)
    da2 = np.sum(g * x, axis=-1) * (a2 > 0)
    dw2 = a1.T @ da2
    da1 = (da2 @ w2.T) * (a1 > 0)
    dw1 = z.T @ da1
    dz = da1 @ w1.T
    dx = g * a2[..., None] + dz[..., None] / x.dtype.type(K)
    return dx, dw1, dw2


def bilinear_pairs(F: int) -> List[Tuple[int, int]]:
    """``itertools.combinations(range(F-1), 2)`` -- the reference pairs only fields 0..F-2
    (FiBiNET/bilinear_interaction_layer.py:24,29,33), giving (F-1)(F-2)/2 outputs."""
    return list(itertools.combinations(range(F - 1), 2))


def bilinear_fwd(x: np.ndarray, w: np.ndarray, type: str) -> np.ndarray:
    """FiBiNET/bilinear_interaction_layer.py:21-40.  x (B,F,K) -> (B,P,K).

    all: w (K,K); each: w (F-1,K,K); interaction: w (F(F-1)/2,K,K) of which the first P are used.
    """
    B, F, K = x.shape
    pairs = bilinear_pairs(F)
    if type == 'all':
        vw = x @ w
        p = [vw[:, i, :] * x[:, j, :] for i, j in pairs]
    elif type == 'each':
        vw = [x[:, i, :] @ w[i] for i in range(F - 1)]
        p = [vw[i] * x[:, j, :] for i, j in pairs]
    elif type == 'interaction':
        p = [(x[:, i, :] @ w[k]) * x[:, j, :] for k, (i, j) in enumerate(pairs)]
    else:
        raise ValueError(f"Bilinear Interaction type must be in ['all','each','interaction'], got '{type}'")
    return np.stack(p, axis=1)


def bilinear_bwd(x, w, type, g):
    """Gradients (dx, dw) of ``bilinear_fwd`` given g (B,P,K)."""
    B, F, K = x.shape
    pairs = bilinear_pairs(F)
    dx = np.zeros_like(x)
    dw = np.zeros_like(w)
    for k, (i, j) in enumerate(pairs):
        wi = w if type == 'all' else (w[i] if type == 'each' else w[k])
        vw = x[:, i, :] @ wi
        dvw = g[:, k, :] * x[:, j, :]
        dx[:, j, :] += g[:, k, :] * vw
        dx[:, i, :] += dvw @ wi.T
        gw = x[:, i, :].T @ dvw
        if type == 'all':
            dw += gw
        elif type == 'each':
            dw[i] += gw
        else:
            dw[k] += gw
    return dx, dw


# --------------------------------------------------------------------------------------
# SURVEY 8f.3 -- tf.train.AdamOptimizer on an IndexedSlices gradient (DeepFM/deepfm.py:246-250)  [TF-internal, A.8]
# --------------------------------------------------------------------------------------


def adam_sparse_apply(var, m, v, rows, values, t, lr, beta1=0.9, beta2=0.999, eps=1e-8, lazy=False):
    """One step.  rows (n,) global row ids (duplicates allowed, summed first), values (n, D).
    Non-lazy = TF's AdamOptimizer._apply_sparse: dense decay of m and v and a dense variable update;
    lazy = LazyAdamOptimizer (DIEN/dien.py:328): only the referenced rows change.  Returns new (var, m, v)."""
    var, m, v = var.astype(np.float64), m.astype(np.float64), v.astype(np.float64)
    g = np.zeros_like(var)
    np.add.at(g, rows, values.astype(np.float64))
    lr_t = lr * np.sqrt(1.0 - beta2 ** t) / (1.0 - beta1 ** t)
    # TF casts beta1_t / beta2_t to the variable dtype and forms (1 - beta_t) in float32 (adam.py _apply_sparse_shared):
    # float32(0.999) is 0.99900001..., so (1 - beta2_t) differs from 1e-3 by 1.3e-5 relative.  The coefficients below
    # are those float32 values; the accumulation itself stays in float64.
    om1 = float(np.float32(1.0) - np.float32(beta1)); om2 = float(np.float32(1.0) - np.float32(beta2))
    beta1 = float(np.float32(beta1)); beta2 = float(np.float32(beta2))
    if lazy:
        idx = np.unique(rows)
        m[idx] = beta1 * m[idx] + om1 * g[idx]
        v[idx] = beta2 * v[idx] + om2 * g[idx] ** 2
        var[idx] -= lr_t * m[idx] / (np.sqrt(v[idx]) + eps)
    else:
        m = beta1 * m + om1 * g
        v = beta2 * v + om2 * g * g
        var = var - lr_t * m / (np.sqrt(v) + eps)
    return var, m, v


# ---- SURVEY 8f.4: BST transformer block (BST/transformer_layer.py:6-79) -------------------------------------------------

BST_PARAM_ORDER = ("position_embedding", "w_q", "w_k", "w_v", "w_o", "ln1_beta", "ln1_gamma", "dense_kernel", "dense_bias",
                   "ln2_beta", "ln2_gamma")


def bst_param_shapes(d, heads, max_length):
    return {"position_embedding": (max_length, d), "w_q": (heads, d, d), "w_k": (heads, d, d), "w_v": (heads, d, d),
            "w_o": (heads * d, d), "ln1_beta": (d,), "ln1_gamma": (d,), "dense_kernel": (d, d), "dense_bias": (d,),
            "ln2_beta": (d,), "ln2_gamma": (d,)}


def _layer_norm_td(x, beta, gamma):
    """tf.contrib.layers.layer_norm defaults on (B,T,d): moments over T AND d, params over d, eps 1e-12 [TF-internal]."""
    mean = x.mean(axis=(1, 2), keepdims=True)
    var = np.mean(np.square(x - mean), axis=(1, 2), keepdims=True)
    inv = (1.0 / np.sqrt(var + 1e-12)) * gamma
    return x * inv + (beta - mean * inv)


def bst_transformer_fwd(queries, keys, values, keys_length, p, heads, use_position_embedding=True):
    """One BST transformer block, float64 except where the reference's float32 arithmetic changes the RESULT:

    transformer_layer.py:28-37  queries/keys += position_embedding[0:T]  (values untouched; the residual at :71 uses the
                                 position-embedded queries because `queries +=` rebinds the name)
    :40-48   per head h: Q = xq @ w_q[h], K = xk @ w_k[h], V = v @ w_v[h], each (T, d)  (d_model == d_k per head)
    :52-57   keys_mask = (1 - sequence_mask(keys_length, T)) * (-2**32 + 1), expanded to (B,1,T,1): it is added along the
             QUERY axis, i.e. the same constant to every entry of a masked row.  Mathematically a no-op for the row softmax;
             in float32 (what the reference runs in) x + (-4294967296) rounds to the same value for every |x| < 256, so a
             masked query row attends UNIFORMLY (1/T).  That float32 effect is reproduced here (the add is done in float32).
    :60-63   softmax(Q K^T / sqrt(d_k) + mask) @ V ;  :66-68 heads concatenated (T, heads*d) @ w_o
    :71-72   layer_norm(all_heads + queries) ; :75-76 leakyrelu(dense(net)) with leak 0.01 ; :78-79 layer_norm(ffn + net).
    """
    q = np.asarray(queries, dtype=np.float64); k = np.asarray(keys, dtype=np.float64); v = np.asarray(values, dtype=np.float64)
    P = {n: np.asarray(a, dtype=np.float64) for n, a in p.items()}
    B, T, d = q.shape
    if use_position_embedding:
        q = q + P["position_embedding"][None, :T, :]
        k = k + P["position_embedding"][None, :T, :]
    masked = (np.arange(T)[None, :] >= np.asarray(keys_length)[:, None])                       # (B,T) query rows
    maskval = np.float32(-2 ** 32 + 1)
    heads_out = []
    for h in range(heads):
        Q = q @ P["w_q"][h]; K = k @ P["w_k"][h]; V = v @ P["w_v"][h]
        S = (Q @ K.transpose(0, 2, 1)) / np.sqrt(d)
        S32 = (S.astype(np.float32) + maskval).astype(np.float64)                             # float32 add, see docstring
        S = np.where(masked[:, :, None], S32, S)
        S = S - S.max(axis=-1, keepdims=True)
        A = np.exp(S); A = A / A.sum(axis=-1, keepdims=True)
        heads_out.append(A @ V)
    all_heads = np.concatenate(heads_out, axis=-1) @ P["w_o"]
    net = _layer_norm_td(all_heads + q, P["ln1_beta"], P["ln1_gamma"])
    f = net @ P["dense_kernel"] + P["dense_bias"]
    f = 0.5 * (1 + 0.01) * f + 0.5 * (1 - 0.01) * np.abs(f)                                   # BST/leakyrelu.py:4-16
    return _layer_norm_td(f + net, P["ln2_beta"], P["ln2_gamma"])


# ---- FFM second-order term (FFM/ffm.py:128-160): field-aware FM, a sibling of FM2 ----------------------------------------

def ffm_partner(i: int, s: int):
    """Field i keeps one sub-embedding per OTHER field: slot s of field i faces field j = s + 1 if s >= i else s, and field j
    faces i through its slot i - 1 if i > j else i  (ffm.py:154-155: embedding_variables[i][j-1], embedding_variables[j][i], i < j)."""
    j = s + 1 if s >= i else s
    return j, (i - 1 if i > j else i)


def ffm_fwd(tile: np.ndarray) -> np.ndarray:
    """tile (B, F, F-1, K): tile[b, i, s, :] = sub-embedding of field i's id for partner slot s (zero vector for a missing id:
    safe_embedding_lookup_sparse on an empty row).  Returns (B, 1): sum_{i<j} <v_i^(j), v_j^(i)>, pairs in the reference's
    loop order (ffm.py:146-160)."""
    B, F = tile.shape[0], tile.shape[1]
    out = np.zeros((B, 1), dtype=tile.dtype)
    for i in range(F - 1):
        for j in range(i + 1, F):
            out = out + np.sum(tile[:, i, j - 1, :] * tile[:, j, i, :], axis=-1, keepdims=True)
    return out


def ffm_bwd(tile: np.ndarray, g: np.ndarray) -> np.ndarray:
    """g (B,) or (B,1) -> d_tile: every (field, slot) position belongs to exactly one pair."""
    B, F = tile.shape[0], tile.shape[1]
    g = g.reshape(B, 1)
    d = np.zeros_like(tile)
    for i in range(F):
        for s in range(F - 1):
            j, sb = ffm_partner(i, s)
            d[:, i, s, :] = g * tile[:, j, sb, :]
    return d
