"""Float64 restatement of DIEN's seq_encoder block (DIEN/dien.py:198-229) with its analytic backward.

Forward, as the reference computes it:
  h_t = GRUCell(nh)(x_t, h_{t-1}) over every t < T from h_{-1} = 0 (TF 1.14 GRUCell: [r, u] = sigmoid([x, h] . Wg + bg),
        c = tanh([x, r*h] . Wc + bc), h' = u*h + (1-u)*c; no sequence_length, so padded positions are processed too);
  a   = softmax_t(where(t < len, h_t . (W e), -2**32 + 1));
  s_t = cell(h_t, s_{t-1}, a_t) for t < len, copied through afterwards (rnn.py _rnn_step, skip_conditionals=True):
        AGRU  (cell 0):  s' = (1-a)*s + a*c                                    (custom_grucell.py:90)
        AUGRU (cell 1):  u' = (1-a)*u;  s' = u'*s + (1-u')*c                    (custom_grucell.py:165-166)
  final_state = s after the last step.  len > T acts as T, len <= 0 as 0.

``skip=True`` computes only the positions t < len of each sample (what the kernels do); ``skip=False`` computes every
position and discards the padded ones with where(), as the reference does.  Every reduction is a fixed-order sum, so the
two forms can be compared bit for bit.
Params are the nine variables in the order of recalgorithm_b200.ops.DIEN_PARAM_ORDER:
  gk (na+nh, 2nh), gb (2nh), ck (na+nh, nh), cb (nh), W (nh, na), egk (2nh, 2nh), egb (2nh), eck (2nh, nh), ecb (nh).
"""
import numpy as np

PAD = -2.0 ** 32 + 1


def mm(x, w):
    """(n, k) . (k, m) with a fixed summation order per element (independent of n)."""
    return (x[:, :, None] * w[None, :, :]).sum(axis=1)


def outer_sum(a, b):
    """sum_n a[n, :, None] * b[n, None, :], rows accumulated in order."""
    out = np.zeros((a.shape[1], b.shape[1]), dtype=a.dtype)
    for i in range(a.shape[0]):
        out = out + a[i][:, None] * b[i][None, :]
    return out


def sig(z):
    return 1.0 / (1.0 + np.exp(-z))


def _gru(x, h, gk, gb, ck, cb):
    nh = h.shape[1]
    v = sig(mm(np.concatenate([x, h], 1), gk) + gb)
    r, u = v[:, :nh], v[:, nh:]
    c = np.tanh(mm(np.concatenate([x, r * h], 1), ck) + cb)
    return u * h + (1 - u) * c, r, u, c


def lengths(seq_len, T):
    return np.clip(np.asarray(seq_len, np.int64), 0, T)


def _rows(act, skip, B):
    return np.nonzero(act)[0] if skip else np.arange(B)


def softmax_masked(scores, L):
    T = scores.shape[1]
    s = np.where(np.arange(T)[None, :] < L[:, None], scores, scores.dtype.type(PAD))
    e = np.exp(s - s.max(1, keepdims=True))
    tot = e[:, 0].copy()
    for t in range(1, T):
        tot = tot + e[:, t]
    return e / tot[:, None]


def dien_fwd(seq, seq_len, tgt, params, cell, skip=True, return_cache=False):
    """-> (final_state (B,nh), attention scores (B,T)) [, cache for dien_bwd]."""
    gk, gb, ck, cb, W, egk, egb, eck, ecb = params
    B, T, na = seq.shape
    nh = W.shape[0]
    L = lengths(seq_len, T)
    dt = seq.dtype
    H = np.full((B, T, nh), np.nan if skip else 0, dt)        # skip: positions never computed stay NaN
    h = np.zeros((B, nh), dt)
    for t in range(T):
        act = t < L
        rows = _rows(act, skip, B) if skip else np.arange(B)  # the extractor has no sequence_length
        if skip:
            h[rows] = _gru(seq[rows, t], h[rows], gk, gb, ck, cb)[0]
        else:
            h = _gru(seq[:, t], h, gk, gb, ck, cb)[0]
        H[rows, t] = h[rows]
    v = mm(tgt, W.T)                                           # W . e_a per sample
    scores = np.where(np.arange(T)[None, :] < L[:, None], (np.nan_to_num(H) * v[:, None, :]).sum(-1), 0)
    A = softmax_masked(scores.astype(dt), L)
    s = np.zeros((B, nh), dt)
    S = np.zeros((B, T, nh), dt)
    for t in range(T):
        act = t < L
        rows = _rows(act, skip, B)
        x, sp, a = H[rows, t], s[rows], A[rows, t][:, None]
        if not skip:
            x = np.nan_to_num(x)
        _, r, u, c = _gru(x, sp, egk, egb, eck, ecb)
        if cell == 1:
            ua = (1 - a) * u
            sn = ua * sp + (1 - ua) * c
        else:
            sn = (1 - a) * sp + a * c
        s[rows] = sn if skip else np.where(act[:, None], sn, sp)
        S[rows, t] = s[rows]
    if return_cache:
        return s, A, dict(H=H, S=S, A=A, v=v, L=L)
    return s, A


def dien_bwd(seq, seq_len, tgt, params, cell, g_final, skip=True):
    """-> (d_seq (B,T,na), d_tgt (B,na), [d of each of the nine params])."""
    gk, gb, ck, cb, W, egk, egb, eck, ecb = params
    B, T, na = seq.shape
    nh = W.shape[0]
    _, A, cc = dien_fwd(seq, seq_len, tgt, params, cell, skip=skip, return_cache=True)
    H, S, v, L = cc["H"], cc["S"], cc["v"], cc["L"]
    H0 = np.nan_to_num(H)
    d = [np.zeros_like(p) for p in params]
    dgk, dgb, dck, dcb, dW, degk, degb, deck, decb = d
    # ---- evolution cell
    dH = np.zeros_like(H0)
    dA = np.zeros((B, T), seq.dtype)
    ds = g_final.copy()
    for t in range(T - 1, -1, -1):
        act = t < L
        rows = _rows(act, skip, B)
        x = H0[rows, t]
        sp = S[rows, t - 1] if t > 0 else np.zeros((len(rows), nh), seq.dtype)
        a = A[rows, t][:, None]
        g = ds[rows] if skip else np.where(act[:, None], ds, 0)
        _, r, u, c = _gru(x, sp, egk, egb, eck, ecb)
        if cell == 1:
            ua = (1 - a) * u
            dua = g * (sp - c)
            dc, dsp, du = g * (1 - ua), g * ua, dua * (1 - a)
            da = -(dua * u).sum(1)
        else:
            dc, dsp, du = g * a, g * (1 - a), np.zeros_like(g)
            da = (g * (c - sp)).sum(1)
        dzc = dc * (1 - c * c)
        din = mm(dzc, eck.T)
        dx, drs = din[:, :nh], din[:, nh:]
        dsp = dsp + drs * r
        dzr = drs * sp * r * (1 - r)
        dzu = du * u * (1 - u)
        dzg = np.concatenate([dzr, dzu], 1)
        din = mm(dzg, egk.T)
        dx, dsp = dx + din[:, :nh], dsp + din[:, nh:]
        degk += outer_sum(np.concatenate([x, sp], 1), dzg)
        degb += dzg.sum(0)
        deck += outer_sum(np.concatenate([x, r * sp], 1), dzc)
        decb += dzc.sum(0)
        dH[rows, t] = dx
        dA[rows, t] = da
        ds[rows] = dsp if skip else np.where(act[:, None], dsp, ds)
    # ---- softmax (masked positions receive no gradient: tf.where routes it to the constant)
    ada = A[:, 0] * dA[:, 0]
    for t in range(1, T):
        ada = ada + A[:, t] * dA[:, t]
    dsc = np.where(np.arange(T)[None, :] < L[:, None], A * (dA - ada[:, None]), 0)
    # ---- extractor
    d_seq = np.zeros_like(seq)
    dv = np.zeros((B, nh), seq.dtype)
    carry = np.zeros((B, nh), seq.dtype)
    for t in range(T - 1, -1, -1):
        act = t < L
        rows = _rows(act, skip, B)
        x = seq[rows, t]
        hp = H0[rows, t - 1] if t > 0 else np.zeros((len(rows), nh), seq.dtype)
        dh = carry[rows] + dH[rows, t] + dsc[rows, t][:, None] * v[rows]
        dv[rows] += dsc[rows, t][:, None] * H0[rows, t]
        _, r, u, c = _gru(x, hp, gk, gb, ck, cb)
        du, dc, dhp = dh * (hp - c), dh * (1 - u), dh * u
        dzc = dc * (1 - c * c)
        din = mm(dzc, ck.T)
        dx, drh = din[:, :na], din[:, na:]
        dhp = dhp + drh * r
        dzr = drh * hp * r * (1 - r)
        dzu = du * u * (1 - u)
        dzg = np.concatenate([dzr, dzu], 1)
        din = mm(dzg, gk.T)
        dx, dhp = dx + din[:, :na], dhp + din[:, na:]
        dgk += outer_sum(np.concatenate([x, hp], 1), dzg)
        dgb += dzg.sum(0)
        dck += outer_sum(np.concatenate([x, r * hp], 1), dzc)
        dcb += dzc.sum(0)
        d_seq[rows, t] = dx
        carry[rows] = dhp
    d_tgt = mm(dv, W)
    dW += outer_sum(dv, tgt)
    return d_seq, d_tgt, d


def init_params(rng, na, nh, dtype=np.float32, bias_scale=None):
    """Glorot-uniform kernels; gate biases ones and candidate biases zeros (the variables' initialisers), or uniform in
    +-bias_scale when given (so that a test exercises the bias gradients away from the initial values)."""
    g = lambda shape: rng.uniform(-1, 1, size=shape) * np.sqrt(6.0 / (shape[0] + shape[1]))
    b = lambda n, base: (rng.uniform(-bias_scale, bias_scale, n) if bias_scale else np.full(n, base))
    p = [g((na + nh, 2 * nh)), b(2 * nh, 1.0), g((na + nh, nh)), b(nh, 0.0), g((nh, na)), g((2 * nh, 2 * nh)), b(2 * nh, 1.0),
         g((2 * nh, nh)), b(nh, 0.0)]
    return [x.astype(dtype) for x in p]
