"""Float64 restatement of DIEN's auxiliary loss (DIEN/dien.py:256-300) with the paper's sign, and its analytic backward
through the seq_encoder block (tests/_dien_ref.py).

With L = clamp(len, 0, T), W = aux_project_matrix (na, nh), q_t = W h_t and the negatives of position t in rows
t*T_neg .. t*T_neg + T_neg - 1 of neg (B, (T-1)*T_neg, na):
  aux_loss = -(1/B) sum_b sum_{t < L-1} [ log sig(q_t . x_{t+1}) + sum_n log(1 - sig(q_t . neg_{t,n})) ]
           =  (1/B) sum_b sum_{t < L-1} [ softplus(-z+_t) + sum_n softplus(z-_{t,n}) ]
-- the negative of the reference's aux_loss.  Positions t >= L-1 are never computed (``reference_form`` computes every
position with tf.log(tf.sigmoid(.)) and masks by multiplication, as the reference does).
"""
import numpy as np

import _dien_ref as R


def softplus(z):
    return np.logaddexp(0.0, z)


def _split(seq, neg, T_neg):
    B, T, na = seq.shape
    return seq[:, 1:], neg.reshape(B, T - 1, T_neg, na)


def counted(seq_len, T):
    """(B, T-1) mask of the positions that carry a term: t < L - 1 (sequence_mask(len - 1, T - 1), dien.py:286)."""
    return np.arange(T - 1)[None, :] < (R.lengths(seq_len, T) - 1)[:, None]


def logits(H, seq, neg, W, T_neg):
    """q (B,T-1,na), z+ (B,T-1), z- (B,T-1,T_neg) from the extractor states H (B,T,nh)."""
    pos, negr = _split(seq, neg, T_neg)
    q = np.nan_to_num(H[:, :-1]) @ W.T
    return q, (q * pos).sum(-1), np.einsum("bti,btni->btn", q, negr)


def aux_fwd(H, seq, seq_len, neg, W, T_neg):
    """aux_loss from the extractor states; per-sample terms summed in position order, samples in batch order."""
    B, T, _ = seq.shape
    _, zp, zn = logits(H, seq, neg, W, T_neg)
    m = counted(seq_len, T)
    term = np.where(m, softplus(-zp) + softplus(zn).sum(-1), 0.0)
    return term.sum() / B if B else 0.0 * term.sum()


def reference_form(H, seq, seq_len, neg, W, T_neg):
    """The reference's arithmetic with its sign flipped: log(sigmoid(.)) at every position, masked by multiplication."""
    B, T, _ = seq.shape
    _, zp, zn = logits(H, seq, neg, W, T_neg)
    sig = lambda z: 1.0 / (1.0 + np.exp(-z))
    m = counted(seq_len, T).astype(seq.dtype)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        pos = (np.log(sig(zp)) * m).sum(1)
        negp = (np.log(1 - sig(zn)) * m[..., None]).sum((1, 2))
    return -np.mean(pos + negp)


def dien_aux_fwd(seq, seq_len, tgt, neg, params, W, cell, T_neg):
    """-> (final_state, attention scores, aux_loss)."""
    fs, A, cc = R.dien_fwd(seq, seq_len, tgt, params, cell, return_cache=True)
    return fs, A, aux_fwd(cc["H"], seq, seq_len, neg, W, T_neg)


def aux_bwd(H, seq, seq_len, neg, W, T_neg, g_aux):
    """-> (d_seq part (B,T,na), d_neg, dL/dH (B,T,nh), d_W) of g_aux * aux_loss."""
    B, T, na = seq.shape
    pos, negr = _split(seq, neg, T_neg)
    q, zp, zn = logits(H, seq, neg, W, T_neg)
    m = counted(seq_len, T)
    s = g_aux / B
    gp = np.where(m, s * (R.sig(zp) - 1.0), 0.0)
    gn = np.where(m[..., None], s * R.sig(zn), 0.0)
    d_seq = np.zeros_like(seq)
    d_seq[:, 1:] = gp[..., None] * q
    d_neg = (gn[..., None] * q[:, :, None, :]).reshape(neg.shape)
    dq = gp[..., None] * pos + np.einsum("btn,btni->bti", gn, negr)
    dH = np.zeros(H.shape, seq.dtype)
    dH[:, :-1] = dq @ W
    dW = np.einsum("bti,btj->ij", dq, np.nan_to_num(H[:, :-1]))
    return d_seq, d_neg, dH, dW


def extractor_bwd(seq, seq_len, params, H, dH):
    """BPTT through the extractor GRU (the last block of R.dien_bwd) from the seeds dH (B,T,nh) = dL/dh_t alone:
    -> (d_seq, [d gk, d gb, d ck, d cb])."""
    gk, gb, ck, cb = params[:4]
    B, T, na = seq.shape
    nh = gb.shape[0] // 2
    L = R.lengths(seq_len, T)
    H0 = np.nan_to_num(H)
    d_seq = np.zeros_like(seq)
    d = [np.zeros_like(p) for p in (gk, gb, ck, cb)]
    carry = np.zeros((B, nh), seq.dtype)
    for t in range(T - 1, -1, -1):
        rows = np.nonzero(t < L)[0]
        x = seq[rows, t]
        hp = H0[rows, t - 1] if t > 0 else np.zeros((len(rows), nh), seq.dtype)
        dh = carry[rows] + dH[rows, t]
        _, r, u, c = R._gru(x, hp, gk, gb, ck, cb)
        du, dc, dhp = dh * (hp - c), dh * (1 - u), dh * u
        dzc = dc * (1 - c * c)
        din = R.mm(dzc, ck.T)
        dx, drh = din[:, :na], din[:, na:]
        dhp = dhp + drh * r
        dzr = drh * hp * r * (1 - r)
        dzu = du * u * (1 - u)
        dzg = np.concatenate([dzr, dzu], 1)
        din = R.mm(dzg, gk.T)
        dx, dhp = dx + din[:, :na], dhp + din[:, na:]
        d[0] += R.outer_sum(np.concatenate([x, hp], 1), dzg)
        d[1] += dzg.sum(0)
        d[2] += R.outer_sum(np.concatenate([x, r * hp], 1), dzc)
        d[3] += dzc.sum(0)
        d_seq[rows, t] = dx
        carry[rows] = dhp
    return d_seq, d


def dien_aux_bwd(seq, seq_len, tgt, neg, params, W, cell, T_neg, g_final, g_aux):
    """Gradients of (final_state, aux_loss) given (g_final (B,nh), g_aux scalar): -> (d_seq, d_neg, d_tgt,
    [d of each of the nine params], d_W).  The backward is linear in the seeds, so it is R.dien_bwd plus the aux terms and
    the extractor's BPTT of their dL/dh."""
    _, _, cc = R.dien_fwd(seq, seq_len, tgt, params, cell, return_cache=True)
    d_seq, d_tgt, dp = R.dien_bwd(seq, seq_len, tgt, params, cell, g_final)
    a_seq, d_neg, dH, dW = aux_bwd(cc["H"], seq, seq_len, neg, W, T_neg, g_aux)
    e_seq, de = extractor_bwd(seq, seq_len, params, cc["H"], dH)
    dp = [p + e for p, e in zip(dp, de)] + list(dp[4:])
    return d_seq + a_seq + e_seq, d_neg, d_tgt, dp, dW
