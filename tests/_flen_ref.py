"""Float64 restatement of FLEN's field-wise bi-interaction (FwBI; Chen et al., arXiv:1911.04690) and its analytic backward.
The reference tree has no FLEN code, so this restatement of the layer's definition (include/ctr_b200.h) is the parity target
of csrc/flen.cu; tests/test_flen_oracle.py checks it against torch.autograd, a brute-force pair loop and, through two
degenerate groupings, against the NFM and FwFM fixtures executed from the reference's own lines."""
import itertools

import numpy as np


def pairs(M):
    """kernel_mf's index order: the row-major strict upper triangle of M x M."""
    return list(itertools.combinations(range(M), 2))


def group_sums(e, group, M):
    """p (B,M,D) = per-group sum of e (B,F,D), q = per-group sum of e*e."""
    e = np.asarray(e, np.float64)
    B, F, D = e.shape
    p = np.zeros((B, M, D))
    q = np.zeros((B, M, D))
    for f, m in enumerate(group):
        p[:, m] += e[:, f]
        q[:, m] += e[:, f] * e[:, f]
    return p, q


def fwbi_fwd(e, group, M, kmf, kfm, bmf, bfm):
    """h (B,D) = sum_{i<j} kmf[pair(i,j)] p_i p_j + bmf + sum_m kfm[m] (p_m^2 - q_m) + bfm."""
    p, q = group_sums(e, group, M)
    kmf, kfm = np.asarray(kmf, np.float64), np.asarray(kfm, np.float64)
    h = np.zeros((p.shape[0], p.shape[2])) + np.asarray(bmf, np.float64)
    for k, (i, j) in enumerate(pairs(M)):
        h += kmf[k] * p[:, i] * p[:, j]
    h_fm = np.asarray(bfm, np.float64) + np.einsum("m,bmd->bd", kfm, p * p - q)
    return h + h_fm


def fwbi_bwd(e, group, M, kmf, kfm, g, d_tile=None):
    """(row_grads (B,F,D), d_kmf, d_kfm, d_bmf, d_bfm) for g = dL/dh (B,D)."""
    e = np.asarray(e, np.float64)
    g = np.asarray(g, np.float64)
    kmf, kfm = np.asarray(kmf, np.float64), np.asarray(kfm, np.float64)
    p, q = group_sums(e, group, M)
    a = np.zeros_like(p)                                   # a_m = sum_{j != m} kmf[pair(m,j)] p_j
    d_kmf = np.zeros(len(kmf))
    for k, (i, j) in enumerate(pairs(M)):
        a[:, i] += kmf[k] * p[:, j]
        a[:, j] += kmf[k] * p[:, i]
        d_kmf[k] = np.sum(g * p[:, i] * p[:, j])
    d_kfm = np.einsum("bd,bmd->m", g, p * p - q)
    grp = np.asarray(group)
    rg = g[:, None, :] * (a[:, grp] + 2.0 * kfm[grp][None, :, None] * (p[:, grp] - e))
    if d_tile is not None:
        rg = rg + np.asarray(d_tile, np.float64)
    db = g.sum(0)
    return rg, d_kmf, d_kfm, db, db.copy()
