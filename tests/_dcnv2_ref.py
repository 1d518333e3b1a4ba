"""Float64 restatement of the DCN-V2 cross network (Wang et al., WWW 2021, arXiv:2008.13535, eq. 1-2) and its analytic
backward, in the row-vector form of include/ctr_b200.h's Row CROSS-V2:

    x_{l+1} = x0 * z_l + x_l,   z_l = x_l . W_l + b_l,   W_l = w[l] (full rank) or w[l] . u[l] (low rank)

with x_0 = xl when given, else x0."""
import numpy as np


def _f64(a):
    return None if a is None else np.asarray(a, dtype=np.float64)


def cross_v2_fwd(x0, w, u, b, xl=None):
    """-> (out (B,d), cache).  w (L,d,d) with u None, or w (L,d,r) and u (L,r,d); b (L,d)."""
    x0, w, u, b = _f64(x0), _f64(w), _f64(u), _f64(b)
    x = x0 if xl is None else _f64(xl)
    xs, zs, ts = [], [], []
    for l in range(w.shape[0]):
        xs.append(x)
        t = None if u is None else x @ w[l]
        z = (x @ w[l] if u is None else t @ u[l]) + b[l]
        ts.append(t)
        zs.append(z)
        x = x0 * z + x
    return x, (x0, xs, zs, ts, xl is not None)


def cross_v2_bwd(cache, w, u, g_out):
    """-> (dx0, dxl | None, dw, du | None, db) given dL/dout."""
    x0, xs, zs, ts, has_xl = cache
    w, u, g = _f64(w), _f64(u), _f64(g_out)
    dx0 = np.zeros_like(x0)
    dw, db = np.zeros_like(w), np.zeros((w.shape[0], x0.shape[1]))
    du = None if u is None else np.zeros_like(u)
    for l in range(w.shape[0] - 1, -1, -1):
        dz = g * x0
        dx0 += g * zs[l]
        db[l] = dz.sum(0)
        if u is None:
            dw[l] = xs[l].T @ dz
            g = g + dz @ w[l].T
        else:
            du[l] = ts[l].T @ dz
            dt = dz @ u[l].T
            dw[l] = xs[l].T @ dt
            g = g + dt @ w[l].T
    if has_xl:
        return dx0, g, dw, du, db
    return dx0 + g, None, dw, du, db
