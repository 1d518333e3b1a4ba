"""Float64 restatement of MMoE's experts, gates and tower sums (MMOE/mmoe.py:207-236) with its analytic backward; the GPU tests
compare the kernels against it, and tests/test_mmoe_oracle.py pins it to the reference-executed fixtures."""
import numpy as np


def softmax(z):
    z = z - z.max(axis=-1, keepdims=True)
    e = np.exp(z)
    return e / e.sum(axis=-1, keepdims=True)


def fwd(x, we, be, wg):
    """x (B,d), we (E,d,H), be (E,H), wg (T,d,E) -> (towers (T,B,H), gates (T,B,E), expert pre-activations a (E,B,H))."""
    a = x @ we + be[:, None, :]                                   # (E,B,H); matmul rather than einsum: BLAS at 65 536 samples
    h = np.maximum(a, 0)
    p = softmax(x @ wg)
    return (p.transpose(1, 0, 2) @ h.transpose(1, 0, 2)).transpose(1, 0, 2), p, a


def bwd(x, we, be, wg, g):
    """(d_x, d_we, d_be, d_wg) for upstream gradient g (T,B,H)."""
    _, p, a = fwd(x, we, be, wg)
    h = np.maximum(a, 0)
    dp = (g.transpose(1, 0, 2) @ h.transpose(1, 2, 0)).transpose(1, 0, 2)                                 # (T,B,E)
    dlogit = p * (dp - (p * dp).sum(-1, keepdims=True))
    dz = (p.transpose(1, 2, 0) @ g.transpose(1, 0, 2)).transpose(1, 0, 2) * (a > 0)                         # (E,B,H)
    d_x = (dz @ we.transpose(0, 2, 1)).sum(0) + (dlogit @ wg.transpose(0, 2, 1)).sum(0)
    return d_x, x.T @ dz, dz.sum(1), x.T @ dlogit


def fixture(z):
    """(x, w_experts, b_experts, w_gates) of a tests/golden/mmoe fixture, in float64."""
    return tuple(np.asarray(z[k], np.float64) for k in ("x", "w_experts", "b_experts", "w_gates"))


def chunked_torch(x, we, be, wg, g, chunk=64, group=128):
    """The same forward and backward in float64 torch on the tensors' device (the GPU tests use it at 65 536 samples, where
    NumPy takes seconds): per-sample (towers (T,B,H), gates (T,B,E), d_x (B,d)), and each batch-reduced gradient as
    (sum over the batch, sum over `chunk`-sample chunks of |chunk sum|) -- the (ref, magnitude) pair of
    test_gpu_layer_variants.chunked_reference, computed for all chunks at once (the batch is zero padded to whole chunks: a
    padded sample has g = 0 and adds nothing)."""
    import torch
    B, d = x.shape
    nc = max(1, -(-B // chunk))
    pad = nc * chunk - B
    x = torch.nn.functional.pad(x, (0, 0, 0, pad))
    g = torch.nn.functional.pad(g, (0, 0, 0, pad))
    a = x @ we + be[:, None, :]
    h = torch.relu(a)
    p = torch.softmax(x @ wg, dim=-1)
    towers = torch.einsum("tbe,ebh->tbh", p, h)
    dp = torch.einsum("tbh,ebh->tbe", g, h)
    dlogit = p * (dp - (p * dp).sum(-1, keepdim=True))
    dz = torch.einsum("tbe,tbh->ebh", p, g) * (a > 0)
    d_x = torch.einsum("ebh,edh->bd", dz, we) + torch.einsum("tbe,tde->bd", dlogit, wg)
    E, T = we.shape[0], wg.shape[0]
    xc, dzc, dlc = x.view(nc, chunk, d), dz.view(E, nc, chunk, -1), dlogit.view(T, nc, chunk, -1)
    red = {k: [0.0, 0.0] for k in ("dwe", "dbe", "dwg")}
    for c0 in range(0, nc, group):
        sl = slice(c0, min(nc, c0 + group))
        parts = {"dwe": torch.einsum("cbd,ecbh->cedh", xc[sl], dzc[:, sl]), "dbe": dzc[:, sl].sum(2).transpose(0, 1),
                 "dwg": torch.einsum("cbd,tcbe->ctde", xc[sl], dlc[:, sl])}
        for k, v in parts.items():
            red[k][0] = red[k][0] + v.sum(0)
            red[k][1] = red[k][1] + v.abs().sum(0)
    per = {"towers": towers[:, :B], "gates": p[:, :B], "dx": d_x[:B]}
    return ({k: v.cpu().numpy() for k, v in per.items()},
            {k: (v[0].cpu().numpy(), v[1].cpu().numpy()) for k, v in red.items()})
