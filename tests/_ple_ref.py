"""Float64 restatement of PLE's expert-gate blocks -- the extraction network (PLE/extraction_network.py:4-85) and the final
experts and gates (PLE/ple.py:185-226) -- with their analytic backward.  The GPU tests compare the kernels against it, and
tests/test_ple_oracle.py pins it to the reference-executed fixtures.

Both blocks are one computation: E = sum n_t + S experts in [task 0 .. task T-1, shared] order, gate t over [task t's
experts, shared experts], and in the extraction network an all-gate over every expert; the gate kernels are concatenated
by columns, w_gates (d, GC).  The final layer returns T outputs (gate t -> output t); the extraction network sums every
gated output into one (B, H).  Written in torch so that the same code runs in float64 on the CPU and, at 65 536 samples,
on the GPU."""
import numpy as np
import torch


def gate_experts(n, S, extraction):
    """Per gate, the experts its columns point at, in column order."""
    es = sum(n)
    e0 = np.cumsum([0] + list(n))
    gates = [list(range(e0[t], e0[t] + n[t])) + list(range(es, es + S)) for t in range(len(n))]
    if extraction:
        gates.append(list(range(es + S)))
    return gates


def fwd(x, we, be, wg, n, S, extraction):
    """x (B,d), we (E,d,H), be (E,H), wg (d,GC) -> (out ((B,H) or (T,B,H)), gates (B,GC), pre-activations a (E,B,H))."""
    a = x @ we + be[:, None, :]
    h = torch.relu(a)
    z = x @ wg
    outs, ps, c = [], [], 0
    for experts in gate_experts(n, S, extraction):
        p = torch.softmax(z[:, c:c + len(experts)], dim=-1)
        ps.append(p)
        outs.append(torch.einsum("bj,jbh->bh", p, h[experts]))
        c += len(experts)
    out = sum(outs) if extraction else torch.stack(outs)
    return out, torch.cat(ps, dim=1), a


def bwd(x, we, be, wg, g, n, S, extraction):
    """(d_x, d_we, d_be, d_wg, dz (E,B,H), dlogit (B,GC)) for the upstream gradient g, shaped as out."""
    _, p, a = fwd(x, we, be, wg, n, S, extraction)
    h = torch.relu(a)
    dz = torch.zeros_like(a)
    dls, c = [], 0
    for gi, experts in enumerate(gate_experts(n, S, extraction)):
        go = g if extraction else g[gi]
        pg = p[:, c:c + len(experts)]
        dp = torch.einsum("bh,jbh->bj", go, h[experts])
        dls.append(pg * (dp - (pg * dp).sum(-1, keepdim=True)))
        dz[experts] += pg.T[:, :, None] * go[None]
        c += len(experts)
    dz = dz * (a > 0)
    dlogit = torch.cat(dls, dim=1)
    d_x = torch.einsum("ebh,edh->bd", dz, we) + dlogit @ wg.T
    return d_x, torch.einsum("bd,ebh->edh", x, dz), dz.sum(1), x.T @ dlogit, dz, dlogit


def hashed_codes(seed, shape, half):
    """Integers in [-half, half] of the given shape from a counter-based hash (splitmix64 of seed and the element index):
    the fixture weights, regenerated here instead of stored, which keeps the archives small.  Plain uint64 arithmetic, so
    the values do not depend on any random-number generator's version."""
    with np.errstate(over="ignore"):
        z = np.arange(int(np.prod(shape)), dtype=np.uint64) + np.uint64(seed) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return ((z % np.uint64(2 * half + 1)).astype(np.int64) - half).reshape(shape)


# (code range, scale) of w_experts, b_experts and w_gates: integer multiples of a power of two, exact in float32;
# expert kernels about glorot-uniform at d = 82..256, H = 256, gates far from uniform
WEIGHT_CODES = ((26, 1 / 256), (25, 1 / 256), (32, 1 / 128))


def fixture_weights(seed, E, d, H, GC):
    """(w_experts (E,d,H), b_experts (E,H), w_gates (d,GC)) of a fixture, float64, from its weight seed."""
    return tuple(hashed_codes(seed + k, shape, half).astype(np.float64) * scale
                 for k, (shape, (half, scale)) in enumerate(zip(((E, d, H), (E, H), (d, GC)), WEIGHT_CODES)))


def fixture(z):
    """(x, w_experts, b_experts, w_gates) of a tests/golden/ple fixture as float64 tensors, and (n, S, extraction)."""
    n, S, extraction = [int(v) for v in z["experts_per_task"]], int(z["num_experts_in_shared"]), bool(z["extraction"])
    x = np.asarray(z["x"], np.float64)
    E, (B, d), H = sum(n) + S, x.shape, z["out_f64"].shape[-1]
    GC = sum(n) + len(n) * S + ((sum(n) + S) if extraction else 0)
    arrays = (x,) + fixture_weights(int(z["weight_seed"]), E, d, H, GC)
    return tuple(torch.from_numpy(a) for a in arrays), (n, S, extraction)
