"""GPU parity: DIEN's interest extractor + attention + interest evolution (csrc/dien.cu) against the reference-executed
fixtures (tests/golden/dien) and the float64 restatement with its analytic backward (tests/_dien_ref.py), over a table of
shapes that reaches all 16 kernels (NHP = 8, 16, 32, 64 x AGRU / AUGRU) at their width, length and batch edges and through
the backward's persistent loop, plus a bitwise check that a sample's outputs do not depend on where it sits in the batch."""
import glob
import os
import sys

import numpy as np
import pytest
import torch

import _dien_ref as R
from _util import GOLDEN, TOL, assert_close, dev, elementwise_excess, relerr
from test_gpu_layer_variants import check_reduced, chunked_reference

pytestmark = pytest.mark.gpu

FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "dien", "*.npz")))
PNAMES = ("gk", "gb", "ck", "cb", "att", "egk", "egb", "eck", "ecb")


def _packed(params):
    return dev(np.concatenate([np.asarray(p, np.float32).reshape(-1) for p in params]))


def _inputs(B, T, na, nh, seed, lens=None):
    rng = np.random.default_rng(seed)
    L = rng.integers(0, T + 1, B) if lens is None else np.resize(np.asarray(lens, np.int64), B)
    seq = (rng.standard_normal((B, T, na)) * 0.7).astype(np.float32)
    seq[np.arange(T)[None, :] >= np.clip(L, 0, T)[:, None]] = 0
    tgt = (rng.standard_normal((B, na)) * 0.7).astype(np.float32)
    params = R.init_params(rng, na, nh, np.float32, bias_scale=0.5)
    g = rng.standard_normal((B, nh)).astype(np.float32)
    return seq, L.astype(np.int64), tgt, params, g


def _f64(a):
    return np.asarray(a, np.float64)


@pytest.mark.parametrize("name", FIXTURES)
def test_dien_fixture_through_ops_and_layers(name):
    from recalgorithm_b200 import layers as L, ops
    z = np.load(os.path.join(GOLDEN, "dien", name + ".npz"), allow_pickle=False)
    cell = 1 if "_augru_" in name else 0
    seq, lens, tgt = z["seq"], z["seq_len"], z["tgt"]
    nh = z["att"].shape[0]
    fs, att, _ = ops.dien_fwd(dev(seq), dev(lens), dev(tgt), _packed([z[k] for k in PNAMES]), nh, cell)
    assert_close(fs, z["final_state_f64"], TOL, f"{name} final_state vs reference (float64)")
    assert_close(att, z["att_f64"][..., 0], TOL, f"{name} attention vs reference (float64)")
    store = L.set_default_store(L.VariableStore(device="cuda", seed=0))
    with L.variable_scope("seq_encoder"):
        L.dien_interest_evolution(dev(seq), dev(lens), dev(tgt), str(nh), "AUGRU" if cell else "AGRU")
    from recalgorithm_b200.ops import DIEN_PARAM_ORDER
    store.assign({"seq_encoder/" + n: z[k] for n, k in zip(DIEN_PARAM_ORDER, PNAMES)})
    with L.variable_scope("seq_encoder"):
        fs2, att2 = L.dien_interest_evolution(dev(seq), dev(lens), dev(tgt), str(nh), "AUGRU" if cell else "AGRU",
                                              return_attention_scores=True)
    assert torch.equal(fs2, fs) and torch.equal(att2[..., 0], att)
    assert sorted(store.vars) == sorted("seq_encoder/" + n for n in DIEN_PARAM_ORDER)


def _nhp(nh):
    """The kernels' width class, dien_nhp (dien.cu:805)."""
    return 8 if nh <= 8 else 16 if nh <= 16 else 32 if nh <= 32 else 64


def _group(nh):
    """(G, SPW): a group of G = min(NHP, 32) lanes runs one sample and a warp runs SPW = 32 / G samples (dien.cu:75)."""
    G = min(_nhp(nh), 32)
    return G, 32 // G


def _lens(T):
    """Lengths cycled over the batch: negative (clamped to 0), 0, 1, 2, T - 1, T and past T, ordered so that the first warps
    of a multi-sample class mix the longest and shortest sequences (mixed warp lengths Lw, dien.cu:347 and :504), then
    every length in turn."""
    return [T, -1, T + 3, 0, T - 1, 1, 2] + list(range(T + 1))


def _resident_batch(nh):
    """A batch that gives every warp of the persistent backward (launch_resident, dien.cu:864) at least two tasks whatever
    occupancy it finds: more than twice the samples of 16 CTAs per SM (2048 threads / 128), 4 warps of SPW samples each,
    on every SM.  The remainder 4 SPW - 1 leaves the last warp (SPW > 1) and the last CTA partly filled."""
    _, spw = _group(nh)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return 2 * 16 * 4 * spw * sms + 4 * spw - 1


# (B, T, na, nh).  The class NHP (dien.cu:805) fixes G and SPW; a CTA holds 4 SPW samples.  Between them the rows of a class
# take nh at both ends of the class, na at 1, G - 1, G, G + 1 and 64 (the input row is spread over the group in slots of G,
# XRow at dien.cu:268, the backward's d x and d target at :685 and :757), T of 1, 2 (the forward prefetches two steps ahead,
# dien.cu:378), 3 and 128, B leaving the last warp and the last CTA partly filled, and B = "resident": _resident_batch, every
# backward warp loops over at least two tasks and accumulates the weight gradients across them (dien.cu:502).
SHAPES = [
    # the first six: one sample, ragged B, the reference shape, wide nh, the largest na and nh, and odd widths
    (1, 1, 16, 8), (333, 7, 16, 8), (1024, 50, 16, 8), (257, 50, 4, 16), (128, 20, 64, 64), (64, 13, 3, 5),
    # NHP = 8: G = 8, SPW = 4; the recurrent weights live in registers (dien.cu:203)
    (333, 2, 7, 1),       # nh = 1, seven dead units per group; na = G - 1; T = 2; last warp 1 of 4, last CTA 13 of 16
    (45, 3, 1, 8),        # nh = 8, the top of the class; na = 1; T = 3; last warp 1 of 4, last CTA 13 of 16
    (30, 5, 8, 3),        # na = G, one whole slot; last warp 2 of 4
    (50, 128, 9, 6),      # na = G + 1, a second slot with one live lane; T = 128; last warp 2 of 4
    (21, 6, 64, 7),       # na = 64, all 8 slots
    ("resident", 4, 9, 8),
    # NHP = 16: G = 16, SPW = 2; the first class with the weights staged in shared memory, padded columns past nh < 16
    (19, 1, 1, 16),       # nh = 16; na = 1; T = 1; last warp 1 of 2, last CTA 3 of 8
    (40, 2, 15, 9),       # nh = 9, the bottom of the class; na = G - 1; T = 2
    (33, 9, 16, 12),      # na = G; last warp 1 of 2
    (27, 3, 17, 9),       # na = G + 1; T = 3; last CTA 3 of 8
    (23, 128, 64, 13),    # na = 64; T = 128
    ("resident", 3, 17, 16),
    # NHP = 32: G = 32, U = 1, SPW = 1; shared-memory weights, padded columns past nh < 32
    (13, 3, 33, 17),      # nh = 17, the bottom of the class; na = G + 1; last CTA 1 of 4
    (30, 2, 1, 32),       # nh = 32; na = 1; T = 2
    (64, 128, 32, 32),    # na = G; T = 128
    (11, 5, 31, 24),      # na = G - 1
    (9, 1, 64, 20),       # na = 64; T = 1
    ("resident", 3, 31, 17),
    # NHP = 64: G = 32, U = 2, SPW = 1; lane g's second unit g + 32 (dien.cu:92) is dead where g + 32 >= nh, at every nh < 64
    (10, 3, 33, 33),      # nh = 33, one live lane in the second slot; na = G + 1; last CTA 2 of 4
    (31, 2, 31, 63),      # nh = 63, one dead lane; na = G - 1; T = 2
    (5, 1, 1, 40),        # na = 1; T = 1
    (15, 128, 32, 63),    # na = G; T = 128
    (30, 4, 64, 50),      # na = 64
    ("resident", 3, 33, 63),
]


def _err(got, want):
    """assert_close's two criteria as one ratio to compare with a tolerance: the larger of max|got - want| / max|want| and
    the worst element of |got - want| / (|want| + rms(want))."""
    return max(relerr(got, want), elementwise_excess(got, want, 1.0))


def test_shape_table_reaches_every_class_and_edge():
    """The table above holds the widths, lengths and batch remainders its comment promises, for every class."""
    assert {nh for *_, nh in SHAPES} >= {1, 8, 9, 16, 17, 32, 33, 63, 64}
    assert {T for _, T, _, _ in SHAPES} >= {1, 2, 3, 128}
    assert set(_lens(7)) >= {-1, 0, 1, 2, 6, 7, 10}
    for nhp in (8, 16, 32, 64):
        rows = [r for r in SHAPES if _nhp(r[3]) == nhp]
        G, spw = _group(rows[0][3])
        assert {na for _, _, na, _ in rows} >= {1, G - 1, G, G + 1, 64}, nhp
        sized = [B for B, *_ in rows if B != "resident"]
        assert spw == 1 or any(B % spw for B in sized), nhp
        assert any(B % (4 * spw) for B in sized), nhp
        assert sum(B == "resident" for B, *_ in rows) == 1, nhp


@pytest.mark.parametrize("cell", [0, 1])
@pytest.mark.parametrize("B,T,na,nh", SHAPES)
def test_dien_fwd_bwd_against_float64(B, T, na, nh, cell):
    """Forward and backward against float64.  final_state, the attention scores, d_seq and d_tgt are per sample and are held to
    TOL element-wise.  The nine weight gradients are batch-reduced (per-CTA shared-memory atomics, then global atomics), so
    they are held to check_reduced's bar over 64-sample chunks.

    At T >= 64 a correct float32 computation of d_seq and d_tgt comes close to TOL: there the bar is TOL or, if larger, 3x the
    worst error of the float32 restatement (tests/_dien_ref.py run in float32 on the same inputs), and both errors are
    printed.  No other output or case gets a looser bar."""
    from recalgorithm_b200 import ops
    if B == "resident":
        B = _resident_batch(nh)
    seq, L, tgt, params, g = _inputs(B, T, na, nh, seed=B + T + na + nh + cell, lens=_lens(T))
    p64 = [_f64(p) for p in params]
    fs, att, ws = ops.dien_fwd(dev(seq), dev(L), dev(tgt), _packed(params), nh, cell)
    d_seq, d_tgt, d_p = ops.dien_bwd(dev(seq), dev(L), dev(tgt), _packed(params), dev(g), nh, cell, ws)
    r_fs, r_att = R.dien_fwd(_f64(seq), L, _f64(tgt), p64, cell)

    def part(lo, hi):
        r_seq, r_tgt, r_p = R.dien_bwd(_f64(seq[lo:hi]), L[lo:hi], _f64(tgt[lo:hi]), p64, cell, _f64(g[lo:hi]))
        return {"d_seq": r_seq, "d_tgt": r_tgt}, dict(zip(PNAMES, r_p))
    per, red = chunked_reference(B, part)

    bars = {"final_state": TOL, "attention scores": TOL, "d_seq": TOL, "d_tgt": TOL}
    restated = {}
    if T >= 64:
        s_seq, s_tgt, _ = R.dien_bwd(seq, L, tgt, params, cell, g)
        for name, s in (("d_seq", s_seq), ("d_tgt", s_tgt)):
            restated[name] = _err(s, per[name])
            bars[name] = max(TOL, 3 * restated[name])
    errs = {"final_state": _err(fs, r_fs), "attention scores": _err(att, r_att), "d_seq": _err(d_seq, per["d_seq"]),
            "d_tgt": _err(d_tgt, per["d_tgt"])}
    case = f"B={B} T={T} na={na} nh={nh} NHP={_nhp(nh)} cell={cell}"
    print(f"{case}: " + ", ".join(f"{k} {v / TOL:.3f} TOL" for k, v in errs.items()) +
          "".join(f"; {k}: kernel {errs[k]:.2e}, float32 restatement {v:.2e}, bar {bars[k]:.2e}" for k, v in restated.items()))
    for name, e in errs.items():
        assert e <= bars[name], f"{case}: {name} error {e:.3e} > bar {bars[name]:.3e}"
    worst = max(check_reduced(got, red[n], f"{case}: d {name}")
                for n, name, got in zip(PNAMES, ops.DIEN_PARAM_ORDER, ops.dien_unpack_params(d_p, na, nh)))
    print(f"{case}: d_params {worst:.3f} of the reduced bar")

    pad = np.arange(T)[None, :] >= np.clip(L, 0, T)[:, None]
    assert torch.count_nonzero(d_seq[dev(pad)]) == 0, "padded positions get exactly 0"
    if cell == 0:
        dp = ops.dien_unpack_params(d_p, na, nh)
        assert torch.count_nonzero(dp[5][:, nh:]) == 0 and torch.count_nonzero(dp[6][nh:]) == 0, "AGRU: u half gets exactly 0"
    again = ops.dien_fwd(dev(seq), dev(L), dev(tgt), _packed(params), nh, cell)[0]
    assert torch.equal(again, fs), "deterministic forward"


@pytest.mark.parametrize("cell", [0, 1])
@pytest.mark.parametrize("nh", [5, 13, 29, 40])
def test_dien_sample_outputs_do_not_depend_on_placement(nh, cell):
    """A sample's final_state, attention scores, d_seq and d_tgt depend on nothing but its own inputs, so they are bit-identical
    whether it runs alone (B = 1), at each lane-group slot s of a warp (warp 1 + s) whose other samples have other lengths, or
    last in the batch, where the last warp (the last CTA at SPW = 1) is partly filled.  A width-G shuffle or a frozen group
    that leaks between the samples of a warp breaks this.  na = G + 1 gives every lane a partly filled second input slot."""
    from recalgorithm_b200 import ops
    G, spw = _group(nh)
    T, na = 9, G + 1
    B = spw * (spw + 2) + (spw - 1 if spw > 1 else 2)
    at = [spw * (1 + s) + s for s in range(spw)] + [B - 1]
    seq1, L1, tgt1, params, g1 = _inputs(1, T, na, nh, seed=nh + cell, lens=[T - 3])
    seq, L, tgt, _, g = _inputs(B, T, na, nh, seed=nh + cell + 1, lens=[T + 3, -1, T, 0, 1, 2, T - 1])
    seq[at], L[at], tgt[at], g[at] = seq1[0], L1[0], tgt1[0], g1[0]
    outs = []
    for s, ln, e, gg in ((seq1, L1, tgt1, g1), (seq, L, tgt, g)):
        fs, att, ws = ops.dien_fwd(dev(s), dev(ln), dev(e), _packed(params), nh, cell)
        d_seq, d_tgt, _ = ops.dien_bwd(dev(s), dev(ln), dev(e), _packed(params), dev(gg), nh, cell, ws)
        outs.append((fs, att, d_seq, d_tgt))
    assert torch.count_nonzero(outs[0][2]) > 0 and torch.count_nonzero(outs[0][3]) > 0
    for name, alone, batch in zip(("final_state", "attention scores", "d_seq", "d_tgt"), *outs):
        for i in at:
            assert torch.equal(batch[i], alone[0]), f"NHP={_nhp(nh)} cell={cell} {name}: sample {i} (warp {i // spw}, " \
                                                    f"slot {i % spw}, B={B}) differs from the sample run alone"


_PROFILE = """
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, "tests")
from _util import dev
from test_gpu_dien import SHAPES, _inputs, _lens, _packed
from recalgorithm_b200 import ops
out = []
for B, T, na, nh in SHAPES:
    B = 70 if B == "resident" else B                                # the kernel depends on nh and the cell only
    for cell in (0, 1):
        seq, L, tgt, params, g = _inputs(B, T, na, nh, seed=0, lens=_lens(T))
        a = (dev(seq), dev(L), dev(tgt), _packed(params))
        ops.dien_bwd(*a, dev(g), nh, cell, ops.dien_fwd(*a, nh, cell)[2])   # first launches (module load) outside the trace
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ops.dien_bwd(*a, dev(g), nh, cell, ops.dien_fwd(*a, nh, cell)[2])
            torch.cuda.synchronize()
        out.append([nh, cell, [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]])
print(json.dumps(out))
"""


def test_shape_table_launches_all_sixteen_kernels():
    """Every row of the table, in both cells, launches exactly the forward and backward kernel of its class, dien_nhp(nh)
    (dien.cu:805), and the table reaches all 16: dien_fwd_kernel and dien_bwd_kernel at NHP = 8, 16, 32, 64 and AGRU / AUGRU.
    The trace is taken in a process of its own, so that this profiler session leaves the test process's profiler as it was."""
    import json
    import re
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    run = subprocess.run([sys.executable, "-c", _PROFILE], cwd=root, capture_output=True, text=True, timeout=900)
    assert run.returncode == 0, run.stderr[-3000:]
    seen = set()
    for nh, cell, names in json.loads(run.stdout.strip().splitlines()[-1]):
        got = {(m[1], int(m[2]), int(m[3])) for n in names for m in [re.search(r"dien_(fwd|bwd)_kernel<(\d+), (\d+)>", n)] if m}
        assert got == {(k, _nhp(nh), cell) for k in ("fwd", "bwd")}, (nh, cell, names)
        seen |= got
    print("launched:", " ".join(f"dien_{k}_kernel<{n}, {c}>" for k, n, c in sorted(seen)))
    assert len(seen) == 16


@pytest.mark.parametrize("cell", [0, 1])
def test_dien_all_zero_lengths(cell):
    from recalgorithm_b200 import ops
    B, T, na, nh = 70, 9, 16, 8
    seq, L, tgt, params, g = _inputs(B, T, na, nh, seed=5, lens=[0])
    fs, att, ws = ops.dien_fwd(dev(seq), dev(L), dev(tgt), _packed(params), nh, cell)
    assert torch.count_nonzero(fs) == 0
    assert torch.all(att == torch.tensor(1.0 / T, device="cuda"))
    d_seq, d_tgt, d_p = ops.dien_bwd(dev(seq), dev(L), dev(tgt), _packed(params), dev(g), nh, cell, ws)
    for t in (d_seq, d_tgt, d_p):
        assert torch.count_nonzero(t) == 0


def test_dien_rejects_out_of_range_shapes():
    from recalgorithm_b200 import _lib, ops
    for B, T, na, nh in ((4, 129, 16, 8), (4, 10, 65, 8), (4, 10, 16, 65)):
        seq, L, tgt, params, g = _inputs(B, T, na, nh, seed=1)
        with pytest.raises(_lib.CtrInvalidArgument) as e:
            ops.dien_fwd(dev(seq), dev(L), dev(tgt), _packed(params), nh, 0)
        assert e.value.code == _lib.CTR_ERR_UNSUPPORTED and "ctr_dien_workspace_bytes" in str(e.value)


@pytest.mark.parametrize("entry", ["ctr_dien_fwd", "ctr_dien_bwd"])
@pytest.mark.parametrize("B,T,na,nh", [(4, 129, 16, 8), (4, 10, 65, 8), (4, 10, 16, 65), (700000, 128, 16, 8)])
def test_dien_entries_reject_out_of_range_shapes(entry, B, T, na, nh):
    """Both compute entries refuse shapes past their bounds themselves (T, na, nh, and B*T*(3nh+2) < 2^31), before touching
    any argument: called through the C ABI with small real buffers and a dummy workspace."""
    from recalgorithm_b200 import _lib
    h = _lib.lib()
    buf = torch.zeros(1 << 16, device="cuda")
    lens = torch.zeros(8, dtype=torch.int64, device="cuda")
    p, ln = buf.data_ptr(), lens.data_ptr()
    if entry == "ctr_dien_fwd":
        rc = h.ctr_dien_fwd(p, ln, p, p, B, T, na, nh, 0, p, p, p, buf.numel() * 4, None)
    else:
        rc = h.ctr_dien_bwd(p, ln, p, p, p, B, T, na, nh, 1, p, p, p, p, buf.numel() * 4, None)
    assert rc == _lib.CTR_ERR_UNSUPPORTED
    msg = h.ctr_last_error().decode()
    assert msg.startswith(entry) and ("unsupported" in msg or "too large" in msg), msg
    torch.cuda.synchronize()


@pytest.mark.parametrize("gru", ["AGRU", "AUGRU", "GRU"])
def test_dien_logit_body(gru):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import model_bodies as M
    from recalgorithm_b200 import autograd, layers as L
    B, T, H, rows = 96, 12, 16, 80
    store = L.set_default_store(L.VariableStore(device="cuda", seed=2))
    gen = torch.Generator(device="cuda").manual_seed(2)
    item = autograd.EmbeddingTables([rows], H, device="cuda")                 # the shared feedid table
    lens = torch.randint(0, T + 1, (B,), device="cuda", generator=gen)
    hist = torch.randint(0, rows, (B, T), device="cuda", generator=gen)
    hist[torch.arange(T, device="cuda")[None, :] >= lens[:, None]] = -1
    tgt = torch.randint(0, rows, (B, 1), device="cuda", generator=gen)
    seq = autograd.lookup(item, hist.reshape(B * T, 1)).reshape(B, T, H)
    target = autograd.lookup(item, tgt).reshape(B, H)
    dense_input = torch.randn(B, 3, device="cuda", generator=gen)
    cat = torch.randn(B, 8, device="cuda", generator=gen)
    y = (torch.rand((B, 1), device="cuda", generator=gen) < 0.3).float()
    logit, att = M.dien_logit(dense_input, cat, target, seq, lens, gru_output_units="8", custom_gru_type=gru)
    assert logit.shape == (B, 1) and att.shape == (B, T, 1) and torch.isfinite(logit).all()
    torch.nn.functional.binary_cross_entropy_with_logits(logit, y).backward()
    assert len(item.grad_slices) == 2 and all(float(s.values.abs().max()) > 0 for s in item.grad_slices)
    names = {"seq_encoder/" + n for n in ("rnn/gru_cell/gates/kernel", "attention_project_matrix", "rnn/gates/kernel",
                                          "rnn/candidate/bias", "fcn/dense/kernel", "fcn/dense_2/kernel")}
    assert names <= set(store.vars)
    for n, v in store.vars.items():
        assert v.grad is not None and torch.isfinite(v.grad).all(), n
    u_half = store.vars["seq_encoder/rnn/gates/kernel"].grad[:, 8:]
    assert (torch.count_nonzero(u_half) == 0) == (gru != "AUGRU")
