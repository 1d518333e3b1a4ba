"""BASELINE configs 2-4 as lookup + interaction chains (hot path only: no dense tail), used by bench.py (`--workload
dcn_cfg2|xdeepfm_cfg3|din_cfg4` and the `configs` key of the default line) and tools/bench_layers.py.

Every builder returns a dict:
    step(ev=None)   one forward+backward pass of the chain on the current stream; `ev` (list of CUDA events, len = n_marks)
                    is recorded between the stages so the caller can split the step per kernel
    outputs         name -> tensor: what the last step computed (bench.py --dump-outputs)
    marks           names of the stages between consecutive events
    B, config       batch and the config keys for the JSON line
    roofline(ms_by_stage, ms_step, peaks) -> dict   the roofline object of the dominant kernel
Tables: 1 M rows per field (SURVEY 8d).  Inputs are created on the device with a fixed seed.
"""
from __future__ import annotations

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from recalgorithm_b200 import ops  # noqa: E402

FP32_FMA_TFLOPS = 132 * 128 * 2 * 1.98e9 / 1e12      # H100 SXM: 132 SMs x 128 FMA lanes x 2 FLOP x 1.98 GHz = 66.9 TFLOP/s (nominal)


def _rn(gen, *s, std=1.0):
    return torch.randn(s, device="cuda", generator=gen) * std


def _rec(ev, i):
    if ev is not None:
        ev[i].record()


def build_dcn_cfg2(rows=1_000_000, B=4096):
    """Config 2: DCN, 30 fields x 16 = 480 wide, 3 cross layers (DCN/dcn.py:157-160)."""
    gen = torch.Generator(device="cuda").manual_seed(1234)
    F, D, L = 30, 16, 3
    d = F * D
    table = _rn(gen, rows * F, D, std=D ** -0.5)
    off = torch.arange(F + 1, device="cuda") * rows
    ids = [torch.randint(0, rows, (B, F), device="cuda", generator=gen) for _ in range(4)]
    w, bb, g = _rn(gen, L, d, std=0.05), _rn(gen, L, d, std=0.05), _rn(gen, B, d)
    k = [0]

    x0, xl = torch.empty((B, d), device="cuda"), torch.empty((B, d), device="cuda")
    outputs = {"x0": x0, "cross_out": xl}

    def step(ev=None):
        k[0] += 1
        _rec(ev, 0)
        ops.embed_cross_fwd(table, off, ids[k[0] % 4], w, bb, x0=x0, out=xl)     # input_layer gather + the cross loop, ONE launch
        _rec(ev, 1)
        dx0, _, dw, db = ops.cross_bwd(x0, w, bb, g)
        outputs.update(d_x0=dx0, d_w=dw, d_b=db)
        _rec(ev, 2)
        # lookup backward of a plain gather (no FM2 term): the IndexedSlices values ARE dx0.view(B,F,D) -- no kernel, no bytes
        _rec(ev, 3)

    bytes_step = B * (F * (8 + 2 * D * 4) + 20 * d)                      # lookup fwd + cross fwd/bwd (20*d); lookup bwd is an alias

    def roofline(ms, ms_step, peaks):
        ach = B * 3 * d * 4 / (ms["cross_bwd"] * 1e-3) / 1e9
        step_gbs = bytes_step / (ms_step * 1e-3) / 1e9
        return {"bound": "hbm", "kernel": "cross_bwd_kernel (all L layers, one launch)", "achieved": ach, "peak": peaks["hbm_gbs"],
                "unit": "GB/s", "frac": ach / peaks["hbm_gbs"], "traffic": None, "algorithmic_bytes_per_launch": B * 3 * d * 4,
                "avg_launch_ms": ms["cross_bwd"], "step_algorithmic_GBps": step_gbs, "step_frac": step_gbs / peaks["hbm_gbs"],
                "step_bytes_per_sample": bytes_step // B,
                "note": "79 MB per step (more than the 50 MB L2); two kernel launches (fused lookup+cross forward, cross backward) + 2 memsets: launch/latency-bound, see DESIGN 4.3"}

    return {"step": step, "outputs": outputs, "marks": ["lookup+cross_fwd", "cross_bwd", "lookup_bwd"], "B": B, "roofline": roofline,
            "config": {"workload": "dcn_cfg2", "model": "DCN lookup + 3 cross layers", "B": B, "F": F, "D": D, "d": d, "L": L,
                       "rows_per_field": rows, "ids": "uniform int64"}, "dtype": "f32"}


def build_xdeepfm_cfg3(rows=1_000_000, B=8192):
    """Config 3: xDeepFM CIN [128,128], 30 fields x 16 (xDeepFM/xdeepfm.py:166-175), 3xTF32 on wgmma."""
    gen = torch.Generator(device="cuda").manual_seed(1234)
    F, D, H = 30, 16, 128
    table = _rn(gen, rows * F, D, std=D ** -0.5)
    off = torch.arange(F + 1, device="cuda") * rows
    ids = [torch.randint(0, rows, (B, F), device="cuda", generator=gen) for _ in range(4)]
    w1, w2 = _rn(gen, F * F, H, std=0.05), _rn(gen, H * F, H, std=0.05)
    gp = _rn(gen, B, 2 * H)
    k = [0]
    outputs = {}

    def step(ev=None):
        k[0] += 1
        _rec(ev, 0)
        x0, _ = ops.embed_fm2_fwd(table, off, ids[k[0] % 4], want_fm2=False)
        _rec(ev, 1)
        x1, p1 = ops.cin_fwd(x0, x0, w1, want_pooled=True)
        x2, p2 = ops.cin_fwd(x0, x1, w2, want_pooled=True)
        _rec(ev, 2)
        g2 = gp[:, H:].unsqueeze(-1).expand(B, H, D).contiguous()          # d(pooled)/d(out) broadcast over D
        dx0b, dx1, dw2 = ops.cin_bwd(x0, x1, w2, g2)
        g1 = dx1 + gp[:, :H].unsqueeze(-1)
        dx0a, dxk, dw1 = ops.cin_bwd(x0, x0, w1, g1.contiguous())
        _rec(ev, 3)
        values = dx0a + dxk + dx0b                                          # sum of the three paths into x0 = the IndexedSlices values
        _rec(ev, 4)
        outputs.update(x2=x2, pooled_1=p1, pooled_2=p2, d_filter_1=dw1, d_filter_2=dw2, d_x0=values)

    flops_fwd = 2.0 * B * D * (F * F * H + H * F * H)
    flops_step = 3.0 * flops_fwd                                          # backward = dX + dW = 2x forward

    def roofline(ms, ms_step, peaks):
        ach = flops_step / ((ms["cin_fwd"] + ms["cin_bwd"]) * 1e-3) / 1e12
        pk = peaks["bf16_tflops_sustained"]
        return {"bound": "tensor", "kernel": "cin_fwd_tc_kernel + cin_bwd_dx/dw_tc_kernel (wgmma kind tf32, 3xTF32)",
                "achieved": ach, "peak": pk, "unit": "TFLOP/s", "frac": ach / pk, "traffic": None,
                "algorithmic_flops_per_step": flops_step, "cin_fwd_ms": ms["cin_fwd"], "cin_bwd_ms": ms["cin_bwd"],
                "executed_over_algorithmic": 3.0, "tf32_rate_over_bf16": 0.5,
                "frac_of_3xtf32_ceiling": ach / (pk * 0.5 / 3.0),
                "note": "fp32-class accuracy costs 3 TF32 MMAs per product at half the bf16 rate: the ceiling of this "
                        "formulation is peak/6; peak = bf16_tflops_sustained (kernels timed inside a step)"}

    return {"step": step, "outputs": outputs, "marks": ["lookup_fwd", "cin_fwd", "cin_bwd", "lookup_bwd"], "B": B, "roofline": roofline,
            "config": {"workload": "xdeepfm_cfg3", "model": "xDeepFM lookup + CIN [128,128]", "B": B, "m": F, "D": D, "cin": [H, H],
                       "rows_per_field": rows, "ids": "uniform int64", "precision": "3xTF32 (fp32-class, <=1e-5)"}, "dtype": "f32 (3xTF32 MMA)"}


def build_din_cfg4(rows=1_000_000, B=4096):
    """Config 4: DIN attention over a 50-step behaviour sequence, H = 16 (DIN/din.py:216-218)."""
    gen = torch.Generator(device="cuda").manual_seed(1234)
    T, Hd = 50, 16
    tab = _rn(gen, rows, Hd, std=0.25)
    off = torch.tensor([0, rows], device="cuda")
    lens = torch.randint(0, T + 1, (B,), device="cuda", generator=gen)
    pad = (torch.arange(T, device="cuda")[None, :] >= lens[:, None]).reshape(-1)
    hists, tgts = [], []
    for _ in range(4):
        h = torch.randint(0, rows, (B * T,), device="cuda", generator=gen)
        h[pad] = -1                                                        # padding -> zero vectors
        hists.append(h.reshape(B, T).contiguous())
        tgts.append(torch.randint(0, rows, (B, 1), device="cuda", generator=gen))
    rng2 = torch.tensor([0, rows], device="cuda")
    ws = [_rn(gen, 4 * Hd, 64, std=0.2), _rn(gen, 64, std=0.1), _rn(gen, 64, 32, std=0.2), _rn(gen, 32, std=0.1),
          _rn(gen, 32, 1, std=0.3), _rn(gen, 1, std=0.1)]
    go = _rn(gen, B, Hd)
    k = [0]
    outputs = {}

    def step(ev=None):
        k[0] += 1
        _rec(ev, 0)
        k3 = ops.embed_seq_fwd(tab, hists[k[0] % 4], rng2)                # (B,T) history: one warp per sample (ctr_embed_seq_fwd)
        q, _ = ops.embed_fm2_fwd(tab, off, tgts[k[0] % 4], want_fm2=False)
        q2 = q.view(B, Hd)
        _rec(ev, 1)
        out, att = ops.din_attention_fwd(q2, k3, lens, *ws, want_weights=True)
        _rec(ev, 2)
        dq, dk, dws = ops.din_attention_bwd(q2, k3, lens, *ws, go, att_w=att)
        _rec(ev, 3)
        outputs.update(out=out, att_weights=att, d_query=dq, d_keys=dk, **{f"d_w{i}": t for i, t in enumerate(dws)})
        # lookup backward of a plain gather: the IndexedSlices values are dk / dq themselves (no kernel, no bytes)
        _rec(ev, 4)

    n_pos = int(lens.sum().item())                                         # positions that reach the MLP (t < keys_length)
    # executed FLOPs: layer 1 folded per sample (H*64 MACs per position instead of 4H*64) + layers 2, 3; backward ~ 2x + the
    # per-sample weight-gradient outer products
    fl_fwd_exec = 2.0 * n_pos * (Hd * 64 + 64 * 32 + 32) + 2.0 * B * (3 * Hd * 64)
    fl_bwd_exec = 2.0 * fl_fwd_exec + 2.0 * n_pos * (Hd * 64 + 64 * 32)
    fl_ref = B * T * 2.0 * (4 * Hd * 64 + 64 * 32 + 32)
    by_fwd = B * (T * Hd * 4 + 8 + 2 * Hd * 4)

    def roofline(ms, ms_step, peaks):
        ach = fl_bwd_exec / (ms["din_bwd"] * 1e-3) / 1e12
        return {"bound": "fp32-fma", "kernel": "din_attention_bwd_kernel", "achieved": ach, "peak": FP32_FMA_TFLOPS, "unit": "TFLOP/s",
                "frac": ach / FP32_FMA_TFLOPS, "traffic": None, "executed_flops_bwd": fl_bwd_exec, "executed_flops_fwd": fl_fwd_exec,
                "reference_counted_flops_fwd": fl_ref, "fwd_TFLOPs_executed": fl_fwd_exec / (ms["din_fwd"] * 1e-3) / 1e12,
                "fwd_GBps": by_fwd / (ms["din_fwd"] * 1e-3) / 1e9, "din_fwd_ms": ms["din_fwd"], "din_bwd_ms": ms["din_bwd"],
                "peak_source": "nominal: 132 SMs x 128 FMA/clk x 2 x 1.98 GHz (no measured fp32 peak in MEASURED_PEAKS.json)",
                "note": "FLOPs are the EXECUTED ones (folded layer 1, masked positions skipped), not the reference's count"}

    return {"step": step, "outputs": outputs, "marks": ["lookup_fwd", "din_fwd", "din_bwd", "lookup_bwd"], "B": B, "roofline": roofline,
            "config": {"workload": "din_cfg4", "model": "DIN lookup + attention", "B": B, "T": T, "H": Hd, "rows": rows,
                       "lengths": "uniform{0..50}", "ids": "uniform int64", "softmax": False}, "dtype": "f32"}


BUILDERS = {"dcn_cfg2": build_dcn_cfg2, "xdeepfm_cfg3": build_xdeepfm_cfg3, "din_cfg4": build_din_cfg4}


def graphed(fn):
    """The same C-ABI calls captured once into a CUDA graph (they only enqueue work on the given stream and never allocate or
    synchronise, so they are capturable as they are); a step is then ONE graph launch."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    return graph.replay
