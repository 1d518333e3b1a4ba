#!/usr/bin/env python
"""Per-layer timings of the non-headline BASELINE configs (2: DCN cross, 3: xDeepFM CIN, 4: DIN attention) and FiBiNET.

Each kernel is timed alone with CUDA events; an L2 flush (a 256 MB write) runs between timed iterations because these
working sets are flushed from the 50 MB L2.  Prints one JSON line per measurement.

    python tools/bench_layers.py [--iters 20] [--only cin,dcn,din,fibinet]     (also: pairwise, bst, adam, pnn, dien, dien_aux, deepcrossing, mmoe, ple, wide, autoint, flen)
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from recalgorithm_b200 import ops  # noqa: E402


def peaks():
    """HBM GB/s and bf16 TFLOP/s: MEASURED_PEAKS.json when present, else the H100 SXM data sheet (bench.measured_peaks)."""
    from bench import measured_peaks
    d = measured_peaks()
    return d["hbm_gbs"], d["bf16_tflops"], d["source"]


def timeit(fn, iters, flush):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        flush.zero_()                                   # 256 MB write: evicts the 50 MB L2
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times), min(times)


def pnn_rows(iters, flush, rn, hbm):
    """IPNN / OPNN forward and backward at the reference batch (1024) and at 65 536, next to plain torch running the same
    feature-row form (fp32 matmul, TF32 off).  Tensor figures are executed 3xTF32 FLOP/s (3 passes x 2 x B x WP x N, WP = the
    feature width 101 padded to 128) against the H100 SXM data-sheet dense TF32 rate (495 TFLOP/s), labelled as such."""
    tf32_peak = 495.0
    F, K, N = 8, 8, 1024
    WP = 128
    iu_f, iu_k = torch.triu_indices(F, F, device="cuda"), torch.triu_indices(K, K, device="cuda")

    def torch_form(e, wlin, wprod, bias, method):
        B = e.shape[0]
        if method == 0:
            q = torch.einsum("bik,bjk->bij", e, e)[:, iu_f[0], iu_f[1]]
            c = torch.where(iu_f[0] == iu_f[1], 1.0, 2.0)
            wq = c[:, None] * (wprod[:, iu_f[0]] * wprod[:, iu_f[1]]).t()
        else:
            s = e.sum(1)
            q = s[:, iu_k[0]] * s[:, iu_k[1]]
            c = torch.where(iu_k[0] == iu_k[1], 1.0, 2.0)
            wq = c[:, None] * wprod[:, iu_k[0], iu_k[1]].t()
        xt = torch.cat([e.reshape(B, -1), q, torch.ones((B, 1), device=e.device)], 1)
        return torch.relu(xt @ torch.cat([wlin, wq, bias[None, :]], 0))

    prev_tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for method, tag in ((0, "ipnn"), (1, "opnn")):
            wlin = rn(F * K, N, std=0.05)
            wprod = rn(N, F, std=0.1) if method == 0 else rn(N, K, K, std=0.1)
            bias = rn(N, std=0.05)
            for B in (1024, 65536):
                e, g = rn(B, F, K, std=K ** -0.5), rn(B, N)
                cfg = {"method": tag.upper(), "B": B, "F": F, "K": K, "N": N}
                out = ops.pnn_fwd(e, wlin, wprod, bias, method)
                flops_fwd = 3 * 2.0 * B * WP * N
                m, bst = timeit(lambda: ops.pnn_fwd(e, wlin, wprod, bias, method), iters, flush)
                line = {"kernel": f"pnn_fwd_{tag}", "config": cfg, "ms_median": m, "ms_best": bst, "l2": "flushed between iterations",
                        "algorithmic_GBps": B * (F * K + N) * 4 / (m * 1e-3) / 1e9, "executed_3xTF32_TFLOPs": flops_fwd / (m * 1e-3) / 1e12,
                        "note": "bytes: read e, write out; FLOPs vs the H100 SXM data-sheet dense TF32 rate (495 TFLOP/s)"}
                line["frac_of_hbm_peak"] = line["algorithmic_GBps"] / hbm
                line["frac_of_tf32_datasheet"] = line["executed_3xTF32_TFLOPs"] / tf32_peak
                print(json.dumps(line), flush=True)
                m, bst = timeit(lambda: ops.pnn_bwd(e, wlin, wprod, out, g, method), iters, flush)
                line = {"kernel": f"pnn_bwd_{tag}", "config": cfg, "ms_median": m, "ms_best": bst, "l2": "flushed between iterations",
                        "algorithmic_GBps": B * (2 * F * K + 4 * N) * 4 / (m * 1e-3) / 1e9,
                        "executed_3xTF32_TFLOPs": 2 * flops_fwd / (m * 1e-3) / 1e12,
                        "note": "bytes: e read, d_e written, g_out and out read once by each of the two GEMM passes"}
                line["frac_of_hbm_peak"] = line["algorithmic_GBps"] / hbm
                line["frac_of_tf32_datasheet"] = line["executed_3xTF32_TFLOPs"] / tf32_peak
                print(json.dumps(line), flush=True)
                ref = torch_form(e, wlin, wprod, bias, method)
                diff = float((ref - out).abs().max() / ref.abs().max())
                m, bst = timeit(lambda: torch_form(e, wlin, wprod, bias, method), iters, flush)
                print(json.dumps({"kernel": f"torch_fp32_fwd_{tag}", "config": cfg, "ms_median": m, "ms_best": bst,
                                  "max_rel_diff_vs_kernel": diff, "within_1e-5": diff <= 1e-5,
                                  "note": "same feature-row form in torch, fp32 matmul, TF32 disabled"}), flush=True)
                ps = [t.clone().requires_grad_() for t in (e, wlin, wprod, bias)]
                ref_out = torch_form(*ps, method)

                def torch_bwd():
                    return torch.autograd.grad(ref_out, ps, g, retain_graph=True)
                grads = torch_bwd()
                kg = ops.pnn_bwd(e, wlin, wprod, out, g, method)
                gdiff = max(float((a - b).abs().max() / b.abs().max()) for a, b in zip(kg, grads))
                m, bst = timeit(torch_bwd, iters, flush)
                print(json.dumps({"kernel": f"torch_fp32_bwd_{tag}", "config": cfg, "ms_median": m, "ms_best": bst,
                                  "max_rel_diff_vs_kernel": gdiff, "within_1e-5": gdiff <= 1e-5,
                                  "note": "autograd of the same torch form (backward only), fp32, TF32 disabled"}), flush=True)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev_tf32


def card():
    """Name and power limit of the GPU the rows are measured on, read in the same run."""
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def dien_rows(iters, flush, hbm):
    """DIEN seq_encoder (ctr_dien_fwd / ctr_dien_bwd) at T = 50, na = 16, nh = 8, lengths uniform in {0..50}, B = 4096 and
    65 536, both cells, next to plain torch running the reference form (a Python loop over T, fp32, TF32 off, autograd
    backward).  Floors: HBM bytes over 3.35 TB/s and FLOPs over the 67 TFLOP/s FP32 data-sheet rate of the H100 SXM (700 W).
    The kernels are bound by the dependent chain of 2*T cell steps per sample, so each row also reports time / (2*T)."""
    T, na, nh = 50, 16, 8
    fp32_peak = 67.0
    print(json.dumps({"dien_card": card()}), flush=True)

    def torch_form(seq, L, tgt, params, cell):
        gk, gb, ck, cb, W, egk, egb, eck, ecb = params

        def gru(x, h, gk, gb, ck, cb):
            v = torch.sigmoid(torch.cat([x, h], 1) @ gk + gb)
            r, u = v[:, :nh], v[:, nh:]
            return u, torch.tanh(torch.cat([x, r * h], 1) @ ck + cb)
        h = seq.new_zeros(seq.shape[0], nh)
        hs = []
        for t in range(T):
            u, c = gru(seq[:, t], h, gk, gb, ck, cb)
            h = u * h + (1 - u) * c
            hs.append(h)
        H = torch.stack(hs, 1)
        mask = torch.arange(T, device=seq.device)[None, :] < L[:, None]
        att = torch.softmax(torch.where(mask, (H @ (tgt @ W.t())[:, :, None])[..., 0], -4294967296.0), dim=1)
        s = seq.new_zeros(seq.shape[0], nh)
        for t in range(T):
            a = att[:, t, None]
            u, c = gru(H[:, t], s, egk, egb, eck, ecb)
            sn = ((1 - a) * u) * s + (1 - (1 - a) * u) * c if cell == 1 else (1 - a) * s + a * c
            s = torch.where(mask[:, t, None], sn, s)
        return s, att

    prev_tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    gen = torch.Generator(device="cuda").manual_seed(50)
    try:
        for B in (4096, 65536):
            L = torch.randint(0, T + 1, (B,), device="cuda", generator=gen)
            seq = torch.randn((B, T, na), device="cuda", generator=gen) * 0.7
            seq[torch.arange(T, device="cuda")[None, :] >= L[:, None]] = 0
            tgt = torch.randn((B, na), device="cuda", generator=gen) * 0.7
            g = torch.randn((B, nh), device="cuda", generator=gen)
            params = [(torch.rand(s, device="cuda", generator=gen) * 2 - 1) * (0.5 if len(s) == 1 else (6.0 / sum(s)) ** 0.5)
                      for s in ops.dien_param_shapes(na, nh)]
            packed = ops.dien_pack_params(params, na, nh)
            steps = int(L.sum())                                    # processed positions (each runs both cells)
            flop_pos = 2 * (3 * nh * (na + nh) + 3 * nh * 2 * nh) + 2 * nh + 30 * nh   # projections + score + gates
            fwd_flops, bwd_flops = steps * flop_pos, 3 * steps * flop_pos            # backward: recompute + two transposes
            fwd_bytes = 4 * (steps * (na + 2 * nh) + B * (T + na + nh) + B * 2)
            bwd_bytes = 4 * (B * T * na + steps * (na + 2 * nh + 1 + 2 * (nh + 1)) + B * (T + 2 * na + nh) + B * 2)
            for cell, tag in ((0, "agru"), (1, "augru")):
                cfg = {"cell": tag.upper(), "B": B, "T": T, "na": na, "nh": nh, "lengths": "uniform 0..50", "mean_len": steps / B}
                fs, att, ws = ops.dien_fwd(seq, L, tgt, packed, nh, cell)
                for kind, fn, flops, nbytes in (
                        ("fwd", lambda: ops.dien_fwd(seq, L, tgt, packed, nh, cell), fwd_flops, fwd_bytes),
                        ("bwd", lambda: ops.dien_bwd(seq, L, tgt, packed, g, nh, cell, ws), bwd_flops, bwd_bytes)):
                    m, bst = timeit(fn, iters, flush)
                    print(json.dumps({"kernel": f"dien_{kind}_{tag}", "config": cfg, "ms_median": m, "ms_best": bst,
                                      "l2": "flushed between iterations", "us_per_dependent_step": m * 1e3 / (2 * T),
                                      "hbm_floor_ms": nbytes / (hbm * 1e9) * 1e3, "fp32_floor_ms": flops / (fp32_peak * 1e12) * 1e3,
                                      "algorithmic_bytes": nbytes, "flops": flops,
                                      "note": "floors: algorithmic bytes / measured-or-datasheet HBM rate, FLOPs / 67 TFLOP/s FP32"}),
                          flush=True)
                ps = [p.clone().requires_grad_() for p in params]
                xs = seq.clone().requires_grad_()
                ts = tgt.clone().requires_grad_()
                ref_s, ref_att = torch_form(xs, L, ts, ps, cell)
                diff = max(float((ref_s.detach() - fs).abs().max() / ref_s.detach().abs().max()),
                           float((ref_att.detach() - att).abs().max() / ref_att.detach().abs().max()))
                m, bst = timeit(lambda: torch_form(seq, L, tgt, params, cell), max(3, iters // 4), flush)
                print(json.dumps({"kernel": f"torch_fp32_fwd_{tag}", "config": cfg, "ms_median": m, "ms_best": bst,
                                  "max_rel_diff_vs_kernel": diff, "within_1e-5": diff <= 1e-5,
                                  "note": "reference form in torch (Python loop over T), fp32, TF32 disabled"}), flush=True)

                def torch_bwd():
                    return torch.autograd.grad(ref_s, [xs, ts] + ps, g, retain_graph=True)
                grads = torch_bwd()
                d_seq, d_tgt, d_p = ops.dien_bwd(seq, L, tgt, packed, g, nh, cell, ws)
                kg = [d_seq, d_tgt] + list(ops.dien_unpack_params(d_p, na, nh))
                gdiff = max(float((a - b).abs().max() / max(float(b.abs().max()), 1e-30)) for a, b in zip(kg, grads))
                m, bst = timeit(torch_bwd, max(3, iters // 4), flush)
                print(json.dumps({"kernel": f"torch_fp32_bwd_{tag}", "config": cfg, "ms_median": m, "ms_best": bst,
                                  "max_rel_diff_vs_kernel": gdiff, "within_1e-5": gdiff <= 1e-5,
                                  "note": "autograd of the same torch form (backward only), fp32, TF32 disabled"}), flush=True)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev_tf32


def dien_aux_rows(iters, flush, hbm):
    """DIEN auxiliary loss at DIEN's reference shape (T = 50, na = 16, nh = 8, lengths uniform in {0..50}) with T_neg = 3, B =
    4096 and 65 536, both cells: ctr_dien_aux_fwd alone, ctr_dien_bwd_aux next to the plain ctr_dien_bwd, and the whole step
    (forward, aux forward, backward) with and without the loss.  HBM floors from shapes: the aux forward reads, per counted
    position (t < len - 1), the positive row, T_neg negative rows and h_t; the aux backward reads the same, writes every
    negative-row gradient (zeros included), the positive-row term of d_seq_input (all B*T rows) and dL/dh_t, and
    ctr_dien_bwd_aux reads that d_seq_input and dL/dh back."""
    import subprocess
    T, na, nh, T_neg = 50, 16, 8, 3
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    print(json.dumps({"dien_aux_card": {"device": torch.cuda.get_device_name(0),
                                        "name, power.limit, clocks.sm, clocks.max.sm": q.stdout.strip() or q.stderr.strip()}}),
          flush=True)
    gen = torch.Generator(device="cuda").manual_seed(50)
    for B in (4096, 65536):
        L = torch.randint(0, T + 1, (B,), device="cuda", generator=gen)
        seq = torch.randn((B, T, na), device="cuda", generator=gen) * 0.7
        seq[torch.arange(T, device="cuda")[None, :] >= L[:, None]] = 0
        neg = torch.randn((B, (T - 1) * T_neg, na), device="cuda", generator=gen) * 0.7
        tgt = torch.randn((B, na), device="cuda", generator=gen) * 0.7
        g = torch.randn((B, nh), device="cuda", generator=gen)
        g_aux = torch.ones((), device="cuda")
        params = [(torch.rand(s, device="cuda", generator=gen) * 2 - 1) * (0.5 if len(s) == 1 else (6.0 / sum(s)) ** 0.5)
                  for s in ops.dien_param_shapes(na, nh)]
        w = (torch.rand((na, nh), device="cuda", generator=gen) * 2 - 1) * (6.0 / (na + nh)) ** 0.5
        packed = ops.dien_pack_params(params, na, nh)
        P = int((L - 1).clamp(min=0).sum())                         # counted positions
        fwd_bytes = 4 * P * (na * (1 + T_neg) + nh) + 8 * B + 8 * B + 8 * B
        bwd_bytes = 4 * (P * (na * (1 + T_neg) + 2 * nh) + B * (T - 1) * T_neg * na + B * T * na) + 8 * B
        extra_bytes = 4 * (B * T * na + P * nh)                     # ctr_dien_bwd_aux re-reads the seeds it adds to
        for cell, tag in ((0, "agru"), (1, "augru")):
            cfg = {"cell": tag.upper(), "B": B, "T": T, "na": na, "nh": nh, "T_neg": T_neg, "lengths": "uniform 0..50",
                   "counted_positions": P}
            _, _, _, ws = ops.dien_fwd_aux(seq, L, tgt, neg, packed, w, nh, cell, T_neg)
            rows = (("dien_aux_fwd", lambda: ops.dien_aux_fwd(seq, neg, L, w, nh, T_neg, ws), fwd_bytes),
                    ("dien_bwd", lambda: ops.dien_bwd(seq, L, tgt, packed, g, nh, cell, ws), None),
                    ("dien_bwd_aux", lambda: ops.dien_bwd_aux(seq, L, tgt, neg, packed, w, g, g_aux, nh, cell, T_neg, ws),
                     bwd_bytes + extra_bytes),
                    ("step_plain", lambda: ops.dien_bwd(seq, L, tgt, packed, g, nh, cell,
                                                        ops.dien_fwd(seq, L, tgt, packed, nh, cell)[2]), None),
                    ("step_aux", lambda: ops.dien_bwd_aux(seq, L, tgt, neg, packed, w, g, g_aux, nh, cell, T_neg,
                                                          ops.dien_fwd_aux(seq, L, tgt, neg, packed, w, nh, cell, T_neg)[3]),
                     None))
            ms = {}
            for name, fn, nbytes in rows:
                m, bst = timeit(fn, iters, flush)
                ms[name] = m
                line = {"kernel": f"{name}_{tag}", "config": cfg, "ms_median": m, "ms_best": bst, "iters": iters,
                        "l2": "flushed between iterations"}
                if nbytes is not None:
                    line.update(hbm_floor_ms=nbytes / (hbm * 1e9) * 1e3, algorithmic_bytes=nbytes)
                print(json.dumps(line), flush=True)
            print(json.dumps({"kernel": f"dien_aux_overhead_{tag}", "config": cfg,
                              "bwd_aux_over_bwd": ms["dien_bwd_aux"] / ms["dien_bwd"] - 1,
                              "step_aux_over_step_plain": ms["step_aux"] / ms["step_plain"] - 1}), flush=True)


def deepcrossing_rows(iters, flush, rn):
    """DeepCrossing residual unit (ctr_residual_unit_fwd / _bwd) at the reference width d = 82, H = 128 and 256, B = 1024 (the
    reference batch) and 65 536, next to plain torch running the same unit (fp32 matmul, TF32 disabled, autograd backward).
    Floors from data-sheet rates of the H100 SXM (700 W), not measured: FLOPs over the 67 TFLOP/s FP32 rate, the executed
    3xTF32 FLOPs (3 passes over DP = 96 inputs, the kernels' padded width) over the 495 TFLOP/s TF32 rate, and x + out
    (forward) or x, out, g, d_x (backward) over 3.35 TB/s of HBM."""
    d, DP = 82, 96
    print(json.dumps({"deepcrossing_card": card()}), flush=True)

    def torch_form(x, w0, b0, w1, b1):
        return torch.relu(x + torch.relu(x @ w0 + b0) @ w1 + b1)

    prev_tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for H in (128, 256):
            lim = (6.0 / (d + H)) ** 0.5
            w0, w1 = (torch.rand(d, H, device="cuda") * 2 - 1) * lim, (torch.rand(H, d, device="cuda") * 2 - 1) * lim
            b0, b1 = rn(H, std=0.1), rn(d, std=0.1)
            for B in (1024, 65536):
                x, g = rn(B, d, std=0.7), rn(B, d)
                cfg = {"B": B, "d": d, "H": H}
                flops = {"fwd": 4.0 * B * d * H, "bwd": 10.0 * B * d * H}       # bwd: gh, dx, dW1, dW0 + the recomputed a
                tc = {"fwd": 3 * 4.0 * B * DP * H, "bwd": 3 * 10.0 * B * DP * H}
                hbm = {"fwd": 2 * B * d * 4, "bwd": 4 * B * d * 4}
                out = ops.residual_unit_fwd(x, w0, b0, w1, b1)
                grads = ops.residual_unit_bwd(x, w0, b0, w1, b1, out, g)
                ps = [t.clone().requires_grad_() for t in (x, w0, b0, w1, b1)]
                ref_out = torch_form(*ps)
                ref_grads = torch.autograd.grad(ref_out, ps, g, retain_graph=True)
                diff = {"fwd": float((ref_out.detach() - out).abs().max() / ref_out.detach().abs().max()),
                        "bwd": max(float((a - b).abs().max() / b.abs().max()) for a, b in zip(grads, ref_grads))}
                runs = {"fwd": (lambda: ops.residual_unit_fwd(x, w0, b0, w1, b1),
                                lambda: torch_form(x, w0, b0, w1, b1)),
                        "bwd": (lambda: ops.residual_unit_bwd(x, w0, b0, w1, b1, out, g),
                                lambda: torch.autograd.grad(ref_out, ps, g, retain_graph=True))}
                for way in ("fwd", "bwd"):
                    m, bst = timeit(runs[way][0], iters, flush)
                    tm, tbst = timeit(runs[way][1], iters, flush)
                    print(json.dumps({
                        "kernel": f"residual_unit_{way}", "config": cfg, "ms_median": m, "ms_best": bst,
                        "torch_fp32_ms_median": tm, "torch_fp32_ms_best": tbst, "speedup_vs_torch": tm / m,
                        "max_norm_rel_diff_vs_torch": diff[way], "l2": "flushed between iterations",
                        "floor_fp32_us": flops[way] / 67e12 * 1e6, "floor_3xtf32_us": tc[way] / 495e12 * 1e6,
                        "floor_hbm_us": hbm[way] / 3.35e12 * 1e6,
                        "note": "floors are data-sheet rates (H100 SXM, 700 W), not measured; torch: same unit, fp32, TF32 off"}),
                        flush=True)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev_tf32



def mmoe_rows(iters, flush, rn):
    """MMoE expert-gate layer (ctr_mmoe_fwd / _bwd) at the reference shape d = 82, E = 3, H = 512, T = 3, B = 1024 and 65 536,
    next to plain torch running the same block (fp32 einsum / softmax, TF32 disabled, autograd backward).  Floors from
    data-sheet rates of the H100 SXM (700 W), not measured: FLOPs over the 67 TFLOP/s FP32 rate, the executed 3xTF32 FLOPs
    (3 passes over DP = 96 inputs and R = E HP + 32 = 1568 units, plus the backward's hidden GEMMs and dW) over the
    495 TFLOP/s TF32 rate, and x + towers + gates (forward) or x, gates, g, d_x and the dz | dlogit round trip (backward)
    over 3.35 TB/s of HBM."""
    d, E, H, T, DP = 82, 3, 512, 3, 96
    R = E * H + 32
    print(json.dumps({"mmoe_card": card()}), flush=True)

    def torch_form(x, we, be, wg):
        h = torch.relu(torch.einsum("bd,edh->ebh", x, we) + be[:, None, :])
        p = torch.softmax(torch.einsum("bd,tde->tbe", x, wg), dim=-1)
        return torch.einsum("tbe,ebh->tbh", p, h), p

    prev_tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        lim_e, lim_g = (6.0 / (d + H)) ** 0.5, (6.0 / (d + E)) ** 0.5
        we = (torch.rand(E, d, H, device="cuda") * 2 - 1) * lim_e
        be = rn(E, H, std=0.1)
        wg = (torch.rand(T, d, E, device="cuda") * 2 - 1) * lim_g
        for B in (1024, 65536):
            x, g = rn(B, d, std=0.7), rn(T, B, H)
            cfg = {"B": B, "d": d, "E": E, "H": H, "T": T}
            fl_fwd = 2.0 * B * d * (E * H + T * E) + 2.0 * B * T * E * H
            flops = {"fwd": fl_fwd, "bwd": 3 * fl_fwd}
            tc = {"fwd": 3 * 2.0 * B * DP * R, "bwd": 3 * 2.0 * B * DP * (3 * R - 32)}   # dx: rows + hidden GEMMs; dW
            hbm = {"fwd": B * (d + T * H + T * E) * 4, "bwd": B * (2 * d + T * E + T * H + 2 * R) * 4}
            towers, gates = ops.mmoe_fwd(x, we, be, wg)
            grads = ops.mmoe_bwd(x, we, be, wg, gates, g)
            ps = [t.clone().requires_grad_() for t in (x, we, be, wg)]
            ref_towers, _ = torch_form(*ps)
            ref_grads = torch.autograd.grad(ref_towers, ps, g, retain_graph=True)
            diff = {"fwd": float((ref_towers.detach() - towers).abs().max() / ref_towers.detach().abs().max()),
                    "bwd": max(float((a - b).abs().max() / b.abs().max()) for a, b in zip(grads, ref_grads))}
            runs = {"fwd": (lambda: ops.mmoe_fwd(x, we, be, wg), lambda: torch_form(x, we, be, wg)),
                    "bwd": (lambda: ops.mmoe_bwd(x, we, be, wg, gates, g),
                            lambda: torch.autograd.grad(ref_towers, ps, g, retain_graph=True))}
            for way in ("fwd", "bwd"):
                m, bst = timeit(runs[way][0], iters, flush)
                tm, tbst = timeit(runs[way][1], iters, flush)
                print(json.dumps({
                    "kernel": f"mmoe_{way}", "config": cfg, "ms_median": m, "ms_best": bst,
                    "torch_fp32_ms_median": tm, "torch_fp32_ms_best": tbst, "speedup_vs_torch": tm / m,
                    "max_norm_rel_diff_vs_torch": diff[way], "l2": "flushed between iterations",
                    "floor_fp32_us": flops[way] / 67e12 * 1e6, "floor_3xtf32_us": tc[way] / 495e12 * 1e6,
                    "floor_hbm_us": hbm[way] / 3.35e12 * 1e6,
                    "note": "floors are data-sheet rates (H100 SXM, 700 W), not measured; torch: same block, fp32, TF32 off"}),
                    flush=True)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev_tf32


def ple_rows(iters, flush, rn):
    """PLE expert-gate blocks (ctr_ple_fwd / _bwd) at the default result.md row, n = 5,5,5 and S = 10 (E = 25), H = 256:
    the extraction network at the input width d = 82 and the final layer at d = H = 256, B = 1024 and 65 536, next to plain
    torch running the same block (fp32 matmul / softmax, TF32 disabled, autograd backward).  The floor is the block's FP32
    FLOPs (expert and gate GEMMs plus the gated sums; the backward counted as 3x) over the data-sheet 67 TFLOP/s of the
    H100 SXM at 700 W, not measured."""
    n, S, H = (5, 5, 5), 10, 256
    E, es = sum(n) + S, sum(n)
    print(json.dumps({"ple_card": card()}), flush=True)

    def gate_lists(ext):
        e0 = [sum(n[:t]) for t in range(len(n))]
        lists = [list(range(e0[t], e0[t] + n[t])) + list(range(es, E)) for t in range(len(n))]
        return lists + ([list(range(E))] if ext else [])

    def torch_form(x, we, be, wg, ext):
        h = torch.relu(x @ we + be[:, None, :])
        z = x @ wg
        outs, c = [], 0
        for experts in gate_lists(ext):
            p = torch.softmax(z[:, c:c + len(experts)], dim=-1)
            outs.append(torch.einsum("bj,jbh->bh", p, h[experts]))
            c += len(experts)
        return sum(outs) if ext else torch.stack(outs)

    prev_tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for d, ext in ((82, True), (256, False)):
            GC = sum(len(g) for g in gate_lists(ext))
            we = (torch.rand(E, d, H, device="cuda") * 2 - 1) * (6.0 / (d + H)) ** 0.5
            be = rn(E, H, std=0.1)
            wg = (torch.rand(d, GC, device="cuda") * 2 - 1) * (6.0 / (d + GC)) ** 0.5
            for B in (1024, 65536):
                x = rn(B, d, std=0.7)
                g = rn(B, H) if ext else rn(len(n), B, H)
                cfg = {"block": "extraction_network" if ext else "final_layer", "B": B, "d": d, "n": list(n), "S": S, "H": H}
                fl_fwd = 2.0 * B * (d * (E * H + GC) + GC * H)
                flops = {"fwd": fl_fwd, "bwd": 3 * fl_fwd}
                out, gates = ops.ple_fwd(x, we, be, wg, n, S, ext)
                grads = ops.ple_bwd(x, we, be, wg, gates, g, n, S, ext)
                ps = [t.clone().requires_grad_() for t in (x, we, be, wg)]
                ref_out = torch_form(*ps, ext)
                ref_grads = torch.autograd.grad(ref_out, ps, g, retain_graph=True)
                diff = {"fwd": float((ref_out.detach() - out).abs().max() / ref_out.detach().abs().max()),
                        "bwd": max(float((a - b).abs().max() / b.abs().max()) for a, b in zip(grads, ref_grads))}
                runs = {"fwd": (lambda: ops.ple_fwd(x, we, be, wg, n, S, ext), lambda: torch_form(x, we, be, wg, ext)),
                        "bwd": (lambda: ops.ple_bwd(x, we, be, wg, gates, g, n, S, ext),
                                lambda: torch.autograd.grad(ref_out, ps, g, retain_graph=True))}
                for way in ("fwd", "bwd"):
                    m, bst = timeit(runs[way][0], iters, flush)
                    tm, tbst = timeit(runs[way][1], iters, flush)
                    print(json.dumps({
                        "kernel": f"ple_{way}", "config": cfg, "ms_median": m, "ms_best": bst,
                        "torch_fp32_ms_median": tm, "torch_fp32_ms_best": tbst, "speedup_vs_torch": tm / m,
                        "max_norm_rel_diff_vs_torch": diff[way], "l2": "flushed between iterations",
                        "floor_fp32_us": flops[way] / 67e12 * 1e6,
                        "note": "floor: data-sheet FP32 rate (H100 SXM, 700 W), not measured; torch: same block, fp32, TF32 off"}),
                        flush=True)
                del out, gates, grads, ps, ref_out, ref_grads
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev_tf32


def wide_rows(iters, flush):
    """Wide & Deep wide part: ctr_crossed_indicator_fwd / _bwd on crossed_column([userid, manual_tag_list]) and ctr_ftrl_apply on
    its kernel, at B = 1024 (the reference batch) and 65 536, num_buckets = 100 000 (the reference) and 10^7.  One userid
    per sample (uniform over 200 000) and 1-12 tags per sample (uniform; the tag count is an assumption, the reference's data is
    not here) over 350 tag ids.  Plain torch runs the same computation on the same GPU: the hash in int64 tensor ops, the
    gather-sum and the scatter with index_add_, FTRL as elementwise ops.  Bytes are what the algorithm moves (ids, offsets,
    one 4-byte kernel entry per cross, the logit; the backward adds the gradient zeroing; FTRL reads 4 and writes 3 arrays)
    over kernel time: the cross kernels are gather / scatter bound, FTRL is HBM bound."""
    print(json.dumps({"wide_card": card()}), flush=True)
    K64 = 0xc6a4a7935bd1e995 - (1 << 64)                       # kMul as a signed int64
    low17 = (1 << 17) - 1

    def mix(x):
        return x ^ ((x >> 47) & low17)                          # logical shift on int64

    def cat64(a, b):
        r = a ^ K64
        r = r ^ (mix(b * K64) * K64)
        r = r * K64
        return mix(mix(r) * K64)

    def umod(h, n):                                             # uint64 h % n, n < 2^31, in int64 arithmetic
        hi, lo = (h >> 32) & 0xFFFFFFFF, h & 0xFFFFFFFF
        return ((hi % n) * ((1 << 32) % n) + lo) % n

    def torch_ids(uid, tags, sample_of_tag, nb):
        return umod(cat64(cat64(torch.full_like(tags, ops.CROSS_HASH_KEY), uid[sample_of_tag]), tags), nb)

    def torch_fwd(uid, tags, sample_of_tag, kernel, bias, B, nb):
        ids = torch_ids(uid, tags, sample_of_tag, nb)
        return torch.zeros(B, device="cuda").index_add_(0, sample_of_tag, kernel[ids]) + bias

    def torch_bwd(uid, tags, sample_of_tag, g, nb):
        ids = torch_ids(uid, tags, sample_of_tag, nb)
        return torch.zeros(nb, device="cuda").index_add_(0, ids, g[sample_of_tag]), g.sum()

    def torch_ftrl(var, acc, lin, g, lr):
        na = acc + g * g
        lin += g - (na.sqrt() - acc.sqrt()) / lr * var
        var.copy_(torch.where(lin.abs() > 0, -lin / (na.sqrt() / lr), torch.zeros_like(var)))
        acc.copy_(na)

    gen = torch.Generator(device="cuda").manual_seed(7)
    for B in (1024, 65536):
        n_tags = torch.randint(1, 13, (B,), device="cuda", generator=gen)
        uid = torch.randint(0, 200000, (B,), device="cuda", generator=gen)
        tags = torch.randint(0, 350, (int(n_tags.sum()),), device="cuda", generator=gen)
        values = torch.cat([uid, tags])
        offsets = torch.stack([torch.arange(B + 1, device="cuda"),
                               B + torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), n_tags.cumsum(0)])]).contiguous()
        sample_of_tag = torch.repeat_interleave(torch.arange(B, device="cuda"), n_tags)
        nnz, crosses = values.numel(), tags.numel()
        for nb in (100000, 10 ** 7):
            kernel = (torch.rand(nb, device="cuda", generator=gen) * 2 - 1) * (6.0 / (nb + 1)) ** 0.5
            bias = torch.full((1,), 0.25, device="cuda")
            g = torch.randn(B, device="cuda", generator=gen)
            cfg = {"B": B, "num_buckets": nb, "K": 2, "crosses": crosses, "tags_per_sample": "uniform 1..12 (assumed)"}
            out = ops.crossed_indicator_fwd(values, offsets, nb, kernel, bias)
            dk, db = ops.crossed_indicator_bwd(values, offsets, nb, g)
            ref_out = torch_fwd(uid, tags, sample_of_tag, kernel, bias, B, nb)
            ref_dk, ref_db = torch_bwd(uid, tags, sample_of_tag, g, nb)
            diff = {"fwd": float((out.reshape(-1) - ref_out).abs().max()), "bwd": float((dk - ref_dk).abs().max())}
            io = nnz * 8 + 2 * (B + 1) * 8
            bytes_ = {"fwd": io + crosses * 4 + B * 4, "bwd": io + B * 4 + nb * 4 + crosses * 4}
            runs = {"fwd": (lambda: ops.crossed_indicator_fwd(values, offsets, nb, kernel, bias),
                            lambda: torch_fwd(uid, tags, sample_of_tag, kernel, bias, B, nb)),
                    "bwd": (lambda: ops.crossed_indicator_bwd(values, offsets, nb, g),
                            lambda: torch_bwd(uid, tags, sample_of_tag, g, nb))}
            for way in ("fwd", "bwd"):
                m, bst = timeit(runs[way][0], iters, flush)
                tm, tbst = timeit(runs[way][1], iters, flush)
                print(json.dumps({
                    "kernel": f"crossed_indicator_{way}", "config": cfg, "ms_median": m, "ms_best": bst,
                    "torch_ms_median": tm, "torch_ms_best": tbst, "speedup_vs_torch": tm / m, "max_abs_diff_vs_torch": diff[way],
                    "algorithmic_GBps": bytes_[way] / (m * 1e-3) / 1e9, "bound": "gather" if way == "fwd" else "scatter (atomics)",
                    "l2": "flushed between iterations", "note": "bytes are algorithmic (4 B per gathered / scattered kernel entry)"}),
                    flush=True)
    for n in (100000, 10 ** 7):
        var = torch.randn(n, device="cuda", generator=gen) * 0.01
        acc, lin = torch.full((n,), 0.1, device="cuda"), torch.zeros(n, device="cuda")
        grad = torch.randn(n, device="cuda", generator=gen)
        tv, ta, tl = var.clone(), acc.clone(), lin.clone()
        ops.ftrl_apply(var, acc, lin, grad, 0.005)
        torch_ftrl(tv, ta, tl, grad, 0.005)
        diff = float((var - tv).abs().max() / tv.abs().max())
        m, bst = timeit(lambda: ops.ftrl_apply(var, acc, lin, grad, 0.005), iters, flush)
        tm, tbst = timeit(lambda: torch_ftrl(tv, ta, tl, grad, 0.005), iters, flush)
        print(json.dumps({
            "kernel": "ftrl_apply", "config": {"n": n, "lr": 0.005, "lr_power": -0.5}, "ms_median": m, "ms_best": bst,
            "torch_ms_median": tm, "torch_ms_best": tbst, "speedup_vs_torch": tm / m, "max_norm_rel_diff_vs_torch": diff,
            "algorithmic_GBps": 28 * n / (m * 1e-3) / 1e9, "frac_of_hbm_3_35TBps": 28 * n / (m * 1e-3) / 3.35e12, "bound": "HBM",
            "l2": "flushed between iterations", "note": "28 B per element (read var, accum, linear, grad; write var, accum, linear)"}),
            flush=True)


def autoint_rows(iters, flush, rn):
    """AutoInt interacting layer (ctr_autoint_fwd / _bwd) at the paper's setting F = 40, H = 2, dk = 32, for the first layer
    (d = 16) and a later one (d = 64), B = 1024 and 65 536; plus DeepCTR's default head width dk = 8 at B = 65 536 (heads
    are padded to 32 columns, so that row spends 4x the padded work).  Each row is timed next to plain torch running the
    same layer: fp32 matmuls with TF32 off, F.scaled_dot_product_attention(..., scale=1.0), the residual matmul and relu,
    autograd for the backward.  Algorithmic FLOPs: projections 2 B F d 4 H dk, attention 4 B H F^2 dk (forward); the
    backward recomputes Q, K, V and the scores and adds dx and dW (2.75x the projections, 2.5x the attention).  Floors from
    data-sheet rates of the H100 SXM (700 W), not measured: 3 x FLOPs (3xTF32) over 495 TFLOP/s, and bytes over 3.35 TB/s
    (forward x + out; backward x, out, g_out, d_x plus the staged projection gradients, written once and read twice)."""
    import torch.nn.functional as Fn
    print(json.dumps({"autoint_card": card()}), flush=True)
    F = 40

    def torch_pre(x, wq, wk, wv, wr, H, dk):
        B = x.shape[0]
        heads = lambda t: t.reshape(B, F, H, dk).transpose(1, 2)
        o = Fn.scaled_dot_product_attention(heads(x @ wq), heads(x @ wk), heads(x @ wv), scale=1.0)
        return o.transpose(1, 2).reshape(B, F, H * dk) + x @ wr

    def torch_form(x, wq, wk, wv, wr, H, dk):
        return torch.relu(torch_pre(x, wq, wk, wv, wr, H, dk))

    prev_tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        shapes = [(d, 2, 32, B) for d in (16, 64) for B in (1024, 65536)] + [(16, 2, 8, 65536)]
        for d, H, dk, B in shapes:
            HD = H * dk
            ws = [rn(d, HD, std=(1.0 / d) ** 0.5) for _ in range(4)]
            x, g = rn(B, F, d), rn(B, F, HD)
            cfg = {"B": B, "F": F, "d": d, "H": H, "dk": dk}
            proj, attn = 2.0 * B * F * d * 4 * HD, 4.0 * B * H * F * F * dk
            flops = {"fwd": proj + attn, "bwd": 2.75 * proj + 2.5 * attn}
            hbm = {"fwd": 4.0 * B * F * (d + HD), "bwd": 4.0 * B * F * (2 * d + 2 * HD) + 3 * 4.0 * B * F * 4 * HD}
            out = ops.autoint_fwd(x, *ws, H, dk)
            grads = ops.autoint_bwd(x, *ws, out, g, H, dk)
            ps = [t.clone().requires_grad_() for t in (x, *ws)]
            ref_out = torch_form(*ps, H, dk)
            ref_grads = torch.autograd.grad(ref_out, ps, g, retain_graph=True)
            # the gradient comparison takes the relu mask from the kernel's out: where the two forwards round to opposite
            # sides of 0, comparing each against its own mask would measure that flip, not the backward
            masked = torch.autograd.grad(torch_pre(*ps, H, dk), ps, g * (out > 0))
            diff = {"fwd": float((ref_out.detach() - out).abs().max() / ref_out.detach().abs().max()),
                    "bwd": max(float((a - b).abs().max() / b.abs().max()) for a, b in zip(grads, masked))}
            del masked
            runs = {"fwd": (lambda: ops.autoint_fwd(x, *ws, H, dk), lambda: torch_form(x, *ws, H, dk)),
                    "bwd": (lambda: ops.autoint_bwd(x, *ws, out, g, H, dk),
                            lambda: torch.autograd.grad(ref_out, ps, g, retain_graph=True))}
            for way in ("fwd", "bwd"):
                m, bst = timeit(runs[way][0], iters, flush)
                tm, tbst = timeit(runs[way][1], iters, flush)
                f_tc, f_hbm = 3 * flops[way] / 495e12 * 1e6, hbm[way] / 3.35e12 * 1e6
                print(json.dumps({
                    "kernel": f"autoint_{way}", "config": cfg, "ms_median": m, "ms_best": bst,
                    "torch_fp32_ms_median": tm, "torch_fp32_ms_best": tbst, "speedup_vs_torch": tm / m,
                    "max_norm_rel_diff_vs_torch": diff[way], "l2": "flushed between iterations",
                    "algorithmic_TFLOPs": flops[way] / (m * 1e-3) / 1e12, "algorithmic_GBps": hbm[way] / (m * 1e-3) / 1e9,
                    "floor_3xtf32_us": f_tc, "floor_hbm_us": f_hbm, "bound": "tensor" if f_tc >= f_hbm else "hbm",
                    "floor_over_kernel": max(f_tc, f_hbm) / (m * 1e3),
                    "note": "floors are data-sheet rates (H100 SXM, 700 W), not measured; torch: same layer, fp32, TF32 off"}),
                    flush=True)
            del out, grads, ps, ref_out, ref_grads
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev_tf32


def flen_rows(iters, flush, rn, gen):
    """FLEN field-wise bi-interaction (ctr_embed_fwbi_fwd / ctr_fwbi_fwd / ctr_fwbi_bwd) at the config-5 tile shape F = 40,
    D = 32 with M = 3 and 8 groups, B = 4 096 and 65 536, over a 40 x 250 000-row table (1.28 GB, far above the 50 MB L2).
    Beside each row, in the same run: ops.embed_bi_fwd / _bwd at the same (B, F, D) (NFM's fused lookup, the same bytes), and
    plain fp32 torch doing the same layer (gather, group sums by einsum, autograd for the backward).  Algorithmic bytes:
    forward ids + rows (+ tile when written) + h; tile-input forward tile + h; backward tile (+ d_tile) + d_h + row_grads.
    The HBM floor is those bytes over the 3.35 TB/s data-sheet figure (H100 SXM, 700 W), not measured."""
    print(json.dumps({"flen_card": card()}), flush=True)
    F, D, rows = 40, 32, 250_000
    table = rn(F * rows, D, std=0.2)
    off = torch.arange(F + 1, dtype=torch.int64, device="cuda") * rows

    def torch_form(e, oh, iu, kmf, kfm, bmf, bfm):
        p, q = torch.einsum("bfd,fm->bmd", e, oh), torch.einsum("bfd,fm->bmd", e * e, oh)
        h = bmf + bfm + torch.einsum("m,bmd->bd", kfm, p * p - q)
        return h + torch.einsum("k,bkd->bd", kmf, p[:, iu[0]] * p[:, iu[1]])

    for M in (3, 8):
        group = [f % M for f in range(F)]
        # the one-hot group matrix and the pair indices are built once, outside the timed calls
        oh = torch.zeros(F, M, device="cuda")
        oh[torch.arange(F), torch.tensor(group)] = 1.0
        iu = torch.triu_indices(M, M, 1, device="cuda")
        w = [rn(M * (M - 1) // 2, std=0.5), rn(M, std=0.5), rn(D, std=0.1), rn(D, std=0.1)]
        for B in (4096, 65536):
            ids = torch.randint(0, rows, (B, F), device="cuda", generator=gen)
            g, dt = rn(B, D), rn(B, F, D)
            cfg = {"B": B, "F": F, "D": D, "M": M, "rows_per_field": rows}
            row, ids_b, h_b = B * F * D * 4, B * F * 8, B * D * 4
            tile, h = ops.embed_fwbi_fwd(table, off, ids, group, *w)
            e = table[off[:-1] + ids].requires_grad_(True)
            wt = [t.clone().requires_grad_(True) for t in w]
            ref_h = torch_form(e, oh, iu, *wt)
            ref_g = torch.autograd.grad(ref_h, [e, *wt], g, retain_graph=True)
            rg = ops.fwbi_bwd(tile, dt, g, group, w[0], w[1])
            diff = {"fwd": float((ref_h.detach() - h).abs().max() / ref_h.detach().abs().max()),
                    "bwd": float((ref_g[0] + dt - rg[0]).abs().max() / (ref_g[0] + dt).abs().max())}

            def torch_fwd():
                return torch_form(table[off[:-1] + ids], oh, iu, *w)
            runs = [
                ("fwbi_fwd_fused_tile", lambda: ops.embed_fwbi_fwd(table, off, ids, group, *w), ids_b + 2 * row + h_b,
                 "embed_bi_fwd_tile", lambda: ops.embed_bi_fwd(table, off, ids), torch_fwd, "fwd"),
                ("fwbi_fwd_fused_no_tile", lambda: ops.embed_fwbi_fwd(table, off, ids, group, *w, want_tile=False),
                 ids_b + row + h_b, "embed_bi_fwd_no_tile", lambda: ops.embed_bi_fwd(table, off, ids, want_tile=False), None, "fwd"),
                ("fwbi_fwd_tile_input", lambda: ops.fwbi_fwd(tile, group, *w), row + h_b, None, None, None, "fwd"),
                ("fwbi_bwd_d_tile", lambda: ops.fwbi_bwd(tile, dt, g, group, w[0], w[1]), 3 * row + h_b,
                 "embed_bi_bwd_d_tile", lambda: ops.embed_bi_bwd(tile, dt, g),
                 lambda: torch.autograd.grad(ref_h, [e, *wt], g, retain_graph=True), "bwd"),
                ("fwbi_bwd_no_d_tile", lambda: ops.fwbi_bwd(tile, None, g, group, w[0], w[1]), 2 * row + h_b,
                 "embed_bi_bwd_no_d_tile", lambda: ops.embed_bi_bwd(tile, None, g), None, "bwd"),
            ]
            for name, fn, by, bi_name, bi_fn, torch_fn, way in runs:
                m, bst = timeit(fn, iters, flush)
                line = {"kernel": name, "config": cfg, "ms_median": m, "ms_best": bst, "algorithmic_GBps": by / (m * 1e-3) / 1e9,
                        "floor_hbm_us": by / 3.35e12 * 1e6, "floor_over_kernel": by / 3.35e12 / (m * 1e-3),
                        "max_norm_rel_diff_vs_torch": diff[way], "l2": "flushed between iterations",
                        "note": "floor from the 3.35 TB/s data sheet (H100 SXM, 700 W), not measured"}
                if bi_fn is not None:
                    bm, _ = timeit(bi_fn, iters, flush)
                    line.update({"embed_bi": bi_name, "embed_bi_ms_median": bm, "over_embed_bi": m / bm})
                if torch_fn is not None:
                    tm, _ = timeit(torch_fn, iters, flush)
                    line.update({"torch_fp32_ms_median": tm, "speedup_vs_torch": tm / m})
                print(json.dumps(line), flush=True)
            del tile, h, e, wt, ref_h, ref_g, rg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--only", default="dcn,cin,din,fibinet")
    ap.add_argument("--sweep", action="store_true", help="bilinear: also time every (columns per lane, tile) variant of the tournament kernels")
    args = ap.parse_args()
    only = set(args.only.split(","))
    torch.cuda.set_device(0)
    gen = torch.Generator(device="cuda").manual_seed(1234)
    rn = lambda *s, std=1.0: torch.randn(s, device="cuda", generator=gen) * std
    flush = torch.empty(64 * 1024 * 1024, device="cuda")
    hbm, tf, src = peaks()

    def emit(name, cfg, med, best, bytes_=None, flops=None, note=""):
        line = {"kernel": name, "config": cfg, "ms_median": med, "ms_best": best, "l2": "flushed between iterations", "note": note}
        if bytes_ is not None:
            line["algorithmic_GBps"] = bytes_ / (med * 1e-3) / 1e9
            line["frac_of_hbm_peak"] = line["algorithmic_GBps"] / hbm
        if flops is not None:
            line["TFLOPs"] = flops / (med * 1e-3) / 1e12
            line["frac_of_bf16_peak"] = line["TFLOPs"] / tf
        line["peak_source"] = src
        print(json.dumps(line), flush=True)

    if "dcn" in only:   # BASELINE config 2: DCN 3 cross layers, 30 fields x 16 = 480, batch 4096
        B, d, L = 4096, 480, 3
        x0, w, b, g = rn(B, d), rn(L, d, std=0.05), rn(L, d, std=0.05), rn(B, d)
        cfg = {"B": B, "d": d, "L": L}
        m, bst = timeit(lambda: ops.cross_fwd(x0, w, b), args.iters, flush)
        emit("cross_fwd", cfg, m, bst, bytes_=B * 2 * d * 4, note="2*d*4 B/sample")
        m, bst = timeit(lambda: ops.cross_bwd(x0, w, b, g), args.iters, flush)
        emit("cross_bwd", cfg, m, bst, bytes_=B * 3 * d * 4, note="3*d*4 B/sample")
        for B2 in (65536,):
            x0b, gb = rn(B2, d), rn(B2, d)
            m, bst = timeit(lambda: ops.cross_fwd(x0b, w, b), args.iters, flush)
            emit("cross_fwd", {"B": B2, "d": d, "L": L}, m, bst, bytes_=B2 * 2 * d * 4)
            m, bst = timeit(lambda: ops.cross_bwd(x0b, w, b, gb), args.iters, flush)
            emit("cross_bwd", {"B": B2, "d": d, "L": L}, m, bst, bytes_=B2 * 3 * d * 4)

    if "cin" in only:   # BASELINE config 3: xDeepFM CIN [128,128], 30 fields, D=16, batch 8192
        B, mm, D, H = 8192, 30, 16, 128
        x0 = rn(B, mm, D, std=0.25)
        w1, w2 = rn(mm * mm, H, std=0.05), rn(H * mm, H, std=0.05)
        x1 = ops.cin_fwd(x0, x0, w1)
        g = rn(B, H, D)
        for prec in (0, 1):
            tag = "3xTF32" if prec == 0 else "1xTF32"
            m, bst = timeit(lambda: ops.cin_fwd(x0, x0, w1, want_pooled=True, precision=prec), args.iters, flush)
            emit(f"cin_fwd_layer1_{tag}", {"B": B, "m": mm, "hk": mm, "D": D, "H": H}, m, bst, flops=2.0 * B * D * mm * mm * H)
            m, bst = timeit(lambda: ops.cin_fwd(x0, x1, w2, want_pooled=True, precision=prec), args.iters, flush)
            emit(f"cin_fwd_layer2_{tag}", {"B": B, "m": mm, "hk": H, "D": D, "H": H}, m, bst, flops=2.0 * B * D * H * mm * H)
        m, bst = timeit(lambda: ops.cin_bwd(x0, x0, w1, g), max(3, args.iters // 4), flush)
        emit("cin_bwd_layer1", {"B": B, "m": mm, "hk": mm, "D": D, "H": H}, m, bst, flops=4.0 * B * D * mm * mm * H)
        m, bst = timeit(lambda: ops.cin_bwd(x0, x1, w2, g), max(3, args.iters // 4), flush)
        emit("cin_bwd_layer2", {"B": B, "m": mm, "hk": H, "D": D, "H": H}, m, bst, flops=4.0 * B * D * H * mm * H)

    if "din" in only:   # BASELINE config 4: DIN attention, seq_len 50, H=16, batch 4096
        B, T, H = 4096, 50, 16
        q, k = rn(B, H, std=0.25), rn(B, T, H, std=0.25)
        lens = torch.randint(0, T + 1, (B,), device="cuda", generator=gen)
        ws = [rn(4 * H, 64, std=0.2), rn(64, std=0.1), rn(64, 32, std=0.2), rn(32, std=0.1), rn(32, 1, std=0.3), rn(1, std=0.1)]
        g = rn(B, H)
        flops_full = B * T * 2.0 * (4 * H * 64 + 64 * 32 + 32)
        for soft in (False, True):
            m, bst = timeit(lambda: ops.din_attention_fwd(q, k, lens, *ws, is_softmax=soft), args.iters, flush)
            emit(f"din_fwd_softmax{int(soft)}", {"B": B, "T": T, "H": H, "lengths": "uniform{0..50}"}, m, bst,
                 bytes_=B * (T * H * 4 + 8 + 2 * H * 4), flops=flops_full,
                 note="FLOPs counted as the reference does them (all T positions, unfolded layer 1)")
            m, bst = timeit(lambda: ops.din_attention_bwd(q, k, lens, *ws, g, is_softmax=soft), args.iters, flush)
            emit(f"din_bwd_softmax{int(soft)}", {"B": B, "T": T, "H": H}, m, bst, flops=2 * flops_full)

    if "fibinet" in only:   # FiBiNET F=30, K=16, r=8 (no BASELINE config; reference defaults)
        B, F, K, r = 4096, 30, 16, 8
        x, w1, w2 = rn(B, F, K, std=0.25), rn(F, r, std=0.3), rn(r, F, std=0.3)
        g = rn(B, F, K)
        m, bst = timeit(lambda: ops.senet_fwd(x, w1, w2), args.iters, flush)
        emit("senet_fwd", {"B": B, "F": F, "K": K, "r": r}, m, bst, bytes_=B * 2 * F * K * 4)
        m, bst = timeit(lambda: ops.senet_bwd(x, w1, w2, g), args.iters, flush)
        emit("senet_bwd", {"B": B, "F": F, "K": K, "r": r}, m, bst, bytes_=B * 3 * F * K * 4)
        P = (F - 1) * (F - 2) // 2
        gp = rn(B, P, K)
        for typ in ("all", "each", "interaction"):
            w = rn(*ops.bilinear_w_shape(F, K, typ), std=0.2)
            variants = [(4, "default (staged all/each, tournament interaction)"), (7, "tournament")]
            if args.sweep:
                variants += [(7 | (kt << 10) | (tile << 4), f"tournament kt={kt} tile={tile}") for kt in (1, 2, 4) for tile in (4, 8, 16)]
            variants += [(8, "round-1 CTA-per-sample kernels")]
            for mask, impl in variants:
                prev = ops.bilinear_set_tournament(mask)
                m, bst = timeit(lambda: ops.bilinear_fwd(x, w, typ), args.iters, flush)
                emit(f"bilinear_fwd_{typ}", {"B": B, "F": F, "K": K, "impl": impl}, m, bst, bytes_=B * (F * K + P * K) * 4)
                m, bst = timeit(lambda: ops.bilinear_bwd(x, w, typ, gp), max(3, args.iters // 4), flush)
                emit(f"bilinear_bwd_{typ}", {"B": B, "F": F, "K": K, "impl": impl}, m, bst, bytes_=B * (2 * F * K + P * K) * 4)
                ops.bilinear_set_tournament(prev)

    if "pairwise" in only:   # SURVEY 8f.4 siblings (FwFM at the config-5 tile shape; AFM at the reference's flag defaults and at F=30)
        B, F, K = 65536, 40, 32
        x, r, g1 = rn(B, F, K, std=0.2), rn(F * (F - 1) // 2, std=0.3), rn(B)
        m_, bst = timeit(lambda: ops.fwfm_fwd(x, r), args.iters, flush)
        emit("fwfm_fwd", {"B": B, "F": F, "K": K}, m_, bst, bytes_=B * F * K * 4, flops=2.0 * B * K * F * (F - 1) / 2)
        m_, bst = timeit(lambda: ops.fwfm_bwd(x, r, g1), args.iters, flush)
        emit("fwfm_bwd", {"B": B, "F": F, "K": K}, m_, bst, bytes_=2 * B * F * K * 4, flops=2.0 * B * K * (F * F + F * (F - 1) / 2))
        for (B, F, K, T) in ((65536, 7, 8, 128), (8192, 30, 16, 8)):
            x, w, b, h, gk = rn(B, F, K, std=0.5), rn(K, T, std=0.3), rn(T, std=0.1), rn(T, std=0.3), rn(B, K)
            P = F * (F - 1) // 2
            m_, bst = timeit(lambda: ops.afm_fwd(x, w, b, h), args.iters, flush)
            emit("afm_fwd", {"B": B, "F": F, "K": K, "T": T}, m_, bst, bytes_=B * (F * K + K) * 4, flops=2.0 * B * P * (K * T + T + K))
            m_, bst = timeit(lambda: ops.afm_bwd(x, w, b, h, gk), args.iters, flush)
            emit("afm_bwd", {"B": B, "F": F, "K": K, "T": T}, m_, bst, bytes_=B * (2 * F * K + K) * 4, flops=2.0 * B * P * (4 * K * T + 2 * T + 4 * K))

    if "bst" in only:   # BST defaults: 50-step history + target = 51 positions, d = 8, 3 heads (BST/bst.py:45-47), batch 4096
        for (B, T, d, H) in ((4096, 51, 8, 3), (4096, 51, 16, 3)):
            x, g = rn(B, T, d), rn(B, T, d)
            klen = torch.randint(1, T + 1, (B,), device="cuda", generator=gen)
            packed = rn(int(ops._lib.lib().ctr_bst_param_count(d, H, T)), std=0.3)
            flops = 2.0 * B * (3 * H * T * d * d + 2 * H * T * T * d + H * T * d * d + T * d * d)
            m_, bst = timeit(lambda: ops.bst_transformer_fwd(x, x, x, klen, packed, H, T), args.iters, flush)
            emit("bst_transformer_fwd", {"B": B, "T": T, "d": d, "heads": H}, m_, bst, bytes_=2 * B * T * d * 4, flops=flops)
            m_, bst = timeit(lambda: ops.bst_transformer_bwd(x, x, x, klen, packed, g, H, T), args.iters, flush)
            emit("bst_transformer_bwd", {"B": B, "T": T, "d": d, "heads": H}, m_, bst, bytes_=5 * B * T * d * 4, flops=3 * flops)

    if "adam" in only:   # SURVEY 8f.3 at BASELINE config 5: the table update that follows the hot path
        from recalgorithm_b200 import autograd, optim
        rows = int(os.environ.get("CTR_BENCH_ROWS", 2_500_000))
        B, F, D = 65536, 40, 32
        tables = autograd.EmbeddingTables([rows] * F, D, device="cuda")
        ids = [torch.randint(0, rows, (B, F), device="cuda", generator=gen) for _ in range(4)]
        vals = rn(B, F, D)
        for lazy in (True, False):
            opt = optim.TableAdam(tables, lr=1e-3, lazy=lazy)
            k = [0]

            def step():
                k[0] += 1
                tables.grad_slices.append(autograd.IndexedSlices(vals.clone(), ids[k[0] % 4], tables.field_row_offset))
                opt.step()
            m_, bst = timeit(step, max(5, args.iters // 2), flush)
            n = B * F
            # algorithmic bytes: ids + values read; (m, v, var) read+written for the referenced rows; dense variant: 6 table streams
            by = n * 8 + n * D * 4 + 6 * n * D * 4 if lazy else 6 * tables.num_rows * D * 4 + n * 8 + n * D * 4
            emit("table_adam_lazy" if lazy else "table_adam_dense", {"B": B, "F": F, "D": D, "rows_per_field": rows}, m_, bst,
                 bytes_=by, note="includes a 336 MB clone of the gradient values per step (the step consumes them)")
            del opt
        # backward + LazyAdam: unfused pair (ctr_embed_fm2_bwd writes row_grads, ctr_adam_indexed_slices re-reads them) vs the
        # fused kernel (ctr_embed_fm2_bwd_adam)
        tile, _ = ops.embed_fm2_fwd(tables.weight, tables.field_row_offset, ids[0])
        d_tile, d_fm2 = rn(B, F, D, std=0.01), rn(B, std=0.01)
        opt_u = optim.TableAdam(tables, lr=1e-3, lazy=True)
        rg = torch.empty_like(tile)

        def unfused():
            k[0] += 1
            ops.embed_fm2_bwd(tile, d_tile, d_fm2, row_grads=rg)
            tables.grad_slices.append(autograd.IndexedSlices(rg, ids[k[0] % 4], tables.field_row_offset))
            opt_u.step()
        m_, bst = timeit(unfused, max(5, args.iters // 2), flush)
        n = B * F
        by_u = n * 8 + 3 * n * D * 4 + n * D * 4 + 6 * n * D * 4
        emit("bwd_plus_lazy_adam_unfused", {"B": B, "F": F, "D": D, "rows_per_field": rows}, m_, bst, bytes_=by_u,
             note="embed_fm2_bwd (read tile, d_tile; write row_grads) + claim/merge/update (read row_grads; RMW m, v, var)")
        del opt_u
        opt_f = optim.TableAdam(tables, lr=1e-3, lazy=True, fused_backward=True)

        def fused():
            k[0] += 1
            opt_f.apply_fused(tile, d_tile, d_fm2, ids[k[0] % 4])
            opt_f.step()
        m_, bst = timeit(fused, max(5, args.iters // 2), flush)
        by_f = n * 8 + 2 * n * D * 4 + 6 * n * D * 4
        emit("bwd_plus_lazy_adam_fused", {"B": B, "F": F, "D": D, "rows_per_field": rows}, m_, bst, bytes_=by_f,
             note="ctr_embed_fm2_bwd_adam: read tile, d_tile; RMW m, v, var; row_grads only for rows with duplicates")

    if "pnn" in only:   # PNN product layer at the reference defaults (F = 8 fields, K = 8, output_dimension 1024); not in the default list
        pnn_rows(args.iters, flush, rn, hbm)
    if "dien" in only:  # DIEN seq_encoder at the reference shape (na = 16, nh = 8) with config 4's T and lengths; not in the default list
        dien_rows(args.iters, flush, hbm)
    if "dien_aux" in only:  # DIEN's auxiliary loss at the same shape with T_neg = 3; not in the default list
        dien_aux_rows(args.iters, flush, hbm)
    if "deepcrossing" in only:  # DeepCrossing residual unit at the reference width (d = 82) and both result.md H; not in the default list
        deepcrossing_rows(args.iters, flush, rn)
    if "mmoe" in only:  # MMoE expert-gate layer at the reference shape (d = 82, E = 3, H = 512, T = 3); not in the default list
        mmoe_rows(args.iters, flush, rn)
    if "ple" in only:   # PLE extraction network (d = 82) and final layer (d = 256) at the default row; not in the default list
        ple_rows(args.iters, flush, rn)
    if "wide" in only:  # Wide & Deep wide part (crossed column, FTRL) at the reference bucket count and 10^7; not in the default list
        wide_rows(args.iters, flush)
    if "autoint" in only:  # AutoInt interacting layer at the paper's setting (F = 40, H = 2, dk = 32, d = 16 and 64); not in the default list
        autoint_rows(args.iters, flush, rn)
    if "flen" in only:  # FLEN field-wise bi-interaction at F = 40, D = 32, M = 3 / 8, beside embed_bi and plain torch; not in the default list
        flen_rows(args.iters, flush, rn, gen)


if __name__ == "__main__" and "--configs" not in sys.argv:
    main()


def config_level():
    """BASELINE configs 2-4 as lookup + interaction chains (hot path only: no dense tail), forward+backward, samples/s.
    Timed as one CUDA-event region per step, L2 flushed between steps; tables 1 M rows per field (SURVEY 8d)."""
    import statistics
    torch.cuda.set_device(0)
    gen = torch.Generator(device="cuda").manual_seed(1234)
    flush = torch.empty(64 * 1024 * 1024, device="cuda")
    rn = lambda *s, std=1.0: torch.randn(s, device="cuda", generator=gen) * std

    def run(name, cfg, B, step, iters=15):
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        ts = []
        for _ in range(iters):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); step(); b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        ms = statistics.median(ts)
        print(json.dumps({"config_level": name, "config": cfg, "ms_per_step": ms, "samples_per_sec": B / (ms * 1e-3),
                          "what": "lookup fwd + interaction fwd + interaction bwd + lookup bwd (IndexedSlices); no dense tail",
                          "l2": "flushed between steps"}), flush=True)

    rows = 1_000_000
    # ---- config 2: DCN, 30 fields x 16, L = 3, B = 4096
    B, F, D, L = 4096, 30, 16, 3
    table = rn(rows * F, D, std=D ** -0.5); off = torch.arange(F + 1, device="cuda") * rows
    ids = torch.randint(0, rows, (B, F), device="cuda", generator=gen)
    w, bb = rn(L, F * D, std=0.05), rn(L, F * D, std=0.05); g = rn(B, F * D)

    def dcn():
        tile, _ = ops.embed_fm2_fwd(table, off, ids, want_fm2=False)
        x0 = tile.view(B, F * D)
        ops.cross_fwd(x0, w, bb)
        dx0, _, _, _ = ops.cross_bwd(x0, w, bb, g)
        ops.embed_fm2_bwd(tile, dx0.view(B, F, D), None)
    run("dcn_cfg2", {"B": B, "F": F, "D": D, "L": L, "rows_per_field": rows}, B, dcn)

    def graphed(fn):
        """The same C-ABI calls captured once into a CUDA graph (they only enqueue work on the given stream and never
        allocate or synchronise, so they are capturable as they are); a step is then ONE graph launch."""
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
    run("dcn_cfg2_cuda_graph", {"B": B, "F": F, "D": D, "L": L, "rows_per_field": rows, "launch": "one CUDA graph replay per step"}, B,
        graphed(dcn))

    # ---- config 3: xDeepFM CIN [128,128], 30 fields x 16, B = 8192
    B, F, D, H = 8192, 30, 16, 128
    ids3 = torch.randint(0, rows, (B, F), device="cuda", generator=gen)
    w1, w2 = rn(F * F, H, std=0.05), rn(H * F, H, std=0.05)
    gp = rn(B, 2 * H)

    def xdeepfm():
        x0, _ = ops.embed_fm2_fwd(table, off, ids3, want_fm2=False)
        x1, p1 = ops.cin_fwd(x0, x0, w1, want_pooled=True)
        x2, p2 = ops.cin_fwd(x0, x1, w2, want_pooled=True)
        g2 = gp[:, H:].unsqueeze(-1).expand(B, H, D).contiguous()          # d(pooled)/d(out) broadcast over D
        dx0b, dx1, _ = ops.cin_bwd(x0, x1, w2, g2)
        g1 = dx1 + gp[:, :H].unsqueeze(-1)
        dx0a, dxk, _ = ops.cin_bwd(x0, x0, w1, g1.contiguous())
        ops.embed_fm2_bwd(x0, (dx0a + dxk + dx0b).contiguous(), None)
    run("xdeepfm_cfg3", {"B": B, "m": F, "D": D, "cin": [H, H], "rows_per_field": rows}, B, xdeepfm)

    # ---- config 4: DIN attention, history T = 50 (one lookup per step), H = 16, B = 4096
    B, T, Hd = 4096, 50, 16
    tab4 = rn(rows, Hd, std=0.25); off4 = torch.tensor([0, rows], device="cuda")
    lens = torch.randint(0, T + 1, (B,), device="cuda", generator=gen)
    hist = torch.randint(0, rows, (B * T, 1), device="cuda", generator=gen)
    hist[(torch.arange(T, device="cuda")[None, :] >= lens[:, None]).reshape(-1)] = -1     # padding -> zero vectors
    tgt = torch.randint(0, rows, (B, 1), device="cuda", generator=gen)
    ws = [rn(4 * Hd, 64, std=0.2), rn(64, std=0.1), rn(64, 32, std=0.2), rn(32, std=0.1), rn(32, 1, std=0.3), rn(1, std=0.1)]
    go = rn(B, Hd)

    def din():
        keys, _ = ops.embed_fm2_fwd(tab4, off4, hist, want_fm2=False)
        q, _ = ops.embed_fm2_fwd(tab4, off4, tgt, want_fm2=False)
        k3, q2 = keys.view(B, T, Hd), q.view(B, Hd)
        out, att = ops.din_attention_fwd(q2, k3, lens, *ws, want_weights=True)
        dq, dk, _ = ops.din_attention_bwd(q2, k3, lens, *ws, go, att_w=att)
        ops.embed_fm2_bwd(keys, dk.view(B * T, 1, Hd), None)
        ops.embed_fm2_bwd(q, dq.view(B, 1, Hd), None)
    run("din_cfg4", {"B": B, "T": T, "H": Hd, "rows": rows, "lengths": "uniform{0..50}"}, B, din)


if __name__ == "__main__" and "--configs" in sys.argv:
    config_level()
