"""Ceilings of the config-5 step (B=65536, F=40, D=32, 12.8 GB table) on the GPU it runs on, each next to the kernel it bounds.

The H100 SXM data sheet gives 3.35 TB/s of HBM3 bandwidth; what a kernel can reach depends on its access pattern (random 128-byte
rows, a 2-read : 1-write stream), so each fused kernel is set against a library kernel with the same bytes and the same pattern.
Prints one JSON line per variant (algorithmic GB/s, and the fraction of the data-sheet or MEASURED_PEAKS.json peak), then one
"device" line (card name, power limit, median SM clock over the run) and one "shares" line (each kernel's time over its ceiling's):
  gather_only      ctr_embed_fm2_fwd with tile=NULL: the same random row reads, 256 KB of output
  fused_fwd        ctr_embed_fm2_fwd (tile + fm2): the forward of bench.py's step
  torch_index      torch.index_select of the same rows (library gather, writes the tile)     -> ceiling of fused_fwd
  stream_copy      torch copy of a tile-sized buffer (streaming read + write)
  fused_bwd        ctr_embed_fm2_bwd (tile + d_tile read, row_grads write): the backward of bench.py's step
  bwd_stream       torch.add(tile, d_tile, out=row_grads): the backward's bytes, no FM2 arithmetic -> ceiling of fused_bwd
  step             bench.py's step: fused_fwd then fused_bwd
L2 (50 MB) is flushed by a 256 MB write before every timed call; the flush is outside the timed region.
"""
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from recalgorithm_b200 import autograd, ops  # noqa: E402


def device_info(clocks):
    """Card name and power limit, read in the same run as the timings (NVML; None where it cannot be read)."""
    info = {"device": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_mhz_median": clocks["sm_mhz"],
            "sm_max_mhz": clocks["sm_max_mhz"], "throttle_reasons": clocks["reasons"], "clock_samples": clocks["samples"]}
    try:
        import pynvml
        pynvml.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        phys = int(vis.split(",")[0]) if vis and vis.split(",")[0].isdigit() else 0
        info["power_limit_w"] = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(phys)) / 1000.0
    except Exception:
        pass
    return info


def main():
    B, F, D, rows = 65536, 40, 32, int(os.environ.get("CTR_BENCH_ROWS", 2_500_000))
    from bench import ClockSampler, measured_peaks        # MEASURED_PEAKS.json, else the H100 SXM data sheet
    peak = measured_peaks()["hbm_gbs"]
    sampler = ClockSampler(0).start()
    gen = torch.Generator(device="cuda").manual_seed(1)
    tables = autograd.EmbeddingTables([rows] * F, D, device="cuda", init=None)
    tables.weight.normal_(0, 1, generator=gen)
    ids = [torch.randint(0, rows, (B, F), device="cuda", generator=gen) for _ in range(8)]
    flat = [(i + tables.field_row_offset[:-1][None, :]).reshape(-1) for i in ids]
    tile = torch.empty((B, F, D), device="cuda"); fm2 = torch.empty((B, 1), device="cuda")
    out2 = torch.empty((B * F, D), device="cuda")
    d_tile = torch.randn((B, F, D), device="cuda", generator=gen) * 0.01
    d_fm2 = torch.randn((B,), device="cuda", generator=gen) * 0.01
    row_grads = torch.empty((B, F, D), device="cuda")
    flush = torch.empty(64 * 1024 * 1024, device="cuda")
    k = [0]

    def t(fn, iters=30):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(iters):
            k[0] += 1
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record(); torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return statistics.median(ts)

    def fwd():
        ops.embed_fm2_fwd(tables.weight, tables.field_row_offset, ids[k[0] % 8], tile=tile, fm2=fm2)

    def bwd():
        ops.embed_fm2_bwd(tile, d_tile, d_fm2, row_grads=row_grads)

    def step():
        fwd(); bwd()

    rows_b, ids_b, tile_b = B * F * D * 4, B * F * 8, B * F * D * 4
    fwd_b, bwd_b = rows_b + ids_b + tile_b, 3 * tile_b
    cases = [
        ("gather_only", lambda: ops.embed_fm2_fwd(tables.weight, tables.field_row_offset, ids[k[0] % 8], want_tile=False, fm2=fm2), rows_b + ids_b),
        ("fused_fwd", fwd, fwd_b),
        ("torch_index", lambda: torch.index_select(tables.weight, 0, flat[k[0] % 8], out=out2), fwd_b),
        ("stream_copy", lambda: out2.copy_(tile.view(B * F, D)), 2 * tile_b),
        ("fused_bwd", bwd, bwd_b),
        ("bwd_stream", lambda: torch.add(tile, d_tile, out=row_grads), bwd_b),
        ("step", step, fwd_b + bwd_b),
    ]
    ms_of = {}
    for name, fn, nbytes in cases:
        ms = ms_of[name] = t(fn)
        print(json.dumps({"variant": name, "ms": ms, "algorithmic_GBps": nbytes / ms / 1e6, "frac_of_hbm_peak": nbytes / ms / 1e6 / peak,
                          "hbm_peak_GBps": peak}), flush=True)
    print(json.dumps({"shares": {"fused_fwd_of_torch_index": ms_of["torch_index"] / ms_of["fused_fwd"],
                                 "fused_fwd_of_gather_only": ms_of["gather_only"] / ms_of["fused_fwd"],
                                 "fused_bwd_of_bwd_stream": ms_of["bwd_stream"] / ms_of["fused_bwd"],
                                 "step_of_ceilings": (ms_of["torch_index"] + ms_of["bwd_stream"]) / ms_of["step"]},
                      "what": "ceiling time over kernel time (1.0 = the kernel runs at its access pattern's measured ceiling)"}), flush=True)
    if "--sweep" in sys.argv:
        # same number of bytes gathered, different row widths: is the random-read rate per ACCESS (row activations) or per byte?
        del tables, tile, out2, flat, d_tile, row_grads
        torch.cuda.empty_cache()
        for Dw in (16, 32, 64, 128):
            Fw = 40 * 32 // Dw
            rows_w = rows * 32 // Dw // (Fw // 40) if Fw >= 40 else rows * 32 // Dw * (40 // Fw)
            tb = autograd.EmbeddingTables([rows_w] * Fw, Dw, device="cuda", init=None)
            tb.weight.normal_(0, 1, generator=gen)
            idw = [torch.randint(0, rows_w, (B, Fw), device="cuda", generator=gen) for _ in range(8)]
            ms = t(lambda: ops.embed_fm2_fwd(tb.weight, tb.field_row_offset, idw[k[0] % 8], want_tile=False, fm2=fm2))
            nb = B * Fw * (Dw * 4 + 8)
            print(json.dumps({"variant": f"gather_only_row{Dw * 4}B", "F": Fw, "rows_per_field": rows_w, "table_GB": tb.weight.numel() * 4 / 1e9,
                              "ms": ms, "algorithmic_GBps": nb / ms / 1e6, "row_reads_per_us": B * Fw / ms / 1e3}), flush=True)
            del tb, idw
            torch.cuda.empty_cache()
    print(json.dumps(device_info(sampler.stop())), flush=True)


if __name__ == "__main__":
    main()
