"""How close is the fused gather to what HBM3e gives RANDOM 128-byte reads?  (config 5: B=65536, F=40, D=32, 12.8 GB table)

Prints one JSON line per variant: algorithmic GB/s and the fraction of the measured streaming peak
  gather_only      ctr_embed_fm2_fwd with tile=NULL: the same random row reads, 256 KB of output  -> the random-read ceiling
  fused_fwd        ctr_embed_fm2_fwd (tile + fm2): what bench.py's roofline reports
  torch_index      torch.index_select of the same rows (library gather, writes the tile)
  stream_copy      torch copy of a tile-sized buffer (streaming read + write)
"""
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from recalgorithm_b200 import autograd, ops  # noqa: E402


def main():
    B, F, D, rows = 65536, 40, 32, int(os.environ.get("CTR_BENCH_ROWS", 2_500_000))
    from bench import measured_peaks                      # MEASURED_PEAKS.json, else the H100 SXM data sheet
    peak = measured_peaks()["hbm_gbs"]
    gen = torch.Generator(device="cuda").manual_seed(1)
    tables = autograd.EmbeddingTables([rows] * F, D, device="cuda", init=None)
    tables.weight.normal_(0, 1, generator=gen)
    ids = [torch.randint(0, rows, (B, F), device="cuda", generator=gen) for _ in range(8)]
    flat = [(i + tables.field_row_offset[:-1][None, :]).reshape(-1) for i in ids]
    tile = torch.empty((B, F, D), device="cuda"); fm2 = torch.empty((B, 1), device="cuda")
    out2 = torch.empty((B * F, D), device="cuda")
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

    rows_b, ids_b, tile_b = B * F * D * 4, B * F * 8, B * F * D * 4
    cases = [
        ("gather_only", lambda: ops.embed_fm2_fwd(tables.weight, tables.field_row_offset, ids[k[0] % 8], want_tile=False, fm2=fm2), rows_b + ids_b),
        ("fused_fwd", lambda: ops.embed_fm2_fwd(tables.weight, tables.field_row_offset, ids[k[0] % 8], tile=tile, fm2=fm2), rows_b + ids_b + tile_b),
        ("torch_index", lambda: torch.index_select(tables.weight, 0, flat[k[0] % 8], out=out2), rows_b + ids_b + tile_b),
        ("stream_copy", lambda: out2.copy_(tile.view(B * F, D)), 2 * tile_b),
    ]
    for name, fn, nbytes in cases:
        ms = t(fn)
        print(json.dumps({"variant": name, "ms": ms, "algorithmic_GBps": nbytes / ms / 1e6, "frac_of_hbm_peak": nbytes / ms / 1e6 / peak,
                          "hbm_peak_GBps": peak}), flush=True)
    if "--sweep" in sys.argv:
        # same number of bytes gathered, different row widths: is the random-read rate per ACCESS (row activations) or per byte?
        del tables, tile, out2, flat
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


if __name__ == "__main__":
    main()
