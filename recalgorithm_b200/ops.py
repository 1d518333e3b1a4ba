"""Thin tensor-level wrappers over the C ABI (device pointers + sizes + the current CUDA stream).

torch is plumbing here: it owns device memory and streams; every computation below is one call
into libctr_b200.so.  Functions validate devices/dtypes and raise instead of falling back.
"""
from __future__ import annotations

import ctypes
import math
from typing import Optional, Tuple

import torch

from . import _lib

F32, I64 = torch.float32, torch.int64


_empty_anchor = {}


def _ptr(t: Optional[torch.Tensor]):
    """Device address of a tensor; None stays NULL (= "output not wanted").  An EMPTY tensor (batch 0) has data_ptr() == 0,
    which the C ABI would read as a missing argument: it gets the address of a small per-device anchor instead -- never
    dereferenced, every entry point returns before launching when its batch dimension is 0."""
    if t is None:
        return None
    if t.numel() == 0:
        a = _empty_anchor.get(t.device)
        if a is None:
            a = _empty_anchor[t.device] = torch.zeros(64, dtype=torch.uint8, device=t.device)
        return a.data_ptr()
    return t.data_ptr()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


I32 = torch.int32


def _chk(t: Optional[torch.Tensor], dtype, name: str, shape=None):
    if t is None:
        return
    if not t.is_cuda:
        raise RuntimeError(f"{name}: expected a CUDA tensor (there is no CPU path)")
    if t.device.index != torch.cuda.current_device():
        # kernels launch on the CURRENT device's current stream: a tensor of another GPU would be touched from the wrong
        # device / stream (single-process multi-GPU callers wrap their calls in `with torch.cuda.device(t.device)`)
        raise RuntimeError(f"{name}: lives on cuda:{t.device.index} but the current device is cuda:{torch.cuda.current_device()}")
    if t.dtype != dtype:
        raise TypeError(f"{name}: expected {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"{name}: must be contiguous")
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name}: expected shape {tuple(shape)}, got {tuple(t.shape)}")


# ------------------------------------------------------------------ Row L + FM2
def embed_fm2_fwd(table: torch.Tensor, field_row_offset: torch.Tensor, ids: torch.Tensor,
                  want_tile: bool = True, want_fm2: bool = True,
                  tile: Optional[torch.Tensor] = None, fm2: Optional[torch.Tensor] = None,
                  ids64_out: Optional[torch.Tensor] = None
                  ) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
    """Fused lookup (+ FM second-order logit).  table (V,D); field_row_offset (F+1,) i64; ids (B,F) i64 -- or i32 (half the
    bytes over PCIe; ``ids64_out`` (B,F) i64 then receives the widened copy for IndexedSlices consumers).
    Returns (tile (B,F,D) | None, fm2 (B,1) | None)."""
    B, F = ids.shape
    D = table.shape[1]
    _chk(table, F32, "table"); _chk(field_row_offset, I64, "field_row_offset", (F + 1,))
    if ids.dtype == I32:
        _chk(ids, I32, "ids"); _chk(ids64_out, I64, "ids64_out", (B, F))
        if want_tile and tile is None:
            tile = torch.empty((B, F, D), dtype=F32, device=table.device)
        if want_fm2 and fm2 is None:
            fm2 = torch.empty((B, 1), dtype=F32, device=table.device)
        _chk(tile, F32, "tile", (B, F, D)); _chk(fm2, F32, "fm2", (B, 1))
        _lib.check(_lib.lib().ctr_embed_fm2_fwd_ids32(_ptr(table), _ptr(field_row_offset), _ptr(ids), B, F, D, _ptr(tile),
                                                      _ptr(fm2), _ptr(ids64_out), _stream()))
        return tile, fm2
    _chk(ids, I64, "ids")
    if want_tile and tile is None:
        tile = torch.empty((B, F, D), dtype=F32, device=table.device)
    if want_fm2 and fm2 is None:
        fm2 = torch.empty((B, 1), dtype=F32, device=table.device)
    _chk(tile, F32, "tile", (B, F, D)); _chk(fm2, F32, "fm2", (B, 1))
    _lib.check(_lib.lib().ctr_embed_fm2_fwd(_ptr(table), _ptr(field_row_offset), _ptr(ids), B, F, D,
                                            _ptr(tile), _ptr(fm2), _stream()))
    return tile, fm2


def embed_fm2_bwd(tile: torch.Tensor, d_tile: Optional[torch.Tensor], d_fm2: Optional[torch.Tensor],
                  row_grads: Optional[torch.Tensor] = None) -> torch.Tensor:
    """IndexedSlices values (B,F,D) of the lookup gradient: d_tile + d_fm2 * (S - e)."""
    B, F, D = tile.shape
    _chk(tile, F32, "tile"); _chk(d_tile, F32, "d_tile", (B, F, D))
    if d_fm2 is not None:
        d_fm2 = d_fm2.reshape(B)
    _chk(d_fm2, F32, "d_fm2", (B,))
    if row_grads is None:
        row_grads = torch.empty_like(tile)
    _chk(row_grads, F32, "row_grads", (B, F, D))
    _lib.check(_lib.lib().ctr_embed_fm2_bwd(_ptr(tile), _ptr(d_tile), _ptr(d_fm2), B, F, D, _ptr(row_grads), _stream()))
    return row_grads


def embed_fm2_lin_fwd(table: torch.Tensor, field_row_offset: torch.Tensor, ids: torch.Tensor, wlin: torch.Tensor,
                      want_tile: bool = True, ids64_out: Optional[torch.Tensor] = None):
    """Lookup + FM2 + fused dense(1) head over the flattened tile: returns (tile | None, fm2 (B,1), lin (B,1)) with
    lin = tile.reshape(B, F*D) @ wlin.  ids int64 or int32 (``ids64_out`` then receives the widened copy)."""
    B, F = ids.shape
    D = table.shape[1]
    _chk(table, F32, "table"); _chk(field_row_offset, I64, "field_row_offset", (F + 1,))
    i32 = ids.dtype == I32
    _chk(ids, I32 if i32 else I64, "ids"); _chk(ids64_out, I64, "ids64_out", (B, F))
    wlin = wlin.reshape(F * D)
    _chk(wlin, F32, "wlin", (F * D,))
    tile = torch.empty((B, F, D), dtype=F32, device=table.device) if want_tile else None
    fm2 = torch.empty((B, 1), dtype=F32, device=table.device)
    lin = torch.empty((B, 1), dtype=F32, device=table.device)
    _lib.check(_lib.lib().ctr_embed_fm2_lin_fwd(_ptr(table), _ptr(field_row_offset), _ptr(ids), int(i32), B, F, D, _ptr(wlin),
                                                _ptr(tile), _ptr(fm2), _ptr(lin), _ptr(ids64_out), _stream()))
    return tile, fm2, lin


def embed_fm2_lin_bwd(tile: torch.Tensor, wlin: torch.Tensor, d_fm2: Optional[torch.Tensor], d_lin: Optional[torch.Tensor],
                      row_grads: Optional[torch.Tensor] = None):
    """Backward of embed_fm2_lin_fwd: (row_grads (B,F,D) = IndexedSlices values, d_wlin (F*D,))."""
    B, F, D = tile.shape
    _chk(tile, F32, "tile")
    wlin = wlin.reshape(F * D)
    _chk(wlin, F32, "wlin", (F * D,))
    if d_fm2 is not None:
        d_fm2 = d_fm2.reshape(B)
    if d_lin is not None:
        d_lin = d_lin.reshape(B)
    _chk(d_fm2, F32, "d_fm2", (B,)); _chk(d_lin, F32, "d_lin", (B,))
    if row_grads is None:
        row_grads = torch.empty_like(tile)
    _chk(row_grads, F32, "row_grads", (B, F, D))
    d_wlin = torch.empty((F * D,), dtype=F32, device=tile.device)
    _lib.check(_lib.lib().ctr_embed_fm2_lin_bwd(_ptr(tile), _ptr(wlin), _ptr(d_fm2), _ptr(d_lin), B, F, D, _ptr(row_grads),
                                                _ptr(d_wlin), _stream()))
    return row_grads, d_wlin


def embed_seq_fwd(table: torch.Tensor, ids: torch.Tensor, row_range: Optional[torch.Tensor] = None,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Sequence lookup: ids (B,T) int64 all index ONE table (rows [row_range[0], row_range[1]) of `table`, default the whole
    table) -> (B,T,D); id < 0 / out of range -> zero row.  The gradient is the IndexedSlices (ids, d_out) as is."""
    B, T = ids.shape
    V, D = table.shape
    _chk(table, F32, "table"); _chk(ids, I64, "ids")
    if row_range is None:
        row_range = torch.tensor([0, V], dtype=I64, device=table.device)
    _chk(row_range, I64, "row_range", (2,))
    if out is None:
        out = torch.empty((B, T, D), dtype=F32, device=table.device)
    _chk(out, F32, "out", (B, T, D))
    _lib.check(_lib.lib().ctr_embed_seq_fwd(_ptr(table), _ptr(row_range), _ptr(ids), B, T, D, _ptr(out), _stream()))
    return out


def sigmoid_ce(logit_a: torch.Tensor, logit_b: Optional[torch.Tensor], labels: torch.Tensor, want_grad: bool = True):
    """Mean sigmoid cross-entropy of (logit_a + logit_b) vs labels and d(loss)/d(logit) in one launch: (loss (1,), d_logit (B,1))."""
    B = logit_a.numel()
    a = logit_a.reshape(B); b = None if logit_b is None else logit_b.reshape(B); y = labels.reshape(B)
    _chk(a, F32, "logit_a"); _chk(b, F32, "logit_b", (B,)); _chk(y, F32, "labels", (B,))
    loss = torch.empty((1,), dtype=F32, device=a.device)
    d = torch.empty((B, 1), dtype=F32, device=a.device) if want_grad else None
    _lib.check(_lib.lib().ctr_sigmoid_ce(_ptr(a), _ptr(b), _ptr(y), B, _ptr(loss), _ptr(d), _stream()))
    return loss, d


def embed_scatter_add(grad_table: torch.Tensor, field_row_offset: torch.Tensor, ids: torch.Tensor,
                      row_grads: torch.Tensor) -> torch.Tensor:
    B, F, D = row_grads.shape
    _chk(grad_table, F32, "grad_table"); _chk(field_row_offset, I64, "field_row_offset", (F + 1,))
    _chk(ids, I64, "ids", (B, F)); _chk(row_grads, F32, "row_grads")
    _lib.check(_lib.lib().ctr_embed_scatter_add(_ptr(grad_table), _ptr(field_row_offset), _ptr(ids), _ptr(row_grads),
                                                B, F, D, _stream()))
    return grad_table


def first_order_fwd(w: torch.Tensor, field_row_offset: torch.Tensor, ids: torch.Tensor, bias: float = 0.0) -> torch.Tensor:
    """DeepFM first-order logit (B,1): bias + sum_f w[row(b,f)].  w (V_total,) = the dense(1) kernel over the indicators."""
    B, F = ids.shape
    _chk(w, F32, "w"); _chk(field_row_offset, I64, "field_row_offset", (F + 1,)); _chk(ids, I64, "ids")
    out = torch.empty((B, 1), dtype=F32, device=w.device)
    _lib.check(_lib.lib().ctr_first_order_fwd(_ptr(w), _ptr(field_row_offset), _ptr(ids), B, F, float(bias), _ptr(out),
                                              _stream()))
    return out


CROSS_HASH_KEY = 0xDECAFCAFFE        # TF's default hash_key of crossed_column / sparse_cross_hashed


def crossed_indicator_fwd(values: torch.Tensor, offsets: torch.Tensor, num_buckets: int, kernel: torch.Tensor, bias: torch.Tensor,
                          hash_key: int = CROSS_HASH_KEY) -> torch.Tensor:
    """Wide logit (B,1) of one hashed crossed column: bias + sum over each sample's crosses of kernel[bucket].  values (nnz,)
    int64 ids of the K keys; offsets (K, B+1) int64 (key k of sample b = values[offsets[k,b]:offsets[k,b+1]]); kernel
    (num_buckets,); bias (1,) read on the device."""
    K, B = offsets.shape[0], offsets.shape[1] - 1
    _chk(values, I64, "values"); _chk(offsets, I64, "offsets"); _chk(kernel, F32, "kernel", (num_buckets,)); _chk(bias, F32, "bias", (1,))
    out = torch.empty((B, 1), dtype=F32, device=kernel.device)
    _lib.check(_lib.lib().ctr_crossed_indicator_fwd(_ptr(values), _ptr(offsets), K, B, num_buckets, hash_key, _ptr(kernel), _ptr(bias),
                                                    _ptr(out), _stream()))
    return out


def crossed_indicator_bwd(values: torch.Tensor, offsets: torch.Tensor, num_buckets: int, d_logit: torch.Tensor,
                          hash_key: int = CROSS_HASH_KEY, want_bias: bool = True):
    """Dense gradients of the wide logit: (d_kernel (num_buckets,), d_bias (1,) | None)."""
    K, B = offsets.shape[0], offsets.shape[1] - 1
    _chk(values, I64, "values"); _chk(offsets, I64, "offsets"); _chk(d_logit, F32, "d_logit")
    if d_logit.numel() != B:
        raise ValueError(f"d_logit: expected {B} elements, got {d_logit.numel()}")
    d_kernel = torch.empty((num_buckets,), dtype=F32, device=d_logit.device)
    d_bias = torch.empty((1,), dtype=F32, device=d_logit.device) if want_bias else None
    _lib.check(_lib.lib().ctr_crossed_indicator_bwd(_ptr(values), _ptr(offsets), K, B, num_buckets, hash_key, _ptr(d_logit),
                                                    _ptr(d_kernel), _ptr(d_bias), _stream()))
    return d_kernel, d_bias


def ftrl_apply(var: torch.Tensor, accum: torch.Tensor, linear: torch.Tensor, grad: torch.Tensor, lr: float, lr_power: float = -0.5,
               l1: float = 0.0, l2: float = 0.0) -> None:
    """TF's dense ApplyFtrl, in place on var, accum and linear (same shape as grad, contiguous)."""
    n = var.numel()
    for t, name in ((var, "var"), (accum, "accum"), (linear, "linear"), (grad, "grad")):
        _chk(t, F32, name, tuple(var.shape))
    _lib.check(_lib.lib().ctr_ftrl_apply(_ptr(var), _ptr(accum), _ptr(linear), _ptr(grad), n, float(lr), float(lr_power), float(l1),
                                         float(l2), _stream()))


def bag_lookup_fwd(table: torch.Tensor, ids: torch.Tensor, offsets: torch.Tensor,
                   out: Optional[torch.Tensor] = None, out_col: int = 0) -> torch.Tensor:
    """Multi-valued lookup, combiner='mean'.  Writes out[:, out_col:out_col+D] of a (B, stride) buffer."""
    V, D = table.shape
    B = offsets.numel() - 1
    _chk(table, F32, "table"); _chk(ids, I64, "ids"); _chk(offsets, I64, "offsets")
    if out is None:
        out = torch.empty((B, D), dtype=F32, device=table.device)
    _chk(out, F32, "out")
    stride = out.shape[1]
    if out_col + D > stride:
        raise ValueError("bag_lookup_fwd: field does not fit in the output row")
    _lib.check(_lib.lib().ctr_bag_lookup_fwd(_ptr(table), V, D, _ptr(ids), _ptr(offsets), B,
                                             out.data_ptr() + 4 * out_col, stride, _stream()))
    return out


def bag_lookup_bwd(d_out: torch.Tensor, out_col: int, V: int, D: int, ids: torch.Tensor,
                   offsets: torch.Tensor) -> torch.Tensor:
    B = offsets.numel() - 1
    _chk(d_out, F32, "d_out"); _chk(ids, I64, "ids"); _chk(offsets, I64, "offsets")
    row_grads = torch.empty((ids.numel(), D), dtype=F32, device=d_out.device)
    _lib.check(_lib.lib().ctr_bag_lookup_bwd(d_out.data_ptr() + 4 * out_col, d_out.shape[1], V, D, _ptr(ids),
                                             _ptr(offsets), B, _ptr(row_grads), _stream()))
    return row_grads


# ------------------------------------------------------------------ Row CROSS
def cross_fwd(x0: torch.Tensor, w: torch.Tensor, b: torch.Tensor, xl_in: Optional[torch.Tensor] = None,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x_L of the cross stack.  x0 (B,d); w, b (L,d); xl_in optional start vector (default x0)."""
    B, d = x0.shape
    L = w.shape[0]
    _chk(x0, F32, "x0"); _chk(w, F32, "w", (L, d)); _chk(b, F32, "b", (L, d)); _chk(xl_in, F32, "xl_in", (B, d))
    if out is None:
        out = torch.empty_like(x0)
    _chk(out, F32, "out", (B, d))
    _lib.check(_lib.lib().ctr_cross_fwd(_ptr(x0), _ptr(xl_in), _ptr(w), _ptr(b), B, d, L, _ptr(out), _stream()))
    return out


def embed_cross_supported(F: int, D: int, L: int) -> bool:
    """Shapes the fused lookup + cross forward covers (ctr_embed_cross_fwd): D % 4 == 0, F*D <= 512, L <= 4."""
    return D % 4 == 0 and F * D <= 512 and 1 <= L <= 4


def embed_cross_fwd(table: torch.Tensor, field_row_offset: torch.Tensor, ids: torch.Tensor, w: torch.Tensor, b: torch.Tensor,
                    x0: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Lookup fused with the cross stack (DCN/dcn.py:153-160): ids (B,F) i64 | i32 -> (x0 (B,F*D), x_L (B,F*D)) in one launch.
    Shapes outside embed_cross_supported() run the lookup kernel followed by the cross kernel (same results)."""
    B, F = ids.shape
    D = table.shape[1]
    d, L = F * D, w.shape[0]
    _chk(table, F32, "table"); _chk(field_row_offset, I64, "field_row_offset", (F + 1,))
    _chk(w, F32, "w", (L, d)); _chk(b, F32, "b", (L, d))
    if ids.dtype not in (I64, I32):
        raise TypeError(f"ids must be int64 or int32, got {ids.dtype}")
    _chk(ids, ids.dtype, "ids")
    if x0 is None:
        x0 = torch.empty((B, d), dtype=F32, device=table.device)
    if out is None:
        out = torch.empty((B, d), dtype=F32, device=table.device)
    _chk(x0, F32, "x0", (B, d)); _chk(out, F32, "out", (B, d))
    if not embed_cross_supported(F, D, L):
        if ids.dtype == I32:
            ids = ids.long()
        embed_fm2_fwd(table, field_row_offset, ids, want_fm2=False, tile=x0.view(B, F, D))
        return x0, cross_fwd(x0, w, b, out=out)
    _lib.check(_lib.lib().ctr_embed_cross_fwd(_ptr(table), _ptr(field_row_offset), _ptr(ids), int(ids.dtype == I32), B, F, D,
                                              _ptr(w), _ptr(b), L, _ptr(x0), _ptr(out), _stream()))
    return x0, out


def cross_bwd(x0, w, b, g_out, xl_in=None):
    """Returns (dx0, dxl_in | None, dw, db)."""
    B, d = x0.shape
    L = w.shape[0]
    _chk(x0, F32, "x0"); _chk(w, F32, "w", (L, d)); _chk(b, F32, "b", (L, d))
    _chk(g_out, F32, "g_out", (B, d)); _chk(xl_in, F32, "xl_in", (B, d))
    dx0 = torch.empty_like(x0)
    dxl = torch.empty_like(x0) if xl_in is not None else None
    dwb = torch.empty((2,) + tuple(w.shape), dtype=F32, device=w.device)     # dw | db back to back: zeroed by one memset
    dw, db = dwb[0], dwb[1]
    _lib.check(_lib.lib().ctr_cross_bwd(_ptr(x0), _ptr(xl_in), _ptr(w), _ptr(b), _ptr(g_out), B, d, L,
                                        _ptr(dx0), _ptr(dxl), _ptr(dw), _ptr(db), _stream()))
    return dx0, dxl, dw, db


# ------------------------------------------------------------------ Row DIN-ATT
def _din_params(H, w1, b1, w2, b2, w3, b3):
    w3 = w3.reshape(32)
    b3 = b3.reshape(1)
    for t, n, s in ((w1, "w1", (4 * H, 64)), (b1, "b1", (64,)), (w2, "w2", (64, 32)), (b2, "b2", (32,)),
                    (w3, "w3", (32,)), (b3, "b3", (1,))):
        _chk(t, F32, n, s)
    return w1, b1, w2, b2, w3, b3


_din_sched = {}


def _din_sched_scratch(B: int, device, balanced: bool):
    """int32[B + 64] schedule scratch of the DIN kernels (longest-first dynamic work distribution), cached per (device, stream):
    two streams running the attention at the same time must not share the sample list."""
    if not balanced or B == 0:
        return None
    key = (device, _stream())
    t = _din_sched.get(key)
    if t is None or t.numel() < B + 64:
        t = _din_sched[key] = torch.empty((B + 64,), dtype=torch.int32, device=device)
    return t


def din_attention_fwd(query, keys, keys_length, w1, b1, w2, b2, w3, b3, is_softmax=False, want_weights=False, balanced=True):
    """DIN attention unit.  query (B,H); keys (B,T,H); keys_length (B,) int64.  Returns out (B,H) [, att_w (B,T)].
    balanced: samples are handed to the warps longest-first from a shared counter instead of round-robin."""
    B, T, H = keys.shape
    _chk(query, F32, "query", (B, H)); _chk(keys, F32, "keys"); _chk(keys_length, I64, "keys_length", (B,))
    w1, b1, w2, b2, w3, b3 = _din_params(H, w1, b1, w2, b2, w3, b3)
    out = torch.empty((B, H), dtype=F32, device=query.device)
    att = torch.empty((B, T), dtype=F32, device=query.device) if want_weights else None
    _lib.check(_lib.lib().ctr_din_attention_fwd(_ptr(query), _ptr(keys) if T > 0 else None, _ptr(keys_length), _ptr(w1),
                                                _ptr(b1), _ptr(w2), _ptr(b2), _ptr(w3), _ptr(b3), B, T, H,
                                                int(bool(is_softmax)), _ptr(out), _ptr(att),
                                                _ptr(_din_sched_scratch(B, query.device, balanced)), _stream()))
    return (out, att) if want_weights else out


def din_attention_bwd(query, keys, keys_length, w1, b1, w2, b2, w3, b3, g_out, is_softmax=False, att_w=None, balanced=True):
    """Returns (d_query, d_keys, [dw1, db1, dw2, db2, dw3, db3]).  att_w: the forward's (B,T) weights (else recomputed)."""
    B, T, H = keys.shape
    _chk(query, F32, "query", (B, H)); _chk(keys, F32, "keys"); _chk(keys_length, I64, "keys_length", (B,))
    _chk(g_out, F32, "g_out", (B, H)); _chk(att_w, F32, "att_w", (B, T))
    w3_shape, b3_shape = w3.shape, b3.shape
    w1, b1, w2, b2, w3, b3 = _din_params(H, w1, b1, w2, b2, w3, b3)
    dq = torch.empty_like(query)
    dk = torch.empty_like(keys)
    sizes = [4 * H * 64, 64, 64 * 32, 32, 32, 1]
    flat = torch.empty((sum(sizes),), dtype=F32, device=query.device)
    _lib.check(_lib.lib().ctr_din_attention_bwd(_ptr(query), _ptr(keys) if T > 0 else None, _ptr(keys_length), _ptr(w1),
                                                _ptr(b1), _ptr(w2), _ptr(b2), _ptr(w3), _ptr(b3), _ptr(g_out), _ptr(att_w), B, T, H,
                                                int(bool(is_softmax)), _ptr(dq), _ptr(dk) if T > 0 else None, _ptr(flat),
                                                _ptr(_din_sched_scratch(B, query.device, balanced)), _stream()))
    parts = list(torch.split(flat, sizes))
    shapes = [(4 * H, 64), (64,), (64, 32), (32,), tuple(w3_shape), tuple(b3_shape)]
    return dq, dk, [p.reshape(s) for p, s in zip(parts, shapes)]


# ------------------------------------------------------------------ Rows SENET / BILINEAR
def senet_fwd(x, w1, w2):
    B, F, K = x.shape
    r = w1.shape[1]
    _chk(x, F32, "x"); _chk(w1, F32, "w1", (F, r)); _chk(w2, F32, "w2", (r, F))
    out = torch.empty_like(x)
    _lib.check(_lib.lib().ctr_senet_fwd(_ptr(x), _ptr(w1), _ptr(w2), B, F, K, r, _ptr(out), _stream()))
    return out


def senet_bwd(x, w1, w2, g_out):
    B, F, K = x.shape
    r = w1.shape[1]
    _chk(x, F32, "x"); _chk(w1, F32, "w1", (F, r)); _chk(w2, F32, "w2", (r, F)); _chk(g_out, F32, "g_out", (B, F, K))
    dx, dw1, dw2 = torch.empty_like(x), torch.empty_like(w1), torch.empty_like(w2)
    _lib.check(_lib.lib().ctr_senet_bwd(_ptr(x), _ptr(w1), _ptr(w2), _ptr(g_out), B, F, K, r, _ptr(dx), _ptr(dw1),
                                        _ptr(dw2), _stream()))
    return dx, dw1, dw2


BILINEAR_TYPES = {"all": 0, "each": 1, "interaction": 2}


def _bilinear_type(type_):
    if type_ not in BILINEAR_TYPES:      # same message as FiBiNET/bilinear_interaction_layer.py:36-38
        raise ValueError(f"Bilinear Interaction type must be in ['all','each','interaction'], got '{type_}'")
    return BILINEAR_TYPES[type_]


def bilinear_w_shape(F, K, type_):
    return {"all": (K, K), "each": (F - 1, K, K), "interaction": (F * (F - 1) // 2, K, K)}[type_]


def bilinear_set_tournament(mask):
    """Tuning hook (see ctr_bilinear_set_rr in include/ctr_b200.h): bits 0..2 route type 'all' / 'each' / 'interaction' through
    the sample-batched tournament kernels (default 4: 'interaction' only; 'all' / 'each' run the staged per-sample kernels),
    bit 3 selects the round-1 kernels for 'all' / 'each'.  Returns the previous mask."""
    return int(_lib.lib().ctr_bilinear_set_rr(int(mask)))


def bilinear_fwd(x, w, type_):
    t = _bilinear_type(type_)
    B, F, K = x.shape
    _chk(x, F32, "x"); _chk(w, F32, "w", bilinear_w_shape(F, K, type_))
    P = (F - 1) * (F - 2) // 2
    out = torch.empty((B, P, K), dtype=F32, device=x.device)
    if B == 0 or P == 0:
        return out
    _lib.check(_lib.lib().ctr_bilinear_fwd(_ptr(x), _ptr(w), B, F, K, t, _ptr(out), _stream()))
    return out


def bilinear_bwd(x, w, type_, g_out):
    t = _bilinear_type(type_)
    B, F, K = x.shape
    P = (F - 1) * (F - 2) // 2
    _chk(x, F32, "x"); _chk(w, F32, "w", bilinear_w_shape(F, K, type_)); _chk(g_out, F32, "g_out", (B, P, K))
    dx, dw = torch.empty_like(x), torch.empty_like(w)
    if B == 0 or P == 0:
        return dx.zero_(), dw.zero_()
    _lib.check(_lib.lib().ctr_bilinear_bwd(_ptr(x), _ptr(w), _ptr(g_out), B, F, K, t, _ptr(dx), _ptr(dw), _stream()))
    return dx, dw


# ------------------------------------------------------------------ Row CIN
_cin_ws = {}


def _cin_workspace(nbytes: int, device) -> Optional[torch.Tensor]:
    """Per-(device, stream) cached scratch for the re-ordered / tf32-split filter (caller-owned, as the ABI requires)."""
    if nbytes == 0:
        return None
    key = (device.index, _stream())
    buf = _cin_ws.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty((nbytes,), dtype=torch.uint8, device=device)
        _cin_ws[key] = buf
    return buf


def cin_fwd(x0: torch.Tensor, xk: torch.Tensor, filt: torch.Tensor, want_pooled: bool = False, precision: int = 0):
    """One CIN layer.  x0 (B,m,D); xk (B,hk,D); filt (hk*m, H).  Returns out (B,H,D) [, pooled (B,H)]."""
    B, m, D = x0.shape
    hk = xk.shape[1]
    H = filt.shape[1]
    _chk(x0, F32, "x0"); _chk(xk, F32, "xk", (B, hk, D)); _chk(filt, F32, "filter", (hk * m, H))
    out = torch.empty((B, H, D), dtype=F32, device=x0.device)
    pooled = torch.empty((B, H), dtype=F32, device=x0.device) if want_pooled else None
    L = _lib.lib()
    nbytes = int(L.ctr_cin_fwd_workspace_bytes(B, m, hk, D, H))
    ws = _cin_workspace(nbytes, x0.device)
    _lib.check(L.ctr_cin_fwd(_ptr(x0), _ptr(xk), _ptr(filt), B, m, hk, D, H, _ptr(out), _ptr(pooled), int(precision),
                             _ptr(ws), nbytes, _stream()))
    return (out, pooled) if want_pooled else out


def cin_bwd(x0, xk, filt, g_out):
    """Returns (dx0, dxk, dfilter)."""
    B, m, D = x0.shape
    hk = xk.shape[1]
    H = filt.shape[1]
    _chk(x0, F32, "x0"); _chk(xk, F32, "xk", (B, hk, D)); _chk(filt, F32, "filter", (hk * m, H))
    _chk(g_out, F32, "g_out", (B, H, D))
    dx0, dxk, dw = torch.empty_like(x0), torch.empty_like(xk), torch.empty_like(filt)
    L = _lib.lib()
    nbytes = int(L.ctr_cin_bwd_workspace_bytes(B, m, hk, D, H))
    ws = _cin_workspace(nbytes, x0.device)
    _lib.check(L.ctr_cin_bwd(_ptr(x0), _ptr(xk), _ptr(filt), _ptr(g_out), B, m, hk, D, H, _ptr(dx0), _ptr(dxk), _ptr(dw),
                             _ptr(ws), nbytes, _stream()))
    return dx0, dxk, dw


# ------------------------------------------------------------------------------------ SURVEY 8f.4: FM2 siblings
def embed_bi_fwd(table: torch.Tensor, field_row_offset: torch.Tensor, ids: torch.Tensor, want_tile: bool = True):
    """Fused lookup + NFM bi-interaction pooling.  Returns (tile (B,F,D) | None, bi (B,D))."""
    B, F = ids.shape
    D = table.shape[1]
    _chk(table, F32, "table"); _chk(field_row_offset, I64, "field_row_offset", (F + 1,)); _chk(ids, I64, "ids")
    tile = torch.empty((B, F, D), dtype=F32, device=table.device) if want_tile else None
    bi = torch.empty((B, D), dtype=F32, device=table.device)
    _lib.check(_lib.lib().ctr_embed_bi_fwd(_ptr(table), _ptr(field_row_offset), _ptr(ids), B, F, D, _ptr(tile), _ptr(bi), _stream()))
    return tile, bi


def embed_bi_bwd(tile: torch.Tensor, d_tile: Optional[torch.Tensor], d_bi: torch.Tensor) -> torch.Tensor:
    """IndexedSlices values (B,F,D): d_tile + d_bi[b,:] * (S - e)."""
    B, F, D = tile.shape
    _chk(tile, F32, "tile"); _chk(d_tile, F32, "d_tile", (B, F, D)); _chk(d_bi, F32, "d_bi", (B, D))
    row_grads = torch.empty_like(tile)
    _lib.check(_lib.lib().ctr_embed_bi_bwd(_ptr(tile), _ptr(d_tile), _ptr(d_bi), B, F, D, _ptr(row_grads), _stream()))
    return row_grads


def _fwbi_args(field_group, F: int, D: int, kernel_mf, kernel_fm, bias_mf=None, bias_fm=None):
    """The host int32 group map (kept alive by the caller while the entry reads it) and M = len(kernel_fm)."""
    M = int(kernel_fm.shape[0]) if kernel_fm.dim() == 1 else -1
    _chk(kernel_fm, F32, "kernel_fm", (M,)); _chk(kernel_mf, F32, "kernel_mf", (M * (M - 1) // 2,))
    _chk(bias_mf, F32, "bias_mf", (D,)); _chk(bias_fm, F32, "bias_fm", (D,))
    groups = [int(g) for g in (field_group.tolist() if torch.is_tensor(field_group) else field_group)]
    if len(groups) != F:
        raise ValueError(f"field_group: expected {F} entries (one per field), got {len(groups)}")
    arr = (ctypes.c_int32 * F)(*groups)
    return arr, M


def embed_fwbi_fwd(table: torch.Tensor, field_row_offset: torch.Tensor, ids: torch.Tensor, field_group, kernel_mf: torch.Tensor,
                   kernel_fm: torch.Tensor, bias_mf: torch.Tensor, bias_fm: torch.Tensor, want_tile: bool = True,
                   ids64_out: Optional[torch.Tensor] = None):
    """Fused lookup + FLEN field-wise bi-interaction.  ids (B,F) int64, or int32 (``ids64_out`` (B,F) i64 then receives the
    widened copy); field_group: F group indices in [0, M), M = len(kernel_fm); kernel_mf (M(M-1)/2,).
    Returns (tile (B,F,D) | None, h (B,D))."""
    B, F = ids.shape
    D = table.shape[1]
    _chk(table, F32, "table"); _chk(field_row_offset, I64, "field_row_offset", (F + 1,))
    i32 = ids.dtype == I32
    _chk(ids, I32 if i32 else I64, "ids"); _chk(ids64_out, I64, "ids64_out", (B, F))
    groups, M = _fwbi_args(field_group, F, D, kernel_mf, kernel_fm, bias_mf, bias_fm)
    tile = torch.empty((B, F, D), dtype=F32, device=table.device) if want_tile else None
    h = torch.empty((B, D), dtype=F32, device=table.device)
    _lib.check(_lib.lib().ctr_embed_fwbi_fwd(_ptr(table), _ptr(field_row_offset), _ptr(ids), int(i32), B, F, D,
                                             ctypes.addressof(groups), M, _ptr(kernel_mf), _ptr(kernel_fm), _ptr(bias_mf),
                                             _ptr(bias_fm), _ptr(tile), _ptr(h), _ptr(ids64_out), _stream()))
    return tile, h


def fwbi_fwd(tile: torch.Tensor, field_group, kernel_mf: torch.Tensor, kernel_fm: torch.Tensor, bias_mf: torch.Tensor,
             bias_fm: torch.Tensor) -> torch.Tensor:
    """FLEN field-wise bi-interaction of a (B,F,D) tile -> h (B,D) (see embed_fwbi_fwd)."""
    _chk(tile, F32, "tile")
    B, F, D = tile.shape
    groups, M = _fwbi_args(field_group, F, D, kernel_mf, kernel_fm, bias_mf, bias_fm)
    h = torch.empty((B, D), dtype=F32, device=tile.device)
    _lib.check(_lib.lib().ctr_fwbi_fwd(_ptr(tile), B, F, D, ctypes.addressof(groups), M, _ptr(kernel_mf), _ptr(kernel_fm),
                                       _ptr(bias_mf), _ptr(bias_fm), _ptr(h), _stream()))
    return h


def fwbi_bwd(tile: torch.Tensor, d_tile: Optional[torch.Tensor], d_h: torch.Tensor, field_group, kernel_mf: torch.Tensor,
             kernel_fm: torch.Tensor):
    """Backward of both FwBI forms: (row_grads (B,F,D) = d_tile + the layer's term -- the IndexedSlices values of the fused
    form --, d_kernel_mf, d_kernel_fm, d_bias_mf, d_bias_fm)."""
    _chk(tile, F32, "tile")
    B, F, D = tile.shape
    _chk(d_tile, F32, "d_tile", (B, F, D)); _chk(d_h, F32, "d_h", (B, D))
    groups, M = _fwbi_args(field_group, F, D, kernel_mf, kernel_fm)
    row_grads = torch.empty_like(tile)
    d_kmf, d_kfm = torch.empty_like(kernel_mf), torch.empty_like(kernel_fm)
    d_bmf, d_bfm = (torch.empty((D,), dtype=F32, device=tile.device) for _ in range(2))
    _lib.check(_lib.lib().ctr_fwbi_bwd(_ptr(tile), _ptr(d_tile), _ptr(d_h), B, F, D, ctypes.addressof(groups), M, _ptr(kernel_mf),
                                       _ptr(kernel_fm), _ptr(row_grads), _ptr(d_kmf), _ptr(d_kfm), _ptr(d_bmf), _ptr(d_bfm),
                                       _stream()))
    return row_grads, d_kmf, d_kfm, d_bmf, d_bfm


def fwfm_fwd(tile: torch.Tensor, r: torch.Tensor) -> torch.Tensor:
    """FwFM second-order logit (B,1).  tile (B,F,K); r (F(F-1)/2,) pair strengths in utils.index_from_upper_triangular order."""
    B, F, K = tile.shape
    _chk(tile, F32, "tile"); _chk(r, F32, "r", (F * (F - 1) // 2,))
    out = torch.empty((B, 1), dtype=F32, device=tile.device)
    _lib.check(_lib.lib().ctr_fwfm_fwd(_ptr(tile), _ptr(r), B, F, K, _ptr(out), _stream()))
    return out


def fwfm_bwd(tile: torch.Tensor, r: torch.Tensor, g: torch.Tensor):
    B, F, K = tile.shape
    g = g.reshape(B)
    _chk(tile, F32, "tile"); _chk(r, F32, "r", (F * (F - 1) // 2,)); _chk(g, F32, "g", (B,))
    d_tile, d_r = torch.empty_like(tile), torch.empty_like(r)
    _lib.check(_lib.lib().ctr_fwfm_bwd(_ptr(tile), _ptr(r), _ptr(g), B, F, K, _ptr(d_tile), _ptr(d_r), _stream()))
    return d_tile, d_r


def afm_fwd(tile: torch.Tensor, w: torch.Tensor, b: torch.Tensor, h: torch.Tensor, want_score: bool = False):
    """AFM attention pooling (B,K) (+ the (B,P) softmax scores).  w (K,T), b (T,), h (T,1) or (T,)."""
    B, F, K = tile.shape
    T = w.shape[1]
    h = h.reshape(T)
    _chk(tile, F32, "tile"); _chk(w, F32, "w", (K, T)); _chk(b, F32, "b", (T,)); _chk(h, F32, "h", (T,))
    pooled = torch.empty((B, K), dtype=F32, device=tile.device)
    score = torch.empty((B, F * (F - 1) // 2), dtype=F32, device=tile.device) if want_score else None
    _lib.check(_lib.lib().ctr_afm_fwd(_ptr(tile), _ptr(w), _ptr(b), _ptr(h), B, F, K, T, _ptr(pooled), _ptr(score), _stream()))
    return (pooled, score) if want_score else pooled


def afm_bwd(tile, w, b, h, g_pooled):
    B, F, K = tile.shape
    T = w.shape[1]
    h_shape = h.shape
    h = h.reshape(T)
    _chk(tile, F32, "tile"); _chk(w, F32, "w", (K, T)); _chk(b, F32, "b", (T,)); _chk(h, F32, "h", (T,)); _chk(g_pooled, F32, "g_pooled", (B, K))
    d_tile, d_w, d_b, d_h = torch.empty_like(tile), torch.empty_like(w), torch.empty_like(b), torch.empty_like(h)
    _lib.check(_lib.lib().ctr_afm_bwd(_ptr(tile), _ptr(w), _ptr(b), _ptr(h), _ptr(g_pooled), B, F, K, T, _ptr(d_tile), _ptr(d_w),
                                      _ptr(d_b), _ptr(d_h), _stream()))
    return d_tile, d_w, d_b, d_h.reshape(h_shape)


# ------------------------------------------------------------------------------------ SURVEY 8f.4: BST transformer block
BST_PARAM_ORDER = ("position_embedding", "w_q", "w_k", "w_v", "w_o", "ln1_beta", "ln1_gamma", "dense_kernel", "dense_bias",
                   "ln2_beta", "ln2_gamma")


def bst_param_shapes(d: int, heads: int, max_length: int):
    return {"position_embedding": (max_length, d), "w_q": (heads, d, d), "w_k": (heads, d, d), "w_v": (heads, d, d),
            "w_o": (heads * d, d), "ln1_beta": (d,), "ln1_gamma": (d,), "dense_kernel": (d, d), "dense_bias": (d,),
            "ln2_beta": (d,), "ln2_gamma": (d,)}


def bst_pack_params(params: dict, d: int, heads: int, max_length: int) -> torch.Tensor:
    """dict of named tensors -> the packed float buffer of ctr_bst_transformer_* (include/ctr_b200.h)."""
    shapes = bst_param_shapes(d, heads, max_length)
    parts = []
    for name in BST_PARAM_ORDER:
        t = params[name]
        if tuple(t.shape) != shapes[name]:
            raise ValueError(f"{name}: expected shape {shapes[name]}, got {tuple(t.shape)}")
        parts.append(t.reshape(-1))
    packed = torch.cat(parts).contiguous()
    assert packed.numel() == _lib.lib().ctr_bst_param_count(d, heads, max_length)
    return packed


def bst_unpack_params(packed: torch.Tensor, d: int, heads: int, max_length: int) -> dict:
    out, o = {}, 0
    for name, shp in bst_param_shapes(d, heads, max_length).items():
        n = 1
        for x in shp:
            n *= x
        out[name] = packed[o:o + n].reshape(shp)
        o += n
    return out


def _bst_args(queries, keys, values, keys_length, packed, heads, max_length):
    B, T, d = queries.shape
    _chk(queries, F32, "queries"); _chk(keys, F32, "keys", (B, T, d)); _chk(values, F32, "values", (B, T, d))
    _chk(keys_length, I64, "keys_length", (B,))
    _chk(packed, F32, "params", (int(_lib.lib().ctr_bst_param_count(d, heads, max_length)),))
    return B, T, d


def bst_transformer_fwd(queries, keys, values, keys_length, packed, heads: int, max_length: int, use_position_embedding: bool = True):
    B, T, d = _bst_args(queries, keys, values, keys_length, packed, heads, max_length)
    out = torch.empty_like(queries)
    _lib.check(_lib.lib().ctr_bst_transformer_fwd(_ptr(queries), _ptr(keys), _ptr(values), _ptr(keys_length), _ptr(packed), B, T, d,
                                                  heads, max_length, int(use_position_embedding), _ptr(out), _stream()))
    return out


def bst_transformer_bwd(queries, keys, values, keys_length, packed, g_out, heads: int, max_length: int,
                        use_position_embedding: bool = True):
    B, T, d = _bst_args(queries, keys, values, keys_length, packed, heads, max_length)
    _chk(g_out, F32, "g_out", (B, T, d))
    dq, dk, dv, dp = torch.empty_like(queries), torch.empty_like(queries), torch.empty_like(queries), torch.empty_like(packed)
    _lib.check(_lib.lib().ctr_bst_transformer_bwd(_ptr(queries), _ptr(keys), _ptr(values), _ptr(keys_length), _ptr(packed),
                                                  _ptr(g_out), B, T, d, heads, max_length, int(use_position_embedding), _ptr(dq),
                                                  _ptr(dk), _ptr(dv), _ptr(dp), _stream()))
    return dq, dk, dv, dp


def ffm_fwd(tile: torch.Tensor) -> torch.Tensor:
    """FFM second-order logit (B,1) from the (B, F, F-1, K) field/slot tile (see include/ctr_b200.h)."""
    B, F, S, K = tile.shape
    if S != F - 1:
        raise ValueError(f"tile: expected shape (B, F, F-1, K), got {tuple(tile.shape)}")
    _chk(tile, F32, "tile")
    out = torch.empty((B, 1), dtype=F32, device=tile.device)
    _lib.check(_lib.lib().ctr_ffm_fwd(_ptr(tile), B, F, K, _ptr(out), _stream()))
    return out


def ffm_bwd(tile: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
    B, F, S, K = tile.shape
    g = g.reshape(B)
    _chk(tile, F32, "tile"); _chk(g, F32, "g", (B,))
    d_tile = torch.empty_like(tile)
    _lib.check(_lib.lib().ctr_ffm_bwd(_ptr(tile), _ptr(g), B, F, K, _ptr(d_tile), _stream()))
    return d_tile


# ------------------------------------------------------------------------------------ PNN product layer
PNN_METHODS = {"IPNN": 0, "OPNN": 1}


def pnn_wprod_shape(F: int, K: int, N: int, method: int):
    """Shape of the product weight: inner_product_w theta (N,F) for IPNN (0), outer_product_w (N,K,K) for OPNN (1)."""
    return (N, F) if method == 0 else (N, K, K)


def _pnn_args(e, wlin, wprod, method):
    if method not in (0, 1):
        raise ValueError(f"method must be 0 (IPNN) or 1 (OPNN), got {method!r}")
    B, F, K = e.shape
    N = wlin.shape[1]
    _chk(e, F32, "e"); _chk(wlin, F32, "wlin", (F * K, N)); _chk(wprod, F32, "wprod", pnn_wprod_shape(F, K, N, method))
    return B, F, K, N


def _pnn_workspace(F, K, N, method, device):
    nbytes = ctypes.c_int64(0)
    _lib.check(_lib.lib().ctr_pnn_workspace_bytes(F, K, N, method, ctypes.byref(nbytes)))
    return _cin_workspace(int(nbytes.value), device), int(nbytes.value)


def pnn_fwd(e: torch.Tensor, wlin: torch.Tensor, wprod: torch.Tensor, bias: torch.Tensor, method: int) -> torch.Tensor:
    """PNN product layer (PNN/pnn.py:125-181): e (B,F,K) field embeddings, wlin (F*K,N), wprod (N,F) | (N,K,K), bias (N,)
    -> product_final = relu(lz + lp + bias) (B,N).  method 0 = IPNN, 1 = OPNN."""
    B, F, K, N = _pnn_args(e, wlin, wprod, method)
    _chk(bias, F32, "bias", (N,))
    out = torch.empty((B, N), dtype=F32, device=e.device)
    ws, nbytes = _pnn_workspace(F, K, N, method, e.device)
    _lib.check(_lib.lib().ctr_pnn_fwd(_ptr(e), _ptr(wlin), _ptr(wprod), _ptr(bias), B, F, K, N, method, _ptr(out), _ptr(ws),
                                      nbytes, _stream()))
    return out


def pnn_bwd(e, wlin, wprod, out, g_out, method: int):
    """Gradients of pnn_fwd given its output `out` (the relu mask) and g_out (B,N): (d_e (B,F,K), d_wlin, d_wprod, d_bias)."""
    B, F, K, N = _pnn_args(e, wlin, wprod, method)
    _chk(out, F32, "out", (B, N)); _chk(g_out, F32, "g_out", (B, N))
    d_e, d_wlin, d_wprod = torch.empty_like(e), torch.empty_like(wlin), torch.empty_like(wprod)
    d_bias = torch.empty((N,), dtype=F32, device=e.device)
    ws, nbytes = _pnn_workspace(F, K, N, method, e.device)
    _lib.check(_lib.lib().ctr_pnn_bwd(_ptr(e), _ptr(wlin), _ptr(wprod), _ptr(out), _ptr(g_out), B, F, K, N, method, _ptr(d_e),
                                      _ptr(d_wlin), _ptr(d_wprod), _ptr(d_bias), _ptr(ws), nbytes, _stream()))
    return d_e, d_wlin, d_wprod, d_bias


# ------------------------------------------------------------------------------------ DIEN interest extractor + evolution
DIEN_CELLS = {"AGRU": 0, "AUGRU": 1}
# the nine variables in the packed order of include/ctr_b200.h (names relative to the caller's seq_encoder scope)
DIEN_PARAM_ORDER = ("rnn/gru_cell/gates/kernel", "rnn/gru_cell/gates/bias", "rnn/gru_cell/candidate/kernel",
                    "rnn/gru_cell/candidate/bias", "attention_project_matrix", "rnn/gates/kernel", "rnn/gates/bias",
                    "rnn/candidate/kernel", "rnn/candidate/bias")


def dien_param_shapes(na: int, nh: int):
    """Shapes of DIEN_PARAM_ORDER for input width na and gru_output_units nh."""
    return ((na + nh, 2 * nh), (2 * nh,), (na + nh, nh), (nh,), (nh, na), (2 * nh, 2 * nh), (2 * nh,), (2 * nh, nh), (nh,))


def dien_pack_params(params, na: int, nh: int) -> torch.Tensor:
    """The nine variables (DIEN_PARAM_ORDER) -> one packed fp32 buffer."""
    for p, s, n in zip(params, dien_param_shapes(na, nh), DIEN_PARAM_ORDER):
        if tuple(p.shape) != s:
            raise ValueError(f"{n}: expected shape {s}, got {tuple(p.shape)}")
    return torch.cat([p.reshape(-1) for p in params]).contiguous()


def dien_unpack_params(packed: torch.Tensor, na: int, nh: int):
    out, o = [], 0
    for s in dien_param_shapes(na, nh):
        n = 1
        for d in s:
            n *= d
        out.append(packed[o:o + n].view(s))
        o += n
    return out


def _dien_args(seq, seq_len, target, packed, nh, cell):
    if cell not in (0, 1):
        raise ValueError(f"cell must be 0 (AGRU) or 1 (AUGRU), got {cell!r}")
    B, T, na = seq.shape
    _chk(seq, F32, "sequnence_input"); _chk(seq_len, I64, "sequnence_length", (B,)); _chk(target, F32, "target_input", (B, na))
    _chk(packed, F32, "params", (sum(math.prod(s) for s in dien_param_shapes(na, nh)),))
    return B, T, na


def dien_workspace(B: int, T: int, na: int, nh: int, device) -> torch.Tensor:
    """The caller-owned workspace of one forward / backward pair (the forward's states and attention weights live there)."""
    nbytes = ctypes.c_int64(0)
    _lib.check(_lib.lib().ctr_dien_workspace_bytes(B, T, na, nh, ctypes.byref(nbytes)))
    return torch.empty((int(nbytes.value),), dtype=torch.uint8, device=device)


def dien_fwd(seq, seq_len, target, packed, nh: int, cell: int):
    """DIEN/dien.py:198-229: (final_state (B,nh), attention scores (B,T), workspace for dien_bwd)."""
    B, T, na = _dien_args(seq, seq_len, target, packed, nh, cell)
    final = torch.empty((B, nh), dtype=F32, device=seq.device)
    scores = torch.empty((B, T), dtype=F32, device=seq.device)
    ws = dien_workspace(B, T, na, nh, seq.device)
    _lib.check(_lib.lib().ctr_dien_fwd(_ptr(seq), _ptr(seq_len), _ptr(target), _ptr(packed), B, T, na, nh, cell, _ptr(final),
                                       _ptr(scores), _ptr(ws), ws.numel(), _stream()))
    return final, scores, ws


def dien_bwd(seq, seq_len, target, packed, g_final, nh: int, cell: int, ws):
    """Gradients of dien_fwd given d final_state (B,nh) and the forward's workspace: (d_seq (B,T,na), d_target (B,na),
    d_packed)."""
    B, T, na = _dien_args(seq, seq_len, target, packed, nh, cell)
    _chk(g_final, F32, "g_final_state", (B, nh))
    d_seq, d_tgt, d_p = torch.empty_like(seq), torch.empty_like(target), torch.empty_like(packed)
    _lib.check(_lib.lib().ctr_dien_bwd(_ptr(seq), _ptr(seq_len), _ptr(target), _ptr(packed), _ptr(g_final), B, T, na, nh, cell,
                                       _ptr(d_seq), _ptr(d_tgt), _ptr(d_p), _ptr(ws), ws.numel(), _stream()))
    return d_seq, d_tgt, d_p


def _dien_aux_args(seq, neg_seq, w_aux, nh, T_neg):
    B, T, na = seq.shape
    if int(T_neg) < 1:
        raise ValueError(f"negative_sample_number must be >= 1, got {T_neg!r}")
    _chk(neg_seq, F32, "neg_sequnence_input", (B, (T - 1) * int(T_neg), na))
    _chk(w_aux, F32, "aux_project_matrix", (na, nh))


def dien_aux_workspace(B: int, T: int, na: int, nh: int, T_neg: int, device) -> torch.Tensor:
    """One workspace for dien_fwd, dien_aux_fwd and dien_bwd_aux: the DIEN workspace plus per-sample partials."""
    nbytes = ctypes.c_int64(0)
    _lib.check(_lib.lib().ctr_dien_aux_workspace_bytes(B, T, na, nh, T_neg, ctypes.byref(nbytes)))
    return torch.empty((int(nbytes.value),), dtype=torch.uint8, device=device)


def dien_fwd_aux(seq, seq_len, target, neg_seq, packed, w_aux, nh: int, cell: int, T_neg: int):
    """DIEN/dien.py:198-229 and the auxiliary loss :256-300 with the paper's sign: (final_state (B,nh), attention scores
    (B,T), aux_loss (), workspace for dien_bwd_aux)."""
    B, T, na = _dien_args(seq, seq_len, target, packed, nh, cell)
    _dien_aux_args(seq, neg_seq, w_aux, nh, T_neg)
    final = torch.empty((B, nh), dtype=F32, device=seq.device)
    scores = torch.empty((B, T), dtype=F32, device=seq.device)
    ws = dien_aux_workspace(B, T, na, nh, T_neg, seq.device)
    _lib.check(_lib.lib().ctr_dien_fwd(_ptr(seq), _ptr(seq_len), _ptr(target), _ptr(packed), B, T, na, nh, cell, _ptr(final),
                                       _ptr(scores), _ptr(ws), ws.numel(), _stream()))
    aux = dien_aux_fwd(seq, neg_seq, seq_len, w_aux, nh, T_neg, ws)
    return final, scores, aux, ws


def dien_aux_fwd(seq, neg_seq, seq_len, w_aux, nh: int, T_neg: int, ws):
    """The auxiliary loss () of the states dien_fwd_aux (or ctr_dien_fwd on this dien_aux_workspace) left in ws."""
    B, T, na = seq.shape
    _chk(seq, F32, "sequnence_input"); _chk(seq_len, I64, "sequnence_length", (B,))
    _dien_aux_args(seq, neg_seq, w_aux, nh, T_neg)
    aux = torch.empty((), dtype=F32, device=seq.device)
    _lib.check(_lib.lib().ctr_dien_aux_fwd(_ptr(seq), _ptr(neg_seq), _ptr(seq_len), _ptr(w_aux), B, T, na, nh, int(T_neg),
                                           _ptr(aux), _ptr(ws), ws.numel(), _stream()))
    return aux


def dien_bwd_aux(seq, seq_len, target, neg_seq, packed, w_aux, g_final, g_aux, nh: int, cell: int, T_neg: int, ws):
    """Gradients of dien_fwd_aux given d final_state (B,nh) and d aux_loss (a device scalar): (d_seq (B,T,na), d_neg_seq,
    d_target (B,na), d_packed, d_w_aux (na,nh))."""
    B, T, na = _dien_args(seq, seq_len, target, packed, nh, cell)
    _dien_aux_args(seq, neg_seq, w_aux, nh, T_neg)
    _chk(g_final, F32, "g_final_state", (B, nh))
    _chk(g_aux, F32, "g_aux_loss", ())
    d_seq, d_neg, d_tgt = torch.empty_like(seq), torch.empty_like(neg_seq), torch.empty_like(target)
    d_p, d_w = torch.empty_like(packed), torch.empty_like(w_aux)
    _lib.check(_lib.lib().ctr_dien_bwd_aux(_ptr(seq), _ptr(neg_seq), _ptr(seq_len), _ptr(target), _ptr(packed), _ptr(w_aux),
                                           _ptr(g_final), _ptr(g_aux), B, T, na, nh, int(T_neg), cell, _ptr(d_seq), _ptr(d_neg),
                                           _ptr(d_tgt), _ptr(d_p), _ptr(d_w), _ptr(ws), ws.numel(), _stream()))
    return d_seq, d_neg, d_tgt, d_p, d_w


# ------------------------------------------------------------------------------------ DeepCrossing residual unit
def residual_unit_workspace(B: int, d: int, H: int, device) -> torch.Tensor:
    """Caller-owned workspace: the prepped weights (B = 0, what the forward needs) plus, for the backward, h and its gradient."""
    nbytes = ctypes.c_int64(0)
    _lib.check(_lib.lib().ctr_residual_unit_workspace_bytes(B, d, H, ctypes.byref(nbytes)))
    return torch.empty((int(nbytes.value),), dtype=torch.uint8, device=device)


def _residual_unit_args(x, w0, b0, w1, b1):
    B, d = x.shape
    H = w0.shape[1]
    _chk(x, F32, "input"); _chk(w0, F32, "w0", (d, H)); _chk(b0, F32, "b0", (H,)); _chk(w1, F32, "w1", (H, d))
    _chk(b1, F32, "b1", (d,))
    return B, d, H


def residual_unit_fwd(x, w0, b0, w1, b1) -> torch.Tensor:
    """DeepCrossing/residual_unit.py:4-21: relu(x + relu(x . w0 + b0) . w1 + b1), x (B,d), w0 (d,H), w1 (H,d) -> (B,d)."""
    B, d, H = _residual_unit_args(x, w0, b0, w1, b1)
    out = torch.empty((B, d), dtype=F32, device=x.device)
    ws = residual_unit_workspace(0, d, H, x.device)
    _lib.check(_lib.lib().ctr_residual_unit_fwd(_ptr(x), _ptr(w0), _ptr(b0), _ptr(w1), _ptr(b1), B, d, H, _ptr(out), _ptr(ws),
                                                ws.numel(), _stream()))
    return out


def residual_unit_bwd(x, w0, b0, w1, b1, out, g_out):
    """Gradients of residual_unit_fwd given its output `out` (the relu mask) and g_out (B,d): (d_x, d_w0, d_b0, d_w1, d_b1).
    The hidden activation is recomputed from x."""
    B, d, H = _residual_unit_args(x, w0, b0, w1, b1)
    _chk(out, F32, "out", (B, d)); _chk(g_out, F32, "g_out", (B, d))
    d_x, d_w0, d_b0, d_w1, d_b1 = (torch.empty_like(t) for t in (x, w0, b0, w1, b1))
    ws = residual_unit_workspace(B, d, H, x.device)
    _lib.check(_lib.lib().ctr_residual_unit_bwd(_ptr(x), _ptr(w0), _ptr(b0), _ptr(w1), _ptr(b1), _ptr(out), _ptr(g_out), B, d,
                                                H, _ptr(d_x), _ptr(d_w0), _ptr(d_b0), _ptr(d_w1), _ptr(d_b1), _ptr(ws),
                                                ws.numel(), _stream()))
    return d_x, d_w0, d_b0, d_w1, d_b1


# ------------------------------------------------------------------------------------ AutoInt interacting layer
def autoint_workspace(B: int, F: int, d: int, H: int, dk: int, device) -> torch.Tensor:
    """Caller-owned workspace: the prepped weights (B = 0, what the forward needs) plus, for the backward, the per-row
    projection gradients (B*F, 4*H*dk)."""
    nbytes = ctypes.c_int64(0)
    _lib.check(_lib.lib().ctr_autoint_workspace_bytes(B, F, d, H, dk, ctypes.byref(nbytes)))
    return torch.empty((int(nbytes.value),), dtype=torch.uint8, device=device)


def _autoint_args(x, wq, wk, wv, wr, heads, dk):
    _chk(x, F32, "input")
    if x.dim() != 3:
        raise ValueError(f"input must be (B, F, d), got shape {tuple(x.shape)}")
    B, F, d = x.shape
    H, dk = int(heads), int(dk)
    for name, w in (("w_query", wq), ("w_key", wk), ("w_value", wv), ("w_res", wr)):
        _chk(w, F32, name, (d, H * dk))
    return B, F, d, H, dk


def autoint_fwd(x, w_query, w_key, w_value, w_res, heads: int, dk: int) -> torch.Tensor:
    """AutoInt interacting layer (arXiv:1810.11921 eq. 5-8): relu(concat_h softmax(Q_h K_h^T) V_h + x . w_res),
    x (B,F,d), each w (d, heads*dk) -> (B, F, heads*dk)."""
    B, F, d, H, dk = _autoint_args(x, w_query, w_key, w_value, w_res, heads, dk)
    out = torch.empty((B, F, H * dk), dtype=F32, device=x.device)
    ws = autoint_workspace(0, F, d, H, dk, x.device)
    _lib.check(_lib.lib().ctr_autoint_fwd(_ptr(x), _ptr(w_query), _ptr(w_key), _ptr(w_value), _ptr(w_res), B, F, d, H, dk,
                                          _ptr(out), _ptr(ws), ws.numel(), _stream()))
    return out


def autoint_bwd(x, w_query, w_key, w_value, w_res, out, g_out, heads: int, dk: int):
    """Gradients of autoint_fwd given its output `out` (the relu mask) and g_out (B,F,heads*dk):
    (d_x, d_w_query, d_w_key, d_w_value, d_w_res).  Q, K, V and the attention are recomputed from x."""
    B, F, d, H, dk = _autoint_args(x, w_query, w_key, w_value, w_res, heads, dk)
    _chk(out, F32, "out", (B, F, H * dk)); _chk(g_out, F32, "g_out", (B, F, H * dk))
    d_x = torch.empty_like(x)
    dws = [torch.empty_like(w) for w in (w_query, w_key, w_value, w_res)]
    ws = autoint_workspace(B, F, d, H, dk, x.device)
    _lib.check(_lib.lib().ctr_autoint_bwd(_ptr(x), _ptr(w_query), _ptr(w_key), _ptr(w_value), _ptr(w_res), _ptr(out),
                                          _ptr(g_out), B, F, d, H, dk, _ptr(d_x), *(_ptr(t) for t in dws), _ptr(ws),
                                          ws.numel(), _stream()))
    return (d_x, *dws)


# ------------------------------------------------------------------------------------ MMoE expert-gate layer
def mmoe_workspace(B: int, d: int, E: int, H: int, T: int, device) -> torch.Tensor:
    """Caller-owned workspace: the prepped weights (B = 0, what the forward needs) plus, for the backward, the expert and
    gate-logit gradients."""
    nbytes = ctypes.c_int64(0)
    _lib.check(_lib.lib().ctr_mmoe_workspace_bytes(B, d, E, H, T, ctypes.byref(nbytes)))
    return torch.empty((int(nbytes.value),), dtype=torch.uint8, device=device)


def _mmoe_args(x, w_experts, b_experts, w_gates):
    _chk(x, F32, "concat_all_input")
    if x.dim() != 2 or w_experts.dim() != 3 or w_gates.dim() != 3:
        raise ValueError("mmoe: x (B,d), w_experts (E,d,H) and w_gates (T,d,E) expected")
    B, d = x.shape
    E, _, H = w_experts.shape
    T = w_gates.shape[0]
    _chk(w_experts, F32, "w_experts", (E, d, H)); _chk(b_experts, F32, "b_experts", (E, H))
    _chk(w_gates, F32, "w_gates", (T, d, E))
    return B, d, E, H, T


def mmoe_fwd(x, w_experts, b_experts, w_gates):
    """MMOE/mmoe.py:207-236: x (B,d), w_experts (E,d,H), b_experts (E,H), w_gates (T,d,E) -> (towers (T,B,H), gates (T,B,E)),
    tower_t = sum_e softmax_e(x . w_gates[t])[e] relu(x . w_experts[e] + b_experts[e])."""
    B, d, E, H, T = _mmoe_args(x, w_experts, b_experts, w_gates)
    towers = torch.empty((T, B, H), dtype=F32, device=x.device)
    gates = torch.empty((T, B, E), dtype=F32, device=x.device)
    ws = mmoe_workspace(0, d, E, H, T, x.device)
    _lib.check(_lib.lib().ctr_mmoe_fwd(_ptr(x), _ptr(w_experts), _ptr(b_experts), _ptr(w_gates), B, d, E, H, T, _ptr(towers),
                                       _ptr(gates), _ptr(ws), ws.numel(), _stream()))
    return towers, gates


def mmoe_bwd(x, w_experts, b_experts, w_gates, gates, g_towers):
    """Gradients of mmoe_fwd given its gates (T,B,E) and g_towers (T,B,H): (d_x, d_w_experts, d_b_experts, d_w_gates).
    The expert outputs are recomputed from x."""
    B, d, E, H, T = _mmoe_args(x, w_experts, b_experts, w_gates)
    _chk(gates, F32, "gates", (T, B, E)); _chk(g_towers, F32, "g_towers", (T, B, H))
    d_x, d_we, d_be, d_wg = (torch.empty_like(t) for t in (x, w_experts, b_experts, w_gates))
    ws = mmoe_workspace(B, d, E, H, T, x.device)
    _lib.check(_lib.lib().ctr_mmoe_bwd(_ptr(x), _ptr(w_experts), _ptr(b_experts), _ptr(w_gates), _ptr(gates), _ptr(g_towers),
                                       B, d, E, H, T, _ptr(d_x), _ptr(d_we), _ptr(d_be), _ptr(d_wg), _ptr(ws), ws.numel(),
                                       _stream()))
    return d_x, d_we, d_be, d_wg


# ------------------------------------------------------------------------------------ PLE expert-gate blocks
def _ple_counts(experts_per_task, num_experts_in_shared, extraction):
    n = [int(v) for v in experts_per_task]
    return (ctypes.c_int64 * max(1, len(n)))(*n), n, int(num_experts_in_shared), 1 if extraction else 0


def ple_gate_width(experts_per_task, num_experts_in_shared, extraction) -> int:
    """GC, the number of gate columns: sum_t (n_t + S), plus the all-gate's sum_t n_t + S in the extraction network."""
    n, S = [int(v) for v in experts_per_task], int(num_experts_in_shared)
    return sum(n) + len(n) * S + ((sum(n) + S) if extraction else 0)


def ple_workspace(B: int, d: int, H: int, experts_per_task, num_experts_in_shared, extraction, device) -> torch.Tensor:
    """Caller-owned workspace: the prepped weights (B = 0, what the forward needs) plus, for the backward, the expert and
    gate-logit gradients."""
    arr, n, S, ext = _ple_counts(experts_per_task, num_experts_in_shared, extraction)
    nbytes = ctypes.c_int64(0)
    _lib.check(_lib.lib().ctr_ple_workspace_bytes(B, d, H, len(n), arr, S, ext, ctypes.byref(nbytes)))
    return torch.empty((int(nbytes.value),), dtype=torch.uint8, device=device)


def _ple_args(x, w_experts, b_experts, w_gates, experts_per_task, num_experts_in_shared, extraction):
    _chk(x, F32, "input")
    if x.dim() != 2 or w_experts.dim() != 3 or w_gates.dim() != 2:
        raise ValueError("ple: x (B,d), w_experts (E,d,H) and w_gates (d,GC) expected")
    B, d = x.shape
    E, _, H = w_experts.shape
    n, S = [int(v) for v in experts_per_task], int(num_experts_in_shared)
    if E != sum(n) + S:
        raise ValueError(f"ple: w_experts holds {E} experts, experts_per_task and num_experts_in_shared give {sum(n) + S}")
    _chk(w_experts, F32, "w_experts", (E, d, H)); _chk(b_experts, F32, "b_experts", (E, H))
    _chk(w_gates, F32, "w_gates", (d, ple_gate_width(n, S, extraction)))
    return B, d, H


def ple_fwd(x, w_experts, b_experts, w_gates, experts_per_task, num_experts_in_shared, extraction):
    """PLE/extraction_network.py:4-85 (extraction = True) or PLE/ple.py:185-226 (False): x (B,d), w_experts (E,d,H) and
    b_experts (E,H) in [task 0 .. task T-1, shared] order, w_gates (d,GC) the gate kernels concatenated by columns ->
    (out, gates (B,GC)).  out is (B,H) for the extraction network, (T,B,H) for the final layer."""
    B, d, H = _ple_args(x, w_experts, b_experts, w_gates, experts_per_task, num_experts_in_shared, extraction)
    arr, n, S, ext = _ple_counts(experts_per_task, num_experts_in_shared, extraction)
    out = torch.empty((B, H) if ext else (len(n), B, H), dtype=F32, device=x.device)
    gates = torch.empty((B, w_gates.shape[1]), dtype=F32, device=x.device)
    ws = ple_workspace(0, d, H, n, S, ext, x.device)
    _lib.check(_lib.lib().ctr_ple_fwd(_ptr(x), _ptr(w_experts), _ptr(b_experts), _ptr(w_gates), B, d, H, len(n), arr, S, ext,
                                      _ptr(out), _ptr(gates), _ptr(ws), ws.numel(), _stream()))
    return out, gates


def ple_bwd(x, w_experts, b_experts, w_gates, gates, g_out, experts_per_task, num_experts_in_shared, extraction):
    """Gradients of ple_fwd given its gates (B,GC) and g_out (shaped as out): (d_x, d_w_experts, d_b_experts, d_w_gates).
    The expert outputs are recomputed from x."""
    B, d, H = _ple_args(x, w_experts, b_experts, w_gates, experts_per_task, num_experts_in_shared, extraction)
    arr, n, S, ext = _ple_counts(experts_per_task, num_experts_in_shared, extraction)
    _chk(gates, F32, "gates", (B, w_gates.shape[1]))
    _chk(g_out, F32, "g_out", (B, H) if ext else (len(n), B, H))
    d_x, d_we, d_be, d_wg = (torch.empty_like(t) for t in (x, w_experts, b_experts, w_gates))
    ws = ple_workspace(B, d, H, n, S, ext, x.device)
    _lib.check(_lib.lib().ctr_ple_bwd(_ptr(x), _ptr(w_experts), _ptr(b_experts), _ptr(w_gates), _ptr(gates), _ptr(g_out), B, d,
                                      H, len(n), arr, S, ext, _ptr(d_x), _ptr(d_we), _ptr(d_be), _ptr(d_wg), _ptr(ws),
                                      ws.numel(), _stream()))
    return d_x, d_we, d_be, d_wg


# ------------------------------------------------------------------------------------ Row MTL: multi-task loss balancing
MTL_METHODS = {"sum": 0, "gradnorm": 1, "uncertainty": 2}   # 1: task_param holds GradNorm's weights w; 2: s = log sigma^2
MTL_MAX_TASKS = 8
F64 = torch.float64


def multitask_sigmoid_ce(logits: torch.Tensor, labels: torch.Tensor, method: int, task_param: Optional[torch.Tensor] = None,
                         want_grad: bool = True):
    """Per-task mean sigmoid cross-entropies of logits / labels (T,B) and the method's total (include/ctr_b200.h, Row MTL):
    (task_loss (T,), total (1,), d_logits (T,B) | None, d_task_param (T,) | None).  d_logits is the unweighted
    (sigmoid(x) - z) / B; d_task_param is d total / d task_param (None for method 0)."""
    T, B = logits.shape
    _chk(logits, F32, "logits"); _chk(labels, F32, "labels", (T, B))
    if method != 0:
        _chk(task_param, F32, "task_param", (T,))
    task_loss = torch.empty((T,), dtype=F32, device=logits.device)
    total = torch.empty((1,), dtype=F32, device=logits.device)
    d_logits = torch.empty((T, B), dtype=F32, device=logits.device) if want_grad else None
    d_param = torch.empty((T,), dtype=F32, device=logits.device) if want_grad and method != 0 else None
    _lib.check(_lib.lib().ctr_multitask_sigmoid_ce(_ptr(logits), _ptr(labels), T, B, int(method),
                                                   _ptr(task_param) if method != 0 else None, _ptr(task_loss), _ptr(total),
                                                   _ptr(d_logits), _ptr(d_param), _stream()))
    return task_loss, total, d_logits, d_param


def _task_rows(grads: torch.Tensor):
    """(T, P, ld) of a (T,P) float32 view whose rows are contiguous (row pitch ld >= P, e.g. a column slice)."""
    if grads.dim() != 2:
        raise ValueError(f"grads: expected (T,P), got shape {tuple(grads.shape)}")
    T, P = grads.shape
    if not (grads.is_cuda and grads.device.index == torch.cuda.current_device() and grads.dtype == F32):
        _chk(grads.contiguous(), F32, "grads")                         # raises the device / dtype error
    ld = grads.stride(0) if T > 1 else P
    if (P > 1 and grads.stride(1) != 1) or ld < P:
        raise ValueError(f"grads: rows must be contiguous with a row pitch >= P, got strides {grads.stride()}")
    return T, P, ld


def multitask_gram(grads: torch.Tensor, gram: Optional[torch.Tensor] = None) -> torch.Tensor:
    """gram (T,T) float64 = grads . grads^T of the per-task gradient rows grads (T,P), deterministic."""
    T, P, ld = _task_rows(grads)
    nbytes = ctypes.c_int64(0)
    _lib.check(_lib.lib().ctr_multitask_gram_workspace_bytes(T, P, ctypes.byref(nbytes)))
    ws = torch.empty((max(int(nbytes.value) // 8, 1),), dtype=F64, device=grads.device)
    if gram is None:
        gram = torch.empty((T, T), dtype=F64, device=grads.device)
    _chk(gram, F64, "gram", (T, T))
    _lib.check(_lib.lib().ctr_multitask_gram(_ptr(grads), T, P, ld, _ptr(gram), _ptr(ws), ws.numel() * 8, _stream()))
    return gram


def pcgrad_combine(grads: torch.Tensor, gram: torch.Tensor, order: torch.Tensor, out: Optional[torch.Tensor] = None,
                   want_coef: bool = False):
    """PCGrad of the per-task gradient rows grads (T,P) given their gram (T,T) float64 and the projection order (T,) int32:
    (out (P,), coef (T,) float64 | None), out = sum_k coef_k grads[k]."""
    T, P, ld = _task_rows(grads)
    _chk(gram, F64, "gram", (T, T)); _chk(order, I32, "order", (T,))
    if out is None:
        out = torch.empty((P,), dtype=F32, device=grads.device)
    _chk(out, F32, "out", (P,))
    coef = torch.empty((T,), dtype=F64, device=grads.device) if want_coef else None
    _lib.check(_lib.lib().ctr_pcgrad_combine(_ptr(grads), T, P, ld, _ptr(gram), _ptr(order), _ptr(out), _ptr(coef), _stream()))
    return out, coef


def gradnorm_update(gram: torch.Tensor, task_loss: torch.Tensor, initial_loss: torch.Tensor, weights: torch.Tensor,
                    alpha: float, lr: float, want_d_weights: bool = False):
    """One GradNorm step on weights (T,) in place from the gram (T,T) float64 of the unweighted per-task gradients, the task
    losses and the initial ones: (grad_loss (1,), d_weights (T,) | None)."""
    T = weights.numel()
    _chk(weights, F32, "weights", (T,)); _chk(gram, F64, "gram", (T, T))
    _chk(task_loss, F32, "task_loss", (T,)); _chk(initial_loss, F32, "initial_loss", (T,))
    grad_loss = torch.empty((1,), dtype=F32, device=weights.device)
    d_w = torch.empty((T,), dtype=F32, device=weights.device) if want_d_weights else None
    _lib.check(_lib.lib().ctr_gradnorm_update(_ptr(gram), _ptr(task_loss), _ptr(initial_loss), T, float(alpha), float(lr),
                                              _ptr(weights), _ptr(grad_loss), _ptr(d_w), _stream()))
    return grad_loss, d_w
