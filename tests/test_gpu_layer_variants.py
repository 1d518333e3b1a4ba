"""Every CUDA-core layer kernel of DCN, DIN, BST, FiBiNET, FwFM, AFM and FFM against float64, at its dispatch boundaries and
with several samples per warp or CTA.

The kernels of csrc/cross.cu, csrc/din_attention.cu, csrc/bst.cu, csrc/fibinet.cu and csrc/pairwise.cu are persistent: the
grid is capped near the SM count and every warp (or CTA) loops over samples (or tiles of samples).  The loop carries the
code that only runs from a worker's second sample on: weight-gradient accumulators kept across samples, the next sample's
loads issued one iteration ahead, double buffers swapped per tile, and the per-CTA merge after the loop.  This file holds
  * a pure-Python mirror of the host dispatch (shape, bilinear mask -> the kernels launched, with template arguments),
  * one table of shapes on both sides of every dispatch boundary, plus rows placed from the device's SM count so that every
    worker of the loop kernels carries at least three samples,
  * a CPU test that the mirror over the table reaches every instantiation the built library contains, except a pinned list
    of instantiations no shape can select, and nothing the library lacks,
  * GPU tests: every row forward and backward against float64, and the launched kernels (torch.profiler) against the mirror,
    with their grids showing that the loop ran at least three times on the SM-placed rows,
  * the C-ABI backward of the cross stack with dw and db in separate allocations.
"""
import json
import os
import re
import shutil
import subprocess
import tempfile
import zlib
from typing import NamedTuple

import numpy as np
import pytest
import torch

from _util import TOL, assert_close, dev, trunc_normal
from oracle import bst_torch
from oracle import layers_np as O

SMS_H100 = 132          # SM count of an H100 SXM: the coverage test places the SM rows for it


# ================================================================================================ dispatch mirror
# ---------------------------------------------------------------------------------------------------------- cross.cu
def cross_vec_n(d):
    """(VEC, N) of with_cross_class, cross.cu:643-655:
        if (d % 4 == 0) { n = (d / 4 + 31) / 32;  N = n <= 1 ? 1 : n <= 2 ? 2 : n <= 4 ? 4 : 8;  VEC = 4 }
        else            { n = (d + 31) / 32;      N = 1, 2, 4, 8, 16 or 32 (the first class >= n);  VEC = 1 }"""
    if d % 4 == 0:
        n = (d // 4 + 31) // 32
        return 4, next(c for c in (1, 2, 4, 8) if n <= c)
    n = (d + 31) // 32
    return 1, next((c for c in (1, 2, 4, 8, 16) if n <= c), 32)


def cross_cpt(vec, n):
    """cross.cu:621  CPT = VEC * N * 32 <= 256 ? 1 : VEC * N * 32 <= 512 ? 2 : 4   (VEC * N * 32: the largest d of the class)."""
    return 1 if vec * n * 32 <= 256 else 2 if vec * n * 32 <= 512 else 4


def cross_bwd_smem(d, L, has_xl, prefetch):
    """cross.cu:578-581  sizeof(float) * (3 L d + (prefetch ? 2 : 1) * (has_xl ? 3 : 2) * CROSS_WARPS d + 2 CROSS_WARPS LMAX)."""
    return 4 * (3 * L * d + (2 if prefetch else 1) * (3 if has_xl else 2) * 8 * d + 2 * 8 * 8)


def cross_reg_smem(d, L, rw):
    """cross.cu:601  sizeof(float) * (2 L d + rw ((L + 1) d + 4))."""
    return 4 * (2 * L * d + rw * ((L + 1) * d + 4))


def cross_fwd_launches(B, d, L):
    """cross.cu:674  if (B == 0) return CTR_OK;   cross.cu:676  launch_cross_fwd<VEC, N> -> cross_fwd_kernel<VEC, N>."""
    return [] if B == 0 else [("cross_fwd_kernel", cross_vec_n(d))]


def cross_bwd_launches(B, d, L, xl, sms):
    """Kernels `ctr_cross_bwd` launches.

    cross.cu:690-694  if (B == 0) { two memsets; return }
    cross.cu:594-595  if constexpr (VEC == 4 && N <= 4) { if (xl_in == nullptr && L <= 4) {
    cross.cu:599-600    wide = B >= sm_count() * 12 * 2 && !(N == 4 && L > 3);  rw = wide ? 12 : 8;
    cross.cu:602        if (smem_r <= 200 * 1024) -> cross_bwd_reg_kernel<N, L, rw>        (cross.cu:613-616: LM = L)
    cross.cu:634-638    pf = VEC == 4 && (N != 8 || cross_bwd_smem(d, L, xl_in != nullptr, true) <= 160 * 1024)
    cross.cu:626        cross_bwd_kernel<VEC, N, CPT, pf, L <= 4 ? 4 : 8>
    """
    if B == 0:
        return []
    vec, n = cross_vec_n(d)
    if vec == 4 and n <= 4 and not xl and L <= 4:
        rw = 12 if B >= sms * 24 and not (n == 4 and L > 3) else 8
        if cross_reg_smem(d, L, rw) <= 200 * 1024:
            return [("cross_bwd_reg_kernel", (n, L, rw))]
    # cross.cu:632-633: below N = 8 (d <= 512) the double-buffered staging always fits 160 KB
    assert vec != 4 or n == 8 or cross_bwd_smem(d, L, xl, True) <= 160 * 1024
    pf = vec == 4 and (n != 8 or cross_bwd_smem(d, L, xl, True) <= 160 * 1024)
    return [("cross_bwd_kernel", (vec, n, cross_cpt(vec, n), pf, 4 if L <= 4 else 8))]


def embed_cross_launches(B, F, D, L, i32):
    """cross.cu:717  unsupported unless D % 4 == 0, F*D <= 512, L <= 4 (ops.embed_cross_fwd then runs lookup + cross_fwd);
    cross.cu:722  if (B == 0) return;   cross.cu:724-729  n = (F*D + 127) / 128 -> N = 1, 2, 3 or 4;
    cross.cu:703-704  embed_cross_fwd_kernel<N, L, IdT>,  IdT = int (ids_are_int32) or long long."""
    assert D % 4 == 0 and F * D <= 512 and L <= 4, "the table has no embed-cross row outside the fused kernel's shapes"
    if B == 0:
        return []
    return [("embed_cross_fwd_kernel", (min((F * D + 127) // 128, 4), L, "int" if i32 else "long long"))]


# ------------------------------------------------------------------------------------------------- din_attention.cu
def din_hp(H):
    """din_attention.cu:681, 734  HP = H <= 4 ? 4 : H <= 8 ? 8 : H <= 16 ? 16 : 32."""
    return 4 if H <= 4 else 8 if H <= 8 else 16 if H <= 16 else 32


def _r4(v):
    return (v + 3) & ~3


def din_fwd_floats(H, T, warps):
    """din_layout(H, T, warps, bwd = false).total, din_attention.cu:45-69."""
    o = 3 * H * 64 + 64 + 64 * 32 + 32 + 36
    return o + warps * _r4(T * H + T + 3 * H) + warps * 4 * 64


def din_bwd_floats(H, HP, T, warps):
    """din_bwd_layout(H, HP, T, warps).total, din_attention.cu:302-336."""
    o = 3 * H * 64 + 64 + 64 * 32 + 32 + 36 + 64 * 32 + 32 + 36
    w = _r4(T * H + T + H + H + T)
    w = _r4(w + 3 * H * 64 + 64)
    w = _r4(w + 64 * (HP + 1))
    w = _r4(w + 64 * 2 + 64 * 2 + 32 * 2)
    return o + warps * w


def din_bwd_warps(H, T):
    """din_attention.cu:736-737  w8 = sizeof(float) * din_bwd_layout(H, HP, T, 8).total <= 220 * 1024; warps = w8 ? 8 : 4."""
    return 8 if 4 * din_bwd_floats(H, din_hp(H), T, 8) <= 220 * 1024 else 4


def din_fwd_launches(B, T, H, balanced):
    """din_attention.cu:696-701  B == 0, T == 0: no kernel;  :702-706  sched_scratch given -> din_schedule_kernel;
    :679  refused above 220 KB;  :718, 693  din_attention_fwd_kernel<HP, 4>."""
    if B == 0 or T == 0:
        return []
    if 4 * din_fwd_floats(H, T, 4) > 220 * 1024:
        return None
    return [("din_schedule_kernel", ())] * balanced + [("din_attention_fwd_kernel", (din_hp(H), 4))]


def din_bwd_launches(B, T, H, balanced):
    """din_attention.cu:723-727  B == 0, T == 0: memsets only;  :728-732  din_schedule_kernel;  :740  refused above 220 KB;
    :766  din_attention_bwd_kernel<HP, warps>."""
    if B == 0 or T == 0:
        return []
    warps = din_bwd_warps(H, T)
    if 4 * din_bwd_floats(H, din_hp(H), T, warps) > 220 * 1024:
        return None
    return [("din_schedule_kernel", ())] * balanced + [("din_attention_bwd_kernel", (din_hp(H), warps))]


# ----------------------------------------------------------------------------------------------------------- bst.cu
def bst_launches(B, d, bwd):
    """bst.cu:404, 419  B == 0: no kernel;  bst.cu:391-396  d in {4, 8, 16, 32, 64} -> bst_kernel<d, BWD>."""
    return [] if B == 0 else [("bst_kernel", (d, bwd))]


# ------------------------------------------------------------------------------------------------------- fibinet.cu
def senet_launches(B, bwd):
    """fibinet.cu:864, 878  B == 0: no kernel;  :866, 880  senet_kernel<BWD>."""
    return [] if B == 0 else [("senet_kernel", (bwd,))]


class RRShape(NamedTuple):
    n: int
    np: int
    rounds: int
    slots: int
    slot0: int


def rr_shape(F):
    """fibinet.cu:317-325."""
    n = F - 1
    np_ = n + 1 if n & 1 else n
    slot0 = 1 if n & 1 else 0
    return RRShape(n, np_, np_ - 1, np_ // 2 - slot0, slot0)


def rr_kt(K, kt_bits=0):
    """fibinet.cu:814-818  kt = g_bilinear_kt > 0 ? g_bilinear_kt : 2;  while (kt > 1 && (K * kt > 64 || K / kt < 2)) kt >>= 1;"""
    kt = kt_bits if kt_bits > 0 else 2
    while kt > 1 and (K * kt > 64 or K // kt < 2):
        kt >>= 1
    return kt


def rr_kt_template(K, kt):
    """fibinet.cu:836-845  kt == 1 -> 1;  kt == 2 -> 2;  else (K <= 16 ? 4 : 2)."""
    return 1 if kt == 1 else 2 if kt == 2 else (4 if K <= 16 else 2)


def rr_threads(F, K, kt):
    """fibinet.cu:821-827  G = min(slots, 256 / lp) (>= 1) groups of lp = K / kt lanes, rounded up to whole warps."""
    lp = K // kt
    G = max(min(rr_shape(F).slots, 256 // lp), 1)
    return (G * lp + 31) // 32 * 32


def rr_tile(F, K, arrays, fixed, budget, tile_bits=0):
    """fibinet.cu:830-834  bs = g_bilinear_tile > 0 ? g_bilinear_tile : 8, halved until fixed + arrays bs F K floats fit."""
    bs = tile_bits if tile_bits > 0 else 8
    while bs >= 1 and fixed + arrays * bs * F * K * 4 > budget:
        bs >>= 1
    return bs


RR_GP = 8               # fibinet.cu:441


def _rr_table_bytes(F):
    sh = rr_shape(F)
    return 4 * _r4(sh.rounds * sh.slots)


def _mask_bits(mask):
    """ctr_bilinear_set_rr, fibinet.cu:899-906: (rr types, old, tile, kt)."""
    return mask & 7, (mask >> 3) & 1, (mask >> 4) & 63, (mask >> 10) & 7


def bilinear_rr_fwd_plan(F, K, mask):
    """(KT, bs, threads, smem) of the forward under `mask`: fibinet.cu:926-931  fixed = pair table;
    bs = rr_tile(.., 1, fixed, 64 KB), else 200 KB (both from the mask's tile bits); 256 threads; kt = rr_kt(K)."""
    _, _, tile, kt = _mask_bits(mask)
    kt = rr_kt(K, kt)
    fixed = _rr_table_bytes(F)
    bs = rr_tile(F, K, 1, fixed, 64 * 1024, tile)
    if bs < 1:
        bs = rr_tile(F, K, 1, fixed, 200 * 1024, tile)
    return rr_kt_template(K, kt), bs, 256, fixed + 4 * bs * F * K


def bilinear_rr_bwd_plan(F, K, mask):
    """(KT, bs, threads, smem) of the dX kernel under `mask`: fibinet.cu:973-981  fixed = pair table + (threads / lp)
    RR_GP K floats;  bs = rr_tile(.., 2, fixed, 72 KB), else 200 KB;  bs = min(bs, RR_GP)."""
    _, _, tile, kt = _mask_bits(mask)
    kt = rr_kt(K, kt)
    threads = rr_threads(F, K, kt)
    fixed = _rr_table_bytes(F) + 4 * (threads // (K // kt)) * RR_GP * K
    bs = rr_tile(F, K, 2, fixed, 72 * 1024, tile)
    if bs < 1:
        bs = rr_tile(F, K, 2, fixed, 200 * 1024, tile)
    bs = min(bs, RR_GP)
    return rr_kt_template(K, kt), bs, threads, fixed + 4 * 2 * bs * F * K


def rr_usable(K, t, mask):
    """fibinet.cu:886-890 (every array the tests pass is 16-byte aligned)."""
    return bool((_mask_bits(mask)[0] >> t) & 1) and K in (8, 16, 32)


def st_usable(K, t, mask):
    """fibinet.cu:893-897."""
    return not _mask_bits(mask)[1] and t <= 1 and K in (8, 16, 32)


BIL_TYPES = {"all": 0, "each": 1, "interaction": 2}


def bilinear_fwd_launches(B, F, K, type_, mask):
    """Kernels `ctr_bilinear_fwd` launches.

    fibinet.cu:923        if (B == 0 || P == 0) return CTR_OK;
    fibinet.cu:925-936    rr_usable -> bs >= 1: bilinear_rr_fwd_kernel<K, KT>  (KT: rr_kt and with_rr)
    fibinet.cu:938-948    st_usable, smem_st = 4 (nw K K + 2 F K + n K) + 4 P <= 200 KB: bilinear_st_fwd_kernel<K, type>
    fibinet.cu:950-954    bilinear_fwd_kernel<type>
    """
    t, n = BIL_TYPES[type_], F - 1
    P = n * (n - 1) // 2
    if B == 0 or P == 0:
        return []
    if rr_usable(K, t, mask):
        KT, bs, _, _ = bilinear_rr_fwd_plan(F, K, mask)
        if bs >= 1:
            return [("bilinear_rr_fwd_kernel", (K, KT))]
    if st_usable(K, t, mask):
        nw = 1 if t == 0 else n
        if 4 * (nw * K * K + 2 * F * K + n * K) + 4 * P <= 200 * 1024:
            return [("bilinear_st_fwd_kernel", (K, t))]
    return [("bilinear_fwd_kernel", (t,))]


def bilinear_bwd_launches(B, F, K, type_, mask):
    """Kernels `ctr_bilinear_bwd` launches; None when it refuses the shape.

    fibinet.cu:965-970    memset dw;  B == 0: return;  P == 0: memset dx, return
    fibinet.cu:971-1001   rr_usable -> bs >= 1: bilinear_rr_bwd_dx_kernel<K, KT>, bilinear_rr_bwd_dw_kernel<K, KT>
    fibinet.cu:1002-1014  type 'interaction': bilinear_bwd_interaction_dx_kernel, bilinear_bwd_interaction_dw_kernel
                          (refused when 4 (2 F K + P K) + 4 P > 200 KB)
    fibinet.cu:1015-1026  st_usable, smem_st = 4 (2 nw K K + 2 F K + 2 P K + 2 n K) <= 200 KB: bilinear_st_bwd_kernel<K, type>
    fibinet.cu:1027-1033  bilinear_bwd_kernel<type>  (refused when 4 (F K + 2 n K + nw K K) > 200 KB)
    """
    t, n = BIL_TYPES[type_], F - 1
    P = n * (n - 1) // 2
    if B == 0 or P == 0:
        return []
    if rr_usable(K, t, mask):
        KT, bs, _, _ = bilinear_rr_bwd_plan(F, K, mask)
        if bs >= 1:
            return [("bilinear_rr_bwd_dx_kernel", (K, KT)), ("bilinear_rr_bwd_dw_kernel", (K, KT))]
    if t == 2:
        if 4 * (2 * F * K + P * K) + 4 * P > 200 * 1024:
            return None
        return [("bilinear_bwd_interaction_dx_kernel", ()), ("bilinear_bwd_interaction_dw_kernel", ())]
    nw = 1 if t == 0 else n
    if st_usable(K, t, mask) and 4 * (2 * nw * K * K + 2 * F * K + 2 * P * K + 2 * n * K) <= 200 * 1024:
        return [("bilinear_st_bwd_kernel", (K, t))]
    if 4 * (F * K + 2 * n * K + nw * K * K) > 200 * 1024:
        return None
    return [("bilinear_bwd_kernel", (t,))]


# ------------------------------------------------------------------------------------------------------ pairwise.cu
def fwfm_launches(B, K, bwd):
    """pairwise.cu:372  B == 0: no kernel;  :374  vec = K % 4 == 0 (the tests' arrays are 16-byte aligned);
    :389-392  fwfm_kernel<BWD, vec>."""
    return [] if B == 0 else [("fwfm_kernel", (bwd, K % 4 == 0))]


def afm_tu(K, T):
    """pairwise.cu:332-342  tu = ceil(T / 32), taken up to the first class >= tu of K's ladder; None: refused (K * TU > 64).
        K 4, 8: 1, 2, 4, 8     K 16: 1, 2, 4     K 32: 1, 2"""
    tu = (T + 31) // 32
    ladder = {4: (1, 2, 4, 8), 8: (1, 2, 4, 8), 16: (1, 2, 4), 32: (1, 2)}.get(K, ())
    return next((c for c in ladder if tu <= c), None)


def afm_launches(B, K, T, bwd):
    """pairwise.cu:398, 412  B == 0: no kernel (before the shape check);  :332-342  afm_kernel<K, TU, BWD>, else refused."""
    if B == 0:
        return []
    TU = afm_tu(K, T)
    return None if TU is None else [("afm_kernel", (K, TU, bwd))]


def ffm_launches(B, bwd):
    """pairwise.cu:421-424  B == 0: no kernel;  ffm_kernel<BWD>."""
    return [] if B == 0 else [("ffm_kernel", (bwd,))]


# ---------------------------------------------------------------------------------------- workers of the loop kernels
# How a kernel hands out work: "warp" kernels loop a warp over samples, "cta" kernels loop a CTA over work items of `unit`
# samples (1, 8 for the staged cross backward, the tile for the tournament kernels).  Kernels not listed here (the
# schedule pass, the weight-gradient kernels over (pair block, batch chunk) grids) do not walk the batch per worker.
WORKERS = {"cross_fwd_kernel": "warp", "cross_bwd_reg_kernel": "warp", "cross_bwd_kernel": "cta", "embed_cross_fwd_kernel": "warp",
           "din_attention_fwd_kernel": "warp", "din_attention_bwd_kernel": "warp", "bst_kernel": "cta", "senet_kernel": "warp",
           "bilinear_fwd_kernel": "cta", "bilinear_bwd_kernel": "cta", "bilinear_bwd_interaction_dx_kernel": "cta",
           "bilinear_st_fwd_kernel": "cta", "bilinear_st_bwd_kernel": "cta", "bilinear_rr_fwd_kernel": "cta",
           "bilinear_rr_bwd_dx_kernel": "cta", "fwfm_kernel": "warp", "afm_kernel": "warp", "ffm_kernel": "warp"}


def ctas_per_sm_bound(threads, smem_bytes):
    """Most CTAs of `threads` threads and `smem_bytes` dynamic shared memory an H100 SM can hold, from the hardware limits
    alone: 2048 threads, 32 CTAs, 228 KB of shared memory of which each CTA also takes 1 KB.  Registers can only lower it,
    so no occupancy query is needed for a batch that gives every worker at least three samples."""
    return max(1, min(32, 2048 // threads, (228 * 1024) // (smem_bytes + 1024)))


def three_passes(workers_per_sm, sms, unit=1, r=5):
    """A batch that gives each of `workers_per_sm * sms` workers at least three items of `unit` samples, the last pass
    partial (r odd)."""
    return 3 * workers_per_sm * sms * unit + r


# ================================================================================================ shape table
class Cross(NamedTuple):
    B: int
    d: int
    L: int
    xl: bool = False

    @property
    def id(self):
        return f"cross-B{self.B}-d{self.d}-L{self.L}" + ("-xl" if self.xl else "")

    def launches(self, sms):
        return [cross_fwd_launches(self.B, self.d, self.L), cross_bwd_launches(self.B, self.d, self.L, self.xl, sms)]


class ECross(NamedTuple):
    B: int
    F: int
    D: int
    L: int
    i32: bool

    @property
    def id(self):
        return f"ecross-B{self.B}-F{self.F}-D{self.D}-L{self.L}-" + ("i32" if self.i32 else "i64")

    def launches(self, sms):
        return [embed_cross_launches(*self)]


class Din(NamedTuple):
    B: int
    T: int
    H: int
    soft: bool = False

    @property
    def id(self):
        return f"din-B{self.B}-T{self.T}-H{self.H}" + ("-softmax" if self.soft else "")

    def launches(self, sms):
        """Both schedules: balanced forward and backward, then the static ones."""
        return [din_fwd_launches(self.B, self.T, self.H, True), din_bwd_launches(self.B, self.T, self.H, True),
                din_fwd_launches(self.B, self.T, self.H, False), din_bwd_launches(self.B, self.T, self.H, False)]


class Bst(NamedTuple):
    B: int
    T: int
    d: int
    heads: int
    pos: bool = True

    @property
    def id(self):
        return f"bst-B{self.B}-T{self.T}-d{self.d}-h{self.heads}" + ("" if self.pos else "-nopos")

    def launches(self, sms):
        return [bst_launches(self.B, self.d, False), bst_launches(self.B, self.d, True)]


class Senet(NamedTuple):
    B: int
    F: int
    K: int
    r: int

    @property
    def id(self):
        return f"senet-B{self.B}-F{self.F}-K{self.K}-r{self.r}"

    def launches(self, sms):
        return [senet_launches(self.B, False), senet_launches(self.B, True)]


class Bil(NamedTuple):
    B: int
    F: int
    K: int
    type: str
    mask: int = 4

    @property
    def id(self):
        return f"bilinear-{self.type}-B{self.B}-F{self.F}-K{self.K}-mask{self.mask}"

    def launches(self, sms):
        return [bilinear_fwd_launches(*self), bilinear_bwd_launches(*self)]


class Fwfm(NamedTuple):
    B: int
    F: int
    K: int

    @property
    def id(self):
        return f"fwfm-B{self.B}-F{self.F}-K{self.K}"

    def launches(self, sms):
        return [fwfm_launches(self.B, self.K, False), fwfm_launches(self.B, self.K, True)]


class Afm(NamedTuple):
    B: int
    F: int
    K: int
    T: int

    @property
    def id(self):
        return f"afm-B{self.B}-F{self.F}-K{self.K}-T{self.T}"

    def launches(self, sms):
        return [afm_launches(self.B, self.K, self.T, False), afm_launches(self.B, self.K, self.T, True)]


class Ffm(NamedTuple):
    B: int
    F: int
    K: int

    @property
    def id(self):
        return f"ffm-B{self.B}-F{self.F}-K{self.K}"

    def launches(self, sms):
        return [ffm_launches(self.B, False), ffm_launches(self.B, True)]


def din_t_switch(H):
    """The shortest history at which the backward of width H drops from 8 to 4 warps per CTA."""
    T = 1
    while din_bwd_warps(H, T) == 8:
        T += 1
    return T


# Boundary rows: small batches (odd, so the last 8-sample tile or pass is partial), one row on each side of every switch.
ROWS = [
    # cross, vector path (d % 4 == 0): N = 1 | 2 | 4 | 8 at d = 128 | 132, 256 | 260, 512 | 516, 1024; L 1-4 and 5-8; xl_in
    Cross(45, 128, 1), Cross(45, 128, 2, True), Cross(45, 128, 6), Cross(37, 132, 2), Cross(37, 132, 4, True),
    Cross(37, 256, 3), Cross(37, 256, 8), Cross(41, 260, 4), Cross(41, 260, 5, True), Cross(41, 512, 1),
    Cross(41, 512, 3, True), Cross(41, 512, 7), Cross(29, 516, 2), Cross(29, 516, 5, True), Cross(29, 1024, 1),
    Cross(29, 1024, 2), Cross(29, 1024, 3), Cross(29, 1024, 8, True),
    # cross, vector path: the 160 KB staging cut-off at d = 768 with xl_in (L 1 fits, L 2 does not); small L and N classes
    Cross(23, 768, 1, True), Cross(23, 768, 2, True), Cross(33, 64, 1), Cross(33, 64, 3), Cross(33, 192, 1), Cross(33, 192, 4),
    Cross(33, 320, 2), Cross(33, 448, 4), Cross(0, 128, 2),
    # cross, scalar path (d % 4 != 0): N = 1 | 2 | 4 | 8 | 16 | 32 at d = 31 | 33, 63 | 65, 127 | 129, 255 | 257, 511 | 513, 1023
    Cross(43, 31, 1), Cross(43, 33, 4, True), Cross(43, 63, 5), Cross(43, 65, 2), Cross(39, 127, 8, True), Cross(39, 129, 3),
    Cross(39, 255, 4), Cross(39, 257, 6, True), Cross(27, 511, 1), Cross(27, 513, 7), Cross(27, 1023, 2, True), Cross(27, 1023, 5),
    Cross(19, 1, 1), Cross(19, 2, 8), Cross(39, 201, 7),
    # cross_bwd_reg_kernel<N, L, 8> (below 24 SMs' worth of samples): N = 1 | 2 | 4 at d = 128, 132 | 256, 260 | 512, L 1..4
    *[Cross(47, d, L) for d in (128, 256, 260) for L in (1, 2, 3, 4)], *[Cross(47, d, L) for d, L in ((132, 1), (512, 2))],
    # fused lookup + cross: N = 1..4 (F*D of 20 | 128, 132 | 256, 260 | 384, 388 | 512) x L 1..4 x int32 / int64 ids
    *[ECross(37, F, D, L, i32) for (F, D), L, i32 in zip([(5, 4), (8, 16), (33, 4), (16, 16), (65, 4), (24, 16), (97, 4),
                                                          (32, 16)] * 4,
                                                         [L for L in (1, 2, 3, 4) for _ in range(8)],
                                                         [bool(i & 1) ^ (i >= 16) for i in range(32)])],
    ECross(0, 8, 16, 2, False),
    # DIN: H at 4 | 5, 8 | 9, 16 | 17, 32; softmax and weighted sum; B = 0 and T = 0
    Din(13, 7, 4), Din(13, 7, 5, True), Din(13, 6, 8, True), Din(13, 6, 9), Din(11, 9, 16), Din(11, 9, 17, True),
    Din(9, 5, 32), Din(9, 5, 32, True), Din(0, 5, 16), Din(7, 0, 16),
    # DIN: the 8 -> 4 warps backward switch at each HP class (the first T whose 8-warp staging exceeds 220 KB)
    *[Din(9, din_t_switch(H) - 1, H, H == 8) for H in (4, 8, 16, 17)],
    *[Din(9, din_t_switch(H), H, H == 16) for H in (4, 8, 16, 17)],
    Din(5, 60, 32, True),
    # BST: every d, forward and backward; B = 0
    Bst(5, 7, 4, 1), Bst(5, 9, 8, 3), Bst(4, 20, 16, 2, False), Bst(3, 17, 32, 2), Bst(3, 11, 64, 1), Bst(2, 6, 64, 1, False),
    Bst(0, 5, 16, 2),
    # SENet; B = 0
    Senet(21, 7, 8, 3), Senet(9, 40, 16, 5), Senet(0, 7, 8, 3),
    # FwFM: K % 4 of 0 and != 0; B = 0
    Fwfm(31, 5, 8), Fwfm(31, 7, 5), Fwfm(17, 40, 16), Fwfm(17, 3, 1), Fwfm(0, 5, 8),
    # AFM: the TU class edges of each K, and one refused T per K; B = 0
    *[Afm(19, 5, K, T) for K, Ts in ((4, (32, 33, 64, 65, 128, 129, 256, 257)), (8, (32, 33, 64, 65, 128, 129, 256, 257)),
                                         (16, (32, 33, 64, 65, 128, 129)), (32, (32, 33, 64, 65))) for T in Ts],
    Afm(0, 5, 8, 16),
    # FFM
    Ffm(23, 5, 4), Ffm(23, 3, 7),
]
# The masks of test_gpu_fibinet.py: 4 (default: tournament kernels for 'interaction'), 7 (tournament kernels for every type),
# 7 with kt = 1, 7 with kt = 4 and 16-sample tiles, 8 (round-1 kernels for 'all' / 'each'), 0 (no tournament kernel).
BIL_MASKS = (4, 7, 7 | 1 << 10, 7 | 4 << 10 | 16 << 4, 8, 0)
# bilinear: K of 8, 16, 32 and 12 (no tournament / staged kernel) x the three types x those masks
ROWS += [Bil(37, 7, K, t, m) for K in (8, 16, 32, 12) for t in ("all", "each", "interaction") for m in BIL_MASKS]
ROWS += [
    Bil(9, 64, 32, "interaction", 4),   # forward tile shrinks to 4 samples (64 KB budget)
    Bil(9, 30, 32, "all", 7),           # backward tile shrinks to 4 < RR_GP (72 KB budget); forward keeps 8
    Bil(9, 9, 32, "each", 7),           # backward tile of RR_GP = 8
    Bil(5, 51, 32, "each", 4),          # staging 50 K x K weights exceeds 200 KB: round-1 forward, backward refused
    Bil(5, 26, 32, "each", 4),          # backward staging exceeds 200 KB: round-1 backward; forward staged
    Bil(5, 25, 32, "each", 4),          # backward staging fits
    Bil(37, 2, 8, "all", 4),            # P = 0: no kernel, dx = 0
]


# Rows placed from the device's SM count: every worker of the backward's loop kernels gets at least three samples (cross,
# DIN and BST forwards too where the same batch does), so every accumulator, prefetch and buffer swap runs past its first
# sample.  The batch is three passes of the most workers the hardware could hold (ctas_per_sm_bound), with the host's own
# caps on the grid where it has them.
def _cross_wide(d, L):
    def make(sms):
        per_sm = min(64, 12 * ctas_per_sm_bound(12 * 32, cross_reg_smem(d, L, 12)))
        row = Cross(three_passes(per_sm, sms), d, L)
        assert row.B >= 24 * sms
        return row
    return make


def _cross_staged(d, L, xl):
    def make(sms):
        pf = cross_vec_n(d)[0] == 4 and cross_bwd_smem(d, L, xl, True) <= 160 * 1024
        per_sm = min(2, ctas_per_sm_bound(256, cross_bwd_smem(d, L, xl, pf)))     # cross.cu:628: at most 2 CTAs per SM
        return Cross(three_passes(per_sm, sms, unit=8), d, L, xl)
    return make


def _din(T, H, soft):
    def make(sms):
        warps = din_bwd_warps(H, T)
        per_sm = warps * ctas_per_sm_bound(warps * 32, 4 * din_bwd_floats(H, din_hp(H), T, warps))
        return Din(three_passes(per_sm, sms), T, H, soft)
    return make


def _bst_ctas(T, d, heads):
    """The backward stages the parameters and their gradient (2 x ctr_bst_param_count floats, bst.cu:144-148, 370-373) next
    to its per-sample arrays, and runs 256 threads: a bound on its CTAs per SM."""
    total = T * d + 4 * heads * d * d + d * d + 5 * d
    return ctas_per_sm_bound(256, 2 * 4 * total)


def _bil(F, K, type_, mask):
    def make(sms):
        row = Bil(1, F, K, type_, mask)
        fwd, bwd = row.launches(sms)
        per_sm = []
        for name, _ in fwd + bwd:
            if name == "bilinear_rr_fwd_kernel":
                _, bs, threads, smem = bilinear_rr_fwd_plan(F, K, mask)
                per_sm.append(bs * ctas_per_sm_bound(threads, smem))
            elif name == "bilinear_rr_bwd_dx_kernel":
                _, bs, threads, smem = bilinear_rr_bwd_plan(F, K, mask)
                per_sm.append(bs * ctas_per_sm_bound(threads, smem))
            elif name in ("bilinear_st_fwd_kernel", "bilinear_st_bwd_kernel"):
                per_sm.append(ctas_per_sm_bound(512, 0))
            elif name == "bilinear_bwd_interaction_dx_kernel":
                per_sm.append(8)                                  # fibinet.cu:1006 capped_grid(B, 8 SMs)
            elif name == "bilinear_bwd_kernel":
                per_sm.append(2)                                  # fibinet.cu:1031 capped_grid(B, 2 SMs)
        return row._replace(B=three_passes(max(per_sm), sms))
    return make


SM_ROWS = {
    # cross_bwd_reg_kernel<N, L, 12>: B >= 24 SMs; N = 1 | 2 | 4 at d = 96 | 160 | 288
    **{f"cross-wide-N{n}-L{L}": _cross_wide(d, L) for n, d in ((1, 96), (2, 160), (4, 288)) for L in (1, 2, 3, 4)
       if not (n == 4 and L == 4)},
    # N = 4 with L = 4 stays at 8 warps (it would spill at 12): two 98 KB CTAs per SM, three samples per warp
    "cross-reg-N4-L4-8warps": lambda sms: Cross(three_passes(8 * ctas_per_sm_bound(256, cross_reg_smem(512, 4, 8)), sms), 512, 4),
    # cross_bwd_kernel: three 8-sample tiles per CTA, so both cp.async buffers are used
    "cross-staged-xl-vec": _cross_staged(128, 2, True),     # <4,1,1,true,4>: x0, xs and g staged per buffer
    "cross-staged-L6-vec": _cross_staged(256, 6, False),    # <4,2,1,true,8>
    "cross-staged-scalar": _cross_staged(129, 3, False),    # <1,8,1,false,4>
    "cross-staged-d1024-pf": _cross_staged(1024, 2, False),     # <4,8,4,true,4>
    "cross-staged-d1024-nopf": _cross_staged(1024, 3, False),   # <4,8,4,false,4>
    "ecross-i32": lambda sms: ECross(three_passes(64, sms), 6, 16, 3, True),
    "ecross-i64": lambda sms: ECross(three_passes(64, sms), 24, 8, 2, False),
    "din-bwd8-H4": _din(5, 4, False),
    "din-bwd8-H16-softmax": _din(4, 16, True),
    "din-bwd4-H32": _din(3, 32, False),
    "din-bwd4-H16-long": lambda sms: _din(din_t_switch(16), 16, False)(sms),
    "bst-d32": lambda sms: Bst(three_passes(_bst_ctas(4, 32, 2), sms), 4, 32, 2),
    "bst-d8": lambda sms: Bst(three_passes(_bst_ctas(6, 8, 3), sms), 6, 8, 3),
    "senet": lambda sms: Senet(three_passes(16, sms), 10, 8, 3),        # fibinet.cu:880 capped_grid(.., 4 SMs) x 4 warps
    "bilinear-rr-interaction": _bil(9, 8, "interaction", 4),
    "bilinear-rr-all": _bil(7, 16, "all", 7),
    "bilinear-rr-kt1": _bil(9, 16, "each", 7 | 1 << 10),
    "bilinear-rr-kt4-tile16": _bil(9, 8, "interaction", 7 | 4 << 10 | 16 << 4),
    "bilinear-st-each": _bil(6, 16, "each", 4),
    "bilinear-st-all": _bil(5, 32, "all", 4),
    "bilinear-round1-interaction": _bil(6, 12, "interaction", 8),
    "fwfm-vec": lambda sms: Fwfm(three_passes(64, sms), 5, 8),
    "fwfm-scalar": lambda sms: Fwfm(three_passes(64, sms), 6, 5),
    "afm-K8-TU1": lambda sms: Afm(three_passes(64, sms), 4, 8, 8),
    "afm-K4-TU8": lambda sms: Afm(three_passes(64, sms), 4, 4, 200),
    "ffm": lambda sms: Ffm(three_passes(64, sms), 4, 4),
}

# BASELINE configurations with a layer here: DCN (3 cross layers, 30 fields x 16, batch 4096) and DIN (T = 50, 16-wide
# keys, batch 4096).
BASELINE_ROWS = [Cross(4096, 480, 3), ECross(4096, 30, 16, 3, False), Din(4096, 50, 16), Din(4096, 50, 16, True)]

# The instantiation each SM row is placed for (test_sm_rows_select_their_kernels).
SM_KERNELS = {
    **{f"cross-wide-N{n}-L{L}": ("cross_bwd_reg_kernel", (n, L, 12)) for n in (1, 2, 4) for L in (1, 2, 3, 4)
       if not (n == 4 and L == 4)},
    "cross-reg-N4-L4-8warps": ("cross_bwd_reg_kernel", (4, 4, 8)),
    "cross-staged-xl-vec": ("cross_bwd_kernel", (4, 1, 1, True, 4)),
    "cross-staged-L6-vec": ("cross_bwd_kernel", (4, 2, 1, True, 8)),
    "cross-staged-scalar": ("cross_bwd_kernel", (1, 8, 1, False, 4)),
    "cross-staged-d1024-pf": ("cross_bwd_kernel", (4, 8, 4, True, 4)),
    "cross-staged-d1024-nopf": ("cross_bwd_kernel", (4, 8, 4, False, 4)),
    "ecross-i32": ("embed_cross_fwd_kernel", (1, 3, "int")),
    "ecross-i64": ("embed_cross_fwd_kernel", (2, 2, "long long")),
    "din-bwd8-H4": ("din_attention_bwd_kernel", (4, 8)),
    "din-bwd8-H16-softmax": ("din_attention_bwd_kernel", (16, 8)),
    "din-bwd4-H32": ("din_attention_bwd_kernel", (32, 4)),
    "din-bwd4-H16-long": ("din_attention_bwd_kernel", (16, 4)),
    "bst-d32": ("bst_kernel", (32, True)),
    "bst-d8": ("bst_kernel", (8, True)),
    "senet": ("senet_kernel", (True,)),
    "bilinear-rr-interaction": ("bilinear_rr_bwd_dx_kernel", (8, 2)),
    "bilinear-rr-all": ("bilinear_rr_bwd_dx_kernel", (16, 2)),
    "bilinear-rr-kt1": ("bilinear_rr_bwd_dx_kernel", (16, 1)),
    "bilinear-rr-kt4-tile16": ("bilinear_rr_bwd_dx_kernel", (8, 4)),
    "bilinear-st-each": ("bilinear_st_bwd_kernel", (16, 1)),
    "bilinear-st-all": ("bilinear_st_bwd_kernel", (32, 0)),
    "bilinear-round1-interaction": ("bilinear_bwd_interaction_dx_kernel", ()),
    "fwfm-vec": ("fwfm_kernel", (True, True)),
    "fwfm-scalar": ("fwfm_kernel", (True, False)),
    "afm-K8-TU1": ("afm_kernel", (8, 1, True)),
    "afm-K4-TU8": ("afm_kernel", (4, 8, True)),
    "ffm": ("ffm_kernel", (True,)),
}


def sm_rows(sms):
    return [make(sms) for make in SM_ROWS.values()]


# ================================================================================================ coverage (CPU)
CORE_KERNELS = ("cross_fwd_kernel", "cross_bwd_kernel", "cross_bwd_reg_kernel", "embed_cross_fwd_kernel",
                "din_schedule_kernel", "din_attention_fwd_kernel", "din_attention_bwd_kernel", "bst_kernel", "senet_kernel",
                "bilinear_fwd_kernel", "bilinear_bwd_kernel", "bilinear_bwd_interaction_dx_kernel",
                "bilinear_bwd_interaction_dw_kernel", "bilinear_rr_fwd_kernel", "bilinear_rr_bwd_dx_kernel",
                "bilinear_rr_bwd_dw_kernel", "bilinear_st_fwd_kernel", "bilinear_st_bwd_kernel", "fwfm_kernel", "afm_kernel",
                "ffm_kernel")


def _instantiations_from_rows(rows, sms):
    found = {}
    for row in rows:
        for call in row.launches(sms):
            for inst in call or []:
                found.setdefault(inst, []).append(row.id)
    return found


def _fmt(inst):
    return f"{inst[0]}<{', '.join(str(a).lower() if isinstance(a, bool) else str(a) for a in inst[1])}>"


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    for home in (os.environ.get("CUDA_HOME"), "/usr/local/cuda"):
        if exe is None and home and os.path.exists(os.path.join(home, "bin", "cuobjdump")):
            exe = os.path.join(home, "bin", "cuobjdump")
    return exe


_MANGLED_TYPES = {"i": "int", "x": "long long"}


def _mangled_args(s):
    """Template arguments at the start of s (after the 'I'): Li4E -> 4, Lb1E -> True, i -> 'int', x -> 'long long'."""
    args = []
    while not s.startswith("E"):
        lit = re.match(r"L([ib])(n?)(\d+)E", s)
        if lit:
            v = (-1 if lit.group(2) else 1) * int(lit.group(3))
            args.append(bool(v) if lit.group(1) == "b" else v)
            s = s[lit.end():]
        else:
            assert s[0] in _MANGLED_TYPES, f"unexpected template argument in {s}"
            args.append(_MANGLED_TYPES[s[0]])
            s = s[1:]
    return tuple(args)


def library_core_instantiations():
    """{(base name, template arguments)} of every kernel in CORE_KERNELS in the built library, read from the mangled names
    (e.g. _ZN3ctr16cross_bwd_kernelILi4ELi1ELi1ELb1ELi4EEEv... -> ("cross_bwd_kernel", (4, 1, 1, True, 4)))."""
    from recalgorithm_b200 import _lib, build
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump is not installed")
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    out = subprocess.run([exe, "-symbols", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found = set()
    for sym in set(re.findall(r"\b_Z\w+", out)):
        for num in re.finditer(r"\d+", sym):                        # <length><identifier> of each nested name
            end = num.end() + int(num.group())
            name = sym[num.end():end]
            if name in CORE_KERNELS and sym[end:end + 1] in ("I", "E"):
                found.add((name, _mangled_args(sym[end + 1:]) if sym[end] == "I" else ()))
                break
    assert {n for n, _ in found} == set(CORE_KERNELS), "kernels missing from the library: " + \
        ", ".join(sorted(set(CORE_KERNELS) - {n for n, _ in found}))
    return found


def test_table_reaches_exactly_the_library_instantiations():
    """The mirror over the shape table (SM rows placed for an H100 SXM) reaches exactly the CUDA-core layer instantiations
    the library has: every one of them, and nothing the library lacks."""
    in_lib = library_core_instantiations()
    reached = _instantiations_from_rows(ROWS + BASELINE_ROWS + sm_rows(SMS_H100), SMS_H100)
    missing = sorted(in_lib - set(reached), key=_fmt)
    unknown = sorted(set(reached) - in_lib, key=_fmt)
    assert not missing, "instantiations no row reaches: " + ", ".join(map(_fmt, missing))
    assert not unknown, "rows predict instantiations the library lacks: " + "; ".join(
        f"{_fmt(i)} (rows {', '.join(reached[i][:3])})" for i in unknown)


def test_shape_sweep_selects_only_library_instantiations():
    """Sweeping the mirror over the whole shape space of the cross, DIN and bilinear backward dispatch (and the bilinear
    forward, with every ctr_bilinear_set_rr mask) selects only instantiations the library has, so no shape outside the
    table can reach a kernel the library does not build."""
    in_lib = library_core_instantiations()
    reached = set()
    for d in range(1, 1025):
        for L in range(1, 9):
            for xl in (False, True):
                for B in (1, 10 ** 6):
                    reached.update(cross_bwd_launches(B, d, L, xl, SMS_H100))
    for H in range(1, 33):
        for T in list(range(1, 400)) + list(range(400, 8193, 7)):
            reached.update(din_bwd_launches(1, T, H, False) or [])
    tuning = [tile << 4 | kt << 10 for tile in (0, 1, 16, 63) for kt in range(8)]       # ctr_bilinear_set_rr's tuning bits
    for K in range(1, 129):
        for F in range(3, 257, 3):
            for t in BIL_TYPES:
                for mask in range(16):
                    for bits in tuning if K in (8, 16, 32) else (0,):       # other K never read them
                        reached.update(bilinear_fwd_launches(1, F, K, t, mask | bits))
                        reached.update(bilinear_bwd_launches(1, F, K, t, mask | bits) or [])
    assert not reached - in_lib, ", ".join(map(_fmt, sorted(reached - in_lib, key=_fmt)))


def test_mirror_sides_of_each_boundary():
    """The table has a row on each side of every dispatch boundary the mirror encodes."""
    rows = ROWS + sm_rows(SMS_H100)
    cross = [r for r in rows if isinstance(r, Cross)]
    for lo, hi in ((128, 129), (256, 257), (512, 513)):
        assert {lo, hi} <= {r.d for r in cross}, (lo, hi)
    assert 1024 in {r.d for r in cross}
    for vec in (1, 4):                                           # d % 4 of 0 and != 0 at each N class
        classes = {cross_vec_n(r.d)[1] for r in cross if cross_vec_n(r.d)[0] == vec}
        assert classes == ({1, 2, 4, 8} if vec == 4 else {1, 2, 4, 8, 16, 32}), (vec, classes)
    for lo, hi in ((32, 33), (64, 65), (128, 129), (256, 257), (512, 513)):    # the scalar-path classes
        assert any(cross_vec_n(r.d) == (1, cross_vec_n(hi)[1]) for r in cross) and hi in {r.d for r in cross}
        assert any(r.d % 4 and (r.d + 31) // 32 == (lo + 31) // 32 for r in cross), lo
    assert {1, 2, 3, 4, 5, 6, 7, 8} <= {r.L for r in cross} and {True, False} == {r.xl for r in cross}
    sms = SMS_H100
    bwd = [cross_bwd_launches(r.B, r.d, r.L, r.xl, sms)[0] for r in cross if r.B]
    assert {k[1][2] for k in bwd if k[0] == "cross_bwd_reg_kernel"} == {8, 12}            # both sides of B = 24 SMs
    assert ("cross_bwd_reg_kernel", (4, 4, 8)) in bwd and any(r.B >= 24 * sms and r.d == 512 and r.L == 4 for r in cross)
    assert {k[1][3] for k in bwd if k[0] == "cross_bwd_kernel" and k[1][0] == 4} == {True, False}   # the 160 KB cut-off
    ec = [r for r in ROWS if isinstance(r, ECross) and r.B]
    assert {embed_cross_launches(*r)[0][1][0] for r in ec} == {1, 2, 3, 4} and {r.L for r in ec} == {1, 2, 3, 4}
    assert {r.i32 for r in ec} == {True, False}
    din = [r for r in rows if isinstance(r, Din)]
    assert {4, 5, 8, 9, 16, 17, 32} <= {r.H for r in din}
    for hp in (4, 8, 16, 32):
        assert {8, 4} <= {din_bwd_warps(r.H, r.T) for r in din if din_hp(r.H) == hp and r.T}, hp
    bst = [r for r in rows if isinstance(r, Bst)]
    assert {4, 8, 16, 32, 64} <= {r.d for r in bst if r.B}
    bil = [r for r in ROWS if isinstance(r, Bil)]
    assert {8, 16, 32} < {r.K for r in bil} and set(BIL_MASKS) == {r.mask for r in bil}
    fwd_bs = {bilinear_rr_fwd_plan(r.F, r.K, r.mask)[1] for r in bil
              if any(k[0] == "bilinear_rr_fwd_kernel" for k in r.launches(sms)[0] or [])}
    bwd_bs = {bilinear_rr_bwd_plan(r.F, r.K, r.mask)[1] for r in bil
              if any(k[0] == "bilinear_rr_bwd_dx_kernel" for k in r.launches(sms)[1] or [])}
    assert {16, 8} <= fwd_bs and min(fwd_bs) < 8 and RR_GP in bwd_bs and min(bwd_bs) < RR_GP, (fwd_bs, bwd_bs)
    kts = {k[1][1] for r in bil for call in r.launches(sms) for k in call or [] if k[0].startswith("bilinear_rr_")}
    assert kts == {1, 2, 4}, kts
    kinds = {k[0] for r in bil for call in r.launches(sms) for k in call or []}
    assert {"bilinear_fwd_kernel", "bilinear_bwd_kernel", "bilinear_st_fwd_kernel", "bilinear_st_bwd_kernel"} <= kinds
    afm = [r for r in ROWS if isinstance(r, Afm) and r.B]
    for K, edges in ((4, (32, 64, 128, 256)), (8, (32, 64, 128, 256)), (16, (32, 64, 128)), (32, (32, 64))):
        Ts = {r.T for r in afm if r.K == K}
        assert all({e, e + 1} <= Ts for e in edges), (K, Ts)
        assert afm_tu(K, max(edges) + 1) is None
    fw = [r for r in rows if isinstance(r, Fwfm)]
    assert {True, False} == {r.K % 4 == 0 for r in fw if r.B}
    for r in sm_rows(sms):                                       # the last pass of every SM row is partial
        assert r.B % 2 == 1


def test_sm_rows_select_their_kernels():
    """CPU: each SM row, placed for an H100 SXM, selects the instantiation it is named for, and every loop-carrying
    backward instantiation among them is a multi-sample one; the GPU trace test checks the same on the device."""
    assert set(SM_KERNELS) == set(SM_ROWS)
    for name, make in SM_ROWS.items():
        row = make(SMS_H100)
        launched = [k for call in row.launches(SMS_H100) for k in call or []]
        assert SM_KERNELS[name] in launched, f"{name}: {row.id} launches {launched}, not {_fmt(SM_KERNELS[name])}"


def test_sm_rows_fill_three_passes():
    """CPU: at the H100 SXM's SM count, the SM-placed rows' batches cover three passes of every worker bound they use."""
    for name, make in SM_ROWS.items():
        row = make(SMS_H100)
        assert row.B >= 3 * SMS_H100, name
    assert cross_bwd_launches(SM_ROWS["cross-reg-N4-L4-8warps"](SMS_H100).B, 512, 4, False, SMS_H100) == \
        [("cross_bwd_reg_kernel", (4, 4, 8))]


# ================================================================================================ float64 references
def _seed(row):
    return zlib.crc32(row.id.encode())


CHUNK = 64


def chunked_reference(B, fn):
    """Runs the float64 oracle `fn(lo, hi) -> (per-sample dict, batch-reduced dict)` over chunks of CHUNK samples.

    Per-sample arrays are concatenated.  A batch-reduced gradient R = sum_c R_c is returned with the magnitude
    M = sum_c |R_c| of its chunks: the kernels add per-sample terms in fp32 (per warp or CTA, then across CTAs with
    atomics), so their rounding error scales with the size of the partial sums they form, not with |R|.  When ~25k
    samples' terms cancel, |R| can be far below those partial sums and a correct kernel misses TOL |R| element-wise.
    M is a float64 stand-in for those partial sums: 64-sample chunks are smaller than any partial sum the kernels form, so
    M is at least as large as the magnitudes their fp32 adds see.  The bar (check_reduced) is TOL max(|R| + rms(R), M),
    which is the plain element-wise bar wherever the chunks do not cancel."""
    per, red, mag = {}, {}, {}
    for lo in range(0, max(B, 1), CHUNK):
        p, r = fn(lo, min(lo + CHUNK, B))
        for k, v in p.items():
            per.setdefault(k, []).append(np.asarray(v, np.float64))
        for k, v in r.items():
            v = np.asarray(v, np.float64)
            red[k] = red.get(k, 0.0) + v
            mag[k] = mag.get(k, 0.0) + np.abs(v)
    return {k: np.concatenate(v) for k, v in per.items()}, {k: (red[k], mag[k]) for k in red}


def check_reduced(got, ref_mag, what):
    """Batch-reduced gradient against float64: |got - R| <= TOL max(|R| + rms(R), M) element-wise (see chunked_reference);
    a gradient whose every chunk is exactly zero must be exactly zero.  Returns the worst |got - R| / bound."""
    ref, mag = ref_mag
    got = got.detach().cpu().double().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
    got = got.reshape(ref.shape)
    rms = float(np.sqrt(np.mean(ref * ref))) if ref.size else 0.0
    bound = TOL * np.maximum(np.abs(ref) + rms, mag)
    err = np.abs(got - ref)
    zero = bound == 0
    assert np.all(got[zero] == 0), f"{what}: {int(np.count_nonzero(got[zero]))} elements must be exactly zero"
    worst = 0.0
    if (~zero).any():
        worst = float((err[~zero] / bound[~zero]).max())
        assert worst <= 1.0, (f"{what}: element-wise error is {worst:.2f}x the bound TOL max(|ref| + rms(ref), "
                              f"sum over 64-sample chunks |chunk ref|) (max error {float(err.max()):.3e})")
    return worst


def _f64(*arrays):
    return [np.asarray(a, np.float64) for a in arrays]


# --------------------------------------------------------------------------------------------------------- per family
def _cross_inputs(row):
    rng = np.random.default_rng(_seed(row))
    x0 = trunc_normal(rng, (row.B, row.d), 0.5)
    w = trunc_normal(rng, (row.L, row.d), (2.0 / row.d) ** 0.5)
    b = trunc_normal(rng, (row.L, row.d), 0.1)
    g = trunc_normal(rng, (row.B, row.d), 1.0)
    xs = trunc_normal(rng, (row.B, row.d), 0.5) if row.xl else None
    return x0, w, b, g, xs


def _cross_reference(row, inputs):
    x0, w, b, g, xs = inputs
    w64, b64 = _f64(w, b)

    def fn(lo, hi):
        if xs is None:
            a0, gg = _f64(x0[lo:hi], g[lo:hi])
            out = O.cross_stack_fwd(a0, w64, b64)[-1]
            dx0, dw, db = O.cross_stack_bwd(a0, w64, b64, gg)
            return {"out": out, "dx0": dx0}, {"dw": dw, "db": db}
        t = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)     # the fuzz test's restatement
        x0t, st, wt, bt = t(x0[lo:hi]), t(xs[lo:hi]), t(w), t(b)
        x = st
        for l in range(row.L):
            x = x0t * (x @ wt[l])[:, None] + bt[l][None, :] + x
        x.backward(torch.tensor(np.asarray(g[lo:hi], np.float64)))
        return ({"out": x.detach().numpy(), "dx0": x0t.grad.numpy(), "dxl": st.grad.numpy()},
                {"dw": wt.grad.numpy(), "db": bt.grad.numpy()})
    return chunked_reference(row.B, fn)


def _run_cross(row, inputs):
    from recalgorithm_b200 import ops
    x0, w, b, g, xs = inputs
    xs_d = dev(xs) if xs is not None else None
    out = ops.cross_fwd(dev(x0), dev(w), dev(b), xl_in=xs_d)
    dx0, dxl, dw, db = ops.cross_bwd(dev(x0), dev(w), dev(b), dev(g), xl_in=xs_d)
    return {"out": out, "dx0": dx0, "dxl": dxl, "dw": dw, "db": db}


def _check_cross(row, inputs, res):
    per, red = _cross_reference(row, inputs)
    if row.B == 0:
        assert res["out"].shape == (0, row.d)
    else:
        assert_close(res["out"], per["out"], TOL, f"{row.id}: forward")
        assert_close(res["dx0"], per["dx0"], TOL, f"{row.id}: dx0")
        if row.xl:
            assert_close(res["dxl"], per["dxl"], TOL, f"{row.id}: dxl_in")
    check_reduced(res["dw"], red["dw"], f"{row.id}: dw")
    check_reduced(res["db"], red["db"], f"{row.id}: db")


def _ecross_inputs(row):
    rng = np.random.default_rng(_seed(row))
    V = 50
    table = trunc_normal(rng, (row.F * V, row.D), 0.5)
    off = (np.arange(row.F + 1) * V).astype(np.int64)
    ids = rng.integers(-1, V, size=(row.B, row.F)).astype(np.int64)        # -1: the zero vector
    d = row.F * row.D
    w = trunc_normal(rng, (row.L, d), (2.0 / d) ** 0.5)
    b = trunc_normal(rng, (row.L, d), 0.1)
    return table, off, ids, w, b


def _run_ecross(row, inputs):
    from recalgorithm_b200 import ops
    table, off, ids, w, b = inputs
    x0, out = ops.embed_cross_fwd(dev(table), dev(off), dev(ids, torch.int32 if row.i32 else torch.int64), dev(w), dev(b))
    return {"x0": x0, "out": out}


def _check_ecross(row, inputs, res):
    table, off, ids, w, b = inputs
    e = O.embedding_lookup(table, ids, off).reshape(row.B, row.F * row.D)
    assert np.array_equal(res["x0"].cpu().numpy(), e), f"{row.id}: the gathered x0 must be bit-exact"
    if row.B:
        assert_close(res["out"], O.cross_stack_fwd(*_f64(e, w, b))[-1], TOL, f"{row.id}: forward")


DIN_PARAMS = ("w1", "b1", "w2", "b2", "w3", "b3")


def _din_inputs(row):
    rng = np.random.default_rng(_seed(row))
    B, T, H = row.B, row.T, row.H
    q = trunc_normal(rng, (B, H), 0.5)
    k = trunc_normal(rng, (B, T, H), 0.5)
    lens = rng.integers(0, T + 1, size=B).astype(np.int64)
    if B:
        lens[0], lens[-1] = 0, T
    ws = [trunc_normal(rng, s, sd) for s, sd in (((4 * H, 64), 0.2), ((64,), 0.1), ((64, 32), 0.2), ((32,), 0.1),
                                                  ((32, 1), 0.3), ((1,), 0.1))]
    g = trunc_normal(rng, (B, H), 1.0)
    # A pre-activation within float32 rounding of 0 may take either side of a relu in the kernel, which changes that
    # position's whole gradient path without any fault (seen at 3.5e-8 in a 9.5k-sample row).  Keys whose layer-1 or
    # layer-2 pre-activation lies closer than 1e-6 to 0 are redrawn.
    w64 = _f64(*ws)
    for _ in range(20):
        qq, kk = _f64(q, k)
        qb = np.broadcast_to(qq[:, None, :], kk.shape)
        p1 = np.concatenate([qb, kk, qb - kk, qb * kk], axis=-1) @ w64[0] + w64[1]
        p2 = np.maximum(p1, 0) @ w64[2] + w64[3]
        near = np.minimum(np.abs(p1).min(-1), np.abs(p2).min(-1)) < 1e-6
        bad = np.argwhere(near & (np.arange(T)[None, :] < lens[:, None]))
        if not len(bad):
            break
        k[bad[:, 0], bad[:, 1]] = trunc_normal(rng, (len(bad), H), 0.5)
    else:
        raise AssertionError(f"{row.id}: could not draw inputs clear of the relu kinks")
    return q, k, lens, ws, g


def _run_din(row, inputs):
    from recalgorithm_b200 import ops
    q, k, lens, ws, g = inputs
    args = (dev(q), dev(k), dev(lens), *[dev(w) for w in ws])
    res = {}
    for tag, balanced in (("", True), ("static_", False)):
        res[tag + "out"] = ops.din_attention_fwd(*args, is_softmax=row.soft, balanced=balanced)
        res[tag + "d_query"], res[tag + "d_keys"], res[tag + "d_params"] = ops.din_attention_bwd(
            *args, dev(g), is_softmax=row.soft, balanced=balanced)
    return res


def _check_din(row, inputs, res):
    q, k, lens, ws, g = inputs
    w64 = _f64(*ws)

    def fn(lo, hi):
        qq, kk, gg = _f64(q[lo:hi], k[lo:hi], g[lo:hi])
        out, c = O.din_attention_fwd(qq, kk, lens[lo:hi], *w64, is_softmax=row.soft, return_cache=True)
        gr = O.din_attention_bwd(qq, kk, lens[lo:hi], *w64, gg, is_softmax=row.soft)
        # scale of the softmax ds terms, ds_bt = w_bt (dw_bt - sum_t' w_bt' dw_bt') / sqrt(H), dw_bt = g_b . k_bt
        # (oracle/layers_np.py:360-364): |ds_bt| <= w_bt (a_bt + A_b) / sqrt(H), a_bt = sum_h |g_bh k_bth|, A_b = sum_t w_bt a_bt
        wt = (c["w"] * c["mask"])[..., 0]
        a = np.einsum("bh,bth->bt", np.abs(gg), np.abs(kk))
        ds_scale = (wt * (a + (wt * a).sum(1, keepdims=True))).sum() / np.sqrt(row.H)
        return {"out": out, "d_query": gr["query"], "d_keys": gr["keys"]}, {**{n: gr[n] for n in DIN_PARAMS},
                                                                            "ds_scale": ds_scale}
    per, red = chunked_reference(row.B, fn)
    for tag in ("", "static_"):
        what = f"{row.id} ({'static' if tag else 'balanced'} schedule)"
        if row.B and row.T:
            assert_close(res[tag + "out"], per["out"], TOL, f"{what}: out")
            assert_close(res[tag + "d_query"], per["d_query"], TOL, f"{what}: d_query")
            assert_close(res[tag + "d_keys"], per["d_keys"], TOL, f"{what}: d_keys")
            dk = res[tag + "d_keys"].cpu().numpy()
            masked = np.arange(row.T)[None, :] >= lens[:, None]
            if row.soft:                      # under softmax a history of length 0 attends uniformly, as in the reference
                masked &= lens[:, None] > 0
            assert np.all(dk[masked] == 0), f"{what}: d_keys of masked positions must be exactly zero"
        for got, name in zip(res[tag + "d_params"], DIN_PARAMS):
            if row.soft and name == "b3":
                # d/db3 = sum_b sum_t ds_bt vanishes analytically under softmax (shift invariance: sum_t ds_bt = 0 per
                # sample), so every chunk is ~0 and the float32 result is rounding alone: of each ds term, whose
                # inputs are the H-term dot product dw and the T-term sum over w dw (error ~ (H + T) eps (a + A) w), and
                # of the sum of the terms.  Both scale with S = sum_{b,t} w_bt (a_bt + A_b) / sqrt(H), the bound on
                # sum |ds_bt| above; TOL S is 170 float32 epsilons of it.
                ref, _ = red["b3"]
                scale = float(red["ds_scale"][0])
                assert abs(float(got.sum()) - float(ref.sum())) <= TOL * scale, \
                    f"{what}: d_b3 = {float(got.sum()):.3e}, float64 {float(ref.sum()):.3e}, allowed {TOL * scale:.3e}"
            else:
                check_reduced(got, red[name], f"{what}: d_{name}")
    # the two schedules assign samples to warps differently; every per-sample result is the same bit for bit
    assert torch.equal(res["out"], res["static_out"]), f"{row.id}: out differs between the schedules"
    assert torch.equal(res["d_query"], res["static_d_query"]), f"{row.id}: d_query differs between the schedules"
    assert torch.equal(res["d_keys"], res["static_d_keys"]), f"{row.id}: d_keys differs between the schedules"


def _bst_inputs(row):
    rng = np.random.default_rng(_seed(row))
    B, T, d, H = row.B, row.T, row.d, row.heads
    q, k, v = (trunc_normal(rng, (B, T, d), 1.0) for _ in range(3))
    lens = rng.integers(0, T + 1, size=B).astype(np.int64)
    if B:
        lens[0], lens[-1] = 0, T
    p = {n: trunc_normal(rng, s, 0.4) for n, s in O.bst_param_shapes(d, H, T).items()}
    p["ln1_gamma"] = 1 + p["ln1_gamma"]
    p["ln2_gamma"] = 1 + p["ln2_gamma"]
    g = trunc_normal(rng, (B, T, d), 1.0)
    return q, k, v, lens, p, g


def _run_bst(row, inputs):
    from recalgorithm_b200 import ops
    q, k, v, lens, p, g = inputs
    packed = ops.bst_pack_params({n: dev(a) for n, a in p.items()}, row.d, row.heads, row.T)
    args = (dev(q), dev(k), dev(v), dev(lens), packed)
    out = ops.bst_transformer_fwd(*args, row.heads, row.T, row.pos)
    dq, dk, dv, dp = ops.bst_transformer_bwd(*args, dev(g), row.heads, row.T, row.pos)
    return {"out": out, "dq": dq, "dk": dk, "dv": dv, "dp": ops.bst_unpack_params(dp, row.d, row.heads, row.T)}


def _check_bst(row, inputs, res):
    q, k, v, lens, p, g = inputs

    def fn(lo, hi):
        if hi == lo:
            return {}, {n: np.zeros(a.shape) for n, a in p.items()}
        out, dq, dk, dv, dp = bst_torch.bst_transformer_bwd(q[lo:hi], k[lo:hi], v[lo:hi], lens[lo:hi], p, row.heads,
                                                            g[lo:hi], use_position_embedding=row.pos)
        return {"out": out, "dq": dq, "dk": dk, "dv": dv}, dp
    per, red = chunked_reference(row.B, fn)
    if row.B:
        assert_close(res["out"], per["out"], TOL, f"{row.id}: forward")
        for n in ("dq", "dk", "dv"):
            assert_close(res[n], per[n], TOL, f"{row.id}: {n}")
    for n in O.BST_PARAM_ORDER:
        check_reduced(res["dp"][n], red[n], f"{row.id}: d_{n}")


def _senet_inputs(row):
    rng = np.random.default_rng(_seed(row))
    x = trunc_normal(rng, (row.B, row.F, row.K), 1.0)
    w1 = trunc_normal(rng, (row.F, row.r), 0.5)
    w2 = trunc_normal(rng, (row.r, row.F), 0.5)
    g = trunc_normal(rng, (row.B, row.F, row.K), 1.0)
    return x, w1, w2, g


def _run_senet(row, inputs):
    from recalgorithm_b200 import ops
    x, w1, w2, g = (dev(a) for a in inputs)
    out = ops.senet_fwd(x, w1, w2)
    dx, dw1, dw2 = ops.senet_bwd(x, w1, w2, g)
    return {"out": out, "dx": dx, "dw1": dw1, "dw2": dw2}


def _check_senet(row, inputs, res):
    x, w1, w2, g = _f64(*inputs)

    def fn(lo, hi):
        dx, dw1, dw2 = O.senet_bwd(x[lo:hi], w1, w2, g[lo:hi])
        return {"out": O.senet_fwd(x[lo:hi], w1, w2), "dx": dx}, {"dw1": dw1, "dw2": dw2}
    per, red = chunked_reference(row.B, fn)
    if row.B:
        assert_close(res["out"], per["out"], TOL, f"{row.id}: forward")
        assert_close(res["dx"], per["dx"], TOL, f"{row.id}: dx")
    check_reduced(res["dw1"], red["dw1"], f"{row.id}: dw1")
    check_reduced(res["dw2"], red["dw2"], f"{row.id}: dw2")


def _bil_inputs(row):
    from recalgorithm_b200 import ops
    rng = np.random.default_rng(_seed(row))
    P = (row.F - 1) * (row.F - 2) // 2
    x = trunc_normal(rng, (row.B, row.F, row.K), 0.5)
    w = trunc_normal(rng, ops.bilinear_w_shape(row.F, row.K, row.type), 0.3)
    g = trunc_normal(rng, (row.B, P, row.K), 1.0)
    return x, w, g


def _run_bil(row, inputs):
    from recalgorithm_b200 import ops
    x, w, g = (dev(a) for a in inputs)
    prev = ops.bilinear_set_tournament(row.mask)
    try:
        out = ops.bilinear_fwd(x, w, row.type)
        dx, dw = ops.bilinear_bwd(x, w, row.type, g)
        torch.cuda.synchronize()
    finally:
        ops.bilinear_set_tournament(prev)
    return {"out": out, "dx": dx, "dw": dw}


def _check_bil(row, inputs, res):
    x, w, g = _f64(*inputs)
    if g.shape[1] == 0:                                   # F = 2: no pair, and the library is not called
        assert res["out"].numel() == 0 and torch.count_nonzero(res["dx"]) == 0 and torch.count_nonzero(res["dw"]) == 0
        return

    def fn(lo, hi):
        dx, dw = O.bilinear_bwd(x[lo:hi], w, row.type, g[lo:hi])
        return {"out": O.bilinear_fwd(x[lo:hi], w, row.type), "dx": dx}, {"dw": dw}
    per, red = chunked_reference(row.B, fn)
    assert_close(res["out"], per["out"], TOL, f"{row.id}: forward")
    assert_close(res["dx"], per["dx"], TOL, f"{row.id}: dx")
    assert torch.count_nonzero(res["dx"][:, -1]) == 0, f"{row.id}: the last field takes no part: its dx must be exactly zero"
    check_reduced(res["dw"], red["dw"], f"{row.id}: dw")


def _pw_inputs(row):
    rng = np.random.default_rng(_seed(row))
    B, F, K = row.B, row.F, row.K
    if isinstance(row, Ffm):
        return trunc_normal(rng, (B, F, F - 1, K), 0.5), trunc_normal(rng, (B, 1), 1.0)
    tile = trunc_normal(rng, (B, F, K), 0.5)
    if isinstance(row, Fwfm):
        return tile, trunc_normal(rng, (F * (F - 1) // 2,), 0.5), trunc_normal(rng, (B, 1), 1.0)
    T = row.T
    return (tile, trunc_normal(rng, (K, T), (2.0 / (K + T)) ** 0.5), trunc_normal(rng, (T,), 0.1),
            trunc_normal(rng, (T, 1), 0.5), trunc_normal(rng, (B, K), 1.0))


def _run_pw(row, inputs):
    from recalgorithm_b200 import ops
    a = [dev(x) for x in inputs]
    if isinstance(row, Ffm):
        out = ops.ffm_fwd(a[0])
        return {"out": out, "d_tile": ops.ffm_bwd(a[0], a[1])}
    if isinstance(row, Fwfm):
        out = ops.fwfm_fwd(a[0], a[1])
        d_tile, d_r = ops.fwfm_bwd(a[0], a[1], a[2])
        return {"out": out, "d_tile": d_tile, "d_r": d_r}
    out = ops.afm_fwd(*a[:4])
    d_tile, d_w, d_b, d_h = ops.afm_bwd(*a)
    return {"out": out, "d_tile": d_tile, "d_w": d_w, "d_b": d_b, "d_h": d_h}


def _check_pw(row, inputs, res):
    a = _f64(*inputs)
    if isinstance(row, Ffm):
        fn = lambda lo, hi: ({"out": O.ffm_fwd(a[0][lo:hi]), "d_tile": O.ffm_bwd(a[0][lo:hi], a[1][lo:hi])}, {})
    elif isinstance(row, Fwfm):
        def fn(lo, hi):
            de, dr = O.fwfm_bwd(a[0][lo:hi], a[1], a[2][lo:hi])
            return {"out": O.fwfm_fwd(a[0][lo:hi], a[1]), "d_tile": de}, {"d_r": dr}
    else:
        def fn(lo, hi):
            de, dw, db, dh = O.afm_bwd(a[0][lo:hi], a[1], a[2], a[3], a[4][lo:hi])
            return {"out": O.afm_fwd(a[0][lo:hi], a[1], a[2], a[3]), "d_tile": de}, {"d_w": dw, "d_b": db, "d_h": dh}
    per, red = chunked_reference(row.B, fn)
    if row.B:
        assert_close(res["out"], per["out"], TOL, f"{row.id}: forward")
        assert_close(res["d_tile"], per["d_tile"], TOL, f"{row.id}: d_tile")
    for name, rm in red.items():
        check_reduced(res[name], rm, f"{row.id}: {name}")


FAMILIES = {Cross: (_cross_inputs, _run_cross, _check_cross), ECross: (_ecross_inputs, _run_ecross, _check_ecross),
            Din: (_din_inputs, _run_din, _check_din), Bst: (_bst_inputs, _run_bst, _check_bst),
            Senet: (_senet_inputs, _run_senet, _check_senet), Bil: (_bil_inputs, _run_bil, _check_bil),
            Fwfm: (_pw_inputs, _run_pw, _check_pw), Afm: (_pw_inputs, _run_pw, _check_pw), Ffm: (_pw_inputs, _run_pw, _check_pw)}


def _refused(row, sms):
    return any(call is None for call in row.launches(sms))


def _execute(row, inputs, sms):
    """Runs the row's calls; a row the mirror says is refused must raise the library's 'unsupported' error."""
    from recalgorithm_b200 import _lib
    run = FAMILIES[type(row)][1]
    if _refused(row, sms):
        with pytest.raises(_lib.CtrError) as err:
            run(row, inputs)
        assert err.value.code == _lib.CTR_ERR_UNSUPPORTED
        torch.cuda.synchronize()
        return None
    res = run(row, inputs)
    torch.cuda.synchronize()
    return res


# ================================================================================================ GPU: parity and dispatch
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _resolve(param):
    return SM_ROWS[param](_sms()) if isinstance(param, str) else param


PARAMS = ROWS + BASELINE_ROWS + list(SM_ROWS)
PARAM_IDS = [p if isinstance(p, str) else p.id for p in PARAMS]


@pytest.mark.gpu
@pytest.mark.parametrize("param", PARAMS, ids=PARAM_IDS)
def test_row_against_float64(param):
    row = _resolve(param)
    make, _, check = FAMILIES[type(row)]
    inputs = make(row)
    res = _execute(row, inputs, _sms())
    if res is not None:
        check(row, inputs, res)


_KERNEL = re.compile(r"ctr::(?:\w+::)*(\w+)(?:<([^<>]*)>)?\(")


def _template_args(text):
    out = []
    for a in (text or "").split(","):
        a = a.strip()
        if a:
            out.append(True if a == "true" else False if a == "false" else int(a) if re.fullmatch(r"-?\d+", a) else a)
    return tuple(out)


def _traced_kernels(fn, expected):
    """[(name, template arguments, grid, block)] of the kernels `fn` launches, in launch order (kineto's chrome trace)."""
    from torch.profiler import ProfilerActivity, profile
    fn()                                                                  # first launches (module load) outside the trace
    for _ in range(3):                       # a session now and then hands back an empty or partial device trace; a new one records
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "trace.json")
            prof.export_chrome_trace(path)
            with open(path) as f:
                events = json.load(f).get("traceEvents", [])
        kernels = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
        out = []
        for e in kernels:
            hit = _KERNEL.search(e["name"])
            if hit:
                args = e.get("args", {})
                out.append((hit.group(1), _template_args(hit.group(2)), args.get("grid"), args.get("block")))
        if kernels and [(n, a) for n, a, _, _ in out] == expected:
            break
    if not kernels and expected:
        pytest.skip("torch.profiler recorded no CUDA kernels on this machine")
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("param", PARAMS, ids=PARAM_IDS)
def test_row_launches_what_the_mirror_predicts(param):
    """The kernels the library launches for the row are the mirror's, in order, with the same template arguments -- this
    keeps the mirror, and with it the coverage claim above, honest.  On the SM-placed rows, the grids of the backward's
    loop kernels also show that every worker had at least three work items, so the loop ran past its first sample."""
    sms = _sms()
    row = _resolve(param)
    inputs = FAMILIES[type(row)][0](row)
    expected = [k for call in row.launches(sms) for k in (call or [])]
    launched = _traced_kernels(lambda: _execute(row, inputs, sms), expected)
    assert [(n, a) for n, a, _, _ in launched] == expected, \
        f"{row.id}: launched {[(n, a) for n, a, _, _ in launched]}, the mirror predicts {expected}"
    if not isinstance(param, str):
        return
    bwd = set(row.launches(sms)[-1 if not isinstance(row, Din) else 1] or [])
    checked = 0
    for name, args, grid, block in launched:
        if (name, args) not in bwd or name not in WORKERS:
            continue
        if grid is None or block is None:
            pytest.skip("the trace does not carry kernel grid / block; the three-pass check needs them")
        workers = grid[0] * (block[0] // 32 if WORKERS[name] == "warp" else 1)
        if name == "cross_bwd_kernel":
            unit = 8
        elif name == "bilinear_rr_fwd_kernel":
            unit = bilinear_rr_fwd_plan(row.F, row.K, row.mask)[1]
        elif name == "bilinear_rr_bwd_dx_kernel":
            unit = bilinear_rr_bwd_plan(row.F, row.K, row.mask)[1]
        else:
            unit = 1
        assert 3 * workers * unit <= row.B, f"{row.id}: {name} ran {workers} workers of {unit} samples for B = {row.B}"
        assert workers < row.B / 2
        checked += 1
    assert checked, f"{row.id}: no loop kernel in the backward"


# ================================================================================================ C ABI: split dw / db
@pytest.mark.gpu
@pytest.mark.parametrize("d,L,xl", [(256, 3, False), (256, 3, True), (130, 6, False)],
                         ids=["register-path", "staged-xl", "staged-scalar"])
def test_cross_bwd_separate_dw_db(d, L, xl):
    """ctr_cross_bwd with dw and db in separate allocations (ops.cross_bwd always puts them back to back and takes the one
    memset branch): both are zeroed by their own memsets and nothing between them is touched."""
    from recalgorithm_b200 import _lib, ops
    sms = _sms()
    row = Cross(3 * 16 * sms + 5, d, L, xl)
    x0, w, b, g, xs = inputs = _cross_inputs(row)
    per, red = _cross_reference(row, inputs)
    n = L * d
    buf = torch.full((4 * n,), float("nan"), device="cuda")          # dw = [0, n), db = [2n, 3n): stale NaN everywhere
    dw, db = buf[:n], buf[2 * n:3 * n]
    x0d, wd, bd, gd = dev(x0), dev(w), dev(b), dev(g)
    xsd = dev(xs) if xl else None
    dx0, dxl = torch.empty_like(x0d), torch.empty_like(x0d) if xl else None
    _lib.check(_lib.lib().ctr_cross_bwd(ops._ptr(x0d), ops._ptr(xsd), ops._ptr(wd), ops._ptr(bd), ops._ptr(gd), row.B, d, L,
                                        ops._ptr(dx0), ops._ptr(dxl), ops._ptr(dw), ops._ptr(db), ops._stream()))
    torch.cuda.synchronize()
    assert cross_bwd_launches(row.B, d, L, xl, sms)[0][0] == ("cross_bwd_reg_kernel" if not xl and L <= 4 and d % 4 == 0
                                                              else "cross_bwd_kernel")
    assert torch.isnan(buf[n:2 * n]).all() and torch.isnan(buf[3 * n:]).all(), "memory between / after dw and db was written"
    assert_close(dx0, per["dx0"], TOL, "dx0")
    if xl:
        assert_close(dxl, per["dxl"], TOL, "dxl_in")
    check_reduced(dw.reshape(L, d), red["dw"], "dw")
    check_reduced(db.reshape(L, d), red["db"], "db")
