"""Every wgmma instantiation of the CIN and PNN kernels against float64, at its tile and dispatch boundaries.

Each tensor-core kernel (csrc/cin.cu, csrc/cin_bwd.cu, csrc/pnn.cu) is a template, and the host picks the instantiation from
the shape.  This file holds
  * a pure-Python mirror of that host dispatch (shape, method, precision -> the kernels launched, with template integers),
  * one table of shapes on both sides of every dispatch boundary,
  * a CPU test that the mirror over the table reaches exactly the `*_tc_kernel` instantiations the built library contains,
  * GPU tests: every row forward and backward against float64, and the launched kernels (torch.profiler) against the mirror,
  * the single-pass TF32 forward (`precision=1`) against an emulation of its rounding, under a bound derived from the
    length of its accumulation chains.
"""
import os
import re
import shutil
import subprocess
import zlib
from typing import NamedTuple

import numpy as np
import pytest
import torch

from _pnn_ref import pnn_bwd as pnn_ref_bwd, pnn_fwd as pnn_ref_fwd
from _util import TOL, assert_close, dev, trunc_normal
from oracle import layers_np as O


# ================================================================================================ dispatch mirror
def _pad3(v):
    return 32 if v <= 32 else 64 if v <= 64 else 128


def cin_fwd_launches(B, m, hk, D, H, precision):
    """Kernels `ctr_cin_fwd` launches, in order: [(base name, template integers)].

    cin.cu:210-211  return m >= 1 && m <= KB && hk >= 1 && H >= 1 && H <= 128 && D >= 1 && D <= 32 && (D & (D - 1)) == 0;
    cin.cu:234      if (B == 0) return CTR_OK;
    cin.cu:236-241  if (!tensor_path_ok(m, hk, D, H)) { ... return launch(..., cin_fwd_simple_kernel, ...); }
    cin.cu:243      const int NP = pad3(H);   tc_ptx.cuh:329  pad3: v <= 32 ? 32 : v <= 64 ? 64 : 128
    cin.cu:249      launch(..., cin_split_filter_kernel, ...)
    cin.cu:261-265  precision 0: PASSES 3, SB 4; precision 1: PASSES 1, SB 6 -> cin_fwd_tc_kernel<PASSES, SB, NP>
    """
    if B == 0:
        return []
    if not (1 <= m <= 32 and hk >= 1 and 1 <= H <= 128 and 1 <= D <= 32 and D & (D - 1) == 0):
        return [("cin_fwd_simple_kernel", ())]
    NP = _pad3(H)
    return [("cin_split_filter_kernel", ()), ("cin_fwd_tc_kernel", (3, 4, NP) if precision == 0 else (1, 6, NP))]


def cin_bwd_launches(B, m, hk, D, H):
    """Kernels `ctr_cin_bwd` launches, in order; None when it refuses the shape (raises CtrError).

    cin_bwd.cu:377      CTR_UNSUPPORTED(D > 256 || H > 256, ...)
    cin_bwd.cu:380      if (B == 0) return CTR_OK;
    cin_bwd.cu:353-354  tensor_path_ok: return m >= 1 && m <= 32 && hk >= 1 && H >= 1 && H <= 128 && (D == 8 || D == 16 || D == 32);
    cin_bwd.cu:383-398  if (!tensor_path_ok(m, hk, D, H)) { launch cin_bwd_dx_kernel, cin_bwd_dw_kernel }
    cin_bwd.cu:402-403  HP = pad_to(H, 32);  NP = pad3(H);   (pad3: v <= 32 ? 32 : v <= 64 ? 64 : 128)
    cin_bwd.cu:406-410  launch split_filter_native_kernel, split_grad_kernel
    cin_bwd.cu:423-431  SB = 3; nkb = HP / 32;  cin_bwd_dx_tc_kernel<SB, nkb>
    cin_bwd.cu:453-455  cin_bwd_dw_tc_kernel<NP, D>
    """
    if D > 256 or H > 256:
        return None
    if B == 0:
        return []
    if 1 <= m <= 32 and hk >= 1 and 1 <= H <= 128 and D in (8, 16, 32):
        return [("split_filter_native_kernel", ()), ("split_grad_kernel", ()),
                ("cin_bwd_dx_tc_kernel", (3, (H + 31) // 32)), ("cin_bwd_dw_tc_kernel", (_pad3(H), D))]
    return [("cin_bwd_dx_kernel", ()), ("cin_bwd_dw_kernel", ())]


def pnn_widths(F, K, N, method):
    """(WX, tensor path?, WP): pnn.cu:618-620  WX = FK + Q + 1;  tc = WX <= 128 && N % 4 == 0;  WP = pad3(WX)."""
    Q = F * (F + 1) // 2 if method == 0 else K * (K + 1) // 2
    WX = F * K + Q + 1
    return WX, WX <= 128 and N % 4 == 0, _pad3(WX)


def pnn_fwd_launches(B, F, K, N, method):
    """Kernels `ctr_pnn_fwd` launches, in order.

    pnn.cu:661          if (B == 0) return CTR_OK;
    pnn.cu:665-666      if (s.tc) { launch pnn_prep_kernel
    pnn.cu:678-682        pnn_fwd_tc_kernel<WP, SB, method>, SB = WP == 32 ? 4 : WP == 64 ? 3 : 2
    pnn.cu:689-696      } else pnn_prep_kernel, pnn_fwd_simple_kernel<method>
    """
    if B == 0:
        return []
    _, tc, WP = pnn_widths(F, K, N, method)
    if tc:
        return [("pnn_prep_kernel", ()), ("pnn_fwd_tc_kernel", (WP, {32: 4, 64: 3, 128: 2}[WP], method))]
    return [("pnn_prep_kernel", ()), ("pnn_fwd_simple_kernel", (method,))]


def pnn_bwd_launches(B, F, K, N, method):
    """Kernels `ctr_pnn_bwd` launches, in order.

    pnn.cu:715-717      if (B > 0 && s.tc) { launch pnn_prep_kernel
    pnn.cu:738            pnn_bwd_dx_tc_kernel<WP, 4, method>
    pnn.cu:741            pnn_bwd_dw_tc_kernel<WP, method>
    pnn.cu:746-764      } else if (B > 0) { pnn_prep_kernel, pnn_bwd_dx_simple_kernel<method>, pnn_bwd_dw_simple_kernel<method> }
    pnn.cu:768          launch pnn_fold_kernel   (always: at B = 0 it writes the zero weight gradients)
    """
    _, tc, WP = pnn_widths(F, K, N, method)
    if B > 0 and tc:
        ks = [("pnn_prep_kernel", ()), ("pnn_bwd_dx_tc_kernel", (WP, 4, method)), ("pnn_bwd_dw_tc_kernel", (WP, method))]
    elif B > 0:
        ks = [("pnn_prep_kernel", ()), ("pnn_bwd_dx_simple_kernel", (method,)), ("pnn_bwd_dw_simple_kernel", (method,))]
    else:
        ks = []
    return ks + [("pnn_fold_kernel", ())]


# The SM-count-dependent schedule parameters the SM-edge rows are placed on.
def cin_row_tiles(B, D):
    """Persistent 128-row tiles of the CIN forward and dX kernels: cin.cu:257-258, cin_bwd.cu:426-427."""
    return (B * D + 127) // 128


def pnn_fwd_nsplit(B, N, sms):
    """pnn.cu:672-675  n_btiles = ceil(B / 128); nsplit = sms / n_btiles clamped to [1, NT], NT = ceil(N / 64)."""
    n_btiles, NT = (B + 127) // 128, (N + 63) // 64
    return min(max(sms // n_btiles, 1), NT)


def pnn_dw_chunks_per_slice(B, N, sms):
    """32-sample chunks per batch slice of pnn_bwd_dw_tc_kernel (8 chunks per accumulation chain): pnn.cu:731-732, 397,
    tc_ptx.cuh:264-268, 377-381."""
    ngroups, chunks = (N + 127) // 128, (B + 31) // 32
    nslices = min(max(sms // ngroups, 1), chunks)
    return -(-chunks // nslices)


def cin_dw_schedule(B, hk, D, sms):
    """(nslices, samples per slice, samples per accumulation chain) of cin_bwd_dw_tc_kernel: cin_bwd.cu:449-452, 200,
    tc_ptx.cuh:264-268, 377-381."""
    ngroups = (hk + 3) // 4
    nslices = min(max(sms // ngroups, 1), B)
    return nslices, -(-B // nslices), 256 // D


# ================================================================================================ shape table
class Cin(NamedTuple):
    B: int
    m: int
    hk: int
    D: int
    H: int
    precision: int = 0          # 1: the forward also runs the single-pass TF32 kernel (the 3xTF32 one always runs)

    @property
    def id(self):
        return f"cin-B{self.B}-m{self.m}-hk{self.hk}-D{self.D}-H{self.H}" + ("-tf32" if self.precision else "")

    def launches(self):
        """Expected kernels of the row's calls: forward (3xTF32), [forward (TF32)], backward (None entry: refused)."""
        calls = [cin_fwd_launches(self.B, self.m, self.hk, self.D, self.H, 0)]
        if self.precision:
            calls.append(cin_fwd_launches(self.B, self.m, self.hk, self.D, self.H, 1))
        calls.append(cin_bwd_launches(self.B, self.m, self.hk, self.D, self.H))
        return calls


class Pnn(NamedTuple):
    B: int
    F: int
    K: int
    N: int
    method: int

    @property
    def id(self):
        wx = pnn_widths(self.F, self.K, self.N, self.method)[0]
        return f"{'ipnn' if self.method == 0 else 'opnn'}-B{self.B}-F{self.F}-K{self.K}-N{self.N}-WX{wx}"

    def launches(self):
        return [pnn_fwd_launches(*self), pnn_bwd_launches(*self)]


# Comments name the instantiations (forward | dX | dW) and the edges each row sits on.  Odd hk around the ring depths: the
# 3xTF32 forward has SB = 4 and 8-block chains, the TF32 forward SB = 6 and 32-block chains, the CIN dX kernel SB = 3.
ROWS = [
    Cin(1, 32, 9, 32, 32),        # <3,4,32> | <3,1> | <32,32>   B = 1, m = 32, H = 32, D = 32; hk = 9: two chains (8 + 1)
    Cin(5, 33, 3, 32, 32),        # m = 33: CUDA-core forward and backward
    Cin(129, 7, 13, 16, 33),      # <3,4,64> | <3,2> | <64,16>   H = 33, B*D = 16.1 tiles
    Cin(128, 10, 17, 16, 64),     # <3,4,64> | <3,2> | <64,16>   H = 64, B*D = 16 full tiles, hk = 17: three chains
    Cin(33, 12, 15, 8, 65),       # <3,4,128> | <3,3> | <128,8>  H = 65
    Cin(31, 8, 11, 8, 96),        # <3,4,128> | <3,3> | <128,8>  H = 96
    Cin(127, 16, 7, 32, 97),      # <3,4,128> | <3,4> | <128,32> H = 97
    Cin(64, 6, 5, 16, 128),       # <3,4,128> | <3,4> | <128,16> H = 128
    Cin(9, 6, 5, 16, 129),        # H = 129: CUDA-core forward and backward
    Cin(4, 5, 4, 8, 256),         # H = 256: the largest H the CUDA-core backward takes
    Cin(2, 3, 2, 8, 257),         # H = 257: backward refused
    Cin(6, 7, 5, 12, 20),         # D = 12: CUDA-core forward and backward
    Cin(3, 6, 4, 64, 40),         # D = 64: CUDA-core forward and backward
    Cin(2, 2, 2, 257, 3),         # D = 257: CUDA-core forward, backward refused
    Cin(300, 9, 6, 1, 24),        # D = 1: <3,4,32>, CUDA-core backward
    Cin(70, 31, 5, 2, 70),        # D = 2: <3,4,128>, CUDA-core backward
    Cin(50, 4, 3, 4, 40),         # D = 4: <3,4,64>, CUDA-core backward
    Cin(65, 11, 1, 8, 16),        # <3,4,32> | <3,1> | <32,8>    hk = 1
    Cin(40, 20, 6, 16, 1),        # <3,4,32> | <3,1> | <32,16>   H = 1
    Cin(20, 13, 9, 8, 50),        # <3,4,64> | <3,2> | <64,8>
    Cin(18, 25, 3, 32, 48),       # <3,4,64> | <3,2> | <64,32>
    Cin(7, 9, 7, 32, 20, 1),      # TF32 <1,6,32>,  hk = 7: the ring of 6 wraps
    Cin(6, 20, 33, 16, 50, 1),    # TF32 <1,6,64>,  hk = 33: two chains (32 + 1)
    Cin(4, 32, 37, 8, 128, 1),    # TF32 <1,6,128>, hk = 37, m = 32
    # PNN, both methods.  Feature-row width WX = F*K + Q + 1 on each side of 32, 64 and 128; N = 96 (forward pad 128, backward
    # pad 96), 200 (partial dW n-group), 4, 30 (N % 4 != 0: CUDA core); B = 0, 1 and around the 128-sample tile and 32-sample
    # dW chunk.
    Pnn(1, 2, 14, 96, 0),         # WX 32:  <32,4,0> | <32,4,0> | <32,0>
    Pnn(127, 1, 31, 200, 0),      # WX 33:  WP 64
    Pnn(128, 3, 19, 4, 0),        # WX 64:  WP 64
    Pnn(32, 4, 8, 96, 0),         # WX 43:  WP 64 mid-class
    Pnn(129, 1, 63, 96, 0),       # WX 65:  WP 128
    Pnn(31, 2, 62, 200, 0),       # WX 128: WP 128
    Pnn(33, 1, 127, 64, 0),       # WX 129: CUDA core
    Pnn(50, 4, 8, 30, 0),         # N = 30: CUDA core
    Pnn(0, 4, 8, 200, 0),         # B = 0
    Pnn(1, 14, 2, 200, 1),        # WX 32:  <32,4,1> | <32,4,1> | <32,1>
    Pnn(127, 31, 1, 96, 1),       # WX 33:  WP 64
    Pnn(128, 7, 6, 200, 1),       # WX 64:  WP 64
    Pnn(32, 8, 4, 200, 1),        # WX 43:  WP 64 mid-class
    Pnn(129, 63, 1, 4, 1),        # WX 65:  WP 128
    Pnn(31, 62, 2, 96, 1),        # WX 128: WP 128
    Pnn(33, 127, 1, 64, 1),       # WX 129: CUDA core
    Pnn(50, 8, 4, 30, 1),         # N = 30: CUDA core
    Pnn(0, 8, 4, 96, 1),          # B = 0
]

# Rows placed on SM-count-dependent switches; built from the device's multiprocessor count at run time.
SM_CASES = ["cin-tile-wrap", "cin-dw-chain-cross", "cin-dw-batch-below-slices",
            "ipnn-nsplit-2", "ipnn-nsplit-1", "opnn-nsplit-2", "opnn-nsplit-1"]


def sm_row(case, sms):
    if case == "cin-tile-wrap":                # n_tiles = SMs + 1 (forward and dX); hk = 7 is no multiple of 3, 4 or 6
        row = Cin(8 * sms + 1, 10, 7, 16, 40, 1)
        assert cin_row_tiles(row.B, row.D) == sms + 1
    elif case == "cin-dw-chain-cross":         # 11 samples per slice (the last one 6): crosses the 8-sample chain of D = 32
        row = Cin((sms // 2) * 11 - 5, 10, 8, 32, 40)
        nslices, per_slice, chain = cin_dw_schedule(row.B, row.hk, row.D, sms)
        assert nslices == sms // 2 and chain < per_slice < 2 * chain
    elif case == "cin-dw-batch-below-slices":  # B below SMs / n-groups: one sample per slice
        row = Cin(sms - 7, 9, 3, 8, 100)
        assert cin_dw_schedule(row.B, row.hk, row.D, sms)[:2] == (row.B, 1)
    else:
        # forward batch tiles on each side of the nsplit 2 -> 1 flip; N = 520: NT = 9 n-tiles split unevenly, three
        # accumulation chains in the dX kernel (17 K-blocks), and dW slices longer than one 8-chunk chain
        method = 0 if case.startswith("ipnn") else 1
        nsplit = int(case[-1])
        B = 128 * (sms // 2) + (0 if nsplit == 2 else 1)
        row = Pnn(B, 4, 8, 520, 0) if method == 0 else Pnn(B, 8, 4, 520, 1)
        assert pnn_fwd_nsplit(row.B, row.N, sms) == nsplit
        assert pnn_dw_chunks_per_slice(row.B, row.N, sms) > 8
    return row


# ================================================================================================ coverage (CPU)
def _tc_instantiations_from_rows(rows):
    found = {}
    for row in rows:
        for call in row.launches():
            for name, args in call or []:
                if name.endswith("_tc_kernel"):
                    found.setdefault((name, args), []).append(row.id)
    return found


def _fmt(inst):
    return f"{inst[0]}<{', '.join(map(str, inst[1]))}>"


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    for home in (os.environ.get("CUDA_HOME"), "/usr/local/cuda"):
        if exe is None and home and os.path.exists(os.path.join(home, "bin", "cuobjdump")):
            exe = os.path.join(home, "bin", "cuobjdump")
    return exe


def library_tc_instantiations():
    """{(base name, template integers)} of every `*_tc_kernel` in the built library, read from the mangled names
    (e.g. _ZN3ctr3pnn17pnn_fwd_tc_kernelILi64ELi3ELi1EEEv... -> ("pnn_fwd_tc_kernel", (64, 3, 1)))."""
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
            if not sym[num.end():end].endswith("_tc_kernel"):
                continue
            args = re.match(r"I((?:Lin?\d+E)+)E", sym[end:])
            assert args or not sym[end:].startswith("I"), f"{sym}: template arguments that are not integers"
            ints = re.findall(r"Li(n?)(\d+)E", args.group(1)) if args else []
            found.add((sym[num.end():end], tuple(-int(v) if neg else int(v) for neg, v in ints)))
    assert found, "no *_tc_kernel symbol found in the library"
    return found


def test_table_reaches_every_tc_instantiation():
    """The mirror over the shape table reaches exactly the library's wgmma instantiations: none is left without a row that
    compares it with float64, and every instantiation the table claims exists."""
    in_lib = library_tc_instantiations()
    reached = _tc_instantiations_from_rows(ROWS)
    missing = sorted(in_lib - set(reached))
    unknown = sorted(set(reached) - in_lib)
    assert not missing, "instantiations no row reaches: " + ", ".join(map(_fmt, missing))
    assert not unknown, "rows predict instantiations the library lacks: " + "; ".join(
        f"{_fmt(i)} (rows {', '.join(reached[i])})" for i in unknown)


def test_mirror_sides_of_each_boundary():
    """The table has a row on each side of every dispatch boundary the mirror encodes."""
    cin = [r for r in ROWS if isinstance(r, Cin)]
    pnn = [r for r in ROWS if isinstance(r, Pnn)]
    for lo, hi in ((32, 33), (64, 65), (96, 97), (128, 129), (256, 257)):
        assert {lo, hi} <= {r.H for r in cin}, (lo, hi)
    assert {32, 33} <= {r.m for r in cin} and {1, 2, 4, 12, 64, 257} <= {r.D for r in cin}
    for method in (0, 1):
        wx = {pnn_widths(r.F, r.K, r.N, r.method)[0] for r in pnn if r.method == method}
        assert {32, 33, 43, 64, 65, 128, 129} <= wx, (method, wx)
        rows = [r for r in pnn if r.method == method]
        assert {0, 1, 31, 32, 33, 127, 128, 129} <= {r.B for r in rows}
        assert {4, 30, 96, 200} <= {r.N for r in rows}
    assert cin_bwd_launches(1, 2, 2, 8, 257) is None and cin_bwd_launches(1, 2, 2, 257, 3) is None


# ================================================================================================ TF32 forward reference
def tf32_rna(x):
    """cvt.rna.tf32.f32 on the bits: round the low 13 mantissa bits to nearest, ties away from zero."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_rz(x):
    """Truncation to TF32 (cvt.rz): the rounding mode a wrong kernel would use instead."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return (u & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_forward_reference(x0, xk, w, rounding=tf32_rna, device="cpu"):
    """float64 sum_{i,j} tf32(fp32(xk[b,i,d] x0[b,j,d])) tf32(w[i*m+j, n]) of the single-pass TF32 forward, and a bound
    on how far a correct kernel may be from it, element by element.  Both (B, H, D).

    The kernel rounds both operands with cvt.rna.tf32, so every product it forms is exact in fp32 (11 x 11 significant
    bits).  It walks K in the order (i, j) with j padded to 32: one K-block per i, four k-steps of 8 j each, and a k-step
    whose 8 j are all >= m adds only zeros and changes nothing.  Each wgmma k-step adds its 8 products into the fp32
    accumulator; the tensor core aligns them to the largest exponent and truncates, so a step that moves the partial sum
    from P_{s-1} to P_s errs by at most 2 ulp of the largest magnitude involved:
        |err_s| <= 2^-22 M_s,   M_s = max(|P_{s-1}|, |P_s|, max_q |a_q w_q|)      (ulp(x) <= 2^-23 |x|).
    The accumulator restarts from zero every 32 K-blocks (cin.cu:262, CHUNK = 32) -- at most 128 k-steps per chain -- and
    each chain's sum A_c is added into the running fp32 total with round-to-nearest, <= 2^-24 |A_c|.  Errors add, so
        |out - ref| <= E = 2^-22 sum_s M_s + 2^-24 sum_c |A_c|,
    which at 128 steps is at most 128 * 2^-22 = 3.1e-5 of the largest partial sum and, since most partials are smaller
    than the largest, lands between 2e-6 and 2e-5 of max|ref| on the table's rows.  A truncating (rz) conversion of the
    operands moves every product by ~2^-11 of itself, 7e-4 to 9e-4 of max|ref| on the same rows;
    test_tf32_bound_separates_rounding_modes checks that separation on these inputs.
    max_q |a_q w_q| is bounded above by max_q |a_q| * max_q |w_q|, which only loosens E."""
    B, m, D = x0.shape
    hk, H = xk.shape[1], w.shape[1]
    S = -(-m // 8)                                                          # k-steps per K-block that carry products
    a = rounding(xk[:, :, None, :] * x0[:, None, :, :])                     # (B, hk, m, D): the fp32 product, then tf32
    a = np.pad(a, ((0, 0), (0, 0), (0, 8 * S - m), (0, 0))).reshape(B, hk, S, 8, D)
    wt = np.pad(rounding(w).reshape(hk, m, H), ((0, 0), (0, 8 * S - m), (0, 0))).reshape(hk, S, 8, H)
    wt = torch.from_numpy(wt).to(device, torch.float64)
    wmax = wt.abs().amax(2)                                                 # (hk, S, H)
    steps_per_chain = 32 * S
    ref = torch.empty((B, H, D), dtype=torch.float64, device=device)
    bound = torch.empty_like(ref)
    chunk = max(1, (1 << 23) // (D * H * hk * S))
    for b0 in range(0, B, chunk):
        ab = torch.from_numpy(a[b0:b0 + chunk]).to(device, torch.float64)
        step = torch.einsum("bisqd,isqn->bdnis", ab, wt).reshape(ab.shape[0], D, H, hk * S)
        pmax = torch.einsum("bisd,isn->bdnis", ab.abs().amax(3), wmax).reshape(step.shape)
        err = torch.zeros(step.shape[:3], dtype=torch.float64, device=device)
        total = torch.zeros_like(err)
        for c0 in range(0, hk * S, steps_per_chain):
            part = torch.cumsum(step[..., c0:c0 + steps_per_chain], -1)
            prev = torch.nn.functional.pad(part[..., :-1], (1, 0))
            ms = torch.maximum(torch.maximum(part.abs(), prev.abs()), pmax[..., c0:c0 + steps_per_chain])
            total = total + part[..., -1]
            err = err + 2.0 ** -22 * ms.sum(-1) + 2.0 ** -24 * total.abs()
        ref[b0:b0 + chunk] = total.permute(0, 2, 1)
        bound[b0:b0 + chunk] = err.permute(0, 2, 1)
    return ref, bound


def _tf32_rows():
    return [r for r in ROWS if isinstance(r, Cin) and r.precision]


@pytest.mark.parametrize("row", _tf32_rows(), ids=lambda r: r.id)
def test_tf32_bound_separates_rounding_modes(row):
    """CPU: on the inputs the GPU test uses, the bound is far tighter than the difference between round-to-nearest and
    truncating conversion, so a kernel that rounded the wrong way would fail it."""
    x0, xk, w, _ = _cin_inputs(row)
    ref, bound = tf32_forward_reference(x0, xk, w)
    ref_rz, _ = tf32_forward_reference(x0, xk, w, rounding=tf32_rz)
    gap = (ref_rz - ref).abs()
    scale = float(ref.abs().max())
    assert float(bound.max()) / scale < 3.2e-5, "the bound is looser than its derivation"
    # a truncating kernel is >= gap - E from the reference: it fails wherever gap > 2E
    assert float((gap > 2 * bound).double().mean()) > 0.5, "the bound does not separate rna from rz on most elements"
    assert float(gap.max()) > 8 * float(bound.max())


# ================================================================================================ GPU: parity and dispatch
def _seed(row):
    return zlib.crc32(row.id.encode())


def _cin_inputs(row):
    rng = np.random.default_rng(_seed(row))
    x0 = trunc_normal(rng, (row.B, row.m, row.D), 0.5)
    xk = trunc_normal(rng, (row.B, row.hk, row.D), 0.5)
    w = trunc_normal(rng, (row.hk * row.m, row.H), 0.2)
    g = trunc_normal(rng, (row.B, row.H, row.D), 1.0)
    return x0, xk, w, g


def _pnn_inputs(row):
    B, F, K, N, method = row
    rng = np.random.default_rng(_seed(row))
    u = lambda shape, lim: rng.uniform(-lim, lim, size=shape).astype(np.float32)
    e = (np.clip(rng.standard_normal((B, F, K)), -2, 2) / np.sqrt(K)).astype(np.float32)
    wlin = u((F * K, N), np.sqrt(6.0 / (F * K + N)))
    wprod = u((N, F), np.sqrt(6.0 / (N + F))) if method == 0 else u((N, K, K), np.sqrt(6.0 / (2 * N * K)))
    bias = u((N,), np.sqrt(3.0 / N))
    g = rng.standard_normal((B, N)).astype(np.float32)
    return e, wlin, wprod, bias, g


def _execute(row, inputs):
    """Runs the row's calls in the order of row.launches(); a refused call must raise the library's error."""
    from recalgorithm_b200 import _lib, ops
    res = {}
    if isinstance(row, Cin):
        x0, xk, w, g = (dev(a) for a in inputs)
        res["out"], res["pooled"] = ops.cin_fwd(x0, xk, w, want_pooled=True)
        if row.precision:
            res["out_tf32"] = ops.cin_fwd(x0, xk, w, precision=1)
        if row.launches()[-1] is None:
            with pytest.raises(_lib.CtrError, match="too large") as err:
                ops.cin_bwd(x0, xk, w, g)
            assert err.value.code == _lib.CTR_ERR_UNSUPPORTED
        else:
            res["dx0"], res["dxk"], res["dw"] = ops.cin_bwd(x0, xk, w, g)
    else:
        e, wlin, wprod, bias, g = (dev(a) for a in inputs)
        res["out"] = out = ops.pnn_fwd(e, wlin, wprod, bias, row.method)
        res["d_e"], res["d_wlin"], res["d_wprod"], res["d_bias"] = ops.pnn_bwd(e, wlin, wprod, out, g, row.method)
    torch.cuda.synchronize()
    return res


def _resolve(param):
    return sm_row(param, torch.cuda.get_device_properties(0).multi_processor_count) if isinstance(param, str) else param


PARAMS = ROWS + SM_CASES
PARAM_IDS = [p if isinstance(p, str) else p.id for p in PARAMS]


def _check_cin(row, inputs, res):
    x0, xk, w, g = (a.astype(np.float64) for a in inputs)
    ref = O.cin_layer_fwd(x0, xk, w)
    assert_close(res["out"], ref, TOL, f"{row.id}: forward (3xTF32)")
    assert_close(res["pooled"], ref.sum(-1), TOL, f"{row.id}: pooled")
    if row.precision:
        tref, bound = tf32_forward_reference(*inputs[:3], device="cuda")
        err = (res["out_tf32"].double() - tref).abs()
        worst = float((err / bound).max())
        assert worst <= 1.0, (f"{row.id}: TF32 forward exceeds its derived bound by {worst:.2f}x "
                              f"(max error {float(err.max()):.3e}, max|ref| {float(tref.abs().max()):.3e})")
    if "dx0" in res:
        ex0, exk, ew = O.cin_layer_bwd(x0, xk, w, g)                  # dfilter: the contraction over the whole batch
        assert_close(res["dx0"], ex0, TOL, f"{row.id}: dx0")
        assert_close(res["dxk"], exk, TOL, f"{row.id}: dxk")
        assert_close(res["dw"], ew, TOL, f"{row.id}: dfilter")


def _check_pnn(row, inputs, res):
    B, F, K, N, method = row
    e, wlin, wprod, bias, g = (a.astype(np.float64) for a in inputs)
    if B == 0:
        assert tuple(res["out"].shape) == (0, N) and tuple(res["d_e"].shape) == (0, F, K)
        for name in ("d_wlin", "d_wprod", "d_bias"):
            assert torch.count_nonzero(res[name]) == 0, f"{row.id}: {name} must be exactly zero at B = 0"
        return
    out = res["out"]
    assert_close(out, pnn_ref_fwd(e, wlin, wprod, bias, method), TOL, f"{row.id}: forward")
    # the relu mask is the kernel's own: pre-activations within rounding of 0 may fall on either side in float64
    mask = out.cpu().numpy() > 0
    r_e, r_wlin, r_wprod, r_bias = pnn_ref_bwd(e, wlin, wprod, bias + 1e6 * (2 * mask - 1), method, np.where(mask, g, 0.0))
    assert_close(res["d_e"], r_e, TOL, f"{row.id}: d_e")
    assert_close(res["d_wlin"], r_wlin, TOL, f"{row.id}: d_linear_w")
    assert_close(res["d_wprod"], r_wprod, TOL, f"{row.id}: d_product_w")
    assert_close(res["d_bias"], r_bias, TOL, f"{row.id}: d_bias")
    if method == 1:
        low = np.tril(np.ones((K, K), bool), -1)
        assert np.all(res["d_wprod"].cpu().numpy()[:, low] == 0), f"{row.id}: OPNN lower triangle must be exactly zero"


@pytest.mark.gpu
@pytest.mark.parametrize("param", PARAMS, ids=PARAM_IDS)
def test_row_against_float64(param):
    row = _resolve(param)
    inputs = _cin_inputs(row) if isinstance(row, Cin) else _pnn_inputs(row)
    res = _execute(row, inputs)
    (_check_cin if isinstance(row, Cin) else _check_pnn)(row, inputs, res)


_KERNEL = re.compile(r"ctr::\w+::(\w+)(?:<([^<>]*)>)?\(")


@pytest.mark.gpu
@pytest.mark.parametrize("param", PARAMS, ids=PARAM_IDS)
def test_row_launches_what_the_mirror_predicts(param):
    """The kernels the library launches for the row (torch.profiler, CUDA activity) are the mirror's, in order, with the
    same template integers -- this keeps the mirror, and with it the coverage claim above, honest."""
    from torch.profiler import ProfilerActivity, profile
    row = _resolve(param)
    inputs = _cin_inputs(row) if isinstance(row, Cin) else _pnn_inputs(row)
    _execute(row, inputs)                                                # first launches (module load) outside the trace
    for _ in range(3):                       # a session now and then hands back an empty device trace; a new one records
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _execute(row, inputs)
        events = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                        key=lambda e: e.time_range.start)
        if events:
            break
    else:
        pytest.skip("torch.profiler recorded no CUDA events on this machine")
    launched = []
    for e in events:
        hit = _KERNEL.search(e.name)
        if hit:
            launched.append((hit.group(1), tuple(int(v) for v in re.findall(r"-?\d+", hit.group(2) or ""))))
    expected = [k for call in row.launches() for k in (call or [])]
    assert launched == expected, f"{row.id}: launched {launched}, the mirror predicts {expected}"
