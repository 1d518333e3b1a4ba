// DIEN interest extractor (GRU) + attention + interest evolution (AGRU / AUGRU), DIEN/dien.py:198-229 with the cells of
// DIEN/custom_grucell.py:19-167, on CUDA cores.
//
// A group of G = min(NHP, 32) lanes runs one sample; lane g owns the hidden units j = g + u*G (u < NHP/G), so a warp runs
// 32/G samples.  The state is broadcast inside the group by width-G shuffles.  Both recurrences stop at the sample's
// length L = clamp(len, 0, T): past it the reference's attention weights are exactly 0 (the masked score is -2^32 and
// exp underflows to 0) and the evolution cell copies its state through, so nothing computed there reaches an output.
// The loops over t run to the warp's longest length with inactive groups frozen, which keeps every shuffle warp-uniform.
//
// The forward keeps the extractor states H, the evolution states S and the attention weights A in the caller's workspace;
// the backward reads them, runs BPTT through the evolution cell, the softmax and the extractor, and accumulates the nine
// weight gradients in shared memory (one global atomic per element per CTA at the end).
//
// The auxiliary loss (DIEN/dien.py:256-300, the paper's sign) reads H from the same workspace: dien_aux_fwd_kernel and
// dien_aux_sum_kernel give the loss, dien_aux_bwd_kernel its row gradients and dL/dh_t, which dien_bwd_aux_kernel -- the
// backward above with the extra terms added instead of overwritten -- carries through BPTT.
//
// Forward weights: the nine recurrent blocks (the extractor's state rows, the evolution cell's input and state rows) are
// held per lane in registers at nh_pad = 8 and staged by the CTA, zero padded, in shared memory above it; the extractor's
// input rows W_x are read through the read-only cache in the projection, which runs outside the recurrent part.  Input rows
// are prefetched two steps ahead.  The backward reads every weight through the read-only cache.
#include <math.h>

#include "ctr_common.cuh"

namespace ctr {
namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int DIEN_WARPS = 4;
constexpr float kMasked = -4294967296.f;   // -2**32 + 1 rounded to fp32 (dien.py:216)

// Offsets of the nine variables in the packed parameter buffer (include/ctr_b200.h).
struct DienParams {
  int gk, gb, ck, cb, att, egk, egb, eck, ecb, total;
};
__host__ __device__ inline DienParams dien_params(int na, int nh) {
  DienParams p;
  int o = 0;
  p.gk = o;  o += (na + nh) * 2 * nh;   // rnn/gru_cell/gates/kernel
  p.gb = o;  o += 2 * nh;               // rnn/gru_cell/gates/bias
  p.ck = o;  o += (na + nh) * nh;       // rnn/gru_cell/candidate/kernel
  p.cb = o;  o += nh;                   // rnn/gru_cell/candidate/bias
  p.att = o; o += nh * na;              // attention_project_matrix
  p.egk = o; o += 2 * nh * 2 * nh;      // rnn/gates/kernel
  p.egb = o; o += 2 * nh;               // rnn/gates/bias
  p.eck = o; o += 2 * nh * nh;          // rnn/candidate/kernel
  p.ecb = o; o += nh;                   // rnn/candidate/bias
  p.total = o;
  return p;
}

__device__ __forceinline__ float sigm(float z) { return 1.f / (1.f + expf(-z)); }

template <int G>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o, G);
  return v;
}
template <int G>
__device__ __forceinline__ float group_max(float v) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL, v, o, G));
  return v;
}
// value of hidden unit k held by the group (unit k lives in lane k % G, slot k / G; U <= 2, selected without indexing so
// that the loops over k need not be fully unrolled)
template <int G, int U>
__device__ __forceinline__ float bcast(const float (&v)[U], int k) {
  static_assert(U == 1 || U == 2, "at most 64 units");
  const float s = (U == 2 && k >= G) ? v[U - 1] : v[0];
  return __shfl_sync(FULL, s, k % G, G);
}

// Per-lane view of one sample: its units, their liveness (j < nh) and the sample's clamped length.
template <int NHP>
struct Lane {
  static constexpr int G = NHP < 32 ? NHP : 32, U = NHP / G, SPW = 32 / G;
  int gl, b, L;
  bool valid;
  int j[U];
  bool live[U];
  __device__ Lane(int warp_task, int B, int T, int nh, const long long* len) {
    const int lane = threadIdx.x & 31;
    gl = lane % G;
    b = warp_task * SPW + lane / G;
    valid = b < B;
    L = 0;
    if (valid) {
      const long long l = len[b];
      L = l <= 0 ? 0 : (l >= T ? T : (int)l);           // len > T: sequence_mask is all-true and the loop runs T steps
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      j[u] = gl + u * G;
      live[u] = valid && j[u] < nh;
    }
  }
  __device__ float w(const float* p, bool ok) const { return ok ? __ldg(p) : 0.f; }
};

// x_t . W_x + b for the extractor's r, u and candidate columns of this lane's units (independent of the recurrence).
template <int NHP>
__device__ __forceinline__ void extractor_proj(const Lane<NHP>& ln, const float* __restrict__ P, const DienParams& o,
                                               const float* __restrict__ xt, bool act, int na, int nh,
                                               float (&pr)[Lane<NHP>::U], float (&pu)[Lane<NHP>::U],
                                               float (&pc)[Lane<NHP>::U]) {
  constexpr int U = Lane<NHP>::U;
#pragma unroll
  for (int u = 0; u < U; ++u) {
    pr[u] = ln.w(P + o.gb + ln.j[u], ln.live[u]);
    pu[u] = ln.w(P + o.gb + nh + ln.j[u], ln.live[u]);
    pc[u] = ln.w(P + o.cb + ln.j[u], ln.live[u]);
  }
  if (!act) return;
#pragma unroll 4
  for (int i = 0; i < na; ++i) {
    const float xi = __ldg(xt + i);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      pr[u] = fmaf(xi, ln.w(P + o.gk + i * 2 * nh + ln.j[u], ln.live[u]), pr[u]);
      pu[u] = fmaf(xi, ln.w(P + o.gk + i * 2 * nh + nh + ln.j[u], ln.live[u]), pu[u]);
      pc[u] = fmaf(xi, ln.w(P + o.ck + i * nh + ln.j[u], ln.live[u]), pc[u]);
    }
  }
}

// One GRU step on the state part: gates r, u from z = proj + h.Wh, candidate c = tanh(pc + (r*h).Wch).  The gate kernel
// (rows [row0, row0 + nh) of a (.., 2nh) matrix) and the candidate kernel (rows [row0, row0 + nh) of a (.., nh) matrix).
template <int NHP, bool NEED_U>
__device__ __forceinline__ void gru_state_part(const Lane<NHP>& ln, const float* __restrict__ gk, const float* __restrict__ ck,
                                               int row0, int nh, const float (&h)[Lane<NHP>::U], float (&zr)[Lane<NHP>::U],
                                               float (&zu)[Lane<NHP>::U], float (&zc)[Lane<NHP>::U],
                                               float (&r)[Lane<NHP>::U], float (&uu)[Lane<NHP>::U],
                                               float (&c)[Lane<NHP>::U], float (&rh)[Lane<NHP>::U]) {
  constexpr int G = Lane<NHP>::G, U = Lane<NHP>::U;
#pragma unroll 8
  for (int k = 0; k < NHP; ++k) {
    if (k < nh) {
      const float hk = bcast<G, U>(h, k);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        zr[u] = fmaf(hk, ln.w(gk + (row0 + k) * 2 * nh + ln.j[u], ln.live[u]), zr[u]);
        if (NEED_U) zu[u] = fmaf(hk, ln.w(gk + (row0 + k) * 2 * nh + nh + ln.j[u], ln.live[u]), zu[u]);
      }
    }
  }
#pragma unroll
  for (int u = 0; u < U; ++u) {
    r[u] = sigm(zr[u]);
    uu[u] = NEED_U ? sigm(zu[u]) : 0.f;
    rh[u] = r[u] * h[u];
  }
#pragma unroll 8
  for (int k = 0; k < NHP; ++k) {
    if (k < nh) {
      const float rk = bcast<G, U>(rh, k);
#pragma unroll
      for (int u = 0; u < U; ++u) zc[u] = fmaf(rk, ln.w(ck + (row0 + k) * nh + ln.j[u], ln.live[u]), zc[u]);
    }
  }
#pragma unroll
  for (int u = 0; u < U; ++u) c[u] = tanhf(zc[u]);
}

// Input part of the evolution cell: its input is the extractor state h_t (nh wide, rows [0, nh) of its kernels).
template <int NHP, bool NEED_U>
__device__ __forceinline__ void evo_input_part(const Lane<NHP>& ln, const float* __restrict__ P, const DienParams& o, int nh,
                                               const float (&x)[Lane<NHP>::U], float (&zr)[Lane<NHP>::U],
                                               float (&zu)[Lane<NHP>::U], float (&zc)[Lane<NHP>::U]) {
  constexpr int G = Lane<NHP>::G, U = Lane<NHP>::U;
#pragma unroll
  for (int u = 0; u < U; ++u) {
    zr[u] = ln.w(P + o.egb + ln.j[u], ln.live[u]);
    zu[u] = NEED_U ? ln.w(P + o.egb + nh + ln.j[u], ln.live[u]) : 0.f;
    zc[u] = ln.w(P + o.ecb + ln.j[u], ln.live[u]);
  }
#pragma unroll 8
  for (int k = 0; k < NHP; ++k) {
    if (k < nh) {
      const float xk = bcast<G, U>(x, k);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        zr[u] = fmaf(xk, ln.w(P + o.egk + k * 2 * nh + ln.j[u], ln.live[u]), zr[u]);
        if (NEED_U) zu[u] = fmaf(xk, ln.w(P + o.egk + k * 2 * nh + nh + ln.j[u], ln.live[u]), zu[u]);
        zc[u] = fmaf(xk, ln.w(P + o.eck + k * nh + ln.j[u], ln.live[u]), zc[u]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------ forward
// The nine blocks of recurrent weights the forward reads at every step, as (offset, leading dimension) in the packed
// parameters: element (k, j) = P[off + k*ld + j] for k, j < nh.  0-2: extractor state rows (r, u, candidate columns);
// 3-5: evolution input rows; 6-8: evolution state rows.
constexpr int NREC = 9;
__device__ __forceinline__ void rec_desc(const DienParams& o, int na, int nh, int m, int& off, int& ld) {
  const int g2 = 2 * nh;
  const int offs[NREC] = {o.gk + na * g2, o.gk + na * g2 + nh, o.ck + na * nh, o.egk, o.egk + nh, o.eck,
                          o.egk + nh * g2, o.egk + nh * g2 + nh, o.eck + nh * nh};
  off = offs[m];
  ld = (m == 2 || m == 5 || m == 8) ? nh : g2;
}
// Below this padded width every lane keeps its columns of all nine blocks in registers (9 * NHP floats); above it the CTA
// stages the blocks, zero padded to NHP x NHP, in shared memory (147 KB at NHP = 64).
__host__ __device__ constexpr bool rec_in_registers(int nhp) { return nhp <= 8; }
template <int NHP>
constexpr size_t rec_smem_bytes() { return rec_in_registers(NHP) ? 0 : sizeof(float) * NREC * NHP * NHP; }

// 0 that the compiler cannot see through.  Where the weights live in shared memory, pointers are re-based on it at every
// step: otherwise the loop-invariant loads are hoisted out of the t loop into more registers than there are, and spill.
__device__ __forceinline__ int opaque_zero() {
  int z = 0;
  asm volatile("" : "+r"(z));
  return z;
}

// This lane's columns of one recurrent block, zero outside nh x nh so that the loops over k need no branch.
template <int NHP>
struct RecMat {
  static constexpr bool REG = rec_in_registers(NHP);
  static constexpr int U = Lane<NHP>::U;
  float r[REG ? NHP : 1][U];
  const float* s;
  __device__ void load(const Lane<NHP>& ln, const float* __restrict__ P, const float* sm, int off, int ld, int nh) {
    if constexpr (REG) {
#pragma unroll
      for (int k = 0; k < NHP; ++k)
#pragma unroll
        for (int u = 0; u < U; ++u) r[k][u] = ln.live[u] && k < nh ? __ldg(P + off + k * ld + ln.j[u]) : 0.f;
    } else {
      s = sm;
    }
  }
  __device__ __forceinline__ float at(const Lane<NHP>& ln, int k, int u) const {
    if constexpr (REG) return r[k][u];
    else return s[k * NHP + ln.j[u]];
  }
};

// z += sum_k in_k * W[k, j] over this lane's units, in_k broadcast inside the group.
template <int NHP>
__device__ __forceinline__ void rec_acc(const Lane<NHP>& ln, const RecMat<NHP>& W, const float (&in)[Lane<NHP>::U],
                                        float (&z)[Lane<NHP>::U]) {
  constexpr int G = Lane<NHP>::G, U = Lane<NHP>::U;
#pragma unroll 8
  for (int k = 0; k < NHP; ++k) {
    const float ik = bcast<G, U>(in, k);
#pragma unroll
    for (int u = 0; u < U; ++u) z[u] = fmaf(ik, W.at(ln, k, u), z[u]);
  }
}
template <int NHP>
__device__ __forceinline__ void rec_acc2(const Lane<NHP>& ln, const RecMat<NHP>& Wa, const RecMat<NHP>& Wb,
                                         const float (&in)[Lane<NHP>::U], float (&za)[Lane<NHP>::U],
                                         float (&zb)[Lane<NHP>::U]) {
  constexpr int G = Lane<NHP>::G, U = Lane<NHP>::U;
#pragma unroll 8
  for (int k = 0; k < NHP; ++k) {
    const float ik = bcast<G, U>(in, k);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      za[u] = fmaf(ik, Wa.at(ln, k, u), za[u]);
      zb[u] = fmaf(ik, Wb.at(ln, k, u), zb[u]);
    }
  }
}

// One input row x_t spread over the group: lane g holds x[g + q*G] (zeros past na, or when the position is not processed).
template <int NHP>
struct XRow {
  static constexpr int RA = (64 + Lane<NHP>::G - 1) / Lane<NHP>::G;
  float v[RA];
  __device__ __forceinline__ void load(const Lane<NHP>& ln, const float* __restrict__ xt, bool act, int na) {
#pragma unroll
    for (int q = 0; q < RA; ++q) {
      const int i = ln.gl + q * Lane<NHP>::G;
      v[q] = act && i < na ? __ldg(xt + i) : 0.f;
    }
  }
};

// x_t . W_x + b for the extractor's r, u and candidate columns of this lane's units, from a row already in registers.
template <int NHP>
__device__ __forceinline__ void proj_row(const Lane<NHP>& ln, const float* __restrict__ P, const DienParams& o,
                                         const XRow<NHP>& x, int na, int nh, float (&pr)[Lane<NHP>::U],
                                         float (&pu)[Lane<NHP>::U], float (&pc)[Lane<NHP>::U]) {
  constexpr int G = Lane<NHP>::G, U = Lane<NHP>::U;
#pragma unroll
  for (int u = 0; u < U; ++u) {
    pr[u] = ln.w(P + o.gb + ln.j[u], ln.live[u]);
    pu[u] = ln.w(P + o.gb + nh + ln.j[u], ln.live[u]);
    pc[u] = ln.w(P + o.cb + ln.j[u], ln.live[u]);
  }
#pragma unroll
  for (int q = 0; q < XRow<NHP>::RA; ++q) {
    if (q * G < na) {                                          // warp-uniform
#pragma unroll 4
      for (int g = 0; g < G; ++g) {
        const int i = q * G + g;
        const float xi = __shfl_sync(FULL, x.v[q], g, G);
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const bool ok = ln.live[u] && i < na;
          pr[u] = fmaf(xi, ln.w(P + o.gk + i * 2 * nh + ln.j[u], ok), pr[u]);
          pu[u] = fmaf(xi, ln.w(P + o.gk + i * 2 * nh + nh + ln.j[u], ok), pu[u]);
          pc[u] = fmaf(xi, ln.w(P + o.ck + i * nh + ln.j[u], ok), pc[u]);
        }
      }
    }
  }
}

// At nh_pad = 8 the weights stay hoisted in registers; wider, the shared-memory blocks and P are re-based on an opaque 0.
template <int NHP>
__device__ __forceinline__ const float* rebase(const float* P, RecMat<NHP> (&W)[NREC], const float* wsm) {
  if constexpr (rec_in_registers(NHP)) {
    return P;
  } else {
    const int z = opaque_zero();
#pragma unroll
    for (int m = 0; m < NREC; ++m) W[m].s = wsm + m * NHP * NHP + z;
    return P + z;
  }
}

// Per step, the dependent chain is only the recurrent part: broadcasts of the state, FMAs against weights already in
// registers (or shared memory), sigmoid / tanh.  Everything that does not depend on the state -- the next input rows x_{t+2}
// (loaded two steps ahead), the projection x_{t+1}.W_x (computed after step t's recurrent part), and, in the evolution
// loop, h_{t+2}, a_{t+2} and the input part h_{t+1}.W_h -- is issued around it.
template <int NHP, int AUGRU>
__global__ void __launch_bounds__(DIEN_WARPS * 32, 1) dien_fwd_kernel(
    const float* __restrict__ x, const long long* __restrict__ len, const float* __restrict__ tgt,
    const float* __restrict__ P, int B, int T, int na, int nh, float* __restrict__ final_state, float* __restrict__ scores,
    float* __restrict__ wsH, float* __restrict__ wsS, float* __restrict__ wsA) {
  using LN = Lane<NHP>;
  constexpr int G = LN::G, U = LN::U, NN = NHP * NHP;
  extern __shared__ float wsm[];
  const DienParams o = dien_params(na, nh);
  if constexpr (!rec_in_registers(NHP)) {
    for (int idx = threadIdx.x; idx < NREC * NN; idx += blockDim.x) {
      const int m = idx / NN, k = (idx / NHP) % NHP, j = idx % NHP;
      int off, ld;
      rec_desc(o, na, nh, m, off, ld);
      wsm[idx] = k < nh && j < nh ? __ldg(P + off + k * ld + j) : 0.f;
    }
    __syncthreads();
  }
  const LN ln(blockIdx.x * DIEN_WARPS + threadIdx.x / 32, B, T, nh, len);
  const int L = ln.L, Lw = __reduce_max_sync(FULL, (unsigned)L);
  const size_t row = (size_t)(ln.valid ? ln.b : 0) * T;
  RecMat<NHP> W[NREC];
#pragma unroll
  for (int m = 0; m < NREC; ++m) {
    int off, ld;
    rec_desc(o, na, nh, m, off, ld);
    W[m].load(ln, P, wsm + m * NN, off, ld, nh);
  }

  // v = attention_project_matrix . target  (score_t = h_t . v)
  float v[U];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    v[u] = 0.f;
    if (ln.live[u])
      for (int i = 0; i < na; ++i) v[u] = fmaf(__ldg(P + o.att + ln.j[u] * na + i), __ldg(tgt + (size_t)ln.b * na + i), v[u]);
  }

  // ---- interest extractor: GRUCell over t < L from a zero state
  float h[U], pr[U], pu[U], pc[U];
#pragma unroll
  for (int u = 0; u < U; ++u) h[u] = 0.f;
  XRow<NHP> xn;
  xn.load(ln, x + row * na, 0 < L, na);
  proj_row<NHP>(ln, P, o, xn, na, nh, pr, pu, pc);
  xn.load(ln, x + (row + 1) * na, 1 < L, na);
  for (int t = 0; t < Lw; ++t) {
    const bool act = t < L;
    const float* Pt = rebase(P, W, wsm);
    XRow<NHP> xf;
    xf.load(ln, x + (row + t + 2) * na, t + 2 < L, na);          // two steps ahead
    float zr[U], zu[U], zc[U], rh[U];
#pragma unroll
    for (int u = 0; u < U; ++u) { zr[u] = pr[u]; zu[u] = pu[u]; zc[u] = pc[u]; }
    rec_acc2<NHP>(ln, W[0], W[1], h, zr, zu);
    float uu[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      uu[u] = sigm(zu[u]);
      rh[u] = sigm(zr[u]) * h[u];
    }
    rec_acc<NHP>(ln, W[2], rh, zc);
    float s = 0.f;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const float c = tanhf(zc[u]);
      const float hn = uu[u] * h[u] + (1.f - uu[u]) * c;
      h[u] = !ln.live[u] ? 0.f : act ? hn : h[u];
      if (act && ln.live[u]) wsH[(row + t) * nh + ln.j[u]] = h[u];
      s = fmaf(h[u], v[u], s);
    }
    proj_row<NHP>(ln, Pt, o, xn, na, nh, pr, pu, pc);            // x_{t+1} . W_x, after the recurrent part
    xn = xf;
    s = group_sum<G>(s);
    if (act && ln.gl == t % G) wsA[row + t] = s;                 // raw score; lane t % G owns position t
  }

  // ---- masked softmax over T (positions t >= L take -2^32 like the reference; their weight is exactly 0 when L >= 1)
  float m = -INFINITY;
  if (ln.valid)
    for (int t = ln.gl; t < T; t += G) m = fmaxf(m, t < L ? wsA[row + t] : kMasked);
  m = group_max<G>(m);
  float sum = 0.f;
  if (ln.valid)
    for (int t = ln.gl; t < T; t += G) sum += expf((t < L ? wsA[row + t] : kMasked) - m);
  sum = group_sum<G>(sum);
  if (ln.valid)
    for (int t = ln.gl; t < T; t += G) {
      const float a = expf((t < L ? wsA[row + t] : kMasked) - m) / sum;
      wsA[row + t] = a;
      if (scores) scores[row + t] = a;
    }
  __syncwarp();

  // ---- interest evolution: AGRU / AUGRU over t < L; the state is copied through past L
  auto load_h = [&](int t, float (&hx)[U]) {
#pragma unroll
    for (int u = 0; u < U; ++u) hx[u] = t < L && ln.live[u] ? wsH[(row + t) * nh + ln.j[u]] : 0.f;
  };
  auto input_part = [&](const float* __restrict__ P, const float (&hx)[U], float (&zr)[U], float (&zu)[U], float (&zc)[U]) {
#pragma unroll
    for (int u = 0; u < U; ++u) {
      zr[u] = ln.w(P + o.egb + ln.j[u], ln.live[u]);
      zu[u] = AUGRU ? ln.w(P + o.egb + nh + ln.j[u], ln.live[u]) : 0.f;
      zc[u] = ln.w(P + o.ecb + ln.j[u], ln.live[u]);
    }
    if (AUGRU) rec_acc2<NHP>(ln, W[3], W[4], hx, zr, zu);
    else rec_acc<NHP>(ln, W[3], hx, zr);
    rec_acc<NHP>(ln, W[5], hx, zc);
  };
  float st[U], hx[U], ir[U], iu[U], ic[U];
#pragma unroll
  for (int u = 0; u < U; ++u) st[u] = 0.f;
  load_h(0, hx);
  input_part(P, hx, ir, iu, ic);
  load_h(1, hx);
  float a_cur = 0 < L ? wsA[row] : 0.f, a_nxt = 1 < L ? wsA[row + 1] : 0.f;
  for (int t = 0; t < Lw; ++t) {
    const bool act = t < L;
    const float* Pt = rebase(P, W, wsm);
    float hf[U];
    load_h(t + 2, hf);                                           // two steps ahead
    const float a_far = t + 2 < L ? wsA[row + t + 2] : 0.f;
    const float a = a_cur;
    float zr[U], zu[U], zc[U], rs[U], uu[U];
#pragma unroll
    for (int u = 0; u < U; ++u) { zr[u] = ir[u]; zu[u] = iu[u]; zc[u] = ic[u]; }
    if (AUGRU) rec_acc2<NHP>(ln, W[6], W[7], st, zr, zu);
    else rec_acc<NHP>(ln, W[6], st, zr);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      uu[u] = AUGRU ? sigm(zu[u]) : 0.f;
      rs[u] = sigm(zr[u]) * st[u];
    }
    rec_acc<NHP>(ln, W[8], rs, zc);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const float c = tanhf(zc[u]);
      float sn;
      if (AUGRU) {
        const float ua = (1.f - a) * uu[u];
        sn = ua * st[u] + (1.f - ua) * c;
      } else {
        sn = (1.f - a) * st[u] + a * c;
      }
      st[u] = !ln.live[u] ? 0.f : act ? sn : st[u];
      if (act && ln.live[u]) wsS[(row + t) * nh + ln.j[u]] = st[u];
    }
    input_part(Pt, hx, ir, iu, ic);                              // h_{t+1} . W_h, after the recurrent part
#pragma unroll
    for (int u = 0; u < U; ++u) hx[u] = hf[u];
    a_cur = a_nxt;
    a_nxt = a_far;
  }
#pragma unroll
  for (int u = 0; u < U; ++u)
    if (ln.live[u]) final_state[(size_t)ln.b * nh + ln.j[u]] = st[u];
}

// ------------------------------------------------------------------------------------------------------------ backward
// AUX: the auxiliary loss's backward (dien_aux_bwd_kernel) has already seeded dL/dh_t into wsDH and its positive-row term
// into d_x; the evolution pass and the extractor pass then add to them instead of overwriting.
#define DIEN_BWD_PARAMS                                                                                                  \
  const float* __restrict__ x, const long long* __restrict__ len, const float* __restrict__ tgt,                        \
      const float* __restrict__ P, const float* __restrict__ g_final, int B, int T, int na, int nh,                     \
      const float* __restrict__ wsH, const float* __restrict__ wsS, const float* __restrict__ wsA,                      \
      float* __restrict__ wsDH, float* __restrict__ wsDA, float* __restrict__ d_x, float* __restrict__ d_tgt,           \
      float* __restrict__ d_P
#define DIEN_BWD_ARGS x, len, tgt, P, g_final, B, T, na, nh, wsH, wsS, wsA, wsDH, wsDA, d_x, d_tgt, d_P

template <int NHP, int AUGRU, bool AUX>
__device__ __forceinline__ void dien_bwd_body(DIEN_BWD_PARAMS) {
  using LN = Lane<NHP>;
  constexpr int G = LN::G, U = LN::U, RMAX = (64 + G - 1) / G;
  extern __shared__ float acc[];                              // d_P, packed like P, summed over this CTA's samples
  const DienParams o = dien_params(na, nh);
  for (int i = threadIdx.x; i < o.total; i += blockDim.x) acc[i] = 0.f;
  __syncthreads();

  const int tasks = (B + LN::SPW - 1) / LN::SPW;
  for (int task = blockIdx.x * DIEN_WARPS + threadIdx.x / 32; task < tasks; task += gridDim.x * DIEN_WARPS) {
    const LN ln(task, B, T, nh, len);
    const int L = ln.L, Lw = __reduce_max_sync(FULL, (unsigned)L);
    const size_t row = (size_t)(ln.valid ? ln.b : 0) * T;
    float v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      v[u] = 0.f;
      if (ln.live[u])
        for (int i = 0; i < na; ++i) v[u] = fmaf(__ldg(P + o.att + ln.j[u] * na + i), __ldg(tgt + (size_t)ln.b * na + i), v[u]);
    }

    // ---- BPTT through the evolution cell: ds = dL/d(state), dx -> wsDH (gradient reaching h_t), da -> wsDA
    float ds[U];
#pragma unroll
    for (int u = 0; u < U; ++u) ds[u] = ln.live[u] ? g_final[(size_t)ln.b * nh + ln.j[u]] : 0.f;
    float sum_ada = 0.f;
    for (int t = Lw - 1; t >= 0; --t) {
      const bool act = t < L;
      const float a = act ? wsA[row + t] : 0.f;
      float xin[U], sp[U], zr[U], zu[U], zc[U], r[U], uu[U], c[U], rs[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const bool ok = act && ln.live[u];
        xin[u] = ok ? wsH[(row + t) * nh + ln.j[u]] : 0.f;
        sp[u] = ok && t > 0 ? wsS[(row + t - 1) * nh + ln.j[u]] : 0.f;
      }
      evo_input_part<NHP, AUGRU == 1>(ln, P, o, nh, xin, zr, zu, zc);
      gru_state_part<NHP, AUGRU == 1>(ln, P + o.egk, P + o.eck, nh, nh, sp, zr, zu, zc, r, uu, c, rs);
      float dzr[U], dzu[U], dzc[U], dsp[U], dxe[U], drs[U], da = 0.f;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const float g = act ? ds[u] : 0.f;
        float dc, du;
        if (AUGRU) {
          const float ua = (1.f - a) * uu[u];
          const float dua = g * (sp[u] - c[u]);
          dc = g * (1.f - ua);
          dsp[u] = g * ua;
          du = dua * (1.f - a);
          da -= dua * uu[u];
        } else {
          dc = g * a;
          dsp[u] = g * (1.f - a);
          du = 0.f;                                          // AGRU never uses u: its gate half gets exactly 0
          da = fmaf(g, c[u] - sp[u], da);
        }
        dzc[u] = dc * (1.f - c[u] * c[u]);
        dzu[u] = du * uu[u] * (1.f - uu[u]);
        dxe[u] = 0.f;
        drs[u] = 0.f;
      }
      da = group_sum<G>(da);
      // d(input rows) = W . dz: this lane's rows are its own unit indices
#pragma unroll 8
      for (int k = 0; k < NHP; ++k) {
        if (k < nh) {
          const float gc = bcast<G, U>(dzc, k);
#pragma unroll
          for (int u = 0; u < U; ++u) {
            dxe[u] = fmaf(ln.w(P + o.eck + ln.j[u] * nh + k, ln.live[u]), gc, dxe[u]);
            drs[u] = fmaf(ln.w(P + o.eck + (nh + ln.j[u]) * nh + k, ln.live[u]), gc, drs[u]);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        dsp[u] = fmaf(drs[u], r[u], dsp[u]);
        dzr[u] = drs[u] * sp[u] * r[u] * (1.f - r[u]);
      }
#pragma unroll 8
      for (int k = 0; k < NHP; ++k) {
        if (k < nh) {
          const float gr = bcast<G, U>(dzr, k);
          const float gu = AUGRU ? bcast<G, U>(dzu, k) : 0.f;
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int rx = ln.j[u] * 2 * nh, rsr = (nh + ln.j[u]) * 2 * nh;
            dxe[u] = fmaf(ln.w(P + o.egk + rx + k, ln.live[u]), gr, dxe[u]);
            dsp[u] = fmaf(ln.w(P + o.egk + rsr + k, ln.live[u]), gr, dsp[u]);
            if (AUGRU) {
              dxe[u] = fmaf(ln.w(P + o.egk + rx + nh + k, ln.live[u]), gu, dxe[u]);
              dsp[u] = fmaf(ln.w(P + o.egk + rsr + nh + k, ln.live[u]), gu, dsp[u]);
            }
          }
        }
      }
      // weight gradients: column j (this lane's units) += input row k * dz_j
#pragma unroll 8
      for (int k = 0; k < NHP; ++k) {
        if (k < nh) {
          const float xk = bcast<G, U>(xin, k), sk = bcast<G, U>(sp, k), rk = bcast<G, U>(rs, k);
#pragma unroll
          for (int u = 0; u < U; ++u) {
            if (act && ln.live[u]) {
              const int j = ln.j[u];
              atomicAdd(acc + o.egk + k * 2 * nh + j, xk * dzr[u]);
              atomicAdd(acc + o.egk + (nh + k) * 2 * nh + j, sk * dzr[u]);
              if (AUGRU) {
                atomicAdd(acc + o.egk + k * 2 * nh + nh + j, xk * dzu[u]);
                atomicAdd(acc + o.egk + (nh + k) * 2 * nh + nh + j, sk * dzu[u]);
              }
              atomicAdd(acc + o.eck + k * nh + j, xk * dzc[u]);
              atomicAdd(acc + o.eck + (nh + k) * nh + j, rk * dzc[u]);
            }
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (act && ln.live[u]) {
          const int j = ln.j[u];
          atomicAdd(acc + o.egb + j, dzr[u]);
          if (AUGRU) atomicAdd(acc + o.egb + nh + j, dzu[u]);
          atomicAdd(acc + o.ecb + j, dzc[u]);
          if constexpr (AUX) wsDH[(row + t) * nh + j] += dxe[u];
          else wsDH[(row + t) * nh + j] = dxe[u];
        }
        if (act) ds[u] = ln.live[u] ? dsp[u] : 0.f;
      }
      if (act) {
        sum_ada = fmaf(a, da, sum_ada);
        if (ln.gl == t % G) wsDA[row + t] = da;
      }
    }
    __syncwarp();

    // ---- BPTT through the softmax and the extractor: dh = carry + dx_evo + dscore * v
    float carry[U], dv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) carry[u] = dv[u] = 0.f;
    for (int t = Lw - 1; t >= 0; --t) {
      const bool act = t < L;
      const float dsc = act ? wsA[row + t] * (wsDA[row + t] - sum_ada) : 0.f;
      float dh[U], hp[U], zr[U], zu[U], zc[U], r[U], uu[U], c[U], rh[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const bool ok = act && ln.live[u];
        const size_t at = (row + t) * nh + ln.j[u];
        dh[u] = ok ? carry[u] + wsDH[at] + dsc * v[u] : 0.f;
        if (ok) dv[u] = fmaf(dsc, wsH[at], dv[u]);
        hp[u] = ok && t > 0 ? wsH[at - nh] : 0.f;
      }
      const float* xt = x + (row + t) * na;
      extractor_proj<NHP>(ln, P, o, xt, act, na, nh, zr, zu, zc);
      gru_state_part<NHP, true>(ln, P + o.gk, P + o.ck, na, nh, hp, zr, zu, zc, r, uu, c, rh);
      float dzr[U], dzu[U], dzc[U], dhp[U], drh[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const float du = dh[u] * (hp[u] - c[u]);
        const float dc = dh[u] * (1.f - uu[u]);
        dhp[u] = dh[u] * uu[u];
        dzc[u] = dc * (1.f - c[u] * c[u]);
        dzu[u] = du * uu[u] * (1.f - uu[u]);
        drh[u] = 0.f;
      }
#pragma unroll 8
      for (int k = 0; k < NHP; ++k) {
        if (k < nh) {
          const float gc = bcast<G, U>(dzc, k);
#pragma unroll
          for (int u = 0; u < U; ++u) drh[u] = fmaf(ln.w(P + o.ck + (na + ln.j[u]) * nh + k, ln.live[u]), gc, drh[u]);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        dhp[u] = fmaf(drh[u], r[u], dhp[u]);
        dzr[u] = drh[u] * hp[u] * r[u] * (1.f - r[u]);
      }
      // d x_t[i] for this lane's rows i = gl + q*G, and the recurrent rows of the gate kernel
      float dxr[RMAX];
#pragma unroll
      for (int q = 0; q < RMAX; ++q) dxr[q] = 0.f;
#pragma unroll 8
      for (int k = 0; k < NHP; ++k) {
        if (k < nh) {
          const float gr = bcast<G, U>(dzr, k), gu = bcast<G, U>(dzu, k), gc = bcast<G, U>(dzc, k);
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int rr = (na + ln.j[u]) * 2 * nh;
            dhp[u] = fmaf(ln.w(P + o.gk + rr + k, ln.live[u]), gr, dhp[u]);
            dhp[u] = fmaf(ln.w(P + o.gk + rr + nh + k, ln.live[u]), gu, dhp[u]);
          }
#pragma unroll
          for (int q = 0; q < RMAX; ++q) {
            const int i = ln.gl + q * G;
            if (i < na && act) {
              float s = dxr[q];
              s = fmaf(__ldg(P + o.gk + i * 2 * nh + k), gr, s);
              s = fmaf(__ldg(P + o.gk + i * 2 * nh + nh + k), gu, s);
              s = fmaf(__ldg(P + o.ck + i * nh + k), gc, s);
              dxr[q] = s;
            }
          }
        }
      }
      if (act) {
#pragma unroll
        for (int q = 0; q < RMAX; ++q) {
          const int i = ln.gl + q * G;
          if (i < na) {
            if constexpr (AUX) d_x[(row + t) * na + i] += dxr[q];
            else d_x[(row + t) * na + i] = dxr[q];
          }
        }
      }
      // weight gradients of the extractor
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (act && ln.live[u]) {
          const int j = ln.j[u];
          for (int i = 0; i < na; ++i) {
            const float xi = __ldg(xt + i);
            atomicAdd(acc + o.gk + i * 2 * nh + j, xi * dzr[u]);
            atomicAdd(acc + o.gk + i * 2 * nh + nh + j, xi * dzu[u]);
            atomicAdd(acc + o.ck + i * nh + j, xi * dzc[u]);
          }
        }
      }
#pragma unroll 8
      for (int k = 0; k < NHP; ++k) {
        if (k < nh) {
          const float hk = bcast<G, U>(hp, k), rk = bcast<G, U>(rh, k);
#pragma unroll
          for (int u = 0; u < U; ++u) {
            if (act && ln.live[u]) {
              const int j = ln.j[u];
              atomicAdd(acc + o.gk + (na + k) * 2 * nh + j, hk * dzr[u]);
              atomicAdd(acc + o.gk + (na + k) * 2 * nh + nh + j, hk * dzu[u]);
              atomicAdd(acc + o.ck + (na + k) * nh + j, rk * dzc[u]);
            }
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (act && ln.live[u]) {
          const int j = ln.j[u];
          atomicAdd(acc + o.gb + j, dzr[u]);
          atomicAdd(acc + o.gb + nh + j, dzu[u]);
          atomicAdd(acc + o.cb + j, dzc[u]);
        }
        if (act) carry[u] = ln.live[u] ? dhp[u] : 0.f;
      }
    }
    // padded positions get exactly 0
    if (ln.valid)
      for (int t = L; t < T; ++t)
        for (int i = ln.gl; i < na; i += G) d_x[(row + t) * na + i] = 0.f;

    // ---- target: v = W_att . e  ->  d e = W_att^T dv (rows i = gl + q*G), d W_att[j, i] += dv_j e_i
    float de[RMAX];
#pragma unroll
    for (int q = 0; q < RMAX; ++q) de[q] = 0.f;
#pragma unroll 8
    for (int k = 0; k < NHP; ++k) {
      if (k < nh) {
        const float g = bcast<G, U>(dv, k);
#pragma unroll
        for (int q = 0; q < RMAX; ++q) {
          const int i = ln.gl + q * G;
          if (i < na && ln.valid) de[q] = fmaf(__ldg(P + o.att + k * na + i), g, de[q]);
        }
      }
    }
    if (ln.valid) {
#pragma unroll
      for (int q = 0; q < RMAX; ++q) {
        const int i = ln.gl + q * G;
        if (i < na) d_tgt[(size_t)ln.b * na + i] = de[q];
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (ln.live[u] && L > 0)
        for (int i = 0; i < na; ++i) atomicAdd(acc + o.att + ln.j[u] * na + i, dv[u] * __ldg(tgt + (size_t)ln.b * na + i));
  }
  __syncthreads();
  for (int i = threadIdx.x; i < o.total; i += blockDim.x) atomicAdd(d_P + i, acc[i]);
}

template <int NHP, int AUGRU>
__global__ void __launch_bounds__(DIEN_WARPS * 32, 1) dien_bwd_kernel(DIEN_BWD_PARAMS) {
  dien_bwd_body<NHP, AUGRU, false>(DIEN_BWD_ARGS);
}
template <int NHP, int AUGRU>
__global__ void __launch_bounds__(DIEN_WARPS * 32, 1) dien_bwd_aux_kernel(DIEN_BWD_PARAMS) {
  dien_bwd_body<NHP, AUGRU, true>(DIEN_BWD_ARGS);
}

// ------------------------------------------------------------------------------------------------------------ auxiliary loss
// DIEN/dien.py:256-300 with the paper's sign: for every position t < L - 1 of a sample, q_t = W h_t (na), z+ = q_t . x_{t+1},
// z-_n = q_t . neg_{t,n}, and the sample's term softplus(-z+) + sum_n softplus(z-_n) = -[log sig(z+) + sum_n log(1 - sig(z-_n))].
// One warp per position (b, t) (persistent CTAs): the positions are independent, and a warp per sample would walk its
// positions one after another, bound by the latency of the dependent loads and warp sums.  Lane l owns the input elements
// i = l and l + 32 (na <= 64), so every row read is coalesced and every dot product is one warp sum.  W (na, nh) is staged
// in shared memory twice: transposed for q = W h (lane i reads its row across j) and as is for the backward's W^T dq (lane j
// reads its column across i).
constexpr int AUX_WARPS = 8;

__device__ __forceinline__ float softplus(float z) { return fmaxf(z, 0.f) + log1pf(expf(-fabsf(z))); }

__device__ __forceinline__ int clamp_len(long long l, int T) { return l <= 0 ? 0 : (l >= T ? T : (int)l); }

// Stages W into wt[j * na + i] (and, if w_rm, into w_rm[i * nh + j] as well).
__device__ __forceinline__ void aux_stage_w(const float* __restrict__ W, int na, int nh, float* wt, float* w_rm) {
  for (int idx = threadIdx.x; idx < na * nh; idx += blockDim.x) {
    const float w = __ldg(W + idx);
    wt[(idx % nh) * na + idx / nh] = w;
    if (w_rm) w_rm[idx] = w;
  }
}

// q = W h for the lane's two rows (0 past na); h0 / h1: the lane's elements j = lane, lane + 32 of h (0 past nh).
__device__ __forceinline__ void aux_q(const float* wt, int na, int nh, float h0, float h1, float& q0, float& q1) {
  const int lane = threadIdx.x & 31;
  q0 = q1 = 0.f;
  for (int j = 0; j < nh; ++j) {
    const float hj = __shfl_sync(FULL, j < 32 ? h0 : h1, j & 31);
    if (lane < na) q0 = fmaf(wt[j * na + lane], hj, q0);
    if (lane + 32 < na) q1 = fmaf(wt[j * na + lane + 32], hj, q1);
  }
}

struct AuxRow {
  float v0, v1;
  __device__ __forceinline__ void load(const float* __restrict__ r, int na) {
    const int lane = threadIdx.x & 31;
    v0 = lane < na ? __ldg(r + lane) : 0.f;
    v1 = lane + 32 < na ? __ldg(r + lane + 32) : 0.f;
  }
  __device__ __forceinline__ float dot(float q0, float q1) const { return warp_sum(fmaf(q1, v1, q0 * v0)); }
};

__device__ __forceinline__ void aux_store(float* __restrict__ r, int na, float v0, float v1) {
  const int lane = threadIdx.x & 31;
  if (lane < na) r[lane] = v0;
  if (lane + 32 < na) r[lane + 32] = v1;
}

// part[b * (T - 1) + t] = the term of position t of sample b, 0 where it does not count.
__global__ void __launch_bounds__(AUX_WARPS * 32) dien_aux_fwd_kernel(
    const float* __restrict__ x, const float* __restrict__ neg, const long long* __restrict__ len,
    const float* __restrict__ W, int B, int T, int na, int nh, int T_neg, const float* __restrict__ wsH,
    float* __restrict__ part) {
  extern __shared__ float wt[];
  aux_stage_w(W, na, nh, wt, nullptr);
  __syncthreads();
  const int lane = threadIdx.x & 31, n = B * (T - 1);
  for (int p = blockIdx.x * AUX_WARPS + threadIdx.x / 32; p < n; p += gridDim.x * AUX_WARPS) {
    const int b = p / (T - 1), t = p % (T - 1);
    float term = 0.f;
    if (t + 1 < clamp_len(len[b], T)) {
      const float* h = wsH + ((size_t)b * T + t) * nh;
      float q0, q1;
      aux_q(wt, na, nh, lane < nh ? h[lane] : 0.f, lane + 32 < nh ? h[lane + 32] : 0.f, q0, q1);
      AuxRow r;
      r.load(x + ((size_t)b * T + t + 1) * na, na);
      term = softplus(-r.dot(q0, q1));
      const float* nr = neg + (size_t)p * T_neg * na;
      for (int k = 0; k < T_neg; ++k) {
        r.load(nr + (size_t)k * na, na);
        term += softplus(r.dot(q0, q1));
      }
    }
    if (lane == 0) part[p] = term;
  }
}

// aux_loss = (sum of the n terms) / B in float64: one CTA, strided partial sums then a fixed tree, so the bits do not depend
// on timing.
constexpr int AUX_SUM_THREADS = 1024;
__global__ void __launch_bounds__(AUX_SUM_THREADS) dien_aux_sum_kernel(const float* __restrict__ part, int n, int B,
                                                                       float* __restrict__ aux_loss) {
  __shared__ double s[AUX_SUM_THREADS];
  double v = 0.0;
  for (int p = threadIdx.x; p < n; p += AUX_SUM_THREADS) v += part[p];
  s[threadIdx.x] = v;
  __syncthreads();
  for (int o = AUX_SUM_THREADS / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) *aux_loss = (float)(s[0] / B);
}

// Backward given g = *g_aux (scale g / B): recomputes q_t and z, writes d_neg (every row, exact zeros at t >= L - 1), the
// positive-row term of d_x (row t + 1 gets g+ q_t; rows 0 and >= L exactly 0), dL/dh_t = W^T dq_t into wsDH (0 at t = L - 1)
// for dien_bwd_aux_kernel, and d_W = sum dq_t (x) h_t (shared-memory sums, one global atomic per element per CTA).
__global__ void __launch_bounds__(AUX_WARPS * 32) dien_aux_bwd_kernel(
    const float* __restrict__ x, const float* __restrict__ neg, const long long* __restrict__ len,
    const float* __restrict__ W, const float* __restrict__ g_aux, int B, int T, int na, int nh, int T_neg,
    const float* __restrict__ wsH, float* __restrict__ wsDH, float* __restrict__ d_x, float* __restrict__ d_neg,
    float* __restrict__ d_W) {
  extern __shared__ float sm[];
  const int nw = na * nh;
  float *wt = sm, *w_rm = sm + nw, *acc = sm + 2 * nw;
  aux_stage_w(W, na, nh, wt, w_rm);
  for (int i = threadIdx.x; i < nw; i += blockDim.x) acc[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const float gs = __ldg(g_aux) / (float)B;
  const int n = B * T;
  for (int p = blockIdx.x * AUX_WARPS + threadIdx.x / 32; p < n; p += gridDim.x * AUX_WARPS) {
    const int b = p / T, t = p % T, L = clamp_len(len[b], T);
    const size_t row = (size_t)b * T;
    if (t == 0) aux_store(d_x + row * na, na, 0.f, 0.f);             // row 0 has no positive term
    if (t == L - 1) {                                                // the last state feeds no aux term
      if (lane < nh) wsDH[(row + t) * nh + lane] = 0.f;
      if (lane + 32 < nh) wsDH[(row + t) * nh + lane + 32] = 0.f;
    }
    if (t + 1 >= T) continue;
    float* dn = d_neg + (((size_t)b * (T - 1) + t) * T_neg) * na;
    if (t + 1 >= L) {                                                // not counted: exact zeros
      for (int k = 0; k < T_neg; ++k) aux_store(dn + (size_t)k * na, na, 0.f, 0.f);
      aux_store(d_x + (row + t + 1) * na, na, 0.f, 0.f);
      continue;
    }
    const float* h = wsH + (row + t) * nh;
    const float h0 = lane < nh ? h[lane] : 0.f, h1 = lane + 32 < nh ? h[lane + 32] : 0.f;
    float q0, q1;
    aux_q(wt, na, nh, h0, h1, q0, q1);
    AuxRow r;
    r.load(x + (row + t + 1) * na, na);
    const float gp = gs * (sigm(r.dot(q0, q1)) - 1.f);
    float dq0 = gp * r.v0, dq1 = gp * r.v1;
    aux_store(d_x + (row + t + 1) * na, na, gp * q0, gp * q1);
    const float* nr = neg + (((size_t)b * (T - 1) + t) * T_neg) * na;
    for (int k = 0; k < T_neg; ++k) {
      r.load(nr + (size_t)k * na, na);
      const float gn = gs * sigm(r.dot(q0, q1));
      aux_store(dn + (size_t)k * na, na, gn * q0, gn * q1);
      dq0 = fmaf(gn, r.v0, dq0);
      dq1 = fmaf(gn, r.v1, dq1);
    }
    // dh_j = sum_i W[i, j] dq_i for the lane's j = lane, lane + 32
    float dh0 = 0.f, dh1 = 0.f;
    for (int i = 0; i < na; ++i) {
      const float dqi = __shfl_sync(FULL, i < 32 ? dq0 : dq1, i & 31);
      if (lane < nh) dh0 = fmaf(w_rm[i * nh + lane], dqi, dh0);
      if (lane + 32 < nh) dh1 = fmaf(w_rm[i * nh + lane + 32], dqi, dh1);
    }
    if (lane < nh) wsDH[(row + t) * nh + lane] = dh0;
    if (lane + 32 < nh) wsDH[(row + t) * nh + lane + 32] = dh1;
    // d_W[i, j] += dq_i h_j
    for (int base = 0; base < nw; base += 32) {
      const int idx = base + lane, i = idx / nh, j = idx % nh;
      const float a0 = __shfl_sync(FULL, dq0, i & 31), a1 = __shfl_sync(FULL, dq1, i & 31);
      const float c0 = __shfl_sync(FULL, h0, j & 31), c1 = __shfl_sync(FULL, h1, j & 31);
      if (idx < nw) atomicAdd(acc + idx, (i < 32 ? a0 : a1) * (j < 32 ? c0 : c1));
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nw; i += blockDim.x) atomicAdd(d_W + i, acc[i]);
}

// ------------------------------------------------------------------------------------------------------------ host
struct DienWs {
  float *H, *S, *A, *DH, *DA;
};
int64_t dien_ws_floats(int64_t B, int64_t T, int64_t nh) { return B * T * (3 * nh + 2); }
DienWs dien_ws(void* ws, int64_t B, int64_t T, int64_t nh) {
  float* p = static_cast<float*>(ws);
  DienWs w;
  w.H = p;
  w.S = w.H + B * T * nh;
  w.A = w.S + B * T * nh;
  w.DH = w.A + B * T;
  w.DA = w.DH + B * T * nh;
  return w;
}

int check_dien(const char* fn, int64_t B, int64_t T, int64_t na, int64_t nh) {
  CTR_REQUIRE(B >= 0 && T >= 1 && na >= 1 && nh >= 1, "%s: bad sizes B=%lld T=%lld na=%lld nh=%lld", fn, (long long)B,
              (long long)T, (long long)na, (long long)nh);
  CTR_UNSUPPORTED(na > 64 || nh > 64 || T > 128, "%s: na=%lld nh=%lld T=%lld unsupported (the kernels cover na <= 64, "
                  "nh <= 64, T <= 128)", fn, (long long)na, (long long)nh, (long long)T);
  CTR_UNSUPPORTED(B * T * (3 * nh + 2) >= (1ll << 31), "%s: B=%lld too large for T=%lld nh=%lld", fn, (long long)B,
                  (long long)T, (long long)nh);
  return CTR_OK;
}

int dien_nhp(int64_t nh) { return nh <= 8 ? 8 : nh <= 16 ? 16 : nh <= 32 ? 32 : 64; }

// The auxiliary loss's workspace: the DIEN workspace, then one float per position t < T - 1 of every sample.
int64_t dien_aux_ws_bytes(int64_t B, int64_t T, int64_t nh) { return (int64_t)sizeof(float) * (dien_ws_floats(B, T, nh) + B * (T - 1)); }

int check_dien_aux(const char* fn, int64_t B, int64_t T, int64_t na, int64_t nh, int64_t T_neg) {
  int rc = check_dien(fn, B, T, na, nh);
  if (rc) return rc;
  CTR_REQUIRE(T_neg >= 1, "%s: T_neg=%lld must be >= 1", fn, (long long)T_neg);
  CTR_UNSUPPORTED(T_neg >= (1ll << 31) || B * (T - 1) * T_neg * na >= (1ll << 31),
                  "%s: B=%lld T=%lld T_neg=%lld na=%lld: more than 2^31 - 1 negative-row elements", fn, (long long)B,
                  (long long)T, (long long)T_neg, (long long)na);
  return CTR_OK;
}

// Persistent grid of warps, one position each, over n positions.
long long dien_aux_ctas(int64_t n) { return (n + AUX_WARPS - 1) / AUX_WARPS; }

}  // namespace
}  // namespace ctr

using namespace ctr;

extern "C" int ctr_dien_workspace_bytes(int64_t B, int64_t T, int64_t na, int64_t nh, int64_t* bytes) {
  int rc = check_dien("ctr_dien_workspace_bytes", B, T, na, nh);
  if (rc) return rc;
  CTR_REQUIRE(bytes, "ctr_dien_workspace_bytes: null argument");
  *bytes = (int64_t)sizeof(float) * dien_ws_floats(B, T, nh);
  return CTR_OK;
}

extern "C" int ctr_dien_fwd(const float* seq_input, const int64_t* seq_length, const float* target_input, const float* params,
                            int64_t B, int64_t T, int64_t na, int64_t nh, int cell_type, float* final_state,
                            float* att_scores, void* workspace, int64_t workspace_bytes, void* stream) {
  int rc = check_dien("ctr_dien_fwd", B, T, na, nh);
  if (rc) return rc;
  CTR_REQUIRE(cell_type == 0 || cell_type == 1, "ctr_dien_fwd: cell_type=%d (0 = AGRU, 1 = AUGRU)", cell_type);
  CTR_REQUIRE(seq_input && seq_length && target_input && params && final_state && workspace,
              "ctr_dien_fwd: null argument");
  CTR_REQUIRE(workspace_bytes >= (int64_t)sizeof(float) * dien_ws_floats(B, T, nh),
              "ctr_dien_fwd: workspace_bytes=%lld < ctr_dien_workspace_bytes()", (long long)workspace_bytes);
  if (B == 0) return CTR_OK;
  const DienWs w = dien_ws(workspace, B, T, nh);
  const int nhp = dien_nhp(nh), spc = DIEN_WARPS * (32 / (nhp < 32 ? nhp : 32));
  const dim3 grid((unsigned)((B + spc - 1) / spc));
  return with_const<8, 16, 32, 64>(nhp, [&](auto NHP) {
    return with_const<0, 1>(cell_type, [&](auto CELL) {
      return launch("ctr_dien_fwd", dien_fwd_kernel<NHP, CELL>, grid, DIEN_WARPS * 32, rec_smem_bytes<NHP>(), as_stream(stream), seq_input,
                    reinterpret_cast<const long long*>(seq_length), target_input, params, (int)B, (int)T, (int)na, (int)nh,
                    final_state, att_scores, w.H, w.S, w.A);
    });
  });
}

extern "C" int ctr_dien_bwd(const float* seq_input, const int64_t* seq_length, const float* target_input, const float* params,
                            const float* g_final_state, int64_t B, int64_t T, int64_t na, int64_t nh, int cell_type,
                            float* d_seq_input, float* d_target_input, float* d_params, void* workspace,
                            int64_t workspace_bytes, void* stream) {
  int rc = check_dien("ctr_dien_bwd", B, T, na, nh);
  if (rc) return rc;
  CTR_REQUIRE(cell_type == 0 || cell_type == 1, "ctr_dien_bwd: cell_type=%d (0 = AGRU, 1 = AUGRU)", cell_type);
  CTR_REQUIRE(seq_input && seq_length && target_input && params && g_final_state && d_seq_input && d_target_input &&
                  d_params && workspace, "ctr_dien_bwd: null argument");
  CTR_REQUIRE(workspace_bytes >= (int64_t)sizeof(float) * dien_ws_floats(B, T, nh),
              "ctr_dien_bwd: workspace_bytes=%lld < ctr_dien_workspace_bytes()", (long long)workspace_bytes);
  const DienParams o = dien_params((int)na, (int)nh);
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(d_params, 0, sizeof(float) * o.total, st));
  if (B == 0) return CTR_OK;
  const DienWs w = dien_ws(workspace, B, T, nh);
  const int nhp = dien_nhp(nh), spw = 32 / (nhp < 32 ? nhp : 32);
  const long long need = ((B + spw - 1) / spw + DIEN_WARPS - 1) / DIEN_WARPS;
  const size_t smem = sizeof(float) * (size_t)o.total;     // <= 209.5 KB at na = nh = 64
  return with_const<8, 16, 32, 64>(nhp, [&](auto NHP) {
    return with_const<0, 1>(cell_type, [&](auto CELL) {
      return launch_resident("ctr_dien_bwd", dien_bwd_kernel<NHP, CELL>, need, DIEN_WARPS * 32, smem, st, seq_input,
                             reinterpret_cast<const long long*>(seq_length), target_input, params, g_final_state, (int)B,
                             (int)T, (int)na, (int)nh, w.H, w.S, w.A, w.DH, w.DA, d_seq_input, d_target_input, d_params);
    });
  });
}

extern "C" int ctr_dien_aux_workspace_bytes(int64_t B, int64_t T, int64_t na, int64_t nh, int64_t T_neg, int64_t* bytes) {
  int rc = check_dien_aux("ctr_dien_aux_workspace_bytes", B, T, na, nh, T_neg);
  if (rc) return rc;
  CTR_REQUIRE(bytes, "ctr_dien_aux_workspace_bytes: null argument");
  *bytes = dien_aux_ws_bytes(B, T, nh);
  return CTR_OK;
}

extern "C" int ctr_dien_aux_fwd(const float* seq_input, const float* neg_seq_input, const int64_t* seq_length,
                                const float* w_aux, int64_t B, int64_t T, int64_t na, int64_t nh, int64_t T_neg,
                                float* aux_loss, void* workspace, int64_t workspace_bytes, void* stream) {
  int rc = check_dien_aux("ctr_dien_aux_fwd", B, T, na, nh, T_neg);
  if (rc) return rc;
  CTR_REQUIRE(seq_input && neg_seq_input && seq_length && w_aux && aux_loss && workspace, "ctr_dien_aux_fwd: null argument");
  CTR_REQUIRE(workspace_bytes >= dien_aux_ws_bytes(B, T, nh),
              "ctr_dien_aux_fwd: workspace_bytes=%lld < ctr_dien_aux_workspace_bytes()", (long long)workspace_bytes);
  cudaStream_t st = as_stream(stream);
  if (B == 0) {
    CTR_CUDA(cudaMemsetAsync(aux_loss, 0, sizeof(float), st));
    return CTR_OK;
  }
  const DienWs w = dien_ws(workspace, B, T, nh);
  float* part = static_cast<float*>(workspace) + dien_ws_floats(B, T, nh);
  const int n = (int)(B * (T - 1));
  if (n > 0)
    rc = launch_resident("ctr_dien_aux_fwd", dien_aux_fwd_kernel, dien_aux_ctas(n), AUX_WARPS * 32,
                       sizeof(float) * (size_t)(na * nh), st, seq_input, neg_seq_input,
                       reinterpret_cast<const long long*>(seq_length), w_aux, (int)B, (int)T, (int)na, (int)nh, (int)T_neg,
                       (const float*)w.H, part);
  if (rc) return rc;
  return launch("ctr_dien_aux_fwd", dien_aux_sum_kernel, dim3(1), dim3(AUX_SUM_THREADS), 0, st, (const float*)part, n, (int)B,
                aux_loss);
}

extern "C" int ctr_dien_bwd_aux(const float* seq_input, const float* neg_seq_input, const int64_t* seq_length,
                                const float* target_input, const float* params, const float* w_aux, const float* g_final_state,
                                const float* g_aux_loss, int64_t B, int64_t T, int64_t na, int64_t nh, int64_t T_neg,
                                int cell_type, float* d_seq_input, float* d_neg_seq_input, float* d_target_input,
                                float* d_params, float* d_w_aux, void* workspace, int64_t workspace_bytes, void* stream) {
  int rc = check_dien_aux("ctr_dien_bwd_aux", B, T, na, nh, T_neg);
  if (rc) return rc;
  CTR_REQUIRE(cell_type == 0 || cell_type == 1, "ctr_dien_bwd_aux: cell_type=%d (0 = AGRU, 1 = AUGRU)", cell_type);
  CTR_REQUIRE(seq_input && neg_seq_input && seq_length && target_input && params && w_aux && g_final_state && g_aux_loss &&
                  d_seq_input && d_neg_seq_input && d_target_input && d_params && d_w_aux && workspace,
              "ctr_dien_bwd_aux: null argument");
  CTR_REQUIRE(workspace_bytes >= (int64_t)sizeof(float) * dien_ws_floats(B, T, nh),
              "ctr_dien_bwd_aux: workspace_bytes=%lld < ctr_dien_workspace_bytes()", (long long)workspace_bytes);
  const DienParams o = dien_params((int)na, (int)nh);
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(d_params, 0, sizeof(float) * o.total, st));
  CTR_CUDA(cudaMemsetAsync(d_w_aux, 0, sizeof(float) * (size_t)(na * nh), st));
  if (B == 0) return CTR_OK;
  const DienWs w = dien_ws(workspace, B, T, nh);
  rc = launch_resident("ctr_dien_bwd_aux", dien_aux_bwd_kernel, dien_aux_ctas(B * T), AUX_WARPS * 32,
                       3 * sizeof(float) * (size_t)(na * nh), st, seq_input, neg_seq_input,
                       reinterpret_cast<const long long*>(seq_length), w_aux, g_aux_loss, (int)B, (int)T, (int)na, (int)nh,
                       (int)T_neg, (const float*)w.H, w.DH, d_seq_input, d_neg_seq_input, d_w_aux);
  if (rc) return rc;
  const int nhp = dien_nhp(nh), spw = 32 / (nhp < 32 ? nhp : 32);
  const long long need = ((B + spw - 1) / spw + DIEN_WARPS - 1) / DIEN_WARPS;
  const size_t smem = sizeof(float) * (size_t)o.total;
  return with_const<8, 16, 32, 64>(nhp, [&](auto NHP) {
    return with_const<0, 1>(cell_type, [&](auto CELL) {
      return launch_resident("ctr_dien_bwd_aux", dien_bwd_aux_kernel<NHP, CELL>, need, DIEN_WARPS * 32, smem, st, seq_input,
                             reinterpret_cast<const long long*>(seq_length), target_input, params, g_final_state, (int)B,
                             (int)T, (int)na, (int)nh, w.H, w.S, w.A, w.DH, w.DA, d_seq_input, d_target_input, d_params);
    });
  });
}
