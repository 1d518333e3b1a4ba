// Peer-memory micro-benchmark for the row-sharded path (SURVEY 8e): how fast can one H100 PULL random 128-byte rows
// from / PUSH 128-byte rows to its NVLink peers, by access method?  Standalone (no torch): one process drives all GPUs.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/peerbench tools/peerbench.cu
//   tools/peerbench [shard_GB=8] [nreq=2621440] [reps=5]
//
// Every GPU runs the same kernel at the same time (all-to-all pattern: rank r pulls from / pushes to all other ranks,
// row -> owner = row % G like the product), so each link direction carries one rank's worth of payload.  Prints one
// JSON line per variant: GB/s of remote payload per rank (max time over ranks, best of `reps`).
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <string>
#include <vector>

#define CK(x)                                                                                   \
  do {                                                                                          \
    cudaError_t e_ = (x);                                                                       \
    if (e_ != cudaSuccess) {                                                                    \
      fprintf(stderr, "%s:%d %s -> %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));      \
      exit(1);                                                                                  \
    }                                                                                           \
  } while (0)

struct Peers {
  float4* base[8];
  int G, logG, me;
};

__device__ __forceinline__ float4 ld_nc_na(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ float4 ld_plain(const float4* p) {
  float4 r;
  asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ float4 ld_relaxed_sys(const float4* p) {
  float4 r;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_cs(float4* p, const float4& v) {
  asm volatile("st.global.cs.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void st_plain(float4* p, const float4& v) {
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// ---- pull with LDG.128: LPR lanes per row (row = LPR*16 bytes), UB row loads in flight per lane ---------------------
template <int LPR, int UB, int HINT>
__global__ void __launch_bounds__(256) pull_ldg(const Peers p, const long long* __restrict__ rows, long long n,
                                                float4* __restrict__ out) {
  const int lane = threadIdx.x & 31, sub = lane / LPR, c = lane % LPR;
  constexpr int RPW = 32 / LPR;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long i0 = warp * (RPW * UB); i0 < n; i0 += nwarps * (RPW * UB)) {
    float4 v[UB];
#pragma unroll
    for (int u = 0; u < UB; ++u) {
      const long long i = i0 + u * RPW + sub;
      v[u] = make_float4(0, 0, 0, 0);
      if (i < n) {
        const long long r = __ldg(rows + i);
        const float4* src = p.base[r & (p.G - 1)] + (size_t)(r >> p.logG) * LPR + c;
        v[u] = HINT == 0 ? ld_nc_na(src) : HINT == 1 ? ld_plain(src) : ld_relaxed_sys(src);
      }
    }
#pragma unroll
    for (int u = 0; u < UB; ++u) {
      const long long i = i0 + u * RPW + sub;
      if (i < n) st_cs(out + (size_t)i * LPR + c, v[u]);
    }
  }
}

// ---- pull shaped like the product kernel (embed_fm2_fwd_kernel<8, SH>): one warp per SAMPLE of F rows; the ids of a 32-field chunk
// are one coalesced 8-byte load per lane, distributed by shuffle; up to 8 row loads per lane in flight, then the tile stores.
template <int HINT>
__global__ void __launch_bounds__(256) pull_sample(const Peers p, const long long* __restrict__ rows, int B, int F,
                                                   float4* __restrict__ out) {
  constexpr int LPR = 8, RPW = 4, UB = 8;
  const int lane = threadIdx.x & 31, sub = lane / LPR, c = lane % LPR;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int b = warp0; b < B; b += nwarps) {
    for (int f0 = 0; f0 < F; f0 += 32) {
      const int nf = min(32, F - f0);
      long long row = -1;
      if (lane < nf) row = __ldg(rows + (size_t)b * F + f0 + lane);
#pragma unroll
      for (int it0 = 0; it0 < LPR; it0 += UB) {
        if (it0 * RPW >= nf) break;
        float4 v[UB];
#pragma unroll
        for (int u = 0; u < UB; ++u) {
          const int fs = (it0 + u) * RPW + sub;
          const long long r = __shfl_sync(0xffffffffu, row, fs);
          v[u] = make_float4(0, 0, 0, 0);
          if (fs < nf && r >= 0) {
            const float4* src = p.base[r & (p.G - 1)] + (size_t)(r >> p.logG) * LPR + c;
            v[u] = HINT == 0 ? ld_nc_na(src) : ld_plain(src);
          }
        }
#pragma unroll
        for (int u = 0; u < UB; ++u) {
          const int fs = (it0 + u) * RPW + sub;
          if (fs < nf) st_cs(out + ((size_t)b * F + f0 + fs) * LPR + c, v[u]);
        }
      }
    }
  }
}

// ---- pull with bulk async copies (TMA unit, non-tensor): each lane fetches one 128-byte row into smem, the warp then
// emits the 32 rows (4 KB, contiguous in `out`) with one bulk store.  NST stages per warp keep NST*32 rows in flight.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n.reg .pred p;\nWAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra DONE_%=;\nbra WAIT_%=;\nDONE_%=:\n}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }

template <int NST, int WARPS>
__global__ void __launch_bounds__(WARPS * 32) pull_bulk(const Peers p, const long long* __restrict__ rows, long long n,
                                                        float4* __restrict__ out) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) unsigned long long bars[WARPS * NST];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char* my = smem + (size_t)warp * NST * 4096;
  if (lane == 0)
    for (int s = 0; s < NST; ++s) mbar_init(smem_u32(&bars[warp * NST + s]), 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncwarp();
  const long long gw = (long long)blockIdx.x * WARPS + warp, nw = (long long)gridDim.x * WARPS;
  const long long nchunks = (n + 31) / 32;
  // chunk k of this warp = global chunk gw + k*nw ; pipeline depth NST
  long long issued = 0, done = 0;
  const long long mine = gw < nchunks ? (nchunks - gw + nw - 1) / nw : 0;
  while (done < mine) {
    while (issued < mine && issued < done + NST) {
      const int s = (int)(issued % NST);
      const long long ch = gw + issued * nw;
      const long long i = ch * 32 + lane;
      // the stage's previous bulk store must have finished READING smem before it is overwritten
      if (lane == 0) bulk_wait_read<0>();
      __syncwarp();
      const int cnt = (int)min(32LL, n - ch * 32);
      if (lane == 0) mbar_expect_tx(smem_u32(&bars[warp * NST + s]), cnt * 128);
      __syncwarp();
      if (i < n) {
        const long long r = __ldg(rows + i);
        const float4* src = p.base[r & (p.G - 1)] + (size_t)(r >> p.logG) * 8;
        bulk_g2s(smem_u32(my + s * 4096 + lane * 128), src, 128, smem_u32(&bars[warp * NST + s]));
      }
      ++issued;
    }
    const int s = (int)(done % NST);
    const long long ch = gw + done * nw;
    mbar_wait(smem_u32(&bars[warp * NST + s]), (uint32_t)((done / NST) & 1));
    const int cnt = (int)min(32LL, n - ch * 32);
    if (lane == 0) {
      bulk_s2g(out + (size_t)ch * 32 * 8, smem_u32(my + s * 4096), cnt * 128);
      bulk_commit();
    }
    __syncwarp();
    ++done;
  }
  if (lane == 0) bulk_wait_read<0>();
}

// ---- push with STG.128: src rows read sequentially from local memory, written to peer rows --------------------------
// dst row index = rows[i] (owner = r % G, local slot r / G): `rows` random = scattered 128 B stores; `rows` = queue order
// (sorted by owner, consecutive slots) = what the gradient push does.
template <int LPR, int UB, int HINT>
__global__ void __launch_bounds__(256) push_stg(const Peers p, const long long* __restrict__ rows, long long n,
                                                const float4* __restrict__ src) {
  const int lane = threadIdx.x & 31, sub = lane / LPR, c = lane % LPR;
  constexpr int RPW = 32 / LPR;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long i0 = warp * (RPW * UB); i0 < n; i0 += nwarps * (RPW * UB)) {
    float4 v[UB];
    long long r[UB];
#pragma unroll
    for (int u = 0; u < UB; ++u) {
      const long long i = i0 + u * RPW + sub;
      r[u] = -1;
      if (i < n) {
        r[u] = __ldg(rows + i);
        v[u] = ld_nc_na(src + (size_t)i * LPR + c);
      }
    }
#pragma unroll
    for (int u = 0; u < UB; ++u) {
      if (r[u] >= 0) {
        float4* dst = p.base[r[u] & (p.G - 1)] + (size_t)(r[u] >> p.logG) * LPR + c;
        if (HINT == 0) st_plain(dst, v[u]); else st_cs(dst, v[u]);
      }
    }
  }
}

// ---- push with bulk stores: the warp stages 32 local rows (4 KB) in smem with one bulk load, then one 128-byte bulk store
// per row to the peer (lane l stores row l).
template <int NST, int WARPS>
__global__ void __launch_bounds__(WARPS * 32) push_bulk(const Peers p, const long long* __restrict__ rows, long long n,
                                                        const float4* __restrict__ src) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) unsigned long long bars[WARPS * NST];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char* my = smem + (size_t)warp * NST * 4096;
  if (lane == 0)
    for (int s = 0; s < NST; ++s) mbar_init(smem_u32(&bars[warp * NST + s]), 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncwarp();
  const long long gw = (long long)blockIdx.x * WARPS + warp, nw = (long long)gridDim.x * WARPS;
  const long long nchunks = (n + 31) / 32;
  const long long mine = gw < nchunks ? (nchunks - gw + nw - 1) / nw : 0;
  long long issued = 0, done = 0;
  while (done < mine) {
    while (issued < mine && issued < done + NST) {
      const int s = (int)(issued % NST);
      const long long ch = gw + issued * nw;
      bulk_wait_read<0>();                            // every lane waits for ITS store of this stage (per-thread groups)
      __syncwarp();
      const int cnt = (int)min(32LL, n - ch * 32);
      if (lane == 0) {
        mbar_expect_tx(smem_u32(&bars[warp * NST + s]), cnt * 128);
        bulk_g2s(smem_u32(my + s * 4096), src + (size_t)ch * 32 * 8, cnt * 128, smem_u32(&bars[warp * NST + s]));
      }
      ++issued;
    }
    const int s = (int)(done % NST);
    const long long ch = gw + done * nw;
    mbar_wait(smem_u32(&bars[warp * NST + s]), (uint32_t)((done / NST) & 1));
    const long long i = ch * 32 + lane;
    if (i < n) {
      const long long r = __ldg(rows + i);
      bulk_s2g(p.base[r & (p.G - 1)] + (size_t)(r >> p.logG) * 8, smem_u32(my + s * 4096 + lane * 128), 128);
    }
    bulk_commit();
    ++done;
  }
  bulk_wait_read<0>();
}

// ----------------------------------------------------------------------------------------------------------------
static uint64_t splitmix(uint64_t& s) {
  uint64_t z = (s += 0x9e3779b97f4a7c15ULL);
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
  return z ^ (z >> 31);
}

struct Ctx {
  int G;
  std::vector<float4*> shard, buf;     // per GPU: table shard (peer-visible), local tile/src buffer
  std::vector<long long*> rows;        // per GPU: request list
  std::vector<cudaStream_t> st;
  std::vector<cudaEvent_t> e0, e1;
  long long n;
  double remote_frac;
};

template <typename F>
static void run(Ctx& c, const char* name, int reps, double bytes_per_row, F launch) {
  float best = 1e30f;
  for (int rep = 0; rep < reps + 1; ++rep) {
    for (int g = 0; g < c.G; ++g) { CK(cudaSetDevice(g)); CK(cudaDeviceSynchronize()); }
    for (int g = 0; g < c.G; ++g) {
      CK(cudaSetDevice(g));
      CK(cudaEventRecord(c.e0[g], c.st[g]));
      launch(g);
      CK(cudaGetLastError());
      CK(cudaEventRecord(c.e1[g], c.st[g]));
    }
    float worst = 0;
    for (int g = 0; g < c.G; ++g) {
      CK(cudaSetDevice(g));
      CK(cudaEventSynchronize(c.e1[g]));
      float ms;
      CK(cudaEventElapsedTime(&ms, c.e0[g], c.e1[g]));
      worst = std::max(worst, ms);
    }
    if (rep > 0) best = std::min(best, worst);
  }
  printf("{\"variant\": \"%s\", \"G\": %d, \"ms\": %.4f, \"remote_GBps_per_rank\": %.1f, \"rows\": %lld, \"remote_frac\": %.3f}\n", name,
         c.G, best, c.n * bytes_per_row * c.remote_frac / (best * 1e-3) / 1e9, c.n, c.remote_frac);
  fflush(stdout);
}

int main(int argc, char** argv) {
  const double shard_gb = argc > 1 ? atof(argv[1]) : 8.0;
  const long long n = argc > 2 ? atoll(argv[2]) : 65536LL * 40;
  const int reps = argc > 3 ? atoi(argv[3]) : 5;
  int ndev = 0;
  CK(cudaGetDeviceCount(&ndev));
  int G = 1;
  while (G * 2 <= ndev && G < 8) G *= 2;
  if (G < 2) { fprintf(stderr, "need >= 2 GPUs\n"); return 2; }
  const long long shard_rows = (long long)(shard_gb * 1e9 / 256) * 2;   // 128-byte rows, even count
  Ctx c;
  c.G = G; c.n = n;
  c.shard.resize(G); c.buf.resize(G); c.rows.resize(G); c.st.resize(G); c.e0.resize(G); c.e1.resize(G);
  for (int g = 0; g < G; ++g) {
    CK(cudaSetDevice(g));
    for (int h = 0; h < G; ++h)
      if (h != g) {
        int can = 0;
        CK(cudaDeviceCanAccessPeer(&can, g, h));
        if (!can) { fprintf(stderr, "no peer access %d->%d\n", g, h); return 2; }
        CK(cudaDeviceEnablePeerAccess(h, 0));
      }
    CK(cudaMalloc(&c.shard[g], (size_t)shard_rows * 128));
    CK(cudaMemset(c.shard[g], 0, (size_t)shard_rows * 128));
    CK(cudaMalloc(&c.buf[g], (size_t)n * 256));
    CK(cudaMemset(c.buf[g], 0, (size_t)n * 256));
    CK(cudaMalloc(&c.rows[g], (size_t)n * 8));
    CK(cudaStreamCreate(&c.st[g]));
    CK(cudaEventCreate(&c.e0[g]));
    CK(cudaEventCreate(&c.e1[g]));
  }
  int logG = 0;
  while ((1 << logG) < G) ++logG;
  std::vector<Peers> peers(G);
  for (int g = 0; g < G; ++g) {
    peers[g].G = G; peers[g].logG = logG; peers[g].me = g;
    for (int h = 0; h < G; ++h) peers[g].base[h] = c.shard[h];
  }
  std::vector<long long> h(n);
  // request lists.  mode 0: uniform random global rows, ALL remote (owner != me); mode 1: uniform incl. local (1/G local);
  // mode 2: sequential remote rows (owner round-robin over peers, consecutive local rows); mode 3: queue order for the push
  // (sorted by owner, consecutive slots per owner)
  auto fill = [&](int mode, int lpr_rows_div) {
    const long long srows = shard_rows / lpr_rows_div;
    for (int g = 0; g < G; ++g) {
      uint64_t s = 1234 + g;
      for (long long i = 0; i < n; ++i) {
        long long owner, lrow;
        if (mode == 0) { owner = (g + 1 + (long long)(splitmix(s) % (G - 1))) % G; lrow = (long long)(splitmix(s) % srows); }
        else if (mode == 1) { owner = (long long)(splitmix(s) % G); lrow = (long long)(splitmix(s) % srows); }
        else if (mode == 2) { owner = (g + 1 + i % (G - 1)) % G; lrow = (i / (G - 1)) % srows; }
        else { const long long per = (n + G - 2) / (G - 1); owner = (g + 1 + i / per) % G; lrow = (long long)g * per + i % per; }
        h[i] = lrow * G + owner;
      }
      CK(cudaSetDevice(g));
      CK(cudaMemcpy(c.rows[g], h.data(), (size_t)n * 8, cudaMemcpyHostToDevice));
    }
    c.remote_frac = mode == 1 ? (double)(G - 1) / G : 1.0;
  };
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int sms = prop.multiProcessorCount;
  printf("{\"info\": \"%s\", \"G\": %d, \"shard_GB\": %.2f, \"rows\": %lld, \"sms\": %d}\n", prop.name, G, shard_rows * 128 / 1e9, n, sms);

#define PULL(LPR, UB, HINT, CTAS, NAME) \
  run(c, NAME, reps, LPR * 16.0, [&](int g) { pull_ldg<LPR, UB, HINT><<<sms * CTAS, 256, 0, c.st[g]>>>(peers[g], c.rows[g], n, c.buf[g]); })
#define PUSH(LPR, UB, HINT, CTAS, NAME) \
  run(c, NAME, reps, LPR * 16.0, [&](int g) { push_stg<LPR, UB, HINT><<<sms * CTAS, 256, 0, c.st[g]>>>(peers[g], c.rows[g], n, c.buf[g]); })

  fill(2, 1);
  PULL(8, 8, 0, 4, "pull_ldg128 SEQ rows nc.na UB8 4cta");
  PULL(8, 8, 1, 4, "pull_ldg128 SEQ rows plain UB8 4cta");
  fill(0, 1);
  PULL(8, 8, 0, 4, "pull_ldg128 random nc.na UB8 4cta");
  PULL(8, 8, 1, 4, "pull_ldg128 random plain UB8 4cta");
  PULL(8, 8, 2, 4, "pull_ldg128 random relaxed.sys UB8 4cta");
  PULL(8, 2, 0, 1, "pull_ldg128 random nc.na UB2 1cta");
  PULL(8, 2, 0, 4, "pull_ldg128 random nc.na UB2 4cta");
  PULL(8, 4, 0, 2, "pull_ldg128 random nc.na UB4 2cta");
  PULL(8, 4, 0, 8, "pull_ldg128 random nc.na UB4 8cta");
  PULL(8, 16, 0, 4, "pull_ldg128 random nc.na UB16 4cta");
  PULL(8, 16, 0, 8, "pull_ldg128 random nc.na UB16 8cta");
  {
    auto k4 = pull_bulk<4, 8>;
    CK(cudaFuncSetAttribute(k4, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 4 * 4096));
    auto k2 = pull_bulk<2, 8>;
    CK(cudaFuncSetAttribute(k2, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 2 * 4096));
    auto k6 = pull_bulk<6, 8>;
    CK(cudaFuncSetAttribute(k6, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 6 * 4096));
    for (int g = 0; g < G; ++g) {
      CK(cudaSetDevice(g));
      CK(cudaFuncSetAttribute(k4, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 4 * 4096));
      CK(cudaFuncSetAttribute(k2, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 2 * 4096));
      CK(cudaFuncSetAttribute(k6, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 6 * 4096));
    }
    run(c, "pull_bulk128 random NST2 1cta(8w)", reps, 128.0, [&](int g) { k2<<<sms, 256, 8 * 2 * 4096, c.st[g]>>>(peers[g], c.rows[g], n, c.buf[g]); });
    run(c, "pull_bulk128 random NST2 3cta(8w)", reps, 128.0, [&](int g) { k2<<<sms * 3, 256, 8 * 2 * 4096, c.st[g]>>>(peers[g], c.rows[g], n, c.buf[g]); });
    run(c, "pull_bulk128 random NST4 1cta(8w)", reps, 128.0, [&](int g) { k4<<<sms, 256, 8 * 4 * 4096, c.st[g]>>>(peers[g], c.rows[g], n, c.buf[g]); });
    run(c, "pull_bulk128 random NST6 1cta(8w)", reps, 128.0, [&](int g) { k6<<<sms, 256, 8 * 6 * 4096, c.st[g]>>>(peers[g], c.rows[g], n, c.buf[g]); });
  }
  fill(1, 1);
  PULL(8, 8, 0, 4, "pull_ldg128 random incl-local nc.na UB8 4cta");
  PULL(8, 8, 1, 4, "pull_ldg128 random incl-local plain UB8 4cta");
  {
    const int Bs = (int)(n / 40);
    run(c, "pull_sample40 (product shape) incl-local plain 3cta", reps, 128.0, [&](int g) { pull_sample<1><<<sms * 3, 256, 0, c.st[g]>>>(peers[g], c.rows[g], Bs, 40, c.buf[g]); });
    run(c, "pull_sample40 (product shape) incl-local plain 4cta", reps, 128.0, [&](int g) { pull_sample<1><<<sms * 4, 256, 0, c.st[g]>>>(peers[g], c.rows[g], Bs, 40, c.buf[g]); });
    run(c, "pull_sample40 (product shape) incl-local plain 6cta", reps, 128.0, [&](int g) { pull_sample<1><<<sms * 6, 256, 0, c.st[g]>>>(peers[g], c.rows[g], Bs, 40, c.buf[g]); });
    run(c, "pull_sample32 (one chunk per sample) incl-local plain 4cta", reps, 128.0, [&](int g) { pull_sample<1><<<sms * 4, 256, 0, c.st[g]>>>(peers[g], c.rows[g], (int)(n / 32), 32, c.buf[g]); });
  }
  fill(0, 2);
  PULL(16, 8, 0, 4, "pull_ldg256 random (256B rows) nc.na UB8 4cta");
  PULL(16, 4, 0, 4, "pull_ldg256 random (256B rows) nc.na UB4 4cta");
  fill(0, 4);
  PULL(32, 4, 0, 4, "pull_ldg512 random (512B rows) nc.na UB4 4cta");

  // ---------------- push
  fill(3, 1);
  PUSH(8, 8, 0, 4, "push_stg128 QUEUE order plain UB8 4cta");
  PUSH(8, 8, 1, 4, "push_stg128 QUEUE order .cs UB8 4cta");
  PUSH(8, 4, 0, 2, "push_stg128 QUEUE order plain UB4 2cta");
  PUSH(8, 2, 0, 8, "push_stg128 QUEUE order plain UB2 8cta");
  fill(0, 1);
  PUSH(8, 8, 0, 4, "push_stg128 random plain UB8 4cta");
  PUSH(8, 8, 1, 4, "push_stg128 random .cs UB8 4cta");
  {
    auto k4 = push_bulk<4, 8>;
    auto k2 = push_bulk<2, 8>;
    for (int g = 0; g < G; ++g) {
      CK(cudaSetDevice(g));
      CK(cudaFuncSetAttribute(k4, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 4 * 4096));
      CK(cudaFuncSetAttribute(k2, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 2 * 4096));
    }
    run(c, "push_bulk128 random NST4 1cta(8w)", reps, 128.0, [&](int g) { k4<<<sms, 256, 8 * 4 * 4096, c.st[g]>>>(peers[g], c.rows[g], n, c.buf[g]); });
    run(c, "push_bulk128 random NST2 3cta(8w)", reps, 128.0, [&](int g) { k2<<<sms * 3, 256, 8 * 2 * 4096, c.st[g]>>>(peers[g], c.rows[g], n, c.buf[g]); });
    fill(3, 1);
    run(c, "push_bulk128 QUEUE order NST4 1cta(8w)", reps, 128.0, [&](int g) { k4<<<sms, 256, 8 * 4 * 4096, c.st[g]>>>(peers[g], c.rows[g], n, c.buf[g]); });
  }
  return 0;
}
