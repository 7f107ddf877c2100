// Warp-specialised, mbarrier-pipelined wgmma GEMM (TF32 in, FP32 accumulate in registers) -- the layer-wise tensor-core
// path (history encoder, DAgger update, network shapes the fused chains do not cover).  Two phases of a tile overlap:
//
//   warps 0-3  PRODUCERS : gather + pad the A operand of tile i+1 into shared-memory stage (i+1)%2 while ...
//   warps 4-7  CONSUMERS : ... one warpgroup issues the wgmma chain of tile i (two 64-row halves), writes its accumulator
//                          fragments over the consumed A stage and fuses bias / activation / act' into coalesced row stores.
//
//   FWD / BWD_DATA: CTA = persistent over 128-row tiles; weights (<= 64 KB) resident in smem; 2 A stages of 66 KB.
//   BWD_WGT      : the grouped weight-gradient kernel (wgrad_group.cuh) with a single GEMM.
//
// The gather index of a tile is prefetched to shared memory first so every operand load is a single round trip,
// and each producer thread keeps 8 independent 16-byte loads in flight.
#pragma once
#include "tc_common.cuh"

namespace dwbc {

constexpr int T2_PROD = 128, T2_EPI = 128;
constexpr int T2_THREADS = T2_PROD + T2_EPI;        // 256: the consumers are warps 4-7, an aligned warpgroup
constexpr int T2_WCH = 64;                          // rows per weight-gradient chunk
constexpr int T2_LDS = TC_MAXN + 4;                 // padded row stride (floats) of the epilogue staging tile: conflict-free float4 rows

__device__ __forceinline__ void t2_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(tc_smem_u32(bar)) : "memory");
}
// named barriers are the warp-aligned form: reconverge the warp first (a lane may still be behind a single-lane mbarrier arrive)
__device__ __forceinline__ void t2_pbar() { __syncwarp(); asm volatile("bar.sync 2, %0;" ::"n"(T2_PROD) : "memory"); }   // producers only
__device__ __forceinline__ void t2_ebar() { __syncwarp(); asm volatile("bar.sync 3, %0;" ::"n"(T2_EPI) : "memory"); }    // epilogue only

// profiling aid: clock64 stamps of CTA events, [grid][64] (set with dwbc_debug_set_tc_cycle_buffer)
__device__ unsigned long long* g_tc_cycles = nullptr;
#define T2_STAMP(slot) do { if (g_tc_cycles && (slot) < 64) g_tc_cycles[blockIdx.x * 64 + (slot)] = clock64(); } while (0)

struct T2Shared {
  uint64_t full[2], empty[2];
  int64_t rowoff[128];     // gathered row offsets (floats) of the tile being filled
};

// the wgmma chain of one 128-row tile: acc[h] = rows [64 h, 64 h + 64) x N columns
template <int N>
__device__ __forceinline__ void t2_mma_tile(float (&acc)[2][64], uint32_t a0, uint32_t b0, int kpad) {
  const uint32_t sbo = (uint32_t)(kpad >> 2) * 128u;
  wg_fence();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    uint64_t ad = tc_desc(a0 + (uint32_t)h * 8u * sbo, 128, sbo), bd = tc_desc(b0, 128, sbo);
    for (int kk = 0; kk < kpad; kk += 8, ad += 16, bd += 16) wg_mma_ss<N>(acc[h], ad, bd, kk > 0);   // one K step = two 16-byte pieces = 256 bytes
  }
  wg_commit();
  wg_wait<0>();
}

// K-major fill by the 128 producer threads, rows addressed through a row-offset table in shared memory
__device__ __forceinline__ void t2_fill_rows(float* smem, const float* base, const int64_t* rowoff, int nrows, int rows_pad, int kvalid, int kpad,
                                             bool vec, int ptid) {
  const int chunks = kpad >> 2, total = rows_pad * chunks;
  for (int b0 = ptid; b0 < total; b0 += 8 * T2_PROD) {
    float4 v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int i = b0 + u * T2_PROD;
      v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (i < total) {
        const int r8 = i & 7, c = (i >> 3) % chunks, g = (i >> 3) / chunks;
        const int r = g * 8 + r8;
        if (r < nrows) {
          const float* src = base + rowoff[r] + 4 * c;
          if (vec && 4 * c + 3 < kvalid) v[u] = ldg_stream(reinterpret_cast<const float4*>(src));
          else {
            if (4 * c + 0 < kvalid) v[u].x = src[0];
            if (4 * c + 1 < kvalid) v[u].y = src[1];
            if (4 * c + 2 < kvalid) v[u].z = src[2];
            if (4 * c + 3 < kvalid) v[u].w = src[3];
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int i = b0 + u * T2_PROD;
      if (i < total) *reinterpret_cast<float4*>(smem + (size_t)i * 4) = v[u];
    }
  }
}
// same fill with cp.async (LDGSTS, 16 B, zero-fill): no register staging, so a producer warp keeps its whole share
// of the tile (64 KB per CTA) in flight.  Requires 16-byte aligned rows and kvalid % 4 == 0.
__device__ __forceinline__ void t2_fill_rows_async(float* smem, const float* base, const int64_t* rowoff, int nrows, int rows_pad, int kvalid,
                                                   int kpad, int ptid) {
  const int chunks = kpad >> 2, total = rows_pad * chunks;
  const uint32_t s0 = tc_smem_u32(smem);
  const int r8 = ptid & 7;                       // T2_PROD % 8 == 0: a thread always serves the same row-in-group
  int c = ptid >> 3, g = 0;                      // (i >> 3) = c + g * chunks, advanced incrementally (no divisions)
  while (c >= chunks) { c -= chunks; ++g; }
#pragma unroll 4
  for (int i = ptid; i < total; i += T2_PROD) {
    const int r = g * 8 + r8;
    const float* src = base;
    int nb = 0;
    if (r < nrows && 4 * c < kvalid) { src = base + rowoff[r] + 4 * c; nb = 16; }
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s0 + (uint32_t)i * 16), "l"(src), "r"(nb) : "memory");
    c += T2_PROD >> 3;
    while (c >= chunks) { c -= chunks; ++g; }
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
}
// transposing K-major fill (source indexed [k][mn])
__device__ __forceinline__ void t2_fill_T(float* smem, const float* base, const int64_t* rowoff, int nk, int kpad, int mnvalid, int mnpad,
                                          bool vec, int ptid) {
  const int chunks = mnpad >> 2, kq = kpad >> 2, cg = (chunks + 3) >> 2, total = (kpad >> 3) * cg * 32;
  for (int b0 = ptid; b0 < total; b0 += 8 * T2_PROD) {
    float4 v[8];
    int cc[8], kk[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int i = b0 + u * T2_PROD;
      const int k8 = i & 7, c4 = (i >> 3) & 3, rest = i >> 5;
      const int c = (rest % cg) * 4 + c4, k = (rest / cg) * 8 + k8;
      cc[u] = (i < total && c < chunks) ? c : -1;
      kk[u] = k;
      v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (cc[u] >= 0 && k < nk) {
        const float* src = base + rowoff[k] + 4 * c;
        if (vec && 4 * c + 3 < mnvalid) v[u] = ldg_stream(reinterpret_cast<const float4*>(src));
        else {
          if (4 * c + 0 < mnvalid) v[u].x = src[0];
          if (4 * c + 1 < mnvalid) v[u].y = src[1];
          if (4 * c + 2 < mnvalid) v[u].z = src[2];
          if (4 * c + 3 < mnvalid) v[u].w = src[3];
        }
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      if (cc[u] < 0) continue;
      const float vv[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
      const int k = kk[u];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int mn = 4 * cc[u] + j;
        smem[((size_t)((mn >> 3) * kq + (k >> 2)) * 8 + (mn & 7)) * 4 + (k & 3)] = vv[j];
      }
    }
  }
}

template <int kMode>
__global__ void __launch_bounds__(T2_THREADS, 1) gemm_tc2_kernel(const GemmArgs g, const int items, const int vecA, const int vecB) {
  extern __shared__ __align__(128) float t2_smem[];
  __shared__ T2Shared sh;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  static_assert(kMode != GEMM_BWD_WGT, "weight gradients run on wgrad_group_kernel");

  if (tid == 0) {
    for (int i = 0; i < 2; ++i) { tc_mbar_init(&sh.full[i], T2_PROD); tc_mbar_init(&sh.empty[i], T2_EPI); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) T2_STAMP(0);
  const int my_items = blockIdx.x < items ? (items - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

  const int N = g.N, K = g.K;
  const int npad = (N + 15) & ~15, kpad = (K + 7) & ~7;
  float* sB = t2_smem;
  float* sA[2] = {t2_smem + TC_MAXN * TC_MAXK, t2_smem + TC_MAXN * TC_MAXK + TC_M * T2_LDS};   // stages double as epilogue staging [128][132]
  if (warp < 4) {
    // ===================== PRODUCERS =====================
    const int ptid = tid;
    // weight operand once (rows of B are plain: no gather)
    if (kMode == GEMM_FWD) {
      for (int r = ptid; r < 128; r += T2_PROD) sh.rowoff[r] = g.B.row(r < N ? r : 0) - g.B.p;
      t2_pbar();
      if ((vecB & 1) && (K & 3) == 0) t2_fill_rows_async(sB, g.B.p, sh.rowoff, N, npad, K, kpad, ptid);
      else t2_fill_rows(sB, g.B.p, sh.rowoff, N, npad, K, kpad, vecB & 1, ptid);
      if (ptid == 0) T2_STAMP(1);
    } else {
      for (int r = ptid; r < 128; r += T2_PROD) sh.rowoff[r] = g.B.row(r < K ? r : 0) - g.B.p;
      t2_pbar();
      t2_fill_T(sB, g.B.p, sh.rowoff, K, kpad, N, npad, vecB & 1, ptid);
    }
    for (int j = 0; j < my_items; ++j) {
      const int it = blockIdx.x + j * gridDim.x, s = j & 1;
      const int64_t m0 = (int64_t)it * TC_M;
      const int rows = (int)min((int64_t)TC_M, (int64_t)g.M - m0);
      t2_pbar();                                        // previous tile's reads of rowoff are done
      if (ptid < TC_M) sh.rowoff[ptid] = ptid < rows ? (g.A.row(m0 + ptid) - g.A.p) : 0;
      tc_mbar_wait(&sh.empty[s], ((j >> 1) & 1) ^ 1);   // stage free (epilogue of tile j-2 done)
      t2_pbar();
      if ((vecA & 1) && (K & 3) == 0) t2_fill_rows_async(sA[s], g.A.p, sh.rowoff, rows, TC_M, K, kpad, ptid);
      else t2_fill_rows(sA[s], g.A.p, sh.rowoff, rows, TC_M, K, kpad, vecA & 1, ptid);
      tc_fence_async_smem();                            // generic-proxy operand writes -> async-proxy reads of the wgmma
      t2_arrive(&sh.full[s]);
      if (ptid == 0) T2_STAMP(2 + j);
    }
  } else {
    // ===================== CONSUMERS: wgmma + epilogue =====================
    // phase A: wgmma, accumulator fragments -> padded staging tile in the (now consumed) A stage;  phase B: warp per row,
    // lane per 4 columns: fully coalesced 512-byte row stores with bias / activation / act' fused.
    const int ew = warp - 4;                       // 0..3
    const int n4 = 4 * lane;
    float bias4[4] = {0.f, 0.f, 0.f, 0.f};
    if (kMode == GEMM_FWD && g.bias)
      for (int qq = 0; qq < 4; ++qq) if (n4 + qq < N) bias4[qq] = __ldg(g.bias + n4 + qq);
    const bool c_al = ((g.ldc & 3) == 0) && ((reinterpret_cast<uintptr_t>(g.C) & 15) == 0);
    const int nw = wg_width(npad);
    for (int j = 0; j < my_items; ++j) {
      const int it = blockIdx.x + j * gridDim.x, s = j & 1;
      const int64_t m0 = (int64_t)it * TC_M;
      const int rows = (int)min((int64_t)TC_M, (int64_t)g.M - m0);
      float* stg = sA[s];
      tc_mbar_wait(&sh.full[s], (j >> 1) & 1);
      if (tid == T2_PROD) T2_STAMP(16 + 4 * j);
      float acc[2][64];
      // (the weight rows past npad of the instruction width are whatever the buffer holds: their output columns are never read)
      if (nw == 32) t2_mma_tile<32>(acc, tc_smem_u32(sA[s]), tc_smem_u32(sB), kpad);
      else if (nw == 64) t2_mma_tile<64>(acc, tc_smem_u32(sA[s]), tc_smem_u32(sB), kpad);
      else t2_mma_tile<128>(acc, tc_smem_u32(sA[s]), tc_smem_u32(sB), kpad);
      t2_ebar();                                   // every warp's part of the wgmma has read the A stage
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float* srow = stg + (size_t)(64 * h + 16 * ew + (lane >> 2)) * T2_LDS + 2 * (lane & 3);
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          if (8 * jj < nw) {
            *reinterpret_cast<float2*>(srow + 8 * jj) = make_float2(acc[h][4 * jj], acc[h][4 * jj + 1]);
            *reinterpret_cast<float2*>(srow + 8 * T2_LDS + 8 * jj) = make_float2(acc[h][4 * jj + 2], acc[h][4 * jj + 3]);
          }
        }
      }
      t2_ebar();
      if (tid == T2_PROD) T2_STAMP(17 + 4 * j);
      if (n4 < N) {
        const bool full = n4 + 3 < N;
        for (int r0 = ew; r0 < rows; r0 += 16) {          // 4 independent rows per iteration (ILP over the dependent exp / store chains)
          float x[4][4], y[4][4];
          bool ok[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int r = r0 + 4 * u;
            ok[u] = r < rows;
            const float4 a = ok[u] ? *reinterpret_cast<const float4*>(stg + (size_t)r * T2_LDS + n4) : make_float4(0.f, 0.f, 0.f, 0.f);
            x[u][0] = a.x; x[u][1] = a.y; x[u][2] = a.z; x[u][3] = a.w;
            y[u][0] = y[u][1] = y[u][2] = y[u][3] = 0.f;
            if (!ok[u]) continue;
            const int64_t m = m0 + r;
            if (g.beta) {
              const float* crow = g.C + m * g.ldc + n4;
              if (full && c_al) { const float4 o = *reinterpret_cast<const float4*>(crow); x[u][0] += o.x; x[u][1] += o.y; x[u][2] += o.z; x[u][3] += o.w; }
              else for (int qq = 0; qq < 4; ++qq) if (n4 + qq < N) x[u][qq] += crow[qq];
            }
            if (kMode == GEMM_BWD_DATA && g.act != ACT_NONE) {
              const float* xr = g.Xact.row(m) + n4;
              if (full && ((reinterpret_cast<uintptr_t>(xr) & 15) == 0)) { const float4 o = *reinterpret_cast<const float4*>(xr); y[u][0] = o.x; y[u][1] = o.y; y[u][2] = o.z; y[u][3] = o.w; }
              else for (int qq = 0; qq < 4; ++qq) if (n4 + qq < N) y[u][qq] = xr[qq];
            }
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
#pragma unroll
            for (int qq = 0; qq < 4; ++qq) {
              float tt = x[u][qq];
              if (kMode == GEMM_FWD) {
                tt += bias4[qq];
                tt = act_f<true>(g.act, tt);   // ex2.approx: 2 ulp, far below the TF32 input rounding
              } else if (g.act != ACT_NONE) tt *= act_df(g.act, y[u][qq]);
              x[u][qq] = tt;
            }
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            if (!ok[u]) continue;
            float* crow = g.C + (m0 + r0 + 4 * u) * g.ldc + n4;
            if (full && c_al) *reinterpret_cast<float4*>(crow) = make_float4(x[u][0], x[u][1], x[u][2], x[u][3]);
            else for (int qq = 0; qq < 4; ++qq) if (n4 + qq < N) crow[qq] = x[u][qq];
          }
        }
      }
      t2_ebar();
      if (tid == T2_PROD) T2_STAMP(18 + 4 * j);
      t2_arrive(&sh.empty[s]);                     // staging (= A stage s) free for the producers
    }
  }
}

template <int kMode>
inline int launch_gemm_tc2(const GemmArgs& g_in, cudaStream_t st) {
  GemmArgs g = g_in;
  if (g.M <= 0 || g.N <= 0 || g.K <= 0) return DWBC_ERR_ARG;
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  }
  const int items = (g.M + TC_M - 1) / TC_M;
  const int grid = items < sms ? items : sms;
  const size_t smem = (size_t)(TC_MAXN * TC_MAXK + 2 * TC_M * T2_LDS) * sizeof(float);   // 196 KB: {B, A0, A1 (padded)}
  static bool attr[2] = {false, false};
  if (!attr[kMode]) {
    if (cudaFuncSetAttribute(gemm_tc2_kernel<kMode>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return DWBC_ERR_LAUNCH;
    attr[kMode] = true;
  }
  gemm_tc2_kernel<kMode><<<grid, T2_THREADS, smem, st>>>(g, items, rowmat_vec_ok(g.A) ? 1 : 0, rowmat_vec_ok(g.B) ? 1 : 0);
  ++dwbc_launch_counter;
  return cudaGetLastError() == cudaSuccess ? DWBC_OK : DWBC_ERR_LAUNCH;
}

// precision of the ActorCritic GEMMs of the current call (defined in mlp.cu): 0 = fp32 CUDA cores (parity anchor), 1 = TF32 wgmma,
// 2 = 3xTF32: the fused chain / grouped weight-gradient kernels compensate the truncation; these layer-wise GEMMs (history encoder,
// DAgger) then run on the exact fp32 kernels
extern thread_local int mlp_precision;

inline int launch_wgrad_one(const GemmArgs& g, cudaStream_t st);   // wgrad_group.cuh

template <int kMode>
inline int dispatch_gemm(const GemmArgs& g, cudaStream_t st) {
  if (mlp_precision == 1 && tc_shape_ok(kMode, g)) {
    if constexpr (kMode == GEMM_BWD_WGT) return launch_wgrad_one(g, st);
    else return launch_gemm_tc2<kMode>(g, st);
  }
  return launch_gemm<kMode>(g, st);
}

// Y = act(beta*Y + X W^T + b)
inline int linear_fwd(RowMat X, const float* W, int64_t ldw, const float* b, float* Y, int64_t ldy, int M, int N, int K,
                      int act, int beta, cudaStream_t st) {
  GemmArgs g{};
  g.A = X; g.B = rowmat(W, ldw); g.C = Y; g.ldc = ldy; g.bias = b; g.act = act; g.beta = beta; g.M = M; g.N = N; g.K = K;
  return dispatch_gemm<GEMM_FWD>(g, st);
}
// dX[M x Nin] = (beta*dX + G[M x Nout] W[Nout x Nin]) * act'(Xact)
inline int linear_bwd_data(RowMat G, const float* W, int64_t ldw, float* dX, int64_t lddx, int M, int Nin, int Nout,
                           int act, RowMat Xact, int beta, cudaStream_t st) {
  GemmArgs g{};
  g.A = G; g.B = rowmat(W, ldw); g.C = dX; g.ldc = lddx; g.act = act; g.Xact = Xact; g.beta = beta; g.M = M; g.N = Nin; g.K = Nout;
  return dispatch_gemm<GEMM_BWD_DATA>(g, st);
}
// dW[Nout x Nin] += G^T X ; db += colsum(G)   (over `rows` rows)
inline int linear_bwd_weight(RowMat G, RowMat X, float* dW, int64_t lddw, float* db, int rows, int Nout, int Nin, cudaStream_t st) {
  GemmArgs g{};
  g.A = G; g.B = X; g.C = dW; g.ldc = lddw; g.dbias = db; g.M = Nout; g.N = Nin; g.K = rows;
  g.k_chunk = simt_wgrad_chunk(Nout, Nin, rows);
  g.part = mlp_wpart;
  return dispatch_gemm<GEMM_BWD_WGT>(g, st);
}

}  // namespace dwbc
