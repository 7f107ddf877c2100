// All weight-gradient GEMMs of one PPO mini-batch in ONE persistent launch (wgmma, TF32).
//
//   dW_l[out x in] += dZ_l^T X_l ,  db_l[out] += colsum(dZ_l)        for every layer l, reduction over the mini-batch rows
//
// A work item is (layer, slab of rows); the host sizes the slabs of each layer by its cost per row so that the items cost about the
// same, and deals them to one persistent CTA per SM, so the split-K epilogue is amortised and there are no launch gaps between layers.
//
// The contraction index is the ROW of both sources, and wgmma takes TF32 operands K-major only.  Chunks of 32 rows are staged in their
// source layout with 16-byte cp.async several chunks ahead; one pass per chunk writes them as K-major tiles (with the zero fill, the
// 3xTF32 low parts and the bias sums), then the two warpgroups, owning output rows [0, 64) and [64, 128), multiply.  Each keeps its
// accumulator in registers over the whole slab and reduces it into dW with vector atomics at the end.
#pragma once
#include <stdlib.h>

#include <algorithm>
#include <cmath>

#include "gemm_tc2.cuh"

namespace dwbc {

constexpr int WG_MAX = 20;
constexpr int WG_THREADS = 256;                   // two warpgroups: every thread copies, transposes and multiplies
constexpr int WG_KC = 32;                         // rows per chunk
constexpr int WG_TILE = WG_KC * 128;              // floats per tile (staged or K-major): 128 features x 32 rows, 16 KB
// staged chunks in flight: {G, X} per stage, then the K-major tiles {G, X} (+ {G_lo, X_lo} in 3xTF32 mode); 14 tiles = 224 KB
template <bool X3> constexpr int wg_stages() { return X3 ? 5 : 6; }
constexpr size_t WG_SMEM = (size_t)14 * WG_TILE * sizeof(float);
static_assert(2 * wg_stages<true>() + 4 <= 14 && 2 * wg_stages<false>() + 2 <= 14, "shared-memory plan");

struct WGItem {
  RowMat G, X;          // dZ [rows x Mo], X [rows x Ni]
  float* dW; int64_t lddw;
  float* db;            // nullable
  int Mo, Ni;
  int nslab, first;     // work items of this GEMM, index of its first item (set by launch_wgrad_group)
};
// Work items are enumerated GEMM by GEMM, GEMMs in the order launch_wgrad_group sorted them (longest item first).
// snake == 0: item e goes to CTA e % grid (round-robin); snake != 0: round j of the deal runs forwards for even j, backwards for odd j.
// Slab s of a GEMM with n slabs covers rows [b(s), b(s + 1)), b(s) = floor(s rows / n) rounded down to a whole chunk, b(n) = rows.
// rev != 0: the slabs of a GEMM are taken from the LAST rows to the first.
struct WGroup { int n, rows, items, snake, rev; WGItem it[WG_MAX]; };

__device__ __forceinline__ void wg_cp16(float* dst, const float* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(tc_smem_u32(dst)), "l"(src) : "memory");
}
// row-major operands whose rows are 16-byte aligned are staged with 16-byte copies, the others with plain loads
__device__ __forceinline__ bool wg_vec(const RowMat& R) {
  return !R.image() && (reinterpret_cast<uintptr_t>(R.p) & 15) == 0 && (R.ld & 3) == 0 && (R.stride_g & 3) == 0;
}
// Stage rows [k0, k0 + 32) of operand R (ncol columns) in its source layout, element (k, f) of the chunk at float
// ((k/8)*32 + f/4)*32 + (k%8)*4 + f%4: a chunk of a 128-row tile image is one contiguous 16 KB block and is copied verbatim; thread t
// copies the 16-byte pieces t/32, t/32 + 8, ... of row k0 + t%32 of a row-major operand, whose address `rp` (nullptr past the slab)
// it looked up beforehand.  Rows past the slab and columns past ncol are left as they are: the transposition masks them.
__device__ __forceinline__ void wg_stage(const RowMat& R, bool vec, int ncol, const float* rp, int64_t k0, float* dst, int tid) {
  if (R.image()) {
    const float* src = R.p + (k0 >> 7) * 16384 + (k0 & 127) * 128;
#pragma unroll
    for (int i = 0; i < WG_TILE / 4 / WG_THREADS; ++i) wg_cp16(dst + 4 * (tid + i * WG_THREADS), src + 4 * (tid + i * WG_THREADS));
    return;
  }
  if (rp == nullptr) return;
  const int k = tid & 31;
  float* d = dst + (k >> 3) * 1024 + (k & 7) * 4;
  if (vec) {
    for (int c = tid >> 5; c < (ncol + 3) >> 2; c += WG_THREADS / 32) wg_cp16(d + c * 32, rp + 4 * c);
  } else {
    for (int f = tid >> 5; f < ncol; f += WG_THREADS / 32) d[(f >> 2) * 32 + (f & 3)] = __ldg(rp + f);
  }
}

// One pass from the staged chunk to the K-major tiles the wgmmas read, element (f, k) at float ((f/8)*8 + k/4)*32 + (f%8)*4 + k%4
// (8 x 4 core matrices, 128 B apart in K, 1 KB apart in f): features [0, W), rows past kvalid and features past ncol as zeros, the low
// parts (3xTF32) into `lo`, and for G the column sums of the chunk into bsum.  A warp takes 8 features x 16 rows per step; lane l
// holds feature l%8 and rows 4 (l/8) .. 4 (l/8) + 3, read in an order rotated by r so that the 32 lanes of each read hit 32 banks.
template <bool X3>
__device__ __forceinline__ void wg_transpose(const float* src, float* hi, float* lo, int W, int ncol, int kvalid, int warp, int lane,
                                             float (&bsum)[4]) {
  const int r = ((lane >> 2) & 1) | ((lane >> 4) << 1);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int u = warp + 8 * j;                   // step: features 8 (u/2) .., rows 16 (u%2) ..
    if (u >= W / 4) break;
    const int f = 8 * (u >> 1) + (lane & 7), k4 = 4 * (u & 1) + (lane >> 3);
    const float* s = src + ((k4 >> 1) * 32 + (f >> 2)) * 32 + 16 * (k4 & 1) + (f & 3);
    float w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) w[i] = s[4 * ((i + r) & 3)];          // w[i] = row 4 k4 + (i + r) % 4
    if (r & 2) { float t = w[0]; w[0] = w[2]; w[2] = t; t = w[1]; w[1] = w[3]; w[3] = t; }
    if (r & 1) { const float t = w[3]; w[3] = w[2]; w[2] = w[1]; w[1] = w[0]; w[0] = t; }
    float4 v;
    const bool fon = f < ncol;
    v.x = fon && 4 * k4 + 0 < kvalid ? w[0] : 0.0f;
    v.y = fon && 4 * k4 + 1 < kvalid ? w[1] : 0.0f;
    v.z = fon && 4 * k4 + 2 < kvalid ? w[2] : 0.0f;
    v.w = fon && 4 * k4 + 3 < kvalid ? w[3] : 0.0f;
    const int o = ((f >> 3) * 8 + k4) * 32 + (f & 7) * 4;
    *reinterpret_cast<float4*>(hi + o) = v;
    if (X3) *reinterpret_cast<float4*>(lo + o) = make_float4(tf32_lo(v.x), tf32_lo(v.y), tf32_lo(v.z), tf32_lo(v.w));
    bsum[j] += (v.x + v.y) + (v.z + v.w);
  }
}

// one chunk of one warpgroup: acc[64 x N] += Gt[64 x 32 rows] Xt[N x 32 rows]^T (3xTF32: + Gt_lo Xt^T + Gt Xt_lo^T), committed
template <int N, bool X3>
__device__ __forceinline__ void wg_mma_chunk(float* acc, uint32_t a0, uint32_t b0, uint32_t al, uint32_t bl) {
  uint64_t ad = tc_desc(a0, 128, 1024), bd = tc_desc(b0, 128, 1024), adl = tc_desc(al, 128, 1024), bdl = tc_desc(bl, 128, 1024);
  wg_fence();
#pragma unroll
  for (int kk = 0; kk < WG_KC; kk += 8) {            // one K step = 8 rows = two core matrices: +256 bytes = +16 in the address field
    wg_mma_ss<N>(acc, ad, bd, 1);
    if (X3) {
      wg_mma_ss<N>(acc, adl, bd, 1);
      wg_mma_ss<N>(acc, ad, bdl, 1);
      adl += 16; bdl += 16;
    }
    ad += 16; bd += 16;
  }
  wg_commit();
}

// rows [k_begin, k_end) of one GEMM, N = the instruction width that covers Ni.  Per chunk c: wait for its copies, transpose it, refill
// its stage with chunk c + stages and multiply it; the copies of the next stages - 1 chunks are in flight all the while.
template <int N, bool X3>
__device__ __forceinline__ void wg_slab(const WGItem& g, int64_t k_begin, int64_t k_end, float* smem, int tid, int warp, int lane) {
  constexpr int NS = wg_stages<X3>();
  const int Mo = g.Mo, Ni = g.Ni, mw = Mo <= 64 ? 64 : 128, wgi = warp >> 2;
  const bool mma_on = 64 * wgi < Mo;
  const bool gvec = wg_vec(g.G), xvec = wg_vec(g.X);
  const int nch = (int)((k_end - k_begin + WG_KC - 1) / WG_KC);
  auto row_of = [&](const RowMat& R, int c) -> const float* {
    const int64_t k = k_begin + (int64_t)c * WG_KC + (tid & 31);
    return !R.image() && c < nch && k < k_end ? R.row(k) : nullptr;
  };
  auto stage = [&](int c, const float* gr, const float* xr) {
    if (c < nch) {
      const int64_t k0 = k_begin + (int64_t)c * WG_KC;
      float* st = smem + (c % NS) * 2 * WG_TILE;
      wg_stage(g.G, gvec, Mo, gr, k0, st, tid);
      wg_stage(g.X, xvec, Ni, xr, k0, st + WG_TILE, tid);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  float acc[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.0f;
  float bsum[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll 1
  for (int c = 0; c < NS; ++c) stage(c, row_of(g.G, c), row_of(g.X, c));
#pragma unroll 1
  for (int c = 0; c < nch; ++c) {
    asm volatile("cp.async.wait_group %0;" ::"n"(NS - 1) : "memory");
    __syncthreads();                                  // chunk c staged by all threads
    const float* gr = row_of(g.G, c + NS);            // gather lookups of the refill, in flight during the transposition
    const float* xr = row_of(g.X, c + NS);
    const float* st = smem + (c % NS) * 2 * WG_TILE;
    float* kt = smem + 2 * NS * WG_TILE;             // {G, X, G_lo, X_lo}: the wgmmas of chunk c - 1 are complete
    const int kvalid = (int)min((int64_t)WG_KC, k_end - k_begin - (int64_t)c * WG_KC);
    wg_transpose<X3>(st, kt, kt + 2 * WG_TILE, mw, Mo, kvalid, warp, lane, bsum);
    float bdummy[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    wg_transpose<X3>(st + WG_TILE, kt + WG_TILE, kt + 3 * WG_TILE, N, Ni, kvalid, warp, lane, bdummy);
    tc_fence_async_smem();                            // generic-proxy tile writes -> async-proxy reads of the wgmma
    __syncthreads();                                  // tiles complete, stage c % NS free
    stage(c + NS, gr, xr);
    if (mma_on) {
      const uint32_t a0 = tc_smem_u32(kt) + (uint32_t)wgi * 8192u, b0 = tc_smem_u32(kt + WG_TILE);
      wg_mma_chunk<N, X3>(acc, a0, b0, a0 + 2u * WG_TILE * 4u, b0 + 2u * WG_TILE * 4u);
      // Awaited here: left in flight over the next transposition (wait<1>), the wgmmas are serialised by ptxas (C7514: the
      // descriptors of the next chunk are defined inside the open pipeline stage).  The copies of the next chunks still fly meanwhile.
      wg_wait<0>();
    }
  }
  // bias gradient: lanes l, l + 8, l + 16, l + 24 hold feature l % 8 of a step; warps 2i and 2i + 1 the two row halves
  if (g.db != nullptr) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float b = bsum[j];
      b += __shfl_xor_sync(0xffffffffu, b, 8);
      b += __shfl_xor_sync(0xffffffffu, b, 16);
      const int f = 8 * ((warp + 8 * j) >> 1) + lane;
      if (lane < 8 && warp + 8 * j < mw / 4 && f < Mo) atomicAdd(g.db + f, b);
    }
  }
  // split-K partial straight from the fragments: lane l holds rows l/4 and l/4 + 8 of its warp's 16, columns 8 jj + 2 (l%4) + {0, 1}
  const bool v2 = (g.lddw & 1) == 0 && (reinterpret_cast<uintptr_t>(g.dW) & 7) == 0;
  if (mma_on) {
#pragma unroll
    for (int jj = 0; jj < N / 8; ++jj) {
      const int col = 8 * jj + 2 * (lane & 3);
      if (col >= Ni) continue;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int row = 64 * wgi + 16 * (warp & 3) + (lane >> 2) + 8 * e;
        if (row >= Mo) continue;
        float* dst = g.dW + (int64_t)row * g.lddw + col;
        const float x0 = acc[4 * jj + 2 * e], x1 = acc[4 * jj + 2 * e + 1];
        if (v2 && col + 1 < Ni) asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(x0), "f"(x1) : "memory");
        else { atomicAdd(dst, x0); if (col + 1 < Ni) atomicAdd(dst + 1, x1); }
      }
    }
  }
}

// X3 = error-compensated mode (3xTF32): the low parts G_lo = G - trunc_tf32(G), X_lo go to two more tiles (the tensor core truncates
// the 13 low mantissa bits of the raw tiles itself), and every chunk is three accumulating products: G^T X + G_lo^T X + G^T X_lo.
template <bool X3>
__global__ void __launch_bounds__(WG_THREADS, 1) wgrad_group_kernel(const __grid_constant__ WGroup grp) {
  extern __shared__ __align__(128) float wg_smem[];
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);      // warp-uniform for ptxas: the wgmma control flow depends on it
  const int nb = (int)gridDim.x, bid = (int)blockIdx.x;
  const int items = grp.items, full = items / nb, rem = items - full * nb;
  const int my_items = grp.snake ? full + ((((full & 1) ? nb - 1 - bid : bid) < rem) ? 1 : 0) : full + (bid < rem ? 1 : 0);
  for (int j = 0; j < my_items; ++j) {
    const int e = j * nb + ((grp.snake && (j & 1)) ? nb - 1 - bid : bid);
    int li = 0;
    while (li + 1 < grp.n && e >= grp.it[li + 1].first) ++li;
    const WGItem& g = grp.it[li];
    int slab_i = e - g.first;
    if (grp.rev) slab_i = g.nslab - 1 - slab_i;
    const int64_t k_begin = (int64_t)slab_i * grp.rows / g.nslab / WG_KC * WG_KC;
    const int64_t k_end = slab_i + 1 == g.nslab ? (int64_t)grp.rows : (int64_t)(slab_i + 1) * grp.rows / g.nslab / WG_KC * WG_KC;
    if (k_end <= k_begin) continue;
    const int nw = wg_width((g.Ni + 15) & ~15);
    if (nw == 32) wg_slab<32, X3>(g, k_begin, k_end, wg_smem, tid, warp, lane);
    else if (nw == 64) wg_slab<64, X3>(g, k_begin, k_end, wg_smem, tid, warp, lane);
    else wg_slab<128, X3>(g, k_begin, k_end, wg_smem, tid, warp, lane);
  }
}

struct WGroupBuilder {
  WGroup g{};
  bool ok = true;
  void add(RowMat G, RowMat X, float* dW, int64_t lddw, float* db, int Mo, int Ni) {
    if (g.n >= WG_MAX || Mo > 128 || Ni > 128 || Mo <= 0 || Ni <= 0) { ok = false; return; }
    WGItem& it = g.it[g.n++];
    it.G = G; it.X = X; it.dW = dW; it.lddw = lddw; it.db = db; it.Mo = Mo; it.Ni = Ni;
  }
};

// Longest slab: the accumulator sums a slab's rows in registers, and longer sums lose accuracy against the fp32 reference
constexpr int64_t WG_MAX_SLAB = 1024;
inline int wg_items_per_cta = 4;                     // tuning aid (dwbc_debug_set_wgrad_items)
inline int wg_reverse = 0;                            // tuning aid (dwbc_debug_set_wgrad_reverse): 0 = slabs from the first rows upwards
inline int wg_snake = 0;                             // tuning aid (dwbc_debug_set_wgrad_snake): 0 = round-robin deal

// Time of one row of a GEMM on the H100 roofline: the operand bytes at 3.35 TB/s or the tensor work padded to the instruction widths
// at 495 TFLOP/s (three products in 3xTF32 mode), whichever is larger.  Only the ratios between GEMMs matter.
inline double wg_row_cost(const WGItem& it, bool x3) {
  auto width = [](const RowMat& R, int ncol) { return R.rpg == 0 ? 128 : (ncol + 3) & ~3; };
  const int mw = it.Mo <= 64 ? 64 : 128, n16 = (it.Ni + 15) & ~15, nw = n16 <= 32 ? 32 : (n16 <= 64 ? 64 : 128);
  const double bytes = 4.0 * (width(it.G, it.Mo) + width(it.X, it.Ni));
  const double flop = 2.0 * mw * nw * (x3 ? 3 : 1);
  return std::max(bytes / 3.35e12, flop / 495e12);
}

// Plan: work items of equal cost, a whole number per CTA.  There are wg_items_per_cta per SM, or more when an item of that cost would be
// longer than WG_MAX_SLAB rows of the cheapest GEMM.  Each GEMM gets a number of slabs proportional to its row cost (largest remainder,
// at least rows / WG_MAX_SLAB, at most one per four chunks), so its slabs are the shorter the more a row costs.  The GEMMs are then ordered
// by the cost of one of their items, longest first, so that items rounded short fill the end of the launch.  At small row counts the
// limits leave fewer items.
inline int launch_wgrad_group(WGroup& g, int rows, bool x3, cudaStream_t st) {
  if (g.n <= 0 || rows <= 0) return DWBC_ERR_ARG;
  g.snake = wg_snake;
  g.rev = wg_reverse;
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  }
  g.rows = rows;
  double cost[WG_MAX], total = 0.0, cmin = 1e30;
  for (int i = 0; i < g.n; ++i) {
    total += cost[i] = wg_row_cost(g.it[i], x3);
    cmin = std::min(cmin, cost[i]);
  }
  const int64_t span = WG_MAX_SLAB - WG_KC;           // rows / n, before the slab bounds are rounded down to whole chunks
  const int64_t per_cta = std::max<int64_t>(wg_items_per_cta, (int64_t)std::ceil((double)rows * total / ((double)sms * span * cmin) - 1e-9));
  const int64_t target = per_cta * sms;
  const int64_t lo = (rows + span - 1) / span, hi = std::max<int64_t>(1, rows / (4 * WG_KC));
  int64_t n[WG_MAX], sum = 0;
  double share[WG_MAX];
  for (int i = 0; i < g.n; ++i) {
    share[i] = (double)target * cost[i] / total;
    n[i] = std::min(hi, std::max(lo, (int64_t)share[i]));
    sum += n[i];
  }
  for (; sum < target; ++sum) {                       // largest remainder first
    int best = -1;
    for (int i = 0; i < g.n; ++i)
      if (n[i] < hi && (best < 0 || share[i] - n[i] > share[best] - n[best])) best = i;
    if (best < 0) break;
    ++n[best];
  }
  double item_cost[WG_MAX];
  for (int i = 0; i < g.n; ++i) {
    g.it[i].nslab = (int)n[i];
    item_cost[i] = cost[i] / (double)n[i];
  }
  int order[WG_MAX];
  for (int i = 0; i < g.n; ++i) order[i] = i;
  std::stable_sort(order, order + g.n, [&](int a, int b) { return item_cost[a] > item_cost[b]; });
  WGItem sorted[WG_MAX];
  int items = 0;
  for (int i = 0; i < g.n; ++i) {
    sorted[i] = g.it[order[i]];
    sorted[i].first = items;
    items += sorted[i].nslab;
  }
  std::copy(sorted, sorted + g.n, g.it);
  g.items = items;
  const int grid = items < sms ? items : sms;
  static bool attr = false;
  if (!attr) {
    if (cudaFuncSetAttribute(wgrad_group_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WG_SMEM) != cudaSuccess ||
        cudaFuncSetAttribute(wgrad_group_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WG_SMEM) != cudaSuccess)
      return DWBC_ERR_LAUNCH;
    attr = true;
  }
  if (x3) wgrad_group_kernel<true><<<grid, WG_THREADS, WG_SMEM, st>>>(g);
  else wgrad_group_kernel<false><<<grid, WG_THREADS, WG_SMEM, st>>>(g);
  ++dwbc_launch_counter;
  return cudaGetLastError() == cudaSuccess ? DWBC_OK : DWBC_ERR_LAUNCH;
}

// one weight gradient on its own (the layer-wise path): dW[M x N] += A^T B over K rows, db += colsum(A)
inline int launch_wgrad_one(const GemmArgs& a, cudaStream_t st) {
  WGroupBuilder b;
  b.add(a.A, a.B, a.C, a.ldc, a.dbias, a.M, a.N);
  if (!b.ok) return DWBC_ERR_ARG;
  return launch_wgrad_group(b.g, a.K, false, st);
}

}  // namespace dwbc
