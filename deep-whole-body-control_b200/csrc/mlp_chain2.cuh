// Fused layer chains of the ActorCritic (AC:86-353) on the Hopper tensor cores (wgmma, TF32 in, FP32 accumulate in registers).
//
//   * A CTA works on one or two 128-row tiles (slots X and Y).  Each slot owns ONE operand tile in shared memory that every op updates
//     in place: two warpgroups multiply the tile with the op's weight image (64 rows each), run the op's epilogue on their accumulator
//     fragments and write the result back into the tile as the next op's operand.  A third warpgroup gives its registers to the workers
//     (setmaxnreg 40 / 232); its first warp streams the weight images in with bulk copies, the image of op i+1 behind the epilogue of op i.
//     All wgmmas of an op form one pipeline: one wait per op, not per instruction.  ptxas silently falls back to fencing and awaiting
//     every wgmma when the control flow around them does not look warp-uniform to it (C7520), which values loaded from shared memory (the
//     queue item, the program's fields) do not: those pass through c2_uni.  The wgmmas of an op are still issued and awaited by the warps
//     that run its epilogue, so nothing of the tensor-core work overlaps that epilogue.  The workers use all 232 registers and spill the
//     prefetched activation chunks of the backward epilogue (x) to local memory around the 3xTF32 wgmmas.
//   * Both slots run the same program, so one weight image per op serves two tiles (half the L2 traffic per tile).
//   * The trunk a second head needs is re-read from the activation buffer the backward pass needs anyway (L2 hit) instead
//     of occupying a second shared-memory tile.
//   * "3xTF32" (precision 2): x = hi + lo with hi = the 19 leading bits the tensor core reads (it TRUNCATES the 13 low mantissa bits
//     of a 32-bit operand) and lo = x - hi (exact in fp32).  D = A_hi W_hi + A_lo W_hi + A_hi W_lo: the first and third products read the
//     fp32 tile / the raw and the "lo" weight image from shared memory, the second takes A_lo as a register operand, formed by each
//     thread from its A fragment for the whole op before / while its wgmmas run (c2_mma_op).  The dropped A_lo W_lo term is 2^-22 relative: fp32-grade results.  The "lo" image occupies the second
//     slot's tile, so 3xTF32 items hold one tile.
//   * The heads' epilogues finish the job (north_star: "log-prob, ratio/clip/min and entropy fused into the epilogue"):
//     rollout: action sampling + two-channel Gaussian log-prob (AC:326-345); update: PPO surrogate / clipped value loss /
//     entropy / privileged-latent regulariser and their gradients w.r.t. the network outputs (PPO:166-221).
//   * Work items (program, tile pair) are handed out through an atomic queue (longest program first).
//
// Tile geometry: [128 rows x 128 k] fp32, element (r, k) at float ((r/8)*32 + k/4)*32 + (r%8)*4 + k%4
// (8-row x 16-byte core matrices, LBO = 128 B, SBO = 4096 B).
#pragma once
#include <stdlib.h>

#include <algorithm>
#include <functional>
#include <vector>

#include "gemm_tc2.cuh"
#include "ppo_terms.cuh"

namespace dwbc {

constexpr int C2_MAX_OPS = 12, C2_MAX_LOADS = 6, C2_MAX_PACK = 36, C2_MAX_PROGS = 4;   // pack items of one launch: forward + backward programs of both networks
constexpr int C2_TILE = 128 * 128;                       // floats per operand tile
constexpr int C2_WORKERS = 8;                            // load / wgmma / epilogue warps: two warpgroups, warp w owns tile rows [16 w, 16 w + 16)
constexpr int C2_H = 2;                                  // column groups of the epilogue: half-warp h takes the 32-column chunks h and h + 2
constexpr int C2_CPW = 4 / C2_H;                         // chunks per thread and op (N <= 128)
constexpr int C2_THREADS = 32 * (C2_WORKERS + 4);        // + a third warpgroup whose first warp (warp 8) copies the weight images
constexpr int C2_REGS_WORKER = 232, C2_REGS_COPY = 40;   // setmaxnreg: 256 x 232 + 128 x 40 = 64 512 of the SM's 65 536 registers
constexpr int C2_KSET = TC_MAXK / 16;                    // 3xTF32: K steps per set of A_lo fragment registers (two sets cover kpad <= 128)
constexpr int C2_NW = 32 * C2_WORKERS;                   // 256 worker threads
constexpr int C2_SMEM_FLOATS = 3 * C2_TILE + 2 * 128 + C2_WORKERS * 1024;    // tile X, tile Y, weight image, two bias slots, transposition buffers

enum { FIN_NONE = 0, FIN_ACT = 1, FIN_PPO = 2, FIN_VALUE = 3, FIN_REG = 4 };

struct C2Load {
  RowMat src;        // rows of the source (already offset to the first column)
  int ncols;         // columns copied (multiple of 4)
  int col0;          // destination column (multiple of 4)
  int zero_to;       // columns [col0 + ncols, zero_to) are zero-filled (K padding of the consuming op)
  int before_op;     // issued once the ops < before_op of the slot have retired (0: with the item)
  int img;           // 1: src.p is a tile-image buffer (RowMat::image): the whole 128 x 128 tile arrives as ONE bulk copy (ncols = 128, col0 = 0)
};
struct C2Op {
  const float* wp;       // packed image: canonical K-major [npad x kpad] weights, then [npad] bias
  const float* wp_lo;    // 3xTF32: image of the low parts (no bias); null otherwise
  float* y;              // global output (nullable), row-major
  int64_t ldy;
  int a_col0, kpad;      // first column of the A window inside the tile (multiple of 4), padded reduction length (multiple of 8)
  int N, npad;           // outputs (npad: multiple of 16)
  int act;               // forward: activation; backward: activation whose derivative multiplies
  int out_col0;          // column of the tile the result is written to (multiple of 32), -1: none
  int mode;              // 0 forward (bias + act), 1 backward ((+ add) * act'(xact))
  const float* xact; int64_t ldx;     // backward: activation OUTPUT [M x ldx] whose derivative multiplies; null: none
  const float* add; int64_t ldadd;    // backward: optional addend [M x ldadd]
  int fin, fin_c;        // epilogue hook of a head's last op and its channel (0 leg, 1 arm)
  int y_img;             // 1: y is a tile-image buffer: the finished tile goes there with one bulk copy (no thread stores)
  int x_img;             // 1: xact is a tile-image buffer
};
struct alignas(16) C2Prog {
  int M, n_loads, n_ops, pad_;
  C2Load ld[C2_MAX_LOADS];
  C2Op op[C2_MAX_OPS];
};
static_assert(sizeof(C2Prog) % 16 == 0, "copied to shared memory in 16-byte pieces");

struct C2Launch {
  int nprog, x3;             // programs (1 or 2), error-compensated mode
  // work items of ONE program: np2 two-tile items over the tiles [0, 2 np2), then ns1 one-tile items over the rest.  All two-tile items (of
  // every program, longest program first) are queued in front of all one-tile items: the tail of a launch is filled with half-size items
  // (launch_chain2 picks ns1 by simulating the queue on the SM count)
  int np2, ns1;
  int rev;                   // tiles are taken from the last one downwards
  int* queue;                // [2] device counters (next item, finished CTAs), zero between launches
  C2Prog p[C2_MAX_PROGS];
  FinArgs fin;
};

// ---- weight packing ---------------------------------------------------------------------------------------------------
// image(n, k) of an op: up to two column segments of the source map into the K window of the tile,
//   transpose = 0: image(n, k) = w[n * ldw + ksrc]     (forward: W [N x K])
//   transpose = 1: image(n, k) = w[ksrc * ldw + n]     (backward: W [Kout x Nin], D = dZ W)
// for k = kdst + j, ksrc = ksrc0 + j, j < len; zero elsewhere and for n >= N.  With `lo` the image of w - trunc_tf32(w) is written too.
struct C2PackSeg { int kdst, ksrc, len; };
struct C2PackItem { const float* w; int64_t ldw; const float* bias; int N, npad, kpad, transpose, nseg; C2PackSeg seg[2]; int64_t dst, dst_lo; };
struct C2PackList { int n; float* out; C2PackItem it[C2_MAX_PACK]; };

__global__ void pack_weights2_kernel(const __grid_constant__ C2PackList pl) {
  const C2PackItem& it = pl.it[blockIdx.y];
  const int wn = it.npad * it.kpad, total = wn + it.npad;
  float* dst = pl.out + it.dst;
  float* dlo = it.dst_lo >= 0 ? pl.out + it.dst_lo : nullptr;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    if (i < wn) {
      const int n = i / it.kpad, k = i - n * it.kpad;
      float v = 0.0f;
      if (n < it.N) {
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          if (s < it.nseg) {
            const int j = k - it.seg[s].kdst;
            if (j >= 0 && j < it.seg[s].len) {
              const int ks = it.seg[s].ksrc + j;
              v = it.transpose ? it.w[(int64_t)ks * it.ldw + n] : it.w[(int64_t)n * it.ldw + ks];
            }
          }
        }
      }
      const size_t o = ((size_t)((n >> 3) * (it.kpad >> 2) + (k >> 2)) * 8 + (n & 7)) * 4 + (k & 3);
      dst[o] = v;
      if (dlo) dlo[o] = tf32_lo(v);
    } else {
      const int n = i - wn;
      dst[i] = (it.bias && n < it.N) ? it.bias[n] : 0.0f;
    }
  }
}

// ---- device helpers ---------------------------------------------------------------------------------------------------
struct C2Shared {
  uint64_t w_full, w_free, ld_bar;
  int item, last;
  float c_reg, rho, ts_w;    // schedule values of the update hooks (FinArgs fields or *FinArgs.sched)
};

// Slot of the update hooks' warp sums: a worker warp owns 16 rows of a tile, so row m belongs to slot m / 16 = 8 tile + warp.  The last
// CTA adds the slots up in slot order (c2_fin_reduce): the sums do not depend on which CTA ran which tile.
constexpr int C2_FIN_PART = 40;
enum { C2P_STD = 0, C2P_SURR = 32, C2P_ENT = 34, C2P_VAL = 36, C2P_REG = 38, C2P_TS = 39 };   // (SURR, ENT, VAL: one per channel)
__device__ __forceinline__ float* c2_fin_slot(const FinArgs& f, int64_t m) { return f.part + (m >> 4) * C2_FIN_PART; }

__device__ __forceinline__ void c2_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(tc_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void c2_bulk_g2s(void* dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(tc_smem_u32(dst_smem)), "l"(src),
               "r"(bytes), "r"(tc_smem_u32(bar))
               : "memory");
}
// shared -> global bulk copy of this thread's bulk group (the tile images of the activations)
__device__ __forceinline__ void c2_bulk_s2g(void* dst, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(tc_smem_u32(src_smem)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void c2_bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }   // sources may be overwritten
__device__ __forceinline__ void c2_bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }         // writes complete
// elect.sync: true in exactly one lane of the (converged) warp
__device__ __forceinline__ bool c2_elect() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
// a value every lane of the (converged) warp holds, in a form the compiler can see is warp-uniform: control flow around wgmma that depends
// on shared-memory loads is "divergent" to ptxas, which then fences and awaits every wgmma on its own (C7520)
__device__ __forceinline__ int c2_uni(int v) { return __shfl_sync(0xffffffffu, v, 0); }
template <int kRegs> __device__ __forceinline__ void c2_reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <int kRegs> __device__ __forceinline__ void c2_reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }
__device__ __forceinline__ void c2_wbar() { __syncwarp(); asm volatile("bar.sync 1, %0;" ::"n"(C2_NW) : "memory"); }     // the worker warps

// ---- fp32 pairs ---------------------------------------------------------------------------------------------------------
// two fp32 values side by side in a 64-bit register, as a 16-byte load delivers them; the arithmetic is element-wise
__device__ __forceinline__ uint64_t c2_pk(float a, float b) { uint64_t r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ void c2_upk(uint64_t p, float& a, float& b) { asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(p)); }
__device__ __forceinline__ uint64_t c2_add2(uint64_t a, uint64_t b) { float a0, a1, b0, b1; c2_upk(a, a0, a1); c2_upk(b, b0, b1); return c2_pk(a0 + b0, a1 + b1); }
__device__ __forceinline__ uint64_t c2_mul2(uint64_t a, uint64_t b) { float a0, a1, b0, b1; c2_upk(a, a0, a1); c2_upk(b, b0, b1); return c2_pk(a0 * b0, a1 * b1); }
// 2^x, flush-to-zero form: ONE MUFU.EX2.  (__expf = ex2.approx.f32 of x * log2 e WITHOUT .ftz, which ptxas wraps in a range test and two
// scaling multiplies per element for results in the denormal range -- irrelevant for e^x - 1.)
__device__ __forceinline__ float c2_ex2(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
constexpr float C2_LOG2E = 1.4426950408889634f;
template <int kAct, bool kFull>
__device__ __forceinline__ void c2_bias_act(float* v, const float* bias, int nvalid) {
  const uint64_t l2e = c2_pk(C2_LOG2E, C2_LOG2E), m1 = c2_pk(-1.0f, -1.0f);
#pragma unroll
  for (int j4 = 0; j4 < 8; ++j4) {
    const float4 b4 = *reinterpret_cast<const float4*>(bias + 4 * j4);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int jj = 4 * j4 + 2 * h;
      float x0, x1;
      c2_upk(c2_add2(c2_pk(v[jj], v[jj + 1]), h ? c2_pk(b4.z, b4.w) : c2_pk(b4.x, b4.y)), x0, x1);
      if (kAct == ACT_ELU) {        // ELU without a select: max(x,0) + (e^{min(x,0)} - 1); 5 instructions per element (9 as scalar code with __expf)
        float e0, e1;
        c2_upk(c2_mul2(c2_pk(fminf(x0, 0.0f), fminf(x1, 0.0f)), l2e), e0, e1);
        c2_upk(c2_add2(c2_add2(c2_pk(c2_ex2(e0), c2_ex2(e1)), m1), c2_pk(fmaxf(x0, 0.0f), fmaxf(x1, 0.0f))), x0, x1);
      } else if (kAct == ACT_SELU) {  // the same form scaled: s max(x,0) + s alpha (e^{min(x,0)} - 1)
        const float e0 = c2_ex2(fminf(x0, 0.0f) * C2_LOG2E) - 1.0f, e1 = c2_ex2(fminf(x1, 0.0f) * C2_LOG2E) - 1.0f;
        x0 = fmaf(SELU_SCALE * SELU_ALPHA, e0, SELU_SCALE * fmaxf(x0, 0.0f));
        x1 = fmaf(SELU_SCALE * SELU_ALPHA, e1, SELU_SCALE * fmaxf(x1, 0.0f));
      } else if (kAct != ACT_NONE) {
        x0 = act_f<true>(kAct, x0); x1 = act_f<true>(kAct, x1);
      }
      v[jj] = (kFull || jj < nvalid) ? x0 : 0.0f;
      v[jj + 1] = (kFull || jj + 1 < nvalid) ? x1 : 0.0f;
    }
  }
}
// v[jj] *= f'(y[jj]) over one 32-column chunk
template <int kAct>
__device__ __forceinline__ void c2_dact(float* v, const float* y) {
#pragma unroll
  for (int jj = 0; jj < 32; ++jj) v[jj] *= act_df(kAct, y[jj]);
}
__device__ __forceinline__ void c2_bias_act_any(float* v, const float* bias, int act, int nvalid) {
  if (act > ACT_TANH) {             // the other hidden activations: one masked form each (nvalid >= 32 masks nothing), to bound the code size
    if (act == ACT_SELU) c2_bias_act<ACT_SELU, false>(v, bias, nvalid);
    else if (act == ACT_RELU) c2_bias_act<ACT_RELU, false>(v, bias, nvalid);
    else if (act == ACT_LRELU) c2_bias_act<ACT_LRELU, false>(v, bias, nvalid);
    else c2_bias_act<ACT_SIGMOID, false>(v, bias, nvalid);
  } else if (nvalid >= 32) {
    if (act == ACT_ELU) c2_bias_act<ACT_ELU, true>(v, bias, 32);
    else if (act == ACT_TANH) c2_bias_act<ACT_TANH, true>(v, bias, 32);
    else c2_bias_act<ACT_NONE, true>(v, bias, 32);
  } else {
    if (act == ACT_ELU) c2_bias_act<ACT_ELU, false>(v, bias, nvalid);
    else if (act == ACT_TANH) c2_bias_act<ACT_TANH, false>(v, bias, nvalid);
    else c2_bias_act<ACT_NONE, false>(v, bias, nvalid);
  }
}

// ---- epilogue hooks: one thread per row, v[0 .. N) = the head's outputs of that row ---------------------------------------
// Both action-group hooks first pull everything they need into registers with independent (8-byte vector) loads, then compute, then
// store: written element by element the compiler had to order every load after the previous store (possible aliasing), i.e. a dozen
// dependent global round trips per row.  A group has at most 16 actions (host check), rows of the [.., n_act] tensors are 8-byte aligned
// at both group offsets when n_act and n_leg are even (host check; else the scalar path).
constexpr int C2_GRP = 16;
__device__ __forceinline__ void c2_ld_group(const float* p, int cnt, bool vec2, float* out) {
  if (vec2) {
#pragma unroll
    for (int i = 0; i < C2_GRP; i += 2)
      if (i < cnt) { const float2 t = *reinterpret_cast<const float2*>(p + i); out[i] = t.x; out[i + 1] = t.y; }
  } else {
#pragma unroll
    for (int i = 0; i < C2_GRP; ++i)
      if (i < cnt) out[i] = p[i];
  }
}
__device__ __forceinline__ void c2_st_group(float* p, int cnt, bool vec2, const float* v) {
  if (vec2) {
#pragma unroll
    for (int i = 0; i < C2_GRP; i += 2)
      if (i < cnt) *reinterpret_cast<float2*>(p + i) = make_float2(v[i], v[i + 1]);
  } else {
#pragma unroll
    for (int i = 0; i < C2_GRP; ++i)
      if (i < cnt) p[i] = v[i];
  }
}
// FIN_ACT (PPO:119-123, AC:326-345): group c = 0 legs (columns [0, n_leg)), 1 arm ([n_leg, n_act))
__device__ __forceinline__ void c2_fin_act(const FinArgs& f, int c, int64_t m, bool on, const float* v) {
  if (!on) return;
  const int off = c == 0 ? 0 : f.n_leg, cnt = c == 0 ? f.n_leg : f.n_act - f.n_leg;
  const bool vec2 = ((f.n_act | f.n_leg) & 1) == 0;
  if (f.actions == nullptr) { c2_st_group(f.mean_out + m * f.n_act + off, cnt, vec2, v); return; }
  float sg[C2_GRP], ep[C2_GRP], ac[C2_GRP], mu[C2_GRP];
  c2_ld_group(f.std + off, cnt, vec2, sg);
  c2_ld_group(f.eps + m * f.n_act + off, cnt, vec2, ep);
  float lp = 0.0f;
#pragma unroll
  for (int i = 0; i < C2_GRP; ++i) {            // compile-time indices keep the arrays in registers
    if (i < cnt) {
      mu[i] = v[i];
      ac[i] = mu[i] + sg[i] * ep[i];
      lp += ppo_logp_term(ac[i], mu[i], sg[i], logf(sg[i]));
    }
  }
  c2_st_group(f.actions + m * f.n_act + off, cnt, vec2, ac);
  c2_st_group(f.mean_out + m * f.n_act + off, cnt, vec2, mu);
  c2_st_group(f.sigma_out + m * f.n_act + off, cnt, vec2, sg);
  f.log_prob[2 * m + c] = lp;
}
// Arm torque supervision of arm joint i on the arm means this hook holds (ppo_torque_term).  Deliberately NOT inlined and scalar-only (no
// array leaves the caller's registers): the optional branch must not cost the hot epilogue anything.
__device__ __noinline__ float2 c2_fin_torque(const FinArgs& f, int64_t src, int cnt, int i, float mu, float ts_w) {
  return ppo_torque_term(f, src, cnt, i, mu, ts_w);
}
// FIN_PPO (AC:341-345, PPO:199-205): log-prob of the stored action, ratio, mixed advantage, clipped surrogate, entropy and
// the gradients w.r.t. the mean (through the tanh, AC:157,170) and std of this group
__device__ __forceinline__ void c2_fin_ppo(const FinArgs& f, int c, int64_t m, bool on, const float* v, int lane, float rho, float ts_w) {
  const int off = c == 0 ? 0 : f.n_leg, cnt = c == 0 ? f.n_leg : f.n_act - f.n_leg;
  const bool vec2 = ((f.n_act | f.n_leg) & 1) == 0;
  const float inv2m = 1.0f / (2.0f * (float)f.rows);
  float l_surr = 0.0f, l_ent = 0.0f, glp = 0.0f, l_ts = 0.0f;
  float sg[C2_GRP], act[C2_GRP], gm[C2_GRP];
  c2_ld_group(f.std + off, cnt, vec2, sg);
  if (on) {
    const int64_t src = f.idx ? f.idx[m] : m;
    c2_ld_group(f.s_actions + src * f.n_act + off, cnt, vec2, act);
    const float2 adv = *reinterpret_cast<const float2*>(f.adv + 2 * src);
    const float old_lp = f.old_logp[2 * src + c];
    float lp = 0.0f;
#pragma unroll
    for (int i = 0; i < C2_GRP; ++i) {
      if (i < cnt) {
        const float ls = logf(sg[i]);
        lp += ppo_logp_term(act[i], v[i], sg[i], ls);
        l_ent += ppo_entropy_term(ls);
      }
    }
    const float ratio = ppo_ratio(lp, old_lp);
    const float2 surr = ppo_surrogate(ppo_mix(adv, c, rho), ratio, f.clip);
    l_surr = surr.x;
    glp = inv2m * surr.y * ratio;
    const int gld = c == 0 ? f.gleg_ld : f.garm_ld;
#pragma unroll
    for (int i = 0; i < C2_GRP; ++i) {
      gm[i] = 0.0f;
      if (i < cnt) gm[i] = ppo_grad_mean(glp, act[i], v[i], sg[i]);
    }
    if (c == 1 && f.ts_target != nullptr) {
#pragma unroll
      for (int i = 0; i < C2_GRP; ++i)
        if (i < cnt) { const float2 t = c2_fin_torque(f, src, cnt, i, v[i], ts_w); l_ts += t.x; gm[i] += t.y; }
    }
    float* grow = c == 0 ? f.g_leg + m * f.gleg_ld : f.g_arm + m * f.garm_ld;
    if ((gld & 3) == 0) {
#pragma unroll
      for (int i = 0; i < C2_GRP; i += 4)
        if (i < gld) *reinterpret_cast<float4*>(grow + i) = make_float4(gm[i], gm[i + 1], gm[i + 2], gm[i + 3]);
    } else {
#pragma unroll
      for (int i = 0; i < C2_GRP; ++i)
        if (i < gld) grow[i] = gm[i];
    }
  }
  float* slot = c2_fin_slot(f, m);
#pragma unroll
  for (int i = 0; i < C2_GRP; ++i) {           // gradient of std: one warp sum per column
    if (i < cnt) {                             // (warp-uniform)
      float gs = 0.0f;
      if (on) gs = ppo_grad_std(glp, act[i], v[i], sg[i], f.c_ent, inv2m);
      gs = warp_sum(gs);
      if (lane == 0) slot[C2P_STD + off + i] = gs;
    }
  }
  const float ss = warp_sum(l_surr * inv2m), se = warp_sum(l_ent * inv2m);
  if (lane == 0) { slot[C2P_SURR + c] = ss; slot[C2P_ENT + c] = se; }
  if (c == 1 && f.ts_target != nullptr) {          // (warp-uniform)
    const float st = warp_sum(l_ts / ((float)f.rows * (float)cnt));
    if (lane == 0) slot[C2P_TS] = st;
  }
}
// FIN_VALUE (PPO:209-216), channel c
__device__ __forceinline__ void c2_fin_value(const FinArgs& f, int c, int64_t m, bool on, float val, int lane) {
  const float inv2m = 1.0f / (2.0f * (float)f.rows);
  float l_val = 0.0f;
  if (on) {
    const int64_t src = f.idx ? f.idx[m] : m;
    const float2 t = ppo_value_term(val, f.old_values[2 * src + c], f.returns[2 * src + c], f.clip, f.clipped_value);
    l_val = t.x;
    f.g_v[m * f.gv_ld + c] = t.y * f.c_value * inv2m;
    if (c == 0) for (int i = 2; i < f.gv_ld; ++i) f.g_v[m * f.gv_ld + i] = 0.0f;     // pad columns are operand columns of the backward pass
  }
  const float s = warp_sum(l_val * inv2m);
  if (lane == 0) c2_fin_slot(f, m)[C2P_VAL + c] = s;
}
// FIN_REG (PPO:174-177): || z_priv - sg(z_hist) ||_2 per row, mean over rows
__device__ __forceinline__ void c2_fin_reg(const FinArgs& f, int64_t m, bool on, const float* v, int lane, float c_reg) {
  const float invm = 1.0f / (float)f.rows;
  float nrm = 0.0f;
  if (on) {
    const int64_t src = f.idx ? f.idx[m] : m;
    const float* zhr = f.zh + (f.zh_by_src ? src : m) * f.zh_ld;
    nrm = ppo_reg_norm<32>(v, zhr, f.latent);
    const float s = ppo_reg_scale(nrm, c_reg, invm);
#pragma unroll
    for (int i = 0; i < 32; ++i)
      if (i < f.gz_ld) f.g_z[m * f.gz_ld + i] = i < f.latent ? s * (v[i] - zhr[i]) : 0.0f;
  }
  const float s = warp_sum(nrm * invm);
  if (lane == 0) c2_fin_slot(f, m)[C2P_REG] = s;
}
// The last CTA of an update's forward launch: the slots of all (tile, warp) pairs in slot order, into the std gradient and the loss
// means.  Worker thread q + 40 p sums field q over the p-th of six contiguous slot ranges; the six range sums are then added in order.
// Fields no hook of this launch wrote (std columns >= n_act, C2P_TS without torque supervision) may hold what a call with more rows left
// in a shared workspace: they are summed like the others but never used.
__device__ __forceinline__ void c2_fin_reduce(const FinArgs& f, int tiles, float* scratch, int tid) {
  constexpr int NPART = 6;
  const int nslot = tiles * C2_WORKERS, q = tid % C2_FIN_PART, p = tid / C2_FIN_PART;
  if (p < NPART) {
    const int b = (int)((int64_t)nslot * p / NPART), e = (int)((int64_t)nslot * (p + 1) / NPART);
    float s = 0.0f;
#pragma unroll 8
    for (int k = b; k < e; ++k) s += __ldcg(f.part + (int64_t)k * C2_FIN_PART + q);
    scratch[p * C2_FIN_PART + q] = s;
  }
  c2_wbar();
  if (tid < C2_FIN_PART) {
    float t = 0.0f;
    for (int i = 0; i < NPART; ++i) t += scratch[i * C2_FIN_PART + tid];
    scratch[NPART * C2_FIN_PART + tid] = t;
  }
  c2_wbar();
  const float* tot = scratch + NPART * C2_FIN_PART;
  if (tid < f.n_act) f.grad_std[tid] += tot[C2P_STD + tid];
  if (tid == 0) {
    f.losses[0] += tot[C2P_SURR] + tot[C2P_SURR + 1];
    f.losses[1] += tot[C2P_VAL] + tot[C2P_VAL + 1];
    f.losses[2] += tot[C2P_REG];
    f.losses[3] += tot[C2P_ENT] + tot[C2P_ENT + 1];
    if (f.ts_target != nullptr) f.losses[4] += tot[C2P_TS];
  }
}

// ---- the kernel -------------------------------------------------------------------------------------------------------
// the wgmma chain of one op on one slot for this warpgroup's 64 rows.  a0 / b0 / b0_lo: shared-memory addresses of the A window (row 0 of
// the warpgroup), the weight image and (3xTF32) the image of the weights' low parts; arow: this thread's first A fragment element.
template <int N>
__device__ __forceinline__ void c2_mma_op(float (&acc)[64], uint32_t a0, uint32_t b0, uint32_t b0_lo, uint32_t wsbo, int nk, bool x3, const float* arow) {
  uint64_t ad = tc_desc(a0, 128, 4096), bd = tc_desc(b0, 128, wsbo);
  if (!x3) {
    wg_fence();
    // one K step (8 columns = two 16-byte pieces) advances both start addresses by 256 bytes: +16 in the descriptors' address field
    for (int k = 0; k < nk; ++k, ad += 16, bd += 16) wg_mma_ss<N>(acc, ad, bd, k > 0);
  } else {
    // D = A_hi W_hi + A_lo W_hi + A_hi W_lo: the tensor core truncates the fp32 tile and the raw image to their high parts itself; A_lo is
    // formed in registers (the A fragment of this thread) and fed as a register operand.  The fragments of a whole op (16 K steps x 4
    // registers) stay live until the op's single wait, in two sets of C2_KSET K steps with a commit group each: the second set is formed
    // while the wgmmas of the first execute, and nothing is awaited inside the op.  (Two smaller sets recycled behind wait<1> made ptxas
    // serialise the wgmmas again: C7511, not enough registers for the pipeline.)
    // Per accumulator the products keep the order hi*hi, lo*hi, hi*lo per K step, K ascending.
    const uint64_t bl = tc_desc(b0_lo, 128, wsbo);
    uint32_t lo[2][C2_KSET][4];
#pragma unroll
    for (int g = 0; g < 2; ++g) {
#pragma unroll
      for (int j = 0; j < C2_KSET; ++j) {
        if (C2_KSET * g + j < nk) {
          const float* ap = arow + (size_t)(C2_KSET * g + j) * 64;          // 8 columns = two pieces of 32 floats
          lo[g & 1][j][0] = __float_as_uint(tf32_lo(ap[0])); lo[g & 1][j][1] = __float_as_uint(tf32_lo(ap[1024]));          // rows +0 / +8 (next 8-row group)
          lo[g & 1][j][2] = __float_as_uint(tf32_lo(ap[32])); lo[g & 1][j][3] = __float_as_uint(tf32_lo(ap[1024 + 32]));    // columns +4
        }
      }
      wg_fence();
#pragma unroll
      for (int j = 0; j < C2_KSET; ++j) {
        const int k = C2_KSET * g + j;
        if (k < nk) {
          wg_mma_ss<N>(acc, ad + 16 * k, bd + 16 * k, k > 0);
          wg_mma_rs<N>(acc, lo[g & 1][j][0], lo[g & 1][j][1], lo[g & 1][j][2], lo[g & 1][j][3], bd + 16 * k, 1);
          wg_mma_ss<N>(acc, ad + 16 * k, bl + 16 * k, 1);
        }
      }
      wg_commit();
    }
  }
  wg_commit();
  wg_wait<0>();
}

// static + dynamic shared memory of the kernel against the 227 KB a block may opt into on sm_90: a field added to C2Op must fail here, not at launch
static_assert(sizeof(C2Prog) + sizeof(C2Shared) + 128 + C2_SMEM_FLOATS * sizeof(float) <= 232448, "chain2_kernel exceeds the shared memory of an SM");

__global__ void __launch_bounds__(C2_THREADS, 1) chain2_kernel(const __grid_constant__ C2Launch L, const int tiles) {
  extern __shared__ __align__(128) float c2_smem[];
  __shared__ C2Shared sh;
  __shared__ __align__(16) C2Prog sprog;
  int cur_prog = -1;
  auto tile = [&](int s) { return c2_smem + s * C2_TILE; };      // operand tile of slot s
  float* wbuf = c2_smem + 2 * C2_TILE;
  float* bias_s = c2_smem + 3 * C2_TILE;                 // two slots of 128 (parity of the CTA-wide op counter)
  float* stage_s = bias_s + 2 * 128;                     // per worker warp: [16 rows][64 columns] transposition buffer of the epilogue
  const int tid = threadIdx.x, lane = tid & 31, warp = c2_uni(tid >> 5);
  if (tid == 0) {
    tc_mbar_init(&sh.w_full, 1);
    tc_mbar_init(&sh.w_free, 1);
    tc_mbar_init(&sh.ld_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    const float* sc = L.fin.sched;
    sh.c_reg = sc ? sc[0] : L.fin.c_reg;
    sh.rho = sc ? sc[1] : L.fin.rho;
    sh.ts_w = sc ? sc[2] : L.fin.ts_w;
  }
  __syncthreads();
  const int n_pair_items = L.np2 * L.nprog;
  const int items = n_pair_items + L.ns1 * L.nprog;
  const bool x3 = L.x3 != 0;

  // running counters, identical in every thread: ops of all items so far (bias slot parity), bulk tile loads (phase of ld_bar)
  uint32_t nop = 0, nld = 0;
  uint32_t nw = 0, nf = 0;          // weight images consumed (phase of w_full: workers) / released (phase of w_free: copy warp)

  // ---- next work item (every thread of the CTA, workers and copy warpgroup alike): false when the queue is empty ----
  int t0, nslots;                                        // first tile, tiles of this item
  auto next_item = [&]() {
    __syncthreads();                                     // everybody is done with the previous item (sh.item may be overwritten)
    if (tid == 0) sh.item = atomicAdd(L.queue, 1);
    __syncthreads();
    const int item = c2_uni(sh.item);
    if (item >= items) return false;
    const bool two = item < n_pair_items;
    const int k = two ? item : item - n_pair_items, per = two ? L.np2 : L.ns1;
    const int pi = k / per;                              // program (0 = the longer one, first)
    t0 = two ? 2 * (k - pi * per) : 2 * L.np2 + (k - pi * per);
    nslots = min(two ? 2 : 1, tiles - t0);
    asm volatile("" : "+r"(nslots));                     // opaque: one body for both item sizes (the compiler cloned the whole item loop otherwise)
    nslots = c2_uni(nslots);
    // the item's program goes to shared memory: read through the kernel parameter, every field access with a run-time op index is an
    // indexed constant-bank load -- a long-scoreboard stall in front of most addresses and predicates of the epilogue
    if (pi != cur_prog) {
      const int4* src = reinterpret_cast<const int4*>(&L.p[pi]);
      int4* dst = reinterpret_cast<int4*>(&sprog);
      for (int k4 = tid; k4 < (int)(sizeof(C2Prog) / 16); k4 += C2_THREADS) dst[k4] = src[k4];
      cur_prog = pi;
      __syncthreads();
    }
    return true;
  };
  const C2Prog& pr = sprog;

  if (warp >= C2_WORKERS) {
    // ===================== weight copies (third warpgroup; its warps 9-11 only take part in the CTA-wide barriers) =====================
    c2_reg_dec<C2_REGS_COPY>();
    while (next_item()) {
      const int nops = c2_uni(pr.n_ops);
      if (warp == C2_WORKERS) {
        // One image is resident at a time: the image (and bias) of op i+1 is fetched as soon as the workers have retired the wgmmas of op i,
        // i.e. behind the epilogue of op i.  3xTF32 items hold one tile (launch_chain2n), so the image of the weights' low parts travels with
        // the raw image into the unused tile of slot 1.
        auto fetch = [&](const C2Op& o, uint32_t slot) {
          const uint32_t wbytes = (uint32_t)(o.npad * o.kpad) * 4u, bbytes = (uint32_t)o.npad * 4u;
          if (c2_elect()) {
            c2_expect_tx(&sh.w_full, wbytes + bbytes + (x3 ? wbytes : 0u));
            c2_bulk_g2s(wbuf, o.wp, wbytes, &sh.w_full);
            c2_bulk_g2s(bias_s + slot * 128, o.wp + (wbytes >> 2), bbytes, &sh.w_full);
            if (x3) c2_bulk_g2s(tile(1), o.wp_lo, wbytes, &sh.w_full);
          }
          __syncwarp();
        };
        fetch(pr.op[0], nop & 1);
        for (int i = 0; i + 1 < nops; ++i) {
          tc_mbar_wait(&sh.w_free, nf & 1); ++nf;          // every wgmma reading image i has retired: the buffer may be refilled
          fetch(pr.op[i + 1], (nop + i + 1) & 1);
        }
        tc_mbar_wait(&sh.w_free, nf & 1); ++nf;
      }
      nop += nops;
    }
  } else {
    // ===================== loads, wgmma and epilogues (two warpgroups) =====================
    c2_reg_inc<C2_REGS_WORKER>();
    while (next_item()) {
      const int nops = c2_uni(pr.n_ops);
      // slot s works on tile tb + s * td: upwards from t0, or (L.rev: the backward launch) downwards from the last tile -- the forward launch
      // that produced the activation images this one reads walked upwards, so its most recent output, still in L2, belongs to the last tiles
      const int tb = L.rev ? tiles - 1 - t0 : t0, td = L.rev ? -1 : 1;
      // wgmma: warp w owns tile rows [16 w, 16 w + 16).  Epilogue: the same rows, thread = (row 16 w + lane % 16, 32-column chunks lane / 16
      // and lane / 16 + 2); the accumulator fragments reach that shape through the warp's transposition buffer, 64 columns at a time.
      const int hh = lane >> 4;
      const int r = warp * 16 + (lane & 15);               // tile row of this thread in the epilogue
      float* const stg = stage_s + warp * 1024;
      constexpr int LRW = 128 / C2_WORKERS, LPS = 32 / LRW;     // load role: rows per warp, piece stride
      const int lrow = warp * LRW + (lane % LRW), lpc = lane / LRW;   // fixed row, 16-byte pieces lpc, lpc + LPS, ...

      // cp.async of one load into the tile of slot s (no waiting); rows beyond the matrix are zero-filled
      auto issue_load = [&](const C2Load& ld, int s, int64_t m0, int rows) {
        float* tl = tile(s);
        const int c40 = ld.col0 >> 2, cpr = ld.ncols >> 2;
        const int z0 = (ld.col0 + ld.ncols) >> 2, z1 = ld.zero_to >> 2;
        float* rowbase = tl + ((size_t)(lrow >> 3) * 32) * 32 + (lrow & 7) * 4;
        for (int cz = z0 + lpc; cz < z1; cz += LPS) *reinterpret_cast<float4*>(rowbase + (size_t)cz * 32) = make_float4(0.f, 0.f, 0.f, 0.f);
        const bool on = lrow < rows;
        const float* src = on ? ld.src.row(m0 + lrow) : ld.src.p;
        const uint32_t d0 = tc_smem_u32(rowbase);
        for (int cc = lpc; cc < cpr; cc += LPS)
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d0 + (uint32_t)(c40 + cc) * 128u), "l"(src + 4 * cc), "r"(on ? 16 : 0)
                       : "memory");
      };
      // loads of the slots that precede op `before`: issue and wait
      auto do_loads = [&](int before, bool sync_first) {
        bool any = false;
        for (int l = 0; l < pr.n_loads; ++l) any |= pr.ld[l].before_op == before;
        if (!any) return false;
        if (sync_first) c2_wbar();                       // every worker has finished writing / copying the tiles the loads overwrite
        int nimg = 0;
        for (int s = 0; s < nslots; ++s) {
          const int64_t m0 = (int64_t)(tb + s * td) * TC_M;
          const int rows = (int)min((int64_t)TC_M, (int64_t)pr.M - m0);
          for (int l = 0; l < pr.n_loads; ++l) {
            if (pr.ld[l].before_op != before) continue;
            if (pr.ld[l].img) ++nimg; else issue_load(pr.ld[l], s, m0, rows);
          }
        }
        if (nimg) {                                      // tile images come back as one bulk copy each (warp-uniform count)
          if (tid == 0) {
            c2_expect_tx(&sh.ld_bar, (uint32_t)nimg * C2_TILE * 4u);
            for (int s = 0; s < nslots; ++s)
              for (int l = 0; l < pr.n_loads; ++l)
                if (pr.ld[l].before_op == before && pr.ld[l].img) c2_bulk_g2s(tile(s), pr.ld[l].src.p + (size_t)(tb + s * td) * C2_TILE, C2_TILE * 4, &sh.ld_bar);
          }
          tc_mbar_wait(&sh.ld_bar, nld & 1);
          ++nld;
        }
        asm volatile("cp.async.wait_all;" ::: "memory");
        return true;
      };

      uint32_t n = nop;
      // ---- item start: the rows a LATER gather of this item will read are pulled into L2 now (its latency is exposed otherwise: the tile
      // columns it fills are still in use), then both slots' initial loads ----
      for (int l = 0; l < pr.n_loads; ++l) {
        const C2Load& ld = pr.ld[l];
        if (ld.before_op == 0 || ld.img) continue;
        for (int s = 0; s < nslots; ++s) {
          const int64_t m0 = (int64_t)(tb + s * td) * TC_M;
          if (m0 + lrow >= pr.M) continue;
          const float* src = ld.src.row(m0 + lrow);
          for (int b = lpc * 32; b < ld.ncols; b += LPS * 32) asm volatile("prefetch.global.L2 [%0];" ::"l"(src + b));
        }
      }
      do_loads(0, false);
      tc_fence_async_smem();                             // generic-proxy tile writes -> async-proxy wgmma / bulk-copy reads (after the barrier below)

      for (int i = 0; i < nops; ++i, ++n) {
        const C2Op& o = pr.op[i];
        bool pending = false;                              // loads that precede op i+1 cover both slots and follow the last slot's epilogue
        bool reload_next = false;                          // an image written earlier is re-read before the next op: those writes must have landed
        for (int l = 0; l < pr.n_loads; ++l) {
          pending |= pr.ld[l].before_op == i + 1;
          reload_next |= pr.ld[l].before_op == i + 1 && pr.ld[l].img != 0;
        }
        // the previous op left a finished tile behind: if its output is a tile image it goes out now, as one 64 KB bulk copy issued right
        // before the wgmmas that read the same tile; it must have read the tile before the epilogue of THIS op may overwrite it
        const bool st_prev = i > 0 && pr.op[i - 1].y_img != 0;
        const int nwid = c2_uni(wg_width(o.npad)), nk = c2_uni(o.kpad >> 3);     // (the control flow around the wgmmas)
        for (int s = 0; s < nslots; ++s) {
          const int64_t m0 = (int64_t)(tb + s * td) * TC_M;
          const int rows = (int)min((int64_t)TC_M, (int64_t)pr.M - m0);
          const bool on = r < rows;
          // backward: the activation chunks whose derivative multiplies, fetched while the wgmmas run
          float x[C2_CPW][32];
          const bool use_x = o.mode == 1 && o.xact != nullptr;
          if (use_x) {
#pragma unroll
            for (int u = 0; u < C2_CPW; ++u) {
              const int c0 = 32 * (hh + u * C2_H);
              // row-major: 32 consecutive floats of the row; tile image: eight 16-byte pieces 128 bytes apart (eight rows share each line)
              const float* xr = o.x_img ? o.xact + (size_t)(tb + s * td) * C2_TILE + ((size_t)((r >> 3) * 32 + (c0 >> 2)) * 8 + (r & 7)) * 4
                                        : o.xact + (m0 + r) * o.ldx + c0;
              const int xst = o.x_img ? 32 : 4;
#pragma unroll
              for (int j4 = 0; j4 < 8; ++j4) {
                float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
                if (on && c0 + 4 * j4 < o.N) t = *reinterpret_cast<const float4*>(xr + xst * j4);
                x[u][4 * j4] = t.x; x[u][4 * j4 + 1] = t.y; x[u][4 * j4 + 2] = t.z; x[u][4 * j4 + 3] = t.w;
              }
            }
          }
          c2_wbar();                                       // the operand tile is complete: loads landed / previous epilogue done (and fenced)
          if (tid == 0 && st_prev) c2_bulk_s2g(pr.op[i - 1].y + (size_t)(tb + s * td) * C2_TILE, tile(s), C2_TILE * 4);
          if (s == 0) { tc_mbar_wait(&sh.w_full, nw & 1); ++nw; }
          float acc[64];
          {
            const uint32_t a0 = tc_smem_u32(tile(s)) + (uint32_t)(warp >> 2) * 8u * 4096u + (uint32_t)(o.a_col0 >> 2) * 128u;
            const uint32_t b0 = tc_smem_u32(wbuf), b0_lo = tc_smem_u32(tile(1)), wsbo = (uint32_t)(o.kpad >> 2) * 128u;
            // A fragment element (row 16 warp + lane / 4, column a_col0 + lane % 4) of this thread
            const float* arow = tile(s) + ((size_t)(2 * warp) * 32 + (o.a_col0 >> 2)) * 32 + (lane >> 2) * 4 + (lane & 3);
            if (nwid == 32) c2_mma_op<32>(acc, a0, b0, b0_lo, wsbo, nk, x3, arow);
            else if (nwid == 64) c2_mma_op<64>(acc, a0, b0, b0_lo, wsbo, nk, x3, arow);
            else c2_mma_op<128>(acc, a0, b0, b0_lo, wsbo, nk, x3, arow);
          }
          if (tid == 0) {
            if (reload_next) c2_bulk_wait_all(); else if (st_prev) c2_bulk_wait_read();
          }
          c2_wbar();                                       // every warp's wgmmas and the bulk copy have read the tile: it may be updated in place
          if (tid == 0 && s + 1 == nslots) t2_arrive(&sh.w_free);
#pragma unroll
          for (int u = 0; u < C2_CPW; ++u) {
            if (64 * u >= nwid) continue;                  // (warp-uniform)
            // fragments of columns [64 u, 64 u + 64) -> transposition buffer (16-byte slot sl of row rr at slot sl ^ rr) -> this thread's chunk
            __syncwarp();
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int sl = 2 * j + ((lane & 3) >> 1), off = (2 * lane) & 3, r0 = lane >> 2;
              *reinterpret_cast<float2*>(stg + r0 * 64 + ((sl ^ r0) << 2) + off) = make_float2(acc[32 * u + 4 * j], acc[32 * u + 4 * j + 1]);
              *reinterpret_cast<float2*>(stg + (r0 + 8) * 64 + ((sl ^ (r0 + 8)) << 2) + off) = make_float2(acc[32 * u + 4 * j + 2], acc[32 * u + 4 * j + 3]);
            }
            __syncwarp();
            const int c0 = 32 * (hh + u * C2_H);            // this thread's u-th chunk
            const bool active = c0 < o.npad;
            float v[32];
#pragma unroll
            for (int j4 = 0; j4 < 8; ++j4) {
              const float4 t = *reinterpret_cast<const float4*>(stg + (lane & 15) * 64 + (((8 * hh + j4) ^ (lane & 15)) << 2));
              v[4 * j4] = t.x; v[4 * j4 + 1] = t.y; v[4 * j4 + 2] = t.z; v[4 * j4 + 3] = t.w;
            }
            if (active) {
              if (o.mode == 0) {
                c2_bias_act_any(v, bias_s + (n & 1) * 128 + c0, o.act, o.N - c0);
              } else {
                if (o.add != nullptr && on) {
                  const float* ar = o.add + (m0 + r) * o.ldadd + c0;
#pragma unroll
                  for (int j4 = 0; j4 < 8; ++j4) {
                    if (c0 + 4 * j4 < o.N) {
                      const float4 t = *reinterpret_cast<const float4*>(ar + 4 * j4);
                      v[4 * j4] += t.x; v[4 * j4 + 1] += t.y; v[4 * j4 + 2] += t.z; v[4 * j4 + 3] += t.w;
                    }
                  }
                }
                if (use_x) {                                   // activation derivatives from the layer's OUTPUTS (act_df)
                  if (o.act == ACT_TANH) {
                    c2_dact<ACT_TANH>(v, x[u]);
                  } else if (o.act == ACT_ELU) {               // ELU'(y) = y > 0 ? 1 : y + 1 = min(y + 1, 1)
#pragma unroll
                    for (int jj = 0; jj < 32; ++jj) v[jj] *= fminf(x[u][jj] + 1.0f, 1.0f);
                  } else if (o.act == ACT_SELU) {
                    c2_dact<ACT_SELU>(v, x[u]);
                  } else if (o.act == ACT_RELU) {
                    c2_dact<ACT_RELU>(v, x[u]);
                  } else if (o.act == ACT_LRELU) {
                    c2_dact<ACT_LRELU>(v, x[u]);
                  } else {
                    c2_dact<ACT_SIGMOID>(v, x[u]);
                  }
                }
                if (o.N - c0 < 32) {                           // ragged last chunk: the pad columns are operand columns of the next op
#pragma unroll
                  for (int jj = 0; jj < 32; ++jj) v[jj] = c0 + jj < o.N ? v[jj] : 0.0f;
                }
              }
              if (o.out_col0 >= 0) {
                float* otile = tile(s) + ((size_t)((r >> 3) * 32 + ((o.out_col0 + c0) >> 2)) * 8 + (r & 7)) * 4;
#pragma unroll
                for (int j4 = 0; j4 < 8; ++j4)
                  *reinterpret_cast<float4*>(otile + (size_t)j4 * 32) = make_float4(v[4 * j4], v[4 * j4 + 1], v[4 * j4 + 2], v[4 * j4 + 3]);
              }
            }
            if (o.fin != FIN_NONE && u == 0) {               // the head's outputs sit in chunk 0: the lanes holding chunk 1 only take part in the warp sums
              const bool fon = on && hh == 0;
              if (o.fin == FIN_ACT) c2_fin_act(L.fin, o.fin_c, m0 + r, fon, v);
              else if (o.fin == FIN_PPO) c2_fin_ppo(L.fin, o.fin_c, m0 + r, fon, v, lane, sh.rho, sh.ts_w);
              else if (o.fin == FIN_VALUE) c2_fin_value(L.fin, o.fin_c, m0 + r, fon, v[0], lane);
              else c2_fin_reg(L.fin, m0 + r, fon, v, lane, sh.c_reg);
            }
            if (active && o.y != nullptr && !o.y_img && on) {       // straight from the registers: 128 contiguous bytes per thread
              float* yr = o.y + (m0 + r) * o.ldy + c0;
              if ((o.ldy & 3) == 0 && (o.N & 3) == 0) {
#pragma unroll
                for (int j4 = 0; j4 < 8; ++j4)
                  if (c0 + 4 * j4 < o.N) *reinterpret_cast<float4*>(yr + 4 * j4) = make_float4(v[4 * j4], v[4 * j4 + 1], v[4 * j4 + 2], v[4 * j4 + 3]);
              } else {
#pragma unroll
                for (int jj = 0; jj < 32; ++jj)
                  if (c0 + jj < o.N) yr[jj] = v[jj];
              }
            }
          }
          tc_fence_async_smem();
          if (pending && i + 1 < nops && s + 1 == nslots) {
            do_loads(i + 1, true);
            tc_fence_async_smem();
          }
        }
      }
      // the last op's tiles: an image output leaves now, and the tiles may be reloaded (next item) only after the copies have read them
      if (pr.op[nops - 1].y_img) {
        c2_wbar();
        if (tid == 0) {
          for (int s = 0; s < nslots; ++s) c2_bulk_s2g(pr.op[nops - 1].y + (size_t)(tb + s * td) * C2_TILE, tile(s), C2_TILE * 4);
          c2_bulk_wait_read();
        }
      }
      nop += nops;
    }
  }
  if (tid == 0) c2_bulk_wait_all();      // the image stores of this CTA have landed
  __threadfence();                       // (and the partial sums of the update hooks)
  __syncthreads();
  if (tid == 0) {                        // the last CTA re-arms the queue for the next launch
    __threadfence();
    sh.last = atomicAdd(L.queue + 1, 1) == (int)gridDim.x - 1;
    if (sh.last) { L.queue[0] = 0; L.queue[1] = 0; __threadfence(); }
  }
  __syncthreads();
  if (sh.last && L.fin.losses != nullptr && warp < C2_WORKERS) c2_fin_reduce(L.fin, tiles, c2_smem, tid);
}


// ---- host side ------------------------------------------------------------------------------------------------------
inline bool c2_aligned(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
constexpr int64_t C2_PACK_FLOATS = (int64_t)2 * C2_MAX_PACK * (C2_TILE + 256);      // raw + low images of every item

inline int launch_pack2(const C2PackList& pl, cudaStream_t st) {
  if (pl.n <= 0) return DWBC_OK;
  pack_weights2_kernel<<<dim3(8, pl.n), 256, 0, st>>>(pl);
  ++dwbc_launch_counter;
  return cudaGetLastError() == cudaSuccess ? DWBC_OK : DWBC_ERR_LAUNCH;
}

// Keeps the pack list and the program in step.  `off` is the running float offset into the packed-weight buffer.
struct C2Builder {
  C2Prog pr{};
  C2PackList* pl;
  int64_t* off;
  bool x3, ok = true;
  C2Builder(C2PackList* pl_, int64_t* off_, int M, bool x3_) : pl(pl_), off(off_), x3(x3_) { pr.M = M; }
  void load(RowMat src, int ncols, int col0, int zero_to, int before_op) {
    if (src.rpg == 0) {                 // tile image: the whole tile, one bulk copy
      if (pr.n_loads >= C2_MAX_LOADS || ncols != 128 || col0 != 0 || zero_to != 128 || !c2_aligned(src.p)) { ok = false; return; }
      pr.ld[pr.n_loads++] = C2Load{src, ncols, col0, zero_to, before_op, 1};
      return;
    }
    if (pr.n_loads >= C2_MAX_LOADS || (ncols & 3) || (col0 & 3) || (zero_to & 3) || zero_to < col0 + ncols || zero_to > 128 || !c2_aligned(src.p) ||
        (src.stride_g & 3) || (src.ld & 3) || src.rpg != 1) { ok = false; return; }
    pr.ld[pr.n_loads++] = C2Load{src, ncols, col0, zero_to, before_op, 0};
  }
  C2Op* push(const float* W, int64_t ldw, const float* bias, int N, int kpad, int transpose, int nseg, C2PackSeg s0, C2PackSeg s1) {
    const int npad = (N + 15) & ~15;
    if (pr.n_ops >= C2_MAX_OPS || pl->n >= C2_MAX_PACK || N <= 0 || N > 128 || kpad <= 0 || kpad > 128 || (kpad & 7)) { ok = false; return nullptr; }
    C2PackItem& it = pl->it[pl->n++];
    it = C2PackItem{W, ldw, bias, N, npad, kpad, transpose, nseg, {s0, s1}, *off, -1};
    C2Op& o = pr.op[pr.n_ops++];
    o = C2Op{};
    o.wp = pl->out ? pl->out + *off : nullptr;
    *off = (*off + (int64_t)npad * kpad + npad + 63) & ~(int64_t)63;       // 256-byte aligned images (bulk copies need 16)
    if (x3) {
      it.dst_lo = *off;
      o.wp_lo = pl->out ? pl->out + *off : nullptr;
      *off = (*off + (int64_t)npad * kpad + 63) & ~(int64_t)63;
    }
    o.kpad = kpad; o.N = N; o.npad = npad;
    return &o;
  }
  // y = act(A[:, a_col0 : a_col0 + kpad] W'^T + b): W [N x ldw]; tile column a_col0 + seg.kdst + j multiplies W[:, seg.ksrc + j]
  // y_img: y is a tile-image buffer (only for full-width outputs written at tile column 0)
  void fwd(const float* W, int64_t ldw, const float* bias, int N, int act, int a_col0, int kpad, int nseg, C2PackSeg s0, C2PackSeg s1, int out_col0,
           float* y, int64_t ldy, int fin = FIN_NONE, int fin_c = 0, bool y_img = false) {
    if (y_img && (N != 128 || out_col0 != 0 || !y || !c2_aligned(y))) { ok = false; return; }
    if ((a_col0 & 3) || a_col0 + kpad > 128 || (out_col0 >= 0 && ((out_col0 & 31) || out_col0 + ((N + 31) & ~31) > 128)) || (fin != FIN_NONE && N > 32)) { ok = false; return; }
    C2Op* o = push(W, ldw, bias, N, kpad, 0, nseg, s0, s1);
    if (!o) return;
    o->y = y; o->ldy = ldy; o->a_col0 = a_col0; o->act = act; o->out_col0 = out_col0; o->mode = 0; o->fin = fin; o->fin_c = fin_c;
    o->y_img = y_img ? 1 : 0;
  }
  // dX[:, :Nin] = (dZ[:, a_col0 : a_col0 + kpad] W' (+ add)) (*) act'(xact): W [Kout x ldw] (row = output feature);
  // tile column a_col0 + seg.kdst + j multiplies row seg.ksrc + j of W
  void bwd(const float* W, int64_t ldw, int Nin, int a_col0, int kpad, C2PackSeg seg, int act, const float* xact, int64_t ldx, const float* add,
           int64_t ldadd, int out_col0, float* y, int64_t ldy, bool x_img = false, bool y_img = false) {
    if ((y_img && (Nin != 128 || out_col0 != 0 || !y)) || (x_img && Nin != 128)) { ok = false; return; }
    if ((a_col0 & 3) || a_col0 + kpad > 128 || (Nin & 3) || (xact && ((ldx & 3) || !c2_aligned(xact))) || (add && ((ldadd & 3) || !c2_aligned(add))) ||
        (out_col0 >= 0 && (out_col0 & 31))) { ok = false; return; }
    C2Op* o = push(W, ldw, nullptr, Nin, kpad, 1, 1, seg, C2PackSeg{0, 0, 0});
    if (!o) return;
    o->y = y; o->ldy = ldy; o->a_col0 = a_col0; o->act = act; o->out_col0 = out_col0; o->mode = 1;
    o->xact = act == ACT_NONE ? nullptr : xact; o->ldx = ldx; o->add = add; o->ldadd = ldadd;
    o->x_img = x_img ? 1 : 0; o->y_img = y_img ? 1 : 0;
  }
  void finish() {
    for (int i = 0; i < pr.n_ops; ++i) {
      C2Op& o = pr.op[i];
      if (o.y && (o.ldy & 3) == 0 && (o.N & 3) == 0 && !c2_aligned(o.y)) ok = false;   // vector stores need 16-byte aligned rows
      // an image written by op i is sent off while op i+1 runs and must have landed before it is re-read: not by a load in front of op i+1
      if (o.y_img)
        for (int l = 0; l < pr.n_loads; ++l)
          if (pr.ld[l].img && pr.ld[l].src.p == o.y && pr.ld[l].before_op <= i + 1) ok = false;
    }
  }
};

// pr1 may be null.  The longer program goes first in the queue.
// ---- how many tiles of a large launch run as one-tile items ---------------------------------------------------------------------------
// A launch of T tiles x P programs on S persistent CTAs: with two-tile items only, the last wave is badly quantised (some CTAs get a second
// long item while the others wait for a short one).  One-tile items are half the work at a worse rate (the weight image serves one tile
// only: factor c2_single_penalty, an estimate), but they fill the tail.  The number of them is chosen by simulating the
// queue (greedy: a CTA that becomes free takes the next item) with a per-op cost model of the epilogue-bound kernel; the choice depends
// only on (tiles, programs), so it is cached.
constexpr double c2_single_penalty = 1.35;               // time of a one-tile item / half the time of a two-tile item
inline double c2_prog_cost(const C2Prog& pr) {
  double c = 0.0;
  for (int i = 0; i < pr.n_ops; ++i) c += 0.3 + (double)pr.op[i].npad / 128.0;       // fixed hand-over + epilogue work ~ output chunks
  return c + 0.3 * pr.n_loads;
}
inline double c2_makespan(int tiles, int nprog, const double* cost, int sms, int ns1) {
  std::vector<double> heap(sms, 0.0);                    // min-heap of the CTAs' free times
  auto take = [&](double c) {
    std::pop_heap(heap.begin(), heap.end(), std::greater<double>());
    heap.back() += c;
    std::push_heap(heap.begin(), heap.end(), std::greater<double>());
  };
  const int np2 = (tiles - ns1 + 1) / 2;
  for (int p = 0; p < nprog; ++p)
    for (int j = 0; j < np2; ++j) take(2 * j + 1 < tiles - ns1 ? cost[p] : 0.5 * c2_single_penalty * cost[p]);   // (an odd last pair holds one tile)
  for (int p = 0; p < nprog; ++p)
    for (int j = 0; j < ns1; ++j) take(0.5 * c2_single_penalty * cost[p]);
  return *std::max_element(heap.begin(), heap.end());
}
inline int c2_pick_singles(int tiles, int nprog, const double* cost, int sms) {
  struct Key { int tiles, nprog, sms; double c0, c1; int ns1; };            // (c1: the sum of the other programs' costs)
  static thread_local Key cache[8];
  static thread_local int ncache = 0;
  double rest = 0.0;
  for (int k = 1; k < nprog; ++k) rest += cost[k] * (1.0 + 1e-3 * k);
  for (int i = 0; i < ncache; ++i) {
    const Key& k = cache[i];
    if (k.tiles == tiles && k.nprog == nprog && k.sms == sms && k.c0 == cost[0] && k.c1 == rest) return k.ns1;
  }
  int best = 0;
  double best_t = c2_makespan(tiles, nprog, cost, sms, 0);
  for (int s1 = 2 - (tiles & 1); s1 <= tiles && s1 <= 2 * sms; s1 += 2) {      // (tiles - s1) even: whole pairs in front
    const double t = c2_makespan(tiles, nprog, cost, sms, s1);
    if (t < best_t * (1.0 - 1e-9)) { best_t = t; best = s1; }
  }
  Key& k = cache[ncache < 8 ? ncache++ : 7];
  k = Key{tiles, nprog, sms, cost[0], rest, best};
  return best;
}

inline int c2_sm_count() {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  }
  return sms;
}

inline int launch_chain2n(const C2Prog* const* prs, int nprog, const FinArgs& fin, bool x3, int* queue, cudaStream_t st, bool rev = false);
inline int launch_chain2(const C2Prog* pr0, const C2Prog* pr1, const FinArgs& fin, bool x3, int* queue, cudaStream_t st, bool rev = false) {
  const C2Prog* prs[2] = {pr0, pr1};
  return launch_chain2n(prs, pr1 ? 2 : 1, fin, x3, queue, st, rev);
}
// up to C2_MAX_PROGS programs over the same rows in one launch; queued longest program first
inline int launch_chain2n(const C2Prog* const* prs, int nprog, const FinArgs& fin, bool x3, int* queue, cudaStream_t st, bool rev) {
  if (nprog < 1 || nprog > C2_MAX_PROGS) return DWBC_ERR_ARG;
  C2Launch L{};
  L.rev = rev ? 1 : 0;
  L.nprog = nprog;
  L.x3 = x3 ? 1 : 0;
  L.queue = queue;
  L.fin = fin;
  int order[C2_MAX_PROGS];
  for (int k = 0; k < nprog; ++k) order[k] = k;
  std::stable_sort(order, order + nprog, [&](int a, int b) { return prs[a]->n_ops > prs[b]->n_ops; });
  for (int k = 0; k < nprog; ++k) L.p[k] = *prs[order[k]];
  for (int k = 0; k < L.nprog; ++k) {
    const C2Prog& pr = L.p[k];
    if (pr.M <= 0 || pr.M != L.p[0].M || pr.n_ops <= 0 || pr.n_ops > C2_MAX_OPS || pr.n_loads < 0 || pr.n_loads > C2_MAX_LOADS) return DWBC_ERR_ARG;
  }
  if (!queue) return DWBC_ERR_ARG;
  const int sms = c2_sm_count();
  const int tiles = (L.p[0].M + TC_M - 1) / TC_M;
  if (tiles * L.nprog <= sms || x3) {                      // small batches (rollout): one tile per item, spread over more SMs; 3xTF32: the
                                                           // second slot's tile holds the image of the weights' low parts
    L.np2 = 0;
    L.ns1 = tiles;
  } else {
    double cost[C2_MAX_PROGS] = {};
    for (int k = 0; k < L.nprog; ++k) cost[k] = c2_prog_cost(L.p[k]);
    L.ns1 = c2_pick_singles(tiles, L.nprog, cost, sms);
    L.np2 = (tiles - L.ns1 + 1) / 2;
  }
  const int items = (L.np2 + L.ns1) * L.nprog;
  const int grid = items < sms ? items : sms;
  const size_t smem = (size_t)C2_SMEM_FLOATS * sizeof(float);
  static bool attr = false;
  if (!attr) {
    if (cudaFuncSetAttribute(chain2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return DWBC_ERR_LAUNCH;
    attr = true;
  }
  chain2_kernel<<<grid, C2_THREADS, smem, st>>>(L, tiles);
  ++dwbc_launch_counter;
  return cudaGetLastError() == cudaSuccess ? DWBC_OK : DWBC_ERR_LAUNCH;
}

}  // namespace dwbc
