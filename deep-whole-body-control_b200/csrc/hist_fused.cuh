// History encoder (StateHistoryEncoder, AC:39-84: Linear 76->30 + act per time step, the tsteps-specific Conv1d stack + act, Flatten,
// Linear 30->latent + act) as ONE exact-fp32 kernel for the inference uses: the regulariser target of PPO.update (PPO:175-176, no
// gradient), rollouts with hist_encoding (AC:207-210) and act_inference.  The layer-wise path needs a GEMM launch per layer plus packing /
// padding kernels and moves the [rows x T x 32] projection through HBM; here a thread owns a row, streams its T x 76 history once (the
// only HBM traffic: 304 B per step), and keeps every intermediate in registers at compile-time indices, one instantiation per variant:
//   * weights sit in shared memory transposed to [input][output], so one 16-byte broadcast load feeds four FMAs of four outputs;
//   * the first (strided) convolution is accumulated as the time steps arrive: step t feeds its tap of each of the at most k1 / s1 open
//     output positions (2, 3, 2 for tsteps 10, 20, 50), so no window of projected steps is kept;
//   * the second convolution keeps the last k2 - 1 finished conv-1 positions -- in shared memory, a ring of k2 - 1 slots per thread,
//     so that the 20- and 50-step variants stay spill-free -- and emits a position as soon as its window is complete; the third
//     (tsteps 50) accumulates its three positions as conv-2 positions arrive; the output layer runs once at the end.
// FMA per row: 34 200 (10 steps), 77 400 (20 steps), 176 000 (50 steps), on the fp32 pipe (the 3xTF32 mode uses it too: exact fp32).
#pragma once
#include "gemm_simt.cuh"

namespace dwbc {

// The conv stacks of StateHistoryEncoder by tsteps (AC:52-70): channels, kernel, stride of conv_layers.0, .2 (, .4).  The projection is
// 30 wide; every stack ends at 3 positions x 10 channels.  check_net (mlp.cu) accepts exactly these rows.
struct HistVariant { int T, nconv, c[3], k[3], s[3]; };
constexpr int HIST_NVAR = 3;
constexpr HistVariant HIST_VARIANTS[HIST_NVAR] = {{10, 2, {20, 10, 0}, {4, 2, 0}, {2, 1, 0}},
                                                  {20, 2, {20, 10, 0}, {6, 4, 0}, {2, 2, 0}},
                                                  {50, 3, {20, 10, 10}, {8, 5, 5}, {4, 1, 1}}};
constexpr int HIST_PROJ = 30, HIST_OUT_POS = 3;
constexpr int hist_out_len(int in, int k, int s) { return (in - k) / s + 1; }

constexpr int HF_THREADS = 128;

// compile-time geometry and shared-memory image (floats) of variant kV:
//   Wp[76][32] bp[32] | W1[k1*30][20] b1[20] | W2[k2*20][12] b2[12] | (W3[k3*10][12] b3[12]) | Wl[3*10][32] bl[32]
template <int kV>
struct HF {
  static constexpr HistVariant V = HIST_VARIANTS[kV];
  static constexpr int T = V.T, NC = V.nconv, K1 = V.k[0], S1 = V.s[0], K2 = V.k[1], S2 = V.s[1], K3 = V.k[2], S3 = V.s[2];
  static constexpr int P1 = hist_out_len(T, K1, S1), P2 = hist_out_len(P1, K2, S2);
  static constexpr int R1 = K1 / S1;                        // open conv-1 positions per step
  static constexpr int TU = (P1 - 1) * S1 + K1;             // time steps conv 1 reads (50 steps: the last two are outside every window)
  static_assert(K1 % S1 == 0 && (NC == 2 ? P2 : hist_out_len(P2, K3, S3)) == HIST_OUT_POS, "history variant geometry");
  static constexpr int WIN_BYTES = (K2 - 1) * 20 * HF_THREADS * 4;   // dynamic shared memory: the conv-2 windows of the CTA's rows
  static constexpr int WP = 0, BP = 76 * 32, W1 = BP + 32, B1 = W1 + K1 * 30 * 20, W2 = B1 + 20, B2 = W2 + K2 * 20 * 12, W3 = B2 + 12,
                       B3 = W3 + K3 * 10 * 12, WL = B3 + (NC == 3 ? 12 : 0), BL = WL + 30 * 32, FLOATS = BL + 32;
};

struct HistFusedArgs {
  const float* wp; const float* bp;     // encoder.0          [30][76], [30]
  const float* w1; const float* b1;     // conv_layers.0      [20][30][k1], [20]
  const float* w2; const float* b2;     // conv_layers.2      [10][20][k2], [10]
  const float* w3; const float* b3;     // conv_layers.4      [10][10][k3], [10] (tsteps 50 only)
  const float* wl; const float* bl;     // linear_output.0    [latent][30] over the channel-major flatten (c * 3 + t), [latent]
  RowMat hist;                          // row r -> first float of its [T][76] history block
  float* out; int64_t ld_out;           // [rows, ld_out]; columns [latent, ld_out) are zero-filled
  int rows, latent;
  int act;                              // hidden activation (ACT_*) after every layer (AC:49-73 apply the one activation throughout)
  int variant;                          // index into HIST_VARIANTS
};

// kAct: the hidden activation, in its precise form (expf / tanhf): this is the exact path
template <int kAct, int kV>
__global__ void __launch_bounds__(HF_THREADS) hist_fused_kernel(const HistFusedArgs a) {
  using G = HF<kV>;
  __shared__ __align__(16) float w[G::FLOATS];
  extern __shared__ __align__(16) float hf_win[];          // [K2 - 1 slots][20 channels][HF_THREADS]: conflict-free per-thread columns
  // ---- weights -> shared memory, transposed to [input][output] (pads zero) ----
  for (int i = threadIdx.x; i < G::FLOATS; i += HF_THREADS) {
    float v = 0.0f;
    if (i < G::BP) { const int in = i >> 5, o = i & 31; if (o < 30) v = a.wp[o * 76 + in]; }
    else if (i < G::W1) { const int o = i - G::BP; if (o < 30) v = a.bp[o]; }
    else if (i < G::B1) { const int j = i - G::W1, row = j / 20, o = j - row * 20, k = row / 30, c = row - k * 30; v = a.w1[(o * 30 + c) * G::K1 + k]; }
    else if (i < G::W2) v = a.b1[i - G::B1];
    else if (i < G::B2) { const int j = i - G::W2, row = j / 12, o = j - row * 12, k = row / 20, c = row - k * 20; if (o < 10) v = a.w2[(o * 20 + c) * G::K2 + k]; }
    else if (i < G::W3) { const int o = i - G::B2; if (o < 10) v = a.b2[o]; }
    else if (i < G::B3) { const int j = i - G::W3, row = j / 12, o = j - row * 12, k = row / 10, c = row - k * 10; if (o < 10) v = a.w3[(o * 10 + c) * G::K3 + k]; }
    else if (i < G::WL) { const int o = i - G::B3; if (o < 10) v = a.b3[o]; }
    else if (i < G::BL) { const int j = i - G::WL, row = j >> 5, o = j & 31, t = row / 10, c = row - t * 10; if (o < a.latent) v = a.wl[o * 30 + c * 3 + t]; }
    else { const int o = i - G::BL; if (o < a.latent) v = a.bl[o]; }
    w[i] = v;
  }
  __syncthreads();
  const int r = blockIdx.x * HF_THREADS + threadIdx.x;
  if (r >= a.rows) return;
  const float* hp = a.hist.row(r);
  // c1[j]: open conv-1 position t / S1 - (R1 - 1) + j.  Finished conv-1 position q sits in ring slot q % (K2 - 1) of win.
  // fin[u]: conv-2 output u (two convs) or conv-3 accumulator u (three convs), then its activation.
  float* win = hf_win + threadIdx.x;
  float c1[G::R1][20], fin[HIST_OUT_POS][12];
#pragma unroll
  for (int o = 0; o < 20; ++o)
#pragma unroll
    for (int j = 0; j < G::R1; ++j) c1[j][o] = j == G::R1 - 1 ? w[G::B1 + o] : 0.0f;
#pragma unroll
  for (int u = 0; u < HIST_OUT_POS; ++u)
#pragma unroll
    for (int o = 0; o < 12; ++o) fin[u][o] = G::NC == 3 ? w[G::B3 + o] : 0.0f;
  float4 xnext = __ldg(reinterpret_cast<const float4*>(hp));
#pragma unroll 1
  for (int t = 0; t < G::TU; ++t) {
    // ---- projection of step t: h = act(Wp x + bp) ----
    float h[32];
#pragma unroll
    for (int o = 0; o < 32; ++o) h[o] = w[G::BP + o];
    // (the whole [T][76] block of a row is contiguous: the next 16 bytes -- of this step or the first of the next one -- are requested
    // before the 128 FMAs of the current four inputs, so a thread always has one load in flight instead of waiting for each in turn)
    const float4* x4p = reinterpret_cast<const float4*>(hp + t * 76);
#pragma unroll 1
    for (int i4 = 0; i4 < 19; ++i4) {
      const float4 x4 = xnext;
      if (t * 19 + i4 + 1 < G::TU * 19) xnext = __ldg(x4p + i4 + 1);
      const float xs[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float4* wr = reinterpret_cast<const float4*>(w + G::WP + (4 * i4 + e) * 32);
#pragma unroll
        for (int o4 = 0; o4 < 8; ++o4) {
          const float4 w4 = wr[o4];
          h[4 * o4] = fmaf(w4.x, xs[e], h[4 * o4]); h[4 * o4 + 1] = fmaf(w4.y, xs[e], h[4 * o4 + 1]);
          h[4 * o4 + 2] = fmaf(w4.z, xs[e], h[4 * o4 + 2]); h[4 * o4 + 3] = fmaf(w4.w, xs[e], h[4 * o4 + 3]);
        }
      }
    }
#pragma unroll
    for (int o = 0; o < 30; ++o) h[o] = act_f<false>(kAct, h[o]);
    // ---- conv 1: step t is tap ph + (R1 - 1 - j) * S1 of open position pn - (R1 - 1) + j ----
    const int pn = t / G::S1, ph = t - pn * G::S1;
#pragma unroll
    for (int j = 0; j < G::R1; ++j) {
      const int pos = pn - (G::R1 - 1) + j;
      if (pos >= 0 && pos < G::P1) {
        const float* wk = w + G::W1 + (ph + (G::R1 - 1 - j) * G::S1) * 30 * 20;
#pragma unroll
        for (int c = 0; c < 30; ++c) {
          const float4* wr = reinterpret_cast<const float4*>(wk + c * 20);
#pragma unroll
          for (int o4 = 0; o4 < 5; ++o4) {
            const float4 w4 = wr[o4];
            c1[j][4 * o4] = fmaf(w4.x, h[c], c1[j][4 * o4]); c1[j][4 * o4 + 1] = fmaf(w4.y, h[c], c1[j][4 * o4 + 1]);
            c1[j][4 * o4 + 2] = fmaf(w4.z, h[c], c1[j][4 * o4 + 2]); c1[j][4 * o4 + 3] = fmaf(w4.w, h[c], c1[j][4 * o4 + 3]);
          }
        }
      }
    }
    if (ph == G::S1 - 1) {
      const int q = pn - (G::R1 - 1);       // the oldest open position has received its last tap
      if (q >= 0) {
#pragma unroll
        for (int o = 0; o < 20; ++o) c1[0][o] = act_f<false>(kAct, c1[0][o]);
        if (q >= G::K2 - 1 && (q - (G::K2 - 1)) % G::S2 == 0) {
          // conv 2 position v = window (conv-1 positions q - K2 + 1 .. q - 1 from the ring, q in c1[0]), taps in order per input channel
          const int v = (q - (G::K2 - 1)) / G::S2;
          int slot[G::K2 - 1];
#pragma unroll
          for (int k = 0; k < G::K2 - 1; ++k) slot[k] = (q - (G::K2 - 1) + k) % (G::K2 - 1) * 20 * HF_THREADS;
          float c2[12];
#pragma unroll
          for (int o = 0; o < 12; ++o) c2[o] = w[G::B2 + o];
#pragma unroll
          for (int c = 0; c < 20; ++c) {
            float xs[G::K2];
#pragma unroll
            for (int k = 0; k < G::K2 - 1; ++k) xs[k] = win[slot[k] + c * HF_THREADS];
            xs[G::K2 - 1] = c1[0][c];
#pragma unroll
            for (int o4 = 0; o4 < 3; ++o4) {
#pragma unroll
              for (int k = 0; k < G::K2; ++k) {
                const float x = xs[k];
                const float4 u = reinterpret_cast<const float4*>(w + G::W2 + (k * 20 + c) * 12)[o4];
                c2[4 * o4] = fmaf(u.x, x, c2[4 * o4]); c2[4 * o4 + 1] = fmaf(u.y, x, c2[4 * o4 + 1]);
                c2[4 * o4 + 2] = fmaf(u.z, x, c2[4 * o4 + 2]); c2[4 * o4 + 3] = fmaf(u.w, x, c2[4 * o4 + 3]);
              }
            }
          }
          if constexpr (G::NC == 2) {
            // positions arrive in order: shift in, so fin[u] ends as position u
#pragma unroll
            for (int o = 0; o < 10; ++o) {
#pragma unroll
              for (int u = 0; u < HIST_OUT_POS - 1; ++u) fin[u][o] = fin[u + 1][o];
              fin[HIST_OUT_POS - 1][o] = act_f<false>(kAct, c2[o]);
            }
          } else {
            // conv 3: position v of conv 2 is tap v - u * S3 of output position u
#pragma unroll
            for (int o = 0; o < 10; ++o) c2[o] = act_f<false>(kAct, c2[o]);
#pragma unroll
            for (int u = 0; u < HIST_OUT_POS; ++u) {
              const int tap = v - u * G::S3;
              if (tap >= 0 && tap < G::K3) {
#pragma unroll
                for (int c = 0; c < 10; ++c) {
                  const float4* wr = reinterpret_cast<const float4*>(w + G::W3 + (tap * 10 + c) * 12);
#pragma unroll
                  for (int o4 = 0; o4 < 3; ++o4) {
                    const float4 u4 = wr[o4];
                    fin[u][4 * o4] = fmaf(u4.x, c2[c], fin[u][4 * o4]); fin[u][4 * o4 + 1] = fmaf(u4.y, c2[c], fin[u][4 * o4 + 1]);
                    fin[u][4 * o4 + 2] = fmaf(u4.z, c2[c], fin[u][4 * o4 + 2]); fin[u][4 * o4 + 3] = fmaf(u4.w, c2[c], fin[u][4 * o4 + 3]);
                  }
                }
              }
            }
          }
        }
        float* wq = win + q % (G::K2 - 1) * 20 * HF_THREADS;
#pragma unroll
        for (int o = 0; o < 20; ++o) wq[o * HF_THREADS] = c1[0][o];
      }
#pragma unroll
      for (int o = 0; o < 20; ++o) {
#pragma unroll
        for (int j = 0; j + 1 < G::R1; ++j) c1[j][o] = c1[j + 1][o];
        c1[G::R1 - 1][o] = w[G::B1 + o];
      }
    }
  }
  if constexpr (G::NC == 3) {
#pragma unroll
    for (int u = 0; u < HIST_OUT_POS; ++u)
#pragma unroll
      for (int o = 0; o < 10; ++o) fin[u][o] = act_f<false>(kAct, fin[u][o]);
  }
  // ---- output layer over the channel-major flatten, position by position ----
  float z[32];
#pragma unroll
  for (int o = 0; o < 32; ++o) z[o] = w[G::BL + o];
#pragma unroll
  for (int u = 0; u < HIST_OUT_POS; ++u) {
#pragma unroll
    for (int c = 0; c < 10; ++c) {
      const float cv = fin[u][c];
      const float4* wr = reinterpret_cast<const float4*>(w + G::WL + (u * 10 + c) * 32);
#pragma unroll
      for (int o4 = 0; o4 < 8; ++o4) {
        const float4 w4 = wr[o4];
        z[4 * o4] = fmaf(w4.x, cv, z[4 * o4]); z[4 * o4 + 1] = fmaf(w4.y, cv, z[4 * o4 + 1]);
        z[4 * o4 + 2] = fmaf(w4.z, cv, z[4 * o4 + 2]); z[4 * o4 + 3] = fmaf(w4.w, cv, z[4 * o4 + 3]);
      }
    }
  }
  float* orow = a.out + (int64_t)r * a.ld_out;
#pragma unroll
  for (int o = 0; o < 32; ++o)
    if (o < a.ld_out) orow[o] = o < a.latent ? act_f<false>(kAct, z[o]) : 0.0f;
}

template <int kAct, int kV>
inline int launch_hist_fused_av(const HistFusedArgs& a, unsigned grid, cudaStream_t st) {
  constexpr int dyn = HF<kV>::WIN_BYTES;
  static bool attr = false;               // static + dynamic shared memory exceeds the 48 KB default for the 20- and 50-step variants
  if (!attr) {
    if (cudaFuncSetAttribute(hist_fused_kernel<kAct, kV>, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn) != cudaSuccess) return DWBC_ERR_LAUNCH;
    attr = true;
  }
  hist_fused_kernel<kAct, kV><<<grid, HF_THREADS, dyn, st>>>(a);
  return DWBC_OK;
}
template <int kV>
inline int launch_hist_fused_v(const HistFusedArgs& a, unsigned grid, cudaStream_t st) {
  switch (a.act) {
    case ACT_ELU: return launch_hist_fused_av<ACT_ELU, kV>(a, grid, st);
    case ACT_SELU: return launch_hist_fused_av<ACT_SELU, kV>(a, grid, st);
    case ACT_RELU: return launch_hist_fused_av<ACT_RELU, kV>(a, grid, st);
    case ACT_LRELU: return launch_hist_fused_av<ACT_LRELU, kV>(a, grid, st);
    case ACT_TANH: return launch_hist_fused_av<ACT_TANH, kV>(a, grid, st);
    case ACT_SIGMOID: return launch_hist_fused_av<ACT_SIGMOID, kV>(a, grid, st);
    default: return DWBC_ERR_UNSUPPORTED;
  }
}

// latent <= 32, ld_out <= 32, history rows 16-byte aligned
inline int launch_hist_fused(const HistFusedArgs& a, cudaStream_t st) {
  if (a.rows <= 0 || a.latent > 32 || a.ld_out > 32 || a.ld_out < a.latent) return DWBC_ERR_UNSUPPORTED;
  const unsigned grid = (a.rows + HF_THREADS - 1) / HF_THREADS;
  int rc = DWBC_ERR_UNSUPPORTED;
  switch (a.variant) {
    case 0: rc = launch_hist_fused_v<0>(a, grid, st); break;
    case 1: rc = launch_hist_fused_v<1>(a, grid, st); break;
    case 2: rc = launch_hist_fused_v<2>(a, grid, st); break;
    default: break;
  }
  if (rc != DWBC_OK) return rc;
  ++dwbc_launch_counter;
  return cudaGetLastError() == cudaSuccess ? DWBC_OK : DWBC_ERR_LAUNCH;
}

}  // namespace dwbc
