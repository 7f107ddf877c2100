// ActorCritic forward / PPO loss / hand-written backward, fp32 CUDA-core path (K5-K8 anchor).
//
// Layer-wise: every nn.Linear (+ its activation) of `rsl_rl/modules/actor_critic.py` is one launch of
// the tile GEMM in gemm_simt.cuh with the bias/activation (forward) or activation derivative
// (backward) fused into its epilogue; the mini-batch gather (RS:189-201) is fused into the
// first-layer operand loads (no gathered batch is materialised); the Conv1d history encoder
// (AC:39-84) is expressed as three more GEMMs over re-packed weights.  The PPO loss
// (PPO:199-221) and its derivative w.r.t. the network outputs is one elementwise kernel.
#include <math.h>

#include <stdlib.h>

#include "hist_fused.cuh"
#include "mlp_chain2.cuh"
#include "wgrad_group.cuh"
#include "dwbc_debug.h"

namespace dwbc {

// precision of the ActorCritic GEMMs of the CURRENT call (DwbcNetCfg.precision, set by every entry point):
// 0 = fp32 CUDA cores (parity anchor), 1 = TF32 wgmma, 2 = 3xTF32 wgmma (error-compensated, fp32-grade)
thread_local int mlp_precision = 0;
// hidden-layer activation of the CURRENT call (DwbcNetCfg.activation as an ACT_* code, set by every entry point): every layer of the
// encoders, backbones and head hidden layers; the actor heads' outputs keep tanh and the critic heads' stay linear
thread_local int mlp_act = 0;
// partial area of the weight-gradient launches of the CURRENT call (gemm_simt.cuh): the workspace's, set by make_plan
thread_local float* mlp_wpart = nullptr;
thread_local int64_t mlp_wpart_cap = 0;

static inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

struct Bump {
  char* base;
  int64_t off;
  float* f(int64_t n) {
    float* p = base ? reinterpret_cast<float*>(base + off) : nullptr;
    off += align_up(n * (int64_t)sizeof(float), 256);
    return p;
  }
};

static inline int last(const int32_t* d, int n) { return d[n - 1]; }

// ---- workspace plan ----------------------------------------------------------------------------
struct Plan {
  // forward activations (saved for backward)
  float* priv[DWBC_MAX_LAYERS];   // priv encoder outputs; the last one is the latent z
  float* ab[DWBC_MAX_LAYERS];     // actor backbone
  float* al[DWBC_MAX_LAYERS];     // actor leg head hidden
  float* aa[DWBC_MAX_LAYERS];     // actor arm head hidden
  float* mean;                    // [rows, mean_ld] tanh outputs (leg | arm)
  float* cb[DWBC_MAX_LAYERS];
  float* cl[DWBC_MAX_LAYERS];
  float* ca[DWBC_MAX_LAYERS];
  float* value;                   // [rows, 2]
  // history encoder (HistGeo: conv i reads rows of width ld[i] and writes positions pos[i + 1] x ld[i + 1])
  float* hproj;                   // [rows*T, 32]
  float* hc[3];                   // conv outputs [rows*pos[i+1], ld[i+1]]: [rows*P1, 20], [rows*P2, 12] (, [rows*3, 12])
  float* zh;                      // [rows, latent]
  float* hw[3]; float* hwl;                // re-packed weights: conv i [c_i][k_i*ld[i]], linear_output [32][36]
  float* wpack;                            // packed weight images of the fused chain kernels (mlp_chain2.cuh)
  int* queue;                              // counters, zero between launches: [0..1] work queue of the chain kernel, [2] ppo_loss_kernel, [3]
                                           // dagger_loss_kernel, [4] ppo_diag_kernel
  float* loss_part;                        // per-block / per-(tile, warp) partial sums of the loss kernels
  float* wpart;                            // per-(GEMM, slab) / per-(split) partials of the weight gradients (wpart_floats)
  // gradients
  float* g_leg; float* g_arm; float* g_vl; float* g_va; float* g_z;   // g_vl / g_va: columns 0 / 1 of one [rows, 4] buffer
  // per-layer pre-activation gradients kept by the fused backward chain for the weight-gradient GEMMs
  float* dza_l[DWBC_MAX_LAYERS]; float* dza_a[DWBC_MAX_LAYERS]; float* dza_b[DWBC_MAX_LAYERS]; float* dzp[DWBC_MAX_LAYERS];
  float* dzc_l[DWBC_MAX_LAYERS]; float* dzc_a[DWBC_MAX_LAYERS]; float* dzc_b[DWBC_MAX_LAYERS];
  float* d0; float* d1; float* d2;         // ping-pong [rows, maxw]
  float* dz;                               // [rows, latent]
  float* dzh;                              // [rows, latent] (dagger)
  float* dh_a[3];                          // im2col-space grads of the conv inputs (dagger) [rows*pos[i+1], k_i*ld[i]]
  float* dh_c[2]; float* dh_proj;          // grads of the conv-2 / conv-3 inputs [rows*pos[i], ld[i]] and of the projection
  float* dhw[3]; float* dhwl;              // grads of the re-packed weights (dagger)
  int mean_ld, maxw, latent;
  int64_t bytes;
};

// The history encoder's variant (a row of HIST_VARIANTS, hist_fused.cuh) with the row widths of the layer-wise path: the projection
// is padded to 32 channels (so 10 steps keep K = 128 for conv 1), conv-1 outputs are 20 wide, later conv outputs 12 (linear_output
// reads 3 x 12).  Conv i is one GEMM over overlapping windows: output position p of a row reads the k_i * ld[i] contiguous floats
// from input position p * s_i on.
struct HistGeo {
  int var, T, nconv;
  int c[3], k[3], s[3];
  int cin[3], ld[4], pos[4];
  int kdim(int i) const { return k[i] * ld[i]; }
};
static int hist_variant(const DwbcNetCfg& n) {
  for (int v = 0; v < HIST_NVAR; ++v) {
    const HistVariant& h = HIST_VARIANTS[v];
    if (n.num_hist != h.T || n.n_hist_conv != h.nconv || n.hist_proj != HIST_PROJ) continue;
    const int32_t got[9] = {n.hist_c1, n.hist_k1, n.hist_s1, n.hist_c2, n.hist_k2, n.hist_s2, n.hist_c3, n.hist_k3, n.hist_s3};
    bool ok = true;
    for (int i = 0; i < 3; ++i) ok = ok && got[3 * i] == h.c[i] && got[3 * i + 1] == h.k[i] && got[3 * i + 2] == h.s[i];
    if (ok) return v;
  }
  return -1;
}
static HistGeo hist_geo(const DwbcNetCfg& n) {
  HistGeo g{};
  g.var = hist_variant(n);
  if (g.var < 0) return g;                  // (every entry point has refused such a net in check_net)
  const HistVariant& h = HIST_VARIANTS[g.var];
  g.T = h.T; g.nconv = h.nconv;
  g.pos[0] = h.T; g.ld[0] = 32;
  for (int i = 0; i < h.nconv; ++i) {
    g.c[i] = h.c[i]; g.k[i] = h.k[i]; g.s[i] = h.s[i];
    g.cin[i] = i == 0 ? HIST_PROJ : h.c[i - 1];
    g.ld[i + 1] = i == 0 ? 20 : 12;
    g.pos[i + 1] = hist_out_len(g.pos[i], h.k[i], h.s[i]);
  }
  return g;
}

static int maxdim(const DwbcNetCfg& n) {
  int m = 32;
  auto up = [&](const int32_t* d, int k) { for (int i = 0; i < k; ++i) m = d[i] > m ? d[i] : m; };
  up(n.priv_dims, n.n_priv_layers); up(n.actor_dims, n.n_actor_layers); up(n.critic_dims, n.n_critic_layers);
  up(n.leg_dims, n.n_leg_layers); up(n.arm_dims, n.n_arm_layers);
  return (int)align_up(m, 4);
}

// activations / pre-activation gradients of 128-wide layers are kept as tile images by the tensor-core path (RowMat::image):
// whole 128-row tiles, so the buffer covers the rows rounded up to a tile
static inline bool img_dim(int d) { return d == 128; }
static inline int64_t act_floats(int64_t rows, int d) { return img_dim(d) ? align_up(rows, 128) * 128 : rows * align_up(d, 4); }
static inline RowMat act_mat(const float* p, int d) { return img_dim(d) ? rowmat_image(p) : rowmat(p, d); }

constexpr int LOSS_PART = 40;              // ppo_loss_kernel, per block: the five loss means, then the std gradient (<= 32)
// partial sums of the loss hooks: one slot per (128-row tile, worker warp) of the chain kernel, one per 128-row block of ppo_loss_kernel
static int64_t loss_part_floats(int64_t rows) {
  static_assert(C2_FIN_PART >= LOSS_PART, "one area serves both");
  return (rows + 127) / 128 * C2_WORKERS * C2_FIN_PART;
}

// Partials of the weight-gradient launches, for every plan a call with `rows` rows can make (any SM count), and
// never fewer for more rows: the largest of
//   the grouped launch: at most wg_max_nslab(rows) slabs per GEMM, and its GEMMs' slots hold at most every parameter (+ alignment);
//   one layer-wise TF32 weight gradient (<= 128 x 128) over at most rows x num_hist rows (the history projection);
//   one split-K CUDA-core weight gradient: CTAs x splits < tiles + 592, tiles <= (d / 64)^2 for the widest operand d.
static int64_t wpart_floats(const DwbcNetCfg& n, int64_t rows) {
  const int64_t group = wg_max_nslab(rows) * (n.num_params + 4 * WG_MAX);
  const int64_t one = wg_max_nslab(rows * n.num_hist) * wg_slot(128, 128);
  const int64_t d = std::max<int64_t>(maxdim(n), std::max(n.num_prop + n.num_priv, 256)), t = ((d + 63) / 64) * ((d + 63) / 64);
  const int64_t simt = (t + 592) * (GT_M * GT_N + GT_M);
  return std::max(group, std::max(one, simt));
}

static Plan make_plan(const DwbcNetCfg& n, int64_t rows, void* ws) {
  Plan p{};
  Bump b{reinterpret_cast<char*>(ws), 0};
  p.queue = reinterpret_cast<int*>(b.f(64));      // FIRST: the same address whatever `rows` is (callers share one workspace between row counts;
                                                  // the counters must stay zero between launches, nothing else may ever be laid over them)
  p.latent = last(n.priv_dims, n.n_priv_layers);
  p.maxw = maxdim(n);
  p.mean_ld = (int)align_up(n.n_leg + n.n_arm, 4);
  for (int i = 0; i < n.n_priv_layers; ++i) p.priv[i] = b.f(rows * align_up(n.priv_dims[i], 4));
  for (int i = 0; i < n.n_actor_layers; ++i) p.ab[i] = b.f(act_floats(rows, n.actor_dims[i]));
  for (int i = 0; i < n.n_leg_layers; ++i) p.al[i] = b.f(act_floats(rows, n.leg_dims[i]));
  for (int i = 0; i < n.n_arm_layers; ++i) p.aa[i] = b.f(act_floats(rows, n.arm_dims[i]));
  p.mean = b.f(rows * p.mean_ld);
  for (int i = 0; i < n.n_critic_layers; ++i) p.cb[i] = b.f(act_floats(rows, n.critic_dims[i]));
  for (int i = 0; i < n.n_leg_layers; ++i) p.cl[i] = b.f(act_floats(rows, n.leg_dims[i]));
  for (int i = 0; i < n.n_arm_layers; ++i) p.ca[i] = b.f(act_floats(rows, n.arm_dims[i]));
  p.value = b.f(rows * 2);
  const HistGeo g = hist_geo(n);
  const bool c3 = g.nconv == 3;            // (the absent third conv takes no space: the 10-step plan is the one it always was)
  p.hproj = b.f(rows * n.num_hist * 32);
  for (int i = 0; i < 3; ++i) p.hc[i] = b.f(i < g.nconv ? rows * g.pos[i + 1] * g.ld[i + 1] : 0);
  p.zh = b.f(rows * align_up(p.latent, 4));
  for (int i = 0; i < 2; ++i) p.hw[i] = b.f(g.c[i] * g.kdim(i));
  p.hw[2] = b.f(c3 ? g.c[2] * g.kdim(2) : 0);
  p.hwl = b.f(32 * 36);
  p.wpack = b.f(C2_PACK_FLOATS);
  p.g_leg = b.f(rows * align_up(n.n_leg, 4)); p.g_arm = b.f(rows * align_up(n.n_arm, 4));
  p.g_vl = b.f(rows * 4); p.g_va = p.g_vl ? p.g_vl + 1 : nullptr; p.g_z = b.f(rows * align_up(p.latent, 4));
  for (int i = 0; i < n.n_leg_layers; ++i) { p.dza_l[i] = b.f(act_floats(rows, n.leg_dims[i])); p.dzc_l[i] = b.f(act_floats(rows, n.leg_dims[i])); }
  for (int i = 0; i < n.n_arm_layers; ++i) { p.dza_a[i] = b.f(act_floats(rows, n.arm_dims[i])); p.dzc_a[i] = b.f(act_floats(rows, n.arm_dims[i])); }
  for (int i = 0; i < n.n_actor_layers; ++i) p.dza_b[i] = b.f(act_floats(rows, n.actor_dims[i]));
  for (int i = 0; i < n.n_critic_layers; ++i) p.dzc_b[i] = b.f(act_floats(rows, n.critic_dims[i]));
  for (int i = 0; i < n.n_priv_layers; ++i) p.dzp[i] = b.f(rows * align_up(n.priv_dims[i], 4));
  p.d0 = b.f(rows * p.maxw); p.d1 = b.f(rows * p.maxw); p.d2 = b.f(rows * p.maxw);
  p.dz = b.f(rows * align_up(p.latent, 4));
  p.dzh = b.f(rows * align_up(p.latent, 4));
  for (int i = 0; i < 3; ++i) p.dh_a[i] = b.f(i < g.nconv ? rows * g.pos[i + 1] * g.kdim(i) : 0);
  p.dh_c[0] = b.f(rows * g.pos[1] * g.ld[1]);
  p.dh_c[1] = b.f(c3 ? rows * g.pos[2] * g.ld[2] : 0);
  p.dh_proj = b.f(rows * n.num_hist * 32);
  for (int i = 0; i < 3; ++i) p.dhw[i] = b.f(i < g.nconv ? g.c[i] * g.kdim(i) : 0);
  p.dhwl = b.f(32 * 36);
  p.loss_part = b.f(loss_part_floats(rows));
  p.wpart = b.f(wpart_floats(n, rows));
  p.bytes = b.off;
  if (ws) { mlp_wpart = p.wpart; mlp_wpart_cap = wpart_floats(n, rows); }     // (the area the weight-gradient launches of this call use)
  return p;
}

// DwbcActivation -> the epilogues' ACT_* code; -1: not an activation the kernels implement
static int hidden_act(int32_t a) {
  switch (a) {
    case DWBC_ACT_ELU: return ACT_ELU;
    case DWBC_ACT_SELU: return ACT_SELU;
    case DWBC_ACT_RELU: return ACT_RELU;
    case DWBC_ACT_LRELU: return ACT_LRELU;
    case DWBC_ACT_TANH: return ACT_TANH;
    case DWBC_ACT_SIGMOID: return ACT_SIGMOID;
    default: return -1;
  }
}

static int check_net(const DwbcNetCfg* n) {
  if (!n || n->abi_version != DWBC_ABI_VERSION || n->precision < 0 || n->precision > 2) return DWBC_ERR_ARG;
  mlp_precision = n->precision;
  mlp_act = hidden_act(n->activation);
  if (mlp_act < 0) return DWBC_ERR_UNSUPPORTED;
  if (n->n_priv_layers < 1 || n->n_priv_layers > DWBC_MAX_LAYERS || n->n_actor_layers < 1 || n->n_actor_layers > DWBC_MAX_LAYERS ||
      n->n_critic_layers < 1 || n->n_critic_layers > DWBC_MAX_LAYERS || n->n_leg_layers < 1 || n->n_leg_layers > DWBC_MAX_LAYERS ||
      n->n_arm_layers < 1 || n->n_arm_layers > DWBC_MAX_LAYERS)
    return DWBC_ERR_UNSUPPORTED;
  // history encoder: the conv stacks of tsteps 10, 20 and 50 (AC:52-70); the reference raises for any other tsteps
  if (hist_variant(*n) < 0) return DWBC_ERR_UNSUPPORTED;
  if (last(n->priv_dims, n->n_priv_layers) > 32 || n->n_leg + n->n_arm > 32) return DWBC_ERR_UNSUPPORTED;
  return DWBC_OK;
}

// ---- history-encoder weight re-packing ---------------------------------------------------------
// conv i [c,cin,k] -> Wi'[c][k*ld+cin] (ld = the row width of its input: 32, 20, 12); linear [L,30] over the channel-major flatten
// (c*3+t) -> Wl'[L][t*12+c].  Pad entries are zero.
struct HistPack {
  float* w[3]; float* wp[3];      // reference-layout and re-packed conv weights (or their gradients)
  int c[3], cin[3], k[3], ld[3];
  int nconv;
  float* wl; float* wlp; int latent;
};
static HistPack hist_pack_args(const HistGeo& g, const float* w0, const float* w1, const float* w2, const float* wl, float* const* wp, float* wlp,
                               int latent) {
  HistPack a{};
  const float* w[3] = {w0, w1, w2};
  for (int i = 0; i < g.nconv; ++i) {
    a.w[i] = const_cast<float*>(w[i]); a.wp[i] = wp[i]; a.c[i] = g.c[i]; a.cin[i] = g.cin[i]; a.k[i] = g.k[i]; a.ld[i] = g.ld[i];
  }
  a.nconv = g.nconv; a.wl = const_cast<float*>(wl); a.wlp = wlp; a.latent = latent;
  return a;
}
static unsigned hist_pack_grid(const HistGeo& g) {
  int n = 32 * 36;
  for (int i = 0; i < g.nconv; ++i) n = g.c[i] * g.kdim(i) > n ? g.c[i] * g.kdim(i) : n;
  return (unsigned)((n + 255) / 256);
}
__global__ void hist_pack_kernel(const HistPack a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  for (int l = 0; l < a.nconv; ++l) {
    const int kd = a.k[l] * a.ld[l];
    if (i < a.c[l] * kd) {
      const int o = i / kd, r = i % kd, k = r / a.ld[l], cin = r % a.ld[l];
      a.wp[l][i] = cin < a.cin[l] ? a.w[l][(o * a.cin[l] + cin) * a.k[l] + k] : 0.0f;
    }
  }
  if (i < a.latent * 36) {
    int j = i / 36, r = i % 36, t = r / 12, c2 = r % 12;
    a.wlp[i] = c2 < 10 ? a.wl[j * 30 + c2 * 3 + t] : 0.0f;
  }
}
// inverse scatter of the re-packed weight gradients (wp, wlp) into the flat gradient (w, wl: reference layouts)
__global__ void hist_unpack_grad_kernel(const HistPack a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  for (int l = 0; l < a.nconv; ++l) {
    const int kd = a.k[l] * a.ld[l];
    if (i < a.c[l] * kd) {
      const int o = i / kd, r = i % kd, k = r / a.ld[l], cin = r % a.ld[l];
      if (cin < a.cin[l]) a.w[l][(o * a.cin[l] + cin) * a.k[l] + k] = a.wp[l][i];
    }
  }
  if (i < a.latent * 36) {
    int j = i / 36, r = i % 36, t = r / 12, c2 = r % 12;
    if (c2 < 10) a.wl[j * 30 + c2 * 3 + t] = a.wlp[i];
  }
}
// col2im of the conv input gradients (overlapping windows) fused with the derivative of the activation `act`:
// dst[m][t][c] = act'(y[m][t][c]) * sum_{t'*stride + k == t} src[(m*To + t')][k*C + c]
__global__ void col2im_dact_kernel(const float* __restrict__ src, const float* __restrict__ y, float* __restrict__ dst, int64_t rows,
                                   int Tin, int C, int ldc, int To, int ksz, int stride, int act) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t total = rows * Tin * ldc;
  if (i >= total) return;
  int c = (int)(i % ldc);
  int t = (int)((i / ldc) % Tin);
  int64_t m = i / ((int64_t)ldc * Tin);
  float s = 0.0f;
  if (c < C) {
    for (int k = 0; k < ksz; ++k) {
      int tt = t - k;
      if (tt < 0 || tt % stride) continue;
      int to = tt / stride;
      if (to >= To) continue;
      s += src[(m * To + to) * (int64_t)(ksz * ldc) + k * ldc + c];
    }
    s *= act_df(act, y[i]);
  }
  dst[i] = s;
}

__global__ void zero_cols_kernel(float* __restrict__ p, int64_t nrows, int ld, int c0) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int w = ld - c0;
  if (i < nrows * w) p[(i / w) * ld + c0 + (i % w)] = 0.0f;
}

// ---- forward ------------------------------------------------------------------------------------
#define TRY(x) do { int rc__ = (x); if (rc__ != DWBC_OK) return rc__; } while (0)

static int hist_forward(const DwbcNetCfg& n, const float* P, const float* obs, const int64_t* idx, int64_t obs_stride, int rows,
                        const Plan& p, cudaStream_t st) {
  const HistGeo g = hist_geo(n);
  const int T = n.num_hist, L = p.latent, Lld = (int)align_up(L, 4);
  hist_pack_kernel<<<hist_pack_grid(g), 256, 0, st>>>(
      hist_pack_args(g, P + n.off_hist_w[1], P + n.off_hist_w[2], P + n.off_hist_w[3], P + n.off_hist_w[4], p.hw, p.hwl, L));
  dwbc_launch_counter += 1 + g.nconv;
  // pad columns of the padded activation buffers are consumed by the next GEMM's K range
  zero_cols_kernel<<<(unsigned)(((int64_t)rows * T * 2 + 255) / 256), 256, 0, st>>>(p.hproj, (int64_t)rows * T, 32, 30);
  for (int i = 1; i < g.nconv; ++i)
    zero_cols_kernel<<<(unsigned)(((int64_t)rows * g.pos[i + 1] * 2 + 255) / 256), 256, 0, st>>>(p.hc[i], (int64_t)rows * g.pos[i + 1], 12, 10);
  RowMat hist = rowmat_grouped(obs + (n.num_obs - T * n.num_prop), idx, T, obs_stride, n.num_prop);
  TRY(linear_fwd(hist, P + n.off_hist_w[0], n.num_prop, P + n.off_hist_b[0], p.hproj, 32, rows * T, 30, n.num_prop, mlp_act, 0, st));  // AC:80
  const float* in = p.hproj;
  for (int i = 0; i < g.nconv; ++i) {                                                                                                   // AC:52-70
    RowMat a = rowmat_grouped(in, nullptr, g.pos[i + 1], (int64_t)g.pos[i] * g.ld[i], g.s[i] * g.ld[i]);
    TRY(linear_fwd(a, p.hw[i], g.kdim(i), P + n.off_hist_b[1 + i], p.hc[i], g.ld[i + 1], rows * g.pos[i + 1], g.c[i], g.kdim(i), mlp_act, 0, st));
    in = p.hc[i];
  }
  TRY(linear_fwd(rowmat(in, 36), p.hwl, 36, P + n.off_hist_b[4], p.zh, Lld, rows, L, 36, mlp_act, 0, st));                              // AC:72
  return DWBC_OK;
}

// history latent only (no intermediates kept): the fused exact-fp32 kernel on the tensor-core precisions (hist_fused.cuh), the layer-wise
// GEMMs on the fp32 anchor path
static int hist_latent_only(const DwbcNetCfg& n, const float* P, const float* obs, const int64_t* idx, int64_t obs_stride, int rows, const Plan& p,
                            float* out, int64_t ld_out, cudaStream_t st) {
  if (mlp_precision == 0 || (obs_stride & 3) || (reinterpret_cast<uintptr_t>(obs) & 15) || (n.num_prop & 3) || ((n.num_obs - n.num_hist * n.num_prop) & 3)) {
    Plan q = p;
    q.zh = out;
    if (ld_out != align_up(p.latent, 4)) return DWBC_ERR_ARG;
    return hist_forward(n, P, obs, idx, obs_stride, rows, q, st);
  }
  HistFusedArgs a{};
  a.wp = P + n.off_hist_w[0]; a.bp = P + n.off_hist_b[0]; a.w1 = P + n.off_hist_w[1]; a.b1 = P + n.off_hist_b[1];
  a.w2 = P + n.off_hist_w[2]; a.b2 = P + n.off_hist_b[2]; a.wl = P + n.off_hist_w[4]; a.bl = P + n.off_hist_b[4];
  a.variant = hist_variant(n);
  if (n.n_hist_conv == 3) { a.w3 = P + n.off_hist_w[3]; a.b3 = P + n.off_hist_b[3]; }
  a.hist = rowmat_gather(obs + (n.num_obs - n.num_hist * n.num_prop), idx, obs_stride);
  a.out = out; a.ld_out = ld_out; a.rows = rows; a.latent = p.latent; a.act = mlp_act;
  return launch_hist_fused(a, st);
}

static int priv_forward(const DwbcNetCfg& n, const float* P, const float* obs, const int64_t* idx, int64_t obs_stride, int rows,
                        const Plan& p, cudaStream_t st) {
  RowMat h = rowmat_gather(obs + n.num_prop, idx, obs_stride);
  int in = n.num_priv;
  for (int l = 0; l < n.n_priv_layers; ++l) {
    int out = n.priv_dims[l], ld = (int)align_up(out, 4);
    TRY(linear_fwd(h, P + n.off_priv_w[l], in, P + n.off_priv_b[l], p.priv[l], ld, rows, out, in, mlp_act, 0, st));  // AC:219-221
    h = rowmat(p.priv[l], ld);
    in = out;
  }
  return DWBC_OK;
}

static int head_forward(const float* P, RowMat h, int in, int nl, const int32_t* dims, int n_out, const int64_t* ow, const int64_t* ob,
                        float* const* acts, float* out, int64_t ldo, int last_act, int rows, cudaStream_t st) {
  for (int l = 0; l < nl; ++l) {
    TRY(linear_fwd(h, P + ow[l], in, P + ob[l], acts[l], dims[l], rows, dims[l], in, mlp_act, 0, st));
    h = rowmat(acts[l], dims[l]);
    in = dims[l];
  }
  return linear_fwd(h, P + ow[nl], in, P + ob[nl], out, ldo, rows, n_out, in, last_act, 0, st);
}

// Actor.forward (AC:204-217); latent z must already be in `z` (row stride zld)
static int actor_forward(const DwbcNetCfg& n, const float* P, const float* obs, const int64_t* idx, int64_t obs_stride, int rows,
                         const float* z, int zld, const Plan& p, cudaStream_t st) {
  RowMat x = rowmat_gather(obs, idx, obs_stride);
  const int in0 = n.num_prop + p.latent;
  // backbone layer 0 over cat([obs_prop, z]) as two accumulating GEMMs (no concat buffer)
  int single = n.n_actor_layers;
  TRY(linear_fwd(x, P + n.off_actor_w[0], in0, P + n.off_actor_b[0], p.ab[0], n.actor_dims[0], rows, n.actor_dims[0], n.num_prop, ACT_NONE, 0, st));
  TRY(linear_fwd(rowmat(z, zld), P + n.off_actor_w[0] + n.num_prop, in0, nullptr, p.ab[0], n.actor_dims[0], rows, n.actor_dims[0], p.latent,
                 mlp_act, 1, st));
  RowMat h = rowmat(p.ab[0], n.actor_dims[0]);
  int in = n.actor_dims[0];
  for (int l = 1; l < single; ++l) {
    TRY(linear_fwd(h, P + n.off_actor_w[l], in, P + n.off_actor_b[l], p.ab[l], n.actor_dims[l], rows, n.actor_dims[l], in, mlp_act, 0, st));
    h = rowmat(p.ab[l], n.actor_dims[l]);
    in = n.actor_dims[l];
  }
  TRY(head_forward(P, h, in, n.n_leg_layers, n.leg_dims, n.n_leg, n.off_aleg_w, n.off_aleg_b, p.al, p.mean, p.mean_ld, ACT_TANH, rows, st));
  TRY(head_forward(P, h, in, n.n_arm_layers, n.arm_dims, n.n_arm, n.off_aarm_w, n.off_aarm_b, p.aa, p.mean + n.n_leg, p.mean_ld, ACT_TANH, rows, st));
  return DWBC_OK;
}

// Critic.forward (AC:280-286)
static int critic_forward(const DwbcNetCfg& n, const float* P, const float* obs, const int64_t* idx, int64_t obs_stride, int rows,
                          const Plan& p, float* value, cudaStream_t st) {
  RowMat h = rowmat_gather(obs, idx, obs_stride);
  int in = n.num_prop + n.num_priv;
  for (int l = 0; l < n.n_critic_layers; ++l) {
    TRY(linear_fwd(h, P + n.off_critic_w[l], in, P + n.off_critic_b[l], p.cb[l], n.critic_dims[l], rows, n.critic_dims[l], in, mlp_act, 0, st));
    h = rowmat(p.cb[l], n.critic_dims[l]);
    in = n.critic_dims[l];
  }
  TRY(head_forward(P, h, in, n.n_leg_layers, n.leg_dims, 1, n.off_cleg_w, n.off_cleg_b, p.cl, value, 2, ACT_NONE, rows, st));
  TRY(head_forward(P, h, in, n.n_arm_layers, n.arm_dims, 1, n.off_carm_w, n.off_carm_b, p.ca, value + 1, 2, ACT_NONE, rows, st));
  return DWBC_OK;
}

// ---- fused forward (tensor-core paths): privileged encoder + actor and the critic as two programs of ONE launch (mlp_chain2.cuh) ----
static inline int pad8(int x) { return (x + 7) & ~7; }
constexpr int C2_COL_PRIV = 32, C2_COL_HID = 64, C2_COL_PROP = 32;     // tile columns of the encoder input / hidden layer and of obs_prop (z sits at 0)

static bool chain_usable(const DwbcNetCfg& n, const Plan& p, const float* obs, int64_t obs_stride) {
  if (mlp_precision == 0) return false;
  auto ok = [](const int32_t* d, int k) { for (int i = 0; i < k; ++i) if (d[i] > 128 || (d[i] & 3)) return false; return true; };
  if (!ok(n.priv_dims, n.n_priv_layers) || !ok(n.actor_dims, n.n_actor_layers) || !ok(n.critic_dims, n.n_critic_layers) ||
      !ok(n.leg_dims, n.n_leg_layers) || !ok(n.arm_dims, n.n_arm_layers))
    return false;
  // tile layout of the actor program: z at columns [0, 32), obs_prop at [32, 32 + num_prop), the encoder works at [32, 64) -> [64, 128) first
  if (n.n_priv_layers != 2 || n.num_priv > 32 || n.priv_dims[0] > 64 || p.latent > 32) return false;
  if ((n.num_prop & 3) || (n.num_priv & 3) || (p.latent & 3) || C2_COL_PROP + n.num_prop > 128 || n.num_prop + n.num_priv > 128) return false;
  if ((obs_stride & 3) || !c2_aligned(obs)) return false;
  if (n.n_leg > C2_GRP || n.n_arm > C2_GRP) return false;      // the epilogue hooks keep one action group in registers
  if (2 + n.n_actor_layers + n.n_leg_layers + n.n_arm_layers + 2 > C2_MAX_OPS) return false;
  if (n.n_critic_layers + n.n_leg_layers + n.n_arm_layers + 2 > C2_MAX_OPS) return false;
  return true;
}

// one head: optional trunk reload (the second head of a program), hidden layers in place, narrow last layer with its epilogue hook
static void chain_head(C2Builder& b, const float* P, const float* trunk, int trunk_ld, bool reload, int in, int nl, const int32_t* dims, int n_out,
                       const int64_t* ow, const int64_t* ob, float* const* acts, bool store, float* out, int64_t ldo, int last_act, int fin, int fin_c) {
  if (reload) b.load(act_mat(trunk, trunk_ld), in, 0, pad8(in), b.pr.n_ops);
  for (int l = 0; l < nl; ++l) {
    b.fwd(P + ow[l], in, P + ob[l], dims[l], mlp_act, 0, pad8(in), 1, C2PackSeg{0, 0, in}, C2PackSeg{0, 0, 0}, 0, store ? acts[l] : nullptr, dims[l],
          FIN_NONE, 0, store && img_dim(dims[l]));
    in = dims[l];
  }
  b.fwd(P + ow[nl], in, P + ob[nl], n_out, last_act, 0, pad8(in), 1, C2PackSeg{0, 0, in}, C2PackSeg{0, 0, 0}, -1, out, ldo, fin, fin_c);
}

// Programs of the forward pass.  z_hist == nullptr: latent from the privileged encoder (computed inside the chain); else the history
// latent [rows, zld].  `loss`: update mode (hooks FIN_REG / FIN_PPO / FIN_VALUE), else rollout mode (FIN_ACT), else none (fin_mode 0).
// keep_mean: the heads' last ops also write the means to Plan::mean in update mode (through the ops' ordinary global output), at row
// stride n_act: the vector stores of an op need 16-byte aligned rows, which stride n_act gives whenever they are taken (n_act and the
// head's N multiples of 4 make n_leg one too), so any action split the update runs on the chains still does.
// With A2 / C2 (inference only: `store` off) the two heads of a network become TWO programs that each recompute the short common part
// (encoder + backbone): a 4096-row rollout then is 4 programs x 32 tiles = 128 one-tile items of at most 6 ops on 128 SMs instead of
// 2 x 32 items of 9 / 7 ops on 64 SMs -- the launch is as long as its longest item.
static int build_forward(const DwbcNetCfg& n, const float* P, const float* obs, const int64_t* idx, int64_t obs_stride, const float* z_hist, int zld,
                         const Plan& p, float* value, bool store, int fin_mode, C2Builder* A, C2Builder* C, C2Builder* A2 = nullptr,
                         C2Builder* C2 = nullptr, bool keep_mean = false) {
  const int Lld = (int)align_up(p.latent, 4);
  if ((A2 || C2) && store) return DWBC_ERR_ARG;
  if (A) {
    const int in0 = n.num_prop + p.latent;
    const int na = n.n_actor_layers;
    // encoder (or the history latent) + backbone; returns the backbone's width.  `keep`: the last backbone layer is stored for a second head
    auto common = [&](C2Builder& B, bool keep) {
      int first_main = 0;
      if (z_hist) {
        B.load(rowmat(z_hist, zld), p.latent, 0, 32, 0);
      } else {
        B.load(rowmat_gather(obs + n.num_prop, idx, obs_stride), n.num_priv, C2_COL_PRIV, C2_COL_PRIV + pad8(n.num_priv), 0);
        B.fwd(P + n.off_priv_w[0], n.num_priv, P + n.off_priv_b[0], n.priv_dims[0], mlp_act, C2_COL_PRIV, pad8(n.num_priv), 1,      // AC:219-221
              C2PackSeg{0, 0, n.num_priv}, C2PackSeg{0, 0, 0}, C2_COL_HID, store ? p.priv[0] : nullptr, align_up(n.priv_dims[0], 4));
        B.fwd(P + n.off_priv_w[1], n.priv_dims[0], P + n.off_priv_b[1], p.latent, mlp_act, C2_COL_HID, pad8(n.priv_dims[0]), 1,
              C2PackSeg{0, 0, n.priv_dims[0]}, C2PackSeg{0, 0, 0}, 0, store ? p.priv[1] : nullptr, Lld, fin_mode == 2 ? FIN_REG : FIN_NONE, 0);
        first_main = 2;
      }
      const int k0 = pad8(C2_COL_PROP + n.num_prop);
      B.load(rowmat_gather(obs, idx, obs_stride), n.num_prop, C2_COL_PROP, k0, first_main);
      // backbone layer 0 over cat([obs_prop, z]) (AC:211): z occupies tile columns [0, latent), obs_prop [32, 32 + num_prop)
      B.fwd(P + n.off_actor_w[0], in0, P + n.off_actor_b[0], n.actor_dims[0], mlp_act, 0, k0, 2, C2PackSeg{0, n.num_prop, p.latent},
            C2PackSeg{C2_COL_PROP, 0, n.num_prop}, 0, (store || (keep && na == 1)) ? p.ab[0] : nullptr, n.actor_dims[0], FIN_NONE, 0,
            img_dim(n.actor_dims[0]) && (store || (keep && na == 1)));
      int in = n.actor_dims[0];
      for (int l = 1; l < na; ++l) {                                                   // AC:211-213
        const bool st = store || (keep && l == na - 1);
        B.fwd(P + n.off_actor_w[l], in, P + n.off_actor_b[l], n.actor_dims[l], mlp_act, 0, pad8(in), 1, C2PackSeg{0, 0, in}, C2PackSeg{0, 0, 0}, 0,
              st ? p.ab[l] : nullptr, n.actor_dims[l], FIN_NONE, 0, img_dim(n.actor_dims[l]) && st);
        in = n.actor_dims[l];
      }
      return in;
    };
    const int fin = fin_mode == 2 ? FIN_PPO : (fin_mode == 1 ? FIN_ACT : FIN_NONE);
    float* mean = fin_mode == 0 || keep_mean ? p.mean : nullptr;      // keep_mean: the update's means for ppo_diag_kernel
    const int64_t mean_ld = fin_mode == 0 ? p.mean_ld : n.n_leg + n.n_arm;
    const int in = common(*A, A2 == nullptr);
    chain_head(*A, P, p.ab[na - 1], in, false, in, n.n_leg_layers, n.leg_dims, n.n_leg, n.off_aleg_w, n.off_aleg_b, p.al, store, mean, mean_ld, ACT_TANH, fin, 0);
    C2Builder& Barm = A2 ? *A2 : *A;
    if (A2) common(*A2, false);
    chain_head(Barm, P, p.ab[na - 1], in, A2 == nullptr, in, n.n_arm_layers, n.arm_dims, n.n_arm, n.off_aarm_w, n.off_aarm_b, p.aa, store,
               mean ? mean + n.n_leg : nullptr, mean_ld, ACT_TANH, fin, 1);
    A->finish();
    if (A2) A2->finish();
    if (!A->ok || (A2 && !A2->ok)) return DWBC_ERR_UNSUPPORTED;
  }
  if (C) {
    const int nc = n.n_critic_layers;
    auto common = [&](C2Builder& B, bool keep) {
      int in = n.num_prop + n.num_priv;
      B.load(rowmat_gather(obs, idx, obs_stride), in, 0, pad8(in), 0);
      for (int l = 0; l < nc; ++l) {                                                   // AC:280-286
        const bool st = store || (keep && l == nc - 1);
        B.fwd(P + n.off_critic_w[l], in, P + n.off_critic_b[l], n.critic_dims[l], mlp_act, 0, pad8(in), 1, C2PackSeg{0, 0, in}, C2PackSeg{0, 0, 0}, 0,
              st ? p.cb[l] : nullptr, n.critic_dims[l], FIN_NONE, 0, img_dim(n.critic_dims[l]) && st);
        in = n.critic_dims[l];
      }
      return in;
    };
    const int fin = fin_mode == 2 ? FIN_VALUE : FIN_NONE;
    const int in = common(*C, C2 == nullptr);
    chain_head(*C, P, p.cb[nc - 1], in, false, in, n.n_leg_layers, n.leg_dims, 1, n.off_cleg_w, n.off_cleg_b, p.cl, store, value, 2, ACT_NONE, fin, 0);
    C2Builder& Barm = C2 ? *C2 : *C;
    if (C2) common(*C2, false);
    chain_head(Barm, P, p.cb[nc - 1], in, C2 == nullptr, in, n.n_arm_layers, n.arm_dims, 1, n.off_carm_w, n.off_carm_b, p.ca, store,
               value + 1, 2, ACT_NONE, fin, 1);
    C->finish();
    if (C2) C2->finish();
    if (!C->ok || (C2 && !C2->ok)) return DWBC_ERR_UNSUPPORTED;
  }
  return DWBC_OK;
}

// ---- rollout sampling + log-prob (AC:326-345, PPO:119-123) of the forward's means [rows, mean_ld] -------------
__global__ void act_finalize_kernel(const FinArgs f, const float* __restrict__ mean_in, int mean_ld) {
  int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= f.rows) return;
  float lp[2] = {0.0f, 0.0f};
  for (int i = 0; i < f.n_act; ++i) {
    const float mu = mean_in[(int64_t)r * mean_ld + i], sg = f.std[i];
    const float a = mu + sg * f.eps[(int64_t)r * f.n_act + i];
    lp[i < f.n_leg ? 0 : 1] += ppo_logp_term(a, mu, sg, logf(sg));
    f.actions[(int64_t)r * f.n_act + i] = a;
    f.mean_out[(int64_t)r * f.n_act + i] = mu;
    f.sigma_out[(int64_t)r * f.n_act + i] = sg;
  }
  f.log_prob[2 * r] = lp[0];
  f.log_prob[2 * r + 1] = lp[1];
}

// ---- PPO loss and its derivative w.r.t. the network outputs (PPO:166-221) ----------------------
// The forward's outputs: means [rows, mean_ld], values [rows, 2], privileged latent zp [rows, f.gz_ld].  f.part: [blocks][LOSS_PART]
// partials, added up in block order by the last block (ticket).
__global__ void __launch_bounds__(128) ppo_loss_kernel(const FinArgs f, const float* mean, int mean_ld, const float* value, const float* zp,
                                                       unsigned* ticket) {
  __shared__ float red[5 + 32][4];
  __shared__ float sched_s[3];            // the schedule values, loaded once per CTA
  if (threadIdx.x == 0) {
    sched_s[0] = f.sched ? f.sched[0] : f.c_reg;
    sched_s[1] = f.sched ? f.sched[1] : f.rho;
    sched_s[2] = f.sched ? f.sched[2] : f.ts_w;
  }
  __syncthreads();
  const float c_reg = sched_s[0], rho = sched_s[1], ts_w = sched_s[2];
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  const bool on = r < f.rows;
  const float inv2m = 1.0f / (2.0f * (float)f.rows), invm = 1.0f / (float)f.rows;
  float l_surr = 0.0f, l_val = 0.0f, l_reg = 0.0f, l_ent = 0.0f, l_ts = 0.0f;
  float gstd[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) gstd[i] = 0.0f;
  if (on) {
    const int64_t src = f.idx ? f.idx[r] : r;
    const float* mu = mean + (int64_t)r * mean_ld;
    const float* act = f.s_actions + src * f.n_act;
    float lp[2] = {0.0f, 0.0f}, ent[2] = {0.0f, 0.0f};
    for (int i = 0; i < f.n_act; ++i) {
      const float sg = f.std[i];
      const int c = i < f.n_leg ? 0 : 1;
      lp[c] += ppo_logp_term(act[i], mu[i], sg, logf(sg));
      ent[c] += ppo_entropy_term(logf(sg));
    }
    const float2 adv = make_float2(f.adv[2 * src], f.adv[2 * src + 1]);
    float glp[2];
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float ratio = ppo_ratio(lp[c], f.old_logp[2 * src + c]);
      const float2 surr = ppo_surrogate(ppo_mix(adv, c, rho), ratio, f.clip);
      l_surr += surr.x;
      glp[c] = inv2m * surr.y * ratio;
      l_ent += ent[c];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      if (i < f.n_act) {
        const float sg = f.std[i], ai = act[i], mi = mu[i];      // loaded once: the compiler cannot rule out that the stores below alias them
        const int c = i < f.n_leg ? 0 : 1;
        float gmu = ppo_grad_mean(glp[c], ai, mi, sg);
        if (c == 1 && f.ts_target != nullptr) {
          const float2 t = ppo_torque_term(f, src, f.n_act - f.n_leg, i - f.n_leg, mi, ts_w);
          l_ts += t.x;
          gmu += t.y;
        }
        if (c == 0) f.g_leg[(int64_t)r * f.gleg_ld + i] = gmu;
        else f.g_arm[(int64_t)r * f.garm_ld + (i - f.n_leg)] = gmu;
        gstd[i] = ppo_grad_std(glp[c], ai, mi, sg, f.c_ent, inv2m);
      }
    }
    float gv[2];
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float2 t = ppo_value_term(value[2 * r + c], f.old_values[2 * src + c], f.returns[2 * src + c], f.clip, f.clipped_value);
      l_val += t.x;
      gv[c] = t.y * (f.c_value * inv2m);
    }
    f.g_v[(int64_t)r * f.gv_ld] = gv[0];
    f.g_v[(int64_t)r * f.gv_ld + 1] = gv[1];
    // pad columns are read as (zero-weighted) operand columns by the tensor-core backward: keep them finite
    for (int i = 2; i < f.gv_ld; ++i) f.g_v[(int64_t)r * f.gv_ld + i] = 0.0f;
    for (int i = f.n_leg; i < f.gleg_ld; ++i) f.g_leg[(int64_t)r * f.gleg_ld + i] = 0.0f;
    for (int i = f.n_act - f.n_leg; i < f.garm_ld; ++i) f.g_arm[(int64_t)r * f.garm_ld + i] = 0.0f;
    const float* zpr = zp + (int64_t)r * f.gz_ld;
    const float* zhr = f.zh + (f.zh_by_src ? src : (int64_t)r) * f.zh_ld;     // precomputed per storage row, or per mini-batch row
    const float nrm = ppo_reg_norm<0>(zpr, zhr, f.latent);
    l_reg = nrm;
    const float s = ppo_reg_scale(nrm, c_reg, invm);
    for (int i = 0; i < f.latent; ++i)
      f.g_z[(int64_t)r * f.gz_ld + i] = s * (zpr[i] - zhr[i]);
  }
  // warp sums -> this block's slot; the last block adds the slots up in block order
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float v4[5] = {l_surr * inv2m, l_val * inv2m, l_reg * invm, l_ent * inv2m, l_ts * invm / (float)max(f.n_act - f.n_leg, 1)};
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    float s = warp_sum(v4[k]);
    if (lane == 0) red[k][w] = s;
  }
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    if (i < f.n_act) {
      float s = warp_sum(gstd[i]);
      if (lane == 0) red[5 + i][w] = s;
    }
  }
  __syncthreads();
  const int nq = 5 + f.n_act, q = threadIdx.x;
  if (q < nq) f.part[(int64_t)blockIdx.x * LOSS_PART + q] = (red[q][0] + red[q][1]) + (red[q][2] + red[q][3]);
  if (!last_block(ticket) || q >= nq) return;
  float s = 0.0f;
  for (int b = 0; b < (int)gridDim.x; ++b) s += __ldcg(f.part + (int64_t)b * LOSS_PART + q);
  if (q >= 5) f.grad_std[q - 5] += s;
  else if (q < 4 || f.ts_target != nullptr) f.losses[q] += s;
}

// DAgger loss PPO:273-276: mean_rows || sg(zp) - zh ||_2 ; writes d/d zh_pre (the derivative of the activation `act` folded in)
__global__ void __launch_bounds__(128) dagger_loss_kernel(const float* __restrict__ zp, const float* __restrict__ zh, int zld, int latent,
                                                          float* __restrict__ g, float* __restrict__ loss, float* part, unsigned* ticket, int rows,
                                                          int act) {
  __shared__ float red[4];
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  float l = 0.0f;
  if (r < rows) {
    const float nrm = ppo_reg_norm<0>(zp + (int64_t)r * zld, zh + (int64_t)r * zld, latent);
    l = nrm / (float)rows;
    const float s = nrm > 0.0f ? 1.0f / ((float)rows * nrm) : 0.0f;
    for (int i = 0; i < latent; ++i) {
      const float y = zh[(int64_t)r * zld + i];
      g[(int64_t)r * zld + i] = -s * (zp[(int64_t)r * zld + i] - y) * act_df(act, y);
    }
  }
  float s = warp_sum(l);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) part[blockIdx.x] = (red[0] + red[1]) + (red[2] + red[3]);      // this block's slot; the last block sums in order
  if (!last_block(ticket) || threadIdx.x != 0) return;
  float t = 0.0f;
  for (int b = 0; b < (int)gridDim.x; ++b) t += __ldcg(part + b);
  *loss += t;
}

// ---- PPO update diagnostics (dwbc_ppo_minibatch_grad_diag) ----------------------------------------
// Per channel c (leg = actions [0, n_leg), arm = the rest), over the M rows of a mini-batch:
//   approx_kl[c]     = mean_rows sum_i log(sg_new / sg_old + 1e-5) + (sg_old^2 + (mu_old - mu_new)^2) / (2 sg_new^2) - 0.5  (rsl_rl's KL)
//   clip_fraction[c] = share of rows whose ratio lies outside [1 - clip, 1 + clip]
// The ratio is the loss's: ppo_logp_term summed in index order over the same new means, std and stored rows, and the loss's ratio and
// clip-range test (ppo_terms.cuh).  The KL terms are evaluated and summed in double.  One partial per 128-row block, added up in block order
// by the last block.
static_assert(DWBC_DIAG_KL_ARM == DWBC_DIAG_KL_LEG + 1 && DWBC_DIAG_CLIP_LEG == DWBC_DIAG_KL_LEG + 2 && DWBC_DIAG_CLIP_ARM == DWBC_DIAG_KL_LEG + 3,
              "ppo_diag_kernel writes its four means to consecutive slots");
struct DiagArgs {
  const float* mean; int mean_ld;         // new means [rows, mean_ld] (the forward's)
  const float* std;                       // new sigma: the std parameters the forward used
  const float* actions; const float* old_logp; const float* old_mu; const float* old_sigma; const int64_t* idx;
  float* out;                             // [DWBC_DIAG_KL_LEG .. DWBC_DIAG_CLIP_ARM] are written
  double* part; unsigned* ticket;         // [blocks][4] partials
  int rows, n_leg, n_act;
  float clip;
};

__global__ void __launch_bounds__(128) ppo_diag_kernel(const DiagArgs a) {
  __shared__ double red[4][4];
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  double v[4] = {0.0, 0.0, 0.0, 0.0};                                            // kl leg, kl arm, outside leg, outside arm
  if (r < a.rows) {
    const int64_t src = a.idx ? a.idx[r] : r;
    const float* mu = a.mean + (int64_t)r * a.mean_ld;
    const float* act = a.actions + src * a.n_act;
    const float* omu = a.old_mu + src * a.n_act;
    const float* osg = a.old_sigma + src * a.n_act;
    float lp[2] = {0.0f, 0.0f};
    for (int i = 0; i < a.n_act; ++i) {
      const float sg = a.std[i];
      const int c = i < a.n_leg ? 0 : 1;
      lp[c] += ppo_logp_term(act[i], mu[i], sg, logf(sg));
      const double sn = sg, so = osg[i], dm = (double)omu[i] - (double)mu[i];
      v[c] += log(sn / so + 1e-5) + (so * so + dm * dm) / (2.0 * sn * sn) - 0.5;
    }
#pragma unroll
    for (int c = 0; c < 2; ++c) v[2 + c] = ppo_inside(ppo_ratio(lp[c], a.old_logp[2 * src + c]), a.clip) ? 0.0 : 1.0;
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double s = warp_sum(v[k]);
    if (lane == 0) red[k][w] = s;
  }
  __syncthreads();
  const int q = threadIdx.x;
  if (q < 4) a.part[(int64_t)blockIdx.x * 4 + q] = (red[q][0] + red[q][1]) + (red[q][2] + red[q][3]);
  if (!last_block(a.ticket) || q >= 4) return;
  double s = 0.0;
  for (int b = 0; b < (int)gridDim.x; ++b) s += __ldcg(a.part + (int64_t)b * 4 + q);
  a.out[DWBC_DIAG_KL_LEG + q] = (float)(s / (double)a.rows);
}

// ---- backward -----------------------------------------------------------------------------------
// Backward of one head: Linear(+ELU) x nl, then Linear -> out.  G_out = d/d(pre-activation of the
// last layer) [rows, n_out].  Accumulates weight grads into `grad`, and adds the head's
// contribution to d(backbone output) into dtrunk (beta_trunk; ELU' of the trunk applied if apply_dact).
static int head_backward(const float* P, float* grad, RowMat G_out, int n_out, int nl, const int32_t* dims, const int64_t* ow,
                         const int64_t* ob, float* const* acts, RowMat trunk, int trunk_dim, float* dtrunk, int beta_trunk,
                         int apply_dact, float* dA, float* dB, int rows, cudaStream_t st) {
  RowMat G = G_out;
  int gout = n_out;
  for (int l = nl; l >= 0; --l) {
    const int in = l == 0 ? trunk_dim : dims[l - 1];
    RowMat X = l == 0 ? trunk : rowmat(acts[l - 1], dims[l - 1]);
    TRY(linear_bwd_weight(G, X, grad + ow[l], in, grad + ob[l], rows, gout, in, st));
    if (l == 0) {
      TRY(linear_bwd_data(G, P + ow[l], in, dtrunk, trunk_dim, rows, in, gout, apply_dact ? mlp_act : ACT_NONE, trunk, beta_trunk, st));
    } else {
      float* d = (l & 1) ? dA : dB;
      TRY(linear_bwd_data(G, P + ow[l], in, d, in, rows, in, gout, mlp_act, X, 0, st));
      G = rowmat(d, in);
      gout = in;
    }
  }
  return DWBC_OK;
}

// ---- fused backward (tensor-core paths): all data-gradient GEMMs of the actor + privileged encoder and of the critic as two
// programs of one launch (mlp_chain2.cuh, backward ops); the per-layer pre-activation gradients they leave behind feed the
// weight-gradient GEMMs (wgrad_group.cuh, MN-major operands).
struct HeadDesc { int nl; const int32_t* dims; const int64_t* ow; const int64_t* ob; float* const* acts; float* const* dz; RowMat g_out; int n_out; };

// data-gradient ops of one head, last layer first.  The head's loss gradient [rows, g_ld] is loaded into tile columns [0, g_ld) right
// before its first op; column g_col + j of that window multiplies row j of the last layer's weights.  The trunk gradient of the
// FIRST head goes to `scratch` unactivated; the second head adds it and applies the trunk's ELU'.
static void chain_head_bwd(C2Builder& b, const float* P, const HeadDesc& hd, const float* g, int g_ld, int g_col, int trunk_dim, const float* trunk,
                           bool second, float* scratch, float* dz_trunk) {
  b.load(rowmat(g, g_ld), g_ld, 0, pad8(g_ld), b.pr.n_ops);
  for (int l = hd.nl; l >= 0; --l) {
    const int in = l == 0 ? trunk_dim : hd.dims[l - 1];
    const int out = l == hd.nl ? hd.n_out : hd.dims[l];
    const bool narrow = l == hd.nl;
    const int kpad = narrow ? pad8(g_ld) : pad8(out);
    const C2PackSeg seg{narrow ? g_col : 0, 0, out};
    if (l > 0)
      b.bwd(P + hd.ow[l], in, in, 0, kpad, seg, mlp_act, hd.acts[l - 1], in, nullptr, 0, 0, hd.dz[l - 1], in, img_dim(in), img_dim(in));
    else if (!second)
      b.bwd(P + hd.ow[0], in, in, 0, kpad, seg, ACT_NONE, nullptr, 0, nullptr, 0, -1, scratch, trunk_dim);
    else
      b.bwd(P + hd.ow[0], in, in, 0, kpad, seg, mlp_act, trunk, trunk_dim, scratch, trunk_dim, 0, dz_trunk, trunk_dim, img_dim(trunk_dim), img_dim(trunk_dim));
  }
}

static void head_wgrad(WGroupBuilder& wb, float* grad, const HeadDesc& hd, RowMat trunk, int trunk_dim) {
  for (int l = hd.nl; l >= 0; --l) {
    const int in = l == 0 ? trunk_dim : hd.dims[l - 1];
    RowMat G = l == hd.nl ? hd.g_out : act_mat(hd.dz[l], hd.dims[l]);
    const int gout = l == hd.nl ? hd.n_out : hd.dims[l];
    RowMat X = l == 0 ? trunk : act_mat(hd.acts[l - 1], hd.dims[l - 1]);
    wb.add(G, X, grad + hd.ow[l], in, grad + hd.ob[l], gout, in);
  }
}

struct BwdDescs { HeadDesc cl, ca, al, aa; };
static BwdDescs bwd_descs(const DwbcNetCfg& n, const Plan& p) {
  const int gleg_ld = (int)align_up(n.n_leg, 4), garm_ld = (int)align_up(n.n_arm, 4);
  BwdDescs d;
  d.cl = HeadDesc{n.n_leg_layers, n.leg_dims, n.off_cleg_w, n.off_cleg_b, p.cl, p.dzc_l, rowmat(p.g_vl, 4), 1};
  d.ca = HeadDesc{n.n_arm_layers, n.arm_dims, n.off_carm_w, n.off_carm_b, p.ca, p.dzc_a, rowmat(p.g_va, 4), 1};
  d.al = HeadDesc{n.n_leg_layers, n.leg_dims, n.off_aleg_w, n.off_aleg_b, p.al, p.dza_l, rowmat(p.g_leg, gleg_ld), n.n_leg};
  d.aa = HeadDesc{n.n_arm_layers, n.arm_dims, n.off_aarm_w, n.off_aarm_b, p.aa, p.dza_a, rowmat(p.g_arm, garm_ld), n.n_arm};
  return d;
}

static int build_backward(const DwbcNetCfg& n, const float* P, const Plan& p, C2Builder& A, C2Builder& C) {
  const int Lld = (int)align_up(p.latent, 4);
  const int gleg_ld = (int)align_up(n.n_leg, 4), garm_ld = (int)align_up(n.n_arm, 4);
  const BwdDescs d = bwd_descs(n, p);
  // ---- critic: both value heads read their column of the [rows, 4] value-gradient buffer ----
  const int cnb = n.n_critic_layers, ctd = n.critic_dims[cnb - 1];
  chain_head_bwd(C, P, d.cl, p.g_vl, 4, 0, ctd, p.cb[cnb - 1], false, p.d1, nullptr);
  chain_head_bwd(C, P, d.ca, p.g_vl, 4, 1, ctd, p.cb[cnb - 1], true, p.d1, p.dzc_b[cnb - 1]);
  for (int l = cnb - 1; l >= 1; --l)
    C.bwd(P + n.off_critic_w[l], n.critic_dims[l - 1], n.critic_dims[l - 1], 0, pad8(n.critic_dims[l]), C2PackSeg{0, 0, n.critic_dims[l]}, mlp_act,
          p.cb[l - 1], n.critic_dims[l - 1], nullptr, 0, 0, p.dzc_b[l - 1], n.critic_dims[l - 1], img_dim(n.critic_dims[l - 1]), img_dim(n.critic_dims[l - 1]));
  C.finish();
  // ---- actor + privileged encoder ----
  const int anb = n.n_actor_layers, atd = n.actor_dims[anb - 1];
  chain_head_bwd(A, P, d.al, p.g_leg, gleg_ld, 0, atd, p.ab[anb - 1], false, p.d0, nullptr);
  chain_head_bwd(A, P, d.aa, p.g_arm, garm_ld, 0, atd, p.ab[anb - 1], true, p.d0, p.dza_b[anb - 1]);
  for (int l = anb - 1; l >= 1; --l)
    A.bwd(P + n.off_actor_w[l], n.actor_dims[l - 1], n.actor_dims[l - 1], 0, pad8(n.actor_dims[l]), C2PackSeg{0, 0, n.actor_dims[l]}, mlp_act,
          p.ab[l - 1], n.actor_dims[l - 1], nullptr, 0, 0, p.dza_b[l - 1], n.actor_dims[l - 1], img_dim(n.actor_dims[l - 1]), img_dim(n.actor_dims[l - 1]));
  const int in0 = n.num_prop + p.latent, np = n.n_priv_layers;
  float* z = p.priv[np - 1];
  // dL/dz = policy path through the latent columns of backbone layer 0 + privileged-latent regulariser (g_z), through the encoder's last ELU
  A.bwd(P + n.off_actor_w[0] + n.num_prop, in0, p.latent, 0, pad8(n.actor_dims[0]), C2PackSeg{0, 0, n.actor_dims[0]}, mlp_act, z, Lld, p.g_z, Lld, 0,
        p.dzp[np - 1], Lld);
  for (int l = np - 1; l >= 1; --l) {
    const int in = n.priv_dims[l - 1], ldin = (int)align_up(in, 4);
    A.bwd(P + n.off_priv_w[l], in, in, 0, pad8(n.priv_dims[l]), C2PackSeg{0, 0, n.priv_dims[l]}, mlp_act, p.priv[l - 1], ldin, nullptr, 0, l - 1 > 0 ? 0 : -1,
          p.dzp[l - 1], ldin);
  }
  A.finish();
  if (!C.ok || !A.ok) return DWBC_ERR_UNSUPPORTED;
  return DWBC_OK;
}

// The chain programs of one entry point and the pack list of their weight images.  b[] = {A, C, A2, C2} for dwbc_policy_act, {C, C2} for
// dwbc_critic_values, {A, C, Ab, Cb} (forward + loss, backward) for dwbc_ppo_minibatch_grad.  The builders point at pl / off: never copied.
struct C2Chains {
  C2PackList pl{};
  int64_t off = 0;
  C2Builder b[4];
  int nprog = 0;
  C2Chains(float* wpack, int rows, bool x3)
      : b{C2Builder(&pl, &off, rows, x3), C2Builder(&pl, &off, rows, x3), C2Builder(&pl, &off, rows, x3), C2Builder(&pl, &off, rows, x3)} {
    pl.out = wpack;
  }
  C2Chains(const C2Chains&) = delete;
  C2Chains& operator=(const C2Chains&) = delete;
};

// THE decision between the fused chains and the layer-wise path, for every entry point: builds all programs the call would launch (host
// code only: nothing is packed or launched) and returns true when the network fits the tile layout (chain_usable) AND every builder
// accepted its ops and loads AND the weight images of all programs fit one pack list (C2_MAX_OPS, C2_MAX_LOADS, C2_MAX_PACK,
// C2_PACK_FLOATS).  A network that passes chain_usable can still fail the latter (e.g. three 128-wide backbone layers per network: 38
// images in the update); it then runs layer-wise like any network with a layer wider than 128.
// what: 0 = dwbc_policy_act (`hist`: the latent comes from the history encoder, in p.zh), 1 = dwbc_critic_values, 2 =
// dwbc_ppo_minibatch_grad (`idx`: its gather index), 3 = dwbc_policy_mean (the actor programs of 0 alone, `hist` as there).  `sms`: the SM
// count the rollout's split into one program per head follows.
static bool plan_chains(C2Chains& c, int what, const DwbcNetCfg& n, const float* P, const float* obs, const int64_t* idx, int64_t obs_stride,
                        bool hist, float* values, const Plan& p, int rows, int sms, bool keep_mean = false) {
  if (!chain_usable(n, p, obs, obs_stride)) return false;
  const int tiles = (rows + TC_M - 1) / TC_M, zld = (int)align_up(p.latent, 4);
  C2Builder* B = c.b;
  int rc;
  if (what == 0) {
    const bool split = 4 * tiles <= sms;       // few tiles (the rollout): one program per HEAD, four short programs spread over 4 x tiles SMs
    rc = build_forward(n, P, obs, nullptr, obs_stride, hist ? p.zh : nullptr, zld, p, values, false, 1, &B[0], &B[1], split ? &B[2] : nullptr,
                       split ? &B[3] : nullptr);
    c.nprog = split ? 4 : 2;
  } else if (what == 1) {
    const bool split = 2 * tiles <= sms;
    rc = build_forward(n, P, obs, nullptr, obs_stride, nullptr, 0, p, values, false, 0, nullptr, &B[0], nullptr, split ? &B[1] : nullptr);
    c.nprog = split ? 2 : 1;
  } else if (what == 3) {
    // Every op of these programs is an op of mode 0's actor programs with the same operands; each program owns whole row tiles, and a
    // trunk stored to p.ab and reloaded for the second head is the fp32 value the split program keeps in its tile.  So the means do not
    // depend on where the two modes split (4 * tiles vs 2 * tiles <= sms).
    const bool split = 2 * tiles <= sms;
    rc = build_forward(n, P, obs, nullptr, obs_stride, hist ? p.zh : nullptr, zld, p, values, false, 1, &B[0], nullptr, split ? &B[1] : nullptr);
    c.nprog = split ? 2 : 1;
  } else {
    rc = build_forward(n, P, obs, idx, obs_stride, nullptr, zld, p, values, true, 2, &B[0], &B[1], nullptr, nullptr, keep_mean);
    if (rc == DWBC_OK) rc = build_backward(n, P, p, B[2], B[3]);
    c.nprog = 2;
  }
  return rc == DWBC_OK && c.off <= C2_PACK_FLOATS;
}

// every layer's weight gradient of both networks in one persistent launch (wgrad_group.cuh)
static bool wgrad_gemms(WGroupBuilder& wb, const DwbcNetCfg& n, float* grad, const DwbcStorage* s, const int64_t* idx, const Plan& p) {
  const int Lld = (int)align_up(p.latent, 4);
  const BwdDescs d = bwd_descs(n, p);
  const int cnb = n.n_critic_layers, ctd = n.critic_dims[cnb - 1];
  const int anb = n.n_actor_layers, atd = n.actor_dims[anb - 1];
  const int in0 = n.num_prop + p.latent, np = n.n_priv_layers;
  float* z = p.priv[np - 1];
  RowMat obs_all = rowmat_gather(s->observations, idx, s->obs_stride);
  head_wgrad(wb, grad, d.cl, act_mat(p.cb[cnb - 1], ctd), ctd);
  head_wgrad(wb, grad, d.ca, act_mat(p.cb[cnb - 1], ctd), ctd);
  for (int l = cnb - 1; l >= 0; --l) {
    const int in = l == 0 ? n.num_prop + n.num_priv : n.critic_dims[l - 1];
    wb.add(act_mat(p.dzc_b[l], n.critic_dims[l]), l == 0 ? obs_all : act_mat(p.cb[l - 1], in), grad + n.off_critic_w[l], in, grad + n.off_critic_b[l],
           n.critic_dims[l], in);
  }
  head_wgrad(wb, grad, d.al, act_mat(p.ab[anb - 1], atd), atd);
  head_wgrad(wb, grad, d.aa, act_mat(p.ab[anb - 1], atd), atd);
  for (int l = anb - 1; l >= 1; --l)
    wb.add(act_mat(p.dza_b[l], n.actor_dims[l]), act_mat(p.ab[l - 1], n.actor_dims[l - 1]), grad + n.off_actor_w[l], n.actor_dims[l - 1],
           grad + n.off_actor_b[l], n.actor_dims[l], n.actor_dims[l - 1]);
  RowMat G0 = act_mat(p.dza_b[0], n.actor_dims[0]);
  wb.add(G0, obs_all, grad + n.off_actor_w[0], in0, grad + n.off_actor_b[0], n.actor_dims[0], n.num_prop);
  wb.add(G0, rowmat(z, Lld), grad + n.off_actor_w[0] + n.num_prop, in0, nullptr, n.actor_dims[0], p.latent);
  for (int l = np - 1; l >= 0; --l) {
    const int in = l == 0 ? n.num_priv : n.priv_dims[l - 1];
    RowMat X = l == 0 ? rowmat_gather(s->observations + n.num_prop, idx, s->obs_stride) : rowmat(p.priv[l - 1], (int)align_up(in, 4));
    wb.add(rowmat(p.dzp[l], (int)align_up(n.priv_dims[l], 4)), X, grad + n.off_priv_w[l], in, grad + n.off_priv_b[l], n.priv_dims[l], in);
  }
  return wb.ok;
}
static int weight_gradients(const DwbcNetCfg& n, float* grad, const DwbcStorage* s, const int64_t* idx, int rows, const Plan& p, cudaStream_t st) {
  WGroupBuilder wb;
  if (!wgrad_gemms(wb, n, grad, s, idx, p)) return DWBC_ERR_UNSUPPORTED;
  return launch_wgrad_group(wb.g, rows, mlp_precision == 2, st);
}

}  // namespace dwbc

using namespace dwbc;

extern "C" int64_t dwbc_workspace_bytes(const DwbcNetCfg* net, int64_t rows) {
  if (check_net(net) != DWBC_OK || rows <= 0) return -1;
  return make_plan(*net, rows, nullptr).bytes;
}

// FinArgs of the rollout hooks and of act_finalize_kernel
static FinArgs fin_rollout(const DwbcNetCfg& n, const float* P, const float* eps, float* actions, float* log_prob, float* mean, float* sigma, int rows) {
  FinArgs f{};
  f.std = P + n.off_std; f.eps = eps; f.actions = actions; f.log_prob = log_prob; f.mean_out = mean; f.sigma_out = sigma;
  f.n_leg = n.n_leg; f.n_act = n.n_leg + n.n_arm; f.rows = rows;
  return f;
}

// FinArgs of the update: the hooks of the forward chains and ppo_loss_kernel.  The loss gradients go to the workspace (g_v: [rows, 4],
// the two value columns, then padding), the privileged latent's at the padded latent stride.
static FinArgs fin_update(const DwbcNetCfg& n, const float* P, const DwbcStorage* s, const int64_t* idx, const DwbcPpoHyper* hp, const float* sched,
                          const Plan& p, float* grad, float* losses, int rows) {
  const int Lld = (int)align_up(p.latent, 4);
  FinArgs f{};
  f.std = P + n.off_std; f.idx = idx; f.s_actions = s->actions; f.old_logp = s->log_prob; f.old_values = s->values; f.returns = s->returns;
  f.adv = s->advantages;
  f.zh = s->hist_latent ? s->hist_latent : p.zh; f.zh_ld = s->hist_latent ? s->hist_latent_ld : Lld; f.zh_by_src = s->hist_latent ? 1 : 0;
  f.g_leg = p.g_leg; f.gleg_ld = (int)align_up(n.n_leg, 4); f.g_arm = p.g_arm; f.garm_ld = (int)align_up(n.n_arm, 4);
  f.g_v = p.g_vl; f.gv_ld = 4; f.g_z = p.g_z; f.gz_ld = Lld;
  f.grad_std = grad + n.off_std; f.losses = losses; f.part = p.loss_part;
  f.n_leg = n.n_leg; f.n_act = n.n_leg + n.n_arm; f.latent = p.latent; f.rows = rows;
  f.clip = hp->clip_param; f.c_value = hp->value_loss_coef; f.c_ent = hp->entropy_coef; f.c_reg = hp->priv_reg_coef; f.rho = hp->mixing_ratio;
  f.clipped_value = hp->use_clipped_value_loss;
  f.ts_target = s->target_arm_torques; f.ts_pos = s->current_arm_dof_pos; f.ts_vel = s->current_arm_dof_vel; f.ts_coef = hp->arm_coefs;
  f.ts_w = hp->torque_supervision_weight; f.sched = sched;
  return f;
}

extern "C" int dwbc_policy_act(const DwbcNetCfg* net, const float* params, const float* obs, int64_t obs_stride, const float* eps,
                               int32_t hist_encoding, float* actions, float* values, float* log_prob, float* mean, float* sigma,
                               int32_t rows, int32_t weights_packed, void* workspace, dwbc_stream_t stream) {
  TRY(check_net(net));
  if (!params || !obs || !eps || !actions || !values || !log_prob || !mean || !sigma || !workspace || rows <= 0) return DWBC_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const DwbcNetCfg& n = *net;
  Plan p = make_plan(n, rows, workspace);
  const float* z;
  int zld = (int)align_up(p.latent, 4);
  const bool x3 = mlp_precision == 2;
  C2Chains ch(p.wpack, rows, x3);
  if (plan_chains(ch, 0, n, params, obs, nullptr, obs_stride, hist_encoding != 0, values, p, rows, c2_sm_count())) {
    if (hist_encoding) TRY(hist_latent_only(n, params, obs, nullptr, obs_stride, rows, p, p.zh, zld, st));
    if (!weights_packed) TRY(launch_pack2(ch.pl, st));       // the images stay valid in the workspace until the parameters change
    const C2Prog* prs[4] = {&ch.b[0].pr, &ch.b[1].pr, &ch.b[2].pr, &ch.b[3].pr};
    return launch_chain2n(prs, ch.nprog, fin_rollout(n, params, eps, actions, log_prob, mean, sigma, rows), x3, p.queue, st);
  }
  if (hist_encoding) {
    TRY(hist_forward(n, params, obs, nullptr, obs_stride, rows, p, st));
    z = p.zh;
  } else {
    TRY(priv_forward(n, params, obs, nullptr, obs_stride, rows, p, st));
    z = p.priv[n.n_priv_layers - 1];
  }
  TRY(actor_forward(n, params, obs, nullptr, obs_stride, rows, z, zld, p, st));
  TRY(critic_forward(n, params, obs, nullptr, obs_stride, rows, p, values, st));
  act_finalize_kernel<<<(rows + 127) / 128, 128, 0, st>>>(fin_rollout(n, params, eps, actions, log_prob, mean, sigma, rows), p.mean, p.mean_ld);
  DWBC_LAUNCH_CHECK();
  return DWBC_OK;
}

// The actor half of dwbc_policy_act: the same ops on the same operands, without the critic programs and the sampling epilogue.  It takes
// the chains exactly when dwbc_policy_act would (mode 0 is planned first: a network whose rollout programs overflow the pack list runs
// layer-wise there, so it must here too), which keeps `mean` bitwise equal to dwbc_policy_act's.
extern "C" int dwbc_policy_mean(const DwbcNetCfg* net, const float* params, const float* obs, int64_t obs_stride, int32_t hist_encoding,
                                float* mean, int32_t rows, int32_t weights_packed, void* workspace, dwbc_stream_t stream) {
  TRY(check_net(net));
  if (!params || !obs || !mean || !workspace || rows <= 0) return DWBC_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const DwbcNetCfg& n = *net;
  Plan p = make_plan(n, rows, workspace);
  const int zld = (int)align_up(p.latent, 4), n_act = n.n_leg + n.n_arm;
  const bool x3 = mlp_precision == 2;
  const int sms = c2_sm_count();
  bool chains;
  {
    C2Chains act(p.wpack, rows, x3);
    chains = plan_chains(act, 0, n, params, obs, nullptr, obs_stride, hist_encoding != 0, p.value, p, rows, sms);
  }
  C2Chains ch(p.wpack, rows, x3);
  if (chains && plan_chains(ch, 3, n, params, obs, nullptr, obs_stride, hist_encoding != 0, p.value, p, rows, sms)) {
    if (hist_encoding) TRY(hist_latent_only(n, params, obs, nullptr, obs_stride, rows, p, p.zh, zld, st));
    if (!weights_packed) TRY(launch_pack2(ch.pl, st));
    const C2Prog* prs[2] = {&ch.b[0].pr, &ch.b[1].pr};
    FinArgs f{};
    f.mean_out = mean; f.n_leg = n.n_leg; f.n_act = n_act; f.rows = rows;
    return launch_chain2n(prs, ch.nprog, f, x3, p.queue, st);
  }
  if (chains) return DWBC_ERR_UNSUPPORTED;          // (cannot happen: the actor programs are a subset of mode 0's; see plan_chains)
  if (hist_encoding) TRY(hist_forward(n, params, obs, nullptr, obs_stride, rows, p, st));
  else TRY(priv_forward(n, params, obs, nullptr, obs_stride, rows, p, st));
  TRY(actor_forward(n, params, obs, nullptr, obs_stride, rows, hist_encoding ? p.zh : p.priv[n.n_priv_layers - 1], zld, p, st));
  if (cudaMemcpy2DAsync(mean, sizeof(float) * n_act, p.mean, sizeof(float) * p.mean_ld, sizeof(float) * n_act, rows, cudaMemcpyDeviceToDevice, st) !=
      cudaSuccess)
    return DWBC_ERR_LAUNCH;
  return DWBC_OK;
}

extern "C" int dwbc_critic_values(const DwbcNetCfg* net, const float* params, const float* obs, int64_t obs_stride, float* values,
                                  int32_t rows, void* workspace, dwbc_stream_t stream) {
  TRY(check_net(net));
  if (!params || !obs || !values || !workspace || rows <= 0) return DWBC_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  Plan p = make_plan(*net, rows, workspace);
  const bool x3 = mlp_precision == 2;
  C2Chains ch(p.wpack, rows, x3);
  if (plan_chains(ch, 1, *net, params, obs, nullptr, obs_stride, false, values, p, rows, c2_sm_count())) {
    TRY(launch_pack2(ch.pl, st));                           // (overwrites the images a previous dwbc_policy_act left behind)
    const C2Prog* prs[2] = {&ch.b[0].pr, &ch.b[1].pr};
    return launch_chain2n(prs, ch.nprog, FinArgs{}, x3, p.queue, st);
  }
  return critic_forward(*net, params, obs, nullptr, obs_stride, rows, p, values, st);
}

extern "C" int dwbc_hist_latent(const DwbcNetCfg* net, const float* params, const float* obs, int64_t obs_stride, float* out, int64_t ld_out,
                                int32_t rows, void* workspace, dwbc_stream_t stream) {
  TRY(check_net(net));
  if (!params || !obs || !out || !workspace || rows <= 0) return DWBC_ERR_ARG;
  Plan p = make_plan(*net, rows, workspace);
  if (ld_out != align_up(p.latent, 4)) return DWBC_ERR_ARG;
  return hist_latent_only(*net, params, obs, nullptr, obs_stride, rows, p, out, ld_out, (cudaStream_t)stream);
}

// sched: optional device (priv_reg_coef, mixing_ratio, torque_supervision_weight) read by the loss kernels in place of hp's fields.
// diag_out: optional (dwbc_ppo_minibatch_grad_diag): the forward also keeps the new means, and ppo_diag_kernel runs behind the loss.
static int ppo_minibatch_grad(const DwbcNetCfg* net, const float* params, const DwbcStorage* s, const int64_t* idx, int32_t M,
                              const DwbcPpoHyper* hp, const float* sched, const float* old_mu, const float* old_sigma, float* grad,
                              float* losses_out, float* diag_out, void* workspace, dwbc_stream_t stream) {
  TRY(check_net(net));
  if (!params || !s || !idx || !hp || !grad || !losses_out || !workspace || M <= 0) return DWBC_ERR_ARG;
  if (diag_out && (!old_mu || !old_sigma)) return DWBC_ERR_ARG;
  if (!s->observations || !s->actions || !s->values || !s->returns || !s->advantages || !s->log_prob) return DWBC_ERR_ARG;
  // torque supervision is on when the storage carries its three tensors (RS:82-84); then the arm coefficients are needed too
  if (s->target_arm_torques && (!s->current_arm_dof_pos || !s->current_arm_dof_vel || !hp->arm_coefs)) return DWBC_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const DwbcNetCfg& n = *net;
  const float* P = params;
  const int rows = M;
  Plan p = make_plan(n, rows, workspace);
  const int Lld = (int)align_up(p.latent, 4);
  // tensor-core path: forward chains with the loss in the heads' epilogues, backward chains, grouped weight gradients.  The weight images
  // of all four programs are packed by ONE launch (the parameters are constant within a mini-batch).
  const bool x3 = mlp_precision == 2;
  C2Chains ch(p.wpack, rows, x3);
  const bool chains = plan_chains(ch, 2, n, P, s->observations, idx, s->obs_stride, false, p.value, p, rows, 0, diag_out != nullptr);
  if (diag_out && !chains) {
    // the diagnostics must never move an update off the chains (other rounding, other speed): refuse rather than fall back
    C2Chains plain(p.wpack, rows, x3);
    if (plan_chains(plain, 2, n, P, s->observations, idx, s->obs_stride, false, p.value, p, rows, 0)) return DWBC_ERR_UNSUPPORTED;
  }
  if (cudaMemsetAsync(grad, 0, sizeof(float) * n.num_params, st) != cudaSuccess) return DWBC_ERR_LAUNCH;
  // the diagnostics of this mini-batch over the forward's means, which both paths leave in Plan::mean (the chains only when asked to: the
  // heads' last ops then write their outputs there at row stride n_act, the layer-wise forward at mean_ld)
  auto diag = [&](int mean_ld) -> int {
    if (!diag_out) return DWBC_OK;
    DiagArgs d{};
    d.mean = p.mean; d.mean_ld = mean_ld; d.std = P + n.off_std;
    d.actions = s->actions; d.old_logp = s->log_prob; d.old_mu = old_mu; d.old_sigma = old_sigma; d.idx = idx;
    d.out = diag_out; d.part = reinterpret_cast<double*>(p.loss_part); d.ticket = reinterpret_cast<unsigned*>(p.queue + 4);
    d.rows = rows; d.n_leg = n.n_leg; d.n_act = n.n_leg + n.n_arm; d.clip = hp->clip_param;
    ppo_diag_kernel<<<(rows + 127) / 128, 128, 0, st>>>(d);
    DWBC_LAUNCH_CHECK();
    return DWBC_OK;
  };

  // forward (the reference evaluates the actor 3x and the priv encoder 3x per mini-batch,
  // PPO:166,174,230; identical values, so each is evaluated once here)
  float* z = p.priv[n.n_priv_layers - 1];
  if (!s->hist_latent) TRY(hist_latent_only(n, P, s->observations, idx, s->obs_stride, rows, p, p.zh, Lld, st));           // PPO:175-176 (no grad)
  const FinArgs f = fin_update(n, P, s, idx, hp, sched, p, grad, losses_out, rows);
  if (chains) {
    TRY(launch_pack2(ch.pl, st));
    TRY(launch_chain2(&ch.b[0].pr, &ch.b[1].pr, f, x3, p.queue, st));
    TRY(diag(n.n_leg + n.n_arm));
    TRY(launch_chain2(&ch.b[2].pr, &ch.b[3].pr, FinArgs{}, x3, p.queue, st, true));      // downwards: the last tiles are still in L2
    return weight_gradients(n, grad, s, idx, rows, p, st);
  }
  TRY(priv_forward(n, P, s->observations, idx, s->obs_stride, rows, p, st));
  TRY(actor_forward(n, P, s->observations, idx, s->obs_stride, rows, z, Lld, p, st));
  TRY(critic_forward(n, P, s->observations, idx, s->obs_stride, rows, p, p.value, st));

  ppo_loss_kernel<<<(rows + 127) / 128, 128, 0, st>>>(f, p.mean, p.mean_ld, p.value, z, reinterpret_cast<unsigned*>(p.queue + 2));
  DWBC_LAUNCH_CHECK();
  TRY(diag(p.mean_ld));

  // ---- critic backward ----
  {
    const int nb = n.n_critic_layers, tdim = n.critic_dims[nb - 1];
    RowMat trunk = rowmat(p.cb[nb - 1], tdim);
    TRY(head_backward(P, grad, rowmat(p.g_vl, 4), 1, n.n_leg_layers, n.leg_dims, n.off_cleg_w, n.off_cleg_b, p.cl, trunk, tdim, p.d2, 0, 0,
                      p.d0, p.d1, rows, st));
    TRY(head_backward(P, grad, rowmat(p.g_va, 4), 1, n.n_arm_layers, n.arm_dims, n.off_carm_w, n.off_carm_b, p.ca, trunk, tdim, p.d2, 1, 1,
                      p.d0, p.d1, rows, st));
    RowMat G = rowmat(p.d2, tdim);
    int gout = tdim;
    for (int l = nb - 1; l >= 0; --l) {
      const int in = l == 0 ? n.num_prop + n.num_priv : n.critic_dims[l - 1];
      RowMat X = l == 0 ? rowmat_gather(s->observations, idx, s->obs_stride) : rowmat(p.cb[l - 1], in);
      TRY(linear_bwd_weight(G, X, grad + n.off_critic_w[l], in, grad + n.off_critic_b[l], rows, gout, in, st));
      if (l > 0) {
        float* d = (l & 1) ? p.d0 : p.d1;
        TRY(linear_bwd_data(G, P + n.off_critic_w[l], in, d, in, rows, in, gout, mlp_act, X, 0, st));
        G = rowmat(d, in);
        gout = in;
      }
    }
  }
  // ---- actor backward ----
  {
    const int nb = n.n_actor_layers, tdim = n.actor_dims[nb - 1];
    RowMat trunk = rowmat(p.ab[nb - 1], tdim);
    TRY(head_backward(P, grad, rowmat(p.g_leg, f.gleg_ld), n.n_leg, n.n_leg_layers, n.leg_dims, n.off_aleg_w, n.off_aleg_b, p.al, trunk, tdim,
                      p.d2, 0, 0, p.d0, p.d1, rows, st));
    TRY(head_backward(P, grad, rowmat(p.g_arm, f.garm_ld), n.n_arm, n.n_arm_layers, n.arm_dims, n.off_aarm_w, n.off_aarm_b, p.aa, trunk, tdim,
                      p.d2, 1, 1, p.d0, p.d1, rows, st));
    RowMat G = rowmat(p.d2, tdim);
    int gout = tdim;
    for (int l = nb - 1; l >= 1; --l) {
      const int in = n.actor_dims[l - 1];
      RowMat X = rowmat(p.ab[l - 1], in);
      TRY(linear_bwd_weight(G, X, grad + n.off_actor_w[l], in, grad + n.off_actor_b[l], rows, gout, in, st));
      float* d = (l & 1) ? p.d0 : p.d1;
      TRY(linear_bwd_data(G, P + n.off_actor_w[l], in, d, in, rows, in, gout, mlp_act, X, 0, st));
      G = rowmat(d, in);
      gout = in;
    }
    // backbone layer 0: input = cat([obs_prop, z])
    const int in0 = n.num_prop + p.latent;
    TRY(linear_bwd_weight(G, rowmat_gather(s->observations, idx, s->obs_stride), grad + n.off_actor_w[0], in0, grad + n.off_actor_b[0], rows,
                          gout, n.num_prop, st));
    TRY(linear_bwd_weight(G, rowmat(z, Lld), grad + n.off_actor_w[0] + n.num_prop, in0, nullptr, rows, gout, p.latent, st));
    // dL/dz = (policy path) + (priv-reg path, already in g_z); then through the ELU of the encoder's last layer
    TRY(linear_bwd_data(G, P + n.off_actor_w[0] + n.num_prop, in0, p.g_z, Lld, rows, p.latent, gout, mlp_act, rowmat(z, Lld), 1, st));
    RowMat Gp = rowmat(p.g_z, Lld);
    int gp = p.latent;
    for (int l = n.n_priv_layers - 1; l >= 0; --l) {
      const int in = l == 0 ? n.num_priv : n.priv_dims[l - 1];
      const int ldin = (int)align_up(in, 4);
      RowMat X = l == 0 ? rowmat_gather(s->observations + n.num_prop, idx, s->obs_stride) : rowmat(p.priv[l - 1], ldin);
      TRY(linear_bwd_weight(Gp, X, grad + n.off_priv_w[l], in, grad + n.off_priv_b[l], rows, gp, in, st));
      if (l > 0) {
        float* d = (l & 1) ? p.d0 : p.d1;
        TRY(linear_bwd_data(Gp, P + n.off_priv_w[l], in, d, ldin, rows, in, gp, mlp_act, X, 0, st));
        Gp = rowmat(d, ldin);
        gp = in;
      }
    }
  }
  return DWBC_OK;
}

extern "C" int dwbc_ppo_minibatch_grad(const DwbcNetCfg* net, const float* params, const DwbcStorage* s, const int64_t* idx, int32_t M,
                                       const DwbcPpoHyper* hp, float* grad, float* losses_out, void* workspace, dwbc_stream_t stream) {
  return ppo_minibatch_grad(net, params, s, idx, M, hp, nullptr, nullptr, nullptr, grad, losses_out, nullptr, workspace, stream);
}

extern "C" int dwbc_ppo_minibatch_grad_sched(const DwbcNetCfg* net, const float* params, const DwbcStorage* s, const int64_t* idx, int32_t M,
                                             const DwbcPpoHyper* hp, const float* sched, float* grad, float* losses_out, void* workspace,
                                             dwbc_stream_t stream) {
  if (!sched) return DWBC_ERR_ARG;
  return ppo_minibatch_grad(net, params, s, idx, M, hp, sched, nullptr, nullptr, grad, losses_out, nullptr, workspace, stream);
}

extern "C" int dwbc_ppo_minibatch_grad_diag(const DwbcNetCfg* net, const float* params, const DwbcStorage* s, const int64_t* idx, int32_t M,
                                            const DwbcPpoHyper* hp, const float* sched, const float* old_mu, const float* old_sigma, float* grad,
                                            float* losses_out, float* diag_out, void* workspace, dwbc_stream_t stream) {
  if (!old_mu || !old_sigma || !diag_out) return DWBC_ERR_ARG;
  return ppo_minibatch_grad(net, params, s, idx, M, hp, sched, old_mu, old_sigma, grad, losses_out, diag_out, workspace, stream);
}

extern "C" int dwbc_dagger_minibatch_grad(const DwbcNetCfg* net, const float* params, const DwbcStorage* s, const int64_t* idx, int32_t M,
                                          float* grad, float* losses_out, void* workspace, dwbc_stream_t stream) {
  TRY(check_net(net));
  if (!params || !s || !s->observations || !idx || !grad || !losses_out || !workspace || M <= 0) return DWBC_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const DwbcNetCfg& n = *net;
  const float* P = params;
  const int rows = M, T = n.num_hist;
  Plan p = make_plan(n, rows, workspace);
  const HistGeo g = hist_geo(n);
  const int L = p.latent, Lld = (int)align_up(L, 4);
  if (cudaMemsetAsync(grad, 0, sizeof(float) * n.num_params, st) != cudaSuccess) return DWBC_ERR_LAUNCH;
  for (int i = 0; i < g.nconv; ++i)
    if (cudaMemsetAsync(p.dhw[i], 0, sizeof(float) * (g.c[i] * g.kdim(i)), st) != cudaSuccess) return DWBC_ERR_LAUNCH;
  if (cudaMemsetAsync(p.dhwl, 0, sizeof(float) * (32 * 36), st) != cudaSuccess) return DWBC_ERR_LAUNCH;
  TRY(priv_forward(n, P, s->observations, idx, s->obs_stride, rows, p, st));             // PPO:273-274 (no grad)
  TRY(hist_forward(n, P, s->observations, idx, s->obs_stride, rows, p, st));             // PPO:275
  dagger_loss_kernel<<<(rows + 127) / 128, 128, 0, st>>>(p.priv[n.n_priv_layers - 1], p.zh, Lld, L, p.dzh, losses_out, p.loss_part,
                                                           reinterpret_cast<unsigned*>(p.queue + 3), rows, mlp_act);
  DWBC_LAUNCH_CHECK();
  // linear_output: zh = act(flat . Wl'^T + b)
  const float* hlast = p.hc[g.nconv - 1];
  RowMat G4 = rowmat(p.dzh, Lld);
  TRY(linear_bwd_weight(G4, rowmat(hlast, 36), p.dhwl, 36, grad + n.off_hist_b[4], rows, L, 36, st));
  TRY(linear_bwd_data(G4, p.hwl, 36, p.d0, 36, rows, 36, L, mlp_act, rowmat(hlast, 36), 0, st));    // d(last conv pre-act) as [rows*3, 12]
  // convs, last first: weight gradient, im2col-space input gradient, then col2im with the input's activation derivative
  const float* gout = p.d0;
  for (int i = g.nconv - 1; i >= 0; --i) {
    const float* in = i == 0 ? p.hproj : p.hc[i - 1];
    float* dst = i == 0 ? p.dh_proj : p.dh_c[i - 1];
    const int rows_o = rows * g.pos[i + 1], kd = g.kdim(i);
    RowMat G = rowmat(gout, g.ld[i + 1]);
    TRY(linear_bwd_weight(G, rowmat_grouped(in, nullptr, g.pos[i + 1], (int64_t)g.pos[i] * g.ld[i], g.s[i] * g.ld[i]), p.dhw[i], kd,
                          grad + n.off_hist_b[1 + i], rows_o, g.c[i], kd, st));
    TRY(linear_bwd_data(G, p.hw[i], kd, p.dh_a[i], kd, rows_o, kd, g.c[i], ACT_NONE, RowMat{}, 0, st));
    int64_t tot = (int64_t)rows * g.pos[i] * g.ld[i];
    col2im_dact_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(p.dh_a[i], in, dst, rows, g.pos[i], g.cin[i], g.ld[i], g.pos[i + 1], g.k[i],
                                                                     g.s[i], mlp_act);
    DWBC_LAUNCH_CHECK();
    gout = dst;
  }
  // projection
  RowMat G1 = rowmat(p.dh_proj, 32);
  RowMat hist = rowmat_grouped(s->observations + (n.num_obs - T * n.num_prop), idx, T, s->obs_stride, n.num_prop);
  TRY(linear_bwd_weight(G1, hist, grad + n.off_hist_w[0], n.num_prop, grad + n.off_hist_b[0], rows * T, 30, n.num_prop, st));
  hist_unpack_grad_kernel<<<hist_pack_grid(g), 256, 0, st>>>(
      hist_pack_args(g, grad + n.off_hist_w[1], grad + n.off_hist_w[2], grad + n.off_hist_w[3], grad + n.off_hist_w[4], p.dhw, p.dhwl, L));
  DWBC_LAUNCH_CHECK();
  return DWBC_OK;
}

// The weight-gradient partials of a debug entry point: `cap` floats of stream-ordered memory, freed behind the launches
template <class F>
static int with_debug_wpart(int64_t cap, cudaStream_t st, F&& launch) {
  void* p = nullptr;
  if (cudaMallocAsync(&p, (size_t)cap * sizeof(float), st) != cudaSuccess) return DWBC_ERR_LAUNCH;
  mlp_wpart = static_cast<float*>(p);
  mlp_wpart_cap = cap;
  const int rc = launch();
  mlp_wpart = nullptr;
  mlp_wpart_cap = 0;
  return cudaFreeAsync(p, st) == cudaSuccess ? rc : DWBC_ERR_LAUNCH;
}

// Debug / test entry: one GEMM of the selected implementation on plain row-major device matrices.
//   mode 0: Y[M,N] = act(X[M,K] W[N,K]^T + b)      mode 1: dX[M,N] = G[M,K] W[K,N]      mode 2: dW[M,N] += G[K,M]^T X[K,N], db += colsum(G)
extern "C" int dwbc_debug_gemm(int mode, int tc, const float* A, int64_t lda, const float* Bm, int64_t ldb, float* C, int64_t ldc,
                               const float* bias, float* dbias, int M, int N, int K, int act, dwbc_stream_t stream) {
  const int saved = mlp_precision;
  mlp_precision = tc;
  int rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (mode == 0) rc = linear_fwd(rowmat(A, lda), Bm, ldb, bias, C, ldc, M, N, K, act, 0, st);
  else if (mode == 1) rc = linear_bwd_data(rowmat(A, lda), Bm, ldb, C, ldc, M, N, K, ACT_NONE, RowMat{}, 0, st);
  else {
    // the partials of the split-K / slab sums in stream-ordered scratch (no workspace here)
    if (M <= 0 || N <= 0 || K <= 0) { mlp_precision = saved; return DWBC_ERR_ARG; }
    const int64_t cap = std::max(simt_wgrad_floats(M, N, K), wg_max_nslab(K) * wg_slot(std::min(M, 128), std::min(N, 128)));
    rc = with_debug_wpart(cap, st, [&] { return linear_bwd_weight(rowmat(A, lda), rowmat(Bm, ldb), C, ldc, dbias, K, M, N, st); });
  }
  mlp_precision = saved;
  return rc;
}

// The chain PROGRAMS a call would launch, described without launching anything (host code only, no GPU; every pointer is formed from the
// fake bases below and never dereferenced).  what: 0 = dwbc_policy_act, 1 = dwbc_critic_values, 2 = forward + loss of dwbc_ppo_minibatch_grad,
// 3 = its backward launch, 4 = dwbc_policy_mean (when dwbc_policy_act runs on the chains), 5 = forward + loss of dwbc_ppo_minibatch_grad_diag
// (2 with the heads' means kept for the diagnostics).  out = [nprog, pack items, then per program:
// n_ops, n_loads, then per op: N, kpad, act, fin, fin_c, out_col0, has_global_output, output_is_tile_image].  Returns the number of ints written, or a negative error code (DWBC_ERR_UNSUPPORTED: the
// configuration does not run on the fused chains).  tests/test_host_cpu.py pins the program structure with it.
extern "C" int dwbc_debug_describe_chain(const DwbcNetCfg* net, int32_t rows, int what, int hist_encoding, int sms, int32_t* out, int32_t out_len) {
  TRY(check_net(net));
  if (rows <= 0 || what < 0 || what > 5 || sms <= 0 || !out) return DWBC_ERR_ARG;
  const DwbcNetCfg& n = *net;
  float* const ws = reinterpret_cast<float*>(uintptr_t(1) << 40);
  const float* const P = reinterpret_cast<const float*>(uintptr_t(2) << 40);
  const float* const obs = reinterpret_cast<const float*>(uintptr_t(3) << 40);
  const int64_t* const idx = what == 2 || what == 3 || what == 5 ? reinterpret_cast<const int64_t*>(uintptr_t(4) << 40) : nullptr;
  Plan p = make_plan(n, rows, ws);
  C2Chains ch(p.wpack, rows, mlp_precision == 2);
  const int mode = what < 2 ? what : (what == 4 ? 3 : 2);
  if (!plan_chains(ch, mode, n, P, obs, idx, n.num_obs, hist_encoding != 0, p.value, p, rows, sms, what == 5)) return DWBC_ERR_UNSUPPORTED;
  const C2Builder* prs = what == 3 ? ch.b + 2 : ch.b;
  int k = 0;
  auto put = [&](int v) { if (k < out_len) out[k] = v; ++k; };
  put(ch.nprog); put(ch.pl.n);
  for (int q = 0; q < ch.nprog; ++q) {
    const C2Prog& pr = prs[q].pr;
    put(pr.n_ops); put(pr.n_loads);
    for (int i = 0; i < pr.n_ops; ++i) {
      const C2Op& o = pr.op[i];
      put(o.N); put(o.kpad); put(o.act); put(o.fin); put(o.fin_c); put(o.out_col0); put(o.y != nullptr); put(o.y_img);
    }
  }
  return k <= out_len ? k : DWBC_ERR_ARG;
}

// The work-item planner of launch_chain2n on its own (host code only, no GPU): for `tiles` row tiles x `nprog` programs of per-two-tile-item
// costs cost[nprog] on `sms` persistent CTAs, the number of two-tile (np2) and one-tile (ns1) items per program it would launch and the
// simulated makespans with (span) and without (span0) one-tile items.  tests/test_host_cpu.py checks coverage and the decision.
extern "C" int dwbc_debug_chain_plan(int tiles, int nprog, const double* cost, int sms, int* np2, int* ns1, double* span, double* span0) {
  if (tiles <= 0 || nprog < 1 || nprog > C2_MAX_PROGS || !cost || sms <= 0 || !np2 || !ns1) return DWBC_ERR_ARG;
  if (tiles * nprog <= sms) { *np2 = 0; *ns1 = tiles; }
  else { *ns1 = c2_pick_singles(tiles, nprog, cost, sms); *np2 = (tiles - *ns1 + 1) / 2; }
  if (span) *span = c2_makespan(tiles, nprog, cost, sms, *np2 ? *ns1 : 0);
  if (span0) *span0 = c2_makespan(tiles, nprog, cost, sms, 0);
  return DWBC_OK;
}
// The grouped weight-gradient launch on caller-described GEMMs (tests/test_gpu_wgrad_group.py)
extern "C" int dwbc_debug_wgrad_group(const DwbcWgradGemm* gemms, int n, int rows, int x3, dwbc_stream_t stream) {
  if (!gemms || n <= 0 || n > WG_MAX || rows <= 0) return DWBC_ERR_ARG;
  auto mat = [](const float* p, const int64_t* idx, int image, int64_t ld) {
    return image ? rowmat_image(p) : (idx ? rowmat_gather(p, idx, ld) : rowmat(p, ld));
  };
  WGroupBuilder b;
  for (int i = 0; i < n; ++i) {
    const DwbcWgradGemm& d = gemms[i];
    if (!d.g || !d.x || !d.dw || (d.g_image && d.g_idx) || (d.x_image && d.x_idx)) return DWBC_ERR_ARG;
    b.add(mat(d.g, d.g_idx, (int)d.g_image, d.g_ld), mat(d.x, d.x_idx, (int)d.x_image, d.x_ld), d.dw, d.lddw, d.db, (int)d.mo, (int)d.ni);
  }
  if (!b.ok) return DWBC_ERR_ARG;
  int64_t slots = 0;
  for (int i = 0; i < n; ++i) slots += wg_slot((int)gemms[i].mo, (int)gemms[i].ni);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return with_debug_wpart(wg_max_nslab(rows) * slots, st, [&] { return launch_wgrad_group(b.g, rows, x3 != 0, st); });
}
extern "C" int dwbc_debug_set_tc_cycle_buffer(unsigned long long* dev_ptr) {
  return cudaMemcpyToSymbol(g_tc_cycles, &dev_ptr, sizeof(dev_ptr)) == cudaSuccess ? DWBC_OK : DWBC_ERR_LAUNCH;
}

// The partial area the grouped weight-gradient launch of dwbc_ppo_minibatch_grad would use on `sms` SMs, and the area
// dwbc_workspace_bytes reserves for it (host code only, no GPU; tests/test_reproducibility_cpu.py checks need <= bound)
extern "C" int dwbc_debug_wgrad_partial_floats(const DwbcNetCfg* net, int32_t rows, int sms, int64_t* need, int64_t* bound) {
  TRY(check_net(net));
  if (rows <= 0 || sms <= 0 || !need || !bound) return DWBC_ERR_ARG;
  float* const ws = reinterpret_cast<float*>(uintptr_t(1) << 40);
  DwbcStorage s{};
  s.observations = reinterpret_cast<const float*>(uintptr_t(2) << 40);
  s.obs_stride = net->num_obs;
  Plan p = make_plan(*net, rows, ws);
  mlp_wpart = nullptr;
  mlp_wpart_cap = 0;
  WGroupBuilder wb;
  if (!wgrad_gemms(wb, *net, ws, &s, reinterpret_cast<const int64_t*>(uintptr_t(3) << 40), p)) return DWBC_ERR_UNSUPPORTED;
  *need = wg_plan(wb.g, rows, mlp_precision == 2, sms);
  *bound = wpart_floats(*net, rows);
  return DWBC_OK;
}
