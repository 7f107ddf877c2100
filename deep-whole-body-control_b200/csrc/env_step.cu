// Fused widowGo1 post-physics step, warp-per-env kernel: ONE kernel launch per sim step (K1 + K2 of SURVEY.md).
//
// Replaces the ~200 ATen launches of WidowGo1.post_physics_step (WG:875-910): derived base
// state, EE-goal generator, command resampling, push, height scan, termination, the reward-term
// stack for both channels, episode sums, reset, observation assembly, history shift, obs clip.
//
// Mapping: one WARP per environment, 4 warps per CTA, any shape and shard size.  The TMA kernel
// (env_step_v2.cu) runs the widowGo1 shapes with 10-step histories on shards that are a multiple of 32;
// this kernel runs everything else.  Both call the per-env functions of env_step_common.cuh on the
// env's rows staged in shared memory: this kernel runs the warp functions with its warp and
// scalar_step() on lane 0.  The history row is read as 128-bit streaming loads issued before anything
// else (so ~86 KB are in flight per SM), re-emitted into obs_buf and shifted in place.  With a device
// step record (a captured step whose step, push decision and curriculum values are read at run time)
// both kernels build their step arguments in shared memory once per CTA (step_args_to_shared).
//
// Compiled with -fmad=false so that discrete decisions (collision rejection, command dead-band,
// termination thresholds) see the same fp32 roundings as the reference's unfused torch arithmetic.
#include <stdlib.h>

#include "env_step_common.cuh"

namespace dwbc {

constexpr int ENV_WARPS = 4;
constexpr int MAX_H4 = 8;  // history row <= 8*32 float4 = 1024 floats in registers; longer rows take the streaming form (kLong)

// shared-memory staging block of one warp (float offsets; S_PRIV and S_PROP 16-byte aligned for the float4 write-out)
enum {
  S_ROOT = 0, S_DOF = 28, S_EE = 76, S_FS = 84, S_TQ = 108, S_ACT = 132, S_AH = 156, S_GS = 348, S_DS = 376, S_SUM = 448,
  S_PRIV = 512, S_PROP = 544, S_CF = 640, S_MASS = 700, S_FRIC = 705, S_MOTOR = 708, S_FEAT = 732, S_RP = 748, S_REW = 752, S_TOTAL = 756
};
static_assert(S_DOF - S_ROOT >= 26 && S_EE - S_DOF >= 2 * DWBC_MAX_DOF && S_GS - S_AH >= 8 * DWBC_MAX_DOF && S_SUM - S_DS >= DWBC_DS &&
                  S_PRIV - S_SUM >= DWBC_MAX_SLOTS && S_MASS - S_CF >= 3 * (4 + 2 * DWBC_MAX_IDX) && S_RP - S_FEAT >= FE_COUNT,
              "staging rows overlap");

// kLong = false: the history row (<= 1024 floats) is loaded into registers before anything else and re-emitted from there.
// kLong = true (history_len * num_prop > 1024, e.g. 20 or 50 steps of 76): the row is streamed at the end instead, in ascending
// 32-float4 chunks: each chunk is loaded, written to obs clipped (WG:992, 1195-1196), and after a __syncwarp written back one num_prop
// row lower (WG:997-999).  In place is safe: the targets of chunk i lie below its end, so chunks <= i have read them already.
// The minimum of 1 CTA per SM keeps ptxas from capping the streaming form at 64 registers, where it spills.
// kDev = true: a launch of dwbc_post_physics_step_device; each CTA builds its step arguments from Ah and the device record `dev` in
// shared memory once.  kDev = false reads Ah directly: building the copy cost an eager launch 0.3-0.4 us (H100 SXM, 700 W).
static_assert(STEP_ARGS_WORDS <= ENV_WARPS * 32, "step_args_to_shared: one word per thread");
template <bool kLong, bool kDev>
__global__ void __launch_bounds__(ENV_WARPS * 32, 1)
env_step_kernel(const __grid_constant__ DwbcEnvCfg cfg, const __grid_constant__ DwbcEnvBuffers B,
                const __grid_constant__ DwbcStepArgs Ah, const DwbcStepDevice* __restrict__ dev) {
  __shared__ __align__(16) float smem[ENV_WARPS * S_TOTAL];
  __shared__ DwbcStepArgs As;
  const DwbcStepArgs& A = kDev ? As : Ah;     // this step's arguments
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int e = blockIdx.x * ENV_WARPS + wid;
  // kDev: the tail CTA of a ragged shard has idle warps; they still write their words of As and reach the barrier below
  const bool active = e < cfg.num_envs;
  if constexpr (!kDev) {
    if (!active) return;
  }
  float* sm = smem + wid * S_TOTAL;
  const int nd = cfg.num_dofs, na = cfg.num_actions, ahl = cfg.action_hist_len, P = cfg.num_prop, H = cfg.history_len;
  const int nbp1 = cfg.num_bodies_p1;
  const int nh4 = (H * P) >> 2, p4 = P >> 2, pp4 = (P + cfg.num_priv) >> 2;
  const int nslots = cfg.n_sum_slots + DWBC_NUM_METRICS;

  // ---- 1. history row: all 128-bit loads in flight first --------------------------------------
  float4* hist4 = reinterpret_cast<float4*>(B.obs_history + (size_t)e * H * P);
  float4 h[kLong ? 1 : MAX_H4];
  if constexpr (!kLong) {
#pragma unroll
    for (int i = 0; i < MAX_H4; ++i) {
      int idx = lane + 32 * i;
      h[i] = active && idx < nh4 ? ldg_stream(hist4 + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  if constexpr (kDev) {
    step_args_to_shared(Ah, dev, &As, threadIdx.x);
    __syncthreads();
    if (!active) return;
  }
  // ---- 2. coalesced staging of the env's rows ----------------------------------------------------
  float* root_g = B.root_states + (size_t)e * 26;
  if (lane < 26) sm[S_ROOT + lane] = root_g[lane];
  float* dof_g = B.dof_state + (size_t)e * 2 * nd;
  for (int i = lane; i < 2 * nd; i += 32) sm[S_DOF + i] = dof_g[i];
  if (lane < 7) sm[S_EE + lane] = __ldg(B.rigid_body_state + ((size_t)e * nbp1 + cfg.gripper_idx) * 13 + lane);
  if (lane < 24) sm[S_FS + lane] = __ldg(B.force_sensor + (size_t)e * 24 + lane);
  if (lane < nd) sm[S_TQ + lane] = __ldg(B.torques + (size_t)e * nd + lane);
  if (lane < na) sm[S_ACT + lane] = __ldg(B.actions + (size_t)e * na + lane);
  float* ah_g = B.action_history + (size_t)e * ahl * na;
  for (int i = lane; i < ahl * na; i += 32) sm[S_AH + i] = ah_g[i];
  float* gs_g = B.goal_state + (size_t)e * DWBC_GS;
  if (lane < DWBC_GS) sm[S_GS + lane] = gs_g[lane];
  float* ds_g = B.derived_state + (size_t)e * DWBC_DS;
  for (int i = DWBC_DS_FEET_AIR_TIME + lane; i < DWBC_DS; i += 32) sm[S_DS + i] = ds_g[i];   // columns below are rewritten every step
  float* sum_g = B.episode_sums + (size_t)e * cfg.sums_stride;
  for (int i = lane; i < nslots; i += 32) sm[S_SUM + i] = sum_g[i];
  if (lane < 5) sm[S_MASS + lane] = __ldg(B.mass_params + (size_t)e * 5 + lane);
  else if (lane == 5) sm[S_FRIC] = __ldg(B.friction + e);
  if (lane < na) sm[S_MOTOR + lane] = __ldg(B.motor_strength + (size_t)e * na + lane);
  {
    const int ncf = 4 + cfg.n_penalized + cfg.n_term_contact;
    for (int i = lane; i < 3 * ncf; i += 32) {
      int b = i / 3, k = i - 3 * b;
      int body = b < 4 ? cfg.feet_idx[b] : (b < 4 + cfg.n_penalized ? cfg.penalized_idx[b - 4] : cfg.term_contact_idx[b - 4 - cfg.n_penalized]);
      sm[S_CF + i] = __ldg(B.contact_forces + ((size_t)e * nbp1 + body) * 3 + k);
    }
  }
  long long ep = B.episode_length[e] + 1;  // WG:875
  __syncwarp();
  const EnvView v{sm + S_ROOT, sm + S_DOF, sm + S_FS, sm + S_TQ, sm + S_ACT, sm + S_AH, sm + S_GS, sm + S_DS, sm + S_SUM, sm + S_EE,
                  sm + S_CF, sm + S_MASS, sm + S_FRIC, sm + S_MOTOR, sm + S_PROP, sm + S_PRIV, sm + S_FEAT, sm + S_RP, sm + S_REW};

  // ---- 3. DOF reductions, height scan, then the scalar step on lane 0 -----------------------------
  dof_features(cfg, v, feature_mask(cfg), cfg.default_dof_pos, nd, na, lane);
  const float gap = cfg.measure_heights ? height_scan(cfg, B, v.root, e, lane) : 0.0f;
  if (lane == 0) v.rp[3] = gap;
  __syncwarp();
  int flags = 0;
  if (lane == 0) flags = scalar_step(cfg, A, v, e, ep);
  __syncwarp();   // orders lane 0's writes to the staged rows before the warp's reads and writes in fix_up() (a shuffle does not)
  flags = __shfl_sync(FULL, flags, 0);
  // ---- 4. goal resample and reset -----------------------------------------------------------------
  if (flags & (F_GOAL_RS | F_RESET)) flags = fix_up(cfg, A, B, v, flags, e, nd, na, ahl, nslots, lane);
  if (flags & F_RESET) {
    ep = 0;
    if constexpr (!kLong) {
#pragma unroll
      for (int i = 0; i < MAX_H4; ++i) h[i] = make_float4(0.f, 0.f, 0.f, 0.f);   // the old history reads as zeros (WG:735)
    }
  }
  __syncwarp();

  // ---- 5. observations (WG:966-1001); this kernel always writes them clipped ----------------------
  assemble_obs(cfg, v, 0, cfg.ig2raisim, cfg.default_dof_pos, INFINITY, nd, na, ahl, lane);
  assemble_obs(cfg, v, 1, cfg.ig2raisim, cfg.default_dof_pos, INFINITY, nd, na, ahl, lane);
  if (lane == 0) v.ds[DWBC_DS_OOB_AGE] = 0.0f;   // no stored history row is known to lie within the clip
  __syncwarp();

  // ---- 6. outputs -------------------------------------------------------------------------------
  const float c = cfg.clip_obs > 0.0f ? cfg.clip_obs : INFINITY;
  float4* obs4 = reinterpret_cast<float4*>(B.obs_buf + (size_t)e * B.obs_stride);
  const float4* prop4 = reinterpret_cast<const float4*>(sm + S_PROP);
  const float4* priv4 = reinterpret_cast<const float4*>(sm + S_PRIV);
  if (lane < pp4) stg_stream(obs4 + lane, clip4(lane < p4 ? prop4[lane] : priv4[lane - p4], c));
  const bool fill = (flags & F_FILL) != 0;
  if constexpr (!kLong) {
#pragma unroll
    for (int i = 0; i < MAX_H4; ++i) {
      int idx = lane + 32 * i;
      if (idx < nh4) stg_stream(obs4 + pp4 + idx, clip4(h[i], c));  // OLD history (WG:992)
    }
    __syncwarp();  // every lane's history loads have been consumed: the in-place shift below is safe
    if (fill) {     // WG:994-996: fill all H rows with the new proprioception
#pragma unroll
      for (int i = 0; i < MAX_H4; ++i) {
        int idx = lane + 32 * i;
        if (idx < nh4) hist4[idx] = prop4[idx % p4];
      }
    } else {        // WG:997-1000: drop the oldest row, append
#pragma unroll
      for (int i = 0; i < MAX_H4; ++i) {
        int idx = lane + 32 * i;
        if (idx >= p4 && idx < nh4) hist4[idx - p4] = h[i];
      }
      if (lane < p4) hist4[nh4 - p4 + lane] = prop4[lane];
    }
  } else {
    const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i0 = 0; i0 < nh4; i0 += 32) {
      const int idx = i0 + lane;
      h[0] = idx < nh4 && !(flags & F_RESET) ? __ldcs(hist4 + idx) : zero4;   // reset: the old history reads as zeros (WG:735)
      if (idx < nh4) stg_stream(obs4 + pp4 + idx, clip4(h[0], c));    // OLD history (WG:992)
      __syncwarp();  // the whole chunk has been read: its targets (and everything below them) may be overwritten
      if (fill) {             // WG:994-996
        if (idx < nh4) hist4[idx] = prop4[idx % p4];
      } else if (idx >= p4 && idx < nh4) {
        hist4[idx - p4] = h[0];                                            // WG:997-999
      }
    }
    if (!fill && lane < p4) hist4[nh4 - p4 + lane] = prop4[lane];          // WG:1000
  }
  if (flags & F_ROOT_DIRTY) { if (lane < 26) root_g[lane] = sm[S_ROOT + lane]; }
  if (flags & F_DOF_DIRTY) {
    for (int i = lane; i < 2 * nd; i += 32) dof_g[i] = sm[S_DOF + i];
    for (int i = lane; i < ahl * na; i += 32) ah_g[i] = sm[S_AH + i];
  }
  if (lane < DWBC_GS) gs_g[lane] = sm[S_GS + lane];
  for (int i = lane; i < DWBC_DS; i += 32) ds_g[i] = sm[S_DS + i];
  for (int i = lane; i < nslots; i += 32) sum_g[i] = sm[S_SUM + i];
  if (lane == 0) {
    B.episode_length[e] = ep;
    store_step(B, e, flags, v.rew[0], v.rew[1]);
  }
  store_heights_obs(cfg, B, e, 1, v.root, lane, 32);
}

__global__ void fill_uniform_kernel(float* out, int n, uint64_t seed, uint64_t step) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;  // one thread per (env, group of 4 columns)
  if (i >= n * (DWBC_RAND_COLS / 4)) return;
  int env = i / (DWBC_RAND_COLS / 4), g = i - env * (DWBC_RAND_COLS / 4);
  uint4 r = philox4x32_10(make_uint4((uint32_t)env, (uint32_t)g, (uint32_t)step, (uint32_t)(step >> 32)),
                          make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  reinterpret_cast<float4*>(out)[i] = make_float4(u01(r.x), u01(r.y), u01(r.z), u01(r.w));
}

// WG:1162-1173: one thread per (env, action)
__global__ void pre_physics_actions_kernel(const float* __restrict__ pol, const int32_t* __restrict__ r2i, float clip,
                                           float* __restrict__ hist, float* __restrict__ actions, int n, int na, int ah, int delay_row) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * na) return;
  int e = i / na, a = i - e * na;
  float* hrow = hist + (size_t)e * ah * na;
  float v = fminf(fmaxf(pol[(size_t)e * na + r2i[a]], -clip), clip);
  // shift the FIFO (each thread owns column a of every row: no cross-thread hazard)
  float prev[8];
  for (int r = 1; r < ah; ++r) prev[r - 1] = hrow[r * na + a];
  for (int r = 0; r < ah - 1; ++r) hrow[r * na + a] = prev[r];
  hrow[(ah - 1) * na + a] = v;
  actions[i] = delay_row == ah - 1 ? v : prev[delay_row];
}

}  // namespace dwbc

using namespace dwbc;

int dwbc_launch_env_step_v2(const DwbcEnvCfg* cfg, const DwbcEnvBuffers* buf, const DwbcStepArgs* args, const DwbcStepDevice* dev, cudaStream_t st);

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// The kernels read a device step record from device memory: device or managed memory, or host memory registered with CUDA and mapped at
// the same address.  A pointer the runtime does not know as one of these (plain host memory, a stale address), or a failed query, is
// refused before anything is launched instead of faulting in the kernel.  Only calls with a record (captures) pay for the query.
static bool device_readable(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    (void)cudaGetLastError();   // not sticky: clear it so that the next launch check does not report it
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged || (a.type == cudaMemoryTypeHost && a.devicePointer == p);
}

// extras['episode'] of one step in a fixed order: block c adds column c of the slots of the envs that reset, in env order (thread t:
// envs t, t + 256, ...; then a fixed tree), column 0 counting them; episode_stats[c] += that sum
// With a device step record (dwbc_post_physics_step_device) block 0 also advances its step: the post-physics kernel before it has used it.
__global__ void __launch_bounds__(256) episode_stats_kernel(const uint8_t* __restrict__ reset, const float* __restrict__ slots, int stride, int n,
                                                            float* __restrict__ stats, DwbcStepDevice* __restrict__ dev) {
  __shared__ float red[256];
  const int c = blockIdx.x;
  if (dev && c == 0 && threadIdx.x == 0) dev->step += 1;
  float s = 0.0f;
  for (int e = threadIdx.x; e < n; e += 256)
    if (reset[e]) s += c == 0 ? 1.0f : slots[(size_t)e * stride + c - 1];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) stats[c] += red[0];
}

static int launch_episode_stats(const DwbcEnvCfg* cfg, const DwbcEnvBuffers* buf, DwbcStepDevice* dev, cudaStream_t st) {
  episode_stats_kernel<<<1 + cfg->n_sum_slots + DWBC_NUM_METRICS, 256, 0, st>>>(buf->reset_buf, buf->episode_scratch, cfg->sums_stride,
                                                                              cfg->num_envs, buf->episode_stats, dev);
  DWBC_LAUNCH_CHECK();
  return DWBC_OK;
}

// dev: optional device step record (dwbc_post_physics_step_device)
static int post_physics_step(const DwbcEnvCfg* cfg, const DwbcEnvBuffers* buf, const DwbcStepArgs* args, DwbcStepDevice* dev,
                             dwbc_stream_t stream) {
  if (!cfg || !buf || !args) return DWBC_ERR_ARG;
  if (cfg->abi_version != DWBC_ABI_VERSION || cfg->num_envs <= 0) return DWBC_ERR_ARG;
  const int nd = cfg->num_dofs, na = cfg->num_actions;
  if (nd > DWBC_MAX_DOF || nd > 24 || na > nd || nd < 14) return DWBC_ERR_UNSUPPORTED;
  if (cfg->num_prop != 2 + 3 + 2 * nd + na + 4 + 3 + 3 + 3) return DWBC_ERR_UNSUPPORTED;  // WG:973-983
  if (cfg->num_priv != 5 + 1 + na) return DWBC_ERR_UNSUPPORTED;                            // WG:987-991
  if ((cfg->num_prop & 3) || (cfg->num_priv & 3) || (buf->obs_stride & 3)) return DWBC_ERR_UNSUPPORTED;
  if (cfg->num_prop > 96 || cfg->history_len < 1) return DWBC_ERR_UNSUPPORTED;
  if (cfg->n_sum_slots + DWBC_NUM_METRICS > DWBC_MAX_SLOTS || cfg->sums_stride < cfg->n_sum_slots + DWBC_NUM_METRICS) return DWBC_ERR_ARG;
  if (cfg->n_leg_terms > DWBC_MAX_TERMS || cfg->n_arm_terms > DWBC_MAX_TERMS) return DWBC_ERR_ARG;
  if (cfg->n_penalized > DWBC_MAX_IDX || cfg->n_term_contact > DWBC_MAX_IDX) return DWBC_ERR_ARG;
  if (cfg->n_collision_samples > 16 || cfg->action_hist_len > 8) return DWBC_ERR_UNSUPPORTED;
  if (cfg->measure_heights && (!buf->height_samples || !buf->measured_heights || cfg->n_height_x > 24 || cfg->n_height_y > 16))
    return DWBC_ERR_ARG;
  if (cfg->terrain_curriculum && (!buf->terrain_levels || !buf->terrain_types || !buf->terrain_origins)) return DWBC_ERR_ARG;
  if (!buf->root_states || !buf->dof_state || !buf->rigid_body_state || !buf->contact_forces || !buf->force_sensor ||
      !buf->torques || !buf->actions || !buf->action_history || !buf->mass_params || !buf->friction || !buf->motor_strength ||
      !buf->env_origins || !buf->box_env_origins_delta_y || !buf->goal_state || !buf->derived_state || !buf->episode_length ||
      !buf->obs_history || !buf->episode_sums || !buf->obs_buf || !buf->rew_buf || !buf->arm_rew_buf || !buf->reset_buf ||
      !buf->time_out_buf || !buf->episode_stats || !buf->episode_scratch || (buf->store_rewards && !buf->store_values))
    return DWBC_ERR_ARG;
  // both kernels move observation rows and history rows in 16-byte vectors
  if (!aligned16(buf->obs_buf) || !aligned16(buf->obs_history)) return DWBC_ERR_UNSUPPORTED;
  if (dev && !device_readable(dev)) return DWBC_ERR_UNSUPPORTED;
  // the TMA kernel (16 envs per CTA, bulk copies) whenever the shard is a multiple of 32 envs and every block is 16-B aligned
  if (cfg->num_envs % 32 == 0 && aligned16(buf->root_states) && aligned16(buf->dof_state) && aligned16(buf->force_sensor) &&
      aligned16(buf->torques) && aligned16(buf->actions) && aligned16(buf->action_history) && aligned16(buf->mass_params) &&
      aligned16(buf->friction) && aligned16(buf->motor_strength) && aligned16(buf->goal_state) && aligned16(buf->derived_state) &&
      aligned16(buf->episode_length) && aligned16(buf->episode_sums) && !args->generic_kernel) {
    const int rc = dwbc_launch_env_step_v2(cfg, buf, args, dev, (cudaStream_t)stream);
    if (rc != DWBC_ERR_UNSUPPORTED) return rc == DWBC_OK ? launch_episode_stats(cfg, buf, dev, (cudaStream_t)stream) : rc;
  }
  const int grid = (cfg->num_envs + ENV_WARPS - 1) / ENV_WARPS;
  const bool long_row = (int64_t)cfg->history_len * cfg->num_prop > MAX_H4 * 128;
  auto kern = long_row ? (dev ? env_step_kernel<true, true> : env_step_kernel<true, false>)
                       : (dev ? env_step_kernel<false, true> : env_step_kernel<false, false>);
  kern<<<grid, ENV_WARPS * 32, 0, (cudaStream_t)stream>>>(*cfg, *buf, *args, dev);
  DWBC_LAUNCH_CHECK();
  return launch_episode_stats(cfg, buf, dev, (cudaStream_t)stream);
}

extern "C" int dwbc_post_physics_step(const DwbcEnvCfg* cfg, const DwbcEnvBuffers* buf, const DwbcStepArgs* args,
                                      dwbc_stream_t stream) {
  return post_physics_step(cfg, buf, args, nullptr, stream);
}

extern "C" int dwbc_post_physics_step_device(const DwbcEnvCfg* cfg, const DwbcEnvBuffers* buf, const DwbcStepArgs* args, DwbcStepDevice* device,
                                             dwbc_stream_t stream) {
  if (!device) return DWBC_ERR_ARG;
  return post_physics_step(cfg, buf, args, device, stream);
}

extern "C" int dwbc_fill_uniform(float* out, int32_t num_envs, uint64_t seed, uint64_t step, dwbc_stream_t stream) {
  if (!out || num_envs <= 0) return DWBC_ERR_ARG;
  int n = num_envs * (DWBC_RAND_COLS / 4);
  fill_uniform_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(out, num_envs, seed, step);
  DWBC_LAUNCH_CHECK();
  return DWBC_OK;
}

extern "C" int dwbc_pre_physics_actions(const float* policy_actions, const int32_t* raisim2ig, float clip_actions,
                                        float* action_history, float* actions, int32_t num_envs, int32_t num_actions,
                                        int32_t action_hist_len, int32_t delay_row, dwbc_stream_t stream) {
  if (!policy_actions || !raisim2ig || !action_history || !actions || num_envs <= 0) return DWBC_ERR_ARG;
  if (action_hist_len < 2 || action_hist_len > 8 || delay_row < 0 || delay_row >= action_hist_len) return DWBC_ERR_UNSUPPORTED;
  int n = num_envs * num_actions;
  pre_physics_actions_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(policy_actions, raisim2ig, clip_actions,
                                                                                 action_history, actions, num_envs, num_actions,
                                                                                 action_hist_len, delay_row);
  DWBC_LAUNCH_CHECK();
  return DWBC_OK;
}

// ---- PD torque controller (WG:1262-1295), SURVEY 8f row f1 ------------------------------------------------------------
__global__ void compute_torques_kernel(const DwbcPdCfg cfg, const float* __restrict__ actions, const float* __restrict__ dof_state,
                                       const float* __restrict__ motor_strength, float* __restrict__ torques, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * cfg.n_dof) return;
  const int e = i / cfg.n_dof, j = i - e * cfg.n_dof;
  float t = 0.0f;                                                          // gripper_torques_zero (WG:1291)
  if (j < cfg.n_act) {
    const float a = actions[(size_t)e * cfg.n_act + j];
    const float scaled = (a * motor_strength[(size_t)e * cfg.n_act + j]) * cfg.action_scale[j];   // WG:1276
    float q = dof_state[((size_t)e * cfg.n_dof + j) * 2];
    if (j == cfg.wrap_dof) q = wrap_pi(q);                                 // WG:1278-1279
    const float qd = dof_state[((size_t)e * cfg.n_dof + j) * 2 + 1];
    t = cfg.p_gains[j] * ((scaled + cfg.default_dof_pos[j]) - q) - cfg.d_gains[j] * qd;           // WG:1281
  }
  const float lim = cfg.torque_limits[j];
  torques[i] = fminf(fmaxf(t, -lim), lim);                                 // WG:1295
}

extern "C" int dwbc_compute_torques(const DwbcPdCfg* cfg, const float* actions, const float* dof_state, const float* motor_strength,
                                    float* torques, int32_t num_envs, dwbc_stream_t stream) {
  if (!cfg || !actions || !dof_state || !motor_strength || !torques || num_envs <= 0) return DWBC_ERR_ARG;
  if (cfg->n_dof <= 0 || cfg->n_dof > DWBC_MAX_DOF || cfg->n_act <= 0 || cfg->n_act > cfg->n_dof || cfg->wrap_dof >= cfg->n_act) return DWBC_ERR_ARG;
  const int total = num_envs * cfg->n_dof;
  compute_torques_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(*cfg, actions, dof_state, motor_strength, torques, num_envs);
  DWBC_LAUNCH_CHECK();
  return DWBC_OK;
}
