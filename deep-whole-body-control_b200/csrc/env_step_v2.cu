// Fused widowGo1 post-physics step, TMA kernel: ONE launch per sim step, 16 envs per CTA, TMA-fed.
//
//  * Every contiguous block of the CTA's 32 envs (history rows 97 KB, root / dof / sensor / torque /
//    action blocks, packed task-state rows, episode sums) is fetched with a 1-D TMA bulk copy
//    (cp.async.bulk, SASS UBLKCP) completing on one mbarrier: no thread issues a load for them.
//  * The history block is re-emitted with bulk stores straight from shared memory, speculatively
//    and at once: obs_buf[:, 100:860] <- old history (WG:992) and history[:, 0:9] <- history[:, 1:10]
//    (WG:997-1000); they overlap with all the arithmetic.  Envs that turn out to be special this step
//    (reset -> zeros / fill; first step of an episode -> fill; a stored row exceeding clip_obs ->
//    clipped copy) are patched with ordinary stores after the bulk group has completed.
//  * Arithmetic is split by shape instead of one serial chain per env (a serial chain per env was
//    latency bound on a ~4 k-instruction dependent chain, profiles/r1_k1_*).  The passes call the per-env
//    functions of env_step_common.cuh, which the warp-per-env kernel (env_step.cu) shares:
//      - "feature pass": a warp per env, a lane per DOF: the sums over DOFs the reward terms need
//        (dof_features);
//      - "scalar pass": one thread per env (warp 0): quaternion algebra, EE-goal interpolation,
//        command resampling, push, termination, reward combination, episode sums (scalar_step);
//      - "fix-up pass": a warp per env with a rare event -- EE-goal resampling with the collision check
//        spread over lanes, and the reset (fix_up);
//      - "assembly pass": a warp per env, a lane per observation column (assemble_obs).
//  * Dimensions are compile-time (widowGo1: 20 dofs, 18 actions, 76-d proprioception, 10-step
//    history): strides fold into immediate offsets.  Other shapes / shard sizes that are not a
//    multiple of 32 run the warp-per-env kernel (env_step.cu).  -fmad=false like it.
#include "env_step_common.cuh"

namespace dwbc {

constexpr int V2_E = 16;                 // envs per CTA: 16 so that TWO CTAs share an SM (one CTA's bulk loads / stores overlap the other's arithmetic)
constexpr int V2_THREADS = 256;
constexpr int V2_CW = 7;                 // compute warps; warp 7 issues the speculative bulk stores
constexpr int V2_CT = V2_CW * 32;
__device__ __forceinline__ void cbar() { asm volatile("bar.sync 1, %0;" ::"n"(V2_CT) : "memory"); }

// ---- TMA / mbarrier PTX ----------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* dst_gmem, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

template <int ND, int NA, int AH, int P, int H, int NPRIV>
struct V2 {
  static constexpr int HP = H * P;
  static constexpr int CFS = 3 * (4 + 2 * DWBC_MAX_IDX);
  // shared-memory carve-up, float offsets; every TMA block is dense [32][cols] and 16-B aligned
  static constexpr int o_hist = 0;
  static constexpr int o_root = o_hist + V2_E * HP;
  static constexpr int o_dof = o_root + V2_E * 26;
  static constexpr int o_fs = o_dof + V2_E * 2 * ND;
  static constexpr int o_tq = o_fs + V2_E * 24;
  static constexpr int o_act = o_tq + V2_E * ND;
  static constexpr int o_ah = o_act + V2_E * NA;
  static constexpr int o_gs = o_ah + V2_E * AH * NA;
  static constexpr int o_ds = o_gs + V2_E * DWBC_GS;
  static constexpr int o_mass = o_ds + V2_E * DWBC_DS;
  static constexpr int o_fric = o_mass + V2_E * 5;
  static constexpr int o_motor = o_fric + V2_E;
  static constexpr int o_eplen = o_motor + V2_E * NA;
  static constexpr int o_ee = o_eplen + V2_E * 2;
  static constexpr int o_cf = o_ee + V2_E * 8;
  static constexpr int o_prop = o_cf + V2_E * CFS;
  static constexpr int o_priv = o_prop + V2_E * P;
  static constexpr int o_feat = o_priv + V2_E * NPRIV;
  static constexpr int o_out = o_feat + V2_E * FE_COUNT;
  static constexpr int o_rp = o_out + V2_E * 2;        // roll, pitch, yaw, sum of height gaps
  static constexpr int o_flags = o_rp + V2_E * 4;
  static constexpr int o_oob = o_flags + V2_E;
  static constexpr int o_sums = o_oob + V2_E;          // [32][stride], runtime stride, last
  static_assert((V2_E * 26) % 4 == 0 && (V2_E * NA) % 4 == 0 && (V2_E * ND) % 4 == 0 && (V2_E * 5) % 4 == 0 && HP % 4 == 0 && P % 4 == 0 &&
                    NPRIV % 4 == 0, "TMA blocks must be multiples of 16 bytes");
};

static_assert(STEP_ARGS_WORDS <= V2_THREADS, "step_args_to_shared: one word per thread");

template <int ND, int NA, int AH, int P, int H, int NPRIV>
__global__ void __launch_bounds__(V2_THREADS, 2)
env_step_v2_kernel(const __grid_constant__ DwbcEnvCfg cfg, const __grid_constant__ DwbcEnvBuffers B, const __grid_constant__ DwbcStepArgs Ah,
                   const DwbcStepDevice* __restrict__ dev) {
  using Ly = V2<ND, NA, AH, P, H, NPRIV>;
  constexpr int HP = Ly::HP, CFS = Ly::CFS;
  extern __shared__ __align__(128) float sm[];
  __shared__ DwbcStepArgs A;      // this step's arguments: the host's, or with `dev` the device record's step / push / curriculum values
  __shared__ __align__(8) uint64_t bar;
  __shared__ int cta_flags;
  __shared__ int feat_mask;
  __shared__ int ig2r_s[DWBC_MAX_DOF];
  __shared__ float defpos_s[DWBC_MAX_DOF];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int e0 = blockIdx.x * V2_E;
  const int stride = cfg.sums_stride, nbp1 = cfg.num_bodies_p1;
  const int nslots = cfg.n_sum_slots + DWBC_NUM_METRICS;
  float* hist_s = sm + Ly::o_hist;
  float* hist_g = B.obs_history + (size_t)e0 * HP;
  float* sums_s = sm + Ly::o_sums;
  int* flags_s = reinterpret_cast<int*>(sm + Ly::o_flags);
  int* oob_s = reinterpret_cast<int*>(sm + Ly::o_oob);
  long long* ep_s = reinterpret_cast<long long*>(sm + Ly::o_eplen);
  auto view = [&](int e) {
    return EnvView{sm + Ly::o_root + e * 26, sm + Ly::o_dof + e * 2 * ND, sm + Ly::o_fs + e * 24, sm + Ly::o_tq + e * ND, sm + Ly::o_act + e * NA,
                   sm + Ly::o_ah + e * AH * NA, sm + Ly::o_gs + e * DWBC_GS, sm + Ly::o_ds + e * DWBC_DS, sums_s + e * stride, sm + Ly::o_ee + e * 8,
                   sm + Ly::o_cf + e * CFS, sm + Ly::o_mass + e * 5, sm + Ly::o_fric + e, sm + Ly::o_motor + e * NA, sm + Ly::o_prop + e * P,
                   sm + Ly::o_priv + e * NPRIV, sm + Ly::o_feat + e * FE_COUNT, sm + Ly::o_rp + 4 * e, sm + Ly::o_out + 2 * e};
  };

  step_args_to_shared(Ah, dev, &A, tid);   // (ordered before every use by the barrier below)
  // ---- 1. TMA loads ------------------------------------------------------------------------------
  if (tid == 0) {
    mbar_init(&bar, 1);
    cta_flags = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    constexpr uint32_t b_hist = V2_E * HP * 4, b_root = V2_E * 26 * 4, b_dof = V2_E * 2 * ND * 4, b_fs = V2_E * 24 * 4, b_tq = V2_E * ND * 4,
                       b_act = V2_E * NA * 4, b_ah = V2_E * AH * NA * 4, b_gs = V2_E * DWBC_GS * 4, b_ds = V2_E * DWBC_DS * 4,
                       b_mass = V2_E * 5 * 4, b_fric = V2_E * 4, b_motor = V2_E * NA * 4, b_ep = V2_E * 8;
    const uint32_t b_sum = V2_E * stride * 4;
    mbar_expect_tx(&bar, b_hist + b_root + b_dof + b_fs + b_tq + b_act + b_ah + b_gs + b_ds + b_sum + b_mass + b_fric + b_motor + b_ep);
    bulk_g2s(sm + Ly::o_root, B.root_states + (size_t)e0 * 26, b_root, &bar);
    bulk_g2s(sm + Ly::o_dof, B.dof_state + (size_t)e0 * 2 * ND, b_dof, &bar);
    bulk_g2s(sm + Ly::o_fs, B.force_sensor + (size_t)e0 * 24, b_fs, &bar);
    bulk_g2s(sm + Ly::o_tq, B.torques + (size_t)e0 * ND, b_tq, &bar);
    bulk_g2s(sm + Ly::o_act, B.actions + (size_t)e0 * NA, b_act, &bar);
    bulk_g2s(sm + Ly::o_ah, B.action_history + (size_t)e0 * AH * NA, b_ah, &bar);
    bulk_g2s(sm + Ly::o_gs, B.goal_state + (size_t)e0 * DWBC_GS, b_gs, &bar);
    bulk_g2s(sm + Ly::o_ds, B.derived_state + (size_t)e0 * DWBC_DS, b_ds, &bar);
    bulk_g2s(sums_s, B.episode_sums + (size_t)e0 * stride, b_sum, &bar);
    bulk_g2s(sm + Ly::o_mass, B.mass_params + (size_t)e0 * 5, b_mass, &bar);
    bulk_g2s(sm + Ly::o_fric, B.friction + e0, b_fric, &bar);
    bulk_g2s(sm + Ly::o_motor, B.motor_strength + (size_t)e0 * NA, b_motor, &bar);
    bulk_g2s(sm + Ly::o_eplen, B.episode_length + e0, b_ep, &bar);
    bulk_g2s(hist_s, hist_g, b_hist, &bar);
  }
  // ---- 2. gathers that are not contiguous per CTA (gripper body row, contact bodies) ------------
  {
    for (int i = tid; i < V2_E * 8; i += V2_THREADS) {
      int e = i >> 3, k = i & 7;
      sm[Ly::o_ee + i] = k < 7 ? __ldg(B.rigid_body_state + ((size_t)(e0 + e) * nbp1 + cfg.gripper_idx) * 13 + k) : 0.0f;
    }
    const int ncf = 4 + cfg.n_penalized + cfg.n_term_contact;
    for (int i = tid; i < V2_E * 3 * ncf; i += V2_THREADS) {
      int e = i / (3 * ncf), r = i - e * 3 * ncf, b = r / 3, k = r - 3 * b;
      int body = b < 4 ? cfg.feet_idx[b] : (b < 4 + cfg.n_penalized ? cfg.penalized_idx[b - 4] : cfg.term_contact_idx[b - 4 - cfg.n_penalized]);
      sm[Ly::o_cf + e * CFS + r] = __ldg(B.contact_forces + ((size_t)(e0 + e) * nbp1 + body) * 3 + k);
    }
    if (tid < V2_E) { sm[Ly::o_rp + 4 * tid + 3] = 0.0f; oob_s[tid] = 0; }
    if (tid < ND) { ig2r_s[tid] = cfg.ig2raisim[tid]; defpos_s[tid] = cfg.default_dof_pos[tid]; }
    if (tid == 64) feat_mask = feature_mask(cfg);
  }
  mbar_wait(&bar, 0);
  __syncthreads();

  const float c = cfg.clip_obs > 0.0f ? cfg.clip_obs : INFINITY;
  constexpr int p4 = P >> 2, pp4 = (P + NPRIV) >> 2, nh4 = HP >> 2;
  // ---- 3. speculative bulk re-emission of the history block: warp 7 is the dedicated store issuer -----
  // (the TMA store queue back-pressures the issuing thread for ~10 k cycles; keep it off the compute warps)
  if (wid == V2_CW) {
    if (lane == 0) {
      for (int e = 0; e < V2_E; ++e) {
        bulk_s2g(B.obs_buf + (size_t)(e0 + e) * B.obs_stride + (P + NPRIV), hist_s + e * HP, HP * 4);   // WG:992 (old history)
        bulk_s2g(hist_g + (size_t)e * HP, hist_s + e * HP + P, (HP - P) * 4);                           // WG:997-999 (shift)
      }
      bulk_commit();
      bulk_wait_all();
    }
  } else {
  // ---- 4. height scan: warp per env ----------------------------------------------------------------
  if (cfg.measure_heights) {
    for (int e = wid; e < V2_E; e += V2_CW) {
      const float gap = height_scan(cfg, B, sm + Ly::o_root + e * 26, e0 + e, lane);
      if (lane == 0) sm[Ly::o_rp + 4 * e + 3] = gap;
    }
  }
  // ---- 5. feature pass: warp per env, lane per DOF, only the reductions an active term needs -------
  for (int e = wid; e < V2_E; e += V2_CW) dof_features(cfg, view(e), feat_mask, defpos_s, ND, NA, lane);
  cbar();

  // assembly of one env's observation columns: part 0 by warps 1..6 WHILE warp 0 runs the scalar pass, part 1 after the fix-up pass
  auto assemble = [&](const int e, const int part) {
    if (assemble_obs(cfg, view(e), part, ig2r_s, defpos_s, c, ND, NA, AH, lane) && lane == 0) oob_s[e] = 1;
  };

  // ---- 6. scalar pass: thread per env (warp 0); warps 1..6 assemble the simulator-only observation columns meanwhile ----
  if (wid >= 1 && wid < V2_CW) {
    for (int e = wid - 1; e < V2_E; e += V2_CW - 1) assemble(e, 0);
  }
  if (tid < V2_E) {
    const long long ep = ep_s[tid] + 1;                                                   // WG:875
    flags_s[tid] = scalar_step(cfg, A, view(tid), e0 + tid, ep);
    ep_s[tid] = ep;
  }
  cbar();

  // ---- 7. fix-up pass: rare events, one warp per flagged env ------------------------------------
  const unsigned fix_list = __ballot_sync(FULL, lane < V2_E && (flags_s[lane] & (F_GOAL_RS | F_RESET)) != 0);   // same value in every warp
  for (int k = wid; k < __popc(fix_list); k += V2_CW) {
    const int e = __fns(fix_list, 0, k + 1);    // k-th flagged env: flagged envs are dealt round-robin to the warps
    const int f = fix_up(cfg, A, B, view(e), flags_s[e], e0 + e, ND, NA, AH, nslots, lane);
    if (lane == 0 && (f & F_RESET)) { flags_s[e] = f; ep_s[e] = 0; }
  }
  cbar();

  // ---- 8. assembly pass, second half: a reset env is re-assembled from its post-reset state first -------------
  for (int e = wid; e < V2_E; e += V2_CW) {
    if (flags_s[e] & F_RESET) {
      if (lane == 0) oob_s[e] = 0;
      __syncwarp();
      assemble(e, 0);
    }
    assemble(e, 1);
  }
  cbar();
  if (tid < V2_E) {
    float* ds = sm + Ly::o_ds + tid * DWBC_DS;
    int f = flags_s[tid];
    const float age = ds[DWBC_DS_OOB_AGE];
    if (age < (float)H) f |= F_OOB;   // a stored history row may exceed the clip: patch obs with the clipped copy
    ds[DWBC_DS_OOB_AGE] = oob_s[tid] ? 0.0f : ((f & F_FILL) ? (float)H : fminf(age + 1.0f, 1.0e6f));
    flags_s[tid] = f;
    if (f & (F_ROOT_DIRTY | F_DOF_DIRTY)) atomicOr(&cta_flags, f & (F_ROOT_DIRTY | F_DOF_DIRTY));
  }
  fence_async_smem();  // generic-proxy writes to the state rows must be visible to the bulk stores below
  cbar();

  // ---- 9. write-out ------------------------------------------------------------------------------
  if (tid == 0) {
    bulk_s2g(B.goal_state + (size_t)e0 * DWBC_GS, sm + Ly::o_gs, V2_E * DWBC_GS * 4);
    bulk_s2g(B.derived_state + (size_t)e0 * DWBC_DS, sm + Ly::o_ds, V2_E * DWBC_DS * 4);
    bulk_s2g(B.episode_sums + (size_t)e0 * stride, sums_s, V2_E * stride * 4);
    bulk_s2g(B.episode_length + e0, sm + Ly::o_eplen, V2_E * 8);
    if (cta_flags & F_ROOT_DIRTY) bulk_s2g(B.root_states + (size_t)e0 * 26, sm + Ly::o_root, V2_E * 26 * 4);
    if (cta_flags & F_DOF_DIRTY) {
      bulk_s2g(B.dof_state + (size_t)e0 * 2 * ND, sm + Ly::o_dof, V2_E * 2 * ND * 4);
      bulk_s2g(B.action_history + (size_t)e0 * AH * NA, sm + Ly::o_ah, V2_E * AH * NA * 4);
    }
    bulk_commit();
  }
  for (int i = tid; i < V2_E * pp4; i += V2_CT) {  // obs[:, 0:100] = clip([prop | priv]); history[:, -1] = prop
    const int e = i / pp4, j = i - e * pp4;
    const float4 v = j < p4 ? reinterpret_cast<const float4*>(sm + Ly::o_prop + e * P)[j]
                            : reinterpret_cast<const float4*>(sm + Ly::o_priv + e * NPRIV)[j - p4];
    stg_stream(reinterpret_cast<float4*>(B.obs_buf + (size_t)(e0 + e) * B.obs_stride) + j, clip4(v, c));
    if (j < p4) reinterpret_cast<float4*>(hist_g + (size_t)e * HP + (HP - P))[j] = v;
  }
  if (tid < V2_E) store_step(B, e0 + tid, flags_s[tid], sm[Ly::o_out + 2 * tid], sm[Ly::o_out + 2 * tid + 1]);
  store_heights_obs(cfg, B, e0, V2_E, sm + Ly::o_root, tid, V2_CT);
  }  // compute warps
  // ---- 10. patch the special envs after the speculative bulk stores have completed (warp 7 waited) ----
  __syncthreads();
  for (int e = wid; e < V2_E; e += V2_THREADS / 32) {
    const int f = flags_s[e];
    if (!(f & (F_RESET | F_FILL | F_OOB))) continue;
    float4* obs4 = reinterpret_cast<float4*>(B.obs_buf + (size_t)(e0 + e) * B.obs_stride) + pp4;
    const float4* h4 = reinterpret_cast<const float4*>(hist_s + e * HP);
    for (int i = lane; i < nh4; i += 32) obs4[i] = (f & F_RESET) ? make_float4(0.f, 0.f, 0.f, 0.f) : clip4(h4[i], c);
    if (f & F_FILL) {
      const float4* prop4 = reinterpret_cast<const float4*>(sm + Ly::o_prop + e * P);
      float4* hg4 = reinterpret_cast<float4*>(hist_g + (size_t)e * HP);
      for (int i = lane; i < nh4; i += 32) hg4[i] = prop4[i % p4];
    }
  }
  if (tid == 0) bulk_wait_all();  // smem must stay alive until the state-row bulk stores have read it
}

}  // namespace dwbc

using namespace dwbc;

// launcher used by dwbc_post_physics_step (env_step.cu); DWBC_ERR_UNSUPPORTED -> caller runs the warp-per-env kernel
int dwbc_launch_env_step_v2(const DwbcEnvCfg* cfg, const DwbcEnvBuffers* buf, const DwbcStepArgs* args, const DwbcStepDevice* dev, cudaStream_t st) {
  using K = V2<20, 18, 4, 76, 10, 24>;
  if (cfg->num_dofs != 20 || cfg->num_actions != 18 || cfg->action_hist_len != 4 || cfg->num_prop != 76 || cfg->history_len != 10 ||
      cfg->num_priv != 24 || (cfg->sums_stride & 3) || cfg->n_collision_samples > 16)
    return DWBC_ERR_UNSUPPORTED;
  const size_t smem = (size_t)(K::o_sums + V2_E * cfg->sums_stride) * sizeof(float);
  if (smem > 110 * 1024) return DWBC_ERR_UNSUPPORTED;      // two CTAs per SM
  auto kern = env_step_v2_kernel<20, 18, 4, 76, 10, 24>;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 110 * 1024) != cudaSuccess) return DWBC_ERR_LAUNCH;
    attr_set = true;
  }
  kern<<<cfg->num_envs / V2_E, V2_THREADS, smem, st>>>(*cfg, *buf, *args, dev);
  DWBC_LAUNCH_CHECK();
  return DWBC_OK;
}
