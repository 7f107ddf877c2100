// Fused widowGo1 post-physics step, v2: ONE launch per sim step, 16 envs per CTA, TMA-fed.
//
//  * Every contiguous block of the CTA's 32 envs (history rows 97 KB, root / dof / sensor / torque /
//    action blocks, packed task-state rows, episode sums) is fetched with a 1-D TMA bulk copy
//    (cp.async.bulk, SASS UBLKCP) completing on one mbarrier: no thread issues a load for them.
//  * The history block is re-emitted with bulk stores straight from shared memory, speculatively
//    and at once: obs_buf[:, 100:860] <- old history (WG:992) and history[:, 0:9] <- history[:, 1:10]
//    (WG:997-1000); they overlap with all the arithmetic.  Envs that turn out to be special this step
//    (reset -> zeros / fill; first step of an episode -> fill; a stored row exceeding clip_obs ->
//    clipped copy) are patched with ordinary stores after the bulk group has completed.
//  * Arithmetic is split by shape instead of one serial chain per env (the v1 / first-v2 profiles were
//    latency bound on a ~4 k-instruction dependent chain, profiles/r1_k1_*):
//      - "feature pass": all 256 threads, one (env, DOF-reduction) pair each: the sums over DOFs the
//        reward terms need (WG:1396-1469, LR:853-886);
//      - "scalar pass": one thread per env (warp 0): quaternion algebra, EE-goal interpolation,
//        command resampling, push, termination, reward combination, episode sums;
//      - "fix-up pass": warp-cooperative handling of the rare events -- EE-goal resampling with the
//        10-sample collision check spread over lanes (WG:1316-1342) and the reset (WG:695-754);
//      - "assembly pass": all threads, one observation column each (WG:966-1001), plus the
//        last_actions / last_dof_vel / last_root_vel copies (WG:908-910).
//  * Dimensions are compile-time (widowGo1: 20 dofs, 18 actions, 76-d proprioception, 10-step
//    history): strides fold into immediate offsets.  Other shapes / shard sizes that are not a
//    multiple of 32 run the generic v1 kernel (env_step.cu).  -fmad=false as in v1.
#include "env_math.cuh"

namespace dwbc {

constexpr int V2_E = 16;                 // envs per CTA: 16 so that TWO CTAs share an SM (one CTA's bulk loads / stores overlap the other's arithmetic)
constexpr int V2_THREADS = 256;
constexpr int V2_CW = 7;                 // compute warps; warp 7 issues the speculative bulk stores
constexpr int V2_CT = V2_CW * 32;
__device__ __forceinline__ void cbar() { asm volatile("bar.sync 1, %0;" ::"n"(V2_CT) : "memory"); }
#define DWBC_DS_OOB_AGE 27 /* derived_state pad column: #most-recent history rows known to be within +-clip_obs */

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

// Philox stream with a one-block cache: consecutive columns share a Philox4x32-10 evaluation.
struct RngC {
  const float* table;
  uint64_t seed, step;
  int env, blk;
  uint4 cur;
  __device__ __forceinline__ float operator()(int col) {
    if (table) return __ldg(table + (size_t)env * DWBC_RAND_COLS + col);
    const int b = col >> 2;
    if (b != blk) {
      cur = philox4x32_10(make_uint4((uint32_t)env, (uint32_t)b, (uint32_t)step, (uint32_t)(step >> 32)),
                          make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
      blk = b;
    }
    const int k = col & 3;
    return u01(k == 0 ? cur.x : (k == 1 ? cur.y : (k == 2 ? cur.z : cur.w)));
  }
};

enum { F_RESET = 1, F_TIMEOUT = 2, F_FILL = 4, F_OOB = 8, F_ROOT_DIRTY = 16, F_DOF_DIRTY = 32, F_GOAL_RS = 64 };
enum { FE_ENERGY_SQ = 0, FE_LEG_ABS, FE_LEG_SUM, FE_ARM_ABS, FE_TORQUE_SQ, FE_DOFVEL_SQ, FE_DOF_ACC, FE_ACT_RATE, FE_HIP_L2, FE_LEG_L2,
       FE_FOOT_Z, FE_POS_LIM, FE_VEL_LIM, FE_TQ_LIM, FE_STAND, FE_COUNT = 16 };

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

// Warp-wide uniform stream for the fix-up pass: lane b holds Philox block b (columns 4b..4b+3) of this env and step,
// evaluated once; any lane reads any column with one shuffle.  MUST be called by all 32 lanes (col may differ per lane).
struct RngW {
  const float* table;
  int env;
  uint4 mine;
  __device__ __forceinline__ float operator()(int col) const {
    if (table) return __ldg(table + (size_t)env * DWBC_RAND_COLS + col);
    const int src = col >> 2, k = col & 3;
    const uint32_t x = __shfl_sync(FULL, mine.x, src), y = __shfl_sync(FULL, mine.y, src), z = __shfl_sync(FULL, mine.z, src),
                   w = __shfl_sync(FULL, mine.w, src);
    return u01(k == 0 ? x : (k == 1 ? y : (k == 2 ? z : w)));
  }
};

// warp-cooperative EE-goal resampling (WG:1316-1332); collision samples spread over lanes (WG:1337-1342)
// Word `tid` of the step arguments a kernel works with: the host's DwbcStepArgs, except that with a device record (CUDA-graph replay) the
// step, the push decision (WG:934) and the curriculum values come from that record.  Threads 0 .. sizeof(DwbcStepArgs) / 4 - 1 take part.
static_assert(offsetof(DwbcStepArgs, generic_kernel) - offsetof(DwbcStepArgs, lin_vel_x) == sizeof(DwbcStepDevice) - offsetof(DwbcStepDevice, lin_vel_x),
              "the curriculum block of DwbcStepDevice mirrors the one of DwbcStepArgs");
static_assert(sizeof(DwbcStepArgs) / 4 <= V2_THREADS && sizeof(DwbcStepArgs) % 4 == 0, "one word per thread");
__device__ __forceinline__ void step_args_to_shared(const DwbcStepArgs& h, const DwbcStepDevice* d, DwbcStepArgs* out, int tid) {
  constexpr int NW = sizeof(DwbcStepArgs) / 4, W_STEP = offsetof(DwbcStepArgs, step) / 4, W_PUSH = offsetof(DwbcStepArgs, do_push) / 4;
  constexpr int W_CUR0 = offsetof(DwbcStepArgs, lin_vel_x) / 4, W_CUR1 = offsetof(DwbcStepArgs, generic_kernel) / 4;
  if (tid >= NW) return;
  uint32_t v = reinterpret_cast<const uint32_t*>(&h)[tid];
  if (d) {
    const uint64_t step = d->step;
    if (tid >= W_CUR0 && tid < W_CUR1) v = reinterpret_cast<const uint32_t*>(d->lin_vel_x)[tid - W_CUR0];
    else if (tid == W_STEP) v = (uint32_t)step;
    else if (tid == W_STEP + 1) v = (uint32_t)(step >> 32);
    else if (tid == W_PUSH) v = (d->push_interval > 0 && step % (uint64_t)d->push_interval == 0) ? 1u : 0u;
  }
  reinterpret_cast<uint32_t*>(out)[tid] = v;
}

__device__ void coop_resample_goal(const DwbcEnvCfg& cfg, const DwbcStepArgs& A, const RngW& rng, float* gs, float yaw, int col_orn, int col_sph,
                                   bool do_orn, int lane) {
  {
    const int l3 = lane < 3 ? lane : 0;
    const float u = rng(col_orn + l3);
    if (do_orn && lane < 3) {
      float d = cfg.delta_orn_span[lane] * u + cfg.delta_orn_lo[lane];
      gs[DWBC_GS_DELTA_ORN + lane] = d;
      gs[DWBC_GS_GOAL_ORN + lane] = wrap_pi(d + (lane == 2 ? yaw : 0.0f));
    }
  }
  V3 start = mk(gs[DWBC_GS_GOAL_SPH], gs[DWBC_GS_GOAL_SPH + 1], gs[DWBC_GS_GOAL_SPH + 2]);
  __syncwarp();
  // The reference tries up to max_goal_tries samples one after the other and keeps the first one whose interpolation path is
  // collision free (else the last one).  The uniforms of try k do not depend on earlier tries, so several tries are evaluated
  // per round, one (try, path sample) pair per lane, and the lowest passing try wins: same result, 4 rounds instead of 10 in
  // the worst case (the slowest CTA of the launch sets the kernel time).
  V3 goal = start;
  const int ns = cfg.n_collision_samples > 0 ? (cfg.n_collision_samples < 32 ? cfg.n_collision_samples : 32) : 1;
  const int tpr = 32 / ns;                                   // tries per round
  const int my_t = lane / ns, my_s = lane - my_t * ns;       // lane -> (try within the round, path sample)
  bool done = false;
  for (int k0 = 0; k0 < cfg.max_goal_tries && !done; k0 += tpr) {
    const int k = k0 + my_t;
    const bool active = my_t < tpr && k < cfg.max_goal_tries;
    const int kc = active ? k : k0;                          // inactive lanes still take part in the shuffles of rng()
    const V3 g = mk(A.goal_l[1] * rng(col_sph + 3 * kc) + A.goal_l[0], A.goal_p[1] * rng(col_sph + 3 * kc + 1) + A.goal_p[0],
                    A.goal_y[1] * rng(col_sph + 3 * kc + 2) + A.goal_y[0]);
    bool hit = false;
    if (active && cfg.n_collision_samples > 0) {
      V3 p = sphere2cart(lerp3(start, g, cfg.collision_t[my_s]));
      bool inside = (p.x < cfg.collision_upper[0] && p.y < cfg.collision_upper[1] && p.z < cfg.collision_upper[2]) &&
                    (p.x > cfg.collision_lower[0] && p.y > cfg.collision_lower[1] && p.z > cfg.collision_lower[2]);
      hit = inside || (p.z < cfg.underground_limit);
    }
    const unsigned hits = __ballot_sync(FULL, hit);
    int win = -1, last = 0;
    for (int t = 0; t < tpr && k0 + t < cfg.max_goal_tries; ++t) {
      const unsigned m = (ns == 32 ? FULL : ((1u << ns) - 1u)) << (t * ns);
      last = t;
      if (win < 0 && (hits & m) == 0) win = t;
    }
    const int src = (win >= 0 ? win : last) * ns;            // first lane of the winning (or, so far, the last) try
    goal = mk(__shfl_sync(FULL, g.x, src), __shfl_sync(FULL, g.y, src), __shfl_sync(FULL, g.z, src));
    done = win >= 0;
  }
  if (lane == 0) {
    V3 gc = sphere2cart(goal);
    gs[DWBC_GS_START_SPH] = start.x; gs[DWBC_GS_START_SPH + 1] = start.y; gs[DWBC_GS_START_SPH + 2] = start.z;
    gs[DWBC_GS_GOAL_SPH] = goal.x; gs[DWBC_GS_GOAL_SPH + 1] = goal.y; gs[DWBC_GS_GOAL_SPH + 2] = goal.z;
    gs[DWBC_GS_GOAL_CART] = gc.x; gs[DWBC_GS_GOAL_CART + 1] = gc.y; gs[DWBC_GS_GOAL_CART + 2] = gc.z;
    gs[DWBC_GS_GOAL_TIMER] = 0.0f;
  }
  __syncwarp();
}

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
    if (tid == 64) {  // which DOF reductions do the active terms need?
      int m = 0;
      for (int ch = 0; ch < 2; ++ch) {
        const int n = ch == 0 ? cfg.n_leg_terms : cfg.n_arm_terms;
        const int32_t* terms = ch == 0 ? cfg.leg_term : cfg.arm_term;
        for (int i = 0; i < n; ++i) {
          switch (terms[i]) {
            case DWBC_TERM_energy_square: m |= 1 << FE_ENERGY_SQ; break;
            case DWBC_TERM_leg_energy_abs_sum: m |= 1 << FE_LEG_ABS; break;
            case DWBC_TERM_leg_energy_sum_abs: case DWBC_TERM_leg_energy: m |= 1 << FE_LEG_SUM; break;
            case DWBC_TERM_arm_energy_abs_sum: m |= 1 << FE_ARM_ABS; break;
            case DWBC_TERM_torques: m |= 1 << FE_TORQUE_SQ; break;
            case DWBC_TERM_dof_vel: m |= 1 << FE_DOFVEL_SQ; break;
            case DWBC_TERM_dof_acc: m |= 1 << FE_DOF_ACC; break;
            case DWBC_TERM_action_rate: m |= 1 << FE_ACT_RATE; break;
            case DWBC_TERM_hip_action_l2: m |= 1 << FE_HIP_L2; break;
            case DWBC_TERM_leg_action_l2: m |= 1 << FE_LEG_L2; break;
            case DWBC_TERM_foot_contacts_z: m |= 1 << FE_FOOT_Z; break;
            case DWBC_TERM_dof_pos_limits: m |= 1 << FE_POS_LIM; break;
            case DWBC_TERM_dof_vel_limits: m |= 1 << FE_VEL_LIM; break;
            case DWBC_TERM_torque_limits: m |= 1 << FE_TQ_LIM; break;
            case DWBC_TERM_stand_still: m |= 1 << FE_STAND; break;
            default: break;
          }
        }
      }
      feat_mask = m;
    }
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
  // ---- 4. height scan (LR:793-829): warp per env, lane per point, gap sum by warp reduction ---------
  if (cfg.measure_heights) {
    const int npts = cfg.n_height_x * cfg.n_height_y;
    for (int e = wid; e < V2_E; e += V2_CW) {
      const float* root = sm + Ly::o_root + e * 26;
      float qy[4] = {0.0f, 0.0f, root[5], root[6]};
      const float n = fmaxf(nsqrt(qy[2] * qy[2] + qy[3] * qy[3]), 1e-9f);     // utils/math.py:38-42 + normalize()
      qy[2] = qy[2] / n; qy[3] = qy[3] / n;
      const float rx = root[0], ry = root[1], rz = root[2];
      float gap = 0.0f;
      float* out = B.measured_heights + (size_t)(e0 + e) * npts;
#pragma unroll 2
      for (int j = lane; j < npts; j += 32) {
        const int ix = j / cfg.n_height_y, iy = j - ix * cfg.n_height_y;
        const V3 pt = quat_apply(qy, mk(cfg.height_x[ix], cfg.height_y[iy], 0.0f));
        const float fx = ((pt.x + rx) + cfg.border_size) / cfg.horizontal_scale;
        const float fy = ((pt.y + ry) + cfg.border_size) / cfg.horizontal_scale;
        long long px = (long long)fx, py = (long long)fy;                   // .long(): truncation toward zero
        px = px < 0 ? 0 : (px > cfg.terrain_rows - 2 ? cfg.terrain_rows - 2 : px);
        py = py < 0 ? 0 : (py > cfg.terrain_cols - 2 ? cfg.terrain_cols - 2 : py);
        const int16_t* hs = B.height_samples + px * cfg.terrain_cols + py;
        const int16_t m = min(min(__ldg(hs), __ldg(hs + cfg.terrain_cols)), __ldg(hs + 1));
        const float hgt = (float)m * cfg.vertical_scale;
        out[j] = hgt;
        gap += rz - hgt;
      }
      gap = warp_sum(gap);
      if (lane == 0) sm[Ly::o_rp + 4 * e + 3] = gap;
    }
  }
  // ---- 5. feature pass: warp per env, lane per DOF, only the reductions an active term needs -------
  for (int e = wid; e < V2_E; e += V2_CW) {
    const float tq = lane < ND ? sm[Ly::o_tq + e * ND + lane] : 0.0f;
    const float dv = lane < ND ? sm[Ly::o_dof + e * 2 * ND + 2 * lane + 1] : 0.0f;
    const float dp = lane < ND ? sm[Ly::o_dof + e * 2 * ND + 2 * lane] : 0.0f;
    const float act = lane < NA ? sm[Ly::o_act + e * NA + lane] : 0.0f;
    const float* ds = sm + Ly::o_ds + e * DWBC_DS;
    float* feat = sm + Ly::o_feat + e * FE_COUNT;
    const float pw = lane < 12 ? tq * dv : 0.0f;
    const int need = feat_mask;
#define FEAT(k, expr) if (need & (1 << (k))) { float r_ = warp_sum(expr); if (lane == 0) feat[k] = r_; }
    FEAT(FE_ENERGY_SQ, pw * pw)                                                                           // WG:1466
    FEAT(FE_LEG_ABS, fabsf(pw))                                                                           // WG:1396
    FEAT(FE_LEG_SUM, pw)                                                                                  // WG:1401,1410
    FEAT(FE_ARM_ABS, (lane >= 12 && lane < ND - 2) ? fabsf(tq * dv) : 0.0f)                               // WG:1414
    FEAT(FE_TORQUE_SQ, tq * tq)                                                                           // WG:1460
    FEAT(FE_DOFVEL_SQ, dv * dv)                                                                           // LR:853
    if (need & (1 << FE_DOF_ACC)) { float a = lane < ND ? (ds[DWBC_DS_LAST_DOF_VEL + lane] - dv) / cfg.dt : 0.0f; a = warp_sum(a * a); if (lane == 0) feat[FE_DOF_ACC] = a; }
    if (need & (1 << FE_ACT_RATE)) { float a = lane < NA ? ds[DWBC_DS_LAST_ACTIONS + lane] - act : 0.0f; a = warp_sum(a * a); if (lane == 0) feat[FE_ACT_RATE] = a; }
    FEAT(FE_HIP_L2, (lane < 12 && lane % 3 == 0) ? act * act : 0.0f)                                      // WG:1379
    FEAT(FE_LEG_L2, lane < 12 ? act * act : 0.0f)                                                         // WG:1405
    if (need & (1 << FE_FOOT_Z)) { float z = lane < 4 ? sm[Ly::o_fs + e * 24 + 6 * lane + 2] : 0.0f; z = warp_sum(z * z); if (lane == 0) feat[FE_FOOT_Z] = z; }
    FEAT(FE_POS_LIM, lane < ND ? -fminf(dp - cfg.dof_pos_lower[lane], 0.0f) + fmaxf(dp - cfg.dof_pos_upper[lane], 0.0f) : 0.0f)
    FEAT(FE_VEL_LIM, lane < ND ? clipf(fabsf(dv) - cfg.dof_vel_limits[lane] * cfg.soft_dof_vel_limit, 0.0f, 1.0f) : 0.0f)
    FEAT(FE_TQ_LIM, lane < ND ? fmaxf(fabsf(tq) - cfg.torque_limits[lane] * cfg.soft_torque_limit, 0.0f) : 0.0f)
    FEAT(FE_STAND, lane < ND ? fabsf(dp - defpos_s[lane]) : 0.0f)
#undef FEAT
  }
  cbar();

  // ---- assembly of one env's observation columns (WG:966-1001, Appendix B): warp per env, lane per column.
  // part 0 = columns that depend only on the simulator state (joint positions / velocities, last action, foot contacts,
  // privileged mass / friction / motor strength): assembled by warps 1..6 WHILE warp 0 runs the scalar pass;
  // part 1 = columns produced by the scalar / fix-up passes (roll-pitch, angular velocity, commands, goal, root velocity).
  auto assemble = [&](const int e, const int part) {
    const float* dof = sm + Ly::o_dof + e * 2 * ND;
    const float* gs = sm + Ly::o_gs + e * DWBC_GS;
    float* ds = sm + Ly::o_ds + e * DWBC_DS;
    float* prop = sm + Ly::o_prop + e * P;
    float* priv = sm + Ly::o_priv + e * NPRIV;
    bool bad = false;
    if (part == 0) {
      if (lane < ND) {            // dof position / velocity columns, last_dof_vel
        const int d = ig2r_s[lane];
        float pos = dof[2 * d];
        if (d == cfg.waist_dof) pos = wrap_pi(pos);
        const float v0 = (pos - defpos_s[d]) * cfg.obs_scale_dof_pos, v1 = dof[2 * d + 1] * cfg.obs_scale_dof_vel;
        prop[5 + lane] = v0;
        prop[5 + ND + lane] = v1;
        bad = !(fabsf(v0) <= c) || !(fabsf(v1) <= c);
        ds[DWBC_DS_LAST_DOF_VEL + lane] = dof[2 * lane + 1];
      }
      if (lane < NA) {            // last applied action column, last_actions, motor strength
        const float v = sm[Ly::o_ah + e * AH * NA + (AH - 1) * NA + ig2r_s[lane]];
        prop[5 + 2 * ND + lane] = v;
        bad = bad || !(fabsf(v) <= c);
        ds[DWBC_DS_LAST_ACTIONS + lane] = sm[Ly::o_act + e * NA + lane];
        priv[6 + lane] = sm[Ly::o_motor + e * NA + lane] - 1.0f;
      }
    }
    {
      constexpr int o = 5 + 2 * ND + NA;
      float v = 0.0f;
      int col = -1;
      if (part == 0) {
        if (lane < 4) {           // foot contacts (WG:1090-1098)
          const float* f = sm + Ly::o_fs + e * 24 + 6 * (lane == 0 ? cfg.feet_perm[0] : (lane == 1 ? cfg.feet_perm[1] : (lane == 2 ? cfg.feet_perm[2] : cfg.feet_perm[3])));
          float nrm = nsqrt(((((f[0] * f[0] + f[1] * f[1]) + f[2] * f[2]) + f[3] * f[3]) + f[4] * f[4]) + f[5] * f[5]);
          v = nrm > 1.5f ? 1.0f : 0.0f; col = o + lane;
        } else if (lane >= 18 && lane < 23) priv[lane - 18] = sm[Ly::o_mass + e * 5 + lane - 18];
        else if (lane == 23) priv[5] = sm[Ly::o_fric + e];
      } else {
        if (lane >= 4 && lane < 6) { v = sm[Ly::o_rp + 4 * e + lane - 4]; col = lane - 4; }
        else if (lane >= 6 && lane < 9) { v = ds[DWBC_DS_BASE_ANG_VEL + lane - 6] * cfg.obs_scale_ang_vel; col = 2 + lane - 6; }
        else if (lane >= 9 && lane < 11) { v = gs[lane - 9] * cfg.obs_scale_lin_vel; col = o + 4 + lane - 9; }
        else if (lane == 11) { v = gs[2] * cfg.obs_scale_ang_vel; col = o + 6; }
        else if (lane >= 12 && lane < 15) { v = gs[(cfg.goal_is_cart ? DWBC_GS_CURR_CART : DWBC_GS_CURR_SPH) + lane - 12]; col = o + 7 + lane - 12; }
        else if (lane >= 15 && lane < 18) { v = gs[DWBC_GS_DELTA_ORN + lane - 15]; col = o + 10 + lane - 15; }
        else if (lane >= 24 && lane < 30) ds[DWBC_DS_LAST_ROOT_VEL + lane - 24] = sm[Ly::o_root + e * 26 + 7 + lane - 24];   // WG:908-910
      }
      if (col >= 0) { prop[col] = v; bad = bad || !(fabsf(v) <= c); }
    }
    if (__any_sync(FULL, bad) && lane == 0) oob_s[e] = 1;
  };

  // ---- 6. scalar pass: thread per env (warp 0); warps 1..6 assemble the simulator-only observation columns meanwhile ----
  if (wid >= 1 && wid < V2_CW) {
    for (int e = wid - 1; e < V2_E; e += V2_CW - 1) assemble(e, 0);
  }
  if (tid < V2_E) {
    const int e = tid, env = e0 + e;
    float* root = sm + Ly::o_root + e * 26;
    float* gs = sm + Ly::o_gs + e * DWBC_GS;
    float* ds = sm + Ly::o_ds + e * DWBC_DS;
    float* sums = sums_s + e * stride;
    float* met = sums + cfg.n_sum_slots;
    const float* feat = sm + Ly::o_feat + e * FE_COUNT;
    const float* ee = sm + Ly::o_ee + e * 8;
    const float* cf = sm + Ly::o_cf + e * CFS;
    RngC rng{A.rand_uniform, A.seed, A.step, env, -1, make_uint4(0, 0, 0, 0)};
    const long long ep = ep_s[e] + 1;                                                     // WG:875
    int flags = 0;
    float r0, p0, yaw;
    {  // derived base state (WG:879-884)
      V3 blv = quat_rotate_inverse(root + 3, mk(root[7], root[8], root[9]));
      V3 bav = quat_rotate_inverse(root + 3, mk(root[10], root[11], root[12]));
      euler_from_quat(root + 3, r0, p0, yaw);
      ds[DWBC_DS_BASE_LIN_VEL] = blv.x; ds[DWBC_DS_BASE_LIN_VEL + 1] = blv.y; ds[DWBC_DS_BASE_LIN_VEL + 2] = blv.z;
      ds[DWBC_DS_BASE_ANG_VEL] = bav.x; ds[DWBC_DS_BASE_ANG_VEL + 1] = bav.y; ds[DWBC_DS_BASE_ANG_VEL + 2] = bav.z;
      ds[DWBC_DS_YAW_EULER] = 0.0f; ds[DWBC_DS_YAW_EULER + 1] = 0.0f; ds[DWBC_DS_YAW_EULER + 2] = yaw;
      ds[DWBC_DS_YAW_QUAT] = 0.0f; ds[DWBC_DS_YAW_QUAT + 1] = 0.0f; ds[DWBC_DS_YAW_QUAT + 2] = nsin(yaw * 0.5f); ds[DWBC_DS_YAW_QUAT + 3] = ncos(yaw * 0.5f);
    }
    {  // EE goal (WG:1344-1350); the sphere resample itself is deferred to the fix-up pass
      float t = clipf(ndiv(gs[DWBC_GS_GOAL_TIMER], gs[DWBC_GS_TRAJ_T]), 0.0f, 1.0f);
      V3 cs = lerp3(mk(gs[DWBC_GS_START_SPH], gs[DWBC_GS_START_SPH + 1], gs[DWBC_GS_START_SPH + 2]),
                    mk(gs[DWBC_GS_GOAL_SPH], gs[DWBC_GS_GOAL_SPH + 1], gs[DWBC_GS_GOAL_SPH + 2]), t);
      V3 cc = sphere2cart(cs);
      gs[DWBC_GS_CURR_SPH] = cs.x; gs[DWBC_GS_CURR_SPH + 1] = cs.y; gs[DWBC_GS_CURR_SPH + 2] = cs.z;
      gs[DWBC_GS_CURR_CART] = cc.x; gs[DWBC_GS_CURR_CART + 1] = cc.y; gs[DWBC_GS_CURR_CART + 2] = cc.z;
      float timer = gs[DWBC_GS_GOAL_TIMER] + 1.0f;
      gs[DWBC_GS_GOAL_TIMER] = timer;
      if (timer > gs[DWBC_GS_TRAJ_TOTAL]) {
        flags |= F_GOAL_RS;
        for (int i = 0; i < 3; ++i) {   // orientation part now: this step's rewards / obs read it (WG:1307-1313)
          float d = cfg.delta_orn_span[i] * rng(DWBC_RAND_GOAL_ORN + i) + cfg.delta_orn_lo[i];
          gs[DWBC_GS_DELTA_ORN + i] = d;
          gs[DWBC_GS_GOAL_ORN + i] = wrap_pi(d + (i == 2 ? yaw : 0.0f));
        }
      }
    }
    if (ep % cfg.resample_interval == 0) {  // WG:922-925, 831-843
      float cx = A.lin_vel_x[1] * rng(DWBC_RAND_CMD) + A.lin_vel_x[0];
      float cy = A.ang_vel_yaw[1] * rng(DWBC_RAND_CMD + 1) + A.ang_vel_yaw[0];
      float keep = (cx > cfg.lin_vel_x_clip || fabsf(cy) > cfg.ang_vel_yaw_clip) ? 1.0f : 0.0f;
      gs[0] = cx * keep; gs[1] = 0.0f * keep; gs[2] = cy * keep;
    }
    const float mean_gap = cfg.measure_heights ? sm[Ly::o_rp + 4 * e + 3] / (float)(cfg.n_height_x * cfg.n_height_y) : 0.0f;
    if (A.do_push) {  // WG:804-814
      float vx = cfg.push_vel[1] * rng(DWBC_RAND_PUSH) + cfg.push_vel[0];
      float vy = cfg.push_vel[1] * rng(DWBC_RAND_PUSH + 1) + cfg.push_vel[0];
      if (((gs[0] + gs[1]) + gs[2]) == 0.0f) { vx *= 2.5f; vy *= 2.5f; }
      root[7] = vx; root[8] = vy;
      flags |= F_ROOT_DIRTY;
    }
    bool time_out, reset;
    {  // termination (WG:937-963)
      bool contact = false;
      for (int i = 0; i < cfg.n_term_contact; ++i) {
        const float* f = cf + 3 * (4 + cfg.n_penalized + i);
        contact = contact || (nsqrt((f[0] * f[0] + f[1] * f[1]) + f[2] * f[2]) > 1.0f);
      }
      const float* g = gs + (cfg.goal_is_cart ? DWBC_GS_CURR_CART : DWBC_GS_CURR_SPH);
      bool r_bad = ((r0 > cfg.term_roll) && (g[2] >= 0.0f)) || ((r0 < -cfg.term_roll) && (g[2] <= 0.0f));
      bool p_bad = ((p0 > cfg.term_pitch) && (g[1] >= 0.0f)) || ((p0 < -cfg.term_pitch) && (g[1] <= 0.0f));
      time_out = ep > cfg.max_episode_length;
      reset = contact || r_bad || p_bad || (root[2] < cfg.term_z) || time_out;
      if (time_out) flags |= F_TIMEOUT;
      if (reset) flags |= F_RESET;
    }
    // rewards (WG:170-205); DOF reductions come from the feature pass
    auto term = [&](int t) -> float {
      float r = 0.0f;
      switch (t) {
        case DWBC_TERM_energy_square: r = feat[FE_ENERGY_SQ]; met[8] += r; break;
        case DWBC_TERM_foot_contacts_z: r = feat[FE_FOOT_Z]; met[9] += r; break;
        case DWBC_TERM_hip_action_l2: r = feat[FE_HIP_L2]; met[6] += r; break;
        case DWBC_TERM_leg_action_l2: r = feat[FE_LEG_L2]; met[6] += r; break;
        case DWBC_TERM_survive: r = 1.0f; break;
        case DWBC_TERM_tracking_ang_vel_yaw_exp: { float x = fabsf(gs[2] - ds[DWBC_DS_BASE_ANG_VEL + 2]); met[2] += x; r = nexp(-x / cfg.tracking_sigma); } break;
        case DWBC_TERM_tracking_ang_vel_yaw_l1: { float x = fabsf(gs[2] - ds[DWBC_DS_BASE_ANG_VEL + 2]); r = -x + fabsf(gs[2]); } break;
        case DWBC_TERM_tracking_lin_vel_x_l1: { float x = fabsf(gs[0] - ds[DWBC_DS_BASE_LIN_VEL]); met[1] += x; r = -x + fabsf(gs[0]); } break;
        case DWBC_TERM_tracking_lin_vel_x_exp: { float x = fabsf(gs[0] - ds[DWBC_DS_BASE_LIN_VEL]); met[1] += x; r = nexp(-x / cfg.tracking_sigma); } break;
        case DWBC_TERM_tracking_lin_vel_y_l2: { float x = gs[1] - ds[DWBC_DS_BASE_LIN_VEL + 1]; r = x * x; } break;
        case DWBC_TERM_tracking_lin_vel_z_l2: { float x = gs[2] - ds[DWBC_DS_BASE_LIN_VEL + 2]; r = x * x; } break;
        case DWBC_TERM_tracking_lin_vel: {
          float ex = gs[0] - ds[DWBC_DS_BASE_LIN_VEL], ey = gs[1] - ds[DWBC_DS_BASE_LIN_VEL + 1];
          r = nexp(-(ex * ex + ey * ey) / cfg.tracking_sigma);
        } break;
        case DWBC_TERM_tracking_ang_vel: { float x = gs[2] - ds[DWBC_DS_BASE_ANG_VEL + 2]; r = nexp(-(x * x) / cfg.tracking_sigma); } break;
        case DWBC_TERM_torques: r = feat[FE_TORQUE_SQ]; met[7] += r; break;
        case DWBC_TERM_leg_energy_abs_sum: r = feat[FE_LEG_ABS]; met[0] += r; break;
        case DWBC_TERM_leg_energy_sum_abs: r = fabsf(feat[FE_LEG_SUM]); break;
        case DWBC_TERM_leg_energy: r = feat[FE_LEG_SUM]; break;
        case DWBC_TERM_arm_energy_abs_sum: r = feat[FE_ARM_ABS]; break;
        case DWBC_TERM_tracking_ee_sphere: {  // WG:1352-1358
          V3 d = mk(ee[0] - root[0], ee[1] - root[1], ee[2] - cfg.z_invariant_offset);
          V3 s = cart2sphere(quat_rotate_inverse(ds + DWBC_DS_YAW_QUAT, d));
          float x = (fabsf(s.x - gs[DWBC_GS_CURR_SPH]) * cfg.sphere_error_scale[0] + fabsf(s.y - gs[DWBC_GS_CURR_SPH + 1]) * cfg.sphere_error_scale[1]) +
                    fabsf(s.z - gs[DWBC_GS_CURR_SPH + 2]) * cfg.sphere_error_scale[2];
          met[4] += x;
          r = nexp(-x / cfg.tracking_ee_sigma);
        } break;
        case DWBC_TERM_tracking_ee_cart: {  // WG:1360-1366
          V3 tv = quat_apply(ds + DWBC_DS_YAW_QUAT, mk(gs[DWBC_GS_CURR_CART], gs[DWBC_GS_CURR_CART + 1], gs[DWBC_GS_CURR_CART + 2]));
          float x = (fabsf(ee[0] - (root[0] + tv.x)) + fabsf(ee[1] - (root[1] + tv.y))) + fabsf(ee[2] - (cfg.z_invariant_offset + tv.z));
          met[3] += x;
          r = nexp(-x / cfg.tracking_ee_sigma);
        } break;
        case DWBC_TERM_tracking_ee_orn:
        case DWBC_TERM_tracking_ee_orn_ry: {  // WG:1368-1394
          float eu[3];
          euler_from_quat(ee + 3, eu[0], eu[1], eu[2]);
          float d0 = wrap_pi(gs[DWBC_GS_GOAL_ORN] - eu[0]), d1 = wrap_pi(gs[DWBC_GS_GOAL_ORN + 1] - eu[1]), d2 = wrap_pi(gs[DWBC_GS_GOAL_ORN + 2] - eu[2]);
          float x;
          if (t == DWBC_TERM_tracking_ee_orn) {
            x = (fabsf(d0) * cfg.orn_error_scale[0] + fabsf(d1) * cfg.orn_error_scale[1]) + fabsf(d2) * cfg.orn_error_scale[2];
          } else {
            x = fabsf(d0 * cfg.orn_error_scale[0]) + fabsf(d2 * cfg.orn_error_scale[2]);
            met[5] += x;
          }
          r = nexp(-x / cfg.tracking_ee_sigma);
        } break;
        case DWBC_TERM_lin_vel_z: r = ds[DWBC_DS_BASE_LIN_VEL + 2] * ds[DWBC_DS_BASE_LIN_VEL + 2]; break;
        case DWBC_TERM_ang_vel_xy: r = ds[DWBC_DS_BASE_ANG_VEL] * ds[DWBC_DS_BASE_ANG_VEL] + ds[DWBC_DS_BASE_ANG_VEL + 1] * ds[DWBC_DS_BASE_ANG_VEL + 1]; break;
        case DWBC_TERM_base_height: { float x = mean_gap - cfg.base_height_target; r = x * x; } break;
        case DWBC_TERM_dof_vel: r = feat[FE_DOFVEL_SQ]; break;
        case DWBC_TERM_dof_acc: r = feat[FE_DOF_ACC]; break;
        case DWBC_TERM_action_rate: r = feat[FE_ACT_RATE]; break;
        case DWBC_TERM_collision: {
          for (int i = 0; i < cfg.n_penalized; ++i) { const float* f = cf + 3 * (4 + i); r += nsqrt((f[0] * f[0] + f[1] * f[1]) + f[2] * f[2]) > 0.1f ? 1.0f : 0.0f; }
        } break;
        case DWBC_TERM_termination: r = (reset && !time_out) ? 1.0f : 0.0f; break;
        case DWBC_TERM_dof_pos_limits: r = feat[FE_POS_LIM]; break;
        case DWBC_TERM_dof_vel_limits: r = feat[FE_VEL_LIM]; break;
        case DWBC_TERM_torque_limits: r = feat[FE_TQ_LIM]; break;
        case DWBC_TERM_feet_air_time: {  // LR:896-908
          for (int f = 0; f < 4; ++f) {
            bool contact = cf[3 * f + 2] > 1.0f;
            bool filt = contact || (ds[DWBC_DS_LAST_CONTACTS + f] != 0.0f);
            float fat = ds[DWBC_DS_FEET_AIR_TIME + f];
            bool first = (fat > 0.0f) && filt;
            fat += cfg.dt;
            r += (fat - 0.5f) * (first ? 1.0f : 0.0f);
            ds[DWBC_DS_LAST_CONTACTS + f] = contact ? 1.0f : 0.0f;
            ds[DWBC_DS_FEET_AIR_TIME + f] = fat * (filt ? 0.0f : 1.0f);
          }
          r *= (nsqrt(gs[0] * gs[0] + gs[1] * gs[1]) > 0.1f) ? 1.0f : 0.0f;
        } break;
        case DWBC_TERM_stumble: {
          bool s = false;
          for (int f = 0; f < 4; ++f) { const float* c = cf + 3 * f; s = s || (nsqrt(c[0] * c[0] + c[1] * c[1]) > 5.0f * fabsf(c[2])); }
          r = s ? 1.0f : 0.0f;
        } break;
        case DWBC_TERM_stand_still: r = feat[FE_STAND] * ((nsqrt(gs[0] * gs[0] + gs[1] * gs[1]) < 0.1f) ? 1.0f : 0.0f); break;
        case DWBC_TERM_feet_contact_forces: {
          for (int f = 0; f < 4; ++f) { const float* c = cf + 3 * f; r += fmaxf(nsqrt((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]) - cfg.max_contact_force, 0.0f); }
        } break;
        default: break;
      }
      return r;
    };
#pragma unroll 1
    for (int ch = 0; ch < 2; ++ch) {
      const int n = ch == 0 ? cfg.n_leg_terms : cfg.n_arm_terms;
      const int32_t* terms = ch == 0 ? cfg.leg_term : cfg.arm_term;
      const int32_t* slots = ch == 0 ? cfg.leg_slot : cfg.arm_slot;
      const float* scales = ch == 0 ? A.leg_scale : A.arm_scale;
      float buf = 0.0f;
      for (int i = 0; i < n; ++i) {
        float r = term(terms[i]) * scales[i];
        buf += r;
        sums[slots[i]] += r;
      }
      if (cfg.only_positive_rewards) buf = fmaxf(buf, 0.0f);
      float ts = ch == 0 ? A.leg_termination_scale : A.arm_termination_scale;
      if (ts != 0.0f && cfg.termination_slot >= 0) {
        float r = ((reset && !time_out) ? 1.0f : 0.0f) * ts;
        buf += r;
        sums[cfg.termination_slot] += r;
      }
      sm[Ly::o_out + 2 * e + ch] = buf / 100.0f;
    }
    sm[Ly::o_rp + 4 * e] = r0; sm[Ly::o_rp + 4 * e + 1] = p0; sm[Ly::o_rp + 4 * e + 2] = yaw;
    if (!reset && ep <= 1) flags |= F_FILL;
    flags_s[e] = flags;
    ep_s[e] = ep;
  }
  cbar();

  // ---- 7. fix-up pass: rare events, one warp per flagged env ------------------------------------
  const unsigned fix_list = __ballot_sync(FULL, lane < V2_E && (flags_s[lane] & (F_GOAL_RS | F_RESET)) != 0);   // same value in every warp
  for (int k = wid; k < __popc(fix_list); k += V2_CW) {
    const int e = __fns(fix_list, 0, k + 1);    // k-th flagged env: flagged envs are dealt round-robin to the warps
    int flags = flags_s[e];
    const int env = e0 + e;
    float* root = sm + Ly::o_root + e * 26;
    float* gs = sm + Ly::o_gs + e * DWBC_GS;
    float* ds = sm + Ly::o_ds + e * DWBC_DS;
    float* dof = sm + Ly::o_dof + e * 2 * ND;
    float* sums = sums_s + e * stride;
    const float yaw = sm[Ly::o_rp + 4 * e + 2];
    RngW rng{A.rand_uniform, env, make_uint4(0, 0, 0, 0)};
    if (!A.rand_uniform && lane < DWBC_RAND_COLS / 4)
      rng.mine = philox4x32_10(make_uint4((uint32_t)env, (uint32_t)lane, (uint32_t)A.step, (uint32_t)(A.step >> 32)),
                               make_uint2((uint32_t)A.seed, (uint32_t)(A.seed >> 32)));
    if (flags & F_GOAL_RS) coop_resample_goal(cfg, A, rng, gs, yaw, DWBC_RAND_GOAL_ORN, DWBC_RAND_GOAL_SPH, false, lane);
    if (flags & F_RESET) {  // WG:695-754
      if (cfg.terrain_curriculum) {  // LR:421-441 (reads the pre-reset root / commands)
        float* org = B.env_origins + (size_t)env * 3;
        float o0 = org[0], o1 = org[1], o2;
        long long lvl = 0;
        const float u_terrain = rng(DWBC_RAND_TERRAIN);
        {
          float dx = root[0] - o0, dy = root[1] - o1;
          float dist = nsqrt(dx * dx + dy * dy);
          bool up = dist > cfg.terrain_env_length / 2.0f;
          bool down = (dist < nsqrt(gs[0] * gs[0] + gs[1] * gs[1]) * cfg.max_episode_length_s * 0.5f) && !up;
          lvl = B.terrain_levels[env] + (up ? 1 : 0) - (down ? 1 : 0);
          if (lvl >= cfg.max_terrain_level) {
            long long rl = (long long)(u_terrain * (float)cfg.max_terrain_level);
            lvl = rl > cfg.max_terrain_level - 1 ? cfg.max_terrain_level - 1 : rl;
          } else if (lvl < 0) {
            lvl = 0;
          }
          const float* to = B.terrain_origins + ((size_t)lvl * cfg.terrain_n_types + B.terrain_types[env]) * 3;
          o0 = to[0]; o1 = to[1]; o2 = to[2];
        }
        __syncwarp();
        if (lane == 0) { B.terrain_levels[env] = lvl; org[0] = o0; org[1] = o1; org[2] = o2; }
        __syncwarp();
      }
      {
        const float u_dof = rng(DWBC_RAND_RST_DOF + (lane < ND ? lane : 0));
        const float u_xy = rng(DWBC_RAND_RST_XY + (lane < 2 ? lane : 0));
        const float u_vel = rng(DWBC_RAND_RST_VEL + ((lane >= 7 && lane < 13) ? lane - 7 : 0));
        const float u_c0 = rng(DWBC_RAND_RST_CMD), u_c1 = rng(DWBC_RAND_RST_CMD + 1);
        if (lane < ND) {  // _reset_dofs WG:816-828
          dof[2 * lane] = cfg.default_dof_pos[lane] * (cfg.dof_reset[1] * u_dof + cfg.dof_reset[0]);
          dof[2 * lane + 1] = 0.0f;
        }
        if (lane < 13) {  // _reset_root_states WG:757-788
          float v = cfg.base_init_state[lane];
          if (lane < 3) v += B.env_origins[(size_t)env * 3 + lane];
          if (lane < 2) v += cfg.origin_perturb[1] * u_xy + cfg.origin_perturb[0];
          if (lane >= 7) v = cfg.init_vel_perturb[1] * u_vel + cfg.init_vel_perturb[0];
          root[lane] = v;
        }
        if (lane == 0 && (flags & F_TIMEOUT)) {  // WG:723-727
          float cx = A.lin_vel_x[1] * u_c0 + A.lin_vel_x[0];
          float cy = A.ang_vel_yaw[1] * u_c1 + A.ang_vel_yaw[0];
          float keep = (cx > cfg.lin_vel_x_clip || fabsf(cy) > cfg.ang_vel_yaw_clip) ? 1.0f : 0.0f;
          gs[0] = cx * keep; gs[1] = 0.0f * keep; gs[2] = cy * keep;
        }
      }
      __syncwarp();
      if (lane == 0) {
        root[13] = cfg.box_x;
        root[14] = root[1] + B.box_env_origins_delta_y[env];
        root[15] = cfg.box_z;
        float r0, p0, y0;
        euler_from_quat(root + 3, r0, p0, y0);   // obs reads the post-reset quaternion (base_quat is a view, WG:535)
        sm[Ly::o_rp + 4 * e] = r0; sm[Ly::o_rp + 4 * e + 1] = p0;
        ep_s[e] = 0;
      }
      __syncwarp();
      coop_resample_goal(cfg, A, rng, gs, yaw, DWBC_RAND_RST_GOAL_ORN, DWBC_RAND_RST_GOAL_SPH, true, lane);
      if (lane < 4) ds[DWBC_DS_FEET_AIR_TIME + lane] = 0.0f;
      float* ah = sm + Ly::o_ah + e * AH * NA;
      for (int i = lane; i < AH * NA; i += 32) ah[i] = 0.0f;
      for (int i = lane; i < nslots; i += 32) {  // extras['episode'] (WG:743-750): this env's slot, added up by episode_stats_kernel
        B.episode_scratch[(size_t)env * cfg.sums_stride + i] = sums[i];
        sums[i] = 0.0f;
      }
      if (lane == 0) flags_s[e] = flags | F_FILL | F_ROOT_DIRTY | F_DOF_DIRTY;
    }
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
  if (tid < V2_E) {
    const int f = flags_s[tid];
    B.rew_buf[e0 + tid] = sm[Ly::o_out + 2 * tid];
    B.arm_rew_buf[e0 + tid] = sm[Ly::o_out + 2 * tid + 1];
    B.reset_buf[e0 + tid] = (f & F_RESET) ? 1 : 0;
    B.time_out_buf[e0 + tid] = (f & F_TIMEOUT) ? 1 : 0;
    if (B.store_rewards) {          // PPO.process_env_step's reward path (PPO:130-134) + dones (RS:102), straight into the storage rows
      const size_t e = (size_t)(e0 + tid);
      const float to = (f & F_TIMEOUT) ? 1.0f : 0.0f;
      B.store_rewards[2 * e] = sm[Ly::o_out + 2 * tid] + B.store_gamma * (B.store_values[2 * e] * to);
      B.store_rewards[2 * e + 1] = sm[Ly::o_out + 2 * tid + 1] + B.store_gamma * (B.store_values[2 * e + 1] * to);
      if (B.store_dones) B.store_dones[e] = (f & F_RESET) ? 1 : 0;
    }
  }
  if (cfg.measure_heights && B.heights_obs) {  // LR:221-223
    const int npts = cfg.n_height_x * cfg.n_height_y;
    for (int i = tid; i < V2_E * npts; i += V2_CT) {
      const int e = i / npts;
      B.heights_obs[(size_t)e0 * npts + i] =
          clipf((sm[Ly::o_root + e * 26 + 2] - 0.5f) - B.measured_heights[(size_t)e0 * npts + i], -1.0f, 1.0f) * cfg.obs_scale_height;
    }
  }
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

// launcher used by dwbc_post_physics_step (env_step.cu); DWBC_ERR_UNSUPPORTED -> caller falls back to v1
int dwbc_launch_env_step_v2(const DwbcEnvCfg* cfg, const DwbcEnvBuffers* buf, const DwbcStepArgs* args, const DwbcStepDevice* dev, cudaStream_t st) {
  using K = V2<20, 18, 4, 76, 10, 24>;
  if (cfg->num_dofs != 20 || cfg->num_actions != 18 || cfg->action_hist_len != 4 || cfg->num_prop != 76 || cfg->history_len != 10 ||
      cfg->num_priv != 24 || (cfg->sums_stride & 3) || cfg->n_collision_samples > 32)
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
