// Per-env logic of the fused post-physics step (WG:865-1001, LR:421-441, LR:793-922), written once for both kernels that run it:
// the TMA kernel (env_step_v2.cu: 16 envs per CTA, work split into passes) and the warp-per-env kernel (env_step.cu: every other
// shape).  Each kernel stages an env's rows in shared memory and describes them with an EnvView; everything here reads and writes
// through that view.  Sizes are int arguments: the TMA kernel passes compile-time constants, so its strides fold into immediates.
// Compiled with -fmad=false: the expressions and summation orders below are the arithmetic both kernels compute, bit for bit.
#pragma once
#include "env_math.cuh"

namespace dwbc {

#define DWBC_DS_OOB_AGE 27 /* derived_state pad column: #most-recent history rows known to be within +-clip_obs */

enum { F_RESET = 1, F_TIMEOUT = 2, F_FILL = 4, F_OOB = 8, F_ROOT_DIRTY = 16, F_DOF_DIRTY = 32, F_GOAL_RS = 64 };
enum { FE_ENERGY_SQ = 0, FE_LEG_ABS, FE_LEG_SUM, FE_ARM_ABS, FE_TORQUE_SQ, FE_DOFVEL_SQ, FE_DOF_ACC, FE_ACT_RATE, FE_HIP_L2, FE_LEG_L2,
       FE_FOOT_Z, FE_POS_LIM, FE_VEL_LIM, FE_TQ_LIM, FE_STAND, FE_COUNT = 16 };

// Word `tid` of the step arguments a kernel works with: the host's DwbcStepArgs, except that with a device record (CUDA-graph replay) the
// step, the push decision (WG:934) and the curriculum values come from that record.  Threads 0 .. STEP_ARGS_WORDS - 1 take part; each
// kernel asserts that its CTA has that many threads.
static_assert(offsetof(DwbcStepArgs, generic_kernel) - offsetof(DwbcStepArgs, lin_vel_x) == sizeof(DwbcStepDevice) - offsetof(DwbcStepDevice, lin_vel_x),
              "the curriculum block of DwbcStepDevice mirrors the one of DwbcStepArgs");
static_assert(sizeof(DwbcStepArgs) % 4 == 0, "one word per thread");
constexpr int STEP_ARGS_WORDS = sizeof(DwbcStepArgs) / 4;
__device__ __forceinline__ void step_args_to_shared(const DwbcStepArgs& h, const DwbcStepDevice* d, DwbcStepArgs* out, int tid) {
  constexpr int W_STEP = offsetof(DwbcStepArgs, step) / 4, W_PUSH = offsetof(DwbcStepArgs, do_push) / 4;
  constexpr int W_CUR0 = offsetof(DwbcStepArgs, lin_vel_x) / 4, W_CUR1 = offsetof(DwbcStepArgs, generic_kernel) / 4;
  if (tid >= STEP_ARGS_WORDS) return;
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

// One env's staged rows (shared memory).
struct EnvView {
  float* root;         // [26] root state: base 0..12, box 13..15
  float* dof;          // [2 nd] (position, velocity) per DOF
  const float* fs;     // [24] foot force sensors
  const float* tq;     // [nd] torques
  const float* act;    // [na] actions
  float* ah;           // [ah_len][na] action history
  float* gs;           // [DWBC_GS] goal_state row
  float* ds;           // [DWBC_DS] derived_state row
  float* sums;         // [n_sum_slots + DWBC_NUM_METRICS] episode sums, then metric sums
  const float* ee;     // gripper rigid-body row: position, quaternion
  const float* cf;     // contact forces (3 each): 4 feet, penalised bodies, termination bodies
  const float* mass;   // [5]
  const float* fric;   // [1]
  const float* motor;  // [na] motor strength
  float* prop;         // [num_prop] observation columns
  float* priv;         // [num_priv] privileged observation columns
  float* feat;         // [FE_COUNT] DOF reductions
  float* rp;           // roll, pitch, yaw, sum of height gaps
  float* rew;          // leg and arm reward of this step
};

// The uniform stream of one env step, value(env, col) = philox(ctr=(env, col/4, step_lo, step_hi), key=seed)[col%4], or the host's
// table when one is given.  One thread's view with a one-block cache: consecutive columns share a Philox4x32-10 evaluation.
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

// Warp-wide uniform stream for the fix-up: lane b holds Philox block b (columns 4b..4b+3) of this env and step,
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

// Which DOF reductions the active reward terms need: bit k for FE_k.
__device__ __forceinline__ int feature_mask(const DwbcEnvCfg& cfg) {
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
  return m;
}

// The sums over DOFs the reward terms need (WG:1396-1469, LR:853-886): warp per env, lane per DOF, only the reductions in `need`;
// lane 0 writes v.feat.  defpos = default_dof_pos.
__device__ __forceinline__ void dof_features(const DwbcEnvCfg& cfg, const EnvView& v, int need, const float* defpos, int nd, int na, int lane) {
  const float tq = lane < nd ? v.tq[lane] : 0.0f;
  const float dv = lane < nd ? v.dof[2 * lane + 1] : 0.0f;
  const float dp = lane < nd ? v.dof[2 * lane] : 0.0f;
  const float act = lane < na ? v.act[lane] : 0.0f;
  const float* ds = v.ds;
  float* feat = v.feat;
  const float pw = lane < 12 ? tq * dv : 0.0f;
#define FEAT(k, expr) if (need & (1 << (k))) { float r_ = warp_sum(expr); if (lane == 0) feat[k] = r_; }
  FEAT(FE_ENERGY_SQ, pw * pw)                                                                           // WG:1466
  FEAT(FE_LEG_ABS, fabsf(pw))                                                                           // WG:1396
  FEAT(FE_LEG_SUM, pw)                                                                                  // WG:1401,1410
  FEAT(FE_ARM_ABS, (lane >= 12 && lane < nd - 2) ? fabsf(tq * dv) : 0.0f)                               // WG:1414
  FEAT(FE_TORQUE_SQ, tq * tq)                                                                           // WG:1460
  FEAT(FE_DOFVEL_SQ, dv * dv)                                                                           // LR:853
  if (need & (1 << FE_DOF_ACC)) { float a = lane < nd ? (ds[DWBC_DS_LAST_DOF_VEL + lane] - dv) / cfg.dt : 0.0f; a = warp_sum(a * a); if (lane == 0) feat[FE_DOF_ACC] = a; }
  if (need & (1 << FE_ACT_RATE)) { float a = lane < na ? ds[DWBC_DS_LAST_ACTIONS + lane] - act : 0.0f; a = warp_sum(a * a); if (lane == 0) feat[FE_ACT_RATE] = a; }
  FEAT(FE_HIP_L2, (lane < 12 && lane % 3 == 0) ? act * act : 0.0f)                                      // WG:1379
  FEAT(FE_LEG_L2, lane < 12 ? act * act : 0.0f)                                                         // WG:1405
  if (need & (1 << FE_FOOT_Z)) { float z = lane < 4 ? v.fs[6 * lane + 2] : 0.0f; z = warp_sum(z * z); if (lane == 0) feat[FE_FOOT_Z] = z; }
  FEAT(FE_POS_LIM, lane < nd ? -fminf(dp - cfg.dof_pos_lower[lane], 0.0f) + fmaxf(dp - cfg.dof_pos_upper[lane], 0.0f) : 0.0f)
  FEAT(FE_VEL_LIM, lane < nd ? clipf(fabsf(dv) - cfg.dof_vel_limits[lane] * cfg.soft_dof_vel_limit, 0.0f, 1.0f) : 0.0f)
  FEAT(FE_TQ_LIM, lane < nd ? fmaxf(fabsf(tq) - cfg.torque_limits[lane] * cfg.soft_torque_limit, 0.0f) : 0.0f)
  FEAT(FE_STAND, lane < nd ? fabsf(dp - defpos[lane]) : 0.0f)
#undef FEAT
}

// Height scan (LR:793-829): warp per env, lane per point.  Writes the env's measured_heights row and returns, in every lane,
// the sum of root_z - height over the points.
__device__ __forceinline__ float height_scan(const DwbcEnvCfg& cfg, const DwbcEnvBuffers& B, const float* root, int env, int lane) {
  const int npts = cfg.n_height_x * cfg.n_height_y;
  float qy[4] = {0.0f, 0.0f, root[5], root[6]};
  const float n = fmaxf(nsqrt(qy[2] * qy[2] + qy[3] * qy[3]), 1e-9f);     // utils/math.py:38-42 + normalize()
  qy[2] = qy[2] / n; qy[3] = qy[3] / n;
  const float rx = root[0], ry = root[1], rz = root[2];
  float gap = 0.0f;
  float* out = B.measured_heights + (size_t)env * npts;
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
  return warp_sum(gap);
}

// One thread per env: derived base state, EE-goal interpolation and timer with the orientation part of an expiring goal's resample,
// command resampling, push, termination, the reward terms of both channels with episode and metric sums.  Needs v.feat and the
// height-gap sum in v.rp[3]; writes v.rp[0..2] (roll, pitch, yaw) and v.rew.  ep = episode length including this step.
// Returns the F_* flags: F_GOAL_RS and F_RESET ask for fix_up().
__device__ __forceinline__ int scalar_step(const DwbcEnvCfg& cfg, const DwbcStepArgs& A, const EnvView& v, int env, long long ep) {
  float* root = v.root;
  float* gs = v.gs;
  float* ds = v.ds;
  float* sums = v.sums;
  float* met = sums + cfg.n_sum_slots;
  const float* feat = v.feat;
  const float* ee = v.ee;
  const float* cf = v.cf;
  RngC rng{A.rand_uniform, A.seed, A.step, env, -1, make_uint4(0, 0, 0, 0)};
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
  {  // EE goal (WG:1344-1350); the sphere resample itself is left to fix_up()
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
  const float mean_gap = cfg.measure_heights ? v.rp[3] / (float)(cfg.n_height_x * cfg.n_height_y) : 0.0f;
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
  // rewards (WG:170-205); DOF reductions come from dof_features()
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
    v.rew[ch] = buf / 100.0f;
  }
  v.rp[0] = r0; v.rp[1] = p0; v.rp[2] = yaw;
  if (!reset && ep <= 1) flags |= F_FILL;
  return flags;
}

// Warp-cooperative EE-goal resampling (WG:1316-1332); collision samples spread over lanes (WG:1337-1342)
static __device__ void coop_resample_goal(const DwbcEnvCfg& cfg, const DwbcStepArgs& A, const RngW& rng, float* gs, float yaw, int col_orn,
                                          int col_sph, bool do_orn, int lane) {
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
  const int ns = cfg.n_collision_samples > 0 ? (cfg.n_collision_samples < 16 ? cfg.n_collision_samples : 16) : 1;   // collision_t[16]
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
      const unsigned m = ((1u << ns) - 1u) << (t * ns);
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

// The rare events of one env, one warp: the sphere part of an expiring goal's resample (F_GOAL_RS) and the reset (F_RESET,
// WG:695-754): terrain curriculum, dof / root reset, commands on time-out, box row, goal, air time, action history and the episode's
// sums moved to its episode_scratch slot.  Returns the flags with F_FILL | F_ROOT_DIRTY | F_DOF_DIRTY added on reset; the caller
// zeroes the episode length and, on reset, the history.
__device__ __forceinline__ int fix_up(const DwbcEnvCfg& cfg, const DwbcStepArgs& A, const DwbcEnvBuffers& B, const EnvView& v, int flags, int env,
                                      int nd, int na, int ah_len, int nslots, int lane) {
  float* root = v.root;
  float* gs = v.gs;
  float* ds = v.ds;
  float* dof = v.dof;
  float* sums = v.sums;
  const float yaw = v.rp[2];
  RngW rng{A.rand_uniform, env, make_uint4(0, 0, 0, 0)};
  if (!A.rand_uniform && lane < DWBC_RAND_COLS / 4)
    rng.mine = philox4x32_10(make_uint4((uint32_t)env, (uint32_t)lane, (uint32_t)A.step, (uint32_t)(A.step >> 32)),
                             make_uint2((uint32_t)A.seed, (uint32_t)(A.seed >> 32)));
  if (flags & F_GOAL_RS) coop_resample_goal(cfg, A, rng, gs, yaw, DWBC_RAND_GOAL_ORN, DWBC_RAND_GOAL_SPH, false, lane);
  if (!(flags & F_RESET)) return flags;
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
    const float u_dof = rng(DWBC_RAND_RST_DOF + (lane < nd ? lane : 0));
    const float u_xy = rng(DWBC_RAND_RST_XY + (lane < 2 ? lane : 0));
    const float u_vel = rng(DWBC_RAND_RST_VEL + ((lane >= 7 && lane < 13) ? lane - 7 : 0));
    const float u_c0 = rng(DWBC_RAND_RST_CMD), u_c1 = rng(DWBC_RAND_RST_CMD + 1);
    if (lane < nd) {  // _reset_dofs WG:816-828
      dof[2 * lane] = cfg.default_dof_pos[lane] * (cfg.dof_reset[1] * u_dof + cfg.dof_reset[0]);
      dof[2 * lane + 1] = 0.0f;
    }
    if (lane < 13) {  // _reset_root_states WG:757-788
      float x = cfg.base_init_state[lane];
      if (lane < 3) x += B.env_origins[(size_t)env * 3 + lane];
      if (lane < 2) x += cfg.origin_perturb[1] * u_xy + cfg.origin_perturb[0];
      if (lane >= 7) x = cfg.init_vel_perturb[1] * u_vel + cfg.init_vel_perturb[0];
      root[lane] = x;
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
    v.rp[0] = r0; v.rp[1] = p0;
  }
  __syncwarp();
  coop_resample_goal(cfg, A, rng, gs, yaw, DWBC_RAND_RST_GOAL_ORN, DWBC_RAND_RST_GOAL_SPH, true, lane);
  if (lane < 4) ds[DWBC_DS_FEET_AIR_TIME + lane] = 0.0f;
  for (int i = lane; i < ah_len * na; i += 32) v.ah[i] = 0.0f;
  for (int i = lane; i < nslots; i += 32) {  // extras['episode'] (WG:743-750): this env's slot, added up by episode_stats_kernel
    B.episode_scratch[(size_t)env * cfg.sums_stride + i] = sums[i];
    sums[i] = 0.0f;
  }
  return flags | F_FILL | F_ROOT_DIRTY | F_DOF_DIRTY;
}

// One env's observation columns (WG:966-1001, Appendix B): warp per env, lane per column.
// part 0 = columns that depend only on the simulator state (joint positions / velocities, last action, foot contacts, privileged
// mass / friction / motor strength) and the last_actions / last_dof_vel copies; part 1 = columns produced by scalar_step() and
// fix_up() (roll-pitch, angular velocity, commands, goal) and the last_root_vel copy (WG:908-910).
// Returns, in every lane, whether a column written lies outside +-c.  ig2r = ig2raisim, defpos = default_dof_pos.
__device__ __forceinline__ bool assemble_obs(const DwbcEnvCfg& cfg, const EnvView& v, int part, const int* ig2r, const float* defpos, float c,
                                             int nd, int na, int ah_len, int lane) {
  const float* dof = v.dof;
  const float* gs = v.gs;
  float* ds = v.ds;
  float* prop = v.prop;
  float* priv = v.priv;
  bool bad = false;
  if (part == 0) {
    if (lane < nd) {            // dof position / velocity columns, last_dof_vel
      const int d = ig2r[lane];
      float pos = dof[2 * d];
      if (d == cfg.waist_dof) pos = wrap_pi(pos);
      const float v0 = (pos - defpos[d]) * cfg.obs_scale_dof_pos, v1 = dof[2 * d + 1] * cfg.obs_scale_dof_vel;
      prop[5 + lane] = v0;
      prop[5 + nd + lane] = v1;
      bad = !(fabsf(v0) <= c) || !(fabsf(v1) <= c);
      ds[DWBC_DS_LAST_DOF_VEL + lane] = dof[2 * lane + 1];
    }
    if (lane < na) {            // last applied action column, last_actions, motor strength
      const float x = v.ah[(ah_len - 1) * na + ig2r[lane]];
      prop[5 + 2 * nd + lane] = x;
      bad = bad || !(fabsf(x) <= c);
      ds[DWBC_DS_LAST_ACTIONS + lane] = v.act[lane];
      priv[6 + lane] = v.motor[lane] - 1.0f;
    }
  }
  {
    const int o = 5 + 2 * nd + na;
    float x = 0.0f;
    int col = -1;
    if (part == 0) {
      if (lane < 4) {           // foot contacts (WG:1090-1098)
        const float* f = v.fs + 6 * (lane == 0 ? cfg.feet_perm[0] : (lane == 1 ? cfg.feet_perm[1] : (lane == 2 ? cfg.feet_perm[2] : cfg.feet_perm[3])));
        float nrm = nsqrt(((((f[0] * f[0] + f[1] * f[1]) + f[2] * f[2]) + f[3] * f[3]) + f[4] * f[4]) + f[5] * f[5]);
        x = nrm > 1.5f ? 1.0f : 0.0f; col = o + lane;
      } else if (lane >= 18 && lane < 23) priv[lane - 18] = v.mass[lane - 18];
      else if (lane == 23) priv[5] = v.fric[0];
    } else {
      if (lane >= 4 && lane < 6) { x = v.rp[lane - 4]; col = lane - 4; }
      else if (lane >= 6 && lane < 9) { x = ds[DWBC_DS_BASE_ANG_VEL + lane - 6] * cfg.obs_scale_ang_vel; col = 2 + lane - 6; }
      else if (lane >= 9 && lane < 11) { x = gs[lane - 9] * cfg.obs_scale_lin_vel; col = o + 4 + lane - 9; }
      else if (lane == 11) { x = gs[2] * cfg.obs_scale_ang_vel; col = o + 6; }
      else if (lane >= 12 && lane < 15) { x = gs[(cfg.goal_is_cart ? DWBC_GS_CURR_CART : DWBC_GS_CURR_SPH) + lane - 12]; col = o + 7 + lane - 12; }
      else if (lane >= 15 && lane < 18) { x = gs[DWBC_GS_DELTA_ORN + lane - 15]; col = o + 10 + lane - 15; }
      else if (lane >= 24 && lane < 30) ds[DWBC_DS_LAST_ROOT_VEL + lane - 24] = v.root[7 + lane - 24];   // WG:908-910
    }
    if (col >= 0) { prop[col] = x; bad = bad || !(fabsf(x) <= c); }
  }
  return __any_sync(FULL, bad);
}

// rew_buf, arm_rew_buf, reset_buf, time_out_buf of one env, and PPO.process_env_step's reward path (PPO:130-134) + dones (RS:102)
// straight into the storage rows.
__device__ __forceinline__ void store_step(const DwbcEnvBuffers& B, int env, int flags, float rew, float arm_rew) {
  B.rew_buf[env] = rew;
  B.arm_rew_buf[env] = arm_rew;
  B.reset_buf[env] = (flags & F_RESET) ? 1 : 0;
  B.time_out_buf[env] = (flags & F_TIMEOUT) ? 1 : 0;
  if (B.store_rewards) {
    const size_t e = (size_t)env;
    const float to = (flags & F_TIMEOUT) ? 1.0f : 0.0f;
    B.store_rewards[2 * e] = rew + B.store_gamma * (B.store_values[2 * e] * to);
    B.store_rewards[2 * e + 1] = arm_rew + B.store_gamma * (B.store_values[2 * e + 1] * to);
    if (B.store_dones) B.store_dones[e] = (flags & F_RESET) ? 1 : 0;
  }
}

// heights_obs (LR:221-223) of envs env0 .. env0 + n - 1, whose post-reset root rows are staged 26 floats apart from `root`;
// thread t of nt.
__device__ __forceinline__ void store_heights_obs(const DwbcEnvCfg& cfg, const DwbcEnvBuffers& B, int env0, int n, const float* root, int t, int nt) {
  if (!cfg.measure_heights || !B.heights_obs) return;
  const int npts = cfg.n_height_x * cfg.n_height_y;
  for (int i = t; i < n * npts; i += nt) {
    const int e = i / npts;
    B.heights_obs[(size_t)env0 * npts + i] = clipf((root[e * 26 + 2] - 0.5f) - B.measured_heights[(size_t)env0 * npts + i], -1.0f, 1.0f) * cfg.obs_scale_height;
  }
}

}  // namespace dwbc
