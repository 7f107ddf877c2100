// Fused widowGo1 post-physics step: ONE kernel launch per sim step (K1 + K2 of SURVEY.md).
//
// Replaces the ~200 ATen launches of WidowGo1.post_physics_step (WG:875-910): derived base
// state, EE-goal generator, command resampling, push, height scan, termination, the reward-term
// stack for both channels, episode sums, reset, observation assembly, history shift, obs clip.
//
// Mapping: one WARP per environment, 4 warps per CTA.  Every env is independent (SURVEY 3.3),
// so all control flow is warp-uniform.  Lane d owns DOF d / obs column groups; the handful of
// scalar quantities (quaternion algebra, goal interpolation, termination) are computed
// redundantly by all lanes from a shared-memory staging block that was filled with coalesced
// loads.  The 3 KB history row is read once as 128-bit streaming loads issued before anything
// else (so ~86 KB are in flight per SM), re-emitted into obs_buf and shifted in place.
//
// HBM-bound: algorithmic bytes 10 653 B / env-step (SURVEY 8d) -> 6.6 us @ 4096 envs at the
// measured 6.57 TB/s.  Compiled with -fmad=false so that discrete decisions (collision
// rejection, command dead-band, termination thresholds) see the same fp32 roundings as the
// reference's unfused torch arithmetic.
#include <stdlib.h>

#include "env_math.cuh"

namespace dwbc {

constexpr int ENV_WARPS = 4;
constexpr int MAX_H4 = 8;  // history row <= 8*32 float4 = 1024 floats in registers; longer rows take the streaming form (kLong)

// shared-memory staging block of one warp (float offsets)
enum {
  S_ROOT = 0, S_DOF = 16, S_EE = 64, S_FS = 80, S_TQ = 104, S_ACT = 128, S_AH = 152, S_GS = 176, S_DS = 204,
  S_SUM = 276, S_PRIV = 340, S_PROP = 372, S_CF = 468, S_TOTAL = 532
};

// WG:1316-1332 for one env; gs = staged goal_state row (all lanes compute, lane 0 commits)
__device__ void resample_goal(const DwbcEnvCfg& cfg, const DwbcStepArgs& A, const Rng& rng, float* gs, float yaw,
                              int col_orn, int col_sph, int lane) {
  float d[3], o[3];
  const float ye[3] = {0.0f, 0.0f, yaw};
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    d[i] = cfg.delta_orn_span[i] * rng(col_orn + i) + cfg.delta_orn_lo[i];
    o[i] = wrap_pi(d[i] + ye[i]);
  }
  V3 start = mk(gs[DWBC_GS_GOAL_SPH], gs[DWBC_GS_GOAL_SPH + 1], gs[DWBC_GS_GOAL_SPH + 2]);
  V3 goal = start;
  for (int k = 0; k < cfg.max_goal_tries; ++k) {
    goal = mk(A.goal_l[1] * rng(col_sph + 3 * k) + A.goal_l[0], A.goal_p[1] * rng(col_sph + 3 * k + 1) + A.goal_p[0],
              A.goal_y[1] * rng(col_sph + 3 * k + 2) + A.goal_y[0]);
    if (!goal_collides(cfg, start, goal)) break;
  }
  V3 gc = sphere2cart(goal);
  __syncwarp();
  if (lane == 0) {
    for (int i = 0; i < 3; ++i) { gs[DWBC_GS_DELTA_ORN + i] = d[i]; gs[DWBC_GS_GOAL_ORN + i] = o[i]; }
    gs[DWBC_GS_START_SPH] = start.x; gs[DWBC_GS_START_SPH + 1] = start.y; gs[DWBC_GS_START_SPH + 2] = start.z;
    gs[DWBC_GS_GOAL_SPH] = goal.x; gs[DWBC_GS_GOAL_SPH + 1] = goal.y; gs[DWBC_GS_GOAL_SPH + 2] = goal.z;
    gs[DWBC_GS_GOAL_CART] = gc.x; gs[DWBC_GS_GOAL_CART + 1] = gc.y; gs[DWBC_GS_GOAL_CART + 2] = gc.z;
    gs[DWBC_GS_GOAL_TIMER] = 0.0f;
  }
  __syncwarp();
}

// WG:831-843
__device__ void resample_commands(const DwbcEnvCfg& cfg, const DwbcStepArgs& A, const Rng& rng, float* gs, int col, int lane) {
  float cx = A.lin_vel_x[1] * rng(col) + A.lin_vel_x[0];
  float cy = A.ang_vel_yaw[1] * rng(col + 1) + A.ang_vel_yaw[0];
  float keep = (cx > cfg.lin_vel_x_clip || fabsf(cy) > cfg.ang_vel_yaw_clip) ? 1.0f : 0.0f;
  __syncwarp();
  if (lane == 0) { gs[0] = cx * keep; gs[1] = 0.0f * keep; gs[2] = cy * keep; }
  __syncwarp();
}

struct TermCtx {
  const DwbcEnvCfg& cfg;
  float* sm;        // staging block
  int lane, nd, na;
  float root_z;
  bool reset, time_out;
  float mean_height_gap;  // mean(root_z - measured_heights) (LR:846) when heights are measured
};

// One reward term for the env of this warp (value identical on all lanes).  Side effects on
// episode_metric_sums (WG:162-167) go to sm[S_SUM + n_sum_slots + metric].
__device__ float eval_term(int term, const TermCtx& c) {
  const DwbcEnvCfg& cfg = c.cfg;
  float* sm = c.sm;
  const int lane = c.lane, nd = c.nd, na = c.na;
  const float tq = lane < nd ? sm[S_TQ + lane] : 0.0f;
  const float dv = lane < nd ? sm[S_DOF + 2 * lane + 1] : 0.0f;
  const float dp = lane < nd ? sm[S_DOF + 2 * lane] : 0.0f;
  const float act = lane < na ? sm[S_ACT + lane] : 0.0f;
  const float* gs = sm + S_GS;
  const float* ds = sm + S_DS;
  float* met = sm + S_SUM + cfg.n_sum_slots;
  const bool l0 = lane == 0;
  float r = 0.0f;
  switch (term) {
    case DWBC_TERM_energy_square: {  // WG:1466-1469
      float e = lane < 12 ? tq * dv : 0.0f;
      r = warp_sum(e * e);
      if (l0) met[8] += r;
    } break;
    case DWBC_TERM_foot_contacts_z: {  // WG:1455-1458
      float f = lane < 4 ? sm[S_FS + 6 * lane + 2] : 0.0f;
      r = warp_sum(f * f);
      if (l0) met[9] += r;
    } break;
    case DWBC_TERM_hip_action_l2: {  // WG:1379-1382
      float a = (lane < 12 && lane % 3 == 0) ? act : 0.0f;
      r = warp_sum(a * a);
      if (l0) met[6] += r;
    } break;
    case DWBC_TERM_leg_action_l2: {  // WG:1405-1408
      float a = lane < 12 ? act : 0.0f;
      r = warp_sum(a * a);
      if (l0) met[6] += r;
    } break;
    case DWBC_TERM_survive: r = 1.0f; break;  // WG:1452-1453
    case DWBC_TERM_tracking_ang_vel_yaw_exp: {  // WG:1441-1444
      float e = fabsf(gs[2] - ds[DWBC_DS_BASE_ANG_VEL + 2]);
      if (l0) met[2] += e;
      r = nexp(-e / cfg.tracking_sigma);
    } break;
    case DWBC_TERM_tracking_ang_vel_yaw_l1: {  // WG:1437-1439
      float e = fabsf(gs[2] - ds[DWBC_DS_BASE_ANG_VEL + 2]);
      r = -e + fabsf(gs[2]);
    } break;
    case DWBC_TERM_tracking_lin_vel_x_l1: {  // WG:1427-1430
      float e = fabsf(gs[0] - ds[DWBC_DS_BASE_LIN_VEL]);
      if (l0) met[1] += e;
      r = -e + fabsf(gs[0]);
    } break;
    case DWBC_TERM_tracking_lin_vel_x_exp: {  // WG:1432-1435
      float e = fabsf(gs[0] - ds[DWBC_DS_BASE_LIN_VEL]);
      if (l0) met[1] += e;
      r = nexp(-e / cfg.tracking_sigma);
    } break;
    case DWBC_TERM_tracking_lin_vel_y_l2: { float e = gs[1] - ds[DWBC_DS_BASE_LIN_VEL + 1]; r = e * e; } break;  // WG:1446
    case DWBC_TERM_tracking_lin_vel_z_l2: { float e = gs[2] - ds[DWBC_DS_BASE_LIN_VEL + 2]; r = e * e; } break;  // WG:1449
    case DWBC_TERM_tracking_lin_vel: {  // WG:1422-1425
      float ex = gs[0] - ds[DWBC_DS_BASE_LIN_VEL], ey = gs[1] - ds[DWBC_DS_BASE_LIN_VEL + 1];
      r = nexp(-(ex * ex + ey * ey) / cfg.tracking_sigma);
    } break;
    case DWBC_TERM_tracking_ang_vel: {  // LR:886-889
      float e = gs[2] - ds[DWBC_DS_BASE_ANG_VEL + 2];
      r = nexp(-(e * e) / cfg.tracking_sigma);
    } break;
    case DWBC_TERM_torques: {  // WG:1460-1464
      r = warp_sum(tq * tq);
      if (l0) met[7] += r;
    } break;
    case DWBC_TERM_leg_energy_abs_sum: {  // WG:1396-1399
      r = warp_sum(lane < 12 ? fabsf(tq * dv) : 0.0f);
      if (l0) met[0] += r;
    } break;
    case DWBC_TERM_leg_energy_sum_abs: r = fabsf(warp_sum(lane < 12 ? tq * dv : 0.0f)); break;  // WG:1401-1403
    case DWBC_TERM_leg_energy: r = warp_sum(lane < 12 ? tq * dv : 0.0f); break;                 // WG:1410-1412
    case DWBC_TERM_arm_energy_abs_sum: r = warp_sum((lane >= 12 && lane < nd - 2) ? fabsf(tq * dv) : 0.0f); break;  // WG:1414
    case DWBC_TERM_tracking_ee_sphere: {  // WG:1352-1358
      V3 d = mk(sm[S_EE] - sm[S_ROOT], sm[S_EE + 1] - sm[S_ROOT + 1], sm[S_EE + 2] - cfg.z_invariant_offset);
      V3 s = cart2sphere(quat_rotate_inverse(ds + DWBC_DS_YAW_QUAT, d));
      float e = (fabsf(s.x - gs[DWBC_GS_CURR_SPH]) * cfg.sphere_error_scale[0] +
                 fabsf(s.y - gs[DWBC_GS_CURR_SPH + 1]) * cfg.sphere_error_scale[1]) +
                fabsf(s.z - gs[DWBC_GS_CURR_SPH + 2]) * cfg.sphere_error_scale[2];
      if (l0) met[4] += e;
      r = nexp(-e / cfg.tracking_ee_sigma);
    } break;
    case DWBC_TERM_tracking_ee_cart: {  // WG:1360-1366
      V3 t = quat_apply(ds + DWBC_DS_YAW_QUAT, mk(gs[DWBC_GS_CURR_CART], gs[DWBC_GS_CURR_CART + 1], gs[DWBC_GS_CURR_CART + 2]));
      float e = (fabsf(sm[S_EE] - (sm[S_ROOT] + t.x)) + fabsf(sm[S_EE + 1] - (sm[S_ROOT + 1] + t.y))) +
                fabsf(sm[S_EE + 2] - (cfg.z_invariant_offset + t.z));
      if (l0) met[3] += e;
      r = nexp(-e / cfg.tracking_ee_sigma);
    } break;
    case DWBC_TERM_tracking_ee_orn:
    case DWBC_TERM_tracking_ee_orn_ry: {  // WG:1368-1394
      float eu[3];
      euler_from_quat(sm + S_EE + 3, eu[0], eu[1], eu[2]);
      float d0 = wrap_pi(gs[DWBC_GS_GOAL_ORN] - eu[0]), d1 = wrap_pi(gs[DWBC_GS_GOAL_ORN + 1] - eu[1]),
            d2 = wrap_pi(gs[DWBC_GS_GOAL_ORN + 2] - eu[2]);
      float e;
      if (term == DWBC_TERM_tracking_ee_orn) {
        e = (fabsf(d0) * cfg.orn_error_scale[0] + fabsf(d1) * cfg.orn_error_scale[1]) + fabsf(d2) * cfg.orn_error_scale[2];
      } else {
        e = fabsf(d0 * cfg.orn_error_scale[0]) + fabsf(d2 * cfg.orn_error_scale[2]);
        if (l0) met[5] += e;
      }
      r = nexp(-e / cfg.tracking_ee_sigma);
    } break;
    case DWBC_TERM_lin_vel_z: r = ds[DWBC_DS_BASE_LIN_VEL + 2] * ds[DWBC_DS_BASE_LIN_VEL + 2]; break;  // LR:832
    case DWBC_TERM_ang_vel_xy:  // LR:836
      r = ds[DWBC_DS_BASE_ANG_VEL] * ds[DWBC_DS_BASE_ANG_VEL] + ds[DWBC_DS_BASE_ANG_VEL + 1] * ds[DWBC_DS_BASE_ANG_VEL + 1];
      break;
    case DWBC_TERM_base_height: { float g = c.mean_height_gap - cfg.base_height_target; r = g * g; } break;  // LR:844-847
    case DWBC_TERM_dof_vel: r = warp_sum(dv * dv); break;                                                  // LR:853
    case DWBC_TERM_dof_acc: {  // LR:857-859
      float a = lane < nd ? (ds[DWBC_DS_LAST_DOF_VEL + lane] - dv) / cfg.dt : 0.0f;
      r = warp_sum(a * a);
    } break;
    case DWBC_TERM_action_rate: {  // LR:861-863
      float a = lane < na ? ds[DWBC_DS_LAST_ACTIONS + lane] - act : 0.0f;
      r = warp_sum(a * a);
    } break;
    case DWBC_TERM_collision: {  // LR:865-867
      float v = 0.0f;
      if (lane < cfg.n_penalized) {
        const float* f = sm + S_CF + 3 * (4 + lane);
        v = sqrtf((f[0] * f[0] + f[1] * f[1]) + f[2] * f[2]) > 0.1f ? 1.0f : 0.0f;
      }
      r = warp_sum(v);
    } break;
    case DWBC_TERM_termination: r = (c.reset && !c.time_out) ? 1.0f : 0.0f; break;  // LR:869-871
    case DWBC_TERM_dof_pos_limits: {  // LR:873-877
      float o = 0.0f;
      if (lane < nd) o = -fminf(dp - cfg.dof_pos_lower[lane], 0.0f) + fmaxf(dp - cfg.dof_pos_upper[lane], 0.0f);
      r = warp_sum(o);
    } break;
    case DWBC_TERM_dof_vel_limits:  // LR:879-882
      r = warp_sum(lane < nd ? clipf(fabsf(dv) - cfg.dof_vel_limits[lane] * cfg.soft_dof_vel_limit, 0.0f, 1.0f) : 0.0f);
      break;
    case DWBC_TERM_torque_limits:  // LR:884-886
      r = warp_sum(lane < nd ? fmaxf(fabsf(tq) - cfg.torque_limits[lane] * cfg.soft_torque_limit, 0.0f) : 0.0f);
      break;
    case DWBC_TERM_feet_air_time: {  // LR:896-908 (stateful: feet_air_time, last_contacts)
      float v = 0.0f;
      if (lane < 4) {
        bool contact = sm[S_CF + 3 * lane + 2] > 1.0f;
        bool filt = contact || (sm[S_DS + DWBC_DS_LAST_CONTACTS + lane] != 0.0f);
        float fat = sm[S_DS + DWBC_DS_FEET_AIR_TIME + lane];
        bool first = (fat > 0.0f) && filt;
        fat += cfg.dt;
        v = (fat - 0.5f) * (first ? 1.0f : 0.0f);
        sm[S_DS + DWBC_DS_LAST_CONTACTS + lane] = contact ? 1.0f : 0.0f;
        sm[S_DS + DWBC_DS_FEET_AIR_TIME + lane] = fat * (filt ? 0.0f : 1.0f);
      }
      r = warp_sum(v) * ((sqrtf(gs[0] * gs[0] + gs[1] * gs[1]) > 0.1f) ? 1.0f : 0.0f);
      __syncwarp();
    } break;
    case DWBC_TERM_stumble: {  // LR:910-913
      bool s = false;
      if (lane < 4) {
        const float* f = sm + S_CF + 3 * lane;
        s = sqrtf(f[0] * f[0] + f[1] * f[1]) > 5.0f * fabsf(f[2]);
      }
      r = __any_sync(FULL, s) ? 1.0f : 0.0f;
    } break;
    case DWBC_TERM_stand_still: {  // LR:915-917
      float s = warp_sum(lane < nd ? fabsf(dp - cfg.default_dof_pos[lane]) : 0.0f);
      r = s * ((sqrtf(gs[0] * gs[0] + gs[1] * gs[1]) < 0.1f) ? 1.0f : 0.0f);
    } break;
    case DWBC_TERM_feet_contact_forces: {  // LR:919-921
      float v = 0.0f;
      if (lane < 4) {
        const float* f = sm + S_CF + 3 * lane;
        v = fmaxf(sqrtf((f[0] * f[0] + f[1] * f[1]) + f[2] * f[2]) - cfg.max_contact_force, 0.0f);
      }
      r = warp_sum(v);
    } break;
    default: break;
  }
  return r;
}

// kLong = false: the history row (<= 1024 floats) is loaded into registers before anything else and re-emitted from there.
// kLong = true (history_len * num_prop > 1024, e.g. 20 or 50 steps of 76): the row is streamed at the end instead, in ascending
// 32-float4 chunks: each chunk is loaded, written to obs clipped (WG:992, 1195-1196), and after a __syncwarp written back one num_prop
// row lower (WG:997-999).  In place is safe: the targets of chunk i lie below its end, so chunks <= i have read them already.
template <bool kLong>
__global__ void __launch_bounds__(ENV_WARPS * 32)
env_step_kernel(const __grid_constant__ DwbcEnvCfg cfg, const __grid_constant__ DwbcEnvBuffers B,
                const __grid_constant__ DwbcStepArgs A) {
  __shared__ __align__(16) float smem[ENV_WARPS * S_TOTAL];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int e = blockIdx.x * ENV_WARPS + wid;
  if (e >= cfg.num_envs) return;
  float* sm = smem + wid * S_TOTAL;
  const int nd = cfg.num_dofs, na = cfg.num_actions, P = cfg.num_prop, H = cfg.history_len;
  const int nbp1 = cfg.num_bodies_p1;
  const int nh4 = (H * P) >> 2, p4 = P >> 2, pp4 = (P + cfg.num_priv) >> 2;
  const int nslots = cfg.n_sum_slots + DWBC_NUM_METRICS;

  // ---- 1. history row: all 128-bit loads in flight first --------------------------------------
  float4* hist4 = reinterpret_cast<float4*>(B.obs_history + (size_t)e * H * P);
  float4 h[kLong ? 1 : MAX_H4];
  bool hist_zeroed = false;                  // (kLong) reset this step: the old history reads as zeros (WG:735)
  if constexpr (!kLong) {
#pragma unroll
    for (int i = 0; i < MAX_H4; ++i) {
      int idx = lane + 32 * i;
      h[i] = idx < nh4 ? ldg_stream(hist4 + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  // ---- 2. coalesced staging of the env's small inputs ------------------------------------------
  float* root_g = B.root_states + (size_t)e * 26;
  if (lane < 13) sm[S_ROOT + lane] = root_g[lane];
  float* dof_g = B.dof_state + (size_t)e * 2 * nd;
  for (int i = lane; i < 2 * nd; i += 32) sm[S_DOF + i] = dof_g[i];
  if (lane < 13) sm[S_EE + lane] = __ldg(B.rigid_body_state + ((size_t)e * nbp1 + cfg.gripper_idx) * 13 + lane);
  if (lane < 24) sm[S_FS + lane] = __ldg(B.force_sensor + (size_t)e * 24 + lane);
  if (lane < nd) sm[S_TQ + lane] = __ldg(B.torques + (size_t)e * nd + lane);
  if (lane < na) sm[S_ACT + lane] = __ldg(B.actions + (size_t)e * na + lane);
  float* ah_g = B.action_history + (size_t)e * cfg.action_hist_len * na;
  if (lane < na) sm[S_AH + lane] = ah_g[(cfg.action_hist_len - 1) * na + lane];
  float* gs_g = B.goal_state + (size_t)e * DWBC_GS;
  if (lane < DWBC_GS) sm[S_GS + lane] = gs_g[lane];
  float* ds_g = B.derived_state + (size_t)e * DWBC_DS;
  for (int i = DWBC_DS_FEET_AIR_TIME + lane; i < DWBC_DS; i += 32) sm[S_DS + i] = ds_g[i];
  float* sum_g = B.episode_sums + (size_t)e * cfg.sums_stride;
  for (int i = lane; i < nslots; i += 32) sm[S_SUM + i] = sum_g[i];
  if (lane < 5) sm[S_PRIV + lane] = __ldg(B.mass_params + (size_t)e * 5 + lane);
  else if (lane == 5) sm[S_PRIV + 5] = __ldg(B.friction + e);
  if (lane < na) sm[S_PRIV + 6 + lane] = __ldg(B.motor_strength + (size_t)e * na + lane) - 1.0f;
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

  Rng rng{A.rand_uniform, A.seed, A.step, e};
  float* gs = sm + S_GS;
  float* ds = sm + S_DS;

  // ---- 3. derived base state (WG:879-884) -------------------------------------------------------
  float yaw;
  {
    const float* q = sm + S_ROOT + 3;
    V3 blv = quat_rotate_inverse(q, mk(sm[S_ROOT + 7], sm[S_ROOT + 8], sm[S_ROOT + 9]));
    V3 bav = quat_rotate_inverse(q, mk(sm[S_ROOT + 10], sm[S_ROOT + 11], sm[S_ROOT + 12]));
    float r0, p0;
    euler_from_quat(q, r0, p0, yaw);
    float cy = ncos(yaw * 0.5f), sy = nsin(yaw * 0.5f);
    __syncwarp();
    if (lane == 0) {
      ds[DWBC_DS_BASE_LIN_VEL] = blv.x; ds[DWBC_DS_BASE_LIN_VEL + 1] = blv.y; ds[DWBC_DS_BASE_LIN_VEL + 2] = blv.z;
      ds[DWBC_DS_BASE_ANG_VEL] = bav.x; ds[DWBC_DS_BASE_ANG_VEL + 1] = bav.y; ds[DWBC_DS_BASE_ANG_VEL + 2] = bav.z;
      ds[DWBC_DS_YAW_EULER] = 0.0f; ds[DWBC_DS_YAW_EULER + 1] = 0.0f; ds[DWBC_DS_YAW_EULER + 2] = yaw;
      ds[DWBC_DS_YAW_QUAT] = 0.0f; ds[DWBC_DS_YAW_QUAT + 1] = 0.0f; ds[DWBC_DS_YAW_QUAT + 2] = sy; ds[DWBC_DS_YAW_QUAT + 3] = cy;
    }
    __syncwarp();
  }
  // ---- 4. EE goal interpolation + timer (WG:1344-1350) ------------------------------------------
  {
    float t = clipf(gs[DWBC_GS_GOAL_TIMER] / gs[DWBC_GS_TRAJ_T], 0.0f, 1.0f);
    V3 cs = lerp3(mk(gs[DWBC_GS_START_SPH], gs[DWBC_GS_START_SPH + 1], gs[DWBC_GS_START_SPH + 2]),
                  mk(gs[DWBC_GS_GOAL_SPH], gs[DWBC_GS_GOAL_SPH + 1], gs[DWBC_GS_GOAL_SPH + 2]), t);
    V3 cc = sphere2cart(cs);
    float timer = gs[DWBC_GS_GOAL_TIMER] + 1.0f;
    bool expired = timer > gs[DWBC_GS_TRAJ_TOTAL];
    __syncwarp();
    if (lane == 0) {
      gs[DWBC_GS_CURR_SPH] = cs.x; gs[DWBC_GS_CURR_SPH + 1] = cs.y; gs[DWBC_GS_CURR_SPH + 2] = cs.z;
      gs[DWBC_GS_CURR_CART] = cc.x; gs[DWBC_GS_CURR_CART + 1] = cc.y; gs[DWBC_GS_CURR_CART + 2] = cc.z;
      gs[DWBC_GS_GOAL_TIMER] = timer;
    }
    __syncwarp();
    if (expired) resample_goal(cfg, A, rng, gs, yaw, DWBC_RAND_GOAL_ORN, DWBC_RAND_GOAL_SPH, lane);
  }
  // ---- 5. callback: command resampling, height scan, push (WG:917-935) --------------------------
  if (ep % cfg.resample_interval == 0) resample_commands(cfg, A, rng, gs, DWBC_RAND_CMD, lane);
  float mean_gap = 0.0f;
  if (cfg.measure_heights) {  // LR:793-829
    const int npts = cfg.n_height_x * cfg.n_height_y;
    float qy[4] = {0.0f, 0.0f, sm[S_ROOT + 5], sm[S_ROOT + 6]};
    float n = fmaxf(sqrtf(qy[2] * qy[2] + qy[3] * qy[3]), 1e-9f);  // utils/math.py:38-42 + normalize()
    qy[2] = qy[2] / n; qy[3] = qy[3] / n;
    float gap = 0.0f;
    for (int i = lane; i < npts; i += 32) {
      int ix = i / cfg.n_height_y, iy = i - ix * cfg.n_height_y;
      V3 pt = quat_apply(qy, mk(cfg.height_x[ix], cfg.height_y[iy], 0.0f));
      float fx = ((pt.x + sm[S_ROOT]) + cfg.border_size) / cfg.horizontal_scale;
      float fy = ((pt.y + sm[S_ROOT + 1]) + cfg.border_size) / cfg.horizontal_scale;
      long long px = (long long)fx, py = (long long)fy;  // .long(): truncation toward zero
      px = px < 0 ? 0 : (px > cfg.terrain_rows - 2 ? cfg.terrain_rows - 2 : px);
      py = py < 0 ? 0 : (py > cfg.terrain_cols - 2 ? cfg.terrain_cols - 2 : py);
      const int16_t* hs = B.height_samples + px * cfg.terrain_cols + py;
      int16_t m = min(min(__ldg(hs), __ldg(hs + cfg.terrain_cols)), __ldg(hs + 1));
      float hgt = (float)m * cfg.vertical_scale;
      B.measured_heights[(size_t)e * npts + i] = hgt;
      gap += sm[S_ROOT + 2] - hgt;
    }
    mean_gap = warp_sum(gap) / (float)npts;
  }
  bool root_dirty = false;
  if (A.do_push) {  // WG:804-814
    float vx = cfg.push_vel[1] * rng(DWBC_RAND_PUSH) + cfg.push_vel[0];
    float vy = cfg.push_vel[1] * rng(DWBC_RAND_PUSH + 1) + cfg.push_vel[0];
    if (((gs[0] + gs[1]) + gs[2]) == 0.0f) { vx *= 2.5f; vy *= 2.5f; }
    __syncwarp();
    if (lane == 0) { sm[S_ROOT + 7] = vx; sm[S_ROOT + 8] = vy; }
    __syncwarp();
    root_dirty = true;
  }
  // ---- 6. termination (WG:937-963) ---------------------------------------------------------------
  bool time_out, reset;
  {
    bool contact = false;
    for (int i = 0; i < cfg.n_term_contact; ++i) {
      const float* f = sm + S_CF + 3 * (4 + cfg.n_penalized + i);
      contact = contact || (sqrtf((f[0] * f[0] + f[1] * f[1]) + f[2] * f[2]) > 1.0f);
    }
    float r0, p0, y0;
    euler_from_quat(sm + S_ROOT + 3, r0, p0, y0);
    const float* g = gs + (cfg.goal_is_cart ? DWBC_GS_CURR_CART : DWBC_GS_CURR_SPH);
    bool r_bad = ((r0 > cfg.term_roll) && (g[2] >= 0.0f)) || ((r0 < -cfg.term_roll) && (g[2] <= 0.0f));
    bool p_bad = ((p0 > cfg.term_pitch) && (g[1] >= 0.0f)) || ((p0 < -cfg.term_pitch) && (g[1] <= 0.0f));
    bool z_bad = sm[S_ROOT + 2] < cfg.term_z;
    time_out = ep > cfg.max_episode_length;
    reset = contact || r_bad || p_bad || z_bad || time_out;
  }
  // ---- 7. rewards (WG:170-205) -------------------------------------------------------------------
  float rew[2];
  {
    TermCtx ctx{cfg, sm, lane, nd, na, sm[S_ROOT + 2], reset, time_out, mean_gap};
#pragma unroll
    for (int ch = 0; ch < 2; ++ch) {
      const int n = ch == 0 ? cfg.n_leg_terms : cfg.n_arm_terms;
      const int32_t* terms = ch == 0 ? cfg.leg_term : cfg.arm_term;
      const int32_t* slots = ch == 0 ? cfg.leg_slot : cfg.arm_slot;
      const float* scales = ch == 0 ? A.leg_scale : A.arm_scale;
      float buf = 0.0f;
      for (int i = 0; i < n; ++i) {
        float r = eval_term(terms[i], ctx) * scales[i];
        buf += r;
        if (lane == 0) sm[S_SUM + slots[i]] += r;
      }
      if (cfg.only_positive_rewards) buf = fmaxf(buf, 0.0f);
      float ts = ch == 0 ? A.leg_termination_scale : A.arm_termination_scale;
      if (ts != 0.0f && cfg.termination_slot >= 0) {
        float r = ((reset && !time_out) ? 1.0f : 0.0f) * ts;
        buf += r;
        if (lane == 0) sm[S_SUM + cfg.termination_slot] += r;
      }
      rew[ch] = buf / 100.0f;
    }
    __syncwarp();
  }
  // ---- 8. reset (WG:695-754) ---------------------------------------------------------------------
  if (reset) {
    if (cfg.terrain_curriculum) {  // LR:421-441 (base-class semantics, SURVEY a21)
      float* org = B.env_origins + (size_t)e * 3;
      float dx = sm[S_ROOT] - org[0], dy = sm[S_ROOT + 1] - org[1];
      float dist = sqrtf(dx * dx + dy * dy);
      bool up = dist > cfg.terrain_env_length / 2.0f;
      bool down = (dist < sqrtf(gs[0] * gs[0] + gs[1] * gs[1]) * cfg.max_episode_length_s * 0.5f) && !up;
      long long lvl = B.terrain_levels[e] + (up ? 1 : 0) - (down ? 1 : 0);
      if (lvl >= cfg.max_terrain_level) {
        long long rl = (long long)(rng(DWBC_RAND_TERRAIN) * (float)cfg.max_terrain_level);
        lvl = rl > cfg.max_terrain_level - 1 ? cfg.max_terrain_level - 1 : rl;
      } else if (lvl < 0) {
        lvl = 0;
      }
      const float* to = B.terrain_origins + ((size_t)lvl * cfg.terrain_n_types + B.terrain_types[e]) * 3;
      float o0 = to[0], o1 = to[1], o2 = to[2];
      __syncwarp();
      if (lane == 0) { B.terrain_levels[e] = lvl; org[0] = o0; org[1] = o1; org[2] = o2; }
      __syncwarp();
    }
    // _reset_dofs WG:816-828
    if (lane < nd) {
      float pos = cfg.default_dof_pos[lane] * (cfg.dof_reset[1] * rng(DWBC_RAND_RST_DOF + lane) + cfg.dof_reset[0]);
      sm[S_DOF + 2 * lane] = pos;
      sm[S_DOF + 2 * lane + 1] = 0.0f;
    }
    // _reset_root_states WG:757-788
    if (lane < 13) {
      float v = cfg.base_init_state[lane];
      if (lane < 3) v += B.env_origins[(size_t)e * 3 + lane];
      if (lane < 2) v += cfg.origin_perturb[1] * rng(DWBC_RAND_RST_XY + lane) + cfg.origin_perturb[0];
      if (lane >= 7) v = cfg.init_vel_perturb[1] * rng(DWBC_RAND_RST_VEL + lane - 7) + cfg.init_vel_perturb[0];
      sm[S_ROOT + lane] = v;
    }
    __syncwarp();
    for (int i = lane; i < 2 * nd; i += 32) dof_g[i] = sm[S_DOF + i];
    if (lane == 0) {
      root_g[13] = cfg.box_x;
      root_g[14] = sm[S_ROOT + 1] + B.box_env_origins_delta_y[e];
      root_g[15] = cfg.box_z;
    }
    root_dirty = true;
    if (time_out) resample_commands(cfg, A, rng, gs, DWBC_RAND_RST_CMD, lane);  // WG:723-727
    resample_goal(cfg, A, rng, gs, yaw, DWBC_RAND_RST_GOAL_ORN, DWBC_RAND_RST_GOAL_SPH, lane);
    // buffers WG:732-740
    if (lane < 4) sm[S_DS + DWBC_DS_FEET_AIR_TIME + lane] = 0.0f;
    if (lane < na) sm[S_AH + lane] = 0.0f;
    for (int i = lane; i < cfg.action_hist_len * na; i += 32) ah_g[i] = 0.0f;
    if constexpr (!kLong) {
#pragma unroll
      for (int i = 0; i < MAX_H4; ++i) h[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
      hist_zeroed = true;
    }
    ep = 0;
    // extras['episode'] means (WG:743-750): the ended episode's sums go to this env's slot; episode_stats_kernel adds them up
    for (int i = lane; i < nslots; i += 32) {
      B.episode_scratch[(size_t)e * cfg.sums_stride + i] = sm[S_SUM + i];
      sm[S_SUM + i] = 0.0f;
    }
    __syncwarp();
  }
  if (root_dirty && lane < 13) root_g[lane] = sm[S_ROOT + lane];

  // ---- 9. observations (WG:966-1001, column map SURVEY Appendix B) ------------------------------
  {
    float r0, p0, y0;
    euler_from_quat(sm + S_ROOT + 3, r0, p0, y0);  // post-reset quaternion (base_quat is a view, WG:535)
    float* prop = sm + S_PROP;
    if (lane == 0) {
      prop[0] = r0; prop[1] = p0;
      for (int i = 0; i < 3; ++i) prop[2 + i] = ds[DWBC_DS_BASE_ANG_VEL + i] * cfg.obs_scale_ang_vel;
    }
    if (lane < nd) {
      int d = cfg.ig2raisim[lane];
      float pos = sm[S_DOF + 2 * d];
      if (d == cfg.waist_dof) pos = wrap_pi(pos);
      prop[5 + lane] = (pos - cfg.default_dof_pos[d]) * cfg.obs_scale_dof_pos;
      prop[5 + nd + lane] = sm[S_DOF + 2 * d + 1] * cfg.obs_scale_dof_vel;
    }
    if (lane < na) prop[5 + 2 * nd + lane] = sm[S_AH + cfg.ig2raisim[lane]];
    const int o = 5 + 2 * nd + na;
    if (lane < 4) {
      const float* f = sm + S_FS + 6 * cfg.feet_perm[lane];
      float nrm = sqrtf(((((f[0] * f[0] + f[1] * f[1]) + f[2] * f[2]) + f[3] * f[3]) + f[4] * f[4]) + f[5] * f[5]);
      prop[o + lane] = nrm > 1.5f ? 1.0f : 0.0f;
    }
    if (lane == 31) {
      prop[o + 4] = gs[0] * cfg.obs_scale_lin_vel;
      prop[o + 5] = gs[1] * cfg.obs_scale_lin_vel;
      prop[o + 6] = gs[2] * cfg.obs_scale_ang_vel;
      const float* g = gs + (cfg.goal_is_cart ? DWBC_GS_CURR_CART : DWBC_GS_CURR_SPH);
      for (int i = 0; i < 3; ++i) { prop[o + 7 + i] = g[i]; prop[o + 10 + i] = gs[DWBC_GS_DELTA_ORN + i]; }
    }
    // tail copies WG:908-910
    if (lane < na) ds[DWBC_DS_LAST_ACTIONS + lane] = sm[S_ACT + lane];
    if (lane < nd) ds[DWBC_DS_LAST_DOF_VEL + lane] = sm[S_DOF + 2 * lane + 1];
    if (lane < 6) ds[DWBC_DS_LAST_ROOT_VEL + lane] = sm[S_ROOT + 7 + lane];
    if (lane == 7) ds[27] = 0.0f;  // DWBC_DS_OOB_AGE (v2 fast-path bookkeeping): v1 always clips, stay conservative
    __syncwarp();
  }
  // ---- 10. outputs -------------------------------------------------------------------------------
  const float c = cfg.clip_obs > 0.0f ? cfg.clip_obs : INFINITY;
  float4* obs4 = reinterpret_cast<float4*>(B.obs_buf + (size_t)e * B.obs_stride);
  const float4* prop4 = reinterpret_cast<const float4*>(sm + S_PROP);
  const float4* priv4 = reinterpret_cast<const float4*>(sm + S_PRIV);
  if (lane < pp4) stg_stream(obs4 + lane, clip4(lane < p4 ? prop4[lane] : priv4[lane - p4], c));
  if constexpr (!kLong) {
#pragma unroll
    for (int i = 0; i < MAX_H4; ++i) {
      int idx = lane + 32 * i;
      if (idx < nh4) stg_stream(obs4 + pp4 + idx, clip4(h[i], c));  // OLD history (WG:992)
    }
    __syncwarp();  // every lane's history loads have been consumed: the in-place shift below is safe
    if (ep <= 1) {  // WG:994-996: fill all H rows with the new proprioception
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
      h[0] = idx < nh4 && !hist_zeroed ? __ldcs(hist4 + idx) : zero4;
      if (idx < nh4) stg_stream(obs4 + pp4 + idx, clip4(h[0], c));    // OLD history (WG:992)
      __syncwarp();  // the whole chunk has been read: its targets (and everything below them) may be overwritten
      if (ep <= 1) {          // WG:994-996
        if (idx < nh4) hist4[idx] = prop4[idx % p4];
      } else if (idx >= p4 && idx < nh4) {
        hist4[idx - p4] = h[0];                                            // WG:997-999
      }
    }
    if (ep > 1 && lane < p4) hist4[nh4 - p4 + lane] = prop4[lane];          // WG:1000
  }
  if (lane < DWBC_GS) gs_g[lane] = sm[S_GS + lane];
  for (int i = lane; i < DWBC_DS; i += 32) ds_g[i] = sm[S_DS + i];
  for (int i = lane; i < nslots; i += 32) sum_g[i] = sm[S_SUM + i];
  if (lane == 0) {
    B.episode_length[e] = ep;
    B.rew_buf[e] = rew[0];
    B.arm_rew_buf[e] = rew[1];
    B.reset_buf[e] = reset ? 1 : 0;
    B.time_out_buf[e] = time_out ? 1 : 0;
    if (B.store_rewards) {          // PPO.process_env_step's reward path (PPO:130-134) + dones (RS:102), straight into the storage rows
      const float to = time_out ? 1.0f : 0.0f;
      B.store_rewards[2 * (size_t)e] = rew[0] + B.store_gamma * (B.store_values[2 * (size_t)e] * to);
      B.store_rewards[2 * (size_t)e + 1] = rew[1] + B.store_gamma * (B.store_values[2 * (size_t)e + 1] * to);
      if (B.store_dones) B.store_dones[e] = reset ? 1 : 0;
    }
  }
  if (cfg.measure_heights && B.heights_obs) {  // LR:221-223
    const int npts = cfg.n_height_x * cfg.n_height_y;
    for (int i = lane; i < npts; i += 32)
      B.heights_obs[(size_t)e * npts + i] =
          clipf((sm[S_ROOT + 2] - 0.5f) - B.measured_heights[(size_t)e * npts + i], -1.0f, 1.0f) * cfg.obs_scale_height;
  }
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
  // v2 (16 envs per CTA, TMA bulk copies) whenever the shard is a multiple of 32 envs and every block is 16-B aligned
  if (cfg->num_envs % 32 == 0 && aligned16(buf->root_states) && aligned16(buf->dof_state) && aligned16(buf->force_sensor) &&
      aligned16(buf->torques) && aligned16(buf->actions) && aligned16(buf->action_history) && aligned16(buf->mass_params) &&
      aligned16(buf->friction) && aligned16(buf->motor_strength) && aligned16(buf->goal_state) && aligned16(buf->derived_state) &&
      aligned16(buf->episode_length) && aligned16(buf->episode_sums) && !args->generic_kernel) {
    const int rc = dwbc_launch_env_step_v2(cfg, buf, args, dev, (cudaStream_t)stream);
    if (rc != DWBC_ERR_UNSUPPORTED) return rc == DWBC_OK ? launch_episode_stats(cfg, buf, dev, (cudaStream_t)stream) : rc;
  }
  if (dev) return DWBC_ERR_UNSUPPORTED;      // the warp-per-env kernel reads the host fields only
  const int grid = (cfg->num_envs + ENV_WARPS - 1) / ENV_WARPS;
  if ((int64_t)cfg->history_len * cfg->num_prop <= MAX_H4 * 128)
    env_step_kernel<false><<<grid, ENV_WARPS * 32, 0, (cudaStream_t)stream>>>(*cfg, *buf, *args);
  else
    env_step_kernel<true><<<grid, ENV_WARPS * 32, 0, (cudaStream_t)stream>>>(*cfg, *buf, *args);
  DWBC_LAUNCH_CHECK();
  return launch_episode_stats(cfg, buf, nullptr, (cudaStream_t)stream);
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
