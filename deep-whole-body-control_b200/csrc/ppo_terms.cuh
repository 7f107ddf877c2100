// Per-row terms of the PPO loss (AC:326-345, PPO:166-239), written once for both paths that compute it: the epilogue hooks of the fused
// chains (c2_fin_act / c2_fin_ppo / c2_fin_value / c2_fin_reg in mlp_chain2.cuh) and the layer-wise kernels of mlp.cu (act_finalize_kernel,
// ppo_loss_kernel, and the ratio and clip test of ppo_diag_kernel).  Each function computes one row's term of one action or channel and
// returns it; the loads, the stores and every reduction stay with the callers, in the order each path sums.  mlp.cu is compiled with FMA
// contraction on, so which multiply-adds fuse depends on how an expression is written: keep each one as it stands, or both paths' bits move.
// Loss terms with a gradient return them as (loss, gradient).
#pragma once
#include "common.cuh"

namespace dwbc {

// everything the update's loss needs, and the rollout's sampling (AC:326-345, PPO:166-221): the arguments of the chains' epilogue hooks and
// of act_finalize_kernel / ppo_loss_kernel
struct FinArgs {
  const float* std;                                          // [n_act]
  // FIN_ACT (rollout): a = mu + std * eps.  actions == nullptr: the mean only (dwbc_policy_mean; eps, log_prob, sigma_out unread)
  const float* eps; float* actions; float* log_prob; float* mean_out; float* sigma_out;
  // FIN_PPO / FIN_VALUE / FIN_REG (update)
  const int64_t* idx;                                        // mini-batch gather index (storage row of mini-batch row r)
  const float* s_actions; const float* old_logp; const float* old_values; const float* returns; const float* adv;
  const float* zh; int64_t zh_ld; int zh_by_src;
  float* g_leg; int gleg_ld; float* g_arm; int garm_ld; float* g_v; int gv_ld; float* g_z; int gz_ld;   // g_v: [rows, gv_ld], value columns 0, 1
  float* grad_std; float* losses;
  float* part;                                               // partial sums (C2_FIN_PART per chain slot, LOSS_PART per ppo_loss_kernel block)
  int n_leg, n_act, latent, rows;
  float clip, c_value, c_ent, c_reg, rho;
  int clipped_value;
  // arm torque supervision (PPO:224-239, fixed gains PPO:318-323); ts_target == nullptr: off.  Rows of [T*N, n_arm] storage tensors,
  // ts_coef = [3][n_arm] default p gains, d gains, default dof positions; ts_w = schedule weight (PPO:304-305); losses[4] += mean loss
  const float* ts_target; const float* ts_pos; const float* ts_vel; const float* ts_coef;
  float ts_w;
  // optional device (c_reg, rho, ts_w) in place of the three fields (dwbc_ppo_minibatch_grad_sched): the kernels load them once per CTA
  // (chain2_kernel into C2Shared, ppo_loss_kernel into shared memory)
  const float* sched;
};

constexpr float LOG_SQRT_2PI = 0.91893853320467274178f;

// One action's term of the Gaussian log-prob (AC:341-345), log_sg = logf(sg).  The rollout, the PPO loss of both paths and ppo_diag_kernel
// sum it over a channel's actions in index order, so the diagnostics see the ratio the loss saw, bit for bit.
__device__ __forceinline__ float ppo_logp_term(float a, float mu, float sg, float log_sg) {
  const float d = a - mu;
  return -(d * d) / (2.0f * (sg * sg)) - log_sg - LOG_SQRT_2PI;
}
// one action's entropy term (AC:326-331; 0.5 log 2pi == log sqrt 2pi)
__device__ __forceinline__ float ppo_entropy_term(float log_sg) { return 0.5f + LOG_SQRT_2PI + log_sg; }

// advantage of channel c (0 leg, 1 arm) mixed with the other channel's (PPO:199-201)
__device__ __forceinline__ float ppo_mix(float2 adv, int c, float rho) { return c == 0 ? adv.x + rho * adv.y : adv.y + rho * adv.x; }
__device__ __forceinline__ float ppo_ratio(float lp, float old_lp) { return expf(lp - old_lp); }     // PPO:202
// the ratio lies within the clip range: the surrogate's gradient passes through the clipped branch, and the row does not count towards
// the diagnostics' clip fraction
__device__ __forceinline__ bool ppo_inside(float ratio, float clip) { return ratio >= 1.0f - clip && ratio <= 1.0f + clip; }
// clipped surrogate max(-mix ratio, -mix clip(ratio)) (PPO:203-205) and its derivative w.r.t. the ratio; at s1 == s2 the mean of the two
// branches' derivatives
__device__ __forceinline__ float2 ppo_surrogate(float mix, float ratio, float clip) {
  const float rc = fminf(fmaxf(ratio, 1.0f - clip), 1.0f + clip);
  const float s1 = -mix * ratio, s2 = -mix * rc;
  const bool inside = ppo_inside(ratio, clip);
  float g;
  if (s1 > s2) g = -mix;
  else if (s1 == s2) g = 0.5f * -mix + (inside ? 0.5f * -mix : 0.0f);
  else g = inside ? -mix : 0.0f;
  return make_float2(fmaxf(s1, s2), g);
}
// gradients of one action's log-prob term scaled by glp = d loss / d log-prob: w.r.t. the pre-tanh mean output (AC:157,170) and, with the
// entropy bonus, w.r.t. the std (inv2m = 1 / (2 rows))
__device__ __forceinline__ float ppo_grad_mean(float glp, float a, float mu, float sg) {
  const float d = a - mu;
  return glp * d / (sg * sg) * (1.0f - mu * mu);
}
__device__ __forceinline__ float ppo_grad_std(float glp, float a, float mu, float sg, float c_ent, float inv2m) {
  const float d = a - mu;
  return glp * ((d * d) / (sg * sg * sg) - 1.0f / sg) - c_ent * inv2m / sg;
}

// Arm torque supervision (PPO:224-239, off in the shipped config WGC:173) of arm joint i of storage row src (cnt arm joints): tau = kp (mu +
// q_default - q) - kd qd (fixed gains, PPO:318-323) on the arm means (PPO:230), loss = w * mean((tau - target)^2) (PPO:236-238).  Returns
// (squared error, d loss / d pre-tanh output).
__device__ __forceinline__ float2 ppo_torque_term(const FinArgs& f, int64_t src, int cnt, int i, float mu, float ts_w) {
  const float kp = f.ts_coef[i];
  const float e = kp * (mu + f.ts_coef[2 * cnt + i] - f.ts_pos[src * cnt + i]) - f.ts_coef[cnt + i] * f.ts_vel[src * cnt + i] - f.ts_target[src * cnt + i];
  return make_float2(e * e, 2.0f * ts_w / ((float)f.rows * (float)cnt) * e * kp * (1.0f - mu * mu));
}

// value loss of one row and channel (PPO:209-216), clipped or not, and its UNSCALED derivative w.r.t. the value: each caller applies
// c_value / (2 rows) in its own order.  At l1 == l2 the mean of the two branches' derivatives.
__device__ __forceinline__ float2 ppo_value_term(float val, float vo, float R, float clip, int clipped) {
  const float l1 = (val - R) * (val - R);
  if (!clipped) return make_float2(l1, 2.0f * (val - R));
  const float dvo = val - vo;
  const float vc = vo + fminf(fmaxf(dvo, -clip), clip);
  const float l2 = (vc - R) * (vc - R);
  const bool inside = dvo >= -clip && dvo <= clip;
  const float g1 = 2.0f * (val - R), g2 = inside ? 2.0f * (vc - R) : 0.0f;
  return make_float2(fmaxf(l1, l2), l1 > l2 ? g1 : (l1 == l2 ? 0.5f * g1 + 0.5f * g2 : g2));
}

// privileged-latent regulariser (PPO:174-177): || z - zh ||_2 of one row, summed in index order over its `latent` entries.  kMax > 0:
// a constant trip count, which the compiler unrolls, so z may be a register array of kMax entries; kMax == 0: a loop over any latent.
// (An explicit #pragma unroll would stop the compiler's own partial unrolling of the kMax == 0 loop, and ppo_loss_kernel then spills.)
template <int kMax>
__device__ __forceinline__ float ppo_reg_norm(const float* z, const float* zh, int latent) {
  float nrm = 0.0f;
  for (int i = 0; i < (kMax > 0 ? kMax : latent); ++i)
    if (i < latent) { const float d = z[i] - zh[i]; nrm += d * d; }
  return sqrtf(nrm);
}
// d (c_reg mean_rows ||z - zh||) / dz = ppo_reg_scale * (z - zh), invm = 1 / rows
__device__ __forceinline__ float ppo_reg_scale(float nrm, float c_reg, float invm) { return nrm > 0.0f ? c_reg * invm / nrm : 0.0f; }

}  // namespace dwbc
