// RolloutStorage.compute_returns (RS:136-150) as one cooperative kernel (K3 + K4 of SURVEY.md):
// two-channel GAE backward scan, thread per (env, channel) serial over T, then the joint
// advantage normalisation (global mean / UNBIASED std over all T*N*2 elements) after a grid
// barrier.  HBM/L2-bound and tiny: 49 B per (t, env) -> 8 MB at T=40, N=4096.
//
// Also PPO.process_env_step's reward path (PPO:130-134).
#include <cooperative_groups.h>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace dwbc {

constexpr int GAE_BLOCK = 64;

// stats layout (DWBC_GAE_STATS doubles): [0..2] = (n, sum, sum of squares), [3] = counter, [4 + 2 b, 4 + 2 b + 1] = partials of block b
constexpr int GAE_PART = 4;

// this block's (sum, sum of squares) -> its own slot
__device__ __forceinline__ void block_partial(double s, double ss, double* stats) {
  __shared__ double red[2][GAE_BLOCK / 32];
  s = warp_sum(s);
  ss = warp_sum(ss);
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) { red[0][w] = s; red[1][w] = ss; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, b = 0;
    for (int i = 0; i < GAE_BLOCK / 32; ++i) { a += red[0][i]; b += red[1][i]; }
    stats[GAE_PART + 2 * blockIdx.x] = a;
    stats[GAE_PART + 2 * blockIdx.x + 1] = b;
  }
}
// The partials of all blocks added up in block order (thread t: blocks t, t + 64, ...; then a fixed tree), the same in every block
__device__ __forceinline__ double2 sum_partials(const double* stats) {
  __shared__ double red[2][GAE_BLOCK];
  double a = 0.0, b = 0.0;
  for (int i = threadIdx.x; i < (int)gridDim.x; i += GAE_BLOCK) {
    a += __ldcg(stats + GAE_PART + 2 * i);
    b += __ldcg(stats + GAE_PART + 2 * i + 1);
  }
  red[0][threadIdx.x] = a;
  red[1][threadIdx.x] = b;
  __syncthreads();
#pragma unroll
  for (int w = GAE_BLOCK / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) { red[0][threadIdx.x] += red[0][threadIdx.x + w]; red[1][threadIdx.x] += red[1][threadIdx.x + w]; }
    __syncthreads();
  }
  return make_double2(red[0][0], red[1][0]);
}

template <bool kFused>
__global__ void __launch_bounds__(GAE_BLOCK)
gae_kernel(const float* __restrict__ rewards, const float* __restrict__ values, const uint8_t* __restrict__ dones,
           const float* __restrict__ last_values, float* __restrict__ returns, float* __restrict__ advantages,
           double* stats, int T, int N, float gamma, float lam) {
  const int C = 2 * N;
  double s = 0.0, ss = 0.0;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < C; j += gridDim.x * blockDim.x) {
    const int env = j >> 1;
    float nxt = last_values[j];
    float adv = 0.0f;
#pragma unroll 8
    for (int t = T - 1; t >= 0; --t) {
      const float r = __ldg(rewards + (size_t)t * C + j);
      const float v = __ldg(values + (size_t)t * C + j);
      const float m = 1.0f - (float)__ldg(dones + (size_t)t * N + env);
      const float delta = r + m * gamma * nxt - v;   // RS:143
      adv = delta + m * gamma * lam * adv;           // RS:144
      const float ret = adv + v;                     // RS:145
      returns[(size_t)t * C + j] = ret;
      const float a = ret - v;                       // RS:148 (returns - values, not `adv` itself)
      advantages[(size_t)t * C + j] = a;
      s += (double)a;
      ss += (double)a * (double)a;
      nxt = v;
    }
  }
  block_partial(s, ss, stats);
  const double n = (double)T * (double)C;
  if constexpr (kFused) {
    __threadfence();
    cg::this_grid().sync();
    const double2 tot = sum_partials(stats);
    if (threadIdx.x == 0 && blockIdx.x == 0) { stats[0] += n; stats[1] += tot.x; stats[2] += tot.y; }
    const double mean = tot.x / n;
    const double var = fmax((tot.y - tot.x * tot.x / n) / (n - 1.0), 0.0);
    const float fm = (float)mean, fd = (float)sqrt(var) + 1e-8f;  // RS:150
    const size_t total = (size_t)T * C;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
      advantages[i] = (__ldcg(advantages + i) - fm) / fd;
  } else {
    if (!last_block(reinterpret_cast<unsigned*>(stats + 3))) return;
    const double2 tot = sum_partials(stats);
    if (threadIdx.x == 0) { stats[0] += n; stats[1] += tot.x; stats[2] += tot.y; }
  }
}

__global__ void normalize_kernel(float* __restrict__ adv, const double* __restrict__ stats, size_t total) {
  const double n = stats[0], sum = stats[1], sq = stats[2];
  const double mean = sum / n;
  const double var = fmax((sq - sum * sum / n) / (n - 1.0), 0.0);
  const float fm = (float)mean, fd = (float)sqrt(var) + 1e-8f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
    adv[i] = (adv[i] - fm) / fd;
}

__global__ void store_rewards_kernel(const float* __restrict__ rew, const float* __restrict__ arm_rew,
                                     const float* __restrict__ values, const uint8_t* __restrict__ time_outs,
                                     const uint8_t* __restrict__ resets, float gamma, float* __restrict__ out,
                                     uint8_t* __restrict__ dones, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float to = time_outs ? (float)time_outs[i] : 0.0f;
  out[2 * i] = rew[i] + gamma * (values[2 * i] * to);          // PPO:133-134
  out[2 * i + 1] = arm_rew[i] + gamma * (values[2 * i + 1] * to);
  if (dones) dones[i] = resets[i] ? 1 : 0;
}

// Explained variance: per channel c the block's sums of R, R^2, R - V and (R - V)^2 (each shifted by row 0's value) in double -> slot 8 b + 4 c + k of scratch (after the
// counter); the last block adds the slots up in block order.
constexpr int EV_BLOCK = 256;
__global__ void __launch_bounds__(EV_BLOCK)
explained_variance_kernel(const float* __restrict__ values, const float* __restrict__ returns, int64_t rows, double* scratch, float* out) {
  __shared__ double red[8][EV_BLOCK / 32];
  // shifted by row 0's R and R - V: no cancellation against a large mean, and exactly 0 for a constant channel
  const double k[4] = {returns[0], returns[0] - (double)values[0], returns[1], returns[1] - (double)values[1]};
  double v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int64_t j = (int64_t)blockIdx.x * EV_BLOCK + threadIdx.x; j < rows; j += (int64_t)gridDim.x * EV_BLOCK) {
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const double R = __ldg(returns + 2 * j + c), r = R - k[2 * c], e = (R - (double)__ldg(values + 2 * j + c)) - k[2 * c + 1];
      v[4 * c] += r; v[4 * c + 1] += r * r; v[4 * c + 2] += e; v[4 * c + 3] += e * e;
    }
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const double s = warp_sum(v[k]);
    if (lane == 0) red[k][w] = s;
  }
  __syncthreads();
  double* part = scratch + 2;
  if (threadIdx.x < 8) {
    double s = 0.0;
    for (int i = 0; i < EV_BLOCK / 32; ++i) s += red[threadIdx.x][i];
    part[8 * blockIdx.x + threadIdx.x] = s;
  }
  if (!last_block(reinterpret_cast<unsigned*>(scratch)) || threadIdx.x >= 2) return;
  const int c = threadIdx.x;
  double t[4] = {0, 0, 0, 0};
  for (int b = 0; b < (int)gridDim.x; ++b)
    for (int k = 0; k < 4; ++k) t[k] += __ldcg(part + 8 * b + 4 * c + k);
  const double n = (double)rows;
  const double var_r = fmax(t[1] / n - (t[0] / n) * (t[0] / n), 0.0), var_e = fmax(t[3] / n - (t[2] / n) * (t[2] / n), 0.0);
  out[c] = var_r > 0.0 ? (float)(1.0 - var_e / var_r) : __int_as_float(0x7fc00000);
}

}  // namespace dwbc

using namespace dwbc;

extern "C" int dwbc_explained_variance(const float* values, const float* returns, int64_t rows, double* scratch, float* out,
                                       dwbc_stream_t stream) {
  if (!values || !returns || !scratch || !out || rows <= 0) return DWBC_ERR_ARG;
  const int64_t blocks = (rows + EV_BLOCK - 1) / EV_BLOCK;
  const int grid = blocks < DWBC_EV_MAX_BLOCKS ? (int)blocks : DWBC_EV_MAX_BLOCKS;   // grid-stride loops cover the rest
  explained_variance_kernel<<<grid, EV_BLOCK, 0, (cudaStream_t)stream>>>(values, returns, rows, scratch, out);
  DWBC_LAUNCH_CHECK();
  return DWBC_OK;
}

extern "C" int dwbc_gae(const float* rewards, const float* values, const uint8_t* dones, const float* last_values,
                        float* returns, float* advantages, double* stats, int32_t T, int32_t N, float gamma, float lam,
                        int32_t normalize, dwbc_stream_t stream) {
  if (!rewards || !values || !dones || !last_values || !returns || !advantages || !stats || T <= 0 || N <= 0) return DWBC_ERR_ARG;
  const int C = 2 * N;
  int grid = (C + GAE_BLOCK - 1) / GAE_BLOCK;
  if (grid > DWBC_GAE_MAX_BLOCKS) grid = DWBC_GAE_MAX_BLOCKS;   // one partial slot per block; grid-stride loops cover the rest
  cudaStream_t st = (cudaStream_t)stream;
  if (normalize && (size_t)T * C > 1) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gae_kernel<true>, GAE_BLOCK, 0);
    const int max_coop = sms * per_sm;
    if (max_coop > 0) {
      if (grid > max_coop) grid = max_coop;  // grid-stride loops cover the rest
      void* args[] = {(void*)&rewards, (void*)&values, (void*)&dones, (void*)&last_values, (void*)&returns,
                      (void*)&advantages, (void*)&stats, (void*)&T, (void*)&N, (void*)&gamma, (void*)&lam};
      cudaError_t e = cudaLaunchCooperativeKernel((const void*)gae_kernel<true>, dim3(grid), dim3(GAE_BLOCK), args, 0, st);
      if (e == cudaSuccess) return DWBC_OK;
      (void)cudaGetLastError();  // fall through to the two-kernel path
    }
    gae_kernel<false><<<grid, GAE_BLOCK, 0, st>>>(rewards, values, dones, last_values, returns, advantages, stats, T, N, gamma, lam);
    DWBC_LAUNCH_CHECK();
    return dwbc_normalize_advantages(advantages, stats, (int64_t)T * C, stream);
  }
  gae_kernel<false><<<grid, GAE_BLOCK, 0, st>>>(rewards, values, dones, last_values, returns, advantages, stats, T, N, gamma, lam);
  DWBC_LAUNCH_CHECK();
  return DWBC_OK;
}

extern "C" int dwbc_normalize_advantages(float* advantages, const double* stats, int64_t count, dwbc_stream_t stream) {
  if (!advantages || !stats || count <= 0) return DWBC_ERR_ARG;
  int grid = (int)((count + 1023) / 1024);
  if (grid > 1184) grid = 1184;
  normalize_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(advantages, stats, (size_t)count);
  DWBC_LAUNCH_CHECK();
  return DWBC_OK;
}

extern "C" int dwbc_store_rewards(const float* rew, const float* arm_rew, const float* values, const uint8_t* time_outs,
                                  const uint8_t* resets, float gamma, float* rewards_out, uint8_t* dones_out,
                                  int32_t num_envs, dwbc_stream_t stream) {
  if (!rew || !arm_rew || !values || !rewards_out || num_envs <= 0 || (dones_out && !resets)) return DWBC_ERR_ARG;
  store_rewards_kernel<<<(num_envs + 255) / 256, 256, 0, (cudaStream_t)stream>>>(rew, arm_rew, values, time_outs, resets, gamma,
                                                                                  rewards_out, dones_out, num_envs);
  DWBC_LAUNCH_CHECK();
  return DWBC_OK;
}
