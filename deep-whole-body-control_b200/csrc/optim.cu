// clip_grad_norm_ + torch.optim.Adam step (PPO:245-246) on the flat parameter buffer (K9), and
// PPO.enforce_min_std (PPO:293-296).  HBM-bound: 7 floats per parameter (28 B) -> 4.7 MB.
#include <math.h>

#include "common.cuh"

namespace dwbc {

// Per-block partial sums of squares: block b writes out[b].  clip_adam_kernel adds them up in block order, so the norm does not depend on
// which block finished first.
__global__ void __launch_bounds__(256) sumsq_kernel(const float* __restrict__ g, int64_t n, float scale, double* __restrict__ out) {
  __shared__ double red[8];
  double s = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = g[i] * scale;
    s += (double)v * (double)v;
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += red[i];
    out[blockIdx.x] = t;
  }
}

struct AdamArgs {
  float* p; float* g; float* m; float* v;
  int64_t n;
  float scale, max_norm, beta1, beta2, eps, step_size, bc2_sqrt;
  const double* sumsq;                   // [nparts] partials of sumsq_kernel
  int nparts;
  float* norm_out;
  const float* bias_row;                 // optional device (step_size, bc2_sqrt) in place of the two fields (dwbc_clip_adam_step_table)
};

// Every block sums the partials itself, in the same fixed order (thread t: partials t, t + 256, ...; then a fixed tree)
__device__ __forceinline__ double sum_partials(const double* __restrict__ part, int n) {
  __shared__ double red[256];
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) s += part[i];
  red[threadIdx.x] = s;
  __syncthreads();
#pragma unroll
  for (int w = 128; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  return red[0];
}

__global__ void __launch_bounds__(256) clip_adam_kernel(const AdamArgs a) {
  const float total = (float)sqrt(sum_partials(a.sumsq, a.nparts));  // clip_grad_norm_: ||g||_2 over all tensors
  const float coef = fminf(a.max_norm / (total + 1e-6f), 1.0f);
  const float step_size = a.bias_row ? a.bias_row[0] : a.step_size, bc2_sqrt = a.bias_row ? a.bias_row[1] : a.bc2_sqrt;
  if (a.norm_out && blockIdx.x == 0 && threadIdx.x == 0) *a.norm_out = total;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
    const float g = (a.g[i] * a.scale) * coef;
    const float m = a.m[i] * a.beta1 + g * (1.0f - a.beta1);
    const float v = a.v[i] * a.beta2 + (g * g) * (1.0f - a.beta2);
    const float denom = sqrtf(v) / bc2_sqrt + a.eps;
    a.g[i] = g;  // leave the clipped gradient behind (what .grad holds after PPO:245)
    a.m[i] = m;
    a.v[i] = v;
    a.p[i] = a.p[i] - step_size * (m / denom);
  }
}

__global__ void min_std_kernel(float* __restrict__ std, const float* __restrict__ min_std, int n) {
  int i = threadIdx.x;
  if (i < n) std[i] = fmaxf(std[i], min_std[i]);
}

}  // namespace dwbc

using namespace dwbc;

// Adam's bias correction of 1-based step `step` as the host computes it: (lr / (1 - beta1^step), sqrt(1 - beta2^step)), double, then float
static void adam_bias_row(const DwbcPpoHyper* hp, int32_t step, float* row) {
  const double bc1 = 1.0 - pow((double)hp->beta1, (double)step), bc2 = 1.0 - pow((double)hp->beta2, (double)step);
  row[0] = (float)((double)hp->lr / bc1);
  row[1] = (float)sqrt(bc2);
}

extern "C" int dwbc_adam_bias_correction(const DwbcPpoHyper* hp, int32_t first_step, int32_t n, float* out) {
  if (!hp || !out || first_step < 1 || n < 0) return DWBC_ERR_ARG;
  for (int32_t i = 0; i < n; ++i) adam_bias_row(hp, first_step + i, out + 2 * i);
  return DWBC_OK;
}

// adam_table: optional device rows (lr / bc1, sqrt(bc2)), row step - 1 read by the kernel in place of the host computation
static int clip_adam_step(float* params, float* grad, float* adam_m, float* adam_v, int64_t first, int64_t count, const DwbcPpoHyper* hp,
                          int32_t step, const float* adam_table, double* norm_scratch, float* grad_norm_out, dwbc_stream_t stream) {
  if (!params || !grad || !adam_m || !adam_v || !hp || !norm_scratch || count <= 0 || first < 0 || step < 1) return DWBC_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const float scale = hp->grad_scale == 0.0f ? 1.0f : hp->grad_scale;
  int grid = (int)((count + 1023) / 1024);
  if (grid > DWBC_NORM_SCRATCH) grid = DWBC_NORM_SCRATCH;
  if (grid < 1) grid = 1;
  sumsq_kernel<<<grid, 256, 0, st>>>(grad + first, count, scale, norm_scratch);
  DWBC_LAUNCH_CHECK();
  float row[2] = {0.0f, 0.0f};
  if (!adam_table) adam_bias_row(hp, step, row);
  AdamArgs a{params + first, grad + first, adam_m + first, adam_v + first, count, scale, hp->max_grad_norm, hp->beta1, hp->beta2,
             hp->adam_eps, row[0], row[1], norm_scratch, grid, grad_norm_out, adam_table ? adam_table + 2 * (int64_t)(step - 1) : nullptr};
  clip_adam_kernel<<<grid, 256, 0, st>>>(a);
  DWBC_LAUNCH_CHECK();
  return DWBC_OK;
}

extern "C" int dwbc_clip_adam_step(float* params, float* grad, float* adam_m, float* adam_v, int64_t first, int64_t count,
                                   const DwbcPpoHyper* hp, int32_t step, double* norm_scratch, float* grad_norm_out,
                                   dwbc_stream_t stream) {
  return clip_adam_step(params, grad, adam_m, adam_v, first, count, hp, step, nullptr, norm_scratch, grad_norm_out, stream);
}

extern "C" int dwbc_clip_adam_step_table(float* params, float* grad, float* adam_m, float* adam_v, int64_t first, int64_t count,
                                         const DwbcPpoHyper* hp, int32_t step, const float* adam_table, double* norm_scratch,
                                         float* grad_norm_out, dwbc_stream_t stream) {
  if (!adam_table) return DWBC_ERR_ARG;
  return clip_adam_step(params, grad, adam_m, adam_v, first, count, hp, step, adam_table, norm_scratch, grad_norm_out, stream);
}

extern "C" int dwbc_enforce_min_std(float* params, int64_t off_std, const float* min_std, int32_t n, dwbc_stream_t stream) {
  if (!params || !min_std || n <= 0 || n > 1024) return DWBC_ERR_ARG;
  min_std_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(params + off_std, min_std, n);
  DWBC_LAUNCH_CHECK();
  return DWBC_OK;
}

unsigned long long dwbc_launch_counter = 0;
extern "C" uint64_t dwbc_launch_count(void) { return dwbc_launch_counter; }

extern "C" const char* dwbc_version(void) { return "dwbc-b200 0.1 (sm_90a, abi 5)"; }

extern "C" int64_t dwbc_step_device_size(void) { return sizeof(DwbcStepDevice); }

extern "C" void dwbc_struct_sizes(int64_t out[6]) {
  out[0] = sizeof(DwbcEnvCfg); out[1] = sizeof(DwbcEnvBuffers); out[2] = sizeof(DwbcStepArgs);
  out[3] = sizeof(DwbcNetCfg); out[4] = sizeof(DwbcPpoHyper); out[5] = sizeof(DwbcStorage);
}
