// Per-step episode bookkeeping of OnPolicyRunner.learn (OPR:140-154) on the device: running returns and lengths per env, and a ring of
// the last C finished episodes in (step, env ascending) order -- rsl_rl's rewbuffer / lenbuffer deques (maxlen C), plus the arm channel.
//
// One CTA of 32 warps.  Warp w owns the contiguous env range [w S, (w + 1) S) (S a multiple of 32), so the rank of a done env among the
// step's dones is a prefix over warps (one shared-memory scan) plus a ballot within the warp: the order is fixed and no atomic is used.
// Phase 1 counts each warp's dones; phase 2 adds the rewards, appends the finished episodes that are among the step's last C dones
// and clears their running sums.  The adds are the plain fp32 adds of the reference, so the results are bitwise those of torch.
#include "common.cuh"

namespace dwbc {

constexpr int EP_WARPS = 32;
constexpr int EP_THREADS = EP_WARPS * 32;
constexpr int EP_BATCH = 4;           // warp steps of 32 envs whose loads are issued together

__global__ void __launch_bounds__(EP_THREADS)
track_episodes_kernel(const float* __restrict__ rew, const float* __restrict__ arm_rew, const uint8_t* __restrict__ dones, int n,
                      float* __restrict__ running, float* __restrict__ ring, int64_t* __restrict__ pos, int cap) {
  __shared__ int warp_first[EP_WARPS + 1];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int span = (n + EP_THREADS - 1) / EP_THREADS * 32;
  const int lo = min(w * span, n), hi = min(lo + span, n);

  int cnt = 0;
#pragma unroll 8
  for (int i = lo + lane; i < hi; i += 32) cnt += dones[i] != 0;
  cnt = __reduce_add_sync(FULL, cnt);
  if (lane == 0) warp_first[w] = cnt;
  __syncthreads();
  if (w == 0) {                       // exclusive scan of the 32 warp counts, in warp order
    const int c = warp_first[lane];
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(FULL, incl, o);
      if (lane >= o) incl += v;
    }
    __syncwarp();
    warp_first[lane] = incl - c;
    if (lane == 31) warp_first[EP_WARPS] = incl;
  }
  __syncthreads();
  const int total = warp_first[EP_WARPS];
  const int first_kept = total > cap ? total - cap : 0;      // earlier dones of this step fall out of the ring within the step
  const int64_t next = pos[0];
  int rank = warp_first[w];
  const unsigned below = (1u << lane) - 1u;

  for (int s = lo; s < hi; s += 32 * EP_BATCH) {
    float r[EP_BATCH], a[EP_BATCH], run[EP_BATCH][3];
    bool d[EP_BATCH];
#pragma unroll
    for (int b = 0; b < EP_BATCH; ++b) {
      const int i = s + b * 32 + lane;
      const bool ok = i < hi;
      r[b] = ok ? rew[i] : 0.f;
      a[b] = ok ? arm_rew[i] : 0.f;
      d[b] = ok && dones[i] != 0;
#pragma unroll
      for (int c = 0; c < 3; ++c) run[b][c] = ok ? running[3 * (size_t)i + c] : 0.f;
    }
#pragma unroll
    for (int b = 0; b < EP_BATCH; ++b) {
      const int i = s + b * 32 + lane;
      float v[3] = {run[b][0] + r[b], run[b][1] + a[b], run[b][2] + 1.0f};   // OPR:147-148
      const unsigned ball = __ballot_sync(FULL, d[b]);
      if (d[b]) {
        const int k = rank + __popc(ball & below);
        if (k >= first_kept) {
          const int64_t slot = (next + (k - first_kept)) % cap;
#pragma unroll
          for (int c = 0; c < 3; ++c) ring[3 * slot + c] = v[c];
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = 0.f;                            // OPR:152-154
      }
      rank += __popc(ball);
      if (i < hi) {
#pragma unroll
        for (int c = 0; c < 3; ++c) running[3 * (size_t)i + c] = v[c];
      }
    }
  }
  __syncthreads();                    // every thread has read pos[0]
  if (threadIdx.x == 0) {
    pos[0] = (next + min(total, cap)) % cap;
    pos[1] += total;
  }
}

}  // namespace dwbc

using namespace dwbc;

extern "C" int dwbc_track_episodes(const float* rew, const float* arm_rew, const uint8_t* dones, int32_t num_envs, float* running,
                                   float* ring, int64_t* ring_pos, int32_t capacity, dwbc_stream_t stream) {
  if (!rew || !arm_rew || !dones || !running || !ring || !ring_pos || num_envs <= 0 || capacity <= 0) return DWBC_ERR_ARG;
  track_episodes_kernel<<<1, EP_THREADS, 0, (cudaStream_t)stream>>>(rew, arm_rew, dones, num_envs, running, ring, ring_pos, capacity);
  DWBC_LAUNCH_CHECK();
  return DWBC_OK;
}
