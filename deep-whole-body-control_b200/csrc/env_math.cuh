// Scalar helpers shared by the post-physics kernels (restated isaacgym.torch_utils math, see
// oracle/torch_utils.py for the definitions and their provenance).
#pragma once
#include <math.h>

#include "common.cuh"

namespace dwbc {

// Out-of-line single copies of the transcendental functions: every call site runs once per env, so the
// kernels are instruction-fetch bound unless the code stays small (29 k SASS instructions when inlined).
static __device__ __noinline__ float nsin(float x) { return sinf(x); }
static __device__ __noinline__ float ncos(float x) { return cosf(x); }
static __device__ __noinline__ float natan2(float y, float x) { return atan2f(y, x); }
static __device__ __noinline__ float nasin(float x) { return asinf(x); }
static __device__ __noinline__ float nexp(float x) { return expf(x); }
static __device__ __noinline__ float nfmod(float x, float y) { return fmodf(x, y); }
static __device__ __noinline__ float ndiv(float x, float y) { return x / y; }
static __device__ __noinline__ float nsqrt(float x) { return sqrtf(x); }

struct V3 { float x, y, z; };
__device__ __forceinline__ V3 mk(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ V3 cross(V3 a, V3 b) { return mk(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }

// isaacgym.torch_utils.quat_rotate_inverse (restated, oracle/torch_utils.py); q = xyzw
static __device__ __noinline__ V3 quat_rotate_inverse(const float* q, V3 v) {
  V3 qv = mk(q[0], q[1], q[2]);
  float qw = q[3];
  float s = 2.0f * (qw * qw) - 1.0f;
  V3 c = cross(qv, v);
  float d = ((qv.x * v.x + qv.y * v.y) + qv.z * v.z);
  return mk((v.x * s - c.x * qw * 2.0f) + qv.x * d * 2.0f, (v.y * s - c.y * qw * 2.0f) + qv.y * d * 2.0f,
            (v.z * s - c.z * qw * 2.0f) + qv.z * d * 2.0f);
}
static __device__ __noinline__ V3 quat_apply(const float* q, V3 v) {
  V3 qv = mk(q[0], q[1], q[2]);
  V3 t = cross(qv, v);
  t = mk(t.x * 2.0f, t.y * 2.0f, t.z * 2.0f);
  V3 c = cross(qv, t);
  return mk((v.x + q[3] * t.x) + c.x, (v.y + q[3] * t.y) + c.y, (v.z + q[3] * t.z) + c.z);
}
static __device__ __noinline__ void euler_from_quat(const float* q, float& roll, float& pitch, float& yaw) {
  float x = q[0], y = q[1], z = q[2], w = q[3];
  roll = natan2(2.0f * (w * x + y * z), 1.0f - 2.0f * (x * x + y * y));
  pitch = nasin(fminf(fmaxf(2.0f * (w * y - z * x), -1.0f), 1.0f));
  yaw = natan2(2.0f * (w * z + x * y), 1.0f - 2.0f * (y * y + z * z));
}
static __device__ __noinline__ V3 sphere2cart(V3 s) {
  float proj = s.x * ncos(s.y);
  return mk(proj * ncos(s.z), proj * nsin(s.z), s.x * nsin(s.y));
}
static __device__ __noinline__ V3 cart2sphere(V3 c) {
  float l = nsqrt((c.x * c.x + c.y * c.y) + c.z * c.z);
  return mk(l, nasin(ndiv(c.z, l)), natan2(c.y, c.x));
}
// torch.remainder(a + pi, 2 pi) - pi  (fmod-based, like ATen)
static __device__ __noinline__ float wrap_pi(float a) {
  const float PI = 3.14159265358979323846f, TWO_PI = 6.28318530717958647692f;
  float r = nfmod(a + PI, TWO_PI);
  if (r != 0.0f && r < 0.0f) r += TWO_PI;
  return r - PI;
}
// torch.lerp
__device__ __forceinline__ float lerpf(float a, float b, float w) {
  float d = b - a;
  return (w < 0.5f) ? a + w * d : b - d * (1.0f - w);
}
__device__ __forceinline__ V3 lerp3(V3 a, V3 b, float w) { return mk(lerpf(a.x, b.x, w), lerpf(a.y, b.y, w), lerpf(a.z, b.z, w)); }
__device__ __forceinline__ float clipf(float v, float lo, float hi) { return fminf(fmaxf(v, lo), hi); }
__device__ __forceinline__ float4 clip4(float4 v, float c) {
  return make_float4(clipf(v.x, -c, c), clipf(v.y, -c, c), clipf(v.z, -c, c), clipf(v.w, -c, c));
}

}  // namespace dwbc
