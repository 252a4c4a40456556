// pfb_common.cuh — shared device helpers for the batched UAV stepper (sm_90a).
//
// Everything here is `PFB_HD` so that tests/hostsim can compile the SAME per-env body with g++ for
// precision studies on a machine without a GPU.  The host build is a test harness only; the product
// library (libpyflyt_b200.so) contains the CUDA kernels and nothing else.
#pragma once

#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define PFB_HD __host__ __device__ __forceinline__
#define PFB_D __device__ __forceinline__
#else
#define PFB_HD inline
#define PFB_D inline
#endif

namespace pfb {

// -------------------------------------------------------------------------------------------------
// Precision policy (see DESIGN.md §precision).  The reference integrates in fp64 end to end; plain
// fp32 misses the 1e-3 m / 1000-step trajectory tolerance by ~10x (SURVEY §7) because attitude
// rounding tilts the thrust vector and is integrated twice.  The attitude quaternion, the position
// and (optionally) the world velocity are therefore carried as fp64 in registers and stored as two
// fp32 words (hi, lo) so the HBM layout stays fp32 SoA.  Everything else — forces, control, aero,
// observations, rewards — is fp32.  The H100 issues non-tensor fp64 at half the fp32 rate.
// -------------------------------------------------------------------------------------------------
#ifndef PFB_Q_DOUBLE
#define PFB_Q_DOUBLE 1
#endif
#ifndef PFB_X_DOUBLE
#define PFB_X_DOUBLE 1
#endif
#ifndef PFB_V_DOUBLE
#define PFB_V_DOUBLE 1
#endif
// Rotation matrix entries: fp64 for the QuadX and rocket bodies (PFB_R_DOUBLE), whose attitude cascades and thrust vectors
// turn fp32 entries into position error that the H100 build carried past the 1e-3 m bar in height-hold modes; fp32 for the
// fixed-wing and dogfight bodies (PFB_FW_R_DOUBLE), whose error floor is the fp32 aerodynamic model (DESIGN.md §5).
#ifndef PFB_R_DOUBLE
#define PFB_R_DOUBLE 1
#endif
#ifndef PFB_FW_R_DOUBLE
#define PFB_FW_R_DOUBLE 0
#endif

#if PFB_Q_DOUBLE
typedef double qreal;
#else
typedef float qreal;
#endif
#if PFB_X_DOUBLE
typedef double xreal;
#else
typedef float xreal;
#endif
#if PFB_V_DOUBLE
typedef double vreal;
#else
typedef float vreal;
#endif

struct Vec3 {
  float x, y, z;
};

PFB_HD Vec3 v3(float x, float y, float z) { return Vec3{x, y, z}; }
PFB_HD Vec3 operator+(Vec3 a, Vec3 b) { return Vec3{a.x + b.x, a.y + b.y, a.z + b.z}; }
PFB_HD Vec3 operator-(Vec3 a, Vec3 b) { return Vec3{a.x - b.x, a.y - b.y, a.z - b.z}; }
PFB_HD Vec3 operator*(float s, Vec3 a) { return Vec3{s * a.x, s * a.y, s * a.z}; }
PFB_HD Vec3 cross(Vec3 a, Vec3 b) {
  return Vec3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
PFB_HD float dot(Vec3 a, Vec3 b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, a.z * b.z)); }

// Row-major body→world rotation.
struct Mat3 {
  float m00, m01, m02, m10, m11, m12, m20, m21, m22;
};
PFB_HD Vec3 mul(const Mat3& R, Vec3 v) {
  return Vec3{fmaf(R.m00, v.x, fmaf(R.m01, v.y, R.m02 * v.z)), fmaf(R.m10, v.x, fmaf(R.m11, v.y, R.m12 * v.z)),
              fmaf(R.m20, v.x, fmaf(R.m21, v.y, R.m22 * v.z))};
}
PFB_HD Vec3 mulT(const Mat3& R, Vec3 v) {
  return Vec3{fmaf(R.m00, v.x, fmaf(R.m10, v.y, R.m20 * v.z)), fmaf(R.m01, v.x, fmaf(R.m11, v.y, R.m21 * v.z)),
              fmaf(R.m02, v.x, fmaf(R.m12, v.y, R.m22 * v.z))};
}

PFB_HD float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
// Single-instruction SFU forms (MUFU.RCP / MUFU.RSQ, flush-to-zero, ~1-2 ulp) without the IEEE
// denormal/overflow fix-up paths: every use below feeds a clipped control value, a reward distance or
// a contact margin, never the integrated trajectory state.
PFB_HD float fast_rcp(float b) {
#if defined(__CUDA_ARCH__)
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(b));
  return r;
#else
  return 1.0f / b;
#endif
}
PFB_HD float fast_div(float a, float b) { return a * fast_rcp(b); }
PFB_HD float fast_rsqrt(float x) {
#if defined(__CUDA_ARCH__)
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
#else
  return 1.0f / sqrtf(x);
#endif
}
PFB_HD float fast_sqrt(float x) {
#if defined(__CUDA_ARCH__)
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
#else
  return sqrtf(x);
#endif
}
// -sign(v) * k * v^2  ==  -k * v * |v|   (boring_bodies.py:115-119, quadx.py:502-506)
PFB_HD float signed_square(float v) { return v * fabsf(v); }

// -------------------------------------------------------------------------------------------------
// Analytic wind field (include/pyflyt_b200.h, PfbWind): wind = base * f(z), evaluated per drag body / lifting surface at
// the link COM like Aviary.wind_field in boring_bodies.py:93-96 and lifting_surfaces.py:88-93.  A member of every vehicle's
// parameter block; kind 0 (still air) costs one uniform branch.
// -------------------------------------------------------------------------------------------------
struct WindParams {
  int kind;  // PFB_WIND_*
  float bx, by, bz;
  float inv_zref, alpha, z0, inv_z0, inv_log;  // inv_log = 1 / ln(z_ref / z0)
};
PFB_HD float wind_profile(const WindParams& w, float z) {
#if defined(__CUDA_ARCH__)
  if (w.kind == 1) return 1.0f;
  if (w.kind == 2) return exp2f(w.alpha * __log2f(fmaxf(z, 0.0f) * w.inv_zref));  // 0 ^ alpha = exp2(-inf) = 0
  if (w.kind == 3) return __logf(fmaxf(z, w.z0) * w.inv_z0) * w.inv_log;
  return __expf(z * w.inv_zref);
#else
  if (w.kind == 1) return 1.0f;
  if (w.kind == 2) return powf(fmaxf(z, 0.0f) * w.inv_zref, w.alpha);
  if (w.kind == 3) return logf(fmaxf(z, w.z0) * w.inv_z0) * w.inv_log;
  return expf(z * w.inv_zref);
#endif
}
// per-substep context: the base wind rotated into the body frame (R^T base) and what is needed for a link's altitude
struct WindCtx {
  Vec3 wb;
  float pz, r20, r21, r22;
};
PFB_HD WindCtx wind_ctx(const WindParams& w, float pz, float m00, float m01, float m02, float m10, float m11, float m12, float m20, float m21,
                        float m22) {
  WindCtx c;
  c.wb = Vec3{m00 * w.bx + m10 * w.by + m20 * w.bz, m01 * w.bx + m11 * w.by + m21 * w.bz, m02 * w.bx + m12 * w.by + m22 * w.bz};
  c.pz = pz; c.r20 = m20; c.r21 = m21; c.r22 = m22;
  return c;
}
// body-frame wind at the link COM r (base frame)
PFB_HD Vec3 wind_body_at(const WindParams& w, const WindCtx& c, float rx, float ry, float rz) {
  const float z = c.pz + c.r20 * rx + c.r21 * ry + c.r22 * rz;
  return wind_profile(w, z) * c.wb;
}

// hi/lo split of an fp64 value into two fp32 words and back
PFB_HD void split_hi_lo(double d, float& hi, float& lo) {
  hi = (float)d;
  lo = (float)(d - (double)hi);
}
PFB_HD double join_hi_lo(float hi, float lo) { return (double)hi + (double)lo; }

// -------------------------------------------------------------------------------------------------
// Philox4x32-10 counter RNG: stateless, keyed by (seed), counter = (env, draw index) — results do
// not depend on how envs are split over GPUs.
// -------------------------------------------------------------------------------------------------
struct U4 {
  uint32_t x, y, z, w;
};

PFB_HD uint32_t mulhi32(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
  return __umulhi(a, b);
#else
  return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32);
#endif
}

PFB_HD U4 philox4x32_10(U4 ctr, uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = mulhi32(M0, ctr.x), lo0 = M0 * ctr.x;
    uint32_t hi1 = mulhi32(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = U4{hi1 ^ ctr.y ^ k0, lo1, hi0 ^ ctr.w ^ k1, lo0};
    k0 += W0;
    k1 += W1;
  }
  return ctr;
}

PFB_HD float u32_to_unit_open(uint32_t u) {
  // (0, 1]: never returns 0 so log() is safe
  return ((float)(u >> 8) + 1.0f) * (1.0f / 16777216.0f);
}

// stream tags of the Philox counters (top byte of the last counter word)
enum { TAG_AVIARY = 0, TAG_ENV_STEP = 1, TAG_RESET = 2, TAG_ACTION = 3 };

// two standard normals from two uniforms (Box–Muller); noise only, so fast intrinsics are fine
PFB_HD void box_muller(uint32_t a, uint32_t b, float& n0, float& n1) {
  float u1 = u32_to_unit_open(a);
  float u2 = u32_to_unit_open(b);
#if defined(__CUDA_ARCH__)
  float r = fast_sqrt(-2.0f * __logf(u1));
  float s, c;
  __sincosf(6.28318530717958647692f * u2, &s, &c);
#else
  float r = sqrtf(-2.0f * logf(u1));
  float s = sinf(6.28318530717958647692f * u2), c = cosf(6.28318530717958647692f * u2);
#endif
  n0 = r * c;
  n1 = r * s;
}

}  // namespace pfb
