// pfb_static.cu — static (fixed-base) bodies of an Aviary handle (DESIGN.md §4h): the reference's
// loadURDF(..., useFixedBase=True) of a landing pad, a helipad or a rooftop, one copy in every drone's world.
//
// The primitive table (pfb::StaticWorld, and pfb::TiltedWorld on solid handles) is host-side here and travels to every step
// launch as a kernel parameter; the poses are field-major device buffers (yaw poses, and full poses on solid handles) that
// only pfb_add_static_body and pfb_set_static_pose write (and pfb_set_static_solid fills, for a handle made solid late).  The
// step kernels themselves live with each vehicle kind (pfb_quadx.cu, pfb_fixedwing.cu, pfb_rocket.cu, pfb_mixed.cu) and run
// when step_statics(h) is set.
#include <cuda_runtime.h>

#include <cmath>

#include "pfb_context.h"

using namespace pfb;

// row b of every drone's world: the pose of body b (x, y, z, cos yaw, sin yaw)
__global__ void __launch_bounds__(kBlock) k_static_fill(float* __restrict__ pose, int body, float x, float y, float z, float c, float s, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  float* q = pose + (int64_t)kStaticPoseRows * body * N + i;
  q[0] = x; q[N] = y; q[2 * N] = z; q[3 * N] = c; q[4 * N] = s;
}

// resetBasePositionAndOrientation of body `body` in the worlds of `mask`: pos / quat place the base inertial frame, at (ox, oy, oz)
// in the link frame.  An upright quaternion (x, y, z, w) ~ (0, 0, qz, qw) is the yaw 2 atan2(qz, qw), whose cosine and sine are
// (w^2 - z^2) / (w^2 + z^2) and 2 w z / (w^2 + z^2); the link frame is at pos - R(yaw) (ox, oy, oz).
__global__ void __launch_bounds__(kBlock) k_static_set_pose(float* __restrict__ pose, int body, const double* __restrict__ pos,
                                                            const double* __restrict__ quat, const uint8_t* __restrict__ mask, double ox,
                                                            double oy, double oz, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  if (mask && !mask[i]) return;
  const double z = quat[4 * i + 2], w = quat[4 * i + 3], d = w * w + z * z;
  const double c = (w * w - z * z) / d, s = 2.0 * w * z / d;
  float* q = pose + (int64_t)kStaticPoseRows * body * N + i;
  q[0] = (float)(pos[3 * i] - (c * ox - s * oy));
  q[N] = (float)(pos[3 * i + 1] - (s * ox + c * oy));
  q[2 * N] = (float)(pos[3 * i + 2] - oz);
  q[3 * N] = (float)c; q[4 * N] = (float)s;
}

// a quaternion (x, y, z, w) whose rotation leaves the z axis vertical: R22 = 1 - 2 (x^2 + y^2) within 1e-9 of 1
static bool upright(const double* q) {
  const double n = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  return n > 0.0 && 2.0 * (q[0] * q[0] + q[1] * q[1]) / n <= 1e-9;
}

// ---- full poses of a solid handle (StaticBodies::d_full, read by TiltedCtx) -------------------------------------------------
// the row-major rotation of quaternion (x, y, z, w), normalised
PFB_HD void quat_rotation(double x, double y, double z, double w, double* r) {
  const double d = 2.0 / (x * x + y * y + z * z + w * w);
  r[0] = 1.0 - d * (y * y + z * z); r[1] = d * (x * y - z * w);       r[2] = d * (x * z + y * w);
  r[3] = d * (x * y + z * w);       r[4] = 1.0 - d * (x * x + z * z); r[5] = d * (y * z - x * w);
  r[6] = d * (x * z - y * w);       r[7] = d * (y * z + x * w);       r[8] = 1.0 - d * (x * x + y * y);
}
struct FullPose { float v[kTiltedPoseRows]; };  // x, y, z, row-major rotation

// rows 12 b .. 12 b + 11 of every drone's world: the pose of body b
__global__ void __launch_bounds__(kBlock) k_static_fill_full(float* __restrict__ full, int body, const __grid_constant__ FullPose p, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  float* q = full + (int64_t)kTiltedPoseRows * body * N + i;
#pragma unroll
  for (int e = 0; e < kTiltedPoseRows; ++e) q[e * N] = p.v[e];
}

// k_static_set_pose's reset with the full rotation R of each quaternion: the link frame is at pos - R (ox, oy, oz)
__global__ void __launch_bounds__(kBlock) k_static_set_full_pose(float* __restrict__ full, int body, const double* __restrict__ pos,
                                                                 const double* __restrict__ quat, const uint8_t* __restrict__ mask, double ox,
                                                                 double oy, double oz, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  if (mask && !mask[i]) return;
  double r[9];
  quat_rotation(quat[4 * i], quat[4 * i + 1], quat[4 * i + 2], quat[4 * i + 3], r);
  float* q = full + (int64_t)kTiltedPoseRows * body * N + i;
  q[0] = (float)(pos[3 * i] - (r[0] * ox + r[1] * oy + r[2] * oz));
  q[N] = (float)(pos[3 * i + 1] - (r[3] * ox + r[4] * oy + r[5] * oz));
  q[2 * N] = (float)(pos[3 * i + 2] - (r[6] * ox + r[7] * oy + r[8] * oz));
#pragma unroll
  for (int e = 0; e < 9; ++e) q[(3 + e) * N] = (float)r[e];
}

// the full poses of bodies 0 .. n_bodies - 1 from their yaw poses (all upright): a handle that becomes solid after its first body
__global__ void __launch_bounds__(kBlock) k_static_full_from_yaw(float* __restrict__ full, const float* __restrict__ pose, int n_bodies, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  for (int b = 0; b < n_bodies; ++b) {
    const float* y = pose + (int64_t)kStaticPoseRows * b * N + i;
    float* q = full + (int64_t)kTiltedPoseRows * b * N + i;
    const float c = y[3 * N], sn = y[4 * N];
    const float v[kTiltedPoseRows] = {y[0], y[N], y[2 * N], c, -sn, 0.0f, sn, c, 0.0f, 0.0f, 0.0f, 1.0f};
#pragma unroll
    for (int e = 0; e < kTiltedPoseRows; ++e) q[e * N] = v[e];
  }
}

// the full-pose buffer of a solid handle with static-body buffers, filled from the yaw poses of the bodies it holds
static int static_alloc_full(PfbContext* h, cudaStream_t st) {
  StaticBodies* b = h->statics;
  if (!b || b->d_full) return 0;
  CUDA_OK(cudaMalloc(&b->d_full, (size_t)kTiltedPoseRows * kMaxStaticBodies * (size_t)h->n * sizeof(float)));
  if (b->n_bodies > 0) {
    k_static_full_from_yaw<<<grid_for(h->n), kBlock, 0, st>>>(b->d_full, b->d_pose, b->n_bodies, h->n);
    LAUNCH_CHECK(h);
  }
  return 0;
}

void static_destroy(PfbContext* h) {
  StaticBodies* b = h->statics;
  if (!b) return;
  if (b->d_pose) cudaFree(b->d_pose);
  if (b->d_bits) cudaFree(b->d_bits);
  if (b->d_full) cudaFree(b->d_full);
  delete b;
  h->statics = nullptr;
}

// the bits are zeroed when the next first body is added
void static_clear(PfbContext* h) {
  if (!h->statics) return;
  h->statics->n_bodies = 0;
  h->statics->world.n_shapes = 0;
  h->statics->tworld.n_shapes = 0;
  h->statics->tilted = false;
}

// Aviary handles only: an env handle keeps its own floor and pad policy
static int require_aviary_statics(PfbHandle h, const char* what) {
  if (!h) return fail("%s: null handle", what);
  if (h->env.env_kind != PFB_ENV_NONE)
    return fail("%s: static bodies are for Aviary handles; an env handle (env kind %d) keeps its own floor and pad", what, h->env.env_kind);
  return 0;
}

extern "C" int pfb_add_static_body(PfbHandle h, const PfbStaticShape* shapes, int n_shapes, const double pos[3], const double quat[4],
                                   const double inertial_origin[3], int* body_id, void* stream) {
  if (require_aviary_statics(h, "pfb_add_static_body")) return -1;
  if (!shapes || !pos || !quat || !body_id) return fail("pfb_add_static_body: null argument");
  if (n_shapes < 1) return fail("pfb_add_static_body: a static body needs at least one collision primitive (box or cylinder), got %d", n_shapes);
  const int have_bodies = h->statics ? h->statics->n_bodies : 0, have_shapes = h->statics ? h->statics->world.n_shapes : 0;
  if (have_bodies >= kMaxStaticBodies) return fail("pfb_add_static_body: at most %d static bodies per handle", kMaxStaticBodies);
  if (have_shapes + n_shapes > kMaxStaticShapes)
    return fail("pfb_add_static_body: at most %d collision primitives over all static bodies of a handle (have %d, adding %d)", kMaxStaticShapes,
                have_shapes, n_shapes);
  // the top-face rule needs upright bodies and primitives; a solid handle takes any orientation (TiltedCtx once one is tilted)
  const bool solid = h->static_solid;
  bool tilted = !upright(quat);
  if (tilted && !solid)
    return fail("pfb_add_static_body: the body must stay upright (only a yaw about the world z axis): tilted static bodies are not modelled "
                "under the top-face rule.  A solid handle (pfb_set_static_solid, solid_static_bodies=True) takes any orientation");
  // each primitive upright in the body frame (a box yawed about its z axis, a cylinder whose axis is z), unless the handle is solid
  for (int k = 0; k < n_shapes; ++k) {
    const PfbStaticShape& s = shapes[k];
    if (s.kind != PFB_SHAPE_BOX && s.kind != PFB_SHAPE_CYLINDER)
      return fail("pfb_add_static_body: primitive %d is a %s; static bodies are boxes and cylinders", k, s.kind == PFB_SHAPE_SPHERE ? "sphere" : "mesh or unknown shape");
    const double* r = s.rot;
    const double tilt = fabs(r[2]) + fabs(r[5]) + fabs(r[6]) + fabs(r[7]) + fabs(r[8] - 1.0);
    if (!(tilt <= 1e-9)) {
      if (!solid)
        return fail("pfb_add_static_body: primitive %d is tilted in its body; only a yaw about the body's z axis is modelled under the top-face "
                    "rule.  A solid handle (pfb_set_static_solid, solid_static_bodies=True) takes any orientation", k);
      tilted = true;
    }
    if (!(s.dims[0] > 0.0 && s.dims[1] > 0.0 && (s.kind == PFB_SHAPE_CYLINDER || s.dims[2] > 0.0)))
      return fail("pfb_add_static_body: primitive %d has a non-positive size", k);
  }
  CUDA_OK(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  if (!h->statics) {  // the handle gets its bodies only once both buffers exist
    float* d_pose = nullptr;
    uint32_t* d_bits = nullptr;
    cudaError_t e = cudaMalloc(&d_pose, (size_t)kStaticPoseRows * kMaxStaticBodies * (size_t)h->n * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&d_bits, (size_t)h->n * sizeof(uint32_t));
    StaticBodies* b = e == cudaSuccess ? new (std::nothrow) StaticBodies() : nullptr;
    if (!b) {
      if (d_pose) cudaFree(d_pose);
      if (d_bits) cudaFree(d_bits);
      return e != cudaSuccess ? fail("allocating the static-body buffers failed: %s", cudaGetErrorString(e)) : fail("out of host memory");
    }
    memset(b, 0, sizeof(*b));
    b->d_pose = d_pose;
    b->d_bits = d_bits;
    h->statics = b;
  }
  StaticBodies* b = h->statics;
  if (solid && static_alloc_full(h, st)) return -1;
  const int body = b->n_bodies;
  // the first body since creation or a full reset: no contact with a static body yet (resetSimulation empties contact_array)
  if (body == 0) CUDA_OK(cudaMemsetAsync(b->d_bits, 0, (size_t)h->n * sizeof(uint32_t), st));
  for (int c = 0; c < 3; ++c) b->inertial[body][c] = inertial_origin ? inertial_origin[c] : 0.0;
  StaticWorld& w = b->world;
  for (int k = 0; k < n_shapes; ++k) {
    const PfbStaticShape& s = shapes[k];
    const int j = w.n_shapes + k;
    w.body[j] = body;
    w.kind[j] = s.kind;
    for (int c = 0; c < 3; ++c) w.at[j][c] = (float)s.at[c];
    const double nrm = std::sqrt(s.rot[0] * s.rot[0] + s.rot[3] * s.rot[3]);  // first column = (cos, sin, 0) of the yaw
    w.cyaw[j] = nrm > 0.0 ? (float)(s.rot[0] / nrm) : 1.0f;  // a tilted primitive's yaw is never read (TiltedCtx)
    w.syaw[j] = nrm > 0.0 ? (float)(s.rot[3] / nrm) : 0.0f;
    TiltedWorld& t = b->tworld;
    t.body[j] = body;
    t.kind[j] = s.kind;
    for (int c = 0; c < 3; ++c) t.at[j][c] = w.at[j][c];
    for (int e = 0; e < 9; ++e) t.rot[j][e] = (float)s.rot[e];
    if (s.kind == PFB_SHAPE_BOX) {
      for (int c = 0; c < 3; ++c) w.half[j][c] = (float)s.dims[c];
    } else {
      w.half[j][0] = w.half[j][1] = (float)s.dims[0];
      w.half[j][2] = (float)s.dims[1];
    }
    for (int c = 0; c < 3; ++c) t.half[j][c] = w.half[j][c];
  }
  const double z = quat[2], qw = quat[3], d = qw * qw + z * z;
  // the yaw pose of a tilted body is never read (TiltedCtx); d = 0 (a half turn about a horizontal axis) keeps it finite
  k_static_fill<<<grid_for(h->n), kBlock, 0, st>>>(b->d_pose, body, (float)pos[0], (float)pos[1], (float)pos[2], d > 0.0 ? (float)((qw * qw - z * z) / d) : 1.0f,
                                                   d > 0.0 ? (float)(2.0 * qw * z / d) : 0.0f, h->n);
  LAUNCH_CHECK(h);
  if (b->d_full) {
    double r[9];
    quat_rotation(quat[0], quat[1], quat[2], quat[3], r);
    FullPose fp;
    for (int c = 0; c < 3; ++c) fp.v[c] = (float)pos[c];
    for (int e = 0; e < 9; ++e) fp.v[3 + e] = (float)r[e];
    k_static_fill_full<<<grid_for(h->n), kBlock, 0, st>>>(b->d_full, body, fp, h->n);
    LAUNCH_CHECK(h);
  }
  b->tilted = b->tilted || tilted;
  w.n_shapes += n_shapes;
  b->tworld.n_shapes += n_shapes;
  b->n_bodies += 1;
  *body_id = body;
  return 0;
}

extern "C" int pfb_set_static_pose(PfbHandle h, int body, const double* pos, const double* quat, const uint8_t* mask, void* stream) {
  if (require_aviary_statics(h, "pfb_set_static_pose")) return -1;
  if (!pos || !quat) return fail("pfb_set_static_pose: null argument");
  const int have = h->statics ? h->statics->n_bodies : 0;
  if (body < 0 || body >= have) return fail("pfb_set_static_pose: no static body %d (the handle has %d)", body, have);
  CUDA_OK(cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  bool tilted = false;
  {  // every masked quaternion upright (or, on a solid handle, whether one is tilted), checked in fp64 on the host before anything changes
    const size_t n = (size_t)h->n;
    double* hq = new (std::nothrow) double[4 * n];
    uint8_t* hm = mask ? new (std::nothrow) uint8_t[n] : nullptr;
    if (!hq || (mask && !hm)) {
      delete[] hq;
      delete[] hm;
      return fail("out of host memory");
    }
    cudaError_t e = cudaMemcpyAsync(hq, quat, 4 * n * sizeof(double), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess && mask) e = cudaMemcpyAsync(hm, mask, n, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    int64_t bad = -1;
    for (int64_t i = 0; e == cudaSuccess && bad < 0 && i < h->n; ++i)
      if ((!hm || hm[i]) && !upright(hq + 4 * i)) {
        tilted = true;
        if (!h->static_solid) bad = i;
      }
    delete[] hq;
    delete[] hm;
    if (e != cudaSuccess) return fail("pfb_set_static_pose: reading the quaternions failed: %s", cudaGetErrorString(e));
    if (bad >= 0)
      return fail("pfb_set_static_pose: quat[%lld] is not upright (only a yaw about the world z axis): tilted static bodies are not modelled "
                  "under the top-face rule.  A solid handle (pfb_set_static_solid, solid_static_bodies=True) takes any orientation",
                  (long long)bad);
  }
  StaticBodies* b = h->statics;
  const double* o = b->inertial[body];
  k_static_set_pose<<<grid_for(h->n), kBlock, 0, st>>>(b->d_pose, body, pos, quat, mask, o[0], o[1], o[2], h->n);
  LAUNCH_CHECK(h);
  if (b->d_full) {
    k_static_set_full_pose<<<grid_for(h->n), kBlock, 0, st>>>(b->d_full, body, pos, quat, mask, o[0], o[1], o[2], h->n);
    LAUNCH_CHECK(h);
  }
  b->tilted = b->tilted || tilted;
  return 0;
}

extern "C" int pfb_get_static_contacts(PfbHandle h, uint32_t* bits, void* stream) {
  if (require_aviary_statics(h, "pfb_get_static_contacts")) return -1;
  if (!bits) return fail("pfb_get_static_contacts: null argument");
  if (!step_statics(h)) return fail("pfb_get_static_contacts: the handle has no static bodies (pfb_add_static_body)");
  CUDA_OK(cudaSetDevice(h->device));
  CUDA_OK(cudaMemcpyAsync(bits, h->statics->d_bits, (size_t)h->n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

extern "C" int pfb_set_static_solid(PfbHandle h, int solid, void* stream) {
  if (require_aviary_statics(h, "pfb_set_static_solid")) return -1;
  if (solid != 0 && solid != 1) return fail("pfb_set_static_solid: solid must be 0 (top faces) or 1 (every face), got %d", solid);
  if (solid == 0 && h->statics && h->statics->tilted)
    return fail("pfb_set_static_solid: the handle holds a tilted static body, primitive or pose since its last reset, which the top-face rule "
                "does not model; reset it first");
  if (solid == 1) {
    CUDA_OK(cudaSetDevice(h->device));
    if (static_alloc_full(h, (cudaStream_t)stream)) return -1;
  }
  h->static_solid = solid == 1;
  return 0;
}
