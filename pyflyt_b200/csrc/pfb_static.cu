// pfb_static.cu — static (fixed-base) bodies of an Aviary handle (DESIGN.md §4h): the reference's
// loadURDF(..., useFixedBase=True) of a landing pad, a helipad or a rooftop, one copy in every drone's world.
//
// The primitive table (pfb::StaticWorld) is host-side here and travels to every step launch as a kernel parameter; the poses are
// a field-major device buffer that only pfb_add_static_body and pfb_set_static_pose write.  The step kernels themselves live
// with each vehicle kind (pfb_quadx.cu, pfb_fixedwing.cu, pfb_rocket.cu, pfb_mixed.cu) and run when step_statics(h) is set.
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

void static_destroy(PfbContext* h) {
  StaticBodies* b = h->statics;
  if (!b) return;
  if (b->d_pose) cudaFree(b->d_pose);
  if (b->d_bits) cudaFree(b->d_bits);
  delete b;
  h->statics = nullptr;
}

// the bits are zeroed when the next first body is added
void static_clear(PfbContext* h) {
  if (!h->statics) return;
  h->statics->n_bodies = 0;
  h->statics->world.n_shapes = 0;
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
  if (!upright(quat))
    return fail("pfb_add_static_body: the body must stay upright (only a yaw about the world z axis): tilted static bodies are not modelled");
  // each primitive upright in the body frame: a box yawed about its z axis, a cylinder whose axis is z
  for (int k = 0; k < n_shapes; ++k) {
    const PfbStaticShape& s = shapes[k];
    if (s.kind != PFB_SHAPE_BOX && s.kind != PFB_SHAPE_CYLINDER)
      return fail("pfb_add_static_body: primitive %d is a %s; static bodies are boxes and cylinders", k, s.kind == PFB_SHAPE_SPHERE ? "sphere" : "mesh or unknown shape");
    const double* r = s.rot;
    const double tilt = fabs(r[2]) + fabs(r[5]) + fabs(r[6]) + fabs(r[7]) + fabs(r[8] - 1.0);
    if (!(tilt <= 1e-9)) return fail("pfb_add_static_body: primitive %d is tilted in its body; only a yaw about the body's z axis is modelled", k);
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
    w.cyaw[j] = (float)(s.rot[0] / nrm);
    w.syaw[j] = (float)(s.rot[3] / nrm);
    if (s.kind == PFB_SHAPE_BOX) {
      for (int c = 0; c < 3; ++c) w.half[j][c] = (float)s.dims[c];
    } else {
      w.half[j][0] = w.half[j][1] = (float)s.dims[0];
      w.half[j][2] = (float)s.dims[1];
    }
  }
  const double z = quat[2], qw = quat[3], d = qw * qw + z * z;
  k_static_fill<<<grid_for(h->n), kBlock, 0, st>>>(b->d_pose, body, (float)pos[0], (float)pos[1], (float)pos[2], (float)((qw * qw - z * z) / d),
                                                   (float)(2.0 * qw * z / d), h->n);
  LAUNCH_CHECK(h);
  w.n_shapes += n_shapes;
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
  {  // every masked quaternion upright, checked in fp64 on the host before anything changes
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
      if ((!hm || hm[i]) && !upright(hq + 4 * i)) bad = i;
    delete[] hq;
    delete[] hm;
    if (e != cudaSuccess) return fail("pfb_set_static_pose: reading the quaternions failed: %s", cudaGetErrorString(e));
    if (bad >= 0)
      return fail("pfb_set_static_pose: quat[%lld] is not upright (only a yaw about the world z axis): tilted static bodies are not modelled",
                  (long long)bad);
  }
  const double* o = h->statics->inertial[body];
  k_static_set_pose<<<grid_for(h->n), kBlock, 0, st>>>(h->statics->d_pose, body, pos, quat, mask, o[0], o[1], o[2], h->n);
  LAUNCH_CHECK(h);
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
