// TEST HARNESS — runs the shared PFB_HD math helpers of pyflyt_b200/csrc one element at a time, so that each can be held
// against an fp64 reference on its own (tests/test_device_math.py).  Built twice from this one file by the `probe` target
// of pyflyt_b200/csrc/Makefile:
//   * nvcc with the product's flags (sm_90a): a grid-stride kernel per helper, arrays are DEVICE pointers;
//   * g++: the same evaluators in a host loop, arrays are HOST pointers (IEEE division / sqrt and libm in the helpers).
// Each evaluator calls the helper and nothing else.  Never linked into libpyflyt_b200.so; the kernels only write results.
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "../../pyflyt_b200/csrc/pfb_rocket.cuh"

static char g_err[512];
static int fail(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return -1;
}
#include "../../pyflyt_b200/csrc/pfb_quadx_host.h"
#include "../../pyflyt_b200/csrc/pfb_fixedwing_host.h"

using namespace pfb;

#if defined(__CUDACC__)
template <class Eval>
__global__ void k_probe(const Eval e, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) e(i);
}
template <class Eval>
static int run(const Eval& e, int64_t n) {
  if (n <= 0) return 0;
  const int64_t blocks = (n + 255) / 256;
  k_probe<<<(unsigned)(blocks < 8192 ? blocks : 8192), 256>>>(e, n);
  cudaError_t err = cudaGetLastError();
  if (err == cudaSuccess) err = cudaDeviceSynchronize();
  return err == cudaSuccess ? 0 : fail("probe kernel: %s", cudaGetErrorString(err));
}
#define PROBE_DEVICE 1
#else
template <class Eval>
static int run(const Eval& e, int64_t n) {
  for (int64_t i = 0; i < n; ++i) e(i);
  return 0;
}
#define PROBE_DEVICE 0
#endif

struct Atan2 {
  const float *y, *x;
  float* out;
  PFB_HD void operator()(int64_t i) const { out[i] = atan2_f(y[i], x[i]); }
};
struct Euler {  // q[n][4] (x, y, z, w) -> roll, pitch, yaw [n][3]
  const float* q;
  float* out;
  PFB_HD void operator()(int64_t i) const {
    const float* p = q + 4 * i;
    euler_from_quat(p[0], p[1], p[2], p[3], out[3 * i], out[3 * i + 1], out[3 * i + 2]);
  }
};
struct RollPitch {  // q[n][4] -> roll, pitch [n][2]
  const float* q;
  float* out;
  PFB_HD void operator()(int64_t i) const {
    const float* p = q + 4 * i;
    roll_pitch_from_quat(p[0], p[1], p[2], p[3], out[2 * i], out[2 * i + 1]);
  }
};
struct HoverAttitude {  // q[n][4] -> the attitude block of the Hover observation: Euler [n][3] or quaternion [n][4]
  const float* q;
  float* out;
  int quaternion;
  PFB_HD void operator()(int64_t i) const {
    QuadXRegs s;
    memset(&s, 0, sizeof(s));
    const float* p = q + 4 * i;
    s.qx = (qreal)p[0]; s.qy = (qreal)p[1]; s.qz = (qreal)p[2]; s.qw = (qreal)p[3];
    HoverParams h;
    memset(&h, 0, sizeof(h));
    h.angle_representation = quaternion;
    const float act[4] = {0.f, 0.f, 0.f, 0.f};
    float obs[21];
    hover_observation(h, s, act, obs);
    const int k = quaternion ? 4 : 3;
    for (int j = 0; j < k; ++j) out[k * i + j] = obs[3 + j];
  }
};
struct QuatFromEuler {  // e[n][3] (roll, pitch, yaw) -> q[n][4]
  const float* e;
  float* out;
  PFB_HD void operator()(int64_t i) const {
    const float* p = e + 3 * i;
    quat_from_euler(p[0], p[1], p[2], out[4 * i], out[4 * i + 1], out[4 * i + 2], out[4 * i + 3]);
  }
};
struct SinCos {
  const float* x;
  float *s, *c;
  PFB_HD void operator()(int64_t i) const { sincos_f(x[i], s[i], c[i]); }
};
struct Surface {  // act[n], vb[n][3], w[n][3] -> F[n][3], T[n][3]; cmd == act, so the actuator lag leaves act as it is
  SurfaceParams sf;
  const float *act, *vb, *w;
  float *F, *T;
  PFB_HD void operator()(int64_t i) const {
    float a = act[i];
    Vec3 f = Vec3{0.f, 0.f, 0.f}, t = Vec3{0.f, 0.f, 0.f};
    surface_force(sf, a, a, Vec3{vb[3 * i], vb[3 * i + 1], vb[3 * i + 2]}, Vec3{w[3 * i], w[3 * i + 1], w[3 * i + 2]}, f, t);
    F[3 * i] = f.x; F[3 * i + 1] = f.y; F[3 * i + 2] = f.z;
    T[3 * i] = t.x; T[3 * i + 1] = t.y; T[3 * i + 2] = t.z;
  }
};
struct BoxMuller {
  const uint32_t *a, *b;
  float *n0, *n1;
  PFB_HD void operator()(int64_t i) const { box_muller(a[i], b[i], n0[i], n1[i]); }
};
struct Wind {
  WindParams w;
  const float* z;
  float* out;
  PFB_HD void operator()(int64_t i) const { out[i] = wind_profile(w, z[i]); }
};
struct Sym3 {  // J[n][6] = (a, b, c, d, e, f) of [[a b c], [b d e], [c e f]], r[n][3] -> J^-1 r [n][3]
  const float *J, *r;
  float* out;
  PFB_HD void operator()(int64_t i) const {
    const float* j = J + 6 * i;
    Vec3 x = solve_sym3(j[0], j[1], j[2], j[3], j[4], j[5], Vec3{r[3 * i], r[3 * i + 1], r[3 * i + 2]});
    out[3 * i] = x.x; out[3 * i + 1] = x.y; out[3 * i + 2] = x.z;
  }
};
struct Fast {  // 0: fast_rcp, 1: fast_rsqrt, 2: fast_sqrt
  int which;
  const float* x;
  float* out;
  PFB_HD void operator()(int64_t i) const { out[i] = which == 0 ? fast_rcp(x[i]) : which == 1 ? fast_rsqrt(x[i]) : fast_sqrt(x[i]); }
};

#define PROBE_API extern "C" __attribute__((visibility("default")))

PROBE_API const char* probe_last_error(void) { return g_err; }
PROBE_API int probe_is_device(void) { return PROBE_DEVICE; }
PROBE_API int probe_atan2(int64_t n, const float* y, const float* x, float* out) { return run(Atan2{y, x, out}, n); }
PROBE_API int probe_euler(int64_t n, const float* q, float* out) { return run(Euler{q, out}, n); }
PROBE_API int probe_roll_pitch(int64_t n, const float* q, float* out) { return run(RollPitch{q, out}, n); }
PROBE_API int probe_hover_attitude(int64_t n, const float* q, int quaternion, float* out) {
  return run(HoverAttitude{q, out, quaternion}, n);
}
PROBE_API int probe_quat_from_euler(int64_t n, const float* e, float* out) { return run(QuatFromEuler{e, out}, n); }
PROBE_API int probe_sincos(int64_t n, const float* x, float* s, float* c) { return run(SinCos{x, s, c}, n); }
// surface `si` of a HOST PfbModel, narrowed as pfb_create narrows it
PROBE_API int probe_surface_force(const PfbModel* m, int si, int64_t n, const float* act, const float* vb, const float* w, float* F, float* T) {
  if (si < 0 || si >= m->n_surfaces) return fail("surface %d out of range", si);
  Surface e;
  pfb_build_surface(m->surfaces[si], e.sf);
  e.act = act; e.vb = vb; e.w = w; e.F = F; e.T = T;
  return run(e, n);
}
PROBE_API int probe_box_muller(int64_t n, const uint32_t* a, const uint32_t* b, float* n0, float* n1) { return run(BoxMuller{a, b, n0, n1}, n); }
// a HOST PfbWind, narrowed as pfb_set_wind narrows it
PROBE_API int probe_wind_profile(const PfbWind* wind, int64_t n, const float* z, float* out) {
  Wind e;
  pfb_narrow_wind(wind, e.w);
  e.z = z; e.out = out;
  return run(e, n);
}
PROBE_API int probe_solve_sym3(int64_t n, const float* J, const float* r, float* out) { return run(Sym3{J, r, out}, n); }
PROBE_API int probe_fast(int which, int64_t n, const float* x, float* out) {
  if (which < 0 || which > 2) return fail("fast helper %d out of range", which);
  return run(Fast{which, x, out}, n);
}
