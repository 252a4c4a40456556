// TEST HARNESS — runs the shared PFB_HD math helpers of pyflyt_b200/csrc one element at a time, so that each can be held
// against an fp64 reference on its own (tests/test_device_math.py; the floor contact solver and flag: tests/test_contact_solver.py).
// Built twice from this one file by the `probe` target of pyflyt_b200/csrc/Makefile:
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

// apply_contact_impulses over a primitive list (ContactParams, or the QuadX table read in place), with the vehicle's own state
// registers: pz[n], R[n][9] (body to world, row-major), world velocity v[n][3], body rate w[n][3], mass M[n], COM offset c[n][3],
// central inertia Ic[n][6] (xx, xy, xz, yy, yz, zz; base frame), surface height top[n] -> world velocity vo[n][3], body rate wo[n][3]
template <class Shapes, class Regs>
struct ContactImpulses {
  Shapes cp;
  float dt;
  const float *pz, *R, *v, *w, *M, *c, *Ic, *top;
  float *vo, *wo;
  PFB_HD void operator()(int64_t i) const {
    Regs s;
    memset(&s, 0, sizeof(s));
    const float* r = R + 9 * i;
    s.R.m00 = r[0]; s.R.m01 = r[1]; s.R.m02 = r[2]; s.R.m10 = r[3]; s.R.m11 = r[4]; s.R.m12 = r[5]; s.R.m20 = r[6]; s.R.m21 = r[7]; s.R.m22 = r[8];
    s.vx = v[3 * i]; s.vy = v[3 * i + 1]; s.vz = v[3 * i + 2];
    s.wx = w[3 * i]; s.wy = w[3 * i + 1]; s.wz = w[3 * i + 2];
    const float* I = Ic + 6 * i;
    apply_contact_impulses(&cp, s, pz[i], top[i], M[i], Vec3{c[3 * i], c[3 * i + 1], c[3 * i + 2]}, I[0], I[1], I[2], I[3], I[4], I[5], dt);
    vo[3 * i] = (float)s.vx; vo[3 * i + 1] = (float)s.vy; vo[3 * i + 2] = (float)s.vz;
    wo[3 * i] = s.wx; wo[3 * i + 1] = s.wy; wo[3 * i + 2] = s.wz;
  }
};
struct GroundContact {  // pz[n], R[n][9], top[n] -> ground_contact flag [n]
  ContactParams cp;
  const float *pz, *R, *top;
  int32_t* out;
  PFB_HD void operator()(int64_t i) const { out[i] = ground_contact(cp, pz[i], R[9 * i + 6], R[9 * i + 7], R[9 * i + 8], top[i]) ? 1 : 0; }
};
struct QuadXGroundContact {  // pz[n], R[n][9] -> quadx_ground_contact flag [n] (the floor only)
  QuadXParams p;
  const float *pz, *R;
  int32_t* out;
  PFB_HD void operator()(int64_t i) const {
    QuadXRegs s;
    memset(&s, 0, sizeof(s));
    s.pz = pz[i];
    s.R.m20 = R[9 * i + 6]; s.R.m21 = R[9 * i + 7]; s.R.m22 = R[9 * i + 8];
    out[i] = quadx_ground_contact(p, s) ? 1 : 0;
  }
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
// the contact solver of a HOST PfbModel, narrowed as pfb_create narrows it: the QuadX table for QuadX models, a ContactParams
// with the fixed-wing or rocket registers otherwise
template <class Shapes, class Regs>
static int run_contact(const Shapes& cp, float dt, int64_t n, const float* pz, const float* R, const float* v, const float* w, const float* M,
                       const float* c, const float* Ic, const float* top, float* vo, float* wo) {
  ContactImpulses<Shapes, Regs> e;
  e.cp = cp; e.dt = dt;
  e.pz = pz; e.R = R; e.v = v; e.w = w; e.M = M; e.c = c; e.Ic = Ic; e.top = top; e.vo = vo; e.wo = wo;
  return run(e, n);
}
PROBE_API int probe_contact_impulses(const PfbModel* m, int64_t n, const float* pz, const float* R, const float* v, const float* w, const float* M,
                                     const float* c, const float* Ic, const float* top, float* vo, float* wo) {
  const float dt = (float)(1.0 / m->physics_hz);
  if (m->kind == PFB_KIND_QUADX) {
    QuadXParams p;
    if (build_quadx_params(*m, p)) return -1;
    return run_contact<QuadXParams, QuadXRegs>(p, dt, n, pz, R, v, w, M, c, Ic, top, vo, wo);
  }
  ContactParams cp;
  memset(&cp, 0, sizeof(cp));
  if (pfb_build_contact(*m, cp)) return -1;
  if (m->kind == PFB_KIND_ROCKET) return run_contact<ContactParams, RocketRegs>(cp, dt, n, pz, R, v, w, M, c, Ic, top, vo, wo);
  return run_contact<ContactParams, FixedwingRegs>(cp, dt, n, pz, R, v, w, M, c, Ic, top, vo, wo);
}
// the contact flag: quadx_ground_contact over the QuadX table (top must be 0: QuadX drones meet the floor only), ground_contact otherwise
PROBE_API int probe_contact_flag(const PfbModel* m, int64_t n, const float* pz, const float* R, const float* top, int32_t* out) {
  if (m->kind == PFB_KIND_QUADX) {
    QuadXGroundContact e;
    if (build_quadx_params(*m, e.p)) return -1;
    e.pz = pz; e.R = R; e.out = out;
    return run(e, n);
  }
  GroundContact e;
  memset(&e.cp, 0, sizeof(e.cp));
  if (pfb_build_contact(*m, e.cp)) return -1;
  e.pz = pz; e.R = R; e.top = top; e.out = out;
  return run(e, n);
}
