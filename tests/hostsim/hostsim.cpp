// TEST HARNESS — compiles the per-env kernel body (pyflyt_b200/csrc/pfb_quadx.cuh) for the HOST so the
// fp32/fp64 precision policy and the control-flow of the CUDA kernels can be studied and unit-tested on
// a machine without a GPU.  Never linked into, loaded by, or reachable from the product package:
// libpyflyt_b200.so contains CUDA kernels only and fails loudly without a device.
// The glue below mirrors the kernels in pfb_quadx.cu one-to-one (same loads, same order, same stores).
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "../../pyflyt_b200/csrc/pfb_quadx.cuh"

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
#include "../../pyflyt_b200/csrc/pfb_rocket_host.h"

using namespace pfb;

struct HostNoise {
  const float* ptr;
  int64_t N;
  void begin_step() {}
  float get(int) {
    float v = *ptr;
    ptr += N;
    return v;
  }
};

#define MODE_SWITCH(mode, BODY)                        \
  switch (mode) {                                      \
    case -1: { constexpr int MODE = -1; BODY; } break; \
    case 0: { constexpr int MODE = 0; BODY; } break;   \
    case 1: { constexpr int MODE = 1; BODY; } break;   \
    case 2: { constexpr int MODE = 2; BODY; } break;   \
    case 3: { constexpr int MODE = 3; BODY; } break;   \
    case 4: { constexpr int MODE = 4; BODY; } break;   \
    case 5: { constexpr int MODE = 5; BODY; } break;   \
    case 6: { constexpr int MODE = 6; BODY; } break;   \
    case 7: { constexpr int MODE = 7; BODY; } break;   \
    default: return fail("bad mode %d", mode);         \
  }

static void hover_params(const PfbEnvConfig* env, HoverParams& h) {
  h.env_step_ratio = env->env_step_ratio;
  h.max_steps = env->max_steps;
  h.angle_representation = env->angle_representation;
  h.sparse_reward = env->sparse_reward;
  h.warmup_steps = env->warmup_steps;
  h.flight_mode = env->flight_mode;
  h.dome2 = (float)(env->flight_dome_size * env->flight_dome_size);
}

#define HS_API extern "C"
HS_API const char* hs_last_error() { return g_err; }
// the counter RNG of the kernels (pfb_common.cuh), for tests/test_philox_replay.py
HS_API void hs_philox(const uint32_t* ctr, uint32_t k0, uint32_t k1, uint32_t* out, float* normals, int64_t n) {
  for (int64_t i = 0; i < n; ++i) {
    U4 r = philox4x32_10(U4{ctr[4 * i], ctr[4 * i + 1], ctr[4 * i + 2], ctr[4 * i + 3]}, k0, k1);
    out[4 * i] = r.x; out[4 * i + 1] = r.y; out[4 * i + 2] = r.z; out[4 * i + 3] = r.w;
    box_muller(r.x, r.y, normals[4 * i], normals[4 * i + 1]);
    box_muller(r.z, r.w, normals[4 * i + 2], normals[4 * i + 3]);
  }
}
HS_API int hs_state_rows() { return QX_ROWS; }
HS_API int hs_istate_rows() { return QI_ROWS; }
HS_API int hs_precision_flags() { return PFB_Q_DOUBLE | (PFB_X_DOUBLE << 1) | (PFB_V_DOUBLE << 2) | (PFB_R_DOUBLE << 3); }

HS_API int hs_reset(const PfbModel* m, float* st, int32_t* ist, float* setpoint, const float* start_pos, const float* start_orn,
             const uint8_t* mask, int64_t N) {
  for (int64_t i = 0; i < N; ++i) {
    if (mask && !mask[i]) continue;
    QuadXRegs s;
    quadx_reset(s, start_pos[3 * i], start_pos[3 * i + 1], start_pos[3 * i + 2], start_orn[3 * i], start_orn[3 * i + 1],
                start_orn[3 * i + 2]);
    quadx_store<7>(st, ist, N, i, s);
    ist[(int64_t)QI_STEP * N + i] = 0;
    for (int k = 0; k < 4; ++k) setpoint[4 * i + k] = 0.f;
  }
  return 0;
}

template <int MODE>
static void set_mode_t(float* st, int32_t* ist, float* setpoint, int64_t N) {
  for (int64_t i = 0; i < N; ++i) {
    QuadXRegs s;
    quadx_load<7>(st, ist, N, i, s);
    for (int k = 0; k < 4; ++k) s.sp[k] = setpoint[4 * i + k];
    quadx_set_mode<MODE>(s);
    quadx_store<7>(st, ist, N, i, s);
    for (int k = 0; k < 4; ++k) setpoint[4 * i + k] = s.sp[k];
  }
}
HS_API int hs_set_mode(int mode, float* st, int32_t* ist, float* setpoint, int64_t N) {
  MODE_SWITCH(mode, (set_mode_t<MODE>(st, ist, setpoint, N)));
  return 0;
}

template <int MODE>
static void aviary_step_t(const QuadXParams& p, float* st, int32_t* ist, const float* setpoint, const float* noise,
                          int n_steps, int64_t N) {
  for (int64_t i = 0; i < N; ++i) {
    QuadXRegs s;
    quadx_load<MODE>(st, ist, N, i, s);
    for (int k = 0; k < 4; ++k) s.sp[k] = setpoint[4 * i + k];
    HostNoise nz{noise + i, N};
    for (int k = 0; k < n_steps; ++k) quadx_aviary_step<MODE>(p, s, nz);
    quadx_store<MODE>(st, ist, N, i, s);
  }
}
HS_API int hs_aviary_step(const PfbModel* m, int mode, float* st, int32_t* ist, const float* setpoint, const float* noise,
                   int n_steps, int64_t N) {
  QuadXParams p;
  if (build_quadx_params(*m, p)) return -1;
  MODE_SWITCH(mode, (aviary_step_t<MODE>(p, st, ist, setpoint, noise, n_steps, N)));
  return 0;
}

HS_API int hs_observe(const float* st, const int32_t* ist, float* drone_state, float* aux, uint8_t* contact, int64_t N) {
  for (int64_t i = 0; i < N; ++i) {
    QuadXRegs s;
    quadx_load<-1>(st, ist, N, i, s);
    quadx_drone_state(s, drone_state + 12 * i, aux + 4 * i);
    contact[i] = (s.flags & FLAG_CONTACT_ARRAY) ? 1 : 0;
  }
  return 0;
}

template <int MODE>
static void env_reset_t(const QuadXParams& p, const HoverParams& h, float* st, int32_t* ist, const float* start_pos,
                        const float* start_orn, const uint8_t* mask, const float* noise, float* obs, int64_t N) {
  const int O = h.angle_representation == 0 ? 20 : 21;
  for (int64_t i = 0; i < N; ++i) {
    if (mask && !mask[i]) continue;
    QuadXRegs s;
    quadx_reset(s, start_pos[3 * i], start_pos[3 * i + 1], start_pos[3 * i + 2], start_orn[3 * i], start_orn[3 * i + 1],
                start_orn[3 * i + 2]);
    quadx_set_mode<MODE>(s);
    HostNoise nz{noise + i, N};
    for (int k = 0; k < h.warmup_steps; ++k) quadx_aviary_step<MODE>(p, s, nz);
    const float zero[4] = {0.f, 0.f, 0.f, 0.f};
    float my_obs[21];
    hover_observation(h, s, zero, my_obs);
    quadx_store<7>(st, ist, N, i, s);
    ist[(int64_t)QI_STEP * N + i] = 0;
    for (int k = 0; k < O; ++k) obs[i * O + k] = my_obs[k];
  }
}
HS_API int hs_env_reset(const PfbModel* m, const PfbEnvConfig* env, float* st, int32_t* ist, const float* start_pos,
                 const float* start_orn, const uint8_t* mask, const float* noise, float* obs, int64_t N) {
  QuadXParams p;
  if (build_quadx_params(*m, p)) return -1;
  HoverParams h;
  hover_params(env, h);
  MODE_SWITCH(env->flight_mode, (env_reset_t<MODE>(p, h, st, ist, start_pos, start_orn, mask, noise, obs, N)));
  return 0;
}

template <int MODE>
static void env_step_t(const QuadXParams& p, const HoverParams& h, float* st, int32_t* ist, const float* actions,
                       const float* noise, float* obs, float* reward, uint8_t* term, uint8_t* trunc, uint8_t* info, int64_t N) {
  const int O = h.angle_representation == 0 ? 20 : 21;
  for (int64_t i = 0; i < N; ++i) {
    QuadXRegs s;
    quadx_load<MODE>(st, ist, N, i, s);
    float act[4];
    for (int k = 0; k < 4; ++k) { act[k] = actions[4 * i + k]; s.sp[k] = act[k]; }
    int step_count = ist[(int64_t)QI_STEP * N + i];
    HostNoise nz{noise + i, N};
    float rew = -0.1f;
    for (int k = 0; k < h.env_step_ratio; ++k) {
      if (s.flags & (FLAG_TERM | FLAG_TRUNC)) break;
      quadx_aviary_step<MODE>(p, s, nz);
      hover_term_trunc_reward(h, s, step_count, rew);
    }
    step_count += 1;
    float my_obs[21];
    hover_observation(h, s, act, my_obs);
    quadx_store<MODE>(st, ist, N, i, s);
    ist[(int64_t)QI_STEP * N + i] = step_count;
    reward[i] = rew;
    term[i] = (s.flags & FLAG_TERM) ? 1 : 0;
    trunc[i] = (s.flags & FLAG_TRUNC) ? 1 : 0;
    info[i] = (uint8_t)(((s.flags & FLAG_OOB) ? 1 : 0) | ((s.flags & FLAG_COLLISION) ? 2 : 0));
    for (int k = 0; k < O; ++k) obs[i * O + k] = my_obs[k];
  }
}
HS_API int hs_env_step(const PfbModel* m, const PfbEnvConfig* env, float* st, int32_t* ist, const float* actions, const float* noise,
                float* obs, float* reward, uint8_t* term, uint8_t* trunc, uint8_t* info, int64_t N) {
  QuadXParams p;
  if (build_quadx_params(*m, p)) return -1;
  HoverParams h;
  hover_params(env, h);
  MODE_SWITCH(env->flight_mode, (env_step_t<MODE>(p, h, st, ist, actions, noise, obs, reward, term, trunc, info, N)));
  return 0;
}

// unit hook: the observation quaternion the kernel reports for attitude q (quaternion representation)
HS_API int hs_obs_quat(const double* q, float* out4) {
  QuadXRegs s;
  memset(&s, 0, sizeof(s));
  s.qx = (qreal)q[0]; s.qy = (qreal)q[1]; s.qz = (qreal)q[2]; s.qw = (qreal)q[3];
  HoverParams h;
  memset(&h, 0, sizeof(h));
  h.angle_representation = 1;
  const float act[4] = {0, 0, 0, 0};
  float obs[21];
  hover_observation(h, s, act, obs);
  for (int k = 0; k < 4; ++k) out4[k] = obs[3 + k];
  return 0;
}

HS_API float hs_atan2(float y, float x) { return atan2_f(y, x); }

// ---- fixedwing (Aviary level) -------------------------------------------------------------------
HS_API int hs_fw_state_rows() { return FW_ROWS; }
HS_API int hs_fw_istate_rows() { return FI_ROWS; }

HS_API int hs_fw_reset(const PfbModel* m, float* st, int32_t* ist, float* setpoint, const float* start_pos, const float* start_orn, int64_t N) {
  FixedwingParams p;
  WaypointParams w;
  if (fw_build_params_impl(*m, nullptr, p, w)) return -1;
  for (int64_t i = 0; i < N; ++i) {
    FixedwingRegs s;
    fixedwing_reset(p, s, start_pos[3 * i], start_pos[3 * i + 1], start_pos[3 * i + 2], start_orn[3 * i], start_orn[3 * i + 1], start_orn[3 * i + 2]);
    fixedwing_store(st, ist, N, i, s);
    ist[(int64_t)FI_STEP * N + i] = 0;
    for (int k = 0; k < 6; ++k) setpoint[6 * i + k] = 0.f;
  }
  return 0;
}

HS_API int hs_fw_aviary_step(const PfbModel* m, int mode, float* st, int32_t* ist, const float* setpoint, const float* noise, int n_steps, int64_t N) {
  FixedwingParams p;
  WaypointParams w;
  if (fw_build_params_impl(*m, nullptr, p, w)) return -1;
  for (int64_t i = 0; i < N; ++i) {
    FixedwingRegs s;
    fixedwing_load(st, ist, N, i, s);
    for (int k = 0; k < 6; ++k) s.sp[k] = setpoint[6 * i + k];
    HostNoise nz{noise + i, N};
    for (int k = 0; k < n_steps; ++k) {
      if (mode == 0) fixedwing_aviary_step<0>(p, s, nz); else fixedwing_aviary_step<-1>(p, s, nz);
    }
    fixedwing_store(st, ist, N, i, s);
  }
  return 0;
}

// the one-basic-block instantiation the step kernels take when the model has all its surfaces and there is no wind
// (fixedwing_substep<FULL>, pfb_fixedwing.cuh): same arithmetic as the generic path, pinned to it by tests/test_fixedwing.py
HS_API int hs_fw_aviary_step_full(const PfbModel* m, int mode, float* st, int32_t* ist, const float* setpoint, const float* noise, int n_steps, int64_t N) {
  FixedwingParams p;
  WaypointParams w;
  if (fw_build_params_impl(*m, nullptr, p, w)) return -1;
  if (!fixedwing_full_model(p)) return fail("hs_fw_aviary_step_full: the model is not complete (surfaces / wind)");
  for (int64_t i = 0; i < N; ++i) {
    FixedwingRegs s;
    fixedwing_load(st, ist, N, i, s);
    for (int k = 0; k < 6; ++k) s.sp[k] = setpoint[6 * i + k];
    HostNoise nz{noise + i, N};
    for (int k = 0; k < n_steps; ++k) {
      if (mode == 0) fixedwing_aviary_step<0, true>(p, s, nz); else fixedwing_aviary_step<-1, true>(p, s, nz);
    }
    fixedwing_store(st, ist, N, i, s);
  }
  return 0;
}

HS_API int hs_fw_observe(const float* st, const int32_t* ist, float* drone_state, float* aux, uint8_t* contact, int64_t N) {
  for (int64_t i = 0; i < N; ++i) {
    FixedwingRegs s;
    fixedwing_load(st, ist, N, i, s);
    fixedwing_drone_state(s, drone_state + 12 * i, aux + 6 * i);
    contact[i] = (s.flags & FLAG_CONTACT_ARRAY) ? 1 : 0;
  }
  return 0;
}

// ---- rocket (Aviary level) ------------------------------------------------------------------------
HS_API int hs_rk_state_rows() { return RK_ROWS; }
HS_API int hs_rk_istate_rows() { return RI_ROWS; }

HS_API int hs_rk_reset(const PfbModel* m, float* st, int32_t* ist, float* setpoint, const float* start_pos, const float* start_orn, int64_t N) {
  RocketParams p;
  LandingParams l;
  if (rk_build_params_impl(*m, nullptr, p, l)) return -1;
  for (int64_t i = 0; i < N; ++i) {
    RocketRegs s;
    rocket_reset(p, s, start_pos[3 * i], start_pos[3 * i + 1], start_pos[3 * i + 2], start_orn[3 * i], start_orn[3 * i + 1], start_orn[3 * i + 2]);
    rocket_store(st, ist, N, i, s);
    ist[(int64_t)RI_STEP * N + i] = 0;
    for (int k = 0; k < 7; ++k) setpoint[7 * i + k] = 0.f;
  }
  return 0;
}

HS_API int hs_rk_set_velocity(float* st, int32_t* ist, const float* lin, const float* ang, int64_t N) {
  for (int64_t i = 0; i < N; ++i) {
    RocketRegs s;
    rocket_load(st, ist, N, i, s);
    s.vx = lin[3 * i]; s.vy = lin[3 * i + 1]; s.vz = lin[3 * i + 2];
    float ox = ang[3 * i], oy = ang[3 * i + 1], oz = ang[3 * i + 2];
    const Rot<rreal>& R = s.R;
    s.wx = (float)R.m00 * ox + (float)R.m10 * oy + (float)R.m20 * oz;
    s.wy = (float)R.m01 * ox + (float)R.m11 * oy + (float)R.m21 * oz;
    s.wz = (float)R.m02 * ox + (float)R.m12 * oy + (float)R.m22 * oz;
    rocket_store(st, ist, N, i, s);
  }
  return 0;
}

HS_API int hs_rk_aviary_step(const PfbModel* m, float* st, int32_t* ist, const float* setpoint, const float* noise, int n_steps, int64_t N) {
  RocketParams p;
  LandingParams l;
  if (rk_build_params_impl(*m, nullptr, p, l)) return -1;
  for (int64_t i = 0; i < N; ++i) {
    RocketRegs s;
    rocket_load(st, ist, N, i, s);
    for (int k = 0; k < 7; ++k) s.sp[k] = setpoint[7 * i + k];
    HostNoise nz{noise + i, N};
    for (int k = 0; k < n_steps; ++k) rocket_aviary_step(p, s, nz, false);
    rocket_store(st, ist, N, i, s);
  }
  return 0;
}

HS_API int hs_rk_observe(const float* st, const int32_t* ist, float* drone_state, float* aux, uint8_t* contact, int64_t N) {
  for (int64_t i = 0; i < N; ++i) {
    RocketRegs s;
    rocket_load(st, ist, N, i, s);
    rocket_drone_state(s, drone_state + 12 * i, aux + 9 * i);
    contact[i] = (s.flags & FLAG_CONTACT_ARRAY) ? 1 : 0;
  }
  return 0;
}
