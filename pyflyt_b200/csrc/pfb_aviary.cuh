// pfb_aviary.cuh — the per-drone bodies of the Aviary operations, one per vehicle kind: the state query, the reset, the
// per-drone set_mode and the base state (set / get), and the world of the Aviary step kernels.  A body works on row j of its
// kind's state region (QuadX warp-tiled, fixed-wing and rocket field-major [F][n] + istate [I][n]) and takes drone u's setpoint
// row (SP floats apart), start pose or base-state rows.  The single-kind kernels call them with j = u = i; the mixed-kind kernels (pfb_mixed.cu) with u = slot_user[j].
// Pointers are passed as parameters, not in structs (a __restrict__ member loses its __restrict__), and a table is bound by
// reference to the kernel's own __grid_constant__ parameter (a copy of it is staged on the stack).
#pragma once

#include "pfb_context.h"
#include "pfb_noise.cuh"

namespace pfb {

// QuadX handles keep their state WARP-TILED (pfb_quadx.cuh) except QuadX-Waypoints, whose kernels (pfb_quadx_wp.cu) still use
// the field-major [F][N] rows + istate; TILED selects the addressing of the kernels both layouts share.
template <int MODE, bool TILED>
__device__ __forceinline__ void qx_load_any(const float* __restrict__ st, const int32_t* __restrict__ ist, int rows, int64_t N, int64_t i,
                                            QuadXRegs& s, int& step_count) {
  if (TILED) {
    quadx_load_tile<MODE, kTileGroupStride>(st + qx_tile_base(i, rows), s, step_count);
  } else {
    quadx_load<MODE>(st, ist, N, i, s);
    step_count = ist[(int64_t)QI_STEP * N + i];
  }
}
template <int MODE, bool TILED>
__device__ __forceinline__ void qx_store_any(float* __restrict__ st, int32_t* __restrict__ ist, int rows, int64_t N, int64_t i,
                                             const QuadXRegs& s, int step_count) {
  if (TILED) {
    quadx_store_tile<MODE, kTileGroupStride>(st + qx_tile_base(i, rows), s, step_count);
  } else {
    quadx_store<MODE>(st, ist, N, i, s);
    ist[(int64_t)QI_STEP * N + i] = step_count;
  }
}

// setpoint row u of a [*][SP] buffer into the drone's registers
template <int SP, int W>
__device__ __forceinline__ void load_setpoint(const float* setpoint, int64_t u, float* sp) {
  if constexpr (SP == 4 && W == 4) {
    float4 v = __ldg(reinterpret_cast<const float4*>(setpoint) + u);
    sp[0] = v.x; sp[1] = v.y; sp[2] = v.z; sp[3] = v.w;
  } else {
#pragma unroll
    for (int c = 0; c < W; ++c) sp[c] = __ldg(setpoint + (int64_t)SP * u + c);
  }
}

// ---- the world an Aviary step kernel flies its drones in (World = NoStatic, StaticCtx, SolidCtx or TiltedCtx, pfb_quadx.cuh)
// The static-body table is the kernel's __grid_constant__ parameter of type WorldTable<World>::T: an empty struct on the
// floor-only path, so that its parameter bank does not carry the StaticWorld.  The kernel binds drone i's world to it in place,
// World w{&table, pose, n, i, 0u}; returned by a helper instead, it moves instructions in some kernels (DESIGN.md §4h).  A
// NoStatic world is never dereferenced (every use in the substeps is behind `if constexpr (World::kOn)`).
template <class World>
struct WorldTable {
  using T = NoStaticTable;
};
template <>
struct WorldTable<StaticCtx> {
  using T = StaticWorld;
};
template <>
struct WorldTable<SolidCtx> {
  using T = StaticWorld;
};
template <>
struct WorldTable<TiltedCtx> {
  using T = TiltedWorld;
};

// ---- Aviary.state(i) / aux_state(i) / contact_array of the drone in row j, and the hi / lo words of its position ------------
// Returns the contact flag.
template <bool TILED>
__device__ __forceinline__ bool qx_query_drone(const float* st, const int32_t* ist, int rows, int64_t n, int64_t j, float* o, float* x, float* hi,
                                               float* lo) {
  QuadXRegs s;
  int step_count;
  qx_load_any<-1, TILED>(st, ist, rows, n, j, s, step_count);
  quadx_drone_state(s, o, x);
  for (int c = 0; c < 3; ++c) {
    hi[c] = st[TILED ? qx_tile_word(j, rows, QX_POS + c) : (QX_POS + c) * n + j];
    lo[c] = st[TILED ? qx_tile_word(j, rows, QX_POS_LO + c) : (QX_POS_LO + c) * n + j];
  }
  return (s.flags & FLAG_CONTACT_ARRAY) != 0;
}
__device__ __forceinline__ bool fw_query_drone(const float* st, const int32_t* ist, int64_t n, int64_t j, float* o, float* x, float* hi, float* lo) {
  FixedwingRegs s;
  fixedwing_load(st, ist, n, j, s);
  fixedwing_drone_state(s, o, x);
  for (int c = 0; c < 3; ++c) {
    hi[c] = st[(FW_POS + c) * n + j];
    lo[c] = st[(FW_POS_LO + c) * n + j];
  }
  return (s.flags & FLAG_CONTACT_ARRAY) != 0;
}
__device__ __forceinline__ bool rk_query_drone(const float* st, const int32_t* ist, int64_t n, int64_t j, float* o, float* x, float* hi, float* lo) {
  RocketRegs s;
  rocket_load(st, ist, n, j, s);
  rocket_drone_state(s, o, x);
  for (int c = 0; c < 3; ++c) {
    hi[c] = st[(RK_POS + c) * n + j];
    lo[c] = st[(RK_POS_LO + c) * n + j];
  }
  return (s.flags & FLAG_CONTACT_ARRAY) != 0;
}

// ---- Aviary.reset of the drone in row j at drone u's start pose (aviary.py:218-312) -----------------------------------------
// The setpoint is the caller's: every kind's reset zeroes it.
template <bool TILED>
__device__ __forceinline__ void qx_reset_drone(float* st, int32_t* ist, int rows, int64_t n, int64_t j, const float* start_pos,
                                               const float* start_orn, int64_t u) {
  QuadXRegs s;  // QuadX.reset (quadx.py:222-231)
  quadx_reset(s, start_pos[3 * u + 0], start_pos[3 * u + 1], start_pos[3 * u + 2], start_orn[3 * u + 0], start_orn[3 * u + 1],
              start_orn[3 * u + 2]);
  qx_store_any<7, TILED>(st, ist, rows, n, j, s, 0);  // mode 7 touches every PID row
}
__device__ __forceinline__ void fw_reset_drone(const FixedwingParams& p, float* st, int32_t* ist, int64_t n, int64_t j, const float* start_pos,
                                               const float* start_orn, int64_t u) {
  FixedwingRegs s;
  fixedwing_reset(p, s, start_pos[3 * u], start_pos[3 * u + 1], start_pos[3 * u + 2], start_orn[3 * u], start_orn[3 * u + 1],
                  start_orn[3 * u + 2]);
  fixedwing_store(st, ist, n, j, s);
  ist[(int64_t)FI_STEP * n + j] = 0;
}
__device__ __forceinline__ void rk_reset_drone(const RocketParams& p, float* st, int32_t* ist, int64_t n, int64_t j, const float* start_pos,
                                               const float* start_orn, int64_t u) {
  RocketRegs s;
  rocket_reset(p, s, start_pos[3 * u], start_pos[3 * u + 1], start_pos[3 * u + 2], start_orn[3 * u], start_orn[3 * u + 1], start_orn[3 * u + 2]);
  rocket_store(st, ist, n, j, s);
  ist[(int64_t)RI_STEP * n + j] = 0;
}

// ---- base state of the drone in row j from / into drone u's rows of the caller's [N][3] / [N][4] arrays (base_state_set,
// base_state_get: pfb_fixedwing.cuh); nullptr = not given / not wanted.  QuadX: Aviary handles only, so always warp-tiled.
template <typename T>
__device__ __forceinline__ void qx_set_base_drone(float* st, int rows, int64_t j, int64_t u, const double* pos, const double* quat, const T* lin,
                                                  const T* ang) {
  float* rec = st + qx_tile_base(j, rows);
  QuadXRegs s;
  int step_count;
  quadx_load_tile<7, kTileGroupStride>(rec, s, step_count);  // mode 7 moves every PID row
  const F4 pwm = ld_f4(rec + 9 * kTileGroupStride);  // the load leaves the last motor command zero: the store puts it back as it was
  s.pwm[0] = pwm.x; s.pwm[1] = pwm.y; s.pwm[2] = pwm.z; s.pwm[3] = pwm.w;
  base_state_set<T>(s, pos ? pos + 3 * u : nullptr, quat ? quat + 4 * u : nullptr, lin ? lin + 3 * u : nullptr, ang ? ang + 3 * u : nullptr);
  quadx_store_tile<7, kTileGroupStride>(rec, s, step_count);
}
template <typename T>
__device__ __forceinline__ void fw_set_base_drone(float* st, int32_t* ist, int64_t n, int64_t j, int64_t u, const double* pos, const double* quat,
                                                  const T* lin, const T* ang) {
  FixedwingRegs s;
  fixedwing_load(st, ist, n, j, s);
  base_state_set<T>(s, pos ? pos + 3 * u : nullptr, quat ? quat + 4 * u : nullptr, lin ? lin + 3 * u : nullptr, ang ? ang + 3 * u : nullptr);
  fixedwing_store(st, ist, n, j, s);
}
template <typename T>
__device__ __forceinline__ void rk_set_base_drone(float* st, int32_t* ist, int64_t n, int64_t j, int64_t u, const double* pos, const double* quat,
                                                  const T* lin, const T* ang) {
  RocketRegs s;
  rocket_load(st, ist, n, j, s);
  base_state_set<T>(s, pos ? pos + 3 * u : nullptr, quat ? quat + 4 * u : nullptr, lin ? lin + 3 * u : nullptr, ang ? ang + 3 * u : nullptr);
  rocket_store(st, ist, n, j, s);
}
__device__ __forceinline__ void qx_get_base_drone(const float* st, int rows, int64_t j, int64_t u, const BaseStateOut& o) {
  QuadXRegs s;
  int step_count;
  quadx_load_tile<-1, kTileGroupStride>(st + qx_tile_base(j, rows), s, step_count);
  base_state_get(s, o.pos ? o.pos + 3 * u : nullptr, o.quat ? o.quat + 4 * u : nullptr, o.lin ? o.lin + 3 * u : nullptr, o.ang ? o.ang + 3 * u : nullptr);
}
__device__ __forceinline__ void fw_get_base_drone(const float* st, const int32_t* ist, int64_t n, int64_t j, int64_t u, const BaseStateOut& o) {
  FixedwingRegs s;
  fixedwing_load(st, ist, n, j, s);
  base_state_get(s, o.pos ? o.pos + 3 * u : nullptr, o.quat ? o.quat + 4 * u : nullptr, o.lin ? o.lin + 3 * u : nullptr, o.ang ? o.ang + 3 * u : nullptr);
}
__device__ __forceinline__ void rk_get_base_drone(const float* st, const int32_t* ist, int64_t n, int64_t j, int64_t u, const BaseStateOut& o) {
  RocketRegs s;
  rocket_load(st, ist, n, j, s);
  base_state_get(s, o.pos ? o.pos + 3 * u : nullptr, o.quat ? o.quat + 4 * u : nullptr, o.lin ? o.lin + 3 * u : nullptr, o.ang ? o.ang + 3 * u : nullptr);
}
// pfb_set_base_state (fp64) or pfb_set_base_velocity (F32) of the drone in row j of kind KIND's region, drone u's inputs
template <bool F32>
__device__ __forceinline__ void set_base_drone(int kind, const BaseStateIn& a, float* st, int32_t* ist, int rows, int64_t n, int64_t j, int64_t u) {
  if (a.mask && !a.mask[u]) return;
  if constexpr (F32) {
    if (kind == 0) qx_set_base_drone<float>(st, rows, j, u, nullptr, nullptr, a.lin32, a.ang32);
    else if (kind == 1) fw_set_base_drone<float>(st, ist, n, j, u, nullptr, nullptr, a.lin32, a.ang32);
    else rk_set_base_drone<float>(st, ist, n, j, u, nullptr, nullptr, a.lin32, a.ang32);
  } else {
    if (kind == 0) qx_set_base_drone<double>(st, rows, j, u, a.pos, a.quat, a.lin, a.ang);
    else if (kind == 1) fw_set_base_drone<double>(st, ist, n, j, u, a.pos, a.quat, a.lin, a.ang);
    else rk_set_base_drone<double>(st, ist, n, j, u, a.pos, a.quat, a.lin, a.ang);
  }
}

// ---- Aviary.set_mode(modes[j]) of the drone in row j (quadx.py:233-373): preset the setpoint, fresh attitude / position PIDs --
// The other kinds keep their state: a fixed-wing's set_mode zeroes its setpoint (fixedwing.py:224-227), a rocket flies mode 0
// only and its set_mode changes nothing (base_drone.py:252-255).
template <int SP>
__device__ __forceinline__ void qx_set_mode_drone(float* st, int rows, int64_t j, const int8_t* modes, float* setpoint, int64_t u) {
  QuadXRegs s;
  int step_count;
  quadx_load_tile<7, kTileGroupStride>(st + qx_tile_base(j, rows), s, step_count);
  if constexpr (SP == 4) {
    float4 sp = reinterpret_cast<const float4*>(setpoint)[u];
    s.sp[0] = sp.x; s.sp[1] = sp.y; s.sp[2] = sp.z; s.sp[3] = sp.w;
  } else {
    for (int c = 0; c < 4; ++c) s.sp[c] = setpoint[(int64_t)SP * u + c];
  }
  quadx_set_mode_any(s, modes[j]);
  quadx_store_tile<7, kTileGroupStride>(st + qx_tile_base(j, rows), s, step_count);
  if constexpr (SP == 4) {
    reinterpret_cast<float4*>(setpoint)[u] = make_float4(s.sp[0], s.sp[1], s.sp[2], s.sp[3]);
  } else {
    for (int c = 0; c < 4; ++c) setpoint[(int64_t)SP * u + c] = s.sp[c];
  }
}

}  // namespace pfb
