// pfb_rocket.cuh — per-env body of the Rocket stepper (one thread = one rocket = one env).
//
// Replaces (paths under /root/reference/PyFlyt/):
//   core/drones/rocket.py:250-332                    update_control / update_physics / update_state
//   core/abstractions/boosters.py:158-263            ignition latch, throttle lag + noise, fuel burn, variable tank
//   core/abstractions/gimbals.py:145-217             2-axis gimbal, Rodrigues rotation of the thrust axis
//   core/abstractions/lifting_surfaces.py            4 finlets (shared with the fixedwing)
//   core/abstractions/boring_bodies.py:78-127        body drag
//   PyBullet stepSimulation (SURVEY §A.3)            composite body whose mass / COM / inertia change every substep
//   gym_envs/rocket_envs/rocket_landing_env.py:129-263, rocket_base_env.py:166-370   Rocket-Landing epilogue
#pragma once

#include "pfb_fixedwing.cuh"

namespace pfb {

struct RocketParams {
  float dt, gravity, vmax;
  int ratio;
  // composite without the fuel tank link + the tank at full load (boosters.py:207-212 rescales it)
  float dry_mass, dry_mc[3], dry_I[9];
  float fuel_total_mass, fuel_pos[3], fuel_max_inertia[3];
  float body_r[3], drag_k[3];
  int n_surfaces;
  SurfaceParams surf[4];
  float booster_r[3], booster_axis[3];
  float booster_lag, booster_noise, booster_min_ratio, booster_max_thrust, fuel_rate;  // fuel_rate = max_fuel_rate / total_fuel
  int reignitable;
  float gimbal_u1[3], gimbal_u2[3], gimbal_lag, gimbal_range[2];
  float start_fuel;
  float noise_loc;
  ContactParams contact;
  WindParams wind;  // analytic wind field; kind 0 = still air
  int contact_response;  // 1: ground / pad contact impulses (PfbEnvConfig.contact_response), 0: contact flag only
};

struct LandingParams {
  int env_step_ratio, max_steps, angle_representation, sparse_reward, warmup_steps;
  int randomize_drop, accelerate_drop;
  float ceiling, max_displacement;
};

enum {
  RK_POS = 0, RK_QUAT = 3, RK_VEL = 7, RK_ANGVEL = 10, RK_ACT = 13 /*4 finlets*/, RK_IGN = 17, RK_FUEL = 18, RK_THR = 19, RK_GIMBAL = 20 /*2*/,
  RK_POS_LO = 22, RK_QUAT_LO = 25, RK_VEL_LO = 29, RK_ROWS = 32
};
enum { RI_STEP = 0, RI_FLAGS = 1, RI_ROWS = 2 };
enum { FLAG_CONTACT_PAD = 128, FLAG_CONTACT_GROUND = 256, FLAG_PAD_OBS = 512 /* landing_pad_contact */ };
constexpr float kPadRadius = 2.0f, kPadTop = 0.15f;  // models/landing_pad.urdf:5-9 at z = 0.1

struct RocketRegs {
  xreal px, py, pz;
  qreal qx, qy, qz, qw;
  vreal vx, vy, vz;
  float wx, wy, wz;
  float act[4];
  float ign, fuel, thr;
  float gim[2];
  float sp[7];
  Rot<rreal> R;
  Vec3 vb;
  uint32_t flags;
};

// Rodrigues rotation of v about unit axis k by angle a: gimbals.py:178-217 (I + sin a W + 2 sin^2(a/2) W^2)
PFB_HD Vec3 rodrigues(Vec3 k, float a, Vec3 v) {
  float sn, cs;
  sincos_f(a, sn, cs);
  Vec3 kv = cross(k, v);
  Vec3 kkv = cross(k, kv);
  return v + sn * kv + (1.0f - cs) * kkv;
}

// symmetric 3x3 solve J x = b by cofactors (J = inertia about the instantaneous COM)
PFB_HD Vec3 solve_sym3(float a, float b, float c, float d, float e, float f, Vec3 r) {
  // J = [[a b c], [b d e], [c e f]]
  float c00 = d * f - e * e, c01 = c * e - b * f, c02 = b * e - c * d;
  float c11 = a * f - c * c, c12 = b * c - a * e, c22 = a * d - b * b;
  float inv = fast_rcp(a * c00 + b * c01 + c * c02);
  return Vec3{(c00 * r.x + c01 * r.y + c02 * r.z) * inv, (c01 * r.x + c11 * r.y + c12 * r.z) * inv, (c02 * r.x + c12 * r.y + c22 * r.z) * inv};
}

// rocket.py:250-278: finlet mixing (rocket.py:152-159) + clip; the rest of the setpoint passes through
PFB_HD void rocket_command(const RocketRegs& s, float* cmd) {
  cmd[0] = clampf(s.sp[1] + s.sp[2], -1.0f, 1.0f);
  cmd[1] = clampf(s.sp[1] - s.sp[2], -1.0f, 1.0f);
  cmd[2] = clampf(s.sp[0] - s.sp[2], -1.0f, 1.0f);
  cmd[3] = clampf(s.sp[0] + s.sp[2], -1.0f, 1.0f);
  cmd[4] = s.sp[3]; cmd[5] = s.sp[4]; cmd[6] = s.sp[5]; cmd[7] = s.sp[6];
}

// one physics substep: update_physics (rocket.py:280-298) + stepSimulation + update_state
// World: NoStatic, StaticCtx or SolidCtx (Aviary handles, with_pad = false), as in quadx_substep.
template <class World = NoStatic>
PFB_HD void rocket_substep(const RocketParams& p, RocketRegs& s, const float* cmd, float xi, bool with_pad, World* world = nullptr) {
  Vec3 F = Vec3{0.f, 0.f, 0.f}, T = Vec3{0.f, 0.f, 0.f};
  const Vec3 w = Vec3{s.wx, s.wy, s.wz};
  const bool windy = p.wind.kind != 0;  // uniform: the parameter block is launch-constant
  WindCtx wc = WindCtx{Vec3{0.f, 0.f, 0.f}, 0.f, 0.f, 0.f, 0.f};
  if (windy) wc = wind_ctx(p.wind, (float)s.pz, (float)s.R.m00, (float)s.R.m01, (float)s.R.m02, (float)s.R.m10, (float)s.R.m11, (float)s.R.m12,
                           (float)s.R.m20, (float)s.R.m21, (float)s.R.m22);
  // body drag (boring_bodies.py:113-127) on the body link, on the velocity through the air (boring_bodies.py:93-96)
  {
    Vec3 r = Vec3{p.body_r[0], p.body_r[1], p.body_r[2]};
    Vec3 v = s.vb + cross(w, r);
    if (windy) v = v - wind_body_at(p.wind, wc, p.body_r[0], p.body_r[1], p.body_r[2]);
    Vec3 Fd = Vec3{-p.drag_k[0] * signed_square(v.x), -p.drag_k[1] * signed_square(v.y), -p.drag_k[2] * signed_square(v.z)};
    F = F + Fd;
    T = T + cross(r, Fd);
  }
  // finlets
  // fully unrolled (4 finlets): independent until summed, and ILP is the only latency hiding at 16 384 envs
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (i < p.n_surfaces) surface_force(p.surf[i], s.act[i], cmd[i], s.vb, w, F, T, windy ? &p.wind : nullptr, &wc);
  }
  // gimbal (gimbals.py:145-176): lag on both axes, thrust axis = R1 (R2 u)
  s.gim[0] = fmaf(p.gimbal_lag, cmd[6] - s.gim[0], s.gim[0]);
  s.gim[1] = fmaf(p.gimbal_lag, cmd[7] - s.gim[1], s.gim[1]);
  Vec3 unit = Vec3{p.booster_axis[0], p.booster_axis[1], p.booster_axis[2]};
  unit = rodrigues(Vec3{p.gimbal_u2[0], p.gimbal_u2[1], p.gimbal_u2[2]}, s.gim[1] * p.gimbal_range[1], unit);
  unit = rodrigues(Vec3{p.gimbal_u1[0], p.gimbal_u1[1], p.gimbal_u1[2]}, s.gim[0] * p.gimbal_range[0], unit);
  // booster (boosters.py:214-263): ignition latch, target throttle, lag, noise, fuel cut-off, fuel burn
  {
    bool latched = (!p.reignitable) && (s.ign != 0.0f);
    s.ign = (latched || cmd[4] > 0.5f) ? 1.0f : 0.0f;
    float target = s.ign * fmaf(cmd[5], 1.0f - p.booster_min_ratio, p.booster_min_ratio);
    float t = fmaf(p.booster_lag, target - s.thr, s.thr);
    t = fmaf(xi * p.booster_noise, t, t);
    t = s.fuel > 0.0f ? t : 0.0f;
    s.thr = t;
    s.fuel = clampf(s.fuel - t * p.fuel_rate * p.dt, 0.0f, 1.0f);
    float thrust = t * p.booster_max_thrust;
    Vec3 Fb = thrust * unit;
    Vec3 rb = Vec3{p.booster_r[0], p.booster_r[1], p.booster_r[2]};
    F = F + Fb;
    T = T + cross(rb, Fb);
  }
  // contacts from the pose at the start of the step: ground plane everywhere, landing pad under the base
  bool touching = false, over_pad = false;
  float top = 0.0f;  // static bodies: the surface height under the drone
  const float pz0 = (float)s.pz;  // altitude at the START of the substep (the contact solver's pose)
  [[maybe_unused]] uint32_t live = 0u;  // SolidCtx: the primitives within reach of the base
  if constexpr (World::kSolid) {
    live = solid_live(*world->w, world->pose, world->n, world->i, (float)s.px, (float)s.py, pz0, p.contact.zmax);
    uint32_t b = ground_contact(p.contact, pz0, (float)s.R.m20, (float)s.R.m21, (float)s.R.m22, 0.0f) ? 1u : 0u;
    if (live) b |= solid_bits(world->w, world->pose, world->n, world->i, live, &p.contact, solid_base(s));
    world->bits |= b;
    touching = b != 0u;
    s.flags = (s.flags & ~(uint32_t)FLAG_CONTACT_PREV) | (touching ? (FLAG_CONTACT_PREV | FLAG_CONTACT_ARRAY) : 0u) |
              ((b & 1u) ? FLAG_CONTACT_GROUND : 0u);
  } else if constexpr (World::kOn) {
    const float pz = (float)s.pz, r20 = (float)s.R.m20, r21 = (float)s.R.m21, r22 = (float)s.R.m22;
    uint32_t b;
    top = static_surface(*world->w, world->pose, world->n, world->i, (float)s.px, (float)s.py, pz, p.contact.zmax,
                         [&](float t) { return ground_contact(p.contact, pz, r20, r21, r22, t); }, b);
    world->bits |= b;
    touching = b != 0u;
    s.flags = (s.flags & ~(uint32_t)FLAG_CONTACT_PREV) | (touching ? (FLAG_CONTACT_PREV | FLAG_CONTACT_ARRAY) : 0u) |
              ((b & 1u) ? FLAG_CONTACT_GROUND : 0u);
  } else {
    const float pz = (float)s.pz, r20 = (float)s.R.m20, r21 = (float)s.R.m21, r22 = (float)s.R.m22;
    bool g = ground_contact(p.contact, pz, r20, r21, r22, 0.0f);
    bool pad = false;
    if (with_pad) {
      float px = (float)s.px, py = (float)s.py;
      over_pad = px * px + py * py <= kPadRadius * kPadRadius;
      if (over_pad) pad = ground_contact(p.contact, pz, r20, r21, r22, kPadTop);
    }
    touching = g || pad;
    s.flags = (s.flags & ~(uint32_t)FLAG_CONTACT_PREV) | ((g || pad) ? (FLAG_CONTACT_PREV | FLAG_CONTACT_ARRAY) : 0u) |
              (g ? FLAG_CONTACT_GROUND : 0u) | (pad ? FLAG_CONTACT_PAD : 0u);
  }
  // composite body with the fuel left AFTER this substep's burn (changeDynamics precedes stepSimulation)
  const float mf = s.fuel * p.fuel_total_mass;
  const float M = p.dry_mass + mf;
  const float inv_M = fast_rcp(M);
  Vec3 mc = Vec3{p.dry_mc[0] + mf * p.fuel_pos[0], p.dry_mc[1] + mf * p.fuel_pos[1], p.dry_mc[2] + mf * p.fuel_pos[2]};
  Vec3 c = inv_M * mc;
  const float fr2 = p.fuel_pos[0] * p.fuel_pos[0] + p.fuel_pos[1] * p.fuel_pos[1] + p.fuel_pos[2] * p.fuel_pos[2];
  // I_O (about the base origin)
  float Ixx = p.dry_I[0] + s.fuel * p.fuel_max_inertia[0] + mf * (fr2 - p.fuel_pos[0] * p.fuel_pos[0]);
  float Iyy = p.dry_I[4] + s.fuel * p.fuel_max_inertia[1] + mf * (fr2 - p.fuel_pos[1] * p.fuel_pos[1]);
  float Izz = p.dry_I[8] + s.fuel * p.fuel_max_inertia[2] + mf * (fr2 - p.fuel_pos[2] * p.fuel_pos[2]);
  float Ixy = p.dry_I[1] - mf * p.fuel_pos[0] * p.fuel_pos[1];
  float Ixz = p.dry_I[2] - mf * p.fuel_pos[0] * p.fuel_pos[2];
  float Iyz = p.dry_I[5] - mf * p.fuel_pos[1] * p.fuel_pos[2];
  // gravity at the COM, Newton-Euler about O:  F' = F - M w x (w x c),  T' = T - w x (I_O w)
  const Rot<rreal>& R = s.R;
  Vec3 gb = Vec3{p.gravity * (float)R.m20, p.gravity * (float)R.m21, p.gravity * (float)R.m22};
  F = F + M * gb;
  T = T + cross(mc, gb);
  Vec3 Iw = Vec3{Ixx * w.x + Ixy * w.y + Ixz * w.z, Ixy * w.x + Iyy * w.y + Iyz * w.z, Ixz * w.x + Iyz * w.y + Izz * w.z};
  Vec3 Fp = F - cross(w, cross(w, mc));
  Vec3 Tp = T - cross(w, Iw);
  // J = I_O - M (|c|^2 E - c c^T) (inertia about the COM):  J wdot = T' - c x F',  a_O = F'/M + c x wdot
  float c2 = dot(c, c);
  Vec3 wdot = solve_sym3(Ixx - M * (c2 - c.x * c.x), Ixy + M * c.x * c.y, Ixz + M * c.x * c.z, Iyy - M * (c2 - c.y * c.y),
                         Iyz + M * c.y * c.z, Izz - M * (c2 - c.z * c.z), Tp - cross(c, Fp));
  Vec3 aO = inv_M * Fp + cross(c, wdot);
  // semi-implicit Euler + exp-map (same state update as rigid_step, accelerations supplied directly)
  rreal ax = R.m00 * (rreal)aO.x + R.m01 * (rreal)aO.y + R.m02 * (rreal)aO.z;
  rreal ay = R.m10 * (rreal)aO.x + R.m11 * (rreal)aO.y + R.m12 * (rreal)aO.z;
  rreal az = R.m20 * (rreal)aO.x + R.m21 * (rreal)aO.y + R.m22 * (rreal)aO.z;
  const vreal dt = (vreal)p.dt;
  s.vx += (vreal)ax * dt; s.vy += (vreal)ay * dt; s.vz += (vreal)az * dt;
  if (fmaxf(fmaxf(fabsf((float)s.vx), fabsf((float)s.vy)), fabsf((float)s.vz)) >= p.vmax) {
    const vreal vmax = (vreal)p.vmax;
    s.vx = fmin(fmax(s.vx, -vmax), vmax); s.vy = fmin(fmax(s.vy, -vmax), vmax); s.vz = fmin(fmax(s.vz, -vmax), vmax);
  }
  s.wx = fmaf(wdot.x, p.dt, s.wx); s.wy = fmaf(wdot.y, p.dt, s.wy); s.wz = fmaf(wdot.z, p.dt, s.wz);
  if (fmaxf(fmaxf(fabsf(s.wx), fabsf(s.wy)), fabsf(s.wz)) > p.vmax * 0.57735f) {
    Mat3 Rf{(float)R.m00, (float)R.m01, (float)R.m02, (float)R.m10, (float)R.m11, (float)R.m12, (float)R.m20, (float)R.m21, (float)R.m22};
    Vec3 wc = quadx_clamp_world_rates(p.vmax, Rf, Vec3{s.wx, s.wy, s.wz});
    s.wx = wc.x; s.wy = wc.y; s.wz = wc.z;
  }
  if constexpr (World::kSolid) {
    if (p.contact_response && touching)
      apply_solid_impulses(&p.contact, s, *world, live, M, c, Ixx - M * (c2 - c.x * c.x), Ixy + M * c.x * c.y, Ixz + M * c.x * c.z,
                           Iyy - M * (c2 - c.y * c.y), Iyz + M * c.y * c.z, Izz - M * (c2 - c.z * c.z), p.dt);
  } else if (p.contact_response && touching)  // contact impulses on the predicted velocities, before the pose is integrated (cold path)
    apply_contact_impulses<World>(&p.contact, s, pz0, World::kOn ? top : (over_pad ? kPadTop : 0.0f), M, c, Ixx - M * (c2 - c.x * c.x), Ixy + M * c.x * c.y, Ixz + M * c.x * c.z,
                           Iyy - M * (c2 - c.y * c.y), Iyz + M * c.y * c.z, Izz - M * (c2 - c.z * c.z), p.dt);
  s.px += (xreal)(s.vx * dt); s.py += (xreal)(s.vy * dt); s.pz += (xreal)(s.vz * dt);
  float h2 = (s.wx * s.wx + s.wy * s.wy + s.wz * s.wz) * (0.25f * p.dt * p.dt);
  float sinc = fmaf(h2, fmaf(h2, fmaf(h2, fmaf(h2, 2.7557319e-6f, -1.9841270e-4f), 8.3333333e-3f), -1.6666667e-1f), 1.0f);
  float scale = 0.5f * p.dt * sinc;
  float cw = fmaf(h2, fmaf(h2, fmaf(h2, fmaf(h2, fmaf(h2, -2.7557319e-7f, 2.4801587e-5f), -1.3888889e-3f), 4.1666667e-2f), -0.5f), 1.0f);
  qreal dx = (qreal)(s.wx * scale), dy = (qreal)(s.wy * scale), dz = (qreal)(s.wz * scale), dw = (qreal)cw;
  qreal nx = s.qw * dx + s.qx * dw + s.qy * dz - s.qz * dy;
  qreal ny = s.qw * dy + s.qy * dw + s.qz * dx - s.qx * dz;
  qreal nz = s.qw * dz + s.qz * dw + s.qx * dy - s.qy * dx;
  qreal nw = s.qw * dw - s.qx * dx - s.qy * dy - s.qz * dz;
  qreal n2 = nx * nx + ny * ny + nz * nz + nw * nw;
#if PFB_Q_DOUBLE
  qreal e = n2 - 1.0;
  qreal inv = 1.0 - 0.5 * e + 0.375 * e * e;
#else
  qreal inv = 1.0f / sqrtf(n2);
#endif
  s.qx = nx * inv; s.qy = ny * inv; s.qz = nz * inv; s.qw = nw * inv;
  body_update_state(s);
}

template <typename NoiseFn, class World = NoStatic>
PFB_HD void rocket_aviary_step(const RocketParams& p, RocketRegs& s, NoiseFn& noise, bool with_pad, World* world = nullptr) {
  s.flags &= ~(uint32_t)(FLAG_CONTACT_ARRAY | FLAG_CONTACT_PAD | FLAG_CONTACT_GROUND);
  if constexpr (World::kOn) world->bits = 0u;
  noise.begin_step();
  float cmd[8];
  rocket_command(s, cmd);
#pragma unroll 1
  for (int u = 0; u < p.ratio; ++u) rocket_substep(p, s, cmd, noise.get(u), with_pad, world);
}
// rocket_aviary_step (no pad) inside an Aviary step of U substeps at several control rates: rocket_command runs before
// substep u when u % r == 0 (r = physics_hz / control_hz of this drone, a divisor of U); draw u of the step.  r == U: the above.
template <typename NoiseFn, class World = NoStatic>
PFB_HD void rocket_aviary_step_rates(const RocketParams& p, RocketRegs& s, int r, int U, NoiseFn& noise, World* world = nullptr) {
  s.flags &= ~(uint32_t)(FLAG_CONTACT_ARRAY | FLAG_CONTACT_PAD | FLAG_CONTACT_GROUND);
  if constexpr (World::kOn) world->bits = 0u;
  noise.begin_step();
  float cmd[8];
#pragma unroll 1
  for (int u = 0; u < U; ++u) {
    if (u % r == 0) rocket_command(s, cmd);
    rocket_substep(p, s, cmd, noise.get(u), false, world);
  }
}

// rocket.py:226-239 + aviary.py:310-311
PFB_HD void rocket_reset(const RocketParams& p, RocketRegs& s, float sx, float sy, float sz, float roll, float pitch, float yaw) {
  s.px = (xreal)sx; s.py = (xreal)sy; s.pz = (xreal)sz;
  {
    qreal hr = (qreal)roll * (qreal)0.5, hp = (qreal)pitch * (qreal)0.5, hy = (qreal)yaw * (qreal)0.5;
    qreal sr = sin(hr), cr = cos(hr), sp = sin(hp), cp = cos(hp), sy_ = sin(hy), cy = cos(hy);
    s.qx = sr * cp * cy - cr * sp * sy_;
    s.qy = cr * sp * cy + sr * cp * sy_;
    s.qz = cr * cp * sy_ - sr * sp * cy;
    s.qw = cr * cp * cy + sr * sp * sy_;
  }
  s.vx = s.vy = s.vz = (vreal)0;
  s.wx = s.wy = s.wz = 0.0f;
#pragma unroll
  for (int k = 0; k < 4; ++k) s.act[k] = 0.0f;
  s.ign = 0.0f; s.fuel = p.start_fuel; s.thr = 0.0f;
  s.gim[0] = s.gim[1] = 0.0f;
#pragma unroll
  for (int k = 0; k < 7; ++k) s.sp[k] = 0.0f;
  s.flags = 0u;
  body_update_state(s);
}

// `st` is field-major [F][N] by default; `rs` / `ci` select an env-major record instead (row stride 1, base already at the
// env's record): the spare post-reset states of the Landing env (pfb_rocket.cu)
PFB_HD void rocket_load(const float* __restrict__ st, const int32_t* __restrict__ ist, int64_t N, int64_t i, RocketRegs& s,
                        int64_t rs = -1, int64_t ci = -1) {
  if (rs < 0) { rs = N; ci = i; }
  auto F = [&](int row) { return st[(int64_t)row * rs + ci]; };
  s.px = join_hi_lo(F(RK_POS + 0), F(RK_POS_LO + 0));
  s.py = join_hi_lo(F(RK_POS + 1), F(RK_POS_LO + 1));
  s.pz = join_hi_lo(F(RK_POS + 2), F(RK_POS_LO + 2));
  s.qx = join_hi_lo(F(RK_QUAT + 0), F(RK_QUAT_LO + 0));
  s.qy = join_hi_lo(F(RK_QUAT + 1), F(RK_QUAT_LO + 1));
  s.qz = join_hi_lo(F(RK_QUAT + 2), F(RK_QUAT_LO + 2));
  s.qw = join_hi_lo(F(RK_QUAT + 3), F(RK_QUAT_LO + 3));
  s.vx = join_hi_lo(F(RK_VEL + 0), F(RK_VEL_LO + 0));
  s.vy = join_hi_lo(F(RK_VEL + 1), F(RK_VEL_LO + 1));
  s.vz = join_hi_lo(F(RK_VEL + 2), F(RK_VEL_LO + 2));
  s.wx = F(RK_ANGVEL + 0); s.wy = F(RK_ANGVEL + 1); s.wz = F(RK_ANGVEL + 2);
#pragma unroll
  for (int k = 0; k < 4; ++k) s.act[k] = F(RK_ACT + k);
  s.ign = F(RK_IGN); s.fuel = F(RK_FUEL); s.thr = F(RK_THR);
  s.gim[0] = F(RK_GIMBAL); s.gim[1] = F(RK_GIMBAL + 1);
  s.flags = (uint32_t)ist[(int64_t)RI_FLAGS * N + i];
  body_update_state(s);
}

PFB_HD void rocket_store(float* __restrict__ st, int32_t* __restrict__ ist, int64_t N, int64_t i, const RocketRegs& s,
                         bool with_flags = true, int64_t rs = -1, int64_t ci = -1) {
  if (rs < 0) { rs = N; ci = i; }
  auto S = [&](int row, float v) { st[(int64_t)row * rs + ci] = v; };
  float hi, lo;
  split_hi_lo(s.px, hi, lo); S(RK_POS + 0, hi); S(RK_POS_LO + 0, lo);
  split_hi_lo(s.py, hi, lo); S(RK_POS + 1, hi); S(RK_POS_LO + 1, lo);
  split_hi_lo(s.pz, hi, lo); S(RK_POS + 2, hi); S(RK_POS_LO + 2, lo);
  split_hi_lo(s.qx, hi, lo); S(RK_QUAT + 0, hi); S(RK_QUAT_LO + 0, lo);
  split_hi_lo(s.qy, hi, lo); S(RK_QUAT + 1, hi); S(RK_QUAT_LO + 1, lo);
  split_hi_lo(s.qz, hi, lo); S(RK_QUAT + 2, hi); S(RK_QUAT_LO + 2, lo);
  split_hi_lo(s.qw, hi, lo); S(RK_QUAT + 3, hi); S(RK_QUAT_LO + 3, lo);
  split_hi_lo(s.vx, hi, lo); S(RK_VEL + 0, hi); S(RK_VEL_LO + 0, lo);
  split_hi_lo(s.vy, hi, lo); S(RK_VEL + 1, hi); S(RK_VEL_LO + 1, lo);
  split_hi_lo(s.vz, hi, lo); S(RK_VEL + 2, hi); S(RK_VEL_LO + 2, lo);
  S(RK_ANGVEL + 0, s.wx); S(RK_ANGVEL + 1, s.wy); S(RK_ANGVEL + 2, s.wz);
#pragma unroll
  for (int k = 0; k < 4; ++k) S(RK_ACT + k, s.act[k]);
  S(RK_IGN, s.ign); S(RK_FUEL, s.fuel); S(RK_THR, s.thr);
  S(RK_GIMBAL, s.gim[0]); S(RK_GIMBAL + 1, s.gim[1]);
  if (with_flags) ist[(int64_t)RI_FLAGS * N + i] = (int32_t)s.flags;
}

// Round the fp64-carried fields to what the state tensor holds (hi + lo fp32 words) and re-derive the body-frame state
PFB_HD void rocket_requantize(RocketRegs& s) {
  float hi, lo;
  split_hi_lo(s.px, hi, lo); s.px = join_hi_lo(hi, lo);
  split_hi_lo(s.py, hi, lo); s.py = join_hi_lo(hi, lo);
  split_hi_lo(s.pz, hi, lo); s.pz = join_hi_lo(hi, lo);
  split_hi_lo(s.qx, hi, lo); s.qx = join_hi_lo(hi, lo);
  split_hi_lo(s.qy, hi, lo); s.qy = join_hi_lo(hi, lo);
  split_hi_lo(s.qz, hi, lo); s.qz = join_hi_lo(hi, lo);
  split_hi_lo(s.qw, hi, lo); s.qw = join_hi_lo(hi, lo);
  split_hi_lo(s.vx, hi, lo); s.vx = join_hi_lo(hi, lo);
  split_hi_lo(s.vy, hi, lo); s.vy = join_hi_lo(hi, lo);
  split_hi_lo(s.vz, hi, lo); s.vz = join_hi_lo(hi, lo);
  body_update_state(s);
}

// Aviary.state(i) (4,3) + aux_state (rocket.py:324-332): finlets x4, ignition, fuel, throttle, gimbal x2
PFB_HD void rocket_drone_state(const RocketRegs& s, float* out12, float* aux9) {
  float roll, pitch, yaw;
  euler_from_quat((float)s.qx, (float)s.qy, (float)s.qz, (float)s.qw, roll, pitch, yaw);
  out12[0] = s.wx; out12[1] = s.wy; out12[2] = s.wz;
  out12[3] = roll; out12[4] = pitch; out12[5] = yaw;
  out12[6] = s.vb.x; out12[7] = s.vb.y; out12[8] = s.vb.z;
  out12[9] = (float)s.px; out12[10] = (float)s.py; out12[11] = (float)s.pz;
#pragma unroll
  for (int k = 0; k < 4; ++k) aux9[k] = s.act[k];
  aux9[4] = s.ign; aux9[5] = s.fuel; aux9[6] = s.thr; aux9[7] = s.gim[0]; aux9[8] = s.gim[1];
}

}  // namespace pfb
