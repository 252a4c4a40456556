// pfb_quadx.cuh — per-env body of the QuadX stepper (one thread = one drone = one env).
//
// Replaces, for N independent single-drone worlds (paths under /root/reference/PyFlyt/):
//   core/aviary.py:506-531                 Aviary.step() substep loop
//   core/drones/quadx.py:401-535           update_control / update_physics / update_state
//   core/abstractions/motors.py:110-195    throttle lag + noise + rpm^2 thrust/torque
//   core/abstractions/boring_bodies.py:78-127   quadratic body drag
//   core/abstractions/pid.py:70-94         PID
//   PyBullet stepSimulation (SURVEY §A.3)  free rigid body, semi-implicit Euler, exp-map quaternion
//   gym_envs/quadx_envs/quadx_hover_env.py:85-138 + quadx_base_env.py:251-301  Hover epilogue
//
// Formulation notes (DESIGN.md §kernel):
//  * Angular velocity is carried in the BODY frame.  Bullet integrates w_world += R wdot_b dt and
//    then q <- dq(w_world dt) * q; because a rotation about w leaves w invariant, the new body-frame
//    rate is exactly w_b + wdot_b dt and dq(w_world dt) * q == q * dq(w_b dt).  The world-frame
//    +-100 rad/s coordinate clamp is applied on a rarely-taken slow path.
//  * Forces are evaluated from the state of the previous update_state (explicit), positions use the
//    NEW velocities (semi-implicit), exactly like the reference.
#pragma once

#include <string.h>

#include "pfb_common.cuh"

namespace pfb {

// fp32 coefficient table, passed BY VALUE as a __grid_constant__ kernel parameter: it lives in the
// constant bank and its fields are used directly as FFMA operands (no shared-memory staging needed
// for uniformly-accessed scalars).
struct QuadXParams {
  float dt;            // 1 / physics_hz
  float ctrl_dt;       // 1 / control_hz
  float inv_ctrl_dt;
  float inv_mass;
  float gravity;       // -9.81
  float vmax;          // 100: btMultiBody max coordinate velocity
  float Ixx, Iyy, Izz;
  float inv_Ixx, inv_Iyy, inv_Izz;
  float motor_x[4], motor_y[4];
  float thrust_k[4];   // thrust_coef * max_rpm^2
  float torque_k[4];   // torque_coef * max_rpm^2 (signed)
  float motor_lag;     // physics_period / tau
  float noise_ratio;
  float noise_loc;     // n_motors: the reference's normal(*shape) quirk, SURVEY §A.4
  float drag_k[3];
  float drag_pqr;
  // PID: [which][kp, ki*T, kd/T, lim][axis]; which = 0 ang_vel 1 ang_pos 2 lin_vel 3 lin_pos 4 z_vel 5 z_pos
  float pid[6][4][3];
  // ground-contact primitives (identity orientation in the body frame)
  int n_shapes;
  int shape_kind[5];
  float shape_dims[5][3];
  float shape_at[5][3];
  float shape_thr[5];
  float contact_zmax;  // base altitude above which no primitive can be within its contact threshold
  int ratio;           // physics substeps per control tick (physics_hz / control_hz)
  WindParams wind;     // analytic wind field; kind 0 = still air
};

struct HoverParams {
  int env_step_ratio;
  int max_steps;
  int angle_representation;  // 0 euler (obs 20), 1 quaternion (obs 21)
  int sparse_reward;
  int warmup_steps;
  int flight_mode;
  float dome2;  // flight_dome_size squared (inf stays inf)
  int ma;       // 1: MAQuadXHover per-agent epilogue (pz_envs/quadx_envs/ma_quadx_hover_env.py)
};

// QuadX-Waypoints constants (gym_envs/quadx_envs/quadx_waypoints_env.py:38-52, utils/waypoint_handler.py)
struct QxWaypointParams {
  int env_step_ratio, max_steps, sparse_reward, warmup_steps;
  int num_targets, use_yaw_targets;
  float dome2, dome, goal_reach_distance, goal_reach_angle, min_height;
};

// PID memory rows inside the state tensor (24 words)
enum { PID_P0 = 0, PID_P1 = 6, PID_P2 = 12, PID_P3 = 16, PID_ZV = 20, PID_ZP = 22, PID_WORDS = 24 };

// QuadX state rows.  Row r is one fp32 word per env.  The row order groups the words a mode-0 env step touches into the
// first 36 rows so that, in the warp-tiled layout (below), they are 9 consecutive 16-byte groups per env.
enum {
  QX_POS = 0,       // 3  position (hi)
  QX_QUAT = 3,      // 4  quaternion x,y,z,w (hi)
  QX_VEL = 7,       // 3  world linear velocity (hi)
  QX_ANGVEL = 10,   // 3  BODY angular velocity
  QX_THR = 13,      // 4  motor throttle (aux_state)
  QX_STEP = 17,     // 1  env step_count, int32 bits   (warp-tiled layout only; the field-major layout keeps it in istate)
  QX_FLAGS = 18,    // 1  flag word, uint32 bits       (same)
  QX_PID0 = 19,     // 6  ang_vel PID: integrals, previous errors
  QX_POS_LO = 25,   // 3
  QX_QUAT_LO = 28,  // 4
  QX_VEL_LO = 32,   // 3  (+ 1 pad word)
  QX_PWM = 36,      // 4  last motor command
  QX_PID1 = 40,     // 18 remaining PID words (ang_pos 6, lin_vel 4, lin_pos 4, z_vel 2, z_pos 2) (+ 2 pad words)
  QX_ROWS = 60
};
// PID word k (0..23, the PID_* offsets above) -> state row
PFB_HD constexpr int qx_pid_row(int k) { return k < 6 ? QX_PID0 + k : QX_PID1 + (k - 6); }

// ---- warp-tiled layout (QuadX-Hover, MAQuadXHover and Aviary-level QuadX handles) ---------------------------------------
// Env i lives in tile i >> 5, lane i & 31.  A tile is G = rows / 4 groups; group g holds rows 4g .. 4g+3 of the tile's 32
// envs as 32 consecutive 16-byte vectors:  word(row r, env i) = st[(((i >> 5) * G + (r >> 2)) * 32 + (i & 31)) * 4 + (r & 3)].
// A warp therefore moves a group with ONE 128-bit access per lane (512 contiguous bytes), every address is the lane's
// record pointer plus an immediate, and the rows a mode touches are one contiguous block of the tile.
// An env-major record (the spare post-reset states) is the same row order with the groups back to back (group stride 4).
constexpr int kTileLanes = 32;
constexpr int kTileGroupStride = kTileLanes * 4;  // floats between consecutive groups of one lane inside a tile
struct alignas(16) F4 { float x, y, z, w; };
PFB_HD F4 ld_f4(const float* p) { return *reinterpret_cast<const F4*>(p); }
PFB_HD void st_f4(float* p, float x, float y, float z, float w) { *reinterpret_cast<F4*>(p) = F4{x, y, z, w}; }
PFB_HD int64_t qx_tile_floats(int rows) { return (int64_t)(rows / 4) * kTileGroupStride; }
// pointer to the first group word of env i (lane record base)
PFB_HD int64_t qx_tile_base(int64_t i, int rows) { return (i >> 5) * qx_tile_floats(rows) + (i & 31) * 4; }
// address of a single word (slow path: accessors, extra rows)
PFB_HD int64_t qx_tile_word(int64_t i, int rows, int r) { return qx_tile_base(i, rows) + (int64_t)(r >> 2) * kTileGroupStride + (r & 3); }
// istate rows [I][N]
enum { QI_STEP = 0, QI_FLAGS = 1, QI_ROWS = 2 };
enum { FLAG_TERM = 1, FLAG_TRUNC = 2, FLAG_OOB = 4, FLAG_COLLISION = 8, FLAG_CONTACT_PREV = 16, FLAG_CONTACT_ARRAY = 32 };
// In-launch autoreset: a tail CTA that resets an env on launch k tags the new episode with FLAG_FRESH0 << (k & 1).  The
// env's regular thread of the SAME launch may read the flags before or after the tail CTA rewrote them (a later wave of
// a large grid): it stands down on TERM/TRUNC (not yet rewritten) and on this launch's tag (already rewritten).  The
// tag of the other parity is from the previous launch and is cleared by the regular thread's store.
enum { FLAG_FRESH0 = 1 << 14, FLAG_FRESH1 = 1 << 15, FLAG_FRESH_ANY = FLAG_FRESH0 | FLAG_FRESH1 };
PFB_HD uint32_t fresh_tag(uint32_t step_seq) { return (uint32_t)FLAG_FRESH0 << (step_seq & 1u); }

template <typename T>
struct Rot {
  T m00, m01, m02, m10, m11, m12, m20, m21, m22;
};

#if PFB_R_DOUBLE
typedef double rreal;
#else
typedef float rreal;
#endif
#if PFB_FW_R_DOUBLE
typedef double fwreal;
#else
typedef float fwreal;
#endif

struct QuadXRegs {
  xreal px, py, pz;
  qreal qx, qy, qz, qw;
  vreal vx, vy, vz;   // world
  float wx, wy, wz;   // body
  float thr[4];
  float pwm[4];
  float pid[PID_WORDS];
  float sp[4];        // setpoint
  // derived by update_state
  Rot<rreal> R;
  Vec3 vb;            // body-frame linear velocity
  uint32_t flags;
};

// p.getMatrixFromQuaternion for a unit quaternion (|q|^2 - 1 ~ 1e-16 after normalisation)
template <typename T, typename Q>
PFB_HD void rot_from_quat(Q x, Q y, Q z, Q w, Rot<T>& R) {
  T X = (T)x, Y = (T)y, Z = (T)z, W = (T)w;
  T xs = X + X, ys = Y + Y, zs = Z + Z;
  T wx = W * xs, wy = W * ys, wz = W * zs;
  T xx = X * xs, xy = X * ys, xz = X * zs;
  T yy = Y * ys, yz = Y * zs, zz = Z * zs;
  R.m00 = (T)1 - (yy + zz); R.m01 = xy - wz; R.m02 = xz + wy;
  R.m10 = xy + wz; R.m11 = (T)1 - (xx + zz); R.m12 = yz - wx;
  R.m20 = xz - wy; R.m21 = yz + wx; R.m22 = (T)1 - (xx + yy);
}

// quadx.py:512-535: body-frame velocities from the world state
PFB_HD void quadx_update_state(QuadXRegs& s) {
  rot_from_quat<rreal>(s.qx, s.qy, s.qz, s.qw, s.R);
  const Rot<rreal>& R = s.R;
  rreal vx = (rreal)s.vx, vy = (rreal)s.vy, vz = (rreal)s.vz;
  s.vb.x = (float)(R.m00 * vx + R.m10 * vy + R.m20 * vz);
  s.vb.y = (float)(R.m01 * vx + R.m11 * vy + R.m21 * vz);
  s.vb.z = (float)(R.m02 * vx + R.m12 * vy + R.m22 * vz);
}

// atan2 without the IEEE-division / denormal slow paths: |error| < 4e-7 rad for max(|x|, |y|) in [FLT_MIN, 2^126)
// (tests/test_device_math.py).  Octant reduction to a = min/max in [0,1], odd minimax polynomial for atan(a), quadrant fix-ups.
// A subnormal max takes a = 0, the nearest multiple of pi/2 in its octant pair (|error| <= pi/4): fast_rcp would flush it to 0
// on the device and overflow on the host, and mn * inf is NaN.  Only a link at rest in still air reaches it, where the
// surface force is ~1e-38 N.  Outside the domain: max >= 2^126 gives a = 0 on the device (the reciprocal is subnormal and
// flushed), and atan2_f(+-0, -0) = +-0 where IEEE atan2 gives +-pi.
PFB_HD float atan2_f(float y, float x) {
  float ax = fabsf(x), ay = fabsf(y);
  float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
  float a = mx >= kFltMin ? fast_div(mn, mx) : 0.0f;
  float t = a * a;
  float r = 0.00282363896258175373077393f;
  r = fmaf(r, t, -0.0159569028764963150024414f);
  r = fmaf(r, t, 0.0425049886107444763183594f);
  r = fmaf(r, t, -0.0748900920152664184570312f);
  r = fmaf(r, t, 0.106347933411598205566406f);
  r = fmaf(r, t, -0.142027363181114196777344f);
  r = fmaf(r, t, 0.199926957488059997558594f);
  r = fmaf(r, t, -0.333331018686294555664062f);
  r = fmaf(r * t, a, a);
  if (ay > ax) r = 1.57079632679489661923f - r;
  if (x < 0.0f) r = 3.14159265358979323846f - r;
  return copysignf(r, y);
}

// p.getEulerFromQuaternion (btQuaternion::getEulerZYX with the +-0.99999 gimbal-lock branch)
// asin(s) is evaluated as atan2(s, sqrt(1 - s^2)): same function on (-1, 1), one polynomial to maintain.
PFB_HD void euler_from_quat(float x, float y, float z, float w, float& roll, float& pitch, float& yaw) {
  float sarg = -2.0f * (x * z - w * y);
  float sqx = x * x, sqy = y * y, sqz = z * z, sqw = w * w;
  float ra = 2.0f * (y * z + w * x), rb = sqw - sqx - sqy + sqz;
  float ya = 2.0f * (x * y + w * z), yb = sqw + sqx - sqy - sqz;
  float pa = sarg, pb = fast_sqrt(fmaxf(0.0f, 1.0f - sarg * sarg));
  float yscale = 1.0f;
  if (fabsf(sarg) >= 0.99999f) {  // gimbal lock: roll = 0, pitch = +-pi/2, yaw = 2 atan2(+-x, -+y)
    float sg = sarg > 0.0f ? 1.0f : -1.0f;
    ra = 0.0f; rb = 1.0f;
    pa = sg; pb = 0.0f;
    ya = -sg * x; yb = sg * y;
    yscale = 2.0f;
  }
  roll = atan2_f(ra, rb);
  pitch = atan2_f(pa, pb);
  yaw = yscale * atan2_f(ya, yb);
}

// roll and pitch only (the Hover reward needs nothing else): quadx_hover_env.py:133-134
PFB_HD void roll_pitch_from_quat(float x, float y, float z, float w, float& roll, float& pitch) {
  float sarg = -2.0f * (x * z - w * y);
  float ra = 2.0f * (y * z + w * x), rb = w * w - x * x - y * y + z * z;
  float pa = sarg, pb = fast_sqrt(fmaxf(0.0f, 1.0f - sarg * sarg));
  if (fabsf(sarg) >= 0.99999f) {
    ra = 0.0f; rb = 1.0f;
    pa = sarg > 0.0f ? 1.0f : -1.0f; pb = 0.0f;
  }
  roll = atan2_f(ra, rb);
  pitch = atan2_f(pa, pb);
}

// p.getQuaternionFromEuler (btQuaternion::setEulerZYX)
PFB_HD void quat_from_euler(float roll, float pitch, float yaw, float& x, float& y, float& z, float& w) {
  float hr = 0.5f * roll, hp = 0.5f * pitch, hy = 0.5f * yaw;
  float sr = sinf(hr), cr = cosf(hr), sp = sinf(hp), cp = cosf(hp), sy = sinf(hy), cy = cosf(hy);
  x = sr * cp * cy - cr * sp * sy;
  y = cr * sp * cy + sr * cp * sy;
  z = cr * cp * sy - sr * sp * cy;
  w = cr * cp * cy + sr * sp * sy;
}

// abstractions/pid.py:70-94 for K axes; mem = [I(K), e_prev(K)]
template <int K>
PFB_HD void pid_step(const float (&g)[4][3], float* mem, const float* state, const float* setpoint, float* out) {
#pragma unroll
  for (int i = 0; i < K; ++i) {
    float error = setpoint[i] - state[i];
    float integral = clampf(fmaf(g[1][i], error, mem[i]), -g[3][i], g[3][i]);
    float derivative = g[2][i] * (error - mem[K + i]);
    mem[i] = integral;
    mem[K + i] = error;
    out[i] = clampf(fmaf(g[0][i], error, integral) + derivative, -g[3][i], g[3][i]);
  }
}

// quadx.py:401-493, specialised on the flight mode at compile time
template <int MODE>
PFB_HD void quadx_update_control(const QuadXParams& p, QuadXRegs& s) {
  if (MODE == -1) {  // direct pwm: no mixing, no saturation handling (quadx.py:432-434)
#pragma unroll
    for (int i = 0; i < 4; ++i) s.pwm[i] = s.sp[i];
    return;
  }
  float a[3] = {s.sp[0], s.sp[1], s.sp[2]};
  float z = s.sp[3];
  const float angvel[3] = {s.wx, s.wy, s.wz};
  float roll = 0.f, pitch = 0.f, yaw = 0.f;
  if (MODE == 1 || MODE >= 3) euler_from_quat((float)s.qx, (float)s.qy, (float)s.qz, (float)s.qw, roll, pitch, yaw);
  const float euler[3] = {roll, pitch, yaw};
  const float linvel[3] = {s.vb.x, s.vb.y, s.vb.z};
  const float pos[3] = {(float)s.px, (float)s.py, (float)s.pz};

  if (MODE == 7) pid_step<2>(p.pid[3], s.pid + PID_P3, pos, a, a);
  if (MODE == 6 || MODE == 7) {  // world -> heading frame (quadx.py:448-451, 460-463)
    float sn = sinf(yaw), c = cosf(yaw);
    float x = c * a[0] + sn * a[1], y = -sn * a[0] + c * a[1];
    a[0] = x; a[1] = y;
  }
  if (MODE >= 4) {
    pid_step<2>(p.pid[2], s.pid + PID_P2, linvel, a, a);
    float t0 = -a[1], t1 = a[0];
    a[0] = t0; a[1] = t1;
  }
  if (MODE == 1 || MODE == 3 || MODE == 7) pid_step<3>(p.pid[1], s.pid + PID_P1, euler, a, a);
  if (MODE == 4 || MODE == 5 || MODE == 6) pid_step<2>(p.pid[1], s.pid + PID_P1, euler, a, a);
  pid_step<3>(p.pid[0], s.pid + PID_P0, angvel, a, a);

  // height chain (quadx.py:470-479)
  if (MODE == 2 || MODE == 3 || MODE == 4 || MODE == 7) pid_step<1>(p.pid[5], s.pid + PID_ZP, &pos[2], &z, &z);
  if (MODE != 0) pid_step<1>(p.pid[4], s.pid + PID_ZV, &linvel[2], &z, &z);
  z = clampf(z, 0.0f, 1.0f);

  // motor mix (quadx.py:130-137, 482-483)
  float m0 = -a[0] - a[1] - a[2] + z;
  float m1 = +a[0] + a[1] - a[2] + z;
  float m2 = +a[0] - a[1] + a[2] + z;
  float m3 = -a[0] + a[1] + a[2] + z;
  // saturation re-scale (quadx.py:485-493)
  float high = fmaxf(fmaxf(m0, m1), fmaxf(m2, m3));
  float low = fminf(fminf(m0, m1), fminf(m2, m3));
  if (high != low) {
    float pwm_max = fminf(high, 1.0f), pwm_min = fmaxf(low, 0.05f);
    float ka = fast_div(pwm_min - low, pwm_max - low);
    float ks = fast_div(high - pwm_max, high - pwm_min);
    m0 += ka * (pwm_max - m0) - ks * (m0 - pwm_min);
    m1 += ka * (pwm_max - m1) - ks * (m1 - pwm_min);
    m2 += ka * (pwm_max - m2) - ks * (m2 - pwm_min);
    m3 += ka * (pwm_max - m3) - ks * (m3 - pwm_min);
  }
  s.pwm[0] = clampf(m0, 0.05f, 1.0f);
  s.pwm[1] = clampf(m1, 0.05f, 1.0f);
  s.pwm[2] = clampf(m2, 0.05f, 1.0f);
  s.pwm[3] = clampf(m3, 0.05f, 1.0f);
}

// lowest point of the collision primitives against the plane z = top (0: the floor), with the relative
// contact-breaking threshold; evaluated on the pose at the START of the substep.
PFB_HD bool quadx_ground_contact(const QuadXParams& p, const QuadXRegs& s, float top = 0.0f) {
  const float pz = (float)s.pz;
  if (pz - top > p.contact_zmax) return false;  // higher than any primitive can reach: the common case
  const float r20 = (float)s.R.m20, r21 = (float)s.R.m21, r22 = (float)s.R.m22;
  bool hit = false;
#pragma unroll 1
  for (int k = 0; k < p.n_shapes; ++k) {
    {
      float cz = pz + r20 * p.shape_at[k][0] + r21 * p.shape_at[k][1] + r22 * p.shape_at[k][2];
      float extent;
      if (p.shape_kind[k] == 0) {
        extent = fabsf(r20) * p.shape_dims[k][0] + fabsf(r21) * p.shape_dims[k][1] + fabsf(r22) * p.shape_dims[k][2];
      } else if (p.shape_kind[k] == 1) {
        extent = p.shape_dims[k][1] * fabsf(r22) + p.shape_dims[k][0] * fast_sqrt(fmaxf(0.0f, 1.0f - r22 * r22));
      } else {
        extent = p.shape_dims[k][0];
      }
      hit = hit || (cz - extent - top < p.shape_thr[k]);
    }
  }
  return hit;
}

// ---- static bodies of an Aviary handle (pfb_add_static_body; DESIGN.md §4h) ---------------------------------------------
// Fixed-base boxes and cylinders, upright once posed.  Every drone's world holds its own copy of each body: the primitive table
// is launch-constant (a kernel parameter), the pose of body b in drone i's world is rows 5 b .. 5 b + 4 (x, y, z, cos yaw,
// sin yaw of the base link frame) of a field-major [5 * kMaxStaticBodies][n] buffer that only pfb_set_static_pose writes.
constexpr int kMaxStaticBodies = 8, kMaxStaticShapes = 16, kStaticPoseRows = 5;  // = PFB_MAX_STATIC_BODIES / _SHAPES
struct StaticWorld {
  int n_shapes;
  int body[kMaxStaticShapes];         // the body primitive k belongs to
  int kind[kMaxStaticShapes];         // PFB_SHAPE_BOX or PFB_SHAPE_CYLINDER
  float at[kMaxStaticShapes][3];      // centre in the body's base link frame
  float cyaw[kMaxStaticShapes], syaw[kMaxStaticShapes];  // yaw of the primitive in that frame
  float half[kMaxStaticShapes][3];    // box: half extents; cylinder: radius, radius, half length
};
// The step bodies take a World: NoStatic (the floor only: the kernels every handle without static bodies launches) or
// StaticCtx (the floor and the static bodies of drone i's world).  bits: what drone i touched during its current Aviary step,
// bit 0 the floor, bit 1 + b static body b.  A step kernel initialises either as World w{&table, pose, n, i, 0u}.
struct NoStaticTable {};
struct NoStatic {
  static constexpr bool kOn = false;
  const NoStaticTable* w;  // StaticCtx's fields, never read
  const float* pose;
  int64_t n, i;
  uint32_t bits;
};
struct StaticCtx {
  static constexpr bool kOn = true;
  const StaticWorld* w;
  const float* pose;
  int64_t n, i;
  uint32_t bits;
};
// pfb_fixedwing.cuh: surface height under a drone and its contact bits
template <class Touch>
PFB_HD float static_surface(const StaticWorld& w, const float* pose, int64_t n, int64_t i, float px, float py, float pz, float reach,
                            Touch&& touch, uint32_t& bits);

// Bullet clamps the WORLD angular-velocity coordinates to +-vmax; that can only bite when a body rate
// exceeds vmax/sqrt(3), so the rotation to the world frame and back lives out of line (cold).  Everything
// is passed BY VALUE so that the caller's register-resident state never has its address taken.
#if defined(__CUDACC__)
static __host__ __device__ __noinline__
#else
inline
#endif
Vec3 quadx_clamp_world_rates(float vmax, Mat3 R, Vec3 w) {
  Vec3 o = mul(R, w);
  o.x = clampf(o.x, -vmax, vmax); o.y = clampf(o.y, -vmax, vmax); o.z = clampf(o.z, -vmax, vmax);
  return mulT(R, o);
}

// Bullet's +-vmax clamp of the world linear velocity (btMultiBody::applyDeltaVeeMultiDof): only ever taken by a body
// falling at the 100 m/s limit.  Out of line for the same reason as above: inlined, the compiler if-converts it into
// ~45 predicated fp64 instructions that occupy issue slots on every substep.
struct Vel3 { vreal x, y, z; };
#if defined(__CUDACC__)
static __host__ __device__ __noinline__
#else
inline
#endif
Vel3 quadx_clamp_world_velocity(vreal vmax, Vel3 v) {
  v.x = fmin(fmax(v.x, -vmax), vmax);
  v.y = fmin(fmax(v.y, -vmax), vmax);
  v.z = fmin(fmax(v.z, -vmax), vmax);
  return v;
}

// contact RESPONSE over a list of collision primitives (pfb_fixedwing.cuh)
template <class Tag = NoStatic, class Shapes, class Regs>
PFB_HD void apply_contact_impulses(const Shapes* cp, Regs& s, float pz0, float top, float M, Vec3 c, float Ixx, float Ixy, float Ixz,
                                   float Iyy, float Iyz, float Izz, float dt);

// One physics substep: update_physics (quadx.py:495-510) + stepSimulation + update_state.
// xi = raw draw of np_random.normal(*throttle.shape)  (one scalar ~ N(4, 1) shared by the motors).
// Written as straight-line code (selects instead of branches): the kernel is instruction-issue bound
// and the I-cache-resident hot loop is what the whole env step runs in.
// CONTACT = the floor pushes back (Aviary handles with contact_response): on a substep whose contact flag is up, contact
// impulses act on the predicted velocities before the pose is integrated (cold path; COM at the base origin, diagonal inertia).
// World: NoStatic, or StaticCtx (the static bodies of this drone's world: flags against each surface under the base, the
// response against the highest of them).
template <bool CONTACT = false, class World = NoStatic>
PFB_HD void quadx_substep(const QuadXParams& p, QuadXRegs& s, float xi, World* world = nullptr) {
  // ---- motors (motors.py:130-155): lag, multiplicative noise, rpm^2 thrust + reaction torque
  float Fz = 0.0f, tx = 0.0f, ty = 0.0f, tz = 0.0f;
  const float gain = xi * p.noise_ratio;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float t = s.thr[i];
    t = fmaf(p.motor_lag, s.pwm[i] - t, t);
    t = fmaf(gain, t, t);
    s.thr[i] = t;
    float a = t * fabsf(t);
    float Ti = p.thrust_k[i] * a;
    Fz += Ti;
    tx = fmaf(p.motor_y[i], Ti, tx);
    ty = fmaf(-p.motor_x[i], Ti, ty);
    tz = fmaf(p.torque_k[i], a, tz);
  }
  // ---- body drag (boring_bodies.py:113-127), body link at the base origin, on the velocity through the AIR
  Vec3 va = s.vb;
  if (p.wind.kind != 0) {  // boring_bodies.py:93-96 (uniform branch: the parameter block is launch-constant)
    const WindCtx wc = wind_ctx(p.wind, (float)s.pz, (float)s.R.m00, (float)s.R.m01, (float)s.R.m02, (float)s.R.m10, (float)s.R.m11,
                                (float)s.R.m12, (float)s.R.m20, (float)s.R.m21, (float)s.R.m22);
    va = va - wind_body_at(p.wind, wc, 0.0f, 0.0f, 0.0f);
  }
  float Fx = -p.drag_k[0] * signed_square(va.x);
  float Fy = -p.drag_k[1] * signed_square(va.y);
  Fz = fmaf(-p.drag_k[2], signed_square(va.z), Fz);
  // ---- rotational drag unless something touched the floor last step (quadx.py:502-510)
  const float kpqr = (s.flags & FLAG_CONTACT_PREV) ? 0.0f : -p.drag_pqr;
  tx = fmaf(kpqr, signed_square(s.wx), tx);
  ty = fmaf(kpqr, signed_square(s.wy), ty);
  tz = fmaf(kpqr, signed_square(s.wz), tz);
  // ---- contact flag from the pose at the start of the step (collision detection precedes
  //      integration inside stepSimulation); aviary.py:523-525
  bool c;
  float top = 0.0f;  // surface height under the drone
  if constexpr (World::kOn) {
    uint32_t b;
    top = static_surface(*world->w, world->pose, world->n, world->i, (float)s.px, (float)s.py, (float)s.pz, p.contact_zmax,
                         [&](float t) { return quadx_ground_contact(p, s, t); }, b);
    world->bits |= b;
    c = b != 0u;
  } else {
    c = quadx_ground_contact(p, s);
  }
  s.flags = (s.flags & ~(uint32_t)FLAG_CONTACT_PREV) | (c ? (FLAG_CONTACT_PREV | FLAG_CONTACT_ARRAY) : 0u);

  // ---- Newton-Euler about the COM (composite COM offset is zero for the quads; inertia diagonal)
  float wdx = (tx - (p.Izz - p.Iyy) * s.wy * s.wz) * p.inv_Ixx;
  float wdy = (ty - (p.Ixx - p.Izz) * s.wz * s.wx) * p.inv_Iyy;
  float wdz = (tz - (p.Iyy - p.Ixx) * s.wx * s.wy) * p.inv_Izz;
  // world acceleration a = R F_b / M + g, velocities first (clamped per coordinate), then positions
  const Rot<rreal>& R = s.R;
  rreal fx = (rreal)(Fx * p.inv_mass), fy = (rreal)(Fy * p.inv_mass), fz = (rreal)(Fz * p.inv_mass);
  rreal ax = R.m00 * fx + R.m01 * fy + R.m02 * fz;
  rreal ay = R.m10 * fx + R.m11 * fy + R.m12 * fz;
  rreal az = R.m20 * fx + R.m21 * fy + R.m22 * fz + (rreal)p.gravity;
  const vreal dt = (vreal)p.dt;
  s.vx += (vreal)ax * dt;
  s.vy += (vreal)ay * dt;
  s.vz += (vreal)az * dt;
  // +-vmax clamp per world coordinate (btMultiBody::applyDeltaVeeMultiDof): tested on the fp32 copy,
  // applied exactly, and only ever taken by a body falling at the 100 m/s limit
  if (fmaxf(fmaxf(fabsf((float)s.vx), fabsf((float)s.vy)), fabsf((float)s.vz)) >= p.vmax) {
    Vel3 c = quadx_clamp_world_velocity((vreal)p.vmax, Vel3{s.vx, s.vy, s.vz});
    s.vx = c.x; s.vy = c.y; s.vz = c.z;
  }
  if (!CONTACT) {  // the contact impulses below change the velocities the positions move with
    s.px += (xreal)(s.vx * dt);
    s.py += (xreal)(s.vy * dt);
    s.pz += (xreal)(s.vz * dt);
  }
  s.wx = fmaf(wdx, p.dt, s.wx);
  s.wy = fmaf(wdy, p.dt, s.wy);
  s.wz = fmaf(wdz, p.dt, s.wz);
  if (fmaxf(fmaxf(fabsf(s.wx), fabsf(s.wy)), fabsf(s.wz)) > p.vmax * 0.57735f) {
    Mat3 Rf{(float)R.m00, (float)R.m01, (float)R.m02, (float)R.m10, (float)R.m11, (float)R.m12, (float)R.m20, (float)R.m21, (float)R.m22};
    Vec3 w = quadx_clamp_world_rates(p.vmax, Rf, Vec3{s.wx, s.wy, s.wz});
    s.wx = w.x; s.wy = w.y; s.wz = w.z;
  }
  if (CONTACT) {
    if (c) apply_contact_impulses<World>(&p, s, (float)s.pz, top, 1.0f / p.inv_mass, Vec3{0.f, 0.f, 0.f}, p.Ixx, 0.0f, 0.0f, p.Iyy, 0.0f, p.Izz, p.dt);
    s.px += (xreal)(s.vx * dt);
    s.py += (xreal)(s.vy * dt);
    s.pz += (xreal)(s.vz * dt);
  }
  // ---- attitude: q <- q * dq(w_b dt).  dq = (w sin(h)/|w|, cos h), h = |w| dt / 2.  With
  // h^2 = |w|^2 dt^2 / 4 <= 0.13 (|w| <= sqrt(3) vmax; checked at create) both factors are short even
  // series in h^2: sin(h)/|w| = dt/2 * sinc(h) and cos(h) — no sqrt, no division, no range reduction,
  // and the series IS Bullet's small-angle branch (btTransformUtil), continued to fp32 round-off.
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
  // |q|^2 = 1 + e with |e| ~ 1e-7 (fp32 increment): 1/sqrt(1+e) = 1 - e/2 + 3e^2/8 (error < 1e-21)
  qreal e = n2 - 1.0;
  qreal inv = 1.0 - 0.5 * e + 0.375 * e * e;
#else
  qreal inv = 1.0f / sqrtf(n2);
#endif
  s.qx = nx * inv; s.qy = ny * inv; s.qz = nz * inv; s.qw = nw * inv;
  // ---- update_state (quadx.py:512-535)
  quadx_update_state(s);
}

// Aviary.step(): one control tick + `ratio` physics substeps (aviary.py:506-531 with one drone).
// Noise protocol: begin_step() prepares the draws of this Aviary step (outside the substep loop),
// get(u) hands out the draw of substep u.
template <int MODE, bool CONTACT = false, typename NoiseFn, class World = NoStatic>
PFB_HD void quadx_aviary_step(const QuadXParams& p, QuadXRegs& s, NoiseFn& noise, World* world = nullptr) {
  s.flags &= ~(uint32_t)FLAG_CONTACT_ARRAY;  // contact_array &= False
  if constexpr (World::kOn) world->bits = 0u;
  noise.begin_step();
  quadx_update_control<MODE>(p, s);
#pragma unroll 1
  for (int u = 0; u < p.ratio; ++u) quadx_substep<CONTACT>(p, s, noise.get(u), world);
}

// quadx.py:233-373: setpoint preset + PID reset on a mode change
template <int MODE>
PFB_HD void quadx_set_mode(QuadXRegs& s) {
  if (MODE == -1) return;
  if (MODE == 0) {
    s.sp[0] = 0.f; s.sp[1] = 0.f; s.sp[2] = 0.f; s.sp[3] = -1.0f;
  } else if (MODE == 1 || MODE == 5 || MODE == 6) {
    s.sp[0] = s.sp[1] = s.sp[2] = s.sp[3] = 0.0f;
  } else if (MODE == 7) {
    float roll, pitch, yaw;
    euler_from_quat((float)s.qx, (float)s.qy, (float)s.qz, (float)s.qw, roll, pitch, yaw);
    s.sp[0] = (float)s.px; s.sp[1] = (float)s.py; s.sp[2] = yaw; s.sp[3] = (float)s.pz;
  } else {
    s.sp[0] = s.sp[1] = s.sp[2] = 0.0f; s.sp[3] = (float)s.pz;
  }
#pragma unroll
  for (int k = 0; k < PID_ZV; ++k) s.pid[k] = 0.0f;  // z_PIDs are not reset by set_mode (quadx.py:196,372)
}

// ---- one flight mode per drone (pfb_set_modes): the mode is a run-time value -------------------------------------------
// Runs BODY with `constexpr int M` = the QuadX flight mode `mode` (-1..7; the caller has checked the range)
#define PFB_QX_MODE_CASES(mode, BODY)               \
  switch (mode) {                                   \
    case -1: { constexpr int M = -1; BODY; } break; \
    case 0: { constexpr int M = 0; BODY; } break;   \
    case 1: { constexpr int M = 1; BODY; } break;   \
    case 2: { constexpr int M = 2; BODY; } break;   \
    case 3: { constexpr int M = 3; BODY; } break;   \
    case 4: { constexpr int M = 4; BODY; } break;   \
    case 5: { constexpr int M = 5; BODY; } break;   \
    case 6: { constexpr int M = 6; BODY; } break;   \
    default: { constexpr int M = 7; BODY; } break;  \
  }

// The control tick of a drone in flight mode `mode`.  Only the control tick branches on the mode: the physics substeps after
// it are the same code for every mode, so a warp whose lanes fly several modes reconverges before them.
PFB_HD void quadx_update_control_any(const QuadXParams& p, QuadXRegs& s, int mode) {
  PFB_QX_MODE_CASES(mode, quadx_update_control<M>(p, s));
}

template <bool CONTACT = false, typename NoiseFn, class World = NoStatic>
PFB_HD void quadx_aviary_step_any(const QuadXParams& p, QuadXRegs& s, int mode, NoiseFn& noise, World* world = nullptr) {
  s.flags &= ~(uint32_t)FLAG_CONTACT_ARRAY;
  if constexpr (World::kOn) world->bits = 0u;
  noise.begin_step();
  quadx_update_control_any(p, s, mode);
#pragma unroll 1
  for (int u = 0; u < p.ratio; ++u) quadx_substep<CONTACT>(p, s, noise.get(u), world);
}

// quadx_aviary_step_any inside an Aviary step of U substeps whose drones run at several control rates (aviary.py:506-529):
// this drone, physics_hz / control_hz = r (a divisor of U, the table's own ratio), runs its control tick before substep u when
// u % r == 0 and takes draw u of the step.  With r == U it is quadx_aviary_step_any.
template <bool CONTACT = false, typename NoiseFn, class World = NoStatic>
PFB_HD void quadx_aviary_step_rates(const QuadXParams& p, QuadXRegs& s, int mode, int r, int U, NoiseFn& noise, World* world = nullptr) {
  s.flags &= ~(uint32_t)FLAG_CONTACT_ARRAY;
  if constexpr (World::kOn) world->bits = 0u;
  noise.begin_step();
#pragma unroll 1
  for (int u = 0; u < U; ++u) {
    if (u % r == 0) quadx_update_control_any(p, s, mode);
    quadx_substep<CONTACT>(p, s, noise.get(u), world);
  }
}

PFB_HD void quadx_set_mode_any(QuadXRegs& s, int mode) { PFB_QX_MODE_CASES(mode, quadx_set_mode<M>(s)); }

// quadx.py:222-231 + aviary.py:310-311: a freshly constructed drone at its start pose
PFB_HD void quadx_reset(QuadXRegs& s, float sx, float sy, float sz, float roll, float pitch, float yaw) {
  s.px = (xreal)sx; s.py = (xreal)sy; s.pz = (xreal)sz;
  {  // getQuaternionFromEuler in the attitude precision
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
  for (int i = 0; i < 4; ++i) { s.thr[i] = 0.0f; s.pwm[i] = 0.0f; s.sp[i] = 0.0f; }
#pragma unroll
  for (int k = 0; k < PID_WORDS; ++k) s.pid[k] = 0.0f;
  s.flags = 0u;
  quadx_update_state(s);
}

// ---- state tensor <-> registers ----------------------------------------------------------------
// MODE-dependent PID rows: only the controllers a mode instantiates are moved.
template <int MODE>
PFB_HD constexpr bool pid_row_used(int k) {
  if (MODE == -1) return false;
  if (k < PID_P1) return true;                                                   // ang_vel
  if (k < PID_P2) {                                                              // ang_pos
    if (MODE == 1 || MODE == 3 || MODE == 7) return true;
    if (MODE >= 4 && MODE <= 6) return (k - PID_P1) < 4;  // two-axis controller: [I0 I1 e0 e1]
    return false;
  }
  if (k < PID_P3) return MODE >= 4;                                              // lin_vel
  if (k < PID_ZV) return MODE == 7;                                              // lin_pos
  if (k < PID_ZP) return MODE != 0;                                              // z_vel
  return MODE == 2 || MODE == 3 || MODE == 4 || MODE == 7;                       // z_pos
}

template <int MODE>
// `st` is field-major [F][N] (row stride N) by default; `rs` / `ci` let a caller read an env-major record instead
// (row stride 1, base already advanced to the env's record): the spare states of the reset pipeline.
PFB_HD void quadx_load(const float* __restrict__ st, const int32_t* __restrict__ ist, int64_t N, int64_t i, QuadXRegs& s,
                       int64_t rs = -1, int64_t ci = -1) {
  if (rs < 0) { rs = N; ci = i; }
  auto F = [&](int row) { return st[(int64_t)row * rs + ci]; };
#if PFB_X_DOUBLE
  s.px = join_hi_lo(F(QX_POS + 0), F(QX_POS_LO + 0));
  s.py = join_hi_lo(F(QX_POS + 1), F(QX_POS_LO + 1));
  s.pz = join_hi_lo(F(QX_POS + 2), F(QX_POS_LO + 2));
#else
  s.px = F(QX_POS + 0); s.py = F(QX_POS + 1); s.pz = F(QX_POS + 2);
#endif
#if PFB_Q_DOUBLE
  s.qx = join_hi_lo(F(QX_QUAT + 0), F(QX_QUAT_LO + 0));
  s.qy = join_hi_lo(F(QX_QUAT + 1), F(QX_QUAT_LO + 1));
  s.qz = join_hi_lo(F(QX_QUAT + 2), F(QX_QUAT_LO + 2));
  s.qw = join_hi_lo(F(QX_QUAT + 3), F(QX_QUAT_LO + 3));
#else
  s.qx = F(QX_QUAT + 0); s.qy = F(QX_QUAT + 1); s.qz = F(QX_QUAT + 2); s.qw = F(QX_QUAT + 3);
#endif
#if PFB_V_DOUBLE
  s.vx = join_hi_lo(F(QX_VEL + 0), F(QX_VEL_LO + 0));
  s.vy = join_hi_lo(F(QX_VEL + 1), F(QX_VEL_LO + 1));
  s.vz = join_hi_lo(F(QX_VEL + 2), F(QX_VEL_LO + 2));
#else
  s.vx = F(QX_VEL + 0); s.vy = F(QX_VEL + 1); s.vz = F(QX_VEL + 2);
#endif
  s.wx = F(QX_ANGVEL + 0); s.wy = F(QX_ANGVEL + 1); s.wz = F(QX_ANGVEL + 2);
#pragma unroll
  // the pwm rows are write-only: every Aviary step starts with a control tick that recomputes pwm before any
  // substep reads it (aviary.py:506-531 with physics_control_ratio == updates_per_step), so they are not loaded
  for (int k = 0; k < 4; ++k) { s.thr[k] = F(QX_THR + k); s.pwm[k] = 0.0f; }
#pragma unroll
  for (int k = 0; k < PID_WORDS; ++k) s.pid[k] = pid_row_used<MODE>(k) ? F(qx_pid_row(k)) : 0.0f;
  s.flags = (uint32_t)ist[(int64_t)QI_FLAGS * N + i];
  quadx_update_state(s);
}

template <int MODE>
PFB_HD void quadx_store(float* __restrict__ st, int32_t* __restrict__ ist, int64_t N, int64_t i, const QuadXRegs& s,
                        bool with_flags = true, int64_t rs = -1, int64_t ci = -1) {
  if (rs < 0) { rs = N; ci = i; }
  auto S = [&](int row, float v) { st[(int64_t)row * rs + ci] = v; };
  float hi, lo;
#if PFB_X_DOUBLE
  split_hi_lo(s.px, hi, lo); S(QX_POS + 0, hi); S(QX_POS_LO + 0, lo);
  split_hi_lo(s.py, hi, lo); S(QX_POS + 1, hi); S(QX_POS_LO + 1, lo);
  split_hi_lo(s.pz, hi, lo); S(QX_POS + 2, hi); S(QX_POS_LO + 2, lo);
#else
  S(QX_POS + 0, s.px); S(QX_POS + 1, s.py); S(QX_POS + 2, s.pz);
#endif
#if PFB_Q_DOUBLE
  split_hi_lo(s.qx, hi, lo); S(QX_QUAT + 0, hi); S(QX_QUAT_LO + 0, lo);
  split_hi_lo(s.qy, hi, lo); S(QX_QUAT + 1, hi); S(QX_QUAT_LO + 1, lo);
  split_hi_lo(s.qz, hi, lo); S(QX_QUAT + 2, hi); S(QX_QUAT_LO + 2, lo);
  split_hi_lo(s.qw, hi, lo); S(QX_QUAT + 3, hi); S(QX_QUAT_LO + 3, lo);
#else
  S(QX_QUAT + 0, s.qx); S(QX_QUAT + 1, s.qy); S(QX_QUAT + 2, s.qz); S(QX_QUAT + 3, s.qw);
#endif
#if PFB_V_DOUBLE
  split_hi_lo(s.vx, hi, lo); S(QX_VEL + 0, hi); S(QX_VEL_LO + 0, lo);
  split_hi_lo(s.vy, hi, lo); S(QX_VEL + 1, hi); S(QX_VEL_LO + 1, lo);
  split_hi_lo(s.vz, hi, lo); S(QX_VEL + 2, hi); S(QX_VEL_LO + 2, lo);
#else
  S(QX_VEL + 0, s.vx); S(QX_VEL + 1, s.vy); S(QX_VEL + 2, s.vz);
#endif
  (void)hi; (void)lo;
  S(QX_ANGVEL + 0, s.wx); S(QX_ANGVEL + 1, s.wy); S(QX_ANGVEL + 2, s.wz);
#pragma unroll
  for (int k = 0; k < 4; ++k) { S(QX_THR + k, s.thr[k]); S(QX_PWM + k, s.pwm[k]); }
#pragma unroll
  for (int k = 0; k < PID_WORDS; ++k)
    if (pid_row_used<MODE>(k)) S(qx_pid_row(k), s.pid[k]);
  if (with_flags) ist[(int64_t)QI_FLAGS * N + i] = (int32_t)s.flags;
}

// ---- warp-tiled / record layout: 16-byte groups -------------------------------------------------------------------------
PFB_HD float f_from_bits(uint32_t u) {
#if defined(__CUDA_ARCH__)
  return __uint_as_float(u);
#else
  float f; memcpy(&f, &u, 4); return f;
#endif
}
PFB_HD uint32_t bits_from_f(float f) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(f);
#else
  uint32_t u; memcpy(&u, &f, 4); return u;
#endif
}
// does MODE move group g (rows 4g .. 4g+3)?  Groups 0-8: pose, velocities, throttles, step / flags, ang_vel PID, lo words;
// 9: pwm (written, never read: every Aviary step starts with a control tick); 10-14: the other controllers' memories
template <int MODE>
PFB_HD constexpr bool qx_group_used(int g) {
  if (g <= 9) return true;
  for (int c = 0; c < 4; ++c) {
    const int k = 6 + 4 * (g - 10) + c;
    if (k < PID_WORDS && pid_row_used<MODE>(k)) return true;
  }
  return false;
}
template <int MODE>
PFB_HD constexpr int qx_groups_moved() {  // groups 0 .. n-1 cover every row MODE touches
  int n = 10;
  for (int g = 10; g < QX_ROWS / 4; ++g)
    if (qx_group_used<MODE>(g)) n = g + 1;
  return n;
}

// `rec` = the env's record base (tile: st + qx_tile_base(i), GS = kTileGroupStride; env-major record: GS = 4).
// Two halves: quadx_fetch_tile issues the 128-bit loads of the groups every mode needs; quadx_unpack_tile turns them into
// registers.  The step kernel runs its noise generator BETWEEN the two so that it executes in the shadow of the loads.
struct QxRaw {
  F4 g0, g1, g2, g3, g4, g5, g6, g7, g8;
};
template <int GS>
PFB_HD QxRaw quadx_fetch_tile(const float* __restrict__ rec) {
  QxRaw r;
  r.g0 = ld_f4(rec + 0 * GS); r.g1 = ld_f4(rec + 1 * GS); r.g2 = ld_f4(rec + 2 * GS); r.g3 = ld_f4(rec + 3 * GS); r.g4 = ld_f4(rec + 4 * GS);
  r.g5 = ld_f4(rec + 5 * GS); r.g6 = ld_f4(rec + 6 * GS); r.g7 = ld_f4(rec + 7 * GS);
#if PFB_V_DOUBLE
  r.g8 = ld_f4(rec + 8 * GS);
#else
  r.g8 = F4{0.f, 0.f, 0.f, 0.f};
#endif
  return r;
}
template <int MODE, int GS>
PFB_HD void quadx_unpack_tile(const QxRaw& r, const float* __restrict__ rec, QuadXRegs& s, int& step_count) {
  const F4 &g0 = r.g0, &g1 = r.g1, &g2 = r.g2, &g3 = r.g3, &g4 = r.g4, &g5 = r.g5, &g6 = r.g6, &g7 = r.g7, &g8 = r.g8;
#if PFB_X_DOUBLE
  s.px = join_hi_lo(g0.x, g6.y); s.py = join_hi_lo(g0.y, g6.z); s.pz = join_hi_lo(g0.z, g6.w);
#else
  s.px = g0.x; s.py = g0.y; s.pz = g0.z;
#endif
#if PFB_Q_DOUBLE
  s.qx = join_hi_lo(g0.w, g7.x); s.qy = join_hi_lo(g1.x, g7.y); s.qz = join_hi_lo(g1.y, g7.z); s.qw = join_hi_lo(g1.z, g7.w);
#else
  s.qx = g0.w; s.qy = g1.x; s.qz = g1.y; s.qw = g1.z;
#endif
#if PFB_V_DOUBLE
  s.vx = join_hi_lo(g1.w, g8.x); s.vy = join_hi_lo(g2.x, g8.y); s.vz = join_hi_lo(g2.y, g8.z);
#else
  s.vx = g1.w; s.vy = g2.x; s.vz = g2.y;
#endif
  s.wx = g2.z; s.wy = g2.w; s.wz = g3.x;
  s.thr[0] = g3.y; s.thr[1] = g3.z; s.thr[2] = g3.w; s.thr[3] = g4.x;
  step_count = (int)bits_from_f(g4.y);
  s.flags = bits_from_f(g4.z);
  const float p0[6] = {g4.w, g5.x, g5.y, g5.z, g5.w, g6.x};
#pragma unroll
  for (int k = 0; k < 6; ++k) s.pid[k] = pid_row_used<MODE>(k) ? p0[k] : 0.0f;
#pragma unroll
  for (int k = 0; k < 4; ++k) s.pwm[k] = 0.0f;
#pragma unroll
  for (int g = 10; g < QX_ROWS / 4; ++g) {
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (qx_group_used<MODE>(g)) {
      const F4 q = ld_f4(rec + g * GS);
      v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int k = 6 + 4 * (g - 10) + c;
      if (k < PID_WORDS) s.pid[k] = pid_row_used<MODE>(k) ? v[c] : 0.0f;
    }
  }
  quadx_update_state(s);
}
template <int MODE, int GS>
PFB_HD void quadx_load_tile(const float* __restrict__ rec, QuadXRegs& s, int& step_count) {
  const QxRaw r = quadx_fetch_tile<GS>(rec);
  quadx_unpack_tile<MODE, GS>(r, rec, s, step_count);
}

template <int MODE, int GS>
PFB_HD void quadx_store_tile(float* __restrict__ rec, const QuadXRegs& s, int step_count) {
  float pxh, pxl, pyh, pyl, pzh, pzl, qxh, qxl, qyh, qyl, qzh, qzl, qwh, qwl, vxh, vxl, vyh, vyl, vzh, vzl;
#if PFB_X_DOUBLE
  split_hi_lo(s.px, pxh, pxl); split_hi_lo(s.py, pyh, pyl); split_hi_lo(s.pz, pzh, pzl);
#else
  pxh = s.px; pyh = s.py; pzh = s.pz; pxl = pyl = pzl = 0.0f;
#endif
#if PFB_Q_DOUBLE
  split_hi_lo(s.qx, qxh, qxl); split_hi_lo(s.qy, qyh, qyl); split_hi_lo(s.qz, qzh, qzl); split_hi_lo(s.qw, qwh, qwl);
#else
  qxh = s.qx; qyh = s.qy; qzh = s.qz; qwh = s.qw; qxl = qyl = qzl = qwl = 0.0f;
#endif
#if PFB_V_DOUBLE
  split_hi_lo(s.vx, vxh, vxl); split_hi_lo(s.vy, vyh, vyl); split_hi_lo(s.vz, vzh, vzl);
#else
  vxh = s.vx; vyh = s.vy; vzh = s.vz; vxl = vyl = vzl = 0.0f;
#endif
  st_f4(rec + 0 * GS, pxh, pyh, pzh, qxh);
  st_f4(rec + 1 * GS, qyh, qzh, qwh, vxh);
  st_f4(rec + 2 * GS, vyh, vzh, s.wx, s.wy);
  st_f4(rec + 3 * GS, s.wz, s.thr[0], s.thr[1], s.thr[2]);
  st_f4(rec + 4 * GS, s.thr[3], f_from_bits((uint32_t)step_count), f_from_bits(s.flags), s.pid[0]);
  st_f4(rec + 5 * GS, s.pid[1], s.pid[2], s.pid[3], s.pid[4]);
  st_f4(rec + 6 * GS, s.pid[5], pxl, pyl, pzl);
  st_f4(rec + 7 * GS, qxl, qyl, qzl, qwl);
#if PFB_V_DOUBLE
  st_f4(rec + 8 * GS, vxl, vyl, vzl, 0.0f);
#endif
  st_f4(rec + 9 * GS, s.pwm[0], s.pwm[1], s.pwm[2], s.pwm[3]);
#pragma unroll
  for (int g = 10; g < QX_ROWS / 4; ++g) {
    if (qx_group_used<MODE>(g)) {
      float v[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int k = 6 + 4 * (g - 10) + c;
        v[c] = k < PID_WORDS ? s.pid[k] : 0.0f;
      }
      st_f4(rec + g * GS, v[0], v[1], v[2], v[3]);
    }
  }
}

// PID words that a step of the uniform MODE kernel leaves as they were (bit k = PID word k).  Its load reads the rows MODE
// uses and zeroes the other rows of the groups it moves, and its store writes those groups back; the rows of the groups it
// does not move keep their memory (the z PIDs of a drone that flies mode 0 or 1 between two height-hold phases).
template <int MODE>
PFB_HD constexpr uint32_t qx_pid_kept() {
  uint32_t m = 0u;
  for (int k = 0; k < PID_WORDS; ++k) {
    const bool moved = k < PID_P1 || qx_group_used<MODE>(10 + (k - PID_P1) / 4);
    if (pid_row_used<MODE>(k) || !moved) m |= 1u << k;
  }
  return m;
}
// After a mode-7 load (every PID row) of a drone in mode `mode`: zero what the uniform kernel of that mode would have loaded
// as zero, so that the per-drone step stores the same state tensor, word for word, as the uniform kernel of the drone's mode
PFB_HD void quadx_mask_pid(QuadXRegs& s, int mode) {
  uint32_t kept = 0u;
  PFB_QX_MODE_CASES(mode, kept = qx_pid_kept<M>());
#pragma unroll
  for (int k = 0; k < PID_WORDS; ++k)
    if (!((kept >> k) & 1u)) s.pid[k] = 0.0f;
}

// Round the fp64-carried fields to what the state tensor holds (hi + lo fp32 words) and re-derive R / body velocity:
// afterwards the registers equal what quadx_store followed by quadx_load would produce.
PFB_HD void quadx_requantize(QuadXRegs& s) {
  float hi, lo;
#if PFB_X_DOUBLE
  split_hi_lo(s.px, hi, lo); s.px = join_hi_lo(hi, lo);
  split_hi_lo(s.py, hi, lo); s.py = join_hi_lo(hi, lo);
  split_hi_lo(s.pz, hi, lo); s.pz = join_hi_lo(hi, lo);
#endif
#if PFB_Q_DOUBLE
  split_hi_lo(s.qx, hi, lo); s.qx = join_hi_lo(hi, lo);
  split_hi_lo(s.qy, hi, lo); s.qy = join_hi_lo(hi, lo);
  split_hi_lo(s.qz, hi, lo); s.qz = join_hi_lo(hi, lo);
  split_hi_lo(s.qw, hi, lo); s.qw = join_hi_lo(hi, lo);
#endif
#if PFB_V_DOUBLE
  split_hi_lo(s.vx, hi, lo); s.vx = join_hi_lo(hi, lo);
  split_hi_lo(s.vy, hi, lo); s.vy = join_hi_lo(hi, lo);
  split_hi_lo(s.vz, hi, lo); s.vz = join_hi_lo(hi, lo);
#endif
  (void)hi; (void)lo;
  quadx_update_state(s);
}

// ---- Aviary.state(i) (4,3) + aux_state -----------------------------------------------------------
PFB_HD void quadx_drone_state(const QuadXRegs& s, float* out12, float* aux4) {
  float roll, pitch, yaw;
  euler_from_quat((float)s.qx, (float)s.qy, (float)s.qz, (float)s.qw, roll, pitch, yaw);
  out12[0] = s.wx; out12[1] = s.wy; out12[2] = s.wz;
  out12[3] = roll; out12[4] = pitch; out12[5] = yaw;
  out12[6] = s.vb.x; out12[7] = s.vb.y; out12[8] = s.vb.z;
  out12[9] = (float)s.px; out12[10] = (float)s.py; out12[11] = (float)s.pz;
#pragma unroll
  for (int k = 0; k < 4; ++k) aux4[k] = s.thr[k];
}

// MAQuadXHover keeps the agent's current and past actions behind the QuadX rows: the observation carries the PAST one, and
// neither is cleared by a reset (ma_quadx_base_env.py:141-150, 326-332)
enum { QM_CUR = QX_ROWS, QM_PAST = QX_ROWS + 4, QM_ROWS = QX_ROWS + 8 };  // groups 15 and 16 of the tile

// ---- QuadX-Hover epilogue ------------------------------------------------------------------------
// quadx_base_env.py:251-266 + quadx_hover_env.py:117-138, evaluated after every Aviary step
PFB_HD void hover_term_trunc_reward(const HoverParams& h, QuadXRegs& s, int step_count, float& reward) {
  if (step_count > h.max_steps) s.flags |= FLAG_TRUNC;
  if (s.flags & FLAG_CONTACT_ARRAY) { reward = -100.0f; s.flags |= FLAG_COLLISION | FLAG_TERM; }
  float px = (float)s.px, py = (float)s.py, pz = (float)s.pz;
  float r2 = px * px + py * py;
  if (r2 + pz * pz > h.dome2) { reward = -100.0f; s.flags |= FLAG_OOB | FLAG_TERM; }  // |x| > dome
  if (!h.sparse_reward) {
    float dz = pz - 1.0f;
    float linear_distance = fast_sqrt(r2 + dz * dz);
    float roll, pitch;
    roll_pitch_from_quat((float)s.qx, (float)s.qy, (float)s.qz, (float)s.qw, roll, pitch);
    float angular_distance = fast_sqrt(roll * roll + pitch * pitch);
    reward -= 0.01f * s.wz * s.wz;
    reward -= linear_distance + angular_distance;
    reward += 1.0f;
  }
}

// quadx_hover_env.py:85-115: [ang_vel, (euler | quat(euler)), lin_vel, lin_pos, action, aux]
// The reference's quaternion observation is getQuaternionFromEuler(getEulerFromQuaternion(q)) — the
// same rotation as q, with the sign that setEulerZYX produces from principal-range angles.  Outside the
// gimbal-lock branch that is +-q, and the sign follows from half-angle tangents (no trig needed).
PFB_HD void hover_observation(const HoverParams& h, const QuadXRegs& s, const float* action, float* obs) {
  const float x = (float)s.qx, y = (float)s.qy, z = (float)s.qz, w = (float)s.qw;
  int o = 0;
  obs[o++] = s.wx; obs[o++] = s.wy; obs[o++] = s.wz;
  if (h.angle_representation == 0) {
    float roll, pitch, yaw;
    euler_from_quat(x, y, z, w, roll, pitch, yaw);
    obs[o++] = roll; obs[o++] = pitch; obs[o++] = yaw;
  } else {
    float sarg = -2.0f * (x * z - w * y);
    float ox, oy, oz, ow;
    if (fabsf(sarg) >= 0.99999f) {  // gimbal lock: the reference rebuilds q from clamped angles
      float roll, pitch, yaw;
      euler_from_quat(x, y, z, w, roll, pitch, yaw);
      quat_from_euler(roll, pitch, yaw, ox, oy, oz, ow);
    } else {
      float sqx = x * x, sqy = y * y, sqz = z * z, sqw = w * w;
      float ra = 2.0f * (y * z + w * x), rb = sqw - sqx - sqy + sqz;  // roll = atan2(ra, rb)
      float ya = 2.0f * (x * y + w * z), yb = sqw + sqx - sqy - sqz;  // yaw  = atan2(ya, yb)
      // w_e = cr cp cy + sr sp sy with cr, cp, cy >= 0: negative only if the sines' product is negative
      // and tan(|roll|/2) tan(|pitch|/2) tan(|yaw|/2) > 1;  tan(a/2) = |sin a| / (1 + cos a)
      float tr_n = fabsf(ra), tr_d = fast_sqrt(ra * ra + rb * rb) + rb;
      float ty_n = fabsf(ya), ty_d = fast_sqrt(ya * ya + yb * yb) + yb;
      float tp_n = fabsf(sarg), tp_d = 1.0f + fast_sqrt(fmaxf(0.0f, 1.0f - sarg * sarg));
      bool sines_negative = (ra * sarg * ya) < 0.0f;
      bool we_negative = sines_negative && (tr_n * tp_n * ty_n > tr_d * tp_d * ty_d);
      float sgn = ((w < 0.0f) != we_negative) ? -1.0f : 1.0f;
      if (w == 0.0f) {  // measure-zero tie: decide on the reference's own formula
        float roll, pitch, yaw;
        euler_from_quat(x, y, z, w, roll, pitch, yaw);
        quat_from_euler(roll, pitch, yaw, ox, oy, oz, ow);
        sgn = (ox * x + oy * y + oz * z) < 0.0f ? -1.0f : 1.0f;
      }
      ox = sgn * x; oy = sgn * y; oz = sgn * z; ow = sgn * w;
    }
    obs[o++] = ox; obs[o++] = oy; obs[o++] = oz; obs[o++] = ow;
  }
  obs[o++] = s.vb.x; obs[o++] = s.vb.y; obs[o++] = s.vb.z;
  obs[o++] = (float)s.px; obs[o++] = (float)s.py; obs[o++] = (float)s.pz;
#pragma unroll
  for (int k = 0; k < 4; ++k) obs[o++] = action[k];
#pragma unroll
  for (int k = 0; k < 4; ++k) obs[o++] = s.thr[k];
}

// ---- MAQuadXHover, one agent (pz_envs/quadx_envs/ma_quadx_hover_env.py) ---------------------------------------------
// compute_term_trunc_reward_info_by_id (:170-206), evaluated after EVERY Aviary step of an env step: rewards add up,
// nothing leaves the loop early (ma_quadx_base_env.py:343-362); the hover point is the agent's start position.
PFB_HD void ma_hover_term_trunc_reward(const HoverParams& h, QuadXRegs& s, int step_count, float sx, float sy, float sz, float& reward) {
  if (step_count > h.max_steps) s.flags |= FLAG_TRUNC;
  if (s.flags & FLAG_CONTACT_ARRAY) { reward -= 100.0f; s.flags |= FLAG_COLLISION | FLAG_TERM; }
  float px = (float)s.px, py = (float)s.py, pz = (float)s.pz;
  if (px * px + py * py + pz * pz > h.dome2) { reward -= 100.0f; s.flags |= FLAG_OOB | FLAG_TERM; }
  if (!h.sparse_reward) {
    float dx = px - sx, dy = py - sy, dz = pz - sz;
    float linear_distance = fast_sqrt(dx * dx + dy * dy + dz * dz);
    float roll, pitch;
    roll_pitch_from_quat((float)s.qx, (float)s.qy, (float)s.qz, (float)s.qw, roll, pitch);
    float angular_distance = fast_sqrt(roll * roll + pitch * pitch);
    reward -= linear_distance + 0.1f * angular_distance;
    reward += 1.0f;
  }
}

// compute_observation_by_id (:119-168): attitude, aux_state (throttles), PAST action, start position
PFB_HD void ma_hover_observation(const HoverParams& h, const QuadXRegs& s, const float* past, float sx, float sy, float sz, float* obs) {
  hover_observation(h, s, s.thr, obs);  // [.., thr (as "action"), thr]: the attitude block and the throttles are in place
  int o = (h.angle_representation == 0 ? 12 : 13) + 4;
#pragma unroll
  for (int k = 0; k < 4; ++k) obs[o++] = past[k];
  obs[o++] = sx; obs[o++] = sy; obs[o++] = sz;
}

// env.step() with random actions (quadx_base_env.py:79-102): uniform in the action box of the flight mode, drawn from env i's
// TAG_ACTION Philox stream.  Rng: the kernels' RngParams (key k0, k1; global id of local env 0 in env_offset_hi:lo)
template <int MODE, class Rng>
PFB_HD void quadx_random_action(const Rng& rng, int64_t i, uint32_t step_seq, float* act) {
  uint64_t g = ((uint64_t)rng.env_offset_hi << 32 | rng.env_offset_lo) + (uint64_t)i;
  U4 r = philox4x32_10(U4{(uint32_t)g, (uint32_t)(g >> 32), step_seq, (uint32_t)TAG_ACTION << 24}, rng.k0, rng.k1);
  const float pi = 3.14159265358979323846f;
  if (MODE == -1) {
    act[0] = 0.8f * u32_to_unit_open(r.x); act[1] = 0.8f * u32_to_unit_open(r.y);
    act[2] = 0.8f * u32_to_unit_open(r.z); act[3] = 0.8f * u32_to_unit_open(r.w);
  } else {
    act[0] = pi * (2.0f * u32_to_unit_open(r.x) - 1.0f); act[1] = pi * (2.0f * u32_to_unit_open(r.y) - 1.0f);
    act[2] = pi * (2.0f * u32_to_unit_open(r.z) - 1.0f); act[3] = 0.8f * u32_to_unit_open(r.w);
  }
}

}  // namespace pfb
