// pfb_fixedwing.cu — Fixedwing kernels (Aviary surface + Fixedwing-Waypoints env) and their launchers.
// Same structure as the QuadX kernels in pfb_quadx.cu: one thread = one env, state in registers between a
// coalesced SoA load and store, obs staged through shared memory, NEXT_STEP autoreset by tail CTAs.
#include <cmath>
#include <cstring>

#include "pfb_aviary.cuh"
#include "pfb_tail_step.cuh"

using namespace pfb;

#include "pfb_fixedwing_host.h"

int fw_build_params(const PfbModel& m, const PfbEnvConfig* env, FixedwingParams& p, WaypointParams& w) {
  return fw_build_params_impl(m, env, p, w);
}

static inline int fw_setpoint_dim(const PfbContext* h) { return h->env.env_kind == PFB_ENV_NONE ? 6 : 4; }
static int fw_obs_dim(const PfbContext* h) { return (h->wp.angle_representation == 0 ? 22 : 23) + 3 * h->wp.num_targets; }

// ---------------------------------------------------------------------------------------------------
// kernels — Aviary surface
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_fw_reset(const __grid_constant__ FixedwingParams p, float* __restrict__ st,
                                                     int32_t* __restrict__ ist, float* __restrict__ setpoint,
                                                     const float* __restrict__ start_pos, const float* __restrict__ start_orn,
                                                     const uint8_t* __restrict__ mask, int sp_dim, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  if (mask && !mask[i]) return;
  fw_reset_drone(p, st, ist, N, i, start_pos, start_orn, i);
  if (setpoint)  // the caller's buffer is [N][sp_dim]: 6 on the Aviary surface, 4 behind an env
    for (int k = 0; k < sp_dim; ++k) setpoint[(int64_t)sp_dim * i + k] = 0.0f;
}

// p.resetBasePositionAndOrientation / p.resetBaseVelocity + update_state (pfb_set_base_state; F32: pfb_set_base_velocity) and
// getBasePositionAndOrientation / getBaseVelocity (pfb_get_base_state)
template <bool F32>
__global__ void __launch_bounds__(kBlock) k_fw_set_base_state(const __grid_constant__ BaseStateIn a, float* __restrict__ st,
                                                              int32_t* __restrict__ ist, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  set_base_drone<F32>(PFB_KIND_FIXEDWING, a, st, ist, 0, N, i, i);
}
__global__ void __launch_bounds__(kBlock) k_fw_get_base_state(const __grid_constant__ BaseStateOut o, const float* __restrict__ st,
                                                              const int32_t* __restrict__ ist, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  fw_get_base_drone(st, ist, N, i, i, o);
}

// n_steps x Aviary.step() in flight mode MODE, or MODE = kModePerDrone: drone i in modes[i] (pfb_set_modes; only the command
// mapping branches on it).  CONTACT: the ground pushes back (Aviary handles with contact_response).  World = StaticCtx: against
// the static bodies of each drone's world (pfb_add_static_body), bits[i] = what drone i touched during its last Aviary step.
// Per-drone modes and static bodies exist on Aviary handles only, whose setpoints are 6 wide; one uniform mode reads sp_dim floats
// (4 behind Fixedwing-Waypoints).
template <int MODE, bool INJECT, bool CONTACT, class World>
__global__ void __launch_bounds__(kBlock, kMinBlocks)
    k_fw_aviary_step(const __grid_constant__ FixedwingParams p, const __grid_constant__ RngParams rng, const __grid_constant__ typename WorldTable<World>::T world,
                     const float* __restrict__ pose, uint32_t* __restrict__ bits, float* __restrict__ st, int32_t* __restrict__ ist,
                     const float* __restrict__ setpoint, const int8_t* __restrict__ modes, const float* __restrict__ noise, int n_steps,
                     uint32_t seq, int sp_dim, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  constexpr bool kPerDrone = MODE == kModePerDrone;
  World w{&world, pose, N, i, 0u};
  int mode = MODE;
  if constexpr (kPerDrone && !World::kOn) mode = modes[i];  // where the mode is read steers ptxas' schedule (DESIGN.md §4h)
  FixedwingRegs s;
  fixedwing_load(st, ist, N, i, s);
  if constexpr (kPerDrone || World::kOn) {
    load_setpoint<6, 6>(setpoint, i, s.sp);
  } else {
#pragma unroll
    for (int k = 0; k < 6; ++k) s.sp[k] = k < sp_dim ? __ldg(setpoint + (int64_t)sp_dim * i + k) : 0.0f;
  }
  if constexpr (kPerDrone && World::kOn) mode = modes[i];
  auto nz = make_noise<INJECT>(noise, N, i, rng, seq, TAG_AVIARY, p.noise_loc, p.ratio);
  if (fixedwing_full_model(p)) {  // launch-uniform: all surfaces, no wind -> the one-basic-block substep (pfb_fixedwing.cuh)
    for (int k = 0; k < n_steps; ++k) fixedwing_aviary_step_any<true, CONTACT>(p, s, mode, nz, &w);
  } else {
    for (int k = 0; k < n_steps; ++k) fixedwing_aviary_step_any<false, CONTACT>(p, s, mode, nz, &w);
  }
  fixedwing_store(st, ist, N, i, s);
  if constexpr (World::kOn) bits[i] = w.bits;
}

__global__ void __launch_bounds__(kBlock) k_fw_observe(const float* __restrict__ st, const int32_t* __restrict__ ist,
                                                       float* __restrict__ drone_state, float* __restrict__ aux,
                                                       uint8_t* __restrict__ contact, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  float o[12], a[6], hi[3], lo[3];
  const bool c = fw_query_drone(st, ist, N, i, o, a, hi, lo);
  if (drone_state)
    for (int k = 0; k < 12; ++k) drone_state[12 * i + k] = o[k];
  if (aux)
    for (int k = 0; k < 6; ++k) aux[6 * i + k] = a[k];
  if (contact) contact[i] = c ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------------
// Fixedwing-Waypoints epilogue
// ---------------------------------------------------------------------------------------------------
constexpr int kWpObsMax = 23 + 3 * kMaxTargets;
constexpr int kWpObsStride = kWpObsMax | 1;

// WaypointHandler.reset (waypoint_handler.py:53-83): polar sampling of the targets, on-device Philox stream
// Target words are addressed as tb[row * ts]: tb = st + i, ts = N for the field-major state tensor, tb = the env's spare
// record, ts = 1 while a spare is being built.
__device__ __forceinline__ void wp_sample_targets(const WaypointParams& w, const RngParams& rng, int64_t i, uint32_t seq,
                                                  float* __restrict__ tb, int64_t ts) {
  uint64_t g = ((uint64_t)rng.env_offset_hi << 32 | rng.env_offset_lo) + (uint64_t)i;
  for (int k = 0; k < w.num_targets; ++k) {
    U4 r = philox4x32_10(U4{(uint32_t)g, (uint32_t)(g >> 32), seq, (4u << 24) | (uint32_t)k}, rng.k0, rng.k1);
    float theta = 6.28318530717958647692f * u32_to_unit_open(r.x);
    float phi = 6.28318530717958647692f * u32_to_unit_open(r.y);
    float dist = 1.0f + (w.dome * 0.9f - 1.0f) * u32_to_unit_open(r.z);
    float st_, ct, sp, cp;
    sincos_f(theta, st_, ct);
    sincos_f(phi, sp, cp);
    float z = fabsf(dist * cp);
    tb[(int64_t)(FW_TARGETS + 3 * k + 0) * ts] = dist * sp * ct;
    tb[(int64_t)(FW_TARGETS + 3 * k + 1) * ts] = dist * sp * st_;
    tb[(int64_t)(FW_TARGETS + 3 * k + 2) * ts] = z > w.min_height ? z : w.min_height;
  }
}

struct WpState {
  float t0x, t0y, t0z;  // next target
  float new_dist;       // WaypointHandler.new_distance
  int first;            // targets reached so far == index of the next target (the list is never shifted)
  bool reached_now;     // a target was reached on the most recent Aviary step
};

__device__ __forceinline__ void wp_load_target0(const float* __restrict__ tb, int64_t ts, WpState& wp) {
  wp.t0x = tb[(int64_t)(FW_TARGETS + 3 * wp.first + 0) * ts];
  wp.t0y = tb[(int64_t)(FW_TARGETS + 3 * wp.first + 1) * ts];
  wp.t0z = tb[(int64_t)(FW_TARGETS + 3 * wp.first + 2) * ts];
}

// compute_state's waypoint part (waypoint_handler.py:120-157): old <- new, new <- |target0 - pos|
__device__ __forceinline__ float wp_update_distance(const FixedwingRegs& s, WpState& wp) {
  float old = wp.new_dist;
  float dx = wp.t0x - (float)s.px, dy = wp.t0y - (float)s.py, dz = wp.t0z - (float)s.pz;
  wp.new_dist = sqrtf(dx * dx + dy * dy + dz * dz);
  return old;
}

// fixedwing_base_env.py:226-244 + fixedwing_waypoints_env.py:169-190
__device__ __forceinline__ void wp_term_trunc_reward(const WaypointParams& w, FixedwingRegs& s, WpState& wp, float old_dist,
                                                     int step_count, float& reward, const float* __restrict__ tb, int64_t ts) {
  if (step_count > w.max_steps) s.flags |= FLAG_TRUNC;
  if (s.flags & FLAG_CONTACT_ARRAY) { reward = -100.0f; s.flags |= FLAG_COLLISION | FLAG_TERM; }
  float px = (float)s.px, py = (float)s.py, pz = (float)s.pz;
  if (px * px + py * py + pz * pz > w.dome2) { reward = -100.0f; s.flags |= FLAG_OOB | FLAG_TERM; }
  if (!w.sparse_reward) {
    float progress = (isinf(old_dist) || isinf(wp.new_dist)) ? 0.0f : old_dist - wp.new_dist;
    reward += fmaxf(3.0f * progress, 0.0f);
    reward += 1.0f / wp.new_dist;
  }
  wp.reached_now = false;
  if (wp.new_dist < w.goal_reach_distance) {  // target_reached (no yaw targets for the fixedwing)
    reward = 100.0f;
    wp.first += 1;  // advance_targets (waypoint_handler.py:176-185): the list head moves, nothing is copied
    wp.reached_now = true;
    if (wp.first == w.num_targets) s.flags |= FLAG_TRUNC | FLAG_ENV_COMPLETE;
    else wp_load_target0(tb, ts, wp);
  }
}

// compute_state (fixedwing_waypoints_env.py:121-167): attitude + action + aux + body-frame target deltas
__device__ __forceinline__ void wp_observation(const WaypointParams& w, const FixedwingRegs& s, const float* action, int first,
                                               const float* __restrict__ tb, int64_t ts, float* obs) {
  const float x = (float)s.qx, y = (float)s.qy, z = (float)s.qz, qw = (float)s.qw;
  float roll, pitch, yaw;
  euler_from_quat(x, y, z, qw, roll, pitch, yaw);
  int o = 0;
  obs[o++] = s.wx; obs[o++] = s.wy; obs[o++] = s.wz;
  if (w.angle_representation == 0) {
    obs[o++] = roll; obs[o++] = pitch; obs[o++] = yaw;
  } else {
    float ox, oy, oz, ow;
    quat_from_euler(roll, pitch, yaw, ox, oy, oz, ow);
    obs[o++] = ox; obs[o++] = oy; obs[o++] = oz; obs[o++] = ow;
  }
  obs[o++] = s.vb.x; obs[o++] = s.vb.y; obs[o++] = s.vb.z;
  obs[o++] = (float)s.px; obs[o++] = (float)s.py; obs[o++] = (float)s.pz;
  for (int k = 0; k < 4; ++k) obs[o++] = action[k];
  for (int k = 0; k < kMaxSurfaces; ++k) obs[o++] = s.act[k];
  obs[o++] = s.thr;
  // target_deltas = (targets - lin_pos) @ R  (waypoint_handler.py:139-142): body-frame deltas
  const Rot<fwreal>& R = s.R;
  for (int k = 0; k < w.num_targets; ++k) {
    float bx = 0.f, by = 0.f, bz = 0.f;
    if (first + k < w.num_targets) {  // remaining targets first, zero padding after
      float dx = tb[(int64_t)(FW_TARGETS + 3 * (first + k) + 0) * ts] - (float)s.px;
      float dy = tb[(int64_t)(FW_TARGETS + 3 * (first + k) + 1) * ts] - (float)s.py;
      float dz = tb[(int64_t)(FW_TARGETS + 3 * (first + k) + 2) * ts] - (float)s.pz;
      bx = (float)R.m00 * dx + (float)R.m10 * dy + (float)R.m20 * dz;
      by = (float)R.m01 * dx + (float)R.m11 * dy + (float)R.m21 * dz;
      bz = (float)R.m02 * dx + (float)R.m12 * dy + (float)R.m22 * dz;
    }
    obs[o++] = bx; obs[o++] = by; obs[o++] = bz;
  }
}

// env.reset() for one env (fixedwing_waypoints_env.py:102-119, fixedwing_base_env.py:126-192); `pose` = the 6 start-pose
// words the caller read (and, when building a spare, recorded), targets go to tb / ts
template <bool INJECT>
__device__ __forceinline__ void wp_reset_env(const FixedwingParams& p, const WaypointParams& w, const RngParams& rng, const float* pose,
                                             const float* __restrict__ reset_targets, const float* __restrict__ noise, uint32_t seq,
                                             int64_t N, int64_t i, float* __restrict__ tb, int64_t ts, FixedwingRegs& s, WpState& wp) {
  fixedwing_reset(p, s, pose[0], pose[1], pose[2], pose[3], pose[4], pose[5]);
  if (reset_targets) {
    for (int k = 0; k < 3 * w.num_targets; ++k) tb[(int64_t)(FW_TARGETS + k) * ts] = reset_targets[(int64_t)i * 3 * w.num_targets + k];
  } else {
    wp_sample_targets(w, rng, i, seq, tb, ts);
  }
  wp.first = 0;
  wp.reached_now = false;
  wp.new_dist = INFINITY;
  wp_load_target0(tb, ts, wp);
  auto nz = make_noise<INJECT>(noise, N, i, rng, seq, TAG_RESET, p.noise_loc, p.ratio);
  for (int k = 0; k < w.warmup_steps; ++k) fixedwing_aviary_step<0>(p, s, nz);
  fixedwing_requantize(s);             // exactly what the state tensor / a spare record will hold
  (void)wp_update_distance(s, wp);     // end_reset -> compute_state
}

// ---- spare post-reset states (pfb_tail_step.cuh): a record holds the FW_* state words INCLUDING the episode's targets and
// new_distance
enum { WSP_ROWS = 64 };

// the Fixedwing-Waypoints env for tail_step (pfb_tail_step.cuh)
template <bool INJECT, bool RANDACT>
struct WpEnv {
  const FixedwingParams& p;
  const WaypointParams& w;
  const RngParams& rng;
  using Regs = FixedwingRegs;
  using Item = WpState;
  static constexpr int kStateRows = FW_ROWS, kSpareRows = WSP_ROWS, kActions = 4, kObsStride = kWpObsStride;
  __device__ __forceinline__ int obs_dim() const { return (w.angle_representation == 0 ? 22 : 23) + 3 * w.num_targets; }
  __device__ __forceinline__ bool pose_keyed() const { return true; }
  __device__ __forceinline__ WpState item(int64_t) const {
    WpState wp;
    return wp;
  }
  // a spare's targets are copied into the state rows: the episode starts at target 0
  __device__ __forceinline__ void load_spare(const float* __restrict__ rec, float* __restrict__ st, int32_t* __restrict__ ist, int64_t N,
                                             int64_t i, FixedwingRegs& s, WpState& wp) const {
    fixedwing_load(rec, ist, N, i, s, 1, 0);
    float* tb = st + i;
    for (int k = 0; k < 3 * w.num_targets; ++k) tb[(int64_t)(FW_TARGETS + k) * N] = rec[FW_TARGETS + k];
    wp.first = 0;
    wp.reached_now = false;
    wp.new_dist = rec[FW_DIST];
  }
  // the targets go to the spare record being built, or to the state rows
  __device__ __forceinline__ void reset(const float* pose, uint32_t nseq, float* __restrict__ rec, float* __restrict__ st, int64_t N, int64_t i,
                                        FixedwingRegs& s, WpState& wp) const {
    wp_reset_env<false>(p, w, rng, pose, nullptr, nullptr, nseq, N, i, rec ? rec : st + i, rec ? 1 : N, s, wp);
  }
  __device__ __forceinline__ void store_spare(float* __restrict__ rec, int32_t* __restrict__ ist, int64_t N, int64_t i, const FixedwingRegs& s,
                                              const WpState& wp) const {
    fixedwing_store(rec, ist, N, i, s, false, 1, 0);
    rec[FW_DIST] = wp.new_dist;
  }
  __device__ __forceinline__ void load(const float* __restrict__ st, const int32_t* __restrict__ ist, int64_t N, int64_t i, FixedwingRegs& s) const {
    fixedwing_load(st, ist, N, i, s);
  }
  __device__ __forceinline__ void action(float* __restrict__ actions, int64_t i, uint32_t step_seq, float* act) const {
    if (RANDACT) {
      fixedwing_random_action(rng, i, step_seq, act);
      reinterpret_cast<float4*>(actions)[i] = make_float4(act[0], act[1], act[2], act[3]);
    } else {
      float4 a4 = __ldg(reinterpret_cast<const float4*>(actions) + i);
      act[0] = a4.x; act[1] = a4.y; act[2] = a4.z; act[3] = a4.w;
    }
  }
  __device__ __forceinline__ void step(const float* __restrict__ st, const int32_t* __restrict__ ist, const float* __restrict__ noise, int64_t N,
                                       int64_t i, uint32_t step_seq, const float* act, FixedwingRegs& s, WpState& wp, int& step_count,
                                       float& rew) const {
    // fixedwing_base_env.py:257-261: the throttle channel is remapped from [-1, 1] to [0, 1]
    s.sp[0] = act[0]; s.sp[1] = act[1]; s.sp[2] = act[2]; s.sp[3] = act[3] * 0.5f + 0.5f;
    step_count = ist[(int64_t)FI_STEP * N + i];
    wp.first = ist[(int64_t)FI_NTARGETS * N + i];
    wp.reached_now = false;
    wp.new_dist = st[(int64_t)FW_DIST * N + i];
    wp_load_target0(st + i, N, wp);
    rew = -0.1f;
    auto nz = make_noise<INJECT>(noise, N, i, rng, step_seq, TAG_ENV_STEP, p.noise_loc, p.ratio);
    const bool full = fixedwing_full_model(p);
#pragma unroll 1
    for (int k = 0; k < w.env_step_ratio; ++k) {
      if (s.flags & (FLAG_TERM | FLAG_TRUNC)) break;
      if (full) fixedwing_aviary_step<0, true>(p, s, nz);
      else fixedwing_aviary_step<0>(p, s, nz);
      float old = wp_update_distance(s, wp);
      wp_term_trunc_reward(w, s, wp, old, step_count, rew, st + i, N);
    }
    step_count += 1;
  }
  // the reference builds the observation in compute_state, BEFORE compute_term_trunc_reward advances the
  // target list: a target reached on the last Aviary step is still the head of the reported list
  __device__ __forceinline__ void observe(const float* __restrict__ st, int64_t N, int64_t i, const float* act, const FixedwingRegs& s,
                                          const WpState& wp, float* row) const {
    wp_observation(w, s, act, wp.first - (wp.reached_now ? 1 : 0), st + i, N, row);
  }
  __device__ __forceinline__ void store(float* __restrict__ st, int32_t* __restrict__ ist, int64_t N, int64_t i, const FixedwingRegs& s,
                                        const WpState& wp, int step_count) const {
    fixedwing_store(st, ist, N, i, s);
    st[(int64_t)FW_DIST * N + i] = wp.new_dist;
    ist[(int64_t)FI_STEP * N + i] = step_count;
    ist[(int64_t)FI_NTARGETS * N + i] = wp.first;
  }
  __device__ __forceinline__ uint8_t info(const FixedwingRegs& s, const WpState& wp) const {
    return (uint8_t)(((s.flags & FLAG_OOB) ? 1 : 0) | ((s.flags & FLAG_COLLISION) ? 2 : 0) | ((s.flags & FLAG_ENV_COMPLETE) ? 4 : 0) |
                     (wp.first << 3));
  }
};

template <bool INJECT, bool RANDACT, bool AUTORESET>
__global__ void __launch_bounds__(kBlock, kAeroBlocks)
    k_fwwp_step(const __grid_constant__ FixedwingParams p, const __grid_constant__ WaypointParams w,
                const __grid_constant__ RngParams rng, float* __restrict__ st, int32_t* __restrict__ ist,
                float* __restrict__ actions, const float* __restrict__ noise, float* __restrict__ obs, float* __restrict__ reward,
                uint8_t* __restrict__ term, uint8_t* __restrict__ trunc, uint8_t* __restrict__ info,
                const float* __restrict__ start_pos, const float* __restrict__ start_orn, const int32_t* __restrict__ prev_count,
                const int32_t* __restrict__ prev_list, int32_t* __restrict__ cur_count, int32_t* __restrict__ cur_list,
                int32_t* __restrict__ next_count, float* __restrict__ spare, int spare_copy, int build, int tail_blocks,
                uint32_t step_seq, int64_t N) {
  tail_step<AUTORESET>(WpEnv<INJECT, RANDACT>{p, w, rng}, st, ist, actions, noise, obs, reward, term, trunc, info, start_pos, start_orn,
                       prev_count, prev_list, cur_count, cur_list, next_count, spare, spare_copy, build, tail_blocks, step_seq, N);
}
// SAME_STEP autoreset: a finishing env is reset in this launch (tail_step_same)
template <bool RANDACT>
__global__ void __launch_bounds__(kBlock, kAeroBlocks)
    k_fwwp_step_same(const __grid_constant__ FixedwingParams p, const __grid_constant__ WaypointParams w, const __grid_constant__ RngParams rng,
                     float* __restrict__ st, int32_t* __restrict__ ist, float* __restrict__ actions, float* __restrict__ obs,
                     float* __restrict__ final_obs, float* __restrict__ reward, uint8_t* __restrict__ term, uint8_t* __restrict__ trunc,
                     uint8_t* __restrict__ info, const float* __restrict__ start_pos, const float* __restrict__ start_orn,
                     int32_t* __restrict__ cur_count, int32_t* __restrict__ cur_list, int32_t* __restrict__ next_count,
                     const float* __restrict__ spare, int spare_copy, uint32_t step_seq, int64_t N) {
  tail_step_same(WpEnv<false, RANDACT>{p, w, rng}, st, ist, actions, nullptr, obs, final_obs, reward, term, trunc, info, start_pos, start_orn,
                 cur_count, cur_list, next_count, spare, spare_copy, step_seq, N);
}

template <bool INJECT>
__global__ void __launch_bounds__(kBlock)
    k_fwwp_reset(const __grid_constant__ FixedwingParams p, const __grid_constant__ WaypointParams w,
                 const __grid_constant__ RngParams rng, float* __restrict__ st, int32_t* __restrict__ ist,
                 const float* __restrict__ start_pos, const float* __restrict__ start_orn, const float* __restrict__ reset_targets,
                 const uint8_t* __restrict__ mask, const float* __restrict__ noise, float* __restrict__ obs, uint32_t seq, int64_t N) {
  __shared__ float smem[kBlock * kWpObsStride];
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  if (i >= N) return;
  if (mask && !mask[i]) return;
  const int O = (w.angle_representation == 0 ? 22 : 23) + 3 * w.num_targets;
  FixedwingRegs s;
  WpState wp;
  const float pose[6] = {start_pos[3 * i], start_pos[3 * i + 1], start_pos[3 * i + 2], start_orn[3 * i], start_orn[3 * i + 1], start_orn[3 * i + 2]};
  wp_reset_env<INJECT>(p, w, rng, pose, reset_targets, noise, seq, N, i, st + i, N, s, wp);
  const float zero[4] = {0.f, 0.f, 0.f, 0.f};
  float* row = smem + threadIdx.x * kWpObsStride;
  wp_observation(w, s, zero, wp.first, st + i, N, row);
  fixedwing_store(st, ist, N, i, s);
  st[(int64_t)FW_DIST * N + i] = wp.new_dist;
  ist[(int64_t)FI_STEP * N + i] = 0;
  ist[(int64_t)FI_NTARGETS * N + i] = wp.first;
  if (obs)
    for (int k = 0; k < O; ++k) obs[i * O + k] = row[k];
}

// ---------------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------------
int fw_reset(PfbContext* h, const uint8_t* mask, cudaStream_t s) {
  k_fw_reset<<<grid_for(h->n), kBlock, 0, s>>>(h->fw, h->buf.state, h->buf.istate, h->buf.setpoint, h->buf.start_pos,
                                               h->buf.start_orn, mask, fw_setpoint_dim(h), h->n);
  LAUNCH_CHECK(h);
  if (!mask) h->mode = 0;
  return 0;
}

int fw_set_mode(PfbContext* h, int mode, cudaStream_t s) {
  const int lo = kModeLo[PFB_KIND_FIXEDWING], hi = kModeHi[PFB_KIND_FIXEDWING];
  if (mode < lo || mode > hi)  // the message of fixedwing.py:216-219
    return fail("`mode` must be between %d and %d or be registered in self.registered_controllers.keys()=dict_keys([]), got %d.", lo, hi, mode);
  if (mode == -1 && fw_setpoint_dim(h) < 6) return fail("mode -1 needs the 6-wide setpoint buffer of the Aviary surface");
  CUDA_OK(cudaMemsetAsync(h->buf.setpoint, 0, (size_t)h->n * fw_setpoint_dim(h) * sizeof(float), s));  // fixedwing.py:224-227
  h->mode = mode;
  return 0;
}

static int fw_set_modes(PfbContext* h, const int8_t*, cudaStream_t s) {
  CUDA_OK(cudaMemsetAsync(h->buf.setpoint, 0, (size_t)h->n * fw_setpoint_dim(h) * sizeof(float), s));  // every drone's set_mode
  h->mode = kModePerDrone;
  return 0;
}

int fw_aviary_step(PfbContext* h, int n_steps, const float* noise, cudaStream_t s) {
  const uint32_t seq = (uint32_t)h->aviary_seq++;
  return aviary_step_launch(h, noise, [&](auto v) {
    using V = decltype(v);
    auto launch = [&](auto mode) {
      k_fw_aviary_step<decltype(mode)::value, V::inject, V::contact, typename V::world><<<grid_for(h->n), kBlock, 0, s>>>(
          h->fw, h->rng, world_table(v), v.pose(), v.bits(), h->buf.state, h->buf.istate, h->buf.setpoint, h->d_modes, noise, n_steps, seq,
          fw_setpoint_dim(h), h->n);
      return 0;
    };
    if (h->mode == kModePerDrone) return launch(std::integral_constant<int, kModePerDrone>{});
    return h->mode == 0 ? launch(std::integral_constant<int, 0>{}) : launch(std::integral_constant<int, -1>{});
  });
}

static int fw_set_base_state(PfbContext* h, const BaseStateIn& a, cudaStream_t s) {
  if (a.lin32 || a.ang32) k_fw_set_base_state<true><<<grid_for(h->n), kBlock, 0, s>>>(a, h->buf.state, h->buf.istate, h->n);
  else k_fw_set_base_state<false><<<grid_for(h->n), kBlock, 0, s>>>(a, h->buf.state, h->buf.istate, h->n);
  LAUNCH_CHECK(h);
  return 0;
}

static int fw_get_base_state(PfbContext* h, const BaseStateOut& o, cudaStream_t s) {
  k_fw_get_base_state<<<grid_for(h->n), kBlock, 0, s>>>(o, h->buf.state, h->buf.istate, h->n);
  LAUNCH_CHECK(h);
  return 0;
}

int fw_observe(PfbContext* h, cudaStream_t s) {
  k_fw_observe<<<grid_for(h->n), kBlock, 0, s>>>(h->buf.state, h->buf.istate, h->buf.drone_state, h->buf.aux_state, h->buf.contact, h->n);
  LAUNCH_CHECK(h);
  return 0;
}

// one launch of k_fwwp_step for tail_env_step / tail_env_reset
static auto fwwp_launcher(PfbContext* h, float* actions, const float* noise) {
  return [=](auto v, const TailLaunch& L) -> int {
    using V = decltype(v);
    if constexpr (V::same) {
      k_fwwp_step_same<V::randact><<<L.grid, kBlock, 0, L.stream>>>(h->fw, h->wp, h->rng, h->buf.state, h->buf.istate, actions, h->buf.obs,
                                                                    h->buf.final_obs, h->buf.reward, h->buf.term, h->buf.trunc, h->buf.info,
                                                                    h->buf.start_pos, h->buf.start_orn, L.cur_count, L.cur_list, L.next_count,
                                                                    L.spare, L.spare_copy, L.seq, h->n);
      return 0;
    }
    k_fwwp_step<V::inject, V::randact, V::autoreset><<<L.grid, kBlock, 0, L.stream>>>(
        h->fw, h->wp, h->rng, h->buf.state, h->buf.istate, actions, noise, h->buf.obs, h->buf.reward, h->buf.term, h->buf.trunc, h->buf.info,
        h->buf.start_pos, h->buf.start_orn, L.prev_count, L.prev_list, L.cur_count, L.cur_list, L.next_count, L.spare, L.spare_copy, L.build,
        L.tail_blocks, L.seq, h->n);
    return 0;
  };
}

static int fw_env_reset(PfbContext* h, const uint8_t* mask, const float* noise, cudaStream_t s) {
  const uint32_t seq = 0x80000000u | (uint32_t)h->reset_seq++;
  auto reset = [&](int g) -> int {
    if (noise)
      k_fwwp_reset<true><<<g, kBlock, 0, s>>>(h->fw, h->wp, h->rng, h->buf.state, h->buf.istate, h->buf.start_pos, h->buf.start_orn,
                                              h->buf.reset_targets, mask, noise, h->buf.obs, seq, h->n);
    else
      k_fwwp_reset<false><<<g, kBlock, 0, s>>>(h->fw, h->wp, h->rng, h->buf.state, h->buf.istate, h->buf.start_pos, h->buf.start_orn,
                                               h->buf.reset_targets, mask, nullptr, h->buf.obs, seq, h->n);
    return 0;
  };
  if (tail_env_reset(h, mask, s, reset, fwwp_launcher(h, h->buf.setpoint, nullptr))) return -1;
  h->mode = 0;
  return 0;
}

static int fw_env_step(PfbContext* h, float* actions, const float* noise, bool randact, size_t, cudaStream_t s) {
  return tail_env_step(h, noise, randact, s, fwwp_launcher(h, actions, noise));
}

const HandleOps kFixedwingAviaryOps = {
    .kind = PFB_KIND_FIXEDWING, .env_kind = PFB_ENV_NONE,
    .state_rows = FW_ROWS, .istate_rows = FI_ROWS, .layout = PFB_LAYOUT_FIELD_MAJOR, .setpoint_dim = 6, .aux_dim = 6,
    .obs_dim = fw_obs_dim,
    .reset = fw_reset, .set_mode = fw_set_mode, .set_modes = fw_set_modes, .aviary_step = fw_aviary_step, .observe = fw_observe,
    .set_base_state = fw_set_base_state, .get_base_state = fw_get_base_state,
};

const HandleOps kFixedwingWaypointsOps = {
    .kind = PFB_KIND_FIXEDWING, .env_kind = PFB_ENV_FIXEDWING_WAYPOINTS,
    .state_rows = FW_ROWS, .istate_rows = FI_ROWS, .layout = PFB_LAYOUT_FIELD_MAJOR, .setpoint_dim = 4, .aux_dim = 6,
    .obs_dim = fw_obs_dim,
    .reset = fw_reset, .set_mode = fw_set_mode, .aviary_step = fw_aviary_step, .observe = fw_observe,
    .env_reset = fw_env_reset, .env_step = fw_env_step,
    .spare_rows = WSP_ROWS, .spare_valid_row = FW_ROWS + SPARE_VALID,
    .invalidate_spares = tail_invalidate_spares,
};
