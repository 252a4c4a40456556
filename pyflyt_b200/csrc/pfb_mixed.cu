// pfb_mixed.cu — Aviary handles whose drones are of several vehicle kinds (pfb_create_mixed; the reference's
// Aviary(drone_type=[...]), aviary.py:139-190): QuadX, fixed-wing and rocket drones stepped by ONE launch.
//
// The handle groups its drones by kind, in stable order: slot t of the kind-grouped order is drone slot_user[t] of the
// caller's order, the QuadX slots first, then the fixed-wing ones, then the rocket ones.  Each kind present has its own region
// of the one state buffer the caller binds, in that kind's own layout (QuadX warp-tiled, fixed-wing and rocket field-major), and
// flies the handle's own tables (qx or qxset, fw, rk), so the wind, reseed, bind, launch-count and destroy entry points serve it
// through their ordinary code.  The step, the state query, the reset and the mode changes are one launch each over all kinds:
// a one-warp CTA takes its kind from its block range, so a warp never diverges by kind, and runs its kind's per-drone body
// (pfb_aviary.cuh) with the user index of its slot.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <new>

#include "pfb_aviary.cuh"

using namespace pfb;

namespace {

constexpr int kKinds = 3;               // PFB_KIND_QUADX, PFB_KIND_FIXEDWING, PFB_KIND_ROCKET
constexpr int kMixedSetpointDim = 7;    // the widest kind (rocket): the caller's setpoint buffer is [N][7]
constexpr int kMixedAuxDim = 9;         // rocket again: the aux buffer is [N][9], zero past a drone's own aux length
constexpr int kMixedPosDim = 6;         // obs buffer of a mixed handle: [N][6] = position hi words, lo words
constexpr int64_t kRegionAlign = 32;    // floats: every kind's state region starts on a 128-byte boundary

}  // namespace

struct MixedKinds {
  int64_t count[kKinds];     // drones of each kind
  int64_t first[kKinds + 1]; // first slot of each kind in the kind-grouped order; first[kKinds] = n
  int32_t* d_slot_user;      // [n] slot -> user index
  int8_t* d_slot_mode;       // [n] flight mode of each slot
  int8_t* h_slot_mode;       // [n] pfb_set_modes' modes in slot order, on their way to d_slot_mode
  uint8_t* h_kind;           // [n] kind of each user drone
  // several control rates (PfbEnvConfig::mixed_control_hz): physics substeps per Aviary step, and the control ratio
  // physics_hz / control_hz of each slot (a divisor of U); d_slot_ratio = nullptr when every drone runs at one rate
  int U;
  uint8_t* d_slot_ratio;
};

// ---------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------
// Where the drones of each kind live: their state regions, the slot -> user map, and the CTA ranges of a launch over all kinds
struct MixedRows {
  float* qx_st;                 // QuadX region, warp-tiled
  float *fw_st, *rk_st;         // fixed-wing and rocket regions, field-major [F][count]
  int32_t *fw_ist, *rk_ist;
  const int32_t* slot_user;
  int64_t n_qx, n_fw, n_rk;
  int cta_qx, cta_fw;           // CTAs of the QuadX range and of the fixed-wing range; the rocket CTAs follow
};

// setpoint floats of each kind; a mixed handle's [N][7] rows are zero past them
__device__ __forceinline__ int kind_setpoint_dim(int kind) { return kind == 0 ? 4 : (kind == 1 ? 6 : 7); }

// The kind of this CTA's block range and this thread's row j of it; -1 past the kind's last drone (the reset and set_mode
// kernels; the step and the state query branch on the block range themselves, which keeps their code as it was)
__device__ __forceinline__ int mixed_row(const MixedRows& r, int64_t& j) {
  const int b = blockIdx.x;
  if (b < r.cta_qx) {
    j = (int64_t)b * kBlock + threadIdx.x;
    return j < r.n_qx ? 0 : -1;
  }
  if (b < r.cta_qx + r.cta_fw) {
    j = (int64_t)(b - r.cta_qx) * kBlock + threadIdx.x;
    return j < r.n_fw ? 1 : -1;
  }
  j = (int64_t)(b - r.cta_qx - r.cta_fw) * kBlock + threadIdx.x;
  return j < r.n_rk ? 2 : -1;
}

// Everything one launch of the mixed step reads.  PS: the QuadX coefficient table (QuadXParams, or QuadXModelSet when the
// QuadX drones fly several models; its index is in QuadX slot order).
template <class PS>
struct MixedStep {
  PS qx;
  FixedwingParams fw;
  RocketParams rk;
  RngParams rng;
  MixedRows r;
  const int8_t* slot_mode;
  const float* setpoint;        // [n][7], user order
  const float* noise;           // [n_steps * ratio][n], user order; nullptr = Philox
  int64_t n;
  int n_steps;
  uint32_t seq;
  const uint8_t* slot_ratio;    // RATES: [n] control ratio of each slot
  int U;                        // RATES: physics substeps per Aviary step
};
// the whole argument travels in the kernel-parameter bank, which holds 32 764 bytes on sm_90
static_assert(sizeof(MixedStep<QuadXModelSet>) <= 32764, "the mixed step's __grid_constant__ argument exceeds the kernel-parameter limit");

// n_steps x Aviary.step() for every drone of a mixed handle.  Drone u draws the noise of drone u of a uniform handle of its
// kind (Philox counter keyed by the USER index, injected column u), and runs the per-drone-mode step of its kind, so each
// drone's trajectory is bit-equal to the one it flies in a uniform handle with the same seed.  CONTACT: the floor pushes back.
// RATES (a handle whose drones run at several control rates): every drone runs the handle's U substeps per Aviary step and
// its control tick on the substeps that are multiples of its slot's ratio; its noise is keyed with U, whatever its own ratio.
// The branches spell out the step bodies of pfb_aviary.cuh rather than call them: called, their pointers and counts are held
// in registers across the step loop instead of being read from the parameter bank where they are used, and the kernel needs
// more stack.
template <bool INJECT, bool CONTACT, bool RATES, class PS>
__global__ void __launch_bounds__(kBlock, kMinBlocks) k_mixed_aviary_step(const __grid_constant__ MixedStep<PS> a) {
  const MixedRows& r = a.r;
  const int b = blockIdx.x;
  if (b < r.cta_qx) {
    const int64_t j = (int64_t)b * kBlock + threadIdx.x;
    if (j >= r.n_qx) return;
    const int64_t u = r.slot_user[j];
    const QuadXParams& p = qx_model(a.qx, j);
    const int mode = a.slot_mode[j];
    QuadXRegs s;
    int step_count;
    quadx_load_tile<7, kTileGroupStride>(r.qx_st + qx_tile_base(j, QX_ROWS), s, step_count);
    quadx_mask_pid(s, mode);
#pragma unroll
    for (int c = 0; c < 4; ++c) s.sp[c] = __ldg(a.setpoint + kMixedSetpointDim * u + c);
    if constexpr (RATES) {
      const int ratio = a.slot_ratio[j];
      auto nz = make_noise<INJECT>(a.noise, a.n, u, a.rng, a.seq, TAG_AVIARY, qx_model0(a.qx).noise_loc, a.U);
      for (int k = 0; k < a.n_steps; ++k) quadx_aviary_step_rates<CONTACT>(p, s, mode, ratio, a.U, nz);
    } else {
      auto nz = make_noise<INJECT>(a.noise, a.n, u, a.rng, a.seq, TAG_AVIARY, qx_model0(a.qx).noise_loc, qx_model0(a.qx).ratio);
      for (int k = 0; k < a.n_steps; ++k) quadx_aviary_step_any<CONTACT>(p, s, mode, nz);
    }
    quadx_store_tile<7, kTileGroupStride>(r.qx_st + qx_tile_base(j, QX_ROWS), s, step_count);
  } else if (b < r.cta_qx + r.cta_fw) {
    const int64_t j = (int64_t)(b - r.cta_qx) * kBlock + threadIdx.x;
    if (j >= r.n_fw) return;
    const int64_t u = r.slot_user[r.n_qx + j];
    const int mode = a.slot_mode[r.n_qx + j];
    const FixedwingParams& p = a.fw;
    FixedwingRegs s;
    fixedwing_load(r.fw_st, r.fw_ist, r.n_fw, j, s);
#pragma unroll
    for (int c = 0; c < 6; ++c) s.sp[c] = __ldg(a.setpoint + kMixedSetpointDim * u + c);
    if constexpr (RATES) {
      const int ratio = a.slot_ratio[r.n_qx + j];
      auto nz = make_noise<INJECT>(a.noise, a.n, u, a.rng, a.seq, TAG_AVIARY, p.noise_loc, a.U);
      if (fixedwing_full_model(p)) {
        for (int k = 0; k < a.n_steps; ++k) fixedwing_aviary_step_rates<true, CONTACT>(p, s, mode, ratio, a.U, nz);
      } else {
        for (int k = 0; k < a.n_steps; ++k) fixedwing_aviary_step_rates<false, CONTACT>(p, s, mode, ratio, a.U, nz);
      }
    } else {
      auto nz = make_noise<INJECT>(a.noise, a.n, u, a.rng, a.seq, TAG_AVIARY, p.noise_loc, p.ratio);
      if (fixedwing_full_model(p)) {
        for (int k = 0; k < a.n_steps; ++k) fixedwing_aviary_step_any<true, CONTACT>(p, s, mode, nz);
      } else {
        for (int k = 0; k < a.n_steps; ++k) fixedwing_aviary_step_any<false, CONTACT>(p, s, mode, nz);
      }
    }
    fixedwing_store(r.fw_st, r.fw_ist, r.n_fw, j, s);
  } else {
    const int64_t j = (int64_t)(b - r.cta_qx - r.cta_fw) * kBlock + threadIdx.x;
    if (j >= r.n_rk) return;
    const int64_t u = r.slot_user[r.n_qx + r.n_fw + j];
    const RocketParams& p = a.rk;
    RocketRegs s;
    rocket_load(r.rk_st, r.rk_ist, r.n_rk, j, s);
#pragma unroll
    for (int c = 0; c < 7; ++c) s.sp[c] = __ldg(a.setpoint + kMixedSetpointDim * u + c);
    if constexpr (RATES) {
      const int ratio = a.slot_ratio[r.n_qx + r.n_fw + j];
      auto nz = make_noise<INJECT>(a.noise, a.n, u, a.rng, a.seq, TAG_AVIARY, p.noise_loc, a.U);
      for (int k = 0; k < a.n_steps; ++k) rocket_aviary_step_rates(p, s, ratio, a.U, nz);
    } else {
      auto nz = make_noise<INJECT>(a.noise, a.n, u, a.rng, a.seq, TAG_AVIARY, p.noise_loc, p.ratio);
      for (int k = 0; k < a.n_steps; ++k) rocket_aviary_step(p, s, nz, false);
    }
    rocket_store(r.rk_st, r.rk_ist, r.n_rk, j, s);
  }
}

// The body of k_mixed_aviary_step with the static bodies of drone u's world, whose bits go to bits[u].  A
// copy rather than a shared body, so that k_mixed_aviary_step stays the code it was.
template <bool INJECT, bool CONTACT, bool RATES, class PS>
__device__ __forceinline__ void mixed_aviary_step_static(const MixedStep<PS>& a, const StaticWorld* world, const float* pose, uint32_t* bits) {
  const MixedRows& r = a.r;
  const int b = blockIdx.x;
  if (b < r.cta_qx) {
    const int64_t j = (int64_t)b * kBlock + threadIdx.x;
    if (j >= r.n_qx) return;
    const int64_t u = r.slot_user[j];
    StaticCtx w{world, pose, a.n, u, 0u};
    const QuadXParams& p = qx_model(a.qx, j);
    const int mode = a.slot_mode[j];
    QuadXRegs s;
    int step_count;
    quadx_load_tile<7, kTileGroupStride>(r.qx_st + qx_tile_base(j, QX_ROWS), s, step_count);
    quadx_mask_pid(s, mode);
#pragma unroll
    for (int c = 0; c < 4; ++c) s.sp[c] = __ldg(a.setpoint + kMixedSetpointDim * u + c);
    if constexpr (RATES) {
      const int ratio = a.slot_ratio[j];
      auto nz = make_noise<INJECT>(a.noise, a.n, u, a.rng, a.seq, TAG_AVIARY, qx_model0(a.qx).noise_loc, a.U);
      for (int k = 0; k < a.n_steps; ++k) quadx_aviary_step_rates<CONTACT>(p, s, mode, ratio, a.U, nz, &w);
    } else {
      auto nz = make_noise<INJECT>(a.noise, a.n, u, a.rng, a.seq, TAG_AVIARY, qx_model0(a.qx).noise_loc, qx_model0(a.qx).ratio);
      for (int k = 0; k < a.n_steps; ++k) quadx_aviary_step_any<CONTACT>(p, s, mode, nz, &w);
    }
    quadx_store_tile<7, kTileGroupStride>(r.qx_st + qx_tile_base(j, QX_ROWS), s, step_count);
    bits[u] = w.bits;
  } else if (b < r.cta_qx + r.cta_fw) {
    const int64_t j = (int64_t)(b - r.cta_qx) * kBlock + threadIdx.x;
    if (j >= r.n_fw) return;
    const int64_t u = r.slot_user[r.n_qx + j];
    StaticCtx w{world, pose, a.n, u, 0u};
    const int mode = a.slot_mode[r.n_qx + j];
    const FixedwingParams& p = a.fw;
    FixedwingRegs s;
    fixedwing_load(r.fw_st, r.fw_ist, r.n_fw, j, s);
#pragma unroll
    for (int c = 0; c < 6; ++c) s.sp[c] = __ldg(a.setpoint + kMixedSetpointDim * u + c);
    if constexpr (RATES) {
      const int ratio = a.slot_ratio[r.n_qx + j];
      auto nz = make_noise<INJECT>(a.noise, a.n, u, a.rng, a.seq, TAG_AVIARY, p.noise_loc, a.U);
      if (fixedwing_full_model(p)) {
        for (int k = 0; k < a.n_steps; ++k) fixedwing_aviary_step_rates<true, CONTACT>(p, s, mode, ratio, a.U, nz, &w);
      } else {
        for (int k = 0; k < a.n_steps; ++k) fixedwing_aviary_step_rates<false, CONTACT>(p, s, mode, ratio, a.U, nz, &w);
      }
    } else {
      auto nz = make_noise<INJECT>(a.noise, a.n, u, a.rng, a.seq, TAG_AVIARY, p.noise_loc, p.ratio);
      if (fixedwing_full_model(p)) {
        for (int k = 0; k < a.n_steps; ++k) fixedwing_aviary_step_any<true, CONTACT>(p, s, mode, nz, &w);
      } else {
        for (int k = 0; k < a.n_steps; ++k) fixedwing_aviary_step_any<false, CONTACT>(p, s, mode, nz, &w);
      }
    }
    fixedwing_store(r.fw_st, r.fw_ist, r.n_fw, j, s);
    bits[u] = w.bits;
  } else {
    const int64_t j = (int64_t)(b - r.cta_qx - r.cta_fw) * kBlock + threadIdx.x;
    if (j >= r.n_rk) return;
    const int64_t u = r.slot_user[r.n_qx + r.n_fw + j];
    StaticCtx w{world, pose, a.n, u, 0u};
    const RocketParams& p = a.rk;
    RocketRegs s;
    rocket_load(r.rk_st, r.rk_ist, r.n_rk, j, s);
#pragma unroll
    for (int c = 0; c < 7; ++c) s.sp[c] = __ldg(a.setpoint + kMixedSetpointDim * u + c);
    if constexpr (RATES) {
      const int ratio = a.slot_ratio[r.n_qx + r.n_fw + j];
      auto nz = make_noise<INJECT>(a.noise, a.n, u, a.rng, a.seq, TAG_AVIARY, p.noise_loc, a.U);
      for (int k = 0; k < a.n_steps; ++k) rocket_aviary_step_rates(p, s, ratio, a.U, nz, &w);
    } else {
      auto nz = make_noise<INJECT>(a.noise, a.n, u, a.rng, a.seq, TAG_AVIARY, p.noise_loc, p.ratio);
      for (int k = 0; k < a.n_steps; ++k) rocket_aviary_step(p, s, nz, false, &w);
    }
    rocket_store(r.rk_st, r.rk_ist, r.n_rk, j, s);
    bits[u] = w.bits;
  }
}

// k_mixed_aviary_step against the static bodies of each drone's world (pfb_add_static_body); bits[u]: what drone u touched during
// its last Aviary step
template <bool INJECT, bool CONTACT, bool RATES, class PS>
__global__ void __launch_bounds__(kBlock, kMinBlocks)
    k_mixed_aviary_step_static(const __grid_constant__ MixedStep<PS> a, const __grid_constant__ StaticWorld world, const float* __restrict__ pose,
                               uint32_t* __restrict__ bits) {
  mixed_aviary_step_static<INJECT, CONTACT, RATES, PS>(a, &world, pose, bits);
}

struct MixedObserve {
  MixedRows r;
  float* drone_state;  // [n][12]
  float* aux;          // [n][9]
  uint8_t* contact;    // [n]
  float* pos;          // [n][6]: position hi words, lo words
};

template <int A>
__device__ __forceinline__ void mixed_write(const MixedObserve& a, int64_t u, const float* o, const float* x, bool contact,
                                            const float* hi, const float* lo) {
  if (a.drone_state)
    for (int c = 0; c < 12; ++c) a.drone_state[12 * u + c] = o[c];
  if (a.aux)
    for (int c = 0; c < kMixedAuxDim; ++c) a.aux[kMixedAuxDim * u + c] = c < A ? x[c < A ? c : 0] : 0.0f;
  if (a.contact) a.contact[u] = contact ? 1 : 0;
  if (a.pos)
    for (int c = 0; c < 3; ++c) {
      a.pos[kMixedPosDim * u + c] = hi[c];
      a.pos[kMixedPosDim * u + 3 + c] = lo[c];
    }
}

// Aviary.state(i) / aux_state(i) / contact_array and the hi + lo position words of every drone, in user order
__global__ void __launch_bounds__(kBlock) k_mixed_observe(const __grid_constant__ MixedObserve a) {
  const MixedRows& r = a.r;
  const int b = blockIdx.x;
  float o[12], hi[3], lo[3];
  if (b < r.cta_qx) {
    const int64_t j = (int64_t)b * kBlock + threadIdx.x;
    if (j >= r.n_qx) return;
    float x[4];
    const bool c = qx_query_drone<true>(r.qx_st, nullptr, QX_ROWS, r.n_qx, j, o, x, hi, lo);
    mixed_write<4>(a, r.slot_user[j], o, x, c, hi, lo);
  } else if (b < r.cta_qx + r.cta_fw) {
    const int64_t j = (int64_t)(b - r.cta_qx) * kBlock + threadIdx.x;
    if (j >= r.n_fw) return;
    float x[6];
    const bool c = fw_query_drone(r.fw_st, r.fw_ist, r.n_fw, j, o, x, hi, lo);
    mixed_write<6>(a, r.slot_user[r.n_qx + j], o, x, c, hi, lo);
  } else {
    const int64_t j = (int64_t)(b - r.cta_qx - r.cta_fw) * kBlock + threadIdx.x;
    if (j >= r.n_rk) return;
    float x[9];
    const bool c = rk_query_drone(r.rk_st, r.rk_ist, r.n_rk, j, o, x, hi, lo);
    mixed_write<9>(a, r.slot_user[r.n_qx + r.n_fw + j], o, x, c, hi, lo);
  }
}

// Aviary.reset: the drones of `mask` (user order; nullptr = every drone) back to their start pose with a zero setpoint.  Every
// setpoint row is rewritten at its kind's width and zeroed past it: zero for a drone that is reset, kept for the others.
__global__ void __launch_bounds__(kBlock) k_mixed_reset(const __grid_constant__ MixedRows r, const __grid_constant__ FixedwingParams fw,
                                                        const __grid_constant__ RocketParams rk, float* __restrict__ setpoint,
                                                        const float* __restrict__ start_pos, const float* __restrict__ start_orn,
                                                        const uint8_t* __restrict__ mask) {
  int64_t j;
  const int k = mixed_row(r, j);
  if (k < 0) return;
  const int64_t u = r.slot_user[(k > 0 ? r.n_qx : 0) + (k > 1 ? r.n_fw : 0) + j];
  const bool reset = !mask || mask[u];
  if (reset) {
    if (k == 0) qx_reset_drone<true>(r.qx_st, nullptr, QX_ROWS, r.n_qx, j, start_pos, start_orn, u);
    else if (k == 1) fw_reset_drone(fw, r.fw_st, r.fw_ist, r.n_fw, j, start_pos, start_orn, u);
    else rk_reset_drone(rk, r.rk_st, r.rk_ist, r.n_rk, j, start_pos, start_orn, u);
  }
  for (int c = reset ? 0 : kind_setpoint_dim(k); c < kMixedSetpointDim; ++c) setpoint[kMixedSetpointDim * u + c] = 0.0f;
}

// Aviary.set_mode: drone u in flight mode slot_mode[t].  Every setpoint row is rewritten as its kind's set_mode leaves it and
// zeroed past the kind's width: the QuadX preset, a fixed-wing's zeros, a rocket's row as it was.
__global__ void __launch_bounds__(kBlock) k_mixed_set_modes(const __grid_constant__ MixedRows r, const int8_t* __restrict__ slot_mode,
                                                            float* __restrict__ setpoint) {
  int64_t j;
  const int k = mixed_row(r, j);
  if (k < 0) return;
  const int64_t u = r.slot_user[(k > 0 ? r.n_qx : 0) + (k > 1 ? r.n_fw : 0) + j];
  if (k == 0) qx_set_mode_drone<kMixedSetpointDim>(r.qx_st, QX_ROWS, j, slot_mode, setpoint, u);
  for (int c = k == 0 ? 4 : (k == 1 ? 0 : 7); c < kMixedSetpointDim; ++c) setpoint[kMixedSetpointDim * u + c] = 0.0f;
}

// p.resetBasePositionAndOrientation / p.resetBaseVelocity + update_state of the drones of `a.mask` (user order; nullptr = every
// drone), F32: pfb_set_base_velocity; and getBasePositionAndOrientation / getBaseVelocity of every drone, in user order
template <bool F32>
__global__ void __launch_bounds__(kBlock) k_mixed_set_base_state(const __grid_constant__ MixedRows r, const __grid_constant__ BaseStateIn a) {
  int64_t j;
  const int k = mixed_row(r, j);
  if (k < 0) return;
  const int64_t u = r.slot_user[(k > 0 ? r.n_qx : 0) + (k > 1 ? r.n_fw : 0) + j];
  if (k == 0) set_base_drone<F32>(0, a, r.qx_st, nullptr, QX_ROWS, r.n_qx, j, u);
  else if (k == 1) set_base_drone<F32>(1, a, r.fw_st, r.fw_ist, 0, r.n_fw, j, u);
  else set_base_drone<F32>(2, a, r.rk_st, r.rk_ist, 0, r.n_rk, j, u);
}
__global__ void __launch_bounds__(kBlock) k_mixed_get_base_state(const __grid_constant__ MixedRows r, const __grid_constant__ BaseStateOut o) {
  int64_t j;
  const int k = mixed_row(r, j);
  if (k < 0) return;
  const int64_t u = r.slot_user[(k > 0 ? r.n_qx : 0) + (k > 1 ? r.n_fw : 0) + j];
  if (k == 0) qx_get_base_drone(r.qx_st, QX_ROWS, j, u, o);
  else if (k == 1) fw_get_base_drone(r.fw_st, r.fw_ist, r.n_fw, j, u, o);
  else rk_get_base_drone(r.rk_st, r.rk_ist, r.n_rk, j, u, o);
}

// ---------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------
static int64_t kind_state_floats(int k, int64_t c) {
  if (k == 0) return ((c + kTileLanes - 1) / kTileLanes) * qx_tile_floats(QX_ROWS);  // whole tiles
  return (int64_t)(k == 1 ? FW_ROWS : RK_ROWS) * c;
}
static int kind_state_rows(int k) { return k == 0 ? (int)QX_ROWS : (k == 1 ? (int)FW_ROWS : (int)RK_ROWS); }
static int kind_istate_rows(int k) { return k == 0 ? (int)QI_ROWS : (k == 1 ? (int)FI_ROWS : (int)RI_ROWS); }
static int grid_of(const MixedKinds* m, int k) { return grid_for(m->count[k]); }

static int mx_state_rows(const PfbContext* h) {
  int r = 0;
  for (int k = 0; k < kKinds; ++k)
    if (h->mixed->count[k] && kind_state_rows(k) > r) r = kind_state_rows(k);
  return r;
}
static int mx_istate_rows(const PfbContext* h) {
  int r = 0;
  for (int k = 0; k < kKinds; ++k)
    if (h->mixed->count[k] && kind_istate_rows(k) > r) r = kind_istate_rows(k);
  return r;
}
// the kinds' regions back to back, QuadX first, each padded to kRegionAlign floats
static int64_t state_offset(const MixedKinds* m, int kind) {
  int64_t off = 0;
  for (int k = 0; k < kind; ++k) off += (kind_state_floats(k, m->count[k]) + kRegionAlign - 1) / kRegionAlign * kRegionAlign;
  return off;
}
static int64_t mx_state_floats(const PfbContext* h) { return state_offset(h->mixed, kKinds); }

// the kinds' regions of the bound buffers: state at state_offset, istate as the kinds' [I_k][count_k] blocks back to back
// (sum <= pfb_istate_rows * n)
static MixedRows rows_of(const PfbContext* h) {
  const MixedKinds* m = h->mixed;
  MixedRows r;
  r.qx_st = h->buf.state;
  r.fw_st = h->buf.state + state_offset(m, 1);
  r.rk_st = h->buf.state + state_offset(m, 2);
  r.fw_ist = h->buf.istate + (int64_t)QI_ROWS * m->count[0];
  r.rk_ist = r.fw_ist + (int64_t)FI_ROWS * m->count[1];
  r.slot_user = m->d_slot_user;
  r.n_qx = m->count[0];
  r.n_fw = m->count[1];
  r.n_rk = m->count[2];
  r.cta_qx = grid_of(m, 0);
  r.cta_fw = grid_of(m, 1);
  return r;
}
static int grid_all(const MixedKinds* m) { return grid_of(m, 0) + grid_of(m, 1) + grid_of(m, 2); }

static int mx_reset(PfbContext* h, const uint8_t* mask, cudaStream_t s) {
  MixedKinds* m = h->mixed;
  k_mixed_reset<<<grid_all(m), kBlock, 0, s>>>(rows_of(h), h->fw, h->rk, h->buf.setpoint, h->buf.start_pos, h->buf.start_orn, mask);
  LAUNCH_CHECK(h);
  if (!mask) CUDA_OK(cudaMemsetAsync(m->d_slot_mode, 0, (size_t)h->n, s));  // a masked reset keeps the modes, as on a single-kind handle
  return 0;
}

// every drone in the modes d_slot_mode holds
static int set_slot_modes(PfbContext* h, cudaStream_t s) {
  MixedKinds* m = h->mixed;
  k_mixed_set_modes<<<grid_all(m), kBlock, 0, s>>>(rows_of(h), m->d_slot_mode, h->buf.setpoint);
  LAUNCH_CHECK(h);
  return 0;
}

static int mx_set_mode(PfbContext* h, int mode, cudaStream_t s) {
  MixedKinds* m = h->mixed;
  for (int64_t u = 0; u < h->n; ++u) {  // nothing changes unless the mode is valid for every drone
    const int k = m->h_kind[u];
    if (mode < kModeLo[k] || mode > kModeHi[k])
      return fail("`mode` must be between %d and %d or be registered in self.registered_controllers.keys()=dict_keys([]), got %d (drone %lld).",
                  kModeLo[k], kModeHi[k], mode, (long long)u);
  }
  CUDA_OK(cudaMemsetAsync(m->d_slot_mode, (int8_t)mode, (size_t)h->n, s));
  return set_slot_modes(h, s);
}

static int mx_set_modes(PfbContext* h, const int8_t* modes, cudaStream_t s) {
  MixedKinds* m = h->mixed;
  for (int64_t u = 0; u < h->n; ++u) {
    const int k = m->h_kind[u];
    if (modes[u] < kModeLo[k] || modes[u] > kModeHi[k])
      return fail("pfb_set_modes: modes[%lld] = %d, must be between %d and %d for this vehicle kind", (long long)u, (int)modes[u], kModeLo[k], kModeHi[k]);
  }
  // h_slot_mode in slot order: the counting sort of pfb_create_mixed again (stable by user index within each kind)
  int64_t next[kKinds] = {m->first[0], m->first[1], m->first[2]};
  for (int64_t u = 0; u < h->n; ++u) m->h_slot_mode[next[m->h_kind[u]]++] = modes[u];
  CUDA_OK(cudaMemcpyAsync(m->d_slot_mode, m->h_slot_mode, (size_t)h->n, cudaMemcpyHostToDevice, s));
  return set_slot_modes(h, s);
}

template <bool INJECT, bool CONTACT, bool RATES, class PS>
static void launch_step(const PfbContext* h, const PS& ps, const float* noise, int n_steps, uint32_t seq, cudaStream_t s) {
  const MixedKinds* m = h->mixed;
  MixedStep<PS> a;
  memset(&a, 0, sizeof(a));
  a.qx = ps;
  a.fw = h->fw;
  a.rk = h->rk;
  a.rng = h->rng;
  a.r = rows_of(h);
  a.slot_mode = m->d_slot_mode;
  a.setpoint = h->buf.setpoint;
  a.noise = noise;
  a.n = h->n;
  a.n_steps = n_steps;
  a.seq = seq;
  a.slot_ratio = m->d_slot_ratio;
  a.U = m->U;
  if (const StaticBodies* sb = step_statics(h))
    k_mixed_aviary_step_static<INJECT, CONTACT, RATES, PS><<<grid_all(m), kBlock, 0, s>>>(a, sb->world, sb->d_pose, sb->d_bits);
  else
    k_mixed_aviary_step<INJECT, CONTACT, RATES, PS><<<grid_all(m), kBlock, 0, s>>>(a);
}

// RATES: several control rates (d_slot_ratio set), chosen by the handle and uniform over the launch
template <bool RATES>
static void launch_steps(const PfbContext* h, const float* noise, int n_steps, uint32_t seq, cudaStream_t s) {
  const bool contact = h->env.contact_response != 0;
  QX_PARAMS_SWITCH(h, (contact ? (noise ? launch_step<true, true, RATES>(h, ps, noise, n_steps, seq, s) : launch_step<false, true, RATES>(h, ps, noise, n_steps, seq, s))
                                : (noise ? launch_step<true, false, RATES>(h, ps, noise, n_steps, seq, s) : launch_step<false, false, RATES>(h, ps, noise, n_steps, seq, s))));
}

static int mx_aviary_step(PfbContext* h, int n_steps, const float* noise, cudaStream_t s) {
  const uint32_t seq = (uint32_t)h->aviary_seq++;
  if (h->mixed->d_slot_ratio) launch_steps<true>(h, noise, n_steps, seq, s);
  else launch_steps<false>(h, noise, n_steps, seq, s);
  LAUNCH_CHECK(h);
  return 0;
}

static int mx_observe(PfbContext* h, cudaStream_t s) {
  MixedObserve a;
  a.r = rows_of(h);
  a.drone_state = h->buf.drone_state;
  a.aux = h->buf.aux_state;
  a.contact = h->buf.contact;
  a.pos = h->buf.obs;
  k_mixed_observe<<<grid_all(h->mixed), kBlock, 0, s>>>(a);
  LAUNCH_CHECK(h);
  return 0;
}

static int mx_set_base_state(PfbContext* h, const BaseStateIn& a, cudaStream_t s) {
  if (a.lin32 || a.ang32) k_mixed_set_base_state<true><<<grid_all(h->mixed), kBlock, 0, s>>>(rows_of(h), a);
  else k_mixed_set_base_state<false><<<grid_all(h->mixed), kBlock, 0, s>>>(rows_of(h), a);
  LAUNCH_CHECK(h);
  return 0;
}

static int mx_get_base_state(PfbContext* h, const BaseStateOut& o, cudaStream_t s) {
  k_mixed_get_base_state<<<grid_all(h->mixed), kBlock, 0, s>>>(rows_of(h), o);
  LAUNCH_CHECK(h);
  return 0;
}

// the hi / lo position words of pfb_observe_state
static int mx_obs_dim(const PfbContext*) { return 6; }

const HandleOps kMixedOps = {
    .kind = -1, .env_kind = PFB_ENV_NONE,
    .layout = PFB_LAYOUT_BY_KIND, .setpoint_dim = 7, .aux_dim = 9,  // the widest kind's (rocket)
    .obs_dim = mx_obs_dim,
    .mixed_state_rows = mx_state_rows, .mixed_istate_rows = mx_istate_rows, .mixed_state_floats = mx_state_floats,
    .reset = mx_reset, .set_mode = mx_set_mode, .set_modes = mx_set_modes, .aviary_step = mx_aviary_step, .observe = mx_observe,
    .set_base_state = mx_set_base_state, .get_base_state = mx_get_base_state,
};

void mx_destroy(PfbContext* h) {
  MixedKinds* m = h->mixed;
  if (!m) return;
  if (m->d_slot_user) cudaFree(m->d_slot_user);
  if (m->d_slot_mode) cudaFree(m->d_slot_mode);
  if (m->d_slot_ratio) cudaFree(m->d_slot_ratio);
  delete[] m->h_slot_mode;
  delete[] m->h_kind;
  delete m;
  h->mixed = nullptr;
}

// The kinds, slots and tables of a mixed handle on a fresh context (pfb_new_context frees everything if this fails)
static int mixed_setup(PfbContext* c, const PfbModel* models, int k, const uint8_t* model_index, const PfbEnvConfig* aviary_cfg) {
  const int64_t n = c->n;
  MixedKinds* m = new (std::nothrow) MixedKinds();
  if (!m) return fail("out of host memory");
  memset(m, 0, sizeof(*m));
  c->mixed = m;
  c->ops = &kMixedOps;
  c->model = models[0];
  c->env.env_kind = PFB_ENV_NONE;
  c->env.contact_response = (aviary_cfg && aviary_cfg->contact_response) ? 1 : 0;
  m->h_kind = new (std::nothrow) uint8_t[n];
  m->h_slot_mode = new (std::nothrow) int8_t[n];
  if (!m->h_kind || !m->h_slot_mode) return fail("out of host memory");
  // QuadX tables in the order `models` lists them; the fixed-wing and rocket table of the handle
  int qx_local[PFB_MAX_QUADX_MODELS + 2];
  PfbModel qx_models[PFB_MAX_QUADX_MODELS];
  int kq = 0, fw_table = -1, rk_table = -1;
  for (int j = 0; j < k; ++j) {
    if (models[j].kind == PFB_KIND_QUADX) { qx_models[kq] = models[j]; qx_local[j] = kq++; }
    else if (models[j].kind == PFB_KIND_FIXEDWING) fw_table = j;
    else rk_table = j;
  }
  for (int64_t i = 0; i < n; ++i) {
    m->h_kind[i] = (uint8_t)models[model_index[i]].kind;
    m->count[m->h_kind[i]] += 1;
  }
  m->first[0] = 0;
  for (int kk = 0; kk < kKinds; ++kk) m->first[kk + 1] = m->first[kk] + m->count[kk];
  // stable counting sort of the drones by kind: slot_user, and the QuadX model index in QuadX slot order
  std::unique_ptr<int32_t[]> slot_user(new (std::nothrow) int32_t[n]);
  std::unique_ptr<uint8_t[]> qx_index(new (std::nothrow) uint8_t[n]);
  if (!slot_user || !qx_index) return fail("out of host memory");
  int64_t next[kKinds] = {m->first[0], m->first[1], m->first[2]};
  for (int64_t i = 0; i < n; ++i) {
    const int64_t t = next[m->h_kind[i]]++;
    slot_user[t] = (int32_t)i;
    if (m->h_kind[i] == PFB_KIND_QUADX) qx_index[t] = (uint8_t)qx_local[model_index[i]];
  }
  CUDA_OK(cudaMalloc(&m->d_slot_user, (size_t)n * sizeof(int32_t)));
  CUDA_OK(cudaMalloc(&m->d_slot_mode, (size_t)n));
  CUDA_OK(cudaMemcpy(m->d_slot_user, slot_user.get(), (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice));
  CUDA_OK(cudaMemset(m->d_slot_mode, 0, (size_t)n));
  const bool rates = aviary_cfg && aviary_cfg->mixed_control_hz;
  QuadXParams tables[PFB_MAX_QUADX_MODELS];
  if (m->count[PFB_KIND_QUADX] && pfb_quadx_tables(qx_models, kq, tables, !rates)) return -1;
  // several control rates: the ratio of every slot, one source for every kind (pfb_create_mixed has checked the rates)
  double slowest = models[0].control_hz;
  for (int j = 1; j < k; ++j) slowest = std::min(slowest, models[j].control_hz);
  m->U = (int)std::lround(models[0].physics_hz / slowest);
  bool several = false;
  for (int j = 0; j < k; ++j) several |= models[j].control_hz != slowest;
  if (rates && several) {
    std::unique_ptr<uint8_t[]> slot_ratio(new (std::nothrow) uint8_t[n]);
    if (!slot_ratio) return fail("out of host memory");
    for (int64_t t = 0; t < n; ++t) {
      const PfbModel& mt = models[model_index[slot_user[t]]];
      slot_ratio[t] = (uint8_t)std::lround(mt.physics_hz / mt.control_hz);
      if (t < m->count[PFB_KIND_QUADX] && slot_ratio[t] != tables[qx_index[t]].ratio)
        return fail("pfb_create_mixed: slot %lld has control ratio %d, its QuadX table %d", (long long)t, (int)slot_ratio[t], tables[qx_index[t]].ratio);
    }
    CUDA_OK(cudaMalloc(&m->d_slot_ratio, (size_t)n));
    CUDA_OK(cudaMemcpy(m->d_slot_ratio, slot_ratio.get(), (size_t)n, cudaMemcpyHostToDevice));
  }
  if (m->count[PFB_KIND_QUADX]) {
    c->qx = tables[0];
    if (kq > 1 && pfb_install_quadx_set(c, tables, kq, qx_index.get(), m->count[PFB_KIND_QUADX])) return -1;
  }
  if (m->count[PFB_KIND_FIXEDWING] && fw_build_params(models[fw_table], nullptr, c->fw, c->wp)) return -1;
  if (m->count[PFB_KIND_ROCKET]) {
    if (rk_build_params(models[rk_table], nullptr, c->rk, c->land)) return -1;
    c->rk.contact_response = c->env.contact_response;
  }
  return 0;
}

extern "C" int pfb_create_mixed(const PfbModel* models, int k, const uint8_t* model_index, int64_t n, const PfbEnvConfig* aviary_cfg, int device,
                                uint64_t seed, PfbHandle* out) {
  // ---- the arguments, before any device is looked up
  if (!models || !model_index || !out) return fail("pfb_create_mixed: null argument");
  if (n <= 0) return fail("n_envs must be positive");
  if (k < 1 || k > PFB_MAX_QUADX_MODELS + 2) return fail("pfb_create_mixed: k = %d, must be in 1..%d", k, PFB_MAX_QUADX_MODELS + 2);
  if (aviary_cfg && aviary_cfg->env_kind != PFB_ENV_NONE)
    return fail("pfb_create_mixed: a mixed-kind handle is an Aviary handle; env kind %d flies one vehicle kind", aviary_cfg->env_kind);
  const bool rates = aviary_cfg && aviary_cfg->mixed_control_hz;
  int tables[kKinds] = {0, 0, 0};
  for (int j = 0; j < k; ++j) {
    const PfbModel& mj = models[j];
    if (mj.abi_version != PFB_ABI_VERSION) return fail("pfb_create_mixed: model %d has ABI %d != library ABI %d", j, mj.abi_version, PFB_ABI_VERSION);
    if (mj.kind < PFB_KIND_QUADX || mj.kind > PFB_KIND_ROCKET) return fail("pfb_create_mixed: model %d has unknown vehicle kind %d", j, mj.kind);
    if (rates) {  // one launch steps every drone with one dt; each drone's control tick falls on whole substeps
      if (mj.physics_hz != models[0].physics_hz)
        return fail("pfb_create_mixed: model %d runs at physics_hz %g, model 0 at %g: every drone of a handle needs the same physics_hz", j, mj.physics_hz,
                    models[0].physics_hz);
      if (!(mj.control_hz > 0.0) || std::fmod(mj.physics_hz, mj.control_hz) != 0.0)
        return fail("pfb_create_mixed: model %d: `physics_hz` (%g) must be multiple of `control_hz` (%g).", j, mj.physics_hz, mj.control_hz);
    } else if (mj.physics_hz != models[0].physics_hz || mj.control_hz != models[0].control_hz)  // one substep count and one dt
      return fail("pfb_create_mixed: model %d runs at physics_hz %g / control_hz %g, model 0 at %g / %g: every drone of a handle needs the same "
                  "physics_hz and control_hz", j, mj.physics_hz, mj.control_hz, models[0].physics_hz, models[0].control_hz);
    tables[mj.kind] += 1;
  }
  if (tables[PFB_KIND_QUADX] > PFB_MAX_QUADX_MODELS)
    return fail("pfb_create_mixed: %d QuadX tables, at most %d", tables[PFB_KIND_QUADX], PFB_MAX_QUADX_MODELS);
  if (rates) {
    // the reference's rule (aviary.py:287-298): sorted, each rate a multiple of the one before; U = physics_hz / slowest in 1..4
    double hz[PFB_MAX_QUADX_MODELS + 2];
    for (int j = 0; j < k; ++j) hz[j] = models[j].control_hz;
    std::sort(hz, hz + k);
    for (int j = 1; j < k; ++j)
      if (std::fmod(hz[j], hz[j - 1]) != 0.0)
        return fail("pfb_create_mixed: control_hz %g and %g: Looprates must form common multiples of each other.", hz[j - 1], hz[j]);
    const double U = models[0].physics_hz / hz[0];
    if (U > 4.0)
      return fail("pfb_create_mixed: physics_hz %g / slowest control_hz %g = %g physics substeps per Aviary step; a handle runs at most 4 (the limit on "
                  "one table's physics_hz / control_hz, applied to the handle)", models[0].physics_hz, hz[0], U);
    // several fixed-wing (rocket) tables are one model at several rates: byte-equal apart from control_hz, and not identical
    for (int j = 0; j < k; ++j)
      for (int l = j + 1; l < k; ++l) {
        if (models[j].kind != models[l].kind || models[j].kind == PFB_KIND_QUADX) continue;
        PfbModel a = models[j], b = models[l];
        a.control_hz = b.control_hz = 0.0;
        if (memcmp(&a, &b, sizeof(PfbModel)) != 0)
          return fail("pfb_create_mixed: %s tables %d and %d differ beyond control_hz; a handle flies one fixed-wing and one rocket model",
                      models[j].kind == PFB_KIND_FIXEDWING ? "fixed-wing" : "rocket", j, l);
        if (models[j].control_hz == models[l].control_hz)
          return fail("pfb_create_mixed: %s tables %d and %d are identical", models[j].kind == PFB_KIND_FIXEDWING ? "fixed-wing" : "rocket", j, l);
      }
  } else if (tables[PFB_KIND_FIXEDWING] > 1 || tables[PFB_KIND_ROCKET] > 1) {
    return fail("pfb_create_mixed: %d fixed-wing and %d rocket tables; a handle flies one fixed-wing and one rocket model", tables[PFB_KIND_FIXEDWING],
                tables[PFB_KIND_ROCKET]);
  }
  for (int64_t i = 0; i < n; ++i)
    if (model_index[i] >= k) return fail("pfb_create_mixed: model_index[%lld] = %d, must be < k = %d", (long long)i, (int)model_index[i], k);
  return pfb_new_context(n, device, seed, out, [&](PfbContext* c) { return mixed_setup(c, models, k, model_index, aviary_cfg); });
}
