// pfb_mixed.cu — Aviary handles whose drones are of several vehicle kinds (pfb_create_mixed; the reference's
// Aviary(drone_type=[...]), aviary.py:139-190): QuadX, fixed-wing and rocket drones stepped by ONE launch.
//
// The handle groups its drones by kind, in stable order: slot t of the kind-grouped order is drone slot_user[t] of the
// caller's order, the QuadX slots first, then the fixed-wing ones, then the rocket ones.  Each kind present is a sub-batch
// with that kind's own state layout (QuadX warp-tiled, fixed-wing and rocket field-major), carved from the one state buffer
// the caller binds, and is held by an ordinary single-kind sub-handle.  Resets, mode changes and the wind are not on the
// hot path: they run the sub-handles' own kernels.  The Aviary step and the state query are one launch each over all kinds:
// a one-warp CTA takes its kind from its block range, so a warp never diverges by kind.
#include <cuda_runtime.h>

#include <cstring>
#include <new>

#include "pfb_context.h"
#include "pfb_noise.cuh"

using namespace pfb;

namespace {

constexpr int kKinds = 3;               // PFB_KIND_QUADX, PFB_KIND_FIXEDWING, PFB_KIND_ROCKET
constexpr int kMixedSetpointDim = 7;    // the widest kind (rocket): the caller's setpoint buffer is [N][7]
constexpr int kMixedAuxDim = 9;         // rocket again: the aux buffer is [N][9], zero past a drone's own aux length
constexpr int kMixedPosDim = 6;         // obs buffer of a mixed handle: [N][6] = position hi words, lo words
constexpr int kSetpointDim[kKinds] = {4, 6, 7};
constexpr int kAuxDim[kKinds] = {4, 6, 9};
constexpr int64_t kRegionAlign = 32;    // floats: every kind's state region starts on a 128-byte boundary

}  // namespace

struct MixedKinds {
  PfbContext* sub[kKinds];   // sub-handle of each kind present (nullptr = no drone of that kind)
  int64_t count[kKinds];     // drones of each kind
  int64_t first[kKinds + 1]; // first slot of each kind in the kind-grouped order; first[kKinds] = n
  int32_t* d_slot_user;      // [n] slot -> user index
  int8_t* d_slot_mode;       // [n] flight mode of each slot
  uint8_t* d_mask;           // [n] a masked reset's mask in slot order
  float* d_sp[kKinds];       // [count][kSetpointDim] the sub-handles' setpoint buffers (their resets / set_mode preset them)
  float* d_pose[kKinds];     // [2][count][3] the sub-handles' start_pos, start_orn
  int8_t* h_slot_mode;       // host copy of d_slot_mode (pfb_set_modes hands slices of it to the sub-handles)
  uint8_t* h_kind;           // [n] kind of each user drone
};

// ---------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------
// What the slot kernels need to find slot t's sub-batch row
struct MixedSlots {
  int64_t first[kKinds + 1];
  int64_t count[kKinds];
  float* sp[kKinds];
  float* pose[kKinds];
};
__device__ __forceinline__ int slot_kind(const MixedSlots& m, int64_t t) { return t < m.first[1] ? 0 : (t < m.first[2] ? 1 : 2); }

// Before a sub-handle reset / mode change: the caller's setpoints, start poses and reset mask in each sub-batch's order
__global__ void __launch_bounds__(kBlock) k_mixed_gather(const MixedSlots m, const int32_t* __restrict__ slot_user,
                                                         const float* __restrict__ setpoint, const float* __restrict__ start_pos,
                                                         const float* __restrict__ start_orn, const uint8_t* __restrict__ mask,
                                                         uint8_t* __restrict__ slot_mask, int64_t n) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int k = slot_kind(m, t);
  const int64_t j = t - m.first[k], u = slot_user[t];
  const int w = k == 0 ? 4 : (k == 1 ? 6 : 7);
  for (int c = 0; c < w; ++c) m.sp[k][w * j + c] = setpoint[kMixedSetpointDim * u + c];
  if (start_pos) {
    for (int c = 0; c < 3; ++c) {
      m.pose[k][3 * j + c] = start_pos[3 * u + c];
      m.pose[k][3 * m.count[k] + 3 * j + c] = start_orn[3 * u + c];
    }
  }
  if (mask) slot_mask[t] = mask[u];
}

// After it: the sub-batch setpoints back into the caller's [N][7] rows, zero past the drone's own length
__global__ void __launch_bounds__(kBlock) k_mixed_scatter_setpoints(const MixedSlots m, const int32_t* __restrict__ slot_user,
                                                                    float* __restrict__ setpoint, int64_t n) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int k = slot_kind(m, t);
  const int64_t j = t - m.first[k], u = slot_user[t];
  const int w = k == 0 ? 4 : (k == 1 ? 6 : 7);
#pragma unroll
  for (int c = 0; c < kMixedSetpointDim; ++c) setpoint[kMixedSetpointDim * u + c] = c < w ? m.sp[k][w * j + c] : 0.0f;
}

// Everything one launch of the mixed step reads.  PS: the QuadX coefficient table (QuadXParams, or QuadXModelSet when the
// QuadX drones fly several models; its index is in QuadX slot order).
template <class PS>
struct MixedStep {
  PS qx;
  FixedwingParams fw;
  RocketParams rk;
  RngParams rng;
  float* qx_st;                 // QuadX sub-batch, warp-tiled
  float *fw_st, *rk_st;         // fixed-wing and rocket sub-batches, field-major [F][count]
  int32_t *fw_ist, *rk_ist;
  const int32_t* slot_user;
  const int8_t* slot_mode;
  const float* setpoint;        // [n][7], user order
  const float* noise;           // [n_steps * ratio][n], user order; nullptr = Philox
  int64_t n, n_qx, n_fw, n_rk;
  int cta_qx, cta_fw;           // CTAs of the QuadX range and of the fixed-wing range; the rocket CTAs follow
  int n_steps;
  uint32_t seq;
};
// the whole argument travels in the kernel-parameter bank, which holds 32 764 bytes on sm_90
static_assert(sizeof(MixedStep<QuadXModelSet>) <= 32764, "the mixed step's __grid_constant__ argument exceeds the kernel-parameter limit");

// n_steps x Aviary.step() for every drone of a mixed handle.  Drone u draws the noise of drone u of a uniform handle of its
// kind (Philox counter keyed by the USER index, injected column u), and runs the per-drone-mode body of its kind, so each
// drone's trajectory is bit-equal to the one it flies in a uniform handle with the same seed.  CONTACT: the floor pushes back.
template <bool INJECT, bool CONTACT, class PS>
__global__ void __launch_bounds__(kBlock, kMinBlocks) k_mixed_aviary_step(const __grid_constant__ MixedStep<PS> a) {
  const int b = blockIdx.x;
  if (b < a.cta_qx) {
    const int64_t j = (int64_t)b * kBlock + threadIdx.x;
    if (j >= a.n_qx) return;
    const int64_t u = a.slot_user[j];
    const QuadXParams& p = qx_model(a.qx, j);
    const int mode = a.slot_mode[j];
    QuadXRegs s;
    int step_count;
    quadx_load_tile<7, kTileGroupStride>(a.qx_st + qx_tile_base(j, QX_ROWS), s, step_count);
    quadx_mask_pid(s, mode);
#pragma unroll
    for (int c = 0; c < 4; ++c) s.sp[c] = __ldg(a.setpoint + kMixedSetpointDim * u + c);
    auto nz = make_noise<INJECT>(a.noise, a.n, u, a.rng, a.seq, TAG_AVIARY, qx_model0(a.qx).noise_loc, qx_model0(a.qx).ratio);
    for (int k = 0; k < a.n_steps; ++k) quadx_aviary_step_any<CONTACT>(p, s, mode, nz);
    quadx_store_tile<7, kTileGroupStride>(a.qx_st + qx_tile_base(j, QX_ROWS), s, step_count);
  } else if (b < a.cta_qx + a.cta_fw) {
    const int64_t j = (int64_t)(b - a.cta_qx) * kBlock + threadIdx.x;
    if (j >= a.n_fw) return;
    const int64_t u = a.slot_user[a.n_qx + j];
    const int mode = a.slot_mode[a.n_qx + j];
    const FixedwingParams& p = a.fw;
    FixedwingRegs s;
    fixedwing_load(a.fw_st, a.fw_ist, a.n_fw, j, s);
#pragma unroll
    for (int c = 0; c < 6; ++c) s.sp[c] = __ldg(a.setpoint + kMixedSetpointDim * u + c);
    auto nz = make_noise<INJECT>(a.noise, a.n, u, a.rng, a.seq, TAG_AVIARY, p.noise_loc, p.ratio);
    if (fixedwing_full_model(p)) {  // launch-uniform, the choice the uniform fixed-wing handle makes
      for (int k = 0; k < a.n_steps; ++k) fixedwing_aviary_step_any<true, CONTACT>(p, s, mode, nz);
    } else {
      for (int k = 0; k < a.n_steps; ++k) fixedwing_aviary_step_any<false, CONTACT>(p, s, mode, nz);
    }
    fixedwing_store(a.fw_st, a.fw_ist, a.n_fw, j, s);
  } else {
    const int64_t j = (int64_t)(b - a.cta_qx - a.cta_fw) * kBlock + threadIdx.x;
    if (j >= a.n_rk) return;
    const int64_t u = a.slot_user[a.n_qx + a.n_fw + j];
    const RocketParams& p = a.rk;
    RocketRegs s;
    rocket_load(a.rk_st, a.rk_ist, a.n_rk, j, s);
#pragma unroll
    for (int c = 0; c < 7; ++c) s.sp[c] = __ldg(a.setpoint + kMixedSetpointDim * u + c);
    auto nz = make_noise<INJECT>(a.noise, a.n, u, a.rng, a.seq, TAG_AVIARY, p.noise_loc, p.ratio);
    for (int k = 0; k < a.n_steps; ++k) rocket_aviary_step(p, s, nz, false);  // the contact response is p.contact_response
    rocket_store(a.rk_st, a.rk_ist, a.n_rk, j, s);
  }
}

struct MixedObserve {
  const float* qx_st;
  const float *fw_st, *rk_st;
  const int32_t *fw_ist, *rk_ist;
  const int32_t* slot_user;
  float* drone_state;  // [n][12]
  float* aux;          // [n][9]
  uint8_t* contact;    // [n]
  float* pos;          // [n][6]: position hi words, lo words
  int64_t n_qx, n_fw, n_rk;
  int cta_qx, cta_fw;
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
  const int b = blockIdx.x;
  float o[12], hi[3], lo[3];
  if (b < a.cta_qx) {
    const int64_t j = (int64_t)b * kBlock + threadIdx.x;
    if (j >= a.n_qx) return;
    QuadXRegs s;
    int step_count;
    quadx_load_tile<-1, kTileGroupStride>(a.qx_st + qx_tile_base(j, QX_ROWS), s, step_count);
    float x[4];
    quadx_drone_state(s, o, x);
    for (int c = 0; c < 3; ++c) {
      hi[c] = a.qx_st[qx_tile_word(j, QX_ROWS, QX_POS + c)];
      lo[c] = a.qx_st[qx_tile_word(j, QX_ROWS, QX_POS_LO + c)];
    }
    mixed_write<4>(a, a.slot_user[j], o, x, (s.flags & FLAG_CONTACT_ARRAY) != 0, hi, lo);
  } else if (b < a.cta_qx + a.cta_fw) {
    const int64_t j = (int64_t)(b - a.cta_qx) * kBlock + threadIdx.x;
    if (j >= a.n_fw) return;
    FixedwingRegs s;
    fixedwing_load(a.fw_st, a.fw_ist, a.n_fw, j, s);
    float x[6];
    fixedwing_drone_state(s, o, x);
    for (int c = 0; c < 3; ++c) {
      hi[c] = a.fw_st[(FW_POS + c) * a.n_fw + j];
      lo[c] = a.fw_st[(FW_POS_LO + c) * a.n_fw + j];
    }
    mixed_write<6>(a, a.slot_user[a.n_qx + j], o, x, (s.flags & FLAG_CONTACT_ARRAY) != 0, hi, lo);
  } else {
    const int64_t j = (int64_t)(b - a.cta_qx - a.cta_fw) * kBlock + threadIdx.x;
    if (j >= a.n_rk) return;
    RocketRegs s;
    rocket_load(a.rk_st, a.rk_ist, a.n_rk, j, s);
    float x[9];
    rocket_drone_state(s, o, x);
    for (int c = 0; c < 3; ++c) {
      hi[c] = a.rk_st[(RK_POS + c) * a.n_rk + j];
      lo[c] = a.rk_st[(RK_POS_LO + c) * a.n_rk + j];
    }
    mixed_write<9>(a, a.slot_user[a.n_qx + a.n_fw + j], o, x, (s.flags & FLAG_CONTACT_ARRAY) != 0, hi, lo);
  }
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

static MixedSlots slots_of(const MixedKinds* m) {
  MixedSlots s;
  for (int k = 0; k <= kKinds; ++k) s.first[k] = m->first[k];
  for (int k = 0; k < kKinds; ++k) {
    s.count[k] = m->count[k];
    s.sp[k] = m->d_sp[k];
    s.pose[k] = m->d_pose[k];
  }
  return s;
}

int mx_state_rows(const PfbContext* h) {
  int r = 0;
  for (int k = 0; k < kKinds; ++k)
    if (h->mixed->count[k] && kind_state_rows(k) > r) r = kind_state_rows(k);
  return r;
}
int mx_istate_rows(const PfbContext* h) {
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
int64_t mx_state_floats(const PfbContext* h) { return state_offset(h->mixed, kKinds); }

int mx_bind(PfbContext* h, const PfbBuffers* b) {
  MixedKinds* m = h->mixed;
  int64_t ioff = 0;
  for (int k = 0; k < kKinds; ++k) {
    if (!m->sub[k]) continue;
    PfbBuffers sb;
    memset(&sb, 0, sizeof(sb));
    sb.state = b->state + state_offset(m, k);
    sb.istate = b->istate + ioff;  // the kinds' [I_k][count_k] blocks back to back: sum <= pfb_istate_rows * n
    ioff += (int64_t)kind_istate_rows(k) * m->count[k];
    sb.setpoint = m->d_sp[k];
    sb.start_pos = m->d_pose[k];
    sb.start_orn = m->d_pose[k] + 3 * m->count[k];
    if (pfb_bind(m->sub[k], &sb)) return -1;
  }
  return 0;
}

static int gather(PfbContext* h, const uint8_t* mask, bool pose, cudaStream_t s) {
  MixedKinds* m = h->mixed;
  k_mixed_gather<<<grid_for(h->n), kBlock, 0, s>>>(slots_of(m), m->d_slot_user, h->buf.setpoint, pose ? h->buf.start_pos : nullptr,
                                                   h->buf.start_orn, mask, m->d_mask, h->n);
  LAUNCH_CHECK(h);
  return 0;
}
static int scatter(PfbContext* h, cudaStream_t s) {
  MixedKinds* m = h->mixed;
  k_mixed_scatter_setpoints<<<grid_for(h->n), kBlock, 0, s>>>(slots_of(m), m->d_slot_user, h->buf.setpoint, h->n);
  LAUNCH_CHECK(h);
  return 0;
}

int mx_reset(PfbContext* h, const uint8_t* mask, cudaStream_t s) {
  MixedKinds* m = h->mixed;
  if (gather(h, mask, true, s)) return -1;
  for (int k = 0; k < kKinds; ++k)
    if (m->sub[k] && pfb_reset(m->sub[k], mask ? m->d_mask + m->first[k] : nullptr, s)) return -1;
  if (scatter(h, s)) return -1;
  if (!mask) {  // every drone back to mode 0 (a masked reset keeps the modes, as on a single-kind handle)
    memset(m->h_slot_mode, 0, (size_t)h->n);
    CUDA_OK(cudaMemsetAsync(m->d_slot_mode, 0, (size_t)h->n, s));
  }
  return 0;
}

static const int kModeLo[kKinds] = {-1, -1, 0}, kModeHi[kKinds] = {7, 0, 0};  // quadx.py:259-262, fixedwing.py:216-219, base_drone.py:252-255

int mx_set_mode(PfbContext* h, int mode, cudaStream_t s) {
  MixedKinds* m = h->mixed;
  for (int64_t u = 0; u < h->n; ++u) {  // nothing changes unless the mode is valid for every drone
    const int k = m->h_kind[u];
    if (mode < kModeLo[k] || mode > kModeHi[k])
      return fail("`mode` must be between %d and %d or be registered in self.registered_controllers.keys()=dict_keys([]), got %d (drone %lld).",
                  kModeLo[k], kModeHi[k], mode, (long long)u);
  }
  if (gather(h, nullptr, false, s)) return -1;
  for (int k = 0; k < kKinds; ++k)
    if (m->sub[k] && pfb_set_mode(m->sub[k], mode, s)) return -1;
  if (scatter(h, s)) return -1;
  memset(m->h_slot_mode, (int8_t)mode, (size_t)h->n);
  CUDA_OK(cudaMemsetAsync(m->d_slot_mode, (int8_t)mode, (size_t)h->n, s));
  return 0;
}

int mx_set_modes(PfbContext* h, const int8_t* modes, cudaStream_t s) {
  MixedKinds* m = h->mixed;
  for (int64_t u = 0; u < h->n; ++u) {
    const int k = m->h_kind[u];
    if (modes[u] < kModeLo[k] || modes[u] > kModeHi[k])
      return fail("pfb_set_modes: modes[%lld] = %d, must be between %d and %d for this vehicle kind", (long long)u, (int)modes[u], kModeLo[k], kModeHi[k]);
  }
  // h_slot_mode in slot order: the counting sort of pfb_create_mixed again (stable by user index within each kind)
  int64_t next[kKinds] = {m->first[0], m->first[1], m->first[2]};
  for (int64_t u = 0; u < h->n; ++u) m->h_slot_mode[next[m->h_kind[u]]++] = modes[u];
  if (gather(h, nullptr, false, s)) return -1;
  for (int k = 0; k < kKinds; ++k)
    if (m->sub[k] && pfb_set_modes(m->sub[k], m->h_slot_mode + m->first[k], s)) return -1;
  if (scatter(h, s)) return -1;
  CUDA_OK(cudaMemcpyAsync(m->d_slot_mode, m->h_slot_mode, (size_t)h->n, cudaMemcpyHostToDevice, s));
  return 0;
}

template <bool INJECT, bool CONTACT, class PS>
static void launch_step(const PfbContext* h, const PS& ps, const float* noise, int n_steps, uint32_t seq, cudaStream_t s) {
  const MixedKinds* m = h->mixed;
  MixedStep<PS> a;
  memset(&a, 0, sizeof(a));
  a.qx = ps;
  if (m->sub[1]) a.fw = m->sub[1]->fw;
  if (m->sub[2]) a.rk = m->sub[2]->rk;
  a.rng = h->rng;
  a.qx_st = m->sub[0] ? m->sub[0]->buf.state : nullptr;
  a.fw_st = m->sub[1] ? m->sub[1]->buf.state : nullptr;
  a.fw_ist = m->sub[1] ? m->sub[1]->buf.istate : nullptr;
  a.rk_st = m->sub[2] ? m->sub[2]->buf.state : nullptr;
  a.rk_ist = m->sub[2] ? m->sub[2]->buf.istate : nullptr;
  a.slot_user = m->d_slot_user;
  a.slot_mode = m->d_slot_mode;
  a.setpoint = h->buf.setpoint;
  a.noise = noise;
  a.n = h->n;
  a.n_qx = m->count[0];
  a.n_fw = m->count[1];
  a.n_rk = m->count[2];
  a.cta_qx = grid_of(m, 0);
  a.cta_fw = grid_of(m, 1);
  a.n_steps = n_steps;
  a.seq = seq;
  const int g = grid_of(m, 0) + grid_of(m, 1) + grid_of(m, 2);
  k_mixed_aviary_step<INJECT, CONTACT, PS><<<g, kBlock, 0, s>>>(a);
}

int mx_aviary_step(PfbContext* h, int n_steps, const float* noise, cudaStream_t s) {
  MixedKinds* m = h->mixed;
  const uint32_t seq = (uint32_t)h->aviary_seq++;
  const bool contact = h->env.contact_response != 0;
  PfbContext* q = m->sub[0];
  if (q && q->qxset) {
    const QuadXModelSet& ps = *q->qxset;
    if (contact) noise ? launch_step<true, true>(h, ps, noise, n_steps, seq, s) : launch_step<false, true>(h, ps, noise, n_steps, seq, s);
    else noise ? launch_step<true, false>(h, ps, noise, n_steps, seq, s) : launch_step<false, false>(h, ps, noise, n_steps, seq, s);
  } else {
    QuadXParams zero;
    if (!q) memset(&zero, 0, sizeof(zero));
    const QuadXParams& ps = q ? q->qx : zero;
    if (contact) noise ? launch_step<true, true>(h, ps, noise, n_steps, seq, s) : launch_step<false, true>(h, ps, noise, n_steps, seq, s);
    else noise ? launch_step<true, false>(h, ps, noise, n_steps, seq, s) : launch_step<false, false>(h, ps, noise, n_steps, seq, s);
  }
  LAUNCH_CHECK(h);
  return 0;
}

int mx_observe(PfbContext* h, cudaStream_t s) {
  const MixedKinds* m = h->mixed;
  MixedObserve a;
  a.qx_st = m->sub[0] ? m->sub[0]->buf.state : nullptr;
  a.fw_st = m->sub[1] ? m->sub[1]->buf.state : nullptr;
  a.fw_ist = m->sub[1] ? m->sub[1]->buf.istate : nullptr;
  a.rk_st = m->sub[2] ? m->sub[2]->buf.state : nullptr;
  a.rk_ist = m->sub[2] ? m->sub[2]->buf.istate : nullptr;
  a.slot_user = m->d_slot_user;
  a.drone_state = h->buf.drone_state;
  a.aux = h->buf.aux_state;
  a.contact = h->buf.contact;
  a.pos = h->buf.obs;
  a.n_qx = m->count[0];
  a.n_fw = m->count[1];
  a.n_rk = m->count[2];
  a.cta_qx = grid_of(m, 0);
  a.cta_fw = grid_of(m, 1);
  k_mixed_observe<<<grid_of(m, 0) + grid_of(m, 1) + grid_of(m, 2), kBlock, 0, s>>>(a);
  LAUNCH_CHECK(h);
  return 0;
}

int mx_set_wind(PfbContext* h, const PfbWind* wind) {
  for (int k = 0; k < kKinds; ++k)
    if (h->mixed->sub[k] && pfb_set_wind(h->mixed->sub[k], wind)) return -1;
  return 0;
}

int mx_reseed(PfbContext* h, uint64_t seed, cudaStream_t s) {
  for (int k = 0; k < kKinds; ++k)
    if (h->mixed->sub[k] && pfb_reseed(h->mixed->sub[k], seed, s)) return -1;
  h->rng.k0 = (uint32_t)seed;
  h->rng.k1 = (uint32_t)(seed >> 32);
  h->aviary_seq = 0;
  return 0;
}

int64_t mx_launches(const PfbContext* h) {
  int64_t c = 0;
  for (int k = 0; k < kKinds; ++k)
    if (h->mixed->sub[k]) c += h->mixed->sub[k]->launches;
  return c;
}

void mx_destroy(PfbContext* h) {
  MixedKinds* m = h->mixed;
  if (!m) return;
  for (int k = 0; k < kKinds; ++k) {
    if (m->sub[k]) pfb_destroy(m->sub[k]);
    if (m->d_sp[k]) cudaFree(m->d_sp[k]);
    if (m->d_pose[k]) cudaFree(m->d_pose[k]);
  }
  if (m->d_slot_user) cudaFree(m->d_slot_user);
  if (m->d_slot_mode) cudaFree(m->d_slot_mode);
  if (m->d_mask) cudaFree(m->d_mask);
  delete[] m->h_slot_mode;
  delete[] m->h_kind;
  delete m;
  h->mixed = nullptr;
}

extern "C" int pfb_create_mixed(const PfbModel* models, int k, const uint8_t* model_index, int64_t n, const PfbEnvConfig* aviary_cfg, int device,
                                uint64_t seed, PfbHandle* out) {
  // ---- the arguments, before any device is looked up
  if (!models || !model_index || !out) return fail("pfb_create_mixed: null argument");
  if (n <= 0) return fail("n_envs must be positive");
  if (k < 1 || k > PFB_MAX_QUADX_MODELS + 2) return fail("pfb_create_mixed: k = %d, must be in 1..%d", k, PFB_MAX_QUADX_MODELS + 2);
  if (aviary_cfg && aviary_cfg->env_kind != PFB_ENV_NONE)
    return fail("pfb_create_mixed: a mixed-kind handle is an Aviary handle; env kind %d flies one vehicle kind", aviary_cfg->env_kind);
  int tables[kKinds] = {0, 0, 0};
  for (int j = 0; j < k; ++j) {
    const PfbModel& mj = models[j];
    if (mj.abi_version != PFB_ABI_VERSION) return fail("pfb_create_mixed: model %d has ABI %d != library ABI %d", j, mj.abi_version, PFB_ABI_VERSION);
    if (mj.kind < PFB_KIND_QUADX || mj.kind > PFB_KIND_ROCKET) return fail("pfb_create_mixed: model %d has unknown vehicle kind %d", j, mj.kind);
    // one launch steps every drone with one substep count and one dt
    if (mj.physics_hz != models[0].physics_hz || mj.control_hz != models[0].control_hz)
      return fail("pfb_create_mixed: model %d runs at physics_hz %g / control_hz %g, model 0 at %g / %g: every drone of a handle needs the same "
                  "physics_hz and control_hz", j, mj.physics_hz, mj.control_hz, models[0].physics_hz, models[0].control_hz);
    tables[mj.kind] += 1;
  }
  if (tables[PFB_KIND_QUADX] > PFB_MAX_QUADX_MODELS)
    return fail("pfb_create_mixed: %d QuadX tables, at most %d", tables[PFB_KIND_QUADX], PFB_MAX_QUADX_MODELS);
  if (tables[PFB_KIND_FIXEDWING] > 1 || tables[PFB_KIND_ROCKET] > 1)
    return fail("pfb_create_mixed: %d fixed-wing and %d rocket tables; a handle flies one fixed-wing and one rocket model", tables[PFB_KIND_FIXEDWING],
                tables[PFB_KIND_ROCKET]);
  for (int64_t i = 0; i < n; ++i)
    if (model_index[i] >= k) return fail("pfb_create_mixed: model_index[%lld] = %d, must be < k = %d", (long long)i, (int)model_index[i], k);
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    return fail("no CUDA device: libpyflyt_b200 has no CPU fallback (%s)", e != cudaSuccess ? cudaGetErrorString(e) : "0 devices");
  if (device < 0 || device >= count) return fail("device %d out of range (have %d)", device, count);
  CUDA_OK(cudaSetDevice(device));

  // ---- the handle
  PfbContext* c = new (std::nothrow) PfbContext();
  MixedKinds* m = new (std::nothrow) MixedKinds();
  if (!c || !m) {
    delete c;
    delete m;
    return fail("out of host memory");
  }
  memset(c, 0, sizeof(*c));
  memset(m, 0, sizeof(*m));
  c->mixed = m;
  c->model = models[0];
  c->env.env_kind = PFB_ENV_NONE;
  c->env.contact_response = (aviary_cfg && aviary_cfg->contact_response) ? 1 : 0;
  c->n = n;
  c->device = device;
  c->rng.k0 = (uint32_t)seed;
  c->rng.k1 = (uint32_t)(seed >> 32);
  auto bail = [&](void) {
    mx_destroy(c);
    delete c;
    return -1;
  };
  m->h_kind = new (std::nothrow) uint8_t[n];
  m->h_slot_mode = new (std::nothrow) int8_t[n];
  int32_t* slot_user = new (std::nothrow) int32_t[n];
  uint8_t* qx_index = new (std::nothrow) uint8_t[n];
  if (!m->h_kind || !m->h_slot_mode || !slot_user || !qx_index) {
    delete[] slot_user;
    delete[] qx_index;
    fail("out of host memory");
    return bail();
  }
  memset(m->h_slot_mode, 0, (size_t)n);
  // QuadX tables in the order `models` lists them; the fixed-wing and rocket table of the handle
  int qx_local[PFB_MAX_QUADX_MODELS + 2];
  PfbModel qx_tables[PFB_MAX_QUADX_MODELS];
  int kq = 0, fw_table = -1, rk_table = -1;
  for (int j = 0; j < k; ++j) {
    if (models[j].kind == PFB_KIND_QUADX) { qx_tables[kq] = models[j]; qx_local[j] = kq++; }
    else if (models[j].kind == PFB_KIND_FIXEDWING) fw_table = j;
    else rk_table = j;
  }
  for (int64_t i = 0; i < n; ++i) {
    m->h_kind[i] = (uint8_t)models[model_index[i]].kind;
    m->count[m->h_kind[i]] += 1;
  }
  m->first[0] = 0;
  for (int kk = 0; kk < kKinds; ++kk) m->first[kk + 1] = m->first[kk] + m->count[kk];
  {  // stable counting sort of the drones by kind
    int64_t next[kKinds] = {m->first[0], m->first[1], m->first[2]};
    for (int64_t i = 0; i < n; ++i) {
      const int64_t t = next[m->h_kind[i]]++;
      slot_user[t] = (int32_t)i;
      if (m->h_kind[i] == PFB_KIND_QUADX) qx_index[t] = (uint8_t)qx_local[model_index[i]];
    }
  }
  PfbEnvConfig cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.env_kind = PFB_ENV_NONE;
  cfg.contact_response = c->env.contact_response;
  int rc = 0;
  for (int kk = 0; kk < kKinds && rc == 0; ++kk) {
    if (!m->count[kk]) continue;
    const PfbModel* mk = kk == PFB_KIND_QUADX ? &qx_tables[0] : &models[kk == PFB_KIND_FIXEDWING ? fw_table : rk_table];
    rc = pfb_create(mk, &cfg, m->count[kk], device, seed, &m->sub[kk]);
    if (rc == 0 && kk == PFB_KIND_QUADX && kq > 1) rc = pfb_set_models(m->sub[kk], qx_tables, kq, qx_index);
    if (rc == 0 && cudaMalloc(&m->d_sp[kk], (size_t)m->count[kk] * kSetpointDim[kk] * sizeof(float)) != cudaSuccess) rc = fail("cudaMalloc failed");
    if (rc == 0 && cudaMalloc(&m->d_pose[kk], (size_t)m->count[kk] * 6 * sizeof(float)) != cudaSuccess) rc = fail("cudaMalloc failed");
  }
  if (rc == 0 && (cudaMalloc(&m->d_slot_user, (size_t)n * sizeof(int32_t)) != cudaSuccess || cudaMalloc(&m->d_slot_mode, (size_t)n) != cudaSuccess ||
                  cudaMalloc(&m->d_mask, (size_t)n) != cudaSuccess))
    rc = fail("cudaMalloc failed");
  if (rc == 0 && (cudaMemcpy(m->d_slot_user, slot_user, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice) != cudaSuccess ||
                  cudaMemset(m->d_slot_mode, 0, (size_t)n) != cudaSuccess))
    rc = fail("cudaMemcpy failed");
  delete[] slot_user;
  delete[] qx_index;
  if (rc) return bail();
  *out = c;
  return 0;
}
