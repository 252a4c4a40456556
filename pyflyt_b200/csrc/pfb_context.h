// pfb_context.h — private to libpyflyt_b200: the handle, error plumbing and launch helpers shared by
// the C-ABI (pfb_lib.cu) and the per-vehicle translation units (pfb_quadx.cu, pfb_fixedwing.cu, ...).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <new>
#include <type_traits>

#include "../../include/pyflyt_b200.h"
#include "pfb_fixedwing.cuh"
#include "pfb_quadx.cuh"
#include "pfb_rocket.cuh"

// thread-local error string (pfb_last_error); returns -1
int pfb_fail(const char* fmt, ...);
#define fail pfb_fail

#define CUDA_OK(expr)                                                                    \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) return fail("%s failed: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)

struct RngParams {
  uint32_t k0, k1;        // Philox key (seed)
  uint32_t env_offset_lo; // global id of local env 0 (multi-GPU sharding keeps streams rank-independent)
  uint32_t env_offset_hi;
};

// pfb_set_base_state / pfb_set_base_velocity / pfb_get_base_state: device arrays in user drone order, [N][3] (quaternions
// [N][4]); nullptr = not given / not wanted.  lin32 / ang32 are the fp32 velocities of pfb_set_base_velocity (every drone).
struct BaseStateIn {
  const uint8_t* mask;  // [N]; nullptr = every drone
  const double *pos, *quat, *lin, *ang;
  const float *lin32, *ang32;
};
struct BaseStateOut {
  double *pos, *quat, *lin, *ang;
};

// ---- mixed-model QuadX handles (pfb_set_models) ------------------------------------------------------------------------
// The kernels that integrate a QuadX drone take their coefficient table as a template type PS, passed BY VALUE as the
// __grid_constant__ kernel parameter:
//   PS = QuadXParams    one table for every env (the only form before mixed models; the K = 1 kernels)
//   PS = QuadXModelSet  up to PFB_MAX_QUADX_MODELS tables + the per-env model index; env i binds m[index[i]].  The tables
//                       stay in the parameter constant bank: a lane's table is read with a register-indexed constant load
// qx_model(ps, i) is env i's table; qx_model0(ps) is table 0, used for the fields that are equal in every table of a set
// (ratio, dt, noise_loc, wind: pfb_set_models checks physics_hz / control_hz and the kind) so that they stay warp-uniform.
constexpr int kMaxQuadXModels = PFB_MAX_QUADX_MODELS;
struct QuadXModelSet {
  pfb::QuadXParams m[kMaxQuadXModels];
  const uint8_t* index;  // device [whole tiles * 32]: model of env i (the tile padding reads model 0)
};
__device__ __forceinline__ const pfb::QuadXParams& qx_model(const pfb::QuadXParams& p, int64_t) { return p; }
__device__ __forceinline__ const pfb::QuadXParams& qx_model(const QuadXModelSet& s, int64_t i) { return s.m[s.index[i]]; }
__device__ __forceinline__ const pfb::QuadXParams& qx_model0(const pfb::QuadXParams& p) { return p; }
__device__ __forceinline__ const pfb::QuadXParams& qx_model0(const QuadXModelSet& s) { return s.m[0]; }
template <class PS>
constexpr bool kUniform = std::is_same<PS, pfb::QuadXParams>::value;

struct PfbContext {
  PfbModel model;
  PfbEnvConfig env;
  int64_t n;
  int device;
  pfb::QuadXParams qx;
  pfb::HoverParams hover;
  pfb::FixedwingParams fw;
  pfb::WaypointParams wp;
  pfb::DogfightParams df;
  pfb::RocketParams rk;
  pfb::LandingParams land;
  RngParams rng;
  PfbBuffers buf;
  bool bound;
  int mode;               // Aviary-level flight mode
  int32_t* d_counters;    // [4] rotating done-list counters: step k appends to [k%4], reads [(k-1)%4], zeroes [(k+1)%4]
  int32_t* d_done_list;   // [4][N] rotating lists of envs (arenas) that finished on a step; list (k-1)%4 is also read by the
                          // side-stream spare rebuild of step k, which step k+2 waits for before list (k+3)%4 is reused
  uint64_t step_seq;      // env.step() calls so far (selects counters/lists, keys the Philox streams)
  uint64_t aviary_seq;    // pfb_aviary_step calls so far
  uint64_t reset_seq;     // pfb_env_reset calls so far
  int64_t launches;
  pfb::QxWaypointParams qwp;
  int sm_count;
  // spare post-reset states (QuadX-Hover: pfb_quadx.cu; tail-CTA kinds: pfb_tail_step.cuh, rebuilt on the side stream)
  float* d_spare;          // spare post-reset states (env-major records), zero-initialised; nullptr = warm-ups run inline
  int2* d_consumed;        // QuadX-Hover fused rollout: (env, episode to rebuild) for every spare a launch consumed
  int fused_ready;         // every env has its spares kRolloutAhead ahead and the step pipeline is drained (cleared by single steps / resets)
  uint32_t same_launches;  // QuadX-Hover SAME_STEP launches so far: launch n appends its top-up list to d_counters[5 + n % 2]
  uint32_t* d_elist;       // QuadX-Hover: [4][N] episode number being built for each done-list entry (builder phase 0 -> phase 1)
  uint32_t* d_episode;     // QuadX-Hover: [N] episode number of each env's current valid spare (its buffer = episode & kSpareMask)
  cudaStream_t side;       // tail-CTA kinds: the spare rebuild runs here, concurrently with the following step launches
  cudaEvent_t ev_step;     // recorded on the caller's stream after a step launch; the side stream waits on it
  cudaEvent_t ev_spare[4]; // ev_spare[k % 4]: spares consumed by step k are rebuilt; step k + 2 waits on it
  int64_t side_launches;
  float* noise_dump;      // optional [substeps per env step][N] device buffer: the step kernel writes every noise draw it hands out (tests)
  // optional per-step CUDA-event pairs around the dominant kernel (bench.py's roofline leg)
  cudaEvent_t* prof_ev;   // [2 * prof_cap]
  int prof_cap;
  int prof_n;
  size_t spare_bytes;     // size of d_spare
  // mixed-model QuadX handle (pfb_set_models with k > 1): the tables and d_model_index; nullptr = every env flies `qx`
  QuadXModelSet* qxset;
  uint8_t* d_model_index;
  // one flight mode per drone (pfb_set_modes; Aviary handles): device [whole tiles * 32], valid while mode == kModePerDrone
  int8_t* d_modes;
  // mixed-kind Aviary handle (pfb_create_mixed, pfb_mixed.cu): the drones of each kind and their slots; nullptr = one kind
  struct MixedKinds* mixed;
  const struct HandleOps* ops;  // what the handle's kind runs, set once at creation
  // static bodies of an Aviary handle (pfb_add_static_body, pfb_static.cu); nullptr until the first one is added
  struct StaticBodies* statics;
};

// ---- static bodies (pfb_static.cu; DESIGN.md §4h) ----------------------------------------------------------------------------
static_assert(pfb::kMaxStaticBodies == PFB_MAX_STATIC_BODIES && pfb::kMaxStaticShapes == PFB_MAX_STATIC_SHAPES, "static-body caps");
struct StaticBodies {
  pfb::StaticWorld world;  // the primitive table every step launch with static bodies takes as a kernel parameter
  int n_bodies;
  double inertial[pfb::kMaxStaticBodies][3];  // each body's base inertial origin in its link frame (pfb_set_static_pose places it)
  float* d_pose;           // [kStaticPoseRows * kMaxStaticBodies][n]: x, y, z, cos yaw, sin yaw of body b in drone i's world
  uint32_t* d_bits;        // [n], user order: bit 0 the floor, bit 1 + b body b, touched during the last Aviary step
};
// The static bodies an Aviary step launch flies against; nullptr = none: the handle launches the kernels it launched before
// static bodies existed
static inline const StaticBodies* step_statics(const PfbContext* h) {
  return (h->statics && h->statics->n_bodies > 0) ? h->statics : nullptr;
}
void static_destroy(PfbContext* h);
void static_clear(PfbContext* h);  // a full pfb_reset: the bodies go, as the reference's resetSimulation removes them

// The device lookup, then a zeroed handle for n drones / envs on `device` with its Philox key and counters, which `setup(c)`
// completes (0 or the result of fail()).  On every failure path everything allocated is freed and *out is left alone.
template <class Setup>
int pfb_new_context(int64_t n, int device, uint64_t seed, PfbContext** out, Setup&& setup) {
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    return fail("no CUDA device: libpyflyt_b200 has no CPU fallback (%s)", e != cudaSuccess ? cudaGetErrorString(e) : "0 devices");
  if (device < 0 || device >= count) return fail("device %d out of range (have %d)", device, count);
  CUDA_OK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CUDA_OK(cudaGetDeviceProperties(&prop, device));
  PfbContext* c = new (std::nothrow) PfbContext();
  if (!c) return fail("out of host memory");
  memset(c, 0, sizeof(*c));
  c->n = n;
  c->device = device;
  c->sm_count = prop.multiProcessorCount;
  c->rng.k0 = (uint32_t)seed;
  c->rng.k1 = (uint32_t)(seed >> 32);
  e = cudaMalloc(&c->d_counters, 8 * sizeof(int32_t));  // [0..3] rotating autoreset counters, [4] ticket of the split dogfight
  if (e == cudaSuccess) e = cudaMemset(c->d_counters, 0, 8 * sizeof(int32_t));
  const int rc = e != cudaSuccess ? fail("allocating the counters failed: %s", cudaGetErrorString(e)) : setup(c);
  if (rc) {
    pfb_destroy(c);
    return -1;
  }
  *out = c;
  return 0;
}

// pfb_lib.cu: the coefficient tables of k QuadX models that one handle flies (one substep ratio, dt and motor count; with
// one_rate = false the control rates may differ: a mixed handle at several rates), and their installation as the handle's
// model set with its current wind and the per-drone index (n entries, padded to whole tiles)
int pfb_quadx_tables(const PfbModel* models, int k, pfb::QuadXParams* tables, bool one_rate = true);
int pfb_install_quadx_set(PfbContext* h, const pfb::QuadXParams* tables, int k, const uint8_t* index_host, int64_t n);

// PfbContext::mode of an Aviary handle whose drones fly the modes in d_modes; pfb_set_mode and a full pfb_reset replace it
constexpr int kModePerDrone = 0x100;

// Runs BODY with PS = the coefficient-table type of the QuadX kernels and `ps` = the value to pass: the handle's table, or its
// model set on a mixed-model handle
#define QX_PARAMS_SWITCH(h, BODY)                                                   \
  if ((h)->qxset) {                                                                 \
    using PS = QuadXModelSet;                                                       \
    const PS& ps = *(h)->qxset;                                                     \
    BODY;                                                                           \
  } else {                                                                          \
    using PS = pfb::QuadXParams;                                                    \
    const PS& ps = (h)->qx;                                                         \
    BODY;                                                                           \
  }

// One warp per CTA: a CTA retires as soon as its own warp is done, so the SM back-fills sooner and the single wave has a
// shorter tail.  448 threads per SM resident (<= 146 regs/thread) for the generic kernels.  The warp-tiled QuadX-Hover
// kernels index their 32-env tile by threadIdx.x and ballot over the full warp, so they depend on this being one warp.
constexpr int kBlock = 32;
static_assert(kBlock == pfb::kTileLanes, "one warp per CTA: the Hover kernels map lane threadIdx.x onto a 32-env tile");
constexpr int kMinBlocks = 448 / kBlock;
// the step kernels of the aerodynamic-surface vehicles (Fixedwing-Waypoints, Dogfight): the batch sizes they run at leave
// < 4 warps per SM, so registers are better spent on interleaving the surfaces than on residency (8 CTAs / SM, up to
// 255 registers, rather than 14 CTAs / SM at 128)
constexpr int kAeroBlocks = 8;

static inline int grid_for(int64_t n) { return (int)((n + kBlock - 1) / kBlock); }

#define LAUNCH_CHECK(h)                                                     \
  do {                                                                      \
    cudaError_t _e = cudaGetLastError();                                    \
    if (_e != cudaSuccess) return fail("kernel launch failed: %s", cudaGetErrorString(_e)); \
    (h)->launches += 1;                                                     \
  } while (0)

// An Aviary handle (no env epilogue) whose config asked for the contact RESPONSE: the QuadX and fixed-wing Aviary steps run
// their CONTACT instantiations.  The rocket carries the switch in RocketParams.contact_response; env handles ignore it.
static inline bool aviary_contact_response(const PfbContext* h) { return h->env.env_kind == PFB_ENV_NONE && h->env.contact_response != 0; }

// per-step bookkeeping shared by every env kind (rotating counters and lists, tail CTAs)
struct StepPlan {
  int32_t *cnt_cur, *cnt_prev, *cnt_next, *list_cur, *list_prev;
  uint32_t seq;
  int tail, grid;
  bool prof;
};
static inline StepPlan plan_step(PfbContext* h) {
  StepPlan p;
  const uint64_t k = h->step_seq;
  // four rotating done lists / counters: step k appends to [k % 4], its tail CTAs (and the side-stream spare rebuild, for the
  // envs that have one) read [(k - 1) % 4], and it zeroes counter [(k + 1) % 4]
  p.cnt_cur = h->d_counters + (k % 4);
  p.cnt_prev = h->d_counters + ((k + 3) % 4);
  p.cnt_next = h->d_counters + ((k + 1) % 4);
  p.list_cur = h->d_done_list + (k % 4) * h->n;
  p.list_prev = h->d_done_list + ((k + 3) % 4) * h->n;
  p.seq = (uint32_t)k;
  // tail CTAs (front of the grid) reset the envs that finished on the previous call; one per SM is
  // plenty for the ~1-3 % of envs that finish per step, and the loop is grid-strided anyway
  p.tail = 0;
  if (h->env.autoreset == PFB_AUTORESET_NEXT_STEP) {  // SAME_STEP resets in the regular lanes: no tail CTAs
    p.tail = h->sm_count;
    int need = grid_for(h->n);
    if (p.tail > need) p.tail = need;
  }
  p.grid = grid_for(h->n) + p.tail;
  p.prof = h->prof_ev && h->prof_n < h->prof_cap;
  return p;
}

// pfb_lib.cu: a masked user reset on an autoreset handle removes the masked envs / arenas from the pending done list
int pfb_drop_masked_done(PfbContext* h, const uint8_t* mask, cudaStream_t s);

// The flight modes each vehicle kind flies, by PFB_KIND_*: QuadX -1..7 (quadx.py:259-262), fixed-wing -1..0 (fixedwing.py:216-219),
// rocket 0 only (base_drone.py:252-255)
constexpr int kModeLo[3] = {-1, -1, 0};
constexpr int kModeHi[3] = {7, 0, 0};

// Runs BODY with `constexpr int MODE` = the QuadX flight mode `mode`
#define PFB_MODE_SWITCH(mode, BODY)                         \
  switch (mode) {                                           \
    case -1: { constexpr int MODE = -1; BODY; } break;      \
    case 0: { constexpr int MODE = 0; BODY; } break;        \
    case 1: { constexpr int MODE = 1; BODY; } break;        \
    case 2: { constexpr int MODE = 2; BODY; } break;        \
    case 3: { constexpr int MODE = 3; BODY; } break;        \
    case 4: { constexpr int MODE = 4; BODY; } break;        \
    case 5: { constexpr int MODE = 5; BODY; } break;        \
    case 6: { constexpr int MODE = 6; BODY; } break;        \
    case 7: { constexpr int MODE = 7; BODY; } break;        \
    default: return fail("`mode` must be between %d and %d, got %d", kModeLo[PFB_KIND_QUADX], kModeHi[PFB_KIND_QUADX], mode); \
  }

// ---- host side of the tail-CTA env kinds (pfb_tail_step.cuh): QuadX-Waypoints, Fixedwing-Waypoints, Rocket-Landing, Dogfight ----
// Each kind passes one generic lambda `launch(StepVariant<INJECT, RANDACT, AUTORESET, SAME>{}, const TailLaunch&)` that launches its
// step kernel and returns 0 or the result of fail(); it serves the step, the side-stream spare rebuild and the build after a reset.
// SAME: the SAME_STEP step kernel (tail_step_same), which reads only the current lists, the spares and spare_copy of L.
template <bool INJECT, bool RANDACT, bool AUTORESET, bool SAME = false>
struct StepVariant {
  static constexpr bool inject = INJECT, randact = RANDACT, autoreset = AUTORESET, same = SAME;
};
struct TailLaunch {
  int grid, tail_blocks;
  float* spare;
  int spare_copy, build;
  const int32_t *prev_count, *prev_list;
  int32_t *cur_count, *cur_list, *next_count;
  uint32_t seq;
  cudaStream_t stream;
};

template <class Launch>
int tail_env_step(PfbContext* h, const float* noise, bool randact, cudaStream_t s, Launch&& launch) {
  const StepPlan pl = plan_step(h);
  float* spare = h->env.autoreset ? h->d_spare : nullptr;
  const bool same = h->env.autoreset == PFB_AUTORESET_SAME_STEP;
  // NEXT_STEP: the rebuild of the spares consumed by step k - 2 must be complete before step k (an env cannot finish again sooner).
  // SAME_STEP: an env reset on step k - 1 may finish again on step k and take its next spare there, so step k waits for the
  // rebuild behind step k - 1
  if (spare && same && h->step_seq >= 1) CUDA_OK(cudaStreamWaitEvent(s, h->ev_spare[(h->step_seq - 1) % 4], 0));
  if (spare && !same && h->step_seq >= 2) CUDA_OK(cudaStreamWaitEvent(s, h->ev_spare[(h->step_seq - 2) % 4], 0));
  if (pl.prof) CUDA_OK(cudaEventRecord(h->prof_ev[2 * h->prof_n], s));
  const TailLaunch L = {pl.grid, pl.tail, spare, (spare && !h->env.inline_reset) ? 1 : 0, 0,
                        pl.cnt_prev, pl.list_prev, pl.cnt_cur, pl.list_cur, pl.cnt_next, pl.seq, s};
  int rc;
  if (same) {
    if (noise) return fail("injected noise (parity mode) is only supported with autoreset = 0");
    rc = randact ? launch(StepVariant<false, true, true, true>{}, L) : launch(StepVariant<false, false, true, true>{}, L);
  } else if (h->env.autoreset) {
    if (noise) return fail("injected noise (parity mode) is only supported with autoreset = 0");
    rc = randact ? launch(StepVariant<false, true, true>{}, L) : launch(StepVariant<false, false, true>{}, L);
  } else {
    rc = noise ? launch(StepVariant<true, false, false>{}, L)
               : (randact ? launch(StepVariant<false, true, false>{}, L) : launch(StepVariant<false, false, false>{}, L));
  }
  if (rc) return rc;
  LAUNCH_CHECK(h);
  if (pl.prof) {
    CUDA_OK(cudaEventRecord(h->prof_ev[2 * h->prof_n + 1], s));
    h->prof_n += 1;
  }
  if (spare) {  // rebuild the spares this launch consumed, on the side stream (ordered behind it), while the next launches run
    CUDA_OK(cudaEventRecord(h->ev_step, s));
    CUDA_OK(cudaStreamWaitEvent(h->side, h->ev_step, 0));
    // NEXT_STEP consumes the spares of the previous step's list in its tail CTAs, SAME_STEP those of its own list
    const int32_t* rb_count = same ? pl.cnt_cur : pl.cnt_prev;
    const int32_t* rb_list = same ? pl.list_cur : pl.list_prev;
    const TailLaunch B = {h->sm_count, h->sm_count, spare, 0, 1, rb_count, rb_list, pl.cnt_cur, pl.list_cur, pl.cnt_next, pl.seq, h->side};
    if (launch(StepVariant<false, false, true>{}, B)) return -1;
    LAUNCH_CHECK(h);
    CUDA_OK(cudaEventRecord(h->ev_spare[h->step_seq % 4], h->side));
  }
  h->step_seq += 1;
  return 0;
}

// ---- host side of the Aviary step (pfb_aviary_step) of every vehicle kind and of the mixed-kind handle ----
// Each kind passes one generic lambda `launch(AviaryVariant<INJECT, CONTACT, World>{sb})` that launches its step kernel and
// returns 0 or the result of fail().  INJECT: injected noise; CONTACT: aviary_contact_response(h); World: pfb::StaticCtx with
// the handle's static bodies `sb` (step_statics), or pfb::NoStatic with sb = nullptr.  The kernel takes world_table(v),
// v.pose() and v.bits().
template <bool INJECT, bool CONTACT, class World>
struct AviaryVariant {
  static constexpr bool inject = INJECT, contact = CONTACT;
  using world = World;
  const StaticBodies* sb;
  const float* pose() const { return sb ? sb->d_pose : nullptr; }
  uint32_t* bits() const { return sb ? sb->d_bits : nullptr; }
};

// the static-body table argument of the step kernel: an empty one for NoStatic (WorldTable, pfb_aviary.cuh)
template <bool INJECT, bool CONTACT>
pfb::NoStaticTable world_table(AviaryVariant<INJECT, CONTACT, pfb::NoStatic>) { return {}; }
template <bool INJECT, bool CONTACT>
const pfb::StaticWorld& world_table(AviaryVariant<INJECT, CONTACT, pfb::StaticCtx> v) { return v.sb->world; }

template <bool INJECT, bool CONTACT, class Launch>
int aviary_step_world(const StaticBodies* sb, Launch& launch) {
  return sb ? launch(AviaryVariant<INJECT, CONTACT, pfb::StaticCtx>{sb}) : launch(AviaryVariant<INJECT, CONTACT, pfb::NoStatic>{nullptr});
}
template <class Launch>
int aviary_step_launch(PfbContext* h, const float* noise, Launch&& launch) {
  const StaticBodies* sb = step_statics(h);
  int rc;
  if (aviary_contact_response(h)) rc = noise ? aviary_step_world<true, true>(sb, launch) : aviary_step_world<false, true>(sb, launch);
  else rc = noise ? aviary_step_world<true, false>(sb, launch) : aviary_step_world<false, false>(sb, launch);
  if (rc) return rc;
  LAUNCH_CHECK(h);
  return 0;
}

// `reset(grid)` launches the kind's reset kernel over every env and returns 0 or the result of fail()
template <class Reset, class Launch>
int tail_env_reset(PfbContext* h, const uint8_t* mask, cudaStream_t s, Reset&& reset, Launch&& launch) {
  const int g = grid_for(h->n);
  float* spare = h->env.autoreset ? h->d_spare : nullptr;
  if (spare) {
    // the spares are rewritten below: the last rebuild must have finished
    if (h->step_seq > 0) CUDA_OK(cudaStreamWaitEvent(s, h->ev_spare[(h->step_seq - 1) % 4], 0));
    if (!mask) CUDA_OK(cudaMemsetAsync(h->d_counters, 0, 4 * sizeof(int32_t), s));  // a full reset empties the autoreset queues
    else if (pfb_drop_masked_done(h, mask, s)) return -1;  // a masked one takes its envs out of the pending done list
  }
  if (reset(g)) return -1;
  LAUNCH_CHECK(h);
  if (spare) {  // every env gets a fresh spare: the step kernel in build mode over all envs, same stream
    const TailLaunch B = {g, g, spare, 0, 1, nullptr, nullptr, nullptr, nullptr, nullptr, 0u, s};
    if (launch(StepVariant<false, false, true>{}, B)) return -1;
    LAUNCH_CHECK(h);
  }
  return 0;
}

// ---- what a handle runs: one constant table per handle kind, which pfb_create picks by (vehicle kind, env kind) and
// pfb_create_mixed sets; the C-ABI entry points check their arguments and call through PfbContext::ops
struct HandleOps {
  int kind, env_kind;  // the pair pfb_create looks the table up by (the mixed table: -1, PFB_ENV_NONE)
  // buffer shape: pfb_state_rows, pfb_istate_rows, pfb_state_layout, pfb_setpoint_dim, pfb_aux_dim, pfb_obs_dim
  int state_rows, istate_rows, layout, setpoint_dim, aux_dim;
  int (*obs_dim)(const PfbContext* h);
  // the mixed table: rows and floats of the kinds present, in place of state_rows, istate_rows and the layout's float count
  int (*mixed_state_rows)(const PfbContext* h);
  int (*mixed_istate_rows)(const PfbContext* h);
  int64_t (*mixed_state_floats)(const PfbContext* h);
  // Aviary surface: every handle has reset, set_mode (which checks `mode` against the kind's range), aviary_step and observe
  int (*reset)(PfbContext* h, const uint8_t* mask, cudaStream_t s);
  int (*set_mode)(PfbContext* h, int mode, cudaStream_t s);
  // pfb_set_modes with modes that differ, on an Aviary handle: a single-kind table runs once d_modes holds the checked modes; the
  // mixed table checks `modes` against each drone's kind itself.  nullptr = every mode list of the kind is uniform (rocket)
  int (*set_modes)(PfbContext* h, const int8_t* modes, cudaStream_t s);
  int (*aviary_step)(PfbContext* h, int n_steps, const float* noise, cudaStream_t s);
  int (*observe)(PfbContext* h, cudaStream_t s);
  // base state: a.lin32 / a.ang32 set = pfb_set_base_velocity, which every table with set_base_state accepts (Aviary handles,
  // and Rocket-Landing, whose reset calls it: rocket_base_env.py:228); the other env handles have neither
  int (*set_base_state)(PfbContext* h, const BaseStateIn& a, cudaStream_t s);
  int (*get_base_state)(PfbContext* h, const BaseStateOut& o, cudaStream_t s);
  // env epilogue, nullptr on Aviary handles.  `dyn_smem`: dynamic shared memory the step launch requests and never touches
  // (pfb_env_step_mapped; only QuadX-Hover's step honours it, 0 = every CTA resident in one wave)
  int (*env_reset)(PfbContext* h, const uint8_t* mask, const float* noise, cudaStream_t s);
  int (*env_step)(PfbContext* h, float* actions, const float* noise, bool randact, size_t dyn_smem, cudaStream_t s);
  int (*env_rollout)(PfbContext* h, int n_steps, cudaStream_t s);  // nullptr = n_steps env_step calls with on-device actions
  // autoreset spares: floats of d_spare per env, offset of a record's valid word (tail-CTA kinds), entries of d_consumed per env
  // (QuadX-Hover builds spares inside its step launches; 0 = rebuilt on the side stream); a wind change runs invalidate_spares
  int spare_rows, spare_valid_row, consumed_rows;
  int (*invalidate_spares)(PfbContext* h, cudaStream_t s);
};

// invalidate_spares of the tail-CTA kinds: every record is marked invalid, so each env's next reset integrates its warm-up inline
inline int tail_invalidate_spares(PfbContext* h, cudaStream_t s) {
  CUDA_OK(cudaMemset2DAsync(h->d_spare + h->ops->spare_valid_row, (size_t)h->ops->spare_rows * sizeof(float), 0, sizeof(float), (size_t)h->n, s));
  return 0;
}

// QuadX translation unit (pfb_quadx.cu): the Aviary surface, which the QuadX-Waypoints table (pfb_quadx_wp.cu) points at too
int qx_reset(PfbContext* h, const uint8_t* mask, cudaStream_t s);
int qx_set_mode(PfbContext* h, int mode, cudaStream_t s);
int qx_aviary_step(PfbContext* h, int n_steps, const float* noise, cudaStream_t s);
int qx_observe(PfbContext* h, cudaStream_t s);

// fixedwing translation unit (pfb_fixedwing.cu): the parameter tables, and the Aviary surface, which the Dogfight table
// (pfb_dogfight.cu) points at too
int fw_build_params(const PfbModel& m, const PfbEnvConfig* env, pfb::FixedwingParams& p, pfb::WaypointParams& w);
int fw_reset(PfbContext* h, const uint8_t* mask, cudaStream_t s);
int fw_set_mode(PfbContext* h, int mode, cudaStream_t s);
int fw_aviary_step(PfbContext* h, int n_steps, const float* noise, cudaStream_t s);
int fw_observe(PfbContext* h, cudaStream_t s);

// rocket translation unit (pfb_rocket.cu)
int rk_build_params(const PfbModel& m, const PfbEnvConfig* env, pfb::RocketParams& p, pfb::LandingParams& l);

// dogfight translation unit (pfb_dogfight.cu): fixedwing vehicles, arenas of 2*team_size adjacent envs
int df_build_params(const PfbEnvConfig* env, pfb::DogfightParams& d);
int df_split_physics(PfbContext* h, const float* actions, const float* noise, float* payload, const uint64_t* peers, int world, int64_t slot0,
                     const uint64_t* peer_flags, int rank, int epoch, int first, int do_reset, int sub, cudaStream_t s);
int df_split_combat(PfbContext* h, const float* table, int64_t first_gid, int64_t num_arenas, int last, const int* wait_flags, int world, int epoch,
                    cudaStream_t s);

// mixed-kind Aviary handles (pfb_mixed.cu)
void mx_destroy(PfbContext* h);

// the tables of the handle kinds, each next to the code it points at
extern const HandleOps kQuadXAviaryOps, kHoverOps, kMAQuadXHoverOps;  // pfb_quadx.cu
extern const HandleOps kQuadXWaypointsOps;                            // pfb_quadx_wp.cu
extern const HandleOps kFixedwingAviaryOps, kFixedwingWaypointsOps;   // pfb_fixedwing.cu
extern const HandleOps kDogfightOps;                                  // pfb_dogfight.cu
extern const HandleOps kRocketAviaryOps, kRocketLandingOps;           // pfb_rocket.cu
extern const HandleOps kMixedOps;                                     // pfb_mixed.cu
