// pfb_context.h — private to libpyflyt_b200: the handle, error plumbing and launch helpers shared by
// the C-ABI (pfb_lib.cu) and the per-vehicle translation units (pfb_quadx.cu, pfb_fixedwing.cu, ...).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
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
};

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

// QuadX state layout: warp-tiled (pfb_quadx.cuh) on every QuadX handle except QuadX-Waypoints (field-major rows + istate)
static inline bool qx_tiled(const PfbContext* h) { return h->model.kind == PFB_KIND_QUADX && h->env.env_kind != PFB_ENV_QUADX_WAYPOINTS; }
static inline int qx_rows(const PfbContext* h) { return h->env.env_kind == PFB_ENV_MA_QUADX_HOVER ? (int)pfb::QM_ROWS : (int)pfb::QX_ROWS; }

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
  if (h->env.autoreset != 0) {
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
    default: return fail("`mode` must be between -1 and 7, got %d", mode); \
  }

// ---- host side of the tail-CTA env kinds (pfb_tail_step.cuh): QuadX-Waypoints, Fixedwing-Waypoints, Rocket-Landing, Dogfight ----
// Each kind passes one generic lambda `launch(StepVariant<INJECT, RANDACT, AUTORESET>{}, const TailLaunch&)` that launches its step
// kernel and returns 0 or the result of fail(); it serves the step, the side-stream spare rebuild and the build after a reset.
template <bool INJECT, bool RANDACT, bool AUTORESET>
struct StepVariant {
  static constexpr bool inject = INJECT, randact = RANDACT, autoreset = AUTORESET;
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
  // the rebuild of the spares consumed by step k - 2 must be complete before step k (an env cannot finish again sooner)
  if (spare && h->step_seq >= 2) CUDA_OK(cudaStreamWaitEvent(s, h->ev_spare[(h->step_seq - 2) % 4], 0));
  if (pl.prof) CUDA_OK(cudaEventRecord(h->prof_ev[2 * h->prof_n], s));
  const TailLaunch L = {pl.grid, pl.tail, spare, (spare && !h->env.inline_reset) ? 1 : 0, 0,
                        pl.cnt_prev, pl.list_prev, pl.cnt_cur, pl.list_cur, pl.cnt_next, pl.seq, s};
  int rc;
  if (h->env.autoreset) {
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
    const TailLaunch B = {h->sm_count, h->sm_count, spare, 0, 1, pl.cnt_prev, pl.list_prev, pl.cnt_cur, pl.list_cur, pl.cnt_next, pl.seq, h->side};
    if (launch(StepVariant<false, false, true>{}, B)) return -1;
    LAUNCH_CHECK(h);
    CUDA_OK(cudaEventRecord(h->ev_spare[h->step_seq % 4], h->side));
  }
  h->step_seq += 1;
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

// QuadX translation unit (pfb_quadx.cu): Aviary surface, QuadX-Hover and MAQuadXHover
int qx_reset(PfbContext* h, const uint8_t* mask, cudaStream_t s);
int qx_set_mode(PfbContext* h, int mode, cudaStream_t s);
int qx_set_modes(PfbContext* h, cudaStream_t s);  // after d_modes holds the modes
int qx_aviary_step(PfbContext* h, int n_steps, const float* noise, cudaStream_t s);
int qx_observe(PfbContext* h, cudaStream_t s);
int hover_spare_rows();     // floats of d_spare per env
int hover_consumed_rows();  // entries of d_consumed per env
int hover_env_reset(PfbContext* h, const uint8_t* mask, const float* noise, cudaStream_t s);
// `dyn_smem`: dynamic shared memory the step launch requests and never touches (pfb_env_step_mapped; 0 = every CTA resident in one wave)
int hover_env_step(PfbContext* h, float* actions, const float* noise, bool randact, size_t dyn_smem, cudaStream_t s);
int hover_env_rollout(PfbContext* h, int n_steps, cudaStream_t s);  // n_steps env steps with on-device actions, fused where it can
// with the device idle: finish the half-built spares, empty their queue and mark every spare record invalid (pfb_set_wind)
int hover_invalidate_spares(PfbContext* h, cudaStream_t s);

// fixedwing translation unit (pfb_fixedwing.cu)
int fw_build_params(const PfbModel& m, const PfbEnvConfig* env, pfb::FixedwingParams& p, pfb::WaypointParams& w);
int fw_state_rows();
int fw_istate_rows();
int fw_obs_dim(const PfbContext* h);
int fw_reset(PfbContext* h, const uint8_t* mask, cudaStream_t s);
int fw_set_mode(PfbContext* h, int mode, cudaStream_t s);
int fw_set_modes(PfbContext* h, cudaStream_t s);  // after d_modes holds the modes: zero the setpoints, flag the handle
int fw_aviary_step(PfbContext* h, int n_steps, const float* noise, cudaStream_t s);
int fw_observe(PfbContext* h, cudaStream_t s);
int fw_env_reset(PfbContext* h, const uint8_t* mask, const float* noise, cudaStream_t s);
int fw_env_step(PfbContext* h, float* actions, const float* noise, bool randact, cudaStream_t s);
int fw_spare_rows();
int fw_spare_valid_row();  // float offset of the valid word in a spare record

// rocket translation unit (pfb_rocket.cu)
int rk_build_params(const PfbModel& m, const PfbEnvConfig* env, pfb::RocketParams& p, pfb::LandingParams& l);
int rk_state_rows();
int rk_istate_rows();
int rk_obs_dim(const PfbContext* h);
int rk_reset(PfbContext* h, const uint8_t* mask, cudaStream_t s);
int rk_set_mode(PfbContext* h, int mode, cudaStream_t s);
int rk_set_velocity(PfbContext* h, const float* lin, const float* ang, cudaStream_t s);
int rk_aviary_step(PfbContext* h, int n_steps, const float* noise, cudaStream_t s);
int rk_observe(PfbContext* h, cudaStream_t s);
int rk_env_reset(PfbContext* h, const uint8_t* mask, const float* noise, cudaStream_t s);
int rk_env_step(PfbContext* h, float* actions, const float* noise, bool randact, cudaStream_t s);
int rk_spare_rows();
int rk_spare_valid_row();  // float offset of the valid word in a spare record

// dogfight translation unit (pfb_dogfight.cu): fixedwing vehicles, arenas of 2*team_size adjacent envs
int df_build_params(const PfbEnvConfig* env, pfb::DogfightParams& d);
int df_obs_dim(const PfbContext* h);
int df_env_reset(PfbContext* h, const uint8_t* mask, const float* noise, cudaStream_t s);
int df_env_step(PfbContext* h, float* actions, const float* noise, bool randact, cudaStream_t s);
int df_spare_rows();
int df_spare_valid_row();  // float offset of the valid word in a spare record
int df_split_physics(PfbContext* h, const float* actions, const float* noise, float* payload, const uint64_t* peers, int world, int64_t slot0,
                     const uint64_t* peer_flags, int rank, int epoch, int first, int do_reset, int sub, cudaStream_t s);
int df_split_combat(PfbContext* h, const float* table, int64_t first_gid, int64_t num_arenas, int last, const int* wait_flags, int world, int epoch,
                    cudaStream_t s);

// QuadX-Waypoints translation unit (pfb_quadx_wp.cu)
int qwp_state_rows();
int qwp_istate_rows();
int qwp_obs_dim(const PfbContext* h);
int qwp_spare_rows();
int qwp_spare_valid_row();  // float offset of the valid word in a spare record
int qwp_env_reset(PfbContext* h, const uint8_t* mask, const float* noise, cudaStream_t s);
int qwp_env_step(PfbContext* h, float* actions, const float* noise, bool randact, cudaStream_t s);
