// pfb_lib.cu — the C-ABI of libpyflyt_b200.so (include/pyflyt_b200.h): argument checks, handle lifetime, and calls through
// the handle's operations table (HandleOps, pfb_context.h) into the vehicle translation units (pfb_quadx.cu, ...).
#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <new>

#include "../../include/pyflyt_b200.h"
#include "pfb_context.h"

using namespace pfb;

// ---------------------------------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
int pfb_fail(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return -1;
}
#include "pfb_quadx_host.h"

// A masked pfb_env_reset on an autoreset handle of the tail-CTA env kinds: an env that finished on the previous step sits in
// the done list the NEXT step's tail CTAs consume; reset by hand, it must not be reset again by them while its regular thread
// steps it (two writers for one env).  Drop the masked entries from that list: in-place compaction by ONE CTA, chunk by chunk
// (a chunk is read completely before anything is written, and the write cursor never passes the read cursor).
__global__ void __launch_bounds__(1024) k_drop_masked_done(int32_t* __restrict__ list, int32_t* __restrict__ count, const uint8_t* __restrict__ mask) {
  __shared__ int kept;
  const int n = *count;
  if (threadIdx.x == 0) kept = 0;
  __syncthreads();
  for (int first = 0; first < n; first += blockDim.x) {
    const int t = first + (int)threadIdx.x;
    const int32_t e = t < n ? list[t] : -1;
    const bool keep = t < n && !mask[e];
    __syncthreads();  // the whole chunk is in registers
    if (keep) list[atomicAdd(&kept, 1)] = e;  // order inside the list does not matter: every entry is an independent env / arena
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = kept;
}
int pfb_drop_masked_done(PfbContext* h, const uint8_t* mask, cudaStream_t s) {
  // SAME_STEP: every finished env was reset by the step that finished it, nothing is pending
  if (!mask || !h->env.autoreset || h->env.autoreset == PFB_AUTORESET_SAME_STEP || !h->d_done_list) return 0;
  const uint64_t k = h->step_seq;  // the next step: its tail CTAs read list [(k - 1) % 4]
  k_drop_masked_done<<<1, 1024, 0, s>>>(h->d_done_list + ((k + 3) % 4) * h->n, h->d_counters + ((k + 3) % 4), mask);
  LAUNCH_CHECK(h);
  return 0;
}

int pfb_quadx_tables(const PfbModel* models, int k, QuadXParams* tables, bool one_rate) {
  for (int j = 0; j < k; ++j) {
    const PfbModel& m = models[j];
    if (m.abi_version != PFB_ABI_VERSION) return fail("pfb_set_models: model %d has ABI %d != library ABI %d", j, m.abi_version, PFB_ABI_VERSION);
    if (m.kind != PFB_KIND_QUADX) return fail("pfb_set_models: model %d is not a QuadX (kind %d)", j, m.kind);
    // every kernel runs ONE substep ratio and one dt per handle
    if (m.physics_hz != models[0].physics_hz || (one_rate && m.control_hz != models[0].control_hz))
      return fail("pfb_set_models: model %d runs at physics_hz %g / control_hz %g, model 0 at %g / %g: every model of a handle needs the same rates", j,
                  m.physics_hz, m.control_hz, models[0].physics_hz, models[0].control_hz);
    memset(&tables[j], 0, sizeof(QuadXParams));
    if (build_quadx_params(m, tables[j]) != 0) return -1;
    if ((one_rate && (tables[j].ratio != tables[0].ratio || tables[j].ctrl_dt != tables[0].ctrl_dt)) || tables[j].dt != tables[0].dt ||
        tables[j].noise_loc != tables[0].noise_loc)
      return fail("pfb_set_models: model %d has a different substep ratio, dt or motor count than model 0", j);
  }
  return 0;
}

int pfb_install_quadx_set(PfbContext* h, const QuadXParams* tables, int k, const uint8_t* index_host, int64_t n) {
  if (!h->qxset) {
    h->qxset = new (std::nothrow) QuadXModelSet();
    if (!h->qxset) return fail("out of host memory");
  }
  memset(h->qxset, 0, sizeof(QuadXModelSet));
  for (int j = 0; j < k; ++j) {
    h->qxset->m[j] = tables[j];
    h->qxset->m[j].wind = h->qx.wind;
  }
  const size_t padded = (size_t)grid_for(n) * kBlock;  // whole tiles: the tile kernels read the index of every lane
  if (!h->d_model_index) CUDA_OK(cudaMalloc(&h->d_model_index, padded));
  CUDA_OK(cudaMemset(h->d_model_index, 0, padded));
  CUDA_OK(cudaMemcpy(h->d_model_index, index_host, (size_t)n, cudaMemcpyHostToDevice));
  h->qxset->index = h->d_model_index;
  return 0;
}

// ---------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------
extern "C" {

const char* pfb_last_error(void) { return g_err; }
int pfb_abi_version(void) { return PFB_ABI_VERSION; }
int pfb_sizeof_model(void) { return (int)sizeof(PfbModel); }
int pfb_sizeof_env_config(void) { return (int)sizeof(PfbEnvConfig); }
int pfb_sizeof_buffers(void) { return (int)sizeof(PfbBuffers); }

// The vehicle tables, env parameters and buffers of a single-kind handle on a fresh context (pfb_new_context frees everything if
// this fails).  `env` = nullptr for an Aviary handle, whose one config field is `aviary_contact`.
static int single_setup(PfbContext* c, const PfbModel* model, const PfbEnvConfig* env, int aviary_contact) {
  const int64_t n_envs = c->n;
  c->model = *model;
  if (env) c->env = *env;
  else c->env.contact_response = aviary_contact;
  if (model->kind == PFB_KIND_QUADX) {
    if (build_quadx_params(*model, c->qx) != 0) return -1;
  } else if (model->kind == PFB_KIND_FIXEDWING) {
    if (fw_build_params(*model, env, c->fw, c->wp) != 0) return -1;
    if (df_build_params(env, c->df) != 0) return -1;
    if (env && env->env_kind == PFB_ENV_DOGFIGHT && (n_envs % (2 * env->team_size)) != 0)
      return fail("n_envs (%lld) must be a multiple of the arena size 2*team_size = %d", (long long)n_envs, 2 * env->team_size);
  } else {
    if (rk_build_params(*model, env, c->rk, c->land) != 0) return -1;
    if (aviary_contact) c->rk.contact_response = 1;
  }
  c->hover.env_step_ratio = env ? env->env_step_ratio : 1;
  c->hover.max_steps = env ? env->max_steps : 0;
  c->hover.angle_representation = env ? env->angle_representation : 1;
  c->hover.sparse_reward = env ? env->sparse_reward : 0;
  c->hover.warmup_steps = env ? env->warmup_steps : 0;
  c->hover.flight_mode = env ? env->flight_mode : 0;
  {
    double dome = env ? env->flight_dome_size : INFINITY;
    c->hover.dome2 = (float)(dome * dome);
  }
  c->hover.ma = (env && env->env_kind == PFB_ENV_MA_QUADX_HOVER) ? 1 : 0;
  if (c->hover.ma && env->autoreset)
    return fail("MAQuadXHover is a per-agent epilogue: arenas are reset by the caller (pfb_env_reset with a mask), autoreset must be 0");
  static const HandleOps* const kSingleKindOps[] = {&kQuadXAviaryOps,     &kHoverOps,    &kMAQuadXHoverOps, &kQuadXWaypointsOps,
                                                    &kFixedwingAviaryOps, &kFixedwingWaypointsOps, &kDogfightOps,
                                                    &kRocketAviaryOps,    &kRocketLandingOps};
  const int env_kind = env ? env->env_kind : PFB_ENV_NONE;
  for (const HandleOps* t : kSingleKindOps)
    if (t->kind == model->kind && t->env_kind == env_kind) c->ops = t;
  if (!c->ops) return fail("env kind %d is not available for vehicle kind %d in this library", env->env_kind, model->kind);
  if (env && env->env_kind == PFB_ENV_QUADX_WAYPOINTS) {
    if (env->num_targets < 1 || env->num_targets > kMaxTargets) return fail("num_targets must be in 1..%d, got %d", kMaxTargets, env->num_targets);
    c->qwp.env_step_ratio = env->env_step_ratio;
    c->qwp.max_steps = env->max_steps;
    c->qwp.sparse_reward = env->sparse_reward;
    c->qwp.warmup_steps = env->warmup_steps;
    c->qwp.num_targets = env->num_targets;
    c->qwp.use_yaw_targets = env->use_yaw_targets ? 1 : 0;
    c->qwp.dome = (float)env->flight_dome_size;
    c->qwp.dome2 = (float)(env->flight_dome_size * env->flight_dome_size);
    c->qwp.goal_reach_distance = (float)env->goal_reach_distance;
    c->qwp.goal_reach_angle = (float)env->goal_reach_angle;
    c->qwp.min_height = 0.1f;  // quadx_waypoints_env.py:88
  }
  CUDA_OK(cudaMalloc(&c->d_done_list, 4 * (size_t)n_envs * sizeof(int32_t)));
  if (env && env->autoreset && c->ops->spare_rows) {
    // spare post-reset states: env-major records (QuadX-Hover: four per env, buffer = episode number & 3, rebuilt by builder
    // CTAs inside the step launches; the other env kinds: one per env, rebuilt on a library-owned side stream)
    c->spare_bytes = (size_t)c->ops->spare_rows * (size_t)n_envs * sizeof(float);
    CUDA_OK(cudaMalloc(&c->d_spare, c->spare_bytes));
    CUDA_OK(cudaMemset(c->d_spare, 0, c->spare_bytes));
    if (c->ops->consumed_rows) {
      CUDA_OK(cudaMalloc(&c->d_consumed, (size_t)c->ops->consumed_rows * (size_t)n_envs * sizeof(int2)));  // (env, episode) per reset of a fused launch
      CUDA_OK(cudaMalloc(&c->d_elist, 4 * (size_t)n_envs * sizeof(uint32_t)));
      CUDA_OK(cudaMemset(c->d_elist, 0, 4 * (size_t)n_envs * sizeof(uint32_t)));
      CUDA_OK(cudaMalloc(&c->d_episode, (size_t)n_envs * sizeof(uint32_t)));
      CUDA_OK(cudaMemset(c->d_episode, 0, (size_t)n_envs * sizeof(uint32_t)));
    } else {
      int prio_lo = 0, prio_hi = 0;  // the rebuild is small and latency-critical: let its CTAs go first when slots free up
      CUDA_OK(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
      CUDA_OK(cudaStreamCreateWithPriority(&c->side, cudaStreamNonBlocking, prio_hi));
      CUDA_OK(cudaEventCreateWithFlags(&c->ev_step, cudaEventDisableTiming));
      for (int k = 0; k < 4; ++k) CUDA_OK(cudaEventCreateWithFlags(&c->ev_spare[k], cudaEventDisableTiming));
    }
  }
  return 0;
}

int pfb_create(const PfbModel* model, const PfbEnvConfig* env, int64_t n_envs, int device, uint64_t seed, PfbHandle* out) {
  if (!model || !out) return fail("pfb_create: null argument");
  if (model->abi_version != PFB_ABI_VERSION) return fail("PfbModel ABI %d != library ABI %d", model->abi_version, PFB_ABI_VERSION);
  if (n_envs <= 0) return fail("n_envs must be positive");
  if (env && env->inline_reset != 0 && env->inline_reset != 1) return fail("inline_reset must be 0 or 1, got %d", env->inline_reset);
  if (model->kind != PFB_KIND_QUADX && model->kind != PFB_KIND_FIXEDWING && model->kind != PFB_KIND_ROCKET)
    return fail("unknown vehicle kind %d", model->kind);
  // An Aviary handle (env kind NONE) takes ONE field from its config, contact_response; every other handle parameter is
  // what env == NULL gives
  int aviary_contact = 0;
  if (env && env->env_kind == PFB_ENV_NONE) {
    aviary_contact = env->contact_response ? 1 : 0;
    env = nullptr;
  }
  if (env && (env->autoreset < PFB_AUTORESET_NONE || env->autoreset > PFB_AUTORESET_SAME_STEP))
    return fail("autoreset must be 0 (none), 1 (NEXT_STEP) or 2 (SAME_STEP), got %d", env->autoreset);
  if (env && env->autoreset == PFB_AUTORESET_SAME_STEP && (env->env_kind == PFB_ENV_MA_QUADX_HOVER || env->env_kind == PFB_ENV_DOGFIGHT))
    return fail("SAME_STEP autoreset (autoreset = 2) is for the single-agent env kinds; MAQuadXHover and MAFixedwingDogfight reset arenas "
                "through pfb_env_reset (MAQuadXHover) or NEXT_STEP (MAFixedwingDogfight)");
  return pfb_new_context(n_envs, device, seed, out, [&](PfbContext* c) { return single_setup(c, model, env, aviary_contact); });
}

int pfb_destroy(PfbHandle h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  mx_destroy(h);
  static_destroy(h);
  if (h->d_spare) {
    if (h->side) {
      cudaStreamSynchronize(h->side);
      cudaStreamDestroy(h->side);
      if (h->ev_step) cudaEventDestroy(h->ev_step);  // a handle whose creation failed may lack them
      for (int k = 0; k < 4; ++k)
        if (h->ev_spare[k]) cudaEventDestroy(h->ev_spare[k]);
    }
    cudaFree(h->d_spare);
    if (h->d_episode) cudaFree(h->d_episode);
    if (h->d_elist) cudaFree(h->d_elist);
    if (h->d_consumed) cudaFree(h->d_consumed);
  }
  cudaFree(h->d_counters);
  cudaFree(h->d_done_list);
  if (h->d_model_index) cudaFree(h->d_model_index);
  if (h->d_modes) cudaFree(h->d_modes);
  delete h->qxset;
  if (h->prof_ev) {
    for (int i = 0; i < 2 * h->prof_cap; ++i) cudaEventDestroy(h->prof_ev[i]);
    delete[] h->prof_ev;
  }
  delete h;
  return 0;
}

int pfb_set_env_offset(PfbHandle h, uint64_t first_global_env) {
  if (!h) return fail("null handle");
  h->rng.env_offset_lo = (uint32_t)first_global_env;
  h->rng.env_offset_hi = (uint32_t)(first_global_env >> 32);
  return 0;
}

// A mixed-kind handle (pfb_create_mixed) carves its state buffer by kind: rows of the widest kind present, PFB_LAYOUT_BY_KIND,
// setpoints and aux of the widest kind (rocket), and its obs buffer receives the hi / lo position words of pfb_observe_state
int pfb_state_rows(PfbHandle h) { return h->ops->mixed_state_rows ? h->ops->mixed_state_rows(h) : h->ops->state_rows; }
int pfb_state_layout(PfbHandle h) { return h ? h->ops->layout : PFB_LAYOUT_FIELD_MAJOR; }
int64_t pfb_state_floats(PfbHandle h) {
  if (!h) return 0;
  if (h->ops->mixed_state_floats) return h->ops->mixed_state_floats(h);
  if (h->ops->layout == PFB_LAYOUT_WARP_TILED) return ((h->n + kTileLanes - 1) / kTileLanes) * qx_tile_floats(h->ops->state_rows);  // whole tiles
  return (int64_t)h->ops->state_rows * h->n;
}
int pfb_istate_rows(PfbHandle h) { return h->ops->mixed_istate_rows ? h->ops->mixed_istate_rows(h) : h->ops->istate_rows; }
int pfb_setpoint_dim(PfbHandle h) { return h->ops->setpoint_dim; }
int pfb_obs_dim(PfbHandle h) { return h->ops->obs_dim(h); }
int pfb_aux_dim(PfbHandle h) { return h->ops->aux_dim; }

int pfb_bind(PfbHandle h, const PfbBuffers* b) {
  if (!h || !b) return fail("pfb_bind: null argument");
  if (!b->state || !b->istate || !b->setpoint || !b->start_pos || !b->start_orn)
    return fail("pfb_bind: state, istate, setpoint, start_pos and start_orn are mandatory");
  if (((uintptr_t)b->setpoint & 15) || ((uintptr_t)b->state & 15)) return fail("pfb_bind: buffers must be 16-byte aligned");
  if (h->env.autoreset == PFB_AUTORESET_SAME_STEP && !b->final_obs)
    return fail("pfb_bind: a SAME_STEP autoreset handle writes the terminal observations to final_obs, which is NULL");
  h->buf = *b;
  h->bound = true;
  return 0;
}

#define REQUIRE_BOUND(h)                                   \
  if (!(h)) return fail("null handle");                    \
  if (!(h)->bound) return fail("buffers not bound: call pfb_bind first"); \
  CUDA_OK(cudaSetDevice((h)->device));


int pfb_reset(PfbHandle h, const uint8_t* mask, void* stream) {
  if (h) h->fused_ready = 0;
  REQUIRE_BOUND(h);
  if (!mask) static_clear(h);  // Aviary.reset calls resetSimulation: the static bodies go with it
  return h->ops->reset(h, mask, (cudaStream_t)stream);
}

int pfb_set_mode(PfbHandle h, int mode, void* stream) {
  REQUIRE_BOUND(h);
  return h->ops->set_mode(h, mode, (cudaStream_t)stream);
}

int pfb_set_modes(PfbHandle h, const int8_t* modes, void* stream) {
  if (!h || !modes) return fail("pfb_set_modes: null argument");
  if (h->ops->env_step)
    return fail("pfb_set_modes: only Aviary handles fly one flight mode per drone; a handle with an env epilogue flies its env's flight_mode");
  REQUIRE_BOUND(h);
  cudaStream_t s = (cudaStream_t)stream;
  if (h->ops == &kMixedOps) return h->ops->set_modes(h, modes, s);  // checks each drone against its own kind
  const int lo = kModeLo[h->model.kind], hi = kModeHi[h->model.kind];
  bool uniform = true;
  for (int64_t i = 0; i < h->n; ++i) {
    if (modes[i] < lo || modes[i] > hi)
      return fail("pfb_set_modes: modes[%lld] = %d, must be between %d and %d for this vehicle kind", (long long)i, (int)modes[i], lo, hi);
    uniform = uniform && modes[i] == modes[0];
  }
  if (uniform) return pfb_set_mode(h, modes[0], stream);  // one mode: the uniform kernels
  const size_t padded = (size_t)grid_for(h->n) * kBlock;  // whole tiles, like d_model_index
  if (!h->d_modes) {
    CUDA_OK(cudaMalloc(&h->d_modes, padded));
    CUDA_OK(cudaMemsetAsync(h->d_modes, 0, padded, s));
  }
  // stream-ordered: a step still queued on `s` reads the previous modes
  CUDA_OK(cudaMemcpyAsync(h->d_modes, modes, (size_t)h->n, cudaMemcpyHostToDevice, s));
  return h->ops->set_modes(h, modes, s);
}

int pfb_aviary_step(PfbHandle h, int n_steps, const float* noise, void* stream) {
  REQUIRE_BOUND(h);
  if (n_steps <= 0) return fail("n_steps must be positive");
  return h->ops->aviary_step(h, n_steps, noise, (cudaStream_t)stream);
}

int pfb_set_base_velocity(PfbHandle h, const float* lin_vel, const float* ang_vel, void* stream) {
  REQUIRE_BOUND(h);
  if (!lin_vel || !ang_vel) return fail("pfb_set_base_velocity: null argument");
  if (!h->ops->set_base_state)
    return fail("pfb_set_base_velocity: only Aviary handles and Rocket-Landing handles; this env builds its autoreset spares from the state");
  const BaseStateIn a = {nullptr, nullptr, nullptr, nullptr, nullptr, lin_vel, ang_vel};
  return h->ops->set_base_state(h, a, (cudaStream_t)stream);
}

// env handles keep autoreset spares and episode bookkeeping built from the state: their base state is the env's business
static int require_aviary(PfbHandle h, const char* what) {
  if (h->env.env_kind != PFB_ENV_NONE)
    return fail("%s: only Aviary handles; an env handle (env kind %d) builds its autoreset spares from the state", what, h->env.env_kind);
  return 0;
}

int pfb_set_base_state(PfbHandle h, const uint8_t* mask, const double* pos, const double* quat, const double* lin_vel, const double* ang_vel,
                       void* stream) {
  REQUIRE_BOUND(h);
  if (require_aviary(h, "pfb_set_base_state")) return -1;
  if (!pos != !quat) return fail("pfb_set_base_state: pos and quat come together (a pose) or not at all");
  if (!pos && !lin_vel && !ang_vel) return 0;
  const BaseStateIn a = {mask, pos, quat, lin_vel, ang_vel, nullptr, nullptr};
  return h->ops->set_base_state(h, a, (cudaStream_t)stream);
}

int pfb_get_base_state(PfbHandle h, double* pos, double* quat, double* lin_vel, double* ang_vel, void* stream) {
  REQUIRE_BOUND(h);
  if (require_aviary(h, "pfb_get_base_state")) return -1;
  if (!pos && !quat && !lin_vel && !ang_vel) return 0;
  const BaseStateOut o = {pos, quat, lin_vel, ang_vel};
  return h->ops->get_base_state(h, o, (cudaStream_t)stream);
}

int pfb_observe_state(PfbHandle h, void* stream) {
  REQUIRE_BOUND(h);
  return h->ops->observe(h, (cudaStream_t)stream);
}

static int require_env(PfbHandle h) {
  if (h->ops == &kMixedOps) return fail("a mixed-kind handle is an Aviary handle: the env entry points fly one vehicle kind");
  if (!h->ops->env_step) return fail("handle was created without an env epilogue");
  if (!h->buf.obs || !h->buf.reward || !h->buf.term || !h->buf.trunc) return fail("obs/reward/term/trunc buffers are not bound");
  return 0;
}

int pfb_env_reset(PfbHandle h, const uint8_t* mask, const float* noise, void* stream) {
  REQUIRE_BOUND(h);
  if (require_env(h)) return -1;
  h->fused_ready = 0;
  return h->ops->env_reset(h, mask, noise, (cudaStream_t)stream);
}

int pfb_sizeof_wind(void) { return (int)sizeof(PfbWind); }

int pfb_set_wind(PfbHandle h, const PfbWind* wind) {
  if (!h) return fail("null handle");
  if (wind && wind->kind != PFB_WIND_NONE) {
    if (wind->kind < PFB_WIND_CONSTANT || wind->kind > PFB_WIND_EXP) return fail("unknown wind kind %d", wind->kind);
    if (!(wind->z_ref > 0.0)) return fail("wind z_ref must be positive");
    if (wind->kind == PFB_WIND_LOG && !(wind->z0 > 0.0 && wind->z0 < wind->z_ref)) return fail("log wind profile needs 0 < z0 < z_ref");
    if (wind->kind == PFB_WIND_POWER && !(wind->alpha >= 0.0)) return fail("power-law wind profile needs alpha >= 0, got %g", wind->alpha);
  }
  WindParams w;
  pfb_narrow_wind(wind, w);
  if (h->d_spare && memcmp(&w, &h->qx.wind, sizeof(w)) != 0) {
    // The spare post-reset states were integrated in the old air.  Nothing may still be building them; then every record is
    // marked invalid but keeps its episode number, so each env's next reset integrates its warm-up inline, under the episode
    // number the spare would have had, in the new air, and the rebuilds that follow it use the new air too.
    CUDA_OK(cudaSetDevice(h->device));
    if (h->side) CUDA_OK(cudaStreamSynchronize(h->side));
    CUDA_OK(cudaDeviceSynchronize());
    if (h->ops->invalidate_spares(h, 0)) return -1;
    CUDA_OK(cudaDeviceSynchronize());
  }
  h->qx.wind = w;
  if (h->qxset)
    for (int j = 0; j < kMaxQuadXModels; ++j) h->qxset->m[j].wind = w;
  h->fw.wind = w;
  h->rk.wind = w;
  return 0;
}

int pfb_set_models(PfbHandle h, const PfbModel* models, int k, const uint8_t* index_host) {
  if (!h || !models || !index_host) return fail("pfb_set_models: null argument");
  if (h->ops == &kMixedOps) return fail("pfb_set_models: a mixed-kind handle takes its models at pfb_create_mixed");
  if (h->model.kind != PFB_KIND_QUADX) return fail("pfb_set_models: only QuadX handles fly several vehicle models");
  if (h->ops == &kMAQuadXHoverOps) return fail("pfb_set_models: MAQuadXHover handles fly one vehicle model");
  if (k < 1 || k > PFB_MAX_QUADX_MODELS) return fail("pfb_set_models: k = %d, must be in 1..%d", k, PFB_MAX_QUADX_MODELS);
  QuadXParams tables[PFB_MAX_QUADX_MODELS];
  if (pfb_quadx_tables(models, k, tables)) return -1;
  for (int64_t i = 0; i < h->n; ++i)
    if (index_host[i] >= k) return fail("pfb_set_models: index[%lld] = %d, must be < k = %d", (long long)i, (int)index_host[i], k);
  CUDA_OK(cudaSetDevice(h->device));
  // The spare post-reset states were integrated with the previous tables: nothing may still be building them, and every record
  // is marked invalid (a reset then integrates its warm-up inline until pfb_env_reset rebuilds them).  QuadX-Hover's builder
  // queues are emptied as a full reset does; QuadX-Waypoints keeps its done list, which its tail CTAs reset the envs from.
  if (h->side) CUDA_OK(cudaStreamSynchronize(h->side));
  CUDA_OK(cudaDeviceSynchronize());
  if (h->d_spare) CUDA_OK(cudaMemset(h->d_spare, 0, h->spare_bytes));
  if (h->d_episode) CUDA_OK(cudaMemset(h->d_counters, 0, 4 * sizeof(int32_t)));
  h->fused_ready = 0;
  const WindParams wind = h->qx.wind;
  h->model = models[0];
  h->qx = tables[0];
  h->qx.wind = wind;
  if (k == 1) {  // uniform again: the handle runs the single-table kernels
    if (h->d_model_index) CUDA_OK(cudaFree(h->d_model_index));
    h->d_model_index = nullptr;
    delete h->qxset;
    h->qxset = nullptr;
    return 0;
  }
  return pfb_install_quadx_set(h, tables, k, index_host, h->n);
}

int pfb_reseed(PfbHandle h, uint64_t seed, void* stream) {
  if (!h) return fail("null handle");
  CUDA_OK(cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  if (h->side) CUDA_OK(cudaStreamSynchronize(h->side));  // no spare rebuild of the old streams may still be in flight
  h->rng.k0 = (uint32_t)seed;
  h->rng.k1 = (uint32_t)(seed >> 32);
  h->fused_ready = 0;
  h->step_seq = 0;
  h->aviary_seq = 0;
  h->reset_seq = 0;
  CUDA_OK(cudaMemsetAsync(h->d_counters, 0, 8 * sizeof(int32_t), s));
  if (h->d_episode) CUDA_OK(cudaMemsetAsync(h->d_episode, 0, (size_t)h->n * sizeof(uint32_t), s));
  // Every spare record was drawn from the old key, and the tail kinds keep each env's episode number inside its record: all of
  // them are invalidated, which rewinds those episode words to 0 (QuadX-Hover's records fail their validity check instead of
  // being taken as warm-ups of episode numbers the new streams have not drawn).  The full pfb_env_reset that follows rebuilds them.
  if (h->d_spare) CUDA_OK(cudaMemsetAsync(h->d_spare, 0, h->spare_bytes, s));
  return 0;
}

int pfb_set_noise_dump(PfbHandle h, float* dump) {
  if (!h) return fail("null handle");
  h->noise_dump = dump;
  return 0;
}

int pfb_env_step(PfbHandle h, const float* actions, const float* noise, void* stream) {
  REQUIRE_BOUND(h);
  if (require_env(h)) return -1;
  if (actions && ((uintptr_t)actions & 15)) return fail("pfb_env_step: actions must be 16-byte aligned");
  return h->ops->env_step(h, actions ? const_cast<float*>(actions) : h->buf.setpoint, noise, false, 0, (cudaStream_t)stream);
}

int pfb_env_rollout(PfbHandle h, int n_steps, void* stream) {
  REQUIRE_BOUND(h);
  if (require_env(h)) return -1;
  if (h->ops->env_rollout) return h->ops->env_rollout(h, n_steps, (cudaStream_t)stream);
  for (int k = 0; k < n_steps; ++k)
    if (h->ops->env_step(h, h->buf.setpoint, nullptr, true, 0, (cudaStream_t)stream)) return -1;
  return 0;
}

int pfb_env_step_host(PfbHandle h, const float* host_actions, float* host_obs, float* host_reward, uint8_t* host_term,
                      uint8_t* host_trunc, void* stream) {
  REQUIRE_BOUND(h);
  if (require_env(h)) return -1;
  if (h->env.autoreset == PFB_AUTORESET_SAME_STEP)
    return fail("pfb_env_step_host: its single obs | reward | term | trunc copy has no room for final_obs; a SAME_STEP autoreset handle "
                "steps through pfb_env_step");
  cudaStream_t s = (cudaStream_t)stream;
  const int O = pfb_obs_dim(h);
  CUDA_OK(cudaMemcpyAsync(h->buf.setpoint, host_actions, (size_t)h->n * pfb_setpoint_dim(h) * sizeof(float), cudaMemcpyHostToDevice, s));
  if (h->ops->env_step(h, h->buf.setpoint, nullptr, false, 0, s)) return -1;
  // obs | reward | term | trunc laid out back to back on both sides (what the Python mirror allocates): one copy, one
  // PCIe transaction stream instead of four latency-bound ones
  const size_t ob = (size_t)h->n * O * sizeof(float), rb = (size_t)h->n * sizeof(float), fb = (size_t)h->n;
  const char* d0 = (const char*)h->buf.obs;
  char* h0 = (char*)host_obs;
  const bool packed = (const char*)h->buf.reward == d0 + ob && (const char*)h->buf.term == d0 + ob + rb && (const char*)h->buf.trunc == d0 + ob + rb + fb &&
                      (char*)host_reward == h0 + ob && (char*)host_term == h0 + ob + rb && (char*)host_trunc == h0 + ob + rb + fb;
  if (packed) {
    CUDA_OK(cudaMemcpyAsync(host_obs, h->buf.obs, ob + rb + 2 * fb, cudaMemcpyDeviceToHost, s));
    return 0;
  }
  CUDA_OK(cudaMemcpyAsync(host_obs, h->buf.obs, ob, cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaMemcpyAsync(host_reward, h->buf.reward, rb, cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaMemcpyAsync(host_term, h->buf.term, fb, cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaMemcpyAsync(host_trunc, h->buf.trunc, fb, cudaMemcpyDeviceToHost, s));
  return 0;
}

// Zero-copy variant of pfb_env_step_host: the step kernel reads the actions from, and writes obs / reward / term / trunc
// straight into, PINNED (device-mapped) host memory.  The PCIe transfers then overlap the launch tile by tile instead of
// bracketing it as two copies; no staging through the bound device buffers.
// The PCIe link is the bottleneck by 10x; with every CTA resident in one wave the bus idles while all warps compute and then
// takes the whole output at once.  Requesting dynamic shared memory the kernel never touches caps the CTAs resident per SM, so
// the step runs as several waves and the output of a wave crosses the bus while the next one computes.
constexpr size_t kMappedDynSmem = 12 * 1024;
int pfb_env_step_mapped(PfbHandle h, const float* host_actions, float* host_obs, float* host_reward, uint8_t* host_term,
                        uint8_t* host_trunc, void* stream) {
  REQUIRE_BOUND(h);
  if (require_env(h)) return -1;
  if (h->env.autoreset == PFB_AUTORESET_SAME_STEP)
    return fail("pfb_env_step_mapped: it writes no final_obs; a SAME_STEP autoreset handle steps through pfb_env_step");
  if (!host_actions || !host_obs || !host_reward || !host_term || !host_trunc) return fail("pfb_env_step_mapped: null argument");
  void *da = nullptr, *dob = nullptr, *dr = nullptr, *dte = nullptr, *dtr = nullptr;
  if (cudaHostGetDevicePointer(&da, (void*)host_actions, 0) != cudaSuccess || cudaHostGetDevicePointer(&dob, host_obs, 0) != cudaSuccess ||
      cudaHostGetDevicePointer(&dr, host_reward, 0) != cudaSuccess || cudaHostGetDevicePointer(&dte, host_term, 0) != cudaSuccess ||
      cudaHostGetDevicePointer(&dtr, host_trunc, 0) != cudaSuccess) {
    cudaGetLastError();
    return fail("pfb_env_step_mapped: the host buffers must be pinned (cudaHostAlloc / cudaHostRegister) memory");
  }
  if (((uintptr_t)da & 15) || ((uintptr_t)dob & 15)) return fail("pfb_env_step_mapped: actions and obs must be 16-byte aligned");
  const PfbBuffers saved = h->buf;
  h->buf.obs = (float*)dob; h->buf.reward = (float*)dr; h->buf.term = (uint8_t*)dte; h->buf.trunc = (uint8_t*)dtr;
  const int rc = h->ops->env_step(h, (float*)da, nullptr, false, kMappedDynSmem, (cudaStream_t)stream);
  h->buf = saved;
  return rc;
}

// ---- MAFixedwingDogfight, split variant: an arena's agents on different ranks (DESIGN.md §7)
int pfb_dogfight_payload_dim(void) { return 20; }

int pfb_dogfight_physics(PfbHandle h, const float* actions, const float* noise, float* payload_out, int first, int do_reset, int aviary_index,
                         void* stream) {
  REQUIRE_BOUND(h);
  if (h->ops != &kDogfightOps) return fail("handle is not a dogfight env");
  if (!payload_out) return fail("pfb_dogfight_physics: null payload buffer");
  return df_split_physics(h, actions ? actions : h->buf.setpoint, noise, payload_out, nullptr, 0, 0, nullptr, 0, 0, first, do_reset, aviary_index,
                          (cudaStream_t)stream);
}

int pfb_dogfight_physics_peer(PfbHandle h, const float* actions, const float* noise, const uint64_t* peer_tables_dev, int world,
                             int64_t slot_offset_floats, const uint64_t* peer_flags_dev, int rank, int epoch, int first, int do_reset,
                             int aviary_index, void* stream) {
  REQUIRE_BOUND(h);
  if (h->ops != &kDogfightOps) return fail("handle is not a dogfight env");
  if (!peer_tables_dev || world < 1) return fail("pfb_dogfight_physics_peer: need the device array of peer table pointers");
  return df_split_physics(h, actions ? actions : h->buf.setpoint, noise, nullptr, peer_tables_dev, world, slot_offset_floats, peer_flags_dev, rank,
                          epoch, first, do_reset, aviary_index, (cudaStream_t)stream);
}

int pfb_dogfight_combat(PfbHandle h, const float* payload_table, int64_t first_global_agent, int64_t num_arenas, int last, void* stream) {
  REQUIRE_BOUND(h);
  if (h->ops != &kDogfightOps) return fail("handle is not a dogfight env");
  if (require_env(h)) return -1;
  return df_split_combat(h, payload_table, first_global_agent, num_arenas, last, nullptr, 0, 0, (cudaStream_t)stream);
}

int pfb_dogfight_combat_wait(PfbHandle h, const float* payload_table, int64_t first_global_agent, int64_t num_arenas, int last,
                             const int32_t* flags, int world, int epoch, void* stream) {
  REQUIRE_BOUND(h);
  if (h->ops != &kDogfightOps) return fail("handle is not a dogfight env");
  if (require_env(h)) return -1;
  if (!flags) return fail("pfb_dogfight_combat_wait: null flag array");
  return df_split_combat(h, payload_table, first_global_agent, num_arenas, last, flags, world, epoch, (cudaStream_t)stream);
}

// One whole env step of the split dogfight with the fused exchange: env_step_ratio x (physics with peer stores + in-kernel
// signal, combat with in-kernel wait).  Nothing between the kernels needs the host, so the step is ONE call.
int pfb_dogfight_split_step(PfbHandle h, const float* actions, const uint64_t* peer_tables_dev, const uint64_t* peer_flags_dev,
                            const float* local_tables, const int32_t* local_flags, int world, int rank, int epoch0,
                            int64_t first_global_agent, int64_t num_arenas, void* stream) {
  REQUIRE_BOUND(h);
  if (h->ops != &kDogfightOps) return fail("handle is not a dogfight env");
  if (require_env(h)) return -1;
  if (!peer_tables_dev || !peer_flags_dev || !local_tables || !local_flags) return fail("pfb_dogfight_split_step: null argument");
  const int64_t na = 2 * num_arenas;
  const int ratio = h->env.env_step_ratio;
  for (int k = 0; k < ratio; ++k) {
    const int epoch = epoch0 + k;          // exchange number, 1-based; its parity selects the half of the double-buffered table
    const int phase = (epoch - 1) & 1;
    if (df_split_physics(h, actions ? actions : h->buf.setpoint, nullptr, nullptr, peer_tables_dev, world, (phase * na + first_global_agent) * 20,
                         peer_flags_dev, rank, epoch, k == 0, 0, k, (cudaStream_t)stream))
      return -1;
    if (df_split_combat(h, local_tables + phase * na * 20, first_global_agent, num_arenas, k == ratio - 1, local_flags, world, epoch,
                        (cudaStream_t)stream))
      return -1;
  }
  return 0;
}

int64_t pfb_launch_count(PfbHandle h) { return h ? h->launches : 0; }

int pfb_profile_begin(PfbHandle h, int capacity) {
  if (!h) return fail("null handle");
  CUDA_OK(cudaSetDevice(h->device));
  if (h->prof_ev) {
    for (int i = 0; i < 2 * h->prof_cap; ++i) cudaEventDestroy(h->prof_ev[i]);
    delete[] h->prof_ev;
    h->prof_ev = nullptr;
  }
  h->prof_cap = 0;
  h->prof_n = 0;
  if (capacity <= 0) return 0;
  h->prof_ev = new (std::nothrow) cudaEvent_t[2 * (size_t)capacity];
  if (!h->prof_ev) return fail("out of host memory");
  for (int i = 0; i < 2 * capacity; ++i) CUDA_OK(cudaEventCreate(&h->prof_ev[i]));
  h->prof_cap = capacity;
  return 0;
}

int pfb_profile_read(PfbHandle h, float* ms_out, int capacity) {
  if (!h) return fail("null handle");
  CUDA_OK(cudaSetDevice(h->device));
  int n = h->prof_n < capacity ? h->prof_n : capacity;
  for (int i = 0; i < n; ++i) CUDA_OK(cudaEventElapsedTime(&ms_out[i], h->prof_ev[2 * i], h->prof_ev[2 * i + 1]));
  return n;
}

}  // extern "C"
