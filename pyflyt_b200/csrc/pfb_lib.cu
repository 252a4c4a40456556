// pfb_lib.cu — the C-ABI of libpyflyt_b200.so (include/pyflyt_b200.h): argument checks, handle lifetime, and dispatch
// to the vehicle translation units (pfb_quadx.cu, pfb_quadx_wp.cu, pfb_fixedwing.cu, pfb_rocket.cu, pfb_dogfight.cu).
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
  if (!mask || !h->env.autoreset || !h->d_done_list) return 0;
  const uint64_t k = h->step_seq;  // the next step: its tail CTAs read list [(k - 1) % 4]
  k_drop_masked_done<<<1, 1024, 0, s>>>(h->d_done_list + ((k + 3) % 4) * h->n, h->d_counters + ((k + 3) % 4), mask);
  LAUNCH_CHECK(h);
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
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    return fail("no CUDA device: libpyflyt_b200 has no CPU fallback (%s)", e != cudaSuccess ? cudaGetErrorString(e) : "0 devices");
  if (device < 0 || device >= count) return fail("device %d out of range (have %d)", device, count);
  CUDA_OK(cudaSetDevice(device));
  PfbContext* c = new (std::nothrow) PfbContext();
  if (!c) return fail("out of host memory");
  memset(c, 0, sizeof(*c));
  c->model = *model;
  if (env) c->env = *env;
  else c->env.contact_response = aviary_contact;
  c->n = n_envs;
  c->device = device;
  if (model->kind == PFB_KIND_QUADX) {
    if (build_quadx_params(*model, c->qx) != 0) { delete c; return -1; }
  } else if (model->kind == PFB_KIND_FIXEDWING) {
    if (fw_build_params(*model, env, c->fw, c->wp) != 0) { delete c; return -1; }
    if (df_build_params(env, c->df) != 0) { delete c; return -1; }
    if (env && env->env_kind == PFB_ENV_DOGFIGHT && (n_envs % (2 * env->team_size)) != 0) {
      delete c;
      return fail("n_envs (%lld) must be a multiple of the arena size 2*team_size = %d", (long long)n_envs, 2 * env->team_size);
    }
  } else {
    if (rk_build_params(*model, env, c->rk, c->land) != 0) { delete c; return -1; }
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
  if (c->hover.ma && env->autoreset) {
    delete c;
    return fail("MAQuadXHover is a per-agent epilogue: arenas are reset by the caller (pfb_env_reset with a mask), autoreset must be 0");
  }
  if (env && env->env_kind != PFB_ENV_NONE) {
    const bool ok = (model->kind == PFB_KIND_QUADX && env->env_kind == PFB_ENV_QUADX_HOVER) ||
                    (model->kind == PFB_KIND_QUADX && env->env_kind == PFB_ENV_QUADX_WAYPOINTS) ||
                    (model->kind == PFB_KIND_QUADX && env->env_kind == PFB_ENV_MA_QUADX_HOVER) ||
                    (model->kind == PFB_KIND_FIXEDWING && env->env_kind == PFB_ENV_FIXEDWING_WAYPOINTS) ||
                    (model->kind == PFB_KIND_FIXEDWING && env->env_kind == PFB_ENV_DOGFIGHT) ||
                    (model->kind == PFB_KIND_ROCKET && env->env_kind == PFB_ENV_ROCKET_LANDING);
    if (!ok) {
      delete c;
      return fail("env kind %d is not available for vehicle kind %d in this library", env->env_kind, model->kind);
    }
  }
  if (env && env->env_kind == PFB_ENV_QUADX_WAYPOINTS) {
    if (env->num_targets < 1 || env->num_targets > kMaxTargets) {
      delete c;
      return fail("num_targets must be in 1..%d, got %d", kMaxTargets, env->num_targets);
    }
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
  c->rng.k0 = (uint32_t)seed;
  c->rng.k1 = (uint32_t)(seed >> 32);
  c->mode = 0;
  cudaDeviceProp prop;
  CUDA_OK(cudaGetDeviceProperties(&prop, device));
  c->sm_count = prop.multiProcessorCount;
  CUDA_OK(cudaMalloc(&c->d_counters, 8 * sizeof(int32_t)));  // [0..3] rotating autoreset counters, [4] ticket of the split dogfight
  CUDA_OK(cudaMemset(c->d_counters, 0, 8 * sizeof(int32_t)));
  CUDA_OK(cudaMalloc(&c->d_done_list, 4 * (size_t)n_envs * sizeof(int32_t)));
  if (env && env->autoreset && (env->env_kind == PFB_ENV_QUADX_HOVER || env->env_kind == PFB_ENV_FIXEDWING_WAYPOINTS ||
                                 env->env_kind == PFB_ENV_QUADX_WAYPOINTS || env->env_kind == PFB_ENV_ROCKET_LANDING ||
                                 env->env_kind == PFB_ENV_DOGFIGHT)) {
    // spare post-reset states: env-major records (QuadX-Hover: four per env, buffer = episode number & 3, rebuilt by builder
    // CTAs inside the step launches; the other env kinds: one per env, rebuilt on a library-owned side stream)
    const bool hover = env->env_kind == PFB_ENV_QUADX_HOVER;
    size_t rec = (size_t)hover_spare_rows();  // floats per env
    if (env->env_kind == PFB_ENV_QUADX_WAYPOINTS) rec = (size_t)qwp_spare_rows();
    else if (env->env_kind == PFB_ENV_FIXEDWING_WAYPOINTS) rec = (size_t)fw_spare_rows();
    else if (env->env_kind == PFB_ENV_ROCKET_LANDING) rec = (size_t)rk_spare_rows();
    else if (env->env_kind == PFB_ENV_DOGFIGHT) rec = (size_t)df_spare_rows();
    c->spare_bytes = rec * (size_t)n_envs * sizeof(float);
    CUDA_OK(cudaMalloc(&c->d_spare, c->spare_bytes));
    CUDA_OK(cudaMemset(c->d_spare, 0, c->spare_bytes));
    if (hover) {
      CUDA_OK(cudaMalloc(&c->d_consumed, (size_t)hover_consumed_rows() * (size_t)n_envs * sizeof(int2)));  // (env, episode) per reset of a fused launch
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
  *out = c;
  return 0;
}

int pfb_destroy(PfbHandle h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  if (h->d_spare) {
    if (h->side) {
      cudaStreamSynchronize(h->side);
      cudaStreamDestroy(h->side);
      cudaEventDestroy(h->ev_step);
      for (int k = 0; k < 4; ++k) cudaEventDestroy(h->ev_spare[k]);
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

static inline bool is_fw(PfbHandle h) { return h->model.kind == PFB_KIND_FIXEDWING; }
static inline bool is_rk(PfbHandle h) { return h->model.kind == PFB_KIND_ROCKET; }
static inline bool is_qwp(PfbHandle h) { return h->model.kind == PFB_KIND_QUADX && h->env.env_kind == PFB_ENV_QUADX_WAYPOINTS; }
static inline bool is_ma(PfbHandle h) { return h->model.kind == PFB_KIND_QUADX && h->env.env_kind == PFB_ENV_MA_QUADX_HOVER; }
static inline bool is_df(PfbHandle h) { return h->model.kind == PFB_KIND_FIXEDWING && h->env.env_kind == PFB_ENV_DOGFIGHT; }
int pfb_state_rows(PfbHandle h) { return is_rk(h) ? rk_state_rows() : (is_fw(h) ? fw_state_rows() : (is_qwp(h) ? qwp_state_rows() : qx_rows(h))); }
int pfb_state_layout(PfbHandle h) { return h && qx_tiled(h) ? PFB_LAYOUT_WARP_TILED : PFB_LAYOUT_FIELD_MAJOR; }
int64_t pfb_state_floats(PfbHandle h) {
  if (!h) return 0;
  if (qx_tiled(h)) return ((h->n + kTileLanes - 1) / kTileLanes) * qx_tile_floats(qx_rows(h));  // padded to whole tiles
  return (int64_t)pfb_state_rows(h) * h->n;
}
int pfb_istate_rows(PfbHandle h) { return is_rk(h) ? rk_istate_rows() : (is_fw(h) ? fw_istate_rows() : (is_qwp(h) ? qwp_istate_rows() : QI_ROWS)); }
int pfb_setpoint_dim(PfbHandle h) { return is_rk(h) ? 7 : ((is_fw(h) && h->env.env_kind == PFB_ENV_NONE) ? 6 : 4); }
int pfb_obs_dim(PfbHandle h) { return is_df(h) ? df_obs_dim(h) : is_rk(h) ? rk_obs_dim(h) : (is_fw(h) ? fw_obs_dim(h) : (is_qwp(h) ? qwp_obs_dim(h) : (h->hover.angle_representation == 0 ? 20 : 21) + (is_ma(h) ? 3 : 0))); }
int pfb_aux_dim(PfbHandle h) { return is_rk(h) ? 9 : (is_fw(h) ? 6 : 4); }

int pfb_bind(PfbHandle h, const PfbBuffers* b) {
  if (!h || !b) return fail("pfb_bind: null argument");
  if (!b->state || !b->istate || !b->setpoint || !b->start_pos || !b->start_orn)
    return fail("pfb_bind: state, istate, setpoint, start_pos and start_orn are mandatory");
  if (((uintptr_t)b->setpoint & 15) || ((uintptr_t)b->state & 15)) return fail("pfb_bind: buffers must be 16-byte aligned");
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
  cudaStream_t s = (cudaStream_t)stream;
  if (is_fw(h)) return fw_reset(h, mask, s);
  if (is_rk(h)) return rk_reset(h, mask, s);
  return qx_reset(h, mask, s);
}

int pfb_set_mode(PfbHandle h, int mode, void* stream) {
  REQUIRE_BOUND(h);
  cudaStream_t s = (cudaStream_t)stream;
  if (is_fw(h)) return fw_set_mode(h, mode, s);
  if (is_rk(h)) return rk_set_mode(h, mode, s);
  return qx_set_mode(h, mode, s);
}

int pfb_set_modes(PfbHandle h, const int8_t* modes, void* stream) {
  if (!h || !modes) return fail("pfb_set_modes: null argument");
  if (h->env.env_kind != PFB_ENV_NONE)
    return fail("pfb_set_modes: only Aviary handles fly one flight mode per drone; a handle with an env epilogue flies its env's flight_mode");
  REQUIRE_BOUND(h);
  const int lo = is_rk(h) ? 0 : -1, hi = is_rk(h) || is_fw(h) ? 0 : 7;  // quadx.py:259-262, fixedwing.py:216-219, rocket: mode 0 only
  bool uniform = true;
  for (int64_t i = 0; i < h->n; ++i) {
    if (modes[i] < lo || modes[i] > hi)
      return fail("pfb_set_modes: modes[%lld] = %d, must be between %d and %d for this vehicle kind", (long long)i, (int)modes[i], lo, hi);
    uniform = uniform && modes[i] == modes[0];
  }
  if (uniform) return pfb_set_mode(h, modes[0], stream);  // one mode: the uniform kernels
  cudaStream_t s = (cudaStream_t)stream;
  const size_t padded = (size_t)grid_for(h->n) * kBlock;  // whole tiles, like d_model_index
  if (!h->d_modes) {
    CUDA_OK(cudaMalloc(&h->d_modes, padded));
    CUDA_OK(cudaMemsetAsync(h->d_modes, 0, padded, s));
  }
  // stream-ordered: a step still queued on `s` reads the previous modes
  CUDA_OK(cudaMemcpyAsync(h->d_modes, modes, (size_t)h->n, cudaMemcpyHostToDevice, s));
  if (is_fw(h)) return fw_set_modes(h, s);
  return qx_set_modes(h, s);
}

int pfb_aviary_step(PfbHandle h, int n_steps, const float* noise, void* stream) {
  REQUIRE_BOUND(h);
  if (n_steps <= 0) return fail("n_steps must be positive");
  cudaStream_t s = (cudaStream_t)stream;
  if (is_fw(h)) return fw_aviary_step(h, n_steps, noise, s);
  if (is_rk(h)) return rk_aviary_step(h, n_steps, noise, s);
  return qx_aviary_step(h, n_steps, noise, s);
}

int pfb_set_base_velocity(PfbHandle h, const float* lin_vel, const float* ang_vel, void* stream) {
  REQUIRE_BOUND(h);
  if (!lin_vel || !ang_vel) return fail("pfb_set_base_velocity: null argument");
  if (is_rk(h)) return rk_set_velocity(h, lin_vel, ang_vel, (cudaStream_t)stream);
  return fail("pfb_set_base_velocity is only built for the rocket (the one vehicle whose env calls resetBaseVelocity)");
}

int pfb_observe_state(PfbHandle h, void* stream) {
  REQUIRE_BOUND(h);
  if (is_fw(h)) return fw_observe(h, (cudaStream_t)stream);
  if (is_rk(h)) return rk_observe(h, (cudaStream_t)stream);
  return qx_observe(h, (cudaStream_t)stream);
}

static int require_env(PfbHandle h) {
  if (h->env.env_kind == PFB_ENV_NONE) return fail("handle was created without an env epilogue");
  if (!h->buf.obs || !h->buf.reward || !h->buf.term || !h->buf.trunc) return fail("obs/reward/term/trunc buffers are not bound");
  return 0;
}

int pfb_env_reset(PfbHandle h, const uint8_t* mask, const float* noise, void* stream) {
  REQUIRE_BOUND(h);
  if (require_env(h)) return -1;
  h->fused_ready = 0;
  cudaStream_t s = (cudaStream_t)stream;
  if (is_df(h)) return df_env_reset(h, mask, noise, s);
  if (is_fw(h)) return fw_env_reset(h, mask, noise, s);
  if (is_rk(h)) return rk_env_reset(h, mask, noise, s);
  if (is_qwp(h)) return qwp_env_reset(h, mask, noise, s);
  return hover_env_reset(h, mask, noise, s);
}

// `dyn_smem`: dynamic shared memory the QuadX-Hover step launch requests and never touches (pfb_env_step_mapped)
static int env_step_impl(PfbHandle h, float* actions, const float* noise, bool randact, size_t dyn_smem, cudaStream_t s) {
  if (is_df(h)) return df_env_step(h, actions, noise, randact, s);
  if (is_fw(h)) return fw_env_step(h, actions, noise, randact, s);
  if (is_rk(h)) return rk_env_step(h, actions, noise, randact, s);
  if (is_qwp(h)) return qwp_env_step(h, actions, noise, randact, s);
  return hover_env_step(h, actions, noise, randact, dyn_smem, s);
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
    if (h->env.env_kind == PFB_ENV_QUADX_HOVER) {
      if (hover_invalidate_spares(h, 0)) return -1;
    } else {
      const int valid = is_df(h) ? df_spare_valid_row() : is_rk(h) ? rk_spare_valid_row() : is_qwp(h) ? qwp_spare_valid_row() : fw_spare_valid_row();
      const size_t rows = (size_t)(is_df(h) ? df_spare_rows() : is_rk(h) ? rk_spare_rows() : is_qwp(h) ? qwp_spare_rows() : fw_spare_rows());
      CUDA_OK(cudaMemset2DAsync(h->d_spare + valid, rows * sizeof(float), 0, sizeof(float), (size_t)h->n, 0));
    }
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
  if (h->model.kind != PFB_KIND_QUADX) return fail("pfb_set_models: only QuadX handles fly several vehicle models");
  if (is_ma(h)) return fail("pfb_set_models: MAQuadXHover handles fly one vehicle model");
  if (k < 1 || k > PFB_MAX_QUADX_MODELS) return fail("pfb_set_models: k = %d, must be in 1..%d", k, PFB_MAX_QUADX_MODELS);
  QuadXParams tables[PFB_MAX_QUADX_MODELS];
  for (int j = 0; j < k; ++j) {
    const PfbModel& m = models[j];
    if (m.abi_version != PFB_ABI_VERSION) return fail("pfb_set_models: model %d has ABI %d != library ABI %d", j, m.abi_version, PFB_ABI_VERSION);
    if (m.kind != PFB_KIND_QUADX) return fail("pfb_set_models: model %d is not a QuadX (kind %d)", j, m.kind);
    // every kernel runs ONE substep ratio and one dt per handle
    if (m.physics_hz != models[0].physics_hz || m.control_hz != models[0].control_hz)
      return fail("pfb_set_models: model %d runs at physics_hz %g / control_hz %g, model 0 at %g / %g: every model of a handle needs the same rates", j,
                  m.physics_hz, m.control_hz, models[0].physics_hz, models[0].control_hz);
    memset(&tables[j], 0, sizeof(QuadXParams));
    if (build_quadx_params(m, tables[j]) != 0) return -1;
    if (tables[j].ratio != tables[0].ratio || tables[j].dt != tables[0].dt || tables[j].ctrl_dt != tables[0].ctrl_dt ||
        tables[j].noise_loc != tables[0].noise_loc)
      return fail("pfb_set_models: model %d has a different substep ratio, dt or motor count than model 0", j);
  }
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
  if (!h->qxset) {
    h->qxset = new (std::nothrow) QuadXModelSet();
    if (!h->qxset) return fail("out of host memory");
  }
  memset(h->qxset, 0, sizeof(QuadXModelSet));
  for (int j = 0; j < k; ++j) {
    h->qxset->m[j] = tables[j];
    h->qxset->m[j].wind = wind;
  }
  const size_t padded = (size_t)grid_for(h->n) * kBlock;  // whole tiles: the tile kernels read the index of every lane
  if (!h->d_model_index) CUDA_OK(cudaMalloc(&h->d_model_index, padded));
  CUDA_OK(cudaMemset(h->d_model_index, 0, padded));
  CUDA_OK(cudaMemcpy(h->d_model_index, index_host, (size_t)h->n, cudaMemcpyHostToDevice));
  h->qxset->index = h->d_model_index;
  return 0;
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
  return env_step_impl(h, actions ? const_cast<float*>(actions) : h->buf.setpoint, noise, false, 0, (cudaStream_t)stream);
}

int pfb_env_rollout(PfbHandle h, int n_steps, void* stream) {
  REQUIRE_BOUND(h);
  if (require_env(h)) return -1;
  if (qx_tiled(h)) return hover_env_rollout(h, n_steps, (cudaStream_t)stream);  // an env handle: QuadX-Hover or MAQuadXHover
  for (int k = 0; k < n_steps; ++k)
    if (env_step_impl(h, h->buf.setpoint, nullptr, true, 0, (cudaStream_t)stream)) return -1;
  return 0;
}

int pfb_env_step_host(PfbHandle h, const float* host_actions, float* host_obs, float* host_reward, uint8_t* host_term,
                      uint8_t* host_trunc, void* stream) {
  REQUIRE_BOUND(h);
  if (require_env(h)) return -1;
  cudaStream_t s = (cudaStream_t)stream;
  const int O = pfb_obs_dim(h);
  CUDA_OK(cudaMemcpyAsync(h->buf.setpoint, host_actions, (size_t)h->n * pfb_setpoint_dim(h) * sizeof(float), cudaMemcpyHostToDevice, s));
  if (env_step_impl(h, h->buf.setpoint, nullptr, false, 0, s)) return -1;
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
  const int rc = env_step_impl(h, (float*)da, nullptr, false, kMappedDynSmem, (cudaStream_t)stream);
  h->buf = saved;
  return rc;
}

// ---- MAFixedwingDogfight, split variant: an arena's agents on different ranks (DESIGN.md §7)
int pfb_dogfight_payload_dim(void) { return 20; }

int pfb_dogfight_physics(PfbHandle h, const float* actions, const float* noise, float* payload_out, int first, int do_reset, int aviary_index,
                         void* stream) {
  REQUIRE_BOUND(h);
  if (!is_df(h)) return fail("handle is not a dogfight env");
  if (!payload_out) return fail("pfb_dogfight_physics: null payload buffer");
  return df_split_physics(h, actions ? actions : h->buf.setpoint, noise, payload_out, nullptr, 0, 0, nullptr, 0, 0, first, do_reset, aviary_index,
                          (cudaStream_t)stream);
}

int pfb_dogfight_physics_peer(PfbHandle h, const float* actions, const float* noise, const uint64_t* peer_tables_dev, int world,
                             int64_t slot_offset_floats, const uint64_t* peer_flags_dev, int rank, int epoch, int first, int do_reset,
                             int aviary_index, void* stream) {
  REQUIRE_BOUND(h);
  if (!is_df(h)) return fail("handle is not a dogfight env");
  if (!peer_tables_dev || world < 1) return fail("pfb_dogfight_physics_peer: need the device array of peer table pointers");
  return df_split_physics(h, actions ? actions : h->buf.setpoint, noise, nullptr, peer_tables_dev, world, slot_offset_floats, peer_flags_dev, rank,
                          epoch, first, do_reset, aviary_index, (cudaStream_t)stream);
}

int pfb_dogfight_combat(PfbHandle h, const float* payload_table, int64_t first_global_agent, int64_t num_arenas, int last, void* stream) {
  REQUIRE_BOUND(h);
  if (!is_df(h)) return fail("handle is not a dogfight env");
  if (require_env(h)) return -1;
  return df_split_combat(h, payload_table, first_global_agent, num_arenas, last, nullptr, 0, 0, (cudaStream_t)stream);
}

int pfb_dogfight_combat_wait(PfbHandle h, const float* payload_table, int64_t first_global_agent, int64_t num_arenas, int last,
                             const int32_t* flags, int world, int epoch, void* stream) {
  REQUIRE_BOUND(h);
  if (!is_df(h)) return fail("handle is not a dogfight env");
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
  if (!is_df(h)) return fail("handle is not a dogfight env");
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
