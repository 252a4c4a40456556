// pfb_quadx.cu — QuadX kernels (Aviary surface, QuadX-Hover and MAQuadXHover envs) and their launchers.
//
// One thread integrates one env; the whole env step (control ticks, physics substeps, reward,
// termination, observation) happens in registers between one coalesced load and one store.
// The Hover step moves a warp's 32-env state tile and observation tile with one TMA bulk copy each.
#include <cuda_runtime.h>

#include "pfb_aviary.cuh"

using namespace pfb;

// ---------------------------------------------------------------------------------------------------
// kernels — Aviary surface
// ---------------------------------------------------------------------------------------------------
// Aviary.reset + QuadX.reset + update_state (aviary.py:218-312, quadx.py:222-231)
template <bool TILED>
__global__ void __launch_bounds__(kBlock) k_quadx_reset(float* __restrict__ st, int32_t* __restrict__ ist, int rows,
                                                        float* __restrict__ setpoint, const float* __restrict__ start_pos,
                                                        const float* __restrict__ start_orn,
                                                        const uint8_t* __restrict__ mask, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  if (mask && !mask[i]) return;
  qx_reset_drone<TILED>(st, ist, rows, N, i, start_pos, start_orn, i);
  if (setpoint) reinterpret_cast<float4*>(setpoint)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// Aviary.set_mode -> QuadX.set_mode (quadx.py:233-373): preset the setpoint, fresh attitude/position PIDs
template <int MODE, bool TILED>
__global__ void __launch_bounds__(kBlock) k_quadx_set_mode(float* __restrict__ st, int32_t* __restrict__ ist, int rows,
                                                           float* __restrict__ setpoint, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  QuadXRegs s;
  int step_count;
  qx_load_any<7, TILED>(st, ist, rows, N, i, s, step_count);
  float4 sp = reinterpret_cast<const float4*>(setpoint)[i];
  s.sp[0] = sp.x; s.sp[1] = sp.y; s.sp[2] = sp.z; s.sp[3] = sp.w;
  quadx_set_mode<MODE>(s);
  qx_store_any<7, TILED>(st, ist, rows, N, i, s, step_count);
  reinterpret_cast<float4*>(setpoint)[i] = make_float4(s.sp[0], s.sp[1], s.sp[2], s.sp[3]);
}

// n_steps x Aviary.step() (aviary.py:480-531) in flight mode MODE, or MODE = kModePerDrone: drone i in modes[i] (pfb_set_modes).
// Per-drone modes move every PID row (the mode-7 set); quadx_mask_pid gives each drone the PID memory the uniform kernel of its
// mode would load, so both store the same words.  CONTACT: the floor pushes back (Aviary handles with contact_response).
// World = StaticCtx: against the static bodies of each drone's world (pfb_add_static_body), bits[i] = what drone i touched
// during its last Aviary step.  TILED = false (field-major state) is QuadX-Waypoints' layout, which has none of the three.
template <int MODE, bool INJECT, bool TILED, class PS, bool CONTACT, class World>
__global__ void __launch_bounds__(kBlock, kMinBlocks)
    k_quadx_aviary_step(const __grid_constant__ PS ps, const __grid_constant__ RngParams rng, const __grid_constant__ typename WorldTable<World>::T world,
                        const float* __restrict__ pose, uint32_t* __restrict__ bits, float* __restrict__ st, int32_t* __restrict__ ist, int rows,
                        const float* __restrict__ setpoint, const int8_t* __restrict__ modes, const float* __restrict__ noise, int n_steps,
                        uint32_t seq, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  constexpr bool kPerDrone = MODE == kModePerDrone;
  constexpr int LM = kPerDrone ? 7 : MODE;  // the PID rows moved
  const QuadXParams& p = qx_model(ps, i);
  World w{&world, pose, N, i, 0u};
  int mode = MODE;
  if constexpr (kPerDrone && !World::kOn) mode = modes[i];  // where the mode is read steers ptxas' schedule (DESIGN.md §4h)
  QuadXRegs s;
  int step_count;
  qx_load_any<LM, TILED>(st, ist, rows, N, i, s, step_count);
  if constexpr (kPerDrone && World::kOn) mode = modes[i];
  if constexpr (kPerDrone) quadx_mask_pid(s, mode);
  float4 sp = __ldg(reinterpret_cast<const float4*>(setpoint) + i);
  s.sp[0] = sp.x; s.sp[1] = sp.y; s.sp[2] = sp.z; s.sp[3] = sp.w;
  auto nz = make_noise<INJECT>(noise, N, i, rng, seq, TAG_AVIARY, qx_model0(ps).noise_loc, qx_model0(ps).ratio);
  for (int k = 0; k < n_steps; ++k) {
    if constexpr (kPerDrone) quadx_aviary_step_any<CONTACT>(p, s, mode, nz, &w);
    else quadx_aviary_step<MODE, CONTACT>(p, s, nz, &w);
  }
  qx_store_any<LM, TILED>(st, ist, rows, N, i, s, step_count);
  if constexpr (World::kOn) bits[i] = w.bits;
}

// ---- one flight mode per drone (pfb_set_modes; Aviary handles, warp-tiled) ----------------------------------------------
// Aviary.set_mode(list): QuadX.set_mode(mode[i]) for every drone i, as k_quadx_set_mode does for one mode
__global__ void __launch_bounds__(kBlock) k_quadx_set_modes(float* __restrict__ st, int rows, float* __restrict__ setpoint,
                                                            const int8_t* __restrict__ modes, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  qx_set_mode_drone<4>(st, rows, i, modes, setpoint, i);
}

// Aviary.state(i) / aux_state(i) / contact_array  -> row-major API buffers
template <bool TILED>
__global__ void __launch_bounds__(kBlock) k_quadx_observe(const float* __restrict__ st, const int32_t* __restrict__ ist, int rows,
                                                          float* __restrict__ drone_state, float* __restrict__ aux,
                                                          uint8_t* __restrict__ contact, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  float o[12], a[4], hi[3], lo[3];
  const bool c = qx_query_drone<TILED>(st, ist, rows, N, i, o, a, hi, lo);
  if (drone_state) {
    float4* d = reinterpret_cast<float4*>(drone_state + 12 * i);
    d[0] = make_float4(o[0], o[1], o[2], o[3]);
    d[1] = make_float4(o[4], o[5], o[6], o[7]);
    d[2] = make_float4(o[8], o[9], o[10], o[11]);
  }
  if (aux) reinterpret_cast<float4*>(aux)[i] = make_float4(a[0], a[1], a[2], a[3]);
  if (contact) contact[i] = c ? 1 : 0;
}

// p.resetBasePositionAndOrientation / p.resetBaseVelocity + update_state (pfb_set_base_state; F32: pfb_set_base_velocity) and
// getBasePositionAndOrientation / getBaseVelocity (pfb_get_base_state); Aviary handles, warp-tiled
template <bool F32>
__global__ void __launch_bounds__(kBlock) k_quadx_set_base_state(const __grid_constant__ BaseStateIn a, float* __restrict__ st, int rows, int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  set_base_drone<F32>(PFB_KIND_QUADX, a, st, nullptr, rows, N, i, i);
}
__global__ void __launch_bounds__(kBlock) k_quadx_get_base_state(const __grid_constant__ BaseStateOut o, const float* __restrict__ st, int rows,
                                                                 int64_t N) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  qx_get_base_drone(st, rows, i, i, o);
}

// ---------------------------------------------------------------------------------------------------
// kernels — QuadX-Hover env (warp-tiled state)
// ---------------------------------------------------------------------------------------------------
// 16 one-warp CTAs (512 threads) per SM resident (<= 128 registers), so that the 2048 CTAs of a 65 536-env step and the builder
// CTAs of the spare rebuild (two per SM) are resident at once or nearly so.  On an H100 a small second wave remains; capping the
// builders to remove it was measured slower, because each builder then carries more of the serial warm-up chains (DESIGN.md §4)
constexpr int kHoverBlocks = 16;
constexpr int kObsMax = 24;  // floats per observation row (20 / 21, + 3 for MAQuadXHover)

// ---- spare post-reset states (DESIGN.md §4, "reset pipeline") ---------------------------------------
// env.reset() = start pose + `warmup_steps` Aviary steps (quadx_base_env.py:149-212): 3.3x the work of an env step and a
// strictly serial chain; run inline, even one finished env stretches the launch to the length of that chain.  So each env
// owns a SPARE, the post-warm-up state of its NEXT episode, with the warm-up noise keyed by (env id, episode number,
// Aviary step) so that it does not matter when it is computed.
//  * An env that finished on call k is reset on call k + 1 BY ITS OWN THREAD: the thread skips the physics loop and, at the
//    end of the launch, swaps the env's spare record in (staged into the warp's dead state-tile buffer by cp.async while the
//    other lanes integrate, kStageFloats below) — every observation row of a warp's tile is written by that warp.
//  * The spare it consumed is rebuilt INSIDE the following two step launches by a few BUILDER CTAs appended to the grid:
//    launch k + 1 (the one that consumes) integrates the first half of the next spare's warm-up, launch k + 2 the second
//    half — each half is shorter than an env step, so the builders never stretch a launch — and the spare is valid again
//    before launch k + 3, the earliest the env can be reset again.  A spare lives in buffer (episode & 3), so the builders
//    never write the record a resetting thread is reading.  One launch per env step: no side stream, no events.
//  * If the start pose was edited since a spare was built, or with inline_reset = 1, the spare is ignored and the warm-up
//    runs inline in the owning thread (same episode number, hence the same result).
// Library-owned: spare[kSpareBufs][N][SP_ROWS] ENV-MAJOR records (the QX_* state rows in record layout, group stride 4, then
// the words below) and episode[N], the episode number of each env's current valid spare (its buffer is episode & kSpareMask).
enum { SP_POSE = QX_ROWS, SP_VALID = QX_ROWS + 6, SP_FLAGS = QX_ROWS + 7, SP_EPISODE = QX_ROWS + 8,
       SP_SETPOINT = QX_ROWS + 12 /* 4: the flight mode's preset setpoint, carried between the two halves of a warm-up */, SP_ROWS = 80 };
static_assert(QX_ROWS % 4 == 0 && QX_ROWS + 16 <= SP_ROWS && SP_ROWS % 4 == 0, "spare record layout");
constexpr int kSpareBufs = 4;  // records per env, buffer = episode & 3: the step pipeline uses two neighbours (one being consumed, one being built);
constexpr uint32_t kSpareMask = kSpareBufs - 1;  // the fused rollout keeps three spares ahead (k_hover_rollout)
constexpr int kWarmSplit = 5;  // Aviary steps integrated by the first builder phase; every warm-up requantizes its state there

// the record of episode e of env i
template <class T>
__device__ __forceinline__ T* spare_rec(T* spare, uint32_t e, int64_t N, int64_t i) {
  return spare + ((int64_t)(e & kSpareMask) * N + i) * SP_ROWS;
}
// the words behind the state rows: the start pose the spare was built for, valid, flags and the episode number
__device__ __forceinline__ void spare_trailer(float* rec, float px, float py, float pz, float ox, float oy, float oz, float valid, uint32_t flags,
                                              uint32_t e) {
  st_f4(rec + SP_POSE, px, py, pz, ox);
  st_f4(rec + SP_POSE + 4, oy, oz, valid, f_from_bits(flags));
  st_f4(rec + SP_POSE + 8, f_from_bits(e), 0.0f, 0.0f, 0.0f);
}
// cp.async.bulk (TMA, 1-D) shared -> global: one instruction moves a warp's whole observation tile
__device__ __forceinline__ void bulk_store_s2g(void* gdst, const void* ssrc, uint32_t bytes) {
  const uint32_t sa = (uint32_t)__cvta_generic_to_shared(ssrc);
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(sa), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// cp.async.bulk (TMA, 1-D) global -> shared with mbarrier completion: the warp's state tile lands asynchronously while
// the warp runs its noise generator; try_wait is the point the loaded data is first needed
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(bar);
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(a), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void bulk_load_g2s(void* sdst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(sdst), b = (uint32_t)__cvta_generic_to_shared(bar);
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(d), "l"(gsrc), "r"(bytes), "r"(b)
               : "memory");
}
// `dep`: values that must have been COMPUTED before the wait starts (the asm consumes them, no instruction is emitted for
// them): keeps work that does not need the tile — the noise generator — in front of the wait instead of behind it
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, float d0 = 0.f, float d1 = 0.f, float d2 = 0.f, float d3 = 0.f,
                                          float d4 = 0.f, float d5 = 0.f, float d6 = 0.f, float d7 = 0.f) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(bar);
  asm volatile(
      "{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}" ::"r"(a),
      "r"(parity), "f"(d0), "f"(d1), "f"(d2), "f"(d3), "f"(d4), "f"(d5), "f"(d6), "f"(d7)
      : "memory");
}
__device__ __forceinline__ void bulk_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
// per-thread asynchronous copies global -> shared (LDGSTS): issued and forgotten, complete in the background, waited for with
// cp_async_wait_all() by the issuing thread, which may then read what it copied
__device__ __forceinline__ void cp_async16(float* sdst, const float* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(sdst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async4(float* sdst, const float* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(sdst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// Staging of spare records (reset by the owning thread): a resetting lane copies its 320-byte record — in the step kernel also the
// start pose the record is checked against — into the warp's state-tile buffer, which is dead once the tile has been unpacked.
// The copies fly while the other lanes integrate; the swap at the end of the step then reads shared memory instead of making two
// or three DEPENDENT trips to L2 / DRAM (valid word -> pose -> state).
constexpr int kStageFloats = SP_ROWS + 8;

// env.reset() integrated inline (quadx_base_env.py:149-212): Aviary steps [from, to) of the warm-up that follows the start
// pose + set_mode.  The state is rounded to what a record holds (hi + lo words) before step kWarmSplit in EVERY path, so a
// warm-up integrated in two launches through a spare record equals one integrated in one go, bit for bit.
// The INLINE form is what the builder CTAs and the reset / build kernels run: `p` must be the kernel's __grid_constant__
// parameter so that the coefficients stay constant-bank operands.
template <int MODE, bool INJECT>
__device__ __forceinline__ void hover_warmup_inline(const QuadXParams& p, QuadXRegs& s, int from, int to, const RngParams& rng,
                                                    const float* __restrict__ noise, int64_t N, int64_t i, uint32_t seq) {
  auto nz = make_noise<INJECT>(noise, N, i, rng, seq, TAG_RESET, p.noise_loc, p.ratio);
  nz.seek((uint32_t)from);
#pragma unroll 1
  for (int k = from; k < to; ++k) {
    if (k == kWarmSplit) quadx_requantize(s);
    quadx_aviary_step<MODE>(p, s, nz);
  }
}
// Out-of-line form for the COLD fallback inside the step role (a spare that cannot be used): everything by value, so the
// caller's register-resident state never has its address taken.  Slow (the coefficient table is read from the stack copy),
// and rare.  A uniform-table kernel must name its __grid_constant__ parameter itself in the call (kUniform below): a copy
// made through a reference to it makes nvcc stage the whole parameter in local memory first, a second 640-byte stack copy.
template <int MODE>
__device__ __noinline__ QuadXRegs hover_warmup_cold(const QuadXParams p, QuadXRegs s, int to, const RngParams rng, int64_t N, int64_t i,
                                                    uint32_t seq) {
  hover_warmup_inline<MODE, false>(p, s, 0, to, rng, nullptr, N, i, seq);
  return s;
}
// a freshly constructed drone in flight mode MODE at its start pose (quadx.py:222-231, quadx_base_env.py:186-207)
template <int MODE>
__device__ __forceinline__ QuadXRegs hover_fresh(float px, float py, float pz, float ox, float oy, float oz) {
  QuadXRegs s;
  quadx_reset(s, px, py, pz, ox, oy, oz);
  quadx_set_mode<MODE>(s);
  return s;
}
// env.reset() without a usable spare, in the step role: the whole warm-up out of line, rounded to exactly what a copied spare
// holds.  A macro, because a uniform-table kernel must name its __grid_constant__ parameters themselves (see hover_warmup_cold)
#define HOVER_RESET_COLD(s, px, py, pz, ox, oy, oz, seq)                                                                         \
  do {                                                                                                                          \
    if constexpr (kUniform<PS>) s = hover_warmup_cold<MODE>(ps, hover_fresh<MODE>(px, py, pz, ox, oy, oz), h.warmup_steps, rng, N, i, seq); \
    else s = hover_warmup_cold<MODE>(p, hover_fresh<MODE>(px, py, pz, ox, oy, oz), h.warmup_steps, rng, N, i, seq);                    \
    quadx_requantize(s);                                                                                                        \
  } while (0)

// the per-env outputs of an env step besides the observation
__device__ __forceinline__ void hover_step_outputs(float* reward, uint8_t* term, uint8_t* trunc, uint8_t* info, int64_t i, float rew, uint32_t flags) {
  reward[i] = rew;
  term[i] = (flags & FLAG_TERM) ? 1 : 0;
  trunc[i] = (flags & FLAG_TRUNC) ? 1 : 0;
  if (info) info[i] = (uint8_t)(((flags & FLAG_OOB) ? 1 : 0) | ((flags & FLAG_COLLISION) ? 2 : 0));
}

// Builder CTAs of the step launch (the first 2 * builders CTAs of the grid): the first `builders` of them (phase 0) start the next
// spare of the envs that are being reset by this launch (done list of the previous launch), the others (phase 1) finish the
// spares started by the previous launch.  ONE copy of the warm-up loop serves both phases.  Each spare is integrated with the
// table of the env it belongs to.
template <int MODE, class PS>
__device__ __forceinline__ void hover_build(const PS& ps, const HoverParams& h, const RngParams& rng, int b, int builders,
                                            const int32_t* __restrict__ b0_count, const int32_t* __restrict__ b0_list,
                                            const int32_t* __restrict__ b1_count, const int32_t* __restrict__ b1_list,
                                            uint32_t* __restrict__ b0_elist, const uint32_t* __restrict__ b1_elist,
                                            const float* __restrict__ start_pos, const float* __restrict__ start_orn,
                                            float* __restrict__ spare, uint32_t* __restrict__ episode, int64_t N) {
  const int phase = b >= builders ? 1 : 0;
  const int slot = b - phase * builders;
  const int32_t* __restrict__ list = phase ? b1_list : b0_list;
  // The builders' chain of DEPENDENT cold loads (count -> list entry -> episode number -> record) is what they wait for while the
  // step CTAs' tile burst saturates DRAM: the first list entry (and, in phase 1, the episode number phase 0 left next to it) is
  // loaded speculatively together with the count — the lists are N entries long, so any index below N is readable
  int t = slot * kBlock + (int)threadIdx.x;
  const int64_t t_spec = t < N ? t : N - 1;
  int32_t i_spec = list[t_spec];
  uint32_t e_spec = phase ? b1_elist[t_spec] : 0u;
  const int t_end = phase ? *b1_count : *b0_count;
  const int split = h.warmup_steps < kWarmSplit ? h.warmup_steps : kWarmSplit;
#pragma unroll 1
  for (; t < t_end; t += builders * kBlock) {
    const int64_t i = i_spec;
    // the spare being built; the one being consumed (episode[i]) lives in the other buffer
    const uint32_t e = phase ? e_spec : episode[i] + 1u;
    float* rec = spare_rec(spare, e, N, i);
    QuadXRegs s;
    float px = 0.f, py = 0.f, pz = 0.f, ox = 0.f, oy = 0.f, oz = 0.f;
    if (phase == 0) {
      px = start_pos[3 * i + 0]; py = start_pos[3 * i + 1]; pz = start_pos[3 * i + 2];
      ox = start_orn[3 * i + 0]; oy = start_orn[3 * i + 1]; oz = start_orn[3 * i + 2];
      s = hover_fresh<MODE>(px, py, pz, ox, oy, oz);
      b0_elist[t] = e;  // read by phase 1 of the next launch (same list, same position)
    } else {
      int dummy;
      quadx_load_tile<7, 4>(rec, s, dummy);
      const F4 sp = ld_f4(rec + SP_SETPOINT);
      s.sp[0] = sp.x; s.sp[1] = sp.y; s.sp[2] = sp.z; s.sp[3] = sp.w;
    }
    hover_warmup_inline<MODE, false>(qx_model(ps, i), s, phase ? split : 0, phase ? h.warmup_steps : split, rng, nullptr, N, i, e);
    quadx_store_tile<7, 4>(rec, s, 0);
    if (phase == 0) {
      spare_trailer(rec, px, py, pz, ox, oy, oz, 0.0f, 0u, e);  // not valid yet
      st_f4(rec + SP_SETPOINT, s.sp[0], s.sp[1], s.sp[2], s.sp[3]);
    } else {
      rec[SP_FLAGS] = f_from_bits(s.flags);
      rec[SP_VALID] = 1.0f;
      episode[i] = e;
    }
    const int tn = t + builders * kBlock;  // more finished envs than builder lanes (a synchronised truncation): next pass
    if (tn < t_end) {
      i_spec = list[tn];
      if (phase) e_spec = b1_elist[tn];
    }
  }
}

// env.step(action) for every env (quadx_base_env.py:269-301 + quadx_hover_env.py), ONE launch, one warp per CTA, one tile
// of 32 envs per warp.
//   RANDACT   actions are drawn on device, uniform in the env's action box (quadx_base_env.py:79-102)
//   AUTORESET gymnasium NEXT_STEP autoreset: an env that finished on the previous call is reset on this one (its action
//             is ignored; obs = first observation of the new episode, reward 0, flags cleared)
template <int MODE, bool INJECT, bool RANDACT, bool AUTORESET, bool MA, class PS>
__global__ void __launch_bounds__(kBlock, kHoverBlocks)
    k_hover_step(const __grid_constant__ PS ps, const __grid_constant__ HoverParams h,
                 const __grid_constant__ RngParams rng, float* __restrict__ st, int rows, float* __restrict__ actions,
                 const float* __restrict__ noise, float* __restrict__ obs, float* __restrict__ reward, uint8_t* __restrict__ term,
                 uint8_t* __restrict__ trunc, uint8_t* __restrict__ info, const float* __restrict__ start_pos,
                 const float* __restrict__ start_orn, int32_t* __restrict__ cur_count, int32_t* __restrict__ cur_list,
                 int32_t* __restrict__ next_count, const int32_t* __restrict__ b0_count, const int32_t* __restrict__ b0_list,
                 const int32_t* __restrict__ b1_count, const int32_t* __restrict__ b1_list, uint32_t* __restrict__ b0_elist,
                 const uint32_t* __restrict__ b1_elist, float* __restrict__ spare, uint32_t* __restrict__ episode, int spare_copy, int builders,
                 float* __restrict__ noise_dump, uint32_t step_seq, int64_t N) {
  // builder CTAs come FIRST in the grid: their serial warm-up chain is the longest thing in the launch, so they must be
  // dispatched at t = 0, not behind the ~2000 step CTAs
  const int n_build = AUTORESET ? 2 * builders : 0;
  if (AUTORESET && (int)blockIdx.x < n_build) {  // builder CTA (CTA-uniform role)
    hover_build<MODE>(ps, h, rng, (int)blockIdx.x, builders, b0_count, b0_list, b1_count, b1_list, b0_elist, b1_elist, start_pos, start_orn, spare,
                      episode, N);
    return;
  }
  const int tile = (int)blockIdx.x - n_build;
  __shared__ __align__(128) float smem[kBlock * kObsMax];
  const int O = (h.angle_representation == 0 ? 20 : 21) + (MA ? 3 : 0);
  const int lane = threadIdx.x;
  const int64_t tile_first = (int64_t)tile * kBlock;
  const int64_t i = tile_first + lane;
  const bool active = i < N;
  const QuadXParams& p = qx_model(ps, i);  // the model index is padded to whole tiles: every lane may read it
  if (AUTORESET && tile == 0 && lane == 0) *next_count = 0;  // arm the counter the NEXT launch appends to
  float* rec = st + qx_tile_base(i, rows);  // the state tensor is padded to whole tiles: every lane may load

  // ---- the warp's state tile (groups 0 .. n-1: everything MODE reads) comes in with ONE cp.async.bulk (TMA) into shared
  //      memory; the noise generator and the action fetch run while it is in flight
  constexpr int kInGroups = qx_groups_moved<MODE>();
  __shared__ __align__(128) float stile[kInGroups * kTileGroupStride];
  __shared__ __align__(8) uint64_t mbar;
  if (lane == 0) {
    mbar_init(&mbar, 1);
    bulk_load_g2s(stile, st + qx_tile_base(tile_first, rows), (uint32_t)(kInGroups * kTileGroupStride * sizeof(float)), &mbar);
  }
  __syncwarp();
  float act[4] = {0.f, 0.f, 0.f, 0.f};
  float past[4] = {0.f, 0.f, 0.f, 0.f};
  auto nz = make_noise<INJECT>(noise, N, active ? i : 0, rng, step_seq, TAG_ENV_STEP, qx_model0(ps).noise_loc, qx_model0(ps).ratio);
  nz.prefetch4();
  if (!INJECT && noise_dump && active) nz.set_dump(noise_dump + i, N);
  if (RANDACT) {
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
    if (active) reinterpret_cast<float4*>(actions)[i] = make_float4(act[0], act[1], act[2], act[3]);
  } else if (active) {
    float4 a4 = __ldg(reinterpret_cast<const float4*>(actions) + i);
    act[0] = a4.x; act[1] = a4.y; act[2] = a4.z; act[3] = a4.w;
  }
  // the episode number of this env's spare, for EVERY lane, in the shadow of the tile load: a lane that turns out to be
  // resetting can then pull its record towards L1 at once (nobody writes episode[i] of a resetting env during this launch)
  uint32_t e_next = (AUTORESET && spare && active) ? episode[i] : 0u;
  QuadXRegs s;
  int step_count;
  mbar_wait(&mbar, 0, nz.dep(0), nz.dep(1), nz.dep(2), nz.dep(3), nz.dep(4), nz.dep(5), nz.dep(6), nz.dep(7));  // the tile has landed
  quadx_load_tile<MODE, kTileGroupStride>(stile + lane * 4, s, step_count);  // LDS.128, conflict-free (lane-contiguous vectors)
  // an env that finished on the previous call: this call is its reset (NEXT_STEP)
  const bool resetting = AUTORESET && active && (s.flags & (FLAG_TERM | FLAG_TRUNC)) != 0;
  const float* staged = nullptr;  // this lane's spare record + start pose in shared memory (see kStageFloats)
  if (AUTORESET && spare) {
    constexpr int kSlots = kInGroups * kTileGroupStride / kStageFloats;
    const unsigned reset_m = __ballot_sync(0xffffffffu, resetting);
    if (reset_m != 0u) {
      __syncwarp();  // every lane has unpacked its part of the tile: the buffer is free
      if (resetting) {
        const float* r = spare_rec(spare, e_next, N, i);
        const int rank = __popc(reset_m & ((1u << lane) - 1u));
        if (rank < kSlots) {
          float* q = stile + rank * kStageFloats;
#pragma unroll
          for (int g = 0; g < SP_ROWS / 4; ++g) cp_async16(q + 4 * g, r + 4 * g);
#pragma unroll
          for (int k = 0; k < 3; ++k) { cp_async4(q + SP_ROWS + k, start_pos + 3 * i + k); cp_async4(q + SP_ROWS + 3 + k, start_orn + 3 * i + k); }
          staged = q;
        } else {  // more resetting lanes than slots (a synchronised truncation): towards L1 at least
          prefetch_l1(r); prefetch_l1(r + 32); prefetch_l1(r + 64); prefetch_l1(r + SP_ROWS - 1);
        }
      }
    }
  }
  int n_aviary = (active && !resetting) ? h.env_step_ratio : 0;
  float rew = -0.1f;
#pragma unroll
  for (int k = 0; k < 4; ++k) s.sp[k] = act[k];
  if (MA) {  // MAQuadXHover: flags are re-evaluated every step, rewards add up from 0, the obs shows the PREVIOUS action
    s.flags &= ~(uint32_t)(FLAG_TERM | FLAG_TRUNC | FLAG_OOB | FLAG_COLLISION);
    rew = 0.0f;
    const F4 cur = ld_f4(rec + (QM_CUR / 4) * kTileGroupStride);
    past[0] = cur.x; past[1] = cur.y; past[2] = cur.z; past[3] = cur.w;
    if (active) {
      st_f4(rec + (QM_PAST / 4) * kTileGroupStride, past[0], past[1], past[2], past[3]);
      st_f4(rec + (QM_CUR / 4) * kTileGroupStride, act[0], act[1], act[2], act[3]);
    }
  }
  float sx = 0.f, sy = 0.f, sz = 0.f;
  if (MA && active) { sx = start_pos[3 * i]; sy = start_pos[3 * i + 1]; sz = start_pos[3 * i + 2]; }
#pragma unroll 1
  for (int k = 0; k < n_aviary; ++k) {
    if (!MA && (s.flags & (FLAG_TERM | FLAG_TRUNC))) break;  // quadx_base_env.py:289-290
    quadx_aviary_step<MODE>(p, s, nz);
    if (MA) ma_hover_term_trunc_reward(h, s, step_count, sx, sy, sz, rew);
    else hover_term_trunc_reward(h, s, step_count, rew);
  }
  step_count += 1;
  if (AUTORESET && __any_sync(0xffffffffu, resetting)) {
    if (resetting) {
      // env.reset(): begin_reset + end_reset (quadx_base_env.py:149-212) — normally a copy of the env's spare
      float px, py, pz, ox, oy, oz;
      if (staged) {
        cp_async_wait_all();
        px = staged[SP_ROWS + 0]; py = staged[SP_ROWS + 1]; pz = staged[SP_ROWS + 2];
        ox = staged[SP_ROWS + 3]; oy = staged[SP_ROWS + 4]; oz = staged[SP_ROWS + 5];
      } else {
        px = start_pos[3 * i + 0]; py = start_pos[3 * i + 1]; pz = start_pos[3 * i + 2];
        ox = start_orn[3 * i + 0]; oy = start_orn[3 * i + 1]; oz = start_orn[3 * i + 2];
      }
      bool hit = false;
      uint32_t nseq = step_seq | 0x40000000u;
      if (spare) {
        nseq = e_next;  // episode number: keys the warm-up noise
        const float* srec = staged ? staged : spare_rec(spare, e_next, N, i);
        const F4 m0 = ld_f4(srec + SP_POSE), m1 = ld_f4(srec + SP_POSE + 4), m2 = ld_f4(srec + SP_POSE + 8);
        hit = spare_copy && m1.z != 0.0f && bits_from_f(m2.x) == e_next && m0.x == px && m0.y == py && m0.z == pz && m0.w == ox && m1.x == oy &&
              m1.y == oz;
        if (hit) {
          int dummy;
          quadx_load_tile<MODE, 4>(srec, s, dummy);
          const F4 pw = ld_f4(srec + QX_PWM);
          s.pwm[0] = pw.x; s.pwm[1] = pw.y; s.pwm[2] = pw.z; s.pwm[3] = pw.w;
          s.flags = bits_from_f(m1.w);
        }
      }
      if (!hit) HOVER_RESET_COLD(s, px, py, pz, ox, oy, oz, nseq);
#pragma unroll
      for (int k = 0; k < 4; ++k) { s.sp[k] = 0.0f; act[k] = 0.0f; }  // self.action = zeros (quadx_base_env.py:165)
      step_count = 0;
      rew = 0.0f;
    }
  }
  float* row = smem + lane * O;  // dense [32][O] tile, written out below by one bulk copy
  if (MA) ma_hover_observation(h, s, past, sx, sy, sz, row);
  else hover_observation(h, s, act, row);
  fence_async_smem();  // generic-proxy writes of this lane -> visible to the bulk-copy (async) proxy
  __syncwarp();
  // ---- this warp's observation tile obs[tile_first .. +rows][O] is contiguous in global memory and 16-byte aligned: ONE
  //      cp.async.bulk (TMA) moves it, issued before the state stores so that the engine's reads of shared memory overlap them
  int64_t nrows = N - tile_first;
  if (nrows > kBlock) nrows = kBlock;
  const uint32_t bytes = (uint32_t)nrows * (uint32_t)O * 4u;
  float* dst = obs + tile_first * O;
  const bool bulk = (bytes & 15u) == 0u;
  if (bulk) {
    if (lane == 0) bulk_store_s2g(dst, smem, bytes);
  } else {  // ragged last tile whose byte count is not a multiple of 16
    for (int j = lane; j < (int)nrows * O; j += kBlock) dst[j] = smem[j];
  }
  if (active) {
    quadx_store_tile<MODE, kTileGroupStride>(rec, s, step_count);
    hover_step_outputs(reward, term, trunc, info, i, rew, s.flags);
  }
  // queue finished episodes: their spares are consumed by the next launch and rebuilt after it
  if (AUTORESET) {
    const bool done = active && (s.flags & (FLAG_TERM | FLAG_TRUNC)) != 0;
    const unsigned m = __ballot_sync(0xffffffffu, done);
    if (done) {
      const int leader = __ffs(m) - 1;
      int base = 0;
      if (lane == leader) base = atomicAdd(cur_count, __popc(m));
      base = __shfl_sync(m, base, leader);
      cur_list[base + __popc(m & ((1u << lane) - 1u))] = (int32_t)i;
    }
  }
  if (bulk && lane == 0) bulk_store_wait_read();  // the CTA's shared memory must outlive the engine's reads
}

// ---------------------------------------------------------------------------------------------------
// Fused rollout (SURVEY 8b: "n_env_steps > 1 = persistent rollout with on-device random actions"): T env steps of every env in
// ONE launch.  A warp loads its tile once, keeps the state in registers for the T steps and stores it once; each step still
// draws its action and noise from the same Philox counters as a single-step launch, integrates, and writes the step's
// observation tile (TMA), reward, flags and the action it drew, so after the launch every output buffer holds the results of
// the LAST of T env steps, like T calls of pfb_env_step.  The state is rounded to the record format at the end of every step —
// what the store / load of two launches does — so a fused launch performs the same arithmetic as T single-step launches; the
// results agree bit for bit except where two compiled copies of the same expression round differently (nvcc contracts
// multiply-adds per inlined copy: ~4e-5 of the env-steps see a one-ulp fp32 difference in a PID term; DESIGN.md 4,
// tests/test_gpu_parity.py::test_fused_rollout_equals_stepwise), and the fused path is pinned to the fp64 oracle on its own
// (tests/test_timed_path_parity.py::test_hover_fused_rollout_matches_oracle).
// Resets: an env that finished on step t takes, on step t + 1, the spare of its next episode out of kSpareBufs records kept
// kRolloutAhead ahead (k_hover_spare_ahead before the first fused launch, k_hover_spare_topup behind every one: all reset work
// stays inside the timed region); a missing spare (more than kRolloutAhead resets of one env inside a launch) is integrated
// inline by the cold path — the same episode number keys the same noise.
// ---------------------------------------------------------------------------------------------------
constexpr int kRolloutAhead = 3;
constexpr int kRolloutMaxSteps = 16;

// one env, one spare: episode `e` of env i, complete warm-up, into its buffer.  k_hover_spare_build keeps its own copy of this
// body: calling it there changes that kernel's SASS (the __restrict__ parameters add alias scopes around its episode[] store)
template <int MODE>
__device__ __forceinline__ void hover_build_full(const QuadXParams& p, const HoverParams& h, const RngParams& rng, const float* __restrict__ start_pos,
                                                 const float* __restrict__ start_orn, float* __restrict__ spare, int64_t N, int64_t i, uint32_t e) {
  float* rec = spare_rec(spare, e, N, i);
  const float px = start_pos[3 * i + 0], py = start_pos[3 * i + 1], pz = start_pos[3 * i + 2];
  const float ox = start_orn[3 * i + 0], oy = start_orn[3 * i + 1], oz = start_orn[3 * i + 2];
  QuadXRegs s = hover_fresh<MODE>(px, py, pz, ox, oy, oz);
  hover_warmup_inline<MODE, false>(p, s, 0, h.warmup_steps, rng, nullptr, N, i, e);
  quadx_store_tile<7, 4>(rec, s, 0);
  spare_trailer(rec, px, py, pz, ox, oy, oz, 1.0f, s.flags, e);
}
// before the first fused launch (or after single-step launches): every env gets the spares episode[i] + 1 .. + kRolloutAhead - 1
// it does not have yet (episode[i] itself is valid by the step pipeline's invariant)
template <int MODE, class PS>
__global__ void __launch_bounds__(kBlock, kHoverBlocks)
    k_hover_spare_ahead(const __grid_constant__ PS ps, const __grid_constant__ HoverParams h, const __grid_constant__ RngParams rng,
                        const float* __restrict__ start_pos, const float* __restrict__ start_orn, float* __restrict__ spare,
                        const uint32_t* __restrict__ episode, int64_t N) {
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  if (i >= N) return;
  const QuadXParams& p = qx_model(ps, i);
  const uint32_t e0 = episode[i];
#pragma unroll 1
  for (int a = 1; a < kRolloutAhead; ++a) {
    const uint32_t e = e0 + (uint32_t)a;
    const float* rec = spare_rec(spare, e, N, i);
    const F4 m0 = ld_f4(rec + SP_POSE), m1 = ld_f4(rec + SP_POSE + 4), m2 = ld_f4(rec + SP_POSE + 8);
    const bool have = m1.z != 0.0f && bits_from_f(m2.x) == e && m0.x == start_pos[3 * i] && m0.y == start_pos[3 * i + 1] && m0.z == start_pos[3 * i + 2] &&
                      m0.w == start_orn[3 * i] && m1.x == start_orn[3 * i + 1] && m1.y == start_orn[3 * i + 2];
    if (!have) hover_build_full<MODE>(p, h, rng, start_pos, start_orn, spare, N, i, e);
  }
}
// behind a fused launch: the spares it consumed, listed as (env, episode to build)
template <int MODE, class PS>
__global__ void __launch_bounds__(kBlock, kHoverBlocks)
    k_hover_spare_topup(const __grid_constant__ PS ps, const __grid_constant__ HoverParams h, const __grid_constant__ RngParams rng,
                        const float* __restrict__ start_pos, const float* __restrict__ start_orn, float* __restrict__ spare,
                        const int32_t* __restrict__ count, const int2* __restrict__ list, int64_t N) {
  const int n = *count;
  for (int t = (int)(blockIdx.x * kBlock + threadIdx.x); t < n; t += (int)(gridDim.x * kBlock)) {
    const int2 en = list[t];
    hover_build_full<MODE>(qx_model(ps, (int64_t)en.x), h, rng, start_pos, start_orn, spare, N, (int64_t)en.x, (uint32_t)en.y);
  }
}
// switching from single-step launches to the fused rollout: the spares whose first half was integrated by the last step launch
// are finished here (phase 1 of hover_build on the list the next step launch would have used), so that episode[] is current
template <int MODE, class PS>
__global__ void __launch_bounds__(kBlock, kHoverBlocks)
    k_hover_drain(const __grid_constant__ PS ps, const __grid_constant__ HoverParams h, const __grid_constant__ RngParams rng,
                  const int32_t* __restrict__ b1_count, const int32_t* __restrict__ b1_list, const uint32_t* __restrict__ b1_elist,
                  const float* __restrict__ start_pos, const float* __restrict__ start_orn, float* __restrict__ spare, uint32_t* __restrict__ episode,
                  int builders, int64_t N) {
  hover_build<MODE>(ps, h, rng, (int)blockIdx.x + builders, builders, b1_count, b1_list, b1_count, b1_list, nullptr, b1_elist, start_pos, start_orn, spare,
                    episode, N);
}

// 14 CTAs per SM: the 2048 tiles of a 65 536-env launch (no builder CTAs here) are still one wave, with 144 registers instead of 128
template <int MODE, class PS>
__global__ void __launch_bounds__(kBlock, 14)
    k_hover_rollout(const __grid_constant__ PS ps, const __grid_constant__ HoverParams h, const __grid_constant__ RngParams rng,
                    float* __restrict__ st, int rows, float* __restrict__ actions, float* __restrict__ obs, float* __restrict__ reward,
                    uint8_t* __restrict__ term, uint8_t* __restrict__ trunc, uint8_t* __restrict__ info, const float* __restrict__ start_pos,
                    const float* __restrict__ start_orn, const float* __restrict__ spare, uint32_t* __restrict__ episode,
                    int32_t* __restrict__ consumed_count, int2* __restrict__ consumed_list, int32_t* __restrict__ last_count,
                    int32_t* __restrict__ last_list, uint32_t step_seq0, int T, int64_t N) {
  const int tile = (int)blockIdx.x;
  __shared__ __align__(128) float smem2[2][kBlock * kObsMax];  // the observation tile of step t leaves by TMA while step t + 1 fills the other one
  constexpr int kInGroups = qx_groups_moved<MODE>();
  __shared__ __align__(128) float stile[kInGroups * kTileGroupStride];
  __shared__ __align__(8) uint64_t mbar;
  const int O = h.angle_representation == 0 ? 20 : 21;
  const int lane = threadIdx.x;
  const int64_t tile_first = (int64_t)tile * kBlock;
  const int64_t i = tile_first + lane;
  const bool active = i < N;
  const QuadXParams& p = qx_model(ps, i);  // the model index is padded to whole tiles: every lane may read it
  float* rec = st + qx_tile_base(i, rows);
  if (lane == 0) {
    mbar_init(&mbar, 1);
    bulk_load_g2s(stile, st + qx_tile_base(tile_first, rows), (uint32_t)(kInGroups * kTileGroupStride * sizeof(float)), &mbar);
  }
  __syncwarp();
  uint32_t e_local = active ? episode[i] : 0u;  // the next spare this env consumes
  float sx = 0.f, sy = 0.f, sz = 0.f, ox = 0.f, oy = 0.f, oz = 0.f;
  if (active) {
    sx = start_pos[3 * i + 0]; sy = start_pos[3 * i + 1]; sz = start_pos[3 * i + 2];
    ox = start_orn[3 * i + 0]; oy = start_orn[3 * i + 1]; oz = start_orn[3 * i + 2];
  }
  QuadXRegs s;
  int step_count;
  mbar_wait(&mbar, 0);
  quadx_load_tile<MODE, kTileGroupStride>(stile + lane * 4, s, step_count);
  __syncwarp();  // the tile buffer is dead from here on: it stages the spare records of resetting lanes (kStageFloats)
  int64_t nrows = N - tile_first;
  if (nrows > kBlock) nrows = kBlock;
  const uint32_t obs_bytes = (uint32_t)nrows * (uint32_t)O * 4u;
  const bool bulk = (obs_bytes & 15u) == 0u;
  float* obs_dst = obs + tile_first * O;
  const uint64_t g = ((uint64_t)rng.env_offset_hi << 32 | rng.env_offset_lo) + (uint64_t)i;
#pragma unroll 1
  for (int t = 0; t < T; ++t) {
    const uint32_t step_seq = step_seq0 + (uint32_t)t;
    // ---- the step's draws: motor noise and the action, same counters as a single-step launch
    auto nz = make_noise<false>(nullptr, N, active ? i : 0, rng, step_seq, TAG_ENV_STEP, qx_model0(ps).noise_loc, qx_model0(ps).ratio);
    nz.prefetch4();
    float act[4];
    {
      U4 r = philox4x32_10(U4{(uint32_t)g, (uint32_t)(g >> 32), step_seq, (uint32_t)TAG_ACTION << 24}, rng.k0, rng.k1);
      const float pi = 3.14159265358979323846f;
      if (MODE == -1) {
        act[0] = 0.8f * u32_to_unit_open(r.x); act[1] = 0.8f * u32_to_unit_open(r.y);
        act[2] = 0.8f * u32_to_unit_open(r.z); act[3] = 0.8f * u32_to_unit_open(r.w);
      } else {
        act[0] = pi * (2.0f * u32_to_unit_open(r.x) - 1.0f); act[1] = pi * (2.0f * u32_to_unit_open(r.y) - 1.0f);
        act[2] = pi * (2.0f * u32_to_unit_open(r.z) - 1.0f); act[3] = 0.8f * u32_to_unit_open(r.w);
      }
      if (active) reinterpret_cast<float4*>(actions)[i] = make_float4(act[0], act[1], act[2], act[3]);
    }
    const bool resetting = active && (s.flags & (FLAG_TERM | FLAG_TRUNC)) != 0;
    // the lanes that reset on this step are known now: their spare record starts its way to L1 and the slot on the top-up list
    // is taken (one atomic per warp) while the other lanes integrate
    const unsigned reset_m = __ballot_sync(0xffffffffu, resetting);
    int reset_base = 0;
    const float* staged = nullptr;  // this lane's spare record in shared memory (the dead state-tile buffer, see kStageFloats)
    if (reset_m != 0u) {
      constexpr int kSlots = kInGroups * kTileGroupStride / SP_ROWS;
      if (resetting) {
        const float* r = spare_rec(spare, e_local, N, i);
        const int rank = __popc(reset_m & ((1u << lane) - 1u));
        if (rank < kSlots) {
          float* q = stile + rank * SP_ROWS;
#pragma unroll
          for (int g = 0; g < SP_ROWS / 4; ++g) cp_async16(q + 4 * g, r + 4 * g);
          staged = q;
        } else {
          prefetch_l1(r); prefetch_l1(r + 32); prefetch_l1(r + 64); prefetch_l1(r + SP_ROWS - 1);
        }
      }
      // one slot range on the top-up list per warp.  Inline PTX: a plain atomicAdd is rewritten by the compiler into its
      // warp-aggregated form, whose broadcast shuffle waits for the atomic's return HERE instead of after the integration
      if (lane == __ffs(reset_m) - 1)
        asm volatile("atom.global.add.u32 %0, [%1], %2;" : "=r"(reset_base) : "l"(consumed_count), "r"(__popc(reset_m)) : "memory");
    }
    const int n_aviary = (active && !resetting) ? h.env_step_ratio : 0;
    float rew = -0.1f;
#pragma unroll
    for (int k = 0; k < 4; ++k) s.sp[k] = act[k];
#pragma unroll 1
    for (int k = 0; k < n_aviary; ++k) {
      if (s.flags & (FLAG_TERM | FLAG_TRUNC)) break;  // quadx_base_env.py:289-290
      quadx_aviary_step<MODE>(p, s, nz);
      hover_term_trunc_reward(h, s, step_count, rew);
    }
    step_count += 1;
    if (reset_m != 0u) {
      if (resetting) {
        if (staged) cp_async_wait_all();
        const float* srec = staged ? staged : spare_rec(spare, e_local, N, i);
        const F4 m0 = ld_f4(srec + SP_POSE), m1 = ld_f4(srec + SP_POSE + 4), m2 = ld_f4(srec + SP_POSE + 8);
        const bool hit = m1.z != 0.0f && bits_from_f(m2.x) == e_local && m0.x == sx && m0.y == sy && m0.z == sz && m0.w == ox && m1.x == oy && m1.y == oz;
        if (hit) {
          int dummy;
          quadx_load_tile<MODE, 4>(srec, s, dummy);
          const F4 pw = ld_f4(srec + QX_PWM);
          s.pwm[0] = pw.x; s.pwm[1] = pw.y; s.pwm[2] = pw.z; s.pwm[3] = pw.w;
          s.flags = bits_from_f(m1.w);
        } else {
          HOVER_RESET_COLD(s, sx, sy, sz, ox, oy, oz, e_local);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) { s.sp[k] = 0.0f; act[k] = 0.0f; }  // self.action = zeros (quadx_base_env.py:165)
        step_count = 0;
        rew = 0.0f;
      }
      // the consumed spares go on the top-up list: (env, episode that takes the freed place kRolloutAhead ahead)
      const int base = __shfl_sync(0xffffffffu, reset_base, __ffs(reset_m) - 1);
      if (resetting) {
        consumed_list[base + __popc(reset_m & ((1u << lane) - 1u))] = make_int2((int)i, (int)(e_local + (uint32_t)kRolloutAhead));
        e_local += 1u;
      }
    }
    // ---- outputs of the step
    float* smem = smem2[t & 1];
    if (bulk && lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");  // the copy that read THIS buffer two steps ago
    __syncwarp();
    hover_observation(h, s, act, smem + lane * O);
    fence_async_smem();
    __syncwarp();
    if (bulk) {
      if (lane == 0) bulk_store_s2g(obs_dst, smem, obs_bytes);
    } else {
      for (int j = lane; j < (int)nrows * O; j += kBlock) obs_dst[j] = smem[j];
    }
    if (active) {
      hover_step_outputs(reward, term, trunc, info, i, rew, s.flags);
    }
    quadx_requantize(s);  // what storing the state and loading it again in the next launch does to the fp64-carried fields
  }
  if (active) {
    quadx_store_tile<MODE, kTileGroupStride>(rec, s, step_count);
    episode[i] = e_local;
  }
  // hand-over to the single-step pipeline: the envs that finished on the LAST step are the done list its next launch expects
  const bool done = active && (s.flags & (FLAG_TERM | FLAG_TRUNC)) != 0;
  const unsigned m = __ballot_sync(0xffffffffu, done);
  if (m != 0u) {
    int base = 0;
    if (lane == __ffs(m) - 1) base = atomicAdd(last_count, __popc(m));
    base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
    if (done) last_list[base + __popc(m & ((1u << lane) - 1u))] = (int32_t)i;
  }
  if (bulk && lane == 0) bulk_store_wait_read();  // the CTA's shared memory must outlive the engine's reads
}

// SAME_STEP autoreset (PFB_AUTORESET_SAME_STEP): T env steps of every env in one launch — T = 1 for pfb_env_step (the caller's
// actions, or RANDACT), up to kRolloutMaxSteps for pfb_env_rollout — on the look-ahead spares of the fused rollout.  Every lane
// integrates every step; a lane whose env finishes writes the step's reward / flags / info from the terminal state and its
// terminal observation row to final_obs, then swaps in the spare of episode e_local (or integrates it cold under the same
// number) and observes the reset state into obs.  At launch, the spares e_local .. e_local + kRolloutAhead - 1 are valid (the
// look-ahead invariant); a fourth reset of one env in a launch finds a stale record and takes the cold path.  After the steps,
// the spares each env needs to be kRolloutAhead ahead again go on the top-up list, which k_hover_spare_topup builds on the
// same stream before the next launch.  The list counter alternates between launches: this launch zeroes the one the next
// appends to (the previous top-up, which read it, has finished).
template <int MODE, bool RANDACT, class PS>
__global__ void __launch_bounds__(kBlock, 14)
    k_hover_same(const __grid_constant__ PS ps, const __grid_constant__ HoverParams h, const __grid_constant__ RngParams rng,
                 float* __restrict__ st, int rows, float* __restrict__ actions, float* __restrict__ obs, float* __restrict__ final_obs,
                 float* __restrict__ reward, uint8_t* __restrict__ term, uint8_t* __restrict__ trunc, uint8_t* __restrict__ info,
                 const float* __restrict__ start_pos, const float* __restrict__ start_orn, const float* __restrict__ spare,
                 uint32_t* __restrict__ episode, int32_t* __restrict__ consumed_count, int2* __restrict__ consumed_list,
                 int32_t* __restrict__ next_consumed_count, int spare_copy, uint32_t step_seq0, int T, int64_t N) {
  const int tile = (int)blockIdx.x;
  __shared__ __align__(128) float smem2[2][kBlock * kObsMax];  // the observation tile of step t leaves by TMA while step t + 1 fills the other one
  constexpr int kInGroups = qx_groups_moved<MODE>();
  __shared__ __align__(128) float stile[kInGroups * kTileGroupStride];
  __shared__ __align__(8) uint64_t mbar;
  const int O = h.angle_representation == 0 ? 20 : 21;
  const int lane = threadIdx.x;
  const int64_t tile_first = (int64_t)tile * kBlock;
  const int64_t i = tile_first + lane;
  const bool active = i < N;
  const QuadXParams& p = qx_model(ps, i);  // the model index is padded to whole tiles: every lane may read it
  float* rec = st + qx_tile_base(i, rows);
  if (tile == 0 && lane == 0) *next_consumed_count = 0;
  if (lane == 0) {
    mbar_init(&mbar, 1);
    bulk_load_g2s(stile, st + qx_tile_base(tile_first, rows), (uint32_t)(kInGroups * kTileGroupStride * sizeof(float)), &mbar);
  }
  __syncwarp();
  const uint32_t e0 = active ? episode[i] : 0u;  // the next spare this env consumes
  uint32_t e_local = e0;
  float sx = 0.f, sy = 0.f, sz = 0.f, ox = 0.f, oy = 0.f, oz = 0.f;
  if (active) {
    sx = start_pos[3 * i + 0]; sy = start_pos[3 * i + 1]; sz = start_pos[3 * i + 2];
    ox = start_orn[3 * i + 0]; oy = start_orn[3 * i + 1]; oz = start_orn[3 * i + 2];
  }
  QuadXRegs s;
  int step_count;
  mbar_wait(&mbar, 0);
  quadx_load_tile<MODE, kTileGroupStride>(stile + lane * 4, s, step_count);
  int64_t nrows = N - tile_first;
  if (nrows > kBlock) nrows = kBlock;
  const uint32_t obs_bytes = (uint32_t)nrows * (uint32_t)O * 4u;
  const bool bulk = (obs_bytes & 15u) == 0u;
  float* obs_dst = obs + tile_first * O;
  const uint64_t g = ((uint64_t)rng.env_offset_hi << 32 | rng.env_offset_lo) + (uint64_t)i;
#pragma unroll 1
  for (int t = 0; t < T; ++t) {
    const uint32_t step_seq = step_seq0 + (uint32_t)t;
    // ---- the step's draws: motor noise and the action, same counters as every other step launch
    auto nz = make_noise<false>(nullptr, N, active ? i : 0, rng, step_seq, TAG_ENV_STEP, qx_model0(ps).noise_loc, qx_model0(ps).ratio);
    nz.prefetch4();
    float act[4] = {0.f, 0.f, 0.f, 0.f};
    if (RANDACT) {
      U4 r = philox4x32_10(U4{(uint32_t)g, (uint32_t)(g >> 32), step_seq, (uint32_t)TAG_ACTION << 24}, rng.k0, rng.k1);
      const float pi = 3.14159265358979323846f;
      if (MODE == -1) {
        act[0] = 0.8f * u32_to_unit_open(r.x); act[1] = 0.8f * u32_to_unit_open(r.y);
        act[2] = 0.8f * u32_to_unit_open(r.z); act[3] = 0.8f * u32_to_unit_open(r.w);
      } else {
        act[0] = pi * (2.0f * u32_to_unit_open(r.x) - 1.0f); act[1] = pi * (2.0f * u32_to_unit_open(r.y) - 1.0f);
        act[2] = pi * (2.0f * u32_to_unit_open(r.z) - 1.0f); act[3] = 0.8f * u32_to_unit_open(r.w);
      }
      if (active) reinterpret_cast<float4*>(actions)[i] = make_float4(act[0], act[1], act[2], act[3]);
    } else if (active) {
      const float4 a4 = __ldg(reinterpret_cast<const float4*>(actions) + i);
      act[0] = a4.x; act[1] = a4.y; act[2] = a4.z; act[3] = a4.w;
    }
    const int n_aviary = active ? h.env_step_ratio : 0;
    float rew = -0.1f;
#pragma unroll
    for (int k = 0; k < 4; ++k) s.sp[k] = act[k];
#pragma unroll 1
    for (int k = 0; k < n_aviary; ++k) {
      if (s.flags & (FLAG_TERM | FLAG_TRUNC)) break;  // quadx_base_env.py:289-290
      quadx_aviary_step<MODE>(p, s, nz);
      hover_term_trunc_reward(h, s, step_count, rew);
    }
    step_count += 1;
    if (active) hover_step_outputs(reward, term, trunc, info, i, rew, s.flags);
    const bool done = active && (s.flags & (FLAG_TERM | FLAG_TRUNC)) != 0;
    // ---- outputs of the step
    float* smem = smem2[t & 1];
    if (bulk && lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");  // the copy that read THIS buffer two steps ago
    __syncwarp();
    float* row = smem + lane * O;
    hover_observation(h, s, act, row);
    if (done) {
      for (int k = 0; k < O; ++k) final_obs[i * O + k] = row[k];
      // env.reset(): begin_reset + end_reset (quadx_base_env.py:149-212), from the spare of episode e_local
      const float* srec = spare_rec(spare, e_local, N, i);
      const F4 m0 = ld_f4(srec + SP_POSE), m1 = ld_f4(srec + SP_POSE + 4), m2 = ld_f4(srec + SP_POSE + 8);
      const bool hit = spare_copy && m1.z != 0.0f && bits_from_f(m2.x) == e_local && m0.x == sx && m0.y == sy && m0.z == sz && m0.w == ox &&
                       m1.x == oy && m1.y == oz;
      if (hit) {
        int dummy;
        quadx_load_tile<MODE, 4>(srec, s, dummy);
        const F4 pw = ld_f4(srec + QX_PWM);
        s.pwm[0] = pw.x; s.pwm[1] = pw.y; s.pwm[2] = pw.z; s.pwm[3] = pw.w;
        s.flags = bits_from_f(m1.w);
      } else {
        HOVER_RESET_COLD(s, sx, sy, sz, ox, oy, oz, e_local);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) { s.sp[k] = 0.0f; act[k] = 0.0f; }  // self.action = zeros (quadx_base_env.py:165)
      step_count = 0;
      e_local += 1u;
      hover_observation(h, s, act, row);
    }
    fence_async_smem();
    __syncwarp();
    if (bulk) {
      if (lane == 0) bulk_store_s2g(obs_dst, smem, obs_bytes);
    } else {
      for (int j = lane; j < (int)nrows * O; j += kBlock) obs_dst[j] = smem[j];
    }
    quadx_requantize(s);  // what storing the state and loading it again in the next launch does to the fp64-carried fields
  }
  if (active) {
    quadx_store_tile<MODE, kTileGroupStride>(rec, s, step_count);
    episode[i] = e_local;
  }
  // the top-up list: the spares e_local .. e_local + kRolloutAhead - 1 that are not valid any more (the ones from
  // e0 + kRolloutAhead on), at most kRolloutAhead per env, in distinct buffers.  One atomic per warp.
  if (spare_copy) {
    const uint32_t first = e_local > e0 + (uint32_t)kRolloutAhead ? e_local : e0 + (uint32_t)kRolloutAhead;
    const int need = active ? (int)(e_local + (uint32_t)kRolloutAhead - first) : 0;
    int incl = need;
#pragma unroll
    for (int off = 1; off < kBlock; off <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += v;
    }
    const int total = __shfl_sync(0xffffffffu, incl, kBlock - 1);
    if (total) {
      int base = 0;
      if (lane == kBlock - 1) base = atomicAdd(consumed_count, total);
      base = __shfl_sync(0xffffffffu, base, kBlock - 1) + incl - need;
      for (int j = 0; j < need; ++j) consumed_list[base + j] = make_int2((int)i, (int)(first + (uint32_t)j));
    }
  }
  if (bulk && lane == 0) bulk_store_wait_read();  // the CTA's shared memory must outlive the engine's reads
}

// After a user reset of every env: each env gets a complete fresh spare (dense warps, all envs).
template <int MODE, class PS>
__global__ void __launch_bounds__(kBlock, kHoverBlocks)
    k_hover_spare_build(const __grid_constant__ PS ps, const __grid_constant__ HoverParams h, const __grid_constant__ RngParams rng,
                        const float* __restrict__ start_pos, const float* __restrict__ start_orn, float* __restrict__ spare,
                        uint32_t* __restrict__ episode, int64_t N) {
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  if (i >= N) return;
  const QuadXParams& p = qx_model(ps, i);
  const uint32_t e = episode[i] + 1u;
  float* rec = spare_rec(spare, e, N, i);
  const float px = start_pos[3 * i + 0], py = start_pos[3 * i + 1], pz = start_pos[3 * i + 2];
  const float ox = start_orn[3 * i + 0], oy = start_orn[3 * i + 1], oz = start_orn[3 * i + 2];
  QuadXRegs s = hover_fresh<MODE>(px, py, pz, ox, oy, oz);
  hover_warmup_inline<MODE, false>(p, s, 0, h.warmup_steps, rng, nullptr, N, i, e);
  quadx_store_tile<7, 4>(rec, s, 0);
  spare_trailer(rec, px, py, pz, ox, oy, oz, 1.0f, s.flags, e);
  episode[i] = e;
}

// env.reset() for all / masked envs
template <int MODE, bool INJECT, class PS>
__global__ void __launch_bounds__(kBlock)
    k_hover_reset(const __grid_constant__ PS ps, const __grid_constant__ HoverParams h,
                  const __grid_constant__ RngParams rng, float* __restrict__ st, int rows,
                  const float* __restrict__ start_pos, const float* __restrict__ start_orn,
                  const uint8_t* __restrict__ mask, const float* __restrict__ noise, float* __restrict__ obs,
                  uint32_t seq, int64_t N) {
  const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  if (i >= N) return;
  if (mask && !mask[i]) return;
  const QuadXParams& p = qx_model(ps, i);
  const int O = (h.angle_representation == 0 ? 20 : 21) + (h.ma ? 3 : 0);
  float row[kObsMax];
  QuadXRegs s = hover_fresh<MODE>(start_pos[3 * i + 0], start_pos[3 * i + 1], start_pos[3 * i + 2], start_orn[3 * i + 0], start_orn[3 * i + 1],
                                  start_orn[3 * i + 2]);
  hover_warmup_inline<MODE, INJECT>(p, s, 0, h.warmup_steps, rng, noise, N, i, seq);
  float* rec = st + qx_tile_base(i, rows);
  const float zero[4] = {0.f, 0.f, 0.f, 0.f};  // self.action = zeros (quadx_base_env.py:165)
  if (h.ma) {  // past_actions is NOT cleared by a reset in the reference: it still holds the previous episode's value
    const F4 pa = ld_f4(rec + (QM_PAST / 4) * kTileGroupStride);
    const float past[4] = {pa.x, pa.y, pa.z, pa.w};
    ma_hover_observation(h, s, past, start_pos[3 * i], start_pos[3 * i + 1], start_pos[3 * i + 2], row);
  } else {
    hover_observation(h, s, zero, row);
  }
  quadx_store_tile<7, kTileGroupStride>(rec, s, 0);
  if (obs) {
#pragma unroll
    for (int k = 0; k < kObsMax; ++k)
      if (k < O) obs[i * O + k] = row[k];
  }
}

// ---------------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------------
// QuadX state layout: warp-tiled (pfb_quadx.cuh) on every QuadX handle except QuadX-Waypoints (field-major rows + istate)
static inline bool qx_tiled(const PfbContext* h) { return h->model.kind == PFB_KIND_QUADX && h->env.env_kind != PFB_ENV_QUADX_WAYPOINTS; }
static inline int qx_rows(const PfbContext* h) { return h->env.env_kind == PFB_ENV_MA_QUADX_HOVER ? (int)QM_ROWS : (int)QX_ROWS; }

int qx_reset(PfbContext* h, const uint8_t* mask, cudaStream_t s) {
  if (qx_tiled(h)) k_quadx_reset<true><<<grid_for(h->n), kBlock, 0, s>>>(h->buf.state, h->buf.istate, qx_rows(h), h->buf.setpoint, h->buf.start_pos, h->buf.start_orn, mask, h->n);
  else k_quadx_reset<false><<<grid_for(h->n), kBlock, 0, s>>>(h->buf.state, h->buf.istate, qx_rows(h), h->buf.setpoint, h->buf.start_pos, h->buf.start_orn, mask, h->n);
  LAUNCH_CHECK(h);
  if (!mask) h->mode = 0;  // QuadX.reset() calls set_mode(0) (quadx.py:224)
  return 0;
}

int qx_set_mode(PfbContext* h, int mode, cudaStream_t s) {
  if (qx_tiled(h)) { PFB_MODE_SWITCH(mode, (k_quadx_set_mode<MODE, true><<<grid_for(h->n), kBlock, 0, s>>>(h->buf.state, h->buf.istate, qx_rows(h), h->buf.setpoint, h->n))); }
  else { PFB_MODE_SWITCH(mode, (k_quadx_set_mode<MODE, false><<<grid_for(h->n), kBlock, 0, s>>>(h->buf.state, h->buf.istate, qx_rows(h), h->buf.setpoint, h->n))); }
  LAUNCH_CHECK(h);
  h->mode = mode;
  return 0;
}

static int qx_set_modes(PfbContext* h, const int8_t*, cudaStream_t s) {
  k_quadx_set_modes<<<grid_for(h->n), kBlock, 0, s>>>(h->buf.state, qx_rows(h), h->buf.setpoint, h->d_modes, h->n);
  LAUNCH_CHECK(h);
  h->mode = kModePerDrone;
  return 0;
}

template <int MODE, bool TILED, class V>
static void qx_launch_step(PfbContext* h, V v, int n_steps, const float* noise, uint32_t seq, cudaStream_t s) {
  QX_PARAMS_SWITCH(h, (k_quadx_aviary_step<MODE, V::inject, TILED, PS, V::contact, typename V::world><<<grid_for(h->n), kBlock, 0, s>>>(
                          ps, h->rng, world_table(v), v.pose(), v.bits(), h->buf.state, h->buf.istate, qx_rows(h), h->buf.setpoint, h->d_modes,
                          noise, n_steps, seq, h->n)));
}

int qx_aviary_step(PfbContext* h, int n_steps, const float* noise, cudaStream_t s) {
  const int mode = h->mode;
  const uint32_t seq = (uint32_t)h->aviary_seq++;
  return aviary_step_launch(h, noise, [&](auto v) {
    using V = decltype(v);
    // per-drone modes, static bodies and the contact response exist on Aviary handles only, which are warp-tiled
    if (mode == kModePerDrone) {
      qx_launch_step<kModePerDrone, true>(h, v, n_steps, noise, seq, s);
    } else if constexpr (V::contact || V::world::kOn) {
      PFB_MODE_SWITCH(mode, (qx_launch_step<MODE, true>(h, v, n_steps, noise, seq, s)));
    } else if (qx_tiled(h)) {
      PFB_MODE_SWITCH(mode, (qx_launch_step<MODE, true>(h, v, n_steps, noise, seq, s)));
    } else {
      PFB_MODE_SWITCH(mode, (qx_launch_step<MODE, false>(h, v, n_steps, noise, seq, s)));
    }
    return 0;
  });
}

int qx_observe(PfbContext* h, cudaStream_t s) {
  if (qx_tiled(h)) k_quadx_observe<true><<<grid_for(h->n), kBlock, 0, s>>>(h->buf.state, h->buf.istate, qx_rows(h), h->buf.drone_state, h->buf.aux_state, h->buf.contact, h->n);
  else k_quadx_observe<false><<<grid_for(h->n), kBlock, 0, s>>>(h->buf.state, h->buf.istate, qx_rows(h), h->buf.drone_state, h->buf.aux_state, h->buf.contact, h->n);
  LAUNCH_CHECK(h);
  return 0;
}

static int qx_set_base_state(PfbContext* h, const BaseStateIn& a, cudaStream_t s) {
  if (a.lin32 || a.ang32) k_quadx_set_base_state<true><<<grid_for(h->n), kBlock, 0, s>>>(a, h->buf.state, qx_rows(h), h->n);
  else k_quadx_set_base_state<false><<<grid_for(h->n), kBlock, 0, s>>>(a, h->buf.state, qx_rows(h), h->n);
  LAUNCH_CHECK(h);
  return 0;
}

static int qx_get_base_state(PfbContext* h, const BaseStateOut& o, cudaStream_t s) {
  k_quadx_get_base_state<<<grid_for(h->n), kBlock, 0, s>>>(o, h->buf.state, qx_rows(h), h->n);
  LAUNCH_CHECK(h);
  return 0;
}

static int hover_obs_dim(const PfbContext* h) { return (h->hover.angle_representation == 0 ? 20 : 21) + (h->hover.ma ? 3 : 0); }

static int hover_env_reset(PfbContext* h, const uint8_t* mask, const float* noise, cudaStream_t s) {
  const int mode = h->hover.flight_mode;
  // resets draw from their own Philox stream; the high bit keeps them apart from in-step autoresets
  const uint32_t seq = 0x80000000u | (uint32_t)h->reset_seq++;
  if (h->d_spare && !mask) CUDA_OK(cudaMemsetAsync(h->d_counters, 0, 4 * sizeof(int32_t), s));  // a full reset empties the rebuild queues
#define HR_ARGS ps, h->hover, h->rng, h->buf.state, qx_rows(h), h->buf.start_pos, h->buf.start_orn, mask, noise, h->buf.obs, seq, h->n
  if (noise) { QX_PARAMS_SWITCH(h, PFB_MODE_SWITCH(mode, (k_hover_reset<MODE, true, PS><<<grid_for(h->n), kBlock, 0, s>>>(HR_ARGS)))); }
  else { QX_PARAMS_SWITCH(h, PFB_MODE_SWITCH(mode, (k_hover_reset<MODE, false, PS><<<grid_for(h->n), kBlock, 0, s>>>(HR_ARGS)))); }
#undef HR_ARGS
  LAUNCH_CHECK(h);
  if (h->d_spare && !mask) {  // every env gets a fresh spare.  A masked reset keeps the spares: they are keyed by (env, episode
                              // number) and stay valid; a masked env simply is not `done` on the next step
    QX_PARAMS_SWITCH(h, PFB_MODE_SWITCH(mode, (k_hover_spare_build<MODE, PS><<<grid_for(h->n), kBlock, 0, s>>>(ps, h->hover, h->rng, h->buf.start_pos,
                                                                                                              h->buf.start_orn, h->d_spare, h->d_episode, h->n))));
    LAUNCH_CHECK(h);
  }
  h->mode = mode;
  return 0;
}

// k_hover_drain over the builder CTAs of a step launch: finish the spares whose first half the last step launch integrated (list
// (k + 2) % 4 of the next step k, with the episode numbers its phase 0 left in d_elist); the caller checks that k >= 2
static int hover_drain(PfbContext* h, cudaStream_t s) {
  const uint64_t k = h->step_seq;
  const int tiles = grid_for(h->n);
  const int builders = h->sm_count < tiles ? h->sm_count : tiles;
  QX_PARAMS_SWITCH(h, PFB_MODE_SWITCH(h->hover.flight_mode, (k_hover_drain<MODE, PS><<<builders, kBlock, 0, s>>>(
                                                                 ps, h->hover, h->rng, h->d_counters + ((k + 2) % 4), h->d_done_list + ((k + 2) % 4) * h->n,
                                                                 h->d_elist + ((k + 2) % 4) * h->n, h->buf.start_pos, h->buf.start_orn, h->d_spare,
                                                                 h->d_episode, builders, h->n))));
  LAUNCH_CHECK(h);
  return 0;
}

// k_hover_spare_topup behind a SAME_STEP or fused launch, same stream: rebuild the `*count` spares it listed in d_consumed
static int hover_topup(PfbContext* h, int32_t* count, cudaStream_t s) {
  const int tiles = grid_for(h->n);
  const int grid = 8 * h->sm_count < tiles ? 8 * h->sm_count : tiles;
  QX_PARAMS_SWITCH(h, PFB_MODE_SWITCH(h->hover.flight_mode, (k_hover_spare_topup<MODE, PS><<<grid, kBlock, 0, s>>>(
                                                                 ps, h->hover, h->rng, h->buf.start_pos, h->buf.start_orn, h->d_spare, count,
                                                                 h->d_consumed, h->n))));
  LAUNCH_CHECK(h);
  return 0;
}

// SAME_STEP: T env steps in one k_hover_same launch, then the top-up of the spares it consumed, on the same stream.  The first
// launch after a reset or a change of the spares brings every env's spares kRolloutAhead ahead (k_hover_spare_ahead); with
// inline_reset = 1 every reset is integrated cold and the spares are left alone.
static int hover_same_launch(PfbContext* h, float* actions, bool randact, int T, cudaStream_t s) {
  const int mode = h->hover.flight_mode;
  const int tiles = grid_for(h->n);
  const int spare_copy = h->env.inline_reset ? 0 : 1;
  if (spare_copy && !h->fused_ready) {
    QX_PARAMS_SWITCH(h, PFB_MODE_SWITCH(mode, (k_hover_spare_ahead<MODE, PS><<<tiles, kBlock, 0, s>>>(ps, h->hover, h->rng, h->buf.start_pos, h->buf.start_orn,
                                                                                                      h->d_spare, h->d_episode, h->n))));
    LAUNCH_CHECK(h);
    h->fused_ready = 1;
  }
  const StepPlan pl = plan_step(h);
  int32_t* cnt = h->d_counters + 5 + (h->same_launches & 1u);
  int32_t* cnt_next = h->d_counters + 5 + ((h->same_launches + 1u) & 1u);
  if (pl.prof) CUDA_OK(cudaEventRecord(h->prof_ev[2 * h->prof_n], s));
#define SAME_ARGS ps, h->hover, h->rng, h->buf.state, qx_rows(h), actions, h->buf.obs, h->buf.final_obs, h->buf.reward, h->buf.term, h->buf.trunc, \
                  h->buf.info, h->buf.start_pos, h->buf.start_orn, h->d_spare, h->d_episode, cnt, h->d_consumed, cnt_next, spare_copy, pl.seq, T, h->n
  if (randact) { QX_PARAMS_SWITCH(h, PFB_MODE_SWITCH(mode, (k_hover_same<MODE, true, PS><<<tiles, kBlock, 0, s>>>(SAME_ARGS)))); }
  else { QX_PARAMS_SWITCH(h, PFB_MODE_SWITCH(mode, (k_hover_same<MODE, false, PS><<<tiles, kBlock, 0, s>>>(SAME_ARGS)))); }
#undef SAME_ARGS
  LAUNCH_CHECK(h);
  if (pl.prof) {
    CUDA_OK(cudaEventRecord(h->prof_ev[2 * h->prof_n + 1], s));
    h->prof_n += 1;
  }
  if (spare_copy && hover_topup(h, cnt, s)) return -1;
  h->same_launches += 1;
  h->step_seq += (uint64_t)T;
  return 0;
}

static int hover_env_step(PfbContext* h, float* actions, const float* noise, bool randact, size_t dyn_smem, cudaStream_t s) {
  const int mode = h->hover.flight_mode;
  if (h->env.autoreset == PFB_AUTORESET_SAME_STEP) {
    if (noise) return fail("injected noise (parity mode) is only supported with autoreset = 0");
    return hover_same_launch(h, actions, randact, 1, s);
  }
  const bool autoreset = h->env.autoreset != 0;
  // step k appends the envs that finish to list k; its builder CTAs start the next spares of list k - 1 (the envs this launch
  // resets) and finish those of list k - 2, next to which phase 0 left the episode numbers it started (d_elist)
  const StepPlan pl = plan_step(h);
  const uint64_t k = h->step_seq;
  int32_t* cnt_b1 = h->d_counters + ((k + 2) % 4);
  int32_t* list_b1 = h->d_done_list + ((k + 2) % 4) * h->n;
  uint32_t* elist_b0 = h->d_elist ? h->d_elist + ((k + 3) % 4) * h->n : nullptr;
  uint32_t* elist_b1 = h->d_elist ? h->d_elist + ((k + 2) % 4) * h->n : nullptr;
  const bool spares = autoreset && h->d_spare != nullptr;
  const int spare_copy = (spares && !h->env.inline_reset) ? 1 : 0;
  const int tiles = grid_for(h->n);
  const int builders = spares ? (h->sm_count < tiles ? h->sm_count : tiles) : 0;
  const int grid = tiles + 2 * builders;
  if (pl.prof) CUDA_OK(cudaEventRecord(h->prof_ev[2 * h->prof_n], s));
#define STEP_ARGS ps, h->hover, h->rng, h->buf.state, qx_rows(h), actions, noise, h->buf.obs, h->buf.reward, h->buf.term, h->buf.trunc,             \
                  h->buf.info, h->buf.start_pos, h->buf.start_orn, pl.cnt_cur, pl.list_cur, pl.cnt_next, pl.cnt_prev, pl.list_prev, cnt_b1, list_b1, \
                  elist_b0, elist_b1, h->d_spare, h->d_episode, spare_copy, builders, h->noise_dump, pl.seq, h->n
  if (autoreset) {
    if (noise) return fail("injected noise (parity mode) is only supported with autoreset = 0");
    if (randact) {
      QX_PARAMS_SWITCH(h, PFB_MODE_SWITCH(mode, (k_hover_step<MODE, false, true, true, false, PS><<<grid, kBlock, dyn_smem, s>>>(STEP_ARGS))));
    } else {
      QX_PARAMS_SWITCH(h, PFB_MODE_SWITCH(mode, (k_hover_step<MODE, false, false, true, false, PS><<<grid, kBlock, dyn_smem, s>>>(STEP_ARGS))));
    }
  } else if (h->hover.ma) {  // one vehicle table (pfb_set_models refuses MAQuadXHover handles)
    if (randact) return fail("MAQuadXHover has no on-device action generator");
    const QuadXParams& ps = h->qx;
    if (noise) { PFB_MODE_SWITCH(mode, (k_hover_step<MODE, true, false, false, true, QuadXParams><<<grid, kBlock, dyn_smem, s>>>(STEP_ARGS))); }
    else { PFB_MODE_SWITCH(mode, (k_hover_step<MODE, false, false, false, true, QuadXParams><<<grid, kBlock, dyn_smem, s>>>(STEP_ARGS))); }
  } else {
    if (noise) {
      QX_PARAMS_SWITCH(h, PFB_MODE_SWITCH(mode, (k_hover_step<MODE, true, false, false, false, PS><<<grid, kBlock, dyn_smem, s>>>(STEP_ARGS))));
    } else if (randact) {
      QX_PARAMS_SWITCH(h, PFB_MODE_SWITCH(mode, (k_hover_step<MODE, false, true, false, false, PS><<<grid, kBlock, dyn_smem, s>>>(STEP_ARGS))));
    } else {
      QX_PARAMS_SWITCH(h, PFB_MODE_SWITCH(mode, (k_hover_step<MODE, false, false, false, false, PS><<<grid, kBlock, dyn_smem, s>>>(STEP_ARGS))));
    }
  }
#undef STEP_ARGS
  LAUNCH_CHECK(h);
  if (pl.prof) {
    CUDA_OK(cudaEventRecord(h->prof_ev[2 * h->prof_n + 1], s));
    h->prof_n += 1;
  }
  h->step_seq += 1;
  h->fused_ready = 0;  // the step pipeline owns the spares again
  return 0;
}

// QuadX-Hover with autoreset: n_steps >= kFusedMinSteps run as fused launches of up to kRolloutMaxSteps env steps (k_hover_rollout)
static bool hover_fused_ok(PfbContext* h) {
  return h->model.kind == PFB_KIND_QUADX && h->env.env_kind == PFB_ENV_QUADX_HOVER && h->env.autoreset != 0 && !h->env.inline_reset &&
         h->d_spare != nullptr && h->d_consumed != nullptr && h->noise_dump == nullptr && !(h->prof_ev && h->prof_n < h->prof_cap);
}
constexpr int kFusedMinSteps = 4;
static int hover_rollout_fused(PfbContext* h, int n_steps, cudaStream_t s) {
  const int mode = h->hover.flight_mode;
  const int tiles = grid_for(h->n);
  if (!h->fused_ready) {
    // finish what the single-step pipeline left half done, then bring every env's spares kRolloutAhead ahead
    if (h->step_seq >= 2 && hover_drain(h, s)) return -1;
    QX_PARAMS_SWITCH(h, PFB_MODE_SWITCH(mode, (k_hover_spare_ahead<MODE, PS><<<tiles, kBlock, 0, s>>>(ps, h->hover, h->rng, h->buf.start_pos, h->buf.start_orn,
                                                                                                      h->d_spare, h->d_episode, h->n))));
    LAUNCH_CHECK(h);
    h->fused_ready = 1;
  }
  while (n_steps > 0) {
    const int T = n_steps < kRolloutMaxSteps ? n_steps : kRolloutMaxSteps;
    const uint64_t k0 = h->step_seq, k_last = k0 + (uint64_t)T - 1;
    CUDA_OK(cudaMemsetAsync(h->d_counters, 0, 8 * sizeof(int32_t), s));  // [0..3] step pipeline lists, [5] spares consumed by this launch
    QX_PARAMS_SWITCH(h, PFB_MODE_SWITCH(mode, (k_hover_rollout<MODE, PS><<<tiles, kBlock, 0, s>>>(
                                                   ps, h->hover, h->rng, h->buf.state, qx_rows(h), h->buf.setpoint, h->buf.obs, h->buf.reward, h->buf.term,
                                                   h->buf.trunc, h->buf.info, h->buf.start_pos, h->buf.start_orn, h->d_spare, h->d_episode, h->d_counters + 5,
                                                   h->d_consumed, h->d_counters + (k_last % 4), h->d_done_list + (k_last % 4) * h->n, (uint32_t)k0, T, h->n))));
    LAUNCH_CHECK(h);
    if (hover_topup(h, h->d_counters + 5, s)) return -1;
    h->step_seq += (uint64_t)T;
    n_steps -= T;
  }
  return 0;
}

// The spares whose first half the last step launch integrated are finished (so that episode[] names each env's next spare) and
// taken off the queue the next launch would finish them from; the envs finished on the last launch stay queued, so that launch
// builds their next spares.  Then every record fails its validity check: each env's next reset runs the cold path under
// episode[i], the number the spare path would have used, and the builders / k_hover_spare_ahead replace the records.
static int hover_invalidate_spares(PfbContext* h, cudaStream_t s) {
  const uint64_t k = h->step_seq;
  if (k >= 2) {
    if (hover_drain(h, s)) return -1;
    CUDA_OK(cudaMemsetAsync(h->d_counters + ((k + 2) % 4), 0, sizeof(int32_t), s));
  }
  CUDA_OK(cudaMemset2DAsync(h->d_spare + SP_VALID, SP_ROWS * sizeof(float), 0, sizeof(float), (size_t)kSpareBufs * h->n, s));
  h->fused_ready = 0;
  return 0;
}

static int hover_env_rollout(PfbContext* h, int n_steps, cudaStream_t s) {
  if (h->env.autoreset == PFB_AUTORESET_SAME_STEP) {  // the same kernel as a single step, kRolloutMaxSteps steps per launch
    for (int k = 0; k < n_steps; k += kRolloutMaxSteps)
      if (hover_same_launch(h, h->buf.setpoint, true, n_steps - k < kRolloutMaxSteps ? n_steps - k : kRolloutMaxSteps, s)) return -1;
    return 0;
  }
  if (n_steps >= kFusedMinSteps && hover_fused_ok(h)) return hover_rollout_fused(h, n_steps, s);
  for (int k = 0; k < n_steps; ++k)
    if (hover_env_step(h, h->buf.setpoint, nullptr, true, 0, s)) return -1;
  return 0;
}

const HandleOps kQuadXAviaryOps = {
    .kind = PFB_KIND_QUADX, .env_kind = PFB_ENV_NONE,
    .state_rows = QX_ROWS, .istate_rows = QI_ROWS, .layout = PFB_LAYOUT_WARP_TILED, .setpoint_dim = 4, .aux_dim = 4,
    .obs_dim = hover_obs_dim,
    .reset = qx_reset, .set_mode = qx_set_mode, .set_modes = qx_set_modes, .aviary_step = qx_aviary_step, .observe = qx_observe,
    .set_base_state = qx_set_base_state, .get_base_state = qx_get_base_state,
};

const HandleOps kHoverOps = {
    .kind = PFB_KIND_QUADX, .env_kind = PFB_ENV_QUADX_HOVER,
    .state_rows = QX_ROWS, .istate_rows = QI_ROWS, .layout = PFB_LAYOUT_WARP_TILED, .setpoint_dim = 4, .aux_dim = 4,
    .obs_dim = hover_obs_dim,
    .reset = qx_reset, .set_mode = qx_set_mode, .aviary_step = qx_aviary_step, .observe = qx_observe,
    .env_reset = hover_env_reset, .env_step = hover_env_step, .env_rollout = hover_env_rollout,
    .spare_rows = SP_ROWS * kSpareBufs,
    .consumed_rows = kRolloutMaxSteps / 2 + 1,  // an env resets at most every second step of a fused launch
    .invalidate_spares = hover_invalidate_spares,
};

// MAQuadXHover: no autoreset, so no spares; its rollout falls back to single steps inside hover_env_rollout
const HandleOps kMAQuadXHoverOps = {
    .kind = PFB_KIND_QUADX, .env_kind = PFB_ENV_MA_QUADX_HOVER,
    .state_rows = QM_ROWS, .istate_rows = QI_ROWS, .layout = PFB_LAYOUT_WARP_TILED, .setpoint_dim = 4, .aux_dim = 4,
    .obs_dim = hover_obs_dim,
    .reset = qx_reset, .set_mode = qx_set_mode, .aviary_step = qx_aviary_step, .observe = qx_observe,
    .env_reset = hover_env_reset, .env_step = hover_env_step, .env_rollout = hover_env_rollout,
};
