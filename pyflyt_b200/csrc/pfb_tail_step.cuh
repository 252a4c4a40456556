// pfb_tail_step.cuh — the step kernel body of the env kinds whose autoreset runs in "tail" CTAs (DESIGN.md §4):
// QuadX-Waypoints, Fixedwing-Waypoints and Rocket-Landing call tail_step() with a per-env policy; the Dogfight, whose work
// items are whole arenas, shares the work-item plan, the done-list append and the observation write-out.
//
// One launch of step k: regular CTAs own one env per thread and skip the envs a tail CTA owns (finished on step k - 1, or
// already rewritten by a tail CTA of this launch: the fresh tag).  The first tail_blocks CTAs reset the envs on the done list
// of step k - 1, normally by copying the env's spare post-reset state, and finished envs of step k go onto the done list of
// step k, so no env has two writers in one launch.  The same kernel in build mode (build = 1: no step, no outputs) computes
// the spares: on the side stream for the envs a step consumed, or for every env after a user reset (prev_list = nullptr).
#pragma once

#include "pfb_context.h"

// Spare post-reset state of one env: an env-major record of Env::kSpareRows floats holding the env's state words in rows
// [0, Env::kStateRows), then this trailer: the start pose it was built for, valid, flags and the episode number that keys
// its draws.  The inline reset of an env without a usable spare uses the same episode number, so both give the same bits.
enum { SPARE_POSE = 0, SPARE_VALID = 6, SPARE_FLAGS = 7, SPARE_EPISODE = 8, SPARE_TRAILER = 9 };

// the work items of this thread: t = t0, t0 + stride, ... < t_end; a tail lane strides over the done list (over every env or
// arena when prev_list is null), a regular lane owns env block_first + threadIdx.x.  Work items are arenas of A envs.
struct TailPlan {
  bool tail;
  int64_t block_first;
  int t0, t_end, stride;
};
template <bool AUTORESET, int A = 1>
__device__ __forceinline__ TailPlan tail_plan(int tail_blocks, int build, const int32_t* __restrict__ prev_count,
                                              const int32_t* __restrict__ prev_list, int32_t* __restrict__ next_count, int64_t N) {
  TailPlan pl;
  pl.tail = AUTORESET && (int)blockIdx.x < tail_blocks;
  pl.block_first = pl.tail ? 0 : (int64_t)((int)blockIdx.x - (AUTORESET ? tail_blocks : 0)) * kBlock;
  if (pl.tail) {
    if (blockIdx.x == 0 && threadIdx.x == 0 && !build) *next_count = 0;  // arm the counter the next launch appends to
    pl.t0 = (blockIdx.x * kBlock + threadIdx.x) / A;
    pl.t_end = prev_list ? *prev_count : (int)(N / A);  // build mode after a user reset: every env
    pl.stride = tail_blocks * kBlock / A;
  } else {
    pl.t0 = 0;
    pl.t_end = (pl.block_first + threadIdx.x < N) ? 1 : 0;
    pl.stride = 1;
  }
  return pl;
}

// warp-aggregated append of id to the done list, for the lanes of `lanes` that pass done: one atomic per warp
__device__ __forceinline__ void done_list_append(unsigned lanes, bool done, int64_t id, int32_t* __restrict__ count,
                                                 int32_t* __restrict__ list) {
  unsigned m = __ballot_sync(lanes, done);
  if (done) {
    int lane = threadIdx.x & 31;
    int leader = __ffs(m) - 1;
    int base = 0;
    if (lane == leader) base = atomicAdd(count, __popc(m));
    base = __shfl_sync(m, base, leader);
    list[base + __popc(m & ((1u << lane) - 1u))] = (int32_t)id;
  }
}

// a tail lane writes its observation row by row; the regular CTAs stage theirs in shared memory (row stride kStride) and
// write the CTA's [rows][O] block with coalesced stores once every lane is done, leaving out the rows of the envs they skipped
__device__ __forceinline__ void obs_write_row(float* __restrict__ obs, int64_t i, int O, const float* row) {
  float* dst = obs + i * O;
  for (int k = 0; k < O; ++k) dst[k] = row[k];
}
template <int kStride>
__device__ __forceinline__ void obs_write_block(float* __restrict__ obs, const float* smem, uint8_t* row_skip, bool skip, int64_t block_first,
                                                int O, int64_t N) {
  row_skip[threadIdx.x] = skip ? 1 : 0;
  __syncthreads();
  int64_t rows = N - block_first;
  if (rows > kBlock) rows = kBlock;
  const int total = (int)rows * O;
  float* dst = obs + block_first * O;
  const int dr = kBlock / O, dc = kBlock - dr * O;
  int r = threadIdx.x / O, c = threadIdx.x - r * O;
  for (int j = threadIdx.x; j < total; j += kBlock) {
    if (!row_skip[r]) dst[j] = smem[r * kStride + c];
    r += dr; c += dc;
    if (c >= O) { c -= O; ++r; }
  }
}

// The step of one launch for an env kind given by the policy Env, which holds references to the kernel's __grid_constant__
// parameter blocks (a copy would be staged on the stack) and provides:
//   Regs, Item                 the vehicle registers (with .flags) and the env's own per-env state
//   kStateRows, kSpareRows     where the spare trailer starts, and the record size
//   kActions, kObsStride       action width, shared-memory row stride of the observation (> its largest width)
//   obs_dim(), pose_keyed()    observation width; whether a spare is only valid for the start pose it was built for
//   item(i)                    per-env set-up before either path
//   load_spare / reset / store_spare    env.reset() from a spare record, inline (into `rec` when building), into `rec`
//   load / action / step       env.step(): the state, the action (drawn when RANDACT), the Aviary steps and the epilogue
//   observe / store / info     the observation row, the state and the info byte after either path
// The pointers stay __restrict__ parameters of the hooks: in a struct they would lose it.
template <bool AUTORESET, class Env>
__device__ __forceinline__ void tail_step(const Env& env, float* __restrict__ st, int32_t* __restrict__ ist, float* __restrict__ actions,
                                          const float* __restrict__ noise, float* __restrict__ obs, float* __restrict__ reward,
                                          uint8_t* __restrict__ term, uint8_t* __restrict__ trunc, uint8_t* __restrict__ info,
                                          const float* __restrict__ start_pos, const float* __restrict__ start_orn,
                                          const int32_t* __restrict__ prev_count, const int32_t* __restrict__ prev_list,
                                          int32_t* __restrict__ cur_count, int32_t* __restrict__ cur_list, int32_t* __restrict__ next_count,
                                          float* __restrict__ spare, int spare_copy, int build, int tail_blocks, uint32_t step_seq, int64_t N) {
  constexpr int R = Env::kStateRows;
  static_assert(R + SPARE_TRAILER <= Env::kSpareRows, "spare record too small");
  __shared__ float smem[kBlock * Env::kObsStride];
  __shared__ uint8_t row_skip[kBlock];
  const int O = env.obs_dim();
  const TailPlan pl = tail_plan<AUTORESET>(tail_blocks, build, prev_count, prev_list, next_count, N);
  bool skip = true;
  float* row = smem + threadIdx.x * Env::kObsStride;
#pragma unroll 1
  for (int t = pl.t0; t < pl.t_end; t += pl.stride) {
    const int64_t i = pl.tail ? (prev_list ? (int64_t)prev_list[t] : (int64_t)t) : pl.block_first + threadIdx.x;
    typename Env::Item x = env.item(i);
    typename Env::Regs s;
    float act[Env::kActions] = {};
    int step_count = 0;
    float rew = 0.0f;
    if (pl.tail) {
      float* rec = spare ? spare + i * Env::kSpareRows : nullptr;
      uint32_t nseq = step_seq | 0x40000000u;
      bool hit = false;
      float pose[6];
#pragma unroll
      for (int k = 0; k < 3; ++k) { pose[k] = start_pos[3 * i + k]; pose[3 + k] = start_orn[3 * i + k]; }
      if (rec) {
        nseq = __float_as_uint(rec[R + SPARE_EPISODE]) + (build ? 1u : 0u);
        hit = !build && spare_copy && rec[R + SPARE_VALID] != 0.0f;
        if (env.pose_keyed()) {
#pragma unroll
          for (int k = 0; k < 6; ++k) hit = hit && (rec[R + SPARE_POSE + k] == pose[k]);
        }
      }
      if (hit) {
        env.load_spare(rec, st, ist, N, i, s, x);
        s.flags = __float_as_uint(rec[R + SPARE_FLAGS]);
      } else {
        if (build) {
          rec[R + SPARE_VALID] = 0.0f;  // invalid until the reset below is stored
#pragma unroll
          for (int k = 0; k < 6; ++k) rec[R + SPARE_POSE + k] = pose[k];
        }
        env.reset(pose, nseq, build ? rec : nullptr, st, N, i, s, x);
      }
      if (build) {
        env.store_spare(rec, ist, N, i, s, x);
        rec[R + SPARE_FLAGS] = __uint_as_float(s.flags);
        rec[R + SPARE_EPISODE] = __uint_as_float(nseq);
        rec[R + SPARE_VALID] = 1.0f;
        continue;
      }
      s.flags |= pfb::fresh_tag(step_seq);
    } else {
      env.load(st, ist, N, i, s);
      if (AUTORESET && (s.flags & (pfb::FLAG_TERM | pfb::FLAG_TRUNC | pfb::fresh_tag(step_seq)))) continue;  // a tail CTA owns this env
      s.flags &= ~(uint32_t)pfb::FLAG_FRESH_ANY;
      env.action(actions, i, step_seq, act);
      env.step(st, ist, noise, N, i, step_seq, act, s, x, step_count, rew);
    }
    env.observe(st, N, i, act, s, x, row);
    env.store(st, ist, N, i, s, x, step_count);
    reward[i] = rew;
    term[i] = (s.flags & pfb::FLAG_TERM) ? 1 : 0;
    trunc[i] = (s.flags & pfb::FLAG_TRUNC) ? 1 : 0;
    if (info) info[i] = env.info(s, x);
    if (pl.tail) {
      obs_write_row(obs, i, O, row);
    } else {
      skip = false;
      if (AUTORESET) done_list_append(__activemask(), (s.flags & (pfb::FLAG_TERM | pfb::FLAG_TRUNC)) != 0, i, cur_count, cur_list);
    }
  }
  if (pl.tail) return;
  obs_write_block<Env::kObsStride>(obs, smem, row_skip, skip, pl.block_first, O, N);
}

// The step of one launch under SAME_STEP autoreset (PFB_AUTORESET_SAME_STEP): no tail CTAs, every lane owns env
// block_first + threadIdx.x.  A lane whose env finishes writes the step's outputs from the terminal state as usual and its
// terminal observation row to final_obs, stores the terminal state, then resets its env in this launch exactly as a tail
// lane of tail_step would on the next one (the spare record, or the inline reset under the record's episode number, so both
// modes give episode e of env i the same bits), observes the reset state into obs and appends the env to the done list of
// this step.  The side-stream rebuild of the consumed spares reads that list; the next step launch waits for it.
template <class Env>
__device__ __forceinline__ void tail_step_same(const Env& env, float* __restrict__ st, int32_t* __restrict__ ist, float* __restrict__ actions,
                                               const float* __restrict__ noise, float* __restrict__ obs, float* __restrict__ final_obs,
                                               float* __restrict__ reward, uint8_t* __restrict__ term, uint8_t* __restrict__ trunc,
                                               uint8_t* __restrict__ info, const float* __restrict__ start_pos, const float* __restrict__ start_orn,
                                               int32_t* __restrict__ cur_count, int32_t* __restrict__ cur_list, int32_t* __restrict__ next_count,
                                               const float* __restrict__ spare, int spare_copy, uint32_t step_seq, int64_t N) {
  constexpr int R = Env::kStateRows;
  static_assert(R + SPARE_TRAILER <= Env::kSpareRows, "spare record too small");
  __shared__ float smem[kBlock * Env::kObsStride];
  __shared__ uint8_t row_skip[kBlock];
  const int O = env.obs_dim();
  const int64_t block_first = (int64_t)blockIdx.x * kBlock;
  const int64_t i = block_first + threadIdx.x;
  if (blockIdx.x == 0 && threadIdx.x == 0) *next_count = 0;  // arm the counter the next launch appends to
  float* row = smem + threadIdx.x * Env::kObsStride;
  if (i < N) {
    typename Env::Item x = env.item(i);
    typename Env::Regs s;
    float act[Env::kActions] = {};
    int step_count = 0;
    float rew = 0.0f;
    env.load(st, ist, N, i, s);
    s.flags &= ~(uint32_t)pfb::FLAG_FRESH_ANY;
    env.action(actions, i, step_seq, act);
    env.step(st, ist, noise, N, i, step_seq, act, s, x, step_count, rew);
    env.observe(st, N, i, act, s, x, row);
    env.store(st, ist, N, i, s, x, step_count);
    reward[i] = rew;
    term[i] = (s.flags & pfb::FLAG_TERM) ? 1 : 0;
    trunc[i] = (s.flags & pfb::FLAG_TRUNC) ? 1 : 0;
    if (info) info[i] = env.info(s, x);
    const bool done = (s.flags & (pfb::FLAG_TERM | pfb::FLAG_TRUNC)) != 0;
    if (done) {
      obs_write_row(final_obs, i, O, row);
      // env.reset(): what a tail lane of tail_step does with this env on the next launch
      const float* rec = spare + i * Env::kSpareRows;
      typename Env::Item y = env.item(i);
      typename Env::Regs r;
      float zero[Env::kActions] = {};
      float pose[6];
#pragma unroll
      for (int k = 0; k < 3; ++k) { pose[k] = start_pos[3 * i + k]; pose[3 + k] = start_orn[3 * i + k]; }
      const uint32_t nseq = __float_as_uint(rec[R + SPARE_EPISODE]);
      bool hit = spare_copy && rec[R + SPARE_VALID] != 0.0f;
      if (env.pose_keyed()) {
#pragma unroll
        for (int k = 0; k < 6; ++k) hit = hit && (rec[R + SPARE_POSE + k] == pose[k]);
      }
      if (hit) {
        env.load_spare(rec, st, ist, N, i, r, y);
        r.flags = __float_as_uint(rec[R + SPARE_FLAGS]);
      } else {
        env.reset(pose, nseq, nullptr, st, N, i, r, y);
      }
      env.observe(st, N, i, zero, r, y, row);
      env.store(st, ist, N, i, r, y, 0);
    }
    done_list_append(__activemask(), done, i, cur_count, cur_list);
  }
  obs_write_block<Env::kObsStride>(obs, smem, row_skip, i >= N, block_first, O, N);
}
