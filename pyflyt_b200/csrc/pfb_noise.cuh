// pfb_noise.cuh — device-side noise sources shared by every vehicle's kernels.
#pragma once

#include "pfb_common.cuh"
#include "pfb_context.h"

using pfb::U4;
using pfb::box_muller;
using pfb::philox4x32_10;

// ---------------------------------------------------------------------------------------------------
// noise sources: raw draws of np_random.normal(*throttle.shape)  (motors.py:134-138)
// ---------------------------------------------------------------------------------------------------
struct InjectedNoise {  // parity tests: the CPU-drawn sequence, [substep][N]
  const float* ptr;
  int64_t N;
  __device__ __forceinline__ void begin_step() {}
  __device__ __forceinline__ void seek(uint32_t) {}  // the caller passes the pointer already positioned
  __device__ __forceinline__ void prefetch4() {}
  __device__ __forceinline__ void set_dump(float*, int64_t) {}
  __device__ __forceinline__ float dep(int) const { return 0.0f; }
  __device__ __forceinline__ float get(int) {
    float v = __ldg(ptr);
    ptr += N;
    return v;
  }
};

// Throughput path: N(noise_loc, 1) from Philox4x32-10, counter = (global env id, call sequence number,
// stream tag | Aviary-step index).  Stateless: nothing is stored per env, and a trajectory does not depend
// on how the batch is sharded over GPUs.  With ratio <= 2 one Philox call (4 words -> 4 normals) serves two
// consecutive Aviary steps (counter = the even step of the pair).  prefetch4() issues the calls of the next four
// Aviary steps at once — the env-step kernels call it before they touch the state they loaded, so that the ~400
// integer instructions of the generator run in the shadow of the state loads instead of inside the physics loop.
// set_dump(): optional [substep][N] buffer that receives every draw handed out (tests replay them through the oracle).
struct PhiloxNoise {
  uint32_t k0, k1, env_lo, env_hi, seq, tag;
  uint32_t step, pre;
  int ratio;
  float loc;
  float n0, n1, n2, n3;  // draws of the current pair of Aviary steps (or of the current step when ratio > 2)
  float m0, m1, m2, m3;  // prefetched draws of the following pair
  float* dump;
  int64_t dump_stride;
  __device__ __forceinline__ void init(const RngParams& r, int64_t i, uint32_t seq_, uint32_t tag_, float loc_, int ratio_) {
    k0 = r.k0; k1 = r.k1;
    uint64_t g = ((uint64_t)r.env_offset_hi << 32 | r.env_offset_lo) + (uint64_t)i;
    env_lo = (uint32_t)g; env_hi = (uint32_t)(g >> 32);
    seq = seq_; tag = tag_ << 24; step = 0; pre = 0; loc = loc_; ratio = ratio_;
    n0 = n1 = n2 = n3 = 0.0f;
    m0 = m1 = m2 = m3 = 0.0f;
    dump = nullptr; dump_stride = 0;
  }
  __device__ __forceinline__ void set_dump(float* d, int64_t stride) { dump = d; dump_stride = stride; }
  __device__ __forceinline__ void draw(uint32_t s, float& a, float& b, float& c, float& d) {
    U4 r = philox4x32_10(U4{env_lo, env_hi, seq, tag | s}, k0, k1);
    box_muller(r.x, r.y, a, b);
    box_muller(r.z, r.w, c, d);
  }
  // continue a stream at Aviary step s (a spare's warm-up is integrated in pieces over several launches)
  __device__ __forceinline__ void seek(uint32_t s) {
    step = s; pre = 0;
    if (ratio <= 2 && (s & 1u)) draw(s - 1u, n0, n1, n2, n3);  // the pair (s-1, s) shares one Philox call
  }
  __device__ __forceinline__ void prefetch4() {
    if (ratio <= 2 && (step & 1u) == 0u) {
      draw(step, n0, n1, n2, n3);
      draw(step + 2u, m0, m1, m2, m3);
      pre = step + 4u;
    }
  }
  __device__ __forceinline__ float dep(int k) const {  // the prefetched draws, for ordering constraints (mbar_wait)
    return k == 0 ? n0 : k == 1 ? n1 : k == 2 ? n2 : k == 3 ? n3 : k == 4 ? m0 : k == 5 ? m1 : k == 6 ? m2 : m3;
  }
  // out-of-line generator for the draws that were not prefetched (long warm-ups, ratio > 2): keeps the physics loop compact
  struct Four { float a, b, c, d; };
  static __device__ __noinline__ Four draw_cold(uint32_t env_lo_, uint32_t env_hi_, uint32_t seq_, uint32_t ctr3, uint32_t k0_, uint32_t k1_) {
    U4 r = philox4x32_10(U4{env_lo_, env_hi_, seq_, ctr3}, k0_, k1_);
    Four f;
    box_muller(r.x, r.y, f.a, f.b);
    box_muller(r.z, r.w, f.c, f.d);
    return f;
  }
  __device__ __forceinline__ void begin_step() {
    bool need = ratio > 2;
    if (!need && (step & 1u) == 0u) {
      if (step < pre) {
        if (step + 2u == pre) { n0 = m0; n1 = m1; n2 = m2; n3 = m3; }  // second prefetched pair moves into place
      } else {
        need = true;
      }
    }
    if (need) {
      const Four f = draw_cold(env_lo, env_hi, seq, tag | step, k0, k1);
      n0 = f.a; n1 = f.b; n2 = f.c; n3 = f.d;
    }
    ++step;
  }
  __device__ __forceinline__ float get(int u) {
    // step was already advanced: odd step-1 -> second half of the 4 normals
    int idx = ratio > 2 ? u : (int)(((step - 1u) & 1u) << 1) + u;
    float lo = (idx & 1) ? n1 : n0, hi = (idx & 1) ? n3 : n2;
    float v = loc + ((idx & 2) ? hi : lo);
    if (dump) { *dump = v; dump += dump_stride; }
    return v;
  }
};

template <bool INJECT>
struct NoiseSel;
template <>
struct NoiseSel<true> {
  typedef InjectedNoise type;
};
template <>
struct NoiseSel<false> {
  typedef PhiloxNoise type;
};

template <bool INJECT>
__device__ __forceinline__ typename NoiseSel<INJECT>::type make_noise(const float* noise, int64_t N, int64_t i,
                                                                      const RngParams& r, uint32_t seq, uint32_t tag,
                                                                      float loc, int ratio);
template <>
__device__ __forceinline__ InjectedNoise make_noise<true>(const float* noise, int64_t N, int64_t i, const RngParams&,
                                                          uint32_t, uint32_t, float, int) {
  return InjectedNoise{noise + i, N};
}
template <>
__device__ __forceinline__ PhiloxNoise make_noise<false>(const float*, int64_t, int64_t i, const RngParams& r,
                                                         uint32_t seq, uint32_t tag, float loc, int ratio) {
  PhiloxNoise n;
  n.init(r, i, seq, tag, loc, ratio);
  return n;
}

