// TEST HARNESS — the host simulator (hostsim.cpp) plus the static bodies of an Aviary handle (DESIGN.md §4h): the static_surface
// helper on its own, and the QuadX Aviary step with the static bodies of each drone's world (StaticCtx, the World of
// the k_quadx_aviary_step<..., StaticCtx> instantiations) over the field-major layout.  The world comes in flat arrays in pfb::StaticWorld's layout.
#include "hostsim.cpp"

static int make_world(int n, const int* body, const int* kind, const float* at, const float* yaw_cs, const float* half, StaticWorld& w) {
  if (n < 0 || n > kMaxStaticShapes) return fail("at most %d static primitives, got %d", kMaxStaticShapes, n);
  memset(&w, 0, sizeof(w));
  w.n_shapes = n;
  for (int k = 0; k < n; ++k) {
    if (body[k] < 0 || body[k] >= kMaxStaticBodies) return fail("bad body %d", body[k]);
    w.body[k] = body[k];
    w.kind[k] = kind[k];
    w.cyaw[k] = yaw_cs[2 * k];
    w.syaw[k] = yaw_cs[2 * k + 1];
    for (int c = 0; c < 3; ++c) { w.at[k][c] = at[3 * k + c]; w.half[k][c] = half[3 * k + c]; }
  }
  return 0;
}

// static_surface at (px, py, pz) of world i, with touch(t) = pz - t < thr; the surface height and the contact bits
HS_API int hs_static_surface(int n, const int* body, const int* kind, const float* at, const float* yaw_cs, const float* half, const float* pose,
                             int64_t n_worlds, int64_t i, float px, float py, float pz, float reach, float thr, float* surf, uint32_t* bits) {
  StaticWorld w;
  if (make_world(n, body, kind, at, yaw_cs, half, w)) return -1;
  *surf = static_surface(w, pose, n_worlds, i, px, py, pz, reach, [&](float t) { return pz - t < thr; }, *bits);
  return 0;
}

// n_steps x Aviary.step() of N QuadX drones in flight mode `mode` against the static bodies of their worlds (pose: [5 * 8][N]),
// with the contact response when `contact`; bits[i] = what drone i touched during its last step
template <int MODE, bool CONTACT>
static void aviary_step_static_t(const QuadXParams& p, const StaticWorld& world, const float* pose, float* st, int32_t* ist, const float* setpoint,
                                 const float* noise, int n_steps, int64_t N, uint32_t* bits) {
  for (int64_t i = 0; i < N; ++i) {
    StaticCtx w{&world, pose, N, i, 0u};
    QuadXRegs s;
    quadx_load<MODE>(st, ist, N, i, s);
    for (int k = 0; k < 4; ++k) s.sp[k] = setpoint[4 * i + k];
    HostNoise nz{noise + i, N};
    for (int k = 0; k < n_steps; ++k) quadx_aviary_step<MODE, CONTACT>(p, s, nz, &w);
    quadx_store<MODE>(st, ist, N, i, s);
    bits[i] = w.bits;
  }
}
HS_API int hs_aviary_step_static(const PfbModel* m, int mode, int contact, int n, const int* body, const int* kind, const float* at, const float* yaw_cs,
                                 const float* half, const float* pose, float* st, int32_t* ist, const float* setpoint, const float* noise, int n_steps,
                                 int64_t N, uint32_t* bits) {
  QuadXParams p;
  if (build_quadx_params(*m, p)) return -1;
  StaticWorld w;
  if (make_world(n, body, kind, at, yaw_cs, half, w)) return -1;
  if (contact) { MODE_SWITCH(mode, (aviary_step_static_t<MODE, true>(p, w, pose, st, ist, setpoint, noise, n_steps, N, bits))); }
  else { MODE_SWITCH(mode, (aviary_step_static_t<MODE, false>(p, w, pose, st, ist, setpoint, noise, n_steps, N, bits))); }
  return 0;
}

// the rocket's Aviary step (no pad of Rocket-Landing) against the static bodies of its world, contact response on
HS_API int hs_rk_aviary_step_static(const PfbModel* m, int n, const int* body, const int* kind, const float* at, const float* yaw_cs, const float* half,
                                    const float* pose, float* st, int32_t* ist, const float* setpoint, const float* noise, int n_steps, int64_t N,
                                    uint32_t* bits) {
  RocketParams p;
  LandingParams l;
  if (rk_build_params_impl(*m, nullptr, p, l)) return -1;
  p.contact_response = 1;
  StaticWorld world;
  if (make_world(n, body, kind, at, yaw_cs, half, world)) return -1;
  for (int64_t i = 0; i < N; ++i) {
    StaticCtx w{&world, pose, N, i, 0u};
    RocketRegs s;
    rocket_load(st, ist, N, i, s);
    for (int k = 0; k < 7; ++k) s.sp[k] = setpoint[7 * i + k];
    HostNoise nz{noise + i, N};
    for (int k = 0; k < n_steps; ++k) rocket_aviary_step(p, s, nz, false, &w);
    rocket_store(st, ist, N, i, s);
    bits[i] = w.bits;
  }
  return 0;
}

// the fixed-wing's Aviary step (flight mode `mode`, the one-basic-block substep when `full`) against the static bodies of its
// world, contact response on
HS_API int hs_fw_aviary_step_static(const PfbModel* m, int mode, int full, int n, const int* body, const int* kind, const float* at,
                                    const float* yaw_cs, const float* half, const float* pose, float* st, int32_t* ist, const float* setpoint,
                                    const float* noise, int n_steps, int64_t N, uint32_t* bits) {
  FixedwingParams p;
  WaypointParams wp;
  if (fw_build_params_impl(*m, nullptr, p, wp)) return -1;
  if (full && !fixedwing_full_model(p)) return fail("hs_fw_aviary_step_static: the model is not complete (surfaces / wind)");
  StaticWorld world;
  if (make_world(n, body, kind, at, yaw_cs, half, world)) return -1;
  for (int64_t i = 0; i < N; ++i) {
    StaticCtx w{&world, pose, N, i, 0u};
    FixedwingRegs s;
    fixedwing_load(st, ist, N, i, s);
    for (int k = 0; k < 6; ++k) s.sp[k] = setpoint[6 * i + k];
    HostNoise nz{noise + i, N};
    for (int k = 0; k < n_steps; ++k) {
      if (full) fixedwing_aviary_step_any<true, true>(p, s, mode, nz, &w);
      else fixedwing_aviary_step_any<false, true>(p, s, mode, nz, &w);
    }
    fixedwing_store(st, ist, N, i, s);
    bits[i] = w.bits;
  }
  return 0;
}
