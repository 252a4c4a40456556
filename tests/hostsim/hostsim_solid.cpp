// TEST HARNESS — the host simulator (hostsim.cpp) plus the solid rule of the static bodies of an Aviary handle (SolidCtx,
// DESIGN.md §4h "solid static bodies"): the helpers on their own (solid_live, solid_point_contact, solid_bits, the solver of
// the rule), and the QuadX, fixed-wing and rocket Aviary steps with SolidCtx over the field-major layout.  The world comes in
// flat arrays in pfb::StaticWorld's layout, as in hostsim_static.cpp.
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

#define HS_WORLD_ARGS int n, const int *body, const int *kind, const float *at, const float *yaw_cs, const float *half, const float *pose
#define HS_MAKE_WORLD(w) \
  StaticWorld w;         \
  if (make_world(n, body, kind, at, yaw_cs, half, w)) return -1

// solid_live at base (px, py, pz) of world i
HS_API int hs_solid_live(HS_WORLD_ARGS, int64_t n_worlds, int64_t i, float px, float py, float pz, float reach, uint32_t* live) {
  HS_MAKE_WORLD(w);
  *live = solid_live(w, pose, n_worlds, i, px, py, pz, reach);
  return 0;
}

// solid_point_contact of world point (x, y, z) of world i against the primitives of `live`: depth, world normal n[3]
HS_API int hs_solid_point_contact(HS_WORLD_ARGS, int64_t n_worlds, int64_t i, uint32_t live, float x, float y, float z, float* depth, float* nrm) {
  HS_MAKE_WORLD(w);
  const SolidContact c = solid_point_contact(w, pose, n_worlds, i, live, x, y, z);
  *depth = c.depth;
  nrm[0] = c.n.x; nrm[1] = c.n.y; nrm[2] = c.n.z;
  return 0;
}

// The QuadX model m at base position base[3], rotation R[9] (row-major, body -> world), in world i: the solid-rule bits
// against the primitives of `live`, and the solver's answer (world velocity v[3], body rate w[3] in; out in vo, wo) over them.
HS_API int hs_solid_bits_solve(const PfbModel* m, HS_WORLD_ARGS, int64_t n_worlds, int64_t i, uint32_t live, const float* base, const float* R,
                               const float* v, const float* w_b, uint32_t* bits, float* vo, float* wo, int* touched) {
  QuadXParams p;
  if (build_quadx_params(*m, p)) return -1;
  HS_MAKE_WORLD(w);
  SolidBase b{base[0], base[1], base[2], {R[0], R[1], R[2], R[3], R[4], R[5], R[6], R[7], R[8]}};
  *bits = solid_bits(&w, pose, n_worlds, i, live, &p, b);
  const Vec3 vbn = Vec3{R[0] * v[0] + R[3] * v[1] + R[6] * v[2], R[1] * v[0] + R[4] * v[1] + R[7] * v[2], R[2] * v[0] + R[5] * v[1] + R[8] * v[2]};
  const SolidCtx ctx{&w, pose, n_worlds, i, 0u};
  const ContactVel cv = solve_contacts_solid(&p, ctx, live, b, vbn, Vec3{w_b[0], w_b[1], w_b[2]}, 1.0f / p.inv_mass, Vec3{0.f, 0.f, 0.f}, p.Ixx, 0.0f,
                                             0.0f, p.Iyy, 0.0f, p.Izz, p.dt);
  vo[0] = cv.vx; vo[1] = cv.vy; vo[2] = cv.vz;
  wo[0] = cv.wx; wo[1] = cv.wy; wo[2] = cv.wz;
  *touched = cv.touched;
  return 0;
}

// n_steps x Aviary.step() of N QuadX drones in flight mode `mode` against the solid static bodies of their worlds (pose:
// [5 * 8][N]), with the contact response when `contact`; bits[i] = what drone i touched during its last step
template <int MODE, bool CONTACT>
static void aviary_step_solid_t(const QuadXParams& p, const StaticWorld& world, const float* pose, float* st, int32_t* ist, const float* setpoint,
                                const float* noise, int n_steps, int64_t N, uint32_t* bits) {
  for (int64_t i = 0; i < N; ++i) {
    SolidCtx w{&world, pose, N, i, 0u};
    QuadXRegs s;
    quadx_load<MODE>(st, ist, N, i, s);
    for (int k = 0; k < 4; ++k) s.sp[k] = setpoint[4 * i + k];
    HostNoise nz{noise + i, N};
    for (int k = 0; k < n_steps; ++k) quadx_aviary_step<MODE, CONTACT>(p, s, nz, &w);
    quadx_store<MODE>(st, ist, N, i, s);
    bits[i] = w.bits;
  }
}
HS_API int hs_aviary_step_solid(const PfbModel* m, int mode, int contact, HS_WORLD_ARGS, float* st, int32_t* ist, const float* setpoint,
                                const float* noise, int n_steps, int64_t N, uint32_t* bits) {
  QuadXParams p;
  if (build_quadx_params(*m, p)) return -1;
  HS_MAKE_WORLD(w);
  if (contact) { MODE_SWITCH(mode, (aviary_step_solid_t<MODE, true>(p, w, pose, st, ist, setpoint, noise, n_steps, N, bits))); }
  else { MODE_SWITCH(mode, (aviary_step_solid_t<MODE, false>(p, w, pose, st, ist, setpoint, noise, n_steps, N, bits))); }
  return 0;
}

// the rocket's Aviary step (no pad of Rocket-Landing) against the solid static bodies of its world, contact response on
HS_API int hs_rk_aviary_step_solid(const PfbModel* m, HS_WORLD_ARGS, float* st, int32_t* ist, const float* setpoint, const float* noise, int n_steps,
                                   int64_t N, uint32_t* bits) {
  RocketParams p;
  LandingParams l;
  if (rk_build_params_impl(*m, nullptr, p, l)) return -1;
  p.contact_response = 1;
  HS_MAKE_WORLD(world);
  for (int64_t i = 0; i < N; ++i) {
    SolidCtx w{&world, pose, N, i, 0u};
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

// the fixed-wing's Aviary step (flight mode `mode`, the one-basic-block substep when `full`) against the solid static bodies
// of its world, contact response on
HS_API int hs_fw_aviary_step_solid(const PfbModel* m, int mode, int full, HS_WORLD_ARGS, float* st, int32_t* ist, const float* setpoint,
                                   const float* noise, int n_steps, int64_t N, uint32_t* bits) {
  FixedwingParams p;
  WaypointParams wp;
  if (fw_build_params_impl(*m, nullptr, p, wp)) return -1;
  if (full && !fixedwing_full_model(p)) return fail("hs_fw_aviary_step_solid: the model is not complete (surfaces / wind)");
  HS_MAKE_WORLD(world);
  for (int64_t i = 0; i < N; ++i) {
    SolidCtx w{&world, pose, N, i, 0u};
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
