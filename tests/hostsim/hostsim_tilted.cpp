// TEST HARNESS — the host simulator (hostsim.cpp) plus the solid rule with full rotation frames (TiltedCtx, DESIGN.md §4h
// "tilted static bodies"): the helpers on their own (solid_live, solid_point_contact, solid_bits, the solver of the rule), and
// the QuadX, fixed-wing and rocket Aviary steps with TiltedCtx over the field-major layout.  The world comes in flat arrays in
// pfb::TiltedWorld's layout: per primitive body, kind, centre, rotation (row-major, primitive -> body) and half sizes, and the
// poses [12 * 8][n] (x, y, z, row-major base link -> world rotation).
#include "hostsim.cpp"

static int make_world(int n, const int* body, const int* kind, const float* at, const float* rot, const float* half, TiltedWorld& w) {
  if (n < 0 || n > kMaxStaticShapes) return fail("at most %d static primitives, got %d", kMaxStaticShapes, n);
  memset(&w, 0, sizeof(w));
  w.n_shapes = n;
  for (int k = 0; k < n; ++k) {
    if (body[k] < 0 || body[k] >= kMaxStaticBodies) return fail("bad body %d", body[k]);
    w.body[k] = body[k];
    w.kind[k] = kind[k];
    for (int e = 0; e < 9; ++e) w.rot[k][e] = rot[9 * k + e];
    for (int c = 0; c < 3; ++c) { w.at[k][c] = at[3 * k + c]; w.half[k][c] = half[3 * k + c]; }
  }
  return 0;
}

#define HS_WORLD_ARGS int n, const int *body, const int *kind, const float *at, const float *rot, const float *half, const float *pose
#define HS_MAKE_WORLD(w) \
  TiltedWorld w;         \
  if (make_world(n, body, kind, at, rot, half, w)) return -1

HS_API int hs_tilted_live(HS_WORLD_ARGS, int64_t n_worlds, int64_t i, float px, float py, float pz, float reach, uint32_t* live) {
  HS_MAKE_WORLD(w);
  *live = solid_live(w, pose, n_worlds, i, px, py, pz, reach);
  return 0;
}

HS_API int hs_tilted_point_contact(HS_WORLD_ARGS, int64_t n_worlds, int64_t i, uint32_t live, float x, float y, float z, float* depth, float* nrm) {
  HS_MAKE_WORLD(w);
  const SolidContact c = solid_point_contact(w, pose, n_worlds, i, live, x, y, z);
  *depth = c.depth;
  nrm[0] = c.n.x; nrm[1] = c.n.y; nrm[2] = c.n.z;
  return 0;
}

// as hs_solid_bits_solve (hostsim_solid.cpp), with TiltedCtx
HS_API int hs_tilted_bits_solve(const PfbModel* m, HS_WORLD_ARGS, int64_t n_worlds, int64_t i, uint32_t live, const float* base, const float* R,
                                const float* v, const float* w_b, uint32_t* bits, float* vo, float* wo, int* touched) {
  QuadXParams p;
  if (build_quadx_params(*m, p)) return -1;
  HS_MAKE_WORLD(w);
  SolidBase b{base[0], base[1], base[2], {R[0], R[1], R[2], R[3], R[4], R[5], R[6], R[7], R[8]}};
  *bits = solid_bits(&w, pose, n_worlds, i, live, &p, b);
  const Vec3 vbn = Vec3{R[0] * v[0] + R[3] * v[1] + R[6] * v[2], R[1] * v[0] + R[4] * v[1] + R[7] * v[2], R[2] * v[0] + R[5] * v[1] + R[8] * v[2]};
  const TiltedCtx ctx{&w, pose, n_worlds, i, 0u};
  const ContactVel cv = solve_contacts_solid(&p, ctx, live, b, vbn, Vec3{w_b[0], w_b[1], w_b[2]}, 1.0f / p.inv_mass, Vec3{0.f, 0.f, 0.f}, p.Ixx, 0.0f,
                                             0.0f, p.Iyy, 0.0f, p.Izz, p.dt);
  vo[0] = cv.vx; vo[1] = cv.vy; vo[2] = cv.vz;
  wo[0] = cv.wx; wo[1] = cv.wy; wo[2] = cv.wz;
  *touched = cv.touched;
  return 0;
}

template <int MODE, bool CONTACT>
static void aviary_step_tilted_t(const QuadXParams& p, const TiltedWorld& world, const float* pose, float* st, int32_t* ist, const float* setpoint,
                                 const float* noise, int n_steps, int64_t N, uint32_t* bits) {
  for (int64_t i = 0; i < N; ++i) {
    TiltedCtx w{&world, pose, N, i, 0u};
    QuadXRegs s;
    quadx_load<MODE>(st, ist, N, i, s);
    for (int k = 0; k < 4; ++k) s.sp[k] = setpoint[4 * i + k];
    HostNoise nz{noise + i, N};
    for (int k = 0; k < n_steps; ++k) quadx_aviary_step<MODE, CONTACT>(p, s, nz, &w);
    quadx_store<MODE>(st, ist, N, i, s);
    bits[i] = w.bits;
  }
}
HS_API int hs_aviary_step_tilted(const PfbModel* m, int mode, int contact, HS_WORLD_ARGS, float* st, int32_t* ist, const float* setpoint,
                                 const float* noise, int n_steps, int64_t N, uint32_t* bits) {
  QuadXParams p;
  if (build_quadx_params(*m, p)) return -1;
  HS_MAKE_WORLD(w);
  if (contact) { MODE_SWITCH(mode, (aviary_step_tilted_t<MODE, true>(p, w, pose, st, ist, setpoint, noise, n_steps, N, bits))); }
  else { MODE_SWITCH(mode, (aviary_step_tilted_t<MODE, false>(p, w, pose, st, ist, setpoint, noise, n_steps, N, bits))); }
  return 0;
}

HS_API int hs_rk_aviary_step_tilted(const PfbModel* m, HS_WORLD_ARGS, float* st, int32_t* ist, const float* setpoint, const float* noise, int n_steps,
                                    int64_t N, uint32_t* bits) {
  RocketParams p;
  LandingParams l;
  if (rk_build_params_impl(*m, nullptr, p, l)) return -1;
  p.contact_response = 1;
  HS_MAKE_WORLD(world);
  for (int64_t i = 0; i < N; ++i) {
    TiltedCtx w{&world, pose, N, i, 0u};
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

HS_API int hs_fw_aviary_step_tilted(const PfbModel* m, int mode, int full, HS_WORLD_ARGS, float* st, int32_t* ist, const float* setpoint,
                                    const float* noise, int n_steps, int64_t N, uint32_t* bits) {
  FixedwingParams p;
  WaypointParams wp;
  if (fw_build_params_impl(*m, nullptr, p, wp)) return -1;
  if (full && !fixedwing_full_model(p)) return fail("hs_fw_aviary_step_tilted: the model is not complete (surfaces / wind)");
  HS_MAKE_WORLD(world);
  for (int64_t i = 0; i < N; ++i) {
    TiltedCtx w{&world, pose, N, i, 0u};
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
