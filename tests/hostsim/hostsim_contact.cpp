// TEST HARNESS — the host simulator (hostsim.cpp) plus the contact RESPONSE of the Aviary steps: the CONTACT = true
// instantiations that k_quadx_aviary_step and k_fw_aviary_step, in one flight mode or per-drone modes
// (pfb_quadx.cu, pfb_fixedwing.cu), run on an Aviary handle created with contact_response, over the field-major layout.
// The rocket needs no new entry point: its parameter block carries the switch (hs_rk_aviary_step_contact sets it).
#include "hostsim.cpp"

template <int MODE>
static void aviary_step_contact_t(const QuadXParams& p, float* st, int32_t* ist, const float* setpoint, const float* noise, int n_steps, int64_t N) {
  for (int64_t i = 0; i < N; ++i) {
    QuadXRegs s;
    quadx_load<MODE>(st, ist, N, i, s);
    for (int k = 0; k < 4; ++k) s.sp[k] = setpoint[4 * i + k];
    HostNoise nz{noise + i, N};
    for (int k = 0; k < n_steps; ++k) quadx_aviary_step<MODE, true>(p, s, nz);
    quadx_store<MODE>(st, ist, N, i, s);
  }
}
HS_API int hs_aviary_step_contact(const PfbModel* m, int mode, float* st, int32_t* ist, const float* setpoint, const float* noise, int n_steps,
                                  int64_t N) {
  QuadXParams p;
  if (build_quadx_params(*m, p)) return -1;
  MODE_SWITCH(mode, (aviary_step_contact_t<MODE>(p, st, ist, setpoint, noise, n_steps, N)));
  return 0;
}

// one flight mode per drone (the glue of hostsim_modes.cpp) with the contact response
HS_API int hs_aviary_step_modes_contact(const PfbModel* m, const int8_t* modes, float* st, int32_t* ist, const float* setpoint, const float* noise,
                                        int n_steps, int64_t N) {
  QuadXParams p;
  if (build_quadx_params(*m, p)) return -1;
  for (int64_t i = 0; i < N; ++i) {
    if (modes[i] < -1 || modes[i] > 7) return fail("bad mode %d", (int)modes[i]);
    QuadXRegs s;
    quadx_load<7>(st, ist, N, i, s);
    quadx_mask_pid(s, modes[i]);
    for (int k = 0; k < 4; ++k) s.sp[k] = setpoint[4 * i + k];
    HostNoise nz{noise + i, N};
    for (int k = 0; k < n_steps; ++k) quadx_aviary_step_any<true>(p, s, modes[i], nz);
    quadx_store<7>(st, ist, N, i, s);
  }
  return 0;
}

// `full`: the one-basic-block substep the kernels take for a complete model in still air (fixedwing_full_model)
HS_API int hs_fw_aviary_step_contact(const PfbModel* m, int mode, int full, float* st, int32_t* ist, const float* setpoint, const float* noise,
                                     int n_steps, int64_t N) {
  FixedwingParams p;
  WaypointParams w;
  if (fw_build_params_impl(*m, nullptr, p, w)) return -1;
  if (full && !fixedwing_full_model(p)) return fail("hs_fw_aviary_step_contact: the model is not complete (surfaces / wind)");
  for (int64_t i = 0; i < N; ++i) {
    FixedwingRegs s;
    fixedwing_load(st, ist, N, i, s);
    for (int k = 0; k < 6; ++k) s.sp[k] = setpoint[6 * i + k];
    HostNoise nz{noise + i, N};
    for (int k = 0; k < n_steps; ++k) {
      if (full) {
        if (mode == 0) fixedwing_aviary_step<0, true, true>(p, s, nz); else fixedwing_aviary_step<-1, true, true>(p, s, nz);
      } else {
        if (mode == 0) fixedwing_aviary_step<0, false, true>(p, s, nz); else fixedwing_aviary_step<-1, false, true>(p, s, nz);
      }
    }
    fixedwing_store(st, ist, N, i, s);
  }
  return 0;
}

HS_API int hs_rk_aviary_step_contact(const PfbModel* m, float* st, int32_t* ist, const float* setpoint, const float* noise, int n_steps, int64_t N) {
  RocketParams p;
  LandingParams l;
  if (rk_build_params_impl(*m, nullptr, p, l)) return -1;
  p.contact_response = 1;
  for (int64_t i = 0; i < N; ++i) {
    RocketRegs s;
    rocket_load(st, ist, N, i, s);
    for (int k = 0; k < 7; ++k) s.sp[k] = setpoint[7 * i + k];
    HostNoise nz{noise + i, N};
    for (int k = 0; k < n_steps; ++k) rocket_aviary_step(p, s, nz, false);
    rocket_store(st, ist, N, i, s);
  }
  return 0;
}
