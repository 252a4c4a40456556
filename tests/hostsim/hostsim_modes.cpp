// TEST HARNESS — the host simulator (hostsim.cpp) plus one flight mode per drone: the glue of k_quadx_set_modes and
// k_quadx_aviary_step<kModePerDrone, ...> (pfb_quadx.cu) over the field-major layout, through the same PFB_HD dispatch helpers
// (quadx_set_mode_any, quadx_aviary_step_any), so that the per-drone control path also runs on the CPU.
#include "hostsim.cpp"

HS_API int hs_set_modes(const int8_t* modes, float* st, int32_t* ist, float* setpoint, int64_t N) {
  for (int64_t i = 0; i < N; ++i) {
    if (modes[i] < -1 || modes[i] > 7) return fail("bad mode %d", (int)modes[i]);
    QuadXRegs s;
    quadx_load<7>(st, ist, N, i, s);
    for (int k = 0; k < 4; ++k) s.sp[k] = setpoint[4 * i + k];
    quadx_set_mode_any(s, modes[i]);
    quadx_store<7>(st, ist, N, i, s);
    for (int k = 0; k < 4; ++k) setpoint[4 * i + k] = s.sp[k];
  }
  return 0;
}

HS_API int hs_aviary_step_modes(const PfbModel* m, const int8_t* modes, float* st, int32_t* ist, const float* setpoint, const float* noise,
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
    for (int k = 0; k < n_steps; ++k) quadx_aviary_step_any(p, s, modes[i], nz);
    quadx_store<7>(st, ist, N, i, s);
  }
  return 0;
}
