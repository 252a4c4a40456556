// TEST HARNESS — the host simulator with the contact response (hostsim_contact.cpp, which includes hostsim.cpp) plus the
// base-state calls: the glue of k_quadx_set_base_state, k_fw_set_base_state, k_rk_set_base_state and their get kernels
// (pfb_quadx.cu, pfb_fixedwing.cu, pfb_rocket.cu; per-drone bodies in pfb_aviary.cuh) over the field-major layout, through the
// same PFB_HD bodies base_state_set / base_state_get (pfb_fixedwing.cuh).  `kind` = PFB_KIND_*; the arrays are [N][3] / [N][4]
// fp64, nullptr = not given / not wanted; mask nullptr = every drone.
#include "hostsim_contact.cpp"

HS_API int hs_set_base_state(int kind, float* st, int32_t* ist, const uint8_t* mask, const double* pos, const double* quat, const double* lin,
                             const double* ang, int64_t N) {
  if (!pos != !quat) return fail("pos and quat come together");
  for (int64_t i = 0; i < N; ++i) {
    if (mask && !mask[i]) continue;
    const double *p = pos ? pos + 3 * i : nullptr, *q = quat ? quat + 4 * i : nullptr;
    const double *l = lin ? lin + 3 * i : nullptr, *a = ang ? ang + 3 * i : nullptr;
    if (kind == PFB_KIND_QUADX) {
      QuadXRegs s;
      quadx_load<7>(st, ist, N, i, s);
      for (int k = 0; k < 4; ++k) s.pwm[k] = st[(int64_t)(QX_PWM + k) * N + i];  // the load leaves the last motor command zero
      base_state_set<double>(s, p, q, l, a);
      quadx_store<7>(st, ist, N, i, s);
    } else if (kind == PFB_KIND_FIXEDWING) {
      FixedwingRegs s;
      fixedwing_load(st, ist, N, i, s);
      base_state_set<double>(s, p, q, l, a);
      fixedwing_store(st, ist, N, i, s);
    } else {
      RocketRegs s;
      rocket_load(st, ist, N, i, s);
      base_state_set<double>(s, p, q, l, a);
      rocket_store(st, ist, N, i, s);
    }
  }
  return 0;
}

HS_API int hs_get_base_state(int kind, const float* st, const int32_t* ist, double* pos, double* quat, double* lin, double* ang, int64_t N) {
  for (int64_t i = 0; i < N; ++i) {
    double *p = pos ? pos + 3 * i : nullptr, *q = quat ? quat + 4 * i : nullptr, *l = lin ? lin + 3 * i : nullptr, *a = ang ? ang + 3 * i : nullptr;
    if (kind == PFB_KIND_QUADX) {
      QuadXRegs s;
      quadx_load<-1>(st, ist, N, i, s);
      base_state_get(s, p, q, l, a);
    } else if (kind == PFB_KIND_FIXEDWING) {
      FixedwingRegs s;
      fixedwing_load(st, ist, N, i, s);
      base_state_get(s, p, q, l, a);
    } else {
      RocketRegs s;
      rocket_load(st, ist, N, i, s);
      base_state_get(s, p, q, l, a);
    }
  }
  return 0;
}
