// pfb_quadx_host.h — host-side narrowing of the fp64 vehicle table (PfbModel) to the fp32 kernel
// parameter block.  Included after a function `static int fail(const char* fmt, ...)` is in scope.
#pragma once

#include <math.h>
#include <string.h>

#include "../../include/pyflyt_b200.h"
#include "pfb_quadx.cuh"

// PfbWind (validated: kind 1..4, z_ref > 0, 0 < z0 < z_ref for the log profile, alpha >= 0) -> the fp32 block every
// vehicle's parameter table carries.  NULL or PFB_WIND_NONE is still air.
static void pfb_narrow_wind(const PfbWind* wind, pfb::WindParams& w) {
  memset(&w, 0, sizeof(w));
  if (!wind || wind->kind == PFB_WIND_NONE) return;
  // alpha = 0 is the constant profile for every z (0^0 = 1); the kernels' exp2(alpha * log2(z)) would give 0 * -inf = NaN at z <= 0
  w.kind = (wind->kind == PFB_WIND_POWER && wind->alpha == 0.0) ? PFB_WIND_CONSTANT : wind->kind;
  w.bx = (float)wind->base[0]; w.by = (float)wind->base[1]; w.bz = (float)wind->base[2];
  w.inv_zref = (float)(1.0 / wind->z_ref);
  w.alpha = (float)wind->alpha;
  if (wind->kind == PFB_WIND_LOG) {
    w.z0 = (float)wind->z0;
    w.inv_z0 = (float)(1.0 / wind->z0);
    w.inv_log = (float)(1.0 / log(wind->z_ref / wind->z0));
  }
}

static int build_quadx_params(const PfbModel& m, pfb::QuadXParams& q) {
  memset(&q, 0, sizeof(q));
  if (m.n_motors != 4) return fail("quadx model must have 4 motors, got %d", m.n_motors);
  for (int k = 0; k < 3; ++k)
    if (m.com[k] != 0.0) return fail("quadx stepper requires the composite COM at the base origin (com[%d]=%g)", k, m.com[k]);
  const double* I = m.inertia;
  if (I[1] != 0 || I[2] != 0 || I[3] != 0 || I[5] != 0 || I[6] != 0 || I[7] != 0)
    return fail("quadx stepper requires a diagonal inertia tensor");
  for (int k = 0; k < 3; ++k)
    if (m.body_pos[k] != 0.0) return fail("quadx stepper requires the drag body link at the base origin");
  q.dt = (float)(1.0 / m.physics_hz);
  q.ctrl_dt = (float)(1.0 / m.control_hz);
  q.inv_ctrl_dt = (float)m.control_hz;
  q.inv_mass = (float)(1.0 / m.mass);
  q.gravity = (float)m.gravity;
  q.vmax = (float)m.max_coord_velocity;
  q.Ixx = (float)I[0]; q.Iyy = (float)I[4]; q.Izz = (float)I[8];
  q.inv_Ixx = (float)(1.0 / I[0]); q.inv_Iyy = (float)(1.0 / I[4]); q.inv_Izz = (float)(1.0 / I[8]);
  for (int i = 0; i < 4; ++i) {
    if (m.motor_pos[i][2] != 0.0 || m.motor_axis[i][0] != 0.0 || m.motor_axis[i][1] != 0.0 || m.motor_axis[i][2] != 1.0)
      return fail("quadx stepper requires motors in the z=0 plane thrusting along +z");
    q.motor_x[i] = (float)m.motor_pos[i][0];
    q.motor_y[i] = (float)m.motor_pos[i][1];
    q.thrust_k[i] = (float)(m.thrust_coef[i] * m.max_rpm[i] * m.max_rpm[i]);
    q.torque_k[i] = (float)(m.torque_coef[i] * m.max_rpm[i] * m.max_rpm[i]);
    if (m.motor_dt_over_tau[i] != m.motor_dt_over_tau[0] || m.motor_noise_ratio[i] != m.motor_noise_ratio[0])
      return fail("quadx stepper requires identical motor tau / noise_ratio");
  }
  q.motor_lag = (float)m.motor_dt_over_tau[0];
  q.noise_ratio = (float)m.motor_noise_ratio[0];
  q.noise_loc = (float)m.n_motors;
  for (int k = 0; k < 3; ++k) q.drag_k[k] = (float)m.drag_const[k];
  q.drag_pqr = (float)m.drag_coef_pqr;
  const double T = 1.0 / m.control_hz;
  for (int w = 0; w < 6; ++w)
    for (int a = 0; a < 3; ++a) {
      q.pid[w][0][a] = (float)m.pid[w][0][a];
      q.pid[w][1][a] = (float)(m.pid[w][1][a] * T);
      q.pid[w][2][a] = (float)(m.pid[w][2][a] / T);
      q.pid[w][3][a] = (float)m.pid[w][3][a];
    }
  if (m.n_shapes > 5) return fail("quadx stepper supports at most 5 collision primitives, got %d", m.n_shapes);
  q.n_shapes = m.n_shapes;
  q.contact_zmax = -1e30f;
  for (int s = 0; s < m.n_shapes; ++s) {
    const PfbShape& sh = m.shapes[s];
    const double id[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (int k = 0; k < 9; ++k)
      if (sh.rot[k] != id[k]) return fail("quadx stepper requires axis-aligned collision primitives");
    q.shape_kind[s] = sh.kind;
    double disc;
    if (sh.kind == PFB_SHAPE_BOX) disc = sqrt(sh.dims[0] * sh.dims[0] + sh.dims[1] * sh.dims[1] + sh.dims[2] * sh.dims[2]);
    else if (sh.kind == PFB_SHAPE_CYLINDER) disc = sqrt(sh.dims[0] * sh.dims[0] + sh.dims[1] * sh.dims[1]);
    else disc = sh.dims[0];
    for (int k = 0; k < 3; ++k) { q.shape_dims[s][k] = (float)sh.dims[k]; q.shape_at[s][k] = (float)sh.at[k]; }
    q.shape_thr[s] = (float)(m.contact_factor * disc);
    {
      double reach = sqrt(sh.at[0] * sh.at[0] + sh.at[1] * sh.at[1] + sh.at[2] * sh.at[2]) + disc + m.contact_factor * disc;
      if ((float)(reach * 1.001) > q.contact_zmax) q.contact_zmax = (float)(reach * 1.001);
    }
  }
  q.ratio = (int)(m.physics_hz / m.control_hz);
  if (q.ratio < 1 || q.ratio > 4) return fail("physics_hz / control_hz must be in 1..4 (got %d)", q.ratio);
  {  // the exp-map series in quadx_substep needs (|w| dt / 2)^2 <= 0.25 with |w| <= sqrt(3) vmax
    double hmax = 0.5 * sqrt(3.0) * m.max_coord_velocity / m.physics_hz;
    if (hmax * hmax > 0.25) return fail("max_coord_velocity * dt too large for the attitude series (h^2 = %g)", hmax * hmax);
  }
  return 0;
}

