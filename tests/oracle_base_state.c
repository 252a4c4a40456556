/* TEST INFRASTRUCTURE — the fp64 oracle (oracle/pfb_oracle.c, included unchanged) plus the base-state reset of a script on top
 * of the reference's Aviary: p.resetBasePositionAndOrientation (fakebullet: the pose, then zero base velocities) and / or
 * p.resetBaseVelocity, then drone.update_state(), for the drones of `mask` (NULL = every drone).  pos [n][3], quat [n][4]
 * (x, y, z, w), lin / ang [n][3] world frame; NULL = not given (pos and quat together).  The contact state of the last step is
 * kept, as getContactPoints reports it until the next stepSimulation.  Built by tests/test_base_state.py with the oracle's
 * flags (oracle/Makefile). */
#include "../oracle/pfb_oracle.c"

void orc_set_base_state(OrcContext* ctx, const uint8_t* mask, const double* pos, const double* quat, const double* lin, const double* ang) {
  for (int64_t i = 0; i < ctx->n; ++i) {
    if (mask && !mask[i]) continue;
    OrcDrone* d = &ctx->d[i];
    if (pos) {
      for (int k = 0; k < 3; ++k) { d->pos[k] = pos[3 * i + k]; d->v[k] = 0.0; d->w[k] = 0.0; }
      for (int k = 0; k < 4; ++k) d->quat[k] = quat[4 * i + k];
    }
    if (lin) for (int k = 0; k < 3; ++k) d->v[k] = lin[3 * i + k];
    if (ang) for (int k = 0; k < 3; ++k) d->w[k] = ang[3 * i + k];
    if (ctx->m.kind == PFB_KIND_QUADX) quadx_update_state(ctx, d);
    else if (ctx->m.kind == PFB_KIND_FIXEDWING) fixedwing_update_state(ctx, d);
    else rocket_update_state(ctx, d);
  }
}
