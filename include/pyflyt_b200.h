/*
 * pyflyt_b200.h — C-ABI of the H100-native batched UAV stepper.
 *
 * This is the drop-in boundary for the ONE hot path of jjshoots/PyFlyt that this project replaces:
 *   Aviary.step()                      PyFlyt/core/aviary.py:480-531
 *   QuadX/Fixedwing/Rocket.update_*    PyFlyt/core/drones/{quadx,fixedwing,rocket}.py
 *   Motors/BoringBodies/LiftingSurfaces/Boosters/Gimbals/PID   PyFlyt/core/abstractions/
 *   PyBullet stepSimulation()          (third party; restated, see DESIGN.md)
 *   env epilogues (obs / reward / term) PyFlyt/gym_envs, PyFlyt/pz_envs
 *
 * The reference has no FFI on this path (it is Python on top of PyBullet's CPython module), so the
 * entry points below are what a maintainer would bind with ctypes from a new `Aviary` backend;
 * INTEGRATION.md shows that stub.  Rules of the boundary:
 *   - plain C types only; every buffer is a raw pointer + the sizes implied by the handle;
 *   - device buffers are OWNED BY THE CALLER (torch tensors on the Python side); the library owns
 *     only its constant model table and a few bytes of bookkeeping;
 *   - every call is asynchronous on the given CUDA stream and never synchronises the device;
 *   - every function returns 0 on success, <0 on error; pfb_last_error() gives the message
 *     (thread-local).  There is NO CPU fallback: without a CUDA device every compute entry fails.
 *
 * Layout convention: SoA, field-major.  A buffer documented as [F][N] holds field f of env i at
 * index f*N + i.  Row-major "API" buffers ([N][K]) are the shapes an RL trainer consumes.
 */
#ifndef PYFLYT_B200_H
#define PYFLYT_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PFB_ABI_VERSION 1

/* ---- vehicle kinds (reference: Aviary.drone_type_mappings, aviary.py:167-170) ------------------- */
#define PFB_KIND_QUADX 0
#define PFB_KIND_FIXEDWING 1
#define PFB_KIND_ROCKET 2

/* ---- env epilogues -------------------------------------------------------------------------------- */
#define PFB_ENV_NONE 0            /* Aviary-level stepping only                                        */
#define PFB_ENV_QUADX_HOVER 1     /* gym_envs/quadx_envs/quadx_hover_env.py                            */
#define PFB_ENV_QUADX_WAYPOINTS 2 /* gym_envs/quadx_envs/quadx_waypoints_env.py                        */
#define PFB_ENV_FIXEDWING_WAYPOINTS 3
#define PFB_ENV_ROCKET_LANDING 4
#define PFB_ENV_DOGFIGHT 5
#define PFB_ENV_MA_QUADX_HOVER 6 /* pz_envs/quadx_envs/ma_quadx_hover_env.py: per-AGENT epilogue (observation with past
                                   * action + start position, rewards summed over the Aviary steps of an env step);
                                   * the arena bookkeeping (who is still alive, reset when all are done) is host-side */

#define PFB_MAX_MOTORS 4
#define PFB_MAX_SURFACES 5
#define PFB_MAX_SHAPES 16
/* Distinct vehicle tables one QuadX handle can fly at once (pfb_set_models).  The K tables travel as ONE kernel argument of
 * K x 640 bytes (fp32 tables), so the cap keeps that argument at 10 KB, well inside the 32 KB kernel-argument limit.      */
#define PFB_MAX_QUADX_MODELS 16

#define PFB_SHAPE_BOX 0
#define PFB_SHAPE_CYLINDER 1
#define PFB_SHAPE_SPHERE 2

/* Static (fixed-base) bodies per Aviary handle, and their collision primitives in all (pfb_add_static_body) */
#define PFB_MAX_STATIC_BODIES 8
#define PFB_MAX_STATIC_SHAPES 16

/* One collision primitive used for the ground / pad contact FLAG (no contact response). */
typedef struct PfbShape {
  int32_t kind;
  int32_t _pad;
  double dims[3]; /* box: half extents; cylinder: radius, half length, -; sphere: radius            */
  double at[3];   /* centre, base inertial frame                                                     */
  double rot[9];  /* row-major rotation of the primitive in the base frame                           */
} PfbShape;

/* One lifting surface (abstractions/lifting_surfaces.py:180-264 precomputed on the host). */
typedef struct PfbSurface {
  double pos[3];        /* link COM in the base frame (point of application)                         */
  double lift_unit[3];
  double drag_unit[3];
  double torque_unit[3];
  double Cl_alpha_3D, aspect, flap_to_chord, aero_tau, eta;
  double alpha_0_base, alpha_stall_P_base, alpha_stall_N_base; /* radians                            */
  double Cd_0, deflection_limit_deg, dt_over_tau, area, chord, half_rho;
} PfbSurface;

/* Host-side, double-precision vehicle table; the library narrows it to fp32 once at pfb_create.     */
typedef struct PfbModel {
  int32_t abi_version;
  int32_t kind;
  double physics_hz;        /* 240 (aviary.py:79)                                                    */
  double control_hz;        /* 120 (quadx.py:27, fixedwing.py:23, rocket.py:35)                      */
  double gravity;           /* -9.81 (aviary.py:226)                                                 */
  double max_coord_velocity;/* 100, btMultiBody::m_maxCoordinateVelocity                             */

  /* composite rigid body about the base origin, base axes (all joints are fixed) */
  double mass;
  double com[3];
  double inertia[9];        /* row-major, about the base origin                                      */

  /* contact flag */
  int32_t n_shapes;
  int32_t _pad0;
  PfbShape shapes[PFB_MAX_SHAPES];
  double contact_factor;    /* 0.02: relative breaking threshold × primitive bounding radius         */

  /* propeller motors (abstractions/motors.py) */
  int32_t n_motors;
  int32_t _pad1;
  double motor_pos[PFB_MAX_MOTORS][3];
  double motor_axis[PFB_MAX_MOTORS][3];
  double thrust_coef[PFB_MAX_MOTORS];
  double torque_coef[PFB_MAX_MOTORS];
  double max_rpm[PFB_MAX_MOTORS];
  double motor_dt_over_tau[PFB_MAX_MOTORS];
  double motor_noise_ratio[PFB_MAX_MOTORS];

  /* body drag (abstractions/boring_bodies.py) + quad rotational drag (quadx.py:502-510) */
  int32_t n_bodies;
  int32_t _pad2;
  double body_pos[3];
  double drag_const[3];     /* 0.5 * 1.225 * Cd * A, per link axis                                   */
  double drag_coef_pqr;

  /* QuadX PID gains (quadx.py:153-197).  index: 0 ang_vel, 1 ang_pos, 2 lin_vel, 3 lin_pos,
   * 4 z_vel, 5 z_pos;  second index: kp, ki, kd, lim;  third: axis.                                 */
  double pid[6][4][3];
  double motor_map[4][4];   /* quadx.py:130-137                                                      */

  /* lifting surfaces (fixedwing: 5, rocket finlets: 4) */
  int32_t n_surfaces;
  int32_t _pad3;
  PfbSurface surfaces[PFB_MAX_SURFACES];

  /* booster + gimbal + fuel tank (rocket; abstractions/boosters.py, gimbals.py) */
  int32_t has_booster;
  int32_t reignitable;
  double booster_pos[3];
  double booster_axis[3];
  double booster_dt_over_tau, booster_noise_ratio;
  double booster_min_thrust, booster_max_thrust;
  double fuel_total_mass, fuel_max_rate;
  double fuel_max_inertia[3];
  double fuel_pos[3];
  double dry_mass;           /* composite without the fuel tank link                                 */
  double dry_first_moment[3];/* sum m_i r_i without the tank                                         */
  double dry_inertia[9];     /* about the base origin, without the tank                              */
  double gimbal_unit1[3], gimbal_unit2[3];
  double gimbal_dt_over_tau;
  double gimbal_range_rad[2];
  double starting_fuel_ratio;
  double starting_velocity[3]; /* fixedwing.py:35,201                                                */
} PfbModel;

/* PfbEnvConfig.autoreset: what pfb_env_step does with an env that terminates or truncates on call k.
 *   NONE       nothing: the caller resets it (pfb_env_reset with a mask)
 *   NEXT_STEP  call k + 1 is its reset: the action is ignored, obs is the first observation of the new episode, reward 0,
 *              both flags 0 (gymnasium's AutoresetMode.NEXT_STEP)
 *   SAME_STEP  call k resets it too: reward, term, trunc and info are the terminal step's, the terminal observation goes to
 *              row i of PfbBuffers.final_obs and obs holds the first observation of the new episode; call k + 1 steps it with
 *              the caller's action (gymnasium's AutoresetMode.SAME_STEP).  QuadX-Hover, QuadX-Waypoints,
 *              Fixedwing-Waypoints and Rocket-Landing only; pfb_env_step_host / pfb_env_step_mapped refuse such a handle.
 * Autoreset episode e of env i starts from the same state in both modes: its warm-up is keyed by (seed, global env id, e).
 * pfb_create refuses any other value. */
#define PFB_AUTORESET_NONE 0
#define PFB_AUTORESET_NEXT_STEP 1
#define PFB_AUTORESET_SAME_STEP 2

/* Env-epilogue constants (gym_envs/quadx_envs/quadx_hover_env.py:29-38 and friends). */
typedef struct PfbEnvConfig {
  int32_t env_kind;          /* PFB_ENV_*                                                            */
  int32_t flight_mode;       /* quadx.py:233-245                                                     */
  int32_t env_step_ratio;    /* 120 / agent_hz                                                       */
  int32_t max_steps;         /* agent_hz * max_duration_seconds                                      */
  int32_t angle_representation; /* 0 euler, 1 quaternion                                             */
  int32_t sparse_reward;
  int32_t autoreset;         /* PFB_AUTORESET_*: 0 none, 1 NEXT_STEP (gymnasium's default), 2 SAME_STEP */
  int32_t warmup_steps;      /* 10 Aviary steps after reset (quadx_base_env.py:209-210)              */
  double flight_dome_size;
  double goal_reach_distance, goal_reach_angle;  /* waypoint envs                                    */
  int32_t num_targets, use_yaw_targets;
  /* Rocket-Landing (gym_envs/rocket_envs/rocket_landing_env.py:33-67, rocket_base_env.py:192-226) */
  double ceiling, max_displacement;
  int32_t randomize_drop, accelerate_drop;
  /* MAFixedwingDogfight (pz_envs/fixedwing_envs/ma_fixedwing_dogfight_env.py:42-62): an arena is
   * 2*team_size CONSECUTIVE envs of the batch; the first team_size of them are team 0                 */
  int32_t team_size;
  int32_t inline_reset;      /* autoreset: 0 = copy the env's spare post-reset state; 1 = integrate every warm-up inside the
                              * step launch instead (same results, longer launches; tests).  pfb_create refuses other values */
  double damage_per_hit, lethal_distance, lethal_angle, aggressiveness, cooperativeness;
  double spawn_min_radius, spawn_max_radius, spawn_min_height, spawn_max_height;
  int32_t contact_response;  /* 1 = ground / pad contact RESPONSE (sequential-impulse normal + Coulomb friction on the collision
                              * primitives' corner / rim points; a restatement, see DESIGN.md), 0 = contact FLAG only.  Read by
                              * Rocket-Landing (a gentle touchdown rests on the pad and reaches env_complete,
                              * rocket_landing_env.py:231-263) and by Aviary handles (env_kind PFB_ENV_NONE: QuadX, fixed-wing and
                              * rocket drones land on, slide along and rest on the floor).  pfb_create reads no other field of a
                              * PFB_ENV_NONE config.  The other env kinds ignore it (they terminate on the first contact).         */
  int32_t mixed_control_hz;  /* 1 = the tables passed to pfb_create_mixed may differ in control_hz (see there).  Read only by
                              * pfb_create_mixed from its PFB_ENV_NONE aviary_cfg; pfb_create and the env kinds ignore it.         */
} PfbEnvConfig;

/* Analytic, time-invariant wind field evaluated IN-KERNEL at every drag body / lifting surface (SURVEY.md 8f item 4).
 * Replaces the Python callback of Aviary.register_wind_field_function (aviary.py:324-334, "for less complicated wind
 * field models (time invariant models)"), which the reference evaluates at each link COM in BoringBodies.state_update
 * (boring_bodies.py:93-96) and LiftingSurfaces.state_update (lifting_surfaces.py:88-93):
 *      wind(x, y, z) = base * f(z)
 *   PFB_WIND_CONSTANT  f = 1
 *   PFB_WIND_POWER     f = (max(z, 0) / z_ref) ^ alpha            (atmospheric power law)
 *   PFB_WIND_LOG       f = ln(max(z, z0) / z0) / ln(z_ref / z0)   (logarithmic boundary layer, 0 below z0)
 *   PFB_WIND_EXP       f = exp(z / z_ref)                          (the field of the reference's tests/test_core.py:275-278)
 * pyflyt_b200.core.wind.AnalyticWind is the same function as a Python callable: hand it to the reference's
 * register_wind_field_function and to BatchedAviary.register_wind_field to fly both in the same air.              */
#define PFB_WIND_NONE 0
#define PFB_WIND_CONSTANT 1
#define PFB_WIND_POWER 2
#define PFB_WIND_LOG 3
#define PFB_WIND_EXP 4
typedef struct PfbWind {
  int32_t kind;
  int32_t _pad;
  double base[3];  /* m/s, world frame */
  double z_ref;
  double alpha;
  double z0;
} PfbWind;

/* Caller-owned DEVICE buffers.  Any pointer may be NULL if the env kind does not use it. */
typedef struct PfbBuffers {
  /* persistent state, fp32 SoA [F][N]; row map is fixed per vehicle kind: see pfb_state_rows()      */
  float* state;
  int32_t* istate;           /* [I][N] int32: step_count, flags, episode counter, ...                */
  /* inputs */
  float* setpoint;           /* [N][S] row-major (S = pfb_setpoint_dim); the caller writes actions /
                              * setpoints here, pfb_reset / pfb_set_mode preset it like the reference  */
  const float* start_pos;    /* [N][3]                                                               */
  const float* start_orn;    /* [N][3] euler                                                         */
  const float* reset_targets;/* [N][3*num_targets] waypoints to install on env reset (nullable: drawn on
                              * device like WaypointHandler.reset, waypoint_handler.py:53-83)          */
  /* outputs of pfb_env_step */
  float* obs;                /* [N][O] row-major                                                     */
  float* reward;             /* [N]                                                                  */
  uint8_t* term;             /* [N]                                                                  */
  uint8_t* trunc;            /* [N]                                                                  */
  uint8_t* info;             /* [N] bit0 out_of_bounds, bit1 collision, bit2 env_complete            */
  float* final_obs;          /* [N][O] SAME_STEP autoreset: row i = terminal observation of env i when it
                              * finished on the last pfb_env_step (other rows untouched); mandatory there,
                              * unused otherwise (NEXT_STEP returns the terminal obs in obs itself)       */
  /* outputs of pfb_observe_state (Aviary.state / aux_state) */
  float* drone_state;        /* [N][12] = state(i) (4,3) flattened: ang_vel_b, euler, lin_vel_b, pos */
  float* aux_state;          /* [N][A]                                                               */
  uint8_t* contact;          /* [N] any ground contact during the last Aviary.step()                 */
} PfbBuffers;

typedef struct PfbContext* PfbHandle;

/* ---- lifecycle ---------------------------------------------------------------------------------- */
const char* pfb_last_error(void);
int pfb_abi_version(void);
int pfb_sizeof_model(void);
int pfb_sizeof_env_config(void);
int pfb_sizeof_buffers(void);

/* Vehicle table from the reference's model files: `<model>.urdf` (fixed joints only; what p.loadURDF(...,
 * URDF_USE_INERTIA_FROM_FILE) reads, base_drone.py:104-122) + `<model>.yaml` (the parameter file the drone constructors read:
 * quadx.py:84-197, fixedwing.py:70-166, rocket.py:82-208, lifting_surfaces.py:180-264).  kind = PFB_KIND_*; physics_hz /
 * control_hz <= 0 select the reference defaults (240 / 120).  Host-only, no CUDA device needed.  Constructor options of the
 * reference (`starting_velocity`, `starting_fuel_ratio`) are left at their defaults: overwrite the fields afterwards.     */
int pfb_model_from_files(int kind, const char* urdf_path, const char* yaml_path, double physics_hz, double control_hz, PfbModel* out);

/* Replaces Aviary.__init__ (aviary.py:69-216) for n_envs independent single-drone worlds. */
int pfb_create(const PfbModel* model, const PfbEnvConfig* env, int64_t n_envs, int device, uint64_t seed,
               PfbHandle* out);
int pfb_destroy(PfbHandle h);
/* Aviary(drone_type=[...]) with drones of several kinds (aviary.py:139-190): drone i flies models[model_index[i]] (host array
 * of n entries, each < k).  Every table has the same physics_hz and control_hz; at most PFB_MAX_QUADX_MODELS QuadX tables,
 * one fixed-wing and one rocket table.  aviary_cfg: NULL, or a PFB_ENV_NONE config of which only contact_response and
 * mixed_control_hz are read.
 * With aviary_cfg->mixed_control_hz = 1 the tables may differ in control_hz (the reference's Aviary with per-drone
 * drone_options control_hz, aviary.py:287-298, 506-529): every table has the same physics_hz, which each control_hz divides;
 * sorted, each distinct rate is a multiple of the one before; U = physics_hz / min(control_hz) is in 1..4.  A QuadX table is
 * one (model, rate) pair (its PIDs use the control period); several fixed-wing, or rocket, tables must be byte-equal apart
 * from control_hz (one model at several rates), and two identical tables are refused.  One pfb_aviary_step step is then U
 * physics substeps u = 0..U-1 for every drone; drone i, with r_i = physics_hz / control_hz_i, runs its control tick before
 * substep u when u % r_i == 0.  Injected noise is [n_steps * U][N] (one draw per drone per substep, whatever its rate);
 * Philox draws are keyed by (seed, i, Aviary step, substep).  If every table has the same control_hz, the flag changes nothing.
 * The handle is an Aviary handle (the env entry points and pfb_set_models refuse it) with:
 *   state     pfb_state_floats() floats, carved by the library into one region per kind (PFB_LAYOUT_BY_KIND): QuadX
 *             warp-tiled, then fixed-wing and rocket field-major, each on a 128-byte boundary; istate [pfb_istate_rows][N];
 *   setpoint  [N][7] (pfb_setpoint_dim): drone i reads its own length (QuadX 4, fixed-wing 6, rocket 7), the rest is zero
 *             after pfb_reset / pfb_set_mode;
 *   aux_state [N][9] (pfb_aux_dim), zero past the drone's own aux length (QuadX 4, fixed-wing 6, rocket 9);
 *   obs       [N][6] (pfb_obs_dim): pfb_observe_state writes the hi and lo fp32 words of each drone's position there.
 * pfb_aviary_step steps every kind in ONE launch.  Drone i draws the noise drone i of a single-kind handle with the same seed
 * draws (Philox stream of env id i, column i of injected noise), so its trajectory is that drone's in such a handle.       */
int pfb_create_mixed(const PfbModel* models, int k, const uint8_t* model_index, int64_t n, const PfbEnvConfig* aviary_cfg, int device,
                     uint64_t seed, PfbHandle* out);
/* env.reset(seed=s) of the reference re-creates np_random: the same seed must give the same episodes.  Re-keys the Philox
 * streams and rewinds every call counter (step / reset / Aviary step numbers, autoreset episode numbers), stream-ordered on
 * `stream`.  It invalidates the spare post-reset states (they hold warm-ups of the old streams): an env handle must follow it
 * with a full pfb_env_reset (mask = NULL), which rebuilds them; an Aviary handle with pfb_reset.                         */
int pfb_reseed(PfbHandle h, uint64_t seed, void* stream);
/* Global index of this handle's env 0 (rank * n_envs when the batch is sharded over GPUs): keeps
 * the Philox streams, and therefore every trajectory, independent of the number of ranks.  Call it before the first
 * pfb_env_reset: the spare post-reset states are keyed to the env ids they were built for.          */
int pfb_set_env_offset(PfbHandle h, uint64_t first_global_env);

/* Several vehicle models in one QuadX handle (Aviary(drone_options=[...]) with one dict per drone, aviary.py:75,196-199):
 * installs k QuadX tables and env i flies models[index_host[i]] (host array of n_envs entries, each < k).  Every table must
 * be QuadX with the same physics_hz and control_hz (one substep ratio per handle), 1 <= k <= PFB_MAX_QUADX_MODELS.  k = 1
 * makes the handle uniform again (the same kernels as a handle created with that table).  An analytic wind set with
 * pfb_set_wind reaches every table, before or after this call.  Not for MAQuadXHover handles.  A set-up call like
 * pfb_create: it synchronises the device, and it invalidates the spare post-reset states; follow it with pfb_env_reset.   */
int pfb_set_models(PfbHandle h, const PfbModel* models, int k, const uint8_t* index_host);

/* Aviary.register_wind_field_function for an analytic field (NULL or kind PFB_WIND_NONE: still air).  Takes effect from the
 * next call on; every vehicle kind.  PFB_WIND_POWER needs alpha >= 0; alpha = 0 is stored as PFB_WIND_CONSTANT (0^0 = 1).
 * On an env handle that keeps spare post-reset states (autoreset), a field that differs from the current one costs a device
 * synchronisation: every spare is marked invalid, so that each env's next reset integrates its warm-up in the new air,
 * under the same episode number, and the spares are rebuilt from there on (the spare and inline_reset paths stay equal).  */
int pfb_set_wind(PfbHandle h, const PfbWind* wind);
int pfb_sizeof_wind(void);

/* Shapes the caller must allocate. */
int pfb_state_rows(PfbHandle h);     /* F of PfbBuffers.state                                         */
/* Layout of PfbBuffers.state.  FIELD_MAJOR: [F][N], word (row r, env i) at r*N + i (fixed-wing, rocket, QuadX-Waypoints).
 * WARP_TILED (every other QuadX handle): env i lives in tile i/32, lane i%32; a tile is F/4 groups of 32 lanes x 4 words:
 * word (r, i) at (((i/32) * (F/4) + r/4) * 32 + i%32) * 4 + r%4.  A warp moves a group with one 128-bit access per lane,
 * and the rows an env step touches are one contiguous block per tile.  pfb_state_floats() is the number of floats to
 * allocate (tiles are padded to 32 envs); step_count and the flag word live in rows 17 / 18 of the tile as int32 bits.  */
#define PFB_LAYOUT_FIELD_MAJOR 0
#define PFB_LAYOUT_WARP_TILED 1
#define PFB_LAYOUT_BY_KIND 2 /* a mixed-kind handle (pfb_create_mixed): one region per vehicle kind, in that kind's layout */
int pfb_state_layout(PfbHandle h);
int64_t pfb_state_floats(PfbHandle h);
int pfb_istate_rows(PfbHandle h);    /* I of PfbBuffers.istate                                        */
int pfb_setpoint_dim(PfbHandle h);   /* S                                                             */
int pfb_obs_dim(PfbHandle h);        /* O                                                             */
int pfb_aux_dim(PfbHandle h);        /* A                                                             */
int pfb_bind(PfbHandle h, const PfbBuffers* buffers);

/* ---- Aviary surface ------------------------------------------------------------------------------ */
/* Aviary.reset + drone.reset + update_state (aviary.py:218-312, quadx.py:222-231).  mask: device
 * [N] uint8, NULL = all envs.  Poses come from the bound start_pos/start_orn.                        */
int pfb_reset(PfbHandle h, const uint8_t* mask, void* stream);
/* Aviary.set_mode (aviary.py:440-458, quadx.py:233-373): same mode for every env; resets the PIDs
 * and presets the bound setpoint buffer rows exactly like the reference.                             */
int pfb_set_mode(PfbHandle h, int mode, void* stream);
/* Aviary.set_mode(list) (aviary.py:440-458): env i gets QuadX/Fixedwing.set_mode(modes[i]), with the setpoint preset and
 * PID reset of its new mode; modes is a host array of n_envs entries.  Aviary handles only (created without an env
 * epilogue).  Ranges: QuadX -1..7, fixed-wing -1..0, rocket 0.  All entries equal: exactly pfb_set_mode(h, modes[0]).
 * Otherwise the following pfb_aviary_step calls fly each env in its own mode, until pfb_set_mode or an unmasked
 * pfb_reset returns the handle to one mode (a masked reset keeps the modes).  Envs 32k .. 32k+31 share a warp: a batch
 * steps fastest when each such tile flies one mode.                                                                      */
int pfb_set_modes(PfbHandle h, const int8_t* modes, void* stream);
/* n_steps × Aviary.step() (aviary.py:480-531).  noise: device [n_steps*updates_per_step][N] raw
 * draws of np_random.normal(*throttle.shape) (motors.py:134-138), or NULL → on-device Philox.        */
int pfb_aviary_step(PfbHandle h, int n_steps, const float* noise, void* stream);
/* p.resetBaseVelocity for every drone (gym_envs/rocket_envs/rocket_base_env.py:228): device [N][3] world-frame linear and
 * angular velocities, fp32.  Every Aviary handle (single-kind or mixed) and Rocket-Landing handles; the body rate the state
 * carries is R^T w in fp32.  The other env handles refuse it.                                                              */
int pfb_set_base_velocity(PfbHandle h, const float* lin_vel, const float* ang_vel, void* stream);
/* p.resetBasePositionAndOrientation(pos, quat) and / or p.resetBaseVelocity(lin_vel, ang_vel), then drone.update_state(), for
 * the drones of `mask` (device [N] uint8, NULL = every drone).  Device fp64 arrays in user drone order: pos [N][3], quat
 * [N][4] (x, y, z, w), lin_vel / ang_vel [N][3], world frame; NULL = not given.  pos and quat come together or not at all.
 * A pose zeroes both velocities, then the velocities given replace them; an input not given keeps its value.  Position,
 * quaternion and velocity land in the hi / lo state words; the angular velocity is stored as the body rate R^T w of the
 * drone's (new) attitude.  Everything else (flags incl. contact, controller memories, actuators, fuel, gimbal, setpoints,
 * flight modes, model index, step count) is kept.  Aviary handles only (single-kind or mixed): env handles refuse it.      */
int pfb_set_base_state(PfbHandle h, const uint8_t* mask, const double* pos, const double* quat, const double* lin_vel, const double* ang_vel,
                       void* stream);
/* getBasePositionAndOrientation / getBaseVelocity of every drone, in user order, into device fp64 arrays (NULL = not wanted):
 * pos [N][3], quat [N][4] (x, y, z, w) and lin_vel [N][3] are the hi + lo sums of the state words, ang_vel [N][3] the world
 * rate R w_body.  Aviary handles only.                                                                                      */
int pfb_get_base_state(PfbHandle h, double* pos, double* quat, double* lin_vel, double* ang_vel, void* stream);
/* Fills drone_state / aux_state / contact (Aviary.state(i), aux_state(i), contact_array).            */
int pfb_observe_state(PfbHandle h, void* stream);

/* ---- static bodies (DESIGN.md §4h): the reference's loadURDF(..., useFixedBase=True) of a landing pad, a helipad or a
 * rooftop.  Aviary handles only.  A body is 1..PFB_MAX_STATIC_SHAPES boxes and cylinders (PfbShape: `at` / `rot` in the
 * body's base link frame; box half extents, cylinder radius and half length), each upright once posed (a box may be yawed,
 * a cylinder's axis is vertical) unless the handle is solid (pfb_set_static_solid), which takes any orientation.  Every drone's world holds its own copy of each body.  A primitive is UNDER drone i when
 * its footprint holds the base's (x, y) and z + R_b >= its top (R_b: the model's contact reach); the contact flag of a body
 * is the drone's flag against the top of each primitive under it, and the contact response (contact_response) runs against
 * the highest surface under the drone (the floor, z = 0, or a top).  This top-face rule is the default: side faces are not
 * solid unless pfb_set_static_solid turns on the solid rule.  pfb_reset with mask = NULL removes every static body
 * (Aviary.reset calls resetSimulation).                                                                                  */
typedef PfbShape PfbStaticShape;
/* Reads the collision primitives of a URDF (fixed joints; boxes, cylinders, spheres) in its base link frame, scaled by
 * global_scaling, and the origin of the base link's inertial frame in that frame (which may be offset, not rotated).
 * *n_shapes = their number; at most `cap` are written (more: an error).  Meshes are refused.                           */
int pfb_static_shapes_from_urdf(const char* urdf_path, double global_scaling, PfbStaticShape* out, int cap, int* n_shapes,
                                double inertial_origin[3]);
/* loadURDF(useFixedBase=True): adds body *body_id = 0, 1, ... to every drone's world with its base LINK frame at pos[3],
 * quat[4] (x, y, z, w; host fp64; upright, or any unit quaternion on a solid handle).  inertial_origin[3] (NULL = 0): the base inertial frame in the link frame, which
 * pfb_set_static_pose places.                                                                                           */
int pfb_add_static_body(PfbHandle h, const PfbStaticShape* shapes, int n_shapes, const double pos[3], const double quat[4],
                        const double inertial_origin[3], int* body_id, void* stream);
/* resetBasePositionAndOrientation of static body `body` in the worlds of the drones of `mask` ([N], NULL = all): device fp64
 * pos [N][3], quat [N][4] (x, y, z, w) of its base INERTIAL frame, as PyBullet's reset places it.  Every quaternion of a
 * drone in the mask must be upright (a yaw about z: 1 - R22 <= 1e-9), else the call fails and changes nothing; a solid handle
 * takes any unit quaternion (the link frame is at pos - R o, R the full rotation).  The check reads the quaternions back to
 * the host: this call synchronises `stream`.                                              */
int pfb_set_static_pose(PfbHandle h, int body, const double* pos, const double* quat, const uint8_t* mask, void* stream);
/* bits[i] (device [N]): what drone i touched during the last pfb_aviary_step, bit 0 the floor, bit 1 + k static body k;
 * zero from the first body added after a full pfb_reset until the next step.                                            */
int pfb_get_static_contacts(PfbHandle h, uint32_t* bits, void* stream);
/* solid = 1: every static primitive is a solid on all of its faces, edges and corners (DESIGN.md §4h, "solid static
 * bodies").  Each candidate point of the drone's collision primitives (8 per box or cylinder) takes the deepest of the floor
 * and the primitives that hold it, with that face's normal, for the contact response; bit 1 + k is set when a candidate point
 * lies inside a primitive of body k grown on every face by the contact threshold.  solid = 0 (the default): the top-face rule
 * above.  A property of the handle: pfb_reset keeps it, and it takes effect at the next pfb_aviary_step.  Aviary handles only;
 * solid must be 0 or 1.  A solid handle takes tilted bodies, primitives and poses (pfb_add_static_body, pfb_set_static_pose);
 * solid = 0 fails while it holds one (until a full pfb_reset).  solid = 1 on a handle that already holds bodies enqueues the
 * fill of their full poses on `stream`.                                                                                   */
int pfb_set_static_solid(PfbHandle h, int solid, void* stream);

/* ---- gymnasium-env surface ----------------------------------------------------------------------- */
/* env.reset(): begin_reset + end_reset (quadx_base_env.py:149-212): pose reset, set_mode, warm-up
 * Aviary steps, first observation.  mask NULL = all.                                                 */
int pfb_env_reset(PfbHandle h, const uint8_t* mask, const float* noise, void* stream);
/* env.step(action) for all envs (quadx_base_env.py:269-301): actions device [N][S] (NULL = the bound
 * setpoint buffer); writes obs / reward / term / trunc / info.                                       */
int pfb_env_step(PfbHandle h, const float* actions, const float* noise, void* stream);
/* Synthetic rollout: n_steps env.step() calls with actions drawn on device (uniform in the env's action box) — "synthetic
 * random-action rollouts" of BASELINE.json.  QuadX-Hover with autoreset runs n_steps >= 4 as FUSED launches of up to 16 env
 * steps (the state stays in registers across the steps; every step's observations, rewards, flags and drawn actions are still
 * written, so afterwards the bound buffers hold the results of the last step, as after n_steps single calls); every other
 * case is one launch per step.  Single steps and fused rollouts can be mixed freely on one handle.                            */
int pfb_env_rollout(PfbHandle h, int n_steps, void* stream);

/* Host-buffer convenience used for the end-to-end measurement: H2D(actions) → pfb_env_step →
 * D2H(obs, reward, term, trunc).  Host pointers should be pinned.  If obs | reward | term | trunc are laid out back to
 * back both in the bound device buffers and in the host pointers, they are returned with a single copy.   */
int pfb_env_step_host(PfbHandle h, const float* host_actions, float* host_obs, float* host_reward,
                      uint8_t* host_term, uint8_t* host_trunc, void* stream);

/* Zero-copy flavour of the same call: the step kernel reads the actions from and writes obs / reward / term / trunc straight
 * into the caller's PINNED host buffers (device-mapped under UVA), so the PCIe traffic overlaps the launch instead of
 * bracketing it with two copies.  Same results, same bytes over the bus.                                              */
int pfb_env_step_mapped(PfbHandle h, const float* host_actions, float* host_obs, float* host_reward,
                        uint8_t* host_term, uint8_t* host_trunc, void* stream);

/* ---- MAFixedwingDogfight with an arena's agents on DIFFERENT ranks (ma_fixedwing_dogfight_env.py:346-465):
 * global agent id = member * num_arenas + arena; this handle owns ids [first_global_agent, +n_envs).  Per Aviary
 * step the caller runs  pfb_dogfight_physics -> all-gather of the payload table (NCCL) -> pfb_dogfight_combat.
 *   physics: integrates one Aviary step (or, with do_reset, the reset + warm-up) and writes
 *            payload_out [n_envs][pfb_dogfight_payload_dim()]; `first` = this is the first Aviary step of an
 *            env.step (actions are latched), `aviary_index` = 0..env_step_ratio-1 (noise stream position);
 *   combat:  payload_table [num_arenas*2][dim] gathered from every rank; `last` = 1 on the last Aviary step of
 *            the env.step (writes obs / reward / term / trunc / info), 2 after a reset (obs only), else 0. */
int pfb_dogfight_payload_dim(void);
int pfb_dogfight_physics(PfbHandle h, const float* actions, const float* noise, float* payload_out, int first, int do_reset,
                         int aviary_index, void* stream);
/* Fused exchange: as pfb_dogfight_physics, but every payload is stored straight into the payload table of EVERY rank
 * (peer_tables_dev: DEVICE array of `world` table base pointers, peer-mapped, e.g. torch symmetric memory) at float offset
 * slot_offset_floats + 20 * local_agent.  No all-gather: the caller follows with a cross-rank barrier on the stream.
 * With peer_flags_dev (DEVICE array of `world` peer-mapped int32[world] flag arrays, zero-initialised) the kernel also
 * signals: when all of its peer stores are fenced it writes `epoch` into entry `rank` of every rank's flag array, and
 * pfb_dogfight_combat_wait spins on its own array until all `world` entries have reached `epoch` — no barrier launch.
 * `epoch` must increase by one per exchange.  peer_flags_dev = NULL: no signalling (the caller barriers).               */
int pfb_dogfight_physics_peer(PfbHandle h, const float* actions, const float* noise, const uint64_t* peer_tables_dev, int world,
                             int64_t slot_offset_floats, const uint64_t* peer_flags_dev, int rank, int epoch, int first, int do_reset,
                             int aviary_index, void* stream);
/* One whole env step (env_step_ratio x physics_peer + combat_wait) in a single call: with in-kernel signalling nothing
 * between the kernels needs the host.  local_tables: this rank's [2][2*num_arenas][20] table, local_flags: its int32[world]
 * flag array; epoch0: number of the step's first exchange (1-based, continuing the count of all earlier exchanges).       */
int pfb_dogfight_split_step(PfbHandle h, const float* actions, const uint64_t* peer_tables_dev, const uint64_t* peer_flags_dev,
                            const float* local_tables, const int32_t* local_flags, int world, int rank, int epoch0,
                            int64_t first_global_agent, int64_t num_arenas, void* stream);
int pfb_dogfight_combat_wait(PfbHandle h, const float* payload_table, int64_t first_global_agent, int64_t num_arenas, int last,
                             const int32_t* flags, int world, int epoch, void* stream);
int pfb_dogfight_combat(PfbHandle h, const float* payload_table, int64_t first_global_agent, int64_t num_arenas, int last,
                        void* stream);
/* Test / audit aid: device buffer [env_step_ratio * updates_per_step][N] (or NULL = off) that receives every motor-noise
 * draw the QuadX-Hover step kernel hands out on the following pfb_env_step calls (overwritten per call): lets a test replay
 * the Philox stream of the timed instantiation through the CPU oracle.                                                  */
int pfb_set_noise_dump(PfbHandle h, float* dump);
/* Number of kernel launches issued by this handle so far (bench.py's gpu_launches).                  */
int64_t pfb_launch_count(PfbHandle h);
/* Measurement aid: record a CUDA-event pair around the dominant kernel of each of the next
 * `capacity` pfb_env_step calls (0 = off); pfb_profile_read returns how many pairs were filled and
 * their durations in ms (call after synchronising the stream).                                       */
int pfb_profile_begin(PfbHandle h, int capacity);
int pfb_profile_read(PfbHandle h, float* ms_out, int capacity);

#ifdef __cplusplus
}
#endif
#endif /* PYFLYT_B200_H */
