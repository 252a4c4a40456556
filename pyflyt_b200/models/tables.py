"""Vehicle coefficient tables: (link table, parameter dict) → ``PfbModel`` (include/pyflyt_b200.h).

The reference builds these numbers inside each drone's constructor from ``<model>.urdf`` +
``<model>.yaml`` (PyFlyt/core/drones/quadx.py:84-196, fixedwing.py:70-166, rocket.py:82-208); here the
same numbers are laid out once, on the host, in double precision, and narrowed to fp32 by the library.
"""

from __future__ import annotations

import ctypes as C
import math
import os

import numpy as np
import yaml

from .urdf import Link, composite_rigid_body, load_urdf_links

PFB_ABI_VERSION = 1
KIND_QUADX, KIND_FIXEDWING, KIND_ROCKET = 0, 1, 2
ENV_NONE, ENV_QUADX_HOVER, ENV_QUADX_WAYPOINTS, ENV_FIXEDWING_WAYPOINTS, ENV_ROCKET_LANDING, ENV_DOGFIGHT, ENV_MA_QUADX_HOVER = range(7)
AUTORESET_NONE, AUTORESET_NEXT_STEP, AUTORESET_SAME_STEP = range(3)  # PfbEnvConfig.autoreset (PFB_AUTORESET_*)
MAX_MOTORS, MAX_SURFACES, MAX_SHAPES = 4, 5, 16
SHAPE_IDS = {"box": 0, "cylinder": 1, "sphere": 2}

_VEHICLE_DIR = os.path.join(os.path.dirname(os.path.realpath(__file__)), "vehicles")

D3 = C.c_double * 3
D9 = C.c_double * 9


class PfbShape(C.Structure):
    _fields_ = [("kind", C.c_int32), ("_pad", C.c_int32), ("dims", D3), ("at", D3), ("rot", D9)]


class PfbSurface(C.Structure):
    _fields_ = [
        ("pos", D3),
        ("lift_unit", D3),
        ("drag_unit", D3),
        ("torque_unit", D3),
        ("Cl_alpha_3D", C.c_double),
        ("aspect", C.c_double),
        ("flap_to_chord", C.c_double),
        ("aero_tau", C.c_double),
        ("eta", C.c_double),
        ("alpha_0_base", C.c_double),
        ("alpha_stall_P_base", C.c_double),
        ("alpha_stall_N_base", C.c_double),
        ("Cd_0", C.c_double),
        ("deflection_limit_deg", C.c_double),
        ("dt_over_tau", C.c_double),
        ("area", C.c_double),
        ("chord", C.c_double),
        ("half_rho", C.c_double),
    ]


class PfbModel(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32),
        ("kind", C.c_int32),
        ("physics_hz", C.c_double),
        ("control_hz", C.c_double),
        ("gravity", C.c_double),
        ("max_coord_velocity", C.c_double),
        ("mass", C.c_double),
        ("com", D3),
        ("inertia", D9),
        ("n_shapes", C.c_int32),
        ("_pad0", C.c_int32),
        ("shapes", PfbShape * MAX_SHAPES),
        ("contact_factor", C.c_double),
        ("n_motors", C.c_int32),
        ("_pad1", C.c_int32),
        ("motor_pos", (C.c_double * 3) * MAX_MOTORS),
        ("motor_axis", (C.c_double * 3) * MAX_MOTORS),
        ("thrust_coef", C.c_double * MAX_MOTORS),
        ("torque_coef", C.c_double * MAX_MOTORS),
        ("max_rpm", C.c_double * MAX_MOTORS),
        ("motor_dt_over_tau", C.c_double * MAX_MOTORS),
        ("motor_noise_ratio", C.c_double * MAX_MOTORS),
        ("n_bodies", C.c_int32),
        ("_pad2", C.c_int32),
        ("body_pos", D3),
        ("drag_const", D3),
        ("drag_coef_pqr", C.c_double),
        ("pid", ((C.c_double * 3) * 4) * 6),
        ("motor_map", (C.c_double * 4) * 4),
        ("n_surfaces", C.c_int32),
        ("_pad3", C.c_int32),
        ("surfaces", PfbSurface * MAX_SURFACES),
        ("has_booster", C.c_int32),
        ("reignitable", C.c_int32),
        ("booster_pos", D3),
        ("booster_axis", D3),
        ("booster_dt_over_tau", C.c_double),
        ("booster_noise_ratio", C.c_double),
        ("booster_min_thrust", C.c_double),
        ("booster_max_thrust", C.c_double),
        ("fuel_total_mass", C.c_double),
        ("fuel_max_rate", C.c_double),
        ("fuel_max_inertia", D3),
        ("fuel_pos", D3),
        ("dry_mass", C.c_double),
        ("dry_first_moment", D3),
        ("dry_inertia", D9),
        ("gimbal_unit1", D3),
        ("gimbal_unit2", D3),
        ("gimbal_dt_over_tau", C.c_double),
        ("gimbal_range_rad", C.c_double * 2),
        ("starting_fuel_ratio", C.c_double),
        ("starting_velocity", D3),
    ]


class PfbEnvConfig(C.Structure):
    _fields_ = [
        ("env_kind", C.c_int32),
        ("flight_mode", C.c_int32),
        ("env_step_ratio", C.c_int32),
        ("max_steps", C.c_int32),
        ("angle_representation", C.c_int32),
        ("sparse_reward", C.c_int32),
        ("autoreset", C.c_int32),
        ("warmup_steps", C.c_int32),
        ("flight_dome_size", C.c_double),
        ("goal_reach_distance", C.c_double),
        ("goal_reach_angle", C.c_double),
        ("num_targets", C.c_int32),
        ("use_yaw_targets", C.c_int32),
        ("ceiling", C.c_double),
        ("max_displacement", C.c_double),
        ("randomize_drop", C.c_int32),
        ("accelerate_drop", C.c_int32),
        ("team_size", C.c_int32),
        ("inline_reset", C.c_int32),
        ("damage_per_hit", C.c_double),
        ("lethal_distance", C.c_double),
        ("lethal_angle", C.c_double),
        ("aggressiveness", C.c_double),
        ("cooperativeness", C.c_double),
        ("spawn_min_radius", C.c_double),
        ("spawn_max_radius", C.c_double),
        ("spawn_min_height", C.c_double),
        ("spawn_max_height", C.c_double),
        ("contact_response", C.c_int32),
        ("mixed_control_hz", C.c_int32),
    ]


# --------------------------------------------------------------------------------------------------
# vehicle files
# --------------------------------------------------------------------------------------------------
def load_vehicle(drone_model: str, model_dir: str | None = None) -> tuple[list[Link], dict]:
    """Returns ``(links, params)`` for a vehicle.

    ``model_dir=None`` reads this package's own table ``models/vehicles/<drone_model>.yaml``;
    otherwise ``<model_dir>/<drone_model>/<drone_model>.{urdf,yaml}`` is parsed, the layout the
    reference uses for custom models (base_drone.py:104-110)."""
    if model_dir is None:
        path = os.path.join(_VEHICLE_DIR, f"{drone_model}.yaml")
        if not os.path.exists(path):
            raise FileNotFoundError(f"no built-in vehicle table for {drone_model!r} ({path})")
        with open(path, "r", encoding="utf-8") as fh:
            doc = yaml.safe_load(fh)
        return [Link.from_dict(d) for d in doc["links"]], doc["params"]
    urdf = os.path.join(model_dir, f"{drone_model}/{drone_model}.urdf")
    param = os.path.join(model_dir, f"{drone_model}/{drone_model}.yaml")
    with open(param, "rb") as fh:
        params = yaml.safe_load(fh)
    return load_urdf_links(urdf), params


def _link(links: list[Link], index: int) -> Link:
    for lk in links:
        if lk.index == index:
            return lk
    raise KeyError(f"vehicle has no link {index}")


def _fill_rigid(m: PfbModel, links: list[Link]):
    M, c, I_O = composite_rigid_body(links)
    m.mass = M
    m.com[:] = c.tolist()
    m.inertia[:] = I_O.reshape(-1).tolist()
    n = 0
    for lk in links:
        for s in lk.shapes:
            if n >= MAX_SHAPES:
                raise ValueError("too many collision primitives")
            sh = m.shapes[n]
            sh.kind = SHAPE_IDS[s.kind]
            if s.kind == "box":
                sh.dims[:] = [0.5 * v for v in s.dims]
            elif s.kind == "cylinder":
                sh.dims[:] = [s.dims[0], 0.5 * s.dims[1], 0.0]
            else:
                sh.dims[:] = [s.dims[0], 0.0, 0.0]
            sh.at[:] = list(s.at)
            sh.rot[:] = np.asarray(s.rot, dtype=np.float64).reshape(-1).tolist()
            n += 1
    m.n_shapes = n
    m.contact_factor = 0.02


def _surface(m_s: PfbSurface, link: Link, lifting_unit, forward_unit, p: dict, physics_period: float):
    """Host precomputation of lifting_surfaces.py:217-262."""
    lift = np.asarray(lifting_unit, dtype=np.float64)
    fwd = np.asarray(forward_unit, dtype=np.float64)
    lift = lift / np.linalg.norm(lift)
    fwd = fwd / np.linalg.norm(fwd)
    chord, span = float(p["chord"]), float(p["span"])
    aspect = span / chord
    flap_to_chord = float(p["flap_to_chord"])
    Cl_alpha_3D = float(p["Cl_alpha_2D"]) * (aspect / (aspect + ((2.0 * (aspect + 4.0)) / (aspect + 2.0))))
    theta_f = math.acos(2.0 * flap_to_chord - 1.0)
    m_s.pos[:] = list(link.com)
    m_s.lift_unit[:] = lift.tolist()
    m_s.drag_unit[:] = fwd.tolist()
    m_s.torque_unit[:] = np.cross(lift, fwd).tolist()
    m_s.Cl_alpha_3D = Cl_alpha_3D
    m_s.aspect = aspect
    m_s.flap_to_chord = flap_to_chord
    m_s.aero_tau = 1.0 - ((theta_f - math.sin(theta_f)) / math.pi)
    m_s.eta = float(p["eta"])
    m_s.alpha_0_base = math.radians(float(p["alpha_0_base"]))
    m_s.alpha_stall_P_base = math.radians(float(p["alpha_stall_P_base"]))
    m_s.alpha_stall_N_base = math.radians(float(p["alpha_stall_N_base"]))
    m_s.Cd_0 = float(p["Cd_0"])
    m_s.deflection_limit_deg = float(p["deflection_limit"])
    m_s.dt_over_tau = physics_period / float(p["tau"])
    m_s.area = chord * span
    m_s.chord = chord
    m_s.half_rho = 0.5 * 1.225


def build_model(
    kind: str,
    drone_model: str | None = None,
    model_dir: str | None = None,
    physics_hz: int = 240,
    control_hz: int = 120,
    **options,
) -> PfbModel:
    """Builds the table for ``kind`` in {"quadx", "fixedwing", "rocket"} (aviary.py:167-170)."""
    defaults = {"quadx": "cf2x", "fixedwing": "fixedwing", "rocket": "rocket"}
    if kind not in defaults:
        raise ValueError(f"unknown drone_type {kind!r}; known: {list(defaults)}")
    if physics_hz % control_hz != 0:
        # base_drone.py:94-97
        raise ValueError(f"`physics_hz` ({physics_hz}) must be multiple of `control_hz` ({control_hz}).")
    drone_model = drone_model or defaults[kind]
    links, params = load_vehicle(drone_model, model_dir)
    dt = 1.0 / physics_hz

    m = PfbModel()
    m.abi_version = PFB_ABI_VERSION
    m.physics_hz = float(physics_hz)
    m.control_hz = float(control_hz)
    m.gravity = -9.81
    m.max_coord_velocity = 100.0
    _fill_rigid(m, links)

    if kind == "quadx":
        m.kind = KIND_QUADX
        mp, dp, cp = params["motor_params"], params["drag_params"], params["control_params"]
        m.n_motors = 4
        max_rpm = math.sqrt(mp["total_thrust"] / (4.0 * mp["thrust_coef"]))  # quadx.py:111-113
        tq = [-mp["torque_coef"], -mp["torque_coef"], +mp["torque_coef"], +mp["torque_coef"]]  # quadx.py:94-101
        for i in range(4):
            m.motor_pos[i][:] = list(_link(links, i).com)
            m.motor_axis[i][:] = [0.0, 0.0, 1.0]
            m.thrust_coef[i] = mp["thrust_coef"]
            m.torque_coef[i] = tq[i]
            m.max_rpm[i] = max_rpm
            m.motor_dt_over_tau[i] = dt / mp["tau"]
            m.motor_noise_ratio[i] = mp["noise_ratio"]
        m.n_bodies = 1
        m.body_pos[:] = list(_link(links, 4).com)  # body_ids=[4], quadx.py:148
        k = 0.5 * 1.225 * dp["drag_coef_xyz"] * dp["drag_area_xyz"]  # boring_bodies.py:63
        m.drag_const[:] = [k, k, k]
        m.drag_coef_pqr = dp["drag_coef_pqr"]
        names = ["ang_vel", "ang_pos", "lin_vel", "lin_pos", "z_vel", "z_pos"]
        for pi, name in enumerate(names):
            for gi, g in enumerate(["kp", "ki", "kd", "lim"]):
                val = cp[name][g]
                vals = list(val) if isinstance(val, (list, tuple)) else [val]
                vals = [float(v) for v in vals] + [0.0] * (3 - len(vals))
                m.pid[pi][gi][:] = vals
        mm = [[-1.0, -1.0, -1.0, +1.0], [+1.0, +1.0, -1.0, +1.0], [+1.0, -1.0, +1.0, +1.0], [-1.0, +1.0, +1.0, +1.0]]
        for i in range(4):
            m.motor_map[i][:] = mm[i]
    elif kind == "fixedwing":
        m.kind = KIND_FIXEDWING
        mp = params["motor_params"]
        m.n_motors = 1
        m.motor_pos[0][:] = list(_link(links, 0).com)
        m.motor_axis[0][:] = [1.0, 0.0, 0.0]
        m.thrust_coef[0] = mp["thrust_coef"]
        m.torque_coef[0] = mp["torque_coef"]
        m.max_rpm[0] = math.sqrt(mp["total_thrust"] / mp["thrust_coef"])  # fixedwing.py:149-151
        m.motor_dt_over_tau[0] = dt / mp["tau"]
        m.motor_noise_ratio[0] = mp["noise_ratio"]
        # order and link ids: fixedwing.py:79-138
        spec = [
            (3, [0, 0, 1], "left_wing_flapped_params"),
            (4, [0, 0, 1], "right_wing_flapped_params"),
            (1, [0, 0, 1], "horizontal_tail_params"),
            (2, [0, 1, 0], "vertical_tail_params"),
            (5, [0, 0, 1], "main_wing_params"),
        ]
        m.n_surfaces = 5
        for si, (lid, lift, key) in enumerate(spec):
            _surface(m.surfaces[si], _link(links, lid), lift, [1, 0, 0], params[key], dt)
        sv = options.get("starting_velocity", [20.0, 0.0, 0.0])  # fixedwing.py:35
        m.starting_velocity[:] = [float(v) for v in sv]
    else:
        m.kind = KIND_ROCKET
        bp, body = params["booster_params"], params["body_params"]
        m.n_bodies = 1
        m.body_pos[:] = list(_link(links, 0).com)  # body_ids=[0], rocket.py:92
        m.drag_const[:] = [
            0.5 * 1.225 * body["drag_coef_x"] * body["area_x"],
            0.5 * 1.225 * body["drag_coef_y"] * body["area_y"],
            0.5 * 1.225 * body["drag_coef_z"] * body["area_z"],
        ]
        # finlets sit on link ids 0,1 (lift +y) and 2,3 (lift +x): rocket.py:113-144 (sic)
        m.n_surfaces = 4
        for si, (lid, lift) in enumerate([(0, [0, 1, 0]), (1, [0, 1, 0]), (2, [1, 0, 0]), (3, [1, 0, 0])]):
            _surface(m.surfaces[si], _link(links, lid), lift, [0, 0, -1], params["finlet_params"], dt)
        m.has_booster = 1
        m.reignitable = 1 if bp["reignitable"] else 0
        m.booster_pos[:] = list(_link(links, 1).com)  # booster_ids=[1], rocket.py:163
        m.booster_axis[:] = [0.0, 0.0, 1.0]
        m.booster_dt_over_tau = dt / bp["booster_tau"]
        m.booster_noise_ratio = bp["noise_ratio"]
        m.booster_min_thrust = bp["min_thrust"]
        m.booster_max_thrust = bp["max_thrust"]
        m.fuel_total_mass = bp["total_fuel"]
        m.fuel_max_rate = bp["max_fuel_rate"]
        m.fuel_max_inertia[:] = [bp["inertia_ixx"], bp["inertia_iyy"], bp["inertia_izz"]]
        tank = _link(links, 0)  # fueltank_ids=[0], rocket.py:164
        m.fuel_pos[:] = list(tank.com)
        Md, cd, Id = composite_rigid_body(links, mass_override={0: 0.0}, inertia_override={0: np.zeros((3, 3))})
        m.dry_mass = Md
        m.dry_first_moment[:] = (Md * cd).tolist()
        m.dry_inertia[:] = Id.reshape(-1).tolist()
        m.gimbal_unit1[:] = [1.0, 0.0, 0.0]
        m.gimbal_unit2[:] = [0.0, 1.0, 0.0]
        m.gimbal_dt_over_tau = dt / bp["gimbal_tau"]
        r = math.radians(bp["gimbal_range_degrees"])
        m.gimbal_range_rad[:] = [r, r]
        m.starting_fuel_ratio = float(options.get("starting_fuel_ratio", 0.05))  # rocket.py:47 default
    return m


MAX_QUADX_MODELS = 16  # PFB_MAX_QUADX_MODELS (include/pyflyt_b200.h)


class ModelSetError(ValueError):
    """A ``drone_options`` sequence the batched stepper cannot fly in one handle (``BatchedAviary`` raises it as
    ``AviaryInitException``)."""


def _options_key(opts: dict) -> str:
    return repr(sorted((str(k), repr(v)) for k, v in opts.items()))


MAX_UPDATES_PER_STEP = 4  # physics steps per Aviary step a handle runs (the library's limit on physics_hz / control_hz)


def check_control_rates(rates, physics_hz: int, mixed_control_hz: bool) -> None:
    """The control rates of one batch.  Without ``mixed_control_hz`` they must all be equal.  With it, they follow the
    reference's rule (aviary.py:287-298): sorted, each rate is an integer multiple of the one before, and an Aviary step is
    ``physics_hz / min(control_hz)`` physics steps, here at most ``MAX_UPDATES_PER_STEP``."""
    rates = sorted({int(r) for r in rates})
    if len(rates) <= 1:
        return
    if not mixed_control_hz:
        raise ModelSetError(f"every drone of a batch needs the same control_hz (one substep ratio per batch; mixed_control_hz=True lets them differ); got {rates}.")
    if any(b % a for a, b in zip(rates, rates[1:])):
        raise AssertionError("Looprates must form common multiples of each other.")  # aviary.py:293-298
    updates = physics_hz // rates[0]
    if updates > MAX_UPDATES_PER_STEP:
        raise ModelSetError(
            f"control_hz {rates} at physics_hz {physics_hz}: an Aviary step of the slowest drone is {updates} physics steps; a batch runs at "
            f"most {MAX_UPDATES_PER_STEP} (the limit on one drone's physics_hz / control_hz)."
        )


def _bytes_but_rate(m: PfbModel) -> bytes:
    """the table's bytes with control_hz zeroed: fixed-wing and rocket tables depend on the rate through nothing else"""
    c = PfbModel.from_buffer_copy(m)
    c.control_hz = 0.0
    return C.string_at(C.addressof(c), C.sizeof(c))


def build_model_set(kind: str, drone_options, physics_hz: int, n: int, mixed_control_hz: bool = False) -> tuple[list[PfbModel], np.ndarray]:
    """Per-drone vehicle tables for ``n`` drones of one ``kind``.

    ``drone_options`` is what the reference's ``Aviary`` takes (aviary.py:75, 196-199): ``None`` or one dict for every drone,
    or a sequence of ``n`` dicts (or ``None``), one per drone.  Returns ``(tables, index)``: the distinct tables and a uint8
    array ``[n]``, drone ``i`` flies ``tables[index[i]]``.  Two drones share a table when their built tables are byte-equal,
    so a sequence that names the same vehicle in two ways still builds one table.

    Raises ``ModelSetError`` for a sequence of the wrong length (the reference's message), for entries with different
    ``control_hz`` (each handle runs one substep ratio), for more than ``MAX_QUADX_MODELS`` distinct QuadX tables and for more
    than one distinct fixed-wing or rocket table.

    ``mixed_control_hz=True`` lets the entries differ in ``control_hz`` under ``check_control_rates`` (an ``AssertionError``
    with the reference's message for rates that do not form common multiples).  A QuadX table is then one (model, rate) pair;
    fixed-wing and rocket tables may differ in ``control_hz`` only, one table per rate."""
    if drone_options is None or isinstance(drone_options, dict):
        entries = [dict(drone_options or {})]
        index = np.zeros(n, dtype=np.int64)
    else:
        seq = list(drone_options)
        if len(seq) != n:  # aviary.py:150-153
            raise ModelSetError(
                f"If multiple `drone_options` ({len(seq)}) are used, must have same number of `drone_options` as number of drones ({n})."
            )
        keys: dict[str, int] = {}
        entries, index = [], np.zeros(n, dtype=np.int64)
        for i, d in enumerate(seq):
            d = dict(d or {})
            key = _options_key(d)
            if key not in keys:
                keys[key] = len(entries)
                entries.append(d)
            index[i] = keys[key]
    if not mixed_control_hz:
        check_control_rates([e.get("control_hz", 120) for e in entries], physics_hz, False)
    tables: list[PfbModel] = []
    by_bytes: dict[bytes, int] = {}
    remap = np.zeros(len(entries), dtype=np.int64)
    for j, e in enumerate(entries):
        opts = dict(e)
        control_hz = int(opts.pop("control_hz", 120))
        m = build_model(kind, opts.pop("drone_model", None), opts.pop("model_dir", None), physics_hz, control_hz, **opts)
        b = C.string_at(C.addressof(m), C.sizeof(m))
        if b not in by_bytes:
            by_bytes[b] = len(tables)
            tables.append(m)
        remap[j] = by_bytes[b]
    if mixed_control_hz:  # after build_model: a control_hz that does not divide physics_hz raises its ValueError first, as in the reference
        check_control_rates([m.control_hz for m in tables], physics_hz, True)
    models = len({_bytes_but_rate(m) for m in tables}) if mixed_control_hz else len(tables)
    if kind != "quadx" and models > 1:
        raise ModelSetError(f"a {kind} batch flies one vehicle model; the drone_options build {models} different ones.")
    if len(tables) > MAX_QUADX_MODELS:
        raise ModelSetError(f"a batch flies at most {MAX_QUADX_MODELS} different vehicle models; the drone_options build {len(tables)}.")
    return tables, remap[index].astype(np.uint8)


KINDS = ("quadx", "fixedwing", "rocket")  # PFB_KIND_QUADX, PFB_KIND_FIXEDWING, PFB_KIND_ROCKET


def build_mixed_model_set(kinds, drone_options, physics_hz: int, n: int, mixed_control_hz: bool = False) -> tuple[list[PfbModel], np.ndarray]:
    """Per-drone vehicle tables for ``n`` drones of several kinds: ``kinds[i]`` is drone ``i``'s ``drone_type``.

    ``drone_options`` is what the reference's ``Aviary`` takes: ``None`` or one dict for every drone, or a sequence of ``n``
    dicts, one per drone.  The sub-sequence of each kind goes through ``build_model_set`` (so each kind keeps its limits: up to
    ``MAX_QUADX_MODELS`` QuadX tables, one fixed-wing and one rocket table).  Returns ``(tables, index)``: the QuadX tables,
    then the fixed-wing table, then the rocket table (those present), and a uint8 array ``[n]``, drone ``i`` flies
    ``tables[index[i]]``.  Every drone must run at the same ``control_hz`` (one launch steps them all with one substep count),
    unless ``mixed_control_hz=True``: then the rates of all kinds together follow ``check_control_rates``, and the fixed-wing
    and rocket tables of each kind follow the QuadX ones in ``build_model_set``'s order, one per rate."""
    kinds = list(kinds)
    if len(kinds) != n:
        raise ModelSetError(f"If multiple `drone_types` are used, must have same number of `drone_types` ({len(kinds)}) as number of drones ({n}).")
    per_drone = not (drone_options is None or isinstance(drone_options, dict))
    if per_drone:
        seq = list(drone_options)
        if len(seq) != n:  # aviary.py:150-153
            raise ModelSetError(
                f"If multiple `drone_options` ({len(seq)}) are used, must have same number of `drone_options` as number of drones ({n})."
            )
    tables: list[PfbModel] = []
    index = np.zeros(n, dtype=np.int64)
    for kind in KINDS:
        ids = [i for i, k in enumerate(kinds) if k == kind]
        if not ids:
            continue
        opts = [seq[i] for i in ids] if per_drone else drone_options
        t, idx = build_model_set(kind, opts, physics_hz, len(ids), mixed_control_hz)
        index[ids] = idx.astype(np.int64) + len(tables)
        tables.extend(t)
    check_control_rates([m.control_hz for m in tables], physics_hz, mixed_control_hz)
    return tables, index.astype(np.uint8)


def model_from_files(kind: str, urdf_path: str, yaml_path: str, physics_hz: int = 240, control_hz: int = 120, **options) -> PfbModel:
    """The same table built INSIDE the C-ABI (``pfb_model_from_files``, pyflyt_b200/csrc/pfb_model_files.cu) from a
    ``<model>.urdf`` + ``<model>.yaml`` pair in the reference's layout (base_drone.py:104-110): what a non-Python caller uses.
    ``options`` are the reference's constructor options (``starting_velocity``, ``starting_fuel_ratio``)."""
    from .._lib import check, lib

    kinds = {"quadx": KIND_QUADX, "fixedwing": KIND_FIXEDWING, "rocket": KIND_ROCKET}
    if kind not in kinds:
        raise ValueError(f"unknown drone_type {kind!r}; known: {list(kinds)}")
    m = PfbModel()
    check(lib().pfb_model_from_files(kinds[kind], os.fsencode(urdf_path), os.fsencode(yaml_path), float(physics_hz), float(control_hz), C.addressof(m)))
    if "starting_velocity" in options and kind == "fixedwing":
        m.starting_velocity[:] = [float(v) for v in options["starting_velocity"]]
    if "starting_fuel_ratio" in options and kind == "rocket":
        m.starting_fuel_ratio = float(options["starting_fuel_ratio"])
    return m


def model_to_dict(m: PfbModel) -> dict:
    """Plain-python view (for tests and debugging)."""

    def conv(v):
        if isinstance(v, C.Array):
            return [conv(x) for x in v]
        if isinstance(v, C.Structure):
            return {n: conv(getattr(v, n)) for n, _ in v._fields_}
        return v

    return conv(m)
