#!/usr/bin/env python
"""Generates tests/golden/*.npz by flying the UNMODIFIED reference (/root/reference/PyFlyt) on the
restated Bullet engine (oracle/fakebullet).  Run in the build container only; the fixtures travel.

Each fixture stores the scenario inputs (setpoints / actions, start pose), the raw
``np_random.normal`` draws the reference consumed (one per component per physics step, SURVEY §A.4)
and the reference's outputs per Aviary step / env step.  The C oracle (oracle/pfb_oracle.c) and the
CUDA path are both replayed against these with the same injected draws.

Scenarios mirror the reference's own tests: tests/test_core.py:13-31 (mode-7 hold),
:65-93 (two set-points), tests/test_gym_envs.py:92-112 (env determinism contract).
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.realpath(__file__)), "..")
sys.path.insert(0, ROOT)
from oracle import ref_in_loop as ril  # noqa: E402

ril.install()
from PyFlyt.core import Aviary  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def fly_quadx(name, mode, drone_model, start_pos, start_orn, setpoint_schedule, n_steps, seed, wind=None):
    """Aviary-level QuadX flight; setpoint_schedule: {step_index: setpoint(4)} applied before step."""
    rng = ril.ScriptedNoise(seed)
    env = Aviary(
        start_pos=np.array([start_pos], dtype=np.float64),
        start_orn=np.array([start_orn], dtype=np.float64),
        drone_type="quadx",
        drone_options=dict(drone_model=drone_model),
        np_random=rng,
    )
    env.set_mode(mode)
    if wind is not None:
        env.register_wind_field_function(wind)  # the UNMODIFIED reference evaluates our AnalyticWind as a plain wind-field function
        env.drones[0].update_state()  # the cached body velocity now sees the wind (update_state runs after every step anyway)
    sp_after_mode = np.array(env.drones[0].setpoint, dtype=np.float64)
    states, auxs, pwms, contacts, raws, sps = [], [], [], [], [], []
    for i in range(n_steps):
        if i in setpoint_schedule:
            env.set_setpoint(0, np.array(setpoint_schedule[i], dtype=np.float64))
        sps.append(np.array(env.drones[0].setpoint, dtype=np.float64))
        env.step()
        d = env.drones[0]
        states.append(np.array(d.state))
        auxs.append(np.array(d.aux_state))
        pwms.append(np.array(d.pwm))
        contacts.append(bool(np.any(env.contact_array[env.planeId])))
        pos, quat = env.getBasePositionAndOrientation(d.Id)
        v, w = env.getBaseVelocity(d.Id)
        raws.append(np.concatenate([pos, quat, v, w]))
    np.savez_compressed(
        os.path.join(OUT, f"{name}.npz"),
        kind="quadx_aviary",
        mode=mode,
        drone_model=drone_model,
        start_pos=np.array(start_pos, dtype=np.float64),
        start_orn=np.array(start_orn, dtype=np.float64),
        setpoint_after_set_mode=sp_after_mode,
        setpoints=np.array(sps),
        noise=np.array(rng.normal_log),
        state=np.array(states),
        aux=np.array(auxs),
        pwm=np.array(pwms),
        contact=np.array(contacts),
        raw=np.array(raws),
        **wind_fields(wind),
    )
    print(name, "final pos", states[-1][3], "draws", len(rng.normal_log))


def fly_quadx_mixed(name, mode, drone_options, start_pos, start_orn, setpoint_schedule, n_steps, seed):
    """Aviary-level flight of several QuadX drones with ONE options dict per drone in one reference Aviary (aviary.py:75,
    196-199).  ``model_dir`` entries are given relative to tests/golden and resolved here; the fixture stores them relative.
    setpoint_schedule: {step_index: [n, 4]} applied before the step.  The noise log holds the draws in the reference's order:
    per physics step, one per drone in drone order."""
    n = len(drone_options)
    resolved = [dict(d, model_dir=os.path.join(OUT, d["model_dir"])) if "model_dir" in d else dict(d) for d in drone_options]
    rng = ril.ScriptedNoise(seed)
    env = Aviary(
        start_pos=np.array(start_pos, dtype=np.float64),
        start_orn=np.array(start_orn, dtype=np.float64),
        drone_type="quadx",
        drone_options=resolved,
        np_random=rng,
    )
    env.set_mode(mode)
    sp_after_mode = np.array([d.setpoint for d in env.drones], dtype=np.float64)
    states, auxs, contacts, sps = [], [], [], []
    for i in range(n_steps):
        if i in setpoint_schedule:
            env.set_all_setpoints(np.array(setpoint_schedule[i], dtype=np.float64))
        sps.append(np.array([d.setpoint for d in env.drones], dtype=np.float64))
        env.step()
        states.append(np.array([d.state for d in env.drones]))
        auxs.append(np.array([d.aux_state for d in env.drones]))
        contacts.append(np.array([bool(env.contact_array[env.planeId, d.Id]) for d in env.drones]))
    np.savez_compressed(
        os.path.join(OUT, f"{name}.npz"),
        kind="quadx_mixed_aviary",
        mode=mode,
        n_drones=n,
        drone_options=json.dumps(drone_options),
        start_pos=np.array(start_pos, dtype=np.float64),
        start_orn=np.array(start_orn, dtype=np.float64),
        setpoint_after_set_mode=sp_after_mode,
        setpoints=np.array(sps),
        noise=np.array(rng.normal_log),
        state=np.array(states),
        aux=np.array(auxs),
        contact=np.array(contacts),
    )
    print(name, "final z", np.array(states[-1])[:, 3, 2], "draws", len(rng.normal_log), "contacts", int(np.sum(contacts)))


def mixed_model_fixtures():
    """Six drones alternating cf2x / primitive_drone, one of the primitive_drone slots flying primitive_tuned (a copy whose
    YAML changes thrust_coef, drag_coef_xyz and an ang_vel gain) loaded through model_dir: three distinct tables.
    No drone touches the floor: QuadX.update_physics drops the rotational drag when getContactPoints() of the WHOLE world is
    non-empty (quadx.py:508-510), so in one reference Aviary a drone's floor contact changes every other drone's flight,
    while the batched stepper gives each drone its own world."""
    opts = [dict(drone_model="cf2x"), dict(drone_model="primitive_drone"), dict(drone_model="cf2x"),
            dict(drone_model="primitive_tuned", model_dir="vehicles"), dict(drone_model="cf2x"), dict(drone_model="primitive_drone")]
    n = len(opts)
    pos = [[10.0 * k, 0.0, 60.0 + 0.5 * k] for k in range(n)]
    orn = [[0.05 * k, -0.04 * k, 0.3 * k] for k in range(n)]
    r = np.random.default_rng(91)
    sched0 = {k: np.concatenate([r.uniform(-0.4, 0.4, (n, 3)), r.uniform(0.2, 0.6, (n, 1))], axis=1) for k in range(0, 300, 60)}
    fly_quadx_mixed("mixed_models_quadx_mode0", 0, opts, pos, orn, sched0, 300, seed=92)
    pos7 = [[10.0 * k, 0.0, 2.0 + 0.5 * k] for k in range(n)]
    sched7 = {k: np.concatenate([r.uniform(-1.0, 1.0, (n, 2)) + np.array(pos7)[:, :2], r.uniform(-0.8, 0.8, (n, 1)), r.uniform(1.0, 4.0, (n, 1))], axis=1)
              for k in range(0, 300, 100)}
    fly_quadx_mixed("mixed_models_quadx_mode7", 7, opts, pos7, orn, sched7, 300, seed=93)


def _setpoint_rows(env):
    """[n, S] setpoints of every drone; fixed-wing mode 0 keeps 4 (fixedwing.py:224-227), padded here to mode -1's 6"""
    rows = [np.atleast_1d(np.asarray(d.setpoint, dtype=np.float64)) for d in env.drones]
    w = max(len(r) for r in rows)
    return np.array([np.concatenate([r, np.zeros(w - len(r))]) for r in rows])


def fly_mixed_modes(name, drone_type, drone_options, start_pos, start_orn, mode_calls, setpoint_fn, n_steps, seed):
    """Aviary-level flight of several drones in one reference Aviary with one flight mode per drone: ``mode_calls`` =
    {step_index: [n] modes}, each applied with ``Aviary.set_mode(list)`` before that step (aviary.py:440-458).
    ``setpoint_fn(step, modes, current)`` returns None or the [n, S] setpoints to apply before the step (after a set_mode call;
    ``current`` = the drones' setpoints at that point).
    The fixture stores the modes of every call and the setpoints each call left."""
    n = len(drone_options)
    rng = ril.ScriptedNoise(seed)
    env = Aviary(
        start_pos=np.array(start_pos, dtype=np.float64),
        start_orn=np.array(start_orn, dtype=np.float64),
        drone_type=drone_type,
        drone_options=[dict(d) for d in drone_options],
        np_random=rng,
    )
    states, auxs, contacts, sps, sp_after = [], [], [], [], []
    modes = None
    for i in range(n_steps):
        if i in mode_calls:
            modes = [int(m) for m in mode_calls[i]]
            env.set_mode(modes)
            sp_after.append(_setpoint_rows(env))
        sp = setpoint_fn(i, modes, _setpoint_rows(env))
        if sp is not None:
            env.set_all_setpoints(np.array(sp, dtype=np.float64))
        sps.append(_setpoint_rows(env))
        env.step()
        states.append(np.array([d.state for d in env.drones]))
        auxs.append(np.array([d.aux_state for d in env.drones], dtype=np.float64))
        contacts.append(np.array([bool(env.contact_array[env.planeId, d.Id]) for d in env.drones]))
    # one reference world: any floor contact would remove every QuadX's rotational drag (quadx.py:508-510)
    assert not np.any(contacts), f"{name}: a drone touched the floor"
    steps = sorted(mode_calls)
    np.savez_compressed(
        os.path.join(OUT, f"{name}.npz"),
        kind=f"{drone_type}_mixed_modes",
        drone_type=drone_type,
        n_drones=n,
        drone_options=json.dumps(drone_options),
        start_pos=np.array(start_pos, dtype=np.float64),
        start_orn=np.array(start_orn, dtype=np.float64),
        mode_steps=np.array(steps),
        modes=np.array([mode_calls[k] for k in steps], dtype=np.int64),
        setpoint_after_set_mode=np.array(sp_after),
        setpoints=np.array(sps),
        noise=np.array(rng.normal_log),
        state=np.array(states),
        aux=np.array(auxs),
        contact=np.array(contacts),
    )
    print(name, "final z", np.array(states[-1])[:, 3, 2], "draws", len(rng.normal_log))


def mixed_mode_fixtures():
    """One flight mode per drone.  QuadX: 18 drones, every mode -1..7 on cf2x and on primitive_drone, re-assigned by
    set_mode(list) at steps 100 and 200: the height-hold drones (modes 2, 3, 4, 7) fly mode 0 or 1 in between and then hold
    height again with the z-PID memory set_mode keeps (quadx.py:196, 372).  Setpoints come from the ranges of the single-mode
    fixtures, heights relative to the start.  Fixed-wing: 4 drones, modes -1 / 0 alternating.  No drone touches the floor."""
    n = 18
    opts = [dict(drone_model="cf2x" if d % 2 == 0 else "primitive_drone") for d in range(n)]
    pos = np.array([[10.0 * d, 0.0, 60.0 + 0.5 * d] for d in range(n)])
    orn = [[0.05 * (d % 5), -0.04 * (d % 4), 0.3 * (d % 7)] for d in range(n)]
    first = [-1 + d // 2 for d in range(n)]
    away = {-1: 3, 0: 7, 1: 2, 2: 0, 3: 1, 4: 0, 5: 4, 6: -1, 7: 1}
    calls = {0: first, 100: [away[m] for m in first], 200: first}
    table = {  # the first / second setpoint of quadx_<model>_mode<m>; heights and mode-7 positions relative to the start
        -1: ([0.3, 0.31, 0.32, 0.3], [0.5, 0.5, 0.45, 0.5]),
        0: ([0.3, -0.2, 0.1, 0.45], [-0.5, 0.4, -0.3, 0.3]),
        1: ([0.2, -0.1, 0.5, 0.3], [-0.2, 0.2, -0.5, -0.2]),
        2: ([0.2, -0.2, 0.3, 1.0], [-0.3, 0.1, 0.0, -1.0]),
        3: ([0.15, -0.1, 0.6, 1.0], [0.0, 0.0, -0.6, -0.5]),
        4: ([0.8, -0.5, 0.3, 1.0], [-0.6, 0.4, -0.2, -0.5]),
        5: ([0.8, -0.5, 0.3, 0.4], [-0.6, 0.4, -0.2, -0.3]),
        6: ([0.9, 0.4, 0.5, 0.3], [-0.5, -0.7, -0.4, -0.2]),
        7: ([1.0, -1.0, 0.8, 1.0], [-0.5, 0.5, -0.8, -1.0]),
    }

    def quadx_sp(i, modes, current):
        if i % 100 == 0:  # a set_mode call's preset is flown for 10 steps; mode -1 keeps the previous setpoint, so it gets pwm now
            out = current.copy()
            for d, m in enumerate(modes):
                if m == -1:
                    out[d] = table[-1][0]
            return out
        if i % 50 != 10 and i % 50 != 0:
            return None
        out = np.zeros((n, 4))
        for d, m in enumerate(modes):
            out[d] = table[m][(i // 50) % 2]
            if m in (2, 3, 4, 7):
                out[d, 3] += pos[d, 2]
            if m == 7:
                out[d, :2] += pos[d, :2]
        return out

    fly_mixed_modes("mixed_modes_quadx", "quadx", opts, pos.tolist(), orn, calls, quadx_sp, 300, seed=95)

    nf = 4
    fw_opts = [dict(drone_model="fixedwing") for _ in range(nf)]
    fw_pos = [[40.0 * d, 0.0, 80.0] for d in range(nf)]
    fw_orn = [[0.05 * d, 0.1, 0.4 * d] for d in range(nf)]
    fw_modes = [-1 if d % 2 == 0 else 0 for d in range(nf)]
    r = np.random.default_rng(96)

    def fw_sp(i, modes, current):
        if i % 40:
            return None
        out = np.zeros((nf, 6))
        for d, m in enumerate(modes):
            if m == -1:
                out[d] = np.concatenate([r.uniform(-0.8, 0.8, 5), r.uniform(0.0, 1.0, 1)])
            else:
                out[d, :4] = np.concatenate([r.uniform(-0.6, 0.6, 3), r.uniform(0.3, 1.0, 1)])
        return out

    fly_mixed_modes("mixed_modes_fixedwing", "fixedwing", fw_opts, fw_pos, fw_orn, {0: fw_modes}, fw_sp, 200, seed=97)


def _padded_rows(rows, w):
    rows = [np.atleast_1d(np.asarray(r, dtype=np.float64)) for r in rows]
    return np.array([np.concatenate([r, np.zeros(w - len(r))]) for r in rows])


def fly_mixed_kinds(name, drone_type, drone_options, start_pos, start_orn, mode_calls, setpoint_fn, n_steps, seed, kind="mixed_kinds"):
    """Aviary-level flight of QuadX, fixed-wing and rocket drones in ONE reference Aviary (``drone_type`` a list,
    aviary.py:139-190, as examples/core/08_mixed_drones.py does): ``mode_calls`` = {step_index: [n] modes}, each applied with
    ``Aviary.set_mode(list)`` before that step; ``setpoint_fn(step, modes)`` returns None or a list of ``n`` per-drone
    setpoints of each drone's own length, applied with ``set_all_setpoints`` (aviary.py:470-478 indexes ``setpoints[i]``).
    Every drone draws one normal per physics step (its motors or its booster), in drone order, so the recorded draws are
    [step][substep][drone], with ``updates_per_step`` substeps (the slowest drone's ratio when the drones' ``control_hz`` differ,
    aviary.py:287-298).  Setpoints are stored padded to 7 columns, aux states to 9."""
    n = len(drone_type)
    rng = ril.ScriptedNoise(seed)
    env = Aviary(
        start_pos=np.array(start_pos, dtype=np.float64),
        start_orn=np.array(start_orn, dtype=np.float64),
        drone_type=list(drone_type),
        drone_options=[dict(d) for d in drone_options],
        np_random=rng,
    )
    states, auxs, contacts, sps, sp_after = [], [], [], [], []
    modes = None
    for i in range(n_steps):
        if i in mode_calls:
            modes = [int(m) for m in mode_calls[i]]
            env.set_mode(modes)
            sp_after.append(_padded_rows([d.setpoint for d in env.drones], 7))
        sp = setpoint_fn(i, modes)
        if sp is not None:
            env.set_all_setpoints([np.array(r, dtype=np.float64) for r in sp])
        sps.append(_padded_rows([d.setpoint for d in env.drones], 7))
        env.step()
        states.append(np.array([d.state for d in env.drones]))
        auxs.append(_padded_rows([d.aux_state for d in env.drones], 9))
        contacts.append(np.array([bool(env.contact_array[env.planeId, d.Id]) for d in env.drones]))
    # one reference world: any floor contact would remove every QuadX's rotational drag (quadx.py:508-510), a coupling that
    # separate worlds cannot have
    assert not np.any(contacts), f"{name}: a drone touched the floor"
    steps = sorted(mode_calls)
    T = n_steps
    noise = np.array(rng.normal_log)
    assert noise.size == T * int(env.updates_per_step) * n, (noise.size, T, n)
    np.savez_compressed(
        os.path.join(OUT, f"{name}.npz"),
        kind=kind,
        drone_type=json.dumps(list(drone_type)),
        n_drones=n,
        drone_options=json.dumps(drone_options),
        start_pos=np.array(start_pos, dtype=np.float64),
        start_orn=np.array(start_orn, dtype=np.float64),
        mode_steps=np.array(steps),
        modes=np.array([mode_calls[k] for k in steps], dtype=np.int64),
        setpoint_after_set_mode=np.array(sp_after),
        setpoints=np.array(sps),
        noise=noise,
        state=np.array(states),
        aux=np.array(auxs),
        contact=np.array(contacts),
    )
    print(name, "final z", np.array(states[-1])[:, 3, 2], "draws", noise.size)


def mixed_kind_fixtures():
    """Rockets, QuadX and fixed-wing drones in one Aviary (the reference's tests/test_core.py::test_mixed_drones with more drones
    and commands).  Rockets upright (roll pi / 2), ignited, with finlet, throttle and gimbal commands; QuadX cf2x and
    primitive_drone in modes 0 and 7; fixed-wing in modes 0 and -1, all re-assigned by a second set_mode(list) at step 150.
    1: the kinds grouped; 2: interleaved r, q, f, q, r, f, ...  No drone touches the floor."""
    qx_opts = [dict(drone_model="cf2x"), dict(drone_model="primitive_drone")]

    def scenario(name, kinds, seed):
        n = len(kinds)
        opts, first, second = [], [], []
        nq = nf = 0
        for k in kinds:
            if k == "quadx":
                opts.append(dict(qx_opts[nq % 2]))
                first.append(0 if (nq // 2) % 2 == 0 else 7)
                nq += 1
            elif k == "fixedwing":
                opts.append(dict(drone_model="fixedwing"))
                first.append(0 if nf % 2 == 0 else -1)
                nf += 1
            else:
                opts.append(dict(drone_model="rocket"))
                first.append(0)
        second = [{0: 7, 7: 0, -1: 0}.get(m, m) if k != "rocket" else 0 for k, m in zip(kinds, first)]
        second = [(-1 if m == 0 else 0) if k == "fixedwing" else m for k, m in zip(kinds, second)]
        pos = np.array([[12.0 * d, 0.0, {"quadx": 40.0, "fixedwing": 80.0, "rocket": 60.0}[k] + 0.5 * d] for d, k in enumerate(kinds)])
        orn = [[np.pi / 2, 0.0, 0.2 * (d % 3)] if k == "rocket" else [0.05 * (d % 3), -0.04 * (d % 2), 0.3 * (d % 5)] for d, k in enumerate(kinds)]
        r = np.random.default_rng(seed)

        def sp_fn(i, modes):
            if i % 50 != 10:
                return None
            out = []
            for d, (k, m) in enumerate(zip(kinds, modes)):
                if k == "rocket":
                    out.append(np.concatenate([r.uniform(-0.5, 0.5, 3), [1.0, r.uniform(0.3, 0.8)], r.uniform(-0.3, 0.3, 2)]))
                elif k == "fixedwing":
                    if m == -1:
                        out.append(np.concatenate([r.uniform(-0.6, 0.6, 5), r.uniform(0.3, 1.0, 1)]))
                    else:
                        out.append(np.concatenate([r.uniform(-0.5, 0.5, 3), r.uniform(0.3, 1.0, 1)]))
                elif m == 7:
                    out.append(np.array([pos[d, 0] + r.uniform(-1, 1), pos[d, 1] + r.uniform(-1, 1), r.uniform(-0.8, 0.8), pos[d, 2] + r.uniform(-1, 1)]))
                else:
                    out.append(np.concatenate([r.uniform(-0.3, 0.3, 3), r.uniform(0.3, 0.45, 1)]))
            return out

        fly_mixed_kinds(name, kinds, opts, pos.tolist(), orn, {0: first, 150: second}, sp_fn, 300, seed=seed)

    scenario("mixed_kinds_grouped", ["rocket"] * 2 + ["quadx"] * 4 + ["fixedwing"] * 2, 101)
    scenario("mixed_kinds_interleaved", ["rocket", "quadx", "fixedwing", "quadx", "rocket", "fixedwing", "quadx", "fixedwing", "rocket", "quadx"], 102)


def rate_fixtures():
    """Drones at different control rates in one reference Aviary (per-drone ``drone_options`` ``control_hz``; the reference's
    tests/test_core.py::test_multi_spawn and examples/core/02_multi_drone.py).  An Aviary step is physics_hz / min(control_hz)
    physics steps and each drone runs its controller on every physics_hz / control_hz-th of them (aviary.py:287-298, 506-529).
    No drone touches the floor."""
    # test_multi_spawn: three cf2x at 60 / 120 / 240 Hz in mode 7, a new height at step 150.  cf2x's gains are tuned for faster
    # control: at 60 or 80 Hz its attitude loop rings after a lateral command and amplifies the round-off difference of two fp64
    # codes to millimetres within a hundred steps, so here (and below) the slow cf2x drones fly the inner-loop modes or climb
    pos = np.array([[-1.0, 0.0, 1.0], [0.0, 0.0, 1.0], [1.0, 0.0, 1.0]])

    def spawn_sp(i, modes):
        if i != 150:
            return None
        return [np.array([p[0], p[1], 0.0, 1.2]) for p in pos]

    fly_mixed_kinds("rates_multi_spawn", ["quadx"] * 3, [dict(control_hz=60), dict(control_hz=120), dict(control_hz=240)], pos.tolist(),
                    np.zeros((3, 3)).tolist(), {0: [7, 7, 7]}, spawn_sp, 300, seed=111, kind="rates")

    # both QuadX models at every rate, in modes -1, 0, 2, 6, 7, re-assigned by one set_mode(list) at step 100
    table = {-1: [0.3, 0.31, 0.32, 0.3], 0: [0.1, -0.05, 0.05, 0.45], 2: [0.1, -0.1, 0.2, 1.0], 6: [0.5, 0.3, 0.3, 0.2], 7: [0.5, -0.5, 0.4, 1.0]}
    combos = [(m, hz) for m in ("cf2x", "primitive_drone") for hz in (60, 120, 240)] + [("primitive_drone", 60), ("cf2x", 120), ("cf2x", 240),
                                                                                      ("primitive_drone", 60)]
    n = 10
    opts = [dict(drone_model=combos[d][0], control_hz=combos[d][1]) for d in range(n)]
    cycle = [-1, 0, 2, 6, 7]
    first = [cycle[d % 5] for d in range(n)]
    second = [cycle[(d + 2) % 5] for d in range(n)]
    pos = np.array([[8.0 * d, 0.0, 60.0 + 0.5 * d] for d in range(n)])
    orn = [[0.05 * (d % 3), -0.04 * (d % 2), 0.3 * (d % 5)] for d in range(n)]

    def modes_sp(i, modes):
        if i % 100 != 0 and i % 100 != 40:
            return None
        out = []
        for d, m in enumerate(modes):
            sp = np.array(table[m]) * (1.0 if i % 100 == 0 else -0.5)
            if m in (2, 7):
                sp[3] = pos[d, 2] + (1.0 if i % 100 == 0 else -0.5)
            if m == 7:
                sp[:2] += pos[d, :2]
            if m == -1:
                sp = np.array(table[-1])
            out.append(sp)
        return out

    fly_mixed_kinds("rates_models_modes", ["quadx"] * n, opts, pos.tolist(), orn, {0: first, 100: second}, modes_sp, 200, seed=112, kind="rates")

    # rockets, QuadX and fixed-wing drones interleaved: QuadX at 60 / 120 / 240 Hz, fixed-wing at 60 / 120 Hz, rockets at 120 / 240 Hz
    kinds = ["rocket", "quadx", "fixedwing", "quadx", "rocket", "fixedwing", "quadx", "fixedwing", "rocket", "quadx"]
    hz = {"quadx": [60, 120, 240], "fixedwing": [60, 120], "rocket": [120, 240]}
    seen = {"quadx": 0, "fixedwing": 0, "rocket": 0}
    opts, first = [], []
    for k in kinds:
        c = hz[k][seen[k] % len(hz[k])]
        opts.append(dict(drone_model={"quadx": "cf2x", "fixedwing": "fixedwing", "rocket": "rocket"}[k], control_hz=c))
        first.append({"quadx": [0, 7, 7, 0][seen[k] % 4], "fixedwing": [0, -1][seen[k] % 2], "rocket": 0}[k])
        seen[k] += 1
    pos = np.array([[12.0 * d, 0.0, {"quadx": 150.0, "fixedwing": 200.0, "rocket": 150.0}[k] + 0.5 * d] for d, k in enumerate(kinds)])
    orn = [[np.pi / 2, 0.0, 0.2 * (d % 3)] if k == "rocket" else [0.05 * (d % 3), -0.04 * (d % 2), 0.3 * (d % 5)] for d, k in enumerate(kinds)]
    r = np.random.default_rng(113)

    def kinds_sp(i, modes):
        if i % 50 != 10:
            return None
        out = []
        for d, (k, m) in enumerate(zip(kinds, modes)):
            if k == "rocket":
                out.append(np.concatenate([r.uniform(-0.5, 0.5, 3), [1.0, r.uniform(0.3, 0.8)], r.uniform(-0.3, 0.3, 2)]))
            elif k == "fixedwing":
                out.append(np.concatenate([r.uniform(-0.6, 0.6, 5), r.uniform(0.3, 1.0, 1)]) if m == -1 else
                           np.concatenate([r.uniform(-0.5, 0.5, 3), r.uniform(0.3, 1.0, 1)]))
            elif m == 7:
                out.append(np.array([pos[d, 0] + r.uniform(-1, 1), pos[d, 1] + r.uniform(-1, 1), r.uniform(-0.8, 0.8), pos[d, 2] + r.uniform(-1, 1)]))
            else:
                out.append(np.concatenate([r.uniform(-0.3, 0.3, 3), r.uniform(0.3, 0.45, 1)]))
        return out

    fly_mixed_kinds("rates_kinds_interleaved", kinds, opts, pos.tolist(), orn, {0: first}, kinds_sp, 300, seed=113, kind="rates")

    # 80 and 240 Hz: three physics steps per Aviary step
    kinds = ["quadx", "quadx", "fixedwing", "rocket", "quadx"]
    opts = [dict(control_hz=80), dict(control_hz=240), dict(control_hz=80), dict(control_hz=240), dict(drone_model="primitive_drone", control_hz=80)]
    pos = np.array([[0.0, 0.0, 30.0], [10.0, 0.0, 30.0], [20.0, 0.0, 80.0], [30.0, 0.0, 60.0], [40.0, 0.0, 30.0]])
    orn = [[0.05, -0.04, 0.3], [0.0, 0.05, -0.2], [0.05, 0.1, 0.4], [np.pi / 2, 0.0, 0.2], [-0.05, 0.0, 0.1]]
    r = np.random.default_rng(114)

    def thirds_sp(i, modes):
        if i % 60 != 0:
            return None
        return [np.concatenate([r.uniform(-0.1, 0.1, 3), r.uniform(0.35, 0.45, 1)]),
                np.concatenate([r.uniform(-0.3, 0.3, 3), r.uniform(0.3, 0.45, 1)]),
                np.concatenate([r.uniform(-0.5, 0.5, 3), r.uniform(0.3, 1.0, 1)]),
                np.concatenate([r.uniform(-0.5, 0.5, 3), [1.0, r.uniform(0.3, 0.8)], r.uniform(-0.3, 0.3, 2)]),
                np.array([pos[4, 0] + r.uniform(-1, 1), pos[4, 1] + r.uniform(-1, 1), r.uniform(-0.5, 0.5), pos[4, 2] + r.uniform(-1, 1)])]

    fly_mixed_kinds("rates_thirds", kinds, opts, pos.tolist(), orn, {0: [0, 0, 0, 0, 7]}, thirds_sp, 240, seed=114, kind="rates")


def wind_fields(wind):
    """npz entries describing an AnalyticWind (absent = still air)"""
    if wind is None:
        return {}
    return dict(wind_kind=wind.kind, wind_base=wind.base, wind_z_ref=wind.z_ref, wind_alpha=wind.alpha, wind_z0=wind.z0)


def fly_vehicle(name, drone_type, drone_model, mode, start_pos, start_orn, setpoint_schedule, n_steps, seed, drone_options=None, pre_hook=None, wind=None):
    """Aviary-level flight of a fixedwing / rocket; setpoint_schedule: {step: setpoint} applied before the step."""
    rng = ril.ScriptedNoise(seed)
    opts = dict(drone_model=drone_model, **(drone_options or {}))
    env = Aviary(
        start_pos=np.array([start_pos], dtype=np.float64),
        start_orn=np.array([start_orn], dtype=np.float64),
        drone_type=drone_type,
        drone_options=opts,
        np_random=rng,
    )
    env.set_mode(mode)
    if wind is not None:
        env.register_wind_field_function(wind)
        env.drones[0].update_state()  # the cached surface / body velocities now see the wind (update_state runs after every step)
    if pre_hook is not None:
        pre_hook(env)
        env.drones[0].update_state()  # resetBaseVelocity alone leaves the drone's cached velocities stale
    d = env.drones[0]
    v0, w0 = env.getBaseVelocity(d.Id)
    sp_dim = len(np.atleast_1d(d.setpoint))
    states, auxs, contacts, raws, sps = [], [], [], [], []
    for i in range(n_steps):
        if i in setpoint_schedule:
            env.set_setpoint(0, np.array(setpoint_schedule[i], dtype=np.float64))
        sps.append(np.array(d.setpoint, dtype=np.float64))
        env.step()
        states.append(np.array(d.state))
        auxs.append(np.array(d.aux_state, dtype=np.float64))
        contacts.append(bool(np.any(env.contact_array[env.planeId])))
        pos, quat = env.getBasePositionAndOrientation(d.Id)
        v, w = env.getBaseVelocity(d.Id)
        raws.append(np.concatenate([pos, quat, v, w]))
    np.savez_compressed(
        os.path.join(OUT, f"{name}.npz"),
        kind=f"{drone_type}_aviary",
        mode=mode,
        drone_type=drone_type,
        drone_model=drone_model,
        drone_options=json.dumps({k: (list(v) if hasattr(v, "__len__") else v) for k, v in (drone_options or {}).items()}),
        start_pos=np.array(start_pos, dtype=np.float64),
        start_orn=np.array(start_orn, dtype=np.float64),
        setpoint_dim=sp_dim,
        start_lin_vel=np.array(v0, dtype=np.float64),
        start_ang_vel=np.array(w0, dtype=np.float64),
        has_pre_hook=pre_hook is not None,
        setpoints=np.array(sps),
        noise=np.array(rng.normal_log),
        state=np.array(states),
        aux=np.array(auxs),
        contact=np.array(contacts),
        raw=np.array(raws),
        **wind_fields(wind),
    )
    print(name, "final pos", states[-1][3], "draws", len(rng.normal_log))


def fly_waypoints(name, seed, n_steps, action_seed, angle_representation="quaternion", sparse=False, num_targets=4,
                  goal_reach_distance=2.0, dome=100.0, action_scale=1.0):
    """FixedwingWaypointsEnv (fixedwing_waypoints_env.py) with scripted actions and user-loop resets."""
    from PyFlyt.gym_envs.fixedwing_envs.fixedwing_waypoints_env import FixedwingWaypointsEnv

    env = FixedwingWaypointsEnv(sparse_reward=sparse, num_targets=num_targets, goal_reach_distance=goal_reach_distance,
                                flight_dome_size=dome, angle_representation=angle_representation)
    rng = ril.ScriptedNoise(seed)
    env._np_random = rng

    def flat(state):
        d = np.asarray(state["target_deltas"], dtype=np.float64).reshape(-1)
        pad = np.zeros(3 * num_targets)
        pad[: len(d)] = d
        return np.concatenate([state["attitude"], pad])

    state0, _ = env.reset()
    targets = [np.array(env.waypoints.targets, dtype=np.float64)]
    arng = np.random.default_rng(action_seed)
    obs, rew, term, trunc, info, acts, episode_start, resets_obs = [], [], [], [], [], [], [], []
    noise_splits = [len(rng.normal_log)]
    for i in range(n_steps):
        a = arng.uniform(-1.0, 1.0, 4) * action_scale
        a[3] = arng.uniform(0.2, 1.0)
        o, r, te, tr, inf = env.step(a)
        acts.append(a); obs.append(flat(o)); rew.append(r); term.append(te); trunc.append(tr)
        info.append(int(inf["out_of_bounds"]) | (int(inf["collision"]) << 1) | (int(inf["env_complete"]) << 2) | (int(inf["num_targets_reached"]) << 3))
        noise_splits.append(len(rng.normal_log))
        if te or tr:
            o2, _ = env.reset()
            targets.append(np.array(env.waypoints.targets, dtype=np.float64))
            resets_obs.append(flat(o2))
            episode_start.append(i + 1)
            noise_splits.append(len(rng.normal_log))
    np.savez_compressed(
        os.path.join(OUT, f"{name}.npz"), kind="fixedwing_waypoints", sparse=sparse, dome=dome, num_targets=num_targets,
        goal_reach_distance=goal_reach_distance, angle_representation=angle_representation, reset_obs=flat(state0),
        targets=np.array(targets), actions=np.array(acts), obs=np.array(obs), reward=np.array(rew), term=np.array(term),
        trunc=np.array(trunc), info=np.array(info), noise=np.array(rng.normal_log), noise_splits=np.array(noise_splits),
        episode_start=np.array(episode_start, dtype=np.int64),
        after_reset_obs=np.array(resets_obs) if resets_obs else np.zeros((0, 23 + 3 * num_targets)),
    )
    print(name, "steps", n_steps, "episodes", len(episode_start) + 1, "max targets reached", max(v >> 3 for v in info), "draws", len(rng.normal_log))


def fly_qx_waypoints(name, seed, n_steps, action_seed, flight_mode=0, angle_representation="quaternion", sparse=False, num_targets=4,
                     use_yaw_targets=False, goal_reach_distance=0.2, goal_reach_angle=0.1, dome=5.0, chase=False, action_scale=1.0):
    """QuadXWaypointsEnv (quadx_waypoints_env.py) with scripted actions and user-loop resets.  ``chase``: in a position
    flight mode (7: x, y, yaw, z) the action is the next target (+ jitter), so that waypoints ARE reached."""
    from PyFlyt.gym_envs.quadx_envs.quadx_waypoints_env import QuadXWaypointsEnv

    env = QuadXWaypointsEnv(sparse_reward=sparse, num_targets=num_targets, use_yaw_targets=use_yaw_targets,
                            goal_reach_distance=goal_reach_distance, goal_reach_angle=goal_reach_angle, flight_mode=flight_mode,
                            flight_dome_size=dome, angle_representation=angle_representation)
    rng = ril.ScriptedNoise(seed)
    env._np_random = rng
    T = 4 if use_yaw_targets else 3

    def flat(state):
        d = np.asarray(state["target_deltas"], dtype=np.float64).reshape(-1)
        pad = np.zeros(T * num_targets)
        pad[: len(d)] = d
        return np.concatenate([state["attitude"], pad])

    def cur_targets():
        t = np.array(env.waypoints.targets, dtype=np.float64).reshape(-1, 3)
        if use_yaw_targets:
            t = np.concatenate([t, np.array(env.waypoints.yaw_targets, dtype=np.float64)[:, None]], axis=-1)
        return t

    state0, _ = env.reset()
    targets = [cur_targets()]
    arng = np.random.default_rng(action_seed)
    obs, rew, term, trunc, info, acts, episode_start, resets_obs = [], [], [], [], [], [], [], []
    noise_splits = [len(rng.normal_log)]
    for i in range(n_steps):
        if chase and len(env.waypoints.targets) > 0:
            t = np.asarray(env.waypoints.targets[0], dtype=np.float64)
            yaw = float(env.waypoints.yaw_targets[0]) if use_yaw_targets else 0.0
            a = np.array([t[0], t[1], yaw, t[2]]) + arng.normal(0.0, 0.02, 4)
        else:
            a = arng.uniform([-np.pi, -np.pi, -np.pi, 0.0], [np.pi, np.pi, np.pi, 0.8]) * np.array([action_scale] * 3 + [1.0])
        o, r, te, tr, inf = env.step(a)
        acts.append(a); obs.append(flat(o)); rew.append(r); term.append(te); trunc.append(tr)
        info.append(int(inf["out_of_bounds"]) | (int(inf["collision"]) << 1) | (int(inf["env_complete"]) << 2) | (int(inf["num_targets_reached"]) << 3))
        noise_splits.append(len(rng.normal_log))
        if te or tr:
            o2, _ = env.reset()
            targets.append(cur_targets())
            resets_obs.append(flat(o2))
            episode_start.append(i + 1)
            noise_splits.append(len(rng.normal_log))
    att = 21 if angle_representation == "quaternion" else 20
    np.savez_compressed(
        os.path.join(OUT, f"{name}.npz"), kind="quadx_waypoints", sparse=sparse, dome=dome, num_targets=num_targets,
        use_yaw_targets=use_yaw_targets, goal_reach_distance=goal_reach_distance, goal_reach_angle=goal_reach_angle, flight_mode=flight_mode,
        angle_representation=angle_representation, reset_obs=flat(state0), targets=np.array(targets), actions=np.array(acts),
        obs=np.array(obs), reward=np.array(rew), term=np.array(term), trunc=np.array(trunc), info=np.array(info),
        noise=np.array(rng.normal_log), noise_splits=np.array(noise_splits), episode_start=np.array(episode_start, dtype=np.int64),
        after_reset_obs=np.array(resets_obs) if resets_obs else np.zeros((0, att + T * num_targets)),
    )
    print(name, "steps", n_steps, "episodes", len(episode_start) + 1, "max targets reached", max(v >> 3 for v in info), "draws", len(rng.normal_log))


def fly_landing(name, seed, n_steps, action_seed, options, angle_representation="quaternion", sparse=False, ignite_p=0.7):
    """RocketLandingEnv (rocket_landing_env.py) with scripted actions and user-loop resets; ``options`` as in
    env.reset(options=...): None = randomised + accelerated drop, {} = the plain 450 m hover-drop."""
    from PyFlyt.gym_envs.rocket_envs.rocket_landing_env import RocketLandingEnv

    env = RocketLandingEnv(sparse_reward=sparse, angle_representation=angle_representation)
    rng = ril.ScriptedNoise(seed)
    env._np_random = rng
    obs0, _ = env.reset(options=None if options is None else dict(options))
    spawns = [np.concatenate([env.start_pos[0], env.start_orn[0]])]
    arng = np.random.default_rng(action_seed)
    lo, hi = env.action_space.low, env.action_space.high
    obs, rew, term, trunc, info, acts, episode_start, resets_obs = [], [], [], [], [], [], [], []
    noise_splits = [len(rng.normal_log)]
    for i in range(n_steps):
        a = arng.uniform(lo, hi)
        a[3] = 1.0 if arng.random() < ignite_p else 0.0
        o, r, te, tr, inf = env.step(a)
        acts.append(a); obs.append(np.array(o)); rew.append(r); term.append(te); trunc.append(tr)
        info.append(int(inf["out_of_bounds"]) | (int(inf["fatal_collision"]) << 1) | (int(inf["env_complete"]) << 2))
        noise_splits.append(len(rng.normal_log))
        if te or tr:
            o2, _ = env.reset(options=None if options is None else dict(options))
            spawns.append(np.concatenate([env.start_pos[0], env.start_orn[0]]))
            resets_obs.append(np.array(o2))
            episode_start.append(i + 1)
            noise_splits.append(len(rng.normal_log))
    np.savez_compressed(
        os.path.join(OUT, f"{name}.npz"), kind="rocket_landing", sparse=sparse, angle_representation=angle_representation,
        randomize_drop=options is None, accelerate_drop=options is None, spawns=np.array(spawns), reset_obs=np.array(obs0),
        actions=np.array(acts), obs=np.array(obs), reward=np.array(rew), term=np.array(term), trunc=np.array(trunc), info=np.array(info),
        noise=np.array(rng.normal_log), noise_splits=np.array(noise_splits), episode_start=np.array(episode_start, dtype=np.int64),
        after_reset_obs=np.array(resets_obs) if resets_obs else np.zeros((0, len(obs0))),
    )
    print(name, "steps", n_steps, "episodes", len(episode_start) + 1, "infos", sorted(set(info)), "draws", len(rng.normal_log))


def fly_touchdown(name, seed, n_steps, descent_rate, ceiling=4.0, max_displacement=20.0, angle_representation="quaternion", lateral=(0.0, 0.0)):
    """RocketLandingEnv brought down onto the pad by a scripted bang-bang ignition law, with the engine's contact RESPONSE
    switched on (oracle/fakebullet World.contact_response): the rocket touches down at `descent_rate`-ish m/s, rests on its
    legs and the UNMODIFIED env reports env_complete (rocket_landing_env.py:231-263).  Same file format as fly_landing."""
    import pybullet as fb  # oracle/fakebullet
    from PyFlyt.gym_envs.rocket_envs.rocket_landing_env import RocketLandingEnv

    fb.World.contact_response = True
    try:
        env = RocketLandingEnv(ceiling=ceiling, max_displacement=max_displacement, angle_representation=angle_representation)
        rng = ril.ScriptedNoise(seed)
        env._np_random = rng
        obs0, _ = env.reset(options=dict(randomize_drop=False, accelerate_drop=False))
        if lateral != (0.0, 0.0):  # a small sideways push: friction has to stop the slide
            env.env.resetBaseVelocity(env.env.drones[0].Id, [lateral[0], lateral[1], 0.0], [0.0, 0.0, 0.0])
        spawns = [np.concatenate([env.start_pos[0], env.start_orn[0]])]
        att = 4 if angle_representation == "quaternion" else 3
        obs_k, acts, obs, rew, term, trunc, info = np.array(obs0), [], [], [], [], [], []
        noise_splits = [len(rng.normal_log)]
        for i in range(n_steps):
            vz, z = obs_k[3 + att + 2], obs_k[3 + att + 3 + 2]
            h = z - 2.425 - 0.15  # leg soles above the pad
            ign = 1.0 if (vz < -(descent_rate + 1.0 * max(h, 0.0)) and h > 0.02) else 0.0
            a = np.array([0.0, 0.0, 0.0, ign, 0.0, 0.0, 0.0])
            o, r, te, tr, inf = env.step(a)
            obs_k = np.array(o)
            acts.append(a); obs.append(obs_k); rew.append(r); term.append(te); trunc.append(tr)
            info.append(int(inf["out_of_bounds"]) | (int(inf["fatal_collision"]) << 1) | (int(inf["env_complete"]) << 2))
            noise_splits.append(len(rng.normal_log))
            if te or tr:
                break
    finally:
        fb.World.contact_response = False
    np.savez_compressed(
        os.path.join(OUT, f"{name}.npz"), kind="rocket_landing", sparse=False, angle_representation=angle_representation,
        randomize_drop=False, accelerate_drop=False, spawns=np.array(spawns), reset_obs=np.array(obs0),
        actions=np.array(acts), obs=np.array(obs), reward=np.array(rew), term=np.array(term), trunc=np.array(trunc), info=np.array(info),
        noise=np.array(rng.normal_log), noise_splits=np.array(noise_splits), episode_start=np.zeros(0, dtype=np.int64),
        after_reset_obs=np.zeros((0, len(obs0))), ceiling=ceiling, max_displacement=max_displacement, contact_response=True,
        start_lin_vel=np.array([lateral[0], lateral[1], 0.0]),
    )
    print(name, "steps", len(acts), "last info", info[-1], "pad contact steps", int(sum(o[-1] for o in obs)), "draws", len(rng.normal_log))


def touchdown_fixtures():
    # SURVEY 8f item 3: gentle touchdowns that must end in env_complete, a hard one that must be a fatal collision
    fly_touchdown("landing_touchdown", seed=81, n_steps=300, descent_rate=0.6)
    fly_touchdown("landing_touchdown_soft_euler", seed=82, n_steps=300, descent_rate=0.3, angle_representation="euler")
    fly_touchdown("landing_touchdown_hard", seed=83, n_steps=300, descent_rate=2.5)


def ground_fixtures():
    """Aviary-level flights that land on, rest on, slide along and take off from the floor, with the engine's contact RESPONSE
    switched on (oracle/fakebullet World.contact_response), replayed by BatchedAviary(contact_response=True).  One drone per
    reference Aviary: the reference drops the rotational drag of every drone of a world once any of them touches
    (quadx.py:508-510), and each batched drone has a world of its own.  The files are named ground_* so that the replays of
    the flag-only fixtures (quadx_*, fixedwing_*, rocket_*) do not pick them up."""
    import pybullet as fb  # oracle/fakebullet

    fb.World.contact_response = True
    try:
        # cf2x take-off from the floor (velocity mode 6): climb to ~1 m, hold, descend, settle on the floor for > 2 s
        fly_quadx("ground_cf2x_takeoff_landing", 6, "cf2x", [0.0, 0.0, 0.01], [0.0, 0.0, 0.0],
                  {0: [0.0, 0.0, 0.0, 0.5], 240: [0.0, 0.0, 0.0, 0.0], 360: [0.0, 0.0, 0.0, -0.4], 660: [0.0, 0.0, 0.0, -0.2]}, 1000, seed=301)
        # primitive_drone dropped tilted with the motors idle: a propeller cylinder's rim strikes first, the airframe tips flat
        fly_quadx("ground_primitive_tilted_drop", -1, "primitive_drone", [0.0, 0.0, 1.5], [0.4, 0.0, 0.0], {0: [0.0, 0.0, 0.0, 0.0]}, 480, seed=302)
        # cf2x pushed sideways by a tilted thrust burst, then motors idle: it touches down sliding and friction stops it
        fly_quadx("ground_cf2x_sliding_touchdown", -1, "cf2x", [0.0, 0.0, 0.1], [0.0, 0.35, 0.0],
                  {0: [0.6, 0.6, 0.6, 0.6], 24: [0.0, 0.0, 0.0, 0.0]}, 600, seed=303)
        # fixed-wing glide at zero throttle from a few metres: belly landing, slides to rest on its box primitives
        fly_vehicle("ground_fixedwing_belly_landing", "fixedwing", "fixedwing", 0, [0.0, 0.0, 3.0], [0.0, 0.05, 0.0], {0: [0.0, 0.1, 0.0, 0.0]},
                    840, seed=304)
        # rocket dropped a short way onto the bare ground, booster off: it rests on its legs
        fly_vehicle("ground_rocket_rest", "rocket", "rocket", 0, [0.0, 0.0, 3.0], [0.0, 0.0, 0.0], {0: [0, 0, 0, 0, 0, 0, 0]}, 360, seed=305)
    finally:
        fb.World.contact_response = False


def fly_base_state(name, drone_type, drone_options, start_pos, start_orn, modes, setpoints, resets, n_steps, seed):
    """Aviary-level flight of ``drone_type`` (a list, one reference Aviary) with base-state resets between ``aviary.step()``
    calls, as a script on top of the Aviary does them: ``resets`` = {step: dict(mask=[n], pos=[n][3], orn=[n][3] Euler, lin=[n][3],
    ang=[n][3])} (keys absent = not given) are applied before that step with ``resetBasePositionAndOrientation`` (then
    ``resetBaseVelocity`` with whatever velocities are given) and ``drones[i].update_state()`` for every masked drone.
    ``modes``: [n] flight modes set once; ``setpoints``: {step: [n] per-drone setpoints} applied with ``set_all_setpoints``.
    The npz stores the reset steps, masks and values (quaternions, x y z w), and per step the states, aux states (padded to 9),
    contact flags and raw base states.  Named base_state_* so that no other replay's glob picks it up."""
    n = len(drone_type)
    rng = ril.ScriptedNoise(seed)
    env = Aviary(start_pos=np.array(start_pos, dtype=np.float64), start_orn=np.array(start_orn, dtype=np.float64), drone_type=list(drone_type),
                 drone_options=[dict(d) for d in drone_options], np_random=rng)
    env.set_mode([int(m) for m in modes])
    R = len(resets)
    r_steps = np.array(sorted(resets), dtype=np.int64)
    r_mask, r_has = np.zeros((R, n), dtype=np.uint8), np.zeros((R, 3), dtype=bool)  # has: pose, lin, ang
    r_pos, r_quat, r_lin, r_ang = np.zeros((R, n, 3)), np.zeros((R, n, 4)), np.zeros((R, n, 3)), np.zeros((R, n, 3))
    r_quat[..., 3] = 1.0
    states, auxs, contacts, raws, sps = [], [], [], [], []
    for i in range(n_steps):
        if i in setpoints:
            env.set_all_setpoints([np.array(r, dtype=np.float64) for r in setpoints[i]])
        if i in resets:
            k, ev = int(np.searchsorted(r_steps, i)), resets[i]
            r_mask[k] = ev["mask"]
            r_has[k] = ["pos" in ev, "lin" in ev, "ang" in ev]
            for d in np.flatnonzero(r_mask[k]):
                drone = env.drones[d]
                if "pos" in ev:
                    r_pos[k, d] = ev["pos"][d]
                    r_quat[k, d] = env.getQuaternionFromEuler(ev["orn"][d])
                    env.resetBasePositionAndOrientation(drone.Id, r_pos[k, d], r_quat[k, d])
                if "lin" in ev or "ang" in ev:
                    r_lin[k, d] = ev["lin"][d] if "lin" in ev else 0.0
                    r_ang[k, d] = ev["ang"][d] if "ang" in ev else 0.0
                    env.resetBaseVelocity(drone.Id, r_lin[k, d] if "lin" in ev else None, r_ang[k, d] if "ang" in ev else None)
                drone.update_state()
        sps.append(_padded_rows([d.setpoint for d in env.drones], 7))
        env.step()
        states.append(np.array([d.state for d in env.drones]))
        auxs.append(_padded_rows([d.aux_state for d in env.drones], 9))
        contacts.append(np.array([bool(env.contact_array[env.planeId, d.Id]) for d in env.drones]))
        raws.append(np.array([np.concatenate([*env.getBasePositionAndOrientation(d.Id), *env.getBaseVelocity(d.Id)]) for d in env.drones]))
    noise = np.array(rng.normal_log)
    assert noise.size == n_steps * int(env.updates_per_step) * n, (noise.size, n_steps, n)
    np.savez_compressed(
        os.path.join(OUT, f"{name}.npz"),
        kind="base_state",
        drone_type=json.dumps(list(drone_type)),
        n_drones=n,
        drone_options=json.dumps(drone_options),
        start_pos=np.array(start_pos, dtype=np.float64),
        start_orn=np.array(start_orn, dtype=np.float64),
        modes=np.array(modes, dtype=np.int64),
        contact_response=bool(__import__("pybullet").World.contact_response),
        reset_steps=r_steps, reset_mask=r_mask, reset_has=r_has, reset_pos=r_pos, reset_quat=r_quat, reset_lin=r_lin, reset_ang=r_ang,
        setpoints=np.array(sps),
        noise=noise,
        state=np.array(states),
        aux=np.array(auxs),
        contact=np.array(contacts),
        raw=np.array(raws),
    )
    print(name, "final pos", np.array(states[-1])[:, 3], "contacts", int(np.sum(contacts)), "draws", noise.size)


def base_state_fixtures():
    """Scripts that move drones by hand between Aviary steps (resetBasePositionAndOrientation / resetBaseVelocity +
    update_state, as rocket_base_env.py:228 and custom task code do), replayed by BatchedAviary.set_base_state."""
    import pybullet as fb  # oracle/fakebullet

    cf2x, prim = dict(drone_model="cf2x"), dict(drone_model="primitive_drone")
    # 1. two QuadX holding (0, 0, 2) in mode 7: one teleported far away and tilted, the other thrown; the PIDs recover with
    #    their memories intact
    hold = {0: [[0.0, 0.0, 0.0, 2.0]] * 2}
    fly_base_state("base_state_quadx", ["quadx", "quadx"], [cf2x, prim], [[0.0, 0.0, 2.0]] * 2, [[0.05, -0.05, 0.2], [-0.04, 0.03, -0.1]], [7, 7], hold,
                   {100: dict(mask=[1, 0], pos=[[6.0, -4.0, 9.0], [0.0] * 3], orn=[[0.5, -0.35, 1.0], [0.0] * 3]),
                    200: dict(mask=[0, 1], lin=[[0.0] * 3, [4.0, 0.0, 3.0]], ang=[[0.0] * 3, [2.0, -1.0, 0.5]])}, 300, seed=401)
    # 2. fixed-wing and acrowing in mode 0, relaunched at 40 m, yaw 1.2, with 20 m/s along the new heading
    for model, sd in (("fixedwing", 402), ("acrowing", 403)):
        relaunch = dict(mask=[1], pos=[[0.0, 0.0, 40.0]], orn=[[0.0, 0.0, 1.2]], lin=[[20.0 * np.cos(1.2), 20.0 * np.sin(1.2), 0.0]])
        fly_base_state(f"base_state_{model}", ["fixedwing"], [dict(drone_model=model)], [[0.0, 0.0, 30.0]], [[0.0, 0.05, 0.0]], [0],
                       {0: [[0.0, 0.1, 0.0, 0.7]], 200: [[0.2, -0.1, 0.1, 0.5]]}, {150: relaunch}, 300, seed=sd)
    # 3. a rocket dropping from 200 m, re-posed upright at 100 m, given (3, -2, -30) m/s and a spin in the same call
    fly_base_state("base_state_rocket", ["rocket"], [dict(drone_model="rocket")], [[0.0, 0.0, 200.0]], [[0.3, -0.2, 0.1]], [0],
                   {0: [[0.2, -0.1, 0.1, 1.0, 0.4, 0.1, -0.1]]},
                   {100: dict(mask=[1], pos=[[5.0, -3.0, 100.0]], orn=[[0.0, 0.0, 0.4]], lin=[[3.0, -2.0, -30.0]], ang=[[0.5, -0.3, 1.0]])}, 300, seed=404)
    # 4. with the contact response, one drone per reference Aviary (as the ground_* fixtures): at rest on the floor, lifted and
    #    tilted by a pose reset, falls and lands again.  The rocket is lifted upright and turned: tilted, it rocks on its legs
    #    for longer than the fixture lasts
    fb.World.contact_response = True
    try:
        fly_base_state("base_state_ground_cf2x", ["quadx"], [cf2x], [[0.0, 0.0, 0.01]], [[0.0, 0.0, 0.0]], [-1], {0: [[0.0] * 4]},
                       {120: dict(mask=[1], pos=[[0.5, -0.3, 1.2]], orn=[[0.4, -0.2, 0.8]])}, 480, seed=405)
        fly_base_state("base_state_ground_fixedwing", ["fixedwing"], [dict(drone_model="fixedwing")], [[0.0, 0.0, 0.5]], [[0.0, 0.0, 0.0]], [0],
                       {0: [[0.0, 0.0, 0.0, 0.0]]}, {200: dict(mask=[1], pos=[[2.0, 1.0, 2.5]], orn=[[0.25, 0.15, 0.5]])}, 720, seed=406)
        fly_base_state("base_state_ground_rocket", ["rocket"], [dict(drone_model="rocket")], [[0.0, 0.0, 3.0]], [[0.0, 0.0, 0.0]], [0], {0: [[0.0] * 7]},
                       {150: dict(mask=[1], pos=[[1.0, -1.0, 2.9]], orn=[[0.0, 0.0, 0.3]])}, 450, seed=407)
    finally:
        fb.World.contact_response = False
    # 5. one Aviary of four kinds, no floor contact: only drones 1 and 3 reset at step 80 (pose and both velocities)
    kinds = ["quadx", "fixedwing", "rocket", "quadx"]
    opts = [cf2x, dict(drone_model="fixedwing"), dict(drone_model="rocket"), prim]
    pos = [[0.0, 0.0, 20.0], [12.0, 0.0, 60.0], [24.0, 0.0, 150.0], [36.0, 0.0, 30.0]]
    orn = [[0.05, -0.04, 0.2], [0.0, 0.05, 0.0], [np.pi / 2, 0.0, 0.2], [-0.03, 0.02, 0.4]]
    sp = {0: [[0.0, 0.0, 0.0, 20.0], [0.1, 0.1, 0.0, 0.7], [0.2, -0.2, 0.1, 1.0, 0.5, 0.1, 0.1], [36.0, 0.0, 0.3, 30.0]]}
    z3 = [0.0] * 3
    fly_base_state("base_state_mixed", kinds, opts, pos, orn, [7, 0, 0, 7], sp,
                   {80: dict(mask=[0, 1, 0, 1], pos=[z3, [10.0, 5.0, 70.0], z3, [33.0, -2.0, 25.0]], orn=[z3, [0.0, 0.05, -0.7], z3, [0.3, 0.1, 0.5]],
                             lin=[z3, [18.0 * np.cos(-0.7), 18.0 * np.sin(-0.7), 0.0], z3, [1.0, -2.0, 0.5]], ang=[z3, [0.1, 0.0, 0.0], z3, [0.5, 0.2, -0.3]])},
                   200, seed=408)


def fly_dogfight(name, seed, n_steps, action_seed, team_size=1, sparse=False, action_scale=0.6, lethal_distance=20.0, lethal_angle=0.07,
                 spawn_min_radius=10.0, spawn_max_radius=50.0, damage_per_hit=0.003, pitch_bias=0.0):
    """MAFixedwingDogfightEnv (pz_envs/fixedwing_envs/ma_fixedwing_dogfight_env.py) with scripted actions; a new
    episode is started whenever every agent is done.  The Aviary's own generator (seeded by reset(seed)) is
    wrapped so that its motor-noise draws are recorded."""
    from PyFlyt.pz_envs.fixedwing_envs.ma_fixedwing_dogfight_env import MAFixedwingDogfightEnv

    env = MAFixedwingDogfightEnv(team_size=team_size, sparse_reward=sparse, lethal_distance=lethal_distance, lethal_angle_radians=lethal_angle,
                                 spawn_min_radius=spawn_min_radius, spawn_max_radius=spawn_max_radius, damage_per_hit=damage_per_hit)
    A = 2 * team_size
    real_default_rng = np.random.default_rng
    loggers = []

    def reset(seed_):
        def patched(s=None):
            lg = ril.ScriptedNoise.__new__(ril.ScriptedNoise)
            lg._rng = real_default_rng(s)
            lg.normal_log = []
            loggers.append(lg)
            return lg
        np.random.default_rng = patched
        try:
            obs, _ = env.reset(seed=seed_)
        finally:
            np.random.default_rng = real_default_rng
        return np.stack([obs[f"uav_{i}"] for i in range(A)])

    def drained():
        lg = loggers[-1]
        out = np.array(lg.normal_log)
        lg.normal_log.clear()
        return out

    arng = real_default_rng(action_seed)
    episodes = []
    ep_seed = seed
    obs0 = reset(ep_seed)
    ep = dict(spawn=np.concatenate([env.start_pos, env.start_orn], axis=1), reset_obs=obs0, reset_noise=drained(), actions=[], obs=[], reward=[], term=[], trunc=[], noise=[])
    for i in range(n_steps):
        alive = set(env.agents)
        act = arng.uniform(-1.0, 1.0, (A, 4)) * action_scale
        act[:, 1] = np.clip(act[:, 1] + pitch_bias, -1.0, 1.0)
        o, r, te, tr, _ = env.step({f"uav_{k}": act[k] for k in range(A) if f"uav_{k}" in alive})
        ep["actions"].append(act)
        ep["noise"].append(drained())
        row = lambda d, default: np.array([d.get(f"uav_{k}", default) for k in range(A)])  # noqa: E731
        ep["obs"].append(np.stack([o.get(f"uav_{k}", np.full(obs0.shape[1], np.nan)) for k in range(A)]))
        ep["reward"].append(row(r, np.nan)); ep["term"].append(row(te, True)); ep["trunc"].append(row(tr, False))
        ep["alive"] = ep.get("alive", []) + [np.array([f"uav_{k}" in alive for k in range(A)])]
        if len(env.agents) == 0:
            episodes.append(ep)
            ep_seed += 1
            obs0 = reset(ep_seed)
            ep = dict(spawn=np.concatenate([env.start_pos, env.start_orn], axis=1), reset_obs=obs0, reset_noise=drained(), actions=[], obs=[], reward=[], term=[], trunc=[], noise=[])
    if ep["actions"]:
        episodes.append(ep)
    flat = {}
    for k, e in enumerate(episodes):
        for key, v in e.items():
            flat[f"ep{k}_{key}"] = np.array(v)
    np.savez_compressed(os.path.join(OUT, f"{name}.npz"), kind="dogfight", team_size=team_size, sparse=sparse, n_episodes=len(episodes),
                        lethal_distance=lethal_distance, lethal_angle=lethal_angle, damage_per_hit=damage_per_hit, **flat)
    print(name, "episodes", len(episodes), "steps", [len(e["actions"]) for e in episodes], "reward range", min(np.nanmin(e["reward"]) for e in episodes), max(np.nanmax(e["reward"]) for e in episodes))


def fly_ma_hover(name, seed, n_steps, action_seed, flight_mode=0, angle_representation="quaternion", sparse=False, dome=10.0,
                 max_duration_seconds=30.0, action_scale=0.3, start_pos=None, agent_hz=40):
    """MAQuadXHoverEnv (pz_envs/quadx_envs/ma_quadx_hover_env.py) with scripted actions; a new episode is started whenever
    every agent is done.  The Aviary's own generator (seeded by reset(seed)) is wrapped so that its draws are recorded."""
    from PyFlyt.pz_envs.quadx_envs.ma_quadx_hover_env import MAQuadXHoverEnv

    kw = dict(sparse_reward=sparse, flight_mode=flight_mode, flight_dome_size=dome, max_duration_seconds=max_duration_seconds,
              angle_representation=angle_representation, agent_hz=agent_hz)
    if start_pos is not None:
        kw.update(start_pos=np.asarray(start_pos, dtype=np.float64), start_orn=np.zeros_like(np.asarray(start_pos, dtype=np.float64)))
    env = MAQuadXHoverEnv(**kw)
    A = len(env.possible_agents)
    real_default_rng = np.random.default_rng
    loggers = []

    def reset(seed_):
        def patched(s=None):
            lg = ril.ScriptedNoise.__new__(ril.ScriptedNoise)
            lg._rng = real_default_rng(s)
            lg.normal_log = []
            loggers.append(lg)
            return lg
        np.random.default_rng = patched
        try:
            obs, _ = env.reset(seed=seed_)
        finally:
            np.random.default_rng = real_default_rng
        return np.stack([obs[f"uav_{i}"] for i in range(A)])

    def drained():
        lg = loggers[-1]
        out = np.array(lg.normal_log)
        lg.normal_log.clear()
        return out

    arng = real_default_rng(action_seed)
    lo, hi = np.array([-np.pi, -np.pi, -np.pi, 0.0]), np.array([np.pi, np.pi, np.pi, 0.8])
    episodes = []
    ep_seed = seed
    obs0 = reset(ep_seed)
    new_ep = lambda o: dict(reset_obs=o, reset_noise=drained(), actions=[], obs=[], reward=[], term=[], trunc=[], noise=[], alive=[])  # noqa: E731
    ep = new_ep(obs0)
    for i in range(n_steps):
        alive = set(env.agents)
        act = arng.uniform(lo, hi, (A, 4)) * np.array([action_scale] * 3 + [1.0])
        o, r, te, tr, _ = env.step({f"uav_{k}": act[k] for k in range(A) if f"uav_{k}" in alive})
        ep["actions"].append(act)
        ep["noise"].append(drained())
        row = lambda d, default: np.array([d.get(f"uav_{k}", default) for k in range(A)])  # noqa: E731
        ep["obs"].append(np.stack([o.get(f"uav_{k}", np.full(obs0.shape[1], np.nan)) for k in range(A)]))
        ep["reward"].append(row(r, np.nan)); ep["term"].append(row(te, True)); ep["trunc"].append(row(tr, False))
        ep["alive"].append(np.array([f"uav_{k}" in alive for k in range(A)]))
        if len(env.agents) == 0:
            episodes.append(ep)
            ep_seed += 1
            ep = new_ep(reset(ep_seed))
    if ep["actions"]:
        episodes.append(ep)
    flat = {}
    for k, e in enumerate(episodes):
        for key, v in e.items():
            flat[f"ep{k}_{key}"] = np.array(v)
    np.savez_compressed(os.path.join(OUT, f"{name}.npz"), kind="ma_quadx_hover", n_agents=A, sparse=sparse, n_episodes=len(episodes), flight_mode=flight_mode,
                        angle_representation=angle_representation, dome=dome, max_duration_seconds=max_duration_seconds, agent_hz=agent_hz,
                        start_pos=np.asarray(env.start_pos, dtype=np.float64), start_orn=np.asarray(env.start_orn, dtype=np.float64), **flat)
    print(name, "episodes", len(episodes), "steps", [len(e["actions"]) for e in episodes], "reward range", min(np.nanmin(e["reward"]) for e in episodes), max(np.nanmax(e["reward"]) for e in episodes))


def fly_hover(name, seed, n_steps, action_seed, angle_representation, flight_mode=0, sparse=False, dome=3.0, action_scale=1.0, wind=None,
              agent_hz=40):
    from PyFlyt.gym_envs.quadx_envs.quadx_hover_env import QuadXHoverEnv

    env = QuadXHoverEnv(
        sparse_reward=sparse, flight_mode=flight_mode, flight_dome_size=dome, angle_representation=angle_representation, agent_hz=agent_hz
    )
    rng = ril.ScriptedNoise(seed)
    env._np_random = rng  # the env hands its generator to the Aviary (quadx_base_env.py:192)
    obs0, _ = env.reset()
    if wind is not None:  # the reference envs have no wind argument: a user attaches the field to the env's Aviary after reset()
        env.env.register_wind_field_function(wind)
        env.env.drones[0].update_state()
    arng = np.random.default_rng(action_seed)
    lo, hi = env.action_space.low, env.action_space.high
    obs, rew, term, trunc, info, acts, episode_start = [], [], [], [], [], [], []
    noise_splits = [len(rng.normal_log)]
    resets_obs = []
    for i in range(n_steps):
        a = arng.uniform(lo, hi) * action_scale
        o, r, te, tr, inf = env.step(a)
        acts.append(a)
        obs.append(o)
        rew.append(r)
        term.append(te)
        trunc.append(tr)
        info.append(int(inf["out_of_bounds"]) | (int(inf["collision"]) << 1) | (int(inf["env_complete"]) << 2))
        noise_splits.append(len(rng.normal_log))
        if te or tr:
            assert wind is None, "wind fixtures are single-episode (a reset re-creates the Aviary without the field)"
            # next-episode reset exactly as a user loop would do it
            o2, _ = env.reset()
            resets_obs.append(o2)
            episode_start.append(i + 1)
            noise_splits.append(len(rng.normal_log))
    np.savez_compressed(
        os.path.join(OUT, f"{name}.npz"),
        kind="quadx_hover",
        flight_mode=flight_mode,
        sparse=sparse,
        dome=dome,
        angle_representation=angle_representation,
        agent_hz=agent_hz,
        reset_obs=obs0,
        actions=np.array(acts),
        obs=np.array(obs),
        reward=np.array(rew),
        term=np.array(term),
        trunc=np.array(trunc),
        info=np.array(info),
        noise=np.array(rng.normal_log),
        noise_splits=np.array(noise_splits),
        episode_start=np.array(episode_start, dtype=np.int64),
        after_reset_obs=np.array(resets_obs) if resets_obs else np.zeros((0, len(obs0))),
        **wind_fields(wind),
    )
    print(name, "steps", n_steps, "episodes", len(episode_start) + 1, "draws", len(rng.normal_log))


def fixedwing_fixtures():
    # Fixedwing (lifting surfaces + one motor), both airframes, mode 0 (RPYT mixing) and -1 (raw surfaces)
    r = np.random.default_rng(21)
    for model in ["fixedwing", "acrowing"]:
        sched0 = {}
        for k in range(0, 600, 40):
            sched0[k] = np.concatenate([r.uniform(-0.6, 0.6, 3), r.uniform(0.3, 1.0, 1)])
        fly_vehicle(f"fixedwing_{model}_mode0", "fixedwing", model, 0, [0, 0, 60.0], [0.05, -0.1, 0.4], sched0, 600, seed=31)
        schedm = {}
        for k in range(0, 400, 50):
            schedm[k] = np.concatenate([r.uniform(-0.8, 0.8, 5), r.uniform(0.0, 1.0, 1)])
        fly_vehicle(f"fixedwing_{model}_mode-1", "fixedwing", model, -1, [0, 0, 80.0], [0.0, 0.2, -1.0], schedm, 400, seed=32)
    # deep stall / tumbling: large attitude offsets and zero airspeed at spawn exercise the post-stall branches
    fly_vehicle(
        "fixedwing_stall", "fixedwing", "fixedwing", 0, [0, 0, 120.0], [1.2, 0.9, -2.0],
        {0: [0.9, -0.9, 0.5, 0.0], 150: [-0.9, 0.9, -0.5, 1.0]}, 500, seed=33, drone_options=dict(starting_velocity=np.array([0.0, 0.0, 0.0])),
    )
    # dive into the floor: contact flag from the link boxes
    fly_vehicle("fixedwing_floor", "fixedwing", "fixedwing", 0, [0, 0, 3.0], [0.0, 0.6, 0.0], {0: [0.0, 0.5, 0.0, 0.2]}, 120, seed=34)
    # Fixedwing-Waypoints env (BASELINE configs[2]); the wide goal radius makes scripted flights reach targets
    fly_waypoints("fwwp_quat_dense", seed=41, n_steps=300, action_seed=5, action_scale=0.3)
    fly_waypoints("fwwp_wide_goal", seed=42, n_steps=400, action_seed=6, goal_reach_distance=70.0, action_scale=0.15, num_targets=3)
    fly_waypoints("fwwp_euler_sparse", seed=43, n_steps=200, action_seed=7, angle_representation="euler", sparse=True, action_scale=0.5)


def rocket_fixtures():
    r = np.random.default_rng(51)

    def sched(n, every, ign_p=0.8):
        out = {}
        for k in range(0, n, every):
            out[k] = np.concatenate([r.uniform(-1, 1, 3), [1.0 if r.random() < ign_p else 0.0], r.uniform(0, 1, 1), r.uniform(-1, 1, 2)])
        return out

    # powered flight from rest: gimbal, fins, throttle changes, full tank (mass/inertia vary slowly)
    fly_vehicle("rocket_powered", "rocket", "rocket", 0, [0, 0, 100.0], [0.05, -0.04, 0.3], sched(600, 40), 600, seed=61)
    # Rocket-Landing style drop: 5 % fuel runs dry (hard cut-off), -100 m/s start hits Bullet's velocity clamp
    def drop(env):
        env.resetBaseVelocity(env.drones[0].Id, [3.0, -2.0, -100.0], [0.2, -0.1, 0.3])
    fly_vehicle("rocket_drop", "rocket", "rocket", 0, [5.0, -8.0, 420.0], [0.2, -0.15, 0.1], sched(500, 25, 0.6), 500, seed=62,
                drone_options=dict(starting_fuel_ratio=0.05), pre_hook=drop)
    # tumbling, engine off: finlets + body drag at large angles of attack
    def spin(env):
        env.resetBaseVelocity(env.drones[0].Id, [20.0, 10.0, -30.0], [1.5, -1.0, 0.5])
    s3 = sched(300, 30, 0.0)
    fly_vehicle("rocket_tumble", "rocket", "rocket", 0, [0, 0, 300.0], [1.0, 0.5, 0.0], s3, 300, seed=63, pre_hook=spin)
    # ground strike (legs / body primitives)
    fly_vehicle("rocket_ground", "rocket", "rocket", 0, [30.0, 0, 6.0], [0.3, 0.0, 0.0], {0: [0, 0, 0, 0, 0, 0, 0]}, 150, seed=64)
    # full tank: the composite mass / COM / inertia change every substep while the booster burns
    fly_vehicle("rocket_full_tank", "rocket", "rocket", 0, [0, 0, 50.0], [0.0, 0.05, 0.0], sched(480, 60, 1.0), 480, seed=65,
                drone_options=dict(starting_fuel_ratio=1.0))
    # Rocket-Landing env (BASELINE configs[3]): randomised accelerated drops (options=None) and the plain drop ({})
    fly_landing("landing_random_drop", seed=71, n_steps=500, action_seed=8, options=None)
    fly_landing("landing_plain_euler", seed=72, n_steps=400, action_seed=9, options={}, angle_representation="euler", ignite_p=0.2)
    fly_landing("landing_sparse", seed=73, n_steps=300, action_seed=10, options=None, sparse=True, ignite_p=0.0)
    # unpowered plain drop straight onto the pad: pad-contact reward, fatal touchdown speed, next episode
    fly_landing("landing_pad_strike", seed=74, n_steps=450, action_seed=11, options={}, ignite_p=0.0)


def quadx_waypoints_fixtures():
    # QuadX-Waypoints (SURVEY 8f #1): rate mode with random actions (crashes, no targets), position mode chasing the
    # targets (reached targets, env_complete), yaw targets, euler + sparse
    fly_qx_waypoints("qxwp_mode0_random", seed=101, n_steps=300, action_seed=21, action_scale=0.3)
    fly_qx_waypoints("qxwp_mode7_chase", seed=102, n_steps=500, action_seed=22, flight_mode=7, chase=True, goal_reach_distance=0.3, num_targets=3)
    fly_qx_waypoints("qxwp_mode7_yaw_targets", seed=103, n_steps=500, action_seed=23, flight_mode=7, chase=True, use_yaw_targets=True,
                     goal_reach_distance=0.4, goal_reach_angle=0.3, num_targets=2)
    fly_qx_waypoints("qxwp_euler_sparse", seed=104, n_steps=200, action_seed=24, angle_representation="euler", sparse=True, action_scale=0.5)


def ma_hover_fixtures():
    # MAQuadXHover (SURVEY 8f #2): default 4 agents; crashes end agents one by one (dead agents keep falling)
    fly_ma_hover("mahover_mode0", seed=201, n_steps=160, action_seed=31)
    fly_ma_hover("mahover_euler_sparse", seed=203, n_steps=120, action_seed=32, angle_representation="euler", sparse=True, action_scale=0.5)
    fly_ma_hover("mahover_mode6_trunc", seed=205, n_steps=100, action_seed=33, flight_mode=6, max_duration_seconds=1.0, action_scale=0.1, dome=10.0)
    fly_ma_hover("mahover_two_agents_small_dome", seed=207, n_steps=140, action_seed=34, dome=2.0, start_pos=[[0.0, 0.0, 1.0], [0.5, 0.5, 1.5]])
    agent_rate_fixtures()


def agent_rate_fixtures():
    # agent rates other than 40 Hz: env_step_ratio 1 (an env step ends halfway through a Philox pair) and 5 (past the four
    # prefetched Aviary steps); a ragged 3-agent arena with euler observations, and mode 1, whose warm-up depends on its noise
    fly_ma_hover("mahover_hz120_three_euler", seed=209, n_steps=300, action_seed=35, angle_representation="euler", dome=2.0,
                 max_duration_seconds=1.5, start_pos=[[0.0, 0.0, 1.0], [1.0, 0.0, 1.5], [-0.5, 0.8, 0.8]], agent_hz=120)
    fly_ma_hover("mahover_hz24_mode1", seed=211, n_steps=90, action_seed=36, flight_mode=1, max_duration_seconds=2.0, dome=3.0, agent_hz=24)
    fly_hover("hover_hz24_mode1", seed=8, n_steps=120, action_seed=5, angle_representation="quaternion", flight_mode=1, action_scale=0.3, agent_hz=24)


def dogfight_fixtures():
    # MAFixedwingDogfight (BASELINE configs[4]): 1-vs-1 arenas; a wide lethal cone makes scripted flights score hits
    fly_dogfight("dogfight_1v1", seed=81, n_steps=260, action_seed=12)
    fly_dogfight("dogfight_1v1_wide_cone", seed=83, n_steps=260, action_seed=13, lethal_distance=150.0, lethal_angle=1.2, action_scale=0.3)
    fly_dogfight("dogfight_1v1_sparse", seed=85, n_steps=150, action_seed=14, sparse=True)
    # nose-down bias: ground collisions (-1000), the survivor's team win (+300), several episodes
    fly_dogfight("dogfight_1v1_crash", seed=91, n_steps=250, action_seed=17, action_scale=0.2, pitch_bias=0.8)
    # heavy damage in a 2-vs-2: deaths by health, team wins, dead agents that keep flying
    fly_dogfight("dogfight_2v2_lethal", seed=87, n_steps=200, action_seed=15, team_size=2, lethal_distance=120.0, lethal_angle=0.9, action_scale=0.3, damage_per_hit=0.05)
    fly_dogfight("dogfight_2v2", seed=87, n_steps=200, action_seed=15, team_size=2, lethal_distance=120.0, lethal_angle=0.9, action_scale=0.3)


def main():
    os.makedirs(OUT, exist_ok=True)
    # A: tests/test_core.py:13-31
    fly_quadx("quadx_mode7_hold", 7, "cf2x", [0, 0, 1], [0, 0, 0], {}, 1000, seed=1)
    # B: tests/test_core.py:65-93 / examples/core/03_control.py
    fly_quadx(
        "quadx_mode7_setpoints", 7, "cf2x", [0, 0, 1], [0, 0, 0],
        {0: [1.0, 0.0, 0.0, 1.0], 500: [0.0, 0.0, np.pi / 4, 2.0]}, 1000, seed=2,
    )
    # every flight mode, both quad models, a tilted start and setpoint changes
    sched = {
        -1: {0: [0.3, 0.31, 0.32, 0.3], 120: [0.5, 0.5, 0.45, 0.5]},
        0: {0: [0.3, -0.2, 0.1, 0.45], 150: [-0.5, 0.4, -0.3, 0.3]},
        1: {0: [0.2, -0.1, 0.5, 0.3], 150: [-0.2, 0.2, -0.5, -0.2]},
        2: {0: [0.2, -0.2, 0.3, 6.0], 150: [-0.3, 0.1, 0.0, 4.0]},
        3: {0: [0.15, -0.1, 0.6, 6.0], 150: [0.0, 0.0, -0.6, 4.5]},
        4: {0: [0.8, -0.5, 0.3, 6.0], 150: [-0.6, 0.4, -0.2, 4.5]},
        5: {0: [0.8, -0.5, 0.3, 0.4], 150: [-0.6, 0.4, -0.2, -0.3]},
        6: {0: [0.9, 0.4, 0.5, 0.3], 150: [-0.5, -0.7, -0.4, -0.2]},
        7: {0: [1.0, -1.0, 0.8, 6.0], 150: [-0.5, 0.5, -0.8, 4.0]},
    }
    for model in ["cf2x", "primitive_drone"]:
        for mode in range(-1, 8):
            fly_quadx(f"quadx_{model}_mode{mode}", mode, model, [0.3, -0.2, 5.0], [0.1, -0.15, 0.7], sched[mode], 300, seed=10 + mode)
    # floor strike: contact flag + "no rotational drag while in contact" (quadx.py:509-510)
    fly_quadx("quadx_floor_contact", 0, "cf2x", [0, 0, 0.3], [0.4, 0.2, 0], {0: [1.0, 2.0, 0.5, 0.05]}, 80, seed=3)
    # long open-sky parity scenario (SURVEY §8d config 1): 3000 Aviary steps = 1000 Hover env-steps
    prng = np.random.default_rng(1)
    sched0 = {}
    for k in range(0, 3000, 30):
        a = prng.uniform([-np.pi, -np.pi, -np.pi, 0.0], [np.pi, np.pi, np.pi, 0.8])
        a[:3] *= 0.3
        sched0[k] = a
    fly_quadx("quadx_mode0_long", 0, "cf2x", [0, 0, 50.0], [0, 0, 0], sched0, 3000, seed=4)
    # Hover env: tests/test_gym_envs.py:92-112 shape (seeded env + scripted actions)
    fly_hover("hover_quat_dense", seed=0, n_steps=400, action_seed=1, angle_representation="quaternion")
    fly_hover("hover_euler_sparse", seed=5, n_steps=200, action_seed=2, angle_representation="euler", sparse=True)
    fly_hover("hover_quat_gentle", seed=6, n_steps=450, action_seed=3, angle_representation="quaternion", action_scale=0.05, dome=50.0)
    fly_hover("hover_mode6", seed=7, n_steps=300, action_seed=4, angle_representation="quaternion", flight_mode=6, action_scale=0.3)


def wind_fixtures():
    """SURVEY 8f item 4: the UNMODIFIED reference flown in an analytic wind (register_wind_field_function, aviary.py:324-334;
    tests/test_core.py:262-290 of the reference does the same with exp(z))."""
    from pyflyt_b200.core.wind import AnalyticWind

    # QuadX, position hold in a power-law boundary layer; the drag body feels it, the controller leans into it
    fly_quadx("wind_quadx_power", 7, "cf2x", [0, 0, 2.0], [0, 0, 0.3], {0: [0.5, -0.5, 0.3, 3.0]}, 400, seed=71,
              wind=AnalyticWind("power", base=(3.0, -1.5, 0.2), z_ref=10.0, alpha=1.0 / 7.0))
    # Fixedwing in a logarithmic profile: every lifting surface sees the wind at its own altitude
    r = np.random.default_rng(72)
    sched = {k: np.concatenate([r.uniform(-0.4, 0.4, 3), r.uniform(0.4, 1.0, 1)]) for k in range(0, 500, 50)}
    fly_vehicle("wind_fixedwing_log", "fixedwing", "fixedwing", 0, [0, 0, 50.0], [0.05, -0.05, 0.4], sched, 500, seed=72,
                wind=AnalyticWind("log", base=(-4.0, 2.0, 0.0), z_ref=10.0, z0=0.03))
    # Rocket: the reference test's own field shape, wind_z = exp(z / z_ref), plus a constant cross wind on a second fixture
    def sched_r(n, every, thr):
        rr = np.random.default_rng(73)
        return {k: np.concatenate([rr.uniform(-0.5, 0.5, 3), [1.0, thr], rr.uniform(-0.5, 0.5, 2)]) for k in range(0, n, every)}
    fly_vehicle("wind_rocket_exp", "rocket", "rocket", 0, [0, 0, 100.0], [0.05, -0.04, 0.3], sched_r(400, 40, 0.8), 400, seed=73,
                wind=AnalyticWind("exp", base=(0.0, 0.0, 1.0), z_ref=60.0))
    fly_vehicle("wind_rocket_constant", "rocket", "rocket", 0, [0, 0, 200.0], [0.1, 0.0, 0.0], sched_r(300, 30, 0.5), 300, seed=74,
                wind=AnalyticWind("constant", base=(6.0, -3.0, 0.5)))
    # one env: QuadX-Hover, a single episode with the field attached to the env's Aviary after reset()
    fly_hover("wind_hover_quat", seed=75, n_steps=80, action_seed=6, angle_representation="quaternion", flight_mode=6, action_scale=0.2, dome=50.0,
              wind=AnalyticWind("constant", base=(2.0, 1.0, 0.0)))


# ---- static bodies (DESIGN.md §4h) ----------------------------------------------------------------------------------------
STATIC_DIR = os.path.join(OUT, "static")


def _static_prims(s):
    """(top, footprint test) of every collision primitive of the fixed-base body s, world frame (fakebullet's pose of s is its base
    inertial frame, the primitives' offsets are relative to it)"""
    Rs = s.R()
    out = []
    for lk in s.links:
        for kind, dims, cr, cR in lk.shapes:
            if kind not in ("box", "cylinder"):
                raise ValueError(f"static body {s.path}: a {kind} (boxes and cylinders only)")
            centre = s.pos + Rs @ cr
            Rw = Rs @ cR
            if kind == "box":
                top = centre[2] + 0.5 * dims[2]
                inside = (lambda c, R, h: lambda x, y: abs(R[0, 0] * (x - c[0]) + R[1, 0] * (y - c[1])) <= h[0]
                          and abs(R[0, 1] * (x - c[0]) + R[1, 1] * (y - c[1])) <= h[1])(centre, Rw, 0.5 * np.asarray(dims))
            else:
                top = centre[2] + 0.5 * dims[1]
                inside = (lambda c, r: lambda x, y: (x - c[0]) ** 2 + (y - c[1]) ** 2 <= r * r)(centre, dims[0])
            out.append((top, inside))
    return out


def _reach(b):
    """the model's contact reach about its base origin: contact_zmax / ContactParams::zmax of the library (pfb_quadx_host.h)"""
    r = 0.0
    for lk in b.links:
        for kind, dims, cr, cR in lk.shapes:
            if kind == "box":
                disc = float(np.linalg.norm(0.5 * np.asarray(dims)))
            elif kind == "cylinder":
                disc = float(np.hypot(dims[0], 0.5 * dims[1]))
            elif kind == "sphere":
                disc = float(dims[0])
            else:
                continue
            r = max(r, (float(np.linalg.norm(cr)) + disc + 0.02 * disc) * 1.001)
    return r


def _tops_under(b, s):
    """tops of the primitives of static body s under free body b: footprint holds the base's (x, y), and z + R_b >= top"""
    x, y, z = b.pos
    return [top for top, inside in _static_prims(s) if inside(x, y) and z + _reach(b) >= top]


class static_rule:
    """The fake client's contact detection and response surface with the static-body rule of DESIGN.md §4h (boxes yawed, the
    height guard, one contact pair per static body), for the fixtures of this group only; oracle/fakebullet keeps its own
    (the untilted cylinder pad of Rocket-Landing) for every other fixture."""

    def __enter__(self):
        import pybullet as fb

        self.fb, self.saved = fb, (fb.World._detect_contacts, fb.World._surface_height)

        def detect(world):
            world.contacts = []
            statics = [s for s in world.bodies.values() if s.fixed_base]
            for b in world.bodies.values():
                if b.fixed_base:
                    continue
                low = b.lowest_point_and_threshold()
                if low is None:
                    continue
                z, thr = low
                for s in statics:
                    if s.is_plane:
                        top = s.pos[2]
                    else:
                        tops = _tops_under(b, s)
                        if not tops:
                            continue
                        top = max(tops)
                    if z - top < thr:
                        world.contacts.append((0, s.uid, b.uid, -1, -1))
                        world.contacts.append((0, b.uid, s.uid, -1, -1))

        def surface(world, b):
            tops = [0.0]
            for s in world.bodies.values():
                if s.fixed_base and not s.is_plane:
                    tops += _tops_under(b, s)
            return max(tops)

        fb.World._detect_contacts, fb.World._surface_height = detect, surface
        fb.World.contact_response = True
        return self

    def __exit__(self, *exc):
        self.fb.World._detect_contacts, self.fb.World._surface_height = self.saved
        self.fb.World.contact_response = False


def fly_static(name, drone_type, drone_options, start_pos, start_orn, mode, bodies, setpoint_schedule, n_steps, seed, poses=None):
    """Each drone in a reference Aviary of its own (its own world), with the static bodies `bodies` = [(urdf file under
    tests/golden/static, basePosition, baseOrientation)] loaded by aviary.loadURDF(useFixedBase=True) and
    register_all_new_bodies(); poses[i] = {body: (pos, quat)} moves body k of drone i's world with resetBasePositionAndOrientation
    (its base inertial frame) before the flight.  Records per drone and step the state, aux state and contact_array[drone.Id, body]
    (bit 0 the floor, bit 1 + k body k) and the raw draws of each world, which the replays inject."""
    n = len(start_pos)
    states, auxs, bits, raws, noises = [], [], [], [], []
    for i in range(n):
        rng = ril.ScriptedNoise(seed + i)
        env = Aviary(start_pos=np.array([start_pos[i]], dtype=np.float64), start_orn=np.array([start_orn[i]], dtype=np.float64),
                     drone_type=drone_type, drone_options=dict(drone_options), np_random=rng)
        ids = [env.loadURDF(os.path.join(STATIC_DIR, f), basePosition=p, baseOrientation=q, useFixedBase=True) for f, p, q in bodies]
        env.register_all_new_bodies()
        for k, (pos, quat) in (poses[i] if poses else {}).items():
            env.resetBasePositionAndOrientation(ids[k], pos, quat)
        env.set_mode(mode)
        d = env.drones[0]
        st, ax, bt, rw = [], [], [], []
        for t in range(n_steps):
            if t in setpoint_schedule:
                env.set_setpoint(0, np.array(setpoint_schedule[t][i] if isinstance(setpoint_schedule[t], dict) else setpoint_schedule[t], dtype=np.float64))
            env.step()
            st.append(np.array(d.state))
            ax.append(np.array(d.aux_state, dtype=np.float64))
            row = env.contact_array[d.Id]
            bt.append(int(row[env.planeId]) | sum(int(row[bid]) << (1 + k) for k, bid in enumerate(ids)))
            pos, quat = env.getBasePositionAndOrientation(d.Id)
            v, w = env.getBaseVelocity(d.Id)
            rw.append(np.concatenate([pos, quat, v, w]))
        states.append(st), auxs.append(ax), bits.append(bt), raws.append(rw), noises.append(np.array(rng.normal_log))
    sched = {str(k): (v if not isinstance(v, dict) else {str(a): list(b) for a, b in v.items()}) for k, v in setpoint_schedule.items()}
    np.savez_compressed(
        os.path.join(OUT, f"{name}.npz"),
        drone_type=drone_type, drone_options=json.dumps(drone_options), mode=mode,
        start_pos=np.array(start_pos, dtype=np.float64), start_orn=np.array(start_orn, dtype=np.float64),
        bodies=json.dumps([(f, list(p), list(q)) for f, p, q in bodies]),
        poses=json.dumps([{str(k): (list(p), list(q)) for k, (p, q) in pz.items()} for pz in poses] if poses else []),
        setpoints=json.dumps({k: np.asarray(v, dtype=np.float64).tolist() if not isinstance(v, dict) else v for k, v in sched.items()}),
        noise=np.stack(noises, axis=-1),  # [draws][n]
        state=np.array(states).transpose(1, 0, 2, 3), aux=np.array(auxs).transpose(1, 0, 2), bits=np.array(bits, dtype=np.uint32).T,
        raw=np.array(raws).transpose(1, 0, 2),
    )
    print(name, "final pos", [s[-1][3] for s in states], "bits", [b[-1] for b in bits], "draws", noises[0].shape)


def static_fixtures():
    """The unmodified reference Aviary with fixed-base bodies (loadURDF + register_all_new_bodies), read through
    contact_array[drone.Id, body], on the fake client with the static-body rule and the contact response (static_rule)."""
    yaw30 = [0.0, 0.0, np.sin(np.pi / 12), np.cos(np.pi / 12)]
    cf2x = dict(drone_model="cf2x")
    with static_rule():
        # cf2x in mode 7: take off from a 1 m platform, cross to a second one yawed 30 degrees, land on it and rest
        fly_static("static_cf2x_platform_hop", "quadx", cf2x, [[0.0, 0.0, 1.02]], [[0.0, 0.0, 0.0]], 7,
                   [("platform_box.urdf", [0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 1.0]), ("platform_box.urdf", [3.0, 1.5, 0.0], yaw30)],
                   {0: [0.0, 0.0, 0.0, 2.0], 240: [3.0, 1.5, 0.0, 2.0], 600: [3.0, 1.5, 0.0, 0.5]}, 960, seed=401)
        # primitive_drone dropped tilted, half over a platform's edge (motors idle)
        fly_static("static_primitive_edge_drop", "quadx", dict(drone_model="primitive_drone"), [[1.0, 0.3, 2.2]], [[0.4, 0.2, 0.0]], -1,
                   [("platform_box.urdf", [0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 1.0])], {0: [0.0, 0.0, 0.0, 0.0]}, 480, seed=402)
        # cf2x flying beside a 4 m tower (30 degrees yawed box) and under its 1.5 m helipad, never touching either
        fly_static("static_cf2x_beside_under", "quadx", cf2x, [[1.0, 0.0, 1.0]], [[0.0, 0.0, 0.0]], 7,
                   [("helipad_tower.urdf", [0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 1.0])],
                   {0: [1.0, 0.0, 0.0, 3.0], 200: [0.0, 1.0, 0.0, 3.5], 400: [-0.8, -0.8, 0.0, 2.0]}, 600, seed=403)
        # fixed-wing gliding onto a runway box, throttle off
        fly_static("static_fixedwing_runway", "fixedwing", dict(drone_model="fixedwing"), [[0.0, 0.0, 1.5]], [[0.0, 0.0, 0.0]], 0,
                   [("runway.urdf", [45.0, 0.0, 0.0], [0.0, 0.0, np.sin(np.pi / 180), np.cos(np.pi / 180)])],
                   {0: [0.0, -0.1, 0.0, 0.0]}, 600, seed=404)
        # rocket dropped onto a pad off the origin, booster off
        fly_static("static_rocket_pad", "rocket", dict(drone_model="rocket"), [[6.3, -4.2, 5.0]], [[0.0, 0.0, 0.0]], 0,
                   [("pad_cylinder.urdf", [6.0, -4.0, 0.0], [0.0, 0.0, 0.0, 1.0])], {0: [0, 0, 0, 0, 0, 0, 0]}, 480, seed=405)
        # per-drone poses: three worlds, the platform moved by resetBasePositionAndOrientation (base inertial frame) in each,
        # cf2x descending onto it near the rotated footprint's edge
        poses = [{0: ([0.5, 0.0, 0.5], [0.0, 0.0, np.sin(0.3), np.cos(0.3)])},
                 {0: ([-1.0, 2.0, 1.0], [0.0, 0.0, np.sin(-0.6), np.cos(-0.6)])},
                 {0: ([2.0, -1.0, 0.2], [0.0, 0.0, np.sin(0.9), np.cos(0.9)])}]
        starts = [[1.2, 0.6, 2.0], [-0.3, 2.6, 2.5], [2.9, -0.4, 1.6]]
        fly_static("static_cf2x_per_drone_poses", "quadx", cf2x, starts, [[0.0, 0.0, 0.0]] * 3, 7,
                   [("platform_box.urdf", [0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 1.0])],
                   {0: {i: [starts[i][0], starts[i][1], 0.0, 0.3] for i in range(3)}}, 600, seed=406, poses=poses)


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    if which in ("all", "quadx"):
        main()
    if which in ("all", "fixedwing"):
        fixedwing_fixtures()
    if which in ("all", "rocket"):
        rocket_fixtures()
    if which in ("all", "dogfight"):
        dogfight_fixtures()
    if which in ("all", "mahover"):
        ma_hover_fixtures()
    if which == "agentrates":  # (included in "mahover")
        agent_rate_fixtures()
    if which in ("all", "qxwp"):
        quadx_waypoints_fixtures()
    if which in ("all", "wind"):
        wind_fixtures()
    if which in ("all", "touchdown"):
        touchdown_fixtures()
    if which in ("all", "mixed"):
        mixed_model_fixtures()
    if which in ("all", "mixedmodes"):
        mixed_mode_fixtures()
    if which in ("all", "ground"):
        ground_fixtures()
    if which in ("all", "mixedkinds"):
        mixed_kind_fixtures()
    if which in ("all", "rates"):
        rate_fixtures()
    if which in ("all", "basestate"):
        base_state_fixtures()
    if which in ("all", "static"):
        static_fixtures()
