"""Drones at different control rates in one batch: ``BatchedAviary(..., mixed_control_hz=True)`` with per-drone
``drone_options`` ``control_hz`` (the reference's tests/test_core.py::test_multi_spawn, examples/core/02_multi_drone.py).

An Aviary step is U = physics_hz / min(control_hz) physics substeps; a drone with r = physics_hz / control_hz runs its control
tick before substep u when u % r == 0 (aviary.py:287-298, 506-529).  Such a drone is the reference drone at its own rate: U / r
Aviary steps of that rate, each on r draws of its column.

CPU: the argument checks and their messages for the Python builders and for pfb_create_mixed, the tables and their order, and
one oracle per drone, composed as above, against the unmodified reference (tests/golden/rates_*.npz, tools/gen_golden.py rates).
GPU: one handle replays the fixtures; a drone of a multi-rate handle is bit for bit the same drone in a handle at its own rate
(injected noise), and the slowest drones bit for bit with Philox noise; one launch per step; 65 536 drones; test_multi_spawn."""
import ctypes as C
import json
import re

import numpy as np
import pytest

from engines import OracleEngine, load_golden
from pyflyt_b200.models import ModelSetError, PfbEnvConfig, PfbModel, build_mixed_model_set, build_model, build_model_set
from test_mixed_kinds import AUX_DIM, HEIGHT_HOLD, SP_DIM, MixedKindEngine, _mode_at, replay_kinds

FIXTURES = ["rates_multi_spawn", "rates_models_modes", "rates_kinds_interleaved", "rates_thirds"]
CF2X, PRIM = dict(drone_model="cf2x"), dict(drone_model="primitive_drone")


def _bytes(m):
    return C.string_at(C.addressof(m), C.sizeof(m))


def _kinds(g):
    return json.loads(str(g["drone_type"]))


def _ratios(opts, physics_hz=240):
    return [physics_hz // int(o.get("control_hz", 120)) for o in opts]


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_model_set_rate_checks():
    rates = lambda *hz: [dict(CF2X, control_hz=h) for h in hz]  # noqa: E731
    # without the option: refused, and the message names the option
    with pytest.raises(ModelSetError, match="control_hz.*mixed_control_hz=True"):
        build_model_set("quadx", rates(60, 120), 240, 2)
    with pytest.raises(ModelSetError, match="control_hz"):
        build_mixed_model_set(["quadx", "rocket"], [dict(control_hz=60), dict(control_hz=120)], 240, 2)
    # the reference's messages and exception types (base_drone.py:94-97, aviary.py:293-298)
    with pytest.raises(AssertionError, match=re.escape("Looprates must form common multiples of each other.")):
        build_model_set("quadx", rates(80, 120), 240, 2, mixed_control_hz=True)
    with pytest.raises(AssertionError, match="Looprates"):
        build_mixed_model_set(["quadx", "fixedwing"], [dict(control_hz=80), dict(control_hz=120)], 240, 2, mixed_control_hz=True)
    with pytest.raises(ValueError, match=re.escape("`physics_hz` (240) must be multiple of `control_hz` (100).")):
        build_model_set("quadx", rates(100, 120), 240, 2, mixed_control_hz=True)
    # at most four physics steps per Aviary step: {30, 120} Hz at 240 Hz needs 8
    with pytest.raises(ModelSetError, match=re.escape("is 8 physics steps; a batch runs at most 4")):
        build_model_set("quadx", rates(30, 120), 240, 2, mixed_control_hz=True)
    with pytest.raises(ModelSetError, match="at most 4"):
        build_mixed_model_set(["quadx", "rocket"], [dict(control_hz=240), dict(control_hz=30)], 240, 2, mixed_control_hz=True)
    # one fixed-wing / rocket model, at one or several rates
    with pytest.raises(ModelSetError, match="one vehicle model"):
        build_model_set("fixedwing", [dict(drone_model="fixedwing", control_hz=60), dict(drone_model="acrowing", control_hz=120)], 240, 2,
                        mixed_control_hz=True)


def test_rate_model_sets_tables_index_and_dedup():
    # QuadX: one table per (model, rate), in the order the entries first name them
    tables, index = build_model_set("quadx", [dict(CF2X, control_hz=60), dict(CF2X, control_hz=120), dict(control_hz=60), dict(PRIM, control_hz=240)],
                                    240, 4, mixed_control_hz=True)
    assert [int(t.control_hz) for t in tables] == [60, 120, 240] and index.tolist() == [0, 1, 0, 2]
    assert _bytes(tables[1]) == _bytes(build_model("quadx", "cf2x", control_hz=120))
    assert _bytes(tables[2]) == _bytes(build_model("quadx", "primitive_drone", control_hz=240))
    # fixed-wing: one model at two rates is two tables, byte-equal apart from control_hz
    tables, index = build_model_set("fixedwing", [dict(control_hz=60), dict(control_hz=120), dict(drone_model="fixedwing", control_hz=60)], 240, 3,
                                    mixed_control_hz=True)
    assert [int(t.control_hz) for t in tables] == [60, 120] and index.tolist() == [0, 1, 0]
    a, b = PfbModel.from_buffer_copy(tables[0]), PfbModel.from_buffer_copy(tables[1])
    a.control_hz = b.control_hz = 0.0
    assert _bytes(a) == _bytes(b)
    # several kinds: the QuadX tables, then the fixed-wing ones, then the rocket ones, each kind in its own first-use order
    kinds = ["rocket", "quadx", "fixedwing", "quadx", "rocket", "fixedwing", "quadx"]
    opts = [dict(control_hz=240), dict(control_hz=60), dict(control_hz=120), dict(PRIM, control_hz=120), dict(control_hz=120), dict(control_hz=60),
            dict(control_hz=60)]
    tables, index = build_mixed_model_set(kinds, opts, 240, 7, mixed_control_hz=True)
    assert [(int(t.kind), int(t.control_hz)) for t in tables] == [(0, 60), (0, 120), (1, 120), (1, 60), (2, 240), (2, 120)]
    assert index.tolist() == [4, 0, 2, 1, 5, 3, 0] and index.dtype == np.uint8
    # equal rates with the option: the tables built without it
    for kw in ({}, dict(mixed_control_hz=True)):
        t, i = build_mixed_model_set(["quadx", "rocket"], [dict(control_hz=60), dict(control_hz=60)], 240, 2, **kw)
        assert [_bytes(m) for m in t] == [_bytes(build_model("quadx", control_hz=60)), _bytes(build_model("rocket", control_hz=60))] and i.tolist() == [0, 1]


def test_aviary_checks_rates_before_the_device():
    from pyflyt_b200.core.aviary import AviaryInitException, BatchedAviary

    z = np.zeros((3, 3))
    spawn = [dict(control_hz=60), dict(control_hz=120), dict(control_hz=240)]
    with pytest.raises(AviaryInitException, match="control_hz"):
        BatchedAviary(z, z, drone_options=spawn)
    with pytest.raises(AviaryInitException, match="env_config"):
        BatchedAviary(z, z, drone_options=spawn, env_config=PfbEnvConfig(), mixed_control_hz=True)
    with pytest.raises(AssertionError, match="Looprates must form common multiples of each other."):
        BatchedAviary(z, z, drone_options=[dict(control_hz=80), dict(control_hz=120), {}], mixed_control_hz=True)
    with pytest.raises(AviaryInitException, match="at most 4"):
        BatchedAviary(z, z, drone_type=["quadx", "rocket", "fixedwing"], drone_options=[dict(control_hz=30), {}, {}], mixed_control_hz=True)


def _lib_or_skip():
    from pyflyt_b200 import _lib

    try:
        return _lib, _lib.lib()
    except _lib.PfbError as e:
        pytest.skip(str(e))


def test_create_mixed_rate_refusals():
    import torch

    _lib, L = _lib_or_skip()
    err = lambda: L.pfb_last_error().decode()  # noqa: E731
    cfg = PfbEnvConfig()
    cfg.mixed_control_hz = 1

    def create(models, index, flag=True):
        tables = (PfbModel * len(models))(*models)
        idx = np.ascontiguousarray(index, dtype=np.uint8)
        h = C.c_void_p()
        rc = L.pfb_create_mixed(tables, len(models), idx.ctypes.data_as(C.c_void_p), len(idx), C.byref(cfg) if flag else None, 0, 1, C.byref(h))
        return rc, h

    q = lambda hz, model="cf2x", phys=240: build_model("quadx", model, physics_hz=phys, control_hz=hz)  # noqa: E731
    f = lambda hz, model="fixedwing": build_model("fixedwing", model, control_hz=hz)  # noqa: E731
    r = lambda hz: build_model("rocket", "rocket", control_hz=hz)  # noqa: E731
    rc, _ = create([q(60), q(120)], [0, 1], flag=False)  # without the flag: today's refusal
    assert rc != 0 and "every drone of a handle needs the same physics_hz and control_hz" in err()
    rc, _ = create([q(120), q(120, phys=480)], [0, 1])
    assert rc != 0 and "every drone of a handle needs the same physics_hz" in err()
    rc, _ = create([q(80), f(120)], [0, 1])
    assert rc != 0 and "Looprates must form common multiples of each other." in err()
    rc, _ = create([q(30), q(120)], [0, 1])
    assert rc != 0 and "= 8 physics substeps per Aviary step; a handle runs at most 4" in err()
    rc, _ = create([q(60), f(60), f(120, "acrowing")], [0, 1, 2])
    assert rc != 0 and "fixed-wing tables 1 and 2 differ beyond control_hz" in err()
    rc, _ = create([r(120), q(60), r(120)], [0, 1, 2])
    assert rc != 0 and "rocket tables 0 and 2 are identical" in err()
    rc, h = create([q(60), q(120, "primitive_drone"), f(60), f(120), r(240), r(120)], [5, 0, 2, 1, 3, 4])
    if torch.cuda.is_available():
        assert rc == 0, err()
        L.pfb_destroy(h)
    else:  # well-formed input: the device lookup is what fails
        assert rc != 0 and "no CPU fallback" in err()


class RateOracle:
    """One oracle per drone at the drone's own rate: an Aviary step of U substeps is U / r of its Aviary steps, each on r draws
    of its column; the contact flag is raised by any of them."""

    def __init__(self, g):
        kinds, opts = _kinds(g), json.loads(str(g["drone_options"]))
        self.kinds, self.ratios = kinds, _ratios(opts)
        self.U = max(self.ratios)
        self.engines = [OracleEngine(build_model(k, o.get("drone_model"), control_hz=int(o.get("control_hz", 120))), None, 1, g["start_pos"][d][None],
                                     g["start_orn"][d][None]) for d, (k, o) in enumerate(zip(kinds, opts))]
        self._contact = np.zeros(len(kinds), dtype=bool)

    def reset(self):
        for e in self.engines:
            e.reset()

    def set_modes(self, modes):
        for e, m in zip(self.engines, modes):
            e.set_mode(int(m))

    def get_setpoints(self):
        out = np.zeros((len(self.engines), 7))
        for d, (e, k) in enumerate(zip(self.engines, self.kinds)):
            out[d, : SP_DIM[k]] = e.o.get_setpoints(SP_DIM[k])[0]
        return out

    def set_setpoints(self, sp):
        for d, (e, k) in enumerate(zip(self.engines, self.kinds)):
            e.set_setpoints(np.asarray(sp[d][: SP_DIM[k]])[None])

    def aviary_step(self, noise):
        assert noise.shape[0] == self.U
        for d, (e, r) in enumerate(zip(self.engines, self.ratios)):
            self._contact[d] = False
            for k in range(self.U // r):
                e.aviary_step(noise[k * r : (k + 1) * r, d][:, None])
                self._contact[d] |= bool(e.contact()[0])

    def state(self):
        return np.concatenate([e.state() for e in self.engines])

    def aux(self):
        out = np.zeros((len(self.engines), 9))
        for d, (e, k) in enumerate(zip(self.engines, self.kinds)):
            out[d, : AUX_DIM[k]] = e.aux()[0]
        return out

    def contact(self):
        return self._contact.copy()


def test_fixtures_cover_the_rates_and_stay_off_the_floor():
    for name in FIXTURES:
        g = load_golden(name)
        opts = json.loads(str(g["drone_options"]))
        ratios = _ratios(opts)
        assert len(set(ratios)) > 1 and not g["contact"].any(), name
        assert g["noise"].size == len(g["state"]) * max(ratios) * int(g["n_drones"])  # one draw per drone per physics step, whatever its rate
    assert sorted(set(_ratios(json.loads(str(load_golden("rates_thirds")["drone_options"]))))) == [1, 3]
    g = load_golden("rates_kinds_interleaved")
    per_kind = {}
    for k, o in zip(_kinds(g), json.loads(str(g["drone_options"]))):
        per_kind.setdefault(k, set()).add(o["control_hz"])
    assert per_kind == {"quadx": {60, 120, 240}, "fixedwing": {60, 120}, "rocket": {120, 240}}


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_reference_rates(name):
    """Each drone of the reference's multi-rate Aviary, replayed by an oracle at its own rate (the bars of
    test_mixed_kinds.py::test_oracle_reproduces_reference_mixed_kinds: 1e-9, 1e-6 for drones that hold height)."""
    g = load_golden(name)
    err = replay_kinds(g, RateOracle(g))
    loose = np.isin(_mode_at(g), HEIGHT_HOLD).any(axis=0)
    assert err["contact_mismatch"].sum() == 0
    for k in ("setpoint", "pos", "euler", "angvel", "linvel", "aux"):
        assert err[k][~loose].max(initial=0.0) < 1e-9, (name, k, err[k])
        assert err[k][loose].max(initial=0.0) < 1e-6, (name, k, err[k])


# ------------------------------------------------------------------------------------------------------------------ GPU
class OwnRateHandles:
    """Every drone of a fixture in a mixed handle where every drone runs at its rate c: U / r_c Aviary steps of it per step of
    the fixture.  A rocket far above the floor joins the drones, so that a handle of QuadX only is a mixed handle as well and
    flies the step kernel of the multi-rate handle, only without several rates."""

    def __init__(self, g):
        from pyflyt_b200.core.aviary import BatchedAviary

        self.kinds, opts = _kinds(g), json.loads(str(g["drone_options"]))
        self.n = len(self.kinds)
        self.rates = np.array([240 // r for r in _ratios(opts)])
        self.U = 240 // int(self.rates.min())
        pos = np.vstack([g["start_pos"], [[0.0, 0.0, 500.0]]]).astype(np.float32)
        orn = np.vstack([g["start_orn"], [[np.pi / 2, 0.0, 0.0]]]).astype(np.float32)
        self.avs = {}
        for c in sorted(set(self.rates.tolist())):
            self.avs[c] = BatchedAviary(pos, orn, drone_type=self.kinds + ["rocket"], drone_options=[dict(o, control_hz=c) for o in opts] + [dict(control_hz=c)])

    def _rows(self, get):
        out = None
        for c, a in self.avs.items():
            v = get(a)[: self.n]
            out = v.copy() if out is None else out
            out[self.rates == c] = v[self.rates == c]
        return out

    def reset(self):
        for a in self.avs.values():
            a.reset()

    def set_modes(self, modes):
        for a in self.avs.values():
            a.set_mode([int(m) for m in modes] + [0])

    def get_setpoints(self):
        return self._rows(lambda a: a.setpoints.cpu().double().numpy())

    def set_setpoints(self, sp):
        for a in self.avs.values():
            a.set_all_setpoints(np.vstack([np.asarray(sp, dtype=np.float32), np.zeros((1, 7), dtype=np.float32)]))

    def aviary_step(self, noise):
        import torch

        nz = torch.as_tensor(np.hstack([noise, np.zeros((self.U, 1))]).astype(np.float32), device="cuda")
        for a in self.avs.values():  # one launch, as the multi-rate handle: a launch carries part of the state in registers
            a.step(self.U // a.updates_per_step, nz)

    def contact(self):  # the last Aviary step of each rate (the fixtures never touch the floor)
        return self._rows(lambda a: a.contact_array.cpu().numpy())

    def state(self):
        return self._rows(lambda a: a.all_states.cpu().double().numpy())

    def aux(self):
        def aux(a):
            a.all_states  # refreshes the observed state
            return a._aux_state.cpu().double().numpy()

        return self._rows(aux)


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_cuda_replays_rate_fixture(name):
    """ONE CUDA handle flies the reference's drones at their several rates.  Every drone flies bit for bit what it flies in a
    handle where every drone runs at its rate (OwnRateHandles: the errors against the reference are the same numbers), and a
    drone that keeps one mode and does not hold position below 120 Hz is within the 1e-3 m of test_mixed_kinds.py::test_cuda_replays_mixed_kind_fixture.  A QuadX
    in mode 7 below 120 Hz (the test_multi_spawn drone at 60 Hz: 3.4 cm; primitive_drone 7 -> 0 at 60 Hz: 24 cm) rings and
    amplifies fp32 rounding, as test_mixed_modes.py documents for single-rate handles, and a drone that changes mode is held to
    5e-3 m (3.4e-3 measured: primitive_drone -1 -> 2 at 240 Hz, a tumbling raw-PWM phase before the height hold); the fp64
    oracle follows the reference to 1e-9 m on the same drones (test_oracle_reproduces_reference_rates)."""
    g = load_golden(name)
    eng = MixedKindEngine(g, mixed_control_hz=True)
    opts = json.loads(str(g["drone_options"]))
    ratios = _ratios(opts)
    assert eng.av.updates_per_step == max(ratios) and eng.av.control_hz.tolist() == [240 // r for r in ratios]
    err = replay_kinds(g, eng)
    own = replay_kinds(g, OwnRateHandles(g))
    for k in err:
        assert np.array_equal(err[k], own[k]), (name, k, err[k], own[k])
    kinds = np.array(_kinds(g))
    print(f"\n[{name}] max |pos - reference| per drone: {np.array2string(err['pos'], precision=2)}")
    assert err["contact_mismatch"].sum() == 0, err["contact_mismatch"]
    assert err["setpoint"].max() < 1e-5, err["setpoint"]
    slow_hold = np.array([k == "quadx" and o.get("control_hz", 120) < 120 for k, o in zip(kinds, opts)]) & (g["modes"] == 7).any(axis=0)
    steady = (g["modes"] == g["modes"][0]).all(axis=0) & ~slow_hold
    assert err["pos"][steady].max(initial=0.0) < 1e-3, err["pos"]
    assert err["pos"][~steady & ~slow_hold].max(initial=0.0) < 5e-3, err["pos"]  # after a set_mode(list): measured 3.4e-3
    assert err["euler"][steady & (kinds != "quadx")].max(initial=0.0) < 1e-3, err["euler"]


RATE_HZ = {"quadx": (60, 120, 240), "fixedwing": (60, 120), "rocket": (120, 240)}


def _rate_setup(n, seed, contact=False):
    """kinds, rates and modes interleaved lane by lane and tile by tile; the setpoints of test_mixed_kinds.py"""
    from test_mixed_kinds import _mixed_setup

    kinds, opts, start, orn, modes, sp = _mixed_setup(n, seed)
    hz = [RATE_HZ[k][(i + i // 32) % len(RATE_HZ[k])] for i, k in enumerate(kinds)]
    opts = [dict(o, control_hz=h) for o, h in zip(opts, hz)]
    if contact:  # dropped onto the floor from low heights (test_mixed_kinds.py::test_mixed_handle_bit_equal_to_single_kind_handles)
        start[:, 2] = np.random.default_rng(1).uniform(0.3, 2.0, n).astype(np.float32)
        rk = np.array(kinds) == "rocket"
        start[rk, 2] = (2.425 + np.random.default_rng(2).uniform(0.05, 2.0, int(rk.sum()))).astype(np.float32)
        orn[rk, :2] = 0.0
        sp[rk] = 0.0
    return kinds, opts, np.array(hz), start, orn, modes, sp


@pytest.mark.gpu
@pytest.mark.parametrize("contact", [False, True])
def test_multi_rate_drone_bit_equal_to_its_own_rate(contact):
    """Injected noise: a drone at rate c of a multi-rate handle (U = 4), stepped t times, holds the state words of the same drone in
    a handle at c stepped t * U / r_c times on the same column of draws, at every step boundary; every kind, several modes."""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    n, steps = 1024 + 45, 40
    kinds, opts, hz, start, orn, modes, sp = _rate_setup(n, 8, contact)
    multi = BatchedAviary(start, orn, drone_type=kinds, drone_options=opts, seed=2, contact_response=contact, mixed_control_hz=True)
    U = multi.updates_per_step
    assert U == 4 and multi.control_hz.tolist() == hz.tolist()
    single = {c: BatchedAviary(start, orn, drone_type=kinds, drone_options=[dict(o, control_hz=c) for o in opts], seed=2, contact_response=contact)
              for c in sorted(set(hz.tolist()))}
    for a in [multi] + list(single.values()):
        a.set_mode(modes)
        a.set_all_setpoints(sp)
    rng = np.random.default_rng(3)
    noise = rng.normal(0.0, 1.0, (steps * U, n)).astype(np.float32)
    noise[:, np.array(kinds) == "quadx"] += 4.0
    nz = torch.as_tensor(noise, device="cuda")
    touched = torch.zeros(n, dtype=torch.bool, device="cuda")
    for t in range(steps):
        chunk = nz[t * U : (t + 1) * U].contiguous()
        multi.step(1, chunk)
        s, aux, pos = multi.all_states.clone(), multi._aux_state.clone(), multi.precise_positions.clone()
        touched |= multi.contact_array
        for c, a in single.items():
            a.step(U // (240 // c), chunk)
            m = torch.as_tensor(hz == c, device="cuda")
            assert torch.equal(s[m], a.all_states[m]), (t, c)
            assert torch.equal(aux[m], a._aux_state[m]), (t, c)
            assert torch.equal(pos[m], a.precise_positions[m]), (t, c)
            if c == 60:  # the slowest drones' Aviary step is the handle's: the contact flags agree too
                assert torch.equal(multi.contact_array[m], a.contact_array[m]), (t, c)
    assert bool(torch.isfinite(multi.all_states).all())
    if contact:
        for k in ("quadx", "fixedwing", "rocket"):
            assert bool(touched[torch.as_tensor(np.array(kinds) == k, device="cuda")].any()), k


@pytest.mark.gpu
def test_slowest_drones_bit_equal_with_philox():
    """Philox noise is keyed by (seed, drone, Aviary step, substep) with the handle's U: the drones at the slowest rate of a
    multi-rate handle are bit for bit the same drones of a handle where every drone runs at that rate (same seed, same U)."""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    n = 2048 + 19
    kinds, opts, hz, start, orn, modes, sp = _rate_setup(n, 4)
    multi = BatchedAviary(start, orn, drone_type=kinds, drone_options=opts, seed=9, mixed_control_hz=True)
    slow = BatchedAviary(start, orn, drone_type=kinds, drone_options=[dict(o, control_hz=60) for o in opts], seed=9)
    assert multi.updates_per_step == slow.updates_per_step == 4
    for a in (multi, slow):
        a.set_mode(modes)
        a.set_all_setpoints(sp)
        a.step(150)
    torch.cuda.synchronize()
    m = torch.as_tensor(hz == 60, device="cuda")
    assert int(m.sum()) > 100
    assert torch.equal(multi.all_states[m], slow.all_states[m]) and torch.equal(multi._aux_state[m], slow._aux_state[m])
    assert torch.equal(multi.precise_positions[m], slow.precise_positions[m])
    assert not torch.equal(multi.all_states[~m], slow.all_states[~m])  # the faster drones fly differently


@pytest.mark.gpu
def test_one_launch_per_step_and_surface():
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    pos = np.array([[-1.0, 0.0, 1.0], [0.0, 0.0, 1.0], [1.0, 0.0, 1.0]])
    av = BatchedAviary(pos, np.zeros_like(pos), drone_options=[dict(control_hz=60), dict(control_hz=120), dict(control_hz=240)], mixed_control_hz=True)
    assert av.kinds == ["quadx"] * 3 and av.setpoints.shape == (3, 7) and av.updates_per_step == 4 and av.step_period == 1.0 / 60
    assert av.control_hz.tolist() == [60, 120, 240]
    c = av.launch_count
    for k in range(5):
        av.step()
        assert av.launch_count == c + k + 1
    av.set_setpoint(1, [0.1, 0.2, 0.3, 0.4])
    assert tuple(av.state(1).shape) == (4, 3) and tuple(av.aux_state(2).shape) == (4,)
    with pytest.raises(ValueError):
        av.set_setpoint(0, [0, 0, 0, 0, 0, 0, 0])
    # all rates equal with the option: the handle built without it
    same = BatchedAviary(pos, np.zeros_like(pos), drone_options=[dict(control_hz=60)] * 3, mixed_control_hz=True)
    assert same.kinds is None and same.setpoints.shape == (3, 4) and same.updates_per_step == 4
    av.reseed(4)
    av.reset()
    assert bool(torch.isfinite(av.all_states).all()) and float(av.setpoints.abs().max()) == 0.0


@pytest.mark.gpu
def test_full_size_rates_repeatable_and_match_oracle():
    """~65 536 drones, kinds and rates interleaved lane by lane: two runs are bit-equal, and a sample follows the oracle at each
    drone's rate over 100 steps of injected noise (the bars of test_mixed_kinds.py::test_full_size_repeatable_and_matches_oracle)."""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    n, steps = 3 * 21846, 100
    kinds, opts, hz, start, orn, modes, sp = _rate_setup(n, 9)
    kinds = [["quadx", "fixedwing", "rocket"][i % 3] for i in range(n)]
    hz = np.array([RATE_HZ[k][(i // 3) % len(RATE_HZ[k])] for i, k in enumerate(kinds)])
    opts = [dict(CF2X, control_hz=int(h)) if k == "quadx" else dict(control_hz=int(h)) for k, h in zip(kinds, hz)]
    ks = np.array(kinds)
    orn[:, 0] = np.where(ks == "rocket", np.pi / 2, orn[:, 0])
    modes = [0] * n
    f = lambda a: a.astype(np.float32).astype(np.float64)  # noqa: E731
    runs = []
    for _ in range(2):
        av = BatchedAviary(start, orn, drone_type=kinds, drone_options=opts, seed=5, mixed_control_hz=True)
        U = av.updates_per_step
        av.set_mode(modes)
        sp = np.zeros((n, 7), dtype=np.float32)
        sp[ks == "quadx", :4] = np.random.default_rng(2).uniform([-1, -1, -1, 0.2], [1, 1, 1, 0.7], (int((ks == "quadx").sum()), 4))
        sp[ks == "rocket"] = [0.1, -0.1, 0.05, 1.0, 0.6, 0.1, -0.1]
        sp[ks == "fixedwing"] = [0.2, -0.1, 0.1, 0.8, 0.0, 0.0, 0.0]
        av.set_all_setpoints(sp)
        noise = f(np.random.default_rng(3).normal(0.0, 1.0, (steps * U, n)))
        noise[:, ks == "quadx"] += 4.0
        nz = torch.as_tensor(noise, dtype=torch.float32, device="cuda")
        for t in range(steps):
            av.step(1, nz[t * U : (t + 1) * U].contiguous())
        torch.cuda.synchronize()
        runs.append((av.all_states.clone(), av._aux_state.clone(), av.setpoints.cpu().double().numpy(), noise))
        del av
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    s = runs[0][0].cpu().double().numpy()
    spn, noise = runs[0][2], runs[0][3]
    U = 4
    for d in np.random.default_rng(4).choice(n, 60, replace=False):
        k, r = kinds[d], 240 // int(hz[d])
        o = OracleEngine(build_model(k, "cf2x" if k == "quadx" else k, control_hz=int(hz[d])), None, 1, f(start[d][None]), f(orn[d][None]))
        o.reset()
        o.set_mode(modes[d])
        o.set_setpoints(spn[d][None, : SP_DIM[k]])
        o.aviary_step(noise[:, d][:, None], n_steps=steps * U // r)
        a = o.state()[0]
        pos_bar, w_bar = (0.5e-3, 2e-3) if k == "quadx" else (1e-3, 1e-2)
        assert np.abs(a[3] - s[d, 3]).max() < pos_bar, (d, k, int(hz[d]), a[3], s[d, 3])
        assert np.abs(a[0] - s[d, 0]).max() < w_bar, (d, k, int(hz[d]), a[0], s[d, 0])


@pytest.mark.gpu
def test_reference_multi_spawn_holds_position():
    """tests/test_core.py::test_multi_spawn of the reference: three QuadX at 60, 120 and 240 Hz, set_mode(7), 1000 steps.  Every
    drone holds its start position (mode 7's preset) to 10 cm, the bar of test_mixed_kinds.py::test_reference_mixed_drones_scenario_with_the_floor."""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    start_pos = np.array([[-1.0, 0.0, 1.0], [0.0, 0.0, 1.0], [1.0, 0.0, 1.0]])
    av = BatchedAviary(start_pos, np.zeros_like(start_pos), drone_type="quadx",
                       drone_options=[dict(control_hz=60), dict(control_hz=120), dict(control_hz=240)], mixed_control_hz=True)
    av.set_mode(7)
    for _ in range(1000):
        av.step()
    s = av.all_states
    assert bool(torch.isfinite(s).all())
    err = (s[:, 3] - torch.as_tensor(start_pos, dtype=torch.float32, device="cuda")).abs().max(dim=1).values
    assert float(err.max()) < 0.1, err
    assert av.physics_steps == 4000 and abs(av.elapsed_time - 1000 / 60) < 1e-9
