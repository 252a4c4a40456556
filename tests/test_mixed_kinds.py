"""Several vehicle kinds in one batch: ``BatchedAviary(drone_type=[...])`` (the reference's aviary.py:139-190,
examples/core/08_mixed_drones.py, tests/test_core.py::test_mixed_drones).

CPU: the argument checks and their messages, the mixed model-set builder, the C-ABI refusals of pfb_create_mixed, and the C
oracle (one per drone) against the unmodified reference flying rockets, QuadX and fixed-wing drones in ONE Aviary
(tests/golden/mixed_kinds_*.npz, tools/gen_golden.py).
GPU: one handle replays the fixtures; drone i of a mixed handle is bit-identical to drone i of a single-kind handle of its kind
(same seed: the Philox streams depend on the drone id, not on the kind); 65 536 drones against the oracle; one launch per step;
the reference's test_mixed_drones scenario with the floor pushing back."""
import ctypes as C
import json
import re

import numpy as np
import pytest

from engines import OracleEngine, build_model, load_golden
from pyflyt_b200.models import ModelSetError, PfbEnvConfig, PfbModel, build_mixed_model_set

FIXTURES = ["mixed_kinds_grouped", "mixed_kinds_interleaved"]
SP_DIM = {"quadx": 4, "fixedwing": 6, "rocket": 7}
AUX_DIM = {"quadx": 4, "fixedwing": 6, "rocket": 9}
HEIGHT_HOLD = (2, 3, 4, 7)
CF2X, PRIM = dict(drone_model="cf2x"), dict(drone_model="primitive_drone")


def _bytes(m):
    return C.string_at(C.addressof(m), C.sizeof(m))


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_aviary_checks_kinds_before_the_device():
    from pyflyt_b200.core.aviary import AviaryInitException, BatchedAviary

    z = np.zeros((3, 3))
    with pytest.raises(AviaryInitException, match=re.escape("If multiple `drone_types` are used, must have same number of `drone_types` (2) as number of drones (3).")):
        BatchedAviary(z, z, drone_type=["quadx", "rocket"])
    with pytest.raises(AviaryInitException, match=re.escape("One of types in `drone_type` ['quadx', 'boat', 'rocket'] is not amongst known types")):
        BatchedAviary(z, z, drone_type=["quadx", "boat", "rocket"])
    with pytest.raises(AviaryInitException, match="control_hz"):
        BatchedAviary(z, z, drone_type=["quadx", "fixedwing", "rocket"], drone_options=[CF2X, dict(control_hz=60), {}])
    with pytest.raises(AviaryInitException, match="one vehicle model"):
        BatchedAviary(np.zeros((4, 3)), np.zeros((4, 3)), drone_type=["quadx", "fixedwing", "fixedwing", "rocket"],
                      drone_options=[CF2X, dict(drone_model="fixedwing"), dict(drone_model="acrowing"), {}])
    with pytest.raises(AviaryInitException, match=re.escape("If multiple `drone_options` (2) are used")):
        BatchedAviary(z, z, drone_type=["quadx", "fixedwing", "rocket"], drone_options=[CF2X, {}])
    with pytest.raises(AviaryInitException, match="env_config"):
        BatchedAviary(z, z, drone_type=["quadx", "fixedwing", "rocket"], env_config=PfbEnvConfig())


def test_mixed_model_set_tables_index_and_dedup():
    kinds = ["rocket", "quadx", "fixedwing", "quadx", "rocket", "quadx"]
    tables, index = build_mixed_model_set(kinds, [{}, CF2X, {}, PRIM, dict(drone_model="rocket"), dict(CF2X)], 240, 6)
    assert [int(t.kind) for t in tables] == [0, 0, 1, 2] and index.dtype == np.uint8
    assert index.tolist() == [3, 0, 2, 1, 3, 0]  # QuadX tables first, then the fixed-wing and the rocket table
    assert _bytes(tables[0]) == _bytes(build_model("quadx", "cf2x")) and _bytes(tables[1]) == _bytes(build_model("quadx", "primitive_drone"))
    assert _bytes(tables[2]) == _bytes(build_model("fixedwing", "fixedwing")) and _bytes(tables[3]) == _bytes(build_model("rocket", "rocket"))
    # None / one dict for every drone: one table per kind present
    tables, index = build_mixed_model_set(["fixedwing", "rocket", "fixedwing"], None, 240, 3)
    assert [int(t.kind) for t in tables] == [1, 2] and index.tolist() == [0, 1, 0]
    with pytest.raises(ModelSetError, match="drone_types"):
        build_mixed_model_set(["quadx", "rocket"], None, 240, 3)


def _lib_or_skip():
    from pyflyt_b200 import _lib

    try:
        return _lib, _lib.lib()
    except _lib.PfbError as e:
        pytest.skip(str(e))


def _create(L, models, index, n=None, cfg=None):
    tables = (PfbModel * len(models))(*models)
    idx = np.ascontiguousarray(index, dtype=np.uint8)
    h = C.c_void_p()
    rc = L.pfb_create_mixed(tables, len(models), idx.ctypes.data_as(C.c_void_p), len(idx) if n is None else n, None if cfg is None else C.byref(cfg), 0, 1, C.byref(h))
    return rc, h


def test_create_mixed_refuses_malformed_input():
    import torch

    _lib, L = _lib_or_skip()
    q, f, r = build_model("quadx", "cf2x"), build_model("fixedwing", "fixedwing"), build_model("rocket", "rocket")
    err = lambda: L.pfb_last_error().decode()  # noqa: E731
    rc, _ = _create(L, [q, f, r], [0, 1, 3])
    assert rc != 0 and "model_index[2] = 3" in err()
    rc, _ = _create(L, [q, f, f, r], [0, 1, 2, 3])
    assert rc != 0 and "one fixed-wing and one rocket model" in err()
    rc, _ = _create(L, [q, f, build_model("rocket", "rocket", control_hz=60)], [0, 1, 2])
    assert rc != 0 and "control_hz" in err()
    rc, _ = _create(L, [q, f, r], [0, 1, 2], n=0)
    assert rc != 0 and "positive" in err()
    cfg = PfbEnvConfig()
    cfg.env_kind = 1
    rc, _ = _create(L, [q, f, r], [0, 1, 2], cfg=cfg)
    assert rc != 0 and "Aviary handle" in err()
    rc, h = _create(L, [q, f, r], [2, 0, 1])
    if torch.cuda.is_available():
        assert rc == 0, err()
        L.pfb_destroy(h)
    else:  # well-formed input: the device lookup is what fails
        assert rc != 0 and "no CPU fallback" in err()


def _fixture_kinds(g):
    return json.loads(str(g["drone_type"]))


def _mode_at(g):
    T, n = len(g["state"]), int(g["n_drones"])
    out = np.zeros((T, n), dtype=int)
    for k, step in enumerate(g["mode_steps"]):
        out[int(step):] = g["modes"][k]
    return out


class _OraclePerDrone:
    """One oracle per drone, each of its own kind: the reference's Aviary loops over its drones the same way."""

    def __init__(self, g):
        kinds, opts = _fixture_kinds(g), json.loads(str(g["drone_options"]))
        self.kinds = kinds
        self.engines = [OracleEngine(build_model(k, o.get("drone_model")), None, 1, g["start_pos"][d][None], g["start_orn"][d][None])
                        for d, (k, o) in enumerate(zip(kinds, opts))]

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
        for d, e in enumerate(self.engines):
            e.aviary_step(noise[:, d][:, None])

    def state(self):
        return np.concatenate([e.state() for e in self.engines])

    def aux(self):
        out = np.zeros((len(self.engines), 9))
        for d, (e, k) in enumerate(zip(self.engines, self.kinds)):
            out[d, : AUX_DIM[k]] = e.aux()[0]
        return out

    def contact(self):
        return np.concatenate([e.contact() for e in self.engines])


def replay_kinds(g, eng):
    """Replays a mixed-kind fixture through ``eng`` (all drones); max abs errors per drone."""
    n, T = int(g["n_drones"]), len(g["state"])
    noise = g["noise"].reshape(T, -1, n)
    calls = {int(s): k for k, s in enumerate(g["mode_steps"])}
    err = {k: np.zeros(n) for k in ("setpoint", "pos", "euler", "angvel", "linvel", "aux")}
    err["contact_mismatch"] = np.zeros(n, dtype=int)
    eng.reset()
    for i in range(T):
        if i in calls:
            k = calls[i]
            eng.set_modes([int(m) for m in g["modes"][k]])
            d = np.abs(eng.get_setpoints() - g["setpoint_after_set_mode"][k]).max(axis=1)
            err["setpoint"] = np.maximum(err["setpoint"], d)
        eng.set_setpoints(g["setpoints"][i])
        eng.aviary_step(noise[i])
        s, ref = eng.state(), g["state"][i]
        d_eul = np.abs((s[:, 1] - ref[:, 1] + np.pi) % (2 * np.pi) - np.pi)
        err["angvel"] = np.maximum(err["angvel"], np.abs(s[:, 0] - ref[:, 0]).max(axis=1))
        err["euler"] = np.maximum(err["euler"], d_eul.max(axis=1))
        err["linvel"] = np.maximum(err["linvel"], np.abs(s[:, 2] - ref[:, 2]).max(axis=1))
        err["pos"] = np.maximum(err["pos"], np.abs(s[:, 3] - ref[:, 3]).max(axis=1))
        err["aux"] = np.maximum(err["aux"], np.abs(eng.aux() - g["aux"][i]).max(axis=1))
        err["contact_mismatch"] += (eng.contact().astype(bool) != g["contact"][i]).astype(int)
    return err


def test_fixtures_cover_every_kind_and_stay_off_the_floor():
    for name in FIXTURES:
        g = load_golden(name)
        kinds = _fixture_kinds(g)
        assert sorted(set(kinds)) == ["fixedwing", "quadx", "rocket"] and not g["contact"].any(), name
        assert g["noise"].size == len(g["state"]) * 2 * int(g["n_drones"])  # one draw per drone per physics step
    assert _fixture_kinds(load_golden("mixed_kinds_interleaved"))[:6] == ["rocket", "quadx", "fixedwing", "quadx", "rocket", "fixedwing"]


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_reference_mixed_kinds(name):
    """Each drone of the reference's mixed-kind Aviary, replayed by an oracle of its own kind (bars of test_oracle_golden.py and
    test_mixed_modes.py: 1e-9, 1e-6 for drones that hold height)."""
    g = load_golden(name)
    err = replay_kinds(g, _OraclePerDrone(g))
    loose = np.isin(_mode_at(g), HEIGHT_HOLD).any(axis=0)
    assert err["contact_mismatch"].sum() == 0
    for k in ("setpoint", "pos", "euler", "angvel", "linvel", "aux"):
        assert err[k][~loose].max(initial=0.0) < 1e-9, (name, k, err[k])
        assert err[k][loose].max(initial=0.0) < 1e-6, (name, k, err[k])


# ------------------------------------------------------------------------------------------------------------------ GPU
class MixedKindEngine:
    """One BatchedAviary over all drones of a fixture."""

    def __init__(self, g, **kw):
        from pyflyt_b200.core.aviary import BatchedAviary

        self.av = BatchedAviary(np.asarray(g["start_pos"], dtype=np.float32), np.asarray(g["start_orn"], dtype=np.float32),
                                drone_type=_fixture_kinds(g), drone_options=json.loads(str(g["drone_options"])), **kw)

    def reset(self):
        self.av.reset()

    def set_modes(self, modes):
        self.av.set_mode(list(modes))

    def get_setpoints(self):
        return self.av.setpoints.cpu().double().numpy()

    def set_setpoints(self, sp):
        self.av.set_all_setpoints(np.asarray(sp, dtype=np.float32))

    def aviary_step(self, noise, n_steps=1):
        import torch

        self.av.step(n_steps, torch.as_tensor(np.ascontiguousarray(noise, dtype=np.float32), device="cuda"))

    def state(self):
        return self.av.all_states.cpu().double().numpy()

    def aux(self):
        self.av.all_states
        return self.av._aux_state.cpu().double().numpy()

    def contact(self):
        return self.av.contact_array.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_cuda_replays_mixed_kind_fixture(name):
    """ONE CUDA handle flies the reference's rockets, QuadX and fixed-wing drones.  Rockets and fixed-wing drones, and QuadX drones
    that keep one mode, to the bars of test_mixed_models.py (1e-3 m).  A QuadX drone that switches between modes 0 and 7 at step
    150 amplifies fp32 rounding in the attitude loop: the fp32 kernel body built for the host (tests/hostsim) ends 0.9 to 2.7 cm
    from the reference on exactly these drones, the device build up to 4.9 cm (interleaved fixture, drone 3), so they are held to
    5 cm here, and to the single-kind kernels bit for bit by test_mixed_handle_bit_equal_to_single_kind_handles."""
    g = load_golden(name)
    eng = MixedKindEngine(g)
    err = replay_kinds(g, eng)
    kinds = np.array(_fixture_kinds(g))
    switched = (kinds == "quadx") & np.isin(g["modes"], (0, 7)).all(axis=0) & (g["modes"][0] != g["modes"][-1])
    print(f"\n[{name}] max |pos - reference| per drone: {np.array2string(err['pos'], precision=2)}")
    assert err["contact_mismatch"].sum() == 0, err["contact_mismatch"]
    assert err["setpoint"].max() < 1e-5, err["setpoint"]
    assert err["pos"][~switched].max() < 1e-3, err["pos"]
    assert err["pos"][switched].max(initial=0.0) < 5e-2, err["pos"]
    assert err["euler"][kinds != "quadx"].max() < 1e-3, err["euler"]


def _interleaved_kinds(n):
    """kinds interleaved both inside a warp (lane by lane) and tile by tile"""
    pattern = ["quadx", "fixedwing", "rocket", "quadx", "quadx", "rocket", "fixedwing"]
    return [pattern[(i + (i // 32)) % len(pattern)] for i in range(n)]


def _mixed_setup(n, seed):
    rng = np.random.default_rng(seed)
    kinds = _interleaved_kinds(n)
    opts = [(CF2X if (i // 3) % 2 == 0 else PRIM) if k == "quadx" else {} for i, k in enumerate(kinds)]
    start = np.column_stack([rng.uniform(-5, 5, n), rng.uniform(-5, 5, n), rng.uniform(30, 60, n)]).astype(np.float32)
    orn = rng.uniform(-0.2, 0.2, (n, 3)).astype(np.float32)
    orn[np.array(kinds) == "rocket", 0] = np.pi / 2
    modes = []
    for i, k in enumerate(kinds):
        modes.append({"quadx": [0, 7, 6, -1][i % 4], "fixedwing": [0, -1][i % 2], "rocket": 0}[k])
    sp = np.zeros((n, 7), dtype=np.float32)
    for i, (k, m) in enumerate(zip(kinds, modes)):
        if k == "rocket":
            sp[i] = [0.1, -0.1, 0.05, 1.0, 0.6, 0.1, -0.1]
        elif k == "fixedwing":
            sp[i, :6] = [0.2, -0.1, 0.1, 0.8, 0.0, 0.0] if m == 0 else [0.1, -0.2, 0.1, 0.05, -0.05, 0.7]
        elif m == 7:
            sp[i, :4] = [start[i, 0] + 1.0, start[i, 1] - 1.0, 0.3, start[i, 2] + 0.5]
        elif m == -1:
            sp[i, :4] = [0.3, 0.31, 0.32, 0.3]
        else:
            sp[i, :4] = [0.1, -0.1, 0.2, 0.4]
    return kinds, opts, start, orn, modes, sp


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["philox", "contact", "wind"])
def test_mixed_handle_bit_equal_to_single_kind_handles(variant):
    """Drone i of a mixed handle (kinds interleaved per lane and per tile, one mode per drone, two QuadX tables, Philox noise)
    against drone i of a single-kind handle of its kind over the same n drones, same seed, same options: bit for bit."""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary
    from pyflyt_b200.core.wind import AnalyticWind

    n, steps = 4096 + 77, 200
    kinds, opts, start, orn, modes, sp = _mixed_setup(n, 7)
    contact = variant == "contact"
    if contact:  # dropped onto the floor from low heights
        start[:, 2] = np.random.default_rng(1).uniform(0.3, 2.0, n).astype(np.float32)
        rk = np.array(kinds) == "rocket"
        # upright rockets: the origin 0.05-2 m above the resting height, where the legs' lowest corners (z = -2.425 in the body)
        # touch the floor; lower, the Baumgarte bias would throw a rocket whose legs start inside the floor out of it
        start[rk, 2] = (2.425 + np.random.default_rng(2).uniform(0.05, 2.0, int(rk.sum()))).astype(np.float32)
        orn[rk, :2] = 0.0
        sp[np.array(kinds) == "rocket"] = 0.0  # not ignited: the rockets drop and rest on the floor
    wind = AnalyticWind("power", base=(3.0, -1.5, 0.2), z_ref=10.0, alpha=1.0 / 7.0) if variant == "wind" else None
    mixed = BatchedAviary(start, orn, drone_type=kinds, drone_options=opts, seed=11, contact_response=contact)
    assert len(mixed.models) == 4
    uniform = {}
    for k in ("quadx", "fixedwing", "rocket"):
        kopts = [o if kk == k else (CF2X if k == "quadx" else {}) for o, kk in zip(opts, kinds)]
        uniform[k] = BatchedAviary(start, orn, drone_type=k, drone_options=kopts if k == "quadx" else None, seed=11, contact_response=contact)
    avs = [mixed] + list(uniform.values())
    for a in avs:
        if wind is not None:
            a.register_wind_field(wind)
        a.reset()
    mixed.set_mode(modes)
    for k, u in uniform.items():
        u.set_mode([m if kk == k else (0) for m, kk in zip(modes, kinds)])
    mixed.set_all_setpoints(sp)
    for k, u in uniform.items():
        u.set_all_setpoints(torch.as_tensor(sp[:, : u.setpoint_dim]))
    touched = None
    for t in range(steps):
        for a in avs:
            a.step(1)
        if t % 10 == 9:
            touched = mixed.contact_array.clone() if touched is None else touched | mixed.contact_array
    torch.cuda.synchronize()
    ks = np.array(kinds)
    s, aux, con = mixed.all_states, mixed._aux_state, mixed.contact_array
    for k, u in uniform.items():
        m = torch.as_tensor(ks == k, device="cuda")
        assert torch.equal(s[m], u.all_states[m]), k
        assert torch.equal(aux[m][:, : u.aux_dim], u.all_aux_states[m]), k
        assert bool((aux[m][:, u.aux_dim :] == 0).all())
        assert torch.equal(con[m], u.contact_array[m]), k
        assert torch.equal(mixed.precise_positions[m], u.precise_positions[m]), k
    assert bool(torch.isfinite(s).all())
    if contact:  # every kind did reach the floor (the contact flags match bit for bit above); the rockets came to rest on their legs
        for k in ("quadx", "fixedwing", "rocket"):
            assert bool(touched[torch.as_tensor(ks == k, device="cuda")].any()), k
        rz = mixed.precise_positions[torch.as_tensor(ks == "rocket", device="cuda"), 2]
        assert bool(con[torch.as_tensor(ks == "rocket", device="cuda")].all()) and float(rz.min()) > 2.3 and float(rz.max()) < 2.5, (rz.min(), rz.max())


@pytest.mark.gpu
def test_mixed_reset_and_set_mode_against_single_kind_handles():
    """Masked and full resets, set_mode(int) and set_mode(list) on a mixed handle against single-kind handles over the same
    drones: the state bit for bit, each setpoint row at its kind's width, and the columns past that width zero, also where they
    held values before.  Steps in between show that the modes are kept or replaced as on the single-kind handles."""
    import torch

    from pyflyt_b200 import _lib
    from pyflyt_b200.core.aviary import BatchedAviary

    n = 256 + 13
    kinds, opts, start, orn, modes, sp = _mixed_setup(n, 5)
    mixed = BatchedAviary(start, orn, drone_type=kinds, drone_options=opts, seed=3)
    uniform = {}
    for k in ("quadx", "fixedwing", "rocket"):
        kopts = [o if kk == k else CF2X for o, kk in zip(opts, kinds)] if k == "quadx" else None
        uniform[k] = BatchedAviary(start, orn, drone_type=k, drone_options=kopts, seed=3)
    avs = [mixed] + list(uniform.values())
    ks = np.array(kinds)
    fill = torch.as_tensor(sp, device="cuda")
    for k, u in uniform.items():  # non-zero columns past each drone's own setpoint length
        fill[torch.as_tensor(ks == k, device="cuda"), u.setpoint_dim :] = 9.0
    mask = torch.as_tensor(np.random.default_rng(6).random(n) < 0.5, dtype=torch.uint8, device="cuda")

    def load_setpoints():
        mixed.setpoints.copy_(fill)
        for u in uniform.values():
            u.setpoints.copy_(fill[:, : u.setpoint_dim])

    def set_modes(ms):
        mixed.set_mode(ms)
        for k, u in uniform.items():
            u.set_mode(ms if isinstance(ms, int) else [m if kk == k else 0 for m, kk in zip(ms, kinds)])

    def same(x, y):  # bit for bit
        return torch.equal(x.contiguous().view(torch.int32), y.contiguous().view(torch.int32))

    def check(what, rows_rewritten=True):
        torch.cuda.synchronize()
        s = mixed.all_states
        for k, u in uniform.items():
            m = torch.as_tensor(ks == k, device="cuda")
            assert same(s[m], u.all_states[m]), (what, k)
            assert same(mixed.setpoints[m][:, : u.setpoint_dim], u.setpoints[m]), (what, k)
            if rows_rewritten:
                assert bool((mixed.setpoints[m][:, u.setpoint_dim :] == 0).all()), (what, k)

    def step_and_check(what):  # a step leaves the setpoint rows as they are
        load_setpoints()
        for a in avs:
            a.step(3)
        check(what, rows_rewritten=False)

    set_modes(modes)
    step_and_check("per-drone modes")
    load_setpoints()
    for a in avs:
        _lib.check(_lib.lib().pfb_reset(a._h, C.c_void_p(mask.data_ptr()), a._s()))
    check("masked reset")
    step_and_check("modes kept by a masked reset")
    load_setpoints()
    set_modes(0)
    check("set_mode(0)")
    step_and_check("mode 0")
    load_setpoints()
    set_modes(modes)
    check("set_mode(list)")
    step_and_check("per-drone modes again")
    load_setpoints()
    for a in avs:
        a.reset()
    check("reset")
    assert float(mixed.setpoints.abs().max()) == 0.0
    step_and_check("mode 0 after a reset")


@pytest.mark.gpu
def test_one_launch_per_step_and_accessors():
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    av = BatchedAviary([[0, 0, 10], [0, 0, 10], [0, 0, 10]], [[np.pi / 2, 0, 0], [0, 0, 0], [0, 0, 0]], drone_type=["rocket", "quadx", "fixedwing"])
    assert av.setpoints.shape == (3, 7) and av.aux_dim == 9
    c = av.launch_count
    for k in range(5):
        av.step()
        assert av.launch_count == c + k + 1
    assert [tuple(a.shape) for a in av.all_aux_states] == [(9,), (4,), (6,)]
    assert tuple(av.aux_state(2).shape) == (6,) and tuple(av.state(0).shape) == (4, 3)
    assert tuple(av.precise_positions.shape) == (3, 3) and av.precise_positions.dtype == torch.float64
    av.set_setpoint(0, [0, 0, 0, 1, 0.5, 0, 0])
    av.set_setpoint(2, [0.1, 0.2, 0.3, 0.4])
    with pytest.raises(ValueError):
        av.set_setpoint(1, [0, 0, 0, 0, 0, 0, 0])
    av.set_all_setpoints([np.zeros(7), [0, 0, 0, 1], np.zeros(6)])
    assert float(av.setpoints[1, 3]) == 1.0
    with pytest.raises(ValueError, match=re.escape("`mode` must be between 0 and 0")):
        av.set_mode(7)  # valid for the QuadX, not for the rocket (drone 0): nothing changes
    av.set_mode([0, 7, -1])
    with pytest.raises(NotImplementedError):
        av.state_row(0)
    with pytest.raises(NotImplementedError):
        av.env_step()
    av.reseed(3)
    av.reset()
    assert bool(torch.isfinite(av.all_states).all()) and float(av.setpoints.abs().max()) == 0.0


@pytest.mark.gpu
def test_full_size_repeatable_and_matches_oracle():
    """~65 536 drones, a third of each kind: two runs are bit-equal, and a sample per kind follows the oracle over 100 steps of
    injected noise."""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    n, steps = 3 * 21846, 100
    kinds, opts, start, orn, modes, sp = _mixed_setup(n, 9)
    kinds = [["quadx", "fixedwing", "rocket"][i % 3] for i in range(n)]
    opts = [CF2X if k == "quadx" else {} for k in kinds]
    orn[:, 0] = np.where(np.array(kinds) == "rocket", np.pi / 2, orn[:, 0])
    modes = [0] * n  # QuadX mode 0: the bars of test_mixed_models.py::test_aviary_4096_alternating_models_match_oracle_per_model
    f = lambda a: a.astype(np.float32).astype(np.float64)  # noqa: E731
    runs = []
    for _ in range(2):
        av = BatchedAviary(start, orn, drone_type=kinds, drone_options=opts, seed=5)
        av.set_mode(modes)
        ks = np.array(kinds)
        sp = np.zeros((n, 7), dtype=np.float32)
        sp[ks == "quadx", :4] = np.random.default_rng(2).uniform([-1, -1, -1, 0.2], [1, 1, 1, 0.7], (int((ks == "quadx").sum()), 4))
        sp[ks == "rocket"] = [0.1, -0.1, 0.05, 1.0, 0.6, 0.1, -0.1]
        sp[ks == "fixedwing"] = [0.2, -0.1, 0.1, 0.8, 0.0, 0.0, 0.0]
        av.set_all_setpoints(sp)
        rng = np.random.default_rng(3)
        noise = f(rng.normal(0.0, 1.0, (steps * av.updates_per_step, n)))
        noise[:, np.array(kinds) == "quadx"] += 4.0  # QuadX motors draw normal(loc = 4) (motors.py:134-138)
        nz = torch.as_tensor(noise, dtype=torch.float32, device="cuda")
        for t in range(steps):
            av.step(1, nz[t * av.updates_per_step : (t + 1) * av.updates_per_step].contiguous())
        torch.cuda.synchronize()
        runs.append((av.all_states.clone(), av._aux_state.clone(), av.setpoints.cpu().double().numpy(), noise))
        del av
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    s = runs[0][0].cpu().double().numpy()
    spn, noise = runs[0][2], runs[0][3]
    sample = np.random.default_rng(4).choice(n, 60, replace=False)
    for d in sample:
        k = kinds[d]
        o = OracleEngine(build_model(k, "cf2x" if k == "quadx" else k), None, 1, f(start[d][None]), f(orn[d][None]))
        o.reset()
        o.set_mode(modes[d])
        o.set_setpoints(spn[d][None, : SP_DIM[k]])
        o.aviary_step(noise[:, d][:, None], n_steps=steps)
        a = o.state()[0]
        pos_bar, w_bar = (0.5e-3, 2e-3) if k == "quadx" else (1e-3, 1e-2)  # QuadX: test_aviary_4096_alternating_models_match_oracle_per_model
        assert np.abs(a[3] - s[d, 3]).max() < pos_bar, (d, k, a[3], s[d, 3])
        assert np.abs(a[0] - s[d, 0]).max() < w_bar, (d, k, a[0], s[d, 0])


@pytest.mark.gpu
def test_reference_mixed_drones_scenario_with_the_floor():
    """tests/test_core.py::test_mixed_drones of the reference without the camera: a rocket, a QuadX and a fixed-wing,
    set_mode([0, 7, 0]), 1000 steps, here with the floor pushing back.  The QuadX holds its mode-7 setpoint."""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    start_pos = np.array([[0.0, 5.0, 5.0], [3.0, 3.0, 1.0], [5.0, 0.0, 1.0]])
    start_orn = np.zeros_like(start_pos)
    av = BatchedAviary(start_pos, start_orn, drone_type=["rocket", "quadx", "fixedwing"], contact_response=True)
    av.set_mode([0, 7, 0])
    target = torch.tensor([3.0, 3.0, 0.0, 1.0], device="cuda")  # mode 7's preset: the drone's start x, y, yaw, z
    assert torch.allclose(av.setpoints[1, :4], target)
    for _ in range(1000):
        av.step()
    s = av.all_states
    assert bool(torch.isfinite(s).all()) and all(bool(torch.isfinite(a).all()) for a in av.all_aux_states)
    assert float((s[1, 3] - target[[0, 1, 3]]).abs().max()) < 0.1, s[1, 3]
