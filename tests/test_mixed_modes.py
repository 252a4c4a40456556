"""One flight mode per drone: ``BatchedAviary.set_mode(list)`` (the reference's aviary.py:440-458) on Aviary handles.

CPU: the C oracle (one oracle per drone) against the unmodified reference flying QuadX drones in every mode -1..7, re-assigned by
two more set_mode(list) calls, and fixed-wing drones in modes -1 / 0, each fixture ONE reference Aviary
(tests/golden/mixed_modes_*.npz, tools/gen_golden.py); the host simulator's per-drone path against the oracle.
GPU: one handle replays the fixtures; drone i of a per-drone handle is bit-identical to drone i of a uniform handle of its
mode (same seed: the Philox streams depend on the drone id, not on the mode); mode sequences against the oracle; refusals."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

from engines import ROOT, CudaEngine, HostSimEngine, OracleEngine, build_model, load_golden

HEIGHT_LOOP = (2, 3, 7)  # modes whose z-velocity PID limit-cycles in the reference: the looser bars of test_oracle_golden.py
# the oracle's 1e-6 bar also covers mode 4: after mode 0 or 1 phases its height chain (z_pos + z_vel PIDs) takes primitive_drone
# to ~1e-7 of the reference
HEIGHT_HOLD = (2, 3, 4, 7)


def _mode_at(g):
    """[T, n] flight mode of every drone on every step of a mixed-mode fixture"""
    T, n = len(g["state"]), int(g["n_drones"])
    out = np.zeros((T, n), dtype=int)
    for k, step in enumerate(g["mode_steps"]):
        out[int(step):] = g["modes"][k]
    return out


def replay_modes(g, engines):
    """Replays a mixed-mode fixture; ``engines`` = [(engine, drone ids it flies)], each engine with a ``set_modes(list)``.
    Max abs errors per drone, and the setpoint error after each set_mode call."""
    n, T = int(g["n_drones"]), len(g["state"])
    sp_dim = g["setpoints"].shape[2]
    noise = g["noise"].reshape(T, -1, n)
    calls = {int(s): k for k, s in enumerate(g["mode_steps"])}
    err = {k: np.zeros(n) for k in ("setpoint0", "setpoint", "pos", "euler", "angvel", "linvel", "aux")}
    err["contact_mismatch"] = np.zeros(n, dtype=int)
    for eng, ids in engines:
        eng.reset()
    for i in range(T):
        if i in calls:
            k = calls[i]
            for eng, ids in engines:
                eng.set_modes([int(m) for m in g["modes"][k][ids]])
                got = eng.get_setpoints()
                w = min(got.shape[1], sp_dim)  # the oracle reports 4 columns; fixed-wing setpoints after set_mode are all zero
                d = np.abs(got[:, :w] - g["setpoint_after_set_mode"][k][ids][:, :w]).max(axis=1)
                err["setpoint"][ids] = np.maximum(err["setpoint"][ids], d)
                if k == 0:
                    err["setpoint0"][ids] = d
        for eng, ids in engines:
            eng.set_setpoints(g["setpoints"][i][ids])
            eng.aviary_step(noise[i][:, ids])
        for eng, ids in engines:
            s, ref = eng.state(), g["state"][i][ids]
            d_eul = np.abs((s[:, 1] - ref[:, 1] + np.pi) % (2 * np.pi) - np.pi)
            err["angvel"][ids] = np.maximum(err["angvel"][ids], np.abs(s[:, 0] - ref[:, 0]).max(axis=1))
            err["euler"][ids] = np.maximum(err["euler"][ids], d_eul.max(axis=1))
            err["linvel"][ids] = np.maximum(err["linvel"][ids], np.abs(s[:, 2] - ref[:, 2]).max(axis=1))
            err["pos"][ids] = np.maximum(err["pos"][ids], np.abs(s[:, 3] - ref[:, 3]).max(axis=1))
            aux = eng.aux()[:, : g["aux"].shape[2]]
            err["aux"][ids] = np.maximum(err["aux"][ids], np.abs(aux - g["aux"][i][ids]).max(axis=1))
            err["contact_mismatch"][ids] += (eng.contact().astype(bool) != g["contact"][i][ids]).astype(int)
    return err


class _PerDrone:
    """One single-mode engine per drone: set_modes(list) = set_mode(mode) on each (the reference's Aviary.set_mode(list))."""

    def __init__(self, make, opts, g):
        self.engines = [make(o, g["start_pos"][d][None], g["start_orn"][d][None]) for d, o in enumerate(opts)]
        self.n = len(self.engines)

    def reset(self):
        for e in self.engines:
            e.reset()

    def set_modes(self, modes):
        for e, m in zip(self.engines, modes):
            e.set_mode(m)

    def get_setpoints(self):
        return np.concatenate([e.get_setpoints() for e in self.engines])

    def set_setpoints(self, sp):
        for d, e in enumerate(self.engines):
            e.set_setpoints(sp[d][None])

    def aviary_step(self, noise, n_steps=1):
        for d, e in enumerate(self.engines):
            e.aviary_step(noise[:, d][:, None], n_steps=n_steps)

    def state(self):
        return np.concatenate([e.state() for e in self.engines])

    def aux(self):
        return np.concatenate([e.aux() for e in self.engines])

    def contact(self):
        return np.concatenate([e.contact() for e in self.engines])


def _opts(g):
    return json.loads(str(g["drone_options"]))


def _model(g, o):
    return build_model(str(g["drone_type"]), o.get("drone_model"))


def _assert_reference_bars(g, err, tag):
    """1e-9 per drone, 1e-6 for drones that spend any of the run in a height-hold mode (test_oracle_golden.py).  The setpoints
    of the first set_mode(list) exactly; the later ones hold the position / yaw of a drone that has flown, to the same bars."""
    loose = np.isin(_mode_at(g), HEIGHT_HOLD).any(axis=0)
    assert err["setpoint0"].max() == 0.0, (tag, err["setpoint0"])
    assert err["contact_mismatch"].sum() == 0, tag
    for k in ("setpoint", "pos", "euler", "angvel", "linvel", "aux"):
        assert err[k][~loose].max() < 1e-9, (tag, k, err[k])
        # primitive_drone 7 -> 1 -> 7: the rates, velocities and throttles of the second position hold reach ~1e-5 (pos < 1e-7)
        assert err[k][loose].max(initial=0.0) < (1e-6 if k in ("setpoint", "pos", "euler") else 1e-4), (tag, k, err[k])


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_quadx_fixture_covers_every_mode_and_the_z_pid_carry_over():
    g = load_golden("mixed_modes_quadx")
    modes = g["modes"]
    assert modes.shape == (3, 18) and sorted(set(modes[0].tolist())) == list(range(-1, 8))
    models = [o["drone_model"] for o in _opts(g)]
    for m in range(-1, 8):  # each mode on both vehicles
        assert {models[d] for d in np.flatnonzero(modes[0] == m)} == {"cf2x", "primitive_drone"}
    hold = (2, 3, 4, 7)
    back = np.isin(modes[0], hold) & np.isin(modes[1], (0, 1)) & np.isin(modes[2], hold)
    assert back.sum() >= 2
    assert not g["contact"].any()
    g = load_golden("mixed_modes_fixedwing")
    assert g["modes"][0].tolist() == [-1, 0, -1, 0] and not g["contact"].any()


@pytest.mark.parametrize("name", ["mixed_modes_quadx", "mixed_modes_fixedwing"])
def test_oracle_reproduces_reference_mixed_modes(name):
    """Each drone of the reference's mixed-mode Aviary, replayed by an oracle of its own; setpoints after every set_mode(list)
    exactly."""
    g = load_golden(name)
    eng = _PerDrone(lambda o, p, r: OracleEngine(_model(g, o), None, 1, p, r), _opts(g), g)
    err = replay_modes(g, [(eng, list(range(eng.n)))])
    _assert_reference_bars(g, err, name)


class HostSimModes(HostSimEngine):
    """HostSimEngine over tests/hostsim/hostsim_modes.cpp: set_modes / aviary_step through the per-drone dispatch helpers."""

    def __init__(self, model, n, start_pos, start_orn):
        super().__init__(model, None, n, start_pos, start_orn)
        self.L = _hostsim_modes_lib()
        self.modes = np.zeros(n, dtype=np.int8)

    def reset(self):
        super().reset()
        self.modes[:] = 0

    def set_modes(self, modes):
        self.modes = np.ascontiguousarray(modes, dtype=np.int8)
        f = C.c_float
        self._chk(self.L.hs_set_modes(self.modes.ctypes.data_as(C.c_void_p), self.st.ctypes.data_as(C.POINTER(f)),
                                      self.ist.ctypes.data_as(C.POINTER(C.c_int32)), self.sp.ctypes.data_as(C.POINTER(f)), C.c_int64(self.n)))

    def aviary_step(self, noise, n_steps=1):
        nz = np.ascontiguousarray(noise, dtype=np.float32)
        f = C.c_float
        self._chk(self.L.hs_aviary_step_modes(C.byref(self.model), self.modes.ctypes.data_as(C.c_void_p), self.st.ctypes.data_as(C.POINTER(f)),
                                              self.ist.ctypes.data_as(C.POINTER(C.c_int32)), self.sp.ctypes.data_as(C.POINTER(f)),
                                              nz.ctypes.data_as(C.POINTER(f)), n_steps, C.c_int64(self.n)))


_HSM = None


def _hostsim_modes_lib():
    global _HSM
    if _HSM is None:
        import subprocess
        import tempfile

        out = os.path.join(tempfile.mkdtemp(prefix="pfb_hostsim_modes_"), "libpfb_hostsim_modes.so")
        src = os.path.join(ROOT, "tests", "hostsim", "hostsim_modes.cpp")
        subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-mfma", "-ffp-contract=fast", "-o", out, src], check=True, capture_output=True)
        _HSM = C.CDLL(out)
        _HSM.hs_last_error.restype = C.c_char_p
    return _HSM


def _fp32_bars(g, err, ids, tag):
    """the bars test_hostsim_parity.py / test_gpu_parity.py use for single modes: per drone, by the modes it flies"""
    loose = np.isin(_mode_at(g), HEIGHT_LOOP).any(axis=0)[ids]
    assert err["contact_mismatch"].sum() == 0, (tag, err["contact_mismatch"])
    assert err["setpoint0"].max() < 1e-6, (tag, err["setpoint0"])
    # 1e-3 in one mode; a drone that re-enters position hold after a mode-1 phase (7 -> 1 -> 7) reaches 1.2e-3 on cf2x
    assert err["pos"][ids][loose].max(initial=0.0) < 1.5e-3, (tag, err["pos"])
    assert err["pos"][ids][~loose].max() < 0.5e-3 and err["euler"][ids][~loose].max() < 1e-3, (tag, err)


def test_hostsim_per_drone_path_matches_reference():
    """The kernel body's per-drone dispatch (quadx_set_mode_any / quadx_aviary_step_any; one engine per model) against the
    reference fixture.  cf2x drones: the bars test_hostsim_parity.py uses for single modes.  primitive_drone drones: this
    scenario (tumbling raw-PWM phases, mode switches mid-flight) amplifies fp32 rounding to centimetres on the single-mode path
    as well, so they are held to the single-mode host path flown drone by drone, bit for bit."""
    g = load_golden("mixed_modes_quadx")
    opts = _opts(g)
    engines, groups = [], {}
    for name in ("cf2x", "primitive_drone"):
        ids = [d for d, o in enumerate(opts) if o["drone_model"] == name]
        groups[name] = ids
        engines.append((HostSimModes(build_model("quadx", name), len(ids), g["start_pos"][ids], g["start_orn"][ids]), ids))
    err = replay_modes(g, engines)
    _fp32_bars(g, err, groups["cf2x"], "hostsim")
    single = _PerDrone(lambda o, p, r: HostSimEngine(_model(g, o), None, 1, p, r), opts, g)
    err1 = replay_modes(g, [(single, list(range(single.n)))])
    for k in ("setpoint", "pos", "euler", "angvel", "linvel", "aux"):
        assert np.array_equal(err[k], err1[k]), k


# ------------------------------------------------------------------------------------------------------------------ GPU
class CudaModes(CudaEngine):
    """CudaEngine over one BatchedAviary with a per-drone ``drone_options`` sequence and ``set_modes(list)``."""

    def __init__(self, drone_type, drone_options, start_pos, start_orn, seed=0):
        import torch

        from pyflyt_b200.core.aviary import BatchedAviary

        self.torch = torch
        self.n = len(drone_options)
        self.av = BatchedAviary(np.asarray(start_pos, dtype=np.float32), np.asarray(start_orn, dtype=np.float32), drone_type=drone_type,
                                drone_options=drone_options, seed=seed)
        self.aux_dim, self.ups, self.obs_dim = self.av.aux_dim, self.av.updates_per_step, self.av.obs_dim

    def set_modes(self, modes):
        self.av.set_mode(list(modes))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mixed_modes_quadx", "mixed_modes_fixedwing"])
def test_cuda_replays_mixed_mode_fixture(name):
    """ONE CUDA handle flies the reference's mixed-mode Aviary.  Fixed-wing and cf2x drones: the bars of
    test_gpu_parity.py::test_flight_modes / test_flight_modes_height_hold by the modes each drone flies.  primitive_drone
    drones (see test_hostsim_per_drone_path_matches_reference): one single-mode handle per drone, flown alongside, bit for bit."""
    g = load_golden(name)
    opts = _opts(g)
    eng = CudaModes(str(g["drone_type"]), opts, g["start_pos"], g["start_orn"])
    err = replay_modes(g, [(eng, list(range(eng.n)))])
    prim = [d for d, o in enumerate(opts) if o.get("drone_model") == "primitive_drone"]
    _fp32_bars(g, err, [d for d in range(eng.n) if d not in prim], name)
    if prim:  # every drone against a single-mode handle of its own: the same errors, bit for bit
        kind = str(g["drone_type"])
        single = _PerDrone(lambda o, p, r: CudaEngine(None, None, 1, p, r, drone_model=o["drone_model"], drone_type=kind), opts, g)
        err1 = replay_modes(g, [(single, list(range(single.n)))])
        for k in ("setpoint", "pos", "euler", "angvel", "linvel", "aux"):
            assert np.array_equal(err[k], err1[k]), k


def _layout(kind, n, rng):
    i = np.arange(n)
    if kind == "tile":
        return -1 + (i // 32) % 9
    if kind == "interleaved":
        return -1 + i % 9
    return rng.integers(-1, 8, n)


def _setpoints(mode, start, rng):
    """[n, 4] random in-range setpoints of ``mode`` (ranges of the single-mode fixtures; heights and mode-7 positions around
    the start)"""
    n = len(start)
    if mode == -1:
        return rng.uniform(0.3, 0.6, (n, 4))
    sp = np.column_stack([rng.uniform(-0.5, 0.5, (n, 3)), rng.uniform(0.2, 0.6, n)])
    if mode in (2, 3, 4, 7):
        sp[:, 3] = start[:, 2] + rng.uniform(-1.0, 1.0, n)
    if mode == 7:
        sp[:, :2] = start[:, :2] + rng.uniform(-1.0, 1.0, (n, 2))
    return sp


def _tile_words(av):
    """[N, rows] raw state words of every drone (warp-tiled [tiles][groups][32][4] -> drone-major)"""
    t = av.state_tensor
    return t.permute(0, 2, 1, 3).reshape(-1, av.state_rows)[: av.num_drones].contiguous().view(__import__("torch").int32)


def _assert_bit_identical(mixed, uniform, modes, tag):
    import torch

    idx = torch.as_tensor(modes, device=mixed.device)
    raw = _tile_words(mixed)
    for m, U in zip(range(-1, 8), uniform):
        sel = idx == m
        assert torch.equal(mixed.all_states[sel], U.all_states[sel]), (tag, m, "all_states")
        assert torch.equal(mixed.all_aux_states[sel], U.all_aux_states[sel]), (tag, m, "aux")
        assert torch.equal(mixed.contact_array[sel], U.contact_array[sel]), (tag, m, "contact")
        assert torch.equal(mixed.setpoints[sel], U.setpoints[sel]), (tag, m, "setpoints")
        assert torch.equal(raw[sel], _tile_words(U)[sel]), (tag, m, "raw state")


@pytest.mark.gpu
@pytest.mark.parametrize("n_models", [1, 2])
@pytest.mark.parametrize("layout", ["tile", "interleaved", "random"])
def test_per_drone_modes_bit_identical_to_uniform_handles(layout, n_models):
    """65 536 drones, one mode per drone, Philox noise: drone i equals drone i of a uniform handle of its mode, bit for bit,
    after set_mode(list) and after every chunk of steps (state words, observations, aux, contact, setpoints)."""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    n = 65536
    rng = np.random.default_rng(5 + n_models)
    start = np.column_stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(20, 30, n)]).astype(np.float32)
    orn = rng.uniform(-0.3, 0.3, (n, 3)).astype(np.float32)
    opts = [dict(drone_model="cf2x" if (i // 2) % 2 == 0 or n_models == 1 else "primitive_drone") for i in range(n)]
    if n_models == 1:
        opts = dict(drone_model="cf2x")
    modes = _layout(layout, n, rng)
    mixed = BatchedAviary(start, orn, drone_options=opts, seed=11)
    uniform = [BatchedAviary(start, orn, drone_options=opts, seed=11) for _ in range(9)]
    assert len(mixed.models) == n_models
    mixed.set_mode(modes.tolist())
    for m, U in zip(range(-1, 8), uniform):
        U.set_mode(m)
    _assert_bit_identical(mixed, uniform, modes, "set_mode")
    dev = mixed.device
    for chunk in (1, 24, 25, 50):
        sps = [_setpoints(m, start, rng).astype(np.float32) for m in range(-1, 8)]
        mixed_sp = np.stack(sps)[modes + 1, np.arange(n)]
        mixed.set_all_setpoints(torch.as_tensor(mixed_sp, device=dev))
        for m, U in zip(range(-1, 8), uniform):
            U.set_all_setpoints(torch.as_tensor(sps[m + 1], device=dev))
        for a in [mixed] + uniform:
            a.step(chunk)
        _assert_bit_identical(mixed, uniform, modes, chunk)
    # the modes really differ in flight
    z = mixed.all_states[:, 3, 2]
    assert float(z.max() - z.min()) > 1.0


def _group_oracles(model, start, orn, keys):
    """one oracle per distinct mode history (row of ``keys``): [(engine, drone ids)]"""
    out = []
    for key in np.unique(keys, axis=0):
        ids = np.flatnonzero((keys == key).all(axis=1))
        out.append((OracleEngine(model, None, len(ids), start[ids], orn[ids]), ids))
    return out


@pytest.mark.gpu
def test_mode_sequence_matches_oracle():
    """set_mode(list) -> steps -> set_mode(int) -> steps -> set_mode(list2) -> reset() -> set_mode(list3) -> steps on 4096 cf2x
    drones against the oracle (bars of test_batch_4096_matches_oracle; 2e-3 for the drones that have flown a height-hold mode, 2, 3,
    4 or 7: under these random height setpoints the height chain of the uniform kernels reaches 1.2e-3 within 60 steps, and
    the velocity error it leaves keeps the position drifting after the drone leaves the mode)."""
    n = 4096
    rng = np.random.default_rng(17)
    f = lambda a: a.astype(np.float32).astype(np.float64)  # noqa: E731
    start = f(np.column_stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(20, 30, n)]))
    orn = f(rng.uniform(-0.3, 0.3, (n, 3)))
    i = np.arange(n)
    list1, list2, list3 = -1 + i % 9, -1 + (i // 9) % 9, -1 + (i + 3) % 9
    model = build_model("quadx", "cf2x")
    cud = CudaModes("quadx", [dict(drone_model="cf2x")] * n, start, orn)
    orcs = _group_oracles(model, start, orn, np.column_stack([list1, list2, list3]))
    loose = np.zeros(n, dtype=bool)

    def run(steps, modes_now):
        nonlocal loose
        loose |= np.isin(modes_now, HEIGHT_HOLD)
        for _ in range(0, steps, 10):
            sps = np.stack([f(_setpoints(m, start, rng)) for m in range(-1, 8)])
            sp = sps[modes_now + 1, i]
            noise = f(rng.normal(4.0, 1.0, (10 * cud.ups, n)))
            cud.set_setpoints(sp)
            cud.aviary_step(noise, n_steps=10)
            for o, ids in orcs:
                o.set_setpoints(sp[ids])
                o.aviary_step(noise[:, ids], n_steps=10)
        a = cud.state()
        for o, ids in orcs:
            b = o.state()
            tol = np.where(loose[ids], 2e-3, 0.5e-3)
            assert (np.abs(a[ids, 3] - b[:, 3]).max(axis=1) < tol).all(), (modes_now[ids[0]], np.abs(a[ids, 3] - b[:, 3]).max())
            assert np.array_equal(o.contact(), cud.contact()[ids])
            if not loose[ids].any():
                assert np.abs(a[ids, 0] - b[:, 0]).max() < 2e-3

    def set_modes(modes):
        cud.set_modes(modes.tolist())
        for o, ids in orcs:
            o.set_mode(int(modes[ids[0]]))  # every drone of a group shares its mode history
        got = cud.get_setpoints()
        for o, ids in orcs:
            assert np.abs(got[ids] - o.get_setpoints()).max() < 2e-3  # mode 7 / height presets hold the drifted pose

    for e in [cud] + [o for o, _ in orcs]:
        e.reset()
    set_modes(list1)
    run(30, list1)
    cud.set_mode(0)  # mode 0: no z-velocity loop to amplify what the first phase left (mode 6's limit cycle, DESIGN.md §5)
    for o, _ in orcs:
        o.set_mode(0)
    run(20, np.full(n, 0))
    set_modes(list2)
    cud.reset()
    for o, _ in orcs:
        o.reset()
    loose[:] = False
    set_modes(list3)
    run(30, list3)


@pytest.mark.gpu
def test_fixedwing_interleaved_modes_bit_identical_to_uniform_handles():
    """4096 fixed-wing drones, modes -1 / 0 interleaved, Philox noise, against a uniform handle of each mode."""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    n = 4096
    rng = np.random.default_rng(23)
    start = np.column_stack([rng.uniform(-5, 5, n), rng.uniform(-5, 5, n), rng.uniform(60, 80, n)]).astype(np.float32)
    orn = np.column_stack([np.zeros(n), rng.uniform(-0.1, 0.1, n), rng.uniform(-np.pi, np.pi, n)]).astype(np.float32)
    modes = np.arange(n) % 2 - 1
    kw = dict(drone_type="fixedwing", seed=9)
    mixed = BatchedAviary(start, orn, **kw)
    uniform = [BatchedAviary(start, orn, **kw) for _ in range(2)]
    mixed.set_mode(modes.tolist())
    for m, U in zip((-1, 0), uniform):
        U.set_mode(m)
    dev = mixed.device
    for chunk in (1, 30, 69):
        sps = [np.column_stack([rng.uniform(-0.8, 0.8, (n, 5)), rng.uniform(0, 1, n)]),
               np.column_stack([rng.uniform(-0.6, 0.6, (n, 3)), rng.uniform(0.3, 1.0, n), np.zeros((n, 2))])]
        sps = [torch.as_tensor(s, dtype=torch.float32, device=dev) for s in sps]
        mixed.set_all_setpoints(torch.where(torch.as_tensor(modes == -1, device=dev)[:, None], sps[0], sps[1]))
        for s, U in zip(sps, uniform):
            U.set_all_setpoints(s)
        for a in [mixed] + uniform:
            a.step(chunk)
        for m, U in zip((-1, 0), uniform):
            sel = torch.as_tensor(modes == m, device=dev)
            assert torch.equal(mixed.all_states[sel], U.all_states[sel]), (chunk, m)
            assert torch.equal(mixed.all_aux_states[sel], U.all_aux_states[sel]), (chunk, m)
            assert torch.equal(mixed.contact_array[sel], U.contact_array[sel]), (chunk, m)
            assert torch.equal(mixed.state_tensor[:, sel], U.state_tensor[:, sel]), (chunk, m)
            assert torch.equal(mixed.istate_tensor[:, sel], U.istate_tensor[:, sel]), (chunk, m)


@pytest.mark.gpu
def test_set_mode_refusals():
    from pyflyt_b200 import _lib
    from pyflyt_b200.core.aviary import BatchedAviary

    z = np.zeros((3, 3), dtype=np.float32)
    z[:, 2] = 10.0
    q = BatchedAviary(z, np.zeros((3, 3)))
    with pytest.raises(AssertionError, match=re.escape("Expected 3 flight_modes, got 2.")):
        q.set_mode([0, 1])
    msg = "`mode` must be between -1 and 7 or be registered in self.registered_controllers.keys()=dict_keys([]), got 8."
    with pytest.raises(ValueError, match=re.escape(msg)):
        q.set_mode([0, 8, 1])
    fw = BatchedAviary(z, np.zeros((3, 3)), drone_type="fixedwing")
    with pytest.raises(ValueError, match=re.escape("`mode` must be between -1 and 0 or be registered")):
        fw.set_mode([-1, 1, 0])
    rk = BatchedAviary(z, np.zeros((3, 3)), drone_type="rocket")
    with pytest.raises(ValueError, match=re.escape("`mode` must be between 0 and 0 or be registered")):
        rk.set_mode([0, 1, 0])
    rk.set_mode([0, 0, 0])  # all zeros: the rocket's one mode
    # the C-ABI refuses an out-of-range entry naming the drone, and a null array
    L = _lib.lib()
    bad = np.array([0, 3, 9], dtype=np.int8)
    with pytest.raises(_lib.PfbError, match=re.escape("modes[2] = 9")):
        _lib.check(L.pfb_set_modes(q._h, bad.ctypes.data_as(C.c_void_p), q._s()))
    with pytest.raises(_lib.PfbError, match="null"):
        _lib.check(L.pfb_set_modes(q._h, None, q._s()))
    # env handles fly their env's flight_mode
    from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverVecEnv

    env = QuadXHoverVecEnv(num_envs=64, seed=0)
    with pytest.raises(_lib.PfbError, match="Aviary handles"):
        env.aviary.set_mode([0, 1] * 32)
    env.close()


@pytest.mark.gpu
def test_uniform_list_and_reset_return_to_the_uniform_kernels():
    """An all-equal list is set_mode(int); set_mode(int) and reset() leave the per-drone path; a masked reset keeps it."""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    n = 2048
    rng = np.random.default_rng(3)
    start = np.column_stack([np.zeros(n), np.zeros(n), rng.uniform(10, 20, n)]).astype(np.float32)
    a, b = BatchedAviary(start, np.zeros((n, 3)), seed=2), BatchedAviary(start, np.zeros((n, 3)), seed=2)
    a.set_mode([7] * n)
    b.set_mode(7)
    a.set_mode((np.arange(n) % 2 * 7).tolist())
    a.set_mode(7)
    for x in (a, b):
        x.step(20)
    assert torch.equal(a.state_tensor, b.state_tensor) and torch.equal(a.setpoints, b.setpoints)
    a.set_mode((np.arange(n) % 2 * 7).tolist())
    a.reset()
    b.reset()
    for x in (a, b):
        x.step(20)
    assert torch.equal(a.state_tensor, b.state_tensor)
