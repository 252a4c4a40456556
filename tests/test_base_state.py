"""Base-state calls on Aviary handles: ``BatchedAviary.set_base_state`` / ``set_base_velocity`` / ``base_state`` (the reference's
resetBasePositionAndOrientation / resetBaseVelocity + ``drone.update_state()`` and getBasePositionAndOrientation /
getBaseVelocity), for a mask of drones, on every kind of Aviary handle.

CPU: the C oracle (with the base-state reset of tests/oracle_base_state.c) and the host build of the per-drone bodies (tests/hostsim/hostsim_base_state.cpp) replay the reference's
scripts that move drones between Aviary steps (tests/golden/base_state_*.npz, tools/gen_golden.py); the argument checks.
GPU: one CUDA handle replays each fixture; a state read from one handle and written into another makes them fly bit for bit
alike; a round trip changes nothing; masked drones keep their modes, models, controller memories and throttles and the others
stay untouched; a mixed handle's resets equal those of single-kind handles."""
import ctypes as C
import glob
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

from engines import GOLDEN, ROOT, HostSimEngine, _p, build_model, load_golden
from pyflyt_b200.models import PfbEnvConfig

FIXTURES = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, "base_state_*.npz")))
SP_DIM = {"quadx": 4, "fixedwing": 6, "rocket": 7}
AUX_DIM = {"quadx": 4, "fixedwing": 6, "rocket": 9}
HEIGHT_HOLD = (2, 3, 4, 7)


def _kinds(g):
    return json.loads(str(g["drone_type"]))


def _options(g):
    return json.loads(str(g["drone_options"]))


def _contact_config():
    e = PfbEnvConfig()
    e.contact_response = 1
    return e


def _reset_args(g, k):
    has = g["reset_has"][k]
    return dict(mask=g["reset_mask"][k], pos=g["reset_pos"][k] if has[0] else None, quat=g["reset_quat"][k] if has[0] else None,
                lin=g["reset_lin"][k] if has[1] else None, ang=g["reset_ang"][k] if has[2] else None)


def replay(g, eng):
    """Replays a base_state fixture through ``eng`` (all drones); max abs errors per drone, and the contact mismatches."""
    n, T = int(g["n_drones"]), len(g["state"])
    noise = g["noise"].reshape(T, -1, n)
    resets = {int(s): k for k, s in enumerate(g["reset_steps"])}
    err = {k: np.zeros(n) for k in ("pos", "euler", "angvel", "linvel", "aux")}
    err["contact_mismatch"] = np.zeros(n, dtype=int)
    eng.reset()
    eng.set_modes([int(m) for m in g["modes"]])
    for i in range(T):
        if i in resets:
            eng.set_base_state(**_reset_args(g, resets[i]))
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


class _PerDrone:
    """One single-drone engine per drone of a fixture, each of its own kind and model: the reference's Aviary loops over its
    drones the same way, and a fixture without floor contact couples none of them."""

    def __init__(self, g, make):
        self.kinds = _kinds(g)
        cfg = _contact_config() if bool(g["contact_response"]) else None
        self.engines = [make(build_model(k, o.get("drone_model")), cfg, g["start_pos"][d][None], g["start_orn"][d][None])
                        for d, (k, o) in enumerate(zip(self.kinds, _options(g)))]

    def reset(self):
        for e in self.engines:
            e.reset()

    def set_modes(self, modes):
        for e, m in zip(self.engines, modes):
            e.set_mode(int(m))

    def set_setpoints(self, sp):
        for d, (e, k) in enumerate(zip(self.engines, self.kinds)):
            e.set_setpoints(np.asarray(sp[d][: SP_DIM[k]])[None])

    def set_base_state(self, mask, pos, quat, lin, ang):
        row = lambda a, d: None if a is None else a[d][None]  # noqa: E731
        for d, e in enumerate(self.engines):
            if mask[d]:
                e.set_base_state(row(pos, d), row(quat, d), row(lin, d), row(ang, d))

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


_ORC = None


def oracle_base_state_lib():
    """tests/oracle_base_state.c: the fp64 oracle with orc_set_base_state, built with the oracle's flags (oracle/Makefile)"""
    global _ORC
    if _ORC is None:
        out = os.path.join(tempfile.mkdtemp(prefix="pfb_oracle_base_state_"), "libpfb_oracle_base_state.so")
        src = os.path.join(ROOT, "tests", "oracle_base_state.c")
        subprocess.run(["/usr/bin/gcc", "-O2", "-fPIC", "-fopenmp", "-ffp-contract=off", "-shared", "-o", out, src, "-lm"], check=True, capture_output=True)
        L = C.CDLL(out)
        vp, dp, u8p = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_uint8)
        L.orc_create.restype = vp
        L.orc_create.argtypes = [vp, vp, C.c_int64, C.c_uint64]
        L.orc_destroy.argtypes = [vp]
        L.orc_updates_per_step.argtypes = [vp]
        L.orc_set_start.argtypes = [vp, dp, dp]
        L.orc_reset.argtypes = [vp, u8p]
        L.orc_set_mode.argtypes = [vp, C.c_int]
        L.orc_set_setpoints.argtypes = [vp, dp, C.c_int]
        L.orc_aviary_step.argtypes = [vp, C.c_int, dp]
        L.orc_get_state.argtypes = [vp, dp]
        L.orc_get_aux.argtypes = [vp, dp, C.c_int]
        L.orc_get_contact.argtypes = [vp, u8p]
        L.orc_set_base_state.argtypes = [vp, u8p, dp, dp, dp, dp]
        _ORC = L
    return _ORC


class _Oracle:
    """One drone on the fp64 oracle (the calls of oracle.oracle.Oracle that the replay needs, plus orc_set_base_state)"""

    def __init__(self, model, cfg, start_pos, start_orn):
        self.L = oracle_base_state_lib()
        self.model, self.cfg = model, cfg
        self.aux_dim = {0: 4, 1: 6, 2: 9}[int(model.kind)]
        self.h = self.L.orc_create(C.byref(model), None if cfg is None else C.byref(cfg), 1, 0)
        assert self.h
        self.L.orc_set_start(self.h, _d(start_pos, 3), _d(start_orn, 3))

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_destroy(self.h)
            self.h = None

    def reset(self):
        self.L.orc_reset(self.h, None)

    def set_mode(self, mode):
        self.L.orc_set_mode(self.h, int(mode))

    def set_setpoints(self, sp):
        sp = np.ascontiguousarray(sp, dtype=np.float64)
        self.L.orc_set_setpoints(self.h, _p(sp, C.c_double), sp.shape[1])

    def set_base_state(self, pos, quat, lin, ang):
        self._keep = [_arr(pos, 3), _arr(quat, 4), _arr(lin, 3), _arr(ang, 3)]
        self.L.orc_set_base_state(self.h, None, *[_p(a, C.c_double) for a in self._keep])

    def aviary_step(self, noise):
        nz = np.ascontiguousarray(noise, dtype=np.float64)
        self.L.orc_aviary_step(self.h, 1, _p(nz, C.c_double))

    def state(self):
        out = np.zeros(12)
        self.L.orc_get_state(self.h, _p(out, C.c_double))
        return out.reshape(1, 4, 3)

    def aux(self):
        out = np.zeros((1, self.aux_dim))
        self.L.orc_get_aux(self.h, _p(out, C.c_double), self.aux_dim)
        return out

    def contact(self):
        out = np.zeros(1, dtype=np.uint8)
        self.L.orc_get_contact(self.h, _p(out, C.c_uint8))
        return out


def _arr(a, w):
    return None if a is None else np.ascontiguousarray(np.reshape(a, (1, w)), dtype=np.float64)


def _d(a, w):
    return _p(_arr(a, w), C.c_double)


_HSB = None


def hostsim_base_state_lib():
    global _HSB
    if _HSB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="pfb_hostsim_base_state_"), "libpfb_hostsim_base_state.so")
        src = os.path.join(ROOT, "tests", "hostsim", "hostsim_base_state.cpp")
        subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-mfma", "-ffp-contract=fast", "-o", out, src], check=True, capture_output=True)
        _HSB = C.CDLL(out)
        _HSB.hs_last_error.restype = C.c_char_p
    return _HSB


class _HostSim(HostSimEngine):
    """HostSimEngine over tests/hostsim/hostsim_base_state.cpp; the Aviary steps of the kernels: the contact response when the
    fixture has it, and the fixed-wing's one-basic-block substep for a complete model in still air"""

    def __init__(self, model, cfg, start_pos, start_orn):
        super().__init__(model, None, 1, start_pos, start_orn)
        self.L = hostsim_base_state_lib()
        self.contact_response = cfg is not None
        self.full_block = self.fw and int(model.n_surfaces) == 5

    def set_base_state(self, pos, quat, lin, ang):
        d = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)  # noqa: E731
        pos, quat, lin, ang = d(pos), d(quat), d(lin), d(ang)
        f64 = C.c_double
        self._chk(self.L.hs_set_base_state(int(self.model.kind), _p(self.st, C.c_float), _p(self.ist, C.c_int32), None, _p(pos, f64), _p(quat, f64),
                                           _p(lin, f64), _p(ang, f64), C.c_int64(self.n)))

    def aviary_step(self, noise, n_steps=1):
        if not self.contact_response:
            return super().aviary_step(noise, n_steps)
        nz = np.ascontiguousarray(noise, dtype=np.float32)
        f, i32, n = C.c_float, C.c_int32, C.c_int64(self.n)
        if self.rk:
            self._chk(self.L.hs_rk_aviary_step_contact(C.byref(self.model), _p(self.st, f), _p(self.ist, i32), _p(self.sp, f), _p(nz, f), n_steps, n))
        elif self.fw:
            self._chk(self.L.hs_fw_aviary_step_contact(C.byref(self.model), self.mode, int(self.full_block), _p(self.st, f), _p(self.ist, i32), _p(self.sp, f),
                                                       _p(nz, f), n_steps, n))
        else:
            self._chk(self.L.hs_aviary_step_contact(C.byref(self.model), self.mode, _p(self.st, f), _p(self.ist, i32), _p(self.sp, f), _p(nz, f), n_steps, n))


def _oracle_bars(g):
    """1e-9 in free flight; 1e-6 for a drone that holds height (the bar of test_mixed_kinds.py) or rests on the floor (the bar of
    the ground_* replays)"""
    tight = np.full(int(g["n_drones"]), 1e-9)
    tight[np.isin(g["modes"], HEIGHT_HOLD)] = 1e-6
    if bool(g["contact_response"]):
        tight[:] = 1e-6
    return tight


# fp32 bars against the reference: the free-flight bars of the GPU parity tests (pos 1e-3 m, euler 1e-3 rad, rates and
# velocities 1e-2), or what the host build of the kernel body shows x5, rounded up, where that is more (the rule of
# test_aviary_ground_contact.py).  A tilted drone dropped into a position hold or onto the floor amplifies fp32 rounding in
# its attitude loop or at each strike.  Host build, max over the drones:   pos      euler    angvel   linvel
#   base_state_quadx (cf2x teleported tilted into mode 7)                   5.3e-5   2.4e-4   4.1e-2   8.7e-4
#   base_state_ground_fixedwing                                             5.4e-4   5.9e-3   8.9e-2   9.3e-2
#   base_state_ground_rocket                                                5.7e-3   4.4e-3   0.12     8.1e-2
#   base_state_mixed (primitive_drone teleported and thrown into mode 7)   2.3e-3   9.8e-3   0.16     6.6e-2
#   the other fixtures                                                      < 8e-6   < 3e-6   < 2e-4   < 7e-6
FREE = dict(pos=1e-3, euler=1e-3, angvel=1e-2, linvel=1e-2)
BARS = {name: FREE for name in FIXTURES}
BARS["base_state_quadx"] = dict(FREE, angvel=0.25)
BARS["base_state_ground_fixedwing"] = dict(pos=3e-3, euler=3e-2, angvel=0.5, linvel=0.5)
BARS["base_state_ground_rocket"] = dict(pos=3e-2, euler=2.5e-2, angvel=0.6, linvel=0.45)
BARS["base_state_mixed"] = dict(pos=1.2e-2, euler=5e-2, angvel=0.8, linvel=0.35)


def _fp32_bars(name, err):
    assert err["contact_mismatch"].sum() == 0, (name, err["contact_mismatch"])
    for k, bar in BARS[name].items():
        assert err[k].max() < bar, (name, k, err[k], bar)


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_fixtures_cover_the_scenarios():
    assert FIXTURES == ["base_state_acrowing", "base_state_fixedwing", "base_state_ground_cf2x", "base_state_ground_fixedwing",
                        "base_state_ground_rocket", "base_state_mixed", "base_state_quadx", "base_state_rocket"]
    for name in FIXTURES:
        g = load_golden(name)
        assert len(g["reset_steps"]) >= 1 and g["reset_mask"].any(), name
        assert g["contact"].any() == bool(g["contact_response"]), name  # the ground fixtures land, the others never touch
    mixed = load_golden("base_state_mixed")
    assert _kinds(mixed) == ["quadx", "fixedwing", "rocket", "quadx"] and mixed["reset_mask"].tolist() == [[0, 1, 0, 1]]


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_replays_base_state_fixture(name):
    g = load_golden(name)
    err = replay(g, _PerDrone(g, _Oracle))
    bar = _oracle_bars(g)
    assert err["contact_mismatch"].sum() == 0, err["contact_mismatch"]
    for k in ("pos", "euler", "angvel", "linvel", "aux"):
        assert (err[k] < bar).all(), (name, k, err[k])


@pytest.mark.parametrize("name", FIXTURES)
def test_hostsim_replays_base_state_fixture(name):
    g = load_golden(name)
    err = replay(g, _PerDrone(g, _HostSim))
    print(f"\n[{name}] host build: " + "  ".join(f"{k} {err[k].max():.1e}" for k in ("pos", "euler", "angvel", "linvel")))
    _fp32_bars(name, err)


def test_hostsim_set_then_get_returns_what_was_set():
    """The host build of the bodies: a pose and velocities written, then read back, come back to the hi + lo rounding; a pose
    alone zeroes both velocities; what is not given keeps its value."""
    L = hostsim_base_state_lib()
    rng = np.random.default_rng(0)
    n = 64
    for kind in (0, 1, 2):
        e = _HostSim(build_model(["quadx", "fixedwing", "rocket"][kind]), None, np.array([[0.0, 0.0, 10.0]]), np.zeros((1, 3)))
        e.n = n
        e.st = np.zeros((e.st.shape[0], n), dtype=np.float32)
        e.ist = np.zeros((e.ist.shape[0], n), dtype=np.int32)
        pos = rng.uniform(-50, 50, (n, 3))
        quat = rng.normal(size=(n, 4))
        quat /= np.linalg.norm(quat, axis=1, keepdims=True)
        lin, ang = rng.uniform(-20, 20, (n, 3)), rng.uniform(-3, 3, (n, 3))
        e.set_base_state(pos, quat, lin, ang)
        out = [np.zeros((n, 3)), np.zeros((n, 4)), np.zeros((n, 3)), np.zeros((n, 3))]
        L.hs_get_base_state(kind, _p(e.st, C.c_float), _p(e.ist, C.c_int32), *[_p(o, C.c_double) for o in out], C.c_int64(n))
        for a, b in zip((pos, quat, lin), out[:3]):
            assert np.abs(a - b).max() <= 1e-13 * max(1.0, np.abs(a).max())
        assert np.abs(out[3] - ang).max() < 1e-5 * 3  # the body rate is fp32
        e.set_base_state(pos[::-1].copy(), quat[::-1].copy(), None, None)
        L.hs_get_base_state(kind, _p(e.st, C.c_float), _p(e.ist, C.c_int32), *[_p(o, C.c_double) for o in out], C.c_int64(n))
        assert not out[2].any() and not out[3].any()
        e.set_base_state(None, None, None, ang)
        L.hs_get_base_state(kind, _p(e.st, C.c_float), _p(e.ist, C.c_int32), *[_p(o, C.c_double) for o in out], C.c_int64(n))
        assert np.abs(out[0] - pos[::-1]).max() < 1e-12 and not out[2].any() and np.abs(out[3] - ang).max() < 3e-5


def test_capi_refuses_bad_calls_before_the_device():
    """pos without quat and env handles are refused with a message; the checks need a bound handle, so without a device the
    handle is NULL and the call says so"""
    from pyflyt_b200 import _lib

    try:
        L = _lib.lib()
    except _lib.PfbError as e:
        pytest.skip(str(e))
    assert L.pfb_set_base_state(None, None, None, None, None, None, None) != 0 and b"null handle" in L.pfb_last_error()
    assert L.pfb_get_base_state(None, None, None, None, None, None) != 0 and b"null handle" in L.pfb_last_error()


# ------------------------------------------------------------------------------------------------------------------ GPU
class CudaBaseStateEngine:
    """One BatchedAviary over all drones of a fixture: a mixed handle for several kinds, a QuadX model set for several QuadX
    models"""

    def __init__(self, g, **kw):
        from pyflyt_b200.core.aviary import BatchedAviary

        kinds, opts = _kinds(g), _options(g)
        one_kind = len(set(kinds)) == 1
        self.av = BatchedAviary(np.asarray(g["start_pos"], dtype=np.float32), np.asarray(g["start_orn"], dtype=np.float32),
                                drone_type=kinds[0] if one_kind else kinds, drone_options=opts[0] if len({json.dumps(o) for o in opts}) == 1 else opts,
                                contact_response=bool(g["contact_response"]), **kw)
        self.kinds = kinds

    def reset(self):
        self.av.reset()

    def set_modes(self, modes):
        self.av.set_mode(list(modes))

    def set_setpoints(self, sp):
        self.av.set_all_setpoints(np.ascontiguousarray(np.asarray(sp)[:, : self.av.setpoint_dim], dtype=np.float32))

    def set_base_state(self, mask, pos, quat, lin, ang):
        self.av.set_base_state(pos=pos, quat=quat, lin_vel=lin, ang_vel=ang, mask=np.asarray(mask, dtype=bool))

    def aviary_step(self, noise):
        import torch

        self.av.step(1, torch.as_tensor(np.ascontiguousarray(noise, dtype=np.float32), device="cuda"))

    def state(self):
        return self.av.all_states.cpu().double().numpy()

    def aux(self):
        self.av.all_states
        a = self.av._aux_state.cpu().double().numpy()
        out = np.zeros((len(self.kinds), 9))
        out[:, : a.shape[1]] = a
        return out

    def contact(self):
        return self.av.contact_array.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_cuda_replays_base_state_fixture(name):
    """One CUDA handle per fixture (the mixed fixture: one mixed handle) within the fp32 bars; contact flags at every step"""
    g = load_golden(name)
    err = replay(g, CudaBaseStateEngine(g))
    print(f"\n[{name}] CUDA: " + "  ".join(f"{k} {err[k].max():.1e}" for k in ("pos", "euler", "angvel", "linvel")))
    _fp32_bars(name, err)


def _kind_setup(kind, n, seed):
    rng = np.random.default_rng(seed)
    start = np.column_stack([rng.uniform(-5, 5, n), rng.uniform(-5, 5, n), rng.uniform(30, 60, n)]).astype(np.float32)
    orn = rng.uniform(-0.2, 0.2, (n, 3)).astype(np.float32)
    if kind == "rocket":
        sp = np.tile(np.array([[0.1, -0.1, 0.05, 1.0, 0.6, 0.1, -0.1]], dtype=np.float32), (n, 1))
        modes = [0] * n
    elif kind == "fixedwing":
        sp = np.tile(np.array([[0.2, -0.1, 0.1, 0.8, 0.0, 0.0]], dtype=np.float32), (n, 1))
        modes = [0] * n
    else:
        modes = [[0, 7, 6, -1][i % 4] for i in range(n)]
        sp = np.zeros((n, 4), dtype=np.float32)
        for i, m in enumerate(modes):
            sp[i] = [start[i, 0] + 1.0, start[i, 1] - 1.0, 0.3, start[i, 2] + 0.5] if m == 7 else ([0.3, 0.31, 0.32, 0.3] if m == -1 else [0.1, -0.1, 0.2, 0.4])
    return start, orn, modes, sp


def _words(av):
    """every state word of a handle, as int32 bits, plus its istate"""
    import torch

    torch.cuda.synchronize()
    return av.state_tensor.reshape(-1).view(torch.int32).clone(), av.istate_tensor.clone()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["quadx", "fixedwing", "rocket", "mixed"])
def test_transplant_flies_bit_for_bit(kind):
    """Two handles with one seed: B starts at pose P, A elsewhere.  Right after reset() B's state, read with base_state(), is
    written into A with set_base_state; B's angular velocity is still zero, so nothing is lost to the body-rate conversion.  A
    then flies bit for bit like B."""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    n = 4096
    if kind == "mixed":
        kinds = [["quadx", "fixedwing", "rocket", "quadx", "rocket"][(i + i // 32) % 5] for i in range(n)]
        start, orn = _kind_setup("quadx", n, 1)[:2]
        modes = [{"quadx": 7, "fixedwing": 0, "rocket": 0}[k] for k in kinds]
        sp = np.zeros((n, 7), dtype=np.float32)
        for i, k in enumerate(kinds):
            sp[i, : SP_DIM[k]] = {"quadx": [start[i, 0] + 1.0, start[i, 1], 0.2, start[i, 2]], "fixedwing": [0.2, -0.1, 0.1, 0.8, 0, 0],
                                  "rocket": [0.1, -0.1, 0.05, 1.0, 0.6, 0.1, -0.1]}[k]
        dt = kinds
    else:
        start, orn, modes, sp = _kind_setup(kind, n, 1)
        dt = kind
    other = start + np.float32(7.0)
    B = BatchedAviary(start, orn, drone_type=dt, seed=5)
    A = BatchedAviary(other, -orn, drone_type=dt, seed=5)
    for av in (A, B):
        av.reset()
        av.set_mode(modes)
    pos, quat, lin, ang = B.base_state()
    assert not bool(ang.any())
    A.set_base_state(pos, quat, lin, ang)
    assert torch.equal(_words(A)[0], _words(B)[0]) and torch.equal(_words(A)[1], _words(B)[1])
    for av in (A, B):
        av.set_all_setpoints(sp)
    for _ in range(100):
        A.step(1)
        B.step(1)
    assert torch.equal(_words(A)[0], _words(B)[0]) and torch.equal(_words(A)[1], _words(B)[1])
    assert torch.equal(A.all_states, B.all_states)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["quadx", "fixedwing", "rocket", "mixed"])
def test_round_trip_changes_nothing(kind):
    """set_base_state(*base_state()) after flight leaves every state word bit-identical except the body angular velocity, which
    goes through R w and back: within 2 ulp of the drone's rate magnitude (a rotation keeps the vector to its own precision, not
    a component far smaller than it)"""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    n = 1000
    kinds = [["quadx", "fixedwing", "rocket"][i % 3] for i in range(n)] if kind == "mixed" else kind
    start, orn, modes, sp = _kind_setup("quadx" if kind == "mixed" else kind, n, 2)
    av = BatchedAviary(start, orn, drone_type=kinds, seed=3)
    if kind == "quadx":
        av.set_mode(modes)
    if kind != "mixed":
        av.set_all_setpoints(sp)
    av.step(60)
    w0, ist0 = av.all_states[:, 0].clone(), av.istate_tensor.clone()
    rest0 = av.all_states[:, 1:].clone()
    aux0 = [a.clone() for a in av.all_aux_states]
    base0 = av.base_state()
    rows0 = None if kind == "mixed" else torch.stack([av.state_row(r) for r in range(av.state_rows)])
    av.set_base_state(*base0)
    assert torch.equal(av.istate_tensor, ist0)
    assert torch.equal(av.all_states[:, 1:], rest0) and all(torch.equal(a, b) for a, b in zip(av.all_aux_states, aux0))
    for x, y in zip(av.base_state()[:3], base0[:3]):
        assert torch.equal(x, y)
    w1 = av.all_states[:, 0]
    ulp = torch.finfo(torch.float32).eps * torch.linalg.vector_norm(w0, dim=1, keepdim=True)
    assert bool(((w1 - w0).abs() <= 2 * ulp).all()), float(((w1 - w0).abs() / ulp.clamp_min(1e-38)).max())
    if rows0 is not None:  # every other word of the state tensor, bit for bit (rows 10-12: QX_ANGVEL = FW_ANGVEL = RK_ANGVEL)
        rows1 = torch.stack([av.state_row(r) for r in range(av.state_rows)])
        keep = [r for r in range(av.state_rows) if r not in (10, 11, 12)]
        assert torch.equal(rows1[keep].view(torch.int32), rows0[keep].view(torch.int32))


@pytest.mark.gpu
def test_masked_reset_keeps_the_rest_quadx_model_set():
    """A QuadX model-set handle with one mode per drone: a masked set_base_state leaves the drones outside the mask bit for
    bit, keeps the masked drones' modes, model indices, PID memories and throttles, and their next steps go on in their modes"""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    n = 1024 + 19
    start, orn, modes, sp = _kind_setup("quadx", n, 4)
    opts = [dict(drone_model="cf2x" if (i // 5) % 2 == 0 else "primitive_drone") for i in range(n)]
    av = BatchedAviary(start, orn, drone_type="quadx", drone_options=opts, seed=8)
    ref = BatchedAviary(start, orn, drone_type="quadx", drone_options=opts, seed=8)
    for a in (av, ref):
        a.set_mode(modes)
        a.set_all_setpoints(sp)
        a.step(50)
    rng = np.random.default_rng(9)
    mask = rng.random(n) < 0.4
    m = torch.as_tensor(mask, device="cuda")
    pos = torch.as_tensor(start + np.float32(3.0), dtype=torch.float64)
    quat = torch.zeros((n, 4), dtype=torch.float64)
    quat[:, 3] = 1.0
    pid_rows = list(range(19, 25)) + list(range(40, 58))
    kept_rows = [13, 14, 15, 16, 17, 18] + pid_rows + [36, 37, 38, 39]  # throttles, step count, flags, PID memories, last motor command
    before = torch.stack([av.state_row(r) for r in range(60)])
    av.set_base_state(pos=pos, quat=quat, lin_vel=np.ones((n, 3)), mask=mask)
    after = torch.stack([av.state_row(r) for r in range(60)])
    same = lambda a, b: torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))  # noqa: E731
    assert same(after[:, ~m], before[:, ~m])
    assert same(after[kept_rows][:, m], before[kept_rows][:, m])
    assert float((av.precise_positions[m] - pos.cuda()[m]).abs().max()) < 1e-12
    assert torch.equal(av.model_index, ref.model_index)
    # the unmasked drones fly on exactly as the untouched handle's; the masked ones in their own modes from the new pose
    av.step(20)
    ref.step(20)
    assert torch.equal(av.all_states[~m], ref.all_states[~m])
    assert bool(torch.isfinite(av.all_states).all())


@pytest.mark.gpu
def test_masked_reset_keeps_the_rest_mixed_rates():
    """The same on a mixed handle whose drones run at several control rates: the drones outside the mask keep their base state
    bit for bit, the masked ones take the new one, and every drone keeps its setpoint and its aux state (throttles, surfaces,
    fuel, gimbal)"""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    n = 512 + 7
    kinds = [["quadx", "fixedwing", "rocket", "quadx"][(i + i // 32) % 4] for i in range(n)]
    rates = [[120, 240, 120, 60][i % 4] for i in range(n)]
    opts = [dict(drone_model="cf2x" if k == "quadx" else k, control_hz=r) if k != "rocket" else dict(control_hz=120) for k, r in zip(kinds, rates)]
    start, orn = _kind_setup("quadx", n, 6)[:2]
    av = BatchedAviary(start, orn, drone_type=kinds, drone_options=opts, seed=2, mixed_control_hz=True)
    ref = BatchedAviary(start, orn, drone_type=kinds, drone_options=opts, seed=2, mixed_control_hz=True)
    modes = [7 if k == "quadx" else 0 for k in kinds]
    sp = np.zeros((n, 7), dtype=np.float32)
    for i, k in enumerate(kinds):
        sp[i, : SP_DIM[k]] = {"quadx": [start[i, 0], start[i, 1], 0.0, start[i, 2] + 1.0], "fixedwing": [0.1, 0.0, 0.0, 0.7, 0, 0],
                              "rocket": [0.1, -0.1, 0.05, 1.0, 0.6, 0.1, -0.1]}[k]
    for a in (av, ref):
        a.set_mode(modes)
        a.set_all_setpoints(sp)
        a.step(30)
    mask = np.random.default_rng(3).random(n) < 0.5
    m = torch.as_tensor(mask, device="cuda")
    rng = np.random.default_rng(4)
    pos = start + rng.uniform(-2, 2, (n, 3))
    quat = rng.normal(size=(n, 4))
    quat /= np.linalg.norm(quat, axis=1, keepdims=True)
    lin, ang = rng.uniform(-5, 5, (n, 3)), rng.uniform(-1, 1, (n, 3))
    sp_before, aux_before = av.setpoints.clone(), [a.clone() for a in av.all_aux_states]
    av.set_base_state(pos, quat, lin, ang, mask=mask)
    p2, q2, l2, w2 = av.base_state()
    p1, q1, l1, w1 = ref.base_state()
    assert torch.equal(p2[~m], p1[~m]) and torch.equal(q2[~m], q1[~m]) and torch.equal(l2[~m], l1[~m]) and torch.equal(w2[~m], w1[~m])
    assert float((p2[m].cpu() - torch.as_tensor(pos)[m.cpu()]).abs().max()) < 1e-12
    assert float((w2[m].cpu() - torch.as_tensor(ang)[m.cpu()]).abs().max()) < 1e-5
    assert torch.equal(av.setpoints, sp_before)
    assert all(torch.equal(a, b) for a, b in zip(av.all_aux_states, aux_before))  # throttles, surfaces, fuel, gimbal kept


@pytest.mark.gpu
def test_mixed_handle_resets_equal_single_kind_handles():
    """Drone i of a mixed handle against drone i of single-kind handles over the same drones, same seed: the same masked
    set_base_state, then 60 steps, bit for bit"""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    n = 2048 + 33
    kinds = [["quadx", "fixedwing", "rocket", "quadx", "quadx", "rocket", "fixedwing"][(i + i // 32) % 7] for i in range(n)]
    ks = np.array(kinds)
    start, orn = _kind_setup("quadx", n, 10)[:2]
    sp = np.zeros((n, 7), dtype=np.float32)
    for i, k in enumerate(kinds):
        sp[i, : SP_DIM[k]] = {"quadx": [0.1, -0.1, 0.2, 0.4], "fixedwing": [0.2, -0.1, 0.1, 0.8, 0, 0], "rocket": [0.1, -0.1, 0.05, 1.0, 0.6, 0.1, -0.1]}[k]
    rng = np.random.default_rng(11)
    mask = rng.random(n) < 0.5
    pos = start.astype(np.float64) + rng.uniform(-3, 3, (n, 3))
    quat = rng.normal(size=(n, 4))
    quat /= np.linalg.norm(quat, axis=1, keepdims=True)
    lin, ang = rng.uniform(-8, 8, (n, 3)), rng.uniform(-2, 2, (n, 3))
    mixed = BatchedAviary(start, orn, drone_type=kinds, seed=4)
    uniform = {k: BatchedAviary(start, orn, drone_type=k, seed=4) for k in ("quadx", "fixedwing", "rocket")}
    avs = [mixed] + list(uniform.values())
    mixed.set_all_setpoints(sp)
    for k, u in uniform.items():
        u.set_all_setpoints(torch.as_tensor(sp[:, : u.setpoint_dim]))
    for a in avs:
        a.step(10)
        a.set_base_state(pos, quat, lin, ang, mask=mask)
    mixed.set_base_velocity(torch.as_tensor(lin[::-1].copy(), dtype=torch.float32), torch.as_tensor(ang[::-1].copy(), dtype=torch.float32))
    for u in uniform.values():
        u.set_base_velocity(torch.as_tensor(lin[::-1].copy(), dtype=torch.float32), torch.as_tensor(ang[::-1].copy(), dtype=torch.float32))
    for a in avs:
        a.step(60)
    torch.cuda.synchronize()
    s = mixed.all_states
    for k, u in uniform.items():
        m = torch.as_tensor(ks == k, device="cuda")
        assert torch.equal(s[m], u.all_states[m]), k
        assert torch.equal(mixed.precise_positions[m], u.precise_positions[m]), k
        assert torch.equal(mixed.contact_array[m], u.contact_array[m]), k
        for x, y in zip(mixed.base_state(), u.base_state()):
            assert torch.equal(x[m], y[m]), k


@pytest.mark.gpu
def test_python_checks_and_refusals():
    import torch

    from pyflyt_b200 import _lib
    from pyflyt_b200.core.aviary import BatchedAviary

    n = 8
    av = BatchedAviary(np.tile([[0.0, 0.0, 5.0]], (n, 1)), np.zeros((n, 3)))
    q = np.tile([[0.0, 0.0, 0.0, 1.0]], (n, 1))
    with pytest.raises(ValueError, match="come together"):
        av.set_base_state(pos=np.zeros((n, 3)))
    with pytest.raises(ValueError, match="shape"):
        av.set_base_state(pos=np.zeros((n, 2)), quat=q)
    with pytest.raises(ValueError, match="shape"):
        av.set_base_state(lin_vel=np.zeros((n + 1, 3)))
    with pytest.raises(ValueError, match="mask"):
        av.set_base_state(lin_vel=np.zeros((n, 3)), mask=np.ones(n - 1, dtype=bool))
    with pytest.raises(ValueError, match="unit"):
        av.set_base_state(pos=np.zeros((n, 3)), quat=q * (1.0 + 2e-6))
    av.set_base_state(pos=np.zeros((n, 3)), quat=q * (1.0 + 5e-7))  # within 1e-6
    # torch input on the device, and a state that all_states / contact_array / precise_positions reflect at once
    p = torch.arange(3 * n, dtype=torch.float64, device="cuda").reshape(n, 3) + 1.0
    av.set_base_state(pos=p, quat=torch.as_tensor(q), lin_vel=torch.ones(n, 3))
    assert torch.equal(av.precise_positions, p)
    assert float((av.all_states[:, 3] - p.float()).abs().max()) == 0.0
    assert float((av.all_states[:, 2] - 1.0).abs().max()) < 1e-6
    hover = PfbEnvConfig()
    hover.env_kind = 1
    hover.env_step_ratio, hover.max_steps, hover.flight_dome_size, hover.angle_representation = 3, 100, 3.0, 1
    env = BatchedAviary(np.tile([[0.0, 0.0, 1.0]], (n, 1)), np.zeros((n, 3)), env_config=hover)
    with pytest.raises(_lib.PfbError, match="only Aviary handles"):
        env.set_base_state(lin_vel=np.zeros((n, 3)))
    with pytest.raises(_lib.PfbError, match="only Aviary handles"):
        env.base_state()
    with pytest.raises(_lib.PfbError, match="Rocket-Landing"):
        env.set_base_velocity(torch.zeros(n, 3), torch.zeros(n, 3))
