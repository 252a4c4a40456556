"""Floor contact RESPONSE on Aviary handles: ``BatchedAviary(contact_response=True)`` for QuadX, fixed-wing and rocket drones.

CPU: the ground_* fixtures (tools/gen_golden.py, group ``ground``: the unmodified reference Aviary on oracle/fakebullet with the
engine's contact response on) end at rest on the floor; the C oracle replays them at fp64 round-off with a kind-NONE config
whose ``contact_response`` is 1; the g++ build of the kernel bodies with CONTACT = true (tests/hostsim/hostsim_contact.cpp)
replays them within fp32 bars, and flies the drops the GPU tests fly against the oracle.
GPU: the CUDA Aviary replays every fixture within the same bars; flight far above the floor is bit-identical with the response on
and off; full-size batches dropped onto the floor come to rest and match the oracle; mixed-model and per-drone-mode handles
equal the matching uniform handles bit for bit; a kind-NONE config with the response off is the handle ``env = NULL`` builds."""
import ctypes as C
import glob
import os
import subprocess
import tempfile

import numpy as np
import pytest

from engines import GOLDEN, ROOT, CudaEngine, HostSimEngine, OracleEngine, _p, build_model, load_golden, replay_aviary, replay_vehicle
from pyflyt_b200.models import PfbEnvConfig

FIXTURES = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, "ground_*.npz")))
REST_STEPS = 120  # the last second of every fixture (control_hz 120)


def contact_config(on=True):
    """an Aviary-handle config (env kind NONE): pfb_create and the oracle read its contact_response"""
    e = PfbEnvConfig()
    e.contact_response = int(bool(on))
    return e


def replay_ground(make_engine, g, every=1):
    """replay_aviary / replay_vehicle with the contact response on: every engine is built from contact_config()"""
    make = lambda model, env, n, sp, so: make_engine(model, contact_config(), n, sp, so)  # noqa: E731
    return replay_aviary(make, g, every) if str(g["kind"]) == "quadx_aviary" else replay_vehicle(make, g, every)


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_fixtures_present():
    names = set(FIXTURES)
    for n in ("ground_cf2x_takeoff_landing", "ground_primitive_tilted_drop", "ground_cf2x_sliding_touchdown", "ground_fixedwing_belly_landing",
              "ground_rocket_rest"):
        assert n in names, n


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_ends_at_rest(name):
    """the reference's drone ends resting on the floor: over the last second it barely moves and its contact flag is up.  The
    bars leave room for the chatter of a resting body: the solver's impulses are not accumulated across iterations, so a
    drone on its primitives keeps rocking at mm/s (primitive_drone on its thin propeller cylinders: ~0.2 rad/s)"""
    g = load_golden(name)
    st, c = g["state"], g["contact"]
    last = st[-REST_STEPS:]
    assert bool(c[-1]) and c[-REST_STEPS:].all(), name
    assert np.abs(last[:, 2]).max() < 0.05, (name, "speed", np.abs(last[:, 2]).max())
    assert np.abs(last[:, 0]).max() < 0.3, (name, "rate", np.abs(last[:, 0]).max())
    assert np.ptp(last[:, 3, 2]) < 1e-3, (name, "height spread", np.ptp(last[:, 3, 2]))
    assert c[: len(c) // 2].any(), name  # the floor is reached well before the end


def test_fixtures_cover_takeoff_and_slide():
    """the take-off fixture leaves the floor and comes back; the sliding touchdown and the belly landing reach the floor with
    a horizontal velocity that friction takes away"""
    g = load_golden("ground_cf2x_takeoff_landing")
    z, c = g["state"][:, 3, 2], g["contact"]
    assert c[0] and z.max() > 0.5 and not c[np.argmax(z)] and c[-1]
    for name in ("ground_cf2x_sliding_touchdown", "ground_fixedwing_belly_landing"):
        g = load_golden(name)
        c, v_world = g["contact"], g["raw"][:, 7:10]  # raw = position, quaternion, world velocity, world rates
        first = int(np.argmax(c))
        assert np.linalg.norm(v_world[first - 1, :2]) > 1.0, (name, v_world[first - 1])
        assert np.linalg.norm(v_world[-1, :2]) < 0.05, (name, v_world[-1])


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_replays_ground_fixture(name):
    """fp64 against fp64 (the bars of test_oracle_golden.py): the oracle's solve_contacts is the engine's _solve_contacts.  The
    rocket takes the looser bar: resting on its legs it chatters (see test_fixture_ends_at_rest), and every impulse amplifies
    the operation-order rounding (1.4e-9 m, 1.9e-7 rad/s seen)"""
    err = replay_ground(OracleEngine, load_golden(name))
    assert err["contact_mismatch"] == 0, err
    tol = 1e-6 if "rocket" in name else 1e-9
    for k in ("pos", "euler", "angvel", "linvel", "aux"):
        assert err[k] < tol, (name, k, err[k])


_HSC = None


def hostsim_contact_lib():
    global _HSC
    if _HSC is None:
        out = os.path.join(tempfile.mkdtemp(prefix="pfb_hostsim_contact_"), "libpfb_hostsim_contact.so")
        src = os.path.join(ROOT, "tests", "hostsim", "hostsim_contact.cpp")
        subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-mfma", "-ffp-contract=fast", "-o", out, src], check=True, capture_output=True)
        _HSC = C.CDLL(out)
        _HSC.hs_last_error.restype = C.c_char_p
    return _HSC


class HostSimContactEngine(HostSimEngine):
    """HostSimEngine whose Aviary steps are the CONTACT = true instantiations (tests/hostsim/hostsim_contact.cpp)"""

    name = "hostsim_contact"

    def __init__(self, model, env=None, n=1, start_pos=None, start_orn=None):
        super().__init__(model, env, n, start_pos, start_orn)
        self.L = hostsim_contact_lib()

    def aviary_step(self, noise, n_steps=1):
        nz = np.ascontiguousarray(noise, dtype=np.float32)
        assert nz.shape == (n_steps * self.ups, self.n)
        f, i32, n = C.c_float, C.c_int32, C.c_int64(self.n)
        if self.rk:
            self._chk(self.L.hs_rk_aviary_step_contact(C.byref(self.model), _p(self.st, f), _p(self.ist, i32), _p(self.sp, f), _p(nz, f), n_steps, n))
        elif self.fw:  # the kernels take the one-basic-block substep for a complete model in still air
            full = int(int(self.model.n_surfaces) == 5)
            self._chk(self.L.hs_fw_aviary_step_contact(C.byref(self.model), self.mode, full, _p(self.st, f), _p(self.ist, i32), _p(self.sp, f), _p(nz, f),
                                                       n_steps, n))
        else:
            self._chk(self.L.hs_aviary_step_contact(C.byref(self.model), self.mode, _p(self.st, f), _p(self.ist, i32), _p(self.sp, f), _p(nz, f), n_steps, n))


# fp32 bars against the reference, per fixture.  What the host build of the kernel body shows (test_hostsim_contact_replays_
# ground_fixture), x5 and rounded up, and never below the free-flight bars of the GPU parity tests (pos 5e-4 m, euler 1e-3 rad,
# rates and velocities 1e-2).  Flight before the first touchdown stays at the free-flight level; each touchdown and tip-over is a
# discontinuous function of the pose that amplifies the fp32 rounding, and a resting drone chatters (test_fixture_ends_at_rest)
# at a phase the rounding decides: hence the rate bars of the tilted drop and the rocket.
#   hostsim seen:                 pos      euler    angvel   linvel
#   ground_cf2x_sliding_touchdown 5.9e-7   6.6e-6   3.6e-4   1.1e-5
#   ground_cf2x_takeoff_landing   5.3e-8   2.4e-8   7.4e-7   2.9e-7
#   ground_fixedwing_belly_landing 3.7e-3  4.2e-5   6.0e-3   2.2e-3
#   ground_primitive_tilted_drop  5.4e-4   7.1e-3   0.62     0.10
#   ground_rocket_rest            6.6e-3   7.0e-3   0.12     0.072
BARS = {
    "ground_cf2x_takeoff_landing": dict(pos=5e-4, euler=1e-3, angvel=1e-2, linvel=1e-2),
    "ground_cf2x_sliding_touchdown": dict(pos=5e-4, euler=1e-3, angvel=1e-2, linvel=1e-2),
    "ground_primitive_tilted_drop": dict(pos=3e-3, euler=4e-2, angvel=3.0, linvel=0.5),
    "ground_fixedwing_belly_landing": dict(pos=2e-2, euler=1e-3, angvel=3e-2, linvel=1.2e-2),
    "ground_rocket_rest": dict(pos=4e-2, euler=4e-2, angvel=0.6, linvel=0.4),
}


def _fp32_bars(name, err):
    assert err["contact_mismatch"] == 0, (name, err["contact_mismatch"])
    for k, bar in BARS[name].items():
        assert err[k] < bar, (name, k, err[k], bar)


@pytest.mark.parametrize("name", FIXTURES)
def test_hostsim_contact_replays_ground_fixture(name):
    """the kernel body with CONTACT = true, compiled for the host, against the reference (no GPU needed)"""
    _fp32_bars(name, replay_ground(HostSimContactEngine, load_golden(name)))


def _drop_batch(kind, n, seed):
    """start poses of a drop: the lowest corner 0.05-2 m above the floor, tilt <= 0.5 rad, any yaw (fp32-exact values).  A spawn
    with a corner below the floor would be pushed out by the Baumgarte bias at up to 0.2 * depth / dt (tens of m/s for a
    fixed-wing's wing tip), so the clearance counts the tilt: the reach of the airframe (cf2x 0.07 m, fixed-wing 1.2 m) times
    sin(tilt) plus its half-thickness"""
    rng = np.random.default_rng(seed)
    f = lambda a: a.astype(np.float32).astype(np.float64)  # noqa: E731
    reach, half = {"quadx": (0.07, 0.01), "fixedwing": (1.2, 0.1)}[kind]
    tilt, az = 0.5 * np.sqrt(rng.uniform(0, 1, n)), rng.uniform(-np.pi, np.pi, n)
    z = half + reach * np.sin(tilt) + rng.uniform(0.05, 2.0, n)
    start = f(np.column_stack([rng.uniform(-5, 5, n), rng.uniform(-5, 5, n), z]))
    orn = f(np.column_stack([tilt * np.cos(az), tilt * np.sin(az), rng.uniform(-np.pi, np.pi, n)]))
    return start, orn


DROP_STEPS = 300  # 2.5 s at 120 Hz
DROP_MODELS = {"quadx": ("quadx", "cf2x", {}), "fixedwing": ("fixedwing", "fixedwing", dict(starting_velocity=np.zeros(3)))}
# a drop's final pose against the oracle's: each strike and tip-over amplifies the fp32 rounding, so the bars come from the host
# build of the kernel body (test_hostsim_drop_matches_oracle: cf2x 1.3e-4 m / 6.4e-3 rad, fixed-wing 8.5e-4 m / 6.8e-3 rad over
# 256 drops) with a margin of ~5x
DROP_BARS = {"quadx": dict(pos=1e-3, euler=4e-2), "fixedwing": dict(pos=5e-3, euler=4e-2)}
# at rest after the drop: speed (m/s) and rate (rad/s) bars for 99 % of the drones, and for every drone.  The cf2x lies still
# (host build, 256 drops: 1e-5 m/s, 1.4e-4 rad/s; an H100 at 65 536 drones: 0.027 m/s at most, a late tip-over); the fixed-wing
# rocks on its boxes (the chatter of test_fixture_ends_at_rest; host build at 16 384 drones: 0.031 / 0.30 for 99 %, 0.049 m/s /
# 0.49 rad/s at most)
REST_BARS = {"quadx": dict(p99=(0.01, 0.05), all=(0.1, 1.0)), "fixedwing": dict(p99=(0.1, 1.0), all=(0.3, 2.0))}


def _drop_engines(kind, make, start, orn):
    dt, name, opts = DROP_MODELS[kind]
    model = build_model(dt, name, **opts)
    e = make(model, contact_config(), len(start), start, orn)
    e.reset()
    e.set_mode(-1)
    e.set_setpoints(np.zeros((len(start), 6 if kind == "fixedwing" else 4)))
    return model, e


def _drop_compare(kind, a, b):
    """max over drones of |pos| and |euler| differences of two (n, 4, 3) states"""
    d_eul = np.abs((a[:, 1] - b[:, 1] + np.pi) % (2 * np.pi) - np.pi)
    return dict(pos=float(np.abs(a[:, 3] - b[:, 3]).max()), euler=float(d_eul.max()))


@pytest.mark.parametrize("kind", ["quadx", "fixedwing"])
def test_hostsim_drop_matches_oracle(kind):
    """256 drops of the GPU drop test, flown by the host build of the kernel body and by the oracle: the evidence behind
    DROP_BARS.  Idle motors (mode -1, zero setpoint) make the noise draws irrelevant: the throttle stays exactly 0."""
    n = 256
    start, orn = _drop_batch(kind, n, 7)
    _, hs = _drop_engines(kind, HostSimContactEngine, start, orn)
    _, orc = _drop_engines(kind, OracleEngine, start, orn)
    noise = np.full((DROP_STEPS * hs.ups, n), 4.0 if kind == "quadx" else 1.0)
    hs.aviary_step(noise, DROP_STEPS)
    orc.aviary_step(noise, DROP_STEPS)
    err = _drop_compare(kind, hs.state(), orc.state())
    for k, bar in DROP_BARS[kind].items():
        assert err[k] < bar, (kind, k, err[k], bar)
    assert orc.contact().all()


# ------------------------------------------------------------------------------------------------------------------ GPU
class ContactCudaEngine(CudaEngine):
    """CudaEngine over BatchedAviary(..., contact_response=True): the Python switch, for every vehicle kind"""

    def __init__(self, model, env, n, start_pos, start_orn):
        import torch

        from pyflyt_b200.core.aviary import BatchedAviary

        kind = {0: "quadx", 1: "fixedwing", 2: "rocket"}[int(model.kind)]
        if kind == "rocket":
            opts = dict(drone_model="rocket", starting_fuel_ratio=float(model.starting_fuel_ratio))
        elif kind == "fixedwing":
            opts = dict(drone_model="acrowing" if abs(model.com[0] + 0.39574468) < 1e-5 else "fixedwing", starting_velocity=list(model.starting_velocity))
        else:
            opts = dict(drone_model="primitive_drone" if abs(model.mass - 1.0) < 1e-12 else "cf2x")
        self.torch = torch
        self.n = n
        sp = np.ascontiguousarray(np.broadcast_to(start_pos, (n, 3)), dtype=np.float32)
        so = np.ascontiguousarray(np.broadcast_to(start_orn, (n, 3)), dtype=np.float32)
        self.av = BatchedAviary(sp, so, drone_type=kind, drone_options=opts, contact_response=True)
        self.aux_dim, self.ups, self.obs_dim = self.av.aux_dim, self.av.updates_per_step, self.av.obs_dim


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_cuda_replays_ground_fixture(name):
    """the CUDA Aviary with contact_response=True, injected noise, within the hostsim-derived bars"""
    _fp32_bars(name, replay_ground(ContactCudaEngine, load_golden(name)))


@pytest.mark.gpu
def test_config_route_equals_kwarg_route():
    """BatchedAviary(env_config=<kind NONE, contact_response 1>) is the handle contact_response=True builds"""
    from engines import make_cuda_engine

    g = load_golden("ground_primitive_tilted_drop")
    a = replay_ground(make_cuda_engine, g)
    b = replay_ground(ContactCudaEngine, g)
    for k in ("pos", "euler", "angvel", "linvel", "aux", "contact_mismatch"):
        assert a[k] == b[k], k


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["quadx", "fixedwing", "rocket"])
def test_kind_none_config_is_the_null_config(kind):
    """pfb_create reads ONLY contact_response from a kind-NONE config: with it 0, and every other field set to values an env
    would use, the handle has the dimensions and steps the state of the handle built with env = NULL, bit for bit"""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    e = PfbEnvConfig()
    e.flight_mode, e.env_step_ratio, e.max_steps, e.angle_representation, e.sparse_reward = 7, 3, 100, 0, 1
    e.warmup_steps, e.flight_dome_size, e.goal_reach_distance, e.num_targets = 10, 2.0, 1.0, 4
    e.ceiling, e.max_displacement, e.randomize_drop, e.accelerate_drop, e.team_size = 10.0, 5.0, 1, 1, 2
    e.contact_response = 0
    n = 1000
    rng = np.random.default_rng(3)
    z0 = {"quadx": 0.5, "fixedwing": 1.0, "rocket": 3.0}[kind]
    start = np.column_stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), z0 + rng.uniform(0, 1, n)]).astype(np.float32)
    orn = rng.uniform(-0.3, 0.3, (n, 3)).astype(np.float32)
    a = BatchedAviary(start, orn, drone_type=kind, seed=5)
    b = BatchedAviary(start, orn, drone_type=kind, seed=5, env_config=e)
    for k in ("obs_dim", "setpoint_dim", "aux_dim", "state_rows", "tiled"):
        assert getattr(a, k) == getattr(b, k), k
    sp = torch.as_tensor(rng.uniform(0, 0.6, (n, a.setpoint_dim)).astype(np.float32), device=a.device)
    for av in (a, b):
        av.set_mode(0)
        av.set_all_setpoints(sp)
        av.step(40)
    assert torch.equal(a.state_tensor, b.state_tensor) and torch.equal(a.istate_tensor, b.istate_tensor)
    assert a.contact_array.any()  # the flag fires (and nothing pushes back) on both
    assert torch.equal(a.all_states, b.all_states) and torch.equal(a.contact_array, b.contact_array)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,n", [("quadx", 65536), ("fixedwing", 16384)])
def test_free_flight_bit_identical(kind, n):
    """drones that never come within contact_zmax of the floor step bit for bit the same with the response on and off"""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    rng = np.random.default_rng(11)
    z = (3.0, 10.0) if kind == "quadx" else (60.0, 100.0)
    start = np.column_stack([rng.uniform(-5, 5, n), rng.uniform(-5, 5, n), rng.uniform(*z, n)]).astype(np.float32)
    orn = rng.uniform(-0.3, 0.3, (n, 3)).astype(np.float32)
    on, off = (BatchedAviary(start, orn, drone_type=kind, seed=9, contact_response=c) for c in (True, False))
    mode = 7 if kind == "quadx" else 0
    for av in (on, off):
        av.set_mode(mode)
    for _ in range(3):
        if kind == "quadx":
            sp = np.column_stack([start[:, :2] + rng.uniform(-1, 1, (n, 2)), rng.uniform(-1, 1, n), start[:, 2] + rng.uniform(-1, 1, n)])
        else:
            sp = np.column_stack([rng.uniform(-0.5, 0.5, (n, 3)), rng.uniform(0.3, 1.0, n), np.zeros((n, 2))])  # mode 0 reads 4 of 6
        sp = torch.as_tensor(sp.astype(np.float32), device=on.device)
        for av in (on, off):
            av.set_all_setpoints(sp)
            av.step(40)
        assert torch.equal(on.state_tensor, off.state_tensor) and torch.equal(on.istate_tensor, off.istate_tensor)
    assert not on.contact_array.any()
    assert float(on.all_states[:, 3, 2].min()) > 1.0


@pytest.mark.gpu
@pytest.mark.parametrize("kind,n", [("quadx", 65536), ("fixedwing", 16384)])
def test_full_batch_drop_comes_to_rest(kind, n):
    """a full batch dropped from 0.05-2 m with tilts up to 0.5 rad, motors idle: after 2.5 s every drone rests on the floor
    (finite, no cf2x deeper than the slop + 5 mm margin, no fixed-wing base below the floor, barely moving, contact flag up);
    256 random drones match the oracle"""
    import torch

    start, orn = _drop_batch(kind, n, 13)
    _, cud = _drop_engines(kind, ContactCudaEngine, start, orn)
    cud.av.step(DROP_STEPS - 2)
    prev = cud.av.all_states.clone()
    cud.av.step(2)
    st = cud.av.all_states
    assert torch.isfinite(st).all()
    v = st[:, 2].abs().amax(dim=1).cpu().numpy()
    w = st[:, 0].abs().amax(dim=1).cpu().numpy()
    dv = (st[:, 2] - prev[:, 2]).abs().amax(dim=1).cpu().numpy()
    seen = dict(v99=np.quantile(v, 0.99), v=v.max(), w99=np.quantile(w, 0.99), w=w.max(), dv=dv.max())
    (v99, w99), (v_all, w_all) = REST_BARS[kind]["p99"], REST_BARS[kind]["all"]
    assert seen["v99"] < v99 and seen["w99"] < w99, seen
    assert seen["v"] < v_all and seen["w"] < w_all and seen["dv"] < v_all, seen
    assert bool(cud.av.contact_array.all())
    pos = cud.av.precise_positions.cpu().numpy()
    assert np.isfinite(pos).all()
    z_min = 0.01 - 0.001 - 0.005 if kind == "quadx" else 0.0  # cf2x: its box's half-height - slop - margin
    assert pos[:, 2].min() > z_min, pos[:, 2].min()
    ids = np.sort(np.random.default_rng(17).choice(n, 256, replace=False))
    _, orc = _drop_engines(kind, OracleEngine, start[ids], orn[ids])
    orc.aviary_step(np.full((DROP_STEPS * orc.ups, 256), 4.0 if kind == "quadx" else 1.0), DROP_STEPS)
    err = _drop_compare(kind, cud.state()[ids], orc.state())
    for k, bar in DROP_BARS[kind].items():
        assert err[k] < bar, (kind, k, err[k], bar)


@pytest.mark.gpu
def test_mixed_models_equal_uniform_handles_with_contact():
    """a model set (cf2x / primitive_drone alternating, test_mixed_models.py's layout) with the response on: drone i equals
    drone i of a uniform handle of its model, bit for bit, through take-offs, drops and landings"""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    n = 4096
    rng = np.random.default_rng(23)
    start = np.column_stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(0.03, 1.0, n)]).astype(np.float32)
    orn = np.column_stack([rng.uniform(-0.3, 0.3, (n, 2)), rng.uniform(-3, 3, n)]).astype(np.float32)
    opts = [dict(drone_model="cf2x" if i % 2 == 0 else "primitive_drone") for i in range(n)]
    mixed = BatchedAviary(start, orn, drone_options=opts, seed=4, contact_response=True)
    uniform = [BatchedAviary(start, orn, drone_options=dict(drone_model=m), seed=4, contact_response=True) for m in ("cf2x", "primitive_drone")]
    assert len(mixed.models) == 2
    idx = torch.as_tensor(np.arange(n) % 2, device=mixed.device)
    for av in [mixed] + uniform:
        av.set_mode(6)
    touched = torch.zeros(n, dtype=torch.bool, device=mixed.device)
    for chunk in range(6):
        sp = np.column_stack([rng.uniform(-0.3, 0.3, (n, 3)), rng.uniform(-0.8, 0.6, n)]).astype(np.float32)
        sp = torch.as_tensor(sp, device=mixed.device)
        for av in [mixed] + uniform:
            av.set_all_setpoints(sp)
            av.step(30)
        touched |= mixed.contact_array
        for j, U in enumerate(uniform):
            sel = idx == j
            assert torch.equal(mixed.all_states[sel], U.all_states[sel]), (chunk, j)
            assert torch.equal(mixed.all_aux_states[sel], U.all_aux_states[sel]), (chunk, j)
            assert torch.equal(mixed.contact_array[sel], U.contact_array[sel]), (chunk, j)
    assert float(touched.float().mean()) > 0.1  # 0.28 seen


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["quadx", "fixedwing"])
def test_per_drone_modes_equal_uniform_handles_with_contact(kind):
    """one mode per drone (test_mixed_modes.py's interleaved layout) with the response on, drones starting on and just above the
    floor: drone i equals drone i of a uniform handle of its mode, bit for bit (state words, observations, contact)"""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary
    from test_mixed_modes import _assert_bit_identical, _layout, _setpoints

    n = 8192 if kind == "quadx" else 4096
    rng = np.random.default_rng(29)
    z = (0.01, 1.0) if kind == "quadx" else (0.05, 2.0)
    start = np.column_stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(*z, n)]).astype(np.float32)
    orn = np.column_stack([rng.uniform(-0.3, 0.3, (n, 2)), rng.uniform(-3, 3, n)]).astype(np.float32)
    opts = dict(drone_model=kind if kind == "fixedwing" else "cf2x")
    modes = _layout("interleaved", n, rng) if kind == "quadx" else -1 + np.arange(n) % 2
    mode_list = list(range(-1, 8)) if kind == "quadx" else [-1, 0]
    mixed = BatchedAviary(start, orn, drone_type=kind, drone_options=opts, seed=8, contact_response=True)
    uniform = [BatchedAviary(start, orn, drone_type=kind, drone_options=opts, seed=8, contact_response=True) for _ in mode_list]
    mixed.set_mode(modes.tolist())
    for m, U in zip(mode_list, uniform):
        U.set_mode(m)
    dev = mixed.device
    touched = torch.zeros(n, dtype=torch.bool, device=dev)
    for chunk in (1, 24, 40, 60):
        if kind == "quadx":
            sps = [_setpoints(m, start, rng).astype(np.float32) for m in mode_list]
        else:
            sps = [np.column_stack([rng.uniform(-0.5, 0.5, (n, 5)), rng.uniform(0.0, 0.3, n)]).astype(np.float32) for _ in mode_list]
        mixed_sp = np.stack(sps)[modes - mode_list[0], np.arange(n)]
        mixed.set_all_setpoints(torch.as_tensor(mixed_sp, device=dev))
        for m, U in enumerate(uniform):
            U.set_all_setpoints(torch.as_tensor(sps[m], device=dev))
        for a in [mixed] + uniform:
            a.step(chunk)
        touched |= mixed.contact_array
        if kind == "quadx":
            _assert_bit_identical(mixed, uniform, modes, chunk)
        else:
            idx = torch.as_tensor(modes, device=dev)
            for m, U in zip(mode_list, uniform):
                sel = idx == m
                assert torch.equal(mixed.all_states[sel], U.all_states[sel]), (chunk, m)
                assert torch.equal(mixed.contact_array[sel], U.contact_array[sel]), (chunk, m)
                for r in range(mixed.state_rows):
                    assert torch.equal(mixed.state_tensor[r][sel], U.state_tensor[r][sel]), (chunk, m, r)
    assert float(touched.float().mean()) > 0.1  # cf2x: 0.19 seen
