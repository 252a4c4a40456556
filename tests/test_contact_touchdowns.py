"""Touchdowns through the Aviary with the floor contact response on, held to the fp64 oracle after EVERY Aviary step.

Every vehicle model meets the floor here: cf2x and primitive_drone dropped from any attitude (inverted and side-on included) with
idle motors, and flown into the floor in mode -1 under asymmetric pwm (impacts up to ~8 m/s, yaw spin, sliding); fixed-wing and
acrowing on their bellies and nose-in, on handles with different ``starting_velocity``; the rocket upright, tilted and side-on
at fuel 0, 0.5 and 1, thrown at the floor with ``set_base_velocity`` (tangential up to 10 m/s, spin up to 3 rad/s); and one
case per kind in an analytic wind.  Every spawn has its lowest candidate contact point at or above the floor (fp64, from the
shapes), so no drone starts inside it and is thrown out by the Baumgarte bias.

The state after each of the first STEPS Aviary steps is compared with the oracle's.  The bars come from the g++ build of the
kernel bodies (HostSimContactEngine) on 256 drones per case (test_hostsim_touchdowns_match_oracle, which runs on any machine);
the GPU test flies 8192 + 45 drones per case through BatchedAviary(contact_response=True) and holds the 99th percentile over
drones to GPU_MARGIN x those bars: every strike and tip-over amplifies the rounding differences between the builds, and in a batch
of thousands a few drones meet a tip-over edge whose side the rounding picks."""
import math

import numpy as np
import pytest

from engines import OracleEngine, build_model
from test_aviary_ground_contact import ContactCudaEngine, HostSimContactEngine, contact_config
from test_contact_solver import candidate_points

STEPS = 60  # 0.5 s at 120 Hz: drops from up to ~1.2 m land, strike and settle or slide inside the window
N_GPU = 8192 + 45
N_HOST = 256


def _rot_from_euler(orn):
    """the rotation PyBullet's getQuaternionFromEuler gives (roll x, pitch y, yaw z; R = Rz Ry Rx), fp64 -> (n, 3, 3)"""
    r, p, y = orn[:, 0], orn[:, 1], orn[:, 2]
    cr, sr, cp, sp, cy, sy = np.cos(r), np.sin(r), np.cos(p), np.sin(p), np.cos(y), np.sin(y)
    return np.stack([np.stack([cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr], -1),
                     np.stack([sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr], -1),
                     np.stack([-sp, cp * sr, cp * cr], -1)], 1)


def _lowest(model, orn):
    """altitude of the lowest candidate contact point below the base origin for each attitude (fp64, >= 0)"""
    P = candidate_points(model)
    return -np.einsum("kj,nij->nki", P, _rot_from_euler(orn))[:, :, 2].min(axis=1)


CASES = {
    # id: (kind, model, options, how the batch is spawned)
    "cf2x_drop": ("quadx", "cf2x", {}, "quad_drop"),
    "primitive_drone_drop": ("quadx", "primitive_drone", {}, "quad_drop"),
    "cf2x_pwm": ("quadx", "cf2x", {}, "quad_pwm"),
    "primitive_drone_pwm": ("quadx", "primitive_drone", {}, "quad_pwm"),
    "fixedwing_v0": ("fixedwing", "fixedwing", dict(starting_velocity=[0.0, 0.0, 0.0]), "wing"),
    "fixedwing_v8": ("fixedwing", "fixedwing", dict(starting_velocity=[8.0, 0.0, 0.0]), "wing"),
    "acrowing_v0": ("fixedwing", "acrowing", dict(starting_velocity=[0.0, 0.0, 0.0]), "wing"),
    "acrowing_v12": ("fixedwing", "acrowing", dict(starting_velocity=[12.0, 0.0, -1.0]), "wing"),
    "rocket_fuel0": ("rocket", "rocket", dict(starting_fuel_ratio=0.0), "rocket"),
    "rocket_fuel0.5": ("rocket", "rocket", dict(starting_fuel_ratio=0.5), "rocket"),
    "rocket_fuel1": ("rocket", "rocket", dict(starting_fuel_ratio=1.0), "rocket"),
}
WIND_CASES = {"quadx": "cf2x_pwm", "fixedwing": "fixedwing_v8", "rocket": "rocket_fuel0.5"}


def spawn(case, n, seed):
    """(model, start, orn, mode, setpoints, base velocity or None, noise) of a case; fp32-exact values"""
    kind, name, opts, how = CASES[case]
    model = build_model(kind, name, **opts)
    rng = np.random.default_rng(seed)
    f = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)  # noqa: E731
    vel = None
    if how.startswith("quad"):  # any attitude: uniform roll and yaw, pitch in [-pi/2, pi/2]
        orn = np.column_stack([rng.uniform(-math.pi, math.pi, n), rng.uniform(-math.pi / 2, math.pi / 2, n), rng.uniform(-math.pi, math.pi, n)])
        orn[: n // 8, 0] = math.pi + rng.normal(0, 0.05, n // 8)  # inverted
        orn[n // 8 : n // 4, 0] = math.pi / 2 + rng.normal(0, 0.05, n // 4 - n // 8)  # side-on
        clear = rng.uniform(0.005, 1.2, n)
        mode = -1
        sp = np.zeros((n, 4)) if how == "quad_drop" else rng.uniform(0.05, 0.9, (n, 4))  # asymmetric pwm: yaw spin and side force
    elif how == "wing":  # belly landings (small pitch and roll) and nose-in (pitched 0.3-0.8 rad down)
        nose = rng.uniform(0, 1, n) < 0.5
        orn = np.column_stack([rng.uniform(-0.3, 0.3, n), np.where(nose, rng.uniform(0.3, 0.8, n), rng.uniform(-0.2, 0.2, n)), rng.uniform(-math.pi, math.pi, n)])
        clear = rng.uniform(0.005, 1.0, n)
        mode = -1
        sp = np.zeros((n, 6))
        sp[:, :5] = rng.uniform(-0.3, 0.3, (n, 5))  # surfaces deflected, motor idle
    else:  # rocket: upright, tilted, side-on; thrown at the floor
        u = rng.uniform(0, 1, n)
        tilt = np.where(u < 0.3, 0.0, np.where(u < 0.7, rng.uniform(0.05, 0.5, n), math.pi / 2 + rng.normal(0, 0.05, n)))
        az = rng.uniform(-math.pi, math.pi, n)
        orn = np.column_stack([tilt * np.cos(az), tilt * np.sin(az), rng.uniform(-math.pi, math.pi, n)])
        clear = rng.uniform(0.005, 1.0, n)
        mode = 0
        sp = np.zeros((n, 7))  # not ignited
        ang = rng.uniform(0, 2 * math.pi, n)
        speed = rng.uniform(0, 10, n)
        lin = np.column_stack([speed * np.cos(ang), speed * np.sin(ang), -rng.uniform(0, 3, n)])
        vel = (f(lin), f(rng.uniform(-3, 3, (n, 3))))
    orn = f(orn)
    z = f(_lowest(model, orn) + clear + 1e-4)
    start = f(np.column_stack([rng.uniform(-5, 5, n), rng.uniform(-5, 5, n), z]))
    assert (start[:, 2] - _lowest(model, orn) > 0).all()  # nothing starts inside the floor
    loc = {"quadx": 4.0, "fixedwing": 1.0, "rocket": 1.0}[kind]
    noise = f(rng.normal(loc, 1.0, (STEPS * int(model.physics_hz // model.control_hz), n)))
    return model, start, orn, mode, f(sp), vel, noise


def _engine(make, case, n, seed, wind=None):
    model, start, orn, mode, sp, vel, noise = spawn(case, n, seed)
    e = make(model, contact_config(), n, start, orn)
    e.reset()
    e.set_mode(mode)
    e.set_setpoints(sp)
    if wind is not None:
        e.set_wind(wind)
    if vel is not None:
        e.set_base_velocity(*vel)
    return e, noise


def _errors(a, b):
    """per-drone |d| of two (n, 4, 3) states: rates, attitude (wrapped), velocity, position"""
    d_eul = np.abs((a[:, 1] - b[:, 1] + np.pi) % (2 * np.pi) - np.pi).max(axis=1)
    return dict(angvel=np.abs(a[:, 0] - b[:, 0]).max(axis=1), euler=d_eul, linvel=np.abs(a[:, 2] - b[:, 2]).max(axis=1), pos=np.abs(a[:, 3] - b[:, 3]).max(axis=1))


def fly(make, case, n, seed, wind=None):
    """steps `make`'s engine and the oracle side by side; per-drone worst error over the steps, the share of (drone, step) contact
    flags that differ and the share of drones that touched the floor"""
    e, noise = _engine(make, case, n, seed, wind)
    o, _ = _engine(OracleEngine, case, n, seed, wind)
    ups = e.ups
    worst = {k: np.zeros(n) for k in ("angvel", "euler", "linvel", "pos")}
    flag_diff, touched = 0, np.zeros(n, bool)
    for t in range(STEPS):
        nz = noise[t * ups : (t + 1) * ups]
        e.aviary_step(nz)
        o.aviary_step(nz)
        for k, v in _errors(e.state(), o.state()).items():
            worst[k] = np.maximum(worst[k], v)
        ce, co = e.contact().astype(bool), o.contact().astype(bool)
        flag_diff += int((ce != co).sum())
        touched |= co
    return worst, flag_diff / (n * STEPS), float(touched.mean())


# The g++ kernel bodies against the oracle, 256 drones per case (test_hostsim_touchdowns_match_oracle): the 99th percentile over
# drones of each drone's worst error over the steps, and the worst drone; each x5, rounded up and never below the free-flight
# bars of the GPU parity tests (pos 5e-4 m, euler 1e-3 rad, rates and velocities 1e-2).  The worst drones of the mode -1 cases
# tumble under full asymmetric thrust after a strike, where the rounding decides which way they go: cf2x_pwm's worst (drone 237
# of the 256, seed 3) stays within 3e-6 of the oracle until it strikes the floor spinning at ~240 rad/s, then is 2.4e-4 and, one
# step later, 1.1 rad/s apart, with no contact flag differing; hence that case's loose worst-drone bars.
#   hostsim seen, p99 / worst:  pos              euler            angvel           linvel
#   cf2x_drop              1.1e-05/8.6e-05  5.1e-04/5.5e-03  5.1e-02/4.3e-01  1.2e-03/2.0e-02
#   primitive_drone_drop   6.4e-07/7.1e-07  1.0e-05/2.2e-05  9.4e-05/1.4e-04  1.3e-05/1.5e-05
#   cf2x_pwm               1.1e-05/4.0e-03  5.8e-05/1.9e-01  5.2e-03/3.9e+01  2.5e-04/1.9e+00
#   primitive_drone_pwm    9.2e-05/1.1e-03  2.5e-03/1.1e-02  3.2e-02/2.7e+00  6.6e-03/2.3e-01
#   fixedwing_v0           6.5e-07/2.7e-06  2.3e-06/1.3e-05  6.7e-05/2.2e-02  2.4e-05/2.6e-03
#   fixedwing_v8           2.5e-05/6.1e-05  2.9e-05/1.4e-04  1.2e-03/6.3e-02  2.3e-04/3.3e-02
#   acrowing_v0            3.4e-07/7.1e-06  6.2e-07/5.0e-05  1.7e-05/1.0e-03  5.0e-06/3.4e-04
#   acrowing_v12           1.2e-05/3.4e-05  2.8e-06/4.8e-06  1.4e-04/1.6e-04  8.3e-05/1.5e-04
#   rocket_fuel0           3.5e-05/6.2e-05  1.6e-04/3.7e-04  7.8e-03/1.0e-01  1.4e-03/1.2e-02
#   rocket_fuel0.5         1.0e-05/1.3e-04  6.3e-05/1.3e-04  2.4e-03/2.9e-02  3.4e-04/4.2e-02
#   rocket_fuel1           3.0e-05/1.1e-04  2.2e-04/6.6e-04  3.3e-02/7.1e-02  5.9e-03/2.1e-02
FREE = dict(pos=5e-4, euler=1e-3, angvel=1e-2, linvel=1e-2)
BARS = {  # case: (p99 bars, worst-drone bars)
    "cf2x_drop": (dict(pos=5e-4, euler=3e-3, angvel=0.3, linvel=1e-2), dict(pos=5e-4, euler=3e-2, angvel=3.0, linvel=0.2)),
    "primitive_drone_drop": (FREE, FREE),
    "cf2x_pwm": (dict(pos=5e-4, euler=1e-3, angvel=3e-2, linvel=1e-2), dict(pos=3e-2, euler=1.0, angvel=200.0, linvel=10.0)),
    "primitive_drone_pwm": (dict(pos=5e-4, euler=2e-2, angvel=0.2, linvel=4e-2), dict(pos=6e-3, euler=6e-2, angvel=20.0, linvel=2.0)),
    "fixedwing_v0": (FREE, dict(pos=5e-4, euler=1e-3, angvel=0.2, linvel=2e-2)),
    "fixedwing_v8": (FREE, dict(pos=5e-4, euler=1e-3, angvel=0.4, linvel=0.2)),
    "acrowing_v0": (FREE, FREE),
    "acrowing_v12": (FREE, FREE),
    "rocket_fuel0": (dict(pos=5e-4, euler=1e-3, angvel=4e-2, linvel=1e-2), dict(pos=5e-4, euler=2e-3, angvel=0.5, linvel=6e-2)),
    "rocket_fuel0.5": (dict(pos=5e-4, euler=1e-3, angvel=2e-2, linvel=1e-2), dict(pos=7e-4, euler=1e-3, angvel=0.2, linvel=0.3)),
    "rocket_fuel1": (dict(pos=5e-4, euler=2e-3, angvel=0.2, linvel=3e-2), dict(pos=6e-4, euler=4e-3, angvel=0.4, linvel=0.2)),
}
FLAG_BAR = 2e-3  # share of (drone, step) contact flags that may differ (host: none; H100: 1e-5 at most)
# The device build differs from the g++ one by the fast-math helpers (fast_rcp, fast_rsqrt, __sincosf: up to ~1.5 ulp,
# tests/test_device_math.py) and by nvcc's FMA contraction, and every strike amplifies those differences as it amplifies fp32
# rounding.  The GPU's 99th percentile is held to GPU_MARGIN x the host's bars.  Measured on an NVIDIA H100 80GB HBM3 (700 W
# power limit), 8237 drones: the p99 of the mode -1 QuadX cases and of the rockets comes to 0.3-0.7 of those bars (rocket at fuel
# 0: angvel 8.6e-2, linvel 3.5e-2), the rest below 0.1.  The worst drone of thousands is a tumble whose direction the rounding
# picks (cf2x mode -1: 160 rad/s apart), so the GPU test holds it to being finite only.
GPU_MARGIN = 5.0


def _check(case, worst, flag_diff, touched, margin=None):
    """margin None: the host bars (p99 and worst drone); else the p99 against margin x the host's p99 bars"""
    assert touched > 0.55, (case, touched)
    assert flag_diff < FLAG_BAR, (case, flag_diff)
    p99, top = BARS[case]
    for k in p99:
        assert np.isfinite(worst[k]).all(), (case, k)
        seen = float(np.quantile(worst[k], 0.99))
        assert seen < (margin or 1.0) * p99[k], (case, k, "p99", seen, (margin or 1.0) * p99[k])
        if margin is None:
            assert float(worst[k].max()) < top[k], (case, k, "worst", float(worst[k].max()), top[k])


@pytest.mark.parametrize("case", list(CASES))
def test_hostsim_touchdowns_match_oracle(case):
    """the evidence behind BARS: the CONTACT = true kernel bodies built by g++ against the oracle, after every step"""
    worst, flag_diff, touched = fly(HostSimContactEngine, case, N_HOST, 3)
    _check(case, worst, flag_diff, touched)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_cuda_touchdowns_match_oracle(case):
    worst, flag_diff, touched = fly(ContactCudaEngine, case, N_GPU, 5)
    print(f"[touchdowns {case}] {N_GPU} drones x {STEPS} steps: p99 / max " + ", ".join(f"{k} {np.quantile(v, 0.99):.2e} / {v.max():.2e}" for k, v in worst.items())
          + f"; contact flags differing {flag_diff:.1e}; touched {touched:.2f}")
    _check(case, worst, flag_diff, touched, GPU_MARGIN)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(WIND_CASES))
def test_cuda_touchdowns_in_wind_match_oracle(kind):
    """one case per kind in a power-law wind with a vertical component"""
    from pyflyt_b200.core.wind import AnalyticWind

    case = WIND_CASES[kind]
    wind = AnalyticWind("power", base=(4.0, -2.0, 0.3), z_ref=10.0, alpha=1.0 / 7.0)
    worst, flag_diff, touched = fly(ContactCudaEngine, case, N_GPU, 6, wind)
    print(f"[touchdowns {case} wind] p99 / max " + ", ".join(f"{k} {np.quantile(v, 0.99):.2e} / {v.max():.2e}" for k, v in worst.items()))
    _check(case, worst, flag_diff, touched, GPU_MARGIN)
