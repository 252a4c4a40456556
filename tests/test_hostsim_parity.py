"""CPU-side check of the KERNEL BODY (pyflyt_b200/csrc/pfb_quadx.cuh compiled with g++ by
tests/hostsim) against the golden vectors: same flight-mode logic, same flags, fp32/fp64 policy within
the trajectory tolerance.  This is a test harness; the product path is CUDA-only."""
import numpy as np
import pytest

from engines import HostSimEngine, OracleEngine, build_model, load_golden, replay_aviary, replay_hover

POS_TOL = 1e-3  # north_star: |dpos| < 1e-3 m over 1000 env-steps


def test_long_mode0_trajectory_within_tolerance():
    err = replay_aviary(HostSimEngine, load_golden("quadx_mode0_long"), every=30)
    assert err["pos"] < POS_TOL, err["pos"]
    assert err["contact_mismatch"] == 0


@pytest.mark.parametrize("mode", [-1, 0, 1, 4, 5, 6])
@pytest.mark.parametrize("model", ["cf2x", "primitive_drone"])
def test_flight_modes(model, mode):
    err = replay_aviary(HostSimEngine, load_golden(f"quadx_{model}_mode{mode}"))
    assert err["setpoint"] < 1e-6 and err["contact_mismatch"] == 0
    assert err["pos"] < 0.5 * POS_TOL and err["euler"] < 1e-3, err


@pytest.mark.parametrize("mode", [2, 3, 7])
def test_flight_modes_with_unstable_height_loop(mode):
    """Modes that run the z-velocity PID (kd/T = 6) limit-cycle in the reference itself on cf2x; rounding
    differences are amplified there, so only the position envelope is asserted."""
    err = replay_aviary(HostSimEngine, load_golden(f"quadx_cf2x_mode{mode}"))
    assert err["contact_mismatch"] == 0 and err["pos"] < POS_TOL, err


def test_floor_contact_flags_and_no_drag_in_contact():
    err = replay_aviary(HostSimEngine, load_golden("quadx_floor_contact"))
    assert err["contact_mismatch"] == 0 and err["pos"] < 1e-5


@pytest.mark.parametrize("name", ["hover_quat_dense", "hover_euler_sparse", "hover_quat_gentle", "hover_mode6", "hover_hz24_mode1"])
def test_hover_env(name):
    err = replay_hover(HostSimEngine, load_golden(name))
    assert err["flag_mismatch"] == 0
    assert err["obs"] < 5e-5 and err["reward"] < 5e-5, err


def test_batch_matches_oracle_on_seeded_inputs():
    n, steps = 32, 240
    rng = np.random.default_rng(7)
    model = build_model("quadx", "cf2x")
    start = np.column_stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(20, 30, n)])
    orn = rng.uniform(-0.3, 0.3, (n, 3))
    start, orn = start.astype(np.float32).astype(np.float64), orn.astype(np.float32).astype(np.float64)
    noise = rng.normal(4.0, 1.0, (steps * 2, n)).astype(np.float32).astype(np.float64)
    engines = [OracleEngine(model, None, n, start, orn), HostSimEngine(model, None, n, start, orn)]
    for e in engines:
        e.reset()
        e.set_mode(0)
    for i in range(0, steps, 20):
        sp = rng.uniform([-1, -1, -1, 0.2], [1, 1, 1, 0.7], (n, 4)).astype(np.float32).astype(np.float64)
        for e in engines:
            e.set_setpoints(sp)
            e.aviary_step(noise[2 * i : 2 * i + 40], n_steps=20)
    a, b = engines[0].state(), engines[1].state()
    assert np.abs(a[:, 3] - b[:, 3]).max() < 1e-4
    assert np.abs(a[:, 0] - b[:, 0]).max() < 1e-4


def test_observation_quaternion_sign_rule():
    """The kernel reports +-q with the sign getQuaternionFromEuler(getEulerFromQuaternion(q)) would give
    (quadx_base_env.py:243), without evaluating any trigonometric function outside gimbal lock."""
    import ctypes as C

    from engines import hostsim_lib, quat_observation_ref, sign_rule_quaternions

    L = hostsim_lib()
    qs = sign_rule_quaternions()
    out = np.zeros(4, dtype=np.float32)
    worst, negatives = 0.0, 0
    for q in qs:
        L.hs_obs_quat(q.ctypes.data_as(C.POINTER(C.c_double)), out.ctypes.data_as(C.POINTER(C.c_float)))
        r = quat_observation_ref(q)
        negatives += int(r[3] < 0)
        worst = max(worst, float(np.abs(out - r).max()))
    assert negatives > 50  # the w_e < 0 branch is exercised
    assert worst < 2e-5, worst  # 1e-5 is the reference's own gimbal-lock snap (|sarg| >= 0.99999)
