"""Parity tests proper: the CUDA path (through the C-ABI) against the golden vectors, the CPU oracle on
seeded inputs, and size-independent properties at BASELINE.json's full size (65 536 envs)."""
import numpy as np
import pytest

from engines import CudaEngine, OracleEngine, build_model, hover_config, load_golden, make_cuda_engine, replay_aviary, replay_hover

pytestmark = pytest.mark.gpu
POS_TOL = 1e-3  # north_star: |dpos| < 1e-3 m over 1000 env-steps (fp32 tolerance vs the fp64 reference)


def test_long_mode0_trajectory_within_tolerance():
    """BASELINE config 1: 1000 Hover env-steps (3000 Aviary steps, 6000 substeps) of mode-0 flight."""
    err = replay_aviary(make_cuda_engine, load_golden("quadx_mode0_long"), every=30)
    assert err["pos"] < POS_TOL, err["pos"]
    assert err["contact_mismatch"] == 0


@pytest.mark.parametrize("mode", [-1, 0, 1, 4, 5, 6])
@pytest.mark.parametrize("model", ["cf2x", "primitive_drone"])
def test_flight_modes(model, mode):
    err = replay_aviary(make_cuda_engine, load_golden(f"quadx_{model}_mode{mode}"), every=3)
    assert err["setpoint"] < 1e-6 and err["contact_mismatch"] == 0
    assert err["pos"] < 0.5 * POS_TOL and err["euler"] < 1e-3, err


@pytest.mark.parametrize("mode", [2, 3, 7])
@pytest.mark.parametrize("model", ["cf2x", "primitive_drone"])
def test_flight_modes_height_hold(model, mode):
    err = replay_aviary(make_cuda_engine, load_golden(f"quadx_{model}_mode{mode}"), every=3)
    assert err["contact_mismatch"] == 0 and err["pos"] < POS_TOL, err


def test_reference_scenarios_mode7():
    """tests/test_core.py:13-31 and :65-93 of the reference (hold, two set-points)."""
    for name in ("quadx_mode7_hold", "quadx_mode7_setpoints"):
        err = replay_aviary(make_cuda_engine, load_golden(name), every=10)
        assert err["pos"] < 1e-4 and err["contact_mismatch"] == 0, (name, err)


def test_floor_contact():
    err = replay_aviary(make_cuda_engine, load_golden("quadx_floor_contact"))
    assert err["contact_mismatch"] == 0 and err["pos"] < 1e-5


@pytest.mark.parametrize("name", ["hover_quat_dense", "hover_euler_sparse", "hover_quat_gentle", "hover_mode6", "hover_hz24_mode1"])
def test_hover_env_golden(name):
    err = replay_hover(make_cuda_engine, load_golden(name))
    assert err["flag_mismatch"] == 0
    assert err["obs"] < 5e-5 and err["reward"] < 5e-5, err


def _seeded_batch(n, seed):
    rng = np.random.default_rng(seed)
    f = lambda a: a.astype(np.float32).astype(np.float64)  # identical, fp32-representable inputs
    start = f(np.column_stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(20, 30, n)]))
    orn = f(rng.uniform(-0.3, 0.3, (n, 3)))
    return rng, f, start, orn


@pytest.mark.parametrize("mode", [0, 6])
def test_batch_4096_matches_oracle(mode):
    """BASELINE config 2 (lower end): 4096 envs, same seeded inputs through oracle and CUDA."""
    n, steps = 4096, 240
    rng, f, start, orn = _seeded_batch(n, 11 + mode)
    model = build_model("quadx", "cf2x")
    noise = f(rng.normal(4.0, 1.0, (steps * 2, n)))
    engines = [OracleEngine(model, None, n, start, orn), CudaEngine(model, None, n, start, orn)]
    for e in engines:
        e.reset()
        e.set_mode(mode)
    lo, hi = ([-1, -1, -1, 0.2], [1, 1, 1, 0.7]) if mode == 0 else ([-1, -1, -0.5, -0.5], [1, 1, 0.5, 0.5])
    for i in range(0, steps, 20):
        sp = f(rng.uniform(lo, hi, (n, 4)))
        for e in engines:
            e.set_setpoints(sp)
            e.aviary_step(noise[2 * i : 2 * i + 40], n_steps=20)
    a, b = engines[0].state(), engines[1].state()
    assert np.abs(a[:, 3] - b[:, 3]).max() < 0.5 * POS_TOL  # 240 Aviary steps, ~50 m travelled
    assert np.abs(a[:, 0] - b[:, 0]).max() < 2e-3
    assert np.array_equal(engines[0].contact(), engines[1].contact())


def test_hover_env_batch_matches_oracle():
    """env.reset + 60 env.step on 4096 envs with scripted actions and injected noise, incl. terminations."""
    n, steps = 4096, 60
    rng, f, _, _ = _seeded_batch(n, 5)
    model = build_model("quadx", "cf2x")
    env = hover_config(0, "quaternion", False, 3.0)
    start, orn = np.tile([[0.0, 0.0, 1.0]], (n, 1)), np.zeros((n, 3))
    orc, cud = OracleEngine(model, env, n, start, orn), CudaEngine(model, env, n, start, orn)
    nz0 = f(rng.normal(4.0, 1.0, (20, n)))
    o0, o1 = orc.env_reset(nz0), cud.env_reset(nz0)
    assert np.abs(o0 - o1).max() < 1e-5
    n_term = 0
    for k in range(steps):
        act = f(rng.uniform([-np.pi, -np.pi, -np.pi, 0.0], [np.pi, np.pi, np.pi, 0.8], (n, 4)) * [0.2, 0.2, 0.2, 1.0])
        nz = f(rng.normal(4.0, 1.0, (6, n)))
        ob0, r0, te0, tr0, in0 = orc.env_step(act, nz)
        ob1, r1, te1, tr1, in1 = cud.env_step(act, nz)
        # an env whose termination decision sits within fp32 rounding of a threshold may flip; none should
        assert np.array_equal(te0, te1) and np.array_equal(tr0, tr1) and np.array_equal(in0, in1), k
        assert np.abs(ob0 - ob1).max() < 1e-4 and np.abs(r0 - r1).max() < 1e-4, k
        n_term = int(te0.sum())
    assert n_term > 0  # the scenario does exercise terminations


def test_full_size_determinism_and_shard_independence():
    """65 536 envs: two runs with one seed are bit-identical, and splitting the batch into two handles
    with env offsets (what each rank does) reproduces the single-handle result exactly."""
    import torch

    from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverVecEnv

    n = 65536

    def run(num, offset):
        env = QuadXHoverVecEnv(num_envs=num, seed=123, env_offset=offset)
        env.reset()
        env.rollout(25)
        torch.cuda.synchronize()
        out = (env.aviary.obs.clone(), env.aviary.reward.clone(), env.aviary.state_tensor.clone(), env.aviary.istate_tensor.clone())
        env.close()
        return out

    a, b = run(n, 0), run(n, 0)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    lo, hi = run(n // 2, 0), run(n // 2, n // 2)
    assert torch.equal(torch.cat([lo[0], hi[0]]), a[0])
    assert torch.equal(torch.cat([lo[1], hi[1]]), a[1])
    assert torch.equal(torch.cat([lo[2], hi[2]], dim=0), a[2])  # warp tiles: [N/32][F/4][32][4]
    assert torch.isfinite(a[0]).all() and torch.isfinite(a[2]).all()


@pytest.mark.parametrize("n_envs", [65536, 393216])  # the second is several waves of CTAs
def test_full_size_autoreset_invariants(n_envs):
    """NEXT_STEP autoreset at 65 536 envs: an env that finished on call k returns, on call k+1, the first
    observation of a new episode (z just under the 1 m start after the 10 warm-up steps), reward 0 and
    cleared flags; nobody is ever left in a finished state for more than one call."""
    import torch

    from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverVecEnv

    env = QuadXHoverVecEnv(num_envs=n_envs, seed=1)
    obs, _ = env.reset()
    assert torch.allclose(obs[:, 10:13], torch.tensor([0.0, 0.0, 1.0], device=obs.device).expand(n_envs, 3), atol=0.05)
    first = obs.clone()
    total_done, prev_done = 0, torch.zeros(n_envs, dtype=torch.bool, device=obs.device)
    for _ in range(40):
        env.rollout(1)
        a = env.aviary
        done = a.term.bool() | a.trunc.bool()
        assert not bool((done & prev_done).any())
        if bool(prev_done.any()):
            z = a.obs[prev_done][:, 12]
            assert bool(((z > 0.9) & (z < 1.0)).all())
            assert bool((a.reward[prev_done] == 0).all())
            assert bool((a.step_counts[prev_done] == 0).all())
            # same start pose, same warm-up dynamics: only the motor-noise draws differ
            assert float((a.obs[prev_done][:, :13] - first[prev_done][:, :13]).abs().max()) < 1e-2
        assert bool((a.reward[done & a.term.bool()] < -50).all())  # -100 overwrite on collision / out of bounds
        total_done += int(done.sum())
        prev_done = done
    assert total_done > 1000  # random actions crash often (SURVEY 8d)
    env.close()


def test_free_fall_closed_form_at_full_size():
    """Mode -1 with zero pwm, drag off: z_k = z0 - g dt^2 k(k+1)/2 for all 65 536 envs."""
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    n, k = 65536, 240
    m = build_model("quadx", "cf2x")
    m.drag_const[:] = [0.0, 0.0, 0.0]
    from pyflyt_b200.core import aviary as _av

    real_build = _av.build_model
    _av.build_model = lambda *a, **kw: m  # hand the edited table to the constructor
    try:
        av = BatchedAviary(np.tile([[0.0, 0.0, 500.0]], (n, 1)), np.zeros((n, 3)))
    finally:
        _av.build_model = real_build
    av.set_mode(-1)
    av.set_all_setpoints(torch.zeros((n, 4), device="cuda"))
    av.step(k // 2, noise=torch.full((k, n), 4.0, device="cuda"))
    z = av.all_states[:, 3, 2].double().cpu().numpy()
    dt, g = 1.0 / 240.0, 9.81
    assert np.abs(z - (500.0 - g * dt * dt * k * (k + 1) / 2.0)).max() < 2e-4
    assert np.ptp(z) == 0.0


def test_host_buffer_entry_matches_device_entry():
    import torch

    from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverVecEnv

    n = 8192
    envs = [QuadXHoverVecEnv(num_envs=n, seed=9), QuadXHoverVecEnv(num_envs=n, seed=9)]
    for e in envs:
        e.reset()
    g = torch.Generator().manual_seed(0)
    act = (torch.rand((n, 4), generator=g) * torch.tensor([0.6, 0.6, 0.6, 0.8])).pin_memory()
    obs_h = torch.empty((n, envs[0].obs_dim)).pin_memory()
    rew_h = torch.empty(n).pin_memory()
    te_h = torch.empty(n, dtype=torch.uint8).pin_memory()
    tr_h = torch.empty(n, dtype=torch.uint8).pin_memory()
    for _ in range(5):
        envs[0].aviary.env_step_host(act, obs_h, rew_h, te_h, tr_h)
        torch.cuda.synchronize()
        ob, r, te, tr, _ = envs[1].step(act.cuda())
        assert torch.equal(ob.cpu(), obs_h) and torch.equal(r.cpu(), rew_h)
        assert torch.equal(te.cpu(), te_h.bool()) and torch.equal(tr.cpu(), tr_h.bool())


def test_single_env_adaptor_signature():
    from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverEnv

    env = QuadXHoverEnv()
    obs, info = env.reset(seed=0)
    assert obs.shape == (21,) and obs.dtype == np.float64 and set(info) == {"out_of_bounds", "collision", "env_complete"}
    obs, rew, term, trunc, info = env.step(np.array([0.0, 0.0, 0.0, 0.4]))
    assert obs.shape == (21,) and isinstance(rew, float) and isinstance(term, bool) and isinstance(trunc, bool)
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode,max_seconds", [(0, 10.0), (6, 0.25), (0, 0.05)])
def test_spare_reset_equals_inline_reset(mode, max_seconds):
    """In-launch autoreset copies the env's spare post-warm-up state, rebuilt on a side stream with noise keyed by
    (env, episode).  It must be bit-identical to integrating every warm-up inside the step launch (inline_reset=True),
    also when the start pose is edited mid-run (stale spares are ignored), with 3-step episodes (max_seconds=0.05), and in
    mode 6 (position control: motors spin during the warm-up; episodes cut to 11 steps so that resets happen)."""
    import torch

    from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverVecEnv

    n = 8192
    rng = np.random.default_rng(3)
    sp = np.zeros((n, 3), dtype=np.float32)
    sp[:, 2] = rng.uniform(0.6, 1.4, n)
    so = np.zeros((n, 3), dtype=np.float32)
    so[:, 2] = rng.uniform(-1, 1, n)
    outs = []
    for inline in (False, True):
        env = QuadXHoverVecEnv(num_envs=n, flight_mode=mode, seed=5, start_pos=sp, start_orn=so, inline_reset=inline, max_duration_seconds=max_seconds)
        env.reset()
        resets, trace = 0, []
        for k in range(90):
            env.rollout(1)
            resets += int((env.aviary.term | env.aviary.trunc).sum())
            trace.append(env.aviary.obs.sum().item())
            if k == 40:  # move every other env's start pose
                env.aviary.start_pos[::2, 2] += 0.25
        torch.cuda.synchronize()
        outs.append((env.aviary.obs.clone(), env.aviary.reward.clone(), env.aviary.state_tensor.clone(), resets, trace))
        env.close()
    a, b = outs
    assert a[3] > n // 4, a[3]  # plenty of resets (position control in mode 6 keeps many envs alive for the whole run)
    assert a[3] == b[3] and a[4] == b[4]
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    # the edited start pose is what later resets use
    env = QuadXHoverVecEnv(num_envs=256, flight_mode=mode, seed=5, max_duration_seconds=0.05)
    env.reset()
    env.aviary.start_pos[:, 2] = 2.0
    for _ in range(12):
        env.rollout(1)
    torch.cuda.synchronize()
    assert float(env.aviary.state_row(2).min()) > 1.5
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("drone_model", ["cf2x", "primitive_drone"])
def test_north_star_parity_4096_envs_1000_env_steps(drone_model):
    """BASELINE.json's bar at scale: |dpos| < 1e-3 m against the fp64 oracle over 1000 env-steps (3000 Aviary steps,
    6000 physics substeps) for 4096 drones flying different scripted rate / thrust commands with the same noise draws.
    The drones start 1.5 km up so that none reaches the floor (a contact flag that flips one substep apart in fp32 and
    fp64 gates the rotational drag and is a legitimate source of divergence, not a precision question); positions are
    read as hi + lo fp64 from the state tensor."""
    n, chunks, per = 4096, 10, 300
    rng = np.random.default_rng(2024)
    f = lambda a: a.astype(np.float32).astype(np.float64)  # noqa: E731
    model = build_model("quadx", drone_model)
    pos0 = f(np.stack([rng.uniform(-2, 2, n), rng.uniform(-2, 2, n), rng.uniform(1500, 1510, n)], axis=-1))
    orn0 = f(np.stack([rng.uniform(-0.2, 0.2, n), rng.uniform(-0.2, 0.2, n), rng.uniform(-3, 3, n)], axis=-1))
    orc = OracleEngine(model, None, n, pos0, orn0)
    cud = CudaEngine(model, None, n, pos0, orn0, drone_model=drone_model)
    for e in (orc, cud):
        e.reset()
        e.set_mode(0)
    err, travelled = np.zeros(n), np.zeros(n)
    prev = pos0.copy()
    for c in range(chunks):
        sp = f(np.concatenate([rng.uniform(-0.6, 0.6, (n, 3)), rng.uniform(0.25, 0.55, (n, 1))], axis=-1))  # body rates, thrust
        noise = f(rng.normal(4.0, 1.0, (per * 2, n)))
        for e in (orc, cud):
            e.set_setpoints(sp)
            e.aviary_step(noise, per)
        p0 = orc.state()[:, 3, :]
        p1 = cud.av.precise_positions.cpu().numpy()  # position rows: hi + lo
        assert p0[:, 2].min() > 10.0  # nobody near the floor
        err = np.maximum(err, np.abs(p0 - p1).max(axis=1))
        travelled += np.linalg.norm(p0 - prev, axis=1)
        prev = p0
    assert np.isfinite(err).all() and err.max() < 1e-3, (err.max(), np.percentile(err, 99))
    assert np.percentile(err, 99) < 4e-4
    assert np.median(travelled) > 50.0  # these are real flights, not hovering drones


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["fixedwing-waypoints", "rocket-landing", "quadx-waypoints"])
def test_masked_reset_on_autoreset_handle_is_not_reset_twice(kind):
    """A finished env that the user resets by hand (masked pfb_env_reset) while autoreset is on must leave the
    pending done list — otherwise the next launch's tail CTA resets it again while its regular thread steps it.  After the
    masked reset + one step every masked env must have been STEPPED (step_count 1, a non-zero reward), deterministically."""
    import torch

    from pyflyt_b200.gym_envs import FixedwingWaypointsVecEnv, QuadXWaypointsVecEnv, RocketLandingVecEnv

    def run():
        if kind == "fixedwing-waypoints":
            env, row = FixedwingWaypointsVecEnv(num_envs=8192, seed=5, max_duration_seconds=0.5), 0
        elif kind == "rocket-landing":
            env, row = RocketLandingVecEnv(num_envs=8192, seed=5, max_duration_seconds=0.4), 0
        else:
            env, row = QuadXWaypointsVecEnv(num_envs=8192, seed=5, max_duration_seconds=0.5), 0
        av = env.aviary
        env.reset()
        checked = 0
        for k in range(40):
            env.rollout(1)
            done = av.term.bool() | av.trunc.bool()
            if bool(done.any()):
                mask = done.clone()
                mask[::7] = True  # plus some envs that were not done
                env.reset(mask=mask.to(torch.uint8))
                env.rollout(1)
                steps = av.istate_tensor[row]
                assert bool((steps[mask] == 1).all()), (k, steps[mask].unique())
                assert bool((av.reward[mask] != 0).all()), k
                checked += int(mask.sum())
        torch.cuda.synchronize()
        out = (av.obs.clone(), av.reward.clone(), av.state_tensor.clone())
        env.close()
        return out, checked

    (a, ca), (b, cb) = run(), run()
    assert ca == cb and ca > 1000
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,n", [(0, 65536), (0, 1000), (6, 8192)])
def test_fused_rollout_equals_stepwise(mode, n):
    """pfb_env_rollout(n >= 4) runs QuadX-Hover as FUSED launches of up to 16 env steps (k_hover_rollout: state in registers across
    the steps, spares kept three ahead and topped up behind every launch); fewer steps run one launch per step.  Same Philox
    counters, same arithmetic: the drawn actions are equal bit for bit, always; the physics agrees bit for bit except where the
    two compiled copies of an expression contract a multiply-add differently (a one-ulp fp32 difference in a PID term a few
    times per 1e5 env-steps, which an env then carries until its next reset).  The two ways of stepping are freely mixed on one
    handle here: the hand-over of the reset pipeline in both directions is part of the test."""
    import torch

    from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverVecEnv

    plan = [16, 16, 5, 1, 1, 23, 1, 40, 4, 2, 64]  # fused chunks (>= 4) and single steps, interleaved
    a = QuadXHoverVecEnv(num_envs=n, seed=21, flight_mode=mode)
    b = QuadXHoverVecEnv(num_envs=n, seed=21, flight_mode=mode)
    a.reset()
    b.reset()
    done_total, worst, diverged_max, inexact_max = 0, 0.0, 0, 0.0
    for chunk in plan:
        a.rollout(chunk)             # fused when chunk >= 4
        for _ in range(chunk):
            b.rollout(1)             # always one launch per step
            done_total += int((b.aviary.term | b.aviary.trunc).sum())
        A, B = a.aviary, b.aviary
        assert torch.equal(A.setpoints, B.setpoints), chunk      # the actions of the last step: pure Philox, no physics
        same = A.state_row_int(17) == B.state_row_int(17)        # same step counter = same reset history
        diverged_max = max(diverged_max, int((~same).sum()))     # a termination decided within an ulp of its threshold
        d = (A.obs.double() - B.obs.double()).abs().amax(dim=1)
        worst = max(worst, float(d[same].max()))
        inexact_max = max(inexact_max, float((d[same] > 0).double().mean()))
        assert torch.equal(A.term[same], B.term[same]) and torch.equal(A.trunc[same], B.trunc[same]), chunk
        assert float((A.reward.double() - B.reward.double()).abs()[same].max()) < 1e-3, chunk
    print(f"\n[fused vs stepwise, mode {mode}, {n} envs, {sum(plan)} steps] {done_total} episodes finished; envs with a different reset history: "
          f"at most {diverged_max}; envs not bit-equal at a checkpoint: at most {inexact_max:.2e} of them; max |obs difference| {worst:.2e}")
    assert done_total > n // 2       # resets everywhere (mode 0: ~6 per env)
    assert diverged_max <= max(2, n // 4096)
    assert inexact_max < 1e-2 and worst < (1e-4 if mode == 0 else 1e-2)  # mode 6: the z-velocity PID limit cycle amplifies an ulp (DESIGN 5)
    a.close()
    b.close()
