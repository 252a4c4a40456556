"""The instantiation bench.py times — Philox noise generated in-kernel, NEXT_STEP autoreset with spare post-reset states —
pinned to the fp64 CPU oracle.  The device streams are stateless (tests/philox_replay.py regenerates them from
(seed, env id, call number, tag)), so the oracle is driven in lock-step with exactly the noise the kernel drew, the actions
it was given and the same reset schedule, at BASELINE.json's full batch (65 536 envs) for 200 env steps (~1e5 autoresets)."""
import numpy as np
import pytest

from engines import OracleEngine, build_model, hover_config
from philox_replay import Streams

pytestmark = pytest.mark.gpu


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float32).astype(np.float64)


@pytest.mark.parametrize("n,steps,randact", [(65536, 200, False), (8192, 120, True)])
def test_hover_philox_autoreset_matches_oracle(n, steps, randact):
    import torch

    from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverVecEnv

    seed = 20240924
    env = QuadXHoverVecEnv(num_envs=n, seed=seed)  # autoreset=True, Philox noise: k_hover_step<0, false, false, true, false>
    av = env.aviary
    dump = torch.zeros((6, n), dtype=torch.float32, device=av.device)
    av.set_noise_dump(dump)
    streams = Streams(seed, n, noise_loc=4.0)
    model = build_model("quadx", "cf2x")
    orc = OracleEngine(model, hover_config(0, "quaternion", False, 3.0), n, np.tile([[0.0, 0.0, 1.0]], (n, 1)), np.zeros((n, 3)))

    obs_g, _ = env.reset()
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(0).astype(np.float64))
    assert np.abs(obs_g.double().cpu().numpy() - obs_o).max() < 1e-5

    rng = np.random.default_rng(1)
    episode = np.ones(n, dtype=np.int64)       # number of the spare an env takes at its next autoreset
    done_prev = np.zeros(n, dtype=bool)
    live = np.ones(n, dtype=bool)              # envs still compared (an env whose termination decision flipped is dropped)
    worst_obs = worst_rew = worst_noise = 0.0
    n_resets = n_done = n_flip = 0
    for k in range(steps):
        if randact:
            env.rollout(1)
            act = av.setpoints.double().cpu().numpy()  # the kernel writes the actions it drew back
            assert np.array_equal(act.astype(np.float32), streams.actions(k))
        else:
            act = _f(rng.uniform([-np.pi, -np.pi, -np.pi, 0.0], [np.pi, np.pi, np.pi, 0.8], (n, 4)))
            env.step(torch.as_tensor(act, dtype=torch.float32, device=av.device))
        og, rg = av.obs.double().cpu().numpy(), av.reward.double().cpu().numpy()
        teg, trg, ig = av.term.cpu().numpy().astype(bool), av.trunc.cpu().numpy().astype(bool), av.info_bits.cpu().numpy()
        # ---- oracle, same step: everyone steps on the replayed noise, then the envs that finished on the previous call are
        #      reset instead (NEXT_STEP): first observation of episode `episode[i]`, reward 0, flags cleared
        nz = streams.step_noise(k)
        oo, ro, teo, tro, io = orc.o.env_step(act, nz.astype(np.float64))
        teo, tro = teo.astype(bool), tro.astype(bool)
        if done_prev.any():
            rz = np.zeros((20, n))
            idx = np.nonzero(done_prev)[0]
            rz[:, idx] = streams.autoreset_noise(episode[idx], envs=idx)
            obs_r = orc.o.env_reset(mask=done_prev.astype(np.uint8), noise=rz)
            oo[done_prev], ro[done_prev], teo[done_prev], tro[done_prev], io[done_prev] = obs_r[done_prev], 0.0, False, False, 0
            episode[idx] += 1
            n_resets += len(idx)
        # ---- the kernel's own draws (dumped) vs the host replay, for the envs that ran all three Aviary steps
        full = ~done_prev & ~(teg | trg)
        worst_noise = max(worst_noise, float(np.abs(dump.cpu().numpy()[:, full] - nz[:, full]).max()))
        # ---- outcomes
        flip = live & ((teg != teo) | (trg != tro))
        if flip.any():  # a termination decided within rounding of its threshold: drop the env from the comparison
            n_flip += int(flip.sum())
            live &= ~flip
        cmp = live
        assert np.array_equal(ig[cmp] & 3, io[cmp] & 3), k
        worst_obs = max(worst_obs, float(np.abs(og[cmp] - oo[cmp]).max()))
        worst_rew = max(worst_rew, float(np.abs(rg[cmp] - ro[cmp]).max()))
        done_prev = teg | trg
        n_done += int(done_prev.sum())
        # (the oracle follows the kernel's reset schedule, which is its own for every env that is still compared)
    print(f"\n[timed-path parity] {n} envs x {steps} steps: {n_done} episodes finished, {n_resets} autoresets, flips {n_flip}; "
          f"max |obs| {worst_obs:.2e}, max |reward| {worst_rew:.2e}, max |noise dump - replay| {worst_noise:.2e}")
    assert n_resets > n  # every env was reset more than once on average
    # the device Box-Muller (__logf / __sincosf / sqrt.approx) is within 2.2e-4 of fp64 over every u1 and every u2
    # (tests/test_device_math.py::test_box_muller_device); the worst is at u1 = 1 - 2^-24, where __logf's absolute error is
    # comparable to -ln u1 = 6e-8 and r = sqrt(-2 ln u1) = 3.5e-4 carries it as a square root
    assert worst_noise < 5e-4
    assert n_flip <= max(2, n // 4096)
    assert worst_obs < 1e-4 and worst_rew < 1e-4
    env.close()


def test_fixedwing_waypoints_philox_autoreset_matches_oracle():
    """The same pin for BASELINE configs[2]: k_fwwp_step with Philox noise (N(1, 1): one motor), device-drawn waypoints and
    NEXT_STEP autoreset through spare post-reset states, 16 384 aircraft x 150 env steps, against the oracle driven with the
    replayed noise AND the replayed waypoint draws (waypoint_handler.py:65-83)."""
    import torch

    from engines import waypoints_config
    from pyflyt_b200.gym_envs.fixedwing_waypoints_env import FixedwingWaypointsVecEnv

    n, steps, seed, T, dome = 16384, 150, 777, 4, 100.0
    env = FixedwingWaypointsVecEnv(num_envs=n, seed=seed, goal_reach_distance=25.0, max_duration_seconds=3.0)  # episodes of <= 90 steps
    av = env.aviary
    streams = Streams(seed, n, noise_loc=1.0)
    model = build_model("fixedwing", "fixedwing")
    cfg = waypoints_config("quaternion", False, T, 25.0, dome, max_duration=3.0)
    orc = OracleEngine(model, cfg, n, np.tile([[0.0, 0.0, 10.0]], (n, 1)), np.zeros((n, 3)))

    obs_g, _ = env.reset()
    tg = streams.waypoint_targets(0x80000000, T, dome, min_height=0.5)  # fixedwing_waypoints_env.py:81
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(0).astype(np.float64), targets=tg.astype(np.float64).reshape(n, -1))
    assert np.abs(obs_g.double().cpu().numpy() - obs_o).max() < 2e-3

    rng = np.random.default_rng(2)
    episode = np.ones(n, dtype=np.int64)
    done_prev = np.zeros(n, dtype=bool)
    live = np.ones(n, dtype=bool)
    worst_obs = worst_rew = 0.0
    n_resets = n_flip = reached = 0
    for k in range(steps):
        act = _f(rng.uniform(-1.0, 1.0, (n, 4)) * [0.5, 0.3, 0.3, 1.0])
        env.step(torch.as_tensor(act, dtype=torch.float32, device=av.device))
        og, rg = av.obs.double().cpu().numpy(), av.reward.double().cpu().numpy()
        teg, trg, ig = av.term.cpu().numpy().astype(bool), av.trunc.cpu().numpy().astype(bool), av.info_bits.cpu().numpy()
        oo, ro, teo, tro, io = orc.o.env_step(act, streams.step_noise(k, 4).astype(np.float64))
        teo, tro = teo.astype(bool), tro.astype(bool)
        if done_prev.any():
            idx = np.nonzero(done_prev)[0]
            rz = np.zeros((20, n))
            rz[:, idx] = streams.autoreset_noise(episode[idx], envs=idx)
            tgr = np.zeros((n, T, 3))
            tgr[idx] = streams.waypoint_targets(episode[idx], T, dome, min_height=0.5, envs=idx)
            obs_r = orc.o.env_reset(mask=done_prev.astype(np.uint8), noise=rz, targets=tgr.reshape(n, -1))
            oo[done_prev], ro[done_prev], teo[done_prev], tro[done_prev], io[done_prev] = obs_r[done_prev], 0.0, False, False, 0
            episode[idx] += 1
            n_resets += len(idx)
        flip = live & ((teg != teo) | (trg != tro) | ((ig >> 3) != (io >> 3)))  # termination / target-reached decisions at a threshold
        n_flip += int(flip.sum())
        live &= ~flip
        worst_obs = max(worst_obs, float(np.abs(og[live] - oo[live]).max()))
        worst_rew = max(worst_rew, float(np.abs(rg[live] - ro[live]).max()))
        reached = max(reached, int((ig >> 3).max()))
        done_prev = teg | trg
    print(f"\n[timed-path parity, fixedwing-waypoints] {n} envs x {steps} steps: {n_resets} autoresets, flips {n_flip}, max targets reached {reached}; "
          f"max |obs| {worst_obs:.2e}, max |reward| {worst_rew:.2e}")
    assert n_resets > n and reached >= 1
    assert n_flip <= n // 1000
    assert worst_obs < 5e-3 and worst_rew < 5e-3  # target deltas are O(100 m) fp32 numbers
    env.close()


@pytest.mark.parametrize("ceiling,max_duration", [(500.0, 2.0), (120.0, 30.0)])
def test_rocket_landing_philox_autoreset_matches_oracle(ceiling, max_duration):
    """The same pin for BASELINE configs[3]: k_land_step with Philox booster noise (N(1, 1)), device-drawn randomised drops
    (rocket_base_env.py:192-199), accelerated drop, contact response on, NEXT_STEP autoreset through spare post-reset states;
    16 384 rockets x 200 env steps against the oracle driven with the replayed noise and the replayed drop poses.
    ceiling 500 / 2 s episodes: every episode ends by truncation in flight; ceiling 120: every rocket reaches the ground (or
    the pad) within a second, so the crash / pad-contact terminations and the contact response are in the comparison."""
    import torch

    from engines import landing_config
    from pyflyt_b200.gym_envs.rocket_landing_env import RocketLandingVecEnv

    n, steps, seed = 16384, 200, 4242
    env = RocketLandingVecEnv(num_envs=n, seed=seed, ceiling=ceiling, max_duration_seconds=max_duration)
    av = env.aviary
    streams = Streams(seed, n, noise_loc=1.0)
    model = build_model("rocket", "rocket", starting_fuel_ratio=0.05)
    cfg = landing_config("quaternion", False, False, True, ceiling=ceiling, max_duration=max_duration, contact_response=True)
    sp, so = streams.drop_poses(0x80000000, ceiling, 200.0)
    sp, so = sp.astype(np.float64), so.astype(np.float64)
    orc = OracleEngine(model, cfg, n, sp, so)

    obs_g, _ = env.reset()
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(0).astype(np.float64))
    assert np.abs(obs_g.double().cpu().numpy() - obs_o).max() < 5e-3

    rng = np.random.default_rng(3)
    episode = np.ones(n, dtype=np.int64)
    done_prev = np.zeros(n, dtype=bool)
    live = np.ones(n, dtype=bool)
    worst_obs = worst_rew = 0.0
    n_resets = n_flip = n_coll = n_pad = 0
    worst_where = None
    loose = np.zeros(n, dtype=bool)
    for k in range(steps):
        act = _f(rng.uniform([-1, -1, -1, 0, 0, -1, -1], [1, 1, 1, 1, 1, 1, 1], (n, 7)))
        env.step(torch.as_tensor(act, dtype=torch.float32, device=av.device))
        og, rg = av.obs.double().cpu().numpy(), av.reward.double().cpu().numpy()
        teg, trg, ig = av.term.cpu().numpy().astype(bool), av.trunc.cpu().numpy().astype(bool), av.info_bits.cpu().numpy()
        oo, ro, teo, tro, io = orc.o.env_step(act, streams.step_noise(k, 3).astype(np.float64))
        teo, tro = teo.astype(bool), tro.astype(bool)
        if done_prev.any():
            idx = np.nonzero(done_prev)[0]
            rz = np.zeros((20, n))
            rz[:, idx] = streams.autoreset_noise(episode[idx], envs=idx)
            p_, o_ = streams.drop_poses(episode[idx], ceiling, 200.0, envs=idx)
            sp[idx], so[idx] = p_, o_
            orc.o.set_start(sp, so)
            obs_r = orc.o.env_reset(mask=done_prev.astype(np.uint8), noise=rz)
            oo[done_prev], ro[done_prev], teo[done_prev], tro[done_prev], io[done_prev] = obs_r[done_prev], 0.0, False, False, 0
            episode[idx] += 1
            n_resets += len(idx)
        flip = live & ((teg != teo) | (trg != tro) | ((ig & 7) != (io & 7)))
        n_flip += int(flip.sum())
        live &= ~flip
        # the step of a crash: both sides terminate (flags compared above), but the post-impact velocities are the output of a
        # stiff impulse iteration on a body arriving at 80+ m/s (0.35 m of penetration per substep): which corner points are
        # inside flips with fp32 rounding.  Gentle contact is pinned by tests/test_contact_response.py; here the crash step's
        # observation / reward stay out of the comparison
        cmp = live & ((ig & 2) == 0)
        dmat = np.abs(og - oo) * cmp[:, None]
        if dmat.max() > worst_obs:
            wi, wc = np.unravel_index(np.argmax(dmat), dmat.shape)
            worst_where = (k, int(wi), int(wc), float(og[wi, wc]), float(oo[wi, wc]), int(ig[wi]), bool(done_prev[wi]), float(og[wi, 12]))
        worst_obs = max(worst_obs, float(np.abs(og[cmp] - oo[cmp]).max()))
        worst_rew = max(worst_rew, float(np.abs(rg[cmp] - ro[cmp]).max()))
        loose |= cmp & ((np.abs(og - oo).max(axis=1) > 5e-3) | (np.abs(rg - ro) > 2e-2))
        n_coll += int(((ig & 2) != 0).sum())
        n_pad += int((og[:, -1] != 0).sum())
        done_prev = teg | trg
    print(f"\n[timed-path parity, rocket-landing ceiling {ceiling:g}] {n} envs x {steps} steps: {n_resets} autoresets, {n_coll} collisions, "
          f"{n_pad} pad-contact observations, flips {n_flip}; max |obs| {worst_obs:.2e} at (step, env, col, gpu, oracle, info, was_reset, z) = {worst_where}, "
          f"max |reward| {worst_rew:.2e}")
    assert n_resets > n
    if ceiling < 200.0:
        assert n_coll > n  # every episode ends on the ground
    assert n_flip <= n // 500
    # positions are O(400 m) fp32 numbers; the reward multiplies velocity differences by 4.  The lifting-surface model is
    # DISCONTINUOUS at the stall angle (lifting_surfaces.py:349-448: attached flow / flat plate): a finlet whose angle of attack
    # sits within fp32 rounding of it takes the other branch for one substep and the episode carries a ~2e-4 rad/s offset from
    # then on (tools/dbg_rocket_env.py shows one such event: 5e-6 -> 5e-4 in a single step, linear growth afterwards).  Such
    # envs are counted, not hidden: at most 0.1 % of them, and never beyond 0.1
    assert loose.mean() < 1e-3, int(loose.sum())
    assert worst_obs < 0.1 and worst_rew < 0.5
    env.close()


@pytest.mark.parametrize("mode,yaw", [(0, False), (7, True)])
def test_quadx_waypoints_philox_autoreset_matches_oracle(mode, yaw):
    """The same pin for QuadX-Waypoints (SURVEY 8f #1): k_qxwp_step with Philox motor noise, device-drawn waypoints (and yaw
    targets), NEXT_STEP autoreset through spare post-reset states; 16 384 envs x 150 env steps."""
    import torch

    from engines import quadx_waypoints_config
    from pyflyt_b200.gym_envs.quadx_waypoints_env import QuadXWaypointsVecEnv

    n, steps, seed, T, dome = 16384, 150, 99, 4, 5.0
    env = QuadXWaypointsVecEnv(num_envs=n, seed=seed, flight_mode=mode, use_yaw_targets=yaw, goal_reach_distance=1.0, goal_reach_angle=3.0,
                               max_duration_seconds=2.0)  # episodes of <= 60 steps
    av = env.aviary
    streams = Streams(seed, n, noise_loc=4.0)
    model = build_model("quadx", "cf2x")
    cfg = quadx_waypoints_config(flight_mode=mode, num_targets=T, use_yaw_targets=yaw, goal_reach_distance=1.0, goal_reach_angle=3.0, dome=dome,
                                 max_duration=2.0)
    orc = OracleEngine(model, cfg, n, np.tile([[0.0, 0.0, 1.0]], (n, 1)), np.zeros((n, 3)))

    obs_g, _ = env.reset()
    tg = streams.waypoint_targets(0x80000000, T, dome, min_height=0.1, yaw=yaw)
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(0).astype(np.float64), targets=tg.astype(np.float64).reshape(n, -1))
    assert np.abs(obs_g.double().cpu().numpy() - obs_o).max() < 1e-4

    rng = np.random.default_rng(5)
    episode = np.ones(n, dtype=np.int64)
    done_prev = np.zeros(n, dtype=bool)
    live = np.ones(n, dtype=bool)
    worst_obs = worst_rew = 0.0
    n_resets = n_flip = reached = 0
    loose = np.zeros(n, dtype=bool)
    for k in range(steps):
        if mode == 7:  # position setpoints inside the dome: the drone chases them, reaches targets, sometimes leaves the dome
            act = _f(rng.uniform([-2.0, -2.0, -1.0, 0.5], [2.0, 2.0, 1.0, 3.0], (n, 4)))
        else:
            act = _f(rng.uniform([-1.0, -1.0, -1.0, 0.0], [1.0, 1.0, 1.0, 0.8], (n, 4)))
        env.step(torch.as_tensor(act, dtype=torch.float32, device=av.device))
        og, rg = av.obs.double().cpu().numpy(), av.reward.double().cpu().numpy()
        teg, trg, ig = av.term.cpu().numpy().astype(bool), av.trunc.cpu().numpy().astype(bool), av.info_bits.cpu().numpy()
        oo, ro, teo, tro, io = orc.o.env_step(act, streams.step_noise(k, 4).astype(np.float64))
        teo, tro = teo.astype(bool), tro.astype(bool)
        if done_prev.any():
            idx = np.nonzero(done_prev)[0]
            rz = np.zeros((20, n))
            rz[:, idx] = streams.autoreset_noise(episode[idx], envs=idx)
            tgr = np.zeros((n, T, 4 if yaw else 3))
            tgr[idx] = streams.waypoint_targets(episode[idx], T, dome, min_height=0.1, envs=idx, yaw=yaw)
            obs_r = orc.o.env_reset(mask=done_prev.astype(np.uint8), noise=rz, targets=tgr.reshape(n, -1))
            oo[done_prev], ro[done_prev], teo[done_prev], tro[done_prev], io[done_prev] = obs_r[done_prev], 0.0, False, False, 0
            episode[idx] += 1
            n_resets += len(idx)
        flip = live & ((teg != teo) | (trg != tro) | ((ig >> 3) != (io >> 3)))
        n_flip += int(flip.sum())
        live &= ~flip
        cols = slice(10, 13) if mode == 7 else slice(None)  # mode 7: the reference's z-velocity PID limit-cycles (DESIGN 5): position envelope
        dobs, drew = np.abs(og[:, cols] - oo[:, cols]).max(axis=1), np.abs(rg - ro)
        worst_obs = max(worst_obs, float(dobs[live].max()))
        worst_rew = max(worst_rew, float(drew[live].max()))
        loose |= live & ((dobs > 1e-3) | (drew > 5e-2))
        reached = max(reached, int((ig >> 3).max()))
        done_prev = teg | trg
    print(f"\n[timed-path parity, quadx-waypoints mode {mode}] {n} envs x {steps} steps: {n_resets} autoresets, flips {n_flip}, max targets reached "
          f"{reached}; max |obs| {worst_obs:.2e}, max |reward| {worst_rew:.2e}")
    assert n_resets > n
    assert n_flip <= n // 500
    if mode == 7:  # chaotic amplification in the limit cycle: 99.5 % of the envs stay inside the tight envelope for the whole run
        assert reached >= 1
        assert loose.mean() < 5e-3, int(loose.sum())
        assert worst_obs < 2e-2 and worst_rew < 0.5
    else:
        assert worst_obs < 5e-4 and worst_rew < 5e-3  # 1 / distance terms amplify a 1e-6 m difference near a target
    env.close()


def test_dogfight_philox_autoreset_matches_oracle():
    """The same pin for BASELINE configs[4] (arena-sharded fused kernel): k_df_step<2> with Philox motor noise, device-drawn
    spawns (_get_start_pos_orn), arena-level NEXT_STEP autoreset through spare post-reset states; 8192 arenas x 2 aircraft x 150
    env steps (2 s episodes: every arena is re-spawned twice) against the oracle driven with the replayed noise and spawns."""
    import torch

    from engines import dogfight_config
    from test_draw_distributions import dogfight_spawns

    from pyflyt_b200.pz_envs import MAFixedwingDogfightVecEnv

    num_arenas, steps, seed = 8192, 150, 2025
    n = 2 * num_arenas
    kw = dict(lethal_distance=150.0, lethal_angle=1.0, damage_per_hit=0.05)
    env = MAFixedwingDogfightVecEnv(num_arenas=num_arenas, seed=seed, lethal_distance=150.0, lethal_angle_radians=1.0, damage_per_hit=0.05,
                                    max_duration_seconds=2.0)
    av = env.aviary
    streams = Streams(seed, n, noise_loc=1.0)
    model = build_model("fixedwing", "acrowing")
    cfg = dogfight_config(1, False, max_duration=2.0, **kw)

    def spawn(seq):
        pos, yaw = dogfight_spawns(seed, num_arenas, seq)
        orn = np.zeros((n, 3))
        orn[:, 2] = yaw.reshape(-1)
        return _f(pos.reshape(n, 3)), _f(orn)

    sp, so = spawn(0x80000000)
    orc = OracleEngine(model, cfg, n, sp, so)
    obs_g, _ = env.reset()
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(0).astype(np.float64))
    assert np.abs(obs_g.double().cpu().numpy() - obs_o).max() < 5e-3

    rng = np.random.default_rng(8)
    episode = np.ones(n, dtype=np.int64)         # per agent, arena-uniform
    agent_done = np.zeros(n, dtype=bool)          # left self.agents in the current episode
    arena_reset = np.zeros(n, dtype=bool)         # per agent: its arena is re-spawned on this call
    live = np.ones(n, dtype=bool)
    worst_obs = worst_rew = 0.0
    n_resets = n_flip = n_hits = 0
    worst_where = None
    for k in range(steps):
        act = _f(np.clip(rng.uniform(-1, 1, (n, 4)) * 0.4 + np.array([0.0, 0.15, 0.0, 0.0]) * (np.arange(n) % 5 == 0)[:, None], -1, 1))
        env.step(torch.as_tensor(act, dtype=torch.float32, device=av.device))
        og, rg = av.obs.double().cpu().numpy(), av.reward.double().cpu().numpy()
        teg, trg = av.term.cpu().numpy().astype(bool), av.trunc.cpu().numpy().astype(bool)
        mem = orc.o.df_get_actions() if arena_reset.any() else None  # a re-spawned arena is NOT stepped on this call: its action memory stays
        oo, ro, teo, tro, io = orc.o.env_step(act, streams.step_noise(k, 4).astype(np.float64))
        teo, tro = teo.astype(bool), tro.astype(bool)
        if arena_reset.any():
            idx = np.nonzero(arena_reset)[0]
            rz = np.zeros((20, n))
            rz[:, idx] = streams.autoreset_noise(episode[idx], envs=idx)
            p_, o_ = spawn(np.where(arena_reset, episode, 0).astype(np.uint32))
            sp[idx], so[idx] = p_[idx], o_[idx]
            orc.o.set_start(sp, so)
            orc.o.df_set_actions(arena_reset, mem)  # before the reset: its first observation shows the surviving past action
            obs_r = orc.o.env_reset(mask=arena_reset.astype(np.uint8), noise=rz)
            oo[arena_reset], ro[arena_reset], teo[arena_reset], tro[arena_reset] = obs_r[arena_reset], 0.0, False, False
            episode[idx] += 1
            agent_done[idx] = False
            n_resets += len(idx) // 2
        cmp = live & ~agent_done                  # agents still in self.agents before this call (re-spawned ones included)
        flip = cmp & ((teg != teo) | (trg != tro))
        n_flip += int(flip.sum())
        live &= ~flip
        # a flipped decision changes the episode of the WHOLE arena from then on
        live = (live.reshape(-1, 2).all(axis=1)[:, None] & np.ones((1, 2), dtype=bool)).reshape(-1)
        cmp &= live
        dmat = np.abs(og - oo) * cmp[:, None]
        if dmat.max() > worst_obs:
            wi, wc = np.unravel_index(np.argmax(dmat), dmat.shape)
            worst_where = (k, int(wi), int(wc), float(og[wi, wc]), float(oo[wi, wc]), bool(arena_reset[wi]), bool(agent_done[wi ^ 1]), int(episode[wi]))
        worst_obs = max(worst_obs, float(dmat.max()))
        worst_rew = max(worst_rew, float(np.abs(rg[cmp] - ro[cmp]).max()))
        n_hits += int((og[cmp][:, 18] < 1.0).sum())
        agent_done |= teg | trg
        agent_done[arena_reset & ~(teg | trg)] = False
        arena_reset = (agent_done.reshape(-1, 2).all(axis=1)[:, None] & np.ones((1, 2), dtype=bool)).reshape(-1)
    print(f"\n[timed-path parity, dogfight] {num_arenas} arenas x 2 x {steps} steps: {n_resets} arena autoresets, flips {n_flip}, hit observations {n_hits}; "
          f"max |obs| {worst_obs:.2e} at (step, agent, col, gpu, oracle, arena_reset_now, opponent_done, episode) = {worst_where}, max |reward| {worst_rew:.2e}")
    assert n_resets > num_arenas
    assert n_flip <= n // 200      # hit / range decisions at fp32 thresholds (lethal cone 1 rad, 150 m): tests/test_dogfight.py allows 2e-3 per step
    assert worst_obs < 2e-2 and worst_rew < 0.1
    env.close()


def test_hover_fused_rollout_matches_oracle():
    """The FUSED rollout (pfb_env_rollout(n >= 4): k_hover_rollout, 16 env steps per launch with the state in registers, on-device
    actions, autoreset from spares kept three ahead) pinned to the fp64 oracle on its own: the oracle is driven step by step with
    the replayed actions (bit-exact Philox replay) and noise, and resets on ITS OWN terminations with the replayed warm-up noise;
    at the end of every fused chunk the two must show the same step counters, flags, observations and rewards."""
    import torch

    from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverVecEnv

    n, seed, chunks = 16384, 77, [16, 16, 7, 16, 32, 16, 16]
    env = QuadXHoverVecEnv(num_envs=n, seed=seed)
    av = env.aviary
    streams = Streams(seed, n, noise_loc=4.0)
    model = build_model("quadx", "cf2x")
    orc = OracleEngine(model, hover_config(0, "quaternion", False, 3.0), n, np.tile([[0.0, 0.0, 1.0]], (n, 1)), np.zeros((n, 3)))
    env.reset()
    orc.o.env_reset(noise=streams.user_reset_noise(0).astype(np.float64))
    episode = np.ones(n, dtype=np.int64)
    done_prev = np.zeros(n, dtype=bool)
    steps_o = np.zeros(n, dtype=np.int64)
    k = 0
    worst_obs = worst_rew = 0.0
    n_resets = desync_max = 0
    for chunk in chunks:
        env.rollout(chunk)
        assert np.array_equal(av.setpoints.cpu().numpy(), streams.actions(k + chunk - 1))  # the last step's actions, written back
        for _ in range(chunk):
            act = streams.actions(k).astype(np.float64)
            oo, ro, teo, tro, io = orc.o.env_step(act, streams.step_noise(k).astype(np.float64))
            teo, tro = teo.astype(bool), tro.astype(bool)
            steps_o += 1
            if done_prev.any():
                idx = np.nonzero(done_prev)[0]
                rz = np.zeros((20, n))
                rz[:, idx] = streams.autoreset_noise(episode[idx], envs=idx)
                obs_r = orc.o.env_reset(mask=done_prev.astype(np.uint8), noise=rz)
                oo[done_prev], ro[done_prev], teo[done_prev], tro[done_prev] = obs_r[done_prev], 0.0, False, False
                episode[idx] += 1
                steps_o[idx] = 0
                n_resets += len(idx)
            done_prev = teo | tro
            k += 1
        og, rg = av.obs.double().cpu().numpy(), av.reward.double().cpu().numpy()
        teg, trg = av.term.cpu().numpy().astype(bool), av.trunc.cpu().numpy().astype(bool)
        same = (av.state_row_int(17).cpu().numpy() == steps_o) & (teg == teo) & (trg == tro)  # same reset history and outcome
        desync_max = max(desync_max, int((~same).sum()))
        worst_obs = max(worst_obs, float(np.abs(og[same] - oo[same]).max()))
        worst_rew = max(worst_rew, float(np.abs(rg[same] - ro[same]).max()))
    print(f"\n[fused rollout vs oracle] {n} envs x {k} steps in chunks {chunks}: {n_resets} oracle resets, envs off the oracle's reset schedule: "
          f"at most {desync_max}; max |obs| {worst_obs:.2e}, max |reward| {worst_rew:.2e}")
    assert n_resets > n
    assert desync_max <= n // 2000   # a termination within rounding of its threshold shifts that env's whole schedule
    assert worst_obs < 1e-4 and worst_rew < 1e-4
    env.close()
