"""The reset streams of the autoreset env kinds away from the shape test_timed_path_parity.py pins (a batch of whole 2048-env
tiles, env offset 0, a 32-bit seed, the seed given at construction):

* oracle pins at ragged batch sizes, with a 64-bit seed and an env offset whose batch straddles 2^32 (the high word of the
  Philox counter), QuadX-Hover in flight mode 1 where the warm-up spins the motors and so depends on its noise;
* reseed: a handle reseeded with s (after running on another seed, spares built ahead) must replay, bit for bit, what a
  fresh handle created with s does;
* ragged shard splits: two handles with matching env offsets must reproduce one handle bit for bit;
* the end-to-end entries (pfb_env_step_mapped, pfb_env_step_host) must produce what pfb_env_step produces.

Oracle batches stay at about a thousand envs so that the whole file runs in minutes."""
import numpy as np
import pytest

import lockstep
from engines import OracleEngine, build_model
from philox_replay import Streams

SEED = (1 << 40) + 0x5EED          # k1 = 256: the high key word is in play
OTHER = 0x1234_5678_9ABC
OFFSET = (1 << 32) - 500           # env ids 2^32 - 500 .. : the batch straddles the counter's high word
KINDS = ["hover", "qxwp", "fwwp", "rocket", "dogfight"]


def make_env(kind, n, seed, env_offset=0, **kw):
    """the env of each kind with episodes short enough that every env autoresets within ~60 steps"""
    if kind == "hover":
        from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverVecEnv

        return QuadXHoverVecEnv(num_envs=n, seed=seed, env_offset=env_offset, **{"max_duration_seconds": 1.0, **kw})
    if kind == "qxwp":
        from pyflyt_b200.gym_envs.quadx_waypoints_env import QuadXWaypointsVecEnv

        return QuadXWaypointsVecEnv(num_envs=n, seed=seed, env_offset=env_offset, goal_reach_distance=1.0, goal_reach_angle=3.0,
                                    **{"max_duration_seconds": 1.0, **kw})
    if kind == "fwwp":
        from pyflyt_b200.gym_envs.fixedwing_waypoints_env import FixedwingWaypointsVecEnv

        return FixedwingWaypointsVecEnv(num_envs=n, seed=seed, env_offset=env_offset, goal_reach_distance=25.0, **{"max_duration_seconds": 1.0, **kw})
    if kind == "rocket":
        from pyflyt_b200.gym_envs.rocket_landing_env import RocketLandingVecEnv

        return RocketLandingVecEnv(num_envs=n, seed=seed, env_offset=env_offset, ceiling=120.0, **{"max_duration_seconds": 1.0, **kw})
    if kind == "dogfight":
        from pyflyt_b200.pz_envs import MAFixedwingDogfightVecEnv

        return MAFixedwingDogfightVecEnv(num_arenas=n // 2, seed=seed, env_offset=env_offset, lethal_distance=150.0, lethal_angle_radians=1.0,
                                         damage_per_hit=0.05, **{"max_duration_seconds": 1.0, **kw})
    if kind == "mahover":
        from pyflyt_b200.pz_envs import MAQuadXHoverVecEnv

        return MAQuadXHoverVecEnv(num_arenas=n // 4, seed=seed, env_offset=env_offset, **{"max_duration_seconds": 1.0, **kw})
    raise ValueError(kind)


# state rows of the action history the multi-agent envs keep across a reset (the reference creates current_actions /
# past_actions in __init__ only): pfb_dogfight.cu DF_PAST / DF_CUR, pfb_quadx.cuh QM_CUR / QM_PAST
ACTION_HISTORY_ROWS = {"dogfight": range(32, 40), "mahover": range(60, 68)}


def scripted_actions(kind, n, rng):
    """float32 [n][action dim] inside each env's action box"""
    if kind in ("hover", "mahover"):
        a = rng.uniform([-np.pi, -np.pi, -np.pi, 0.0], [np.pi, np.pi, np.pi, 0.8], (n, 4))
    elif kind == "qxwp":
        a = rng.uniform([-1.0, -1.0, -1.0, 0.0], [1.0, 1.0, 1.0, 0.8], (n, 4))
    elif kind == "fwwp":
        a = rng.uniform(-1.0, 1.0, (n, 4)) * [0.5, 0.3, 0.3, 1.0]
    elif kind == "rocket":
        a = rng.uniform([-1, -1, -1, 0, 0, -1, -1], [1, 1, 1, 1, 1, 1, 1], (n, 7))
    else:
        a = np.clip(rng.uniform(-1, 1, (n, 4)) * 0.4 + np.array([0.0, 0.15, 0.0, 0.0]) * (np.arange(n) % 5 == 0)[:, None], -1, 1)
    return np.ascontiguousarray(a, dtype=np.float32)


def snapshot(env):
    """every output and the whole per-env state of a handle, on the host; warp-tiled state through state_row (the tile padding
    is not state)"""
    import torch

    torch.cuda.synchronize()
    av = env.aviary
    out = {"obs": av.obs.cpu().clone(), "reward": av.reward.cpu().clone(), "term": av.term.cpu().clone(), "trunc": av.trunc.cpu().clone(),
           "info": av.info_bits.cpu().clone(), "istate": av.istate_tensor.cpu().clone()}
    if av.tiled:
        out["state"] = torch.stack([av.state_row(r).cpu() for r in range(av.state_rows)])
    else:
        out["state"] = av.state_tensor.cpu().clone()
    if hasattr(env, "alive"):
        out["alive"] = env.alive.cpu().clone()
    return out


def assert_same(a, b, where):
    import torch

    for key in a:
        assert torch.equal(a[key], b[key]), (where, key)


# ---------------------------------------------------------------------------------------------------------------------------
# 1. oracle pins at the edges
def test_hover_mode1_warmup_depends_on_its_noise():
    """Guard against a vacuous pin: the first observation after a warm-up must depend on the warm-up's noise by far more than the
    1e-4 bar, or a wrong reset key would pass.  In mode 1 the warm-up holds vz = 0 with spinning motors; in mode 0 (thrust preset
    to -1) the two draws differ only by ~1e-3 in the velocity and motor columns."""
    from engines import hover_config

    n = 256
    st = Streams(SEED, n, env_offset=OFFSET)
    spread = {}
    for mode in (0, 1):
        obs = []
        for noise in (st.user_reset_noise(0), st.autoreset_noise(np.ones(n, dtype=np.int64))):
            orc = OracleEngine(build_model("quadx", "cf2x"), hover_config(mode), n, np.tile([[0.0, 0.0, 1.0]], (n, 1)), np.zeros((n, 3)))
            obs.append(orc.env_reset(noise.astype(np.float64)))
        spread[mode] = np.abs(obs[0] - obs[1]).max(axis=1)
    print(f"\n[warm-up noise sensitivity] per-env max |obs(draw a) - obs(draw b)|: mode 0 median {np.median(spread[0]):.2e}; "
          f"mode 1 min {spread[1].min():.2e}, median {np.median(spread[1]):.2e}, share > 1e-3 {(spread[1] > 1e-3).mean():.3f}")
    assert np.median(spread[1]) > 100 * 1e-4
    assert (spread[1] > 10 * 1e-4).mean() > 0.9


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1000, 33])
@pytest.mark.parametrize("path", ["step", "fused"])
def test_hover_mode1_matches_oracle_at_the_edges(n, path):
    """QuadX-Hover, mode 1 (angle setpoints and vz: random angles crash often, so many resets), a 64-bit seed, the batch
    straddling env id 2^32, a partial last warp tile (n = 1000: 8 lanes; n = 33: one lane); single-step launches with the noise
    dump and the RANDACT draws compared, and the fused rollout with its three-ahead spares."""
    offset = (1 << 32) - min(500, n // 2)
    env = make_env("hover", n, SEED, offset, flight_mode=1)
    # the mode-0 bar.  Measured single-step on an H100 (400 W power limit), no flips in either case:
    #   1 s episodes (used here): max 4.9e-5; per-env max quantiles 50 / 99 / 99.9 % 3.9e-6 / 2.3e-5 / 4.4e-5; fused: max 1.3e-5
    #   2 s episodes: max 1.6e-4; quantiles 4.5e-6 / 4.2e-5 / 1.4e-4, 3 envs of 1000 (and 1 of 33) above 1e-4.  Longer
    #   episodes let the attitude loop amplify rounding around the random angle setpoints; 1 s episodes keep the bar tight
    bar = 1e-4
    if path == "step":
        run = lockstep.hover_step(env, SEED, 100, env_offset=offset, obs_bar=bar)
    else:
        run = lockstep.hover_fused(env, SEED, [16, 16, 7, 16, 32, 16], env_offset=offset, obs_bar=bar)
    env.close()
    assert run.reset_obs < 1e-5, run.summary()
    if path == "step":
        assert run.worst_noise < 5e-4, run.summary()
    run.check(min_resets=n)
    assert run.extra["episodes"] >= 3, run.summary()  # some env is on its third episode: spares rotate through their buffers


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["qxwp", "fwwp", "rocket", "dogfight"])
def test_tail_kinds_match_oracle_at_the_edges(kind):
    """The tail-CTA kinds at a ragged batch (a partial last CTA: the obs_write_block row clamp; fewer CTAs than SMs: every tail
    CTA count), a 64-bit seed and the batch straddling env id 2^32; waypoints, drop poses and spawns replayed into the oracle."""
    n = 1034 if kind == "dogfight" else 1000  # 517 arenas
    if kind == "qxwp":
        env = make_env(kind, n, SEED, OFFSET, max_duration_seconds=2.0)
        run = lockstep.quadx_waypoints(env, SEED, 150, env_offset=OFFSET)
        bar0 = 1e-4
    elif kind == "fwwp":
        env = make_env(kind, n, SEED, OFFSET, max_duration_seconds=3.0)
        run = lockstep.fixedwing_waypoints(env, SEED, 150, env_offset=OFFSET)
        bar0 = 2e-3
    elif kind == "rocket":
        env = make_env(kind, n, SEED, OFFSET, max_duration_seconds=30.0)
        run = lockstep.rocket_landing(env, SEED, 200, env_offset=OFFSET)
        bar0 = 5e-3
    else:
        env = make_env(kind, n, SEED, OFFSET, max_duration_seconds=2.0)
        run = lockstep.dogfight(env, SEED, 150, env_offset=OFFSET)
        bar0 = 5e-3
    env.close()
    assert run.reset_obs < bar0, run.summary()
    run.check(min_resets=n // 2 if kind == "dogfight" else n)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hover", "fwwp"])
def test_second_user_reset_matches_oracle(kind):
    """A second full reset: its warm-up is keyed by user-reset number 1 (0x80000000 | 1), and each env's autoreset episode count
    continues from the first reset's spares (the first autoreset takes episode 2)."""
    n = 1000
    if kind == "hover":
        env = make_env(kind, n, SEED, OFFSET, flight_mode=1)
        env.reset()
        run = lockstep.hover_step(env, SEED, 60, env_offset=OFFSET, reset_seq=1, episode0=2)
        bar0 = 1e-5
    else:
        env = make_env(kind, n, SEED, OFFSET, max_duration_seconds=1.0)
        env.reset()
        run = lockstep.fixedwing_waypoints(env, SEED, 60, env_offset=OFFSET, reset_seq=1, episode0=2)
        bar0 = 2e-3
    env.close()
    assert run.reset_obs < bar0, run.summary()
    run.check(min_resets=n)


# ---------------------------------------------------------------------------------------------------------------------------
# 2. reseed
def _reseed_case(kind, via, mode=0, fused=False, n=1000, K=60):
    """a fresh handle with SEED against a handle that ran on OTHER (spares built, fused ones ahead; envs mid-episode) and was
    then reseeded with SEED and fully reset: K steps, bit for bit"""
    import torch

    kw = {"flight_mode": mode} if kind == "hover" else {}
    plan = [16, 16, 8, 16, 4] if fused else [1] * K  # Hover: env steps per rollout call

    def drive(env, reset):
        rng = np.random.default_rng(11)
        obs, _ = reset()
        shots = [snapshot(env)]
        if kind == "hover":
            for steps in plan:
                env.rollout(steps)  # on-device actions: keyed by (seed, env, step number), so both sides draw the same
                shots.append(snapshot(env))
        else:
            for _ in range(K):
                env.step(torch.as_tensor(scripted_actions(kind, env.aviary.num_drones, rng), device=env.device))
                shots.append(snapshot(env))
        return shots

    fresh = make_env(kind, n, SEED, **kw)
    want = drive(fresh, fresh.reset)
    assert int((fresh.aviary.step_counts.cpu() < sum(plan)).sum()) > 0  # the replayed calls include autoresets
    fresh.close()

    env = make_env(kind, n, OTHER, **kw)
    env.reset()
    rng = np.random.default_rng(5)
    if kind == "hover":
        env.rollout(16)
        env.rollout(3)
        env.rollout(17)  # fused launches: spares built up to three episodes ahead; 36 steps < the 40-step episodes
    else:
        for _ in range(45):
            env.step(torch.as_tensor(scripted_actions(kind, env.aviary.num_drones, rng), device=env.device))
    if kind in ACTION_HISTORY_ROWS:
        # the observation shows the past action, and a reset keeps both the current and the past one, as in the reference: a
        # reseed replays a fresh handle only from an empty history.  Zero actions until every agent's history is zero (an
        # agent needs two steps of its own; a re-spawned arena skips the call it is re-spawned on, a culled agent waits for
        # its arena's reset)
        zero = torch.zeros((env.aviary.num_drones, 4), device=env.device)
        for _ in range(200):
            env.step(zero)
            if not any(bool(env.aviary.state_row(r).any()) for r in ACTION_HISTORY_ROWS[kind]):
                break
        assert not any(bool(env.aviary.state_row(r).any()) for r in ACTION_HISTORY_ROWS[kind])
    torch.cuda.synchronize()
    mid = ~(env.aviary.term.bool() | env.aviary.trunc.bool())
    assert bool(mid.any())  # envs in the middle of an episode at the reseed

    if via == "aviary":
        def reset():
            env.aviary.reseed(SEED)
            return env.reset()
    else:
        def reset():
            return env.reset(seed=SEED)
    got = drive(env, reset)
    env.close()
    assert len(got) == len(want)
    for k, (a, b) in enumerate(zip(want, got)):
        if k == 0:  # reset() returns the observation and info; reward and the flags still hold the last step's
            a, b = ({key: v for key, v in x.items() if key not in ("reward", "term", "trunc")} for x in (a, b))
        assert_same(a, b, f"{kind} via {via}: call {k}")


@pytest.mark.gpu
@pytest.mark.parametrize("via", ["aviary", "vecenv"])
@pytest.mark.parametrize("kind", ["qxwp", "fwwp", "rocket", "dogfight", "mahover"])
def test_reseed_replays_a_fresh_handle(kind, via):
    """every tail-CTA kind, and MAQuadXHover (no spares: its arenas reset from the host with a mask)"""
    _reseed_case(kind, via, n=1034 if kind == "dogfight" else (1032 if kind == "mahover" else 1000))


@pytest.mark.gpu
@pytest.mark.parametrize("via", ["aviary", "vecenv"])
@pytest.mark.parametrize("mode,fused", [(0, False), (0, True), (1, False), (1, True)])
def test_hover_reseed_replays_a_fresh_handle(mode, fused, via):
    """mode 1: the warm-up depends on its noise, so a spare left from the old seed shows; fused: spares three episodes ahead"""
    _reseed_case("hover", via, mode=mode, fused=fused)


@pytest.mark.gpu
def test_reset_seed_with_mask_is_refused():
    import torch

    env = make_env("hover", 64, SEED)
    with pytest.raises(ValueError):
        env.reset(seed=1, mask=torch.ones(64, dtype=torch.uint8, device=env.device))
    env.close()


# ---------------------------------------------------------------------------------------------------------------------------
# 3. ragged shard split
@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_ragged_shard_split_equals_one_handle(kind):
    """one handle of n envs against two handles split at a point that is not a multiple of 32 (arena-aligned for the dogfight),
    env offsets base and base + split with the batch straddling 2^32: bit for bit, autoresets included"""
    import torch

    n, split = (1034, 502) if kind == "dogfight" else (1000, 397)
    base = (1 << 32) - 450
    whole = make_env(kind, n, SEED, base)
    parts = [make_env(kind, split, SEED, base), make_env(kind, n - split, SEED, base + split)]
    for e in [whole] + parts:
        e.reset()
    rng = np.random.default_rng(3)
    plan = [1, 1, 1, 16, 7, 1, 1, 16, 1, 5] if kind == "hover" else [1] * 60
    for k, steps in enumerate(plan):
        if kind == "hover":
            for e in [whole] + parts:
                e.rollout(steps)
        else:
            act = torch.as_tensor(scripted_actions(kind, n, rng), device=whole.device)
            whole.step(act)
            parts[0].step(act[:split].clone())
            parts[1].step(act[split:].clone())  # a fresh, 16-byte aligned buffer
        a, lo, hi = snapshot(whole), snapshot(parts[0]), snapshot(parts[1])
        for key in a:
            dim = 1 if key in ("state", "istate") else 0
            assert torch.equal(a[key], torch.cat([lo[key], hi[key]], dim=dim)), (kind, k, key)
    assert int(a["info"].numel()) == n
    for e in [whole] + parts:
        e.close()


# ---------------------------------------------------------------------------------------------------------------------------
# 4. mapped and host steps
@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["slab", "separate"])
@pytest.mark.parametrize("entry,kind,n", [("mapped", k, 1034 if k == "dogfight" else 1000) for k in KINDS] + [("mapped", "hover", 65536)]
                         + [("host", k, 1034 if k == "dogfight" else 1000) for k in KINDS if k != "hover"])
def test_end_to_end_entries_equal_device_step(entry, kind, n, layout):
    """pfb_env_step_mapped (the kernels read the pinned actions and write obs / reward / term / trunc into pinned host memory,
    with dynamic shared memory that spreads the launch over several waves) and pfb_env_step_host (copies around the launch)
    against pfb_env_step on a twin handle, 64 steps with autoresets: the outputs, info and state bit for bit"""
    import torch

    envs = [make_env(kind, n, SEED), make_env(kind, n, SEED)]
    for e in envs:
        e.reset()
    av, ref = envs[0].aviary, envs[1].aviary
    O = av.obs_dim
    if layout == "slab":
        slab = torch.zeros(av.out_slab_bytes(n, O), dtype=torch.uint8).pin_memory()
        bufs = av.slab_views(slab, n, O)
    else:
        bufs = (torch.zeros((n, O)).pin_memory(), torch.zeros(n).pin_memory(), torch.zeros(n, dtype=torch.uint8).pin_memory(),
                torch.zeros(n, dtype=torch.uint8).pin_memory())
    rng = np.random.default_rng(7)
    resets = 0
    for k in range(64):
        act = torch.from_numpy(scripted_actions(kind, n, rng)).pin_memory()
        (av.env_step_mapped if entry == "mapped" else av.env_step_host)(act, *bufs)
        ref.env_step(act.to(ref.device))
        torch.cuda.synchronize()
        obs, rew, te, tr = bufs
        assert torch.equal(obs, ref.obs.cpu()) and torch.equal(rew, ref.reward.cpu()), (k, "obs / reward")
        assert torch.equal(te, ref.term.cpu()) and torch.equal(tr, ref.trunc.cpu()), (k, "term / trunc")
        assert torch.equal(av.info_bits.cpu(), ref.info_bits.cpu()), (k, "info")
        resets += int((te | tr).sum())
    a, b = snapshot(envs[0]), snapshot(envs[1])
    assert torch.equal(a["state"], b["state"]) and torch.equal(a["istate"], b["istate"])
    assert resets > n // 2
    for e in envs:
        e.close()
