"""TEST INFRASTRUCTURE — lock-step drivers of the fp64 oracle for the autoreset env kinds.

Each driver runs one VecEnv handle with Philox noise and NEXT_STEP autoreset through spare post-reset states, and steps the
oracle alongside it with exactly what the kernel consumed: the replayed noise (tests/philox_replay.py), the same actions (the
replayed RANDACT draws where Streams has them, scripted ones otherwise) and the same reset schedule, each autoreset keyed by
the env's episode number.  They generalise the loops of tests/test_timed_path_parity.py to any batch size, 64-bit seed, env
offset (the global id of env 0), flight mode, first user-reset number (``reset_seq``: the count of earlier full
``env_reset`` calls since the handle was created or reseeded) and first autoreset episode number (``episode0``: a full
reset continues each env's episode count, so it is 1 + the number of episodes the env started since creation or reseed).

An env whose termination decision sits within fp32 rounding of its threshold takes the other branch on one side; from then on
the two follow different episodes, so it is dropped from the comparison and counted as a flip.  ``Run.check()`` holds the
flips, the "loose" envs and the worst differences to the per-kind bars of test_timed_path_parity.py; a flip budget never goes
below 2, so small batches are not held to a zero-flip bar.

Every driver takes an optional wind schedule ``{env step: AnalyticWind | None}``: each entry is registered on the handle's
Aviary and set on the oracle before that env step (the step's index in the driver's loop; entry 0 before ``env.reset()``),
so a wind can be present from the start, or registered, changed and cleared between autoresets.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from engines import OracleEngine, build_model
from philox_replay import Streams, philox4x32_10, unit_open


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float32).astype(np.float64)


def _host(av):
    return (av.obs.double().cpu().numpy(), av.reward.double().cpu().numpy(), av.term.cpu().numpy().astype(bool),
            av.trunc.cpu().numpy().astype(bool), av.info_bits.cpu().numpy())


@dataclass
class Run:
    """What one lock-step run saw, and the bars it is held to."""
    kind: str
    n: int
    obs_bar: float
    rew_bar: float
    flip_per: int                  # flip budget: max(2, n // flip_per)
    loose_frac: float = 0.0        # share of envs allowed outside the tight envelope (0: no envelope)
    live: np.ndarray = None
    loose: np.ndarray = None
    n_flip: int = 0
    n_resets: int = 0
    worst_obs: float = 0.0
    worst_rew: float = 0.0
    worst_noise: float = 0.0
    reset_obs: float = 0.0         # |gpu - oracle| of the observation after the user reset
    reached: int = 0
    extra: dict = field(default_factory=dict)
    env_worst: np.ndarray = None   # per env: the largest observation difference it showed while compared

    def __post_init__(self):
        self.live = np.ones(self.n, dtype=bool)
        self.loose = np.zeros(self.n, dtype=bool)
        self.env_worst = np.zeros(self.n)

    def flips(self, flip):
        flip = self.live & flip
        self.n_flip += int(flip.sum())
        self.live &= ~flip

    def compare(self, dobs, drew, cmp, loose_obs=None, loose_rew=None):
        """dobs [n] per-env max |obs difference|, drew [n]; cmp: the envs compared on this step"""
        self.env_worst = np.maximum(self.env_worst, np.where(cmp, dobs, 0.0))
        if cmp.any():
            self.worst_obs = max(self.worst_obs, float(dobs[cmp].max()))
            self.worst_rew = max(self.worst_rew, float(drew[cmp].max()))
        if loose_obs is not None:
            self.loose |= cmp & ((dobs > loose_obs) | (drew > loose_rew))

    def summary(self) -> str:
        return (f"[lockstep {self.kind}] n {self.n}: {self.n_resets} autoresets, flips {self.n_flip}, loose {int(self.loose.sum())}, "
                f"reached {self.reached}; user reset |obs| {self.reset_obs:.2e}, max |obs| {self.worst_obs:.2e}, max |reward| {self.worst_rew:.2e}, "
                f"max |noise dump - replay| {self.worst_noise:.2e}; per-env max |obs| quantiles 50/99/99.9 % "
                f"{np.quantile(self.env_worst, [0.5, 0.99, 0.999]).round(8).tolist()} {self.extra}")

    def check(self, min_resets: int):
        print("\n" + self.summary())
        assert self.n_resets >= min_resets, self.summary()
        assert self.n_flip <= max(2, self.n // self.flip_per), self.summary()
        if self.loose_frac:
            assert self.loose.mean() <= max(self.loose_frac, 2.0 / self.n), self.summary()
        assert self.worst_obs < self.obs_bar and self.worst_rew < self.rew_bar, self.summary()


def oracle_config(env):
    """the env's own PfbEnvConfig for the oracle, which runs no autoreset of its own (the drivers reset it) and draws no spawn
    poses (the drivers install the replayed ones)"""
    c = type(env.config).from_buffer_copy(env.config)
    c.autoreset, c.inline_reset, c.randomize_drop = 0, 0, 0
    return c


def _apply_wind(wind, k, env, orc):
    """the schedule's entry for env step k, if any, on the handle and on the oracle (whose set_wind refreshes the link air
    velocities, as the kernels derive them from the state in every substep)"""
    if wind and k in wind:
        env.aviary.register_wind_field(wind[k])
        orc.set_wind(wind[k])


def _autoreset_noise(streams, episode, idx, n):
    rz = np.zeros((20, n))
    rz[:, idx] = streams.autoreset_noise(episode[idx], envs=idx)
    return rz


# ---------------------------------------------------------------------------------------------------------- QuadX-Hover
def hover_oracle(env, n):
    return OracleEngine(build_model("quadx", "cf2x"), oracle_config(env), n, np.tile([[0.0, 0.0, 1.0]], (n, 1)), np.zeros((n, 3)))


def hover_step(env, seed: int, steps: int, *, env_offset: int = 0, reset_seq: int = 0, episode0: int = 1, obs_bar: float = 1e-4, wind: dict | None = None) -> Run:
    """Single-step launches (``rollout(1)``: on-device RANDACT actions, compared bit for bit with the replay), the kernel's noise
    dumped and compared with the replay, the oracle reset on the kernel's schedule."""
    import torch

    av, n, mode, ratio = env.aviary, env.num_envs, env.flight_mode, env.config.env_step_ratio
    run = Run("hover step", n, obs_bar, obs_bar, 4096)
    dump = torch.zeros((2 * ratio, n), dtype=torch.float32, device=av.device)  # two draws per Aviary step
    av.set_noise_dump(dump)
    streams = Streams(seed, n, env_offset=env_offset, noise_loc=4.0)
    orc = hover_oracle(env, n)
    _apply_wind(wind, 0, env, orc)
    obs_g, _ = env.reset()
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(reset_seq).astype(np.float64))
    run.reset_obs = float(np.abs(obs_g.double().cpu().numpy() - obs_o).max())
    episode = np.full(n, episode0, dtype=np.int64)
    done_prev = np.zeros(n, dtype=bool)
    for k in range(steps):
        if k:
            _apply_wind(wind, k, env, orc)
        env.rollout(1)
        act_g = av.setpoints.cpu().numpy()
        act = streams.actions(k, mode)
        assert np.array_equal(act_g, act), k
        og, rg, teg, trg, ig = _host(av)
        nz = streams.step_noise(k, ratio)
        oo, ro, teo, tro, io = orc.o.env_step(act.astype(np.float64), nz.astype(np.float64))
        teo, tro = teo.astype(bool), tro.astype(bool)
        if done_prev.any():
            idx = np.nonzero(done_prev)[0]
            obs_r = orc.o.env_reset(mask=done_prev.astype(np.uint8), noise=_autoreset_noise(streams, episode, idx, n))
            oo[done_prev], ro[done_prev], teo[done_prev], tro[done_prev], io[done_prev] = obs_r[done_prev], 0.0, False, False, 0
            episode[idx] += 1
            run.n_resets += len(idx)
        full = ~done_prev & ~(teg | trg)  # the envs that ran every Aviary step of the env step
        if full.any():
            run.worst_noise = max(run.worst_noise, float(np.abs(dump.cpu().numpy()[:, full] - nz[:, full]).max()))
        run.flips((teg != teo) | (trg != tro))
        assert np.array_equal(ig[run.live] & 3, io[run.live] & 3), k
        run.compare(np.abs(og - oo).max(axis=1), np.abs(rg - ro), run.live)
        done_prev = teg | trg
    av.set_noise_dump(None)
    run.extra["episodes"] = int(episode.max())
    return run


def hover_fused(env, seed: int, chunks, *, env_offset: int = 0, reset_seq: int = 0, episode0: int = 1, obs_bar: float = 1e-4, wind: dict | None = None) -> Run:
    """The fused rollout (chunks of >= 4 env steps: k_hover_rollout with spares kept three ahead): the oracle runs step by step
    on the replayed actions and noise and resets on its OWN terminations; at the end of every chunk the step counters, flags,
    observations and rewards must agree.  An env off the oracle's schedule counts as a flip."""
    av, n, mode = env.aviary, env.num_envs, env.flight_mode
    run = Run("hover fused", n, obs_bar, obs_bar, 2000)
    streams = Streams(seed, n, env_offset=env_offset, noise_loc=4.0)
    orc = hover_oracle(env, n)
    _apply_wind(wind, 0, env, orc)
    obs_g, _ = env.reset()
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(reset_seq).astype(np.float64))
    run.reset_obs = float(np.abs(obs_g.double().cpu().numpy() - obs_o).max())
    episode = np.full(n, episode0, dtype=np.int64)
    done_prev = np.zeros(n, dtype=bool)
    steps_o = np.zeros(n, dtype=np.int64)
    k = 0
    assert not wind or set(wind) <= {0, *np.cumsum(chunks)[:-1].tolist()}, "the wind can only change between fused launches"
    for chunk in chunks:
        if k:
            _apply_wind(wind, k, env, orc)
        env.rollout(chunk)
        assert np.array_equal(av.setpoints.cpu().numpy(), streams.actions(k + chunk - 1, mode))  # the last step's actions, written back
        for _ in range(chunk):
            oo, ro, teo, tro, io = orc.o.env_step(streams.actions(k, mode).astype(np.float64), streams.step_noise(k).astype(np.float64))
            teo, tro = teo.astype(bool), tro.astype(bool)
            steps_o += 1
            if done_prev.any():
                idx = np.nonzero(done_prev)[0]
                obs_r = orc.o.env_reset(mask=done_prev.astype(np.uint8), noise=_autoreset_noise(streams, episode, idx, n))
                oo[done_prev], ro[done_prev], teo[done_prev], tro[done_prev] = obs_r[done_prev], 0.0, False, False
                episode[idx] += 1
                steps_o[idx] = 0
                run.n_resets += len(idx)
            done_prev = teo | tro
            k += 1
        og, rg, teg, trg, _ = _host(av)
        run.flips((av.state_row_int(17).cpu().numpy() != steps_o) | (teg != teo) | (trg != tro))
        run.compare(np.abs(og - oo).max(axis=1), np.abs(rg - ro), run.live)
    run.extra["episodes"] = int(episode.max())
    return run


# ------------------------------------------------------------------------------------------------------- QuadX-Waypoints
def quadx_waypoints(env, seed: int, steps: int, *, env_offset: int = 0, reset_seq: int = 0, episode0: int = 1, rng_seed: int = 5, wind: dict | None = None) -> Run:
    """Scripted actions; device-drawn waypoints (and yaw targets) replayed into the oracle."""
    import torch

    av, n, c = env.aviary, env.num_envs, env.config
    mode, yaw, T, dome = c.flight_mode, bool(c.use_yaw_targets), c.num_targets, c.flight_dome_size
    if mode == 7:  # the reference's z-velocity PID limit-cycles (DESIGN 5): a position envelope
        run = Run("quadx-waypoints", n, 2e-2, 0.5, 500, loose_frac=5e-3)
    else:
        run = Run("quadx-waypoints", n, 5e-4, 5e-3, 500)
    streams = Streams(seed, n, env_offset=env_offset, noise_loc=4.0)
    orc = OracleEngine(build_model("quadx", "cf2x"), oracle_config(env), n, np.tile([[0.0, 0.0, 1.0]], (n, 1)), np.zeros((n, 3)))
    _apply_wind(wind, 0, env, orc)
    obs_g, _ = env.reset()
    tg = streams.waypoint_targets(0x80000000 | reset_seq, T, dome, min_height=0.1, yaw=yaw)
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(reset_seq).astype(np.float64), targets=tg.astype(np.float64).reshape(n, -1))
    run.reset_obs = float(np.abs(obs_g.double().cpu().numpy() - obs_o).max())
    rng = np.random.default_rng(rng_seed)
    episode = np.full(n, episode0, dtype=np.int64)
    done_prev = np.zeros(n, dtype=bool)
    for k in range(steps):
        if k:
            _apply_wind(wind, k, env, orc)
        if mode == 7:
            act = _f(rng.uniform([-2.0, -2.0, -1.0, 0.5], [2.0, 2.0, 1.0, 3.0], (n, 4)))
        else:
            act = _f(rng.uniform([-1.0, -1.0, -1.0, 0.0], [1.0, 1.0, 1.0, 0.8], (n, 4)))
        env.step(torch.as_tensor(act, dtype=torch.float32, device=av.device))
        og, rg, teg, trg, ig = _host(av)
        oo, ro, teo, tro, io = orc.o.env_step(act, streams.step_noise(k, 4).astype(np.float64))
        teo, tro = teo.astype(bool), tro.astype(bool)
        if done_prev.any():
            idx = np.nonzero(done_prev)[0]
            tgr = np.zeros((n, T, 4 if yaw else 3))
            tgr[idx] = streams.waypoint_targets(episode[idx], T, dome, min_height=0.1, envs=idx, yaw=yaw)
            obs_r = orc.o.env_reset(mask=done_prev.astype(np.uint8), noise=_autoreset_noise(streams, episode, idx, n), targets=tgr.reshape(n, -1))
            oo[done_prev], ro[done_prev], teo[done_prev], tro[done_prev], io[done_prev] = obs_r[done_prev], 0.0, False, False, 0
            episode[idx] += 1
            run.n_resets += len(idx)
        run.flips((teg != teo) | (trg != tro) | ((ig >> 3) != (io >> 3)))
        cols = slice(10, 13) if mode == 7 else slice(None)
        run.compare(np.abs(og[:, cols] - oo[:, cols]).max(axis=1), np.abs(rg - ro), run.live, 1e-3, 5e-2)
        run.reached = max(run.reached, int((ig >> 3).max()))
        done_prev = teg | trg
    return run


# ---------------------------------------------------------------------------------------------------- Fixedwing-Waypoints
def fixedwing_waypoints(env, seed: int, steps: int, *, env_offset: int = 0, reset_seq: int = 0, episode0: int = 1, obs_bar: float = 5e-3,
                        wind: dict | None = None) -> Run:
    """On-device RANDACT actions (U(-1, 1)^4, compared bit for bit with the replay on every env that stepped); device-drawn
    waypoints replayed into the oracle."""
    av, n, T, dome = env.aviary, env.num_envs, env.config.num_targets, env.config.flight_dome_size
    run = Run("fixedwing-waypoints", n, obs_bar, 5e-3, 1000)  # target deltas are O(100 m) fp32 numbers
    streams = Streams(seed, n, env_offset=env_offset, noise_loc=1.0)
    orc = OracleEngine(build_model("fixedwing", "fixedwing"), oracle_config(env), n, np.tile([[0.0, 0.0, 10.0]], (n, 1)), np.zeros((n, 3)))
    _apply_wind(wind, 0, env, orc)
    obs_g, _ = env.reset()
    tg = streams.waypoint_targets(0x80000000 | reset_seq, T, dome, min_height=0.5)
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(reset_seq).astype(np.float64), targets=tg.astype(np.float64).reshape(n, -1))
    run.reset_obs = float(np.abs(obs_g.double().cpu().numpy() - obs_o).max())
    episode = np.full(n, episode0, dtype=np.int64)
    done_prev = np.zeros(n, dtype=bool)
    for k in range(steps):
        if k:
            _apply_wind(wind, k, env, orc)
        env.rollout(1)
        act = streams.uniform_actions(k)
        assert np.array_equal(av.setpoints.cpu().numpy()[~done_prev], act[~done_prev]), k  # a resetting env draws no action
        og, rg, teg, trg, ig = _host(av)
        oo, ro, teo, tro, io = orc.o.env_step(act.astype(np.float64), streams.step_noise(k, 4).astype(np.float64))
        teo, tro = teo.astype(bool), tro.astype(bool)
        if done_prev.any():
            idx = np.nonzero(done_prev)[0]
            tgr = np.zeros((n, T, 3))
            tgr[idx] = streams.waypoint_targets(episode[idx], T, dome, min_height=0.5, envs=idx)
            obs_r = orc.o.env_reset(mask=done_prev.astype(np.uint8), noise=_autoreset_noise(streams, episode, idx, n), targets=tgr.reshape(n, -1))
            oo[done_prev], ro[done_prev], teo[done_prev], tro[done_prev], io[done_prev] = obs_r[done_prev], 0.0, False, False, 0
            episode[idx] += 1
            run.n_resets += len(idx)
        run.flips((teg != teo) | (trg != tro) | ((ig >> 3) != (io >> 3)))
        run.compare(np.abs(og - oo).max(axis=1), np.abs(rg - ro), run.live)
        run.reached = max(run.reached, int((ig >> 3).max()))
        done_prev = teg | trg
    return run


# --------------------------------------------------------------------------------------------------------- Rocket-Landing
def rocket_landing(env, seed: int, steps: int, *, env_offset: int = 0, reset_seq: int = 0, episode0: int = 1, rng_seed: int = 3, wind: dict | None = None) -> Run:
    """Scripted actions; device-drawn randomised drops replayed into the oracle.  The crash step's observation and reward stay
    out of the comparison (a stiff impulse iteration on an 80 m/s impact: see test_timed_path_parity.py); envs that carry a
    stall-branch offset are counted as loose."""
    import torch

    av, n, ceiling = env.aviary, env.num_envs, env.config.ceiling
    run = Run("rocket-landing", n, 0.1, 0.5, 500, loose_frac=1e-3)
    streams = Streams(seed, n, env_offset=env_offset, noise_loc=1.0)
    sp, so = streams.drop_poses(0x80000000 | reset_seq, ceiling, 200.0)
    sp, so = sp.astype(np.float64), so.astype(np.float64)
    orc = OracleEngine(build_model("rocket", "rocket", starting_fuel_ratio=0.05), oracle_config(env), n, sp, so)
    _apply_wind(wind, 0, env, orc)
    obs_g, _ = env.reset()
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(reset_seq).astype(np.float64))
    run.reset_obs = float(np.abs(obs_g.double().cpu().numpy() - obs_o).max())
    rng = np.random.default_rng(rng_seed)
    episode = np.full(n, episode0, dtype=np.int64)
    done_prev = np.zeros(n, dtype=bool)
    for k in range(steps):
        if k:
            _apply_wind(wind, k, env, orc)
        act = _f(rng.uniform([-1, -1, -1, 0, 0, -1, -1], [1, 1, 1, 1, 1, 1, 1], (n, 7)))
        env.step(torch.as_tensor(act, dtype=torch.float32, device=av.device))
        og, rg, teg, trg, ig = _host(av)
        oo, ro, teo, tro, io = orc.o.env_step(act, streams.step_noise(k, 3).astype(np.float64))
        teo, tro = teo.astype(bool), tro.astype(bool)
        if done_prev.any():
            idx = np.nonzero(done_prev)[0]
            sp[idx], so[idx] = streams.drop_poses(episode[idx], ceiling, 200.0, envs=idx)
            orc.o.set_start(sp, so)
            obs_r = orc.o.env_reset(mask=done_prev.astype(np.uint8), noise=_autoreset_noise(streams, episode, idx, n))
            oo[done_prev], ro[done_prev], teo[done_prev], tro[done_prev], io[done_prev] = obs_r[done_prev], 0.0, False, False, 0
            episode[idx] += 1
            run.n_resets += len(idx)
        run.flips((teg != teo) | (trg != tro) | ((ig & 7) != (io & 7)))
        cmp = run.live & ((ig & 2) == 0)
        run.compare(np.abs(og - oo).max(axis=1), np.abs(rg - ro), cmp, 5e-3, 2e-2)
        done_prev = teg | trg
    return run


# ------------------------------------------------------------------------------------------------------------- Dogfight
def dogfight_spawns(streams: Streams, seq, rmin=10.0, rmax=50.0, A=2):
    """df_reset_agent's random spawn (pfb_dogfight.cu): one base angle per arena from the stream of the arena's first agent
    (tag 6, word 0), radius / height / heading jitter per agent (tag 6 | 1); [n][3] positions and [n][3] orientations"""
    n = streams.n
    li = np.arange(n) % A
    first = np.arange(n) - li
    seq = np.broadcast_to(np.asarray(seq, dtype=np.uint32), (n,))
    a = philox4x32_10(streams.env_lo[first], streams.env_hi[first], seq, np.uint32(6 << 24), streams.k0, streams.k1)
    b = philox4x32_10(streams.env_lo, streams.env_hi, seq, np.uint32((6 << 24) | 1), streams.k0, streams.k1)
    two_pi = np.float32(6.28318530717958647692)
    rad = (two_pi / np.float32(A)) * li.astype(np.float32) + two_pi * unit_open(a[0])
    radius = np.float32(rmin) + np.float32(rmax - rmin) * unit_open(b[0])
    height = np.float32(rmin) + np.float32(rmax - rmin) * unit_open(b[1])
    yaw = rad + unit_open(b[2]) * np.float32(0.39269908169872414)
    pos = np.stack([radius * np.cos(rad), radius * np.sin(rad), height], axis=1)
    orn = np.zeros((n, 3))
    orn[:, 2] = yaw
    return _f(pos), _f(orn)


def dogfight(env, seed: int, steps: int, *, env_offset: int = 0, reset_seq: int = 0, episode0: int = 1, rng_seed: int = 8, wind: dict | None = None) -> Run:
    """1-vs-1 arenas, scripted actions, device-drawn spawns replayed into the oracle; an arena is re-spawned once both of its
    agents have left, and a flipped decision drops the whole arena."""
    import torch

    av, n = env.aviary, env.num_agents
    run = Run("dogfight", n, 2e-2, 0.1, 200)
    streams = Streams(seed, n, env_offset=env_offset, noise_loc=1.0)
    sp, so = dogfight_spawns(streams, 0x80000000 | reset_seq)
    orc = OracleEngine(build_model("fixedwing", "acrowing"), oracle_config(env), n, sp, so)
    _apply_wind(wind, 0, env, orc)
    obs_g, _ = env.reset()
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(reset_seq).astype(np.float64))
    run.reset_obs = float(np.abs(obs_g.double().cpu().numpy() - obs_o).max())
    rng = np.random.default_rng(rng_seed)
    episode = np.full(n, episode0, dtype=np.int64)   # per agent, arena-uniform
    agent_done = np.zeros(n, dtype=bool)   # left self.agents in the current episode
    arena_reset = np.zeros(n, dtype=bool)  # per agent: its arena is re-spawned on this call
    pairs = lambda m: (m.reshape(-1, 2).all(axis=1)[:, None] & np.ones((1, 2), dtype=bool)).reshape(-1)  # noqa: E731
    for k in range(steps):
        if k:
            _apply_wind(wind, k, env, orc)
        act = _f(np.clip(rng.uniform(-1, 1, (n, 4)) * 0.4 + np.array([0.0, 0.15, 0.0, 0.0]) * (np.arange(n) % 5 == 0)[:, None], -1, 1))
        env.step(torch.as_tensor(act, dtype=torch.float32, device=av.device))
        og, rg, teg, trg, _ = _host(av)
        mem = orc.o.df_get_actions() if arena_reset.any() else None  # a re-spawned arena is not stepped on this call
        oo, ro, teo, tro, _ = orc.o.env_step(act, streams.step_noise(k, 4).astype(np.float64))
        teo, tro = teo.astype(bool), tro.astype(bool)
        if arena_reset.any():
            idx = np.nonzero(arena_reset)[0]
            p_, o_ = dogfight_spawns(streams, np.where(arena_reset, episode, 0).astype(np.uint32))
            sp[idx], so[idx] = p_[idx], o_[idx]
            orc.o.set_start(sp, so)
            orc.o.df_set_actions(arena_reset, mem)
            obs_r = orc.o.env_reset(mask=arena_reset.astype(np.uint8), noise=_autoreset_noise(streams, episode, idx, n))
            oo[arena_reset], ro[arena_reset], teo[arena_reset], tro[arena_reset] = obs_r[arena_reset], 0.0, False, False
            episode[idx] += 1
            agent_done[idx] = False
            run.n_resets += len(idx) // 2
        cmp = ~agent_done
        run.flips(cmp & ((teg != teo) | (trg != tro)))
        run.live = pairs(run.live)  # a flipped decision changes the episode of the whole arena
        cmp &= run.live
        run.compare(np.abs(og - oo).max(axis=1), np.abs(rg - ro), cmp)
        agent_done |= teg | trg
        agent_done[arena_reset & ~(teg | trg)] = False
        arena_reset = pairs(agent_done)
    return run
