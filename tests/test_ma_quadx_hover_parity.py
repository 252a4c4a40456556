"""MAQuadXHover on its timed path (k_hover_step<MODE, ..., MA = true> with Philox noise, k_hover_reset for the masked arena
resets of MAQuadXHoverVecEnv's SAME_STEP autoreset) pinned to the fp64 oracle.

``Arenas`` restates the reference's PettingZoo parallel API (ma_quadx_base_env.py:309-372) in numpy on top of the oracle's
per-agent env: an agent leaves ``self.agents`` once it terminates or truncates, the culled agents are stepped with a zero
action and have no reward, and an arena is reset with a mask once all of its agents are done.  It does not import
pyflyt_b200.pz_envs: the torch bookkeeping there is under test as well.  It is first checked against the unmodified reference
(the mahover_* fixtures), then it judges the CUDA env, driven with the noise the kernels drew (tests/philox_replay.py):

* every step's reset call draws its warm-up noise from seq = 0x80000000 | reset_seq, and MAQuadXHoverVecEnv.step makes that
  call on every step, even when no arena is done, so reset_seq counts steps;
* the action memory (QM_CUR / QM_PAST) survives a reset, so the first observation of an episode shows the action of the
  previous episode's second-to-last step;
* the euler observation row of 23 floats makes a ragged last tile whose byte count is not a multiple of 16 (the per-float
  store loop of k_hover_step) whenever the agent count is not a multiple of 4;
* agent rates of 120, 60, 24 and 10 Hz (env_step_ratio 1, 2, 5, 12) cross the Philox pair and prefetch boundaries of
  PhiloxNoise; QuadX-Hover's timed path is pinned at the same rates.
"""
import glob
import os

import numpy as np
import pytest

from engines import GOLDEN, OracleEngine, build_model, fixture_agent_hz, load_golden, ma_hover_config
from philox_replay import Streams

FIX = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "mahover_*.npz")))
SEED = (1 << 40) + 0x5EED  # k1 = 256: the high key word is in play
GPU_BAR = 1e-4             # the obs / reward bar of the Hover timed-path pin


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float32).astype(np.float64)


class Arenas:
    """``num_arenas`` arenas of ``len(start_pos)`` agents on the fp64 oracle, with the arena bookkeeping of the reference's
    PettingZoo env and MAQuadXHoverVecEnv's SAME_STEP autoreset.  Noise comes from ``streams`` unless it is passed in."""

    def __init__(self, cfg, start_pos, start_orn, num_arenas, streams=None):
        self.A, self.G = len(start_pos), int(num_arenas)
        self.n = self.A * self.G
        self.ratio, self.warmup = int(cfg.env_step_ratio), int(cfg.warmup_steps)
        sp, so = np.tile(start_pos, (self.G, 1)), np.tile(start_orn, (self.G, 1))
        self.orc = OracleEngine(build_model("quadx", "cf2x"), cfg, self.n, sp, so).o
        self.streams = streams
        self.alive = np.ones(self.n, dtype=bool)
        self.reset_seq = 0  # pfb_env_reset calls so far: the key of the next reset's warm-up noise
        self.step_seq = 0   # env steps so far: the key of the next step's motor noise
        self.last_noise = None

    def reset(self, noise=None):
        """env.reset(): every arena"""
        if noise is None:
            noise = self.streams.user_reset_noise(self.reset_seq, self.warmup)
        self.reset_seq += 1
        self.alive[:] = True
        return self.orc.env_reset(noise=np.asarray(noise, dtype=np.float64))

    def reset_noise(self, seq, idx):
        """[warm-up draws][n] with the columns of the agents ``idx`` filled from the reset stream ``seq``"""
        rz = np.zeros((2 * self.warmup, self.n))
        rz[:, idx] = self.streams.user_reset_noise(seq, self.warmup, envs=idx)
        return rz

    def step(self, actions, noise=None, reset_noise=None, autoreset=True):
        """One MAQuadXHoverVecEnv.step.  ``reset_noise(seq, idx)`` -> [warm-up draws][n] (default: the reset stream ``seq``).
        Returns obs, reward, term, trunc, info bits and a dict with ``was_alive``, ``alive``, ``reset`` and ``final_obs``."""
        if noise is None:
            noise = self.streams.step_noise(self.step_seq, self.ratio)
        self.step_seq += 1
        self.last_noise = noise
        was_alive = self.alive.copy()
        act = np.asarray(actions, dtype=np.float64) * was_alive[:, None]  # current_actions *= 0 for the culled agents
        obs, rew, te, tr, info = self.orc.env_step(act, np.asarray(noise, dtype=np.float64))
        rew = np.where(was_alive, rew, 0.0)
        term = te.astype(bool) | ~was_alive
        trunc = tr.astype(bool) & was_alive
        self.alive &= ~(term | trunc)  # cull for the next round (ma_quadx_base_env.py:365-370)
        mask = np.zeros(self.n, dtype=bool)
        final_obs = obs.copy()
        if autoreset:
            mask = np.repeat(~self.alive.reshape(self.G, self.A).any(axis=1), self.A)
            seq = self.reset_seq
            self.reset_seq += 1  # the reset call is made on every step, with an empty mask too
            if mask.any():
                idx = np.nonzero(mask)[0]
                rz = self.reset_noise(seq, idx) if reset_noise is None else reset_noise(seq, idx)
                obs_r = self.orc.env_reset(mask=mask.astype(np.uint8), noise=rz)
                obs = np.where(mask[:, None], obs_r, obs)
            self.alive |= mask
        return obs, rew, term, trunc, info, dict(was_alive=was_alive, alive=self.alive.copy(), reset=mask, final_obs=final_obs)


# ---------------------------------------------------------------------------------------------------------------------------
# 1. the harness against the reference
def test_fixtures_cover_the_agent_rates():
    rates = {fixture_agent_hz(load_golden(name)) for name in FIX}
    assert {40, 120, 24} <= rates, rates


@pytest.mark.parametrize("name", FIX)
def test_harness_reproduces_reference(name):
    """The harness decides who is alive and when an arena resets; it must reproduce the fixture's alive / term / trunc sequences
    and episode boundaries, with the bars of test_ma_quadx_hover.py::test_oracle_reproduces_reference."""
    g = load_golden(name)
    A, E = int(g["n_agents"]), int(g["n_episodes"])
    cfg = ma_hover_config(int(g["flight_mode"]), str(g["angle_representation"]), bool(g["sparse"]), float(g["dome"]), fixture_agent_hz(g),
                          float(g["max_duration_seconds"]))
    har = Arenas(cfg, g["start_pos"], g["start_orn"], 1)
    obs = har.reset(g["ep0_reset_noise"].reshape(-1, A))
    worst_obs, worst_rew = float(np.abs(obs - g["ep0_reset_obs"]).max()), 0.0
    for k in range(E):
        T = len(g[f"ep{k}_actions"])
        for i in range(T):
            alive = g[f"ep{k}_alive"][i]
            assert np.array_equal(har.alive, alive), (k, i)

            def next_episode_noise(seq, idx):  # (the last recorded episode may end with the run: its successor is not recorded)
                return g[f"ep{k + 1}_reset_noise"].reshape(-1, A) if k + 1 < E else np.zeros((2 * har.warmup, A))

            ob, r, te, tr, _, ex = har.step(g[f"ep{k}_actions"][i], g[f"ep{k}_noise"][i].reshape(-1, A), next_episode_noise)
            assert np.array_equal(te, g[f"ep{k}_term"][i]) and np.array_equal(tr, g[f"ep{k}_trunc"][i]), (k, i)
            # an episode ends once all of its agents are done, and the next one starts in the same step
            assert ex["reset"].all() or not ex["reset"].any()
            if k + 1 < E:
                assert bool(ex["reset"].any()) == (i == T - 1), (k, i)
            else:
                assert not ex["reset"].any() or i == T - 1, (k, i)
            worst_obs = max(worst_obs, float(np.abs(ex["final_obs"][alive] - g[f"ep{k}_obs"][i][alive]).max()))
            worst_rew = max(worst_rew, float(np.abs(r[alive] - g[f"ep{k}_reward"][i][alive]).max()))
            assert (r[~alive] == 0).all()
            if ex["reset"].any() and k + 1 < E:
                worst_obs = max(worst_obs, float(np.abs(ob - g[f"ep{k + 1}_reset_obs"]).max()))
        if k + 1 < E:
            assert har.alive.all()
    assert worst_obs < 1e-7 and worst_rew < 1e-6, (worst_obs, worst_rew)


# ---------------------------------------------------------------------------------------------------------------------------
# 2. vacuity guards: the first observation after a masked reset depends on the reset key and on the action memory
def test_masked_reset_depends_on_its_key_and_the_action_memory():
    """In mode 1 the warm-up holds vz = 0 with spinning motors, so its observation depends on its noise.  A wrong reset key,
    a cleared past action or swapped current / past actions must move the first observation after a masked reset by more than
    100 x the bar the GPU tests below hold it to, or the pin would not see them."""
    G, A = 64, 4
    start = np.array([[-1.0, -1.0, 1.0], [1.0, -1.0, 1.0], [-1.0, 1.0, 1.0], [1.0, 1.0, 1.0]])
    streams = Streams(SEED, G * A, env_offset=(1 << 32) - 100)
    rng = np.random.default_rng(4)
    acts = [_f(rng.uniform([-0.3, -0.3, -1.0, -0.5], [0.3, 0.3, 1.0, 0.5], (G * A, 4))) for _ in range(3)]

    def first_obs(variant):
        har = Arenas(ma_hover_config(flight_mode=1), start, np.zeros_like(start), G, streams)
        har.reset()
        for a in acts:
            har.step(a, autoreset=False)
        assert har.alive.all()
        seq = har.reset_seq + {"key-1": -1, "key+1": 1}.get(variant, 0)
        mem = har.orc.df_get_actions()  # past | current
        if variant == "cleared":
            mem[:, :4] = 0.0
        elif variant == "swapped":
            mem = np.concatenate([mem[:, 4:], mem[:, :4]], axis=1)
        har.orc.df_set_actions(None, mem)
        mask = np.ones(har.n, dtype=np.uint8)
        return har.orc.env_reset(mask=mask, noise=har.reset_noise(seq, np.arange(har.n)))

    base = first_obs("kept")
    past = slice(17, 21)  # quaternion row: ang_vel 3, quaternion 4, lin_vel 3, lin_pos 3, throttle 4, past action 4, start 3
    assert np.allclose(base[:, past], acts[-2]), "the first observation shows the second-to-last action"
    spread = {v: np.abs(first_obs(v) - base).max(axis=1) for v in ("key-1", "key+1", "cleared", "swapped")}
    print("\n[masked-reset sensitivity] per-agent max |obs(variant) - obs(kept)|: "
          + ", ".join(f"{v} min {s.min():.2e} median {np.median(s):.2e}" for v, s in spread.items()))
    for v in ("key-1", "key+1"):
        assert np.median(spread[v]) > 100 * GPU_BAR and (spread[v] > 10 * GPU_BAR).mean() > 0.9, v
    for v in ("cleared", "swapped"):
        assert spread[v].min() > 100 * GPU_BAR, v


# ---------------------------------------------------------------------------------------------------------------------------
# 3. the CUDA env against the harness
def _host(x):
    return x.double().cpu().numpy() if x.is_floating_point() else x.cpu().numpy()


def lockstep_ma(env, start_pos, seed, steps, act_fn, *, env_offset=0, rng_seed=0, cols=None, loose_obs=None, loose_rew=None):
    """Drives ``env`` (a fresh MAQuadXHoverVecEnv with Philox noise and autoreset) and the harness with the same actions, the
    replayed noise and each side's own alive / reset decisions, and compares every output on every step.  A termination or
    truncation that flips within rounding changes the arena's whole schedule: the arena is dropped and counted, as it is when
    the Aviary step in which an agent first leaves the dome or touches the floor differs (the reward then differs by a whole
    -100 penalty while both sides terminate).  The observation buffer is filled with NaN before every step, so a value the
    kernels did not write shows.  ``cols``: the observation columns held to the bar (None: all); ``loose_obs`` / ``loose_rew``: the tight envelope whose outliers are
    counted per agent."""
    import torch

    av = env.aviary
    G, A, n = env.num_arenas, env.agents_per_arena, env.num_agents
    ratio = int(env.config.env_step_ratio)
    cfg = type(env.config).from_buffer_copy(env.config)
    streams = Streams(seed, n, env_offset=env_offset, noise_loc=4.0)
    har = Arenas(cfg, np.asarray(start_pos, dtype=np.float64), np.zeros((A, 3)), G, streams)
    dump = torch.zeros((2 * ratio, n), dtype=torch.float32, device=av.device)  # two draws per Aviary step
    av.set_noise_dump(dump)
    obs_g, info = env.reset()
    obs_o = har.reset()
    s = dict(reset_obs=float(np.abs(_host(obs_g) - obs_o).max()), obs=0.0, rew=0.0, noise=0.0, final=0.0, rew_abs=0.0, flips=0, resets=0, culled=0,
             where=None, flip_events=[])
    assert s["reset_obs"] < GPU_BAR, s
    live_arena = np.ones(G, dtype=bool)
    loose = np.zeros(n, dtype=bool)
    alive_prev_g = np.ones(n, dtype=bool)
    agent_worst = np.zeros(n)
    cols = slice(None) if cols is None else cols
    rng = np.random.default_rng(rng_seed)
    for k in range(steps):
        act = _f(act_fn(rng, n))
        av.obs.fill_(float("nan"))
        og, rg, teg, trg, info = env.step(torch.as_tensor(act, dtype=torch.float32, device=av.device))
        og, rg, teg, trg = _host(og), _host(rg), _host(teg), _host(trg)
        ig, alive_g, reset_g, final_g = _host(av.info_bits), _host(info["alive"]), _host(info["reset"]), _host(info["final_obs"])
        oo, ro, teo, tro, io, ex = har.step(act)
        assert np.isfinite(og).all(), (k, np.nonzero(~np.isfinite(og)))
        # the GPU's own bookkeeping: a culled agent has reward exactly 0 and term set
        culled = ~alive_prev_g
        assert (rg[culled] == 0.0).all() and teg[culled].all() and not trg[culled].any(), k
        s["culled"] += int(culled.sum())
        # the kernel's draws vs the replay (every agent runs every Aviary step of every env step)
        s["noise"] = max(s["noise"], float(np.abs(_host(dump) - har.last_noise).max()))
        # a flipped decision drops the whole arena
        wa = ex["was_alive"]
        flip_agent = wa & ((teg != teo) | (trg != tro) | (np.abs(rg - ro) > 50.0)) & np.repeat(live_arena, A)
        for w in np.nonzero(flip_agent)[0][: max(0, 3 - len(s["flip_events"]))]:
            p = ex["final_obs"][w, 9:12] if har.orc.obs_dim == 23 else ex["final_obs"][w, 10:13]  # the oracle's position
            s["flip_events"].append(dict(step=k, agent=int(w), term=(bool(teg[w]), bool(teo[w])), trunc=(bool(trg[w]), bool(tro[w])),
                                         reward=(float(rg[w]), float(ro[w])), info=(int(ig[w]), int(io[w])), z=float(p[2]), r=float(np.linalg.norm(p))))
        flip = flip_agent.reshape(G, A).any(axis=1)
        s["flips"] += int(flip.sum())
        live_arena &= ~flip
        live = np.repeat(live_arena, A)
        assert np.array_equal(alive_prev_g[live], wa[live]), k
        assert np.array_equal(teg[live], teo[live]) and np.array_equal(trg[live], tro[live]), k
        assert np.array_equal(alive_g[live], ex["alive"][live]) and np.array_equal(reset_g[live], ex["reset"][live]), k
        cmp = live & wa  # the agents in self.agents before this step
        assert np.array_equal(ig[cmp] & 3, io[cmp] & 3), k
        shown = live & (wa | ex["reset"])  # ... and every agent of an arena that starts a new episode
        dobs = np.where(shown, np.abs(og[:, cols] - oo[:, cols]).max(axis=1), 0.0)
        # the reward adds -100 for every Aviary step an agent spends out of bounds or on the floor (-1200 per env step at 10 Hz,
        # where Hover's reward stops at the first): fp32 keeps 4 ulps of such a sum (2^-21 of it), which is not counted
        drew = np.where(cmp, np.maximum(np.abs(rg - ro) - 2.0**-21 * np.abs(ro), 0.0), 0.0)
        s["rew_abs"] = max(s["rew_abs"], float(np.abs(rg - ro)[cmp].max(initial=0.0)))
        if dobs.max() > s["obs"]:
            w = int(np.argmax(dobs))
            c = int(np.argmax(np.abs(og[w, cols] - oo[w, cols])))
            s["where"] = dict(step=k, agent=w, col=c, gpu=float(og[w, cols][c]), oracle=float(oo[w, cols][c]), reset=bool(ex["reset"][w]))
        agent_worst = np.maximum(agent_worst, dobs)
        s["obs"], s["rew"] = max(s["obs"], float(dobs.max())), max(s["rew"], float(drew.max()))
        fin = live & wa & ex["reset"]  # the terminal observations of the agents that finished their arena's episode
        if fin.any():
            s["final"] = max(s["final"], float(np.abs(final_g[fin][:, cols] - ex["final_obs"][fin][:, cols]).max()))
        if loose_obs is not None:
            loose |= (dobs > loose_obs) | (drew > loose_rew)
        s["resets"] += int(ex["reset"][live].sum()) // A
        alive_prev_g = alive_g
    av.set_noise_dump(None)
    s["loose"] = int(loose.sum())
    s["live_arenas"] = int(live_arena.sum())
    s["quantiles"] = np.quantile(agent_worst, [0.5, 0.99, 0.999]).tolist()
    s["above_bar"] = int((agent_worst > GPU_BAR).sum())
    return s


def _summary(tag, n, steps, s):
    return (f"\n[ma-hover {tag}] {n} agents x {steps} steps: {s['resets']} arena resets, flips {s['flips']}, culled agent-steps {s['culled']}, "
            f"loose {s.get('loose', 0)}; reset |obs| {s['reset_obs']:.2e}, max |obs| {s['obs']:.2e} at {s['where']}, max |final_obs| {s['final']:.2e}, "
            f"max |reward| {s['rew']:.2e} beyond 4 fp32 ulps ({s['rew_abs']:.2e} in all), max |noise dump - replay| {s['noise']:.2e}; "
            f"per-agent max |obs| quantiles 50/99/99.9 % {np.round(s['quantiles'], 8).tolist()}, {s['above_bar']} agents above {GPU_BAR:g}; "
            f"flips {s['flip_events']}")


def _rate_actions(rng, n):  # the Hover pin's box: random body rates and thrust, every step different
    return rng.uniform([-np.pi, -np.pi, -np.pi, 0.0], [np.pi, np.pi, np.pi, 0.8], (n, 4))


DEFAULT_START = np.array([[-1.0, -1.0, 1.0], [1.0, -1.0, 1.0], [-1.0, 1.0, 1.0], [1.0, 1.0, 1.0]])


def _check(s, n, num_arenas, obs_bar=GPU_BAR, rew_bar=GPU_BAR, min_resets=None):
    assert s["resets"] > (num_arenas if min_resets is None else min_resets), s
    # the device Box-Muller is within 2.2e-4 of fp64 (tests/test_device_math.py::test_box_muller_device)
    assert s["noise"] < 5e-4, s
    assert s["flips"] <= max(2, n // 4096), s
    assert s["obs"] < obs_bar and s["final"] < obs_bar and s["rew"] < rew_bar, s


@pytest.mark.gpu
def test_full_batch_timed_path_matches_oracle():
    """16 384 arenas x 4 agents (65 536 agents), Philox noise, 1 s episodes in a 3 m dome: arenas end at different steps and
    every arena is reset several times in 200 steps."""
    from pyflyt_b200.pz_envs import MAQuadXHoverVecEnv

    G, steps = 16384, 200
    env = MAQuadXHoverVecEnv(num_arenas=G, seed=SEED, max_duration_seconds=1.0, flight_dome_size=3.0)
    s = lockstep_ma(env, DEFAULT_START, SEED, steps, _rate_actions, rng_seed=1)
    env.close()
    print(_summary("full batch", 4 * G, steps, s))
    _check(s, 4 * G, G, min_resets=2 * G)


# mode -> action box (flight_mode 6: velocity setpoints; 7: position setpoints around the dome's centre)
MODE_BOX = {-1: ([0.0] * 4, [0.8] * 4), 0: ([-np.pi, -np.pi, -np.pi, 0.0], [np.pi, np.pi, np.pi, 0.8]),
            1: ([-np.pi, -np.pi, -np.pi, -1.0], [np.pi, np.pi, np.pi, 1.0]), 6: ([-2.0, -2.0, -1.0, -1.0], [2.0, 2.0, 1.0, 1.0]),
            7: ([-2.0, -2.0, -1.0, 0.5], [2.0, 2.0, 1.0, 3.0])}


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["quaternion-dense", "euler-sparse"])
@pytest.mark.parametrize("mode", [-1, 0, 1, 6, 7])
def test_flight_modes_match_oracle(mode, form):
    """2048 arenas x 4 agents x 120 steps in each flight mode and observation form.

    Mode 1 (roll / pitch setpoints up to +-pi, yaw rate, vz): the attitude loop amplifies rounding around random angle
    setpoints (test_reset_streams.py measures it on QuadX-Hover: per-env 99.9 % quantile 4.4e-5 in 1000 envs).  Over 8192
    agents one reaches 1.34e-4, in a yaw rate of -3.03 rad/s (H100 80GB HBM3, 700 W power limit; three agents above 1e-4,
    per-agent 99.9 % quantile 8.1e-5): all but 0.1 % of the agents are held to the 1e-4 bar, and every agent to 1e-3.  Modes 6 and 7 run the reference's z-velocity PID, which limit-cycles on cf2x (DESIGN.md 5;
    test_ma_quadx_hover.py::test_cuda_matches_reference loosens its bar for it): a rounding difference grows along the cycle,
    so these modes are held to the QuadX-Waypoints mode-7 envelope instead: position columns within 1e-3 and rewards within
    5e-2 for all but 0.5 % of the agents, and at most 2e-2 / 0.5 anywhere.  The printed line shows the spread."""
    from pyflyt_b200.pz_envs import MAQuadXHoverVecEnv

    G, steps = 2048, 120
    euler = form.startswith("euler")
    lo, hi = MODE_BOX[mode]
    env = MAQuadXHoverVecEnv(num_arenas=G, seed=SEED + mode, max_duration_seconds=1.0, flight_dome_size=3.0, flight_mode=mode,
                             angle_representation="euler" if euler else "quaternion", sparse_reward=euler)
    limit_cycle = mode in (6, 7)
    p0 = 9 if euler else 10
    kw = dict(cols=slice(p0, p0 + 3), loose_obs=1e-3, loose_rew=5e-2) if limit_cycle else {}
    if mode == 1:
        kw = dict(loose_obs=GPU_BAR, loose_rew=GPU_BAR)
    s = lockstep_ma(env, DEFAULT_START, SEED + mode, steps, lambda rng, n: rng.uniform(lo, hi, (n, 4)), rng_seed=10 + mode, **kw)
    env.close()
    print(_summary(f"mode {mode} {form}", 4 * G, steps, s))
    if limit_cycle:
        assert s["loose"] <= 5e-3 * 4 * G, s
        _check(s, 4 * G, G, obs_bar=2e-2, rew_bar=0.5)
    elif mode == 1:
        assert s["loose"] <= 1e-3 * 4 * G, s
        _check(s, 4 * G, G, obs_bar=1e-3, rew_bar=1e-3)
    else:
        _check(s, 4 * G, G)


RAGGED = {3: np.array([[-1.0, 0.0, 1.0], [1.0, 0.0, 1.0], [0.0, 1.2, 1.5]]), 2: np.array([[0.0, 0.0, 1.0], [0.5, 0.5, 1.5]])}


@pytest.mark.gpu
@pytest.mark.parametrize("env_offset", [0, 4093])
@pytest.mark.parametrize("euler", [True, False])
@pytest.mark.parametrize("A,G", [(3, 11), (3, 345), (2, 17)])
def test_ragged_arenas_match_oracle(A, G, euler, env_offset):
    """3- and 2-agent arenas: N = 33, 1035, 34 agents, a partial last tile of 1, 11 or 2 rows.  With euler observations (23
    floats) its byte count is not a multiple of 16, so k_hover_step writes it with the per-float loop instead of the bulk copy."""
    from pyflyt_b200.pz_envs import MAQuadXHoverVecEnv

    steps = 100
    env = MAQuadXHoverVecEnv(num_arenas=G, start_pos=RAGGED[A], seed=SEED, env_offset=env_offset, max_duration_seconds=1.0, flight_dome_size=3.0,
                             angle_representation="euler" if euler else "quaternion")
    n = A * G
    assert euler == ((n % 32) * env.obs_dim * 4 % 16 != 0)
    s = lockstep_ma(env, RAGGED[A], SEED, steps, _rate_actions, env_offset=env_offset, rng_seed=A * G)
    env.close()
    print(_summary(f"{G} arenas of {A}, {'euler' if euler else 'quaternion'}, offset {env_offset}", n, steps, s))
    _check(s, n, G)


@pytest.mark.gpu
@pytest.mark.parametrize("agent_hz", [120, 60, 24, 10])
def test_agent_rates_match_oracle(agent_hz):
    """env_step_ratio 1 (an env step ends halfway through a Philox pair), 2, 5 and 12 (past the four prefetched Aviary steps:
    the cold draws); the noise dump holds 2 x env_step_ratio draws per agent and step."""
    from pyflyt_b200.pz_envs import MAQuadXHoverVecEnv

    G, steps = 2048, 120
    env = MAQuadXHoverVecEnv(num_arenas=G, seed=SEED, agent_hz=agent_hz, max_duration_seconds=0.25, flight_dome_size=3.0)
    assert env.config.env_step_ratio == 120 // agent_hz
    s = lockstep_ma(env, DEFAULT_START, SEED, steps, _rate_actions, rng_seed=agent_hz)
    env.close()
    print(_summary(f"{agent_hz} Hz", 4 * G, steps, s))
    _check(s, 4 * G, G)


@pytest.mark.gpu
@pytest.mark.parametrize("agent_hz", [120, 60, 24, 10])
def test_hover_agent_rates_match_oracle(agent_hz):
    """QuadX-Hover's timed path (NEXT_STEP autoreset through spare post-reset states, on-device actions) at the same rates."""
    import lockstep
    from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverVecEnv

    n = 8192
    env = QuadXHoverVecEnv(num_envs=n, seed=SEED, agent_hz=agent_hz, max_duration_seconds=0.25)
    assert env.config.env_step_ratio == 120 // agent_hz
    run = lockstep.hover_step(env, SEED, 120)
    env.close()
    assert run.reset_obs < 1e-5, run.summary()
    assert run.worst_noise < 5e-4, run.summary()
    run.check(min_resets=n)
