"""TEST INFRASTRUCTURE — lock-step drivers of the fp64 oracle for handles built with SAME_STEP autoreset
(``autoreset_mode="same_step"``): the drivers of tests/lockstep.py, with an env that finishes on call k reset on call k itself.

The oracle steps every env; its terminal observation is compared with the row the kernel wrote to final_obs (and the step's
reward and flags as usual); then the oracle resets the envs the kernel finished, with the same episode-keyed warm-up noise,
targets and drop poses as under NEXT_STEP, and that reset observation is compared with obs.  The bars, flip budgets and
``Run.check()`` are those of tests/lockstep.py.
"""
from __future__ import annotations

import numpy as np

from engines import OracleEngine, build_model
from lockstep import Run, _apply_wind, _autoreset_noise, _f, _host, hover_oracle, oracle_config
from philox_replay import Streams


def _same_step(env, run, orc, steps, act_fn, noise_fn, reset_fn, flag_fn, wind=None, cmp_fn=None, loose=(None, None)):
    import torch

    av, n = env.aviary, env.num_envs
    episode = np.full(n, run.extra.pop("episode0"), dtype=np.int64)
    for k in range(steps):
        if k:
            _apply_wind(wind, k, env, orc)
        act = act_fn(k)
        if act is None:  # on-device RANDACT draws: every env draws its action on every call
            env.rollout(1)
            act = run.extra["randact"](k)
            assert np.array_equal(av.setpoints.cpu().numpy(), act), k
        else:
            env.step(torch.as_tensor(act, dtype=torch.float32, device=av.device))
        og, rg, teg, trg, ig = _host(av)
        fo = av.final_obs.double().cpu().numpy()
        oo, ro, teo, tro, io = orc.o.env_step(act.astype(np.float64), noise_fn(k))
        teo, tro = teo.astype(bool), tro.astype(bool)
        done = teg | trg
        run.flips((teg != teo) | (trg != tro) | (flag_fn(ig) != flag_fn(io)))
        cmp = run.live if cmp_fn is None else run.live & cmp_fn(ig)
        term_obs = np.where(done[:, None], fo, og)  # the step's own observation: final_obs for the finished envs
        run.compare(np.abs(term_obs - oo).max(axis=1), np.abs(rg - ro), cmp, *loose)
        if done.any():
            idx = np.nonzero(done)[0]
            obs_r = reset_fn(done, idx, episode)
            episode[idx] += 1
            run.n_resets += len(idx)
            d = np.abs(og - obs_r).max(axis=1)
            run.compare(np.where(done, d, 0.0), np.zeros(n), run.live & done)
            run.extra["reset_obs_max"] = max(run.extra.get("reset_obs_max", 0.0), float(d[run.live & done].max(initial=0.0)))
    run.extra["episodes"] = int(episode.max())
    return run


def hover_same_step(env, seed: int, steps: int, *, env_offset: int = 0, reset_seq: int = 0, episode0: int = 1, obs_bar: float = 1e-4,
                    wind: dict | None = None) -> Run:
    """hover_step on a SAME_STEP handle: single-step launches with on-device RANDACT actions"""
    n, mode = env.num_envs, env.flight_mode
    run = Run("hover same-step", n, obs_bar, obs_bar, 4096)
    streams = Streams(seed, n, env_offset=env_offset, noise_loc=4.0)
    orc = hover_oracle(env, n)
    _apply_wind(wind, 0, env, orc)
    obs_g, _ = env.reset()
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(reset_seq).astype(np.float64))
    run.reset_obs = float(np.abs(obs_g.double().cpu().numpy() - obs_o).max())
    run.extra.update(episode0=episode0, randact=lambda k: streams.actions(k, mode))

    def reset(done, idx, episode):
        return orc.o.env_reset(mask=done.astype(np.uint8), noise=_autoreset_noise(streams, episode, idx, n))

    return _same_step(env, run, orc, steps, lambda k: None, lambda k: streams.step_noise(k).astype(np.float64), reset, lambda b: b & 3, wind)


def hover_same_fused(env, seed: int, chunks, *, env_offset: int = 0, reset_seq: int = 0, episode0: int = 1, obs_bar: float = 1e-4) -> Run:
    """hover_fused on a SAME_STEP handle (rollout(chunk): k_hover_same, up to 16 env steps per launch): the oracle resets on its
    own terminations in the step that ends them; at the end of every chunk the step counters, flags, observations, rewards and,
    for the envs that finished on the chunk's last step, the terminal observations must agree"""
    av, n, mode = env.aviary, env.num_envs, env.flight_mode
    run = Run("hover same-step fused", n, obs_bar, obs_bar, 2000)
    streams = Streams(seed, n, env_offset=env_offset, noise_loc=4.0)
    orc = hover_oracle(env, n)
    obs_g, _ = env.reset()
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(reset_seq).astype(np.float64))
    run.reset_obs = float(np.abs(obs_g.double().cpu().numpy() - obs_o).max())
    episode = np.full(n, episode0, dtype=np.int64)
    steps_o = np.zeros(n, dtype=np.int64)
    k = 0
    for chunk in chunks:
        env.rollout(chunk)
        assert np.array_equal(av.setpoints.cpu().numpy(), streams.actions(k + chunk - 1, mode))
        for _ in range(chunk):
            oo, ro, teo, tro, io = orc.o.env_step(streams.actions(k, mode).astype(np.float64), streams.step_noise(k).astype(np.float64))
            teo, tro = teo.astype(bool), tro.astype(bool)
            steps_o += 1
            done = teo | tro
            fo_o = oo.copy()
            if done.any():
                idx = np.nonzero(done)[0]
                obs_r = orc.o.env_reset(mask=done.astype(np.uint8), noise=_autoreset_noise(streams, episode, idx, n))
                oo[done] = obs_r[done]
                episode[idx] += 1
                steps_o[idx] = 0
                run.n_resets += len(idx)
            k += 1
        og, rg, teg, trg, _ = _host(av)
        fo = av.final_obs.double().cpu().numpy()
        run.flips((av.state_row_int(17).cpu().numpy() != steps_o) | (teg != teo) | (trg != tro))
        run.compare(np.abs(og - oo).max(axis=1), np.abs(rg - ro), run.live)
        run.compare(np.abs(fo - fo_o).max(axis=1), np.zeros(n), run.live & done)
    run.extra["episodes"] = int(episode.max())
    return run


def quadx_waypoints_same_step(env, seed: int, steps: int, *, env_offset: int = 0, reset_seq: int = 0, episode0: int = 1, rng_seed: int = 5) -> Run:
    """quadx_waypoints on a SAME_STEP handle (modes other than 7)"""
    n, c = env.num_envs, env.config
    yaw, T, dome = bool(c.use_yaw_targets), c.num_targets, c.flight_dome_size
    run = Run("quadx-waypoints same-step", n, 5e-4, 5e-3, 500)
    streams = Streams(seed, n, env_offset=env_offset, noise_loc=4.0)
    orc = OracleEngine(build_model("quadx", "cf2x"), oracle_config(env), n, np.tile([[0.0, 0.0, 1.0]], (n, 1)), np.zeros((n, 3)))
    obs_g, _ = env.reset()
    tg = streams.waypoint_targets(0x80000000 | reset_seq, T, dome, min_height=0.1, yaw=yaw)
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(reset_seq).astype(np.float64), targets=tg.astype(np.float64).reshape(n, -1))
    run.reset_obs = float(np.abs(obs_g.double().cpu().numpy() - obs_o).max())
    run.extra["episode0"] = episode0
    rng = np.random.default_rng(rng_seed)

    def reset(done, idx, episode):
        tgr = np.zeros((n, T, 4 if yaw else 3))
        tgr[idx] = streams.waypoint_targets(episode[idx], T, dome, min_height=0.1, envs=idx, yaw=yaw)
        return orc.o.env_reset(mask=done.astype(np.uint8), noise=_autoreset_noise(streams, episode, idx, n), targets=tgr.reshape(n, -1))

    return _same_step(env, run, orc, steps, lambda k: _f(rng.uniform([-1.0, -1.0, -1.0, 0.0], [1.0, 1.0, 1.0, 0.8], (n, 4))),
                      lambda k: streams.step_noise(k, 4).astype(np.float64), reset, lambda b: b >> 3, loose=(1e-3, 5e-2))


def fixedwing_waypoints_same_step(env, seed: int, steps: int, *, env_offset: int = 0, reset_seq: int = 0, episode0: int = 1,
                                  obs_bar: float = 5e-3, wind: dict | None = None) -> Run:
    """fixedwing_waypoints on a SAME_STEP handle: on-device RANDACT actions, drawn by every env on every call"""
    n, T, dome = env.num_envs, env.config.num_targets, env.config.flight_dome_size
    run = Run("fixedwing-waypoints same-step", n, obs_bar, 5e-3, 1000)
    streams = Streams(seed, n, env_offset=env_offset, noise_loc=1.0)
    orc = OracleEngine(build_model("fixedwing", "fixedwing"), oracle_config(env), n, np.tile([[0.0, 0.0, 10.0]], (n, 1)), np.zeros((n, 3)))
    _apply_wind(wind, 0, env, orc)
    obs_g, _ = env.reset()
    tg = streams.waypoint_targets(0x80000000 | reset_seq, T, dome, min_height=0.5)
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(reset_seq).astype(np.float64), targets=tg.astype(np.float64).reshape(n, -1))
    run.reset_obs = float(np.abs(obs_g.double().cpu().numpy() - obs_o).max())
    run.extra.update(episode0=episode0, randact=streams.uniform_actions)

    def reset(done, idx, episode):
        tgr = np.zeros((n, T, 3))
        tgr[idx] = streams.waypoint_targets(episode[idx], T, dome, min_height=0.5, envs=idx)
        return orc.o.env_reset(mask=done.astype(np.uint8), noise=_autoreset_noise(streams, episode, idx, n), targets=tgr.reshape(n, -1))

    return _same_step(env, run, orc, steps, lambda k: None, lambda k: streams.step_noise(k, 4).astype(np.float64), reset, lambda b: b >> 3, wind)


def rocket_landing_same_step(env, seed: int, steps: int, *, env_offset: int = 0, reset_seq: int = 0, episode0: int = 1, rng_seed: int = 3) -> Run:
    """rocket_landing on a SAME_STEP handle; the crash step's terminal observation and reward stay out of the comparison"""
    n, ceiling = env.num_envs, env.config.ceiling
    run = Run("rocket-landing same-step", n, 0.1, 0.5, 500, loose_frac=1e-3)
    streams = Streams(seed, n, env_offset=env_offset, noise_loc=1.0)
    sp, so = streams.drop_poses(0x80000000 | reset_seq, ceiling, 200.0)
    sp, so = sp.astype(np.float64), so.astype(np.float64)
    orc = OracleEngine(build_model("rocket", "rocket", starting_fuel_ratio=0.05), oracle_config(env), n, sp, so)
    obs_g, _ = env.reset()
    obs_o = orc.o.env_reset(noise=streams.user_reset_noise(reset_seq).astype(np.float64))
    run.reset_obs = float(np.abs(obs_g.double().cpu().numpy() - obs_o).max())
    run.extra["episode0"] = episode0
    rng = np.random.default_rng(rng_seed)

    def reset(done, idx, episode):
        sp[idx], so[idx] = streams.drop_poses(episode[idx], ceiling, 200.0, envs=idx)
        orc.o.set_start(sp, so)
        return orc.o.env_reset(mask=done.astype(np.uint8), noise=_autoreset_noise(streams, episode, idx, n))

    return _same_step(env, run, orc, steps, lambda k: _f(rng.uniform([-1, -1, -1, 0, 0, -1, -1], [1, 1, 1, 1, 1, 1, 1], (n, 7))),
                      lambda k: streams.step_noise(k, 3).astype(np.float64), reset, lambda b: b & 7, cmp_fn=lambda ig: (ig & 2) == 0, loose=(5e-3, 2e-2))
