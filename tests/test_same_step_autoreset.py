"""gymnasium's SAME_STEP autoreset (PfbEnvConfig.autoreset = PFB_AUTORESET_SAME_STEP, ``autoreset_mode="same_step"``) for
QuadX-Hover, QuadX-Waypoints, Fixedwing-Waypoints and Rocket-Landing: an env that finishes on call k is reset inside call k,
its terminal observation goes to ``final_obs``.

CPU: the config builder, the facade's mode parsing, the header constants and the C-ABI refusals that come before the device
lookup.  GPU: each kind against the fp64 oracle reset in the same step (tests/lockstep_same.py, the bars of the NEXT_STEP drivers),
NEXT_STEP and SAME_STEP handles against each other, the spare path against inline_reset with episodes ending on every call, and
the other entry points."""
import ctypes
import os
import re

import numpy as np
import pytest

from pyflyt_b200 import _lib
from pyflyt_b200.core.env_base import env_config
from pyflyt_b200.models import build_model
from pyflyt_b200.models import tables

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "pyflyt_b200.h")
KINDS = ["hover", "qxwp", "fwwp", "rocket"]


@pytest.fixture(scope="module")
def L():
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    return _lib.lib()


# ------------------------------------------------------------------------------------------------------------------- CPU
def _cfg(**kw):
    args = dict(agent_hz=40, max_duration_seconds=10.0, angle_representation="quaternion", sparse_reward=False, autoreset=True, flight_dome_size=3.0)
    args.update(kw)
    return env_config(tables.ENV_QUADX_HOVER, **args)


def test_env_config_modes():
    assert _cfg().autoreset == 1
    assert _cfg(autoreset_mode="next_step").autoreset == 1
    assert _cfg(autoreset_mode="same_step").autoreset == 2
    assert _cfg(autoreset=False, autoreset_mode="same_step").autoreset == 0
    assert bytes(_cfg()) == bytes(_cfg(autoreset_mode="next_step"))  # the default config is what it was
    a, b = _cfg(), _cfg(autoreset_mode="same_step")
    a.autoreset = 2
    assert bytes(a) == bytes(b)  # the mode changes that one field only


@pytest.mark.parametrize("mode", ["NextStep", "SameStep", "same-step", "", None, 2, True])
def test_env_config_refuses_other_modes(mode):
    with pytest.raises(ValueError, match="autoreset_mode must be one of"):
        _cfg(autoreset_mode=mode)


def test_vecenv_refuses_a_bad_mode_before_touching_a_device():
    from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverVecEnv

    with pytest.raises(ValueError, match="autoreset_mode"):
        QuadXHoverVecEnv(num_envs=4, autoreset_mode="sameStep", device="cuda:99")


def test_header_autoreset_values_match_python():
    text = open(HEADER).read()
    found = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define PFB_AUTORESET_(\w+) (\d+)", text)}
    assert found == {"NONE": tables.AUTORESET_NONE, "NEXT_STEP": tables.AUTORESET_NEXT_STEP, "SAME_STEP": tables.AUTORESET_SAME_STEP}
    assert (tables.AUTORESET_NONE, tables.AUTORESET_NEXT_STEP, tables.AUTORESET_SAME_STEP) == (0, 1, 2)


def test_facade_mode_parsing():
    from pyflyt_b200.gym_envs import vector

    assert vector.PyFlytVectorEnv.metadata["autoreset_mode"] == vector._NEXT_STEP  # the class default stays NEXT_STEP
    for value in ("NextStep", "SameStep", "Disabled"):
        assert vector.parse_autoreset_mode(value) == value
        assert vector.parse_autoreset_mode(vector._MODES[value]) == value
    for bad in ("next_step", "same_step", "SAME_STEP", None, 1):
        with pytest.raises(ValueError, match="AutoresetMode"):
            vector.parse_autoreset_mode(bad)


@pytest.mark.parametrize("value", [3, -1, 100])
def test_create_refuses_unknown_autoreset(L, value):
    """The check comes before the device lookup, so it is the same with and without a GPU."""
    from engines import hover_config

    env = hover_config(autoreset=True)
    env.autoreset = value
    h = ctypes.c_void_p()
    assert L.pfb_create(ctypes.byref(build_model("quadx")), ctypes.byref(env), 8, 0, 0, ctypes.byref(h)) != 0 and not h.value
    assert L.pfb_last_error() == f"autoreset must be 0 (none), 1 (NEXT_STEP) or 2 (SAME_STEP), got {value}".encode()


@pytest.mark.parametrize("kind", ["mahover", "dogfight"])
def test_create_refuses_same_step_for_the_arena_kinds(L, kind):
    from engines import dogfight_config, hover_config

    if kind == "mahover":
        env, model = hover_config(autoreset=True), build_model("quadx")
        env.env_kind = tables.ENV_MA_QUADX_HOVER
    else:
        env, model = dogfight_config(), build_model("fixedwing", "acrowing")
    env.autoreset = 2
    h = ctypes.c_void_p()
    assert L.pfb_create(ctypes.byref(model), ctypes.byref(env), 8, 0, 0, ctypes.byref(h)) != 0 and not h.value
    assert L.pfb_last_error().startswith(b"SAME_STEP autoreset (autoreset = 2) is for the single-agent env kinds")


# ------------------------------------------------------------------------------------------------------------------- GPU
def make_env(kind, n, seed, mode="same_step", env_offset=0, **kw):
    """each kind with short episodes (every env autoresets within ~60 steps), as tests/test_reset_streams.py builds them"""
    base = dict(num_envs=n, seed=seed, env_offset=env_offset, autoreset_mode=mode)
    if kind == "hover":
        from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverVecEnv

        return QuadXHoverVecEnv(**base, **{"max_duration_seconds": 1.0, **kw})
    if kind == "qxwp":
        from pyflyt_b200.gym_envs.quadx_waypoints_env import QuadXWaypointsVecEnv

        return QuadXWaypointsVecEnv(**base, goal_reach_distance=1.0, goal_reach_angle=3.0, **{"max_duration_seconds": 1.0, **kw})
    if kind == "fwwp":
        from pyflyt_b200.gym_envs.fixedwing_waypoints_env import FixedwingWaypointsVecEnv

        return FixedwingWaypointsVecEnv(**base, goal_reach_distance=25.0, **{"max_duration_seconds": 1.0, **kw})
    if kind == "rocket":
        from pyflyt_b200.gym_envs.rocket_landing_env import RocketLandingVecEnv

        return RocketLandingVecEnv(**base, ceiling=120.0, **{"max_duration_seconds": 1.0, **kw})
    raise ValueError(kind)


def _drive(env, k, actions):
    """call k: on-device RANDACT draws (rollout(1)) or the given scripted actions"""
    import torch

    if actions is None:
        env.rollout(1)
    else:
        env.step(torch.as_tensor(actions[k], dtype=torch.float32, device=env.device))


def _scripted(kind, n, steps, seed=11):
    """the actions both handles of a comparison take: on-device draws (None) for the RANDACT-driven kinds"""
    rng = np.random.default_rng(seed)
    if kind == "qxwp":
        return rng.uniform([-1.0, -1.0, -1.0, 0.0], [1.0, 1.0, 1.0, 0.8], (steps, n, 4)).astype(np.float32)
    if kind == "rocket":
        return rng.uniform([-1, -1, -1, 0, 0, -1, -1], [1, 1, 1, 1, 1, 1, 1], (steps, n, 7)).astype(np.float32)
    return None


def _outputs(env):
    a = env.aviary
    return [t.clone() for t in (a.obs, a.reward, a.term, a.trunc, a.info_bits, a.final_obs)]


@pytest.mark.gpu
def test_hover_same_step_matches_oracle_single_step():
    import lockstep_same as lockstep

    env = make_env("hover", 65536, 20240924, max_duration_seconds=10.0)
    run = lockstep.hover_same_step(env, 20240924, 120)
    run.check(min_resets=100)
    env.close()


@pytest.mark.gpu
def test_hover_same_step_matches_oracle_fused():
    import lockstep_same as lockstep

    env = make_env("hover", 65536, 77, max_duration_seconds=10.0)
    run = lockstep.hover_same_fused(env, 77, [16, 16, 7, 16, 32, 16, 16])
    run.check(min_resets=100)
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["step", "fused"])
def test_hover_same_step_ragged_offset(path):
    """a ragged batch and a shard offset whose env ids straddle 2^32"""
    import lockstep_same as lockstep

    n, seed, offset = 4133, 0x1234_5678_9ABC, (1 << 32) - 500
    env = make_env("hover", n, seed, env_offset=offset)
    if path == "step":
        run = lockstep.hover_same_step(env, seed, 100, env_offset=offset)
    else:
        run = lockstep.hover_same_fused(env, seed, [16, 16, 7, 16, 32, 16], env_offset=offset)
    run.check(min_resets=n)
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["step", "fused"])
def test_hover_same_step_model_set_equals_uniform_handles(path):
    """cf2x / primitive_drone interleaved per env (the QuadXModelSet instantiations), ragged N and a shard offset, against two
    uniform SAME_STEP handles with the same seed: every env follows the handle of its model"""
    import torch

    n, seed, offset = 4133, 21, (1 << 32) - 500
    opts = [dict(drone_model="cf2x") if i % 2 == 0 else dict(drone_model="primitive_drone") for i in range(n)]
    mixed = make_env("hover", n, seed, env_offset=offset, drone_options=opts)
    uniform = [make_env("hover", n, seed, env_offset=offset, drone_options=dict(drone_model=m)) for m in ("cf2x", "primitive_drone")]
    idx = mixed.aviary.model_index
    assert len(mixed.aviary.models) == 2
    for e in [mixed] + uniform:
        e.reset()
    finished, worst = 0, 0.0
    for k in range(12 if path == "fused" else 120):
        for e in [mixed] + uniform:
            e.rollout(16 if path == "fused" else 1)
        m = mixed.aviary
        finished += int((m.term | m.trunc).sum())
        for j, U in enumerate(uniform):
            sel = idx == j
            u = U.aviary
            assert torch.equal(m.term[sel], u.term[sel]) and torch.equal(m.trunc[sel], u.trunc[sel]), k
            fin = sel & (m.term | m.trunc).bool()
            worst = max(worst, float((m.obs[sel] - u.obs[sel]).abs().max()), float((m.final_obs[fin] - u.final_obs[fin]).abs().max()) if fin.any() else 0.0)
    print(f"\n[same-step model set vs uniform, {path}] {finished} finished; max |difference| {worst:.2e}")
    assert finished > (n if path == "step" else n // 4) and worst < 1e-4
    for e in [mixed] + uniform:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["qxwp", "fwwp", "rocket"])
def test_tail_kinds_same_step_match_oracle(kind):
    import lockstep_same as lockstep

    seed = 20240925
    if kind == "qxwp":
        env = make_env(kind, 4096, seed)
        run = lockstep.quadx_waypoints_same_step(env, seed, 150)
    elif kind == "fwwp":
        env = make_env(kind, 4096, seed)
        run = lockstep.fixedwing_waypoints_same_step(env, seed, 150)
    else:
        env = make_env(kind, 4096, seed)
        run = lockstep.rocket_landing_same_step(env, seed, 200)
    run.check(min_resets=4096)
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_next_and_same_step_agree(kind):
    """Same seed, same actions: bit-identical outputs up to each env's first finish (SAME's final_obs = NEXT's obs on that
    call), and the first observation of every autoreset episode that both handles reach is bit-identical.

    Rocket-Landing is held to a bar instead: its step body compiled into the SAME_STEP kernel rounds some states differently
    from the NEXT_STEP kernel's copy (two compiled copies of one expression may contract multiply-adds differently), so an env
    whose finishing decision then differs is dropped, within a budget, and the rest agree to 5e-3."""
    import torch

    n, steps, seed = 2048, 150, 31
    nxt, same = make_env(kind, n, seed, "next_step"), make_env(kind, n, seed, "same_step")
    acts = _scripted(kind, n, steps)
    o_n, _ = nxt.reset()
    o_s, _ = same.reset()
    assert torch.equal(o_n, o_s)
    first_n, first_s = {}, {}  # (env, autoreset episode) -> its first observation
    ep_n, ep_s = np.zeros(n, dtype=np.int64), np.zeros(n, dtype=np.int64)
    before = torch.ones(n, dtype=torch.bool, device=nxt.device)  # no env has finished yet
    done_prev_n = np.zeros(n, dtype=bool)
    worst, n_flip = 0.0, 0
    for k in range(steps):
        _drive(nxt, k, acts)
        _drive(same, k, acts)
        on, rn, tn, trn, inn, _ = _outputs(nxt)
        os_, rs, ts, trs, ins, fs = _outputs(same)
        fin = (ts | trs).bool()
        b = before
        if kind == "rocket":
            flip = b & ((tn != ts) | (trn != trs) | (inn != ins))
            n_flip += int(flip.sum())
            b = b & ~flip
            fin = fin & b
            live = b & ~fin
            if b.any():
                worst = max(worst, float((rn[b] - rs[b]).abs().max()), float((on[live] - os_[live]).abs().max()) if live.any() else 0.0,
                            float((on[fin] - fs[fin]).abs().max()) if fin.any() else 0.0)
        else:
            assert torch.equal(rn[b], rs[b]) and torch.equal(tn[b], ts[b]) and torch.equal(trn[b], trs[b]) and torch.equal(inn[b], ins[b]), k
            live = b & ~fin
            assert torch.equal(on[live], os_[live]), k
            assert torch.equal(on[b & fin], fs[b & fin]), k
        before = b & ~fin
        # first observations: NEXT shows episode e on the call after the finish, SAME on the finishing call
        on_h, os_h, fin_h = on.cpu().numpy(), os_.cpu().numpy(), fin.cpu().numpy()
        for i in np.nonzero(done_prev_n)[0]:
            ep_n[i] += 1
            first_n[(i, ep_n[i])] = on_h[i]
        for i in np.nonzero(fin_h)[0]:
            ep_s[i] += 1
            first_s[(i, ep_s[i])] = os_h[i]
        done_prev_n = (tn | trn).bool().cpu().numpy()
    both = set(first_n) & set(first_s)
    assert len(both) >= n // 2, len(both)
    if kind == "rocket":
        first = max(float(np.abs(first_n[key] - first_s[key]).max()) for key in both)
        print(f"\n[{kind}] {n_flip} finishing decisions differ; max |difference| before the first finish {worst:.2e}; {len(both)} autoreset "
              f"episodes reached by both handles, max |first observation difference| {first:.2e}")
        assert n_flip <= max(2, n // 500) and worst < 5e-3 and first < 5e-3
    else:
        bad = [key for key in both if not np.array_equal(first_n[key], first_s[key])]
        print(f"\n[{kind}] {len(both)} autoreset episodes reached by both handles, {len(bad)} first observations differ")
        assert not bad, bad[:5]
    nxt.close()
    same.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("chunk", [1, 16])
def test_spare_path_equals_inline_with_episodes_ending_every_call(kind, chunk):
    """Episodes of one or two agent steps: every env resets every call or every second call, so a reused or half-built spare
    shows.  A SAME_STEP handle with spares and one with inline_reset agree bit for bit (QuadX-Hover: single steps and fused
    launches of 16, where the fourth reset of an env in a launch takes the cold path)."""
    import torch

    if chunk > 1 and kind != "hover":
        pytest.skip("the tail kinds run a rollout as single steps")
    n, seed = 3000, 5
    kw = dict(max_duration_seconds=0.05 if kind != "rocket" else 0.1)
    if kind == "fwwp":
        kw["agent_hz"] = 30
    a, b = make_env(kind, n, seed, **kw), make_env(kind, n, seed, inline_reset=True, **kw)
    acts = _scripted(kind, n, 40)
    assert torch.equal(a.reset()[0], b.reset()[0])
    resets = 0
    for k in range(0, 40, chunk):
        if chunk == 1:
            _drive(a, k, acts)
            _drive(b, k, acts)
        else:
            a.rollout(chunk)
            b.rollout(chunk)
        for x, y in zip(_outputs(a), _outputs(b)):
            assert torch.equal(x, y), k
        resets += int((a.aviary.term | a.aviary.trunc).sum())
    assert resets >= 5 * n // chunk
    a.close()
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_entry_points_on_a_same_step_handle(kind):
    """A wind change mid-run and a masked reset keep the spare and inline paths equal; reset(seed=s) twice replays the same
    episodes; the host and mapped step entry points are refused."""
    import torch

    from pyflyt_b200.core.wind import AnalyticWind

    n, seed, steps = 1024, 9, 60
    a, b = make_env(kind, n, seed), make_env(kind, n, seed, inline_reset=True)
    acts = _scripted(kind, n, steps)
    mask = torch.zeros(n, dtype=torch.bool, device=a.device)
    mask[::7] = True

    def run(seed_):
        outs = []
        for e in (a, b):
            e.reset(seed=seed_)
        for k in range(steps):
            if k == 20:
                for e in (a, b):
                    e.aviary.register_wind_field(AnalyticWind("constant", [1.5, -0.5, 0.0]))
            if k == 35:
                for e in (a, b):
                    e.reset(mask=mask)
            for e in (a, b):
                _drive(e, k, acts)
            xa, xb = _outputs(a), _outputs(b)
            for x, y in zip(xa, xb):
                assert torch.equal(x, y), k
            outs.append(xa)
        for e in (a, b):
            e.aviary.register_wind_field(None)
        return outs

    first, second = run(123), run(123)
    for x, y in zip(first, second):
        for u, v in zip(x[:5], y[:5]):
            assert torch.equal(u, v)
        fin = (x[2] | x[3]).bool()  # final_obs rows are written for the envs that finished only
        assert torch.equal(x[5][fin], y[5][fin])
    av = a.aviary
    pinned = [torch.zeros_like(t, device="cpu").pin_memory() for t in (av.setpoints, av.obs, av.reward, av.term, av.trunc)]
    with pytest.raises(_lib.PfbError, match="pfb_env_step_host"):
        av.env_step_host(*pinned)
    with pytest.raises(_lib.PfbError, match="pfb_env_step_mapped"):
        av.env_step_mapped(*pinned)
    a.close()
    b.close()


@pytest.mark.gpu
def test_bind_refuses_a_same_step_handle_without_final_obs():
    env = make_env("hover", 64, 1)
    b = _lib.PfbBuffers.from_buffer_copy(env.aviary._buffers)
    b.final_obs = None
    assert _lib.lib().pfb_bind(env.aviary._h, ctypes.byref(b)) != 0
    assert b"final_obs" in _lib.lib().pfb_last_error()
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("stem", ["QuadX-Hover", "QuadX-Waypoints", "Fixedwing-Waypoints", "Rocket-Landing"])
def test_facade_same_step(stem):
    """Through PyFlytVectorEnv: a finished env's returned obs is its reset observation, and info["final_obs"][mask] is what a
    NEXT_STEP facade returned as obs on that call; per-instance metadata; DISABLED resets only the masked envs."""
    import torch

    from pyflyt_b200.gym_envs import vector

    n, seed = 1024, 3
    kw = {"max_duration_seconds": 1.0}
    if stem == "Rocket-Landing":
        kw["ceiling"] = 120.0
    nxt = vector.PyFlytVectorEnv(f"PyFlyt/{stem}-v4", n, seed=seed, **kw)
    same = vector.PyFlytVectorEnv(f"PyFlyt/{stem}-v4", n, seed=seed, autoreset_mode="SameStep", **kw)
    assert nxt.metadata["autoreset_mode"] == vector._MODES["NextStep"] and same.metadata["autoreset_mode"] == vector._MODES["SameStep"]
    nxt.reset()
    same.reset()
    rng = np.random.default_rng(0)
    lo, hi = same.single_action_space.low, same.single_action_space.high
    checked = 0
    while checked == 0:
        act = torch.as_tensor(rng.uniform(lo, hi, (n, len(lo))).astype(np.float32), device=same.device)
        o_n, r_n, te_n, tr_n, i_n = nxt.step(act)
        o_s, r_s, te_s, tr_s, i_s = same.step(act)
        m = i_s["_final_obs"]
        assert torch.equal(m, te_s | tr_s) and i_s["final_obs"].shape == o_s.shape
        if m.any():
            assert torch.equal(i_s["final_obs"][m], o_n[m])
            assert torch.equal(o_s[m], same.env.aviary.obs[m])
            checked += int(m.sum())
            break
        assert torch.equal(o_n, o_s) and torch.equal(r_n, r_s)
    assert "final_obs" not in i_n
    # the finished envs' returned obs is the reset observation: the next NEXT_STEP call shows the same rows
    o_n2, *_ = nxt.step(act)
    assert torch.equal(o_n2[m], o_s[m])
    nxt.close()
    same.close()
    off = vector.PyFlytVectorEnv(f"PyFlyt/{stem}-v4", 64, seed=seed, autoreset_mode=vector._MODES["Disabled"], **kw)
    assert off.metadata["autoreset_mode"] == vector._MODES["Disabled"] and off.env.config.autoreset == 0
    o0, _ = off.reset()
    o0 = o0.clone()
    for _ in range(3):
        off.step(np.zeros((64, len(off.single_action_space.low)), dtype=np.float32))
    before = off.env.aviary.obs.clone()
    mask = np.zeros(64, dtype=bool)
    mask[::5] = True
    o1, _ = off.reset(options={"reset_mask": mask})
    mt = torch.as_tensor(mask, device=o1.device)
    assert torch.equal(o1[~mt], before[~mt])
    off.close()
