"""The batched envs' constructor surface, on the CPU: argument refusals (type and message) and the ``PfbEnvConfig`` each env
builds from its defaults.  ``BatchedAviary`` is replaced by a recorder, so nothing here needs a GPU."""

import pytest
import torch

import engines
from pyflyt_b200.models import PfbEnvConfig

HZ_MSG = "`agent_hz` must be round denominator of 120, try 40 or 60."
RENDER_MSG = "rendering is out of scope for the batched stepper (SURVEY.md §2 row 21)"
ANGLE_MSG = "angle_representation must be either `euler` or `quaternion`, not rpy"


@pytest.fixture
def recorder(monkeypatch):
    """Replaces ``BatchedAviary`` where the envs build it; returns the list of the keyword arguments of every construction."""
    from pyflyt_b200.core import env_base
    from pyflyt_b200.pz_envs import ma_fixedwing_dogfight_split

    calls = []

    class Recorder:
        def __init__(self, start_pos, start_orn, **kwargs):
            calls.append(dict(kwargs, start_pos=start_pos, start_orn=start_orn))
            self.device = torch.device("cpu")
            self.obs_dim = 21

    monkeypatch.setattr(env_base, "BatchedAviary", Recorder)
    monkeypatch.setattr(ma_fixedwing_dogfight_split, "BatchedAviary", Recorder)
    return calls


def env_class(name):
    from pyflyt_b200 import gym_envs, pz_envs

    return getattr(gym_envs, name, None) or getattr(pz_envs, name)


GYM = ["QuadXHoverVecEnv", "QuadXWaypointsVecEnv", "FixedwingWaypointsVecEnv", "RocketLandingVecEnv"]
MA = ["MAQuadXHoverVecEnv", "MAFixedwingDogfightVecEnv"]

REFUSALS = (
    [(n, dict(agent_hz=50), ValueError, HZ_MSG) for n in GYM]
    + [(n, dict(agent_hz=50), AssertionError, HZ_MSG) for n in MA]
    + [(n, dict(render_mode="human"), ValueError, RENDER_MSG) for n in GYM + MA]
    + [(n, dict(angle_representation="rpy"), ValueError, ANGLE_MSG) for n in GYM + ["MAQuadXHoverVecEnv"]]
    + [(n, dict(flight_mode=m), ValueError, f"`mode` must be between -1 and 7, got {m}.") for n in GYM[:2] for m in (-2, 8)]
    + [("FixedwingWaypointsVecEnv", dict(flight_mode=m), ValueError, "Fixedwing-Waypoints is built for flight mode 0 (the env's 4-dim action box)")
       for m in (-1, 1)]
    + [(n, dict(inline_reset=2), ValueError, "inline_reset must be a bool, got 2") for n in GYM + ["MAFixedwingDogfightVecEnv"]]
    # checked in the reference's order: agent_hz before render_mode before angle_representation before the flight mode
    + [("QuadXHoverVecEnv", dict(agent_hz=50, render_mode="human", angle_representation="rpy", flight_mode=8), ValueError, HZ_MSG),
       ("QuadXWaypointsVecEnv", dict(render_mode="human", angle_representation="rpy", flight_mode=8), ValueError, RENDER_MSG),
       ("RocketLandingVecEnv", dict(angle_representation="rpy", inline_reset=2), ValueError, ANGLE_MSG)]
)


@pytest.mark.parametrize("name,kwargs,exc,msg", REFUSALS)
def test_constructor_refusals(recorder, name, kwargs, exc, msg):
    with pytest.raises(exc) as e:
        env_class(name)(**kwargs)
    assert type(e.value) is exc and str(e.value) == msg
    assert recorder == []


def test_split_dogfight_refuses_agent_hz(recorder):
    from pyflyt_b200.pz_envs import MAFixedwingDogfightSplitEnv

    with pytest.raises(AssertionError):
        MAFixedwingDogfightSplitEnv(2, agent_hz=50, single_rank=True)
    assert recorder == []


# default construction -> (the engines.py config of the kind, the fields where the env's defaults differ from the helper's)
DEFAULTS = {
    "QuadXHoverVecEnv": (engines.hover_config, dict(autoreset=1, inline_reset=0)),
    "QuadXWaypointsVecEnv": (engines.quadx_waypoints_config, dict(autoreset=1, inline_reset=0)),
    "FixedwingWaypointsVecEnv": (engines.waypoints_config, dict(autoreset=1, inline_reset=0)),
    "RocketLandingVecEnv": (engines.landing_config, dict(autoreset=1, inline_reset=0, randomize_drop=1, accelerate_drop=1, contact_response=1)),
    "MAQuadXHoverVecEnv": (engines.ma_hover_config, dict()),
    "MAFixedwingDogfightVecEnv": (engines.dogfight_config, dict(autoreset=1, inline_reset=0, randomize_drop=1)),
    # the reference draws the spawn heights from the radius range (sic), and the split env keeps that
    "MAFixedwingDogfightSplitEnv": (engines.dogfight_config, dict(spawn_min_height=10.0, spawn_max_height=50.0)),
}


@pytest.mark.parametrize("name", sorted(DEFAULTS))
def test_default_config(recorder, name):
    helper, env_only = DEFAULTS[name]
    env = env_class(name)(2, single_rank=True) if name.endswith("SplitEnv") else env_class(name)()
    expected = helper()
    for field, value in env_only.items():
        setattr(expected, field, value)
    for field, _ in PfbEnvConfig._fields_:
        assert getattr(env.config, field) == getattr(expected, field), field
    assert bytes(env.config) == bytes(expected)
    assert len(recorder) == 1 and recorder[0]["env_config"] is env.config
