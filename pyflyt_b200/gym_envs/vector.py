"""gymnasium ``VectorEnv`` facade over the batched envs (SURVEY.md §8f item 2): N reference envs behind the API that
SB3 / CleanRL-style trainers consume — ``num_envs``, ``single_observation_space`` / ``single_action_space`` and their
batched versions, ``reset(seed=, options=) -> (obs, info)``, ``step(actions) -> (obs, reward, terminated, truncated, info)``
with gymnasium's NEXT_STEP (default), SAME_STEP or DISABLED autoreset (``metadata["autoreset_mode"]``, per instance), ``close()``.

Tensors are returned ZERO-COPY by default: ``obs``/``reward``/``terminated``/``truncated`` are views of the device buffers the
CUDA step kernel writes (valid until the next ``step``; clone what you store).  ``output="numpy"`` copies them to the host
for trainers that want arrays.  Subclasses ``gymnasium.vector.VectorEnv`` when gymnasium is importable.

The ids are the reference's (PyFlyt/gym_envs/__init__.py:8-43) plus the ``-v2`` aliases BASELINE.json uses; the waypoint
envs return the flat observation of the reference's ``FlattenWaypointEnv(context_length=num_targets)`` wrapper
(gym_envs/utils/flatten_waypoint_env.py): attitude, then the body-frame deltas of the remaining targets, zero-padded.
"""

from __future__ import annotations

from typing import Any

import numpy as np
import torch

from . import spaces

try:  # pragma: no cover - not installable in the build image
    from gymnasium.vector import VectorEnv as _Base
    from gymnasium.vector.vector_env import AutoresetMode

    _NEXT_STEP = AutoresetMode.NEXT_STEP
    _MODES = {m.value: m for m in AutoresetMode}
except Exception:
    _Base = object
    _NEXT_STEP = "NextStep"
    _MODES = {m: m for m in ("NextStep", "SameStep", "Disabled")}
# gymnasium's AutoresetMode values -> the batched envs' (autoreset, autoreset_mode) arguments
_ENV_AUTORESET = {"NextStep": (True, "next_step"), "SameStep": (True, "same_step"), "Disabled": (False, "next_step")}


def parse_autoreset_mode(mode) -> str:
    """gymnasium's ``AutoresetMode`` member or its string value (``"NextStep"``, ``"SameStep"``, ``"Disabled"``) -> the value."""
    value = getattr(mode, "value", mode)
    if value not in _ENV_AUTORESET:
        raise ValueError(f"autoreset_mode must be a gymnasium AutoresetMode or one of {list(_ENV_AUTORESET)}, got {mode!r}")
    return value

# id stem -> (module, VecEnv class, single-env adaptor module:class)
ENV_TABLE = {
    "QuadX-Hover": ("pyflyt_b200.gym_envs.quadx_hover_env", "QuadXHoverVecEnv", "pyflyt_b200.gym_envs.quadx_hover_env:QuadXHoverEnv"),
    "QuadX-Waypoints": ("pyflyt_b200.gym_envs.quadx_waypoints_env", "QuadXWaypointsVecEnv", "pyflyt_b200.gym_envs.single_env:QuadXWaypointsEnv"),
    "Fixedwing-Waypoints": ("pyflyt_b200.gym_envs.fixedwing_waypoints_env", "FixedwingWaypointsVecEnv", "pyflyt_b200.gym_envs.single_env:FixedwingWaypointsEnv"),
    "Rocket-Landing": ("pyflyt_b200.gym_envs.rocket_landing_env", "RocketLandingVecEnv", "pyflyt_b200.gym_envs.single_env:RocketLandingEnv"),
}
VERSIONS = ("v4", "v2")  # the reference's current ids and the aliases BASELINE.json quotes


def env_ids() -> list[str]:
    return [f"PyFlyt/{stem}-{v}" for stem in ENV_TABLE for v in VERSIONS]


def _stem(env_id: str) -> str:
    name = env_id.split("/", 1)[1] if "/" in env_id else env_id
    stem, _, ver = name.rpartition("-")
    if stem not in ENV_TABLE or ver not in VERSIONS:
        raise ValueError(f"unknown env id {env_id!r}; the batched stepper provides {env_ids()}")
    return stem


class PyFlytVectorEnv(_Base):
    """``num_envs`` copies of one reference env, stepped by one CUDA launch per ``step``."""

    metadata = {"render_modes": [], "autoreset_mode": _NEXT_STEP}

    def __init__(self, env_id: str, num_envs: int, output: str = "torch", device: str | torch.device = "cuda:0", seed: int | None = None,
                 autoreset_mode=_NEXT_STEP, **env_kwargs: Any):
        """``autoreset_mode``: gymnasium's ``AutoresetMode`` or its string value.  NEXT_STEP (default) and SAME_STEP run the
        reset inside the step launch; under SAME_STEP ``info["final_obs"]`` / ``info["_final_obs"]`` carry the terminal
        observations.  DISABLED leaves finished envs alone until ``reset(options={"reset_mask": mask})`` resets the masked ones."""
        if output not in ("torch", "numpy"):
            raise ValueError("output must be 'torch' (zero-copy device tensors) or 'numpy'")
        mode = parse_autoreset_mode(autoreset_mode)
        mod, cls, _ = ENV_TABLE[_stem(env_id)]
        self.spec_id = env_id
        self.output = output
        self.metadata = {**type(self).metadata, "autoreset_mode": _MODES[mode]}
        autoreset, env_mode = _ENV_AUTORESET[mode]
        self.env = getattr(__import__(mod, fromlist=[cls]), cls)(num_envs=int(num_envs), seed=seed, autoreset=autoreset, autoreset_mode=env_mode,
                                                                 device=device, **env_kwargs)
        self.num_envs = int(num_envs)
        self.device = self.env.device
        dt = np.float32
        self.single_observation_space = spaces.Box(low=-np.inf, high=np.inf, shape=(self.env.obs_dim,), dtype=dt)
        self.single_action_space = spaces.Box(low=self.env.action_low.astype(dt), high=self.env.action_high.astype(dt), dtype=dt)
        self.observation_space = spaces.batch_box(self.single_observation_space, self.num_envs)
        self.action_space = spaces.batch_box(self.single_action_space, self.num_envs)
        self.closed = False

    # ------------------------------------------------------------------
    def _out(self, x: torch.Tensor):
        return x if self.output == "torch" else x.cpu().numpy()

    def _info(self, info: dict) -> dict:
        return {k: self._out(v) for k, v in info.items()}

    def reset(self, *, seed: int | list[int] | None = None, options: dict | None = None):
        """A seed re-keys the random streams of the batch: the same seed gives the same episodes (gymnasium's contract,
        tests/test_gym_envs.py:92-112 of the reference).  The zero-copy tensors stay the same buffers across a seeded reset."""
        if isinstance(seed, (list, tuple)):
            seed = seed[0]
        mask = (options or {}).get("reset_mask")
        if mask is not None:  # gymnasium's DISABLED contract: reset only the masked envs
            mask = torch.as_tensor(np.asarray(mask) if not torch.is_tensor(mask) else mask, device=self.device).reshape(self.num_envs).bool()
        obs, info = self.env.reset(seed=seed, mask=mask)
        return self._out(obs), self._info(info)

    def step(self, actions):
        if not torch.is_tensor(actions):
            actions = torch.as_tensor(np.asarray(actions, dtype=np.float32), device=self.device)
        actions = actions.to(device=self.device, dtype=torch.float32).reshape(self.num_envs, -1).contiguous()
        obs, rew, term, trunc, info = self.env.step(actions)
        return self._out(obs), self._out(rew), self._out(term), self._out(trunc), self._info(info)

    def close(self, **kwargs):
        if not self.closed:
            self.env.close()
            self.closed = True

    def close_extras(self, **kwargs):  # gymnasium.vector.VectorEnv.close() calls this
        if not self.closed:
            self.env.close()
            self.closed = True

    @property
    def unwrapped(self):
        return self

    def __repr__(self):
        return f"PyFlytVectorEnv({self.spec_id}, num_envs={self.num_envs})"


def make_vec(env_id: str, num_envs: int, **kwargs) -> PyFlytVectorEnv:
    """``gymnasium.make_vec``-style constructor: ``make_vec("PyFlyt/QuadX-Hover-v4", 65536)``."""
    return PyFlytVectorEnv(env_id, num_envs, **kwargs)


def make(env_id: str, **kwargs):
    """``gymnasium.make`` for the ids of this package (single env, the reference's numpy-in / numpy-out signature); with
    gymnasium installed ``gymnasium.make(id)`` works too (the ids are registered at import)."""
    _, _, entry = ENV_TABLE[_stem(env_id)]
    mod, cls = entry.split(":")
    return getattr(__import__(mod, fromlist=[cls]), cls)(**kwargs)


def register_all() -> int:
    """Registers every id with gymnasium (single-env entry point + vector entry point); returns how many were registered
    (0 without gymnasium)."""
    try:
        from gymnasium.envs.registration import register, registry
    except Exception:
        return 0
    count = 0
    for stem, (_, _, entry) in ENV_TABLE.items():
        for v in VERSIONS:
            env_id = f"PyFlyt/{stem}-{v}"
            if env_id in registry:
                continue
            register(id=env_id, entry_point=entry,
                     vector_entry_point=lambda num_envs=1, _id=env_id, **kw: PyFlytVectorEnv(_id, num_envs, **kw))
            count += 1
    return count
