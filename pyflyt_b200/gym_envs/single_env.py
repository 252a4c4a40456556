"""Single-env adaptors with the reference's call signatures (numpy in, numpy out) on top of the batched envs.

They exist so that code written against ``PyFlyt.gym_envs`` runs unchanged for smoke tests and evaluation loops; the
throughput path is the ``*VecEnv`` classes.  Observation layouts follow the reference:

* ``QuadXWaypointsEnv`` / ``FixedwingWaypointsEnv``: ``{"attitude": (A,), "target_deltas": (k, T)}`` with k = targets left
  (quadx_waypoints_env.py:95-110, fixedwing_waypoints_env.py:88-101);
* ``QuadXHoverEnv`` / ``RocketLandingEnv``: flat vector (quadx_hover_env.py:85-116, rocket_landing_env.py:129-188).
"""

from __future__ import annotations

from typing import Any

import numpy as np
import torch

from . import spaces


class _SingleEnv:
    _vec_cls = None
    _action_dim = 4

    def __init__(self, **kwargs):
        kwargs.setdefault("autoreset", False)
        self._vec = self._vec_cls(num_envs=1, **kwargs)
        self.action_space = spaces.Box(low=self._vec.action_low, high=self._vec.action_high, dtype=np.float64)
        self.observation_space = self._make_observation_space()

    def _make_observation_space(self):
        return spaces.Box(low=-np.inf, high=np.inf, shape=(self._vec.obs_dim,), dtype=np.float64)

    def _info(self, info) -> dict:
        out = {}
        for k, v in info.items():
            x = v[0].item()
            out[k] = bool(x) if v.dtype == torch.bool else int(x)
        return out

    def _obs(self, obs: torch.Tensor, info: dict):
        return obs[0].double().cpu().numpy()

    def reset(self, *, seed: None | int = None, options: None | dict[str, Any] = dict()):
        obs, info = self._vec.reset(seed=seed)  # the same seed replays the same episode (gymnasium's contract)
        info = self._info(info)
        return self._obs(obs, info), info

    def step(self, action: np.ndarray):
        a = torch.as_tensor(np.asarray(action, dtype=np.float32).reshape(1, self._action_dim), device=self._vec.device)
        obs, rew, term, trunc, info = self._vec.step(a)
        info = self._info(info)
        return self._obs(obs, info), float(rew[0].item()), bool(term[0].item()), bool(trunc[0].item()), info

    def close(self):
        self._vec.close()


class _WaypointsMixin:
    _attitude_dim = {"quadx": (20, 21), "fixedwing": (22, 23)}

    def _make_observation_space(self):  # quadx_waypoints_env.py:95-110, fixedwing_waypoints_env.py:88-101
        v = self._vec
        a = self._attitude_dim[self._vehicle][1 if v.config.angle_representation == 1 else 0]
        t = 4 if getattr(v, "use_yaw_targets", False) else 3
        return spaces.Dict({
            "attitude": spaces.Box(low=-np.inf, high=np.inf, shape=(a,), dtype=np.float64),
            "target_deltas": spaces.Sequence(spaces.Box(low=-np.inf, high=np.inf, shape=(t,), dtype=np.float64), stack=True),
        })

    def _obs(self, obs: torch.Tensor, info: dict):
        v = self._vec
        quat = v.config.angle_representation == 1
        a = self._attitude_dim[self._vehicle][1 if quat else 0]
        t = 4 if getattr(v, "use_yaw_targets", False) else 3
        flat = obs[0].double().cpu().numpy()
        # remaining targets come first, zero rows pad the tail (a real delta that is exactly zero has measure zero); the
        # count can exceed num_targets - num_targets_reached by one: the observation is built before the list advances
        rows = flat[a:].reshape(v.num_targets, t)
        k = int(np.any(rows != 0.0, axis=1).sum())
        return {"attitude": flat[:a], "target_deltas": rows[:k]}


def _make(name, vec_import, vehicle=None, action_dim=4, doc="", **attrs):
    def _vec_cls(*a, **k):
        mod, cls = vec_import
        return getattr(__import__(mod, fromlist=[cls]), cls)(*a, **k)

    bases = (_WaypointsMixin, _SingleEnv) if vehicle else (_SingleEnv,)
    return type(name, bases, {"_vec_cls": staticmethod(_vec_cls), "_action_dim": action_dim, "_vehicle": vehicle, "__doc__": doc, **attrs})


QuadXHoverEnv = _make("QuadXHoverEnv", ("pyflyt_b200.gym_envs.quadx_hover_env", "QuadXHoverVecEnv"),
                      doc="gym_envs/quadx_envs/quadx_hover_env.py:15-138 for one env.", metadata={"render_modes": [], "render_fps": 30})
QuadXWaypointsEnv = _make("QuadXWaypointsEnv", ("pyflyt_b200.gym_envs.quadx_waypoints_env", "QuadXWaypointsVecEnv"), "quadx",
                          doc="gym_envs/quadx_envs/quadx_waypoints_env.py:14-212 for one env.")
FixedwingWaypointsEnv = _make("FixedwingWaypointsEnv", ("pyflyt_b200.gym_envs.fixedwing_waypoints_env", "FixedwingWaypointsVecEnv"), "fixedwing",
                              doc="gym_envs/fixedwing_envs/fixedwing_waypoints_env.py:16-190 for one env.")
RocketLandingEnv = _make("RocketLandingEnv", ("pyflyt_b200.gym_envs.rocket_landing_env", "RocketLandingVecEnv"), None, action_dim=7,
                         doc="gym_envs/rocket_envs/rocket_landing_env.py:17-263 for one env.")
