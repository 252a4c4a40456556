"""Fixedwing-Waypoints on the batched stepper (BASELINE.json configs[2]).

N copies of the reference's ``FixedwingWaypointsEnv``
(/root/reference/PyFlyt/gym_envs/fixedwing_envs/fixedwing_waypoints_env.py:16-190 on top of
fixedwing_base_env.py:16-278 and gym_envs/utils/waypoint_handler.py) advanced by one fused launch per
``step``: 4 Aviary steps (8 physics substeps of 5 lifting surfaces + motor + composite rigid body), the
waypoint bookkeeping, reward, termination and the observation.

The reference returns a Dict observation {"attitude" (23), "target_deltas" (k, 3) with k = targets left};
here it is one tensor ``[N, 23 + 3*num_targets]``: attitude, then the body-frame deltas of the remaining
targets in order, zero-padded.  ``info["num_targets_reached"]`` carries the count.
"""

from __future__ import annotations

from typing import Literal

import numpy as np
import torch

from ..core.aviary import BatchedAviary
from ..models import PfbEnvConfig
from ..models.tables import ENV_FIXEDWING_WAYPOINTS


class FixedwingWaypointsVecEnv:
    metadata = {"render_modes": [], "render_fps": 30}

    def __init__(
        self,
        num_envs: int = 1,
        sparse_reward: bool = False,
        num_targets: int = 4,
        goal_reach_distance: float = 2.0,
        flight_mode: int = 0,
        flight_dome_size: float = 100.0,
        max_duration_seconds: float = 120.0,
        angle_representation: Literal["euler", "quaternion"] = "quaternion",
        agent_hz: int = 30,
        render_mode: None | str = None,
        drone_options: dict | None = None,
        autoreset: bool = True,
        seed: int | None = None,
        device: str | torch.device = "cuda:0",
        env_offset: int = 0,
        inline_reset: bool = False,
    ):
        if 120 % agent_hz != 0:  # fixedwing_base_env.py:47-52
            lowest = int(120 / (int(120 / agent_hz) + 1))
            highest = int(120 / int(120 / agent_hz))
            raise ValueError(f"`agent_hz` must be round denominator of 120, try {lowest} or {highest}.")
        if render_mode is not None:
            raise ValueError("rendering is out of scope for the batched stepper (SURVEY.md §2 row 21)")
        if angle_representation not in ("euler", "quaternion"):
            raise ValueError(f"angle_representation must be either `euler` or `quaternion`, not {angle_representation}")
        if flight_mode != 0:
            raise ValueError("Fixedwing-Waypoints is built for flight mode 0 (the env's 4-dim action box)")
        self.num_envs = int(num_envs)
        self.num_targets = int(num_targets)
        cfg = PfbEnvConfig()
        cfg.env_kind = ENV_FIXEDWING_WAYPOINTS
        cfg.flight_mode = 0
        cfg.env_step_ratio = int(120 / agent_hz)
        cfg.max_steps = int(agent_hz * max_duration_seconds)
        cfg.angle_representation = 0 if angle_representation == "euler" else 1
        cfg.sparse_reward = int(bool(sparse_reward))
        cfg.autoreset = int(bool(autoreset))
        cfg.warmup_steps = 10  # fixedwing_base_env.py:187-188
        cfg.flight_dome_size = float(flight_dome_size)
        cfg.goal_reach_distance = float(goal_reach_distance)
        cfg.goal_reach_angle = float("inf")
        cfg.num_targets = self.num_targets
        cfg.use_yaw_targets = 0
        cfg.inline_reset = int(bool(inline_reset))  # tests: spare-copy resets must equal inline ones bit for bit
        self.config = cfg
        sp = np.tile(np.array([[0.0, 0.0, 10.0]]), (self.num_envs, 1))  # fixedwing_waypoints_env.py:63
        so = np.zeros((self.num_envs, 3))
        self.aviary = BatchedAviary(sp, so, drone_type="fixedwing", drone_options=drone_options, seed=seed, device=device, env_config=cfg, env_offset=env_offset)
        self.device = self.aviary.device
        self.obs_dim = self.aviary.obs_dim
        self.action_low, self.action_high = -np.ones(4), np.ones(4)  # fixedwing_base_env.py:79-81
        self.autoreset = bool(autoreset)

    def _info(self):
        bits = self.aviary.info_bits
        return {
            "out_of_bounds": (bits & 1).bool(),
            "collision": (bits & 2).bool(),
            "env_complete": (bits & 4).bool(),
            "num_targets_reached": (bits >> 3).int(),
        }

    def reset(self, *, seed: int | None = None, options: dict | None = None, mask=None, noise=None, targets=None):
        obs = self.aviary.env_reset(mask=mask, noise=noise, targets=targets, seed=seed)
        if mask is None:
            self.aviary.info_bits.zero_()
        return obs, self._info()

    def step(self, actions: torch.Tensor, noise=None):
        a = self.aviary
        if not (torch.is_tensor(actions) and actions.is_cuda and actions.dtype == torch.float32 and actions.is_contiguous()):
            a.setpoints.copy_(torch.as_tensor(actions, dtype=torch.float32, device=self.device).reshape(self.num_envs, 4))
            actions = None
        a.env_step(actions=actions, noise=noise)
        return a.obs, a.reward, a.term.bool(), a.trunc.bool(), self._info()

    def rollout(self, n_steps: int) -> None:
        self.aviary.env_rollout(n_steps)

    def close(self) -> None:
        self.aviary.disconnect()
