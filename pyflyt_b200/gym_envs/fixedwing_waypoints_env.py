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

from ..core.env_base import WaypointsVecEnv, check_env_args, env_config
from ..models.tables import ENV_FIXEDWING_WAYPOINTS


class FixedwingWaypointsVecEnv(WaypointsVecEnv):
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
        autoreset_mode: str = "next_step",
    ):
        check_env_args(agent_hz, render_mode, angle_representation)  # fixedwing_base_env.py:47-52
        if flight_mode != 0:
            raise ValueError("Fixedwing-Waypoints is built for flight mode 0 (the env's 4-dim action box)")
        self.num_envs = int(num_envs)
        self.num_targets = int(num_targets)
        cfg = env_config(ENV_FIXEDWING_WAYPOINTS, agent_hz=agent_hz, max_duration_seconds=max_duration_seconds,
                         angle_representation=angle_representation, sparse_reward=sparse_reward, autoreset=autoreset,
                         flight_dome_size=flight_dome_size, inline_reset=inline_reset, autoreset_mode=autoreset_mode, goal_reach_distance=float(goal_reach_distance),
                         goal_reach_angle=float("inf"), num_targets=self.num_targets, use_yaw_targets=0)
        sp = np.tile(np.array([[0.0, 0.0, 10.0]]), (self.num_envs, 1))  # fixedwing_waypoints_env.py:63
        so = np.zeros((self.num_envs, 3))
        super().__init__(cfg, sp, so, "fixedwing", drone_options=drone_options, seed=seed, device=device, env_offset=env_offset)
        self.action_low, self.action_high = -np.ones(4), np.ones(4)  # fixedwing_base_env.py:79-81
        self.autoreset = bool(autoreset)
