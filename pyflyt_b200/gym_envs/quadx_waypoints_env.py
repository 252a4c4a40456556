"""QuadX-Waypoints on the batched stepper (SURVEY.md §8f, first widening row).

N copies of the reference's ``QuadXWaypointsEnv``
(/root/reference/PyFlyt/gym_envs/quadx_envs/quadx_waypoints_env.py:14-212 on top of quadx_base_env.py:17-301 and
gym_envs/utils/waypoint_handler.py) advanced by one fused launch per ``step``: 4 Aviary steps, the waypoint
bookkeeping (optionally with yaw targets), reward, termination and the observation.

The reference returns a Dict observation {"attitude" (21), "target_deltas" (k, 3 or 4) with k = targets left};
here it is one tensor ``[N, 21 + T*num_targets]`` (T = 4 with ``use_yaw_targets``): attitude, then the body-frame
deltas (and yaw errors) of the remaining targets in order, zero-padded.  ``info["num_targets_reached"]`` carries the
count.
"""

from __future__ import annotations

from typing import Literal, Sequence

import numpy as np
import torch

from ..core.env_base import WaypointsVecEnv, check_env_args, env_config
from ..models.tables import ENV_QUADX_WAYPOINTS


class QuadXWaypointsVecEnv(WaypointsVecEnv):
    def __init__(
        self,
        num_envs: int = 1,
        sparse_reward: bool = False,
        num_targets: int = 4,
        use_yaw_targets: bool = False,
        goal_reach_distance: float = 0.2,
        goal_reach_angle: float = 0.1,
        flight_mode: int = 0,
        flight_dome_size: float = 5.0,
        max_duration_seconds: float = 10.0,
        angle_representation: Literal["euler", "quaternion"] = "quaternion",
        agent_hz: int = 30,
        render_mode: None | str = None,
        drone_options: dict | Sequence[dict] | None = None,  # a sequence: one vehicle model per env (BatchedAviary)
        autoreset: bool = True,
        seed: int | None = None,
        device: str | torch.device = "cuda:0",
        env_offset: int = 0,
        inline_reset: bool = False,
        autoreset_mode: str = "next_step",
    ):
        check_env_args(agent_hz, render_mode, angle_representation)
        if flight_mode < -1 or flight_mode > 7:
            raise ValueError(f"`mode` must be between -1 and 7, got {flight_mode}.")
        self.num_envs = int(num_envs)
        self.num_targets = int(num_targets)
        self.use_yaw_targets = bool(use_yaw_targets)
        self.flight_mode = int(flight_mode)
        cfg = env_config(ENV_QUADX_WAYPOINTS, agent_hz=agent_hz, max_duration_seconds=max_duration_seconds,
                         angle_representation=angle_representation, sparse_reward=sparse_reward, autoreset=autoreset,
                         flight_dome_size=flight_dome_size, inline_reset=inline_reset, autoreset_mode=autoreset_mode, flight_mode=self.flight_mode,
                         goal_reach_distance=float(goal_reach_distance), goal_reach_angle=float(goal_reach_angle),
                         num_targets=self.num_targets, use_yaw_targets=int(self.use_yaw_targets))
        sp = np.tile(np.array([[0.0, 0.0, 1.0]]), (self.num_envs, 1))  # quadx_waypoints_env.py:71
        so = np.zeros((self.num_envs, 3))
        super().__init__(cfg, sp, so, "quadx", drone_options=drone_options, seed=seed, device=device, env_offset=env_offset)
        if self.flight_mode == -1:  # quadx_base_env.py:79-102
            self.action_low, self.action_high = np.zeros(4), np.ones(4) * 0.8
        else:
            self.action_low, self.action_high = np.array([-np.pi, -np.pi, -np.pi, 0.0]), np.array([np.pi, np.pi, np.pi, 0.8])
        self.autoreset = bool(autoreset)
