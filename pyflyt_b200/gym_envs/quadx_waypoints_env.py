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

from ..core.aviary import BatchedAviary
from ..models import PfbEnvConfig
from ..models.tables import ENV_QUADX_WAYPOINTS


class QuadXWaypointsVecEnv:
    metadata = {"render_modes": [], "render_fps": 30}

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
    ):
        if 120 % agent_hz != 0:  # quadx_base_env.py:47-52
            lowest = int(120 / (int(120 / agent_hz) + 1))
            highest = int(120 / int(120 / agent_hz))
            raise ValueError(f"`agent_hz` must be round denominator of 120, try {lowest} or {highest}.")
        if render_mode is not None:
            raise ValueError("rendering is out of scope for the batched stepper (SURVEY.md §2 row 21)")
        if angle_representation not in ("euler", "quaternion"):  # quadx_base_env.py:66-69
            raise ValueError(f"angle_representation must be either `euler` or `quaternion`, not {angle_representation}")
        if flight_mode < -1 or flight_mode > 7:
            raise ValueError(f"`mode` must be between -1 and 7, got {flight_mode}.")
        self.num_envs = int(num_envs)
        self.num_targets = int(num_targets)
        self.use_yaw_targets = bool(use_yaw_targets)
        self.flight_mode = int(flight_mode)
        cfg = PfbEnvConfig()
        cfg.env_kind = ENV_QUADX_WAYPOINTS
        cfg.flight_mode = self.flight_mode
        cfg.env_step_ratio = int(120 / agent_hz)
        cfg.max_steps = int(agent_hz * max_duration_seconds)
        cfg.angle_representation = 0 if angle_representation == "euler" else 1
        cfg.sparse_reward = int(bool(sparse_reward))
        cfg.autoreset = int(bool(autoreset))
        cfg.warmup_steps = 10  # quadx_base_env.py:209-210
        cfg.flight_dome_size = float(flight_dome_size)
        cfg.goal_reach_distance = float(goal_reach_distance)
        cfg.goal_reach_angle = float(goal_reach_angle)
        cfg.num_targets = self.num_targets
        cfg.use_yaw_targets = int(self.use_yaw_targets)
        cfg.inline_reset = int(bool(inline_reset))  # tests: spare-copy resets must equal inline ones bit for bit
        self.config = cfg
        sp = np.tile(np.array([[0.0, 0.0, 1.0]]), (self.num_envs, 1))  # quadx_waypoints_env.py:71
        so = np.zeros((self.num_envs, 3))
        self.aviary = BatchedAviary(sp, so, drone_type="quadx", drone_options=drone_options, seed=seed, device=device, env_config=cfg, env_offset=env_offset)
        self.device = self.aviary.device
        self.obs_dim = self.aviary.obs_dim
        if self.flight_mode == -1:  # quadx_base_env.py:79-102
            self.action_low, self.action_high = np.zeros(4), np.ones(4) * 0.8
        else:
            self.action_low, self.action_high = np.array([-np.pi, -np.pi, -np.pi, 0.0]), np.array([np.pi, np.pi, np.pi, 0.8])
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
        """``targets``: optional [N, num_targets, 3 or 4] waypoints (x, y, z[, yaw]); default = drawn on device."""
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
