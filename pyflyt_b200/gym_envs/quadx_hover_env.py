"""QuadX-Hover on the batched stepper.

``QuadXHoverVecEnv`` is N copies of the reference's ``QuadXHoverEnv``
(/root/reference/PyFlyt/gym_envs/quadx_envs/quadx_hover_env.py:15-138 on top of
quadx_base_env.py:16-301) advanced by ONE fused kernel launch per ``step``: 3 Aviary steps (6 physics
substeps, 3 control ticks), reward accumulation, termination / truncation and the observation are all
computed in registers.  Constructor arguments, observation layout, action box, reward and termination
rules are the reference's; tensors replace numpy arrays and every output has a leading env axis.

``drone_options`` may be a sequence of ``num_envs`` dicts: env ``i`` then flies its own vehicle model (``BatchedAviary``).

``QuadXHoverEnv`` is the single-env, numpy-in/numpy-out adaptor with the reference's exact
``reset``/``step`` signature (what ``gymnasium.make("PyFlyt/QuadX-Hover-v4")`` returns).
"""

from __future__ import annotations

from typing import Any, Literal, Sequence

import numpy as np
import torch

from ..core.env_base import VecEnv, check_env_args, env_config
from ..models.tables import ENV_QUADX_HOVER
from .single_env import QuadXHoverEnv  # noqa: F401  (the gymnasium entry point names this module)


class QuadXHoverVecEnv(VecEnv):
    def __init__(
        self,
        num_envs: int = 1,
        sparse_reward: bool = False,
        flight_mode: int = 0,
        flight_dome_size: float = 3.0,
        max_duration_seconds: float = 10.0,
        angle_representation: Literal["euler", "quaternion"] = "quaternion",
        agent_hz: int = 40,
        render_mode: None | str = None,
        start_pos: np.ndarray | None = None,
        start_orn: np.ndarray | None = None,
        drone_options: dict[str, Any] | Sequence[dict[str, Any]] | None = None,
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
        self.flight_mode = int(flight_mode)
        self.sparse_reward = bool(sparse_reward)
        self.autoreset = bool(autoreset)
        cfg = env_config(ENV_QUADX_HOVER, agent_hz=agent_hz, max_duration_seconds=max_duration_seconds, angle_representation=angle_representation,
                         sparse_reward=sparse_reward, autoreset=autoreset, flight_dome_size=flight_dome_size, inline_reset=inline_reset, autoreset_mode=autoreset_mode,
                         flight_mode=self.flight_mode)
        self.flight_dome_size = cfg.flight_dome_size
        self.max_steps = cfg.max_steps
        self.env_step_ratio = cfg.env_step_ratio
        self.angle_representation = cfg.angle_representation

        sp = np.array([[0.0, 0.0, 1.0]]) if start_pos is None else np.asarray(start_pos, dtype=np.float64)
        so = np.array([[0.0, 0.0, 0.0]]) if start_orn is None else np.asarray(start_orn, dtype=np.float64)
        sp = np.ascontiguousarray(np.broadcast_to(sp.reshape(-1, 3) if sp.size == 3 else sp, (self.num_envs, 3)))
        so = np.ascontiguousarray(np.broadcast_to(so.reshape(-1, 3) if so.size == 3 else so, (self.num_envs, 3)))
        super().__init__(cfg, sp, so, "quadx", drone_options=drone_options, seed=seed, device=device, env_offset=env_offset)
        # action box (quadx_base_env.py:79-102)
        if self.flight_mode == -1:
            self.action_low = np.zeros(4)
            self.action_high = np.ones(4) * 0.8
        else:
            self.action_low = np.array([-np.pi, -np.pi, -np.pi, 0.0])
            self.action_high = np.array([np.pi, np.pi, np.pi, 0.8])
        self.single_observation_shape = (self.obs_dim,)
        self.single_action_shape = (4,)
