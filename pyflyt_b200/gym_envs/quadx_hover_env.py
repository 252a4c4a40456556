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

from ..core.aviary import BatchedAviary
from ..models import PfbEnvConfig
from ..models.tables import ENV_QUADX_HOVER


class QuadXHoverVecEnv:
    metadata = {"render_modes": [], "render_fps": 30}

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
        inline_reset: bool | int = False,
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
        self.flight_mode = int(flight_mode)
        self.flight_dome_size = float(flight_dome_size)
        self.max_steps = int(agent_hz * max_duration_seconds)
        self.env_step_ratio = int(120 / agent_hz)
        self.sparse_reward = bool(sparse_reward)
        self.angle_representation = 0 if angle_representation == "euler" else 1
        self.autoreset = bool(autoreset)

        cfg = PfbEnvConfig()
        cfg.env_kind = ENV_QUADX_HOVER
        cfg.flight_mode = self.flight_mode
        cfg.env_step_ratio = self.env_step_ratio
        cfg.max_steps = self.max_steps
        cfg.angle_representation = self.angle_representation
        cfg.sparse_reward = int(self.sparse_reward)
        cfg.autoreset = int(self.autoreset)
        cfg.warmup_steps = 10  # quadx_base_env.py:209-210
        cfg.flight_dome_size = self.flight_dome_size
        # 0: finished envs take their spare post-reset state, spares rebuilt on the library's side stream; 1: every warm-up is
        # integrated inside the step launch (tests: must equal the spare path bit for bit); 2: spares, rebuilt on the caller's stream
        cfg.inline_reset = int(inline_reset)
        self.config = cfg

        sp = np.array([[0.0, 0.0, 1.0]]) if start_pos is None else np.asarray(start_pos, dtype=np.float64)
        so = np.array([[0.0, 0.0, 0.0]]) if start_orn is None else np.asarray(start_orn, dtype=np.float64)
        sp = np.ascontiguousarray(np.broadcast_to(sp.reshape(-1, 3) if sp.size == 3 else sp, (self.num_envs, 3)))
        so = np.ascontiguousarray(np.broadcast_to(so.reshape(-1, 3) if so.size == 3 else so, (self.num_envs, 3)))
        self.aviary = BatchedAviary(
            sp, so, drone_type="quadx", drone_options=drone_options, seed=seed, device=device, env_config=cfg, env_offset=env_offset
        )
        self.device = self.aviary.device
        self.obs_dim = self.aviary.obs_dim
        # action box (quadx_base_env.py:79-102)
        if self.flight_mode == -1:
            self.action_low = np.zeros(4)
            self.action_high = np.ones(4) * 0.8
        else:
            self.action_low = np.array([-np.pi, -np.pi, -np.pi, 0.0])
            self.action_high = np.array([np.pi, np.pi, np.pi, 0.8])
        self.single_observation_shape = (self.obs_dim,)
        self.single_action_shape = (4,)

    # ------------------------------------------------------------------
    def _info(self) -> dict[str, torch.Tensor]:
        bits = self.aviary.info_bits
        return {
            "out_of_bounds": (bits & 1).bool(),
            "collision": (bits & 2).bool(),
            "env_complete": (bits & 4).bool(),
        }

    def reset(self, *, seed: int | None = None, options: dict | None = None, mask: torch.Tensor | None = None, noise=None):
        """env.reset() for every env (or the masked ones): quadx_hover_env.py:70-83.  ``seed`` re-keys the random streams of the
        whole batch first (``BatchedAviary.reseed``): the same seed then replays the same episodes."""
        obs = self.aviary.env_reset(mask=mask, noise=noise, seed=seed)
        if mask is None:
            self.aviary.info_bits.zero_()
        return obs, self._info()

    def step(self, actions: torch.Tensor, noise=None):
        """env.step(action) for every env: quadx_base_env.py:269-301.  With ``autoreset`` (gymnasium's
        default NEXT_STEP mode) an env that terminated / truncated on the previous call is reset on this
        one: its action is ignored and it returns the first observation of the new episode with reward 0
        and both flags False — all inside the same kernel launch."""
        a = self.aviary
        if not (torch.is_tensor(actions) and actions.is_cuda and actions.dtype == torch.float32 and actions.is_contiguous()):
            a.setpoints.copy_(torch.as_tensor(actions, dtype=torch.float32, device=self.device).reshape(self.num_envs, 4))
            actions = None
        a.env_step(actions=actions, noise=noise)
        return a.obs, a.reward, a.term.bool(), a.trunc.bool(), self._info()

    def rollout(self, n_steps: int) -> None:
        """n_steps env steps with on-device uniform random actions (benchmark shape of BASELINE.json).  With autoreset, 4 or more
        steps run as fused launches of up to 16 env steps each (``pfb_env_rollout``); the buffers then hold the last step's results."""
        self.aviary.env_rollout(n_steps)

    def close(self) -> None:
        self.aviary.disconnect()


class QuadXHoverEnv:
    """Single-env adaptor: numpy in / numpy out, the reference's signature
    (quadx_hover_env.py:29-83, quadx_base_env.py:269-301)."""

    metadata = {"render_modes": [], "render_fps": 30}

    def __init__(self, **kwargs):
        kwargs.setdefault("autoreset", False)
        self._seed = kwargs.pop("seed", None)
        self._kwargs = kwargs
        self._vec = QuadXHoverVecEnv(num_envs=1, seed=self._seed, **kwargs)
        from . import spaces

        n = self._vec.obs_dim
        self.observation_space = spaces.Box(low=-np.inf, high=np.inf, shape=(n,), dtype=np.float64)
        self.action_space = spaces.Box(low=self._vec.action_low, high=self._vec.action_high, dtype=np.float64)

    def _np_info(self, info):
        return {k: bool(v[0].item()) for k, v in info.items()}

    def reset(self, *, seed: None | int = None, options: None | dict[str, Any] = dict()):
        if seed is not None:  # the same seed must replay the same episode (gymnasium contract; tests/test_gym_envs.py:92-112)
            self._seed = int(seed)
            self._vec.aviary.reseed(self._seed)
        obs, info = self._vec.reset()
        return obs[0].double().cpu().numpy(), self._np_info(info)

    def step(self, action: np.ndarray):
        a = torch.as_tensor(np.asarray(action, dtype=np.float32).reshape(1, 4), device=self._vec.device)
        obs, rew, term, trunc, info = self._vec.step(a)
        return obs[0].double().cpu().numpy(), float(rew[0].item()), bool(term[0].item()), bool(trunc[0].item()), self._np_info(info)

    def close(self):
        self._vec.close()
