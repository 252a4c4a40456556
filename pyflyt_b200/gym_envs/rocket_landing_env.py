"""Rocket-Landing on the batched stepper (BASELINE.json configs[3]).

N copies of the reference's ``RocketLandingEnv``
(/root/reference/PyFlyt/gym_envs/rocket_envs/rocket_landing_env.py:17-263 on top of rocket_base_env.py:17-391):
one fused launch per ``step`` runs 3 Aviary steps (6 physics substeps of body drag + 4 finlets + gimballed
booster with fuel burn + variable-mass composite body), the landing reward, termination rules and the
30-float observation.

Contact (SURVEY.md §8f #3): with ``contact_response`` (default) the legs and the body push back against the pad and the
ground — sequential-impulse normal + Coulomb friction on the collision primitives' corner / rim points, a restatement of a
Bullet-like solver (DESIGN.md §4) — so a touchdown below 1 m/s RESTS on the pad and the env reports ``env_complete`` like the
reference's (tests/test_contact_response.py flies three touchdown episodes of the unmodified reference env through it).
``contact_response=False`` keeps the round-1 behaviour: contact is a flag only.
"""

from __future__ import annotations

from typing import Literal

import numpy as np
import torch

from ..core.aviary import BatchedAviary
from ..models import PfbEnvConfig
from ..models.tables import ENV_ROCKET_LANDING


class RocketLandingVecEnv:
    metadata = {"render_modes": [], "render_fps": 30}

    def __init__(
        self,
        num_envs: int = 1,
        sparse_reward: bool = False,
        ceiling: float = 500.0,
        max_displacement: float = 200.0,
        max_duration_seconds: float = 30.0,
        angle_representation: Literal["euler", "quaternion"] = "quaternion",
        agent_hz: int = 40,
        render_mode: None | str = None,
        randomize_drop: bool = True,
        accelerate_drop: bool = True,
        autoreset: bool = True,
        seed: int | None = None,
        device: str | torch.device = "cuda:0",
        env_offset: int = 0,
        inline_reset: bool = False,
        contact_response: bool = True,
    ):
        """``randomize_drop`` / ``accelerate_drop`` are the reference's ``reset(options=...)`` switches
        (rocket_landing_env.py:94-98: both on when ``options=None``).  ``contact_response`` (default on): the legs / body push back
        against the pad and the ground (sequential-impulse contact with friction, a restatement of Bullet's, DESIGN.md), so a
        gentle touchdown RESTS on the pad and the env can report ``env_complete`` like the reference; off = contact flag only."""
        if 120 % agent_hz != 0:
            lowest = int(120 / (int(120 / agent_hz) + 1))
            highest = int(120 / int(120 / agent_hz))
            raise ValueError(f"`agent_hz` must be round denominator of 120, try {lowest} or {highest}.")
        if render_mode is not None:
            raise ValueError("rendering is out of scope for the batched stepper (SURVEY.md §2 row 21)")
        if angle_representation not in ("euler", "quaternion"):
            raise ValueError(f"angle_representation must be either `euler` or `quaternion`, not {angle_representation}")
        self.num_envs = int(num_envs)
        cfg = PfbEnvConfig()
        cfg.env_kind = ENV_ROCKET_LANDING
        cfg.flight_mode = 0
        cfg.env_step_ratio = int(120 / agent_hz)
        cfg.max_steps = int(agent_hz * max_duration_seconds)
        cfg.angle_representation = 0 if angle_representation == "euler" else 1
        cfg.sparse_reward = int(bool(sparse_reward))
        cfg.autoreset = int(bool(autoreset))
        cfg.warmup_steps = 10
        cfg.ceiling = float(ceiling)
        cfg.max_displacement = float(max_displacement)
        cfg.randomize_drop = int(bool(randomize_drop))
        cfg.accelerate_drop = int(bool(accelerate_drop))
        cfg.flight_dome_size = float("inf")
        cfg.inline_reset = int(bool(inline_reset))  # tests: spare-copy resets must equal inline ones bit for bit
        cfg.contact_response = int(bool(contact_response))
        self.config = cfg
        sp = np.tile(np.array([[0.0, 0.0, ceiling * 0.9]]), (self.num_envs, 1))  # rocket_landing_env.py:60
        so = np.zeros((self.num_envs, 3))
        self.aviary = BatchedAviary(sp, so, drone_type="rocket", drone_options=dict(starting_fuel_ratio=0.05), seed=seed, device=device,
                                    env_config=cfg, env_offset=env_offset)
        self.device = self.aviary.device
        self.obs_dim = self.aviary.obs_dim
        self.action_low = np.array([-1.0, -1.0, -1.0, 0.0, 0.0, -1.0, -1.0])  # rocket_base_env.py:82-107
        self.action_high = np.ones(7)

    def _info(self):
        bits = self.aviary.info_bits
        return {"out_of_bounds": (bits & 1).bool(), "fatal_collision": (bits & 2).bool(), "env_complete": (bits & 4).bool()}

    def reset(self, *, seed: int | None = None, options: dict | None = None, mask=None, noise=None):
        obs = self.aviary.env_reset(mask=mask, noise=noise, seed=seed)
        if mask is None:
            self.aviary.info_bits.zero_()
        return obs, self._info()

    def step(self, actions: torch.Tensor, noise=None):
        a = self.aviary
        if not (torch.is_tensor(actions) and actions.is_cuda and actions.dtype == torch.float32 and actions.is_contiguous()):
            a.setpoints.copy_(torch.as_tensor(actions, dtype=torch.float32, device=self.device).reshape(self.num_envs, 7))
            actions = None
        a.env_step(actions=actions, noise=noise)
        return a.obs, a.reward, a.term.bool(), a.trunc.bool(), self._info()

    def rollout(self, n_steps: int) -> None:
        self.aviary.env_rollout(n_steps)

    def close(self) -> None:
        self.aviary.disconnect()
