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

from ..core.env_base import VecEnv, check_env_args, env_config
from ..models.tables import ENV_ROCKET_LANDING


class RocketLandingVecEnv(VecEnv):
    _info_flags = (("out_of_bounds", 1), ("fatal_collision", 2), ("env_complete", 4))

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
        autoreset_mode: str = "next_step",
        contact_response: bool = True,
    ):
        """``randomize_drop`` / ``accelerate_drop`` are the reference's ``reset(options=...)`` switches
        (rocket_landing_env.py:94-98: both on when ``options=None``).  ``contact_response`` (default on): the legs / body push back
        against the pad and the ground (sequential-impulse contact with friction, a restatement of Bullet's, DESIGN.md), so a
        gentle touchdown RESTS on the pad and the env can report ``env_complete`` like the reference; off = contact flag only."""
        check_env_args(agent_hz, render_mode, angle_representation)
        self.num_envs = int(num_envs)
        cfg = env_config(ENV_ROCKET_LANDING, agent_hz=agent_hz, max_duration_seconds=max_duration_seconds,
                         angle_representation=angle_representation, sparse_reward=sparse_reward, autoreset=autoreset,
                         flight_dome_size=float("inf"), inline_reset=inline_reset, autoreset_mode=autoreset_mode, ceiling=float(ceiling),
                         max_displacement=float(max_displacement), randomize_drop=int(bool(randomize_drop)),
                         accelerate_drop=int(bool(accelerate_drop)), contact_response=int(bool(contact_response)))
        sp = np.tile(np.array([[0.0, 0.0, ceiling * 0.9]]), (self.num_envs, 1))  # rocket_landing_env.py:60
        so = np.zeros((self.num_envs, 3))
        super().__init__(cfg, sp, so, "rocket", drone_options=dict(starting_fuel_ratio=0.05), seed=seed, device=device, env_offset=env_offset)
        self.action_low = np.array([-1.0, -1.0, -1.0, 0.0, 0.0, -1.0, -1.0])  # rocket_base_env.py:82-107
        self.action_high = np.ones(7)
