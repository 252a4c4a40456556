"""MAFixedwingDogfight on the batched stepper (BASELINE.json configs[4]).

``num_arenas`` copies of the reference's ``MAFixedwingDogfightEnv``
(/root/reference/PyFlyt/pz_envs/fixedwing_envs/ma_fixedwing_dogfight_env.py:20-833 on top of
ma_fixedwing_base_env.py:17-408), each with ``2 * team_size`` acrowing aircraft.  One fused launch per ``step``
runs 4 Aviary steps for every aircraft and, after each of them, the pairwise combat state (separation, engagement
angle, hits, healths), the engagement / boundary rewards and the termination rules; the agents of an arena sit in
adjacent lanes of a warp and exchange what they need with shuffles.

Tensors are agent-major: ``[num_arenas * A, ...]`` with the agents of arena ``g`` at rows ``g*A .. g*A + A-1`` and the
first ``team_size`` of them on team 0; ``.view(num_arenas, A, -1)`` gives the per-arena layout.  The PettingZoo dict
API of the reference maps to it as ``obs[f"uav_{k}"] == obs.view(num_arenas, A, -1)[:, k]``.

Differences from the reference that a user must know: aircraft never collide with each other (the restated engine
detects ground contact only; the reference also terminates on mid-air contact), ``flatten_observation=True`` only,
``assisted_flight=True`` only, team_size 1 or 2.  With ``autoreset`` an arena whose agents have all finished is
re-spawned on the next call (NEXT_STEP), inside the same launch.
"""

from __future__ import annotations

import numpy as np
import torch

from ..core.env_base import VecEnv, check_env_args, env_config
from ..models.tables import ENV_DOGFIGHT


class MAFixedwingDogfightVecEnv(VecEnv):
    metadata = {"render_modes": [], "name": "ma_fixedwing_dogfight"}
    _info_flags = (("out_of_bounds", 1), ("collision", 2), ("dead", 4), ("team_win", 8))

    def __init__(
        self,
        num_arenas: int = 1,
        team_size: int = 1,
        spawn_min_radius: float = 10.0,
        spawn_max_radius: float = 50.0,
        spawn_min_height: float = 20.0,
        spawn_max_height: float = 50.0,
        damage_per_hit: float = 0.003,
        lethal_distance: float = 20.0,
        lethal_angle_radians: float = 0.07,
        assisted_flight: bool = True,
        aggressiveness: float = 0.5,
        cooperativeness: float = 0.5,
        sparse_reward: bool = False,
        flatten_observation: bool = True,
        flight_dome_size: float = 800.0,
        max_duration_seconds: float = 60.0,
        agent_hz: int = 30,
        render_mode: None | str = None,
        autoreset: bool = True,
        random_spawn: bool = True,
        seed: int | None = None,
        device: str | torch.device = "cuda:0",
        env_offset: int = 0,
        inline_reset: bool = False,
    ):
        check_env_args(agent_hz, render_mode, hz_error=AssertionError)  # ma_fixedwing_base_env.py:43-48
        if not assisted_flight or not flatten_observation:
            raise ValueError("the fused dogfight kernel is built for assisted_flight=True, flatten_observation=True")
        if team_size not in (1, 2):
            raise ValueError("the fused dogfight kernel supports team_size 1 or 2")
        self.num_arenas, self.team_size = int(num_arenas), int(team_size)
        self.agents_per_arena = 2 * self.team_size
        self.num_agents = self.num_arenas * self.agents_per_arena
        self.possible_agents = [f"uav_{r}" for r in range(self.agents_per_arena)]
        cfg = env_config(ENV_DOGFIGHT, agent_hz=agent_hz, max_duration_seconds=max_duration_seconds,
                         angle_representation="euler",  # ma_fixedwing_dogfight_env.py:92
                         sparse_reward=sparse_reward, autoreset=autoreset, flight_dome_size=flight_dome_size, inline_reset=inline_reset,
                         team_size=self.team_size, damage_per_hit=float(damage_per_hit), lethal_distance=float(lethal_distance),
                         lethal_angle=float(lethal_angle_radians), aggressiveness=float(aggressiveness),
                         cooperativeness=float(cooperativeness), spawn_min_radius=float(spawn_min_radius),
                         spawn_max_radius=float(spawn_max_radius), spawn_min_height=float(spawn_min_height),
                         spawn_max_height=float(spawn_max_height),
                         randomize_drop=int(bool(random_spawn)))  # draw the spawn on device like _get_start_pos_orn
        n = self.num_agents
        super().__init__(cfg, np.zeros((n, 3)), np.zeros((n, 3)), "fixedwing", drone_options=dict(drone_model="acrowing"), seed=seed,
                         device=device, env_offset=env_offset)

    def _info(self):
        info = super()._info()
        info["health"] = self.aviary.state_tensor[30]  # DF_HEALTH row
        return info

    def set_spawn(self, start_pos, start_orn):
        """Explicit spawn poses [num_agents, 3] used by reset() when ``random_spawn=False``."""
        self.aviary.start_pos.copy_(torch.as_tensor(start_pos, dtype=torch.float32, device=self.device).reshape(-1, 3))
        self.aviary.start_orn.copy_(torch.as_tensor(start_orn, dtype=torch.float32, device=self.device).reshape(-1, 3))

    def reset(self, *, seed: int | None = None, options: dict | None = None, noise=None):
        return self._reset(noise=noise, seed=seed)
