"""MAQuadXHover on the batched stepper (SURVEY.md §8f, second widening row).

``num_arenas`` copies of the reference's ``MAQuadXHoverEnv``
(/root/reference/PyFlyt/pz_envs/quadx_envs/ma_quadx_hover_env.py:13-206 on top of ma_quadx_base_env.py:17-372), each
with ``A = len(start_pos)`` quadrotors.  The per-agent part (3 Aviary steps, rewards summed over them, termination rules,
observation with the PAST action and the agent's start position) is the fused CUDA step with env kind 6; the arena
bookkeeping of the PettingZoo parallel API — who is still in ``self.agents``, zero actions for the culled agents, a new
episode once every agent of an arena is done — is a handful of tensor ops here, with no host synchronisation.

Tensors are agent-major: ``[num_arenas * A, ...]`` with the agents of arena ``g`` at rows ``g*A .. g*A + A-1``; the
reference's dicts map to it as ``obs[f"uav_{k}"] == obs.view(num_arenas, A, -1)[:, k]``.

Differences a user must know: the quadrotors of an arena do not collide with each other (the restated engine detects
floor contact only); with ``autoreset`` an arena whose agents are all done is reset inside the same ``step`` call and the
returned observation of its agents is the first one of the new episode (gymnasium's SAME_STEP mode).
"""

from __future__ import annotations

from typing import Literal

import numpy as np
import torch

from ..core.env_base import AviaryEnv, check_env_args, env_config
from ..models.tables import ENV_MA_QUADX_HOVER

_DEFAULT_START = np.array([[-1.0, -1.0, 1.0], [1.0, -1.0, 1.0], [-1.0, 1.0, 1.0], [1.0, 1.0, 1.0]])  # ma_quadx_hover_env.py:39-41


class MAQuadXHoverVecEnv(AviaryEnv):
    metadata = {"render_modes": [], "name": "ma_quadx_hover"}
    _info_flags = (("out_of_bounds", 1), ("collision", 2))

    def __init__(
        self,
        num_arenas: int = 1,
        start_pos: np.ndarray = _DEFAULT_START,
        start_orn: np.ndarray | None = None,
        sparse_reward: bool = False,
        flight_mode: int = 0,
        flight_dome_size: float = 10.0,
        max_duration_seconds: float = 30.0,
        angle_representation: Literal["euler", "quaternion"] = "quaternion",
        agent_hz: int = 40,
        render_mode: None | str = None,
        autoreset: bool = True,
        seed: int | None = None,
        device: str | torch.device = "cuda:0",
        env_offset: int = 0,
    ):
        check_env_args(agent_hz, render_mode, angle_representation, hz_error=AssertionError)  # ma_quadx_base_env.py:47-52
        start_pos = np.asarray(start_pos, dtype=np.float64).reshape(-1, 3)
        start_orn = np.zeros_like(start_pos) if start_orn is None else np.asarray(start_orn, dtype=np.float64).reshape(-1, 3)
        assert start_orn.shape == start_pos.shape
        self.num_arenas, self.agents_per_arena = int(num_arenas), len(start_pos)
        self.num_agents = self.num_arenas * self.agents_per_arena
        self.possible_agents = [f"uav_{r}" for r in range(self.agents_per_arena)]
        self.autoreset = bool(autoreset)
        cfg = env_config(ENV_MA_QUADX_HOVER, agent_hz=agent_hz, max_duration_seconds=max_duration_seconds,
                         angle_representation=angle_representation, sparse_reward=sparse_reward,
                         autoreset=False,  # arenas are reset from here, with a mask
                         flight_dome_size=flight_dome_size, flight_mode=int(flight_mode))
        sp, so = np.tile(start_pos, (self.num_arenas, 1)), np.tile(start_orn, (self.num_arenas, 1))
        super().__init__(cfg, sp, so, "quadx", seed=seed, device=device, env_offset=env_offset)
        n = self.num_agents
        self.alive = torch.ones(n, dtype=torch.bool, device=self.device)  # the agents still in self.agents
        self._mask = torch.zeros(n, dtype=torch.uint8, device=self.device)
        self._act = torch.zeros((n, 4), dtype=torch.float32, device=self.device)

    def _info(self):
        info = super()._info()
        info["alive"] = self.alive
        return info

    def reset(self, *, seed: int | None = None, options: dict | None = None, noise=None):
        obs, info = self._reset(noise=noise, seed=seed)
        self.alive.fill_(True)
        return obs, info

    def step(self, actions: torch.Tensor, noise=None):
        """``actions`` [num_agents, 4].  Returns (obs, reward, term, trunc, info); rows of culled agents hold their frozen
        last values with reward 0 and term = True (the reference simply has no entry for them)."""
        a = self.aviary
        actions = torch.as_tensor(actions, dtype=torch.float32, device=self.device).reshape(self.num_agents, 4)
        torch.mul(actions, self.alive[:, None], out=self._act)  # current_actions *= 0 for the agents not in self.agents
        was_alive = self.alive.clone()
        a.env_step(actions=self._act, noise=noise)
        term, trunc = a.term.bool(), a.trunc.bool()
        reward = a.reward * was_alive
        term = term | ~was_alive
        trunc = trunc & was_alive
        self.alive &= ~(term | trunc)  # cull for the next round (ma_quadx_base_env.py:365-370)
        if self.autoreset:
            A = self.agents_per_arena
            done = ~self.alive.view(self.num_arenas, A).any(dim=1)
            self._mask.copy_(done.repeat_interleave(A))
            # SAME_STEP autoreset overwrites the rows of a finished arena with the first observation of its next episode: keep the
            # terminal observation (gymnasium's info["final_obs"]; bootstrapping on truncation needs it)
            torch.where(self._mask.bool()[:, None], a.obs, a.final_obs, out=a.final_obs)
            a.env_reset(mask=self._mask)  # no-op for the arenas that are still running; writes their first observation otherwise
            self.alive |= self._mask.bool()
        info = self._info()
        if self.autoreset:
            info["final_obs"] = a.final_obs      # valid in the rows where info["reset"] is set
            info["reset"] = self._mask.bool()
        return a.obs, reward, term, trunc, info
