"""MAFixedwingDogfight with the two aircraft of an arena on DIFFERENT ranks (BASELINE.json configs[4] as written:
"NCCL all-gather for inter-agent distance").

The default :class:`MAFixedwingDogfightVecEnv` shards whole arenas over ranks and needs no collective; this variant
exists for the layout the benchmark names, where a learner keeps team 0 on one set of GPUs and team 1 on another.
Global agent id ``gid = member * num_arenas + arena``; rank ``r`` of ``world`` owns the contiguous slice
``[r * n_local, (r + 1) * n_local)`` with ``n_local = 2 * num_arenas / world``.  Every Aviary step is

    pfb_dogfight_physics  ->  all_gather_into_tensor(payload [n_local, 20])  ->  pfb_dogfight_combat

(ma_fixedwing_dogfight_env.py:346-465 `_compute_agent_states` is the part that reads other agents).  1-vs-1 arenas,
no autoreset (``reset`` is a collective call), explicit or host-drawn spawns.  With ``group=None`` and no initialised
process group it runs single-rank (the "gather" is a copy), which is how the parity tests drive it on one GPU.

``exchange="peer"`` fuses the exchange into the physics kernel: the payload table lives in symmetric (peer-mapped)
memory, every rank's kernel stores its payloads straight into ALL ranks' tables over NVLink, and the only thing left
between the two kernels is a cross-rank barrier — no all-gather launch, no staging buffer:

    pfb_dogfight_physics_peer (peer stores)  ->  symmetric-memory barrier  ->  pfb_dogfight_combat

The table is double-buffered by Aviary-step parity: a rank that runs ahead writes the other half while a slower rank
still reads its own.  ``exchange="peer-signal"`` also removes the barrier launch: the last CTA of the physics kernel raises
this rank's flag in every rank's (symmetric) flag array, and the combat kernel spins on its own array before it reads.
"""

from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist

from ..core.aviary import BatchedAviary
from ..core.env_base import env_config
from ..models.tables import ENV_DOGFIGHT

PAYLOAD = 20


def split_agent_range(num_arenas: int, rank: int, world_size: int) -> tuple[int, int]:
    """Global agent ids owned by ``rank``; the all-gather needs equal slices, so 2*num_arenas % world_size == 0."""
    total = 2 * int(num_arenas)
    if total % world_size:
        raise ValueError(f"2 * num_arenas = {total} must be divisible by the world size {world_size}")
    n_local = total // world_size
    return rank * n_local, (rank + 1) * n_local


def spawn_poses(num_arenas: int, spawn_min_radius: float, spawn_max_radius: float, seed: int) -> tuple[np.ndarray, np.ndarray]:
    """ma_fixedwing_dogfight_env.py:177-217 for every arena, in global-agent order [2 * num_arenas, 3] (same on all ranks)."""
    rs = np.random.RandomState(seed)
    base = rs.uniform(0.0, 2 * np.pi, size=(1, num_arenas))
    rad = np.pi * np.arange(2)[:, None] + base  # pi / team_size * index, team_size = 1
    radius = rs.uniform(spawn_min_radius, spawn_max_radius, size=(2, num_arenas))
    height = rs.uniform(spawn_min_radius, spawn_max_radius, size=(2, num_arenas))  # (sic) the reference uses the radius range
    pos = np.stack([radius * np.cos(rad), radius * np.sin(rad), height], axis=-1).reshape(-1, 3)
    orn = np.zeros_like(pos)
    orn[:, 2] = (rad + rs.random_sample((2, num_arenas)) * np.pi / 8.0).reshape(-1)
    return pos, orn


class MAFixedwingDogfightSplitEnv:
    def __init__(self, num_arenas: int, damage_per_hit: float = 0.003, lethal_distance: float = 20.0, lethal_angle_radians: float = 0.07,
                 aggressiveness: float = 0.5, cooperativeness: float = 0.5, sparse_reward: bool = False, flight_dome_size: float = 800.0,
                 max_duration_seconds: float = 60.0, agent_hz: int = 30, spawn_min_radius: float = 10.0, spawn_max_radius: float = 50.0,
                 seed: int | None = None, device: str | torch.device = "cuda:0", group=None, single_rank: bool = False,
                 exchange: str = "nccl"):
        assert 120 % agent_hz == 0
        self.group = group
        self.distributed = dist.is_available() and dist.is_initialized() and not single_rank
        self.rank = dist.get_rank(group) if self.distributed else 0
        self.world = dist.get_world_size(group) if self.distributed else 1
        self.num_arenas = int(num_arenas)
        self.first_gid, end = split_agent_range(num_arenas, self.rank, self.world)
        self.n_local = end - self.first_gid
        self.seed = 0 if seed is None else int(seed)
        self.spawn = (float(spawn_min_radius), float(spawn_max_radius))
        cfg = env_config(ENV_DOGFIGHT, agent_hz=agent_hz, max_duration_seconds=max_duration_seconds, angle_representation="euler",
                         sparse_reward=sparse_reward, autoreset=False, flight_dome_size=flight_dome_size, team_size=1,
                         damage_per_hit=float(damage_per_hit), lethal_distance=float(lethal_distance), lethal_angle=float(lethal_angle_radians),
                         aggressiveness=float(aggressiveness), cooperativeness=float(cooperativeness),
                         spawn_min_radius=self.spawn[0], spawn_max_radius=self.spawn[1],
                         spawn_min_height=self.spawn[0], spawn_max_height=self.spawn[1])  # (sic) heights take the radius range, as spawn_poses
        self.config = cfg
        n = self.n_local
        # env_offset = first global agent id: the noise streams are keyed by gid, so they do not depend on the world size
        self.aviary = BatchedAviary(np.zeros((n, 3)), np.zeros((n, 3)), drone_type="fixedwing", drone_options=dict(drone_model="acrowing"),
                                    seed=seed, device=device, env_config=cfg, env_offset=self.first_gid)
        self.device = self.aviary.device
        self.payload = torch.zeros(n, PAYLOAD, device=self.device)
        self.table = torch.zeros(2 * self.num_arenas, PAYLOAD, device=self.device)
        self.ratio = cfg.env_step_ratio
        self.collectives = 0
        self._resets = 0
        assert exchange in ("nccl", "peer", "peer-signal")
        self.exchange = exchange
        self._symm = None
        if exchange in ("peer", "peer-signal"):
            na = 2 * self.num_arenas
            if self.world > 1:
                import torch.distributed._symmetric_memory as symm_mem

                grp = group if group is not None else dist.group.WORLD
                self._tables = symm_mem.empty((2, na, PAYLOAD), dtype=torch.float32, device=self.device)
                self._tables.zero_()
                self._symm = symm_mem.rendezvous(self._tables, grp)
                ptrs = [int(p) for p in self._symm.buffer_ptrs]
                self._flags = symm_mem.empty((32,), dtype=torch.int32, device=self.device)
                self._flags.zero_()
                self._symm_flags = symm_mem.rendezvous(self._flags, grp)
                fptrs = [int(p) for p in self._symm_flags.buffer_ptrs]
                self._symm.barrier(channel=0)  # everybody's tables and flags are zeroed before anyone stores into them
            else:
                self._tables = torch.zeros((2, na, PAYLOAD), dtype=torch.float32, device=self.device)
                ptrs = [self._tables.data_ptr()]
                self._flags = torch.zeros(32, dtype=torch.int32, device=self.device)
                fptrs = [self._flags.data_ptr()]
            self._peers = torch.tensor(ptrs, dtype=torch.int64, device=self.device)
            self._peer_flags = torch.tensor(fptrs, dtype=torch.int64, device=self.device)

    def _gather(self) -> None:
        if self.world > 1:
            dist.all_gather_into_tensor(self.table, self.payload, group=self.group)
        else:
            self.table.copy_(self.payload)
        self.collectives += 1

    def _physics(self, **kw) -> torch.Tensor:
        """One Aviary step (or the reset) + the exchange; returns the payload table to read."""
        a = self.aviary
        if self.exchange == "nccl":
            a.dogfight_physics(self.payload, **kw)
            self._gather()
            return self.table
        phase = self.collectives & 1
        na = 2 * self.num_arenas
        self.collectives += 1
        if self.exchange == "peer-signal":
            a.dogfight_physics_peer(self._peers, self.world, (phase * na + self.first_gid) * PAYLOAD, peer_flags=self._peer_flags, rank=self.rank,
                                    epoch=self.collectives, **kw)
            return self._tables[phase]
        a.dogfight_physics_peer(self._peers, self.world, (phase * na + self.first_gid) * PAYLOAD, **kw)
        if self._symm is not None:
            self._symm.barrier(channel=0)  # every rank's peer stores have landed; enqueued on the current stream
        return self._tables[phase]

    def _combat(self, table: torch.Tensor, last: int) -> None:
        if self.exchange == "peer-signal":
            self.aviary.dogfight_combat_wait(table, self.first_gid, self.num_arenas, last, self._flags, self.world, self.collectives)
        else:
            self.aviary.dogfight_combat(table, self.first_gid, self.num_arenas, last)

    def reset(self, start_pos=None, start_orn=None, noise=None):
        """Collective.  ``start_pos`` / ``start_orn``: [2 * num_arenas, 3] in global-agent order (all ranks pass the same)."""
        if start_pos is None:
            start_pos, start_orn = spawn_poses(self.num_arenas, *self.spawn, seed=self.seed + self._resets)
        self._resets += 1
        a = self.aviary
        sl = slice(self.first_gid, self.first_gid + self.n_local)
        a.start_pos.copy_(torch.as_tensor(np.asarray(start_pos, dtype=np.float32)[sl], device=self.device))
        a.start_orn.copy_(torch.as_tensor(np.asarray(start_orn, dtype=np.float32)[sl], device=self.device))
        table = self._physics(noise=noise, do_reset=True)
        self._combat(table, last=2)
        a.info_bits.zero_()
        return a.obs

    def step(self, actions: torch.Tensor, noise: torch.Tensor | None = None):
        """``actions`` [n_local, 4] for this rank's agents; ``noise`` (parity tests) [ratio * 2, n_local]."""
        a = self.aviary
        actions = torch.as_tensor(actions, dtype=torch.float32, device=self.device).contiguous()
        if self.exchange == "peer-signal" and noise is None:  # nothing between the kernels needs the host: one call
            a.dogfight_split_step(actions, self._peers, self._peer_flags, self._tables, self._flags, self.world, self.rank, self.collectives + 1,
                                  self.first_gid, self.num_arenas)
            self.collectives += self.ratio
            return a.obs, a.reward, a.term.bool(), a.trunc.bool()
        for k in range(self.ratio):
            nz = None if noise is None else noise[2 * k:]
            table = self._physics(actions=actions, noise=nz, first=(k == 0), aviary_index=k)
            self._combat(table, last=int(k == self.ratio - 1))
        return a.obs, a.reward, a.term.bool(), a.trunc.bool()

    def close(self) -> None:
        self.aviary.disconnect()
