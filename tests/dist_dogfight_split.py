"""torchrun worker for the split dogfight (one process per GPU, NCCL): every rank steps its slice of the agents, the
payload table is all-gathered each Aviary step, and the result must equal the single-rank run of the same arenas.
Launched by tests/test_dogfight_split.py; also usable by hand:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29533 tests/dist_dogfight_split.py
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from pyflyt_b200.pz_envs import MAFixedwingDogfightSplitEnv, spawn_poses  # noqa: E402


def scenario(num_arenas, steps, seed=5):
    rng = np.random.default_rng(seed)
    n = 2 * num_arenas
    pos, orn = spawn_poses(num_arenas, 10.0, 50.0, seed)
    orn[:num_arenas:2, 2] += np.pi  # every other arena: member 0 turns inwards
    orn[num_arenas::2, 2] += np.pi
    nz0 = rng.normal(1.0, 1.0, (20, n)).astype(np.float32)
    acts = (rng.uniform(-1, 1, (steps, n, 4)) * 0.4).astype(np.float32)
    nz = rng.normal(1.0, 1.0, (steps, 8, n)).astype(np.float32)
    return pos, orn, nz0, acts, nz


def run(num_arenas, steps, device, single_rank=False, exchange="nccl", wind=None):
    """``wind``: an AnalyticWind registered on the rank's Aviary before the reset, or None"""
    pos, orn, nz0, acts, nz = scenario(num_arenas, steps)
    env = MAFixedwingDogfightSplitEnv(num_arenas, seed=3, device=device, lethal_distance=150.0, lethal_angle_radians=1.0, damage_per_hit=0.05,
                                      single_rank=single_rank, exchange=exchange)
    if wind is not None:
        env.aviary.register_wind_field(wind)
    lo, hi = env.first_gid, env.first_gid + env.n_local
    dev = env.device
    out = [env.reset(pos, orn, noise=torch.as_tensor(nz0[:, lo:hi].copy(), device=dev)).clone()]
    rew, term = [], []
    for k in range(steps):
        o, r, te, tr = env.step(torch.as_tensor(acts[k, lo:hi].copy(), device=dev), noise=torch.as_tensor(nz[k][:, lo:hi].copy(), device=dev))
        out.append(o.clone()); rew.append(r.clone()); term.append(te.clone())
    return torch.stack(out), torch.stack(rew), torch.stack(term), env


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl")
    num_arenas, steps = 4096, 20
    exchange = os.environ.get("PFB_SPLIT_EXCHANGE", "nccl")
    obs, rew, term, env = run(num_arenas, steps, f"cuda:{torch.cuda.current_device()}", exchange=exchange)
    lo, hi = env.first_gid, env.first_gid + env.n_local
    # gather everything on every rank and compare with a local single-rank run of all agents
    def gather(x):
        parts = [torch.empty_like(x) for _ in range(world)]
        dist.all_gather(parts, x.contiguous())
        return torch.cat(parts, dim=1)
    g_obs, g_rew, g_term = gather(obs), gather(rew), gather(term.to(torch.uint8))
    if rank == 0:
        s_obs, s_rew, s_term, _ = run(num_arenas, steps, "cuda:0", single_rank=True)
        assert torch.equal(g_obs, s_obs), float((g_obs - s_obs).abs().max())
        assert torch.equal(g_rew, s_rew) and torch.equal(g_term, s_term.to(torch.uint8))
        assert int(s_term.sum()) > 0
        print(f"SPLIT_OK world={world} exchange={exchange} collectives={env.collectives} terminations={int(s_term[-1].sum())}")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
