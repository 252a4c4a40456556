"""QuadX-Hover env-steps/s with several vehicle models in one batch (``drone_options`` = one dict per env).  Same method as
bench.py's per-step leg: the L2 flushed before every timed step, a CUDA-event pair around each ``rollout(1)`` (one step launch,
autoreset with the spare pipeline, on-device random actions); then the fused ``rollout(16)``.  One JSON line per layout:

    uniform      every env flies cf2x (the single-table kernels)
    k2_tile      cf2x / primitive_drone, one model per 32-env tile (every warp reads one table)
    k2_env       cf2x / primitive_drone interleaved per env (every warp reads both tables)
    k16_random   16 tables (cf2x and primitive_drone variants that differ in drag), drawn at random per env
    k16_tile     the same 16 tables and counts, envs sorted by model (a tile holds one model, or two at a boundary)

    python tools/bench_mixed_models.py [--envs 65536] [--steps 100] [--warmup 10]

The variant vehicle files go to a temporary directory; nothing is written to the tree."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
VEHICLES = os.path.join(ROOT, "tests", "golden", "vehicles")


def variants(tmp, k):
    """k vehicle dirs under tmp: cf2x and primitive_drone copies whose drag_coef_xyz differ."""
    out = []
    for j in range(k):
        base = "cf2x" if j % 2 == 0 else "primitive_drone"
        name = f"{base}_v{j}"
        os.makedirs(os.path.join(tmp, name))
        shutil.copy(os.path.join(VEHICLES, base, f"{base}.urdf"), os.path.join(tmp, name, f"{name}.urdf"))
        text = open(os.path.join(VEHICLES, base, f"{base}.yaml")).read()
        key = "drag_coef_xyz:"
        i = text.index(key)
        end = text.index("\n", i)
        value = float(text[i + len(key) : end]) * (1.0 + 0.02 * j)
        with open(os.path.join(tmp, name, f"{name}.yaml"), "w") as fh:
            fh.write(text[:i] + f"{key} {value!r}" + text[end:])
        out.append(dict(drone_model=name, model_dir=tmp))
    return out


def time_rollout(env, chunk, K, W, dev):
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    for _ in range(W):
        env.rollout(chunk)
    torch.cuda.synchronize(dev)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(K)]
    for k in range(K):
        flush.fill_(float(k))
        ev[k][0].record()
        env.rollout(chunk)
        ev[k][1].record()
    torch.cuda.synchronize(dev)
    return sum(a.elapsed_time(b) for a, b in ev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverVecEnv

    dev = torch.device("cuda", 0)
    n, K, W = args.envs, args.steps, args.warmup
    cf2x, prim = dict(drone_model="cf2x"), dict(drone_model="primitive_drone")
    tmp = tempfile.mkdtemp(prefix="pfb_variants_")
    try:
        layouts = {
            "uniform": cf2x,
            "k2_tile": [cf2x if (i // 32) % 2 == 0 else prim for i in range(n)],
            "k2_env": [cf2x if i % 2 == 0 else prim for i in range(n)],
        }
        v16 = variants(tmp, 16)
        pick = np.random.default_rng(0).integers(0, 16, n)
        layouts["k16_random"] = [v16[j] for j in pick]
        layouts["k16_tile"] = [v16[j] for j in np.sort(pick)]  # the same envs per model, grouped: 32-env tiles see one table (mostly)
        prop = torch.cuda.get_device_properties(dev)
        try:  # read-only query: the power limit is part of the number
            q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
        except (OSError, subprocess.SubprocessError):
            q = ""
        for name, opts in layouts.items():
            if args.only and name not in args.only.split(","):
                continue
            env = QuadXHoverVecEnv(num_envs=n, seed=0, drone_options=opts, device=dev)
            env.reset()
            ms1 = time_rollout(env, 1, K, W, dev)
            ms16 = time_rollout(env, 16, max(1, K // 16), 2, dev)
            k = len(env.aviary.models)
            env.close()
            print(json.dumps({"layout": name, "models": k, "envs": n, "gpu": prop.name, "power_limit_w,sm_max_mhz": q,
                              "env_steps_per_s": n * K / (ms1 * 1e-3), "ms_per_step": ms1 / K,
                              "fused_env_steps_per_s": n * 16 * max(1, K // 16) / (ms16 * 1e-3)}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
