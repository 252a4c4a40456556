"""Per-step cost of SAME_STEP autoreset (``autoreset_mode="same_step"``) against NEXT_STEP, for the four env kinds at the batch
sizes bench.py and tools/bench_workloads.py use.  Same method as bench.py's per-step leg: the L2 flushed before every timed
call, a CUDA-event pair around it, the median over the calls.  Two legs per (kind, mode):

    step       rollout(1): one env step with on-device random actions (one step launch; QuadX-Hover SAME_STEP adds the top-up
               launch, the tail kinds add the side-stream rebuild)
    rollout16  rollout(16), reported per env step (QuadX-Hover: one fused launch of 16 steps; the tail kinds: 16 single steps)

One JSON line per (kind, mode), with the device, its power limit and its SM clock.

    python tools/bench_same_step.py [--steps 100] [--warmup 10] [--only hover]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

KINDS = {  # kind -> (VecEnv class path, envs per GPU, extra constructor arguments)
    "QuadX-Hover": ("pyflyt_b200.gym_envs.quadx_hover_env:QuadXHoverVecEnv", 65536),
    "QuadX-Waypoints": ("pyflyt_b200.gym_envs.quadx_waypoints_env:QuadXWaypointsVecEnv", 65536),
    "Fixedwing-Waypoints": ("pyflyt_b200.gym_envs.fixedwing_waypoints_env:FixedwingWaypointsVecEnv", 16384),
    "Rocket-Landing": ("pyflyt_b200.gym_envs.rocket_landing_env:RocketLandingVecEnv", 16384),
}


def device_info():
    """name, power limit and SM clocks, read (not set) through nvidia-smi"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock_idle": sm, "sm_clock_max": sm_max}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(0)}


def median_ms(fn, K, W, dev):
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    for _ in range(W):
        fn()
    torch.cuda.synchronize(dev)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(K)]
    for k in range(K):
        flush.fill_(float(k))
        ev[k][0].record()
        fn()
        ev[k][1].record()
    torch.cuda.synchronize(dev)
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    info = device_info()
    for kind, (path, n) in KINDS.items():
        if args.only and args.only.lower() not in kind.lower():
            continue
        mod, cls = path.split(":")
        Env = getattr(__import__(mod, fromlist=[cls]), cls)
        for mode in ("next_step", "same_step"):
            env = Env(num_envs=n, seed=1, device=dev, autoreset_mode=mode)
            env.reset()
            l0 = env.aviary.launch_count
            env.rollout(1)
            launches = env.aviary.launch_count - l0
            finished = []
            for _ in range(50):
                env.rollout(1)
                finished.append(int((env.aviary.term | env.aviary.trunc).sum()))
            step = median_ms(lambda: env.rollout(1), args.steps, args.warmup, dev)
            r16 = median_ms(lambda: env.rollout(16), max(args.steps // 4, 10), max(args.warmup // 4, 2), dev) / 16
            line = {"kind": kind, "autoreset_mode": mode, "envs": n, "step_us": round(step * 1e3, 2), "rollout16_us_per_step": round(r16 * 1e3, 2),
                    "env_steps_per_s_step": n / (step * 1e-3), "env_steps_per_s_rollout16": n / (r16 * 1e-3), "launches_per_step": launches,
                    "finished_per_step_mean": float(np.mean(finished)), "steps": args.steps, "l2": "flushed before every timed call", **info}
            print(json.dumps(line), flush=True)
            env.close()


if __name__ == "__main__":
    main()
