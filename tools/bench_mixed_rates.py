"""Cost of flying the drones of one batch at several control rates (``BatchedAviary(..., mixed_control_hz=True)``).

A third of the drones of each kind.  Three batches over the same drones, each a mixed handle stepped by one launch per
``step``, all with U = 4 physics substeps per Aviary step, so that they integrate the same physics:
  uniform      every drone at 60 Hz (one control tick per Aviary step);
  tiled        QuadX at 60 / 120 / 240 Hz, fixed-wing at 60 / 120 Hz, rockets at 120 / 240 Hz, one rate per 32-drone tile of
               each kind (a warp runs its control ticks together);
  interleaved  the same rates, changing from drone to drone: the lanes of a warp run their control ticks on different substeps.
CUDA events around ``step(n_steps)`` with the library's Philox motor noise, after warm-up; the median of ``--reps``, in µs per
Aviary step.  Sizes: 3 (the reference's examples/core/02_multi_drone.py has three drones), 3 x 1 024 and 3 x 21 845 (~65 536).
One JSON line per size:

    python tools/bench_mixed_rates.py [--n-steps 10] [--reps 30] [--warmup 5]

Nothing is written to the tree."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

KINDS = ("quadx", "fixedwing", "rocket")
RATES = {"quadx": (60, 120, 240), "fixedwing": (60, 120), "rocket": (120, 240)}


def time_steps(av, n_steps, reps, warmup):
    for _ in range(warmup):
        av.step(n_steps)
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        av.step(n_steps)
        b.record()
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in ev)
    return 1e3 * ms[len(ms) // 2] / n_steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    from pyflyt_b200.core.aviary import BatchedAviary

    dev = torch.device("cuda", 0)
    prop = torch.cuda.get_device_properties(dev)
    try:  # read-only query: the power limit is part of the number
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    rng = np.random.default_rng(0)
    for per_kind in (1, 1024, 21845):
        n = 3 * per_kind
        kinds = [KINDS[i % 3] for i in range(n)]
        j = np.arange(n) // 3  # index of the drone among those of its kind: the handle's slot order within the kind
        rates = {
            "uniform": [60] * n,
            "tiled": [RATES[k][(j[i] // 32) % len(RATES[k])] for i, k in enumerate(kinds)],
            "interleaved": [RATES[k][j[i] % len(RATES[k])] for i, k in enumerate(kinds)],
        }
        ks = np.array(kinds)
        start = np.column_stack([rng.uniform(-5, 5, n), rng.uniform(-5, 5, n), rng.uniform(200, 300, n)]).astype(np.float32)
        orn = np.zeros((n, 3), dtype=np.float32)
        orn[ks == "rocket", 0] = np.pi / 2
        sp = np.zeros((n, 7), dtype=np.float32)  # QuadX mode 7 holding its start, fixed-wing at 0.8 throttle, rockets ignited at 0.6
        sp[ks == "quadx", :4] = np.column_stack([start[ks == "quadx", 0], start[ks == "quadx", 1], np.zeros(int((ks == "quadx").sum())), start[ks == "quadx", 2]])
        sp[ks == "fixedwing", 3] = 0.8
        sp[ks == "rocket", 3:5] = [1.0, 0.6]
        modes = [7 if k == "quadx" else 0 for k in kinds]
        out = {"drones": n, "n_steps": args.n_steps, "gpu": prop.name, "power_limit_w,sm_max_mhz": q}
        for name, hz in rates.items():
            av = BatchedAviary(start, orn, drone_type=kinds, drone_options=[dict(control_hz=int(h)) for h in hz], seed=0, device=dev, mixed_control_hz=True)
            assert av.updates_per_step == 4
            av.set_mode(modes)
            av.set_all_setpoints(sp)
            out[f"{name}_us_per_step"] = time_steps(av, args.n_steps, args.reps, args.warmup)
            del av
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
