"""What the floor contact response (``BatchedAviary(contact_response=True)``) costs an Aviary step.  The median of CUDA-event
pairs around ``step(n_steps)`` with the library's Philox motor noise, after warm-up; one JSON line per case, for cf2x at
--drones and fixed-wing at --fw-drones:

    a_off_free     contact off, free flight far above the floor
    b_on_free      contact on, the same free flight (the solver is never entered: its branch is cold)
    c_on_resting   contact on, every drone resting on the floor (the solver runs on every substep of every drone)
    d_on_one_per_tile  contact on, one resting drone per 32-drone tile, the rest in free flight (every warp waits for one solver)

(a) and (b) are timed alternately, --pairs times each, to show the run-to-run spread next to their difference.

    python tools/bench_contact_response.py [--drones 65536] [--fw-drones 16384] [--n-steps 10] [--reps 20] [--warmup 5]

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


def time_steps(av, n_steps, reps, warmup, dev):
    for _ in range(warmup):
        av.step(n_steps)
    torch.cuda.synchronize(dev)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        av.step(n_steps)
        b.record()
    torch.cuda.synchronize(dev)
    ms = sorted(a.elapsed_time(b) for a, b in ev)
    return ms[len(ms) // 2]  # median launch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--drones", type=int, default=65536)
    ap.add_argument("--fw-drones", type=int, default=16384)
    ap.add_argument("--n-steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--pairs", type=int, default=3)
    args = ap.parse_args()
    from pyflyt_b200.core.aviary import BatchedAviary

    dev = torch.device("cuda", 0)
    prop = torch.cuda.get_device_properties(dev)
    try:  # read-only query: the power limit and clock are part of the number
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""

    def build(kind, n, contact, resting):
        """free flight at 40-60 m (cf2x: mode 7 position hold; fixed-wing: mode 0 cruise); `resting` drones start on the floor
        in mode -1 with idle motors (cf2x) or zero throttle (fixed-wing) and stay there"""
        rng = np.random.default_rng(0)
        start = np.column_stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(40, 60, n)]).astype(np.float32)
        rest_z = 0.009 if kind == "quadx" else 0.1
        start[resting, 2] = rest_z
        opts = dict(drone_model="cf2x") if kind == "quadx" else dict(drone_model="fixedwing")
        av = BatchedAviary(start, np.zeros((n, 3), dtype=np.float32), drone_type=kind, drone_options=opts, seed=0, device=dev, contact_response=contact)
        if kind == "quadx":
            modes = np.where(resting, -1, 7)
            sp = np.column_stack([start[:, :2], np.zeros(n), start[:, 2]])
            sp[resting] = 0.0
        else:
            modes = np.zeros(n, dtype=int)
            sp = np.column_stack([np.zeros((n, 3)), np.where(resting, 0.0, 0.6), np.zeros((n, 2))])
        av.set_mode(int(modes[0]) if (modes == modes[0]).all() else modes.tolist())
        av.set_all_setpoints(torch.as_tensor(sp, dtype=torch.float32, device=dev))
        av.step(60)  # resting drones settle onto the floor
        return av

    def report(case, kind, n, av, ms):
        z = av.all_states[:, 3, 2]
        print(json.dumps({"case": case, "kind": kind, "drones": n, "n_steps": args.n_steps, "gpu": prop.name, "power_limit_w,sm_mhz,sm_max_mhz": q,
                          "ms_per_launch": ms, "drone_steps_per_s": n * args.n_steps / (ms * 1e-3),
                          "in_contact": int(av.contact_array.sum()), "min_z": float(z.min())}), flush=True)

    for kind, n in (("quadx", args.drones), ("fixedwing", args.fw_drones)):
        none = np.zeros(n, dtype=bool)
        avs = {"a_off_free": build(kind, n, False, none), "b_on_free": build(kind, n, True, none)}
        for _ in range(args.pairs):
            for case in ("a_off_free", "b_on_free"):
                report(case, kind, n, avs[case], time_steps(avs[case], args.n_steps, args.reps, args.warmup, dev))
        del avs
        for case, resting in (("c_on_resting", np.ones(n, dtype=bool)), ("d_on_one_per_tile", np.arange(n) % 32 == 0)):
            av = build(kind, n, True, resting)
            report(case, kind, n, av, time_steps(av, args.n_steps, args.reps, args.warmup, dev))
            del av


if __name__ == "__main__":
    main()
