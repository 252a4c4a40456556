"""What static bodies (``BatchedAviary.loadURDF``, DESIGN.md §4h) cost an Aviary step.  The median of CUDA-event pairs around
``step(n_steps)`` with the library's Philox motor noise, after warm-up; one JSON line per case: QuadX (cf2x, mode 7 position
hold) at --drones and fixed-wing (mode 0 cruise) and rocket (unpowered, falling from 400-600 m) at --fw-drones, with 0, 1 and 8 static bodies,
with the contact response off and on.  The bodies are 1 m platforms spread around the drones, each drone's world holding them at
the same poses; the drones fly high above them, so the surface test runs on every substep but no contact is made (the cost of
the bodies, not of the solver).  Each case is timed --pairs times, interleaved with the others, to show the run-to-run spread.

    python tools/bench_static_bodies.py [--drones 65536] [--fw-drones 16384] [--n-steps 10] [--reps 20] [--warmup 5] [--pairs 2]

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
PLATFORM = os.path.join(ROOT, "tests", "golden", "static", "platform_box.urdf")


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
    ap.add_argument("--pairs", type=int, default=2)
    args = ap.parse_args()
    from pyflyt_b200.core.aviary import BatchedAviary

    dev = torch.device("cuda", 0)
    prop = torch.cuda.get_device_properties(dev)
    try:  # read-only query: the power limit and clock are part of the number
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""

    def build(kind, n, contact, bodies):
        rng = np.random.default_rng(0)
        lo, hi = (400.0, 600.0) if kind == "rocket" else (40.0, 60.0)  # an unpowered rocket falls: it must not reach the floor while timed
        start = np.column_stack([rng.uniform(-10, 10, n), rng.uniform(-10, 10, n), rng.uniform(lo, hi, n)]).astype(np.float32)
        av = BatchedAviary(start, np.zeros((n, 3), dtype=np.float32), drone_type=kind, seed=0, device=dev, contact_response=contact)
        for k in range(bodies):
            a = 2 * np.pi * k / 8
            av.loadURDF(PLATFORM, [8.0 * np.cos(a), 8.0 * np.sin(a), 0.0], [0.0, 0.0, np.sin(a / 2), np.cos(a / 2)])
        if kind == "quadx":
            av.set_mode(7)
            av.set_all_setpoints(torch.as_tensor(np.column_stack([start[:, :2], np.zeros(n), start[:, 2]]), dtype=torch.float32, device=dev))
        elif kind == "fixedwing":
            av.set_mode(0)
            av.set_all_setpoints(torch.as_tensor(np.tile([0.0, 0.0, 0.0, 0.6, 0.0, 0.0], (n, 1)), dtype=torch.float32, device=dev))
        return av

    for kind, n in (("quadx", args.drones), ("fixedwing", args.fw_drones), ("rocket", args.fw_drones)):
        cases = {(contact, bodies): build(kind, n, contact, bodies) for contact in (False, True) for bodies in (0, 1, 8)}
        for _ in range(args.pairs):
            for (contact, bodies), av in cases.items():
                ms = time_steps(av, args.n_steps, args.reps, args.warmup, dev)
                print(json.dumps({"kind": kind, "drones": n, "static_bodies": bodies, "contact_response": contact, "n_steps": args.n_steps,
                                  "gpu": prop.name, "power_limit_w,sm_mhz,sm_max_mhz": q, "ms_per_launch": ms,
                                  "drone_steps_per_s": n * args.n_steps / (ms * 1e-3), "in_contact": int(av.contact_array.sum())}), flush=True)
        del cases


if __name__ == "__main__":
    main()
