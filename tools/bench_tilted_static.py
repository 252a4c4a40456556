"""What the solid rule in full rotation frames (TiltedCtx: a ``solid_static_bodies=True`` handle that holds a tilted body,
DESIGN.md §4h "tilted static bodies") costs an Aviary step, next to the same scene on the yaw frames of SolidCtx.  Each case is
one scene built twice: plus one body 1000 m away, upright (the handle launches SolidCtx) or pitched 0.3 rad (TiltedCtx).  The
median of CUDA-event pairs around ``step(n_steps)`` with the library's Philox motor noise, after warm-up; one JSON line per case:

* ``far``: QuadX (cf2x, mode 7 position hold) at --drones, fixed-wing (mode 0 cruise) and rocket (unpowered, falling from
  400-600 m) at --fw-drones, 40 m or more above 1 wall or 7 walls (with the far body: 2 or 8 bodies), contact response off
  and on.  The cull keeps every primitive out of the candidate tests: this is the cost of the cull itself, which reads 12 pose
  words per primitive with TiltedCtx and 5 with SolidCtx.
* ``near``: cf2x hovering inside the cull distance above a platform under each drone, clear of its grown top.
* ``slide``: cf2x pushed by its position hold against a wall 0.3 m ahead, contact response on.

The two rules of a case are timed --pairs times, interleaved, to show the run-to-run spread.

    python tools/bench_tilted_static.py [--drones 65536] [--fw-drones 16384] [--n-steps 10] [--reps 20] [--warmup 5] [--pairs 2]

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
STATIC = os.path.join(ROOT, "tests", "golden", "static")
WALL, PLATFORM = os.path.join(STATIC, "wall_box.urdf"), os.path.join(STATIC, "platform_box.urdf")
FAR_UPRIGHT, FAR_TILTED = [0.0, 0.0, 0.0, 1.0], [0.0, float(np.sin(0.15)), 0.0, float(np.cos(0.15))]


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

    def aviary(kind, start, contact):
        n = len(start)
        return BatchedAviary(start.astype(np.float32), np.zeros((n, 3), dtype=np.float32), drone_type=kind, seed=0, device=dev,
                             contact_response=contact, solid_static_bodies=True)

    def far_body(av, tilted):  # the last body loaded: it decides SolidCtx or TiltedCtx
        av.loadURDF(WALL, [1000.0, 1000.0, 0.0], FAR_TILTED if tilted else FAR_UPRIGHT)

    def hold(av, sp):
        av.set_mode(7)
        av.set_all_setpoints(torch.as_tensor(sp, dtype=torch.float32, device=dev))

    def far(kind, n, contact, tilted, bodies):
        rng = np.random.default_rng(0)
        lo, hi = (400.0, 600.0) if kind == "rocket" else (40.0, 60.0)  # an unpowered rocket falls: it must not reach the floor while timed
        start = np.column_stack([rng.uniform(-10, 10, n), rng.uniform(-10, 10, n), rng.uniform(lo, hi, n)])
        av = aviary(kind, start, contact)
        for k in range(bodies - 1):
            a = 2 * np.pi * k / 8
            av.loadURDF(WALL, [8.0 * np.cos(a), 8.0 * np.sin(a), 0.0], [0.0, 0.0, np.sin(a / 2), np.cos(a / 2)])
        if kind == "quadx":
            hold(av, np.column_stack([start[:, :2], np.zeros(n), start[:, 2]]))
        elif kind == "fixedwing":
            av.set_mode(0)
            av.set_all_setpoints(torch.as_tensor(np.tile([0.0, 0.0, 0.0, 0.6, 0.0, 0.0], (n, 1)), dtype=torch.float32, device=dev))
        far_body(av, tilted)
        return av

    def near(n, tilted):
        rng = np.random.default_rng(1)
        xy = rng.uniform(-50, 50, (n, 2))
        av = aviary("quadx", np.column_stack([xy, np.full(n, 1.0)]), True)
        # the contact reach of the model about its base (contact_zmax), and the lowest a level drone's grown primitives reach
        m, reach, low = av.model, 0.0, 0.0
        for k in range(m.n_shapes):
            sh = m.shapes[k]
            disc = float(np.sqrt(sh.dims[0] ** 2 + sh.dims[1] ** 2 + sh.dims[2] ** 2)) if sh.kind == 0 else float(np.hypot(sh.dims[0], sh.dims[1]))
            reach = max(reach, (float(np.linalg.norm(list(sh.at))) + disc * (1.0 + float(m.contact_factor))) * 1.001)
            low = max(low, float(sh.dims[2] if sh.kind == 0 else sh.dims[1]) - float(sh.at[2]) + float(m.contact_factor) * disc)
        h = low + 0.75 * (reach - low)  # above the top: inside the cull distance, clear of the grown top
        av.loadURDF(PLATFORM, [0.0, 0.0, 0.0])
        av.set_static_pose(0, np.column_stack([xy, np.full(n, 0.5)]))  # the 1 m platform's inertial frame: its top at 1 m
        far_body(av, tilted)
        av.set_base_state(np.column_stack([xy, np.full(n, 1.5 + h)]), np.tile([0.0, 0.0, 0.0, 1.0], (n, 1)))
        hold(av, np.column_stack([xy, np.zeros(n), np.full(n, 1.0 + h)]))
        av.step(960)  # spin up 0.5 m higher, then descend to the held height and settle
        return av

    def slide(n, tilted):
        rng = np.random.default_rng(2)
        xy = rng.uniform(-50, 50, (n, 2))
        av = aviary("quadx", np.column_stack([xy, np.full(n, 1.0)]), True)
        av.loadURDF(WALL, [0.0, 0.0, 0.0])
        yaw = rng.uniform(-0.3, 0.3, n)
        av.set_static_pose(0, np.column_stack([xy[:, 0] + 0.4, xy[:, 1], np.full(n, 1.5)]),
                           np.column_stack([np.zeros(n), np.zeros(n), np.sin(yaw / 2), np.cos(yaw / 2)]))
        far_body(av, tilted)
        hold(av, np.column_stack([xy[:, 0] + 4.0, xy[:, 1], np.zeros(n), np.full(n, 1.0)]))
        av.step(240)  # pressed against the wall
        return av

    def report(case, kind, n, rule, contact, bodies, av):
        ms = time_steps(av, args.n_steps, args.reps, args.warmup, dev)
        bits = av.contact_bodies()
        print(json.dumps({"case": case, "kind": kind, "drones": n, "rule": rule, "static_bodies": bodies, "contact_response": contact,
                          "n_steps": args.n_steps, "gpu": prop.name, "power_limit_w,sm_mhz,sm_max_mhz": q, "ms_per_launch": ms,
                          "drone_steps_per_s": n * args.n_steps / (ms * 1e-3), "touching_a_body": int(bits[:, 1:].any(dim=1).sum()),
                          "touching_the_floor": int(bits[:, 0].sum())}), flush=True)

    for kind, n in (("quadx", args.drones), ("fixedwing", args.fw_drones), ("rocket", args.fw_drones)):
        cases = {(contact, tilted, bodies): far(kind, n, contact, tilted, bodies) for contact in (False, True) for tilted in (False, True) for bodies in (2, 8)}
        for _ in range(args.pairs):
            for (contact, tilted, bodies), av in cases.items():
                report("far", kind, n, "tilted" if tilted else "solid", contact, bodies, av)
        del cases
    n = args.drones
    for case, make in (("near", near), ("slide", slide)):
        cases = {tilted: make(n, tilted) for tilted in (False, True)}
        for _ in range(args.pairs):
            for tilted, av in cases.items():
                report(case, "quadx", n, "tilted" if tilted else "solid", True, 2, av)
        del cases


if __name__ == "__main__":
    main()
