"""The floor contact solver on its own, contact by contact, against the fp64 oracle.

``apply_contact_impulses`` (pyflyt_b200/csrc/pfb_fixedwing.cuh) solves the contact in fp32, in the BODY frame, with a cofactor
inverse of the central inertia; ``solve_contacts`` (oracle/pfb_oracle.c) solves it in fp64 in the WORLD frame with ``inv3`` on
the rotated tensor.  tests/probe/pfb_probe.cu runs the product helper one case at a time (over the QuadX table for cf2x and
primitive_drone, over a ContactParams with the fixed-wing or rocket registers otherwise), built by nvcc for the H100 and by g++;
the oracle runs through ``orc_solve_contacts``.  The contact FLAG (``ground_contact``, ``quadx_ground_contact``) is held to
``detect_contact_at`` the same way.

The cases (seeded, below) put the lowest candidate point of every model at the depths where the solver branches (0 +- 1-4
ulp, 1e-6, the slop +- 4 ulp, then 2e-3 ... 5e-2), in orientations where several candidate points are equally deep (flat face
down, upside down, edge down, cylinders whose lowest rim point lies half-way between two candidate points, the rocket on its
side) and in uniform random ones, with approach speeds up to the 100 m/s clamp and body rates up to the rate clamp.  Tangential
input speeds run from 0 through the band (1e-12, 1e-9] where the fp64 solver applies friction and the fp32 one does not, past
it (1e-8 ... 5e-7 m/s) to 10 m/s, and around the friction-cone edge.  Both solvers test their friction threshold on a point's
slip AFTER its normal impulse, which adds the slip of the rotation that impulse starts: the band rows keep that slip in the band
or near it, but do not place it a given number of ulp from 1e-9.  The rocket flies at fuel 0, 0.5 and 1 with the composite
mass, COM and inertia of its step.

What is compared, case by case:
  * post-solve velocity and rate, |dv| + |dw| reach, relative to the case's scale |v| + |w| reach + bias + erp * tol / dt + 1e-8
    (reach = farthest candidate point from the COM, bias = the Baumgarte velocity of the lowest point, tol = 8 fp32 ulp of the
    altitudes a depth is formed from: the Baumgarte velocity of a depth the fp32 solver can only know to that tolerance; 1e-8
    m/s: the slides below 1e-9 m/s the fp32 solver leaves unbraked);
  * a case with a candidate point within a few ulp of depth 0 (marked by the generator in fp64) may match the fp64 result of
    either side of that branch: the oracle is also run with the base a few ulp higher and lower.  A flat face can have some of
    its equally deep corners in contact and others not.  These cases are held to the same bar as every other case off the slop;
  * the bias max(depth - slop, 0) is continuous, as are the normal impulse max(0, jn0) and the friction cap min(sp / kt, mu jn),
    so those edges take no either-side rule.  The cases within a few ulp of the slop get a bar of their own: at rest their
    whole result is the rounding of the fp32 depth times erp / dt;
  * a case with no speed and the lowest point well inside the slop (no bias on either side) must come out exactly at rest;
  * cases whose speeds all lie in the (1e-12, 1e-9] band, their lowest point well inside the slop, are held to
    |dv| + |dw| reach <= a multiple of their speed;
  * contact flags are equal except within 4 fp32 ulp of the threshold, on poses from 0 to 1024 ulp and 1e-5 m to 30 m away
    from it.

The CPU tests hold the g++ build to the bars it measures here, with margin; the GPU tests hold the device build to at most 2x the
host result and print one ``[device-math contact ...]`` line each."""
import math

import numpy as np
import pytest

from engines import build_model
from test_device_math import Probe

F32 = np.float32
EPS32 = float(np.finfo(F32).eps)
ERP, SLOP, MU = 0.2, 0.001, 0.5
# the fp32 solver leaves a point sliding at up to 1e-9 m/s unbraked where the fp64 one brakes it from 1e-12 m/s: a velocity
# floor of every case's scale, ten times that for the candidate points it can happen at
SLIDE_FLOOR = 1e-8
PAD_TOP = 0.15

# (id, vehicle kind, model, rocket fuel ratio)
MODELS = [("cf2x", "quadx", "cf2x", None), ("primitive_drone", "quadx", "primitive_drone", None), ("fixedwing", "fixedwing", "fixedwing", None),
          ("acrowing", "fixedwing", "acrowing", None), ("rocket_fuel0", "rocket", "rocket", 0.0), ("rocket_fuel0.5", "rocket", "rocket", 0.5),
          ("rocket_fuel1", "rocket", "rocket", 1.0)]
MODEL_IDS = [m[0] for m in MODELS]


def f32(a):
    return np.asarray(a, dtype=F32).astype(np.float64)


# ---- geometry and the composite body, fp64 ---------------------------------------------------------------------------------
def candidate_points(model):
    """the solver's candidate points in the base frame (8 per box or cylinder: corners, 4 + 4 rim points) -> (K, 3)"""
    pts = []
    for s in range(model.n_shapes):
        sh = model.shapes[s]
        if sh.kind > 1:
            continue
        rot, at, d = np.array(sh.rot).reshape(3, 3), np.array(sh.at), np.array(sh.dims)
        for j in range(8):
            sz = 1.0 if j & 4 else -1.0
            if sh.kind == 0:
                q = [(1.0 if j & 1 else -1.0) * d[0], (1.0 if j & 2 else -1.0) * d[1], sz * d[2]]
            else:
                cs = [(1, 0), (0, 1), (-1, 0), (0, -1)][j & 3]
                q = [d[0] * cs[0], d[0] * cs[1], sz * d[1]]
            pts.append(rot @ np.array(q) + at)
    return np.array(pts)


def composite(model, fuel):
    """(M, c, I_O, Ic): mass, COM offset, inertia about the base origin and about the COM (base frame), as the step forms them;
    the rocket's from its fuel ratio (tank mass fuel * total at fuel_pos, tank inertia fuel * fuel_max_inertia)"""
    if int(model.kind) == 2:
        mf = fuel * model.fuel_total_mass
        M = model.dry_mass + mf
        r = np.array(model.fuel_pos)
        c = (np.array(model.dry_first_moment) + mf * r) / M
        I_O = np.array(model.dry_inertia).reshape(3, 3) + mf * (r @ r * np.eye(3) - np.outer(r, r)) + np.diag(fuel * np.array(model.fuel_max_inertia))
    else:
        M, c, I_O = float(model.mass), np.array(model.com), np.array(model.inertia).reshape(3, 3)
    Ic = I_O - M * (c @ c * np.eye(3) - np.outer(c, c))
    return M, c, I_O, Ic


def axis_angle(axis, angle):
    a = np.asarray(axis, dtype=np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * K @ K


def random_rotations(rng, n):
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    x, y, z, w = q.T
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], 1)


def orientations(kind, rng):
    """(R, tag) pairs, R body to world rounded to fp32: special attitudes of the vehicle kind, then uniform SO(3).  A yaw in
    front leaves the third row (all the depths see) as it is; where two candidate points are equally low by symmetry their
    third-row weights are made bit-equal in fp32 so that both builds see them at one depth"""
    out = []
    special = [("flat", np.eye(3)), ("upside_down", axis_angle([1, 0, 0], math.pi))]
    for ax in ([1, 0, 0], [0, 1, 0]):  # edge down
        for s in (1, -1):
            special.append(("edge", axis_angle(ax, s * math.pi / 4)))
    corner = math.atan(1 / math.sqrt(2))
    for sx, sy in ((1, 1), (-1, 1), (1, -1)):  # a single corner lowest
        special.append(("corner", axis_angle([1, 0, 0], sx * corner) @ axis_angle([0, 1, 0], sy * math.pi / 4)))
        special.append(("corner", axis_angle([1, 0, 0], sx * 0.3) @ axis_angle([0, 1, 0], sy * 0.45)))
    for phi in (math.pi / 4, 3 * math.pi / 4, -math.pi / 4):  # cylinders: the lowest rim point half-way between two candidates
        for tilt in (0.05, 0.4, 1.2):
            special.append(("rim45", axis_angle([-math.sin(phi), math.cos(phi), 0.0], tilt)))
    if kind == "rocket":  # lying on its side
        for ax in ([1, 0, 0], [0, 1, 0], [1, 1, 0], [1, -2, 0]):
            special.append(("side", axis_angle(ax, math.pi / 2)))
        special.append(("side", axis_angle([1, 0, 0], math.pi / 2 + 0.2)))
    for tag, R in special:
        R = axis_angle([0, 0, 1], rng.uniform(-math.pi, math.pi)) @ R
        R = f32(R)
        if tag == "rim45":  # |R20| = |R21| = sin(tilt) / sqrt(2): the rim points +x and +-y are equally low
            R[2, 1] = math.copysign(abs(R[2, 0]), R[2, 1])
        out.append((R, tag))
    for R in random_rotations(rng, 48):
        out.append((f32(R), "so3"))
    return out


def _depth_offsets():
    """signed depths of the lowest candidate point: (kind, value) where kind 'ulp0' / 'ulpslop' counts fp32 ulps of the base
    altitude from depth 0 / the slop"""
    offs = [("ulp0", k) for k in (-4, -2, -1, 1, 2, 4)] + [("depth", 1e-6)] + [("ulpslop", k) for k in (-4, -1, 0, 1, 4)]
    return offs + [("depth", d) for d in (2e-3, 5e-3, 1e-2, 2e-2, 5e-2)]


def _unit(rng, n=1):
    u = rng.normal(size=(n, 3))
    return u / np.linalg.norm(u, axis=1, keepdims=True)


def solver_cases(kind, name, fuel, seed=0):
    """the seeded case set of one model: dict of fp64 arrays holding fp32 values (pz, R, v world, w body, top), the composite
    body, and per case the fp64 marks: near (a candidate point within a few ulp of depth 0), atslop (one within a few ulp of
    the slop, none near depth 0), band (every speed in (1e-12, 1e-9]), the depth and bias of the lowest point and the reach"""
    model = build_model(kind, name)
    M, c, I_O, Ic = composite(model, fuel)
    P = candidate_points(model)
    reach = float(np.linalg.norm(f32(P) - c, axis=1).max())
    vmax, wmax = float(model.max_coord_velocity), float(model.max_coord_velocity) * 0.57735
    dt = 1.0 / model.physics_hz
    rng = np.random.default_rng(seed)
    tops = (0.0,) if kind == "quadx" else (0.0, PAD_TOP)  # QuadX drones meet the floor only
    Ic_inv = np.linalg.inv(Ic)
    rows = []
    for R, tag in orientations(kind, rng):
        zrel = (f32(P) @ R.T)[:, 2]
        zlow = float(zrel.min())
        for top in tops:
            for okind, val in _depth_offsets():
                if okind == "depth":
                    pz = float(F32(top - zlow - val))
                else:
                    base = F32(top - zlow - (SLOP if okind == "ulpslop" else 0.0))
                    pz = float(base + F32(val) * np.spacing(base)) if val else float(base)
                # velocities: structured rows, then random ones
                vels = []
                vn_list = (0.0, 0.01, 0.3, 1.0, 3.0, 8.0, 30.0, 99.9, -0.5)  # approach speeds (negative: separating)
                for vn in rng.choice(vn_list, 3, replace=False):
                    t = _unit(rng)[0]
                    t[2] = 0.0
                    t /= np.linalg.norm(t)
                    vt = float(rng.choice([0.0, 1e-3, 0.1, 1.0, 3.0, 10.0]))
                    wmag = float(rng.choice([0.0, 0.5, 5.0, wmax * 0.999]))
                    vels.append((np.array([0, 0, -vn]) + vt * t, wmag * _unit(rng)[0]))
                vels.append((np.zeros(3), np.zeros(3)))
                if okind == "depth" and val > SLOP:  # the friction-cone edge sp = mu jn kt at the lowest point, after its normal impulse
                    rw = R @ (f32(P[int(np.argmin(zrel))]) - c)
                    Iw = R @ Ic_inv @ R.T
                    t = np.array([math.cos(a := rng.uniform(-math.pi, math.pi)), math.sin(a), 0.0])
                    rn, rt = np.cross(rw, [0, 0, 1.0]), np.cross(rw, t)
                    vn = float(rng.choice([0.0, 0.3, 3.0]))
                    jn = (ERP * (val - SLOP) * model.physics_hz + vn) / (1 / M + rn @ Iw @ rn)
                    edge = MU * jn * (1 / M + rt @ Iw @ rt)
                    slip = np.cross(jn * Iw @ rn, rw)  # what the normal impulse's rotation adds at the point
                    slip[2] = 0.0
                    for fac in (0.98, 1.0, 1.02):
                        vels.append((np.array([0.0, 0.0, -vn]) + fac * edge * t - slip, np.zeros(3)))
                # the friction band, and tiny slides just above it (only where the normal speed is tiny too: bias 0, no rotation
                # from the solve to swamp them)
                if okind == "ulp0" or (okind == "depth" and val < SLOP):
                    t = _unit(rng)[0]
                    t[2] = 0.0
                    t /= np.linalg.norm(t)
                    for vt in (1e-11, 3e-10, 1e-9 * (1 - 2 * EPS32), 1e-9, 1e-9 * (1 + 2 * EPS32), 1e-8, 1e-7, 5e-7):
                        vels.append((np.array([0.0, 0.0, -float(rng.uniform(0.2, 1.0)) * vt]) + vt * t, np.zeros(3)))
                for v, w in vels:
                    rows.append((pz, R, f32(v), f32(w), top, tag))
    n = len(rows)
    pz = np.array([r[0] for r in rows])
    R = np.stack([r[1] for r in rows])
    v = np.stack([r[2] for r in rows])
    w = np.stack([r[3] for r in rows])
    top = np.array([r[4] for r in rows])
    tag = np.array([r[5] for r in rows])
    # fp64 marks from the fp32 inputs
    zr = np.einsum("kj,nij->nki", f32(P), R)[:, :, 2]  # (n, K)
    depth = top[:, None] - (pz[:, None] + zr)
    scale_z = np.abs(pz) + np.abs(top) + np.abs(zr).max(axis=1)
    tol = 8 * EPS32 * scale_z
    near = (np.abs(depth) <= tol[:, None]).any(axis=1)
    atslop = (np.abs(depth - SLOP) <= tol[:, None]).any(axis=1) & ~near
    dlow = depth.max(axis=1)
    bias = ERP * np.maximum(dlow - SLOP, 0.0) / dt
    speed = np.linalg.norm(v, axis=1) + np.linalg.norm(w, axis=1) * reach
    band = (speed > 0) & (speed <= 1e-9 * (1 + 8 * EPS32) * 2)
    # the fp32 depth is known to a few ulp of the altitudes it is formed from: so is the Baumgarte velocity erp * depth / dt
    dfloor = ERP * tol / dt
    return dict(model=model, M=M, c=c, I_O=I_O, Ic=Ic, reach=reach, dt=dt, n=n, pz=pz, R=R, v=v, w=w, top=top, tag=tag, near=near, atslop=atslop, tol=tol,
                depth=dlow, bias=bias, dfloor=dfloor, speed=speed, band=band & (dlow < 0.5 * SLOP))


def _oracle(cs, pz):
    from oracle.oracle import solve_contacts

    n = cs["n"]
    w_world = np.einsum("nij,nj->ni", cs["R"], cs["w"])
    vo, wo, touched = solve_contacts(cs["model"], pz, cs["R"].reshape(n, 9), cs["v"], w_world, np.full(n, cs["M"]), cs["c"], cs["I_O"].reshape(9), cs["top"],
                                     cs["dt"])
    return vo, np.einsum("nji,nj->ni", cs["R"], wo), touched  # the rate back in the body frame (R^T w)


def measure_solver(p, kind, name, fuel):
    """worst relative error of the probe against the oracle over the case set, and where it occurred"""
    cs = solver_cases(kind, name, fuel)
    n, Ic, c = cs["n"], cs["Ic"], cs["c"]
    ic6 = np.array([Ic[0, 0], Ic[0, 1], Ic[0, 2], Ic[1, 1], Ic[1, 2], Ic[2, 2]])
    vk, wk = p.contact_impulses(cs["model"], cs["pz"], cs["R"], cs["v"], cs["w"], np.full(n, cs["M"]), np.tile(c, (n, 1)), np.tile(ic6, (n, 1)), cs["top"])
    vk, wk = vk.astype(np.float64), wk.astype(np.float64)
    vo, wo, touched = _oracle(cs, cs["pz"])
    reach = cs["reach"]

    err = np.linalg.norm(vk - vo, axis=1) + np.linalg.norm(wk - wo, axis=1) * reach
    near = cs["near"]
    if near.any():  # either side of the depth-0 branch: the fp64 result with the base a few ulp higher or lower
        for s in (-2.0, 2.0):
            v1, w1, _ = _oracle(cs, cs["pz"] + s * cs["tol"])
            e1 = np.linalg.norm(vk - v1, axis=1) + np.linalg.norm(wk - w1, axis=1) * reach
            err[near] = np.minimum(err[near], e1[near])
    band = cs["band"]
    scale = cs["speed"] + cs["bias"] + cs["dfloor"] + SLIDE_FLOOR
    still = (cs["speed"] == 0) & (cs["depth"] < 0.5 * SLOP)  # no speed and no bias on either side: nothing may move
    rel = err / scale

    def worst(sel):
        i = int(np.argmax(np.where(sel, rel, -1.0)))
        at = dict(tag=str(cs["tag"][i]), depth=float(cs["depth"][i]), top=float(cs["top"][i]), v=cs["v"][i].round(4).tolist(), w=cs["w"][i].round(3).tolist())
        return float(rel[i]) if sel.any() else 0.0, at

    far, at = worst(~band & ~still & ~cs["atslop"])
    slop, slop_at = worst(~band & ~still & cs["atslop"])
    return dict(n=n, worst=far, at=at, slop=slop, slop_at=slop_at, n_slop=int(cs["atslop"].sum()), band=float((err[band] / cs["speed"][band]).max()), n_band=int(band.sum()),
                still=float(err[still].max()) if still.any() else 0.0, nonfinite=int((~np.isfinite(vk)).any(axis=1).sum() + (~np.isfinite(wk)).any(axis=1).sum()),
                touched=float(touched.mean()), n_near=int(near.sum()), tags=sorted(set(cs["tag"].tolist())))


# the g++ build against fp64, rel = (|dv| + |dw| reach) / scale: what it measures here, x ~4 and rounded up.  The first bar holds
# every case off the slop edge, the cases within a few ulp of depth 0 (after the either-side rule) among them; the second the cases
# with a candidate point within a few ulp of the slop.  There the bias erp * max(depth - slop, 0) / dt is continuous, but a
# depth the fp32 solver forms to a few ulp of the altitudes is all the bias there is: at rest the whole result is that rounding
# times erp / dt, and the scale's erp * tol / dt term is what it is measured against.  Seen: cf2x 2.4e-4 / 6.5e-2,
# primitive_drone 4.4e-5 / 4.3e-2, fixedwing 1.3e-4 / 5.1e-2, acrowing 1.3e-4 / 6.9e-2, rocket (fuel 0, 0.5, 1) 3.1e-3 / 0.38.
SOLVER_HOST_BAR = {"cf2x": (1e-3, 0.15), "primitive_drone": (2e-4, 0.1), "fixedwing": (6e-4, 0.1), "acrowing": (6e-4, 0.15), "rocket": (2e-2, 0.8)}
BAND_BAR = 12.0  # |dv| + |dw| reach <= BAND_BAR x speed in the friction band (seen: 1.7 cf2x ... 8.0 rocket)


@pytest.mark.parametrize("mid,kind,name,fuel", MODELS, ids=MODEL_IDS)
def test_contact_solver_host_matches_oracle(mid, kind, name, fuel):
    m = measure_solver(Probe(False), kind, name, fuel)
    far, slop = SOLVER_HOST_BAR[name]
    assert m["nonfinite"] == 0, m
    assert m["worst"] < far and m["slop"] < slop, m
    assert m["n_near"] > 0.2 * m["n"] and m["n_slop"] > 0.1 * m["n"], m
    assert m["band"] < BAND_BAR and m["n_band"] > 0, m
    assert m["still"] == 0.0, m
    assert 0.3 < m["touched"] < 1.0, m  # both sides of depth 0 are flown


@pytest.mark.gpu
@pytest.mark.parametrize("mid,kind,name,fuel", MODELS, ids=MODEL_IDS)
def test_contact_solver_device(mid, kind, name, fuel):
    h, d = measure_solver(Probe(False), kind, name, fuel), measure_solver(Probe(True), kind, name, fuel)
    print(f"[device-math contact {mid}] {d['n']} cases: rel (|dv| + |dw| reach) / scale: device {d['worst']:.3e} at {d['at']}, host {h['worst']:.3e}; "
          f"({d['n_near']} within a few ulp of depth 0); {d['n_slop']} within a few ulp of the slop: device {d['slop']:.3e}, host {h['slop']:.3e}; "
          f"{d['n_band']} in the friction band: "
          f"device {d['band']:.2e} x speed, host {h['band']:.2e}; {d['nonfinite']} non-finite")
    assert d["nonfinite"] == 0, d
    assert d["worst"] <= 2.0 * max(h["worst"], 1e-6) and d["slop"] <= 2.0 * max(h["slop"], 1e-6), (d, h)
    assert d["band"] < BAND_BAR and d["still"] == 0.0, d


# ---- the contact flag --------------------------------------------------------------------------------------------------------
FLAG_ULPS = 4  # a flag may differ from fp64 this close to its threshold, in fp32 ulp of the terms it is formed from


def flag_cases(kind, name, seed=1):
    """poses whose base altitude sits at the flag threshold pz* (some shape within contact_factor * disc of `top`) + 0 ... 8,
    16, 64, 256, 1024 fp32 ulp of pz* either way, +- 1e-5 ... 30 m; with each pose's distance from pz* in fp32 ulp of the largest term the
    threshold is formed from (pz*, top, and each shape's centre height and extent)"""
    model = build_model(kind, name)
    rng = np.random.default_rng(seed)
    tops = (0.0,) if kind == "quadx" else (0.0, PAD_TOP)
    rows = []
    for R, _ in orientations(kind, rng):
        for top in tops:
            thr, terms = [], [abs(top)]
            for s in range(model.n_shapes):
                sh = model.shapes[s]
                d = np.array(sh.dims)
                Rz = R[2] @ np.array(sh.rot).reshape(3, 3)
                if sh.kind == 0:
                    ext, disc = np.abs(Rz) @ d, math.sqrt(d @ d)
                elif sh.kind == 1:
                    ext, disc = d[1] * abs(Rz[2]) + d[0] * math.sqrt(max(0.0, 1 - Rz[2] ** 2)), math.hypot(d[0], d[1])
                else:
                    ext, disc = d[0], d[0]
                cz = R[2] @ np.array(sh.at)
                thr.append(model.contact_factor * disc - (cz - ext))
                terms += [abs(cz), abs(ext)]
            star = top + max(thr)
            unit = float(np.spacing(F32(max(terms + [abs(star)]))))
            base = F32(star)
            for k in list(range(-8, 9)) + [s * k for k in (16, 64, 256, 1024) for s in (-1, 1)]:
                rows.append((float(base + F32(k) * np.spacing(base)), R, top, star, unit))
            for dz in (1e-5, 1e-4, 1e-2, 0.1, 1.0, 30.0):
                rows += [(float(F32(star + dz)), R, top, star, unit), (float(F32(star - dz)), R, top, star, unit)]
    pz = np.array([r[0] for r in rows])
    R = np.stack([r[1] for r in rows])
    top = np.array([r[2] for r in rows])
    ulps = np.abs(pz - np.array([r[3] for r in rows])) / np.array([r[4] for r in rows])
    return model, pz, R, top, ulps


def measure_flag(p, kind, name):
    from oracle.oracle import contact_flag

    model, pz, R, top, ulps = flag_cases(kind, name)
    fk = p.contact_flag(model, pz, R, top)
    fo = contact_flag(model, pz, R.reshape(-1, 9), top)
    differ = fk != fo
    return dict(n=len(pz), differ=int(differ.sum()), worst_ulps=float(ulps[differ].max()) if differ.any() else 0.0, n_close=int((ulps <= 8).sum()),
                up=float(fo.mean()))


FLAG_MODELS = [m[:3] for m in MODELS[:5]]


@pytest.mark.parametrize("mid,kind,name", FLAG_MODELS, ids=[m[0] for m in FLAG_MODELS])
def test_contact_flag_host_matches_oracle(mid, kind, name):
    m = measure_flag(Probe(False), kind, name)
    assert m["worst_ulps"] <= FLAG_ULPS and 0.3 < m["up"] < 0.7, m


@pytest.mark.gpu
@pytest.mark.parametrize("mid,kind,name", FLAG_MODELS, ids=[m[0] for m in FLAG_MODELS])
def test_contact_flag_device(mid, kind, name):
    h, m = measure_flag(Probe(False), kind, name), measure_flag(Probe(True), kind, name)
    print(f"[device-math contact flag {mid}] {m['n']} poses ({m['n_close']} within 8 ulp of the threshold): {m['differ']} flags differ from fp64, "
          f"the farthest {m['worst_ulps']:.2f} ulp from the threshold (host {h['differ']}, {h['worst_ulps']:.2f} ulp)")
    assert m["worst_ulps"] <= FLAG_ULPS and 0.3 < m["up"] < 0.7, m


def test_case_generator_covers_the_edges():
    """the generator does put points at the branches it claims: depth 0 +- ulp (marked near), the slop, the band, the pad"""
    cs = solver_cases("rocket", "rocket", 0.5)
    assert cs["near"].sum() > 100 and cs["band"].sum() > 100
    assert {"flat", "upside_down", "edge", "corner", "rim45", "side", "so3"} <= set(cs["tag"].tolist())
    assert (cs["top"] == PAD_TOP).any() and (np.abs(cs["v"][:, 2]) > 90).any() and (np.linalg.norm(cs["w"], axis=1) > 50).any()
    d = cs["depth"]
    assert ((d > 0) & (d < 1e-6)).any() and ((d < 0) & (d > -1e-6)).any() and (np.abs(d - SLOP) < 1e-8).any() and (d > 0.04).any()
