"""Tilted static bodies in the Aviary: on a handle with ``solid_static_bodies=True``, ``loadURDF`` takes any ``baseOrientation``,
URDF collision primitives any ``rpy`` and ``set_static_pose`` any unit quaternion (ramps, race gates, bars).  The step kernels run
the solid rule in full rotation frames (TiltedCtx; DESIGN.md §4h, "tilted static bodies") once a tilted body, primitive or pose
is on the handle; upright scenes keep SolidCtx.

CPU (g++ build, tests/hostsim/hostsim_tilted.cpp): each face of a box turned by a full rotation, the tie orders and the
cylinder's radial / top / bottom choice in rotated frames; rotating a primitive and a query point together rotates the normal and
keeps the depth; on yaw-only frames the TiltedCtx helpers give the SolidCtx bits, depths and normals; the cull against the
uncalled helper on random tilted poses; the host build replays every ``tilted_*`` fixture.
GPU: the CUDA Aviary replays every fixture; refusals on default handles and through the C-ABI; an upright scene stepped through
TiltedCtx against SolidCtx; a mixed handle equals the single-kind handles; a masked tilted pose leaves the other worlds;
``reset()`` clears the flag; the friction cone on ramps; 8 192 QuadX at randomly tilted walls; a 4-gate course."""
import ctypes as C
import glob
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

from engines import GOLDEN, ROOT, load_golden

STATIC = os.path.join(GOLDEN, "static")
WALL, RAMP, GATE, BAR, PLATFORM = (os.path.join(STATIC, f) for f in ("wall_box.urdf", "ramp_slab.urdf", "race_gate.urdf", "bar_cylinder.urdf",
                                                                     "platform_box.urdf"))
FAR = (1000.0, 1000.0, 0.0)
f32, i32, u32 = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint32)

_HS = None


def hs():
    global _HS
    if _HS is None:
        out = os.path.join(tempfile.mkdtemp(prefix="pfb_hostsim_tilted_"), "libpfb_hostsim_tilted.so")
        src = os.path.join(ROOT, "tests", "hostsim", "hostsim_tilted.cpp")
        subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-mfma", "-ffp-contract=fast", "-o", out, src], check=True, capture_output=True)
        _HS = C.CDLL(out)
        _HS.hs_last_error.restype = C.c_char_p
    return _HS


def rot(roll, pitch, yaw):
    """R = Rz(yaw) Ry(pitch) Rx(roll), PyBullet's getMatrixFromQuaternion(getQuaternionFromEuler(...))"""
    cr, sr, cp, sp, cy, sy = np.cos(roll), np.sin(roll), np.cos(pitch), np.sin(pitch), np.cos(yaw), np.sin(yaw)
    return np.array([[cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr], [sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr], [-sp, cp * sr, cp * cr]])


def quat(roll, pitch, yaw):
    cr, sr, cp, sp, cy, sy = np.cos(roll / 2), np.sin(roll / 2), np.cos(pitch / 2), np.sin(pitch / 2), np.cos(yaw / 2), np.sin(yaw / 2)
    return [sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy]


def quat_matrix(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def random_rotation(rng):
    q = rng.normal(size=4)
    return quat_matrix(q / np.linalg.norm(q))


class TWorld:
    """A static world in the flat layout of tests/hostsim/hostsim_tilted.cpp: primitives (body, kind, centre, rotation in the body,
    half sizes) and the poses of the bodies in each of n worlds ([12 * 8][n]: x, y, z, row-major rotation of the base link frame)."""

    def __init__(self, n=1):
        self.n = n
        self.body, self.kind, self.at, self.rot, self.half = [], [], [], [], []
        self.pose = np.zeros((12 * 8, n), dtype=np.float32)
        for b in range(8):
            self.pose[12 * b + 3:12 * b + 12] = np.eye(3).reshape(9, 1)
        self.n_bodies = 0

    def add(self, prims, pos=(0.0, 0.0, 0.0), R=np.eye(3)):
        b = self.n_bodies
        for kind, at, Rp, half in prims:
            self.body.append(b)
            self.kind.append(kind)
            self.at.append(at)
            self.rot.append(np.asarray(Rp, dtype=np.float64).reshape(9))
            self.half.append(half)
        self.n_bodies += 1
        self.place(b, pos, R)
        return b

    def place(self, b, pos, R, cols=slice(None)):
        shape = (-1,) if isinstance(cols, int) else (-1, 1)
        self.pose[12 * b:12 * b + 3, cols] = np.asarray(pos, dtype=np.float64).reshape(shape)
        self.pose[12 * b + 3:12 * b + 12, cols] = np.asarray(R, dtype=np.float64).reshape(shape)

    def args(self):
        self._keep = [np.ascontiguousarray(np.asarray(a, dtype=t).reshape(-1)) for a, t in
                      ((self.body, np.int32), (self.kind, np.int32), (self.at, np.float32), (self.rot, np.float32), (self.half, np.float32))]
        self._keep.append(np.ascontiguousarray(self.pose))
        return [len(self.body)] + [k.ctypes.data_as(i32 if k.dtype == np.int32 else f32) for k in self._keep]

    @property
    def all(self):
        return (1 << len(self.body)) - 1


def contact(world, x, y, z, live=None, i=0):
    d, nrm = C.c_float(0), (C.c_float * 3)()
    live = world.all if live is None else live
    f = C.c_float
    assert hs().hs_tilted_point_contact(*world.args(), C.c_int64(world.n), C.c_int64(i), C.c_uint32(live), f(x), f(y), f(z), C.byref(d), nrm) == 0
    return d.value, np.array(nrm[:])


def live_of(world, x, y, z, reach, i=0):
    out = C.c_uint32(0)
    f = C.c_float
    assert hs().hs_tilted_live(*world.args(), C.c_int64(world.n), C.c_int64(i), f(x), f(y), f(z), f(reach), C.byref(out)) == 0
    return out.value


def bits_solve(model, world, live, base, R, v, w):
    bits, vo, wo, t = C.c_uint32(0), (C.c_float * 3)(), (C.c_float * 3)(), C.c_int(0)
    keep = [np.ascontiguousarray(a, dtype=np.float32).reshape(-1) for a in (base, R, v, w)]
    assert hs().hs_tilted_bits_solve(C.byref(model), *world.args(), C.c_int64(world.n), C.c_int64(0), C.c_uint32(live),
                                     *[k.ctypes.data_as(f32) for k in keep], C.byref(bits), vo, wo, C.byref(t)) == 0
    return bits.value, np.array(vo[:], dtype=np.float32), np.array(wo[:], dtype=np.float32), t.value


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_faces_of_a_rotated_box():
    """each face of a box turned by a full rotation (body and primitive both tilted): the depth to that face and its outward
    normal, the primitive-frame normal turned by the primitive's world rotation"""
    Rb, Rp = rot(0.4, -0.3, 0.7), rot(0.2, 0.5, -0.1)
    Rw = Rb @ Rp
    w = TWorld()
    pos, at = np.array([2.0, -1.0, 3.0]), np.array([0.3, 0.1, 0.5])
    w.add([(0, tuple(at), Rp, (0.5, 1.0, 0.8))], pos=tuple(pos), R=Rb)
    centre = pos + Rb @ at
    for local, normal, depth in (((0.45, 0.0, 0.0), (1, 0, 0), 0.05), ((-0.42, 0.1, 0.2), (-1, 0, 0), 0.08), ((0.0, 0.93, 0.2), (0, 1, 0), 0.07),
                                 ((0.1, -0.96, -0.1), (0, -1, 0), 0.04), ((0.1, 0.2, 0.77), (0, 0, 1), 0.03), ((0.2, 0.1, -0.79), (0, 0, -1), 0.01)):
        d, n = contact(w, *(centre + Rw @ np.array(local)))
        np.testing.assert_allclose(d, depth, atol=3e-6)
        np.testing.assert_allclose(n, Rw @ np.array(normal, dtype=np.float64), atol=2e-6)
    d, n = contact(w, *(centre + Rw @ np.array([0.6, 0.0, 0.0])))
    assert n.tolist() == [0.0, 0.0, 1.0] and d < 0  # outside: the floor's contact


def test_tie_orders_in_a_rotated_frame():
    """the box's ties (+z, then +-x, then +-y, then -z) and the cylinder's (top, radial, bottom; +x on the axis) hold in the
    primitive's own frame whatever its rotation (rotations by quarter turns, exact in fp32, so that the ties stay exact)"""
    R = np.array([[0.0, 0.0, 1.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])  # x -> y -> z -> x: no primitive axis stays vertical
    w = TWorld()
    w.add([(0, (0.0, 0.0, 0.0), np.eye(3), (1.0, 1.0, 1.0))], pos=(0.0, 0.0, 5.0), R=R)
    c = np.array([0.0, 0.0, 5.0])
    for local, normal in (((0.5, 0.5, 0.5), (0, 0, 1)), ((-0.5, -0.5, 0.0), (-1, 0, 0)), ((0.0, -0.5, -0.5), (0, -1, 0)), ((0.0, 0.0, 0.0), (0, 0, 1)),
                          ((0.0, 0.0, -0.8), (0, 0, -1))):
        np.testing.assert_allclose(contact(w, *(c + R @ np.array(local, dtype=np.float64)))[1], R @ np.array(normal, dtype=np.float64), atol=2e-6)
    Rc = np.array([[0.0, 1.0, 0.0], [0.0, 0.0, -1.0], [-1.0, 0.0, 0.0]])  # a horizontal bar: its axis along world -x
    w2 = TWorld()
    w2.add([(1, (0.0, 0.0, 0.0), np.eye(3), (0.25, 0.25, 0.5))], pos=(0.0, 0.0, 3.0), R=Rc)
    c = np.array([0.0, 0.0, 3.0])
    for local, normal in (((0.0, 0.0, 0.4), (0, 0, 1)), ((0.1, 0.0, 0.0), (1, 0, 0)), ((0.0, 0.0, -0.4), (0, 0, -1)),
                          ((0.0, 0.0, 0.0), (1, 0, 0)),            # on the axis: rho < 1e-6 -> +x of the primitive
                          ((0.0, 0.25 - 0.25, 0.25), (0, 0, 1)),   # top 0.25 = radial 0.25: the top
                          ((0.0, -0.0, -0.25), (1, 0, 0))):        # radial 0.25 (on the axis: +x) = bottom 0.25: radial
        d, n = contact(w2, *(c + Rc @ np.array(local, dtype=np.float64)))
        np.testing.assert_allclose(n, Rc @ np.array(normal, dtype=np.float64), atol=2e-6, err_msg=str(local))


def test_rotating_primitive_and_point_together():
    """a random rotation Q applied to a primitive's pose and to a query point: the depth is kept and the normal turns with Q"""
    rng = np.random.default_rng(21)
    for _ in range(300):
        kind = int(rng.integers(0, 2))
        half = tuple(rng.uniform(0.2, 1.0, 3)) if kind == 0 else (0.6, 0.6, float(rng.uniform(0.2, 1.0)))
        Rp, Q = random_rotation(rng), random_rotation(rng)
        p = rng.uniform(-1, 1, 3) * np.array([half[0], half[1], half[2]])
        c = np.array([0.0, 0.0, 20.0])  # high above the floor
        a, b = TWorld(), TWorld()
        a.add([(kind, (0.0, 0.0, 0.0), np.eye(3), half)], pos=tuple(c), R=Rp)
        b.add([(kind, (0.0, 0.0, 0.0), np.eye(3), half)], pos=tuple(c), R=Q @ Rp)
        da, na = contact(a, *(c + Rp @ p))
        db, nb = contact(b, *(c + Q @ Rp @ p))
        if da < 0 or db < 0:  # a point at the boundary may round outside in one of them
            continue
        np.testing.assert_allclose(db, da, atol=1e-5)
        if da > 1e-2:  # the normal of a shallow point, or of one near a cylinder's axis, is as good as the fp32 frame
            np.testing.assert_allclose(nb, Q @ na, atol=1e-4)


def _solid_lib():
    from test_solid_static_bodies import hs as solid_hs

    return solid_hs()


def _yaw_pair(rng, n_bodies=3):
    """the same upright world in both layouts: (TWorld, the SolidCtx World of test_solid_static_bodies)"""
    from test_solid_static_bodies import World

    t, s = TWorld(), World()
    for _ in range(n_bodies):
        prims = []
        for _ in range(int(rng.integers(1, 3))):
            kind = int(rng.integers(0, 2))
            half = tuple(rng.uniform(0.2, 1.0, 3)) if kind == 0 else (0.4, 0.4, float(rng.uniform(0.2, 1.0)))
            prims.append((kind, tuple(rng.uniform(-0.5, 0.5, 2)) + (float(rng.uniform(0.3, 1.5)),), float(rng.uniform(-np.pi, np.pi)), half))
        pos, yaw = tuple(rng.uniform(-2, 2, 2)) + (0.0,), float(rng.uniform(-np.pi, np.pi))
        s.add(prims, pos=pos, yaw=yaw)
        t.add([(k, at, rot(0, 0, py), h) for k, at, py, h in prims], pos=pos, R=rot(0, 0, yaw))
    return t, s


def test_yaw_frames_match_solid_ctx():
    """on upright bodies and primitives the TiltedCtx helpers give the SolidCtx bits and depths, and normals within fp32 ulps"""
    from test_solid_static_bodies import _bits_solve, _cf2x, contact as solid_contact

    rng = np.random.default_rng(22)
    m = _cf2x()
    hits = 0
    for _ in range(40):
        t, s = _yaw_pair(rng)
        for _ in range(20):
            p = rng.uniform([-3, -3, 0.0], [3, 3, 2.5])
            dt_, nt = contact(t, *p)
            ds, ns = solid_contact(s, *p)
            assert abs(dt_ - ds) <= 4e-6 and np.allclose(nt, ns, atol=1e-6), (p, dt_, ds, nt, ns)
            hits += ds > 0 and ns[2] != 1.0
            R = rot(*rng.uniform(-0.5, 0.5, 2), rng.uniform(-np.pi, np.pi))
            v, wb = rng.normal(0, 2, 3), rng.normal(0, 3, 3)
            bt = bits_solve(m, t, t.all, p, R, v, wb)
            bs = _bits_solve(m, s, s.all, p, R, v, wb)
            assert bt[0] == bs[0] and bt[3] == bs[3]
            np.testing.assert_allclose(bt[1], bs[1], atol=2e-4, rtol=1e-4)
    assert hits > 20


def _reach(model):
    from test_solid_static_bodies import _reach as r

    return r(model)


def test_cull_equals_uncalled_helper():
    """random cf2x poses around every primitive of a tilted world (a pitched ramp, a gate turned by roll, pitch and yaw, a bar):
    the bits and solved velocities over the primitives the cull keeps equal those over every primitive, bit for bit"""
    from test_solid_static_bodies import _cf2x

    m = _cf2x()
    reach = _reach(m)
    w = TWorld()
    w.add([(0, (0.0, 0.0, -0.05), np.eye(3), (2.0, 1.0, 0.05))], pos=(2.0, 0.5, 1.0), R=rot(0.0, 0.4, 0.3))
    gate = [(0, (0.0, 0.0, -0.225), np.eye(3), (0.025, 0.25, 0.025)), (0, (0.0, -0.225, 0.0), np.eye(3), (0.025, 0.025, 0.2)),
            (0, (0.0, 0.225, 0.0), np.eye(3), (0.025, 0.025, 0.2)), (0, (0.0, 0.0, 0.225), np.eye(3), (0.025, 0.25, 0.025))]
    w.add(gate, pos=(-1.0, -2.0, 1.0), R=rot(0.2, 0.3, 1.0))
    w.add([(1, (0.0, 0.0, 1.0), rot(np.pi / 2, 0, 0), (0.05, 0.05, 1.5))], pos=(-3.0, 3.0, 0.0), R=rot(0.0, 0.0, -0.5))
    rng = np.random.default_rng(23)
    centres = [(2.0, 0.5, 1.0), (-1.0, -2.0, 1.0), (-3.0, 3.0, 1.0)]
    halves = [(2.2, 2.2, 1.0), (0.3, 0.3, 0.3), (1.6, 1.6, 0.2)]
    seen_hit, seen_cull = 0, 0
    for k in range(len(centres)):
        for _ in range(300):
            base = np.array(centres[k]) + rng.uniform(-1, 1, 3) * (np.array(halves[k]) + 2.0 * reach)
            R = rot(*rng.uniform(-0.6, 0.6, 2), rng.uniform(-np.pi, np.pi))
            v, wb = rng.normal(0, 2, 3), rng.normal(0, 3, 3)
            live = live_of(w, *base, reach)
            a = bits_solve(m, w, live, base, R, v, wb)
            b = bits_solve(m, w, w.all, base, R, v, wb)
            assert a[0] == b[0] and a[3] == b[3] and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32)) and np.array_equal(a[2].view(np.uint32), b[2].view(np.uint32))
            seen_hit += b[0] > 1
            seen_cull += live != w.all
    assert seen_hit > 15 and seen_cull > 300


# ------------------------------------------------------------------------------------------------------------------ fixtures
# tests/golden/tilted_*.npz (tools/gen_golden.py, group ``tilted``): the unmodified reference Aviary with tilted fixed-base bodies
# (loadURDF with a baseOrientation, a URDF collision rpy, resetBasePositionAndOrientation), each drone in an Aviary of its own,
# read through contact_array[drone.Id, body], with the contact response, on the fake client with the solid rule (fp64).  The host
# build and the CUDA Aviary replay them with the reference's draws injected: contact bits exact at every step, state within fp32
# bars: what the host build shows, x5 and rounded up, never below the free-flight bars (pos 5e-4 m, euler 1e-3 rad, rates and
# velocities 1e-2).  Host seen:
#                                  pos      euler    angvel   linvel
#   tilted_cf2x_gate_bar           8.6e-4   9.4e-3   0.81     2.4e-2
#   tilted_cf2x_gate_pass          6.8e-5   1.4e-5   1.7e-3   4.0e-3
#   tilted_cf2x_per_drone_poses    1.4e-4   3.7e-3   0.64     1.9e-2
#   tilted_cf2x_ramp_rest          1.6e-7   7.2e-7   6.9e-5   3.6e-6
#   tilted_cf2x_ramp_slide         4.3e-6   6.5e-5   1.2e-3   7.2e-5
#   tilted_fixedwing_rolled_wall   7.5e-3   1.4e-2   2.7      0.56
#   tilted_primitive_bar_drop      9.7e-5   1.6e-3   0.36     2.6e-2
#   tilted_rocket_pad              3.0e-3   4.7e-3   0.15     3.9e-2
TILTED_FIXTURES = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, "tilted_*.npz")))
TILTED_BARS = {
    "tilted_cf2x_gate_bar": dict(pos=4.3e-3, euler=4.7e-2, angvel=4.1, linvel=0.12),
    "tilted_cf2x_gate_pass": dict(pos=5e-4, euler=1e-3, angvel=1e-2, linvel=2e-2),
    "tilted_cf2x_per_drone_poses": dict(pos=7e-4, euler=1.9e-2, angvel=3.2, linvel=9.5e-2),
    "tilted_cf2x_ramp_rest": dict(pos=5e-4, euler=1e-3, angvel=1e-2, linvel=1e-2),
    "tilted_cf2x_ramp_slide": dict(pos=5e-4, euler=1e-3, angvel=1e-2, linvel=1e-2),
    "tilted_fixedwing_rolled_wall": dict(pos=3.8e-2, euler=7e-2, angvel=14.0, linvel=2.8),
    "tilted_primitive_bar_drop": dict(pos=5e-4, euler=8e-3, angvel=1.8, linvel=0.13),
    "tilted_rocket_pad": dict(pos=1.5e-2, euler=2.4e-2, angvel=0.75, linvel=0.2),
}


def _fixture_world(g):
    """the fixture's static bodies as the flat TWorld of the host build: primitives read by the library's URDF reader, body k of
    drone i's world at its loadURDF pose, or at the pose resetBasePositionAndOrientation gave its base inertial frame"""
    from test_static_bodies import read_shapes

    n = len(g["start_pos"])
    w = TWorld(n)
    inertial = []
    for f, pos, q in json.loads(str(g["bodies"])):
        rc, shapes, io = read_shapes(os.path.join(STATIC, f), with_inertial=True)
        assert rc == 0
        inertial.append(io)
        prims = [(s.kind, tuple(s.at), np.array(s.rot[:]).reshape(3, 3), tuple(s.dims) if s.kind == 0 else (s.dims[0], s.dims[0], s.dims[1])) for s in shapes]
        w.add(prims, pos=tuple(pos), R=quat_matrix(np.array(q) / np.linalg.norm(q)))
    for i, pz in enumerate(json.loads(str(g["poses"]))):
        for k, (pos, q) in pz.items():
            R = quat_matrix(np.array(q) / np.linalg.norm(q))
            w.place(int(k), tuple(np.array(pos) - R @ inertial[int(k)]), R, cols=i)
    return w


def _replay(g, cuda):
    from test_static_bodies import _errors, _setpoint_at

    kind, n, T = str(g["drone_type"]), len(g["start_pos"]), len(g["state"])
    states, bits = np.zeros((T, n, 4, 3)), np.zeros((T, n), dtype=np.uint32)
    noise = g["noise"].reshape(T, -1, n).astype(np.float32)
    if cuda:
        import torch
        from pyflyt_b200.core.aviary import BatchedAviary

        av = BatchedAviary(g["start_pos"], g["start_orn"], drone_type=kind, drone_options=json.loads(str(g["drone_options"])), seed=0,
                           contact_response=True, solid_static_bodies=True)
        for f, pos, q in json.loads(str(g["bodies"])):
            av.loadURDF(os.path.join(STATIC, f), pos, q)
        moved = {}
        for i, pz in enumerate(json.loads(str(g["poses"]))):
            for k, (pos, q) in pz.items():
                moved.setdefault(int(k), (np.zeros((n, 3)), np.tile([0.0, 0.0, 0.0, 1.0], (n, 1)), np.zeros(n, dtype=bool)))
                moved[int(k)][0][i], moved[int(k)][1][i], moved[int(k)][2][i] = pos, q, True
        for k, (pos, q, mask) in moved.items():
            av.set_static_pose(k, pos, q, mask=mask)
        av.set_mode(int(g["mode"]))
        nz = torch.as_tensor(noise, device=av.device)
        for t in range(T):
            sp = _setpoint_at(g, t, n)
            if sp is not None:
                rows = np.zeros((n, av.setpoint_dim))
                rows[:, : sp.shape[1]] = sp
                av.set_all_setpoints(rows)
            av.step(1, noise=nz[t].contiguous())
            states[t] = av.all_states.cpu().numpy()
            cb = av.contact_bodies().cpu().numpy()
            bits[t] = (cb * (1 << np.arange(cb.shape[1]))).sum(axis=1)
        return _errors(g, states, bits)
    from engines import HostSimEngine, build_model

    model = build_model(kind, **json.loads(str(g["drone_options"])))
    eng = HostSimEngine(model, None, n=n, start_pos=g["start_pos"], start_orn=g["start_orn"])
    eng.reset()
    eng.set_mode(int(g["mode"]))
    w = _fixture_world(g)
    a = w.args()
    full = int(kind == "fixedwing" and int(model.n_surfaces) == 5)
    L = hs()
    for t in range(T):
        sp = _setpoint_at(g, t, n)
        if sp is not None:
            eng.set_setpoints(sp)
        nz = np.ascontiguousarray(noise[t])
        b = np.zeros(n, dtype=np.uint32)
        args = (*a, eng.st.ctypes.data_as(f32), eng.ist.ctypes.data_as(i32), eng.sp.ctypes.data_as(f32), nz.ctypes.data_as(f32), 1, C.c_int64(n),
                b.ctypes.data_as(u32))
        if kind == "quadx":
            rc = L.hs_aviary_step_tilted(C.byref(model), eng.mode, 1, *args)
        elif kind == "fixedwing":
            rc = L.hs_fw_aviary_step_tilted(C.byref(model), eng.mode, full, *args)
        else:
            rc = L.hs_rk_aviary_step_tilted(C.byref(model), *args)
        assert rc == 0, L.hs_last_error()
        states[t], bits[t] = eng.state(), b
    return _errors(g, states, bits)


def test_tilted_fixtures_present():
    assert set(TILTED_FIXTURES) == set(TILTED_BARS) and len(TILTED_FIXTURES) >= 8


def test_fixtures_touch_what_they_say():
    """the flights do what their names say: a rest and a slide on the ramps, a gate crossed without a bit and a bar struck"""
    b = {n: load_golden(n)["bits"] for n in TILTED_FIXTURES}
    assert not b["tilted_cf2x_gate_pass"].any() and (b["tilted_cf2x_gate_bar"] & 2).any()
    for n in ("tilted_cf2x_ramp_rest", "tilted_cf2x_ramp_slide", "tilted_primitive_bar_drop", "tilted_fixedwing_rolled_wall", "tilted_rocket_pad"):
        assert (b[n] & 2).any(), n
    rest, slide = load_golden("tilted_cf2x_ramp_rest")["state"], load_golden("tilted_cf2x_ramp_slide")["state"]
    assert abs(rest[-1, 0, 3, 0]) < 0.1 and rest[-1, 0, 3, 2] > 0.9 and slide[-1, 0, 3, 0] > 1.0


def _check(name, err):
    assert err["bits_mismatch"] == 0, (name, err)
    for k, bar in TILTED_BARS[name].items():
        assert err[k] < bar, (name, k, err[k], bar)


@pytest.mark.parametrize("name", sorted(TILTED_BARS))
def test_host_replays_tilted_fixture(name):
    """the g++ build of the TiltedCtx steps replays the reference: contact bits at every step, state within the fp32 bars"""
    _check(name, _replay(load_golden(name), cuda=False))


# ------------------------------------------------------------------------------------------------------------------ GPU
def _aviary(n=4, kind="quadx", contact=True, seed=3, start=None, solid=True, **kw):
    from pyflyt_b200.core.aviary import BatchedAviary

    if start is None:
        start = np.column_stack([np.linspace(-1, 1, n), np.zeros(n), np.full(n, 1.0)])
    return BatchedAviary(start, np.zeros((n, 3)), drone_type=kind, seed=seed, contact_response=contact, solid_static_bodies=solid, **kw)


def _state_bytes(av):
    import torch

    torch.cuda.synchronize()
    return av.state_tensor.detach().cpu().numpy().view(np.uint32).copy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(TILTED_BARS))
def test_cuda_replays_tilted_fixture(name):
    """the CUDA Aviary with solid_static_bodies=True replays the reference on tilted bodies: bits at every step, the same bars"""
    _check(name, _replay(load_golden(name), cuda=True))


@pytest.mark.gpu
def test_refusals():
    """default handles refuse tilt as before (with a pointer to the solid option); a solid handle takes it, and then refuses to
    go back to the top-face rule until a reset"""
    import torch
    from pyflyt_b200 import _lib as L

    tilt = quat(0.1, 0.0, 0.0)
    av = _aviary(solid=False)
    with pytest.raises(L.PfbError, match="upright") as e:
        av.loadURDF(PLATFORM, [0, 0, 0], tilt)
    assert "solid_static_bodies" in str(e.value)
    with tempfile.TemporaryDirectory() as tmp:
        t = os.path.join(tmp, "t.urdf")
        with open(t, "w") as f:
            f.write('<robot name="t"><link name="b"><collision><origin rpy="0.3 0 0"/><geometry><box size="1 1 1"/></geometry></collision></link></robot>')
        with pytest.raises(L.PfbError, match="tilted"):
            av.loadURDF(t, [0, 0, 0])
        s = _aviary(solid=True)
        assert s.loadURDF(t, [0, 0, 0]) == 0  # a tilted primitive on a solid handle
    av.loadURDF(PLATFORM, [0, 0, 0])
    with pytest.raises(ValueError, match="upright") as e:
        av.set_static_pose(0, [0.0, 0.0, 0.0], tilt)
    assert "solid_static_bodies=True" in str(e.value)
    pos = torch.zeros((4, 3), dtype=torch.float64, device=av.device)
    q = torch.tensor([[0.0, 0.0, 0.0, 1.0]] * 3 + [tilt], dtype=torch.float64, device=av.device)
    lib = L.lib()
    assert lib.pfb_set_static_pose(av._h, 0, C.c_void_p(pos.data_ptr()), C.c_void_p(q.data_ptr()), None, None) != 0
    assert b"quat[3] is not upright" in lib.pfb_last_error()
    # the solid handle: tilted poses through the C-ABI, then no way back to the top-face rule until reset()
    b = _aviary(solid=True)
    b.loadURDF(PLATFORM, [0, 0, 0])
    assert lib.pfb_set_static_solid(b._h, 0, None) == 0 and lib.pfb_set_static_solid(b._h, 1, None) == 0  # upright: either rule
    assert lib.pfb_set_static_pose(b._h, 0, C.c_void_p(pos.data_ptr()), C.c_void_p(q.data_ptr()), None, None) == 0
    assert lib.pfb_set_static_solid(b._h, 0, None) != 0 and b"tilted" in lib.pfb_last_error()
    b.reset()
    assert lib.pfb_set_static_solid(b._h, 0, None) == 0 and lib.pfb_set_static_solid(b._h, 1, None) == 0
    c = _aviary(solid=True)
    c.loadURDF(PLATFORM, [0, 0, 0], tilt)
    assert lib.pfb_set_static_solid(c._h, 0, None) != 0


def _wall_flight(av, n, start):
    av.set_mode(7)
    av.set_all_setpoints(np.column_stack([np.full(n, 4.0), start[:, 1], np.zeros(n), np.full(n, 1.0)]))


@pytest.mark.gpu
def test_upright_scene_through_tilted_ctx():
    """an upright scene (a wall, a pillar-free platform) stepped through TiltedCtx, forced by one extra tilted body 1000 m away,
    against the same scene on SolidCtx (the extra body upright): the same bits at every step, the state within fp32 bars"""
    n = 32
    rng = np.random.default_rng(31)
    start = np.column_stack([np.zeros(n), rng.uniform(-2, 2, n), np.full(n, 1.0)])
    a, b = _aviary(n, start=start), _aviary(n, start=start)
    for av in (a, b):
        av.loadURDF(WALL, [1.5, 0.0, 0.0], quat(0.0, 0.0, 0.3))
        av.loadURDF(PLATFORM, [-2.0, 0.0, 0.0])
    a.loadURDF(RAMP, FAR, quat(0.0, 0.4, 0.0))
    b.loadURDF(RAMP, FAR)
    for av in (a, b):
        _wall_flight(av, n, start)
    worst = 0.0
    for _ in range(300):
        a.step(1)
        b.step(1)
        assert np.array_equal(a.contact_bodies().cpu().numpy(), b.contact_bodies().cpu().numpy())
        worst = max(worst, float(np.abs(a.all_states.cpu().numpy()[:, 3] - b.all_states.cpu().numpy()[:, 3]).max()))
    assert a.contact_bodies().cpu().numpy()[:, 1].any() and worst < 2e-2, worst


@pytest.mark.gpu
def test_mixed_handle_equals_single_kind_handles():
    """a mixed-kind Aviary among tilted bodies: every drone flies bit for bit as in a single-kind handle of its kind"""
    import torch
    from pyflyt_b200.core.aviary import BatchedAviary

    kinds = ["quadx", "rocket", "fixedwing", "quadx", "rocket", "quadx"]
    n = len(kinds)
    start = np.column_stack([np.zeros(n), np.arange(n) * 8.0, np.full(n, 1.2)])
    start[1] = (0.0, 8.0, 2.5)  # rocket 1 dropped onto the ramp
    bodies = [(WALL, [1.5, 0.0, 0.0], quat(0.0, 0.3, 0.2)), (RAMP, [0.0, 8.0, 1.0], quat(0.0, 0.35, 0.0)), (BAR, [1.5, 40.0, 0.2], quat(0.0, 0.0, 0.0))]
    sp = np.zeros((n, 7), dtype=np.float32)
    sp[:, 0], sp[:, 1], sp[:, 3] = 4.0, start[:, 1], 1.2
    qx = np.array([k == "quadx" for k in kinds])
    fw_sp = np.array([0.0, 0.0, 0.0, 0.8, 0.0, 0.0], dtype=np.float32)
    mixed = BatchedAviary(start, np.zeros((n, 3)), drone_type=kinds, seed=11, contact_response=True, solid_static_bodies=True)
    for u, p, q in bodies:
        mixed.loadURDF(u, p, q)
    mixed.set_mode([7 if k == "quadx" else 0 for k in kinds])
    allsp = np.where(qx[:, None], sp, 0.0)
    allsp[2, :6] = fw_sp
    mixed.set_all_setpoints(allsp)
    mixed.step(300)
    pm, qm, lm, am = mixed.base_state()
    bits_m = mixed.contact_bodies().cpu().numpy()
    for kind in ("quadx", "fixedwing", "rocket"):
        idx = [i for i, k in enumerate(kinds) if k == kind]
        single = BatchedAviary(start, np.zeros((n, 3)), drone_type=kind, seed=11, contact_response=True, solid_static_bodies=True)
        for u, p, q in bodies:
            single.loadURDF(u, p, q)
        single.set_mode(7 if kind == "quadx" else 0)
        width = {"quadx": 4, "fixedwing": 6, "rocket": 7}[kind]
        ssp = sp[:, :4] if kind == "quadx" else (np.tile(fw_sp, (n, 1)) if kind == "fixedwing" else np.zeros((n, width), dtype=np.float32))
        single.set_all_setpoints(ssp)
        single.step(300)
        ps, qs, ls, as_ = single.base_state()
        for x, y in ((pm, ps), (qm, qs), (lm, ls), (am, as_)):
            assert torch.equal(x[idx], y[idx]), kind
        assert np.array_equal(bits_m[idx], single.contact_bodies().cpu().numpy()[idx]), kind
    assert bits_m[0, 1]  # drone 0 against the pitched wall


@pytest.mark.gpu
def test_masked_tilted_pose_leaves_other_worlds():
    n = 64
    rng = np.random.default_rng(35)
    start = np.column_stack([np.zeros(n), rng.uniform(-2, 2, n), np.full(n, 1.0)])
    a, b = _aviary(n, start=start), _aviary(n, start=start)
    for av in (a, b):
        av.loadURDF(WALL, [1.5, 0, 0])
        av.loadURDF(RAMP, FAR, quat(0.0, 0.4, 0.0))  # both handles on TiltedCtx from the start
        _wall_flight(av, n, start)
    mask = rng.random(n) < 0.5
    b.set_static_pose(0, np.tile([1.6, 0.0, 1.5], (n, 1)), np.tile(quat(0.3, 0.4, 0.2), (n, 1)), mask=mask)
    a.step(360)
    b.step(360)
    sa, sb = a.all_states.cpu().numpy(), b.all_states.cpu().numpy()
    assert np.array_equal(sa[~mask], sb[~mask]) and not np.array_equal(sa[mask], sb[mask])
    cb = b.contact_bodies().cpu().numpy()
    assert np.array_equal(cb[~mask], a.contact_bodies().cpu().numpy()[~mask])


@pytest.mark.gpu
def test_reset_clears_the_tilted_flag():
    """after reset() an upright scene runs bit for bit like a fresh solid handle (SolidCtx again)"""
    start = np.array([[0.0, 0.0, 1.0], [0.0, 1.0, 1.0]])
    a, b = _aviary(2, start=start), _aviary(2, start=start)
    a.loadURDF(RAMP, [0.0, 0.0, 0.5], quat(0.0, 0.3, 0.0))
    a.step(10)
    b.step(10)  # the same number of step launches: the noise streams are keyed by it
    for av in (a, b):
        av.reset()
        av.loadURDF(WALL, [1.5, 0.0, 0.0], quat(0.0, 0.0, 0.4))
        av.set_mode(7)
        av.set_all_setpoints([[4.0, 0.0, 0.0, 1.0], [4.0, 1.0, 0.0, 1.0]])
        av.step(300)
    assert np.array_equal(_state_bytes(a), _state_bytes(b)) and a.contact_bodies().cpu().numpy()[:, 1].all()


@pytest.mark.gpu
def test_friction_cone_on_ramps():
    """cf2x dropped with idle motors on ramps pitched either side of the friction angle atan(0.5) = 26.6 degrees: under it every
    drone rests on the slope, over it every one slides off"""
    n = 64
    rng = np.random.default_rng(37)
    out = {}
    for pitch in (0.35, 0.55):
        start = np.column_stack([rng.uniform(-0.5, 0.5, n), rng.uniform(-0.5, 0.5, n), np.full(n, 1.4)])
        av = _aviary(n, start=start)
        av.loadURDF(RAMP, [0.0, 0.0, 1.0], quat(0.0, pitch, 0.0))
        av.set_mode(-1)
        av.set_all_setpoints(np.zeros((n, 4)))
        av.step(360)
        p = av.all_states.cpu().numpy()[:, 3]
        out[pitch] = (p[:, 0] - start[:, 0], p[:, 2])
    assert (np.abs(out[0.35][0]) < 0.15).all() and (out[0.35][1] > 0.7).all()
    assert (out[0.55][0] > 1.0).all()


@pytest.mark.gpu
def test_no_drone_crosses_its_tilted_wall():
    """8 192 QuadX, each world with its own wall pose (random position, yaw within 40 degrees of square to the flight, roll and
    pitch up to 0.4 rad), each drone sent 4 m past it: none ends on the far side of its wall"""
    n, T = 8192, 600
    rng = np.random.default_rng(39)
    xy = rng.uniform(-50, 50, (n, 2))
    ang = np.column_stack([rng.uniform(-0.4, 0.4, n), rng.uniform(-0.4, 0.4, n), rng.uniform(-0.7, 0.7, n)])
    dist = rng.uniform(1.5, 2.5, n)
    start = np.column_stack([xy[:, 0] - dist, xy[:, 1] + rng.uniform(-1.0, 1.0, n), np.full(n, 1.0)])
    a = _aviary(n, start=start)
    a.loadURDF(WALL, [0.0, 0.0, 0.0])
    q = np.array([quat(*r) for r in ang])
    a.set_static_pose(0, np.column_stack([xy, np.full(n, 1.5)]), q)
    a.set_mode(7)
    a.set_all_setpoints(np.column_stack([xy[:, 0] + 4.0, start[:, 1], np.zeros(n), np.full(n, 1.0)]))
    hit = np.zeros(n, dtype=bool)
    for _ in range(T // 30):
        a.step(30)
        hit |= a.contact_bodies().cpu().numpy()[:, 1]
    p = a.all_states.cpu().numpy()[:, 3].astype(np.float64)
    R = np.array([quat_matrix(x) for x in q])
    lx = np.einsum("ni,ni->n", R[:, :, 0], p - np.column_stack([xy, np.full(n, 1.5)]))  # along the wall's own x axis
    assert hit.mean() > 0.9 and (lx < -0.1).all(), (hit.sum(), lx.max())


def _gate_course(rng):
    """QuadXGatesEnv.generate_gates: 4 gates, distances 4-6 m, angles up to (0, 0.3, 1.0) rad from the previous gate"""
    pos, ang = np.array([0.0, 0.0, 1.0]), np.zeros(3)
    gates = []
    for d, a in zip(rng.uniform(4.0, 6.0, 4), rng.uniform(-1.0, 1.0, (4, 3)) * [0.0, 0.3, 1.0]):
        old, new = quat_matrix(quat(*ang)), quat_matrix(quat(*a))
        pos = pos + new @ old @ np.array([0.0, d, 0.0])
        ang = ang + a
        gates.append((pos.copy(), quat(*ang)))
    return gates


@pytest.mark.gpu
def test_gate_course():
    """a 4-gate course (16 primitives, the cap) placed by the reference's generate_gates recipe: drones flown level through the
    opening of a gate set no gate bit; drones flown the same way through a gate's top bar set that gate's bit"""
    n = 64
    gates = _gate_course(np.random.default_rng(41))
    start, sp, which, bar = np.zeros((n, 3)), np.zeros((n, 4)), np.arange(n) % 4, np.arange(n) % 8 >= 4
    for i in range(n):
        c, q = gates[which[i]]
        G = quat_matrix(q)
        h = G[:, 0] * [1.0, 1.0, 0.0]
        h /= np.linalg.norm(h)
        off = np.array([0.0, 0.0, 0.17]) + (0.225 * G[:, 2] if bar[i] else 0.0)
        start[i], tgt = c - 1.5 * h + off, c + 1.5 * h + off
        sp[i] = (tgt[0], tgt[1], 0.0, tgt[2])
    av = _aviary(n, start=start)
    for c, q in gates:
        av.loadURDF(GATE, c.tolist(), q)
    av.set_mode(7)
    av.set_all_setpoints(sp)
    seen = np.zeros((n, 5), dtype=bool)
    for _ in range(300):
        av.step(1)
        seen |= av.contact_bodies().cpu().numpy()
    assert not seen[~bar, 1:].any()
    assert all(seen[i, 1 + which[i]] for i in range(n) if bar[i])
