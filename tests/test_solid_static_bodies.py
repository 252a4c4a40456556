"""Solid static bodies in the Aviary: ``BatchedAviary(..., solid_static_bodies=True)`` makes every face, edge and corner of a
static body solid (SolidCtx in the step kernels; DESIGN.md §4h, "solid static bodies"), where the default rule only has top faces.

CPU: the helpers of the rule through a g++ build (tests/hostsim/hostsim_solid.cpp): the face of each side of a yawed box and the
fp32 boundaries of inside / outside, every tie order, the cylinder's radial / top / bottom choice and its axis, the floor against
a primitive; the cull against the uncalled helper on random poses near every primitive (no bit and no impulse differs); g++
builds of the QuadX, fixed-wing and rocket steps with SolidCtx: a cf2x flown at a wall is flagged and stopped in front of it, a
fixed-wing stops at a 1 m thick wall, a rocket dropped against the side of a pad is pushed off it, bodies out of reach fly the
floor-only step bit for bit.
GPU: the CUDA steps against the host build on the same walls (bits exact, state within fp32 bars); refusals; with every body out
of reach each handle kind flies bit for bit like the option off; a mixed handle equals the single-kind handles; a masked
``set_static_pose`` leaves the other worlds bit for bit; 8 192 QuadX flown at walls at randomised per-world poses never end on
the far side; ``reset()`` keeps the option and removes the bodies."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from engines import GOLDEN, ROOT

STATIC = os.path.join(GOLDEN, "static")
WALL, PILLAR, THICK = (os.path.join(STATIC, f) for f in ("wall_box.urdf", "pillar_cylinder.urdf", "thick_wall.urdf"))
PLATFORM, PAD, TOWER = (os.path.join(STATIC, f) for f in ("platform_box.urdf", "pad_cylinder.urdf", "helipad_tower.urdf"))
FAR = (1000.0, 1000.0, 0.0)  # out of reach of every drone of these tests
f32, i32, u32 = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint32)

_HS = None


def hs():
    global _HS
    if _HS is None:
        out = os.path.join(tempfile.mkdtemp(prefix="pfb_hostsim_solid_"), "libpfb_hostsim_solid.so")
        src = os.path.join(ROOT, "tests", "hostsim", "hostsim_solid.cpp")
        subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-mfma", "-ffp-contract=fast", "-o", out, src], check=True, capture_output=True)
        _HS = C.CDLL(out)
        _HS.hs_last_error.restype = C.c_char_p
    return _HS


class World:
    """A static world in the flat layout of tests/hostsim/hostsim_solid.cpp: primitives (body, kind, centre, yaw, half sizes) and
    the poses of the bodies in each of n worlds ([5 * 8][n]: x, y, z, cos yaw, sin yaw of the base link frame)."""

    def __init__(self, n=1):
        self.n = n
        self.body, self.kind, self.at, self.yaw, self.half = [], [], [], [], []
        self.pose = np.zeros((5 * 8, n), dtype=np.float32)
        self.pose[3::5] = 1.0
        self.n_bodies = 0

    def add(self, prims, pos=(0.0, 0.0, 0.0), yaw=0.0):
        b = self.n_bodies
        for kind, at, pyaw, half in prims:
            self.body.append(b)
            self.kind.append(kind)
            self.at.append(at)
            self.yaw.append((np.cos(pyaw), np.sin(pyaw)))
            self.half.append(half)
        self.n_bodies += 1
        self.place(b, pos, yaw)
        return b

    def place(self, b, pos, yaw, cols=slice(None)):
        self.pose[5 * b + 0, cols], self.pose[5 * b + 1, cols], self.pose[5 * b + 2, cols] = pos
        self.pose[5 * b + 3, cols], self.pose[5 * b + 4, cols] = np.cos(yaw), np.sin(yaw)

    def args(self):
        self._keep = [np.ascontiguousarray(np.asarray(a, dtype=t).reshape(-1)) for a, t in
                      ((self.body, np.int32), (self.kind, np.int32), (self.at, np.float32), (self.yaw, np.float32), (self.half, np.float32))]
        self._keep.append(np.ascontiguousarray(self.pose))
        ptrs = [k.ctypes.data_as(i32 if k.dtype == np.int32 else f32) for k in self._keep]
        return [len(self.body)] + ptrs

    @property
    def all(self):
        return (1 << len(self.body)) - 1


def contact(world, x, y, z, live=None, i=0):
    d, nrm = C.c_float(0), (C.c_float * 3)()
    live = world.all if live is None else live
    f = C.c_float
    assert hs().hs_solid_point_contact(*world.args(), C.c_int64(world.n), C.c_int64(i), C.c_uint32(live), f(x), f(y), f(z), C.byref(d), nrm) == 0
    return d.value, np.array(nrm[:])


def live_of(world, x, y, z, reach, i=0):
    out = C.c_uint32(0)
    f = C.c_float
    assert hs().hs_solid_live(*world.args(), C.c_int64(world.n), C.c_int64(i), f(x), f(y), f(z), f(reach), C.byref(out)) == 0
    return out.value


def f32_step(x, k=1):
    x = np.float32(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, np.float32(np.inf if k > 0 else -np.inf))
    return float(x)


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_box_faces_of_a_yawed_box():
    """each face of a box yawed 30 degrees by its body and 15 more by itself: the depth to that face and its outward normal"""
    w = World()
    yaw = np.pi / 6 + np.pi / 12
    w.add([(0, (0.0, 0.0, 1.0), np.pi / 12, (0.5, 1.0, 1.0))], pos=(2.0, -1.0, 0.0), yaw=np.pi / 6)
    c, s = np.cos(yaw), np.sin(yaw)
    centre = np.array([2.0, -1.0, 1.0])
    for local, normal, depth in (((0.45, 0.0, 1.0), (1, 0, 0), 0.05), ((-0.42, 0.1, 0.8), (-1, 0, 0), 0.08), ((0.0, 0.93, 1.2), (0, 1, 0), 0.07),
                                 ((0.1, -0.96, 0.9), (0, -1, 0), 0.04), ((0.1, 0.2, 1.97), (0, 0, 1), 0.03), ((0.2, 0.1, 0.01), (0, 0, -1), 0.01)):
        lx, ly, lz = local[0], local[1], local[2] - 1.0
        p = centre + [c * lx - s * ly, s * lx + c * ly, lz]
        d, n = contact(w, *p)
        nw = np.array([c * normal[0] - s * normal[1], s * normal[0] + c * normal[1], normal[2]])
        np.testing.assert_allclose(d, depth if normal != (0, 0, -1) else max(depth, -p[2]), atol=2e-6)
        if normal != (0, 0, -1):  # the bottom face lies on the floor: the floor (depth -z) is as deep and wins the tie
            np.testing.assert_allclose(n, nw, atol=1e-6)
    d, n = contact(w, *(centre + [c * 0.6, s * 0.6, 0.0]))  # outside, beside the +x face
    assert n.tolist() == [0.0, 0.0, 1.0] and d < 0  # the floor's contact: 1 m below


def test_inside_outside_boundaries():
    """on a face the point is inside (depth 0); one fp32 ulp outside it is not; the floor is the answer there"""
    w = World()
    w.add([(0, (0.0, 0.0, 2.0), 0.0, (1.0, 2.0, 0.5))], pos=(3.0, 0.0, 0.0))
    assert contact(w, 4.0, 0.0, 2.0) == (0.0, pytest.approx([1.0, 0.0, 0.0]))
    d, n = contact(w, f32_step(4.0), 0.0, 2.0)
    assert d == np.float32(-2.0) and n.tolist() == [0.0, 0.0, 1.0]
    d, n = contact(w, f32_step(4.0, -1), 0.0, 2.0)
    assert d > 0 and n.tolist() == [1.0, 0.0, 0.0]
    assert contact(w, 3.0, 0.0, 2.5)[1].tolist() == [0.0, 0.0, 1.0] and contact(w, 3.0, 0.0, 2.5)[0] == 0.0
    assert contact(w, 3.0, 0.0, f32_step(2.5))[0] == np.float32(-f32_step(2.5))
    assert contact(w, 3.0, 2.0, 2.0)[1].tolist() == [0.0, 1.0, 0.0]
    assert contact(w, 3.0, f32_step(2.0), 2.0)[1].tolist() == [0.0, 0.0, 1.0]


def test_box_tie_order():
    """equal depths go to +z, then +-x, then +-y, then -z"""
    w = World()
    w.add([(0, (0.0, 0.0, 5.0), 0.0, (1.0, 1.0, 1.0))])
    assert contact(w, 0.5, 0.5, 5.5)[1].tolist() == [0.0, 0.0, 1.0]    # +z, +x and +y at 0.5
    assert contact(w, -0.5, -0.5, 5.0)[1].tolist() == [-1.0, 0.0, 0.0]  # -x and -y at 0.5
    assert contact(w, 0.0, -0.5, 4.5)[1].tolist() == [0.0, -1.0, 0.0]   # -y and -z at 0.5
    assert contact(w, 0.0, 0.0, 5.0)[1].tolist() == [0.0, 0.0, 1.0]     # the centre: all six at 1
    assert contact(w, 0.0, 0.0, 4.2)[1].tolist() == [0.0, 0.0, -1.0]
    assert contact(w, 0.0, 0.3, 4.6)[1].tolist() == [0.0, 0.0, -1.0]


def test_cylinder_choice_and_axis():
    """radial, top and bottom depths: the least wins, ties to top then radial then bottom; on the axis the radial normal is +x of
    the primitive, turned by its yaw"""
    w = World()
    yaw = 0.4
    w.add([(1, (0.0, 0.0, 2.0), yaw, (0.5, 0.5, 1.0))], pos=(1.0, 1.0, 0.0))
    d, n = contact(w, 1.4, 1.0, 2.0)
    np.testing.assert_allclose([d, *n], [0.1, 1.0, 0.0, 0.0], atol=1e-6)
    d, n = contact(w, 1.0, 1.3, 2.9)
    np.testing.assert_allclose([d, *n], [0.1, 0.0, 0.0, 1.0], atol=1e-6)
    d, n = contact(w, 1.0, 1.0, 1.05)
    np.testing.assert_allclose([d, *n], [0.05, 0.0, 0.0, -1.0], atol=1e-6)
    d, n = contact(w, 1.0, 1.5 - 0.25, 2.75)  # radial 0.25 = top 0.25: the top
    assert n.tolist() == [0.0, 0.0, 1.0]
    d, n = contact(w, 1.0, 1.0 - 0.25, 1.25)  # radial 0.25 = bottom 0.25: radial
    np.testing.assert_allclose(n, [0.0, -1.0, 0.0], atol=1e-6)
    w2 = World()
    w2.add([(1, (0.0, 0.0, 0.5), yaw, (0.25, 0.25, 0.5))], pos=(0.0, 0.0, 3.0))  # radius 0.25 < half length: the axis goes radial
    d, n = contact(w2, 0.0, 0.0, 3.5)
    np.testing.assert_allclose([d, *n], [0.25, np.cos(yaw), np.sin(yaw), 0.0], atol=1e-6)


def test_floor_against_primitive():
    """the deepest of the floor and the primitives; the floor wins a tie, then the primitive first in table order"""
    w = World()
    w.add([(0, (0.0, 0.0, 0.0), 0.0, (1.0, 1.0, 0.5))])  # half sunk into the floor
    w.add([(0, (0.0, 0.0, 0.0), 0.0, (1.0, 1.0, 0.5))])  # the same box again, body 1
    assert contact(w, 0.0, 0.0, -0.25)[1].tolist() == [0.0, 0.0, 1.0] and contact(w, 0.0, 0.0, -0.25)[0] == 0.25  # tie: the floor
    d, n = contact(w, 0.0, 0.0, -0.1)  # floor 0.1; the box's nearest face is its bottom, 0.4 deep: deeper, it wins
    assert d == np.float32(0.4) and n.tolist() == [0.0, 0.0, -1.0]
    d, n = contact(w, 0.0, 0.0, 0.1)
    assert d == np.float32(0.4) and n.tolist() == [0.0, 0.0, 1.0]
    d, n = contact(w, 0.95, 0.0, -0.4)  # floor 0.4, +x face 0.05: the floor
    assert d == np.float32(0.4) and n.tolist() == [0.0, 0.0, 1.0]
    d, n = contact(w, 0.95, 0.0, -0.01)  # floor 0.01 < +x 0.05: box 0 (table order beats the identical box 1)
    np.testing.assert_allclose([d, *n], [0.05, 1.0, 0.0, 0.0], atol=1e-6)
    assert contact(w, 0.95, 0.0, -0.01, live=0b10)[0] == pytest.approx(0.05, abs=1e-6)
    assert contact(w, 0.95, 0.0, -0.01, live=0b00)[0] == np.float32(0.01)  # nothing live: the floor


def _cf2x():
    from engines import build_model

    return build_model("quadx", "cf2x")


def _rot(roll, pitch, yaw):
    cr, sr, cp, sp, cy, sy = np.cos(roll), np.sin(roll), np.cos(pitch), np.sin(pitch), np.cos(yaw), np.sin(yaw)
    return np.array([[cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr], [sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr], [-sp, cp * sr, cp * cr]])


def _bits_solve(model, world, live, base, R, v, w):
    bits, vo, wo, t = C.c_uint32(0), (C.c_float * 3)(), (C.c_float * 3)(), C.c_int(0)
    arr = lambda a: np.ascontiguousarray(a, dtype=np.float32)  # noqa: E731
    keep = [arr(base), arr(R).reshape(-1), arr(v), arr(w)]
    assert hs().hs_solid_bits_solve(C.byref(model), *world.args(), C.c_int64(world.n), C.c_int64(0), C.c_uint32(live),
                                    *[k.ctypes.data_as(f32) for k in keep], C.byref(bits), vo, wo, C.byref(t)) == 0
    return bits.value, np.array(vo[:], dtype=np.float32), np.array(wo[:], dtype=np.float32), t.value


def _reach(model):
    """the model's contact reach about its base origin, as the library computes it (contact_zmax)"""
    r = 0.0
    for k in range(model.n_shapes):
        sh = model.shapes[k]
        d = np.sqrt(sum(sh.dims[c] ** 2 for c in range(3))) if sh.kind == 0 else (np.sqrt(sh.dims[0] ** 2 + sh.dims[1] ** 2) if sh.kind == 1 else sh.dims[0])
        r = max(r, float(np.float32((np.linalg.norm(list(sh.at)) + d + model.contact_factor * d) * 1.001)))
    return r


def test_cull_equals_uncalled_helper():
    """random cf2x poses around every primitive of a world (a yawed wall, a pillar, a tower of a box and a cylinder): the bits and
    the solver's velocities over the primitives the cull keeps equal those over every primitive, bit for bit"""
    m = _cf2x()
    reach = _reach(m)
    w = World()
    w.add([(0, (0.0, 0.0, 1.5), 0.2, (0.1, 3.0, 1.5))], pos=(2.0, 0.5, 0.0), yaw=0.3)
    w.add([(1, (0.0, 0.0, 2.0), 0.0, (0.3, 0.3, 2.0))], pos=(-1.0, -2.0, 0.0))
    w.add([(0, (0.0, 0.0, 2.0), np.pi / 6, (1.0, 1.0, 2.0)), (1, (0.5, 0.0, 4.05), 0.0, (0.8, 0.8, 0.05))], pos=(-3.0, 3.0, 0.0), yaw=-0.5)
    rng = np.random.default_rng(11)
    centres = [(2.0, 0.5, 1.5), (-1.0, -2.0, 2.0), (-3.0, 3.0, 2.0), (-3.0 + 0.5 * np.cos(-0.5), 3.0 + 0.5 * np.sin(-0.5), 4.05)]
    halves = [(3.0, 3.0, 1.6), (0.4, 0.4, 2.1), (1.5, 1.5, 2.1), (0.9, 0.9, 0.2)]
    seen_hit, seen_cull = 0, 0
    for k in range(len(centres)):
        for _ in range(300):
            base = np.array(centres[k]) + rng.uniform(-1, 1, 3) * (np.array(halves[k]) + 2.5 * reach)
            R = _rot(*rng.uniform(-0.6, 0.6, 2), rng.uniform(-np.pi, np.pi))
            v, wb = rng.normal(0, 2, 3), rng.normal(0, 3, 3)
            live = live_of(w, *base, reach)
            a = _bits_solve(m, w, live, base, R, v, wb)
            b = _bits_solve(m, w, w.all, base, R, v, wb)
            assert a[0] == b[0] and a[3] == b[3] and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32)) and np.array_equal(a[2].view(np.uint32), b[2].view(np.uint32))
            seen_hit += b[0] > 1
            seen_cull += live != w.all
    assert seen_hit > 100 and seen_cull > 300  # the poses touch bodies, and the cull drops primitives


def _hs_engine(kind, n, start, orn=None):
    from engines import HostSimEngine, build_model

    eng = HostSimEngine(build_model(kind) if kind != "quadx" else build_model("quadx", "cf2x"), None, n=n, start_pos=start,
                        start_orn=np.zeros((n, 3)) if orn is None else orn)
    eng.reset()
    return eng


def _hs_step(eng, kind, world, noise, contact=True, mode=None):
    L = hs()
    bits = np.zeros(eng.n, dtype=np.uint32)
    nz = np.ascontiguousarray(noise, dtype=np.float32)
    ptr = lambda a, t=f32: a.ctypes.data_as(t)  # noqa: E731
    if kind == "quadx":
        rc = L.hs_aviary_step_solid(C.byref(eng.model), eng.mode, int(contact), *world.args(), ptr(eng.st), ptr(eng.ist, i32), ptr(eng.sp), ptr(nz), 1,
                                    C.c_int64(eng.n), ptr(bits, u32))
    elif kind == "fixedwing":
        full = int(int(eng.model.n_surfaces) == 5)
        rc = L.hs_fw_aviary_step_solid(C.byref(eng.model), eng.mode if mode is None else mode, full, *world.args(), ptr(eng.st), ptr(eng.ist, i32), ptr(eng.sp),
                                       ptr(nz), 1, C.c_int64(eng.n), ptr(bits, u32))
    else:
        rc = L.hs_rk_aviary_step_solid(C.byref(eng.model), *world.args(), ptr(eng.st), ptr(eng.ist, i32), ptr(eng.sp), ptr(nz), 1, C.c_int64(eng.n), ptr(bits, u32))
    assert rc == 0, L.hs_last_error()
    return bits


def test_host_out_of_reach_is_floor_step():
    """bodies out of reach: the solid step is the floor-only step, bit for bit, through touchdowns on the floor"""
    from test_aviary_ground_contact import hostsim_contact_lib

    n, T = 8, 240
    rng = np.random.default_rng(1)
    start = np.column_stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(0.3, 1.0, n)])
    a, b = _hs_engine("quadx", n, start), _hs_engine("quadx", n, start)
    sp = np.column_stack([start[:, 0], start[:, 1], np.zeros(n), np.full(n, -0.5)])
    for e in (a, b):
        e.set_mode(7)
        e.set_setpoints(sp)
    w = World(n)
    w.add([(0, (0.0, 0.0, 0.5), 0.0, (1.0, 1.0, 0.5))], pos=FAR)
    w.add([(1, (0.0, 0.0, 2.0), 0.0, (0.5, 0.5, 2.0))], pos=(0.0, 0.0, 50.0))
    noise = rng.normal(4.0, 1.0, size=(T, a.ups, n))
    Lc = hostsim_contact_lib()
    for t in range(T):
        bits = _hs_step(a, "quadx", w, noise[t])
        nz = np.ascontiguousarray(noise[t], dtype=np.float32)
        assert Lc.hs_aviary_step_contact(C.byref(b.model), b.mode, b.st.ctypes.data_as(f32), b.ist.ctypes.data_as(i32), b.sp.ctypes.data_as(f32),
                                         nz.ctypes.data_as(f32), 1, C.c_int64(n)) == 0
        assert np.array_equal(a.st.view(np.uint32), b.st.view(np.uint32)), t
        assert np.array_equal(bits & 1, b.contact().astype(np.uint32)) and not (bits >> 1).any()


def _wall_world(n, x=1.5, yaw=0.0):
    """wall_box.urdf (0.2 m x 6 m x 3 m) with its base link frame at (x, 0, 0), yawed"""
    w = World(n)
    w.add([(0, (0.0, 0.0, 1.5), 0.0, (0.1, 3.0, 1.5))], pos=(x, 0.0, 0.0), yaw=yaw)
    return w


def test_host_cf2x_stops_at_wall():
    """cf2x in mode 7 sent 4 m past a wall 1.5 m ahead (straight, and yawed 30 degrees): flagged, stopped in front of it, holding
    against it; without the response it is flagged and flies through"""
    for yaw in (0.0, np.pi / 6):
        n, T = 3, 480
        start = np.column_stack([np.zeros(n), np.array([-0.5, 0.0, 0.5]), np.full(n, 1.0)])
        a = _hs_engine("quadx", n, start)
        a.set_mode(7)
        a.set_setpoints(np.column_stack([np.full(n, 4.0), start[:, 1], np.zeros(n), np.full(n, 1.0)]))
        w = _wall_world(n, yaw=yaw)
        noise = np.random.default_rng(3).normal(4.0, 1.0, size=(T, a.ups, n))
        hit = np.zeros(n, dtype=bool)
        for t in range(T):
            bits = _hs_step(a, "quadx", w, noise[t])
            hit |= (bits & 2) != 0
        p = a.state()[:, 3]
        lx = np.cos(yaw) * (p[:, 0] - 1.5) + np.sin(yaw) * p[:, 1]  # along the wall's normal: its near face is at -0.1
        assert hit.all() and (bits & 2).all(), yaw
        assert (lx < -0.1).all() and (lx > -0.2).all(), (yaw, lx)
    b = _hs_engine("quadx", 1, np.array([[0.0, 0.0, 1.0]]))
    b.set_mode(7)
    b.set_setpoints(np.array([[4.0, 0.0, 0.0, 1.0]]))
    w = _wall_world(1)
    noise = np.random.default_rng(3).normal(4.0, 1.0, size=(480, b.ups, 1))
    hit = False
    for t in range(480):
        hit |= bool(_hs_step(b, "quadx", w, noise[t], contact=False)[0] & 2)
    assert hit and b.state()[0, 3, 0] > 3.0  # flagged on the way through: the flags do not need the response


def test_host_fixedwing_stops_at_thick_wall():
    """a fixed-wing in level flight into a 1 m thick wall 20 m ahead is flagged and does not reach its far side"""
    n, T = 2, 360
    start = np.column_stack([np.zeros(n), np.array([-1.0, 1.0]), np.full(n, 5.0)])
    a = _hs_engine("fixedwing", n, start)
    a.set_mode(0)
    a.set_setpoints(np.tile([0.0, 0.0, 0.0, 0.8, 0.0, 0.0], (n, 1)))
    w = World(n)
    w.add([(0, (0.0, 0.0, 10.0), 0.0, (0.5, 20.0, 10.0))], pos=(20.0, 0.0, 0.0))
    noise = np.random.default_rng(5).normal(4.0, 1.0, size=(T, a.ups, n))
    hit = np.zeros(n, dtype=bool)
    for t in range(T):
        hit |= (_hs_step(a, "fixedwing", w, noise[t], mode=0) & 2) != 0
    s = a.state()
    assert hit.all() and (s[:, 3, 0] < 19.6).all(), s[:, 3]


def test_host_rocket_against_pad_side():
    """a rocket dropped beside a 1 m high pad, its base 5 cm outside the side face and its rim over the top: flagged against
    the pad, it lands on the edge and tips away from the pad"""
    n, T = 1, 240
    start = np.array([[2.05, 0.0, 4.0]])
    a = _hs_engine("rocket", n, start)
    w = World(n)
    w.add([(1, (0.0, 0.0, 0.5), 0.0, (2.0, 2.0, 0.5))])
    noise = np.random.default_rng(4).normal(4.0, 1.0, size=(T, a.ups, n))
    seen = 0
    for t in range(T):
        seen |= int(_hs_step(a, "rocket", w, noise[t])[0])
    s = a.state()
    assert seen & 2 and np.isfinite(s).all()
    # its rim lands on the pad's top edge and it tips away from the pad: moving outward, base well above the top, not inside
    assert s[0, 3, 0] > 2.3 and s[0, 2, 0] > 0.5 and s[0, 3, 2] > 3.0, s[0]


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


def test_null_handle_refused():
    from pyflyt_b200 import _lib as L

    assert L.lib().pfb_set_static_solid(None, 1, None) != 0 and b"null handle" in L.lib().pfb_last_error()


@pytest.mark.gpu
def test_refusals():
    from pyflyt_b200 import _lib as L
    from pyflyt_b200.core.aviary import AviaryInitException, BatchedAviary
    from engines import hover_config

    av = _aviary(solid=False)
    assert av.solid_static_bodies is False
    rc = L.lib().pfb_set_static_solid(av._h, 2, None)
    assert rc != 0 and b"must be 0" in L.lib().pfb_last_error()
    with pytest.raises(AviaryInitException, match="solid_static_bodies"):
        BatchedAviary(np.zeros((2, 3)) + [0, 0, 1], np.zeros((2, 3)), env_config=hover_config(), solid_static_bodies=True)
    env = BatchedAviary(np.zeros((2, 3)) + [0, 0, 1], np.zeros((2, 3)), env_config=hover_config())
    rc = L.lib().pfb_set_static_solid(env._h, 1, None)
    assert rc != 0 and b"Aviary handles" in L.lib().pfb_last_error()
    with pytest.raises(AttributeError):
        av.solid_static_bodies = True


KINDS = [
    ("quadx", {}, 7),
    ("quadx", {}, [7, 0, 6, -1]),
    ("quadx", dict(drone_options=[{"drone_model": "cf2x"}, {"drone_model": "primitive_drone"}] * 2), 7),
    ("quadx", dict(drone_options=[{"drone_model": "cf2x"}, {"drone_model": "primitive_drone"}] * 2), [7, 0, 6, -1]),
    ("fixedwing", {}, 0),
    ("fixedwing", {}, [0, -1, 0, -1]),
    ("rocket", {}, 0),
    (["quadx", "fixedwing", "rocket", "quadx"], {}, 0),
    (["quadx", "fixedwing", "rocket", "quadx"], dict(drone_options=[{"control_hz": 120}, {"control_hz": 120}, {"control_hz": 120}, {"control_hz": 60}],
                                                     mixed_control_hz=True), 0),
]


@pytest.mark.gpu
@pytest.mark.parametrize("contact", [False, True])
@pytest.mark.parametrize("case", range(len(KINDS)))
def test_out_of_reach_is_bit_for_bit(case, contact):
    """with every body out of reach (far away, or high above) a handle with solid bodies steps bit for bit like one with the
    option off and no bodies"""
    kind, kw, mode = KINDS[case]
    start = np.array([[0.0, 0.0, 0.3], [1.0, 0.0, 2.0], [-1.0, 1.0, 0.05], [0.5, -0.5, 5.0]])
    a, b = _aviary(kind=kind, contact=contact, start=start, **kw), _aviary(kind=kind, contact=contact, start=start, solid=False, **kw)
    assert a.solid_static_bodies and not b.solid_static_bodies
    a.loadURDF(WALL, FAR)
    a.loadURDF(TOWER, [0.0, 0.0, 60.0])
    for av in (a, b):
        av.set_mode(mode)
        av.step(150)
    assert np.array_equal(_state_bytes(a), _state_bytes(b))
    ca, cb = a.contact_bodies().cpu().numpy(), b.contact_array.cpu().numpy()
    assert ca.shape == (4, 3) and np.array_equal(ca[:, 0], cb) and not ca[:, 1:].any()


def _cuda_vs_host(kind, start, setpoints, mode, T, urdf, pose, yaw, world):
    """the CUDA Aviary and the host build side by side with the same injected draws: the contact bits at every step, and the
    largest position difference"""
    import torch

    n = len(start)
    av = _aviary(n, kind=kind, start=start, seed=0)
    av.loadURDF(urdf, pose, [0.0, 0.0, np.sin(yaw / 2), np.cos(yaw / 2)])
    eng = _hs_engine(kind, n, start)
    for e in (av, eng):
        e.set_mode(mode)
    av.set_all_setpoints(setpoints)
    eng.set_setpoints(setpoints)
    rng = np.random.default_rng(9)
    worst, seen = 0.0, 0
    for t in range(T):
        nz = rng.normal(4.0, 1.0, size=(eng.ups, n)).astype(np.float32)
        av.step(1, torch.as_tensor(nz, device=av.device))
        hb = _hs_step(eng, kind, world, nz, mode=mode)
        gb = av.contact_bodies().cpu().numpy()
        assert np.array_equal(gb[:, 0], (hb & 1) != 0) and np.array_equal(gb[:, 1], (hb & 2) != 0), t
        seen |= int(np.bitwise_or.reduce(hb))
        worst = max(worst, float(np.abs(av.all_states.cpu().numpy()[:, 3].astype(np.float64) - eng.state()[:, 3]).max()))
    return worst, seen


@pytest.mark.gpu
def test_cuda_matches_host_build():
    """cf2x into a wall (straight and yawed 30 degrees), a fixed-wing into a 1 m thick wall, a rocket dropped against a pad's
    side: the CUDA steps flag what the g++ build flags at every step, and their positions stay near it.  Only the position is
    compared, with wide bars: these flights run on long after the impact, pinned against the face, where the fp32 rounding of
    the two builds grows (cf2x: 2.4e-3 m seen on an H100).  The per-component comparison with the reference is the fixture
    replays below."""
    n = 3
    start = np.column_stack([np.zeros(n), np.array([-0.5, 0.0, 0.5]), np.full(n, 1.0)])
    sp = np.column_stack([np.full(n, 4.0), start[:, 1], np.zeros(n), np.full(n, 1.0)]).astype(np.float32)
    for yaw in (0.0, np.pi / 6):
        worst, seen = _cuda_vs_host("quadx", start, sp, 7, 360, WALL, [1.5, 0.0, 0.0], yaw, _wall_world(n, yaw=yaw))
        assert seen & 2 and worst < 1.5e-2, (yaw, worst)
    fw_start = np.column_stack([np.zeros(2), np.array([-1.0, 1.0]), np.full(2, 5.0)])
    w = World(2)
    w.add([(0, (0.0, 0.0, 10.0), 0.0, (0.5, 20.0, 10.0))], pos=(20.0, 0.0, 0.0))
    worst, seen = _cuda_vs_host("fixedwing", fw_start, np.tile([0.0, 0.0, 0.0, 0.8, 0.0, 0.0], (2, 1)).astype(np.float32), 0, 240, THICK,
                                [20.0, 0.0, 0.0], 0.0, w)
    assert seen & 2 and worst < 0.35, worst
    w = World(1)
    w.add([(1, (0.0, 0.0, 0.5), 0.0, (2.0, 2.0, 0.5))])
    with tempfile.TemporaryDirectory() as tmp:
        drum = os.path.join(tmp, "drum.urdf")
        with open(drum, "w") as f:
            f.write('<robot name="d"><link name="b"><collision><origin xyz="0 0 0.5"/><geometry><cylinder radius="2" length="1"/></geometry>'
                    "</collision></link></robot>")
        worst, seen = _cuda_vs_host("rocket", np.array([[2.05, 0.0, 4.0]]), np.zeros((1, 7), dtype=np.float32), 0, 120, drum, [0.0, 0.0, 0.0], 0.0, w)
    assert seen & 2 and worst < 5e-2, worst


@pytest.mark.gpu
def test_mixed_handle_equals_single_kind_handles():
    """a mixed-kind Aviary flying into walls and a pillar: every drone flies bit for bit as in a single-kind handle of its kind"""
    import torch
    from pyflyt_b200.core.aviary import BatchedAviary

    kinds = ["quadx", "rocket", "fixedwing", "quadx", "rocket", "quadx"]
    n = len(kinds)
    start = np.column_stack([np.zeros(n), np.arange(n) * 8.0, np.full(n, 1.2)])
    start[1, :2] = (1.65, 0.0)  # rocket 1 falls beside the wall's far face, in its own world
    bodies = [(WALL, [1.5, 0.0, 0.0]), (PILLAR, [1.5, 40.0, 0.0]), (THICK, [15.0, 16.0, 0.0])]
    sp = np.zeros((n, 7), dtype=np.float32)
    sp[:, 0], sp[:, 1], sp[:, 3] = 4.0, start[:, 1], 1.2  # the QuadX rows: 4 m ahead, past the wall and the pillar
    qx = np.array([k == "quadx" for k in kinds])
    fw_sp = np.array([0.0, 0.0, 0.0, 0.8, 0.0, 0.0], dtype=np.float32)
    mixed = BatchedAviary(start, np.zeros((n, 3)), drone_type=kinds, seed=11, contact_response=True, solid_static_bodies=True)
    for u, p in bodies:
        mixed.loadURDF(u, p)
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
        for u, p in bodies:
            single.loadURDF(u, p)
        single.set_mode(7 if kind == "quadx" else 0)
        width = {"quadx": 4, "fixedwing": 6, "rocket": 7}[kind]
        ssp = sp[:, :4] if kind == "quadx" else (np.tile(fw_sp, (n, 1)) if kind == "fixedwing" else np.zeros((n, width), dtype=np.float32))
        single.set_all_setpoints(ssp)
        single.step(300)
        ps, qs, ls, as_ = single.base_state()
        for x, y in ((pm, ps), (qm, qs), (lm, ls), (am, as_)):
            assert torch.equal(x[idx], y[idx]), kind
        assert np.array_equal(bits_m[idx], single.contact_bodies().cpu().numpy()[idx]), kind
    assert bits_m[0, 1] and bits_m[5, 2]  # drone 0 against the wall, drone 5 against the pillar
    assert (pm[0, 0] < 1.4) and (pm[5, 0] < 1.2)


@pytest.mark.gpu
def test_masked_set_static_pose_leaves_other_worlds():
    n = 64
    rng = np.random.default_rng(5)
    start = np.column_stack([np.zeros(n), rng.uniform(-2, 2, n), np.full(n, 1.0)])
    a, b = _aviary(n, start=start), _aviary(n, start=start)
    for av in (a, b):
        av.loadURDF(WALL, [1.5, 0, 0])
        av.set_mode(7)
        av.set_all_setpoints(np.column_stack([np.full(n, 4.0), start[:, 1], np.zeros(n), np.full(n, 1.0)]))
    mask = rng.random(n) < 0.5
    b.set_static_pose(0, np.tile([30.0, 0.0, 1.5], (n, 1)), np.tile([0.0, 0.0, np.sin(0.3), np.cos(0.3)], (n, 1)), mask=mask)
    a.step(480)
    b.step(480)
    sa, sb = a.all_states.cpu().numpy(), b.all_states.cpu().numpy()
    assert np.array_equal(sa[~mask], sb[~mask])
    assert (sa[:, 3, 0] < 1.4).all() and (np.abs(sb[mask, 3, 0] - 4.0) < 0.2).all()  # the moved wall is out of the masked drones' way
    cb = b.contact_bodies().cpu().numpy()
    assert not cb[mask, 1].any() and cb[~mask, 1].all()


@pytest.mark.gpu
def test_no_drone_crosses_its_wall():
    """8 192 QuadX, each world with its own wall pose (random x, y, yaw within 40 degrees of square to the flight), each drone
    sent 4 m past it at about 2 m/s: every one is flagged, and none ends on the far side of its wall"""
    n, T = 8192, 600
    rng = np.random.default_rng(7)
    xy = rng.uniform(-50, 50, (n, 2))
    yaw = rng.uniform(-0.7, 0.7, n)
    dist = rng.uniform(1.0, 2.5, n)
    start = np.column_stack([xy[:, 0] - dist, xy[:, 1] + rng.uniform(-1.0, 1.0, n), np.full(n, 1.0)])
    a = _aviary(n, start=start)
    a.loadURDF(WALL, [0.0, 0.0, 0.0])
    q = np.zeros((n, 4))
    q[:, 2], q[:, 3] = np.sin(yaw / 2), np.cos(yaw / 2)
    a.set_static_pose(0, np.column_stack([xy, np.full(n, 1.5)]), q)
    a.set_mode(7)
    a.set_all_setpoints(np.column_stack([xy[:, 0] + 4.0, start[:, 1], np.zeros(n), np.full(n, 1.0)]))
    hit = np.zeros(n, dtype=bool)
    for _ in range(T // 30):
        a.step(30)
        hit |= a.contact_bodies().cpu().numpy()[:, 1]
    p = a.all_states.cpu().numpy()[:, 3].astype(np.float64)
    # signed distance along the wall's own x axis from its centre plane: < 0 on the drones' side
    lx = np.cos(yaw) * (p[:, 0] - xy[:, 0]) + np.sin(yaw) * (p[:, 1] - xy[:, 1])
    assert hit.all() and (lx < -0.1).all(), (hit.sum(), lx.max())


@pytest.mark.gpu
def test_reset_keeps_option_and_removes_bodies():
    start = np.array([[0.0, 0.0, 1.0]])
    a, b = _aviary(1, start=start), _aviary(1, start=start, solid=False)
    a.loadURDF(WALL, [1.5, 0.0, 0.0])
    a.step(10)
    b.step(10)  # the same number of step launches: the noise streams are keyed by it
    a.reset()
    b.reset()
    assert a.solid_static_bodies and a.static_bodies == [] and a.contact_bodies().shape == (1, 1)
    for av in (a, b):
        av.set_mode(7)
        av.set_all_setpoints([[4.0, 0.0, 0.0, 1.0]])
        av.step(480)
    assert np.array_equal(_state_bytes(a), _state_bytes(b))  # the wall is gone: a flies through like b
    a.reset()
    a.loadURDF(WALL, [1.5, 0.0, 0.0])
    a.set_mode(7)
    a.set_all_setpoints([[4.0, 0.0, 0.0, 1.0]])
    a.step(480)  # solid again after the reset: stopped by the wall
    assert a.contact_bodies().cpu().numpy()[0, 1] and a.all_states.cpu().numpy()[0, 3, 0] < 1.4


# ------------------------------------------------------------------------------------------------------------------ fixtures
# tests/golden/solid_*.npz (tools/gen_golden.py, group ``solid``): the unmodified reference Aviary with loadURDF(useFixedBase=True)
# + register_all_new_bodies(), each drone in an Aviary of its own, read through contact_array[drone.Id, body] (bits), with the
# contact response, on the fake client with the solid rule (solid_rule, fp64).  The host build and the CUDA Aviary replay them
# with the reference's draws injected: the contact bits exactly at every step, the state within fp32 bars.
import glob  # noqa: E402

from engines import load_golden  # noqa: E402

SOLID_FIXTURES = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, "solid_*.npz")))
# fp32 bars against the reference: what the host build shows, x5 and rounded up, never below the free-flight bars of the GPU
# parity tests (pos 5e-4 m, euler 1e-3 rad, rates and velocities 1e-2), as the static_* replays.  An impact on a wall and the
# drone pinned against it amplify the fp32 rounding (the wall flights end 0.25 s after the impact for that reason).  Host seen:
#                                  pos      euler    angvel   linvel
#   solid_cf2x_per_drone_poses     3.6e-4   1.5e-2   0.85     3.2e-2
#   solid_cf2x_pillar_slide        2.8e-6   5.4e-6   1.6e-4   1.1e-4
#   solid_cf2x_step_straddle       5.5e-7   1.2e-5   6.7e-4   3.1e-5
#   solid_cf2x_wall                1.4e-4   1.0e-2   0.70     1.9e-2
#   solid_cf2x_wall_yawed          1.1e-3   3.1e-2   0.84     5.4e-2
#   solid_fixedwing_wall           9.9e-4   1.3e-3   2.3e-2   1.8e-2
#   solid_primitive_edge_drop      1.0e-4   1.7e-3   0.33     2.7e-2
#   solid_rocket_pad_side          8.9e-7   3.0e-7   1.3e-6   2.6e-5
SOLID_BARS = {
    "solid_cf2x_per_drone_poses": dict(pos=2e-3, euler=8e-2, angvel=4.5, linvel=0.16),
    "solid_cf2x_pillar_slide": dict(pos=5e-4, euler=1e-3, angvel=1e-2, linvel=1e-2),
    "solid_cf2x_step_straddle": dict(pos=5e-4, euler=1e-3, angvel=1e-2, linvel=1e-2),
    "solid_cf2x_wall": dict(pos=7e-4, euler=6e-2, angvel=3.5, linvel=0.1),
    "solid_cf2x_wall_yawed": dict(pos=6e-3, euler=0.16, angvel=4.5, linvel=0.27),
    "solid_fixedwing_wall": dict(pos=5e-3, euler=7e-3, angvel=0.12, linvel=0.1),
    "solid_primitive_edge_drop": dict(pos=6e-4, euler=9e-3, angvel=1.7, linvel=0.14),
    "solid_rocket_pad_side": dict(pos=5e-4, euler=1e-3, angvel=1e-2, linvel=1e-2),
}


def _replay(g, cuda):
    import json

    from test_static_bodies import _errors, _fixture_world, _setpoint_at

    kind, n, T = str(g["drone_type"]), len(g["start_pos"]), len(g["state"])
    states, bits = np.zeros((T, n, 4, 3)), np.zeros((T, n), dtype=np.uint32)
    noise = g["noise"].reshape(T, -1, n).astype(np.float32)
    if cuda:
        import torch
        from pyflyt_b200.core.aviary import BatchedAviary

        av = BatchedAviary(g["start_pos"], g["start_orn"], drone_type=kind, drone_options=json.loads(str(g["drone_options"])), seed=0,
                           contact_response=True, solid_static_bodies=True)
        for f, pos, quat in json.loads(str(g["bodies"])):
            av.loadURDF(os.path.join(STATIC, f), pos, quat)
        moved = {}
        for i, pz in enumerate(json.loads(str(g["poses"]))):
            for k, (pos, quat) in pz.items():
                moved.setdefault(int(k), (np.zeros((n, 3)), np.tile([0.0, 0.0, 0.0, 1.0], (n, 1)), np.zeros(n, dtype=bool)))
                moved[int(k)][0][i], moved[int(k)][1][i], moved[int(k)][2][i] = pos, quat, True
        for k, (pos, quat, mask) in moved.items():
            av.set_static_pose(k, pos, quat, mask=mask)
        av.set_mode(int(g["mode"]))
        nz = torch.as_tensor(noise, device=av.device)
        for t in range(T):
            sp = _setpoint_at(g, t, n)
            if sp is not None:  # the fixed-wing's 4-wide setpoint fills the first columns of the Aviary's 6
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
    (k, *prims), pose = _fixture_world(g).args()
    full = int(kind == "fixedwing" and int(model.n_surfaces) == 5)
    L = hs()
    for t in range(T):
        sp = _setpoint_at(g, t, n)
        if sp is not None:
            eng.set_setpoints(sp)
        nz = np.ascontiguousarray(noise[t])
        b = np.zeros(n, dtype=np.uint32)
        args = (k, *prims, pose, eng.st.ctypes.data_as(f32), eng.ist.ctypes.data_as(i32), eng.sp.ctypes.data_as(f32), nz.ctypes.data_as(f32), 1,
                C.c_int64(n), b.ctypes.data_as(u32))
        if kind == "quadx":
            rc = L.hs_aviary_step_solid(C.byref(model), eng.mode, 1, *args)
        elif kind == "fixedwing":
            rc = L.hs_fw_aviary_step_solid(C.byref(model), eng.mode, full, *args)
        else:
            rc = L.hs_rk_aviary_step_solid(C.byref(model), *args)
        assert rc == 0, L.hs_last_error()
        states[t], bits[t] = eng.state(), b
    return _errors(g, states, bits)


def test_solid_fixtures_present():
    assert set(SOLID_FIXTURES) == set(SOLID_BARS) and len(SOLID_FIXTURES) >= 8


def _check(name, err):
    assert err["bits_mismatch"] == 0, (name, err)
    for k, bar in SOLID_BARS[name].items():
        assert err[k] < bar, (name, k, err[k], bar)


@pytest.mark.parametrize("name", sorted(SOLID_BARS))
def test_host_replays_solid_fixture(name):
    """the g++ build of the solid-rule steps replays the reference: contact bits at every step, state within the fp32 bars"""
    _check(name, _replay(load_golden(name), cuda=False))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SOLID_BARS))
def test_cuda_replays_solid_fixture(name):
    """the CUDA Aviary with solid_static_bodies=True replays the reference: bits at every step, the same bars"""
    _check(name, _replay(load_golden(name), cuda=True))
