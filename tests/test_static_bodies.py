"""Static bodies in the Aviary: ``BatchedAviary.loadURDF(..., useFixedBase=True)`` of pads, platforms and runways, their per-world
poses (``set_static_pose``), their contact flags (``contact_bodies``) and the opt-in contact response on their top faces
(DESIGN.md §4h).

Fixtures (tests/golden/static_*.npz, tools/gen_golden.py group ``static``): the unmodified reference Aviary with loadURDF +
register_all_new_bodies, read through contact_array[drone.Id, body]; the host build and the CUDA Aviary replay them, bits exact.
CPU: the URDF reader; the surface rule of ``static_surface`` at its boundaries (footprint edge, ``z + R_b = top``, offset primitives
in yawed bodies) through a g++ build of the helper (tests/hostsim/hostsim_static.cpp); g++ builds of the QuadX, fixed-wing and
rocket steps with static bodies: the fixture replays, and landings on a platform, runway or pad as on the floor shifted up by its
height; out of reach, the floor-only step bit for bit.
GPU: the fixture replays; every refusal; handles whose static bodies are out of reach step bit for bit like handles without them,
for every Aviary handle kind; a masked ``set_static_pose`` leaves the other drones' worlds bit for bit; 8 192 QuadX at randomised
per-world poses land on their platform or pass beside its rotated edge; a fixed-wing on a runway and a rocket on a pad off the
origin fly as on the shifted floor; a mixed handle equals the single-kind handles; ``reset()`` removes the bodies and their bits."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from engines import GOLDEN, ROOT

STATIC = os.path.join(GOLDEN, "static")
PLATFORM, PAD, RUNWAY, TOWER = (os.path.join(STATIC, f) for f in ("platform_box.urdf", "pad_cylinder.urdf", "runway.urdf", "helipad_tower.urdf"))
FAR = (1000.0, 1000.0, 0.0)  # out of reach of every drone of these tests


def _header_define(name):
    with open(os.path.join(ROOT, "include", "pyflyt_b200.h")) as f:
        for line in f:
            if line.startswith(f"#define {name} "):
                return int(line.split()[2])
    raise KeyError(name)


def _lib():
    from pyflyt_b200 import _lib as L

    return L.lib()


_HS = None


def hostsim_static_lib():
    global _HS
    if _HS is None:
        out = os.path.join(tempfile.mkdtemp(prefix="pfb_hostsim_static_"), "libpfb_hostsim_static.so")
        src = os.path.join(ROOT, "tests", "hostsim", "hostsim_static.cpp")
        subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-mfma", "-ffp-contract=fast", "-o", out, src], check=True, capture_output=True)
        _HS = C.CDLL(out)
        _HS.hs_last_error.restype = C.c_char_p
    return _HS


def _urdf(tmp, name, geometry):
    p = os.path.join(tmp, name)
    with open(p, "w") as f:
        f.write(f'<?xml version="1.0"?><robot name="x"><link name="base"><collision><origin xyz="0 0 0"/><geometry>{geometry}</geometry>'
                "</collision></link></robot>")
    return p


def read_shapes(path, scaling=1.0, with_inertial=False):
    from pyflyt_b200.models import PfbShape

    shapes = (PfbShape * 16)()
    n = C.c_int(0)
    io = (C.c_double * 3)()
    rc = _lib().pfb_static_shapes_from_urdf(path.encode(), float(scaling), shapes, 16, C.byref(n), io)
    out = rc, [shapes[k] for k in range(n.value)]
    return out + (np.array(io[:]),) if with_inertial else out


class World:
    """A static world in the flat layout of tests/hostsim/hostsim_static.cpp: primitives (body, kind, centre, yaw, half sizes)
    and the poses of the bodies in each of n worlds ([5 * 8][n]: x, y, z, cos yaw, sin yaw)."""

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
        i32, f32 = C.POINTER(C.c_int32), C.POINTER(C.c_float)
        self._keep = [np.ascontiguousarray(np.asarray(a, dtype=t).reshape(-1)) for a, t in
                      ((self.body, np.int32), (self.kind, np.int32), (self.at, np.float32), (self.yaw, np.float32), (self.half, np.float32))]
        self._keep.append(np.ascontiguousarray(self.pose))
        ptrs = [k.ctypes.data_as(i32 if k.dtype == np.int32 else f32) for k in self._keep]
        return [len(self.body)] + ptrs[:5], ptrs[5]


def surface(world, px, py, pz, reach=0.1, thr=0.01, i=0):
    L = hostsim_static_lib()
    (n, *prims), pose = world.args()
    s, b = C.c_float(0), C.c_uint32(0)
    f = C.c_float
    assert L.hs_static_surface(n, *prims, pose, C.c_int64(world.n), C.c_int64(i), f(px), f(py), f(pz), f(reach), f(thr), C.byref(s), C.byref(b)) == 0
    return s.value, b.value


def f32_up(x, k=1):
    x = np.float32(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, np.float32(np.inf if k > 0 else -np.inf))
    return float(x)


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_caps_match_header():
    from pyflyt_b200.core import aviary

    assert aviary.MAX_STATIC_BODIES == _header_define("PFB_MAX_STATIC_BODIES") == 8
    assert aviary.MAX_STATIC_SHAPES == _header_define("PFB_MAX_STATIC_SHAPES") == 16


def test_urdf_reader_link_frame_and_scaling():
    rc, sh = read_shapes(PLATFORM)
    assert rc == 0 and len(sh) == 1
    assert sh[0].kind == 0 and list(sh[0].dims) == [1.0, 1.0, 0.5] and list(sh[0].at) == [0.0, 0.0, 0.5]  # base LINK frame, half sizes
    rc, sh = read_shapes(PAD, 2.0)
    assert rc == 0 and sh[0].kind == 1
    np.testing.assert_allclose([sh[0].dims[0], sh[0].dims[1], sh[0].at[2]], [4.0, 0.1, 0.1], rtol=0, atol=1e-15)
    rc, sh = read_shapes(TOWER)
    assert rc == 0 and [s.kind for s in sh] == [0, 1]
    np.testing.assert_allclose(list(sh[1].at), [0.0, 0.0, 4.05], atol=1e-15)  # the pad link, through the fixed joint
    np.testing.assert_allclose([sh[0].rot[0], sh[0].rot[3], sh[0].rot[8]], [np.cos(np.pi / 6), np.sin(np.pi / 6), 1.0], atol=1e-15)


def test_urdf_reader_refuses_meshes_and_reports_spheres():
    with tempfile.TemporaryDirectory() as tmp:
        rc, _ = read_shapes(_urdf(tmp, "mesh.urdf", '<mesh filename="pad.obj"/>'))
        assert rc != 0 and b"other than a box, a cylinder or a sphere" in _lib().pfb_last_error()
        rc, sh = read_shapes(_urdf(tmp, "sphere.urdf", '<sphere radius="1"/>'))
        assert rc == 0 and sh[0].kind == 2  # pfb_add_static_body refuses it


def test_upright_rule():
    from pyflyt_b200.core.aviary import _upright_error

    yaw = 0.7
    assert _upright_error([0.0, 0.0, np.sin(yaw / 2), np.cos(yaw / 2)]) <= 1e-15
    assert _upright_error([np.sin(1e-3), 0.0, 0.0, np.cos(1e-3)]) > 1e-9


def test_surface_footprint_edges():
    """(px, py) on a box's edge is under it and the next fp32 offset outside is not; a cylinder's rim likewise"""
    w = World()
    w.add([(0, (0.0, 0.0, 0.5), 0.0, (1.0, 2.0, 0.5))], pos=(3.0, -1.0, 0.0))
    assert surface(w, 4.0, -1.0, 1.0)[0] == 1.0
    assert surface(w, f32_up(4.0), -1.0, 1.0)[0] == 0.0  # dx = 1 + 4.8e-7
    assert surface(w, 3.0, 1.0, 1.0)[0] == 1.0
    assert surface(w, 3.0, f32_up(1.0), 1.0)[0] == 1.0  # dy = 2 + 1.2e-7 rounds to 2 in fp32: still on the edge
    assert surface(w, 3.0, f32_up(1.0, 2), 1.0)[0] == 0.0  # dy = 2 + 2.4e-7: the next fp32 past the edge
    c = World()
    c.add([(1, (0.0, 0.0, 0.05), 0.0, (2.0, 2.0, 0.05))], pos=(-5.0, 0.0, 0.0))
    assert surface(c, -3.0, 0.0, 0.2)[0] == np.float32(0.1)
    assert surface(c, f32_up(-3.0), 0.0, 0.2)[0] == 0.0  # dx = 2 + 2.4e-7


def test_surface_yawed_rectangle():
    """a box yawed 30 degrees by its body and 60 more by itself = 90 degrees: the long side runs along world y"""
    w = World()
    w.add([(0, (0.0, 0.0, 0.5), np.pi / 3, (3.0, 0.5, 0.5))], pos=(0.0, 0.0, 0.0), yaw=np.pi / 6)
    assert surface(w, 0.0, 2.9, 1.2)[0] == 1.0
    assert surface(w, 2.9, 0.0, 1.2)[0] == 0.0
    assert surface(w, 0.45, -2.9, 1.2)[0] == 1.0
    assert surface(w, 0.55, 0.0, 1.2)[0] == 0.0


def test_surface_offset_primitive_in_yawed_body():
    """a primitive offset from its body's origin turns with the body's yaw, and its own yaw adds to it: probes that a sign error
    in either sine would move to the other side"""
    w = World()
    yaw = np.pi / 6  # +30 degrees: the primitive at (2, 0) of the body lands at (2 cos 30, +2 sin 30) = (1.732, +1.0)
    w.add([(0, (2.0, 0.0, 0.5), np.pi / 6, (0.8, 0.1, 0.5))], pos=(0.0, 0.0, 0.0), yaw=yaw)  # long axis at +60 degrees
    cx, cy = 2.0 * np.cos(yaw), 2.0 * np.sin(yaw)
    assert surface(w, cx, cy, 1.05)[0] == 1.0
    assert surface(w, cx, -cy, 1.05)[0] == 0.0  # the body yawed -30 degrees would put it here
    a = np.pi / 3
    assert surface(w, cx + 0.7 * np.cos(a), cy + 0.7 * np.sin(a), 1.05)[0] == 1.0  # along the long axis, +60 degrees
    assert surface(w, cx + 0.7 * np.cos(a), cy - 0.7 * np.sin(a), 1.05)[0] == 0.0  # -60 degrees: off the 0.1 m half width
    assert surface(w, cx + 0.7 * np.cos(0.0), cy, 1.05)[0] == 0.0  # the primitive's own yaw ignored: off as well


def test_surface_height_guard():
    """a primitive is under the drone only while z + R_b >= its top: at equality it is, one fp32 ulp lower it is not"""
    w = World()
    w.add([(0, (0.0, 0.0, 1.5), 0.0, (1.0, 1.0, 0.5))])  # top at 2
    reach = 0.25
    assert surface(w, 0.0, 0.0, 1.75, reach)[0] == 2.0
    assert surface(w, 0.0, 0.0, f32_up(1.75, -1), reach)[0] == 0.0
    assert surface(w, 0.0, 0.0, f32_up(1.75, 1), reach)[0] == 2.0


def test_surface_highest_top_and_bits():
    """two bodies stacked under the drone: the surface is the higher top; each body's bit follows its own top's flag"""
    w = World()
    w.add([(1, (0.0, 0.0, 0.05), 0.0, (2.0, 2.0, 0.05))])       # body 0: a pad, top 0.1
    w.add([(0, (0.0, 0.0, 0.25), 0.0, (0.5, 0.5, 0.25))])       # body 1: a block, top 0.5
    s, b = surface(w, 0.0, 0.0, 0.505, reach=0.2, thr=0.01)
    assert s == 0.5 and b == 0b100  # touching the block only
    s, b = surface(w, 1.0, 0.0, 0.105, reach=0.2, thr=0.01)
    assert s == np.float32(0.1) and b == 0b010
    s, b = surface(w, 5.0, 0.0, 0.005, reach=0.2, thr=0.01)
    assert s == 0.0 and b == 0b001  # the floor


def test_surface_per_world_pose():
    w = World(n=3)
    b = w.add([(0, (0.0, 0.0, 0.5), 0.0, (1.0, 1.0, 0.5))], pos=FAR)
    w.place(b, (10.0, 0.0, 0.0), 0.0, cols=1)
    assert surface(w, 10.0, 0.0, 1.0, i=0)[0] == 0.0
    assert surface(w, 10.0, 0.0, 1.0, i=1)[0] == 1.0
    assert surface(w, 10.0, 0.0, 1.0, i=2)[0] == 0.0


def _hs_quadx(n, start_pos):
    """the host simulator's QuadX Aviary (cf2x) with the floor-only and the static-body steps, contact response on"""
    from engines import HostSimEngine, build_model

    eng = HostSimEngine(build_model("quadx", "cf2x"), None, n=n, start_pos=start_pos, start_orn=np.zeros((n, 3)))
    eng.reset()
    return eng


def _hs_step_static(eng, world, noise, n_steps=1, contact=True):
    L = hostsim_static_lib()
    (n, *prims), pose = world.args()
    bits = np.zeros(eng.n, dtype=np.uint32)
    f, i32 = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    nz = np.ascontiguousarray(noise, dtype=np.float32)
    rc = L.hs_aviary_step_static(C.byref(eng.model), eng.mode, int(contact), n, *prims, pose, eng.st.ctypes.data_as(f), eng.ist.ctypes.data_as(i32),
                                 eng.sp.ctypes.data_as(f), nz.ctypes.data_as(f), n_steps, C.c_int64(eng.n), bits.ctypes.data_as(C.POINTER(C.c_uint32)))
    assert rc == 0, L.hs_last_error()
    return bits


def _hs_step_floor(eng, noise, n_steps=1):
    from test_aviary_ground_contact import hostsim_contact_lib

    L = hostsim_contact_lib()
    f, i32 = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    nz = np.ascontiguousarray(noise, dtype=np.float32)
    assert L.hs_aviary_step_contact(C.byref(eng.model), eng.mode, eng.st.ctypes.data_as(f), eng.ist.ctypes.data_as(i32), eng.sp.ctypes.data_as(f),
                                    nz.ctypes.data_as(f), n_steps, C.c_int64(eng.n)) == 0


def test_host_out_of_reach_is_floor_step():
    """bodies out of reach: the static-body step is the floor-only step, bit for bit, through a touchdown on the floor"""
    n, T = 8, 240
    rng = np.random.default_rng(1)
    start = np.column_stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(0.3, 1.0, n)])
    a, b = _hs_quadx(n, start), _hs_quadx(n, start)
    a.set_mode(7)
    b.set_mode(7)
    sp = np.column_stack([start[:, 0], start[:, 1], np.zeros(n), np.full(n, -0.5)])
    a.set_setpoints(sp)
    b.set_setpoints(sp)
    w = World(n)
    w.add([(0, (0.0, 0.0, 0.5), 0.0, (1.0, 1.0, 0.5))], pos=FAR)
    w.add([(1, (0.0, 0.0, 2.0), 0.0, (0.5, 0.5, 2.0))], pos=(0.0, 0.0, 50.0))  # above the drones: its top is out of reach
    noise = rng.normal(4.0, 1.0, size=(T, a.ups, n))
    for t in range(T):
        bits = _hs_step_static(a, w, noise[t])
        _hs_step_floor(b, noise[t])
        assert np.array_equal(a.st.view(np.uint32), b.st.view(np.uint32)), t
        assert np.array_equal(bits & 1, b.contact().astype(np.uint32)) and not (bits >> 1).any()


def test_host_platform_landing_is_shifted_floor_landing():
    """QuadX drones descending onto a 1 m platform (mode 7, target below the top) land and rest as drones descending onto the
    floor from 1 m lower: position within the fp32 bars of a 1 m offset, the platform's bit up and the floor's down"""
    n, T, h = 6, 480, 1.0
    rng = np.random.default_rng(2)
    start = np.column_stack([rng.uniform(-0.8, 0.8, n), rng.uniform(-0.8, 0.8, n), rng.uniform(0.3, 0.8, n)])
    plat = _hs_quadx(n, start + [0.0, 0.0, h])
    floor = _hs_quadx(n, start)
    for e, dz in ((plat, h), (floor, 0.0)):
        e.set_mode(7)
        e.set_setpoints(np.column_stack([start[:, 0], start[:, 1], np.zeros(n), np.full(n, dz - 0.3)]))
    w = World(n)
    w.add([(0, (0.0, 0.0, 0.5), 0.0, (1.0, 1.0, 0.5))])
    noise = rng.normal(4.0, 1.0, size=(T, plat.ups, n))
    for t in range(T):
        bits = _hs_step_static(plat, w, noise[t])
        _hs_step_floor(floor, noise[t])
    sa, sb = plat.state(), floor.state()
    np.testing.assert_allclose(sa[:, 3, 2] - h, sb[:, 3, 2], atol=2e-4)
    np.testing.assert_allclose(sa[:, 3, :2], sb[:, 3, :2], atol=2e-4)
    np.testing.assert_allclose(sa[:, :3], sb[:, :3], atol=2e-3)
    assert (bits == 0b10).all() and (floor.contact() == 1).all()
    assert np.abs(sa[:, 2]).max() < 1e-2  # at rest


def test_host_rocket_on_pad_is_shifted_floor_landing():
    """the rocket's Aviary step with a static pad (StaticCtx in rocket_substep): dropped onto a pad off the origin it rests on the
    pad's top as it rests on the floor 0.1 m lower, with the pad's bit up and the floor's down"""
    from engines import HostSimEngine, build_model
    from test_aviary_ground_contact import hostsim_contact_lib

    n, T = 3, 480
    start = np.column_stack([np.full(n, 6.0) + [0.0, 0.5, -0.5], np.full(n, -4.0), np.full(n, 5.0)])
    pad, floor = (HostSimEngine(build_model("rocket"), None, n=n, start_pos=start - [0.0, 0.0, dz], start_orn=np.zeros((n, 3))) for dz in (0.0, 0.1))
    pad.reset()
    floor.reset()
    w = World(n)
    w.add([(1, (0.0, 0.0, 0.05), 0.0, (2.0, 2.0, 0.05))], pos=(6.0, -4.0, 0.0))
    L, Lc = hostsim_static_lib(), hostsim_contact_lib()
    f, i32, u32 = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint32)
    noise = np.random.default_rng(4).normal(4.0, 1.0, size=(T, pad.ups, n)).astype(np.float32)
    bits = np.zeros(n, dtype=np.uint32)
    for t in range(T):
        (k, *prims), pose = w.args()
        nz = np.ascontiguousarray(noise[t])
        assert L.hs_rk_aviary_step_static(C.byref(pad.model), k, *prims, pose, pad.st.ctypes.data_as(f), pad.ist.ctypes.data_as(i32), pad.sp.ctypes.data_as(f),
                                          nz.ctypes.data_as(f), 1, C.c_int64(n), bits.ctypes.data_as(u32)) == 0
        assert Lc.hs_rk_aviary_step_contact(C.byref(floor.model), floor.st.ctypes.data_as(f), floor.ist.ctypes.data_as(i32), floor.sp.ctypes.data_as(f),
                                            nz.ctypes.data_as(f), 1, C.c_int64(n)) == 0
    sa, sb = pad.state(), floor.state()
    # the drop's bounce runs at another altitude, so its rounding differs: a few 1e-4 m of height at the end (still settling),
    # and about 1 cm of the slide the bounce starts
    np.testing.assert_allclose(sa[:, 3, 2] - 0.1, sb[:, 3, 2], atol=2e-3)
    np.testing.assert_allclose(sa[:, 3, :2], sb[:, 3, :2], atol=2e-2)
    assert (bits == 0b10).all() and (floor.contact() == 1).all()


def test_host_fixedwing_runway_landing_is_shifted_floor_landing():
    """the fixed-wing's Aviary step with a static runway (StaticCtx in fixedwing_substep): gliding onto a runway 0.5 m high, yawed
    2 degrees off its path, it lands and slides as on the floor 0.5 m lower, with the runway's bit up and the floor's down"""
    from engines import HostSimEngine, build_model
    from test_aviary_ground_contact import hostsim_contact_lib

    n, T = 4, 600
    start = np.column_stack([np.zeros(n), np.linspace(-1.0, 1.0, n), np.full(n, 1.5)])
    a, b = (HostSimEngine(build_model("fixedwing"), None, n=n, start_pos=start - [0.0, 0.0, dz], start_orn=np.zeros((n, 3))) for dz in (0.0, 0.5))
    for e in (a, b):
        e.reset()
        e.set_mode(0)
        e.set_setpoints(np.tile([0.0, -0.1, 0.0, 0.0, 0.0, 0.0], (n, 1)))
    w = World(n)
    w.add([(0, (0.0, 0.0, 0.25), 0.0, (40.0, 4.0, 0.25))], pos=(45.0, 0.0, 0.0), yaw=np.deg2rad(2.0))
    L, Lc = hostsim_static_lib(), hostsim_contact_lib()
    f, i32, u32 = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint32)
    full = int(int(a.model.n_surfaces) == 5)
    noise = np.random.default_rng(6).normal(4.0, 1.0, size=(T, a.ups, n)).astype(np.float32)
    bits = np.zeros(n, dtype=np.uint32)
    for t in range(T):
        (k, *prims), pose = w.args()
        nz = np.ascontiguousarray(noise[t])
        assert L.hs_fw_aviary_step_static(C.byref(a.model), 0, full, k, *prims, pose, a.st.ctypes.data_as(f), a.ist.ctypes.data_as(i32), a.sp.ctypes.data_as(f),
                                          nz.ctypes.data_as(f), 1, C.c_int64(n), bits.ctypes.data_as(u32)) == 0
        assert Lc.hs_fw_aviary_step_contact(C.byref(b.model), 0, full, b.st.ctypes.data_as(f), b.ist.ctypes.data_as(i32), b.sp.ctypes.data_as(f),
                                            nz.ctypes.data_as(f), 1, C.c_int64(n)) == 0
    sa, sb = a.state(), b.state()
    np.testing.assert_allclose(sa[:, 3, 2] - 0.5, sb[:, 3, 2], atol=2e-4)
    np.testing.assert_allclose(sa[:, 3, :2], sb[:, 3, :2], atol=2e-3)
    assert (sa[:, 3, 0] > 60.0).all() and (bits == 0b10).all() and (b.contact() == 1).all()  # landed, and slid along the runway


# ------------------------------------------------------------------------------------------------------------------ GPU
def _aviary(n=4, kind="quadx", contact=True, seed=3, start=None, **kw):
    from pyflyt_b200.core.aviary import BatchedAviary

    if start is None:
        start = np.column_stack([np.linspace(-1, 1, n), np.zeros(n), np.full(n, 1.0)])
    return BatchedAviary(start, np.zeros((n, 3)), drone_type=kind, seed=seed, contact_response=contact, **kw)


def _state_bytes(av):
    import torch

    torch.cuda.synchronize()
    return av.state_tensor.detach().cpu().numpy().view(np.uint32).copy()


@pytest.mark.gpu
def test_refusals():
    from pyflyt_b200 import _lib as L
    from pyflyt_b200.core.aviary import AviaryInitException, BatchedAviary

    av = _aviary()
    tilt = [np.sin(0.05), 0.0, 0.0, np.cos(0.05)]
    with pytest.raises(L.PfbError, match="upright"):
        av.loadURDF(PLATFORM, [0, 0, 0], tilt)
    with pytest.raises(ValueError, match="useFixedBase"):
        av.loadURDF(PLATFORM, [0, 0, 0], useFixedBase=False)
    with tempfile.TemporaryDirectory() as tmp:
        with pytest.raises(L.PfbError, match="sphere"):
            av.loadURDF(_urdf(tmp, "s.urdf", '<sphere radius="1"/>'), [0, 0, 0])
        with pytest.raises(L.PfbError, match="other than a box"):
            av.loadURDF(_urdf(tmp, "m.urdf", '<mesh filename="x.obj"/>'), [0, 0, 0])
        tilted = os.path.join(tmp, "t.urdf")
        with open(tilted, "w") as f:
            f.write('<robot name="t"><link name="b"><collision><origin rpy="0.3 0 0"/><geometry><box size="1 1 1"/></geometry></collision></link></robot>')
        with pytest.raises(L.PfbError, match="tilted"):
            av.loadURDF(tilted, [0, 0, 0])
    assert av.static_bodies == []
    for k in range(8):
        assert av.loadURDF(PLATFORM, [100.0 * (k + 1), 0, 0]) == k
    with pytest.raises(L.PfbError, match="at most 8 static bodies"):
        av.loadURDF(PLATFORM, [0, 0, 0])
    av.reset()
    with tempfile.TemporaryDirectory() as tmp:
        seven = os.path.join(tmp, "seven.urdf")  # seven boxes on fixed joints
        links = "".join(f'<link name="l{k}"><collision><geometry><box size="1 1 1"/></geometry></collision></link>' for k in range(7))
        joints = "".join(f'<joint name="j{k}" type="fixed"><parent link="l0"/><child link="l{k}"/><origin xyz="{k} 0 0"/></joint>' for k in range(1, 7))
        with open(seven, "w") as f:
            f.write(f'<robot name="seven">{links}{joints}</robot>')
        av.loadURDF(seven, [100.0, 0, 0])
        av.loadURDF(seven, [200.0, 0, 0])
    av.loadURDF(TOWER, [300.0, 0, 0])  # 16 primitives: the cap
    with pytest.raises(L.PfbError, match="at most 16 collision primitives"):
        av.loadURDF(PLATFORM, [0, 0, 0])
    with pytest.raises(ValueError, match="upright"):
        av.set_static_pose(0, [0.0, 0.0, 0.0], tilt)
    with pytest.raises(ValueError, match="no static body"):
        av.set_static_pose(9, [0.0, 0.0, 0.0])
    import torch  # the C-ABI checks the quaternions itself, and changes nothing when one is tilted

    pos = torch.zeros((4, 3), dtype=torch.float64, device=av.device)
    quat = torch.tensor([[0.0, 0.0, 0.0, 1.0]] * 3 + [tilt], dtype=torch.float64, device=av.device)
    rc = _lib().pfb_set_static_pose(av._h, 0, C.c_void_p(pos.data_ptr()), C.c_void_p(quat.data_ptr()), None, None)
    assert rc != 0 and b"quat[3] is not upright" in _lib().pfb_last_error()
    mask = torch.tensor([1, 1, 1, 0], dtype=torch.uint8, device=av.device)  # the tilted one is not in the mask: accepted
    assert _lib().pfb_set_static_pose(av._h, 0, C.c_void_p(pos.data_ptr()), C.c_void_p(quat.data_ptr()), C.c_void_p(mask.data_ptr()), None) == 0
    from engines import hover_config

    env = BatchedAviary(np.zeros((2, 3)) + [0, 0, 1], np.zeros((2, 3)), env_config=hover_config())
    with pytest.raises(AviaryInitException, match="Aviary handles"):
        env.loadURDF(PLATFORM, [0, 0, 0])
    shapes = (__import__("pyflyt_b200.models", fromlist=["PfbShape"]).PfbShape * 1)()
    shapes[0].kind, shapes[0].dims[0], shapes[0].dims[1], shapes[0].dims[2] = 0, 1.0, 1.0, 1.0
    shapes[0].rot[0] = shapes[0].rot[4] = shapes[0].rot[8] = 1.0
    body = C.c_int(-1)
    rc = _lib().pfb_add_static_body(env._h, shapes, 1, (C.c_double * 3)(0, 0, 0), (C.c_double * 4)(0, 0, 0, 1), None, C.byref(body), None)
    assert rc != 0 and b"Aviary handles" in _lib().pfb_last_error()


KINDS = [
    ("quadx", {}, 7),
    ("quadx", {}, [7, 0, 6, -1]),
    ("quadx", dict(drone_options=[{"drone_model": "cf2x"}, {"drone_model": "primitive_drone"}] * 2), 7),
    ("fixedwing", {}, 0),
    ("fixedwing", {}, [0, -1, 0, -1]),
    ("rocket", {}, 0),
    (["quadx", "fixedwing", "rocket", "quadx"], {}, 0),
]


@pytest.mark.gpu
@pytest.mark.parametrize("contact", [False, True])
@pytest.mark.parametrize("case", range(len(KINDS)))
def test_out_of_reach_is_bit_for_bit(case, contact):
    """a handle whose static bodies are out of reach (far away, or high above) steps bit for bit like one without them"""
    kind, kw, mode = KINDS[case]
    start = np.array([[0.0, 0.0, 0.3], [1.0, 0.0, 2.0], [-1.0, 1.0, 0.05], [0.5, -0.5, 5.0]])
    a, b = _aviary(kind=kind, contact=contact, start=start, **kw), _aviary(kind=kind, contact=contact, start=start, **kw)
    a.loadURDF(PLATFORM, FAR)
    a.loadURDF(TOWER, [0.0, 0.0, 60.0])
    a.register_all_new_bodies()
    for av in (a, b):
        av.set_mode(mode)
        av.step(150)
    assert np.array_equal(_state_bytes(a), _state_bytes(b))
    ca, cb = a.contact_bodies().cpu().numpy(), b.contact_array.cpu().numpy()
    assert ca.shape == (4, 3) and np.array_equal(ca[:, 0], cb) and not ca[:, 1:].any()
    assert np.array_equal(a.contact_array.cpu().numpy(), cb)


@pytest.mark.gpu
def test_masked_set_static_pose_leaves_other_worlds():
    n = 64
    rng = np.random.default_rng(5)
    start = np.column_stack([rng.uniform(-0.5, 0.5, n), rng.uniform(-0.5, 0.5, n), np.full(n, 1.5)])
    a, b = _aviary(n, start=start), _aviary(n, start=start)
    for av in (a, b):
        av.loadURDF(PLATFORM, [0, 0, 0])
        av.set_mode(7)
        av.set_all_setpoints(np.column_stack([start[:, :2], np.zeros(n), np.full(n, 0.5)]))
    mask = rng.random(n) < 0.5
    b.set_static_pose(0, np.tile([30.0, 0.0, 0.0], (n, 1)), np.tile([0.0, 0.0, np.sin(0.3), np.cos(0.3)], (n, 1)), mask=mask)
    a.step(360)
    b.step(360)
    sa, sb = a.all_states.cpu().numpy(), b.all_states.cpu().numpy()
    assert np.array_equal(sa[~mask], sb[~mask])
    za, zb = sa[:, 3, 2], sb[:, 3, 2]
    # the moved platform is gone from the masked drones' worlds: they hold their target height 0.5 over the empty floor
    assert (za > 0.95).all() and (np.abs(zb[mask] - 0.5) < 0.1).all()
    cb = b.contact_bodies().cpu().numpy()
    assert not cb[mask].any() and cb[~mask, 1].all() and not cb[~mask, 0].any()


def _shifted_pair(n, kind, top, start, pad_pose, urdf, setpoints, mode, T, yaw=None):
    """a handle whose drones fly over static bodies and one whose drones fly the same start `top` lower over the floor"""
    a = _aviary(n, kind=kind, start=start)
    b = _aviary(n, kind=kind, start=start - np.column_stack([np.zeros(n), np.zeros(n), top]))
    a.loadURDF(urdf, [0.0, 0.0, -10.0])
    q = np.zeros((n, 4))
    q[:, 3] = 1.0
    if yaw is not None:
        q[:, 2], q[:, 3] = np.sin(yaw / 2), np.cos(yaw / 2)
    a.set_static_pose(0, pad_pose, q)
    for av, dz in ((a, top), (b, 0.0)):
        av.set_mode(mode)
        if setpoints is not None:
            av.set_all_setpoints(setpoints(dz))
        av.step(T)
    return a, b


@pytest.mark.gpu
def test_quadx_touchdowns_at_randomised_poses():
    """8 192 QuadX, each world with its own platform pose (random x, y, height, yaw), each drone descending from up to 1.27 m off
    the platform's centre in x and y, so that the rotated square's edge decides: a drone over it lands and rests as the same drone
    does on the floor shifted down by the platform's top; one beside it sinks past the top to its target 0.3 m below it.  Drones within 5 mm of the edge, where
    the descent's drift decides, are left out."""
    n, T = 8192, 480
    rng = np.random.default_rng(7)
    top = rng.uniform(0.2, 3.0, n)
    yaw = rng.uniform(-np.pi, np.pi, n)
    xy = rng.uniform(-20, 20, (n, 2))
    off = rng.uniform(-1.27, 1.27, (n, 2))
    start = np.column_stack([xy + off, top + rng.uniform(0.2, 1.0, n)])
    # in the platform's own axes (a 1 m half-size square): rotate the offset by -yaw
    lx, ly = np.cos(yaw) * off[:, 0] + np.sin(yaw) * off[:, 1], -np.sin(yaw) * off[:, 0] + np.cos(yaw) * off[:, 1]
    margin = 1.0 - np.maximum(np.abs(lx), np.abs(ly))  # > 0: over the platform
    over, beside = margin > 5e-3, margin < -5e-3
    assert over.sum() > 3000 and beside.sum() > 1000
    pose = np.column_stack([xy, top - 0.5])  # the base inertial frame, at the middle of the 1 m high box (platform_box.urdf)
    sp = lambda dz: np.column_stack([start[:, :2], np.zeros(n), np.broadcast_to(dz, n) - 0.3])  # noqa: E731
    a, b = _shifted_pair(n, "quadx", top, start, pose, PLATFORM, sp, 7, T, yaw=yaw)
    sa, sb = a.all_states.cpu().numpy().astype(np.float64), b.all_states.cpu().numpy().astype(np.float64)
    np.testing.assert_allclose(sa[over, 3, 2] - top[over], sb[over, 3, 2], atol=1e-3)
    np.testing.assert_allclose(sa[over, 3, :2], sb[over, 3, :2], atol=1e-3)
    ca = a.contact_bodies().cpu().numpy()
    assert ca[over, 1].all() and not ca[over, 0].any() and b.contact_array.cpu().numpy()[over].all()
    assert not ca[beside, 1].any() and (sa[beside, 3, 2] < np.maximum(top[beside] - 0.2, 0.05)).all()  # below its top, untouched
    assert np.abs(sa[over, 2]).max() < 2e-2  # at rest


@pytest.mark.gpu
def test_fixedwing_belly_landing_on_runway():
    """fixed-wings gliding down onto a runway box (80 m x 8 m, top 0.5 m, yawed 2 degrees off their path, its near end 5 m ahead)
    land and slide on it as on the floor 0.5 m lower"""
    n, T = 4, 600
    start = np.column_stack([np.zeros(n), np.linspace(-1.0, 1.0, n), np.full(n, 1.5)])
    from pyflyt_b200.core.aviary import BatchedAviary

    a = BatchedAviary(start, np.zeros((n, 3)), drone_type="fixedwing", seed=3, contact_response=True)
    b = BatchedAviary(start - [0, 0, 0.5], np.zeros((n, 3)), drone_type="fixedwing", seed=3, contact_response=True)
    yaw = np.deg2rad(2.0)
    a.loadURDF(RUNWAY, [45.0, 0.0, 0.0], [0.0, 0.0, np.sin(yaw / 2), np.cos(yaw / 2)])
    for av in (a, b):
        av.set_mode(0)
        av.set_all_setpoints(np.tile([0.0, -0.1, 0.0, 0.0, 0.0, 0.0], (n, 1)))  # throttle off
        av.step(T)
    sa, sb = a.all_states.cpu().numpy().astype(np.float64), b.all_states.cpu().numpy().astype(np.float64)
    msg = f"positions {sa[:, 3].tolist()} / {sb[:, 3].tolist()}"
    np.testing.assert_allclose(sa[:, 3, 2] - 0.5, sb[:, 3, 2], atol=1e-3, err_msg=msg)  # 5x the host bars
    np.testing.assert_allclose(sa[:, 3, :2], sb[:, 3, :2], atol=1e-2, err_msg=msg)
    ca = a.contact_bodies().cpu().numpy()
    assert ca[:, 1].all() and not ca[:, 0].any(), ca


@pytest.mark.gpu
def test_rocket_on_pad_off_origin():
    """a rocket dropped onto a pad at (6, -4) lands and settles on its top, as one dropped onto the floor 0.1 m lower (its base
    origin rests about 2.4 m above its bottom; the tall body still rocks a little after 4 s)"""
    n, T = 3, 480
    start = np.column_stack([np.full(n, 6.0) + [0.0, 0.5, -0.5], np.full(n, -4.0), np.full(n, 5.0)])
    from pyflyt_b200.core.aviary import BatchedAviary

    a = BatchedAviary(start, np.zeros((n, 3)), drone_type="rocket", seed=3, contact_response=True)
    b = BatchedAviary(start - [0, 0, 0.1], np.zeros((n, 3)), drone_type="rocket", seed=3, contact_response=True)
    a.loadURDF(PAD, [6.0, -4.0, 0.0])
    for av in (a, b):
        av.step(T)
    sa, sb = a.all_states.cpu().numpy().astype(np.float64), b.all_states.cpu().numpy().astype(np.float64)
    msg = f"positions {sa[:, 3].tolist()} / {sb[:, 3].tolist()}, velocities {sa[:, 2].tolist()}"
    np.testing.assert_allclose(sa[:, 3, 2] - 0.1, sb[:, 3, 2], atol=1e-2, err_msg=msg)  # 5x the host bar
    ca = a.contact_bodies().cpu().numpy()
    assert ca[:, 1].all() and not ca[:, 0].any(), (ca, msg)


@pytest.mark.gpu
def test_mixed_handle_equals_single_kind_handles():
    """a mixed-kind Aviary with two pads: every drone flies bit for bit as in a single-kind handle of its kind with the same pads"""
    import torch

    kinds = ["quadx", "rocket", "fixedwing", "quadx", "rocket", "quadx"]
    n = len(kinds)
    start = np.column_stack([np.arange(n) * 5.0, np.zeros(n), np.full(n, 1.2)])
    from pyflyt_b200.core.aviary import BatchedAviary

    mixed = BatchedAviary(start, np.zeros((n, 3)), drone_type=kinds, seed=11, contact_response=True)
    for av in (mixed,):
        av.loadURDF(PAD, [0.0, 0.0, 0.0])
        av.loadURDF(PLATFORM, [15.0, 0.0, 0.0])
    mixed.set_mode([7 if k == "quadx" else 0 for k in kinds])
    sp = np.zeros((n, 7), dtype=np.float32)
    sp[:, 0], sp[:, 3] = start[:, 0], -0.5  # the QuadX rows: descend at their start (x, y) onto whatever is under them
    qx_rows = [i for i, k in enumerate(kinds) if k == "quadx"]
    mixed.set_all_setpoints(np.where(np.isin(np.arange(n), qx_rows)[:, None], sp, 0.0))
    mixed.step(300)
    pm, qm, lm, am = mixed.base_state()
    bits_m = mixed.contact_bodies().cpu().numpy()
    for kind in ("quadx", "fixedwing", "rocket"):
        idx = [i for i, k in enumerate(kinds) if k == kind]
        single = BatchedAviary(start, np.zeros((n, 3)), drone_type=kind, seed=11, contact_response=True)
        single.loadURDF(PAD, [0.0, 0.0, 0.0])
        single.loadURDF(PLATFORM, [15.0, 0.0, 0.0])
        single.set_mode(7 if kind == "quadx" else 0)
        width = {"quadx": 4, "fixedwing": 6, "rocket": 7}[kind]
        single.set_all_setpoints(sp[:, :width] if kind == "quadx" else np.zeros((n, width), dtype=np.float32))
        single.step(300)
        ps, qs, ls, as_ = single.base_state()
        for x, y in ((pm, ps), (qm, qs), (lm, ls), (am, as_)):
            assert torch.equal(x[idx], y[idx]), kind
        assert np.array_equal(bits_m[idx], single.contact_bodies().cpu().numpy()[idx]), kind
    assert bits_m[0, 1] and bits_m[3, 2]  # drone 0 on the pad, drone 3 on the platform


@pytest.mark.gpu
def test_reset_removes_bodies():
    start = np.array([[0.0, 0.0, 1.5]])
    a, b = _aviary(1, start=start), _aviary(1, start=start)
    a.loadURDF(PLATFORM, [0.0, 0.0, 0.0])
    a.step(100)
    b.step(100)  # the same number of step launches: the noise streams are keyed by it
    assert a.contact_bodies().shape == (1, 2)
    a.reset()
    b.reset()
    assert a.static_bodies == [] and a.contact_bodies().shape == (1, 1)
    for av in (a, b):
        av.set_mode(7)
        av.set_all_setpoints([[0.0, 0.0, 0.0, -0.5]])
        av.step(480)
    assert np.array_equal(_state_bytes(a), _state_bytes(b))  # the platform is gone: a lands on the floor like b
    assert a.loadURDF(PAD, [0.0, 0.0, 0.0]) == 0  # scripts reload their bodies after reset()
    a.reset()
    a.loadURDF(PLATFORM, [0.0, 0.0, 0.0])
    a.step(100)  # lands on the platform
    assert a.contact_bodies().cpu().numpy()[0, 1]
    a.reset()
    a.loadURDF(PLATFORM, [0.0, 0.0, 0.0])
    assert not a.contact_bodies().cpu().numpy().any()  # resetSimulation empties contact_array: no bits of the last step survive


# ------------------------------------------------------------------------------------------------------------------ fixtures
# tests/golden/static_*.npz (tools/gen_golden.py, group ``static``): the unmodified reference Aviary with loadURDF(useFixedBase=
# True) + register_all_new_bodies(), each drone in an Aviary of its own, read through contact_array[drone.Id, body] (bits), with
# the contact response, on the fake client with the static-body rule.  The host build and the CUDA Aviary replay them with the
# reference's draws injected: the contact bits exactly at every step, the state within fp32 bars.
import glob  # noqa: E402
import json  # noqa: E402

from engines import load_golden  # noqa: E402

STATIC_FIXTURES = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, "static_*.npz")))
SP_DIM = {"quadx": 4, "fixedwing": 6, "rocket": 7}
# fp32 bars against the reference: what the host build shows, x5 and rounded up, never below the free-flight bars of the GPU
# parity tests (pos 5e-4 m, euler 1e-3 rad, rates and velocities 1e-2), as the ground_* replays.  Each touchdown, tip-over and
# bounce amplifies the fp32 rounding, and a resting body chatters at a phase the rounding decides; the rocket's 5 m drop onto the
# pad bounces hardest.  Host build seen:  pos      euler    angvel   linvel
#   static_cf2x_beside_under            2.0e-5   2.6e-5   1.5e-3   6.2e-4
#   static_cf2x_per_drone_poses         1.1e-4   4.3e-6   5.4e-5   4.6e-3
#   static_cf2x_platform_hop            9.2e-5   1.9e-3   0.29     9.4e-3
#   static_fixedwing_runway             2.2e-3   2.3e-5   5.1e-3   2.0e-3
#   static_primitive_edge_drop          1.7e-4   2.7e-3   0.35     3.0e-2
#   static_rocket_pad                   6.4e-2   2.5e-2   0.21     0.37
STATIC_BARS = {
    "static_cf2x_beside_under": dict(pos=5e-4, euler=1e-3, angvel=1e-2, linvel=1e-2),
    "static_cf2x_per_drone_poses": dict(pos=1e-3, euler=1e-3, angvel=1e-2, linvel=3e-2),
    "static_cf2x_platform_hop": dict(pos=5e-4, euler=1e-2, angvel=1.5, linvel=5e-2),
    "static_fixedwing_runway": dict(pos=2e-2, euler=1e-3, angvel=3e-2, linvel=1.2e-2),
    "static_primitive_edge_drop": dict(pos=1e-3, euler=2e-2, angvel=2.0, linvel=0.2),
    "static_rocket_pad": dict(pos=0.35, euler=0.13, angvel=1.1, linvel=1.9),
}


def _fixture_world(g):
    """the fixture's static bodies as the flat World of the host build: primitives read by the library's URDF reader, body k of
    drone i's world at its loadURDF pose, or at the pose resetBasePositionAndOrientation gave its base inertial frame"""
    n = len(g["start_pos"])
    w = World(n)
    inertial = []
    for f, pos, quat in json.loads(str(g["bodies"])):
        rc, shapes, io = read_shapes(os.path.join(STATIC, f), with_inertial=True)
        assert rc == 0
        inertial.append(io)
        prims = []
        for s in shapes:
            half = tuple(s.dims) if s.kind == 0 else (s.dims[0], s.dims[0], s.dims[1])
            prims.append((s.kind, tuple(s.at), float(np.arctan2(s.rot[3], s.rot[0])), half))
        w.add(prims, pos=tuple(pos), yaw=2.0 * np.arctan2(quat[2], quat[3]))
    for i, pz in enumerate(json.loads(str(g["poses"]))):
        for k, (pos, quat) in pz.items():
            yaw = 2.0 * np.arctan2(quat[2], quat[3])
            o = inertial[int(k)]
            link = np.array(pos) - [np.cos(yaw) * o[0] - np.sin(yaw) * o[1], np.sin(yaw) * o[0] + np.cos(yaw) * o[1], o[2]]
            w.place(int(k), tuple(link), yaw, cols=i)
    return w


def _setpoint_at(g, t, n):
    sched = json.loads(str(g["setpoints"]))
    if str(t) not in sched:
        return None
    v = sched[str(t)]
    return np.array([v[str(i)] for i in range(n)] if isinstance(v, dict) else [v] * n, dtype=np.float64)


def _errors(g, states, bits):
    ref = g["state"]  # [T][n][4][3]
    err = {k: float(np.max(np.abs(states[:, :, r] - ref[:, :, r]))) for k, r in (("angvel", 0), ("linvel", 2), ("pos", 3))}
    err["euler"] = float(np.max(np.abs(np.angle(np.exp(1j * (states[:, :, 1] - ref[:, :, 1]))))))  # modulo 2 pi
    err["bits_mismatch"] = int(np.sum(bits != g["bits"]))
    return err


def replay_host(g):
    from engines import HostSimEngine, build_model

    kind, n, T = str(g["drone_type"]), len(g["start_pos"]), len(g["state"])
    model = build_model(kind, **json.loads(str(g["drone_options"])))
    eng = HostSimEngine(model, None, n=n, start_pos=g["start_pos"], start_orn=g["start_orn"])
    eng.reset()
    eng.set_mode(int(g["mode"]))
    w = _fixture_world(g)
    L = hostsim_static_lib()
    f, i32, u32 = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint32)
    noise = g["noise"].reshape(T, -1, n).astype(np.float32)
    states, bits = np.zeros((T, n, 4, 3)), np.zeros((T, n), dtype=np.uint32)
    full = int(kind == "fixedwing" and int(model.n_surfaces) == 5)
    for t in range(T):
        sp = _setpoint_at(g, t, n)
        if sp is not None:
            eng.set_setpoints(sp)
        (k, *prims), pose = w.args()
        nz = np.ascontiguousarray(noise[t])
        b = np.zeros(n, dtype=np.uint32)
        args = (k, *prims, pose, eng.st.ctypes.data_as(f), eng.ist.ctypes.data_as(i32), eng.sp.ctypes.data_as(f), nz.ctypes.data_as(f), 1, C.c_int64(n),
                b.ctypes.data_as(u32))
        if kind == "quadx":
            rc = L.hs_aviary_step_static(C.byref(model), eng.mode, 1, *args)
        elif kind == "fixedwing":
            rc = L.hs_fw_aviary_step_static(C.byref(model), eng.mode, full, *args)
        else:
            rc = L.hs_rk_aviary_step_static(C.byref(model), *args)
        assert rc == 0, L.hs_last_error()
        states[t], bits[t] = eng.state(), b
    return _errors(g, states, bits)


def replay_cuda(g):
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary

    kind, n, T = str(g["drone_type"]), len(g["start_pos"]), len(g["state"])
    av = BatchedAviary(g["start_pos"], g["start_orn"], drone_type=kind, drone_options=json.loads(str(g["drone_options"])), seed=0,
                       contact_response=True)
    for f, pos, quat in json.loads(str(g["bodies"])):
        av.loadURDF(os.path.join(STATIC, f), pos, quat)
    av.register_all_new_bodies()
    moved = {}
    for i, pz in enumerate(json.loads(str(g["poses"]))):
        for k, (pos, quat) in pz.items():
            moved.setdefault(int(k), (np.zeros((n, 3)), np.tile([0.0, 0.0, 0.0, 1.0], (n, 1)), np.zeros(n, dtype=bool)))
            moved[int(k)][0][i], moved[int(k)][1][i], moved[int(k)][2][i] = pos, quat, True
    for k, (pos, quat, mask) in moved.items():
        av.set_static_pose(k, pos, quat, mask=mask)
    av.set_mode(int(g["mode"]))
    noise = torch.as_tensor(g["noise"].reshape(T, -1, n).astype(np.float32), device=av.device)
    states, bits = np.zeros((T, n, 4, 3)), np.zeros((T, n), dtype=np.uint32)
    for t in range(T):
        sp = _setpoint_at(g, t, n)
        if sp is not None:  # the fixed-wing's 4-wide setpoint fills the first columns of the Aviary's 6
            rows = np.zeros((n, av.setpoint_dim))
            rows[:, : sp.shape[1]] = sp
            av.set_all_setpoints(rows)
        av.step(1, noise=noise[t].contiguous())
        states[t] = av.all_states.cpu().numpy()
        cb = av.contact_bodies().cpu().numpy()
        bits[t] = (cb * (1 << np.arange(cb.shape[1]))).sum(axis=1)
    return _errors(g, states, bits)


def test_static_fixtures_present():
    assert len(STATIC_FIXTURES) == len(STATIC_BARS) and set(STATIC_FIXTURES) == set(STATIC_BARS)


@pytest.mark.parametrize("name", sorted(STATIC_BARS))
def test_host_replays_static_fixture(name):
    """the g++ build of the static-body steps replays the reference: contact bits at every step, state within the fp32 bars"""
    err = replay_host(load_golden(name))
    assert err["bits_mismatch"] == 0, (name, err)
    for k, bar in STATIC_BARS[name].items():
        assert err[k] < bar, (name, k, err[k], bar)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(STATIC_BARS))
def test_cuda_replays_static_fixture(name):
    """the CUDA Aviary (loadURDF, set_static_pose, contact_bodies) replays the reference: bits at every step, the same bars"""
    err = replay_cuda(load_golden(name))
    assert err["bits_mismatch"] == 0, (name, err)
    for k, bar in STATIC_BARS[name].items():
        assert err[k] < bar, (name, k, err[k], bar)
