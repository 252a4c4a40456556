"""The shared math helpers of pyflyt_b200/csrc, one at a time, against fp64 at the inputs where fast GPU math and the host build
part ways (tests/probe/pfb_probe.cu runs each helper element-wise).

Every helper runs three ways: on the H100 (``rcp.approx.ftz``, ``rsqrt.approx.ftz``, ``sqrt.approx.ftz``, ``__logf``,
``__log2f``, ``__expf``, ``__sincosf``), built by g++ (IEEE division and square root, libm) and in fp64.  The device-vs-fp64
gap is what the GPU tests hold; the host-vs-fp64 gap, printed beside it, is what the algorithm costs without the fast forms.
The CPU tests hold the g++ build to the same bars.  Each GPU test prints one ``[device-math ...]`` line with its worst error.

The lock-step suites remain the check of the helpers inside the step kernels, where nvcc may contract FMAs differently."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from engines import ROOT, build_model, euler_zyx_ref, quat_from_euler_ref, sign_rule_quaternions
from pyflyt_b200.core.wind import AnalyticWind

F32 = np.float32
FLT_MIN = float(np.finfo(F32).tiny)
FLT_MAX = float(np.finfo(F32).max)
TWO_PI = 2.0 * math.pi

# ---- the probe libraries ----------------------------------------------------------------------------------------------------
_BUILD = os.path.join(ROOT, "oracle", "_build")
_LIBS = {}


def _lib(device: bool):
    """libpfb_probe.so (nvcc, sm_90a) or libpfb_probe_host.so (g++), built by __graft_entry__.build() into oracle/_build.
    A missing library is built here once; a build that fails is a test failure, never a skip."""
    name = "libpfb_probe.so" if device else "libpfb_probe_host.so"
    if name in _LIBS:
        return _LIBS[name]
    path = os.path.join(_BUILD, name)
    if not os.path.exists(path):
        subprocess.run(["make", "-C", os.path.join(ROOT, "pyflyt_b200", "csrc"), "probe"], check=True, capture_output=True)
    L = C.CDLL(path)
    vp, i64, i32 = C.c_void_p, C.c_int64, C.c_int
    L.probe_last_error.restype = C.c_char_p
    L.probe_atan2.argtypes = [i64, vp, vp, vp]
    L.probe_euler.argtypes = [i64, vp, vp]
    L.probe_roll_pitch.argtypes = [i64, vp, vp]
    L.probe_hover_attitude.argtypes = [i64, vp, i32, vp]
    L.probe_quat_from_euler.argtypes = [i64, vp, vp]
    L.probe_sincos.argtypes = [i64, vp, vp, vp]
    L.probe_surface_force.argtypes = [vp, i32, i64, vp, vp, vp, vp, vp]
    L.probe_box_muller.argtypes = [i64, vp, vp, vp, vp]
    L.probe_wind_profile.argtypes = [vp, i64, vp, vp]
    L.probe_solve_sym3.argtypes = [i64, vp, vp, vp]
    L.probe_fast.argtypes = [i32, i64, vp, vp]
    L.probe_contact_impulses.argtypes = [vp, i64] + [vp] * 10
    L.probe_contact_flag.argtypes = [vp, i64, vp, vp, vp, vp]
    assert L.probe_is_device() == int(device), path
    _LIBS[name] = L
    return L


class Probe:
    """Calls one probe entry on numpy inputs and returns numpy outputs; the device build gets CUDA copies."""

    def __init__(self, device: bool):
        self.device = device
        self.L = _lib(device)
        self.name = "device" if device else "host"

    def __call__(self, fn, pre, ins, outs, mid=()):
        """fn(*pre, n, *ins, *mid, *outs); ``ins`` numpy arrays with n rows, ``outs`` (row width, dtype) pairs."""
        n = len(ins[0])
        if self.device:
            import torch

            keep = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in ins]
            res = [torch.empty((n, w), dtype=torch.float32 if dt == F32 else torch.int32, device="cuda") for w, dt in outs]
            ptrs = [t.data_ptr() for t in keep] + list(mid) + [t.data_ptr() for t in res]
        else:
            keep = [np.ascontiguousarray(a) for a in ins]
            res = [np.zeros((n, w), dtype=dt) for w, dt in outs]
            ptrs = [a.ctypes.data for a in keep] + list(mid) + [a.ctypes.data for a in res]
        rc = getattr(self.L, fn)(*pre, n, *ptrs)
        assert rc == 0, self.L.probe_last_error().decode()
        out = [r.cpu().numpy() if self.device else r for r in res]
        return [o[:, 0] if o.shape[1] == 1 else o for o in out]

    def atan2(self, y, x):
        return self(fn="probe_atan2", pre=(), ins=[F32(y), F32(x)], outs=[(1, F32)])[0]

    def euler(self, q):
        return self("probe_euler", (), [F32(q)], [(3, F32)])[0]

    def roll_pitch(self, q):
        return self("probe_roll_pitch", (), [F32(q)], [(2, F32)])[0]

    def hover_attitude(self, q, quaternion):
        return self("probe_hover_attitude", (), [F32(q)], [(4 if quaternion else 3, F32)], mid=(int(quaternion),))[0]

    def quat_from_euler(self, e):
        return self("probe_quat_from_euler", (), [F32(e)], [(4, F32)])[0]

    def sincos(self, x):
        return self("probe_sincos", (), [F32(x)], [(1, F32), (1, F32)])

    def surface(self, model, si, act, vb, w):
        return self("probe_surface_force", (C.byref(model), si), [F32(act), F32(vb), F32(w)], [(3, F32), (3, F32)])

    def box_muller(self, a, b):
        return self("probe_box_muller", (), [np.uint32(a), np.uint32(b)], [(1, F32), (1, F32)])

    def wind(self, wind_struct, z):
        return self("probe_wind_profile", (C.byref(wind_struct),), [F32(z)], [(1, F32)])[0]

    def solve_sym3(self, J, r):
        return self("probe_solve_sym3", (), [F32(J), F32(r)], [(3, F32)])[0]

    def fast(self, which, x):
        return self("probe_fast", (int(which),), [F32(x)], [(1, F32)])[0]

    def contact_impulses(self, model, pz, R, v, w, M, c, Ic, top):
        """apply_contact_impulses: world velocity v and body rate w after the solve (tests/test_contact_solver.py)"""
        ins = [F32(pz), F32(R).reshape(-1, 9), F32(v), F32(w), F32(M), F32(c), F32(Ic), F32(top)]
        return self("probe_contact_impulses", (C.byref(model),), ins, [(3, F32), (3, F32)])

    def contact_flag(self, model, pz, R, top):
        return self("probe_contact_flag", (C.byref(model),), [F32(pz), F32(R).reshape(-1, 9), F32(top)], [(1, np.int32)])[0].astype(bool)


def _f64(a):
    return np.asarray(a, dtype=F32).astype(np.float64)


# ---- atan2_f ------------------------------------------------------------------------------------------------------------------
ATAN2_BAR = 4e-7  # pfb_quadx.cuh: atan2_f (the g++ build reaches 3.2e-7 near the diagonal of the third quadrant)


def atan2_inputs():
    """(y, x) fp32: every sign pair of {+-0, +-2^-149, +-FLT_MIN, +-1, +-2^125}; 2^22 angles on the unit circle; ratios within
    8 ulp of 1 and of the octant edges (0 and inf), every sign; the circle scaled to radii 2^-149 .. 2^125."""
    sp = np.array([0.0, 2.0**-149, FLT_MIN, 1.0, 2.0**125], dtype=F32)
    sp = np.concatenate([sp, -sp])
    y0, x0 = np.meshgrid(sp, sp)
    th = np.linspace(-math.pi, math.pi, 1 << 22, endpoint=False) + 0.5 * TWO_PI / (1 << 22)
    y1, x1 = F32(np.sin(th)), F32(np.cos(th))
    one = F32(1.0)
    k = np.arange(-8, 9)
    ulps = one + k.astype(F32) * np.spacing(one)  # ratio ~ 1 (the diagonal)
    tiny = k[k > 0].astype(F32) * F32(2.0**-24)  # ratio ~ 0 (the axes)
    ys, xs = [y0.ravel(), y1], [x0.ravel(), x1]
    for r in (ulps, tiny):
        for sy in (1, -1):
            for sx in (1, -1):
                ys += [sy * r, sy * np.ones_like(r)]
                xs += [sx * np.ones_like(r), sx * r]
    ang = th[:: (1 << 22) // 2048]
    for e in range(-149, 126):
        s = 2.0**e
        ys.append(F32(np.sin(ang) * s))
        xs.append(F32(np.cos(ang) * s))
    return np.concatenate(ys).astype(F32), np.concatenate(xs).astype(F32)


def measure_atan2(p):
    y, x = atan2_inputs()
    out = p.atan2(y, x).astype(np.float64)
    ref = np.arctan2(_f64(y), _f64(x))
    # atan2_f(+-0, -0) = +-0 where IEEE atan2 gives +-pi: the octant reduction sees a = 0 and x < 0 is false for -0
    zz = (y == 0) & (x == 0) & np.signbit(x)
    assert np.array_equal(out[zz], np.copysign(0.0, _f64(y[zz]))), out[zz]
    keep = ~zz
    mx = np.maximum(np.abs(_f64(y)), np.abs(_f64(x)))
    nonfinite = int((~np.isfinite(out) & keep).sum())
    err = np.abs(out - ref)
    err[~keep] = 0.0
    err[~np.isfinite(err)] = np.inf
    # a subnormal max(|x|, |y|) takes the nearest multiple of pi/2 in its octant pair (atan2_f's comment): held to pi/4
    sub = keep & (mx < FLT_MIN) & (mx > 0)
    worst_sub = float(err[sub].max())
    err[sub] = 0.0
    i = int(np.argmax(err))
    return dict(nonfinite=nonfinite, worst=float(err[i]), at=(float(y[i]), float(x[i])), n=int(keep.sum()), worst_subnormal=worst_sub)


def test_atan2_host():
    m = measure_atan2(Probe(False))
    assert m["nonfinite"] == 0 and m["worst"] <= ATAN2_BAR and m["worst_subnormal"] <= math.pi / 4 + ATAN2_BAR, m


@pytest.mark.gpu
def test_atan2_device():
    h, d = measure_atan2(Probe(False)), measure_atan2(Probe(True))
    print(f"[device-math atan2_f] {d['n']} inputs: device max |err| {d['worst']:.3e} rad at (y, x) = {d['at']} for max(|x|, |y|) >= FLT_MIN, "
          f"{d['worst_subnormal']:.3e} below; {d['nonfinite']} non-finite; host {h['worst']:.3e}")
    assert d["nonfinite"] == 0, d
    assert d["worst"] <= ATAN2_BAR and d["worst_subnormal"] <= math.pi / 4 + ATAN2_BAR, d


# ---- Euler angles and the Hover attitude block ---------------------------------------------------------------------------------
QUAT_OBS_BAR = 2e-5  # the host bar of test_hostsim_parity.py::test_observation_quaternion_sign_rule
EULER_BAR = 4e-6  # roll / pitch / yaw where |sarg| <= 0.999 (well away from gimbal lock)
# roll_pitch_from_quat against euler_from_quat: the same expressions, contracted into FMAs independently; near gimbal lock
# ra and rb are O(sqrt(1 - sarg^2)) differences of O(1) products, so one rounding moves roll by ~1e-5
RP_CALM_BAR, RP_BAR = 1e-6, 5e-5


def attitude_quaternions():
    """fp32 unit quaternions: the 24 000 of the sign-rule test, a dense band at |sarg| in [0.9999, 1] and w = 0."""
    rng = np.random.default_rng(11)
    base = sign_rule_quaternions()
    n = 20000
    s = rng.uniform(0.9999, 1.0, n) * rng.choice([-1.0, 1.0], n)
    pitch = np.arcsin(s)
    band = np.array([quat_from_euler_ref(r, p, y) for r, p, y in zip(rng.uniform(-math.pi, math.pi, n), pitch, rng.uniform(-math.pi, math.pi, n))])
    band *= rng.choice([-1.0, 1.0], (n, 1))
    w0 = rng.normal(size=(4000, 4))
    w0[:, 3] = 0.0
    q = np.vstack([base, band, w0 / np.linalg.norm(w0, axis=1, keepdims=True)])
    return F32(q)


def _obs_ref(q, lock):
    roll, pitch, yaw = euler_zyx_ref(q, lock)
    return quat_from_euler_ref(roll, pitch, yaw)


def measure_attitude(p):
    q = attitude_quaternions()
    q64 = _f64(q)
    sarg = -2.0 * (q64[:, 0] * q64[:, 2] - q64[:, 3] * q64[:, 1])
    obs = p.hover_attitude(q, True).astype(np.float64)
    # within a few fp32 ulp of the +-0.99999 snap the fp32 and fp64 sarg may take different branches: accept either branch
    edge = np.abs(np.abs(sarg) - 0.99999) < 4 * 2.0**-24
    err = np.empty(len(q))
    negatives = 0
    for i in range(len(q)):
        r = _obs_ref(q64[i], None)
        negatives += int(r[3] < 0)
        e = np.abs(obs[i] - r).max()
        if edge[i]:
            e = min(e, np.abs(obs[i] - _obs_ref(q64[i], not (abs(sarg[i]) >= 0.99999))).max())
        err[i] = e
    eul = p.euler(q).astype(np.float64)
    rp = p.roll_pitch(q).astype(np.float64)
    eobs = p.hover_attitude(q, False).astype(np.float64)
    calm = np.abs(sarg) <= 0.999
    ref = np.array([euler_zyx_ref(v) for v in q64[calm]])
    d = np.abs(eul[calm] - ref)
    d[:, [0, 2]] = np.minimum(d[:, [0, 2]], TWO_PI - d[:, [0, 2]])  # roll / yaw at +-pi
    i = int(np.argmax(err))
    rp_diff = np.abs(rp - eul[:, :2]).max(axis=1)
    return dict(worst_quat=float(err[i]), at=q[i].tolist(), negatives=negatives, edge=int(edge.sum()), finite=bool(np.isfinite(obs).all() and np.isfinite(eul).all()),
                worst_euler=float(d.max()), rp_vs_euler=float(rp_diff.max()), rp_vs_euler_calm=float(rp_diff[calm].max()),
                eobs_vs_euler=float(np.abs(eobs - eul).max()), n=len(q))


def test_attitude_host():
    m = measure_attitude(Probe(False))
    assert m["finite"] and m["negatives"] > 50, m
    assert m["worst_quat"] < QUAT_OBS_BAR and m["worst_euler"] < EULER_BAR, m
    assert m["rp_vs_euler_calm"] <= RP_CALM_BAR and m["rp_vs_euler"] <= RP_BAR and m["eobs_vs_euler"] == 0.0, m


@pytest.mark.gpu
def test_attitude_device():
    h, d = measure_attitude(Probe(False)), measure_attitude(Probe(True))
    print(f"[device-math attitude] {d['n']} quaternions ({d['edge']} at the gimbal-lock snap, {d['negatives']} with w_e < 0): device quaternion obs "
          f"{d['worst_quat']:.3e} at {d['at']}, Euler (|sarg| <= 0.999) {d['worst_euler']:.3e}, roll/pitch helper vs Euler {d['rp_vs_euler_calm']:.1e} (all {d['rp_vs_euler']:.1e}); "
          f"host {h['worst_quat']:.3e} / {h['worst_euler']:.3e}")
    assert d["finite"] and d["negatives"] > 50, d
    assert d["worst_quat"] < QUAT_OBS_BAR and d["worst_euler"] < EULER_BAR, d
    assert d["rp_vs_euler_calm"] <= RP_CALM_BAR and d["rp_vs_euler"] <= RP_BAR and d["eobs_vs_euler"] == 0.0, d


# ---- quat_from_euler / sincos_f ------------------------------------------------------------------------------------------------
QFE_BAR = 4e-7
SINCOS_BAR = 2e-7  # pfb_fixedwing.cuh: sincos_f


def measure_quat_from_euler(p):
    rng = np.random.default_rng(5)
    n = 1 << 18
    e = np.column_stack([rng.uniform(-math.pi, math.pi, n), rng.uniform(-math.pi / 2, math.pi / 2, n), rng.uniform(-math.pi, math.pi, n)])
    edges = np.array([0.0, math.pi, -math.pi, math.pi / 2, -math.pi / 2], dtype=F32)
    g = np.array(np.meshgrid(edges, edges, edges)).reshape(3, -1).T
    e = F32(np.vstack([e, g]))
    out = p.quat_from_euler(e).astype(np.float64)
    ref = np.array([quat_from_euler_ref(*v) for v in _f64(e)])
    err = np.abs(out - ref).max(axis=1)
    return dict(worst=float(err.max()), at=e[int(np.argmax(err))].tolist(), finite=bool(np.isfinite(out).all()))


def sincos_inputs():
    x = np.linspace(-6.5, 6.5, 1 << 22, dtype=np.float64)
    k = np.arange(-4, 5) * (math.pi / 2)
    near = [F32(v) for v in k]
    ulp = []
    for v in near:
        s = np.spacing(np.abs(v)) if v != 0 else F32(2.0**-149)
        ulp += [v + j * s for j in range(-4, 5)]
    return np.concatenate([F32(x), np.array(ulp, dtype=F32)])


def measure_sincos(p):
    x = sincos_inputs()
    s, c = p.sincos(x)
    xs = _f64(x)
    es, ec = np.abs(s - np.sin(xs)), np.abs(c - np.cos(xs))
    i = int(np.argmax(np.maximum(es, ec)))
    return dict(worst=float(max(es.max(), ec.max())), at=float(x[i]), finite=bool(np.isfinite(s).all() and np.isfinite(c).all()))


def test_quat_from_euler_and_sincos_host():
    q, s = measure_quat_from_euler(Probe(False)), measure_sincos(Probe(False))
    assert q["finite"] and q["worst"] < QFE_BAR, q
    assert s["finite"] and s["worst"] < SINCOS_BAR, s


@pytest.mark.gpu
def test_quat_from_euler_and_sincos_device():
    hq, hs = measure_quat_from_euler(Probe(False)), measure_sincos(Probe(False))
    dq, ds = measure_quat_from_euler(Probe(True)), measure_sincos(Probe(True))
    print(f"[device-math quat_from_euler] device {dq['worst']:.3e} at {dq['at']}, host {hq['worst']:.3e}")
    print(f"[device-math sincos_f] |x| <= 6.5 and k pi/2 +- 4 ulp: device {ds['worst']:.3e} at x = {ds['at']}, host {hs['worst']:.3e}")
    assert dq["finite"] and dq["worst"] < QFE_BAR, dq
    assert ds["finite"] and ds["worst"] < SINCOS_BAR, ds


# ---- surface_force ---------------------------------------------------------------------------------------------------------
SURFACE_MODELS = [("fixedwing", "fixedwing"), ("fixedwing", "acrowing"), ("rocket", "rocket")]
# speeds (m/s): 0; h2 = lifting^2 + forward^2 underflowing to 0; h2 subnormal; h2 at FLT_MIN; then normal flight
TINY_SPEEDS = [0.0, 1e-24, 1e-21, 1e-20, 3e-20, 1.1e-19]
SPEEDS = [1e-3, 0.5, 7.0, 30.0, 100.0]
ACTUATIONS = [-1.0, -0.5, 0.0, 0.5, 1.0]
SURFACE_HOST_BAR = 1e-4  # |dF| / (Q_area area), |dT| / (Q_area area (|r| + chord)): the g++ build reaches 4.6e-5 (acrowing)


def _stall_angles(sf, act):
    """fp64 alpha_stall_N / alpha_stall_P of a PfbSurface at actuation act (lifting_surfaces.py:349-448)"""
    defl = act * sf.deflection_limit_deg * math.pi / 180.0
    dcl = sf.Cl_alpha_3D * sf.aero_tau * sf.eta * defl
    a0 = sf.alpha_0_base - dcl / sf.Cl_alpha_3D
    clp = sf.Cl_alpha_3D * (sf.alpha_stall_P_base - sf.alpha_0_base) + sf.flap_to_chord * dcl
    cln = sf.Cl_alpha_3D * (sf.alpha_stall_N_base - sf.alpha_0_base) + sf.flap_to_chord * dcl
    return a0 + cln / sf.Cl_alpha_3D, a0 + clp / sf.Cl_alpha_3D


def surface_inputs(sf):
    """(act, vb, w, alpha, speed, near_stall): the alpha circle at 4096 angles plus +-4 ulp around each stall angle and +-pi/2,
    every actuation, every speed; w = 0 except on a random quarter of the normal-speed rows"""
    lift, fwd = np.array(sf.lift_unit), np.array(sf.drag_unit)
    circle = np.linspace(-math.pi, math.pi, 4096, endpoint=False)
    rows = []
    for act in ACTUATIONS:
        sn, sp = _stall_angles(sf, act)
        special = []
        for a in (sn, sp, math.pi / 2, -math.pi / 2):
            af = F32(a)
            special += [float(af + j * np.spacing(np.abs(af))) for j in range(-4, 5)]
        alphas = np.concatenate([circle, special])
        near = np.zeros(len(alphas), bool)
        near[len(circle):len(circle) + 18] = True
        for s in TINY_SPEEDS + SPEEDS:
            rows.append((np.full(len(alphas), act), alphas, np.full(len(alphas), s), near))
    act = np.concatenate([r[0] for r in rows])
    alpha = np.concatenate([r[1] for r in rows])
    speed = np.concatenate([r[2] for r in rows])
    near = np.concatenate([r[3] for r in rows])
    # alpha = atan2(-lifting, forward): v = s (cos a fwd - sin a lift)
    vb = speed[:, None] * (np.cos(alpha)[:, None] * fwd[None, :] - np.sin(alpha)[:, None] * lift[None, :])
    w = np.zeros_like(vb)
    rng = np.random.default_rng(2)
    spin = (speed >= 0.5) & (rng.uniform(size=len(speed)) < 0.25)
    w[spin] = rng.normal(0.0, 0.05, (int(spin.sum()), 3)) * speed[spin, None]
    return F32(act), F32(vb), F32(w), alpha, speed, near


def measure_surface(p, kind, name):
    from oracle.oracle import surface_wrench

    model = build_model(kind, name)
    worst = dict(F=0.0, T=0.0, nonfinite=0, tiny=0.0, near=0, at=None)
    for si in range(model.n_surfaces):
        sf = model.surfaces[si]
        act, vb, w, alpha, speed, near = surface_inputs(sf)
        F, T = p.surface(model, si, act, vb, w)
        F0, T0 = surface_wrench(model, si, _f64(act), _f64(vb), _f64(w))
        worst["nonfinite"] += int((~np.isfinite(F)).any(axis=1).sum() + (~np.isfinite(T)).any(axis=1).sum())
        v = _f64(vb) + np.cross(_f64(w), np.array(sf.pos))
        qa = sf.half_rho * sf.area * (v * v).sum(axis=1)  # Q_area of the fp32 inputs, fp64
        eF = np.abs(F - F0).max(axis=1)
        eT = np.abs(T - T0).max(axis=1)
        if near.any():  # either side of the stall discontinuity: the fp64 values a few ulp of alpha away
            for dth in (-1e-5, 1e-5):
                rot = np.cos(dth) * _f64(vb) + np.sin(dth) * np.cross(np.array(sf.torque_unit), _f64(vb))
                F1, T1 = surface_wrench(model, si, _f64(act), rot, _f64(w))
                eF[near] = np.minimum(eF[near], np.abs(F - F1).max(axis=1)[near])
                eT[near] = np.minimum(eT[near], np.abs(T - T1).max(axis=1)[near])
        arm = float(np.linalg.norm(sf.pos)) + sf.chord
        normal = speed >= 1e-3
        rF, rT = eF[normal] / qa[normal], eT[normal] / (qa[normal] * arm)
        i = int(np.argmax(rF))
        if rF[i] > worst["F"]:
            worst["F"], worst["at"] = float(rF[i]), (si, float(act[normal][i]), float(alpha[normal][i]), float(speed[normal][i]))
        worst["T"] = max(worst["T"], float(rT.max()))
        tiny = ~normal
        worst["tiny"] = max(worst["tiny"], float(np.nan_to_num(np.maximum(eF[tiny], eT[tiny]), nan=np.inf).max()))
        worst["near"] += int(near.sum())
    return worst


@pytest.mark.parametrize("kind,name", SURFACE_MODELS)
def test_surface_force_host_matches_oracle(kind, name):
    m = measure_surface(Probe(False), kind, name)
    assert m["nonfinite"] == 0, m
    assert m["F"] < SURFACE_HOST_BAR and m["T"] < SURFACE_HOST_BAR and m["tiny"] < 1e-30, m


@pytest.mark.gpu
@pytest.mark.parametrize("kind,name", SURFACE_MODELS)
def test_surface_force_device(kind, name):
    h, d = measure_surface(Probe(False), kind, name), measure_surface(Probe(True), kind, name)
    print(f"[device-math surface_force {name}] |dF| / (Q_area area): device {d['F']:.3e} at (surface, act, alpha, speed) = {d['at']}, host {h['F']:.3e}; "
          f"|dT| device {d['T']:.3e}, host {h['T']:.3e}; speeds < 1e-3 m/s max |dF|, |dT| {d['tiny']:.1e}; {d['nonfinite']} non-finite; "
          f"{d['near']} inputs within 4 ulp of a stall angle or +-pi/2")
    assert d["nonfinite"] == 0, d
    assert d["F"] <= 2.0 * max(h["F"], 1e-6) and d["T"] <= 2.0 * max(h["T"], 1e-6), (d, h)
    assert d["tiny"] < 1e-30, d


# ---- box_muller --------------------------------------------------------------------------------------------------------------
NOISE_BAR = 5e-4  # the bar test_timed_path_parity.py holds the device noise dump to
FIXED_WORDS = np.array([0x00000000, 0x3FFFFF00, 0x7FFFFF00, 0xBFFFFF00, 0xFFFFFF00, 0x12345600], dtype=np.uint32)


def _unit(words):
    return ((words >> 8).astype(np.float64) + 1.0) * 2.0**-24


def measure_box_muller(p):
    """every u1 (2^24) against the fixed u2 words, then every u2 against the fixed u1 words"""
    every = np.arange(1 << 24, dtype=np.uint32) << 8
    worst, at, nan = 0.0, None, 0
    for fixed_is_b in (True, False):
        for fw in FIXED_WORDS:
            fixed = np.full(len(every), fw, dtype=np.uint32)
            a, b = (every, fixed) if fixed_is_b else (fixed, every)
            n0, n1 = p.box_muller(a, b)
            u1, u2 = _unit(a), _unit(b)
            r = np.sqrt(-2.0 * np.log(u1))
            e = np.maximum(np.abs(n0 - r * np.cos(TWO_PI * u2)), np.abs(n1 - r * np.sin(TWO_PI * u2)))
            nan += int((~np.isfinite(n0)).sum() + (~np.isfinite(n1)).sum())
            e[~np.isfinite(e)] = np.inf
            i = int(np.argmax(e))
            if e[i] > worst:
                worst, at = float(e[i]), (float(u1[i]), float(u2[i]))
    return dict(worst=worst, at=at, nonfinite=nan)


def test_box_muller_host():
    m = measure_box_muller(Probe(False))
    assert m["nonfinite"] == 0 and m["worst"] < 1e-5, m


@pytest.mark.gpu
def test_box_muller_device():
    h, d = measure_box_muller(Probe(False)), measure_box_muller(Probe(True))
    print(f"[device-math box_muller] all 2^24 u1 x {len(FIXED_WORDS)} u2, all 2^24 u2 x {len(FIXED_WORDS)} u1: device max |n - n_fp64| {d['worst']:.3e} "
          f"at (u1, u2) = {d['at']}, {d['nonfinite']} non-finite; host {h['worst']:.3e}")
    assert d["nonfinite"] == 0, d
    assert d["worst"] < NOISE_BAR, d


# ---- wind_profile ------------------------------------------------------------------------------------------------------------
WIND_CASES = [("constant", 1.0 / 7.0), ("power", 0.1), ("power", 1.0 / 7.0), ("power", 0.5), ("power", 2.0), ("log", 1.0 / 7.0), ("exp", 1.0 / 7.0)]
Z_REF, Z0 = 10.0, 0.125
WIND_BAR = 2e-6  # relative over max(1, |ln f|), where f > 1e-6; for the log profile the error of ln(u) over max(1, ln u)


def wind_inputs():
    z = [np.linspace(-10.0, 1e4, 1 << 20), np.geomspace(1e-30, 1e4, 1 << 16)]
    special = [0.0, -0.0, 2.0**-149, -(2.0**-149), 1e-40, FLT_MIN, Z0, Z_REF]
    for v in (Z0, Z_REF):
        f = F32(v)
        special += [float(f + j * np.spacing(f)) for j in range(-4, 5)]
    return F32(np.concatenate(z + [np.array(special)]))


def _wind_ref(kind, alpha, z):
    z = _f64(z)
    if kind == "constant":
        return np.ones_like(z)
    if kind == "power":
        return np.power(np.maximum(z, 0.0) / Z_REF, alpha)
    if kind == "log":
        return np.log(np.maximum(z, Z0) / Z0) / math.log(Z_REF / Z0)
    with np.errstate(over="ignore"):
        return np.exp(z / Z_REF)


def measure_wind(p, kind, alpha):
    w = AnalyticWind(kind, base=(1.0, 0.0, 0.0), z_ref=Z_REF, alpha=alpha, z0=Z0).as_struct()
    z = wind_inputs()
    f = p.wind(w, z).astype(np.float64)
    ref = _wind_ref(kind, alpha, z)
    fits = ref < FLT_MAX * (1.0 - 1e-6)  # the fp64 value has an fp32 neighbour: the helper must be finite there
    nonfinite = int((~np.isfinite(f) & fits).sum())
    zero_miss = int((f[ref == 0.0] != 0.0).sum())
    # z / z_ref below FLT_MIN (|z| < ~1e-37 m) is subnormal in fp32, on both builds: there the power law only has to stay in
    # [0, f(z_ref FLT_MIN)], the value it rises to at the first normal argument
    under = (kind == "power") & (np.abs(_f64(z)) < Z_REF * FLT_MIN)
    f_edge = float(_wind_ref(kind, alpha, np.array([Z_REF * FLT_MIN], dtype=F32))[0]) if kind == "power" else 0.0
    under_miss = int(((f[under] < 0.0) | (f[under] > f_edge * (1.0 + WIND_BAR))).sum())
    sel = fits & (ref > 1e-6) & ~under
    if kind == "log":
        # the error of ln(u), u = max(z, z0) / z0, over max(1, ln u): __logf's bound is ABSOLUTE near u = 1 (2^-21.41 on [0.5, 2])
        L = math.log(Z_REF / Z0)
        rel = np.abs(f[sel] - ref[sel]) * L / np.maximum(1.0, ref[sel] * L)
    else:
        # relative error over the condition of the profile in its argument: |d ln f / d ln(z / z_ref)| is |ln f| for the exponential
        rel = np.abs(f[sel] - ref[sel]) / (ref[sel] * np.maximum(1.0, np.abs(np.log(ref[sel]))))
    rel[~np.isfinite(rel)] = np.inf
    i = int(np.argmax(rel))
    return dict(worst=float(rel[i]), at=float(z[sel][i]), nonfinite=nonfinite, zero_miss=zero_miss, under_miss=under_miss)


@pytest.mark.parametrize("kind,alpha", WIND_CASES)
def test_wind_profile_host(kind, alpha):
    m = measure_wind(Probe(False), kind, alpha)
    assert m["nonfinite"] == 0 and m["zero_miss"] == 0 and m["under_miss"] == 0 and m["worst"] < WIND_BAR, m


@pytest.mark.gpu
@pytest.mark.parametrize("kind,alpha", WIND_CASES)
def test_wind_profile_device(kind, alpha):
    h, d = measure_wind(Probe(False), kind, alpha), measure_wind(Probe(True), kind, alpha)
    what = "|d ln u| / max(1, ln u)" if kind == "log" else "relative error / max(1, |ln f|)"
    print(f"[device-math wind_profile {kind} alpha={alpha:.4g}] {what} where f > 1e-6: device {d['worst']:.3e} at z = {d['at']:.6g}, "
          f"host {h['worst']:.3e}; {d['zero_miss']} non-zero where fp64 is 0, {d['nonfinite']} non-finite, {d['under_miss']} out of range at subnormal z / z_ref")
    assert d["nonfinite"] == 0 and d["zero_miss"] == 0 and d["under_miss"] == 0, d
    assert d["worst"] < WIND_BAR, d


# ---- solve_sym3 --------------------------------------------------------------------------------------------------------------
SYM3_C = 4.0  # |x - x_fp64| / |x_fp64| <= SYM3_C * cond(J) * 2^-22


def rocket_com_inertia(n):
    """J about the COM of the rocket at n fuel fractions in [0, 1] (pfb_rocket.cuh rocket_substep), fp64 rounded to fp32 entries
    (a, b, c, d, e, f) of [[a b c], [b d e], [c e f]]"""
    m = build_model("rocket", "rocket")
    fuel = np.concatenate([np.linspace(0.0, 1.0, n - 2), [0.0, 1.0]])
    fp, dI = np.array(m.fuel_pos), np.array(m.dry_inertia)
    mf = fuel * m.fuel_total_mass
    M = m.dry_mass + mf
    mc = np.array(m.dry_first_moment)[None, :] + mf[:, None] * fp[None, :]
    c = mc / M[:, None]
    fr2 = float(fp @ fp)
    fmi = np.array(m.fuel_max_inertia)
    Ixx = dI[0] + fuel * fmi[0] + mf * (fr2 - fp[0] ** 2)
    Iyy = dI[4] + fuel * fmi[1] + mf * (fr2 - fp[1] ** 2)
    Izz = dI[8] + fuel * fmi[2] + mf * (fr2 - fp[2] ** 2)
    Ixy, Ixz, Iyz = dI[1] - mf * fp[0] * fp[1], dI[2] - mf * fp[0] * fp[2], dI[5] - mf * fp[1] * fp[2]
    c2 = (c * c).sum(axis=1)
    J = np.column_stack([Ixx - M * (c2 - c[:, 0] ** 2), Ixy + M * c[:, 0] * c[:, 1], Ixz + M * c[:, 0] * c[:, 2], Iyy - M * (c2 - c[:, 1] ** 2),
                         Iyz + M * c[:, 1] * c[:, 2], Izz - M * (c2 - c[:, 2] ** 2)])
    return F32(J)


def measure_sym3(p):
    n = 100000
    J = rocket_com_inertia(n)
    r = F32(np.random.default_rng(9).normal(size=(n, 3)))
    x = p.solve_sym3(J, r).astype(np.float64)
    a, b, c, d, e, f = _f64(J).T
    A = np.stack([np.stack([a, b, c], -1), np.stack([b, d, e], -1), np.stack([c, e, f], -1)], 1)
    x0 = np.linalg.solve(A, _f64(r)[:, :, None])[:, :, 0]
    rel = np.linalg.norm(x - x0, axis=1) / np.linalg.norm(x0, axis=1)
    kappa = np.linalg.cond(A)
    ratio = rel / (kappa * 2.0**-22)
    i = int(np.argmax(ratio))
    return dict(worst_ratio=float(ratio[i]), rel=float(rel[i]), kappa=float(kappa[i]), kappa_max=float(kappa.max()), finite=bool(np.isfinite(x).all()))


def test_solve_sym3_host():
    m = measure_sym3(Probe(False))
    assert m["finite"] and m["worst_ratio"] < SYM3_C, m


@pytest.mark.gpu
def test_solve_sym3_device():
    h, d = measure_sym3(Probe(False)), measure_sym3(Probe(True))
    print(f"[device-math solve_sym3] rocket COM inertia at 1e5 fuel fractions (cond <= {d['kappa_max']:.1f}): device max |dx|/|x| / (cond 2^-22) = {d['worst_ratio']:.3f} "
          f"(|dx|/|x| {d['rel']:.2e} at cond {d['kappa']:.1f}); host {h['worst_ratio']:.3f}")
    assert d["finite"] and d["worst_ratio"] < SYM3_C, d


# ---- fast_rcp / fast_rsqrt / fast_sqrt ---------------------------------------------------------------------------------------
SPECIAL = np.array([0.0, -0.0, 2.0**-149, -(2.0**-149), FLT_MIN / 2, FLT_MIN, 1.0, 2.0**126, FLT_MAX, np.inf], dtype=F32)
SPECIAL_NAMES = ["0", "-0", "2^-149", "-2^-149", "FLT_MIN/2", "FLT_MIN", "1", "2^126", "FLT_MAX", "inf"]
FAST = [("fast_rcp", lambda x: 1.0 / x), ("fast_rsqrt", lambda x: 1.0 / np.sqrt(x)), ("fast_sqrt", np.sqrt)]
# ulp bars over the normal inputs whose result is normal: rcp.approx.f32 and sqrt.approx.f32 within 1 ulp (the PTX ISA);
# rsqrt.approx.f32 relative error 2^-22.9, up to 2.1 ulp where the result's mantissa is near 2; the host's 1 / sqrtf rounds twice
FAST_ULP = [1.0, 2.0, 1.0]
# what the device returns for SPECIAL (sm_90a, the .ftz forms): a subnormal input is a signed zero
DEVICE_SPECIAL = {
    "fast_rcp": [np.inf, -np.inf, np.inf, -np.inf, np.inf, 2.0**126, 1.0, 2.0**-126, 0.0, 0.0],
    "fast_rsqrt": [np.inf, -np.inf, np.inf, -np.inf, np.inf, 2.0**63, 1.0, 2.0**-63, float(F32(1.0 / math.sqrt(FLT_MAX))), 0.0],
    "fast_sqrt": [0.0, -0.0, 0.0, -0.0, 0.0, 2.0**-63, 1.0, 2.0**63, float(F32(math.sqrt(FLT_MAX))), np.inf],
}


def normal_sweep():
    rng = np.random.default_rng(4)
    bits = (rng.integers(1, 255, 1 << 20).astype(np.uint32) << 23) | rng.integers(0, 1 << 23, 1 << 20).astype(np.uint32)
    return bits.view(F32)


def measure_fast(p):
    x = normal_sweep()
    out = {}
    for k, (name, ref) in enumerate(FAST):
        xs = x[x < 2.0**126] if name == "fast_rcp" else x  # above 2^126 the reciprocal is subnormal: the table below
        y = p.fast(k, xs).astype(np.float64)
        r = ref(_f64(xs))
        ulp = np.spacing(np.abs(F32(r))).astype(np.float64)
        e = np.abs(y - r) / ulp
        i = int(np.argmax(e))
        with np.errstate(divide="ignore", invalid="ignore"):
            out[name] = dict(ulp=float(e[i]), at=float(xs[i]), special=p.fast(k, SPECIAL).astype(np.float64).tolist())
    return out


def test_fast_forms_host():
    m = measure_fast(Probe(False))
    for k, (name, _) in enumerate(FAST):
        assert m[name]["ulp"] <= FAST_ULP[k], (name, m[name])


@pytest.mark.gpu
def test_fast_forms_device():
    h, d = measure_fast(Probe(False)), measure_fast(Probe(True))
    for k, (name, _) in enumerate(FAST):
        table = ", ".join(f"{a} -> {b:.9g}" for a, b in zip(SPECIAL_NAMES, d[name]["special"]))
        print(f"[device-math {name}] normal inputs: device {d[name]['ulp']:.3f} ulp at {d[name]['at']:.9g}, host {h[name]['ulp']:.3f} ulp; device: {table}")
    for k, (name, _) in enumerate(FAST):
        assert d[name]["ulp"] <= FAST_ULP[k], (name, d[name])
        got, want = np.array(d[name]["special"]), np.array(DEVICE_SPECIAL[name])
        assert np.array_equal(got, want) and np.array_equal(np.signbit(got), np.signbit(want)), (name, got.tolist())
