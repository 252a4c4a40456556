"""TEST INFRASTRUCTURE — ctypes binding of oracle/pfb_oracle.c (the fp64 CPU restatement).

Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs may import this module.
"""

from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.realpath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libpfb_oracle.so")
_lib = None


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "pfb_oracle.c")
    hdr = os.path.join(_HERE, "..", "include", "pyflyt_b200.h")
    stale = (
        force
        or not os.path.exists(_LIB_PATH)
        or os.path.getmtime(_LIB_PATH) < max(os.path.getmtime(src), os.path.getmtime(hdr))
    )
    if stale:
        subprocess.run(["make", "-C", _HERE, "-B" if force else "-s"], check=True, capture_output=True)
    return _LIB_PATH


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        L = C.CDLL(_LIB_PATH)
        vp, i64, u64, dp, u8p = C.c_void_p, C.c_int64, C.c_uint64, C.POINTER(C.c_double), C.POINTER(C.c_uint8)
        L.orc_create.restype = vp
        L.orc_create.argtypes = [vp, vp, i64, u64]
        L.orc_destroy.argtypes = [vp]
        L.orc_set_start.argtypes = [vp, dp, dp]
        L.orc_df_get_actions.argtypes = [vp, dp]
        L.orc_df_set_actions.argtypes = [vp, C.POINTER(C.c_uint8), dp]
        L.orc_set_wind.argtypes = [vp, vp]
        L.orc_wind_field.argtypes = [vp, i64, dp, dp]
        L.orc_surface_wrench.argtypes = [vp, C.c_int, i64, dp, dp, dp, dp, dp]
        L.orc_solve_contacts.argtypes = [vp, i64, dp, dp, dp, dp, dp, dp, dp, dp, C.c_double, dp, dp, u8p]
        L.orc_contact_flag.argtypes = [vp, i64, dp, dp, dp, u8p]
        L.orc_reset.argtypes = [vp, u8p]
        L.orc_set_mode.argtypes = [vp, C.c_int]
        L.orc_set_setpoints.argtypes = [vp, dp, C.c_int]
        L.orc_get_setpoints.argtypes = [vp, dp, C.c_int]
        L.orc_aviary_step.argtypes = [vp, C.c_int, dp]
        L.orc_get_raw.argtypes = [vp, dp, dp, dp, dp]
        L.orc_set_base_velocity.argtypes = [vp, dp, dp]
        L.orc_update_state.argtypes = [vp]
        L.orc_get_state.argtypes = [vp, dp]
        L.orc_get_aux.argtypes = [vp, dp, C.c_int]
        L.orc_get_pwm.argtypes = [vp, dp]
        L.orc_get_contact.argtypes = [vp, u8p]
        L.orc_env_reset.argtypes = [vp, u8p, dp, dp]
        L.orc_env_reset_targets.argtypes = [vp, u8p, dp, dp, dp]
        L.orc_obs_dim.argtypes = [vp]
        L.orc_env_step.argtypes = [vp, dp, dp, dp, dp, u8p, u8p, u8p]
        L.orc_env_rollout.restype = i64
        L.orc_env_rollout.argtypes = [vp, C.c_int]
        L.orc_set_num_threads.argtypes = [C.c_int]
        _lib = L
    return _lib


def _dp(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))


def _u8(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_uint8))


def surface_wrench(model, si: int, actuation, vb, w):
    """Lifting surface ``si`` of ``model`` on its own, in fp64: actuation[n] (after the lag), base-origin velocity vb[n][3]
    and body rate w[n][3] (base frame, still air) -> force F[n][3] and torque T[n][3] about the base origin, base frame."""
    L = lib()
    act = np.ascontiguousarray(actuation, dtype=np.float64).reshape(-1)
    vb = np.ascontiguousarray(vb, dtype=np.float64).reshape(-1, 3)
    w = np.ascontiguousarray(w, dtype=np.float64).reshape(-1, 3)
    assert len(vb) == len(act) and len(w) == len(act)
    F, T = np.zeros((len(act), 3)), np.zeros((len(act), 3))
    L.orc_surface_wrench(C.byref(model), int(si), len(act), _dp(act), _dp(vb), _dp(w), _dp(F), _dp(T))
    return F, T


def _rows(a, n, width):
    """`a` as n contiguous fp64 rows of `width` values (n values for width 1), a scalar or a single row broadcast"""
    a = np.asarray(a, dtype=np.float64)
    if width == 1:
        return np.ascontiguousarray(np.broadcast_to(a, (n,)))
    return np.ascontiguousarray(np.broadcast_to(a.reshape(-1, width), (n, width)))


def solve_contacts(model, pz, R, v, w, M, c, I_O, top, dt):
    """The floor contact solver of ``model`` on its own, in fp64, for n cases: base altitude pz[n], rotation R[n][3][3] (body
    to world), world velocity v[n][3] and world rate w[n][3], composite mass M[n], COM offset c[n][3] and inertia about the base
    origin I_O[n][3][3] (base frame), surface height top[n], time step dt -> (v, w, touched) after the solve.  Scalars and
    single rows broadcast over the n cases."""
    L = lib()
    pz = np.ascontiguousarray(np.atleast_1d(np.asarray(pz, dtype=np.float64)))
    n = len(pz)
    R, v, w, c, I_O = (_rows(a, n, k) for a, k in ((R, 9), (v, 3), (w, 3), (c, 3), (I_O, 9)))
    M, top = _rows(M, n, 1), _rows(top, n, 1)
    vo, wo, touched = np.zeros((n, 3)), np.zeros((n, 3)), np.zeros(n, dtype=np.uint8)
    L.orc_solve_contacts(C.byref(model), n, _dp(pz), _dp(R), _dp(v), _dp(w), _dp(M), _dp(c), _dp(I_O), _dp(top), float(dt), _dp(vo), _dp(wo), _u8(touched))
    return vo, wo, touched.astype(bool)


def contact_flag(model, pz, R, top):
    """detect_contact_at of ``model`` for n poses: base altitude pz[n], rotation R[n][3][3], surface height top[n] -> bool[n]"""
    pz = np.ascontiguousarray(np.atleast_1d(np.asarray(pz, dtype=np.float64)))
    n = len(pz)
    out = np.zeros(n, dtype=np.uint8)
    lib().orc_contact_flag(C.byref(model), n, _dp(pz), _dp(_rows(R, n, 9)), _dp(_rows(top, n, 1)), _u8(out))
    return out.astype(bool)


class Oracle:
    """N independent single-drone worlds stepped on the CPU in fp64."""

    def __init__(self, model, env_config=None, n: int = 1, seed: int = 0, start_pos=None, start_orn=None):
        L = lib()
        assert L.orc_sizeof_model() == C.sizeof(model), "PfbModel layout mismatch between Python and C"
        if env_config is not None:
            assert L.orc_sizeof_env_config() == C.sizeof(env_config)
        self.model, self.env_config, self.n = model, env_config, int(n)
        self._h = L.orc_create(C.byref(model), C.byref(env_config) if env_config is not None else None, self.n, seed)
        if not self._h:
            raise RuntimeError("orc_create failed (ABI mismatch?)")
        self.updates_per_step = L.orc_updates_per_step(C.c_void_p(self._h))
        sp = np.zeros((self.n, 3)) if start_pos is None else np.ascontiguousarray(np.broadcast_to(start_pos, (self.n, 3)), dtype=np.float64)
        so = np.zeros((self.n, 3)) if start_orn is None else np.ascontiguousarray(np.broadcast_to(start_orn, (self.n, 3)), dtype=np.float64)
        L.orc_set_start(self._h, _dp(sp), _dp(so))
        self.obs_dim = L.orc_obs_dim(C.c_void_p(self._h)) if env_config is not None else 21

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_destroy(self._h)
            self._h = None

    # --- Aviary level
    def reset(self, mask=None):
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        lib().orc_reset(self._h, _u8(m))

    def set_mode(self, mode: int):
        lib().orc_set_mode(self._h, int(mode))

    def set_wind(self, wind):
        """wind: pyflyt_b200.core.wind.AnalyticWind or None"""
        if wind is None:
            lib().orc_set_wind(self._h, None)
        else:
            w = wind.as_struct()
            lib().orc_set_wind(self._h, C.byref(w))

    def wind_field(self, pos):
        """the field set with set_wind at world points pos[m][3] -> [m][3]"""
        p = np.ascontiguousarray(pos, dtype=np.float64).reshape(-1, 3)
        out = np.zeros_like(p)
        lib().orc_wind_field(self._h, len(p), _dp(p), _dp(out))
        return out

    def set_setpoints(self, sp):
        sp = np.ascontiguousarray(sp, dtype=np.float64)
        lib().orc_set_setpoints(self._h, _dp(sp), sp.shape[1])

    def get_setpoints(self, dim=4):
        out = np.zeros((self.n, dim))
        lib().orc_get_setpoints(self._h, _dp(out), dim)
        return out

    def aviary_step(self, n_steps: int = 1, noise=None):
        nz = None
        if noise is not None:
            nz = np.ascontiguousarray(noise, dtype=np.float64)
            assert nz.shape == (n_steps * self.updates_per_step, self.n), nz.shape
        lib().orc_aviary_step(self._h, n_steps, _dp(nz))

    def set_base_velocity(self, lin, ang):
        lin = np.ascontiguousarray(np.broadcast_to(lin, (self.n, 3)), dtype=np.float64)
        ang = np.ascontiguousarray(np.broadcast_to(ang, (self.n, 3)), dtype=np.float64)
        lib().orc_set_base_velocity(self._h, _dp(lin), _dp(ang))

    def update_state(self):
        lib().orc_update_state(self._h)

    def raw(self):
        pos, quat, v, w = np.zeros((self.n, 3)), np.zeros((self.n, 4)), np.zeros((self.n, 3)), np.zeros((self.n, 3))
        lib().orc_get_raw(self._h, _dp(pos), _dp(quat), _dp(v), _dp(w))
        return pos, quat, v, w

    def state(self):
        out = np.zeros((self.n, 12))
        lib().orc_get_state(self._h, _dp(out))
        return out.reshape(self.n, 4, 3)

    def aux_state(self, dim=4):
        out = np.zeros((self.n, dim))
        lib().orc_get_aux(self._h, _dp(out), dim)
        return out

    def pwm(self):
        out = np.zeros((self.n, 4))
        lib().orc_get_pwm(self._h, _dp(out))
        return out

    def contact(self):
        out = np.zeros(self.n, dtype=np.uint8)
        lib().orc_get_contact(self._h, _u8(out))
        return out

    # --- gym env level
    def env_reset(self, mask=None, noise=None, targets=None):
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        nz = None if noise is None else np.ascontiguousarray(noise, dtype=np.float64)
        obs = np.zeros((self.n, self.obs_dim))
        if targets is not None:
            tg = np.ascontiguousarray(targets, dtype=np.float64).reshape(self.n, -1)
            lib().orc_env_reset_targets(self._h, _u8(m), _dp(nz), _dp(tg), _dp(obs))
        else:
            lib().orc_env_reset(self._h, _u8(m), _dp(nz), _dp(obs))
        return obs

    def set_start(self, start_pos, start_orn):
        sp = np.ascontiguousarray(np.broadcast_to(start_pos, (self.n, 3)), dtype=np.float64)
        so = np.ascontiguousarray(np.broadcast_to(start_orn, (self.n, 3)), dtype=np.float64)
        lib().orc_set_start(self._h, _dp(sp), _dp(so))

    def df_get_actions(self):
        """MAFixedwingDogfight and MAQuadXHover: [N][8] past_action | current_action of every agent"""
        out = np.zeros((self.n, 8))
        lib().orc_df_get_actions(self._h, _dp(out))
        return out

    def df_set_actions(self, mask, values):
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        v = np.ascontiguousarray(values, dtype=np.float64).reshape(self.n, 8)
        lib().orc_df_set_actions(self._h, _u8(m), _dp(v))

    def env_step(self, actions, noise=None):
        a = np.ascontiguousarray(actions, dtype=np.float64)
        nz = None if noise is None else np.ascontiguousarray(noise, dtype=np.float64)
        obs = np.zeros((self.n, self.obs_dim))
        rew = np.zeros(self.n)
        term, trunc, info = (np.zeros(self.n, dtype=np.uint8) for _ in range(3))
        lib().orc_env_step(self._h, _dp(a), _dp(nz), _dp(obs), _dp(rew), _u8(term), _u8(trunc), _u8(info))
        return obs, rew, term, trunc, info

    def env_rollout(self, n_steps: int) -> int:
        return int(lib().orc_env_rollout(self._h, int(n_steps)))
