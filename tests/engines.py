"""Test-side adapters giving the CPU oracle, the host-compiled kernel body and the CUDA product one
common surface, so that every golden fixture is replayed through identical code.

* ``OracleEngine``  — oracle/pfb_oracle.c, fp64 (the checker).
* ``HostSimEngine`` — tests/hostsim: the kernel body of pyflyt_b200/csrc compiled with g++ (precision
  studies / logic checks without a GPU; NOT a product path).
* ``CudaEngine``    — the product: pyflyt_b200.BatchedAviary → libpyflyt_b200.so on cuda:0.
"""

from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.realpath(__file__)), "..")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from pyflyt_b200.models import PfbEnvConfig, build_model  # noqa: E402


def euler_zyx_ref(q, lock=None):
    """(roll, pitch, yaw) of the quaternion q = (x, y, z, w) in fp64, as p.getEulerFromQuaternion gives them
    (btQuaternion::getEulerZYX with its +-0.99999 gimbal-lock branch).  ``lock`` True / False forces the gimbal-lock / regular
    branch (a quaternion whose sarg rounds to either side of the snap)."""
    import math

    x, y, z, w = (float(v) for v in q)
    sarg = -2.0 * (x * z - w * y)
    if lock is None:
        lock = abs(sarg) >= 0.99999
    if lock:
        if sarg < 0.0:
            return 0.0, -0.5 * math.pi, 2.0 * math.atan2(x, -y)
        return 0.0, 0.5 * math.pi, 2.0 * math.atan2(-x, y)
    sarg = min(max(sarg, -1.0), 1.0)
    return (math.atan2(2.0 * (y * z + w * x), w * w - x * x - y * y + z * z), math.asin(sarg),
            math.atan2(2.0 * (x * y + w * z), w * w + x * x - y * y - z * z))


def quat_from_euler_ref(roll, pitch, yaw):
    """p.getQuaternionFromEuler (btQuaternion::setEulerZYX) in fp64 -> (x, y, z, w)."""
    import math

    cy, sy, cp, sp = math.cos(yaw / 2), math.sin(yaw / 2), math.cos(pitch / 2), math.sin(pitch / 2)
    cr, sr = math.cos(roll / 2), math.sin(roll / 2)
    return np.array([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy])


def quat_observation_ref(q):
    """The reference's quaternion observation getQuaternionFromEuler(getEulerFromQuaternion(q)) (quadx_base_env.py:243), fp64."""
    return quat_from_euler_ref(*euler_zyx_ref(q))


def sign_rule_quaternions():
    """24 000 unit quaternions [n][4] (x, y, z, w), fp64: 20 000 uniform on the sphere, then 4 000 from Euler angles with large
    roll / yaw and steep pitch (where the observation's w_e < 0) up to near gimbal lock, each with a random sign."""
    rng = np.random.default_rng(3)
    qs = rng.normal(size=(20000, 4))
    eul = np.column_stack([rng.uniform(-np.pi, np.pi, 4000), rng.uniform(-1.5705, 1.5705, 4000), rng.uniform(-np.pi, np.pi, 4000)])
    extra = [quat_from_euler_ref(r, p, y) * rng.choice([-1.0, 1.0]) for r, p, y in eul]
    qs = np.vstack([qs, np.array(extra)])
    return qs / np.linalg.norm(qs, axis=1, keepdims=True)


def hover_config(flight_mode=0, angle_representation="quaternion", sparse=False, dome=3.0, agent_hz=40, max_duration=10.0, autoreset=False):
    e = PfbEnvConfig()
    e.env_kind = 1
    e.flight_mode = int(flight_mode)
    e.env_step_ratio = int(120 / agent_hz)
    e.max_steps = int(agent_hz * max_duration)
    e.angle_representation = 1 if angle_representation == "quaternion" else 0
    e.sparse_reward = int(bool(sparse))
    e.autoreset = int(bool(autoreset))
    e.warmup_steps = 10
    e.flight_dome_size = float(dome)
    return e


class OracleEngine:
    name = "oracle"

    def __init__(self, model, env=None, n=1, start_pos=None, start_orn=None):
        from oracle.oracle import Oracle

        self.o = Oracle(model, env, n=n, start_pos=start_pos, start_orn=start_orn)
        self.n = n
        self.ups = self.o.updates_per_step
        self.aux_dim = {0: 4, 1: 6, 2: 9}[int(model.kind)]

    def reset(self):
        self.o.reset()

    def set_mode(self, mode):
        self.o.set_mode(mode)

    def set_setpoints(self, sp):
        self.o.set_setpoints(sp)

    def get_setpoints(self):
        return self.o.get_setpoints()

    def set_wind(self, wind):
        self.o.set_wind(wind)
        self.o.update_state()  # the fixtures call drone.update_state() after registering the field

    def set_base_velocity(self, lin, ang):
        self.o.set_base_velocity(lin, ang)
        self.o.update_state()  # the fixtures call drone.update_state() after resetBaseVelocity

    def set_start(self, pos, orn):
        self.o.set_start(pos, orn)

    def aviary_step(self, noise, n_steps=1):
        self.o.aviary_step(n_steps, noise)

    def state(self):
        return self.o.state()

    def aux(self, dim=None):
        return self.o.aux_state(dim or self.aux_dim)

    def contact(self):
        return self.o.contact()

    def env_reset(self, noise, targets=None):
        return self.o.env_reset(noise=noise, targets=targets)

    def env_step(self, actions, noise):
        return self.o.env_step(actions, noise)


_HS = None


def hostsim_lib(flags: str = ""):
    """Builds (if stale) and loads tests/_build/libpfb_hostsim<tag>.so; ``flags`` e.g. "-DPFB_V_DOUBLE=0"."""
    global _HS
    tag = "".join(ch for ch in flags if ch.isalnum())
    out = os.path.join(ROOT, "tests", "_build", f"libpfb_hostsim{tag}.so")
    src = os.path.join(ROOT, "tests", "hostsim", "hostsim.cpp")
    deps = [src] + [os.path.join(ROOT, "pyflyt_b200", "csrc", f) for f in ("pfb_common.cuh", "pfb_quadx.cuh", "pfb_quadx_host.h", "pfb_fixedwing.cuh", "pfb_fixedwing_host.h", "pfb_rocket.cuh", "pfb_rocket_host.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        cmd = ["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-mfma", "-ffp-contract=fast"] + flags.split() + ["-o", out, src]
        subprocess.run(cmd, check=True, capture_output=True)
    L = C.CDLL(out)
    L.hs_last_error.restype = C.c_char_p
    return L


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


class HostSimEngine:
    name = "hostsim"

    def __init__(self, model, env=None, n=1, start_pos=None, start_orn=None, flags: str = ""):
        self.L = hostsim_lib(flags)
        self.model, self.env, self.n = model, env, n
        self.ups = int(model.physics_hz / model.control_hz)
        self.fw = int(model.kind) == 1
        self.rk = int(model.kind) == 2
        pre = "hs_rk_" if self.rk else ("hs_fw_" if self.fw else "hs_")
        self.st = np.zeros((getattr(self.L, pre + "state_rows")(), n), dtype=np.float32)
        self.ist = np.zeros((getattr(self.L, pre + "istate_rows")(), n), dtype=np.int32)
        self.sp = np.zeros((n, 7 if self.rk else (6 if self.fw else 4)), dtype=np.float32)
        self.aux_dim = 9 if self.rk else (6 if self.fw else 4)
        self.start_pos = np.ascontiguousarray(np.broadcast_to(np.zeros(3) if start_pos is None else start_pos, (n, 3)), dtype=np.float32)
        self.start_orn = np.ascontiguousarray(np.broadcast_to(np.zeros(3) if start_orn is None else start_orn, (n, 3)), dtype=np.float32)
        self.mode = 0
        self.obs_dim = 21 if (env is not None and env.angle_representation == 1) else 20

    def _chk(self, rc):
        if rc != 0:
            raise RuntimeError(self.L.hs_last_error().decode())

    def reset(self):
        f, i32 = C.c_float, C.c_int32
        if self.fw or self.rk:
            fn = self.L.hs_rk_reset if self.rk else self.L.hs_fw_reset
            self._chk(fn(C.byref(self.model), _p(self.st, f), _p(self.ist, i32), _p(self.sp, f), _p(self.start_pos, f), _p(self.start_orn, f), C.c_int64(self.n)))
            self.mode = 0
            return
        self._chk(self.L.hs_reset(C.byref(self.model), _p(self.st, f), _p(self.ist, i32), _p(self.sp, f), _p(self.start_pos, f), _p(self.start_orn, f), None, C.c_int64(self.n)))
        self.mode = 0

    def set_base_velocity(self, lin, ang):
        lin = np.ascontiguousarray(np.broadcast_to(lin, (self.n, 3)), dtype=np.float32)
        ang = np.ascontiguousarray(np.broadcast_to(ang, (self.n, 3)), dtype=np.float32)
        self._chk(self.L.hs_rk_set_velocity(_p(self.st, C.c_float), _p(self.ist, C.c_int32), _p(lin, C.c_float), _p(ang, C.c_float), C.c_int64(self.n)))

    def set_mode(self, mode):
        if self.rk:
            self.mode = int(mode)
            return
        if self.fw:
            self.sp[...] = 0.0
            self.mode = int(mode)
            return
        self._chk(self.L.hs_set_mode(int(mode), _p(self.st, C.c_float), _p(self.ist, C.c_int32), _p(self.sp, C.c_float), C.c_int64(self.n)))
        self.mode = int(mode)

    def set_setpoints(self, sp):
        sp = np.asarray(sp, dtype=np.float32)
        self.sp[:, : sp.shape[1]] = sp

    def get_setpoints(self):
        return self.sp.astype(np.float64)

    def aviary_step(self, noise, n_steps=1):
        nz = np.ascontiguousarray(noise, dtype=np.float32)
        assert nz.shape == (n_steps * self.ups, self.n)
        if self.rk:
            self._chk(self.L.hs_rk_aviary_step(C.byref(self.model), _p(self.st, C.c_float), _p(self.ist, C.c_int32), _p(self.sp, C.c_float), _p(nz, C.c_float), n_steps, C.c_int64(self.n)))
            return
        if self.fw:
            fn = self.L.hs_fw_aviary_step_full if getattr(self, "full_block", False) else self.L.hs_fw_aviary_step
            self._chk(fn(C.byref(self.model), self.mode, _p(self.st, C.c_float), _p(self.ist, C.c_int32), _p(self.sp, C.c_float), _p(nz, C.c_float), n_steps, C.c_int64(self.n)))
            return
        self._chk(self.L.hs_aviary_step(C.byref(self.model), self.mode, _p(self.st, C.c_float), _p(self.ist, C.c_int32), _p(self.sp, C.c_float), _p(nz, C.c_float), n_steps, C.c_int64(self.n)))

    def _observe(self):
        ds = np.zeros((self.n, 12), dtype=np.float32)
        aux = np.zeros((self.n, self.aux_dim), dtype=np.float32)
        con = np.zeros(self.n, dtype=np.uint8)
        if self.rk:
            self._chk(self.L.hs_rk_observe(_p(self.st, C.c_float), _p(self.ist, C.c_int32), _p(ds, C.c_float), _p(aux, C.c_float), _p(con, C.c_uint8), C.c_int64(self.n)))
            return ds, aux, con
        if self.fw:
            self._chk(self.L.hs_fw_observe(_p(self.st, C.c_float), _p(self.ist, C.c_int32), _p(ds, C.c_float), _p(aux, C.c_float), _p(con, C.c_uint8), C.c_int64(self.n)))
            return ds, aux, con
        self._chk(self.L.hs_observe(_p(self.st, C.c_float), _p(self.ist, C.c_int32), _p(ds, C.c_float), _p(aux, C.c_float), _p(con, C.c_uint8), C.c_int64(self.n)))
        return ds, aux, con

    def state(self):
        return self._observe()[0].reshape(self.n, 4, 3).astype(np.float64)

    def aux(self):
        return self._observe()[1].astype(np.float64)

    def contact(self):
        return self._observe()[2]

    def precise_pos(self):
        """hi + lo position words (the fp64 value the kernel carries)."""
        return (self.st[0:3].astype(np.float64) + self.st[25:28].astype(np.float64)).T  # QX_POS + QX_POS_LO rows

    def env_reset(self, noise, targets=None):
        nz = np.ascontiguousarray(noise, dtype=np.float32)
        obs = np.zeros((self.n, self.obs_dim), dtype=np.float32)
        self._chk(self.L.hs_env_reset(C.byref(self.model), C.byref(self.env), _p(self.st, C.c_float), _p(self.ist, C.c_int32), _p(self.start_pos, C.c_float), _p(self.start_orn, C.c_float), None, _p(nz, C.c_float), _p(obs, C.c_float), C.c_int64(self.n)))
        return obs.astype(np.float64)

    def env_step(self, actions, noise):
        a = np.ascontiguousarray(actions, dtype=np.float32)
        nz = np.ascontiguousarray(noise, dtype=np.float32)
        obs = np.zeros((self.n, self.obs_dim), dtype=np.float32)
        rew = np.zeros(self.n, dtype=np.float32)
        term, trunc, info = (np.zeros(self.n, dtype=np.uint8) for _ in range(3))
        self._chk(self.L.hs_env_step(C.byref(self.model), C.byref(self.env), _p(self.st, C.c_float), _p(self.ist, C.c_int32), _p(a, C.c_float), _p(nz, C.c_float), _p(obs, C.c_float), _p(rew, C.c_float), _p(term, C.c_uint8), _p(trunc, C.c_uint8), _p(info, C.c_uint8), C.c_int64(self.n)))
        return obs.astype(np.float64), rew.astype(np.float64), term, trunc, info


# ----------------------------------------------------------------------------------------------------
# fixture replays (shared by every engine)
# ----------------------------------------------------------------------------------------------------
GOLDEN = os.environ.get("PFB_GOLDEN_DIR", os.path.join(ROOT, "tests", "golden"))


def load_golden(name):
    return np.load(os.path.join(GOLDEN, name if name.endswith(".npz") else name + ".npz"))


def fixture_agent_hz(g):
    """the agent rate a Hover / MAQuadXHover fixture was flown at (fixtures that do not record it: the default, 40 Hz)"""
    return int(g["agent_hz"]) if "agent_hz" in g.files else 40


def fixture_wind(g):
    """the AnalyticWind a fixture was flown in (None = still air)"""
    if "wind_kind" not in g.files:
        return None
    from pyflyt_b200.core.wind import AnalyticWind

    return AnalyticWind(str(g["wind_kind"]), base=g["wind_base"], z_ref=float(g["wind_z_ref"]), alpha=float(g["wind_alpha"]), z0=float(g["wind_z0"]))


def replay_aviary(make_engine, g, every=1):
    """Replays a quadx_aviary fixture; returns dict of max abs errors vs the reference's outputs."""
    model = build_model("quadx", str(g["drone_model"]))
    eng = make_engine(model, None, 1, g["start_pos"][None], g["start_orn"][None])
    eng.reset()
    eng.set_mode(int(g["mode"]))
    if fixture_wind(g) is not None:
        eng.set_wind(fixture_wind(g))
    T = len(g["state"])
    noise = g["noise"].reshape(T, eng.ups)
    err = dict(setpoint=float(np.abs(eng.get_setpoints()[0] - g["setpoint_after_set_mode"]).max()), pos=0.0, euler=0.0, angvel=0.0, linvel=0.0, aux=0.0, contact_mismatch=0)
    pos_err_t = np.zeros(T)
    for i in range(T):
        eng.set_setpoints(g["setpoints"][i][None])
        eng.aviary_step(noise[i][:, None])
        if i % every and i != T - 1:
            continue
        s = eng.state()[0]
        ref = g["state"][i]
        d_eul = np.abs((s[1] - ref[1] + np.pi) % (2 * np.pi) - np.pi)
        err["angvel"] = max(err["angvel"], float(np.abs(s[0] - ref[0]).max()))
        err["euler"] = max(err["euler"], float(d_eul.max()))
        err["linvel"] = max(err["linvel"], float(np.abs(s[2] - ref[2]).max()))
        pe = float(np.abs(s[3] - ref[3]).max())
        pos_err_t[i] = pe
        err["pos"] = max(err["pos"], pe)
        err["aux"] = max(err["aux"], float(np.abs(eng.aux()[0] - g["aux"][i]).max()))
        err["contact_mismatch"] += int(bool(eng.contact()[0]) != bool(g["contact"][i]))
    err["pos_err_t"] = pos_err_t
    return err


def replay_hover(make_engine, g):
    """Replays a quadx_hover fixture (env.reset + scripted env.step + user-loop resets)."""
    model = build_model("quadx", "cf2x")
    env = hover_config(int(g["flight_mode"]), str(g["angle_representation"]), bool(g["sparse"]), float(g["dome"]), fixture_agent_hz(g))
    eng = make_engine(model, env, 1, np.array([[0.0, 0.0, 1.0]]), np.zeros((1, 3)))
    noise, splits = g["noise"], g["noise_splits"]
    cursor = {"i": 0}

    def take():
        k = cursor["i"]
        seg = noise[(splits[k - 1] if k > 0 else 0) : splits[k]]
        cursor["i"] += 1
        return seg

    per_step = env.env_step_ratio * eng.ups
    obs = eng.env_reset(take()[:, None])
    if fixture_wind(g) is not None:  # attached to the env's Aviary after reset()
        eng.set_wind(fixture_wind(g))
    err = dict(obs=float(np.abs(obs[0] - g["reset_obs"]).max()), reward=0.0, flag_mismatch=0, episodes=0)
    ep_starts = set(g["episode_start"].tolist())
    k = 0
    for i in range(len(g["actions"])):
        seg = take()
        full = np.zeros((per_step, 1))
        full[: len(seg), 0] = seg  # an early break consumes fewer draws
        ob, r, te, tr, inf = eng.env_step(g["actions"][i][None], full)
        err["obs"] = max(err["obs"], float(np.abs(ob[0] - g["obs"][i]).max()))
        err["reward"] = max(err["reward"], float(abs(r[0] - g["reward"][i])))
        err["flag_mismatch"] += int(bool(te[0]) != bool(g["term"][i])) + int(bool(tr[0]) != bool(g["trunc"][i])) + int(int(inf[0]) != int(g["info"][i]))
        if (i + 1) in ep_starts:
            ob2 = eng.env_reset(take()[:, None])
            err["obs"] = max(err["obs"], float(np.abs(ob2[0] - g["after_reset_obs"][k]).max()))
            k += 1
            err["episodes"] += 1
    return err


class CudaEngine:
    """The product path: pyflyt_b200.BatchedAviary -> ctypes -> libpyflyt_b200.so on cuda:0."""

    name = "cuda"

    def __init__(self, model_or_name, env=None, n=1, start_pos=None, start_orn=None, drone_model="cf2x", seed=0, drone_type="quadx", drone_options=None):
        import torch

        from pyflyt_b200.core.aviary import BatchedAviary

        self.torch = torch
        self.n = n
        sp = np.ascontiguousarray(np.broadcast_to(np.zeros(3) if start_pos is None else start_pos, (n, 3)), dtype=np.float32)
        so = np.ascontiguousarray(np.broadcast_to(np.zeros(3) if start_orn is None else start_orn, (n, 3)), dtype=np.float32)
        self.av = BatchedAviary(sp, so, drone_type=drone_type, drone_options=dict(drone_model=drone_model, **(drone_options or {})), seed=seed, env_config=env)
        self.aux_dim = self.av.aux_dim
        self.ups = self.av.updates_per_step
        self.obs_dim = self.av.obs_dim

    def _dev(self, a):
        return self.torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32), device=self.av.device)

    def reset(self):
        self.av.reset()

    def set_mode(self, mode):
        self.av.set_mode(mode)

    def set_setpoints(self, sp):
        sp = np.asarray(sp, dtype=np.float32)
        full = np.zeros((self.n, self.av.setpoint_dim), dtype=np.float32)
        full[:, : sp.shape[1]] = sp
        self.av.set_all_setpoints(self._dev(full))

    def get_setpoints(self):
        return self.av.setpoints.double().cpu().numpy()

    def set_wind(self, wind):
        self.av.register_wind_field(wind)

    def set_base_velocity(self, lin, ang):
        lin = self._dev(np.broadcast_to(lin, (self.n, 3)))
        ang = self._dev(np.broadcast_to(ang, (self.n, 3)))
        self.av.set_base_velocity(lin, ang)

    def set_start(self, pos, orn):
        self.av.start_pos.copy_(self._dev(np.broadcast_to(pos, (self.n, 3))))
        self.av.start_orn.copy_(self._dev(np.broadcast_to(orn, (self.n, 3))))

    def aviary_step(self, noise, n_steps=1):
        self.av.step(n_steps, noise=self._dev(noise))

    def state(self):
        return self.av.all_states.double().cpu().numpy()

    def aux(self):
        return self.av.all_aux_states.double().cpu().numpy()

    def contact(self):
        return self.av.contact_array.cpu().numpy().astype(np.uint8)

    def env_reset(self, noise, targets=None):
        tg = None if targets is None else self._dev(np.asarray(targets).reshape(self.n, -1))
        return self.av.env_reset(noise=self._dev(noise), targets=tg).double().cpu().numpy()

    def env_step(self, actions, noise):
        self.av.env_step(actions=self._dev(actions), noise=self._dev(noise))
        a = self.av
        return (a.obs.double().cpu().numpy(), a.reward.double().cpu().numpy(), a.term.cpu().numpy(), a.trunc.cpu().numpy(), a.info_bits.cpu().numpy())


def make_cuda_engine(model, env, n, start_pos, start_orn):
    """Adapter with the (model, env, n, start_pos, start_orn) factory signature used by the replays."""
    if int(model.kind) == 2:
        return CudaEngine(model, env, n, start_pos, start_orn, drone_model="rocket", drone_type="rocket",
                          drone_options=dict(starting_fuel_ratio=float(model.starting_fuel_ratio)))
    if int(model.kind) == 1:
        name = "acrowing" if abs(model.com[0] + 0.39574468) < 1e-5 else "fixedwing"
        return CudaEngine(model, env, n, start_pos, start_orn, drone_model=name, drone_type="fixedwing",
                          drone_options=dict(starting_velocity=list(model.starting_velocity)))
    name = "primitive_drone" if abs(model.mass - 1.0) < 1e-12 else "cf2x"
    return CudaEngine(model, env, n, start_pos, start_orn, drone_model=name)


def model_for_fixture(g):
    import json

    kind = str(g["drone_type"]) if "drone_type" in g.files else "quadx"
    opts = json.loads(str(g["drone_options"])) if "drone_options" in g.files else {}
    return build_model(kind, str(g["drone_model"]), **opts)


def replay_vehicle(make_engine, g, every=1):
    """Replays a fixedwing_aviary / rocket_aviary fixture; max abs errors vs the reference's outputs."""
    model = model_for_fixture(g)
    eng = make_engine(model, None, 1, g["start_pos"][None], g["start_orn"][None])
    eng.reset()
    eng.set_mode(int(g["mode"]))
    if fixture_wind(g) is not None:
        eng.set_wind(fixture_wind(g))
    if "has_pre_hook" in g.files and bool(g["has_pre_hook"]):
        eng.set_base_velocity(g["start_lin_vel"][None], g["start_ang_vel"][None])  # p.resetBaseVelocity + drone.update_state()
    T = len(g["state"])
    noise = g["noise"].reshape(T, -1)
    err = dict(pos=0.0, euler=0.0, angvel=0.0, linvel=0.0, aux=0.0, contact_mismatch=0)
    for i in range(T):
        eng.set_setpoints(g["setpoints"][i][None])
        eng.aviary_step(noise[i][:, None])
        if i % every and i != T - 1:
            continue
        s = eng.state()[0]
        ref = g["state"][i]
        d_eul = np.abs((s[1] - ref[1] + np.pi) % (2 * np.pi) - np.pi)
        err["angvel"] = max(err["angvel"], float(np.abs(s[0] - ref[0]).max()))
        err["euler"] = max(err["euler"], float(d_eul.max()))
        err["linvel"] = max(err["linvel"], float(np.abs(s[2] - ref[2]).max()))
        err["pos"] = max(err["pos"], float(np.abs(s[3] - ref[3]).max()))
        err["aux"] = max(err["aux"], float(np.abs(eng.aux()[0][: len(g["aux"][i])] - g["aux"][i]).max()))
        err["contact_mismatch"] += int(bool(eng.contact()[0]) != bool(g["contact"][i]))
    return err


def waypoints_config(angle_representation="quaternion", sparse=False, num_targets=4, goal_reach_distance=2.0, dome=100.0,
                     agent_hz=30, max_duration=120.0, autoreset=False):
    e = PfbEnvConfig()
    e.env_kind = 3
    e.flight_mode = 0
    e.env_step_ratio = int(120 / agent_hz)
    e.max_steps = int(agent_hz * max_duration)
    e.angle_representation = 1 if angle_representation == "quaternion" else 0
    e.sparse_reward = int(bool(sparse))
    e.autoreset = int(bool(autoreset))
    e.warmup_steps = 10
    e.flight_dome_size = float(dome)
    e.goal_reach_distance = float(goal_reach_distance)
    e.goal_reach_angle = float("inf")
    e.num_targets = int(num_targets)
    e.use_yaw_targets = 0
    return e


def quadx_waypoints_config(g_or_none=None, *, flight_mode=0, angle_representation="quaternion", sparse=False, num_targets=4,
                           use_yaw_targets=False, goal_reach_distance=0.2, goal_reach_angle=0.1, dome=5.0, agent_hz=30,
                           max_duration=10.0, autoreset=False):
    """QuadXWaypointsEnv.__init__ defaults (quadx_waypoints_env.py:38-52)."""
    e = PfbEnvConfig()
    e.env_kind = 2
    e.flight_mode = int(flight_mode)
    e.env_step_ratio = int(120 / agent_hz)
    e.max_steps = int(agent_hz * max_duration)
    e.angle_representation = 1 if angle_representation == "quaternion" else 0
    e.sparse_reward = int(bool(sparse))
    e.autoreset = int(bool(autoreset))
    e.warmup_steps = 10
    e.flight_dome_size = float(dome)
    e.goal_reach_distance = float(goal_reach_distance)
    e.goal_reach_angle = float(goal_reach_angle)
    e.num_targets = int(num_targets)
    e.use_yaw_targets = int(bool(use_yaw_targets))
    return e


def replay_waypoints(make_engine, g):
    """Replays a fixedwing_waypoints / quadx_waypoints fixture: env.reset (targets injected) + scripted env.step +
    user-loop resets."""
    if str(g["kind"]) == "quadx_waypoints":
        model = build_model("quadx", "cf2x")
        env = quadx_waypoints_config(flight_mode=int(g["flight_mode"]), angle_representation=str(g["angle_representation"]), sparse=bool(g["sparse"]),
                                     num_targets=int(g["num_targets"]), use_yaw_targets=bool(g["use_yaw_targets"]),
                                     goal_reach_distance=float(g["goal_reach_distance"]), goal_reach_angle=float(g["goal_reach_angle"]), dome=float(g["dome"]))
        eng = make_engine(model, env, 1, np.array([[0.0, 0.0, 1.0]]), np.zeros((1, 3)))
    else:
        model = build_model("fixedwing", "fixedwing")
        env = waypoints_config(str(g["angle_representation"]), bool(g["sparse"]), int(g["num_targets"]), float(g["goal_reach_distance"]), float(g["dome"]))
        eng = make_engine(model, env, 1, np.array([[0.0, 0.0, 10.0]]), np.zeros((1, 3)))
    noise, splits = g["noise"], g["noise_splits"]
    cursor = {"i": 0}

    def take():
        k = cursor["i"]
        seg = noise[(splits[k - 1] if k > 0 else 0) : splits[k]]
        cursor["i"] += 1
        return seg

    per_step = env.env_step_ratio * eng.ups
    obs = eng.env_reset(take()[:, None], targets=g["targets"][0][None])
    p0 = 10 if str(g["angle_representation"]) == "quaternion" else 9  # lin_pos columns of the attitude block
    err = dict(obs=float(np.abs(obs[0] - g["reset_obs"]).max()), pos=0.0, reward=0.0, flag_mismatch=0, episodes=0)
    ep_starts = set(g["episode_start"].tolist())
    k = 0
    for i in range(len(g["actions"])):
        seg = take()
        full = np.zeros((per_step, 1))
        full[: len(seg), 0] = seg
        ob, r, te, tr, inf = eng.env_step(g["actions"][i][None], full)
        err["obs"] = max(err["obs"], float(np.abs(ob[0] - g["obs"][i]).max()))
        err["pos"] = max(err["pos"], float(np.abs(ob[0][p0 : p0 + 3] - g["obs"][i][p0 : p0 + 3]).max()))
        err["reward"] = max(err["reward"], float(abs(r[0] - g["reward"][i])))
        err["flag_mismatch"] += int(bool(te[0]) != bool(g["term"][i])) + int(bool(tr[0]) != bool(g["trunc"][i])) + int(int(inf[0]) != int(g["info"][i]))
        if (i + 1) in ep_starts:
            k += 1
            ob2 = eng.env_reset(take()[:, None], targets=g["targets"][k][None])
            err["obs"] = max(err["obs"], float(np.abs(ob2[0] - g["after_reset_obs"][k - 1]).max()))
            err["episodes"] += 1
    return err


def landing_config(angle_representation="quaternion", sparse=False, randomize_drop=False, accelerate_drop=False, ceiling=500.0,
                   max_displacement=200.0, agent_hz=40, max_duration=30.0, autoreset=False, contact_response=False):
    e = PfbEnvConfig()
    e.env_kind = 4
    e.flight_mode = 0
    e.env_step_ratio = int(120 / agent_hz)
    e.max_steps = int(agent_hz * max_duration)
    e.angle_representation = 1 if angle_representation == "quaternion" else 0
    e.sparse_reward = int(bool(sparse))
    e.autoreset = int(bool(autoreset))
    e.warmup_steps = 10
    e.ceiling = float(ceiling)
    e.max_displacement = float(max_displacement)
    e.randomize_drop = int(bool(randomize_drop))
    e.accelerate_drop = int(bool(accelerate_drop))
    e.flight_dome_size = float("inf")
    e.contact_response = int(bool(contact_response))
    return e


def replay_landing(make_engine, g, max_steps=None):
    """Replays a rocket_landing fixture: every episode's spawn pose is installed explicitly."""
    model = build_model("rocket", "rocket", starting_fuel_ratio=0.05)  # rocket_landing_env.py:104
    extra = {k: (float(g[k]) if k != "contact_response" else bool(g[k])) for k in ("ceiling", "max_displacement", "contact_response") if k in g.files}
    env = landing_config(str(g["angle_representation"]), bool(g["sparse"]), False, bool(g["accelerate_drop"]), **extra)
    sp = g["spawns"]
    eng = make_engine(model, env, 1, sp[0][None, :3], sp[0][None, 3:])
    noise, splits = g["noise"], g["noise_splits"]
    cursor = {"i": 0}

    def take():
        k = cursor["i"]
        seg = noise[(splits[k - 1] if k > 0 else 0) : splits[k]]
        cursor["i"] += 1
        return seg

    per_step = env.env_step_ratio * eng.ups
    obs = eng.env_reset(take()[:, None])
    if fixture_wind(g) is not None:  # attached to the env's Aviary after reset()
        eng.set_wind(fixture_wind(g))
    err = dict(obs=float(np.abs(obs[0] - g["reset_obs"]).max()), reward=0.0, flag_mismatch=0, episodes=0)
    ep_starts = set(g["episode_start"].tolist())
    k = 0
    T = len(g["actions"]) if max_steps is None else min(max_steps, len(g["actions"]))
    for i in range(T):
        seg = take()
        full = np.zeros((per_step, 1))
        full[: len(seg), 0] = seg
        ob, r, te, tr, inf = eng.env_step(g["actions"][i][None], full)
        err["obs"] = max(err["obs"], float(np.abs(ob[0] - g["obs"][i]).max()))
        err["reward"] = max(err["reward"], float(abs(r[0] - g["reward"][i])))
        err["flag_mismatch"] += int(bool(te[0]) != bool(g["term"][i])) + int(bool(tr[0]) != bool(g["trunc"][i])) + int(int(inf[0]) != int(g["info"][i]))
        if (i + 1) in ep_starts:
            k += 1
            eng.set_start(sp[k][None, :3], sp[k][None, 3:])
            ob2 = eng.env_reset(take()[:, None])
            err["obs"] = max(err["obs"], float(np.abs(ob2[0] - g["after_reset_obs"][k - 1]).max()))
            err["episodes"] += 1
    return err


def dogfight_config(team_size=1, sparse=False, lethal_distance=20.0, lethal_angle=0.07, damage_per_hit=0.003, aggressiveness=0.5,
                    cooperativeness=0.5, dome=800.0, agent_hz=30, max_duration=60.0, autoreset=False,
                    spawn_min_radius=10.0, spawn_max_radius=50.0, spawn_min_height=20.0, spawn_max_height=50.0):
    e = PfbEnvConfig()
    e.env_kind = 5
    e.flight_mode = 0
    e.env_step_ratio = int(120 / agent_hz)
    e.max_steps = int(agent_hz * max_duration)
    e.angle_representation = 0
    e.sparse_reward = int(bool(sparse))
    e.autoreset = int(bool(autoreset))
    e.warmup_steps = 10
    e.flight_dome_size = float(dome)
    e.team_size = int(team_size)
    e.damage_per_hit, e.lethal_distance, e.lethal_angle = float(damage_per_hit), float(lethal_distance), float(lethal_angle)
    e.aggressiveness, e.cooperativeness = float(aggressiveness), float(cooperativeness)
    e.spawn_min_radius, e.spawn_max_radius = float(spawn_min_radius), float(spawn_max_radius)
    e.spawn_min_height, e.spawn_max_height = float(spawn_min_height), float(spawn_max_height)
    return e


def replay_dogfight(make_engine, g):
    """Replays a dogfight fixture arena by arena: spawn poses and noise injected, dead agents keep flying."""
    ts = int(g["team_size"])
    A = 2 * ts
    model = build_model("fixedwing", "acrowing")  # ma_fixedwing_base_env.py:192-195
    env = dogfight_config(ts, bool(g["sparse"]), float(g["lethal_distance"]), float(g["lethal_angle"]), float(g["damage_per_hit"]) if "damage_per_hit" in g.files else 0.003)
    err = dict(obs=0.0, reward=0.0, flag_mismatch=0, episodes=int(g["n_episodes"]))
    eng = None
    for k in range(int(g["n_episodes"])):
        spawn = g[f"ep{k}_spawn"]
        if eng is None:
            eng = make_engine(model, env, A, spawn[:, :3], spawn[:, 3:])
        else:
            eng.set_start(spawn[:, :3], spawn[:, 3:])
        per_sub = A
        rn = g[f"ep{k}_reset_noise"].reshape(-1, per_sub)
        obs = eng.env_reset(rn)
        err["obs"] = max(err["obs"], float(np.abs(obs - g[f"ep{k}_reset_obs"]).max()))
        T = len(g[f"ep{k}_actions"])
        for i in range(T):
            nz = g[f"ep{k}_noise"][i].reshape(-1, per_sub)
            ob, r, te, tr, _ = eng.env_step(g[f"ep{k}_actions"][i], nz)
            alive = g[f"ep{k}_alive"][i]
            ref_o, ref_r = g[f"ep{k}_obs"][i], g[f"ep{k}_reward"][i]
            err["obs"] = max(err["obs"], float(np.abs(ob[alive] - ref_o[alive]).max()))
            err["reward"] = max(err["reward"], float(np.abs(r[alive] - ref_r[alive]).max()))
            err["flag_mismatch"] += int((te[alive].astype(bool) != g[f"ep{k}_term"][i][alive]).sum()) + int((tr[alive].astype(bool) != g[f"ep{k}_trunc"][i][alive]).sum())
    return err


def ma_hover_config(flight_mode=0, angle_representation="quaternion", sparse=False, dome=10.0, agent_hz=40, max_duration=30.0):
    """MAQuadXHoverEnv.__init__ defaults (ma_quadx_hover_env.py:37-60); per-agent env kind 6 (no in-kernel autoreset: the
    arena bookkeeping is host-side)."""
    e = PfbEnvConfig()
    e.env_kind = 6
    e.flight_mode = int(flight_mode)
    e.env_step_ratio = int(120 / agent_hz)
    e.max_steps = int(agent_hz * max_duration)
    e.angle_representation = 1 if angle_representation == "quaternion" else 0
    e.sparse_reward = int(bool(sparse))
    e.autoreset = 0
    e.warmup_steps = 10
    e.flight_dome_size = float(dome)
    return e


def replay_ma_hover(make_engine, g):
    """Replays a ma_quadx_hover fixture: one engine env per agent, noise injected; the agents the reference has culled
    are stepped with a zero action (their outputs are not compared)."""
    A = int(g["n_agents"])
    model = build_model("quadx", "cf2x")
    env = ma_hover_config(int(g["flight_mode"]), str(g["angle_representation"]), bool(g["sparse"]), float(g["dome"]), fixture_agent_hz(g),
                         float(g["max_duration_seconds"]))
    eng = make_engine(model, env, A, g["start_pos"], g["start_orn"])
    err = dict(obs=0.0, pos=0.0, reward=0.0, flag_mismatch=0, episodes=int(g["n_episodes"]))
    p0 = 10 if str(g["angle_representation"]) == "quaternion" else 9
    for k in range(int(g["n_episodes"])):
        obs = eng.env_reset(g[f"ep{k}_reset_noise"].reshape(-1, A))
        err["obs"] = max(err["obs"], float(np.abs(obs - g[f"ep{k}_reset_obs"]).max()))
        for i in range(len(g[f"ep{k}_actions"])):
            alive = g[f"ep{k}_alive"][i]
            act = g[f"ep{k}_actions"][i] * alive[:, None]  # current_actions *= 0 for the agents not in self.agents
            ob, r, te, tr, _ = eng.env_step(act, g[f"ep{k}_noise"][i].reshape(-1, A))
            ref_o, ref_r = g[f"ep{k}_obs"][i], g[f"ep{k}_reward"][i]
            err["obs"] = max(err["obs"], float(np.abs(ob[alive] - ref_o[alive]).max()))
            err["pos"] = max(err["pos"], float(np.abs(ob[alive][:, p0 : p0 + 3] - ref_o[alive][:, p0 : p0 + 3]).max()))
            err["reward"] = max(err["reward"], float(np.abs(r[alive] - ref_r[alive]).max()))
            err["flag_mismatch"] += int((te[alive].astype(bool) != g[f"ep{k}_term"][i][alive]).sum()) + int((tr[alive].astype(bool) != g[f"ep{k}_trunc"][i][alive]).sum())
    return err
