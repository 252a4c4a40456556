"""``BatchedAviary`` — N independent single-drone worlds stepped in lock-step on one GPU.

Mirrors the surface of the reference's ``Aviary`` that its environments use
(/root/reference/PyFlyt/core/aviary.py): ctor kwargs ``start_pos``/``start_orn``/``drone_type``/
``drone_options``/``seed``/``physics_hz`` (:69-83), ``reset`` (:218), ``step`` (:480), ``state(i)`` (:335),
``aux_state(i)`` (:353), ``all_states`` (:372), ``set_mode`` (:440), ``set_setpoint`` (:460),
``set_all_setpoints`` (:470), ``contact_array`` (:322), counters (:227-229, :528-531), and the Bullet client's base-state
calls that scripts on top of the Aviary use: ``resetBasePositionAndOrientation`` / ``resetBaseVelocity`` followed by
``drone.update_state()`` (``set_base_state``, ``set_base_velocity``) and ``getBasePositionAndOrientation`` /
``getBaseVelocity`` (``base_state``), by drone index and mask rather than body id — with one difference in meaning: drone
``i`` lives in its OWN world (the reference puts them in one Bullet world), so ``contact_array[i]`` is "drone i touched the
floor during the last step".

``drone_options`` may be a sequence with one dict per drone, as in the reference (aviary.py:75): a QuadX batch then flies up
to ``MAX_QUADX_MODELS`` different vehicle tables (``models``), drone ``i`` the table ``model_index[i]``.  All of them run at
the same ``control_hz`` unless ``mixed_control_hz=True`` (below).  Drones ``32 k .. 32 k + 31`` share one warp: a batch runs
fastest when each such tile flies one model (DESIGN.md §4a).

The floor: the reference's Aviary is a PyBullet world, so a drone that reaches the floor stands on it.  Here, by default, the
floor only raises ``contact_array`` and a drone keeps falling through ``z = 0`` (the envs end an episode on the first
contact, so they never need more).  ``contact_response=True`` makes the floor push back on QuadX, fixed-wing and rocket
drones: contact impulses with Coulomb friction on the corners / rim points of each drone's collision primitives, so drones
take off from, land on, slide along and rest on the floor (DESIGN.md §4c).

``drone_type`` may be a list with one kind per drone, as in the reference (aviary.py:139-190, examples/core/08_mixed_drones.py):
a batch then flies QuadX, fixed-wing and rocket drones together, all stepped by one CUDA launch (DESIGN.md §4d).  Every drone
keeps its own kind's surface: ``set_setpoint(i, sp)`` takes drone ``i``'s own setpoint length (QuadX 4, fixed-wing 4 or 6,
rocket 7) and ``state(i)`` / ``aux_state(i)`` return its own aux length (4, 6 or 9); ``setpoints`` is ``[N, 7]`` and
``all_aux_states`` a list of ``N`` tensors.  Each kind's drones take their tables from their own ``drone_options`` entries (up
to ``MAX_QUADX_MODELS`` QuadX models, one fixed-wing and one rocket model), and every drone runs at one ``control_hz`` unless
``mixed_control_hz=True`` (below).  Such a batch is an Aviary only: no ``env_config``, no ``state_row``.  Drone ``i`` draws the random stream drone ``i`` of a single-kind batch with the same seed draws, so it flies
exactly as it would there.

``mixed_control_hz=True`` lets the drones' ``drone_options`` differ in ``control_hz``, as in the reference's
examples/core/02_multi_drone.py (three QuadX at 60, 120 and 240 Hz): the rates must form common multiples (the reference's
``AssertionError`` otherwise), ``updates_per_step`` and ``step_period`` follow the slowest rate (at most 4 physics steps per
Aviary step), and drone ``i`` runs its controller on the physics steps that are multiples of ``physics_hz / control_hz[i]``.
Such a batch is a mixed handle whatever its kinds, with the surface described above (``setpoints`` ``[N, 7]``); a batch whose
rates turn out equal is the batch built without the option (DESIGN.md §4e).

Static bodies: ``loadURDF(fileName, basePosition, baseOrientation, useFixedBase=True)`` (then ``register_all_new_bodies()``, kept
for script compatibility) puts a landing pad, a helipad or a rooftop into every drone's world, as the reference's
``aviary.loadURDF`` does; ``set_static_pose`` moves a body in the worlds of a mask of drones, and ``contact_bodies()`` says
which body each drone touched.  Up to ``MAX_STATIC_BODIES`` bodies of ``MAX_STATIC_SHAPES`` boxes and cylinders in all,
upright; only their top faces are solid (DESIGN.md §4h).  ``reset()`` removes them, as the reference's ``resetSimulation`` does.

All state is held in caller-visible ``torch`` tensors; the CUDA library (libpyflyt_b200.so) only sees
raw device pointers.  There is no CPU path.
"""

from __future__ import annotations

import ctypes as C
import os
from typing import Any, Sequence

import numpy as np
import torch

from .. import _lib
from ..models import ModelSetError, PfbEnvConfig, PfbModel, PfbShape, build_mixed_model_set, build_model, build_model_set

_KINDS = ("quadx", "fixedwing", "rocket")
_MODE_RANGE = {"quadx": (-1, 7), "fixedwing": (-1, 0), "rocket": (0, 0)}  # quadx.py:259-262, fixedwing.py:216-219, base_drone.py:252-255
_SETPOINT_LEN = {"quadx": (4,), "fixedwing": (4, 6), "rocket": (7,)}
_AUX_LEN = {"quadx": 4, "fixedwing": 6, "rocket": 9}
MAX_STATIC_BODIES = 8  # PFB_MAX_STATIC_BODIES
MAX_STATIC_SHAPES = 16  # PFB_MAX_STATIC_SHAPES


def _upright_error(quat: np.ndarray) -> float:
    """Largest 1 - R22 over unit quaternions (x, y, z, w): 0 for a pure yaw."""
    q = np.asarray(quat, dtype=np.float64).reshape(-1, 4)
    n = np.sum(q * q, axis=1)
    return float(np.max(2.0 * (q[:, 0] ** 2 + q[:, 1] ** 2) / n)) if len(q) else 0.0


def _check_mode(kind: str, mode: int) -> None:
    lo, hi = _MODE_RANGE[kind]
    if mode < lo or mode > hi:
        # quadx.py:259-262, fixedwing.py:216-219, base_drone.py:252-255
        raise ValueError(f"`mode` must be between {lo} and {hi} or be registered in self.registered_controllers.keys()=dict_keys([]), got {mode}.")


class AviaryInitException(Exception):
    """Same role as PyFlyt.core.aviary.AviaryInitException (aviary.py:21-44)."""

    def __init__(self, message: str = "AviaryInitException"):
        self.message = message
        super().__init__(self.message)

    def __str__(self) -> str:
        return f"Aviary Error: {self.message}"


def _stream_ptr(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


class BatchedAviary:
    def __init__(
        self,
        start_pos,
        start_orn,
        drone_type: str = "quadx",
        drone_options: dict[str, Any] | Sequence[dict[str, Any]] | None = None,
        physics_hz: int = 240,
        seed: None | int = None,
        device: str | torch.device = "cuda:0",
        env_config: PfbEnvConfig | None = None,
        env_offset: int = 0,
        contact_response: bool = False,
        mixed_control_hz: bool = False,
    ):
        """``contact_response``: the floor pushes back (contact impulses + Coulomb friction) instead of only raising
        ``contact_array``.  The reference always responds, since every ``Aviary`` is a PyBullet world; here it is opt-in so
        that a handle built without it steps exactly as before, and so that flight far above the floor never pays for the
        solver.  Aviary handles only: an env handle (``env_config``) has its own contact policy.

        ``mixed_control_hz``: the drones' ``drone_options`` may differ in ``control_hz``, as in the reference's
        tests/test_core.py::test_multi_spawn (DESIGN.md §4e).  An Aviary step is then ``physics_hz / min(control_hz)`` physics
        steps, and each drone runs its controller every ``physics_hz / control_hz`` of them.  Opt-in so that a batch built
        without it keeps refusing different rates.  Aviary handles only: an env flies one drone at one rate."""
        start_pos = np.asarray(start_pos, dtype=np.float32)
        start_orn = np.asarray(start_orn, dtype=np.float32)
        # shape checks with the reference's messages (aviary.py:120-131)
        if start_pos.ndim != 2 or start_pos.shape[-1] != 3:
            raise AviaryInitException(f"start_pos must be shape (n, 3), currently {start_pos.shape}.")
        if start_orn.shape != start_pos.shape:
            raise AviaryInitException(f"start_orn must be same shape as start_pos, currently {start_orn.shape}.")
        if mixed_control_hz and env_config is not None:
            raise AviaryInitException("mixed_control_hz is an Aviary-handle option; an env handle (env_config) flies one drone at one control_hz.")
        kinds = None  # one vehicle kind per drone (a list that holds more than one kind), else None
        if isinstance(drone_type, (tuple, list)):
            if len(set(drone_type)) != 1:
                # the reference's checks and messages (aviary.py:140-148, 178-186)
                if len(drone_type) != start_pos.shape[0]:
                    raise AviaryInitException(
                        f"If multiple `drone_types` are used, must have same number of `drone_types` ({len(drone_type)}) as number of drones ({start_pos.shape[0]})."
                    )
                if not all(dt in _KINDS for dt in drone_type):
                    raise AviaryInitException(f"One of types in `drone_type` {drone_type} is not amongst known types {dict.fromkeys(_KINDS).keys()}.")
                if env_config is not None:
                    raise AviaryInitException("a batch of several vehicle kinds is an Aviary only; an env handle (env_config) flies one kind.")
                kinds = [str(k) for k in drone_type]
            else:
                drone_type = drone_type[0]
        if kinds is None and drone_type not in ("quadx", "fixedwing", "rocket"):
            raise AviaryInitException(f"Can't find `drone_type` {drone_type} amongst known types ['quadx', 'fixedwing', 'rocket'].")
        # one options dict per drone (aviary.py:75, 196-199): the distinct vehicle tables + the model index of every drone
        models, index = None, None
        if kinds is not None:
            try:
                models, index = build_mixed_model_set(kinds, drone_options, physics_hz, int(start_pos.shape[0]), mixed_control_hz)
            except ModelSetError as e:
                raise AviaryInitException(str(e)) from None
        elif drone_options is not None and not isinstance(drone_options, dict):
            try:
                models, index = build_model_set(drone_type, drone_options, physics_hz, int(start_pos.shape[0]), mixed_control_hz)
            except ModelSetError as e:
                raise AviaryInitException(str(e)) from None
        # different control rates: a mixed handle, whether the batch flies one kind or several
        multi_rate = models is not None and len({float(m.control_hz) for m in models}) > 1
        if multi_rate and kinds is None:
            kinds = [str(drone_type)] * int(start_pos.shape[0])
        if not torch.cuda.is_available():
            raise _lib.PfbError("pyflyt_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback.")
        self.device = torch.device(device)
        self.num_drones = int(start_pos.shape[0])
        self.drone_type = drone_type if kinds is None else kinds
        self.kinds = kinds
        self.physics_hz = int(physics_hz)
        self.physics_period = 1.0 / physics_hz
        if models is None:
            opts = dict(drone_options or {})
            control_hz = int(opts.pop("control_hz", 120))
            self.model = build_model(drone_type, opts.pop("drone_model", None), opts.pop("model_dir", None), physics_hz, control_hz, **opts)
            self.models = [self.model]
        else:
            control_hz = int(min(m.control_hz for m in models))  # the slowest drone sets the Aviary step (aviary.py:288-289)
            self.model = models[0]
            self.models = models
        # [N] control rate of every drone
        self.control_hz = np.full(self.num_drones, control_hz, dtype=np.int64) if index is None else np.array([int(models[k].control_hz) for k in index], dtype=np.int64)
        if contact_response:
            if env_config is not None:
                raise AviaryInitException("contact_response is an Aviary-handle option; an env handle (env_config) keeps its own contact policy.")
            env_config = PfbEnvConfig()  # env kind NONE: pfb_create reads only contact_response from it
            env_config.contact_response = 1
        if multi_rate:
            if env_config is None:
                env_config = PfbEnvConfig()  # env kind NONE: pfb_create_mixed reads contact_response and mixed_control_hz
            env_config.mixed_control_hz = 1
        self.contact_response = bool(contact_response)
        self.mixed_control_hz = bool(mixed_control_hz)
        self.env_config = env_config
        self.updates_per_step = int(physics_hz / control_hz)  # aviary.py:288-289
        self.step_period = 1.0 / control_hz
        self.seed = 0 if seed is None else int(seed)

        L = _lib.lib()
        self._h = C.c_void_p()
        dev_index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        if kinds is not None:  # drone i flies models[index[i]], each kind in its own region of the state buffer
            tables = (PfbModel * len(models))(*models)
            idx = np.ascontiguousarray(index, dtype=np.uint8)
            _lib.check(L.pfb_create_mixed(tables, len(models), idx.ctypes.data_as(C.c_void_p), self.num_drones,
                                          C.byref(env_config) if env_config is not None else None, dev_index, self.seed, C.byref(self._h)))
        else:
            _lib.check(L.pfb_create(C.byref(self.model), C.byref(env_config) if env_config is not None else None, self.num_drones, dev_index, self.seed, C.byref(self._h)))
        _lib.check(L.pfb_set_env_offset(self._h, int(env_offset)))
        n, dev = self.num_drones, self.device
        if kinds is None and len(self.models) > 1:  # drone i flies self.models[model_index[i]]; one table keeps the handle as pfb_create made it
            tables = (PfbModel * len(models))(*models)
            idx = np.ascontiguousarray(index, dtype=np.uint8)
            _lib.check(L.pfb_set_models(self._h, tables, len(models), idx.ctypes.data_as(C.c_void_p)))
        self.model_index = torch.as_tensor(np.zeros(n, dtype=np.uint8) if index is None else index, dtype=torch.uint8, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)
        self.obs_dim = L.pfb_obs_dim(self._h)
        self.setpoint_dim = L.pfb_setpoint_dim(self._h)
        self.aux_dim = L.pfb_aux_dim(self._h)
        # persistent state: fp32 SoA, field-major [F][N] or warp-tiled [N/32][F/4][32][4] (include/pyflyt_b200.h)
        self.state_rows = int(L.pfb_state_rows(self._h))
        self.tiled = int(L.pfb_state_layout(self._h)) == 1
        if kinds is not None:  # one flat buffer; the library carves it into one region per kind, each in that kind's layout
            self.state_tensor = torch.zeros((int(L.pfb_state_floats(self._h)),), **f32)
            self._setpoint_len = [_SETPOINT_LEN[k] for k in kinds]
            self._aux_len = [_AUX_LEN[k] for k in kinds]
        elif self.tiled:
            self.state_tensor = torch.zeros((int(L.pfb_state_floats(self._h)) // (self.state_rows * 32), self.state_rows // 4, 32, 4), **f32)
        else:
            self.state_tensor = torch.zeros((self.state_rows, n), **f32)
        self.istate_tensor = torch.zeros((L.pfb_istate_rows(self._h), n), dtype=torch.int32, device=dev)
        self.setpoints = torch.zeros((n, self.setpoint_dim), **f32)
        self.start_pos = torch.from_numpy(start_pos).to(dev).contiguous()
        self.start_orn = torch.from_numpy(start_orn).to(dev).contiguous()
        # obs | reward | term | trunc live in ONE slab: pfb_env_step_host then returns them with a single D2H copy
        self._out_slab = torch.zeros(self.out_slab_bytes(n, self.obs_dim), dtype=torch.uint8, device=dev)
        self.obs, self.reward, self.term, self.trunc = self.slab_views(self._out_slab, n, self.obs_dim)
        self.info_bits = torch.zeros((n,), dtype=torch.uint8, device=dev)
        self.final_obs = torch.zeros((n, self.obs_dim), **f32)
        self._drone_state = torch.zeros((n, 12), **f32)
        self._aux_state = torch.zeros((n, self.aux_dim), **f32)
        self._contact = torch.zeros((n,), dtype=torch.uint8, device=dev)
        b = _lib.PfbBuffers()
        b.state, b.istate = self.state_tensor.data_ptr(), self.istate_tensor.data_ptr()
        b.setpoint, b.start_pos, b.start_orn = self.setpoints.data_ptr(), self.start_pos.data_ptr(), self.start_orn.data_ptr()
        b.obs, b.reward, b.term, b.trunc = self.obs.data_ptr(), self.reward.data_ptr(), self.term.data_ptr(), self.trunc.data_ptr()
        b.info, b.final_obs = self.info_bits.data_ptr(), self.final_obs.data_ptr()
        b.drone_state, b.aux_state, b.contact = self._drone_state.data_ptr(), self._aux_state.data_ptr(), self._contact.data_ptr()
        b.reset_targets = None
        self._reset_targets = None
        self._buffers = b
        _lib.check(L.pfb_bind(self._h, C.byref(b)))
        self._state_fresh = False
        self.static_bodies: list[str] = []  # the URDF of each static body (loadURDF), by body index
        self.reset()

    # ------------------------------------------------------------------ lifecycle
    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                _lib.lib().pfb_destroy(h)
            except Exception:
                pass
            self._h = None

    def disconnect(self) -> None:
        self.__del__()

    def _s(self):
        return C.c_void_p(_stream_ptr(self.device))

    # ------------------------------------------------------------------ Aviary surface
    def reset(self) -> None:
        """aviary.py:218-312: every drone back to its start pose, mode 0, zero setpoint."""
        _lib.check(_lib.lib().pfb_reset(self._h, None, self._s()))
        self.static_bodies = []  # pfb_reset removed them (resetSimulation)
        self.physics_steps = 0
        self.aviary_steps = 0
        self.elapsed_time = 0.0
        self._state_fresh = False

    def set_mode(self, flight_modes: int | Sequence[int]) -> None:
        """aviary.py:440-458: one mode for every drone, or a list / tuple with one mode per drone.

        A list whose entries differ flies each drone in its own mode until the next ``set_mode(int)`` or ``reset()`` (Aviary
        handles only; an env flies its ``flight_mode``).  Drones ``32 k .. 32 k + 31`` share one warp: a batch steps fastest
        when each such tile flies one mode (DESIGN.md §4b).

        Every drone's mode is checked against its own kind's range first, and the first invalid one raises its kind's
        ``ValueError`` with nothing changed.  (On a batch of several kinds the reference's loop, aviary.py:454-458, would already
        have set the mode of the drones before that one.)"""
        kinds = self.kinds if self.kinds is not None else [self.drone_type] * self.num_drones
        if isinstance(flight_modes, (list, tuple)):
            if len(flight_modes) != self.num_drones:
                raise AssertionError(f"Expected {self.num_drones} flight_modes, got {len(flight_modes)}.")
            modes = [int(m) for m in flight_modes]
            for kind, m in zip(kinds, modes):  # every drone's set_mode checks its own mode (aviary.py:455-456)
                _check_mode(kind, m)
            # one mode on a single-kind batch: the uniform kernels; a batch of several kinds keeps one mode per drone
            if self.kinds is not None or len(set(modes)) != 1:
                arr = np.ascontiguousarray(modes, dtype=np.int8)
                _lib.check(_lib.lib().pfb_set_modes(self._h, arr.ctypes.data_as(C.c_void_p), self._s()))
                self._state_fresh = False
                return
            flight_modes = modes[0]
        mode = int(flight_modes)
        for kind in dict.fromkeys(kinds):  # the kinds in drone order: the first drone that refuses raises
            _check_mode(kind, mode)
        _lib.check(_lib.lib().pfb_set_mode(self._h, mode, self._s()))
        self._state_fresh = False

    def _setpoint_row(self, index: int, setpoint) -> torch.Tensor:
        """Drone ``index``'s setpoint of its own length, zero-padded to the 7 columns of a batch of several kinds."""
        sp = torch.as_tensor(setpoint, dtype=torch.float32).reshape(-1)
        allowed = self._setpoint_len[index]
        if sp.numel() not in allowed:
            raise ValueError(f"drone {index} is a {self.kinds[index]}: its setpoint has length {' or '.join(map(str, allowed))}, got {sp.numel()}.")
        row = torch.zeros(self.setpoint_dim, dtype=torch.float32)
        row[: sp.numel()] = sp
        return row

    def set_setpoint(self, index: int, setpoint) -> None:
        if self.kinds is not None:
            self.setpoints[index] = self._setpoint_row(index, setpoint).to(self.device)
            return
        self.setpoints[index] = torch.as_tensor(setpoint, dtype=torch.float32, device=self.device)

    def set_all_setpoints(self, setpoints) -> None:
        """A batch of several kinds takes a padded ``[N, 7]`` array or a sequence of ``N`` per-drone setpoints (aviary.py:477-478
        indexes ``setpoints[i]``)."""
        if self.kinds is not None and not (hasattr(setpoints, "shape") and tuple(setpoints.shape) == (self.num_drones, self.setpoint_dim)):
            if len(setpoints) != self.num_drones:
                raise ValueError(f"Expected {self.num_drones} setpoints, got {len(setpoints)}.")
            setpoints = torch.stack([self._setpoint_row(i, sp) for i, sp in enumerate(setpoints)])
        self.setpoints.copy_(torch.as_tensor(setpoints, dtype=torch.float32, device=self.device))

    def step(self, n_steps: int = 1, noise: torch.Tensor | None = None) -> None:
        """``n_steps`` x Aviary.step() (aviary.py:480-531).  ``noise``: optional device tensor
        [n_steps*updates_per_step, N] of raw ``np_random.normal`` draws (parity tests)."""
        ptr = None
        if noise is not None:
            assert noise.dtype == torch.float32 and noise.is_cuda and noise.is_contiguous()
            assert tuple(noise.shape) == (n_steps * self.updates_per_step, self.num_drones), tuple(noise.shape)
            ptr = C.c_void_p(noise.data_ptr())
        _lib.check(_lib.lib().pfb_aviary_step(self._h, int(n_steps), ptr, self._s()))
        self.physics_steps += n_steps * self.updates_per_step
        self.aviary_steps += n_steps
        self.elapsed_time = self.physics_steps / self.physics_hz
        self._state_fresh = False

    def set_base_velocity(self, lin_vel: torch.Tensor, ang_vel: torch.Tensor) -> None:
        """``p.resetBaseVelocity`` for every drone (used by rocket_base_env.py:228): [N, 3] world-frame velocities, taken in
        fp32.  The state then carries the body rate R^T w, computed in fp32.  Like the env scripts that call it, it does not
        zero anything else; ``set_base_state`` is the fp64, masked form."""
        lin = torch.as_tensor(lin_vel, dtype=torch.float32, device=self.device).reshape(self.num_drones, 3).contiguous()
        ang = torch.as_tensor(ang_vel, dtype=torch.float32, device=self.device).reshape(self.num_drones, 3).contiguous()
        _lib.check(_lib.lib().pfb_set_base_velocity(self._h, C.c_void_p(lin.data_ptr()), C.c_void_p(ang.data_ptr()), self._s()))
        self._state_fresh = False

    def _rows64(self, x, width: int, name: str) -> torch.Tensor | None:
        if x is None:
            return None
        t = torch.as_tensor(x, dtype=torch.float64, device=self.device)
        if tuple(t.shape) != (self.num_drones, width):
            raise ValueError(f"{name} must be shape ({self.num_drones}, {width}), got {tuple(t.shape)}.")
        return t.contiguous()

    def set_base_state(self, pos=None, quat=None, lin_vel=None, ang_vel=None, mask=None) -> None:
        """``p.resetBasePositionAndOrientation(id, pos, quat)`` and / or ``p.resetBaseVelocity(id, lin_vel, ang_vel)``, then
        ``drone.update_state()``, for the drones of ``mask`` ([N] bool; None = every drone).  ``pos`` [N, 3], ``quat`` [N, 4]
        (x, y, z, w, PyBullet's order; unit norm to 1e-6), ``lin_vel`` / ``ang_vel`` [N, 3] in the world frame, numpy or
        torch, taken in fp64; None = not given.  ``pos`` and ``quat`` come together.  A pose zeroes both velocities, as
        Bullet's reset does, and the velocities given then replace them; what is not given keeps its value.  Flight modes,
        setpoints, controller memories, motor throttles, surfaces, fuel, gimbal, model index, step count and the contact flags
        are kept (DESIGN.md §4g).  Aviary handles only."""
        if (pos is None) != (quat is None):
            raise ValueError("pos and quat come together (resetBasePositionAndOrientation sets both) or not at all.")
        p, q = self._rows64(pos, 3, "pos"), self._rows64(quat, 4, "quat")
        lv, av = self._rows64(lin_vel, 3, "lin_vel"), self._rows64(ang_vel, 3, "ang_vel")
        if q is not None:
            err = float((torch.linalg.vector_norm(q, dim=1) - 1.0).abs().max())
            if not err <= 1e-6:
                raise ValueError(f"quat must be unit quaternions (x, y, z, w): a norm differs from 1 by {err:.3g} (> 1e-6).")
        m = None
        if mask is not None:
            m = torch.as_tensor(mask, device=self.device)
            if tuple(m.shape) != (self.num_drones,):
                raise ValueError(f"mask must be shape ({self.num_drones},), got {tuple(m.shape)}.")
            m = m.to(torch.uint8).contiguous()
        ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
        _lib.check(_lib.lib().pfb_set_base_state(self._h, ptr(m), ptr(p), ptr(q), ptr(lv), ptr(av), self._s()))
        self._state_fresh = False

    def base_state(self) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """``getBasePositionAndOrientation`` / ``getBaseVelocity`` of every drone: fp64 device tensors position [N, 3],
        quaternion [N, 4] (x, y, z, w), world linear velocity [N, 3] (the hi + lo words the kernels carry) and world angular
        velocity [N, 3] (R w_body).  ``set_base_state(*base_state())`` writes the same state back."""
        n, f64 = self.num_drones, dict(dtype=torch.float64, device=self.device)
        pos, quat, lin, ang = torch.empty((n, 3), **f64), torch.empty((n, 4), **f64), torch.empty((n, 3), **f64), torch.empty((n, 3), **f64)
        _lib.check(_lib.lib().pfb_get_base_state(self._h, C.c_void_p(pos.data_ptr()), C.c_void_p(quat.data_ptr()), C.c_void_p(lin.data_ptr()),
                                                 C.c_void_p(ang.data_ptr()), self._s()))
        return pos, quat, lin, ang

    # ------------------------------------------------------------------ static bodies (DESIGN.md §4h)
    def loadURDF(self, fileName: str, basePosition=(0.0, 0.0, 0.0), baseOrientation=None, useFixedBase: bool = True,
                 globalScaling: float = 1.0) -> int:
        """The reference's ``aviary.loadURDF`` of a fixed-base body (a landing pad, a helipad, a rooftop), placed in every drone's
        world with its base link frame at ``basePosition`` / ``baseOrientation`` (x, y, z, w; None = identity).  Returns the
        body index ``k``: column ``1 + k`` of ``contact_bodies()``.  The body must be boxes and cylinders joined by fixed joints,
        upright once posed (a yaw only); spheres, meshes, tilted poses and ``useFixedBase=False`` are refused.  Aviary handles
        only."""
        if self.env_config is not None and self.env_config.env_kind != 0:
            raise AviaryInitException("static bodies are for Aviary handles; an env handle (env_config) keeps its own floor and pad.")
        if not useFixedBase:
            raise ValueError("only fixed-base bodies (useFixedBase=True) can be loaded: a free body would need contact between bodies.")
        pos = np.asarray(basePosition, dtype=np.float64).reshape(-1)
        quat = np.asarray((0.0, 0.0, 0.0, 1.0) if baseOrientation is None else baseOrientation, dtype=np.float64).reshape(-1)
        if pos.shape != (3,) or quat.shape != (4,):
            raise ValueError(f"basePosition must have 3 entries and baseOrientation 4, got {pos.shape[0]} and {quat.shape[0]}.")
        if not abs(float(np.linalg.norm(quat)) - 1.0) <= 1e-6:
            raise ValueError("baseOrientation must be a unit quaternion (x, y, z, w).")
        path = str(fileName)
        if not os.path.isfile(path):
            raise FileNotFoundError(f"cannot find the URDF {fileName!r}")
        L = _lib.lib()
        shapes = (PfbShape * MAX_STATIC_SHAPES)()
        n = C.c_int(0)
        inertial = (C.c_double * 3)()
        _lib.check(L.pfb_static_shapes_from_urdf(path.encode(), float(globalScaling), shapes, MAX_STATIC_SHAPES, C.byref(n), inertial))
        body = C.c_int(-1)
        p3, q4 = (C.c_double * 3)(*pos), (C.c_double * 4)(*quat)
        _lib.check(L.pfb_add_static_body(self._h, shapes, n.value, p3, q4, inertial, C.byref(body), self._s()))
        self.static_bodies.append(path)
        return int(body.value)

    def register_all_new_bodies(self) -> None:
        """The reference registers new bodies for its contact array (aviary.py:314-320); here every loaded body is registered
        by ``loadURDF``.  Kept so that scripts run unchanged."""

    def set_static_pose(self, body: int, pos, quat=None, mask=None) -> None:
        """``resetBasePositionAndOrientation`` of static body ``body`` in the worlds of the drones of ``mask`` ([N] bool; None =
        every drone): ``pos`` [N, 3] or [3], ``quat`` [N, 4] or [4] (x, y, z, w; None = identity), fp64, upright (a yaw only).
        As in PyBullet, the pose is that of the body's base INERTIAL frame (``loadURDF``'s ``basePosition`` places its base link
        frame; the two differ by the inertial origin of the URDF's base link).  Each drone's world keeps its own pose, so every
        drone may get a different one (randomised pads)."""
        n = self.num_drones
        if not 0 <= int(body) < len(self.static_bodies):
            raise ValueError(f"no static body {body}: {len(self.static_bodies)} loaded since the last reset().")
        p = np.broadcast_to(np.asarray(pos, dtype=np.float64), (n, 3)) if np.asarray(pos).ndim == 1 else np.asarray(pos, dtype=np.float64)
        q = np.asarray((0.0, 0.0, 0.0, 1.0) if quat is None else quat, dtype=np.float64)
        q = np.broadcast_to(q, (n, 4)) if q.ndim == 1 else q
        if p.shape != (n, 3) or q.shape != (n, 4):
            raise ValueError(f"pos must be shape ({n}, 3) or (3,) and quat ({n}, 4) or (4,), got {p.shape} and {q.shape}.")
        err = float(np.max(np.abs(np.linalg.norm(q, axis=1) - 1.0))) if n else 0.0
        if not err <= 1e-6:
            raise ValueError(f"quat must be unit quaternions (x, y, z, w): a norm differs from 1 by {err:.3g} (> 1e-6).")
        if not _upright_error(q) <= 1e-9:
            raise ValueError("static bodies stay upright: quat must be a yaw about the world z axis (tilted static bodies are not modelled).")
        pt = torch.as_tensor(np.ascontiguousarray(p), device=self.device)
        qt = torch.as_tensor(np.ascontiguousarray(q), device=self.device)
        m = None
        if mask is not None:
            m = torch.as_tensor(mask, device=self.device)
            if tuple(m.shape) != (n,):
                raise ValueError(f"mask must be shape ({n},), got {tuple(m.shape)}.")
            m = m.to(torch.uint8).contiguous()
        _lib.check(_lib.lib().pfb_set_static_pose(self._h, int(body), C.c_void_p(pt.data_ptr()), C.c_void_p(qt.data_ptr()),
                                                  None if m is None else C.c_void_p(m.data_ptr()), self._s()))

    def contact_bodies(self) -> torch.Tensor:
        """(N, 1 + M) bool, M = static bodies loaded: column 0 the floor, column 1 + k static body k, touched during the last
        ``step()`` — the reference's ``contact_array[drone.Id, body_id]``.  ``contact_array`` is their ``any``."""
        if not self.static_bodies:
            return self.contact_array.reshape(-1, 1)
        bits = torch.empty((self.num_drones,), dtype=torch.int32, device=self.device)
        _lib.check(_lib.lib().pfb_get_static_contacts(self._h, C.c_void_p(bits.data_ptr()), self._s()))
        cols = torch.arange(1 + len(self.static_bodies), dtype=torch.int32, device=self.device)
        return ((bits[:, None] >> cols[None, :]) & 1).bool()

    def _refresh(self):
        if not self._state_fresh:
            _lib.check(_lib.lib().pfb_observe_state(self._h, self._s()))
            self._state_fresh = True

    @property
    def all_states(self) -> torch.Tensor:
        """(N, 4, 3): ang_vel (body), euler, lin_vel (body), position — aviary.py:372-393."""
        self._refresh()
        return self._drone_state.view(self.num_drones, 4, 3)

    @property
    def all_aux_states(self) -> torch.Tensor | list[torch.Tensor]:
        """(N, A) tensor; a batch of several kinds returns a list of ``N`` tensors of each drone's own aux length (aviary.py:396-411)."""
        self._refresh()
        if self.kinds is not None:
            return [self._aux_state[i, : self._aux_len[i]] for i in range(self.num_drones)]
        return self._aux_state

    def state(self, index: int) -> torch.Tensor:
        return self.all_states[index]

    def aux_state(self, index: int) -> torch.Tensor:
        if self.kinds is not None:
            self._refresh()
            return self._aux_state[index, : self._aux_len[index]]
        return self.all_aux_states[index]

    @property
    def contact_array(self) -> torch.Tensor:
        """(N,) bool: contact with the floor or any static body during the last step (aviary.py:322, 523-525, per world; the
        reference's ``np.any(contact_array[drone.Id])``)."""
        self._refresh()
        return self._contact.bool()

    # ------------------------------------------------------------------ raw state access (tests, debugging)
    def _single_kind(self, what: str) -> None:
        if self.kinds is not None:
            raise NotImplementedError(f"{what} is not available on a batch of several vehicle kinds (drone_type={sorted(set(self.kinds))}).")

    def state_row(self, row: int) -> torch.Tensor:
        """[N] fp32 copy-free view (field-major) or gathered copy (warp-tiled) of state row ``row``."""
        self._single_kind("state_row (a kind-specific state layout)")
        if not self.tiled:
            return self.state_tensor[row]
        return self.state_tensor[:, row // 4, :, row % 4].reshape(-1)[: self.num_drones]

    def state_row_int(self, row: int) -> torch.Tensor:
        """[N] int32: a row that holds integer bits (warp-tiled layout: 17 = step_count, 18 = flags)."""
        return self.state_row(row).contiguous().view(torch.int32)

    @property
    def precise_positions(self) -> torch.Tensor:
        """(N, 3) float64 world positions as the kernels carry them: hi + lo fp32 words of the state tensor."""
        if self.kinds is not None:  # pfb_observe_state writes the hi and lo words into obs [N, 6]
            self._refresh()
            return self.obs[:, :3].double() + self.obs[:, 3:6].double()
        lo = {"quadx": 25, "fixedwing": 19, "rocket": 22}[self.drone_type]
        return torch.stack([self.state_row(k).double() + self.state_row(lo + k).double() for k in range(3)], dim=1)

    @property
    def step_counts(self) -> torch.Tensor:
        """[N] int32 env step counters."""
        return self.state_row_int(17) if self.tiled else self.istate_tensor[0]

    def register_wind_field(self, wind) -> None:
        """``Aviary.register_wind_field_function`` (aviary.py:324-334) for an analytic field: ``wind`` is a
        :class:`pyflyt_b200.core.wind.AnalyticWind` (the same object is a valid wind-field function for the reference) or ``None``
        for still air.  Arbitrary Python callbacks cannot run inside the step kernel (DESIGN.md, out of scope)."""
        from .wind import AnalyticWind, PfbWind

        if wind is None:
            _lib.check(_lib.lib().pfb_set_wind(self._h, None))
            self.wind_field = None
            return
        if not isinstance(wind, AnalyticWind):
            raise TypeError("the batched stepper evaluates the wind inside the CUDA kernels: pass a pyflyt_b200.core.wind.AnalyticWind")
        L = _lib.lib()
        assert L.pfb_sizeof_wind() == C.sizeof(PfbWind)
        w = wind.as_struct()
        _lib.check(L.pfb_set_wind(self._h, C.byref(w)))
        self.wind_field = wind

    register_wind_field_function = register_wind_field

    def reseed(self, seed: int) -> None:
        """``env.reset(seed=s)``: re-key the random streams and rewind every call counter, so that the same seed replays the same
        episodes (the reference re-creates ``np_random``, aviary.py:108-117).  The spare post-reset states built from the old
        streams are dropped: follow with a full ``env_reset()`` (no mask) or ``reset()``."""
        self.seed = int(seed)
        _lib.check(_lib.lib().pfb_reseed(self._h, self.seed, self._s()))

    def set_noise_dump(self, buf: torch.Tensor | None) -> None:
        """Test aid: ``buf`` [env_step_ratio * updates_per_step, N] fp32 receives every motor-noise draw of the following
        QuadX-Hover ``env_step`` calls (None = off)."""
        self._single_kind("set_noise_dump")
        self._noise_dump = buf
        _lib.check(_lib.lib().pfb_set_noise_dump(self._h, None if buf is None else C.c_void_p(buf.data_ptr())))

    @property
    def launch_count(self) -> int:
        return int(_lib.lib().pfb_launch_count(self._h))

    # ------------------------------------------------------------------ fused env surface
    def env_reset(self, mask: torch.Tensor | None = None, noise: torch.Tensor | None = None, targets: torch.Tensor | None = None,
                  seed: int | None = None) -> torch.Tensor:
        """env.reset() for all / masked envs.  ``targets`` [N, 3*num_targets] installs explicit waypoints
        (parity tests); by default they are drawn on device like ``WaypointHandler.reset``.  ``seed``: ``reseed(seed)`` first;
        that rewinds every env, so it resets the whole batch and takes no ``mask``."""
        self._single_kind("env_reset")
        if seed is not None:
            if mask is not None:
                raise ValueError("reset(seed=...) re-keys the random streams of every env: it resets the whole batch and takes no mask")
            self.reseed(seed)
        if targets is not None:
            self._reset_targets = torch.as_tensor(targets, dtype=torch.float32, device=self.device).reshape(self.num_drones, -1).contiguous()
            self._buffers.reset_targets = self._reset_targets.data_ptr()
            _lib.check(_lib.lib().pfb_bind(self._h, C.byref(self._buffers)))
        elif self._reset_targets is not None:
            self._reset_targets = None
            self._buffers.reset_targets = None
            _lib.check(_lib.lib().pfb_bind(self._h, C.byref(self._buffers)))
        m = None if mask is None else C.c_void_p(mask.to(torch.uint8).contiguous().data_ptr())
        nz = None if noise is None else C.c_void_p(noise.data_ptr())
        _lib.check(_lib.lib().pfb_env_reset(self._h, m, nz, self._s()))
        self._state_fresh = False
        return self.obs

    def env_step(self, actions: torch.Tensor | None = None, noise: torch.Tensor | None = None) -> None:
        """One fused env.step() for every env; ``actions`` [N, S] fp32 on this device (None = ``self.setpoints``)."""
        self._single_kind("env_step")
        act = None
        if actions is not None:
            assert actions.is_cuda and actions.dtype == torch.float32 and actions.is_contiguous()
            assert tuple(actions.shape) == (self.num_drones, self.setpoint_dim), tuple(actions.shape)
            act = C.c_void_p(actions.data_ptr())
        nz = None if noise is None else C.c_void_p(noise.data_ptr())
        _lib.check(_lib.lib().pfb_env_step(self._h, act, nz, self._s()))
        self._state_fresh = False

    @staticmethod
    def out_slab_bytes(n: int, obs_dim: int) -> int:
        return n * obs_dim * 4 + n * 4 + n + n

    @staticmethod
    def slab_views(slab: torch.Tensor, n: int, obs_dim: int):
        """(obs [n, O] f32, reward [n] f32, term [n] u8, trunc [n] u8) views of a contiguous uint8 slab (device or pinned host)."""
        o = n * obs_dim * 4
        obs = slab[:o].view(torch.float32).view(n, obs_dim)
        reward = slab[o : o + 4 * n].view(torch.float32)
        term = slab[o + 4 * n : o + 5 * n]
        trunc = slab[o + 5 * n : o + 6 * n]
        return obs, reward, term, trunc

    def dogfight_physics(self, payload: torch.Tensor, actions: torch.Tensor | None = None, noise: torch.Tensor | None = None,
                         first: bool = False, do_reset: bool = False, aviary_index: int = 0) -> None:
        """Split dogfight, half 1: integrate one Aviary step (or reset + warm-up) and publish ``payload`` [N, 20]."""
        self._single_kind("dogfight_physics")
        act = None if actions is None else C.c_void_p(actions.data_ptr())
        nz = None if noise is None else C.c_void_p(noise.data_ptr())
        _lib.check(_lib.lib().pfb_dogfight_physics(self._h, act, nz, C.c_void_p(payload.data_ptr()), int(first), int(do_reset), int(aviary_index), self._s()))
        self._state_fresh = False

    def dogfight_physics_peer(self, peer_tables: torch.Tensor, world: int, slot_offset_floats: int, actions: torch.Tensor | None = None,
                              noise: torch.Tensor | None = None, first: bool = False, do_reset: bool = False, aviary_index: int = 0,
                              peer_flags: torch.Tensor | None = None, rank: int = 0, epoch: int = 0) -> None:
        """Split dogfight, half 1 with the exchange fused in: every payload is stored straight into all ranks' tables
        (``peer_tables``: int64 device tensor of ``world`` peer-mapped base pointers)."""
        self._single_kind("dogfight_physics_peer")
        act = None if actions is None else C.c_void_p(actions.data_ptr())
        nz = None if noise is None else C.c_void_p(noise.data_ptr())
        fl = None if peer_flags is None else C.c_void_p(peer_flags.data_ptr())
        _lib.check(_lib.lib().pfb_dogfight_physics_peer(self._h, act, nz, C.c_void_p(peer_tables.data_ptr()), int(world), int(slot_offset_floats),
                                                        fl, int(rank), int(epoch), int(first), int(do_reset), int(aviary_index), self._s()))
        self._state_fresh = False

    def dogfight_combat_wait(self, table: torch.Tensor, first_global_agent: int, num_arenas: int, last: int, flags: torch.Tensor,
                             world: int, epoch: int) -> None:
        """Split dogfight, half 2, waiting in-kernel until every rank's physics kernel has raised its flag to ``epoch``."""
        self._single_kind("dogfight_combat_wait")
        _lib.check(_lib.lib().pfb_dogfight_combat_wait(self._h, C.c_void_p(table.data_ptr()), int(first_global_agent), int(num_arenas), int(last),
                                                       C.c_void_p(flags.data_ptr()), int(world), int(epoch), self._s()))
        self._state_fresh = False

    def dogfight_split_step(self, actions: torch.Tensor, peer_tables: torch.Tensor, peer_flags: torch.Tensor, tables: torch.Tensor,
                            flags: torch.Tensor, world: int, rank: int, epoch0: int, first_global_agent: int, num_arenas: int) -> None:
        """A whole env step of the split dogfight (fused exchange, in-kernel signalling) in one library call."""
        self._single_kind("dogfight_split_step")
        _lib.check(_lib.lib().pfb_dogfight_split_step(self._h, C.c_void_p(actions.data_ptr()), C.c_void_p(peer_tables.data_ptr()),
                                                      C.c_void_p(peer_flags.data_ptr()), C.c_void_p(tables.data_ptr()), C.c_void_p(flags.data_ptr()),
                                                      int(world), int(rank), int(epoch0), int(first_global_agent), int(num_arenas), self._s()))
        self._state_fresh = False

    def dogfight_combat(self, table: torch.Tensor, first_global_agent: int, num_arenas: int, last: int) -> None:
        """Split dogfight, half 2: combat state from the all-gathered payload ``table`` [2 * num_arenas, 20]."""
        self._single_kind("dogfight_combat")
        _lib.check(_lib.lib().pfb_dogfight_combat(self._h, C.c_void_p(table.data_ptr()), int(first_global_agent), int(num_arenas), int(last), self._s()))
        self._state_fresh = False

    def profile_begin(self, capacity: int) -> None:
        _lib.check(_lib.lib().pfb_profile_begin(self._h, int(capacity)))

    def profile_read(self, capacity: int) -> list[float]:
        buf = (C.c_float * capacity)()
        n = _lib.lib().pfb_profile_read(self._h, buf, capacity)
        if n < 0:
            _lib.check(n)
        return [float(buf[i]) for i in range(n)]

    def env_rollout(self, n_steps: int) -> None:
        _lib.check(_lib.lib().pfb_env_rollout(self._h, int(n_steps), self._s()))
        self._state_fresh = False

    def env_step_mapped(self, actions: torch.Tensor, obs: torch.Tensor, reward: torch.Tensor, term: torch.Tensor, trunc: torch.Tensor) -> None:
        """Zero-copy end-to-end step: the kernel reads ``actions`` from and writes the results into PINNED host tensors."""
        self._single_kind("env_step_mapped")
        self._single_kind("env_rollout")
        for t in (actions, obs, reward, term, trunc):
            assert not t.is_cuda and t.is_contiguous() and t.is_pinned()
        _lib.check(_lib.lib().pfb_env_step_mapped(self._h, C.c_void_p(actions.data_ptr()), C.c_void_p(obs.data_ptr()), C.c_void_p(reward.data_ptr()), C.c_void_p(term.data_ptr()), C.c_void_p(trunc.data_ptr()), self._s()))
        self._state_fresh = False

    def env_step_host(self, actions: torch.Tensor, obs: torch.Tensor, reward: torch.Tensor, term: torch.Tensor, trunc: torch.Tensor) -> None:
        """Pinned-host in, pinned-host out (the end-to-end path bench.py times)."""
        self._single_kind("env_step_host")
        for t in (actions, obs, reward, term, trunc):
            assert not t.is_cuda and t.is_contiguous()
        _lib.check(_lib.lib().pfb_env_step_host(self._h, C.c_void_p(actions.data_ptr()), C.c_void_p(obs.data_ptr()), C.c_void_p(reward.data_ptr()), C.c_void_p(term.data_ptr()), C.c_void_p(trunc.data_ptr()), self._s()))
        self._state_fresh = False
