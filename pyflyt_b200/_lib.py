"""ctypes binding of libpyflyt_b200.so (include/pyflyt_b200.h).  There is no CPU fallback: if the
CUDA library is missing or no device is present, every compute entry raises."""

from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.realpath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libpyflyt_b200.so")
_lib = None


class PfbError(RuntimeError):
    """An error reported by libpyflyt_b200 (pfb_last_error)."""


class PfbBuffers(C.Structure):
    _fields_ = [
        ("state", C.c_void_p),
        ("istate", C.c_void_p),
        ("setpoint", C.c_void_p),
        ("start_pos", C.c_void_p),
        ("start_orn", C.c_void_p),
        ("reset_targets", C.c_void_p),
        ("obs", C.c_void_p),
        ("reward", C.c_void_p),
        ("term", C.c_void_p),
        ("trunc", C.c_void_p),
        ("info", C.c_void_p),
        ("final_obs", C.c_void_p),
        ("drone_state", C.c_void_p),
        ("aux_state", C.c_void_p),
        ("contact", C.c_void_p),
    ]


def build(verbose: bool = False) -> str:
    """Compiles pyflyt_b200/csrc for the H100 (sm_90a) into pyflyt_b200/lib (nvcc cross-compiles without a GPU)."""
    cuda_home = os.environ.get("CUDA_HOME") or os.environ.get("CUDA_PATH") or "/usr/local/cuda"
    nvcc = shutil.which("nvcc") or os.path.join(cuda_home, "bin", "nvcc")
    if not os.path.exists(nvcc):
        raise PfbError("nvcc not found: cannot build libpyflyt_b200.so")
    jobs = str(min(8, os.cpu_count() or 1))
    r = subprocess.run(["make", "-j", jobs, "-C", os.path.join(_HERE, "csrc"), f"NVCC={nvcc}"], capture_output=True, text=True)
    if r.returncode != 0:
        raise PfbError("building libpyflyt_b200.so failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stdout)
    return LIB_PATH


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise PfbError(
            f"{LIB_PATH} is missing.  Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C pyflyt_b200/csrc`).  pyflyt_b200 has no CPU fallback."
        )
    L = C.CDLL(LIB_PATH)
    vp, i64, u64, i32 = C.c_void_p, C.c_int64, C.c_uint64, C.c_int
    L.pfb_last_error.restype = C.c_char_p
    L.pfb_create.argtypes = [vp, vp, i64, i32, u64, C.POINTER(vp)]
    L.pfb_create_mixed.argtypes = [vp, i32, vp, i64, vp, i32, u64, C.POINTER(vp)]
    L.pfb_model_from_files.argtypes = [i32, C.c_char_p, C.c_char_p, C.c_double, C.c_double, vp]
    L.pfb_destroy.argtypes = [vp]
    L.pfb_set_env_offset.argtypes = [vp, u64]
    for name in ("pfb_state_rows", "pfb_istate_rows", "pfb_setpoint_dim", "pfb_obs_dim", "pfb_aux_dim", "pfb_state_layout"):
        getattr(L, name).argtypes = [vp]
    L.pfb_state_floats.restype = i64
    L.pfb_state_floats.argtypes = [vp]
    L.pfb_set_noise_dump.argtypes = [vp, vp]
    L.pfb_reseed.argtypes = [vp, u64, vp]
    L.pfb_set_wind.argtypes = [vp, vp]
    L.pfb_set_models.argtypes = [vp, vp, i32, vp]
    L.pfb_bind.argtypes = [vp, vp]
    L.pfb_reset.argtypes = [vp, vp, vp]
    L.pfb_set_mode.argtypes = [vp, i32, vp]
    L.pfb_set_modes.argtypes = [vp, vp, vp]
    L.pfb_aviary_step.argtypes = [vp, i32, vp, vp]
    L.pfb_observe_state.argtypes = [vp, vp]
    L.pfb_static_shapes_from_urdf.argtypes = [C.c_char_p, C.c_double, vp, i32, vp, vp]
    L.pfb_add_static_body.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp]
    L.pfb_set_static_pose.argtypes = [vp, i32, vp, vp, vp, vp]
    L.pfb_get_static_contacts.argtypes = [vp, vp, vp]
    L.pfb_set_base_velocity.argtypes = [vp, vp, vp, vp]
    L.pfb_set_base_state.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    L.pfb_get_base_state.argtypes = [vp, vp, vp, vp, vp, vp]
    L.pfb_env_reset.argtypes = [vp, vp, vp, vp]
    L.pfb_env_step.argtypes = [vp, vp, vp, vp]
    L.pfb_env_rollout.argtypes = [vp, i32, vp]
    L.pfb_env_step_host.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    L.pfb_env_step_mapped.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    L.pfb_dogfight_physics.argtypes = [vp, vp, vp, vp, i32, i32, i32, vp]
    L.pfb_dogfight_combat.argtypes = [vp, vp, i64, i64, i32, vp]
    L.pfb_dogfight_physics_peer.argtypes = [vp, vp, vp, vp, i32, i64, vp, i32, i32, i32, i32, i32, vp]
    L.pfb_dogfight_combat_wait.argtypes = [vp, vp, i64, i64, i32, vp, i32, i32, vp]
    L.pfb_dogfight_split_step.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, i32, i64, i64, vp]
    L.pfb_launch_count.restype = i64
    L.pfb_launch_count.argtypes = [vp]
    L.pfb_profile_begin.argtypes = [vp, i32]
    L.pfb_profile_read.argtypes = [vp, vp, i32]
    if L.pfb_sizeof_buffers() != C.sizeof(PfbBuffers):
        raise PfbError("PfbBuffers layout mismatch between Python and libpyflyt_b200.so")
    _lib = L
    return L


def check(rc: int) -> None:
    if rc != 0:
        raise PfbError(lib().pfb_last_error().decode("utf-8", "replace"))


EXPORTS = [
    "pfb_last_error", "pfb_abi_version", "pfb_sizeof_model", "pfb_sizeof_env_config", "pfb_sizeof_buffers",
    "pfb_model_from_files", "pfb_create", "pfb_create_mixed", "pfb_destroy", "pfb_set_env_offset", "pfb_state_rows", "pfb_state_layout", "pfb_state_floats", "pfb_set_noise_dump", "pfb_reseed", "pfb_set_wind", "pfb_sizeof_wind", "pfb_set_models",
    "pfb_istate_rows", "pfb_setpoint_dim",
    "pfb_obs_dim", "pfb_aux_dim", "pfb_bind", "pfb_reset", "pfb_set_mode", "pfb_set_modes", "pfb_aviary_step", "pfb_observe_state",
    "pfb_set_base_velocity", "pfb_set_base_state", "pfb_get_base_state",
    "pfb_static_shapes_from_urdf", "pfb_add_static_body", "pfb_set_static_pose", "pfb_get_static_contacts",
    "pfb_env_reset", "pfb_env_step", "pfb_env_rollout", "pfb_env_step_host", "pfb_env_step_mapped", "pfb_launch_count",
    "pfb_profile_begin", "pfb_profile_read", "pfb_dogfight_payload_dim", "pfb_dogfight_physics", "pfb_dogfight_physics_peer", "pfb_dogfight_combat", "pfb_dogfight_combat_wait", "pfb_dogfight_split_step",
]  # every symbol include/pyflyt_b200.h declares
