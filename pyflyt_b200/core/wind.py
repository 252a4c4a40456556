"""Analytic, time-invariant wind fields (SURVEY.md 8f item 4).

``AnalyticWind`` is BOTH a plain Python wind-field function with the reference's signature — ``wind(time, position[n, 3])
-> [n, 3]``, what ``Aviary.register_wind_field_function`` accepts (/root/reference/PyFlyt/core/aviary.py:324-334) — and the
parameter block the CUDA kernels evaluate in place of that callback (``PfbWind`` in include/pyflyt_b200.h):

    wind(x, y, z) = base * f(z)
      constant   f = 1
      power      f = (max(z, 0) / z_ref) ** alpha      # alpha >= 0; alpha = 0 is the constant profile (0 ** 0 = 1)
      log        f = ln(max(z, z0) / z0) / ln(z_ref / z0)
      exp        f = exp(z / z_ref)          # tests/test_core.py:275-278 of the reference: base = (0, 0, 1), z_ref = 1
"""

from __future__ import annotations

import ctypes as C

import numpy as np

KINDS = {"none": 0, "constant": 1, "power": 2, "log": 3, "exp": 4}


class PfbWind(C.Structure):
    _fields_ = [("kind", C.c_int32), ("_pad", C.c_int32), ("base", C.c_double * 3), ("z_ref", C.c_double), ("alpha", C.c_double), ("z0", C.c_double)]


class AnalyticWind:
    def __init__(self, kind: str = "constant", base=(0.0, 0.0, 0.0), z_ref: float = 10.0, alpha: float = 1.0 / 7.0, z0: float = 0.03):
        if kind not in KINDS:
            raise ValueError(f"wind kind must be one of {sorted(KINDS)}, got {kind!r}")
        if z_ref <= 0.0 or (kind == "log" and not (0.0 < z0 < z_ref)):
            raise ValueError("z_ref must be positive and, for the log profile, 0 < z0 < z_ref")
        if kind == "power" and not alpha >= 0.0:  # a negative exponent makes the wind infinite at the floor
            raise ValueError(f"the power-law profile needs alpha >= 0, got {alpha}")
        self.kind, self.base = kind, np.asarray(base, dtype=np.float64).reshape(3)
        self.z_ref, self.alpha, self.z0 = float(z_ref), float(alpha), float(z0)

    def profile(self, z: np.ndarray) -> np.ndarray:
        z = np.asarray(z, dtype=np.float64)
        if self.kind == "none":
            return np.zeros_like(z)
        if self.kind == "constant":
            return np.ones_like(z)
        if self.kind == "power":
            return (np.maximum(z, 0.0) / self.z_ref) ** self.alpha
        if self.kind == "log":
            return np.log(np.maximum(z, self.z0) / self.z0) / np.log(self.z_ref / self.z0)
        return np.exp(z / self.z_ref)

    def __call__(self, time: float, position: np.ndarray) -> np.ndarray:
        position = np.asarray(position, dtype=np.float64)
        return self.profile(position[:, 2])[:, None] * self.base[None, :]

    def as_struct(self) -> PfbWind:
        w = PfbWind()
        w.kind = KINDS[self.kind]
        for k in range(3):
            w.base[k] = float(self.base[k])
        w.z_ref, w.alpha, w.z0 = self.z_ref, self.alpha, self.z0
        return w
