"""TEST INFRASTRUCTURE — NumPy restatement of the device-side random streams of libpyflyt_b200 (pyflyt_b200/csrc/pfb_common.cuh:
philox4x32_10, u32_to_unit_open, box_muller; pfb_noise.cuh: PhiloxNoise; pfb_quadx.cu: the RANDACT action mapping of k_hover_step).

The kernels are stateless: every draw is a pure function of (seed, global env id, call sequence number, stream tag, Aviary
step).  That lets a test regenerate exactly the noise / action streams the TIMED instantiation of the step kernel consumes
(Philox noise, NEXT_STEP autoreset) and drive the fp64 CPU oracle with them in lock-step.  Integer parts are bit-exact; the
Box-Muller transform uses the device's fast intrinsics (__logf, __sincosf, sqrt.approx) on the GPU and libm here, so normals
agree to ~1e-6, which the noise-dump test pins (tests/test_timed_path_parity.py).
"""
from __future__ import annotations

import numpy as np

TAG_AVIARY, TAG_ENV_STEP, TAG_RESET, TAG_ACTION = 0, 1, 2, 3
M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0: int, k1: int):
    """Philox4x32-10 (Salmon et al., SC'11) on arrays of uint32 counters; returns four uint32 arrays."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & MASK for c in (c0, c1, c2, c3))
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    k0, k1 = int(k0) & 0xFFFFFFFF, int(k1) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = M0 * c0, M1 * c2
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & MASK, p1 >> np.uint64(32), p1 & MASK
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint64(k0), lo1, hi0 ^ c3 ^ np.uint64(k1), lo0
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return tuple(c.astype(np.uint32) for c in (c0, c1, c2, c3))


def unit_open(u):
    """(0, 1]: ((u >> 8) + 1) * 2^-24 — exact in float32."""
    return ((np.asarray(u, dtype=np.uint32) >> np.uint32(8)).astype(np.float32) + np.float32(1.0)) * np.float32(1.0 / 16777216.0)


def box_muller(a, b):
    u1, u2 = unit_open(a).astype(np.float64), unit_open(b).astype(np.float64)
    r = np.sqrt(-2.0 * np.log(u1))
    ang = np.float32(6.28318530717958647692).astype(np.float64) * u2
    return (r * np.cos(ang)).astype(np.float32), (r * np.sin(ang)).astype(np.float32)


class Streams:
    """The streams of one handle: key = seed (k0 = low word, k1 = high word), counters start at the global env id."""

    def __init__(self, seed: int, n_envs: int, env_offset: int = 0, noise_loc: float = 4.0, ratio: int = 2):
        self.k0, self.k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
        g = np.arange(n_envs, dtype=np.uint64) + np.uint64(env_offset)
        self.env_lo, self.env_hi = (g & MASK).astype(np.uint32), (g >> np.uint64(32)).astype(np.uint32)
        self.n, self.loc, self.ratio = n_envs, np.float32(noise_loc), ratio
        assert ratio <= 2, "ratio > 2 draws one Philox call per Aviary step (not needed by the tests)"

    def _four(self, seq, tag: int, pair_step: int, envs=None):
        lo = self.env_lo if envs is None else self.env_lo[envs]
        hi = self.env_hi if envs is None else self.env_hi[envs]
        seq = np.broadcast_to(np.asarray(seq, dtype=np.uint32), lo.shape)
        r = philox4x32_10(lo, hi, seq, np.uint32((tag << 24) | pair_step), self.k0, self.k1)
        n0, n1 = box_muller(r[0], r[1])
        n2, n3 = box_muller(r[2], r[3])
        return n0, n1, n2, n3

    def noise(self, seq, tag: int, n_aviary: int, envs=None) -> np.ndarray:
        """[n_aviary * ratio][len(envs)] float32 raw draws N(loc, 1): what NoiseFn.get() hands out, in order."""
        m = self.n if envs is None else len(envs)
        out = np.zeros((n_aviary * self.ratio, m), dtype=np.float32)
        for a in range(0, n_aviary, 2):
            four = self._four(seq, tag, a, envs)
            for s in range(2):
                if a + s >= n_aviary:
                    break
                for u in range(self.ratio):
                    out[(a + s) * self.ratio + u] = self.loc + four[2 * s + u]
        return out

    def step_noise(self, step_seq: int, env_step_ratio: int = 3, envs=None):
        return self.noise(step_seq, TAG_ENV_STEP, env_step_ratio, envs)

    def user_reset_noise(self, reset_seq: int, warmup: int = 10, envs=None):
        """pfb_env_reset: seq = 0x80000000 | number of earlier pfb_env_reset calls"""
        return self.noise(0x80000000 | reset_seq, TAG_RESET, warmup, envs)

    def autoreset_noise(self, episode, warmup: int = 10, envs=None):
        """spare post-reset states: seq = the env's episode number (1 for the first autoreset after a user reset)"""
        return self.noise(episode, TAG_RESET, warmup, envs)

    def waypoint_targets(self, seq, num_targets: int, dome: float, min_height: float = 0.1, envs=None, yaw: bool = False) -> np.ndarray:
        """WaypointHandler.reset (gym_envs/utils/waypoint_handler.py:65-90) as the kernels draw it (pfb_fixedwing.cu wp_sample_targets,
        pfb_quadx_wp.cu qw_sample_targets): stream tag 4, counter word 3 = (4 << 24) | target index; [len(envs)][num_targets][3]
        (or [..][4] with `yaw`: the yaw target U(-pi, pi) from the fourth word of the same Philox call)"""
        lo = self.env_lo if envs is None else self.env_lo[envs]
        hi = self.env_hi if envs is None else self.env_hi[envs]
        seq = np.broadcast_to(np.asarray(seq, dtype=np.uint32), lo.shape)
        out = np.zeros((len(lo), num_targets, 4 if yaw else 3), dtype=np.float32)
        two_pi = np.float32(6.28318530717958647692)
        for k in range(num_targets):
            r = philox4x32_10(lo, hi, seq, np.uint32((4 << 24) | k), self.k0, self.k1)
            theta, phi = two_pi * unit_open(r[0]), two_pi * unit_open(r[1])
            dist = np.float32(1.0) + np.float32(dome * 0.9 - 1.0) * unit_open(r[2])
            out[:, k, 0] = dist * np.sin(phi) * np.cos(theta)
            out[:, k, 1] = dist * np.sin(phi) * np.sin(theta)
            z = np.abs(dist * np.cos(phi))
            out[:, k, 2] = np.where(z > min_height, z, np.float32(min_height))
            if yaw:
                out[:, k, 3] = np.float32(-3.14159265358979323846) + two_pi * unit_open(r[3])
        return out

    def drop_poses(self, seq, ceiling: float, max_displacement: float, envs=None):
        """options["randomize_drop"] (rocket_base_env.py:192-199) as k_land_step / k_land_reset draw it (pfb_rocket.cu
        landing_reset_env_inline): stream tag 5, two Philox calls; returns (start_pos [m][3], start_orn [m][3]) float32"""
        lo = self.env_lo if envs is None else self.env_lo[envs]
        hi = self.env_hi if envs is None else self.env_hi[envs]
        seq = np.broadcast_to(np.asarray(seq, dtype=np.uint32), lo.shape)
        a = philox4x32_10(lo, hi, seq, np.uint32(5 << 24), self.k0, self.k1)
        b = philox4x32_10(lo, hi, seq, np.uint32((5 << 24) | 1), self.k0, self.k1)
        one, two = np.float32(1.0), np.float32(2.0)
        rng_ = np.float32(max_displacement) * np.float32(0.1)
        pos = np.stack([rng_ * (two * unit_open(a[0]) - one), rng_ * (two * unit_open(a[1]) - one),
                        np.float32(ceiling) * (np.float32(0.8) + np.float32(0.1) * unit_open(a[2]))], axis=1)
        orn = np.stack([np.float32(0.3) * (two * unit_open(b[k]) - one) for k in range(3)], axis=1)
        return pos.astype(np.float32), orn.astype(np.float32)

    def uniform_actions(self, step_seq: int) -> np.ndarray:
        """RANDACT of the fixed-wing envs: U(-1, 1)^4"""
        r = philox4x32_10(self.env_lo, self.env_hi, np.uint32(step_seq), np.uint32(TAG_ACTION << 24), self.k0, self.k1)
        return np.stack([np.float32(2.0) * unit_open(x) - np.float32(1.0) for x in r], axis=1)

    def actions(self, step_seq: int, mode: int = 0) -> np.ndarray:
        """RANDACT: uniform in the env's action box (quadx_base_env.py:79-102)"""
        r = philox4x32_10(self.env_lo, self.env_hi, np.uint32(step_seq), np.uint32(TAG_ACTION << 24), self.k0, self.k1)
        u = [unit_open(x) for x in r]
        pi, two, one = np.float32(3.14159265358979323846), np.float32(2.0), np.float32(1.0)
        if mode == -1:
            return np.stack([np.float32(0.8) * x for x in u], axis=1)
        return np.stack([pi * (two * u[0] - one), pi * (two * u[1] - one), pi * (two * u[2] - one), np.float32(0.8) * u[3]], axis=1)
