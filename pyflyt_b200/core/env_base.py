"""What the batched envs share: the reference bases' argument checks, the ``PfbEnvConfig`` fields every env kind fills the
same way, and the ``reset`` / ``step`` / ``rollout`` / ``close`` surface around one ``BatchedAviary``.

It lives in ``core`` rather than ``gym_envs`` because importing ``gym_envs`` registers the gymnasium ids, and the PettingZoo
envs build on it too."""

from __future__ import annotations

import torch

from ..models import PfbEnvConfig
from ..models.tables import AUTORESET_NEXT_STEP, AUTORESET_SAME_STEP
from .aviary import BatchedAviary

# env_config's autoreset_mode -> PfbEnvConfig.autoreset when autoreset is on
AUTORESET_MODES = {"next_step": AUTORESET_NEXT_STEP, "same_step": AUTORESET_SAME_STEP}


def check_env_args(agent_hz: int, render_mode: None | str, angle_representation: str = "quaternion", hz_error: type = ValueError) -> None:
    """The reference bases' constructor checks (quadx_base_env.py:47-52, 66-69), with their messages.  ``hz_error``: the gym
    bases raise ``ValueError`` for ``agent_hz``, the PettingZoo bases ``AssertionError`` (ma_quadx_base_env.py:47-52)."""
    if 120 % agent_hz != 0:
        lowest = int(120 / (int(120 / agent_hz) + 1))
        highest = int(120 / int(120 / agent_hz))
        raise hz_error(f"`agent_hz` must be round denominator of 120, try {lowest} or {highest}.")
    if render_mode is not None:
        raise ValueError("rendering is out of scope for the batched stepper (SURVEY.md §2 row 21)")
    if angle_representation not in ("euler", "quaternion"):
        raise ValueError(f"angle_representation must be either `euler` or `quaternion`, not {angle_representation}")


def env_config(env_kind: int, *, agent_hz: int, max_duration_seconds: float, angle_representation: str, sparse_reward: bool,
               autoreset: bool, flight_dome_size: float, inline_reset: bool = False, autoreset_mode: str = "next_step",
               **fields) -> PfbEnvConfig:
    """The ``PfbEnvConfig`` of an env of kind ``env_kind``: the fields every kind derives from its constructor arguments, then
    the kind-specific ``fields`` as given.

    ``inline_reset`` (autoreset kinds): integrate every post-reset warm-up inside the step launch instead of copying the env's
    spare post-reset state.  The results are the same bit for bit; the tests compare the two paths.

    ``autoreset_mode`` (with ``autoreset``): ``"next_step"``, gymnasium's NEXT_STEP (a finished env is reset on the next
    call, which ignores its action), or ``"same_step"``, gymnasium's SAME_STEP (it is reset inside the call that finishes it,
    which returns the terminal observation in ``final_obs``)."""
    if inline_reset not in (0, 1):
        raise ValueError(f"inline_reset must be a bool, got {inline_reset!r}")
    if autoreset_mode not in AUTORESET_MODES:
        raise ValueError(f"autoreset_mode must be one of {sorted(AUTORESET_MODES)}, got {autoreset_mode!r}")
    cfg = PfbEnvConfig()
    cfg.env_kind = env_kind
    cfg.env_step_ratio = int(120 / agent_hz)
    cfg.max_steps = int(agent_hz * max_duration_seconds)
    cfg.angle_representation = 0 if angle_representation == "euler" else 1
    cfg.sparse_reward = int(bool(sparse_reward))
    cfg.autoreset = AUTORESET_MODES[autoreset_mode] if autoreset else 0
    cfg.warmup_steps = 10  # Aviary steps after a reset: quadx_base_env.py:209-210, fixedwing_base_env.py:187-188
    cfg.flight_dome_size = float(flight_dome_size)
    cfg.inline_reset = int(inline_reset)
    for name, value in fields.items():
        setattr(cfg, name, value)
    return cfg


class AviaryEnv:
    """A batch of envs stepped by one ``BatchedAviary`` built from ``config``.  ``_info_flags`` lists the ``(key, bit)`` pairs
    that ``info`` decodes from the aviary's info bits."""

    _info_flags: tuple[tuple[str, int], ...] = (("out_of_bounds", 1), ("collision", 2), ("env_complete", 4))

    def __init__(self, config: PfbEnvConfig, start_pos, start_orn, drone_type: str, drone_options=None, seed: int | None = None,
                 device: str | torch.device = "cuda:0", env_offset: int = 0):
        self.config = config
        self.aviary = BatchedAviary(start_pos, start_orn, drone_type=drone_type, drone_options=drone_options, seed=seed, device=device,
                                    env_config=config, env_offset=env_offset)
        self.device = self.aviary.device
        self.obs_dim = self.aviary.obs_dim

    def _info(self) -> dict[str, torch.Tensor]:
        bits = self.aviary.info_bits
        return {key: (bits & bit).bool() for key, bit in self._info_flags}

    def _reset(self, mask: torch.Tensor | None = None, **kwargs):
        obs = self.aviary.env_reset(mask=mask, **kwargs)
        if mask is None:
            self.aviary.info_bits.zero_()
        return obs, self._info()

    def close(self) -> None:
        self.aviary.disconnect()


class VecEnv(AviaryEnv):
    """An ``AviaryEnv`` whose autoreset, if any, runs inside the step launch."""

    metadata = {"render_modes": [], "render_fps": 30}

    def reset(self, *, seed: int | None = None, options: dict | None = None, mask: torch.Tensor | None = None, noise=None):
        """env.reset() for every env, or for the envs where ``mask`` is set.  ``seed`` first re-keys the random streams of the
        whole batch (``BatchedAviary.reseed``): the same seed then replays the same episodes."""
        return self._reset(mask=mask, noise=noise, seed=seed)

    @property
    def same_step(self) -> bool:
        """Whether a finished env is reset inside the step that finishes it (``autoreset_mode="same_step"``)."""
        return self.config.autoreset == AUTORESET_SAME_STEP

    def step(self, actions: torch.Tensor, noise=None):
        """env.step(action) for every env.  With ``autoreset`` (gymnasium's default NEXT_STEP mode) an env that terminated or
        truncated on the previous call is reset on this one: its action is ignored and it returns the first observation of the
        new episode with reward 0 and both flags False, all inside the same kernel launch.

        With ``autoreset_mode="same_step"`` (gymnasium's SAME_STEP) an env that terminates or truncates on this call is reset
        on it too: the returned observation is the first one of its new episode, while reward, terminated, truncated and the
        other info keys are those of the step that finished it (so ``info`` holds its terminal flags; there is no
        ``final_info``).  ``info["final_obs"]`` is a zero-copy [N, O] view of its terminal observations, valid where
        ``info["_final_obs"]`` (= terminated | truncated) is set."""
        a = self.aviary
        if not (torch.is_tensor(actions) and actions.is_cuda and actions.dtype == torch.float32 and actions.is_contiguous()):
            a.setpoints.copy_(torch.as_tensor(actions, dtype=torch.float32, device=self.device).reshape(a.setpoints.shape))
            actions = None
        a.env_step(actions=actions, noise=noise)
        term, trunc, info = a.term.bool(), a.trunc.bool(), self._info()
        if self.same_step:
            info["final_obs"] = a.final_obs
            info["_final_obs"] = term | trunc
        return a.obs, a.reward, term, trunc, info

    def rollout(self, n_steps: int) -> None:
        """n_steps env steps with on-device uniform random actions (the benchmark's workload); the buffers then hold the last
        step's results.  QuadX-Hover with autoreset runs 4 or more steps as fused launches of up to 16 env steps each."""
        self.aviary.env_rollout(n_steps)


class WaypointsVecEnv(VecEnv):
    """A ``VecEnv`` with a list of waypoints per env: ``info["num_targets_reached"]`` counts the ones reached."""

    def _info(self) -> dict[str, torch.Tensor]:
        info = super()._info()
        info["num_targets_reached"] = (self.aviary.info_bits >> 3).int()
        return info

    def reset(self, *, seed: int | None = None, options: dict | None = None, mask: torch.Tensor | None = None, noise=None, targets=None):
        """``targets``: optional [N, num_targets, 3 or 4] waypoints (x, y, z[, yaw]); by default they are drawn on device."""
        return self._reset(mask=mask, noise=noise, targets=targets, seed=seed)
