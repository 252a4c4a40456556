"""The Aviary of a QuadX-Waypoints env keeps its drones field-major ([F][N] rows + istate), while a plain QuadX Aviary keeps
them warp-tiled.  ``env.aviary.step(n)`` runs the field-major (untiled) instantiations of the QuadX Aviary step, which no env
step reaches: this pins them, flown from the same reset, seed and setpoints, to the plain Aviary's drones."""
import numpy as np
import pytest


@pytest.mark.gpu
@pytest.mark.parametrize("mode", range(-1, 8))
@pytest.mark.parametrize("inject", [False, True])
def test_waypoints_aviary_step_matches_plain_aviary(mode, inject):
    import torch

    from pyflyt_b200.core.aviary import BatchedAviary
    from pyflyt_b200.gym_envs import QuadXWaypointsVecEnv

    n, seed, steps = 4099, 11, 3  # a ragged last tile on the warp-tiled side
    env = QuadXWaypointsVecEnv(num_envs=n, seed=seed, flight_mode=mode)
    wp = env.aviary
    assert not wp.tiled
    plain = BatchedAviary(np.tile([[0.0, 0.0, 1.0]], (n, 1)), np.zeros((n, 3)), seed=seed)
    assert plain.tiled
    rng = np.random.default_rng(mode + 2)
    lo, hi = (0.0, 0.8) if mode == -1 else (-0.5, 0.5)
    for av in (wp, plain):
        av.reset()
        av.set_mode(mode)
    for k in range(steps):
        sp = torch.as_tensor(rng.uniform(lo, hi, (n, 4)).astype(np.float32), device=plain.device)
        noise = None
        if inject:
            noise = torch.as_tensor(rng.normal(size=(10 * plain.updates_per_step, n)).astype(np.float32), device=plain.device)
        for av in (wp, plain):
            av.set_all_setpoints(sp)
            av.step(10, noise=noise)
        a, b = wp.all_states, plain.all_states
        assert torch.isfinite(b).all()
        assert torch.equal(a, b), f"step {k}: max |diff| {float((a - b).abs().max()):.3g}"
        assert torch.equal(wp.contact_array, plain.contact_array)
