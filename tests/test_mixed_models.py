"""Several QuadX vehicle models in one batch (``drone_options`` = one dict per drone, the reference's aviary.py:75, 196-199).

CPU: the model-set builder and its refusals, and the C oracle against the unmodified reference flying cf2x, primitive_drone
and a third vehicle loaded through ``model_dir`` in ONE Aviary (tests/golden/mixed_models_*.npz, tools/gen_golden.py).
GPU: the mixed-model kernels against the fixture, against the oracle per model, and env i of a mixed handle against env i of
a uniform handle of its model (same seed: the Philox streams depend on the env id, not on the model)."""
import json
import os
import re

import numpy as np
import pytest

from engines import GOLDEN, CudaEngine, OracleEngine, build_model, load_golden
from pyflyt_b200.models import MAX_QUADX_MODELS, ModelSetError, build_model_set

FIXTURES = ["mixed_models_quadx_mode0", "mixed_models_quadx_mode7"]
CF2X, PRIM = dict(drone_model="cf2x"), dict(drone_model="primitive_drone")
TUNED = dict(drone_model="primitive_tuned", model_dir=os.path.join(GOLDEN, "vehicles"))


def _bytes(m):
    import ctypes as C

    return C.string_at(C.addressof(m), C.sizeof(m))


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_model_set_two_tables_and_index():
    tables, index = build_model_set("quadx", [CF2X, PRIM, CF2X], 240, 3)
    assert len(tables) == 2 and index.dtype == np.uint8 and index.tolist() == [0, 1, 0]
    assert _bytes(tables[0]) == _bytes(build_model("quadx", "cf2x"))
    assert _bytes(tables[1]) == _bytes(build_model("quadx", "primitive_drone"))


def test_model_set_deduplicates_by_table_bytes():
    # equal dicts, a None entry and a dict that names the default model all build the cf2x table
    tables, index = build_model_set("quadx", [CF2X, dict(CF2X), None, {}, TUNED, PRIM], 240, 6)
    assert len(tables) == 3 and index.tolist() == [0, 0, 0, 0, 1, 2]
    assert _bytes(tables[1]) != _bytes(tables[2])  # primitive_tuned really differs from primitive_drone
    # one dict (or None) for every drone: one table
    for opts in (CF2X, None):
        tables, index = build_model_set("quadx", opts, 240, 5)
        assert len(tables) == 1 and index.tolist() == [0] * 5
    # a sequence whose entries build one fixed-wing table is accepted
    tables, index = build_model_set("fixedwing", [dict(drone_model="fixedwing"), {}], 240, 2)
    assert len(tables) == 1 and index.tolist() == [0, 0]


def test_model_set_refusals():
    with pytest.raises(ModelSetError, match=re.escape("If multiple `drone_options` (2) are used, must have same number of `drone_options` as number of drones (3).")):
        build_model_set("quadx", [CF2X, PRIM], 240, 3)
    with pytest.raises(ModelSetError, match="control_hz"):
        build_model_set("quadx", [dict(CF2X, control_hz=120), dict(PRIM, control_hz=60)], 240, 2)
    with pytest.raises(ModelSetError, match="one vehicle model"):
        build_model_set("fixedwing", [dict(drone_model="fixedwing"), dict(drone_model="acrowing")], 240, 2)


def test_model_set_cap(tmp_path):
    """More distinct tables than the library holds is refused; the cap is the header's PFB_MAX_QUADX_MODELS."""
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "pyflyt_b200.h")).read()
    assert int(re.search(r"#define PFB_MAX_QUADX_MODELS (\d+)", header).group(1)) == MAX_QUADX_MODELS
    src = os.path.join(GOLDEN, "vehicles", "primitive_drone")
    text = open(os.path.join(src, "primitive_drone.yaml")).read()
    urdf = open(os.path.join(src, "primitive_drone.urdf")).read()
    opts = []
    for k in range(MAX_QUADX_MODELS + 1):  # primitive_drone variants that differ in drag_coef_xyz
        name = f"variant{k}"
        os.makedirs(tmp_path / name)
        (tmp_path / name / f"{name}.urdf").write_text(urdf)
        (tmp_path / name / f"{name}.yaml").write_text(text.replace("drag_coef_xyz: 2.0", f"drag_coef_xyz: {1.0 + 0.05 * k}"))
        opts.append(dict(drone_model=name, model_dir=str(tmp_path)))
    tables, index = build_model_set("quadx", opts[:MAX_QUADX_MODELS], 240, MAX_QUADX_MODELS)
    assert len(tables) == MAX_QUADX_MODELS and index.tolist() == list(range(MAX_QUADX_MODELS))
    with pytest.raises(ModelSetError, match=f"at most {MAX_QUADX_MODELS}"):
        build_model_set("quadx", opts, 240, len(opts))


def test_aviary_checks_sequences_before_the_device():
    from pyflyt_b200.core.aviary import AviaryInitException, BatchedAviary

    z = np.zeros((3, 3))
    with pytest.raises(AviaryInitException, match=re.escape("If multiple `drone_options` (2) are used")):
        BatchedAviary(z, z, drone_options=[CF2X, PRIM])
    with pytest.raises(AviaryInitException, match="control_hz"):
        BatchedAviary(z, z, drone_options=[CF2X, PRIM, dict(CF2X, control_hz=60)])
    with pytest.raises(AviaryInitException, match="one vehicle model"):
        BatchedAviary(z, z, drone_type="fixedwing", drone_options=[dict(drone_model="fixedwing"), dict(drone_model="acrowing"), {}])


def _fixture_options(g):
    return [dict(d, model_dir=os.path.join(GOLDEN, d["model_dir"])) if "model_dir" in d else d for d in json.loads(str(g["drone_options"]))]


def _model(opts):
    return build_model("quadx", opts.get("drone_model"), opts.get("model_dir"))


def replay_mixed(g, engines):
    """Replays a mixed-model fixture; ``engines`` = [(engine, drone ids it flies)].  Max abs errors per drone."""
    n, T, mode = int(g["n_drones"]), len(g["state"]), int(g["mode"])
    noise = g["noise"].reshape(T, -1, n)
    err = {k: np.zeros(n) for k in ("setpoint", "pos", "euler", "angvel", "linvel", "aux")}
    err["contact_mismatch"] = np.zeros(n, dtype=int)
    for eng, ids in engines:
        eng.reset()
        eng.set_mode(mode)
        err["setpoint"][ids] = np.abs(eng.get_setpoints()[:, :4] - g["setpoint_after_set_mode"][ids]).max(axis=1)
    for i in range(T):
        for eng, ids in engines:
            eng.set_setpoints(g["setpoints"][i][ids])
            eng.aviary_step(noise[i][:, ids])
        for eng, ids in engines:
            s, ref = eng.state(), g["state"][i][ids]
            d_eul = np.abs((s[:, 1] - ref[:, 1] + np.pi) % (2 * np.pi) - np.pi)
            err["angvel"][ids] = np.maximum(err["angvel"][ids], np.abs(s[:, 0] - ref[:, 0]).max(axis=1))
            err["euler"][ids] = np.maximum(err["euler"][ids], d_eul.max(axis=1))
            err["linvel"][ids] = np.maximum(err["linvel"][ids], np.abs(s[:, 2] - ref[:, 2]).max(axis=1))
            err["pos"][ids] = np.maximum(err["pos"][ids], np.abs(s[:, 3] - ref[:, 3]).max(axis=1))
            err["aux"][ids] = np.maximum(err["aux"][ids], np.abs(eng.aux()[:, :4] - g["aux"][i][ids]).max(axis=1))
            err["contact_mismatch"][ids] += (eng.contact().astype(bool) != g["contact"][i][ids]).astype(int)
    return err


def test_mixed_fixtures_cover_three_tables():
    for name in FIXTURES:
        g = load_golden(name)
        tables, index = build_model_set("quadx", _fixture_options(g), 240, int(g["n_drones"]))
        assert len(tables) == 3 and sorted(set(index.tolist())) == [0, 1, 2], name


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_reference_mixed_aviary(name):
    """Each drone of the reference's multi-model Aviary, replayed by an oracle of its own model (bars of
    test_oracle_golden.py: 1e-9, 1e-6 in the height-hold modes)."""
    g = load_golden(name)
    opts = _fixture_options(g)
    engines = [(OracleEngine(_model(o), None, 1, g["start_pos"][d][None], g["start_orn"][d][None]), [d]) for d, o in enumerate(opts)]
    err = replay_mixed(g, engines)
    tol = 1e-6 if int(g["mode"]) in (2, 3, 7) else 1e-9
    assert err["setpoint"].max() == 0.0
    assert err["contact_mismatch"].sum() == 0
    for k in ("pos", "euler", "angvel", "linvel", "aux"):
        assert err[k].max() < tol, (name, k, err[k])


# ------------------------------------------------------------------------------------------------------------------ GPU
class MixedCudaEngine(CudaEngine):
    """CudaEngine over ONE BatchedAviary built with a per-drone ``drone_options`` sequence."""

    def __init__(self, drone_options, start_pos, start_orn, env=None, seed=0):
        import torch

        from pyflyt_b200.core.aviary import BatchedAviary

        self.torch = torch
        self.n = len(drone_options)
        self.av = BatchedAviary(np.asarray(start_pos, dtype=np.float32), np.asarray(start_orn, dtype=np.float32), drone_options=drone_options,
                                seed=seed, env_config=env)
        self.aux_dim, self.ups, self.obs_dim = self.av.aux_dim, self.av.updates_per_step, self.av.obs_dim


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_cuda_replays_mixed_fixture(name):
    """ONE CUDA handle flies the reference's three vehicles (bars of test_flight_modes / test_flight_modes_height_hold)."""
    g = load_golden(name)
    opts = _fixture_options(g)
    eng = MixedCudaEngine(opts, g["start_pos"], g["start_orn"])
    assert len(eng.av.models) == 3
    err = replay_mixed(g, [(eng, list(range(len(opts))))])
    assert err["contact_mismatch"].sum() == 0, err["contact_mismatch"]
    if int(g["mode"]) in (2, 3, 7):
        assert err["pos"].max() < 1e-3, err["pos"]
    else:
        assert err["setpoint"].max() < 1e-6
        assert err["pos"].max() < 0.5e-3 and err["euler"].max() < 1e-3, err


def _alternating(n):
    return [CF2X if i % 2 == 0 else PRIM for i in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 6])
def test_aviary_4096_alternating_models_match_oracle_per_model(mode):
    """4096 seeded envs, cf2x / primitive_drone alternating, against one oracle per model (bars of
    test_batch_4096_matches_oracle).  In mode 6 primitive_drone's z-velocity PID limit cycle amplifies fp32 rounding past these
    bars on the uniform kernels as well (DESIGN.md §5; ~0.09 m here), so there its envs are held to a uniform primitive_drone
    handle on the same inputs, bit for bit, and cf2x to the oracle."""
    n, steps = 4096, 240
    rng = np.random.default_rng(31 + mode)
    f = lambda a: a.astype(np.float32).astype(np.float64)  # noqa: E731
    start = f(np.column_stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), rng.uniform(20, 30, n)]))
    orn = f(rng.uniform(-0.3, 0.3, (n, 3)))
    cud = MixedCudaEngine(_alternating(n), start, orn)
    idx = cud.av.model_index.cpu().numpy()
    assert idx.tolist() == [i % 2 for i in range(n)]
    groups = [np.flatnonzero(idx == j) for j in range(2)]
    orcs = [OracleEngine(cud.av.models[j], None, len(ids), start[ids], orn[ids]) for j, ids in enumerate(groups)]
    if mode == 6:
        orcs[1] = CudaEngine(None, None, len(groups[1]), start[groups[1]], orn[groups[1]], drone_model="primitive_drone")
    noise = f(rng.normal(4.0, 1.0, (steps * 2, n)))
    for e in [cud] + orcs:
        e.reset()
        e.set_mode(mode)
    lo, hi = ([-1, -1, -1, 0.2], [1, 1, 1, 0.7]) if mode == 0 else ([-1, -1, -0.5, -0.5], [1, 1, 0.5, 0.5])
    for i in range(0, steps, 20):
        sp = f(rng.uniform(lo, hi, (n, 4)))
        cud.set_setpoints(sp)
        cud.aviary_step(noise[2 * i : 2 * i + 40], n_steps=20)
        for o, ids in zip(orcs, groups):
            o.set_setpoints(sp[ids])
            o.aviary_step(noise[2 * i : 2 * i + 40][:, ids], n_steps=20)
    b = cud.state()
    for o, ids in zip(orcs, groups):
        a = o.state()
        if isinstance(o, CudaEngine):
            assert np.array_equal(a, b[ids]) and np.array_equal(o.aux(), cud.aux()[ids])
        assert np.abs(a[:, 3] - b[ids, 3]).max() < 0.5e-3
        assert np.abs(a[:, 0] - b[ids, 0]).max() < 2e-3
        assert np.array_equal(o.contact(), cud.contact()[ids])
    # the two models really fly differently under the same commands
    assert np.abs(b[groups[0][:200], 3] - b[groups[1][:200], 3]).max() > 1.0


def _compare_to_uniform(mixed, uniform, idx, tag, worst_bar):
    """Env i of the mixed handle against env i of the uniform handle of its model: bars of test_fused_rollout_equals_stepwise."""
    import torch

    A = mixed.aviary
    same_all, worst, inexact, n = [], 0.0, 0.0, A.num_drones
    for j, U in enumerate(u.aviary for u in uniform):
        m = idx == j
        same = (A.step_counts == U.step_counts) & m
        assert int((m & ~same).sum()) <= max(2, n // 4096), (tag, j, int((m & ~same).sum()))
        d = (A.obs.double() - U.obs.double()).abs().amax(dim=1)
        worst = max(worst, float(d[same].max()))
        inexact = max(inexact, float((d[same] > 0).double().sum()) / max(1, int(m.sum())))
        assert torch.equal(A.term[same], U.term[same]) and torch.equal(A.trunc[same], U.trunc[same]), (tag, j)
        assert float((A.reward.double() - U.reward.double()).abs()[same].max()) < 1e-3, (tag, j)
        same_all.append(same)
    assert inexact < 1e-2 and worst < worst_bar, (tag, inexact, worst)
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("mode,variant", [(0, "plan"), (6, "plan"), (0, "inline_reset"), (0, "host")])
def test_hover_mixed_equals_uniform_handles(mode, variant):
    """QuadX-Hover at 65 536 envs, cf2x / primitive_drone interleaved per env, against two uniform handles with the same seed.
    "plan": the fused / single-step plan of test_fused_rollout_equals_stepwise (spare pipeline, fused rollout, hand-overs);
    "inline_reset": every warm-up integrated inside the step launch; "host": pfb_env_step_host with scripted actions."""
    import torch

    from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverVecEnv

    n = 65536
    kw = dict(num_envs=n, seed=21, flight_mode=mode, inline_reset=(variant == "inline_reset"))
    mixed = QuadXHoverVecEnv(drone_options=_alternating(n), **kw)
    uniform = [QuadXHoverVecEnv(drone_options=CF2X, **kw), QuadXHoverVecEnv(drone_options=PRIM, **kw)]
    envs = [mixed] + uniform
    idx = mixed.aviary.model_index
    assert len(mixed.aviary.models) == 2 and bool((idx == torch.arange(n, device=idx.device) % 2).all())
    for e in envs:
        e.reset()
    done_total, worst = 0, 0.0
    bar = 1e-4 if mode == 0 else 1e-2
    if variant == "host":
        g = torch.Generator().manual_seed(0)
        bufs = [(torch.empty((n, mixed.obs_dim)).pin_memory(), torch.empty(n).pin_memory(), torch.empty(n, dtype=torch.uint8).pin_memory(),
                 torch.empty(n, dtype=torch.uint8).pin_memory()) for _ in envs]
        for k in range(60):
            act = ((torch.rand((n, 4), generator=g) * 2 - 1) * torch.tensor([0.6, 0.6, 0.6, 0.0]) + torch.tensor([0.0, 0.0, 0.0, 0.45])).pin_memory()
            for e, b in zip(envs, bufs):
                e.aviary.env_step_host(act, *b)
            torch.cuda.synchronize()
            for e, b in zip(envs, bufs):  # the host results are the bound device buffers' copies
                assert torch.equal(e.aviary.obs.cpu(), b[0]) and torch.equal(e.aviary.reward.cpu(), b[1])
            done_total += int((mixed.aviary.term | mixed.aviary.trunc).sum())
            worst = max(worst, _compare_to_uniform(mixed, uniform, idx, k, bar))
    else:
        plan = [16, 16, 5, 1, 1, 23, 1, 40, 4, 2, 64]
        for chunk in plan:
            for e in envs:
                e.rollout(chunk)
            done_total += int((mixed.aviary.term | mixed.aviary.trunc).sum())
            for U in uniform:  # the actions of the last step: pure Philox, the same for every handle
                assert torch.equal(mixed.aviary.setpoints, U.aviary.setpoints), chunk
            worst = max(worst, _compare_to_uniform(mixed, uniform, idx, chunk, bar))
    print(f"\n[mixed vs uniform, mode {mode}, {variant}] finished at checkpoints: {done_total}; max |obs difference| {worst:.2e}")
    assert done_total > 0
    for e in envs:
        e.close()


@pytest.mark.gpu
def test_quadx_waypoints_mixed_equals_uniform_handles():
    import torch

    from pyflyt_b200.gym_envs.quadx_waypoints_env import QuadXWaypointsVecEnv

    n = 16384
    kw = dict(num_envs=n, seed=8, max_duration_seconds=1.0)
    mixed = QuadXWaypointsVecEnv(drone_options=_alternating(n), **kw)
    uniform = [QuadXWaypointsVecEnv(drone_options=CF2X, **kw), QuadXWaypointsVecEnv(drone_options=PRIM, **kw)]
    envs = [mixed] + uniform
    idx = mixed.aviary.model_index
    for e in envs:
        e.reset()
    done_total = 0
    for k in range(70):
        for e in envs:
            e.rollout(1)
        done_total += int((mixed.aviary.term | mixed.aviary.trunc).sum())
        A = mixed.aviary
        for j, U in enumerate(u.aviary for u in uniform):
            m = idx == j
            same = (A.istate_tensor[0] == U.istate_tensor[0]) & m  # same step counter = same reset history
            # the drawn actions (an env reset by a tail CTA draws none on that step)
            assert torch.equal(A.setpoints[same], U.setpoints[same]), k
            if k % 10 == 9:
                assert int((m & ~same).sum()) <= 2, (k, j)
                d = (A.obs.double() - U.obs.double()).abs().amax(dim=1)
                assert float(d[same].max()) < 1e-4, (k, j)
                assert torch.equal(A.term[same], U.term[same]) and torch.equal(A.trunc[same], U.trunc[same])
    assert done_total > n // 4
    for e in envs:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("order", ["wind_then_models", "models_then_wind"])
def test_wind_reaches_every_model(order):
    """An analytic wind registered before or after the models are installed acts on every table of the set: the mixed handle
    matches two uniform handles in the same air."""
    import ctypes as C

    import torch

    from pyflyt_b200 import _lib
    from pyflyt_b200.core.aviary import BatchedAviary
    from pyflyt_b200.core.wind import AnalyticWind
    from pyflyt_b200.models import PfbModel

    n, steps = 2048, 120
    wind = AnalyticWind("power", base=(4.0, -2.0, 0.5), z_ref=10.0, alpha=1.0 / 7.0)
    start = np.column_stack([np.zeros(n), np.zeros(n), np.linspace(5, 15, n)]).astype(np.float32)
    orn = np.zeros((n, 3), dtype=np.float32)
    mixed = BatchedAviary(start, orn, drone_options=_alternating(n), seed=3)
    if order == "wind_then_models":  # re-install the models on a handle that already has the wind
        mixed.register_wind_field(wind)
        tables = (PfbModel * 2)(*mixed.models)
        idx = mixed.model_index.cpu().numpy().astype(np.uint8)
        _lib.check(_lib.lib().pfb_set_models(mixed._h, tables, 2, idx.ctypes.data_as(C.c_void_p)))
    else:
        mixed.register_wind_field(wind)
    uniform = [BatchedAviary(start, orn, drone_options=o, seed=3) for o in (CF2X, PRIM)]
    for u in uniform:
        u.register_wind_field(wind)
    calm = BatchedAviary(start, orn, drone_options=_alternating(n), seed=3)
    avs = [mixed, calm] + uniform
    for a in avs:
        a.reset()
        a.set_mode(7)
        a.set_all_setpoints(torch.as_tensor(np.column_stack([np.zeros((n, 3)), start[:, 2]]), dtype=torch.float32, device="cuda"))
    for _ in range(steps):
        for a in avs:
            a.step(1)
    s = mixed.all_states
    idx = mixed.model_index
    for j, u in enumerate(uniform):
        m = idx == j
        assert float((s[m] - u.all_states[m]).abs().max()) < 1e-5, j
    assert float((s[:, 3, :2] - calm.all_states[:, 3, :2]).abs().max()) > 1e-3  # the wind does push the drones


@pytest.mark.gpu
def test_sequence_with_one_table_is_the_uniform_handle():
    """A per-env sequence that builds one table is bit-identical to today's dict-constructed handle."""
    import torch

    from pyflyt_b200.gym_envs.quadx_hover_env import QuadXHoverVecEnv

    n = 8192
    a = QuadXHoverVecEnv(num_envs=n, seed=4, drone_options=dict(drone_model="primitive_drone"))
    b = QuadXHoverVecEnv(num_envs=n, seed=4, drone_options=[dict(drone_model="primitive_drone")] * (n // 2) + [dict(PRIM)] * (n // 2))
    assert len(b.aviary.models) == 1
    for e in (a, b):
        e.reset()
    for chunk in (1, 8, 1, 16):
        for e in (a, b):
            e.rollout(chunk)
        torch.cuda.synchronize()
        assert torch.equal(a.aviary.obs, b.aviary.obs) and torch.equal(a.aviary.state_tensor, b.aviary.state_tensor)
        assert torch.equal(a.aviary.reward, b.aviary.reward) and torch.equal(a.aviary.term, b.aviary.term)
    a.close()
    b.close()
