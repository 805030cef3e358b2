"""Observation normalization on the GPU: the moments update against the float64 Welford / Chan
reference (tests/obs_norm_reference.py) across its shape envelope, successive updates and
bit-identical reruns; wdb_obs_normalize against the float32 restatement bit for bit; the
one-launch rollout's normalizing kinds (raw observations in the batch, the first layer's
input equal to wdb_obs_normalize of them, identity statistics equal to the plain kinds bit for
bit); and Trainer runs with the key on (A2C, PPO, per-policy statistics, checkpoints,
evaluation)."""
import ctypes
import importlib
import json
import os
import socket

import numpy as np
import pytest
import torch

from obs_norm_reference import batch_moments, chan, normalize_f32, shift_scale

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _lib():
    from warp_drive_b200 import lib as wlib

    return wlib, wlib.load()


def _state(F):
    return {"count": torch.zeros((), dtype=torch.float64, device="cuda"),
            "mean": torch.zeros(F, dtype=torch.float64, device="cuda"),
            "m2": torch.zeros(F, dtype=torch.float64, device="cuda"),
            "shift": torch.zeros(F, device="cuda"), "scale": torch.ones(F, device="cuda")}


def _ptrs(wlib, st):
    return [wlib.ptr(st[k]) for k in ("count", "mean", "m2", "shift", "scale")]


def _update(st, x):
    wlib, L = _lib()
    rows, F = x.shape
    scratch = torch.empty(max(1, int(L.wdb_obs_moments_scratch_doubles(rows, F))),
                          dtype=torch.float64, device="cuda")
    wlib.check(L.wdb_obs_moments_update(wlib.stream_ptr(), wlib.ptr(x), rows, F,
                                        wlib.ptr(scratch), *_ptrs(wlib, st)), "update")


def _data(rows, F, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    scale = torch.rand(F, device="cuda", generator=g) * 2 + 0.1
    sign = torch.where(torch.rand(F, device="cuda", generator=g) < 0.5, -1.0, 1.0)
    offset = sign * (torch.rand(F, device="cuda", generator=g) * 3 + 1)
    return torch.randn(rows, F, device="cuda", generator=g) * scale + offset


def _check_state(st, ref):
    n, mean, m2 = ref
    assert float(st["count"]) == n
    dm, dm2 = st["mean"].cpu().numpy(), st["m2"].cpu().numpy()
    assert (np.abs(dm - mean) <= 1e-12 * np.abs(mean)).all(), np.abs(dm - mean).max()
    assert (np.abs(dm2 - m2) <= 1e-12 * np.abs(m2) + 1e-300).all(), np.abs(dm2 - m2).max()
    # shift and scale are the float32 of the device's own float64 statistics
    shift, scale = shift_scale(float(st["count"]), dm, dm2)
    assert np.array_equal(st["shift"].cpu().numpy(), shift)
    assert np.array_equal(st["scale"].cpu().numpy(), scale)


def _bits(t):
    return t.reshape(-1).view(torch.int64 if t.dtype == torch.float64 else torch.int32)


SHAPES = [(r, f) for r in (1, 17, 100_000, 2_100_000) for f in (1, 3, 63, 64, 1024)
          if not (r == 2_100_000 and f == 1024)]     # (8.6 GB of batch; the host reference)


@pytest.mark.parametrize("rows,F", SHAPES)
def test_moments_update_matches_float64_reference(rows, F):
    n_updates = 2 if rows * F > 10**7 else 3
    batches = [_data(rows, F, seed=rows + F + k) for k in range(n_updates)]
    runs = []
    for _ in range(2):                                   # two identical runs
        st = _state(F)
        ref = (0.0, np.zeros(F), np.zeros(F))
        for x in batches:
            _update(st, x)
            torch.cuda.synchronize()
            ref = chan(ref, batch_moments(x.cpu().numpy()))
            _check_state(st, ref)
        runs.append({k: v.clone() for k, v in st.items()})
    for k in runs[0]:
        assert torch.equal(_bits(runs[0][k]), _bits(runs[1][k])), k


def test_no_samples_is_the_identity():
    wlib, L = _lib()
    st = _state(5)
    st["shift"].fill_(7.0)
    st["scale"].fill_(7.0)
    _update(st, torch.empty(0, 5, device="cuda"))
    torch.cuda.synchronize()
    assert float(st["count"]) == 0
    assert torch.equal(st["shift"], torch.zeros(5, device="cuda"))
    assert torch.equal(st["scale"], torch.ones(5, device="cuda"))
    # a merge of records that hold no rows changes nothing either
    rec = torch.zeros((2, 11), dtype=torch.float64, device="cuda")
    wlib.check(L.wdb_obs_moments_merge(wlib.stream_ptr(), wlib.ptr(rec), 2, 5,
                                       *_ptrs(wlib, st)), "merge")
    torch.cuda.synchronize()
    assert float(st["count"]) == 0 and torch.equal(st["scale"], torch.ones(5, device="cuda"))
    # bad shapes and pointers are refused without a launch
    assert L.wdb_obs_moments_update(None, None, 4, 0, None, *_ptrs(wlib, st)) != 0
    assert L.wdb_obs_moments_merge(None, None, 1, 5, *_ptrs(wlib, st)) != 0
    assert L.wdb_obs_normalize(None, None, None, 1, 5, None, None, ctypes.c_float(1.0)) != 0
    x = torch.zeros(2, 5, device="cuda")
    for clip in (0.0, -1.0, float("inf"), float("nan")):
        assert L.wdb_obs_normalize(None, wlib.ptr(x), wlib.ptr(x), 2, 5, wlib.ptr(st["shift"]),
                                   wlib.ptr(st["scale"]), ctypes.c_float(clip)) != 0


def test_rank_records_merged_in_order_match_the_whole_batch():
    """What two GPUs do: each rank's batch record, then the gathered records merged in rank
    order -- within the reference bound of the moments of the concatenated batch, and the same
    bits on a rerun."""
    wlib, L = _lib()
    F = 37
    parts = [_data(50_000, F, seed=1), _data(30_001, F, seed=2)]
    out = []
    for _ in range(2):
        recs = torch.empty((2, 2 * F + 1), dtype=torch.float64, device="cuda")
        for r, x in enumerate(parts):
            scratch = torch.empty(int(L.wdb_obs_moments_scratch_doubles(x.shape[0], F)),
                                  dtype=torch.float64, device="cuda")
            wlib.check(L.wdb_obs_moments_batch(wlib.stream_ptr(), wlib.ptr(x), x.shape[0], F,
                                               wlib.ptr(scratch), wlib.ptr(recs[r])), "batch")
        st = _state(F)
        wlib.check(L.wdb_obs_moments_merge(wlib.stream_ptr(), wlib.ptr(recs), 2, F,
                                           *_ptrs(wlib, st)), "merge")
        torch.cuda.synchronize()
        ref = chan(batch_moments(parts[0].cpu().numpy()), batch_moments(parts[1].cpu().numpy()))
        _check_state(st, ref)
        out.append(st)
    for k in out[0]:
        assert torch.equal(out[0][k], out[1][k]), k


@pytest.mark.parametrize("rows,F", [(1, 1), (17, 3), (4096, 63), (1000, 1024), (100_000, 7)])
def test_normalize_is_the_float32_restatement_bit_for_bit(rows, F):
    wlib, L = _lib()
    g = torch.Generator(device="cuda").manual_seed(rows + F)
    x = torch.randn(rows, F, device="cuda", generator=g) * 10
    x.view(-1)[::7] *= 1e30                              # large magnitudes, clamped
    x.view(-1)[::11] = 0.0
    shift = torch.randn(F, device="cuda", generator=g)
    scale = torch.rand(F, device="cuda", generator=g) * 3
    for clip in (0.5, 5.0, 1e30):
        y = torch.empty_like(x)
        wlib.check(L.wdb_obs_normalize(wlib.stream_ptr(), wlib.ptr(x), wlib.ptr(y), rows, F,
                                       wlib.ptr(shift), wlib.ptr(scale), ctypes.c_float(clip)),
                   "normalize")
        want = normalize_f32(x.cpu().numpy(), shift.cpu().numpy(), scale.cpu().numpy(), clip)
        assert np.array_equal(y.cpu().numpy().view(np.uint32), want.view(np.uint32)), clip


# ------------------------------------------------------------------------ one-launch rollout
ENVS = {"cartpole": ("warp_drive_b200.envs.single_agent.cartpole",
                     "CUDAClassicControlCartPoleEnv", False),
        "mountain_car": ("warp_drive_b200.envs.single_agent.classic_control",
                         "CUDAClassicControlMountainCarEnv", False),
        "acrobot": ("warp_drive_b200.envs.single_agent.classic_control",
                    "CUDAClassicControlAcrobotEnv", False),
        "pendulum": ("warp_drive_b200.envs.single_agent.classic_control",
                     "CUDAClassicControlPendulumEnv", True),
        "continuous_mountain_car": ("warp_drive_b200.envs.single_agent.classic_control",
                                    "CUDAClassicControlContinuousMountainCarEnv", True)}


def _build(name, E, T, fused, model_kw, fc_dims=(32, 32), pool=8, seed=11):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.managers.function_manager import CUDASampler
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.training.rollout import RolloutEngine
    from warp_drive_b200.training.utils.data_loader import create_and_push_data_placeholders

    mod, cls, continuous = ENVS[name]
    env = getattr(importlib.import_module(mod), cls)(
        episode_length=30, env_backend="b200", reset_pool_size=pool, seed=seed)
    w = EnvWrapper(env, num_envs=E, env_backend="b200")
    w.reset_all_envs()
    pm = {"shared": [0]}
    s = CUDASampler(w.cuda_function_manager)
    create_and_push_data_placeholders(env_wrapper=w, action_sampler=s,
                                      policy_tag_to_agent_id_map=pm,
                                      training_batch_size_per_env=T)
    s.init_random(seed)
    if pool >= 2:
        w.init_reset_pool(seed=5)
    torch.manual_seed(0)
    kind = "fully_connected_gaussian" if continuous else "fully_connected"
    cfg = dict({"type": kind, "fc_dims": list(fc_dims), "log_std_init": -0.4}, **model_kw)
    model = ModelFactory.create(kind)(w, cfg, "shared", pm).cuda().eval()
    st = w.cuda_data_manager.data_on_device_via_torch("state")
    g = torch.Generator(device="cuda").manual_seed(3)
    st.add_(0.05 * (torch.rand(st.shape, device="cuda", generator=g) - 0.5))
    eng = RolloutEngine(w, {"shared": model}, pm, s, T, use_cuda_graph=False,
                        use_fused_step=fused)
    return w, eng, s, model


def _set_statistics(model, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    F = model.obs_shift.numel()
    model.obs_shift.copy_(torch.randn(F, device="cuda", generator=g) * 0.5)
    model.obs_scale.copy_(torch.rand(F, device="cuda", generator=g) * 4 + 0.5)


def _hooks(name, T, E, A, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if ENVS[name][2]:
        return {"normals": torch.randn((T, E), device="cuda", generator=g),
                "probs_out": torch.zeros((T, E), device="cuda")}
    return {"uniforms": torch.rand((T, E), device="cuda", generator=g).clamp_min(1e-7),
            "probs_out": torch.zeros((T, E, A), device="cuda")}


def _normalize(model, x):
    from warp_drive_b200.training import obs_norm

    return obs_norm.normalize(model, x.contiguous())


@pytest.mark.parametrize("name", list(ENVS))
def test_normalizing_kind_keeps_raw_observations_and_normalizes_the_input(name):
    """obs_batch[t] is, bit for bit, the observation the env step wrote at t (a generic-path
    replica stepped with the recorded actions); the recorded probabilities / mean equal the
    torch forward of the normalized observation."""
    E, T = 160, 24
    kw = {"normalize_observations": True, "observation_clip": 1.5}
    wa, ea, sa, ma = _build(name, E, T, True, kw)
    wb, eb, sb, mb = _build(name, E, T, False, kw)
    assert ea.sa is not None and ea.sa.normalizing, "the whole-rollout kernel is not in use"
    assert eb.sa is None and not eb.fused_forward
    _set_statistics(ma, 1)
    _set_statistics(mb, 1)
    dma, dmb = wa.cuda_data_manager, wb.cuda_data_manager
    A = int(ma.output_dims[0])
    for it in range(2):
        hooks = _hooks(name, T, E, A, seed=10 + it)
        ea.sa.launch(T, t0=0, record=True, **hooks)
        torch.cuda.synchronize()
        obs_b = dma.data_on_device_via_torch("processed_observations_batch_shared")
        act_b = dma.data_on_device_via_torch("sampled_actions_batch_shared")
        for t in range(T):
            obs = dmb.data_on_device_via_torch("observations")
            assert torch.equal(obs, obs_b[t]), (it, t)
            with torch.no_grad():
                want = mb(obs)[0][0]
            got = hooks["probs_out"][t]
            assert torch.allclose(want.reshape(got.shape), got, atol=2e-6, rtol=1e-5), (it, t)
            dmb.data_on_device_via_torch("sampled_actions").view(E).copy_(act_b[t].view(E))
            wb.step_all_envs()
            eb.bookkeep(t)
            wb.reset_only_done_envs()
        # clamped inputs occurred
        assert (_normalize(ma, obs_b.view(-1, obs_b.shape[-1])).abs() == 1.5).any()
        for k in ("state", "observations", "_timestep_", "_done_", "rewards"):
            assert torch.equal(dma.data_on_device_via_torch(k), dmb.data_on_device_via_torch(k)), k


@pytest.mark.parametrize("name", ["pendulum", "continuous_mountain_car"])
def test_first_layer_input_is_wdb_obs_normalize_bit_for_bit(name):
    """A Gaussian policy whose mean is exactly its normalized input feature i (hidden layer
    [relu(x), relu(-x)], head e_i - e_{F+i}, zero biases): the recorded mean equals
    wdb_obs_normalize of the batch's raw row, bit for bit."""
    E, T = 96, 20
    w, eng, s, m = _build(name, E, T, True, {"normalize_observations": True,
                                             "observation_clip": 2.0},
                          fc_dims=(2 * ENVS_F[name],))
    F = ENVS_F[name]
    _set_statistics(m, 2)
    with torch.no_grad():
        l1 = m.fc["0"][0]
        l1.weight.copy_(torch.cat([torch.eye(F), -torch.eye(F)]).cuda())
        l1.bias.zero_()
        m.policy_head.bias.zero_()
    obs_b = w.cuda_data_manager.data_on_device_via_torch("processed_observations_batch_shared")
    for i in range(F):
        with torch.no_grad():
            head = torch.zeros(1, 2 * F)
            head[0, i], head[0, F + i] = 1.0, -1.0
            m.policy_head.weight.copy_(head.cuda())
        hooks = _hooks(name, T, E, 1, seed=20 + i)
        eng.sa.launch(T, t0=0, record=True, **hooks)
        torch.cuda.synchronize()
        want = _normalize(m, obs_b.reshape(-1, F))[:, i].view(T, E)
        assert torch.equal(hooks["probs_out"], want), i


ENVS_F = {"cartpole": 4, "mountain_car": 2, "acrobot": 6, "pendulum": 3,
          "continuous_mountain_car": 2}


@pytest.mark.parametrize("name", ["mountain_car", "acrobot", "pendulum"])
def test_identity_statistics_give_the_plain_kind_bit_for_bit(name):
    """No samples yet (shift 0, scale 1) and a clip no input reaches: the normalizing kind
    records exactly what the plain kind, which runs without the key, records."""
    E, T = 160, 24
    wa, ea, _, ma = _build(name, E, T, True, {"normalize_observations": True,
                                              "observation_clip": 1e30})
    wb, eb, _, mb = _build(name, E, T, True, {})
    assert ea.sa.normalizing and not eb.sa.normalizing
    for pa, pb in zip(ma.parameters(), mb.parameters()):
        assert torch.equal(pa, pb)
    A = int(ma.output_dims[0])
    for it in range(2):
        ha, hb = _hooks(name, T, E, A, 30 + it), _hooks(name, T, E, A, 30 + it)
        ea.sa.launch(T, t0=0, record=True, **ha)
        eb.sa.launch(T, t0=0, record=True, **hb)
        torch.cuda.synchronize()
        assert torch.equal(ha["probs_out"], hb["probs_out"])
        for k in ("processed_observations_batch_shared", "sampled_actions_batch_shared",
                  "rewards_batch_shared", "done_flags_batch", "state", "observations"):
            assert torch.equal(wa.cuda_data_manager.data_on_device_via_torch(k),
                               wb.cuda_data_manager.data_on_device_via_torch(k)), k


# ------------------------------------------------------------------------ Trainer
def _single_trainer(tmp_path, config, algo, E, T, L, iters, ppo_epochs=False):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent import classic_control as cc
    from warp_drive_b200.training.trainer import Trainer, load_run_config

    cfg = load_run_config(config)
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, num_episodes=E * T * iters // L,
                          seed=7)
    cfg["trainer"].pop("neg_pos_env_ratio", None)
    cfg["env"].update(episode_length=L, reset_pool_size=64)
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1, model_params_save_freq=1)
    pol = cfg["policy"]["shared"]
    pol["algorithm"] = algo
    if algo == "PPO":
        pol.setdefault("clip_param", 0.2)
    if ppo_epochs:
        pol.update(num_epochs=2, num_mini_batches=4, gae_lambda=0.95)
    pol["model"]["normalize_observations"] = True
    name = "Pendulum" if "pendulum" in config else "MountainCar"
    env = getattr(cc, f"CUDAClassicControl{name}Env")(**cfg["env"])
    wrapper = EnvWrapper(env, num_envs=E, env_backend="numba")
    return Trainer(env_wrapper=wrapper, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                   results_dir=algo, verbose=False)


def _stats(model):
    return {k: getattr(model, k).detach().clone()
            for k in ("obs_count", "obs_mean", "obs_m2", "obs_shift", "obs_scale")}


def _iterate_and_check(trainer, n_iters):
    """Run iterations by hand: after each, the statistics are the reference merge of that
    rollout's raw batch into the previous ones; the rollout saw the previous ones."""
    dm = trainer.cuda_envs.cuda_data_manager
    refs = {p: (0.0, np.zeros(m.obs_mean.numel()), np.zeros(m.obs_mean.numel()))
            for p, m in trainer.models.items()}
    for it in range(n_iters):
        before = {p: _stats(m) for p, m in trainer.models.items()}
        trainer._generate_rollout_batch()
        batches = {p: dm.data_on_device_via_torch(
            f"processed_observations_batch_{p}").clone() for p in trainer.models}
        trainer._update_model_params(it)
        torch.cuda.synchronize()
        for p, m in trainer.models.items():
            x = batches[p].cpu().numpy().reshape(-1, m.obs_mean.numel())
            refs[p] = chan(refs[p], batch_moments(x))
            st = {"count": m.obs_count, "mean": m.obs_mean, "m2": m.obs_m2,
                  "shift": m.obs_shift, "scale": m.obs_scale}
            _check_state(st, refs[p])
            # the batch is the raw observations: never all inside the clip's identity
            assert float(m.obs_count) == float(before[p]["obs_count"]) + x.shape[0]
    return refs


@pytest.mark.parametrize("config,algo,epochs", [("single_mountain_car_obs_norm", "A2C", False),
                                                ("single_pendulum_ppo", "PPO", True)])
def test_trainer_updates_the_statistics_after_each_iteration(config, algo, epochs, tmp_path):
    trainer = _single_trainer(tmp_path, config, algo, E=256, T=16, L=32, iters=3,
                              ppo_epochs=epochs)
    assert trainer.engine.sa is not None and trainer.engine.sa.normalizing
    model = trainer.models["shared"]
    assert float(model.obs_count) == 0
    _iterate_and_check(trainer, 3)
    assert all(torch.isfinite(p).all() for p in model.parameters())
    # evaluation leaves the statistics alone
    before = _stats(model)
    trainer.evaluate_episodes()
    torch.cuda.synchronize()
    for k, v in _stats(model).items():
        assert torch.equal(v, before[k]), k
    # a checkpoint carries them
    trainer.save_model_checkpoint(0)
    ckpts = [p for p in os.listdir(trainer.save_dir) if p.endswith(".state_dict")]
    path = os.path.join(trainer.save_dir, max(ckpts, key=trainer._checkpoint_timestep))
    saved = torch.load(path, map_location="cpu")
    for k, v in before.items():
        assert torch.equal(saved[k], v.cpu()), k
    ptrs = {k: getattr(model, k).data_ptr() for k in before}
    with torch.no_grad():
        for k in before:
            getattr(model, k).fill_(3.0)
    trainer.load_model_checkpoint({"shared": path})
    for k, v in before.items():
        assert torch.equal(getattr(model, k), v), k
        assert getattr(model, k).data_ptr() == ptrs[k], k      # restored in place
    trainer.train()
    lines = [json.loads(l) for l in open(os.path.join(trainer.save_dir, "results.json"))]
    assert all(np.isfinite(rec["shared"]["Total loss"]) for rec in lines)


def test_multi_policy_generic_path_keeps_per_policy_statistics(tmp_path):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.tag_gridworld import CUDATagGridWorld
    from warp_drive_b200.training.trainer import Trainer, load_run_config

    E, T = 64, 10
    cfg = load_run_config("tag_gridworld")
    cfg["env"].update(grid_length=10, episode_length=40)
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, seed=5, num_episodes=E * 3)
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1, model_params_save_freq=100)
    pol = cfg["policy"].pop("shared")
    pol["model"].update(normalize_observations=True, observation_clip=5.0)
    cfg["policy"] = {p: json.loads(json.dumps(pol)) for p in ("tagger", "runner")}
    env = CUDATagGridWorld(**cfg["env"])
    wrapper = EnvWrapper(env, num_envs=E, env_backend="pycuda")
    pm = {"tagger": sorted(env.taggers), "runner": sorted(env.runners)}
    trainer = Trainer(env_wrapper=wrapper, config=cfg, policy_tag_to_agent_id_map=pm,
                      results_dir="grid", verbose=False)
    assert trainer.engine.sa is None and trainer.engine.fused is None
    assert not trainer.engine.fused_forward
    refs = _iterate_and_check(trainer, 2)
    for p, ids in pm.items():
        assert refs[p][0] == 2 * T * E * len(ids)
    a, b = (trainer.models[p].obs_mean for p in pm)
    assert not torch.equal(a, b)


# ------------------------------------------------------------------------ two GPUs
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import copy

    import torch.distributed as dist
    import yaml

    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.tag_continuous import TagContinuous
    from warp_drive_b200.training.trainer import Trainer
    from warp_drive_b200.training.utils.distributed import init_process_group

    torch.cuda.set_device(rank)
    init_process_group("nccl", device_id=rank)
    root = os.path.dirname(HERE)
    with open(os.path.join(root, "warp_drive_b200", "training", "run_configs",
                           "tag_continuous.yaml"), encoding="utf8") as fp:
        cfg = yaml.safe_load(fp)
    cfg["env"].update(num_taggers=2, num_runners=8, episode_length=20)
    cfg["trainer"].update(num_envs=16, train_batch_size=16 * 5, num_episodes=4, seed=7)
    for p in cfg["policy"].values():
        p["model"].update(fc_dims=[32, 32], normalize_observations=True)
    cfg["saving"].update(basedir=f"/tmp/obs_norm_nccl_{port}", name="n", tag=f"rank{rank}",
                         metrics_log_freq=1000, model_params_save_freq=1000)
    env = TagContinuous(**cfg["env"])
    w = EnvWrapper(env, num_envs=16, env_backend="b200")
    pm = {"runner": sorted(env.runners), "tagger": sorted(env.taggers)}
    tr = Trainer(w, copy.deepcopy(cfg), pm, num_devices=world, device_id=rank, verbose=False)
    same, moved = True, True
    w.reset_all_envs()
    tr.engine.resync_observations()
    for it in range(tr.num_iters):
        tr._generate_rollout_batch()
        tr._update_model_params(it)
        flat = torch.cat([getattr(tr.models[p], k).double().reshape(-1) for p in tr.policies
                          for k in ("obs_count", "obs_mean", "obs_m2", "obs_shift",
                                    "obs_scale")])
        both = [torch.zeros_like(flat) for _ in range(world)]
        dist.all_gather(both, flat)
        same = same and bool(torch.equal(both[0].view(torch.int64), both[1].view(torch.int64)))
        moved = moved and float(tr.models["runner"].obs_count) == (it + 1) * world * 16 * 5 * 8
    out.put((rank, same, moved))
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_hold_bit_identical_statistics():
    import torch.multiprocessing as mp

    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, out)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(out.get(timeout=600) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert all(r[1] for r in res), "the ranks' statistics differ"
    assert all(r[2] for r in res), "the statistics did not count both ranks' rows"
