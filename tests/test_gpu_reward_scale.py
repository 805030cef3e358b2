"""Running reward scaling on the GPU: wdb_discounted_return_scan against the float32
restatement (tests/reward_scale_reference.py) bit for bit, with its carry in and out, guard
regions and reruns; and Trainer runs with scale_rewards on every rollout path and both update
paths, where the rewards the update receives are the reference's scaled batch bit for bit and
the statistics the float64 reference of every return so far (key off: the raw batch itself),
through checkpoints, train() and evaluation, and on two GPUs."""
import ctypes
import json
import os
import socket

import numpy as np
import pytest
import torch

from obs_norm_reference import shift_scale
from reward_scale_reference import RunningReturns, scale_f32, scan_f32

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
_STATS = ("return_count", "return_mean", "return_m2", "return_shift", "return_scale")


def _lib():
    from warp_drive_b200 import lib as wlib

    return wlib, wlib.load()


def _bits(t):
    return t.reshape(-1).view(torch.int64 if t.dtype == torch.float64 else torch.int32)


def _scan_inputs(T, E, Np, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rewards = torch.randn((T, E, Np), device="cuda", generator=g) * 4 - 2
    u = torch.rand((T, E), device="cuda", generator=g)
    done = (u < 0.15).to(torch.int32) + (u < 0.03).to(torch.int32)      # 0, 1 and 2
    done[0, 0::5] = 1                                                   # done at t = 0
    done[T - 1, 1::5] = 1                                               # at t = T - 1
    if T > 2:
        done[1:3, 2::5] = 2                                             # consecutive steps
    carry = torch.randn((E, Np), device="cuda", generator=g) * 30
    return rewards, done.contiguous(), carry


def _guarded(n, fill=-12345.0):
    """A float32 buffer of n elements inside 64 guard elements on either side."""
    buf = torch.full((n + 128,), fill, device="cuda")
    return buf, buf[64:64 + n]


@pytest.mark.parametrize("T", [1, 7, 250])
@pytest.mark.parametrize("E,Np", [(333, 1), (77, 5), (1001, 3)])
def test_scan_is_the_float32_restatement_bit_for_bit(T, E, Np):
    wlib, L = _lib()
    rewards, done, carry0 = _scan_inputs(T, E, Np, seed=T * 7 + E + Np)
    gamma = 0.95
    want, want_carry = scan_f32(rewards.cpu().numpy(), done.cpu().numpy(), gamma,
                                carry0.cpu().numpy())
    runs = []
    for _ in range(2):                                   # a relaunch gives the same bits
        ret_buf, ret = _guarded(T * E * Np)
        carry_buf, carry = _guarded(E * Np)
        carry.copy_(carry0.reshape(-1))
        wlib.check(L.wdb_discounted_return_scan(
            wlib.stream_ptr(), wlib.ptr(rewards), wlib.ptr(done), T, E, Np,
            ctypes.c_float(gamma), wlib.ptr(carry), wlib.ptr(ret)), "scan")
        torch.cuda.synchronize()
        assert np.array_equal(ret.cpu().numpy().view(np.uint32),
                              want.reshape(-1).view(np.uint32))
        assert np.array_equal(carry.cpu().numpy().view(np.uint32),
                              want_carry.reshape(-1).view(np.uint32))
        for buf in (ret_buf, carry_buf):
            assert torch.all(buf[:64] == -12345.0) and torch.all(buf[-64:] == -12345.0)
        runs.append((ret_buf.clone(), carry_buf.clone()))
    assert torch.equal(_bits(runs[0][0]), _bits(runs[1][0]))
    assert torch.equal(_bits(runs[0][1]), _bits(runs[1][1]))


def test_scan_refuses_bad_shapes_and_pointers():
    wlib, L = _lib()
    r = torch.zeros((2, 3, 1), device="cuda")
    d = torch.zeros((2, 3), dtype=torch.int32, device="cuda")
    c = torch.zeros(3, device="cuda")
    out = torch.zeros_like(r)
    p = [wlib.ptr(r), wlib.ptr(d), wlib.ptr(c), wlib.ptr(out)]
    g = ctypes.c_float(0.9)
    ok = L.wdb_discounted_return_scan(None, p[0], p[1], 2, 3, 1, g, p[2], p[3])
    assert ok == 0
    for k in range(4):
        q = list(p)
        q[k] = None
        assert L.wdb_discounted_return_scan(None, q[0], q[1], 2, 3, 1, g, q[2], q[3]) != 0
    for T, E, Np in ((0, 3, 1), (2, 0, 1), (2, 3, 0), (-1, 3, 1)):
        assert L.wdb_discounted_return_scan(None, p[0], p[1], T, E, Np, g, p[2], p[3]) != 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------ Trainer
def _single_trainer(tmp_path, config, E, T, L, iters, policy_kw, tag, algo=None):
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
    if algo:
        pol["algorithm"] = algo
    pol.update(policy_kw)
    name = {"pendulum": "Pendulum", "mountain_car": "MountainCar", "cartpole": "CartPole"}[
        next(k for k in ("pendulum", "mountain_car", "cartpole") if k in config)]
    env = getattr(cc, f"CUDAClassicControl{name}Env")(**cfg["env"])
    wrapper = EnvWrapper(env, num_envs=E, env_backend="numba")
    return Trainer(env_wrapper=wrapper, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                   results_dir=tag, verbose=False)


def _spy(trainer):
    """Record the rewards tensor each trained policy's update receives."""
    seen = {}
    for p, algo in trainer.trainers.items():
        loss, prep = algo.compute_loss_and_metrics, algo.prepare_batch

        def loss_spy(*a, _p=p, _f=loss, **kw):
            seen[_p] = a[2]
            return _f(*a, **kw)

        def prep_spy(*a, _p=p, _f=prep, **kw):
            seen[_p] = a[3]
            return _f(*a, **kw)

        algo.compute_loss_and_metrics, algo.prepare_batch = loss_spy, prep_spy
    return seen


def _check_stats(model, ref):
    n, mean, m2 = ref.stats
    assert float(model.return_count) == n
    dm, dm2 = model.return_mean.cpu().numpy(), model.return_m2.cpu().numpy()
    assert (np.abs(dm - mean) <= 1e-12 * np.abs(mean) + 1e-300).all(), (dm, mean)
    assert (np.abs(dm2 - m2) <= 1e-12 * np.abs(m2) + 1e-300).all(), (dm2, m2)
    # shift and scale are the float32 of the device's own float64 statistics
    shift, scale = shift_scale(float(model.return_count), dm, dm2)
    assert np.array_equal(model.return_shift.cpu().numpy(), shift)
    assert np.array_equal(model.return_scale.cpu().numpy(), scale)


def _references(trainer):
    out = {}
    for p, scaler in trainer._reward_scalers.items():
        E, Np = scaler.carry.shape
        out[p] = RunningReturns(E, Np, trainer.config["policy"][p]["gamma"], scaler.clip)
    return out


def _iterate_and_check(trainer, refs, n_iters):
    """Run iterations by hand: after each, the rewards the update received are the reference's
    scaled batch bit for bit, the raw batch is untouched, the carry is the reference's and the
    statistics the reference merge of every return so far."""
    dm = trainer.cuda_envs.cuda_data_manager
    seen = _spy(trainer)
    for it in range(n_iters):
        seen.clear()
        trainer._generate_rollout_batch()
        done = dm.data_on_device_via_torch("done_flags_batch").clone()
        raw = {p: dm.data_on_device_via_torch(f"rewards_batch_{p}").clone() for p in refs}
        trainer._update_model_params(it)
        torch.cuda.synchronize()
        assert set(seen) == set(trainer.policies_to_train)
        for p, ref in refs.items():
            model, scaler = trainer.models[p], trainer._reward_scalers[p]
            returns = ref.step(raw[p].cpu().numpy(), done.cpu().numpy())
            assert np.array_equal(scaler.returns.cpu().numpy().view(np.uint32),
                                  returns.view(np.uint32)), (p, it)
            assert np.array_equal(scaler.carry.cpu().numpy().view(np.uint32),
                                  ref.carry.view(np.uint32)), (p, it)
            _check_stats(model, ref)
            want = scale_f32(raw[p].cpu().numpy(), model.return_scale.cpu().numpy(), ref.clip)
            got = seen[p]
            assert got.data_ptr() == scaler.scaled.data_ptr()
            assert np.array_equal(got.cpu().numpy().view(np.uint32), want.view(np.uint32))
            assert torch.equal(dm.data_on_device_via_torch(f"rewards_batch_{p}"), raw[p])


def _check_train_eval_and_checkpoint(trainer, refs):
    """train() starts from a zero carry, evaluation zeroes it and leaves the statistics alone,
    and a checkpoint carries the statistics."""
    carries = []
    orig = trainer._generate_rollout_batch

    def rollout_spy():
        carries.append({p: s.carry.clone() for p, s in trainer._reward_scalers.items()})
        return orig()

    assert any(bool(s.carry.any()) for s in trainer._reward_scalers.values())
    trainer._generate_rollout_batch = rollout_spy
    trainer.train()
    trainer._generate_rollout_batch = orig
    torch.cuda.synchronize()
    assert len(carries) == trainer.num_iters
    assert all(not bool(c.any()) for c in carries[0].values())
    lines = [json.loads(l) for l in open(os.path.join(trainer.save_dir, "results.json"))]
    for rec in lines:
        for p in refs:
            assert np.isfinite(rec[p]["Total loss"]) and rec[p]["Reward scale"] > 0
    model = trainer.models[next(iter(refs))]
    assert lines[-1][next(iter(refs))]["Reward scale"] == float(model.return_scale)
    stats = {p: {k: getattr(trainer.models[p], k).clone() for k in _STATS} for p in refs}
    trainer.evaluate_episodes()
    torch.cuda.synchronize()
    for p, s in trainer._reward_scalers.items():
        assert not bool(s.carry.any())
        for k in _STATS:
            assert torch.equal(getattr(trainer.models[p], k), stats[p][k]), k
    # the checkpoint round trip, in place
    p = next(iter(refs))
    trainer.save_model_checkpoint(0)
    ckpts = [f for f in os.listdir(trainer.save_dir)
             if f.startswith(f"{p}_") and f.endswith(".state_dict")]
    path = os.path.join(trainer.save_dir, max(ckpts, key=trainer._checkpoint_timestep))
    saved = torch.load(path, map_location="cpu")
    ptrs = {k: getattr(model, k).data_ptr() for k in _STATS}
    for k in _STATS:
        assert torch.equal(saved[k], stats[p][k].cpu()), k
    with torch.no_grad():
        for k in _STATS:
            getattr(trainer.models[p], k).fill_(3.0)
    trainer.load_model_checkpoint({p: path})
    for k in _STATS:
        assert torch.equal(getattr(trainer.models[p], k), stats[p][k]), k
        assert getattr(trainer.models[p], k).data_ptr() == ptrs[k], k


def test_one_launch_pendulum_ppo_gae_minibatches(tmp_path):
    trainer = _single_trainer(tmp_path, "single_pendulum_ppo_scaled", E=256, T=16, L=40,
                              iters=3, policy_kw={"num_epochs": 2, "num_mini_batches": 2},
                              tag="ppo")
    assert trainer.engine.sa is not None and trainer._minibatch_steps == 4
    refs = _references(trainer)
    assert refs["shared"].clip == 10.0
    _iterate_and_check(trainer, refs, 3)
    _check_train_eval_and_checkpoint(trainer, refs)


@pytest.mark.parametrize("config", ["single_mountain_car", "single_cartpole"])
def test_one_launch_a2c_single_step(config, tmp_path):
    trainer = _single_trainer(tmp_path, config, E=200, T=12, L=30, iters=3,
                              policy_kw={"scale_rewards": True, "reward_clip": 2.5,
                                         "gamma": 0.99},
                              tag="a2c", algo="A2C")
    assert trainer.engine.sa is not None and trainer._minibatch_steps is None
    refs = _references(trainer)
    _iterate_and_check(trainer, refs, 3)
    _check_train_eval_and_checkpoint(trainer, refs)


def _scaled_policies(cfg, clips):
    pol = cfg["policy"].pop("shared", None)
    if pol is not None:
        cfg["policy"] = {p: json.loads(json.dumps(pol)) for p in clips}
    for p, clip in clips.items():
        cfg["policy"][p].update(scale_rewards=True, reward_clip=clip)
    cfg["policy"][next(iter(clips))]["gamma"] = 0.9


def test_two_policy_generic_path_keeps_per_policy_statistics(tmp_path):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.tag_gridworld import CUDATagGridWorld
    from warp_drive_b200.training.trainer import Trainer, load_run_config

    E, T = 64, 10
    cfg = load_run_config("tag_gridworld")
    cfg["env"].update(grid_length=10, episode_length=40)
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, seed=5, num_episodes=E * 3)
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1, model_params_save_freq=1)
    _scaled_policies(cfg, {"tagger": 10.0, "runner": 1.0})
    env = CUDATagGridWorld(**cfg["env"])
    wrapper = EnvWrapper(env, num_envs=E, env_backend="pycuda")
    pm = {"tagger": sorted(env.taggers), "runner": sorted(env.runners)}
    trainer = Trainer(env_wrapper=wrapper, config=cfg, policy_tag_to_agent_id_map=pm,
                      results_dir="grid", verbose=False)
    assert trainer.engine.sa is None and trainer.engine.fused is None
    refs = _references(trainer)
    _iterate_and_check(trainer, refs, 3)
    for p, ids in pm.items():
        assert refs[p].stats[0] == 3 * T * E * len(ids)
    assert float(trainer.models["tagger"].return_m2) != float(trainer.models["runner"].return_m2)
    _check_train_eval_and_checkpoint(trainer, refs)


def test_fused_tag_continuous_step(tmp_path):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.tag_continuous import TagContinuous
    from warp_drive_b200.training.trainer import Trainer, load_run_config

    cfg = load_run_config("tag_continuous")
    cfg["trainer"].update(num_envs=32, train_batch_size=32 * 25, num_episodes=96, seed=3)
    cfg["env"].update(num_taggers=2, num_runners=10, episode_length=50)
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1, model_params_save_freq=1)
    _scaled_policies(cfg, {"runner": 10.0, "tagger": 3.0})
    env = TagContinuous(**cfg["env"])
    wrapper = EnvWrapper(env, num_envs=32, env_backend="pycuda")
    pm = {"runner": sorted(env.runners), "tagger": sorted(env.taggers)}
    trainer = Trainer(env_wrapper=wrapper, config=cfg, policy_tag_to_agent_id_map=pm,
                      results_dir="t", verbose=False)
    assert trainer.engine.fused is not None            # the single-launch timestep is in use
    refs = _references(trainer)
    _iterate_and_check(trainer, refs, 3)
    _check_train_eval_and_checkpoint(trainer, refs)


def test_key_off_passes_the_raw_batch_and_registers_nothing(tmp_path):
    trainer = _single_trainer(tmp_path, "single_pendulum_ppo_gae", E=128, T=8, L=40, iters=2,
                              policy_kw={"num_epochs": 1, "num_mini_batches": 2}, tag="off")
    assert trainer._reward_scalers == {}
    model = trainer.models["shared"]
    assert not any(k.startswith("return_") for k in model.state_dict())
    dm = trainer.cuda_envs.cuda_data_manager
    seen = _spy(trainer)
    trainer._generate_rollout_batch()
    trainer._update_model_params(0)
    own = dm.data_on_device_via_torch("rewards_batch_shared")
    assert seen["shared"].data_ptr() == own.data_ptr() and seen["shared"].shape == own.shape


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
        p["scale_rewards"] = True
    cfg["saving"].update(basedir=f"/tmp/reward_scale_nccl_{port}", name="n", tag=f"rank{rank}",
                         metrics_log_freq=1000, model_params_save_freq=1000)
    env = TagContinuous(**cfg["env"])
    w = EnvWrapper(env, num_envs=16, env_backend="b200")
    pm = {"runner": sorted(env.runners), "tagger": sorted(env.taggers)}
    tr = Trainer(w, copy.deepcopy(cfg), pm, num_devices=world, device_id=rank, verbose=False)
    same, counted = True, True
    tr._reset_all_envs()
    tr.engine.resync_observations()
    for it in range(tr.num_iters):
        tr._generate_rollout_batch()
        tr._update_model_params(it)
        flat = torch.cat([getattr(tr.models[p], k).double().reshape(-1) for p in tr.policies
                          for k in _STATS])
        both = [torch.zeros_like(flat) for _ in range(world)]
        dist.all_gather(both, flat)
        same = same and bool(torch.equal(both[0].view(torch.int64), both[1].view(torch.int64)))
        counted = counted and float(tr.models["runner"].return_count) == (it + 1) * world * 16 * 5 * 8
    out.put((rank, same, counted))
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
