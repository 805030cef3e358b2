"""TrainerDDPG's fused update (wdb_ddpg_update + FlatAdam, algorithms/fused_ddpg.py) against
its torch autograd update from identical trainer state; path selection, launches and host
synchronisation of a fused iteration; the fall-back shapes; the gradient arena; two ranks."""
import copy
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

_ENVS = {"single_pendulum": "CUDAClassicControlPendulumEnv",
         "single_continuous_mountain_car": "CUDAClassicControlContinuousMountainCarEnv"}


def _trainer(tmp_path, config="single_pendulum", E=256, T=8, model=None, policy=None,
             num_devices=1, device_id=0):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent import classic_control as cc
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_ddpg import TrainerDDPG

    cfg = load_run_config(config)
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, num_episodes=E * 4, seed=11)
    cfg["trainer"]["evaluator"] = False
    cfg["env"].update(episode_length=32, reset_pool_size=64)
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1000,
                         model_params_save_freq=1000)
    pol = cfg["policy"]["shared"]
    for kind in ("actor", "critic"):
        pol["model"][kind].update((model or {}).get(kind, {}))
    pol.update(policy or {})
    env = getattr(cc, _ENVS[config])(**cfg["env"])
    w = EnvWrapper(env, num_envs=E, env_backend="numba")
    return TrainerDDPG(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                       results_dir=f"r{device_id}", verbose=False, num_devices=num_devices,
                       device_id=device_id)


def _state(tr):
    p = "shared"
    nets = (tr.actor_models[p], tr.critic_models[p], tr.target_actor_models[p],
            tr.target_critic_models[p])
    return ([t.detach().clone() for m in nets for t in m.parameters()],
            [copy.deepcopy(o.state_dict()) for o in (tr.actor_optimizers[p],
                                                     tr.critic_optimizers[p])],
            dict(tr.current_timestep))


def _restore(tr, state):
    params, opts, ts = state
    p = "shared"
    nets = (tr.actor_models[p], tr.critic_models[p], tr.target_actor_models[p],
            tr.target_critic_models[p])
    with torch.no_grad():
        for t, v in zip([t for m in nets for t in m.parameters()], params):
            t.copy_(v)
    for o, s in zip((tr.actor_optimizers[p], tr.critic_optimizers[p]), opts):
        o.load_state_dict(s)
    tr.current_timestep.update(ts)


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def test_fused_update_matches_the_torch_update(tmp_path):
    tr = _trainer(tmp_path)
    assert "shared" in tr.fused_updates
    algo = tr.trainers["shared"]
    for _ in range(2):                         # fill the ring (capacity T + n_step - 1)
        tr._generate_rollout_batch()
    assert tr.engine.isfull()
    start = _state(tr)
    results = {}
    for fused in (True, False):
        _restore(tr, start)
        algo.use_fused_update = fused
        metrics = tr._update_model_params(0)["shared"]        # a logging iteration
        one = _state(tr)[0]
        for it in range(1, 10):
            tr._update_model_params(it)
        results[fused] = (metrics, one, _state(tr)[0])
    algo.use_fused_update = True
    (m_f, one_f, ten_f), (m_t, one_t, ten_t) = results[True], results[False]
    for a, b in zip(one_f, one_t):
        assert _rel(a, b) <= 1e-5
    for a, b in zip(ten_f, ten_t):
        assert torch.isfinite(a).all() and _rel(a, b) <= 1e-3
    assert m_f.keys() == m_t.keys()
    for k in m_t:
        # the episodic sums restart after the first run's logging iteration
        if isinstance(m_t[k], float) and not k.startswith("Mean episodic"):
            assert m_f[k] == pytest.approx(m_t[k], rel=1e-5, abs=1e-5, nan_ok=True), k


@pytest.mark.parametrize("config", list(_ENVS))
def test_fused_iteration_launches_no_sync_and_learns(config, tmp_path):
    from warp_drive_b200 import lib as wlib

    # tau = 0 freezes the targets: the returns on a frozen ring stay fixed
    tr = _trainer(tmp_path, config, policy={"lr": {"actor": 1e-3, "critic": 1e-3}, "tau": 0.0})
    assert "shared" in tr.fused_updates
    for _ in range(2):
        tr._generate_rollout_batch()
    tr._update_model_params(1)                 # warm-up (allocations, kernel attributes)
    torch.cuda.synchronize()
    before = wlib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        tr._update_model_params(1)             # not a logging iteration
    finally:
        torch.cuda.set_sync_debug_mode(0)
    # wdb_ddpg_update (2) + per network clipping norm and Adam (2 x 2)
    assert wlib.launch_count() - before == 6
    # a frozen ring: the update descends actor loss + critic loss (the critic's gradient is
    # that of both, as in the reference; alone, the critic loss can rise when the rewards are
    # small, as ContinuousMountainCar's are)
    first = tr._update_model_params(0)["shared"]["Total loss"]
    for it in range(1, 200):
        tr._update_model_params(it)
    last = tr._update_model_params(0)["shared"]["Total loss"]
    assert np.isfinite(last) and last < first


@pytest.mark.parametrize("model,policy", [
    ({"actor": {"fc_dims": [65, 64]}}, None),
    ({"critic": {"fc_dims": [8, 8, 8, 8]}}, None),
    (None, {"normalize_return": True}),
], ids=["width65", "four_hidden", "normalize_return"])
def test_unsupported_shapes_fall_back_to_torch(model, policy, tmp_path):
    from warp_drive_b200 import lib as wlib

    tr = _trainer(tmp_path, model=model, policy=policy, E=64)
    assert tr.fused_updates == {}
    for _ in range(2):
        tr._generate_rollout_batch()
    torch.cuda.synchronize()
    before = wlib.launch_count()
    tr._update_model_params(1)
    torch.cuda.synchronize()
    # torch update + FlatAdam only: clipping norm and Adam for each network
    assert wlib.launch_count() - before == 4
    assert all(torch.isfinite(p).all() for p in tr.actor_models["shared"].parameters())


def test_dict_observation_with_action_mask_is_not_fused(tmp_path):
    from warp_drive_b200.training.algorithms.fused_ddpg import fused_ddpg_supported
    from warp_drive_b200.utils import spaces

    tr = _trainer(tmp_path, E=64)
    actor = copy.deepcopy(tr.actor_models["shared"])
    critic = tr.critic_models["shared"]
    args = (tr.trainers["shared"], actor, critic, 64, 1, tr.ring_capacity, tr.n_step)
    assert fused_ddpg_supported(*args)
    actor.observation_space = spaces.Dict({"obs": actor.observation_space})
    actor.action_mask = torch.ones(64, 1, 1, device="cuda")
    assert not fused_ddpg_supported(*args)


def test_every_grad_is_a_view_into_the_arena(tmp_path):
    tr = _trainer(tmp_path, E=64)
    arena = tr._arena_grads
    lo, hi = arena.data_ptr(), arena.data_ptr() + arena.numel() * 4
    n = 0
    for models in (tr.actor_models, tr.critic_models):
        for p in models["shared"].parameters():
            assert p.grad is not None and lo <= p.grad.data_ptr() < hi
            assert p.grad.data_ptr() + p.grad.numel() * 4 <= hi
            n += 1
    assert n == 12
    for _ in range(2):
        tr._generate_rollout_batch()
    tr._update_model_params(1)
    assert arena.abs().sum() > 0


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, basedir, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import torch.distributed as dist

    from warp_drive_b200.training.utils.distributed import init_process_group

    torch.cuda.set_device(rank)
    init_process_group("nccl", device_id=rank)
    tr = _trainer(basedir, E=64, num_devices=world, device_id=rank)
    tr.train()
    flat = torch.cat([p.detach().reshape(-1) for m in (tr.actor_models, tr.critic_models,
                                                       tr.target_actor_models,
                                                       tr.target_critic_models)
                      for p in m["shared"].parameters()])
    both = [torch.zeros_like(flat) for _ in range(world)]
    dist.all_gather(both, flat)
    out.put((rank, bool(torch.equal(both[0], both[1])), bool(torch.isfinite(flat).all())))
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_rank_ddpg_training_keeps_ranks_identical(tmp_path):
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, str(tmp_path), out))
             for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(out.get(timeout=600) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert all(r[1] and r[2] for r in res)
