"""TrainerTD3 on Pendulum and ContinuousMountainCar: the fused update (wdb_td3_critic_update /
wdb_td3_actor_update + FlatAdam, algorithms/fused_td3.py) against the torch autograd update from
identical trainer state and noise; launches and host synchronisation of critic-only and actor
iterations; the delayed actor and targets; learning on a frozen ring; the fall-back shapes; the
gradient arena; checkpoints; two ranks."""
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
_NETS = ("actor_models", "critic_models", "critic2_models", "target_actor_models",
         "target_critic_models", "target_critic2_models")


def _trainer(tmp_path, config="single_pendulum", E=256, T=8, model=None, policy=None,
             num_devices=1, device_id=0):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent import classic_control as cc
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_td3 import TrainerTD3

    cfg = load_run_config(config)
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, num_episodes=E * 4, seed=11)
    cfg["trainer"]["evaluator"] = False
    cfg["env"].update(episode_length=32, reset_pool_size=64)
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1000,
                         model_params_save_freq=1000)
    pol = cfg["policy"]["shared"]
    pol.update(algorithm="TD3", target_noise=0.2, target_noise_clip=0.5, policy_delay=2)
    for kind in ("actor", "critic"):
        pol["model"][kind].update((model or {}).get(kind, {}))
    pol.update(policy or {})
    env = getattr(cc, _ENVS[config])(**cfg["env"])
    w = EnvWrapper(env, num_envs=E, env_backend="numba")
    return TrainerTD3(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                      results_dir=f"r{device_id}", verbose=False, num_devices=num_devices,
                      device_id=device_id)


def _params(tr):
    return [t.detach().clone() for n in _NETS for t in getattr(tr, n)["shared"].parameters()]


def _state(tr):
    p = "shared"
    return (_params(tr),
            [copy.deepcopy(o.state_dict()) for o in (tr.actor_optimizers[p],
                                                     tr.critic_optimizers[p])],
            dict(tr.current_timestep), dict(tr.update_count),
            tr._noise_generator.get_state())


def _restore(tr, state):
    params, opts, ts, counts, gen = state
    p = "shared"
    with torch.no_grad():
        for t, v in zip([t for n in _NETS for t in getattr(tr, n)[p].parameters()], params):
            t.copy_(v)
    for o, s in zip((tr.actor_optimizers[p], tr.critic_optimizers[p]), opts):
        o.load_state_dict(s)
    tr.current_timestep.update(ts)
    tr.update_count.update(counts)
    tr._noise_generator.set_state(gen)


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _filled(tmp_path, config, **kw):
    tr = _trainer(tmp_path, config, **kw)
    for _ in range(2):                         # fill the ring (capacity T + n_step - 1)
        tr._generate_rollout_batch()
    assert tr.engine.isfull()
    return tr


@pytest.mark.parametrize("config", list(_ENVS))
def test_fused_update_matches_the_torch_update(config, tmp_path):
    tr = _filled(tmp_path, config)
    assert "shared" in tr.fused_updates
    algo = tr.trainers["shared"]
    start = _state(tr)
    results = {}
    for fused in (True, False):
        _restore(tr, start)
        algo.use_fused_update = fused
        m_critic = tr._update_model_params(0)["shared"]        # update 1: critic only
        one = _params(tr)
        m_actor = tr._update_model_params(0)["shared"]         # update 2: critic + actor
        two = _params(tr)
        for it in range(1, 9):
            tr._update_model_params(it)
        results[fused] = (m_critic, m_actor, one, two, _params(tr))
    algo.use_fused_update = True
    f, t = results[True], results[False]
    for k in (2, 3):
        for a, b in zip(f[k], t[k]):
            assert _rel(a, b) <= 1e-5
    for a, b in zip(f[4], t[4]):
        assert torch.isfinite(a).all() and _rel(a, b) <= 1e-3
    for mf, mt in ((f[0], t[0]), (f[1], t[1])):
        assert mf.keys() == mt.keys()
        for k in mt:
            if isinstance(mt[k], float) and not k.startswith("Mean episodic"):
                assert mf[k] == pytest.approx(mt[k], rel=1e-5, abs=1e-5, nan_ok=True), k
    assert "Actor loss" in f[1] and "Actor loss" not in f[0]


@pytest.mark.parametrize("config", list(_ENVS))
def test_iterations_launch_no_sync_delay_the_actor_and_learn(config, tmp_path):
    from warp_drive_b200 import lib as wlib

    # tau = 0 freezes the targets: the returns on a frozen ring stay fixed
    tr = _filled(tmp_path, config, policy={"lr": {"actor": 1e-3, "critic": 1e-3}, "tau": 0.0})
    assert "shared" in tr.fused_updates
    tr._update_model_params(1)                 # warm-up (allocations, kernel attributes)
    tr._update_model_params(1)
    torch.cuda.synchronize()
    actor_opt = tr.actor_optimizers["shared"]
    for expect_actor in (False, True):
        actor = [p.detach().clone() for p in tr.actor_models["shared"].parameters()]
        steps = actor_opt.step_count
        before = wlib.launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            tr._update_model_params(1)         # not a logging iteration
        finally:
            torch.cuda.set_sync_debug_mode(0)
        # critic pass (2) + twin-critic clipping norm and Adam (2); an actor update adds the
        # actor pass (2) and the actor's clipping norm and Adam (2)
        assert wlib.launch_count() - before == (8 if expect_actor else 4)
        assert actor_opt.step_count == steps + int(expect_actor)
        same = all(torch.equal(a, b) for a, b in
                   zip(actor, tr.actor_models["shared"].parameters()))
        assert same != expect_actor
    first = tr._update_model_params(0)["shared"]["Critic loss"]
    for it in range(1, 200):
        tr._update_model_params(it)
    last = tr._update_model_params(0)["shared"]["Critic loss"]
    assert np.isfinite(last) and last < first


def test_targets_move_only_on_actor_updates(tmp_path):
    tr = _filled(tmp_path, "single_pendulum")
    p = "shared"
    targets = (tr.target_actor_models[p], tr.target_critic_models[p],
               tr.target_critic2_models[p])

    def snap():
        return [t.detach().clone() for m in targets for t in m.parameters()]

    for k in range(1, 5):
        before = snap()
        tr._update_model_params(1)
        moved = [not torch.equal(a, b) for a, b in zip(before, snap())]
        assert any(moved) if k % 2 == 0 else not any(moved), k
        assert tr.update_count[p] == k


@pytest.mark.parametrize("model,policy", [
    ({"actor": {"fc_dims": [65, 64]}}, None),
    ({"critic": {"fc_dims": [64, 64, 64]}}, None),
], ids=["width65", "three_hidden_64"])
def test_unsupported_shapes_fall_back_to_torch(model, policy, tmp_path):
    from warp_drive_b200 import lib as wlib

    tr = _trainer(tmp_path, model=model, policy=policy, E=64)
    assert tr.fused_updates == {}
    for _ in range(2):
        tr._generate_rollout_batch()
    # torch gradients + FlatAdam only: clipping norm and Adam of the twin critic on the
    # critic-only update, and of the actor too on the next
    for expect in (2, 4):
        torch.cuda.synchronize()
        before = wlib.launch_count()
        tr._update_model_params(1)
        torch.cuda.synchronize()
        assert wlib.launch_count() - before == expect
    assert all(torch.isfinite(p).all() for p in tr.actor_models["shared"].parameters())


def test_every_grad_is_a_view_into_the_arena(tmp_path):
    tr = _trainer(tmp_path, E=64)
    arena = tr._arena_grads
    lo, hi = arena.data_ptr(), arena.data_ptr() + arena.numel() * 4
    n = 0
    for models in (tr.actor_models, tr.critic_models, tr.critic2_models):
        for p in models["shared"].parameters():
            assert p.grad is not None and lo <= p.grad.data_ptr() < hi
            assert p.grad.data_ptr() + p.grad.numel() * 4 <= hi
            n += 1
    assert n == 18
    twin = tr.critic_optimizers["shared"]
    assert len(twin.param_list) == 12          # one optimizer over both critics
    for _ in range(2):
        tr._generate_rollout_batch()
    tr._update_model_params(1)
    assert twin.grads.abs().sum() > 0


def test_checkpoint_round_trip(tmp_path):
    tr = _filled(tmp_path, "single_pendulum")
    tr._update_model_params(1)
    tr._update_model_params(1)
    tr.save_model_checkpoint(0)
    ts = tr.current_timestep["shared"]
    paths = {k: os.path.join(tr.save_dir, f"shared_{k}_{ts}.state_dict")
             for k in ("actor", "critic", "critic2")}
    assert all(os.path.isfile(v) for v in paths.values())
    saved = {k: [t.detach().clone() for t in getattr(tr, f"{k}_models")["shared"].parameters()]
             for k in ("actor", "critic", "critic2")}
    fresh = _trainer(tmp_path / "b")
    fresh.load_model_checkpoint({"shared": paths})
    assert fresh.current_timestep["shared"] == ts
    for k in ("actor", "critic", "critic2"):
        got = list(getattr(fresh, f"{k}_models")["shared"].parameters())
        assert all(torch.equal(a, b) for a, b in zip(got, saved[k]))
    got = list(fresh.target_critic2_models["shared"].parameters())
    assert all(torch.equal(a, b) for a, b in zip(got, saved["critic2"]))
    # without critic2 the checkpoint loads as a DDPG one: actor and Q1
    other = _trainer(tmp_path / "c")
    other.load_model_checkpoint({"shared": {k: paths[k] for k in ("actor", "critic")}})
    got = list(other.critic_models["shared"].parameters())
    assert all(torch.equal(a, b) for a, b in zip(got, saved["critic"]))


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
    flat = torch.cat([p.detach().reshape(-1) for n in _NETS
                      for p in getattr(tr, n)["shared"].parameters()])
    both = [torch.zeros_like(flat) for _ in range(world)]
    dist.all_gather(both, flat)
    out.put((rank, bool(torch.equal(both[0], both[1])), bool(torch.isfinite(flat).all())))
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_rank_td3_training_keeps_ranks_identical(tmp_path):
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
