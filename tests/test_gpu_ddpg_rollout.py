"""GPU tests of the whole-rollout kernel for the continuous-action single-agent envs
(wdb_single_agent_rollout with WDB_SA_CONTINUOUS_MOUNTAIN_CAR / WDB_SA_PENDULUM: the DDPG
rollout of single_continuous_mountain_car.yaml / single_pendulum.yaml).

The one-launch rollout must record exactly what the separate calls of the generic path
produce when they are teacher-forced with its mean and its normals: the stand-alone OU sampler
(wdb_sample_ou_process), the stand-alone step kernels (pinned bit for bit to the reference's
numba binaries in test_gpu_classic_control.py), the generic bookkeeping and the reset kernel.
The in-kernel float32 actor forward is checked against the torch module at 1e-5.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

ENVS = {"pendulum": "CUDAClassicControlPendulumEnv",
        "continuous_mountain_car": "CUDAClassicControlContinuousMountainCarEnv"}
OU = {"damping": 0.3, "stddev": 0.5, "scale": 0.8}


def _build(name, E, T, pool, fused, fc_dims=(32, 32), episode_length=30, seed=11, ring=None):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent import classic_control as cc
    from warp_drive_b200.managers.function_manager import CUDASampler
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.training.models.fully_connected_actor_critic import ActorAsPolicy
    from warp_drive_b200.training.rollout import RolloutEngine
    from warp_drive_b200.training.trainer_ddpg import RingRolloutEngine
    from warp_drive_b200.training.utils.data_loader import create_and_push_data_placeholders

    env = getattr(cc, ENVS[name])(
        episode_length=episode_length, env_backend="b200", reset_pool_size=pool, seed=seed)
    w = EnvWrapper(env, num_envs=E, env_backend="b200")
    w.reset_all_envs()
    pm = {"shared": [0]}
    s = CUDASampler(w.cuda_function_manager)
    create_and_push_data_placeholders(env_wrapper=w, action_sampler=s,
                                      policy_tag_to_agent_id_map=pm,
                                      training_batch_size_per_env=ring or T)
    s.init_random(seed)
    if pool >= 2:
        w.init_reset_pool(seed=5)
    torch.manual_seed(0)
    cfg = {"type": "fully_connected_actor", "fc_dims": list(fc_dims), "output_w": 2.0,
           "output_b": 0.25}
    actor = ModelFactory.create("fully_connected_actor")(w, cfg, "shared", pm).cuda().eval()
    models = {"shared": ActorAsPolicy(actor)}
    # spread the initial states so that different replicas take different branches
    st = w.cuda_data_manager.data_on_device_via_torch("state")
    g = torch.Generator(device="cuda").manual_seed(3)
    st.add_(0.05 * (torch.rand(st.shape, device="cuda", generator=g) - 0.5))
    if ring is None:
        eng = RolloutEngine(w, models, pm, s, T, use_cuda_graph=False, use_fused_step=fused)
    else:
        eng = RingRolloutEngine(w, models, pm, s, T, ring_capacity=ring)
    return w, eng, s, actor


@pytest.mark.parametrize("name", ["pendulum", "continuous_mountain_car"])
@pytest.mark.parametrize("pool", [0, 8])
def test_one_launch_ddpg_rollout_equals_separate_calls(name, pool):
    E, T = 192, 24
    wa, ea, sa, ma = _build(name, E, T, pool, fused=True)
    wb, eb, sb, mb = _build(name, E, T, pool, fused=False)
    assert ea.sa is not None and ea.sa.continuous, "the whole-rollout kernel is not in use"
    assert eb.sa is None and eb.fused is None
    dma, dmb = wa.cuda_data_manager, wb.cuda_data_manager
    g = torch.Generator(device="cuda").manual_seed(9)
    n_done = 0
    for it in range(4):                      # 96 steps > 3 episodes of 30 steps
        normals = torch.randn((T, E), device="cuda", generator=g)
        mean = torch.zeros((T, E), device="cuda")
        ea.sa.launch(T, t0=0, record=True, normals=normals, probs_out=mean, **OU)
        torch.cuda.synchronize()
        obs_b = dma.data_on_device_via_torch("processed_observations_batch_shared")
        act_b = dma.data_on_device_via_torch("sampled_actions_batch_shared")
        rew_b = dma.data_on_device_via_torch("rewards_batch_shared")
        done_b = dma.data_on_device_via_torch("done_flags_batch")
        for t in range(T):
            # the env B is in exactly the state A recorded
            obs = dmb.data_on_device_via_torch("observations")
            assert torch.equal(obs, obs_b[t]), (it, t)
            with torch.no_grad():
                want = mb(obs)[0]
            assert torch.allclose(want.view(E), mean[t], atol=1e-5, rtol=1e-5), (it, t)
            # the stand-alone OU sampler on A's mean and normals draws A's actions
            sb.sample(dmb, mean[t].view(E, 1, 1).contiguous(), "sampled_actions",
                      normals=normals[t].contiguous(), **OU)
            assert torch.equal(dmb.data_on_device_via_torch("sampled_actions"), act_b[t]), (it, t)
            wb.step_all_envs()
            eb.bookkeep(t)
            assert torch.equal(dmb.data_on_device_via_torch("rewards_batch_shared")[t], rew_b[t])
            assert torch.equal(dmb.data_on_device_via_torch("done_flags_batch")[t], done_b[t])
            n_done += int((done_b[t] > 0).sum())
            wb.reset_only_done_envs()
        for k in ("state", "observations", "_timestep_", "_done_", "rewards",
                  "sampled_actions", "sampled_actions_ou_state"):
            assert torch.equal(dma.data_on_device_via_torch(k), dmb.data_on_device_via_torch(k)), k
    assert n_done >= 2 * E
    assert int(ea.num_completed_episodes) == int(eb.num_completed_episodes) == n_done
    assert int(ea.episodic_step_sum) == int(eb.episodic_step_sum)
    ra, rb = float(ea.episodic_reward_sum["shared"]), float(eb.episodic_reward_sum["shared"])
    assert abs(ra - rb) <= 1e-3 * max(1.0, abs(rb))
    assert torch.equal(ea.step_running_sum, eb.step_running_sum)


def test_device_rng_matches_the_ou_sampler_stream():
    """Without injected normals the kernel draws from the sampler's Philox streams exactly like
    wdb_sample_ou_process (stream = env, one draw per timestep); with scale = 0 it draws nothing
    and leaves the OU state alone."""
    E, T = 64, 8
    wa, ea, sa, ma = _build("pendulum", E, T, 0, fused=True)
    wb, eb, sb, mb = _build("pendulum", E, T, 0, fused=False)
    dma, dmb = wa.cuda_data_manager, wb.cuda_data_manager
    mean = torch.zeros((T, E), device="cuda")
    ea.sa.launch(T, t0=0, record=True, probs_out=mean, **OU)
    act_b = dma.data_on_device_via_torch("sampled_actions_batch_shared")
    for t in range(T):
        sb.sample(dmb, mean[t].view(E, 1, 1).contiguous(), "sampled_actions", **OU)
        assert torch.equal(dmb.data_on_device_via_torch("sampled_actions"), act_b[t]), t
    assert torch.equal(sa.rng_state, sb.rng_state)           # same final stream offsets
    ou = dma.data_on_device_via_torch("sampled_actions_ou_state")
    assert torch.equal(ou, dmb.data_on_device_via_torch("sampled_actions_ou_state"))
    assert float(ou.abs().max()) > 0

    rng0, ou0 = sa.rng_state.clone(), ou.clone()
    ea.sa.launch(T, t0=0, record=True, probs_out=mean, damping=0.3, stddev=0.5, scale=0.0)
    torch.cuda.synchronize()
    assert torch.equal(sa.rng_state, rng0)
    assert torch.equal(ou, ou0)
    assert torch.equal(act_b.view(T, E), mean)               # the mean itself, no noise


def test_ring_rollouts_land_in_the_ring_slots():
    """A RingRolloutEngine (capacity T + 4) writes each rollout at slots cursor .. cursor + T - 1
    (mod capacity) with at most two launches: its time-ordered window equals the last
    `capacity` timesteps of a plain engine that ran the same steps from the same seeds."""
    from warp_drive_b200 import lib as wlib

    E, T, n_roll = 96, 5, 4
    cap = T + 4
    wr, er, sr, mr = _build("continuous_mountain_car", E, T, 8, fused=True, ring=cap)
    wp, ep, sp, mp = _build("continuous_mountain_car", E, T * n_roll, 8, fused=True)
    assert er.sa is not None and ep.sa is not None
    launches = []
    for _ in range(n_roll):
        cursor = er.ring_cursor
        torch.cuda.synchronize()
        c0 = wlib.launch_count()
        er.rollout(**OU)
        launches.append(wlib.launch_count() - c0)
        assert launches[-1] == (1 if cursor + T <= cap else 2), (cursor, launches)
    assert 2 in launches and 1 in launches
    ep.rollout(**OU)
    torch.cuda.synchronize()
    assert er.isfull()
    for name in ("processed_observations_batch_shared", "sampled_actions_batch_shared",
                 "rewards_batch_shared", "done_flags_batch"):
        full = wp.cuda_data_manager.data_on_device_via_torch(name)
        assert torch.equal(er.unroll(name), full[-cap:]), name
    for k in ("state", "observations", "_timestep_", "_done_", "sampled_actions_ou_state"):
        assert torch.equal(wr.cuda_data_manager.data_on_device_via_torch(k),
                           wp.cuda_data_manager.data_on_device_via_torch(k)), k
    # a single ring step goes to the mapped slot, not to slot t
    dm = wr.cuda_data_manager
    slot = er._slot(0)
    assert slot != 0
    obs_b = dm.data_on_device_via_torch("processed_observations_batch_shared")
    obs0, slot0 = dm.data_on_device_via_torch("observations").clone(), obs_b[0].clone()
    c0 = wlib.launch_count()
    er.step(0, **OU)
    torch.cuda.synchronize()
    assert wlib.launch_count() == c0 + 1
    assert torch.equal(obs_b[slot], obs0) and torch.equal(obs_b[0], slot0)


@pytest.mark.parametrize("config,cls", [
    ("single_pendulum", "CUDAClassicControlPendulumEnv"),
    ("single_continuous_mountain_car", "CUDAClassicControlContinuousMountainCarEnv")])
def test_reference_configs_select_the_one_launch_rollout(config, cls, tmp_path):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent import classic_control as cc
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_ddpg import TrainerDDPG

    def trainer(fc_dims=None):
        E, T = 128, 5
        cfg = load_run_config(config)
        cfg["trainer"].update(num_envs=E, train_batch_size=E * T, num_episodes=E)
        cfg["env"].update(episode_length=20, reset_pool_size=64)
        cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1, model_params_save_freq=100)
        if fc_dims is not None:
            cfg["policy"]["shared"]["model"]["actor"]["fc_dims"] = fc_dims
        w = EnvWrapper(getattr(cc, cls)(**cfg["env"]), num_envs=E, env_backend="numba")
        return w, TrainerDDPG(env_wrapper=w, config=cfg,
                              policy_tag_to_agent_id_map={"shared": [0]}, results_dir="r",
                              verbose=False)

    w, tr = trainer()
    assert tr.engine.sa is not None and tr.engine.sa.continuous
    tr.train()
    # the generic evaluation path still works after fused rollouts (same state arrays)
    reward_sum, step_sum = tr.evaluate_episodes(scale=0)
    assert torch.isfinite(reward_sum["shared"]).all()
    assert int(step_sum["shared"].min()) >= 1 and int(step_sum["shared"].max()) <= 20
    # an actor too wide for the per-env forward keeps the generic path and still trains
    w, tr = trainer(fc_dims=[256, 256])
    assert tr.engine.sa is None
    tr.train()
    acts = w.cuda_data_manager.data_on_device_via_torch("sampled_actions_batch_shared")
    assert torch.isfinite(acts).all()


def test_discrete_engines_are_unaffected():
    import importlib

    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.managers.function_manager import CUDASampler
    from warp_drive_b200.training.models.fully_connected import FullyConnected
    from warp_drive_b200.training.rollout import RolloutEngine
    from warp_drive_b200.training.utils.data_loader import create_and_push_data_placeholders

    env = importlib.import_module("warp_drive_b200.envs.single_agent.cartpole") \
        .CUDAClassicControlCartPoleEnv(episode_length=30, env_backend="b200", seed=1)
    w = EnvWrapper(env, num_envs=64, env_backend="b200")
    w.reset_all_envs()
    pm = {"shared": [0]}
    s = CUDASampler(w.cuda_function_manager)
    create_and_push_data_placeholders(env_wrapper=w, action_sampler=s,
                                      policy_tag_to_agent_id_map=pm, training_batch_size_per_env=4)
    s.init_random(1)
    cfg = {"type": "fully_connected", "fc_dims": [32, 32], "model_ckpt_filepath": ""}
    eng = RolloutEngine(w, {"shared": FullyConnected(w, cfg, "shared", pm).cuda()}, pm, s, 4,
                        use_cuda_graph=False)
    assert eng.sa is not None and not eng.sa.continuous
    assert eng._sa_params_ok({"use_argmax": True}) and not eng._sa_params_ok({"scale": 1.0})


def test_invalid_continuous_rollouts_are_refused_without_a_launch():
    from warp_drive_b200 import lib as wlib

    E, T = 32, 4
    w, eng, s, m = _build("pendulum", E, T, 0, fused=True)
    eng.sa.launch(T, **OU)                     # fills the struct with live pointers
    torch.cuda.synchronize()
    L = wlib.load()
    base = eng.sa.r
    # a too-wide head gets real [2, H] weights so that even a wrong acceptance stays in bounds
    H = int(base.dims[base.n_hidden])
    w2, b2 = torch.zeros((2, H), device="cuda"), torch.zeros(2, device="cuda")

    def variant(**fields):
        r = wlib.SaRollout.from_buffer_copy(base)
        r.n_envs = 1
        for k, v in fields.items():
            if k == "head":
                r.dims[r.n_hidden + 1] = 2
                r.w[r.n_hidden], r.b[r.n_hidden] = wlib.ptr(w2), wlib.ptr(b2)
            elif k == "obs_dim":
                r.dims[0] = v
            else:
                setattr(r, k, v)
        return r

    cases = {"state_dim": variant(state_dim=3), "obs_dim": variant(obs_dim=2),
             "ou_state": variant(ou_state=None), "head": variant(head=True),
             "kind": variant(env_kind=5)}
    for what, r in cases.items():
        c0 = wlib.launch_count()
        assert L.wdb_single_agent_rollout(wlib.stream_ptr(), ctypes.byref(r)) != 0, what
        assert wlib.launch_count() == c0, what
    # the bypass (scale < 1e-8) needs no OU state; the unmodified struct launches
    for r in (variant(ou_state=None, ou_scale=0.0), variant()):
        c0 = wlib.launch_count()
        assert L.wdb_single_agent_rollout(wlib.stream_ptr(), ctypes.byref(r)) == 0
        assert wlib.launch_count() == c0 + 1
    torch.cuda.synchronize()
