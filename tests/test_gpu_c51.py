"""Categorical DQN (C51) on the GPU: the native pass (wdb_c51_update_sampled) against the float64
reference (tests/c51_reference.py) over its shape envelope, its weighted form, reproducibility
and guard regions, the torch fallback outside the envelope, and TrainerDQN with a
`fully_connected_categorical_q` on CartPole -- fused against torch gradients, the launches of a
non-logging iteration, QR-DQN's and IQN's launches left as they were, the one-launch rollout
against the per-step path, MountainCar's fallback to the per-step path, and prioritized
replay."""
import numpy as np
import pytest
import torch

import c51_reference as ref
import dqn_update_reference as dref
from test_ddpg_update_reference_cpu import layers
from test_gpu_ddpg_update_exact import _guarded
from test_gpu_dqn import _dev, _guard_grads, _rel, _ring32, _untouched

pytestmark = pytest.mark.gpu

DEV = "cuda"
REL = 2e-4                                 # norm-wise float32 against float64, as QR-DQN's tests


def _c51_model(dims=(64, 64), N=51, v_min=0.0, v_max=100.0):
    return {"type": "fully_connected_categorical_q", "fc_dims": list(dims), "num_atoms": N,
            "v_min": v_min, "v_max": v_max, "model_ckpt_filepath": ""}


def _trainer(tmp_path, E=64, T=8, name="r", pool=64, env="cartpole", **over):
    """test_gpu_dqn._trainer's CartPole run, with a categorical model and no huber_delta."""
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.cartpole import CUDAClassicControlCartPoleEnv
    from warp_drive_b200.envs.single_agent.mountain_car import CUDAClassicControlMountainCarEnv
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import TrainerDQN

    cfg = load_run_config("single_cartpole_dqn")
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, num_episodes=E * 40, seed=11,
                          replay_slots_per_env=203, replay_batch_rows=333,
                          updates_per_iteration=3, replay_warmup_slots=20)
    cfg["trainer"].update(over.pop("trainer", {}))
    model = over.pop("model", _c51_model())
    if model["type"] == "fully_connected_categorical_q":
        cfg["policy"]["shared"].pop("huber_delta", None)
    cfg["policy"]["shared"].update(over, model=model)
    cfg["trainer"]["evaluator"] = False
    cfg["env"].update(episode_length=32, reset_pool_size=pool)
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1000,
                         model_params_save_freq=100000)
    cls = CUDAClassicControlCartPoleEnv if env == "cartpole" else CUDAClassicControlMountainCarEnv
    w = EnvWrapper(cls(**cfg["env"], seed=17), num_envs=E, env_backend="numba")
    return TrainerDQN(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                      results_dir=name, verbose=False)


def _support(q_net):
    return q_net.support.detach().cpu().double().numpy(), q_net.delta_z


def _pick(models, ring, B, n_step, seed, double_q):
    """B windows whose bootstrap action has an expectation margin of 1e-3 and whose hidden
    pre-activations in all three forwards lie off the ReLU kink (float32 cannot flip either)."""
    g = np.random.default_rng(seed)
    C, E, Np = ring[0].shape[:3]
    n = 8 * B + 8
    w = np.stack([g.integers(0, C, n), g.integers(0, E * Np, n)], axis=1).astype(np.int32)
    w[0] = (C - 1, E * Np - 1)                         # wraps the physical end of the ring
    obs, _, _, _, boot_obs = dref.gather(ring, w, n_step, Np)
    Lq, Lt = layers(models[0]), layers(models[1])
    margin = np.minimum(np.minimum(dref.relu_margin(Lq, obs), dref.relu_margin(Lt, boot_obs)),
                        dref.relu_margin(Lq, boot_obs))
    keep = margin > 1e-4
    z, dz = _support(models[0])
    chooser = ref.c51_sampled(models, ring, w, n_step, 0.97, double_q, z, dz)["chooser"]
    top = np.sort(chooser, axis=1)
    keep &= top[:, -1] - top[:, -2] > 1e-3
    w = w[keep][:B].copy()
    if B > 2:
        w[2] = w[1]                                    # a duplicate
    assert len(w) == B and (w[:, 0] + n_step >= C).any()    # a window wraps the ring
    return w


# (B, n_step, C, E, Np, F, A, N, hidden dims)
SHAPES = [(1, 3, 9, 4, 1, 4, 2, 51, [64, 64]),
          (333, 3, 40, 6, 1, 4, 2, 51, [64, 64]),   # the run config's shape
          (300, 1, 5, 3, 2, 6, 3, 2, [16]),
          (129, 2, 30, 4, 1, 3, 4, 64, [8]),
          (513, 4, 11, 5, 3, 4, 3, 13, [5, 7, 9]),
          (64, 3, 12, 4, 1, 4, 3, 51, []),
          (50, 3, 12, 4, 1, 63, 2, 32, [64, 64]),
          (40, 3, 12, 4, 1, 4, 3, 51, [64, 64])]


@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("shape", SHAPES,
                         ids=[f"B{s[0]}_F{s[5]}_A{s[6]}_N{s[7]}_L{len(s[8])}" for s in SHAPES])
def test_c51_pass_matches_the_float64_reference(shape, double_q):
    from warp_drive_b200.training.algorithms.dqn import CategoricalDQN
    from warp_drive_b200.training.algorithms.fused_dqn import FusedC51Update

    B, n_step, C, E, Np, F, A, N, dims = shape
    gamma = 0.97
    q_net, target = ref.make_c51_models(F, A, dims, N=N, v_min=-3.0, v_max=4.0, seed=B)
    with torch.no_grad():
        for p in target.parameters():
            p.add_(0.3 * torch.randn_like(p))
    q_net, target = q_net.float(), target.float()
    ring = _ring32(C, E, Np, F, A, B)
    windows = _pick((q_net, target), ring, B, n_step, B, double_q)
    z, dz = _support(q_net)
    weights = np.random.default_rng(B).uniform(0.1, 1.0, B).astype(np.float32)
    algo = CategoricalDQN(gamma, n_step=n_step, double_q=double_q)
    wants = [ref.c51_sampled((q_net, target), ring, windows, n_step, gamma, double_q, z, dz, wt)
             for wt in (None, weights)]
    if B > 8:                                  # atom targets clamp at both ends
        assert (wants[0]["tz"] == z[0]).any() and (wants[0]["tz"] == z[-1]).any()
    q_net, target = q_net.to(DEV), target.to(DEV)
    fused = FusedC51Update(algo, q_net, target, E, Np, C, B)
    w = torch.from_numpy(windows).to(DEV)
    results = []
    for want, wt in zip(wants, (None, torch.from_numpy(weights).to(DEV))):
        guards = _guard_grads(q_net)
        outs = [_guarded((B,), DEV) for _ in range(2)]
        guards += [b for b, _ in outs]
        sums = fused.launch(*_dev(ring), w, tuple(v for _, v in outs), wt).clone()
        first = [p.grad.clone() for p in q_net.parameters()]
        names = [n for n, _ in q_net.named_parameters()]
        for name, got, key in zip(names, first, want["grads"]):
            assert _rel(got, key) <= REL, name
        assert _rel(outs[0][1], want["qbar"]) <= REL and _rel(outs[1][1], want["rbar"]) <= REL
        assert float(sums[0]) == pytest.approx(want["sum_loss"], rel=REL)
        assert float(sums[1]) == pytest.approx(want["sum_q"], rel=REL, abs=REL * B)
        assert _untouched(guards)
        again = fused.launch(*_dev(ring), w, tuple(v for _, v in outs), wt)
        assert all(torch.equal(a, p.grad) for a, p in zip(first, q_net.parameters()))
        assert torch.equal(sums, again)
        results.append((first, sums, [v.clone() for _, v in outs]))
    # unit weights: the unweighted pass bit for bit
    _guard_grads(q_net)
    outs = [torch.empty(B, device=DEV) for _ in range(2)]
    sums = fused.launch(*_dev(ring), w, tuple(outs), torch.ones(B, device=DEV))
    plain_grads, plain_sums, plain_outs = results[0]
    assert all(torch.equal(a, p.grad) for a, p in zip(plain_grads, q_net.parameters()))
    assert torch.equal(sums, plain_sums)
    assert all(torch.equal(a, b) for a, b in zip(outs, plain_outs))


def test_outside_the_envelope_the_torch_update_trains(tmp_path):
    from warp_drive_b200.training.algorithms.dqn import CategoricalDQN
    from warp_drive_b200.training.algorithms.fused_dqn import fused_c51_supported

    # a third hidden layer of 64 beside a head of 2 x 51: shared memory runs out
    model = _c51_model(dims=(64, 64, 64))
    q, _ = ref.make_c51_models(4, 2, [64, 64, 64], N=51)
    assert not fused_c51_supported(CategoricalDQN(0.99, n_step=3), q.float(), 16, 1, 203, 333)
    tr = _trainer(tmp_path, E=16, model=model)
    assert isinstance(tr.trainers["shared"], CategoricalDQN)
    assert "shared" not in tr.fused_updates
    before = [p.detach().clone() for p in tr.q_models["shared"].parameters()]
    for it in range(6):
        tr._generate_rollout_batch()
        m = tr._update_model_params(0 if it == 5 else 1)
    assert {"Q loss", "Mean Q value", "Mean return", "Epsilon"} <= set(m["shared"])
    after = list(tr.q_models["shared"].parameters())
    assert all(torch.isfinite(p).all() for p in after)
    assert any(not torch.equal(a, b) for a, b in zip(before, after))


# ------------------------------------------------------------------------ the trainer
def test_trainer_fused_and_torch_gradients_agree(tmp_path):
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.dqn import CategoricalDQN
    from warp_drive_b200.training.algorithms.fused_dqn import FusedC51Update

    tr = _trainer(tmp_path)
    assert isinstance(tr.trainers["shared"], CategoricalDQN)
    assert isinstance(tr.fused_updates["shared"], FusedC51Update)
    assert tr.engine.sa is not None and tr.engine.q_network    # the one-launch rollout
    for it in range(3):
        tr._generate_rollout_batch()
    acts = tr.engine._tensor("sampled_actions_batch_shared")
    assert int(acts.min()) >= 0 and int(acts.max()) <= 1
    tr._sample_replay_windows("shared")
    grads, metrics = {}, {}
    for fused in (True, False):
        tr.trainers["shared"].use_fused_update = fused
        if fused:
            metrics[fused] = tr._fused_q_gradients("shared", tr.fused_updates["shared"], True)
        else:
            metrics[fused] = tr._torch_q_gradients("shared", True)
        grads[fused] = [p.grad.clone() for p in tr.q_models["shared"].parameters()]
    tr.trainers["shared"].use_fused_update = True
    names = [n for n, _ in tr.q_models["shared"].named_parameters()]
    for name, a, b in zip(names, grads[True], grads[False]):
        assert float((a - b).norm() / b.norm().clamp_min(1e-30)) <= 1e-5, name
    assert metrics[True].keys() == metrics[False].keys() == {"Q loss", "Mean Q value",
                                                             "Mean return"}
    for k in metrics[True]:
        assert metrics[True][k] == pytest.approx(metrics[False][k], rel=1e-5, abs=1e-6), k
    # a non-logging iteration: DQN's launches and no host wait
    tr._update_model_params(1)
    torch.cuda.synchronize()
    counts = []
    for _ in range(2):
        n0 = wlib.launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            tr._update_model_params(1)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        counts.append(wlib.launch_count() - n0)
    assert counts == [3 * (1 + 2 + 2)] * 2             # windows, the pass, clipping + Adam
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        tr._update_model_params(1)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    assert any("c51_kernel" in n for n in names), names


@pytest.mark.parametrize("model,kernel", [
    ({"type": "fully_connected_quantile_q", "fc_dims": [64, 64], "num_quantiles": 32,
      "model_ckpt_filepath": ""}, "qr_dqn_kernel"),
    ({"type": "fully_connected_iqn", "fc_dims": [64, 64], "model_ckpt_filepath": ""},
     "iqn_kernel")], ids=["qr_dqn", "iqn"])
def test_other_distributional_configs_keep_their_launches(model, kernel, tmp_path):
    from warp_drive_b200 import lib as wlib

    tr = _trainer(tmp_path, model=model)
    for it in range(3):
        tr._generate_rollout_batch()
        tr._update_model_params(1)
    torch.cuda.synchronize()
    n0 = wlib.launch_count()
    tr._update_model_params(1)
    assert wlib.launch_count() - n0 == 3 * (1 + 2 + 2)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        tr._update_model_params(1)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    assert any(kernel in n for n in names), names
    assert not any("c51" in n for n in names), names


def _two_engines(tmp_path, E=64):
    a = _trainer(tmp_path, E=E, name="a", pool=0)
    b = _trainer(tmp_path, E=E, name="b", pool=0)
    assert a.engine.sa is not None and a.engine.sa.categorical
    b.engine.sa = None
    for x, y in zip(a.q_models["shared"].parameters(), b.q_models["shared"].parameters()):
        assert torch.equal(x, y)
    return a, b


def test_one_launch_and_per_step_rollouts_agree(tmp_path):
    """epsilon = 1: identical sequences.  epsilon = 0: the one-launch path's Q values agree with
    q_values to 1e-4, and both take its first argmax; envs are compared while every step so far
    had a margin of 3e-4 between the two Q values."""
    a, b = _two_engines(tmp_path)
    names = ["sampled_actions_batch_shared", "rewards_batch_shared", "done_flags_batch",
             "processed_observations_batch_shared"]
    for _ in range(5):
        a.engine.rollout(epsilon=1.0)
        b.engine.rollout(epsilon=1.0)
        for n in names:
            assert torch.equal(a.engine._tensor(n), b.engine._tensor(n)), n
    # a changed head: the one-launch path must read the live weights
    for tr in (a, b):
        with torch.no_grad():
            torch.manual_seed(3)
            h = tr.q_models["shared"].policy_head.weight
            h.add_(0.5 * torch.randn_like(h))
    E = 64
    q = torch.empty((1, E, 2), device=DEV)
    clean = torch.ones(E, dtype=torch.bool, device=DEV)
    for _ in range(40):
        obs = a.engine._tensor("observations")[:, 0].clone()
        a.engine.sa.launch(1, record=False, probs_out=q, epsilon=0.0)
        b.engine.step(-1, epsilon=0.0)
        with torch.no_grad():
            want = a.q_models["shared"].q_values(obs)
        assert float((q[0] - want).abs().max()) <= 1e-4
        clean &= (want[:, 0] - want[:, 1]).abs() > 3e-4  # beyond the two paths' difference
        ea = a.engine._tensor("sampled_actions")[:, 0, 0]
        eb = b.engine._tensor("sampled_actions")[:, 0, 0]
        assert torch.equal(ea[clean], eb[clean])
        assert torch.equal(ea[clean], want[clean].argmax(dim=-1).to(torch.int32))
    assert float(clean.float().mean()) > 0.8


def test_mountain_car_falls_back_to_the_per_step_rollout_and_trains(tmp_path):
    tr = _trainer(tmp_path, E=16, env="mountain_car", model=_c51_model(v_min=-100.0, v_max=0.0))
    assert tr.engine.sa is None                          # 3 x 51 atoms: over the weight cap
    assert "shared" in tr.fused_updates                  # the update still runs natively
    before = [p.detach().clone() for p in tr.q_models["shared"].parameters()]
    for it in range(6):
        tr._generate_rollout_batch()
        m = tr._update_model_params(0 if it == 5 else 1)
    assert {"Q loss", "Mean Q value", "Mean return", "Epsilon"} <= set(m["shared"])
    assert all(np.isfinite(m["shared"][k]) for k in ("Q loss", "Mean Q value", "Mean return"))
    acts = tr.engine._tensor("sampled_actions_batch_shared")
    assert int(acts.min()) >= 0 and int(acts.max()) <= 2
    after = list(tr.q_models["shared"].parameters())
    assert all(torch.isfinite(p).all() for p in after)
    assert any(not torch.equal(a, b) for a, b in zip(before, after))


def test_prioritized_c51_writes_finite_priorities(tmp_path):
    per = {"prioritized_replay": True, "priority_beta": [[0, 0.4], [10 ** 5, 1.0]]}
    tr = _trainer(tmp_path, E=16, trainer=per)
    assert "shared" in tr.fused_updates
    st = tr.priority_stores["shared"]
    C = tr.ring_capacity
    for it in range(30):                                # 240 slots > 203: wraps
        tr._generate_rollout_batch()
        m = tr._update_model_params(0 if it in (5, 29) else 1)
        if it in (5, 29):
            m = m["shared"]
            want = {"Q loss", "Mean Q value", "Mean return", "Epsilon", "Priority beta",
                    "Mean IS weight", "Max priority"}
            assert want <= set(m), it
            assert all(np.isfinite(m[k]) for k in want), it
    assert tr.engine.ring_filled == C
    for net in tr._all_networks("shared"):
        assert all(torch.isfinite(p).all() for p in net.parameters())
    alpha, eps = tr.prioritized["alpha"], tr.prioritized["epsilon"]
    w = tr.replay_windows["shared"].long()
    leaves = st.leaves[w[:, 0] * 16 + w[:, 1]]
    assert bool(torch.isfinite(leaves).all()) and bool((leaves > 0).all())
    want = ((st.q_values - st.returns).abs() + eps) ** alpha
    assert bool((leaves >= want * (1 - 1e-5)).all())
    assert np.isfinite(float(st.p_max)) and float(st.p_max) > 0
