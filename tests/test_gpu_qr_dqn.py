"""Quantile-regression DQN on the GPU: the native pass (wdb_qr_dqn_update_sampled) against the
float64 reference (tests/qr_dqn_reference.py), its weighted form, and TrainerDQN with a
`fully_connected_quantile_q` on CartPole -- fused against torch gradients, the torch fallback
outside the envelope, the one-launch rollout against the per-step path, and training through
the ring's wrap with and without prioritized replay."""
import numpy as np
import pytest
import torch

import dqn_update_reference as dref
import qr_dqn_reference as ref
from test_gpu_ddpg_update_exact import _guarded
from test_gpu_dqn import _dev, _guard_grads, _rel, _ring32, _trainer, _untouched

pytestmark = pytest.mark.gpu

DEV = "cuda"
REL = 2e-4                                 # norm-wise float32 against float64, as DQN's tests


def _qr_model(N=32, dims=(64, 64)):
    return {"type": "fully_connected_quantile_q", "fc_dims": list(dims), "num_quantiles": N,
            "model_ckpt_filepath": ""}


def _pick_windows(models, ring, B, n_step, seed, double_q, N):
    """B windows whose bootstrap action has a mean-quantile margin of 1e-3 and whose hidden
    pre-activations in all three forwards lie off the ReLU kink (float32 cannot flip either;
    the quantile Huber gradient is continuous in every u_ij)."""
    from test_ddpg_update_reference_cpu import layers

    g = np.random.default_rng(seed)
    C, E, Np = ring[0].shape[:3]
    w = np.stack([g.integers(0, C, 8 * B + 8), g.integers(0, E * Np, 8 * B + 8)],
                 axis=1).astype(np.int32)
    w[0] = (C - 1, E * Np - 1)                         # wraps the physical end of the ring
    obs, _, _, _, boot_obs = dref.gather(ring, w, n_step, Np)
    Lq, Lt = layers(models[0]), layers(models[1])
    margin = np.minimum(np.minimum(dref.relu_margin(Lq, obs), dref.relu_margin(Lt, boot_obs)),
                        dref.relu_margin(Lq, boot_obs))
    keep = margin > 1e-4
    means = ref.qr_dqn_sampled(models, ring, w, n_step, 0.9, 1.0, double_q, N)["chooser"].mean(2)
    if means.shape[1] > 1:
        top = np.sort(means, axis=1)
        keep &= top[:, -1] - top[:, -2] > 1e-3
    w = w[keep][:B].copy()
    if B > 2:
        w[2] = w[1]                                    # a duplicate
    assert len(w) == B
    return w


# (B, n_step, C, E, Np, F, A, N, hidden dims)
SHAPES = [(1, 3, 9, 4, 1, 4, 2, 32, [64, 64]), (37, 3, 40, 6, 1, 4, 2, 8, [64, 64]),
          (300, 1, 5, 3, 2, 6, 3, 21, [16]), (129, 2, 30, 4, 1, 3, 4, 16, []),
          (4099, 4, 11, 5, 3, 4, 3, 2, [5, 7, 9])]


def _case(shape, double_q):
    B, n_step, C, E, Np, F, A, N, dims = shape
    q_net, target = ref.make_qr_models(F, A, N, dims, seed=B)
    with torch.no_grad():
        for p in target.parameters():
            p.add_(0.3 * torch.randn_like(p))
    q_net, target = q_net.float(), target.float()
    ring = _ring32(C, E, Np, F, A, B)
    windows = _pick_windows((q_net, target), ring, B, n_step, B, double_q, N)
    probe = ref.qr_dqn_sampled((q_net, target), ring, windows, n_step, 0.97, 1.0, double_q, N)
    kappa = float(np.median(np.abs(probe["u"])))
    return q_net, target, ring, windows, kappa


@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"B{s[0]}_N{s[7]}" for s in SHAPES])
def test_qr_dqn_pass_matches_the_float64_reference(shape, double_q):
    from warp_drive_b200.training.algorithms.dqn import QuantileDQN
    from warp_drive_b200.training.algorithms.fused_dqn import FusedQRDQNUpdate

    B, n_step, C, E, Np, F, A, N, dims = shape
    gamma = 0.97
    q_net, target, ring, windows, kappa = _case(shape, double_q)
    weights = np.random.default_rng(B).uniform(0.1, 1.0, B).astype(np.float32)
    algo = QuantileDQN(gamma, n_step=n_step, double_q=double_q, huber_delta=kappa)
    wants = [ref.qr_dqn_sampled((q_net, target), ring, windows, n_step, gamma, kappa, double_q,
                                N, wt) for wt in (None, weights)]
    q_net, target = q_net.to(DEV), target.to(DEV)
    fused = FusedQRDQNUpdate(algo, q_net, target, E, Np, C, B)
    w = torch.from_numpy(windows).to(DEV)
    results = []
    for want, wt in zip(wants, (None, torch.from_numpy(weights).to(DEV))):
        guards = _guard_grads(q_net)
        outs = [_guarded((B,), DEV) for _ in range(2)]
        guards += [b for b, _ in outs]
        sums = fused.launch(*_dev(ring), w, tuple(v for _, v in outs), wt).clone()
        first = [p.grad.clone() for p in q_net.parameters()]
        for got, key in zip(first, want["grads"]):
            assert _rel(got, key) <= REL
        assert _rel(outs[0][1], want["qbar"]) <= REL and _rel(outs[1][1], want["rbar"]) <= REL
        assert float(sums[0]) == pytest.approx(want["sum_loss"], rel=REL)
        assert float(sums[1]) == pytest.approx(want["sum_q"], rel=REL, abs=REL * B)
        assert _untouched(guards)
        again = fused.launch(*_dev(ring), w, tuple(v for _, v in outs), wt)
        assert all(torch.equal(a, p.grad) for a, p in zip(first, q_net.parameters()))
        assert torch.equal(sums, again)
        results.append((first, sums, [v.clone() for _, v in outs]))
    # unit weights: the unweighted pass bit for bit
    guards = _guard_grads(q_net)
    outs = [torch.empty(B, device=DEV) for _ in range(2)]
    sums = fused.launch(*_dev(ring), w, tuple(outs), torch.ones(B, device=DEV))
    plain_grads, plain_sums, plain_outs = results[0]
    assert all(torch.equal(a, p.grad) for a, p in zip(plain_grads, q_net.parameters()))
    assert torch.equal(sums, plain_sums)
    assert all(torch.equal(a, b) for a, b in zip(outs, plain_outs))


def test_more_than_one_agent_per_env():
    """Np = 3 through the ring: sampled agent rows map to env = row // Np in the kernel as in
    the torch loss on the gathered windows."""
    from warp_drive_b200.training.algorithms.dqn import QuantileDQN
    from warp_drive_b200.training.algorithms.fused_dqn import FusedQRDQNUpdate

    n_step, C, E, Np, F, A, N, B, gamma = 3, 50, 7, 3, 4, 3, 16, 500, 0.95
    q_net, target = [m.float().to(DEV) for m in ref.make_qr_models(F, A, N, [32, 32], seed=9)]
    ring = _dev(_ring32(C, E, Np, F, A, 9))
    g = np.random.default_rng(9)
    windows = torch.from_numpy(np.stack([g.integers(0, C, B), g.integers(0, E * Np, B)],
                                        axis=1).astype(np.int32)).to(DEV)
    algo = QuantileDQN(gamma, n_step=n_step, double_q=True, huber_delta=0.7)
    for p in q_net.parameters():
        p.grad = torch.zeros_like(p)
    FusedQRDQNUpdate(algo, q_net, target, E, Np, C, B).launch(*ring, windows)
    fused = [p.grad.clone() for p in q_net.parameters()]
    s, n = windows[:, 0].long(), windows[:, 1].long()
    steps = (s[None] + torch.arange(n_step + 1, device=DEV)[:, None]) % C
    obs, actions, rewards, done = ring
    o = obs.reshape(C, -1, F)
    q_net.zero_grad()
    loss, _, _ = algo.loss(q_net, target, o[s, n], actions.reshape(C, -1)[s, n][:, None],
                           rewards.reshape(C, -1)[steps[:-1], n],
                           done[steps[:-1], n // Np].float(), o[steps[-1], n])
    loss.backward()
    for a, p in zip(fused, q_net.parameters()):
        assert float((a - p.grad).norm() / p.grad.norm().clamp_min(1e-30)) <= 1e-4


# ------------------------------------------------------------------------ the trainer
def test_trainer_fused_and_torch_gradients_agree(tmp_path):
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.dqn import QuantileDQN
    from warp_drive_b200.training.algorithms.fused_dqn import FusedQRDQNUpdate

    tr = _trainer(tmp_path, model=_qr_model())
    assert isinstance(tr.trainers["shared"], QuantileDQN)
    assert isinstance(tr.fused_updates["shared"], FusedQRDQNUpdate)
    assert tr.engine.sa is not None and tr.engine.q_network    # the one-launch rollout
    for it in range(3):
        tr._generate_rollout_batch()
    acts = tr.engine._tensor("sampled_actions_batch_shared")
    assert int(acts.min()) >= 0 and int(acts.max()) <= 1      # CartPole's 2 actions, not A * N
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
    for a, b in zip(grads[True], grads[False]):
        assert float((a - b).norm() / b.norm().clamp_min(1e-30)) <= 1e-4
    assert metrics[True].keys() == metrics[False].keys() == {"Q loss", "Mean Q value",
                                                             "Mean return"}
    for k in metrics[True]:
        assert metrics[True][k] == pytest.approx(metrics[False][k], rel=1e-4, abs=1e-5), k
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


def test_outside_the_envelope_the_torch_update_trains(tmp_path):
    tr = _trainer(tmp_path, E=16, model=_qr_model(N=33))       # head 2 * 33 = 66 > 64
    assert "shared" not in tr.fused_updates
    before = [p.detach().clone() for p in tr.q_models["shared"].parameters()]
    for it in range(6):
        tr._generate_rollout_batch()
        m = tr._update_model_params(0 if it == 5 else 1)
    assert {"Q loss", "Mean Q value", "Mean return", "Epsilon"} <= set(m["shared"])
    after = list(tr.q_models["shared"].parameters())
    assert all(torch.isfinite(p).all() for p in after)
    assert any(not torch.equal(a, b) for a, b in zip(before, after))


def _two_engines(tmp_path, E=64):
    a = _trainer(tmp_path, E=E, name="a", pool=0, model=_qr_model())
    b = _trainer(tmp_path, E=E, name="b", pool=0, model=_qr_model())
    assert a.engine.sa is not None
    b.engine.sa = None
    for x, y in zip(a.q_models["shared"].parameters(), b.q_models["shared"].parameters()):
        assert torch.equal(x, y)
    return a, b


def test_one_launch_and_per_step_rollouts_agree(tmp_path):
    """epsilon = 1: identical sequences.  epsilon = 0: both take the first argmax of the mean
    quantile from the same collapsed head; envs are compared while every step so far had a
    margin of 1e-4 between the two Q-bar values (the one-launch path records them)."""
    a, b = _two_engines(tmp_path)
    names = ["sampled_actions_batch_shared", "rewards_batch_shared", "done_flags_batch",
             "processed_observations_batch_shared"]
    for _ in range(5):
        a.engine.rollout(epsilon=1.0)
        b.engine.rollout(epsilon=1.0)
        for n in names:
            assert torch.equal(a.engine._tensor(n), b.engine._tensor(n)), n
    # a changed head: the one-launch path must read the collapsed head of the live weights
    for tr in (a, b):
        with torch.no_grad():
            torch.manual_seed(3)
            tr.q_models["shared"].policy_head.weight.add_(
                0.5 * torch.randn_like(tr.q_models["shared"].policy_head.weight))
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
        clean &= (q[0, :, 0] - q[0, :, 1]).abs() > 1e-4
        ea = a.engine._tensor("sampled_actions")[:, 0, 0]
        eb = b.engine._tensor("sampled_actions")[:, 0, 0]
        assert torch.equal(ea[clean], eb[clean])
        assert torch.equal(ea[clean], q[0, clean].argmax(dim=-1).to(torch.int32))
    assert float(clean.float().mean()) > 0.8


_PER = {"prioritized_replay": True, "priority_beta": [[0, 0.4], [10 ** 5, 1.0]]}


@pytest.mark.parametrize("prioritized", [False, True], ids=["uniform", "prioritized"])
def test_trainer_trains_through_the_ring_wrap(prioritized, tmp_path):
    tr = _trainer(tmp_path, E=16, model=_qr_model(),
                  trainer=dict(_PER) if prioritized else {})
    assert "shared" in tr.fused_updates
    st = tr.priority_stores.get("shared")
    assert (st is not None) == prioritized
    C = tr.ring_capacity
    for it in range(30):                                # 240 slots > 203: wraps
        tr._generate_rollout_batch()
        m = tr._update_model_params(0 if it in (5, 29) else 1)
        if it in (5, 29):                               # logging iterations after the warm-up
            m = m["shared"]
            want = {"Q loss", "Mean Q value", "Mean return", "Epsilon", "Replay buffer fill"}
            if prioritized:
                want |= {"Priority beta", "Mean IS weight", "Max priority"}
            assert want <= set(m), it
            assert all(np.isfinite(m[k]) for k in want), it
    assert tr.engine.ring_filled == C and tr.engine.ring_cursor == (30 * 8) % C
    for net in tr._all_networks("shared"):
        assert all(torch.isfinite(p).all() for p in net.parameters())
    if prioritized:
        # the priorities of the last update's windows are (|Q-bar - R-bar| + eps)^alpha
        alpha, eps = tr.prioritized["alpha"], tr.prioritized["epsilon"]
        w = tr.replay_windows["shared"].long()
        leaves = st.leaves[w[:, 0] * 16 + w[:, 1]]
        want = ((st.q_values - st.returns).abs() + eps) ** alpha
        assert bool((leaves >= want * (1 - 1e-5)).all())
        assert float(st.p_max) > 0
