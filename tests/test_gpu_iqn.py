"""Implicit quantile networks on the GPU: the native pass (wdb_iqn_update_sampled) against the
float64 reference (tests/iqn_reference.py) over its shape envelope, its weighted form,
reproducibility and guard regions, and TrainerDQN with a `fully_connected_iqn` on CartPole --
fused against torch gradients from the same levels, the one-launch rollout against the per-step
path, prioritized replay, the launches of a non-logging iteration, and QR-DQN's launches left as
they were."""
import numpy as np
import pytest
import torch

import dqn_update_reference as dref
import iqn_reference as ref
from test_gpu_ddpg_update_exact import _guarded
from test_gpu_dqn import _dev, _guard_grads, _rel, _ring32, _trainer, _untouched

pytestmark = pytest.mark.gpu

DEV = "cuda"
REL = 2e-4                                 # norm-wise float32 against float64, as QR-DQN's tests


def _iqn_model(dims=(64, 64), n_cos=64, N=32, NP=32, K=32):
    return {"type": "fully_connected_iqn", "fc_dims": list(dims), "num_cosines": n_cos,
            "num_tau_samples": N, "num_tau_prime_samples": NP, "num_quantile_samples": K,
            "model_ckpt_filepath": ""}


def _pick(models, ring, B, n_step, seed, double_q):
    """B windows and their levels [B, N + N'] whose bootstrap action has a collapsed-head margin
    of 1e-3 and whose pre-activations -- the trunks in all three forwards and the online
    embedding at the row's levels -- lie off the ReLU kink (float32 cannot flip either)."""
    g = np.random.default_rng(seed)
    C, E, Np = ring[0].shape[:3]
    n = 8 * B + 8
    w = np.stack([g.integers(0, C, n), g.integers(0, E * Np, n)], axis=1).astype(np.int32)
    w[0] = (C - 1, E * Np - 1)                         # wraps the physical end of the ring
    q = models[0]
    taus = g.uniform(0.0, 1.0, (n, q.num_tau_samples + q.num_tau_prime_samples))
    taus = taus.astype(np.float32)
    obs, _, _, _, boot_obs = dref.gather(ring, w, n_step, Np)
    trunks = [[(a, b) for a, b in ref.parts(m)[0]] + [ref.parts(m)[1]] for m in models]
    margin = np.minimum(np.minimum(dref.relu_margin(trunks[0], obs),
                                   dref.relu_margin(trunks[1], boot_obs)),
                        dref.relu_margin(trunks[0], boot_obs))
    E_, e_ = ref.parts(q)[2]
    pre = ref.cos_features(taus[:, :q.num_tau_samples].astype(np.float64), E_.shape[1]) @ E_.T
    margin = np.minimum(margin, np.abs(pre + e_).min(axis=(1, 2)))
    keep = margin > 1e-4
    chooser = ref.iqn_sampled(models, ring, w, n_step, 0.9, 1.0, double_q, taus)["chooser"]
    if chooser.shape[1] > 1:
        top = np.sort(chooser, axis=1)
        keep &= top[:, -1] - top[:, -2] > 1e-3
    w, taus = w[keep][:B].copy(), taus[keep][:B].copy()
    if B > 2:
        w[2], taus[2] = w[1], taus[1]                  # a duplicate
    assert len(w) == B
    return w, taus


# (B, n_step, C, E, Np, F, A, n_cos, N, N', K, hidden dims)
SHAPES = [(1, 3, 9, 4, 1, 4, 2, 64, 32, 32, 32, [64, 64]),
          (37, 3, 40, 6, 1, 4, 2, 64, 8, 8, 32, [64, 64]),
          (300, 1, 5, 3, 2, 6, 3, 16, 64, 5, 256, [16]),
          (129, 2, 30, 4, 1, 3, 4, 1, 1, 64, 1, [8]),
          (513, 4, 11, 5, 3, 4, 3, 7, 13, 3, 9, [5, 7, 9]),
          (64, 3, 12, 4, 1, 4, 64, 64, 32, 32, 32, [64, 64]),
          (50, 3, 12, 4, 1, 63, 16, 64, 32, 32, 32, [64, 64]),
          (40, 3, 12, 4, 1, 4, 16, 64, 16, 16, 32, [64, 64, 64])]


def _case(shape, double_q):
    B, n_step, C, E, Np, F, A, n_cos, N, NP, K, dims = shape
    q_net, target = ref.make_iqn_models(F, A, dims, n_cos=n_cos, N=N, NP=NP, K=K, seed=B)
    with torch.no_grad():
        for p in target.parameters():
            p.add_(0.3 * torch.randn_like(p))
        for net in (q_net, target):            # most embedding units active
            net.tau_embedding.bias.add_(0.3)
    q_net, target = q_net.float(), target.float()
    ring = _ring32(C, E, Np, F, A, B)
    windows, taus = _pick((q_net, target), ring, B, n_step, B, double_q)
    probe = ref.iqn_sampled((q_net, target), ring, windows, n_step, 0.97, 1.0, double_q, taus)
    kappa = float(np.median(np.abs(probe["u"])))
    return q_net, target, ring, windows, taus, kappa


@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("shape", SHAPES,
                         ids=[f"B{s[0]}_F{s[5]}_A{s[6]}_N{s[8]}" for s in SHAPES])
def test_iqn_pass_matches_the_float64_reference(shape, double_q):
    from warp_drive_b200.training.algorithms.dqn import ImplicitQuantileDQN
    from warp_drive_b200.training.algorithms.fused_dqn import FusedIQNUpdate

    B, n_step, C, E, Np, F, A, n_cos, N, NP, K, dims = shape
    gamma = 0.97
    q_net, target, ring, windows, taus, kappa = _case(shape, double_q)
    weights = np.random.default_rng(B).uniform(0.1, 1.0, B).astype(np.float32)
    algo = ImplicitQuantileDQN(gamma, n_step=n_step, double_q=double_q, huber_delta=kappa)
    wants = [ref.iqn_sampled((q_net, target), ring, windows, n_step, gamma, kappa, double_q,
                             taus, wt) for wt in (None, weights)]
    q_net, target = q_net.to(DEV), target.to(DEV)
    fused = FusedIQNUpdate(algo, q_net, target, E, Np, C, B)
    w = torch.from_numpy(windows).to(DEV)
    t = torch.from_numpy(taus).to(DEV)
    results = []
    for want, wt in zip(wants, (None, torch.from_numpy(weights).to(DEV))):
        guards = _guard_grads(q_net)
        outs = [_guarded((B,), DEV) for _ in range(2)]
        guards += [b for b, _ in outs]
        sums = fused.launch(*_dev(ring), w, tuple(v for _, v in outs), wt, taus=t).clone()
        first = [p.grad.clone() for p in q_net.parameters()]
        names = [n for n, _ in q_net.named_parameters()]
        for name, got, key in zip(names, first, want["grads"]):
            assert _rel(got, key) <= REL, name
        assert _rel(outs[0][1], want["qbar"]) <= REL and _rel(outs[1][1], want["rbar"]) <= REL
        assert float(sums[0]) == pytest.approx(want["sum_loss"], rel=REL)
        assert float(sums[1]) == pytest.approx(want["sum_q"], rel=REL, abs=REL * B)
        assert _untouched(guards)
        again = fused.launch(*_dev(ring), w, tuple(v for _, v in outs), wt, taus=t)
        assert all(torch.equal(a, p.grad) for a, p in zip(first, q_net.parameters()))
        assert torch.equal(sums, again)
        results.append((first, sums, [v.clone() for _, v in outs]))
    # unit weights: the unweighted pass bit for bit
    _guard_grads(q_net)
    outs = [torch.empty(B, device=DEV) for _ in range(2)]
    sums = fused.launch(*_dev(ring), w, tuple(outs), torch.ones(B, device=DEV), taus=t)
    plain_grads, plain_sums, plain_outs = results[0]
    assert all(torch.equal(a, p.grad) for a, p in zip(plain_grads, q_net.parameters()))
    assert torch.equal(sums, plain_sums)
    assert all(torch.equal(a, b) for a, b in zip(outs, plain_outs))


# ------------------------------------------------------------------------ the trainer
def test_trainer_fused_and_torch_gradients_agree(tmp_path):
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.dqn import ImplicitQuantileDQN
    from warp_drive_b200.training.algorithms.fused_dqn import FusedIQNUpdate

    tr = _trainer(tmp_path, model=_iqn_model())
    assert isinstance(tr.trainers["shared"], ImplicitQuantileDQN)
    assert isinstance(tr.fused_updates["shared"], FusedIQNUpdate)
    assert tr.engine.sa is not None and tr.engine.q_network    # the one-launch rollout
    assert tr.iqn_taus["shared"].shape == (333, 64)
    for it in range(3):
        tr._generate_rollout_batch()
    acts = tr.engine._tensor("sampled_actions_batch_shared")
    assert int(acts.min()) >= 0 and int(acts.max()) <= 1
    tr._sample_replay_windows("shared")
    tr.iqn_taus["shared"].uniform_(generator=tr._tau_generator)
    taus = tr.iqn_taus["shared"].clone()
    assert 0.0 <= float(taus.min()) and float(taus.max()) < 1.0
    grads, metrics = {}, {}
    for fused in (True, False):
        tr.trainers["shared"].use_fused_update = fused
        if fused:
            metrics[fused] = tr._fused_q_gradients("shared", tr.fused_updates["shared"], True)
        else:
            metrics[fused] = tr._torch_q_gradients("shared", True)
        grads[fused] = [p.grad.clone() for p in tr.q_models["shared"].parameters()]
    assert torch.equal(tr.iqn_taus["shared"], taus)     # both read the same levels
    tr.trainers["shared"].use_fused_update = True
    names = [n for n, _ in tr.q_models["shared"].named_parameters()]
    for name, a, b in zip(names, grads[True], grads[False]):
        assert float((a - b).norm() / b.norm().clamp_min(1e-30)) <= 1e-5, name
    assert metrics[True].keys() == metrics[False].keys() == {"Q loss", "Mean Q value",
                                                             "Mean return"}
    for k in metrics[True]:
        assert metrics[True][k] == pytest.approx(metrics[False][k], rel=1e-5, abs=1e-6), k
    # a non-logging iteration: DQN's launches (the levels are one torch draw) and no host wait
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
    assert not torch.equal(tr.iqn_taus["shared"], taus)   # fresh levels every update


def test_quantile_q_config_keeps_its_launches(tmp_path):
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.dqn import QuantileDQN
    from warp_drive_b200.training.algorithms.fused_dqn import FusedQRDQNUpdate

    tr = _trainer(tmp_path, model={"type": "fully_connected_quantile_q", "fc_dims": [64, 64],
                                   "num_quantiles": 32, "model_ckpt_filepath": ""})
    assert type(tr.trainers["shared"]) is QuantileDQN
    assert type(tr.fused_updates["shared"]) is FusedQRDQNUpdate and not tr.iqn_taus
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
    assert any("qr_dqn_kernel" in n for n in names), names
    assert not any("iqn" in n for n in names), names


def _two_engines(tmp_path, E=64):
    a = _trainer(tmp_path, E=E, name="a", pool=0, model=_iqn_model())
    b = _trainer(tmp_path, E=E, name="b", pool=0, model=_iqn_model())
    assert a.engine.sa is not None
    b.engine.sa = None
    for x, y in zip(a.q_models["shared"].parameters(), b.q_models["shared"].parameters()):
        assert torch.equal(x, y)
    return a, b


def test_one_launch_and_per_step_rollouts_agree(tmp_path):
    """epsilon = 1: identical sequences.  epsilon = 0: both take the first argmax of the
    collapsed head of the live weights, the argmax of q_values; envs are compared while every
    step so far had a margin of 3e-4 between the two Q values."""
    a, b = _two_engines(tmp_path)
    names = ["sampled_actions_batch_shared", "rewards_batch_shared", "done_flags_batch",
             "processed_observations_batch_shared"]
    for _ in range(5):
        a.engine.rollout(epsilon=1.0)
        b.engine.rollout(epsilon=1.0)
        for n in names:
            assert torch.equal(a.engine._tensor(n), b.engine._tensor(n)), n
    # a changed embedding: the one-launch path must read the collapsed head of the live weights
    for tr in (a, b):
        with torch.no_grad():
            torch.manual_seed(3)
            e = tr.q_models["shared"].tau_embedding.weight
            e.add_(0.5 * torch.randn_like(e))
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


def test_prioritized_iqn_writes_finite_priorities(tmp_path):
    per = {"prioritized_replay": True, "priority_beta": [[0, 0.4], [10 ** 5, 1.0]]}
    tr = _trainer(tmp_path, E=16, model=_iqn_model(), trainer=per)
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
