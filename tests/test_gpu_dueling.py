"""Dueling Q networks on the GPU: wdb_dueling_fold / wdb_dueling_unfold_grads against the float64
reference (tests/dueling_reference.py), the native DQN and C51 updates of a dueling network
against the float64 reference of the plain pass on its folded twin, reproducibility and guard
regions, and TrainerDQN with dueling heads on CartPole -- fused against torch gradients, the
launches of a non-logging update, the one-launch rollout against the per-step path, the fallback
outside the envelope, prioritized replay and a checkpoint round-trip."""
import ctypes

import numpy as np
import pytest
import torch

import c51_reference as cref
import dqn_update_reference as dref
import dueling_reference as ref
import per_reference as pref
from test_dueling_cpu import make_dueling
from test_gpu_c51 import _pick as _pick_c51
from test_gpu_c51 import _trainer
from test_gpu_ddpg_update_exact import _guarded
from test_gpu_dqn import _delta_off_the_kink, _dev, _guard_grads, _pick_windows, _rel, _ring32
from test_gpu_dqn import _untouched

pytestmark = pytest.mark.gpu

DEV = "cuda"
REL = 2e-4                                 # norm-wise float32 against float64, as C51's tests


def _close(got, want, rel=1e-3, floor=REL):
    """Per element: |got - want| <= rel |want| + floor max |want|."""
    got = got.detach().double().cpu().numpy() if torch.is_tensor(got) else got
    bound = rel * np.abs(want) + floor * max(float(np.abs(want).max()), 1e-30)
    return bool((np.abs(got - want) <= bound).all())


def _param_keys(head):
    """The dueling_reference names of a DuelingHead's parameters, in parameter order."""
    if head.stream_dim:
        return [p + s for p in ("value_h", "value_o", "adv_h", "adv_o") for s in "wb"]
    return [p + s for p in ("value_o", "adv_o") for s in "wb"]


def _guard_fold(fold):
    guards = []
    for group in (fold.layers, fold.grads or []):
        for i, (w, b) in enumerate(group):
            (gw, vw), (gb, vb) = _guarded(tuple(w.shape), DEV), _guarded(tuple(b.shape), DEV)
            group[i] = (vw, vb)
            guards += [gw, gb]
    return guards


# (A, N, S, H)
FOLD_SHAPES = [(2, 1, 32, 64), (3, 1, 0, 16), (2, 51, 32, 64), (3, 13, 8, 7), (4, 64, 0, 8),
               (1, 1, 4, 4), (3, 51, 16, 64)]


@pytest.mark.parametrize("shape", FOLD_SHAPES, ids=[f"A{s[0]}_N{s[1]}_S{s[2]}_H{s[3]}"
                                                    for s in FOLD_SHAPES])
def test_fold_and_unfold_match_the_float64_reference(shape):
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.fused_dqn import DuelingFold, fold

    A, N, S, H = shape
    q = make_dueling(4, A, N, [H], S, seed=A + N + S).float().to(DEV)
    t = make_dueling(4, A, N, [H], S, seed=99).float().to(DEV)
    on, tg = DuelingFold(q, grads=True), DuelingFold(t)
    guards = _guard_fold(on) + _guard_fold(tg) + _guard_grads(q)
    fold(on, tg)
    for model, f in ((q, on), (t, tg)):
        p = ref.stream_params(model.policy_head)
        scale = max(float(np.abs(v).max()) for v in p.values())
        for (w, b), (rw, rb) in zip(f.layers, ref.fold(p, A, N, S)):
            for got, want in ((w, rw), (b, rb)):
                err = np.abs(got.double().cpu().numpy() - want)
                assert (err <= 1e-6 * (np.abs(want) + scale)).all()
    first = [(w.clone(), b.clone()) for w, b in on.layers]
    fold(on, tg)
    assert all(torch.equal(a, w) and torch.equal(c, b) for (a, c), (w, b) in zip(first, on.layers))
    # unfold random folded gradients onto the streams
    g = torch.Generator(device=DEV).manual_seed(A * N + S)
    for w, b in on.grads:
        w.copy_(torch.randn(w.shape, generator=g, device=DEV))
        b.copy_(torch.randn(b.shape, generator=g, device=DEV))
    _lib = wlib.load()
    wlib.check(_lib.wdb_dueling_unfold_grads(wlib.stream_ptr(), ctypes.byref(on.struct())))
    want = ref.unfold([(w.double().cpu().numpy(), b.double().cpu().numpy()) for w, b in on.grads],
                      A, N, S)
    head_params = list(q.policy_head.parameters())
    scale = max(float(w.abs().max()) for pair in on.grads for w in pair)
    for p, key in zip(head_params, _param_keys(q.policy_head)):
        err = np.abs(p.grad.double().cpu().numpy() - want[key])
        assert (err <= 1e-6 * (np.abs(want[key]) + A * scale)).all(), key
    again = [p.grad.clone() for p in head_params]
    wlib.check(_lib.wdb_dueling_unfold_grads(wlib.stream_ptr(), ctypes.byref(on.struct())))
    assert all(torch.equal(a, p.grad) for a, p in zip(again, head_params))
    assert _untouched(guards)
    # a NULL required pointer: refused, nothing launched
    n0 = wlib.launch_count()
    bad = on.struct()
    bad.ow = None
    assert _lib.wdb_dueling_fold(wlib.stream_ptr(), ctypes.byref(bad), None) == 1
    bad = on.struct()
    bad.adv_gob = None
    assert _lib.wdb_dueling_unfold_grads(wlib.stream_ptr(), ctypes.byref(bad)) == 1
    assert wlib.launch_count() == n0


def _twins(q_net, target, categorical, dims, F, A, N):
    """Plain float64 networks holding the folded layers of (q_net, target): the networks the
    pass runs."""
    from warp_drive_b200.training.algorithms.fused_dqn import folded_widths

    widths = folded_widths(q_net)
    pair = (cref.make_c51_models(F, A, widths, N=N, v_min=-3.0, v_max=4.0) if categorical
            else dref.make_q_models(F, A, widths))
    for src, twin in zip((q_net, target), pair):
        head = src.policy_head
        layers = [(src.fc[str(i)][0].weight, src.fc[str(i)][0].bias) for i in range(len(dims))]
        layers = [(w.detach().double().cpu().numpy(), b.detach().double().cpu().numpy())
                  for w, b in layers]
        layers += ref.fold(ref.stream_params(head), A, N, head.stream_dim)
        dst = [(twin.fc[str(i)][0].weight, twin.fc[str(i)][0].bias)
               for i in range(len(twin.fc))] + [(twin.policy_head.weight, twin.policy_head.bias)]
        with torch.no_grad():
            for (w, b), (dw, db) in zip(layers, dst):
                dw.copy_(torch.from_numpy(w))
                db.copy_(torch.from_numpy(b))
    return pair


def _unfolded(want_grads, q_net, n_trunk, A, N):
    """The reference gradients of the dueling network's parameters, in parameter order."""
    trunk = want_grads[:2 * n_trunk]
    folded = want_grads[2 * n_trunk:]
    head = q_net.policy_head
    streams = ref.unfold(list(zip(folded[0::2], folded[1::2])), A, N, head.stream_dim)
    return trunk + [streams[k] for k in _param_keys(head)]


# (B, n_step, C, E, Np, F, A, N, trunk dims, S); N = 1: DQN
GRAD_SHAPES = [(333, 3, 40, 6, 1, 4, 2, 1, [64], 32),
               (300, 1, 5, 3, 2, 6, 3, 1, [16, 16], 8),
               (129, 3, 30, 4, 1, 3, 4, 1, [8], 0),
               (333, 3, 40, 6, 1, 4, 2, 51, [64], 32),
               (200, 1, 12, 4, 1, 4, 3, 13, [16], 8),
               (64, 3, 12, 4, 1, 4, 3, 51, [], 0)]


@pytest.mark.parametrize("weighted", [False, True], ids=["uniform", "weighted"])
@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("shape", GRAD_SHAPES, ids=[
    f"{'dqn' if s[7] == 1 else 'c51'}_B{s[0]}_n{s[1]}_A{s[6]}_N{s[7]}_L{len(s[8])}_S{s[9]}"
    for s in GRAD_SHAPES])
def test_dueling_update_matches_the_float64_reference(shape, double_q, weighted):
    from warp_drive_b200.training.algorithms.dqn import DQN, CategoricalDQN
    from warp_drive_b200.training.algorithms.fused_dqn import (
        FusedDuelingUpdate, fused_dueling_supported)

    B, n_step, C, E, Np, F, A, N, dims, S = shape
    categorical = N > 1
    gamma = 0.97
    extra = {"v_min": -3.0, "v_max": 4.0} if categorical else {}
    q_net = make_dueling(F, A, N, dims, S, seed=B, **extra)
    target = make_dueling(F, A, N, dims, S, seed=B, **extra)
    with torch.no_grad():
        for p in target.parameters():
            p.add_(0.3 * torch.randn_like(p))
    q_net, target = q_net.float(), target.float()
    twins = _twins(q_net, target, categorical, dims, F, A, N)
    ring = _ring32(C, E, Np, F, A, B)
    wts = np.random.default_rng(B).uniform(0.1, 1.0, B).astype(np.float32)
    if categorical:
        windows = _pick_c51(twins, ring, B, n_step, B, double_q)
        z, dz = twins[0].support.double().numpy(), twins[0].delta_z
        want = cref.c51_sampled(twins, ring, windows, n_step, gamma, double_q, z, dz,
                                wts if weighted else None)
        algo = CategoricalDQN(gamma, n_step=n_step, double_q=double_q)
        want_q = want["qbar"]
    else:
        windows = _pick_windows(twins, ring, B, n_step, B, double_q)
        probe = dref.dqn_sampled(twins, ring, windows, n_step, gamma, 1e9, double_q)
        delta = _delta_off_the_kink(probe["diff"])
        want = (pref.dqn_weighted(twins, ring, windows, wts.astype(np.float64), n_step, gamma,
                                  delta, double_q) if weighted
                else dref.dqn_sampled(twins, ring, windows, n_step, gamma, delta, double_q))
        algo = DQN(gamma, n_step=n_step, double_q=double_q, huber_delta=delta)
        want_q = want["q"]
    wants = _unfolded(want["grads"], q_net, len(dims), A, N)
    q_net, target = q_net.to(DEV), target.to(DEV)
    assert fused_dueling_supported(algo, q_net, E, Np, C, B)
    fused = FusedDuelingUpdate(algo, q_net, target, E, Np, C, B)
    guards = _guard_grads(q_net) + _guard_fold(fused.online) + _guard_fold(fused.target)
    outs = [_guarded((B,), DEV) for _ in range(2)]
    guards += [b for b, _ in outs]
    w = torch.from_numpy(windows).to(DEV)
    weights = torch.from_numpy(wts).to(DEV) if weighted else None
    sums = fused.launch(*_dev(ring), w, tuple(v for _, v in outs), weights).clone()
    first = [p.grad.clone() for p in q_net.parameters()]
    names = [n for n, _ in q_net.named_parameters()]
    for name, got, key in zip(names, first, wants):
        assert _rel(got, key) <= REL, name
        assert _close(got, key), name
    assert _rel(outs[0][1], want_q) <= REL
    assert _untouched(guards)
    again = fused.launch(*_dev(ring), w, tuple(v for _, v in outs), weights)
    assert all(torch.equal(a, p.grad) for a, p in zip(first, q_net.parameters()))
    assert torch.equal(sums, again)
    if not weighted:                           # unit weights: the unweighted pass bit for bit
        outs2 = [torch.empty(B, device=DEV) for _ in range(2)]
        sums2 = fused.launch(*_dev(ring), w, tuple(outs2), torch.ones(B, device=DEV))
        assert all(torch.equal(a, p.grad) for a, p in zip(first, q_net.parameters()))
        assert torch.equal(sums2, sums)
        assert torch.equal(outs2[0], outs[0][1]) and torch.equal(outs2[1], outs[1][1])


# ------------------------------------------------------------------------ the trainer
def _dueling_model(kind, dims=(64,), S=32):
    m = {"type": kind, "fc_dims": list(dims), "dueling": True, "stream_fc_dims": [S] if S else [],
         "model_ckpt_filepath": ""}
    if kind == "fully_connected_categorical_q":
        m.update(num_atoms=51, v_min=0.0, v_max=100.0)
    return m


KINDS = ["fully_connected_q", "fully_connected_categorical_q"]


@pytest.mark.parametrize("kind", KINDS, ids=["dqn", "c51"])
def test_trainer_fused_and_torch_gradients_agree(kind, tmp_path):
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.fused_dqn import FusedDuelingUpdate

    tr = _trainer(tmp_path, model=_dueling_model(kind))
    assert isinstance(tr.fused_updates["shared"], FusedDuelingUpdate)
    assert tr.engine.sa is not None and tr.engine.q_network    # the one-launch rollout
    for it in range(3):
        tr._generate_rollout_batch()
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
    assert any(n.startswith("policy_head.advantage") for n in names)
    for name, a, b in zip(names, grads[True], grads[False]):
        assert float((a - b).norm() / b.norm().clamp_min(1e-30)) <= 1e-5, name
    for k in metrics[True]:
        assert metrics[True][k] == pytest.approx(metrics[False][k], rel=1e-5, abs=1e-6), k
    # a non-logging update: windows, fold, the pass, unfold, clipping + Adam; no host wait
    tr._update_model_params(1)
    torch.cuda.synchronize()
    for _ in range(2):
        n0 = wlib.launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            tr._update_model_params(1)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert wlib.launch_count() - n0 == 3 * (1 + 1 + 2 + 1 + 2)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        tr._update_model_params(1)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    assert any("dueling_fold_kernel" in n for n in names), names
    assert any("dueling_unfold_kernel" in n for n in names), names
    pass_kernel = "c51_kernel" if "categorical" in kind else "dqn_pass_kernel"
    assert any(pass_kernel in n for n in names), names


@pytest.mark.parametrize("kind", KINDS, ids=["dqn", "c51"])
def test_one_launch_and_per_step_rollouts_agree(kind, tmp_path):
    """epsilon = 1: identical sequences.  epsilon = 0, after an optimizer step and a change to
    the stream parameters: the one-launch path's Q values agree with q_values to 1e-4, and
    both paths take its first argmax where the margin exceeds 3e-4."""
    a = _trainer(tmp_path, E=64, name="a", pool=0, model=_dueling_model(kind))
    b = _trainer(tmp_path, E=64, name="b", pool=0, model=_dueling_model(kind))
    assert a.engine.sa is not None
    b.engine.sa = None
    names = ["sampled_actions_batch_shared", "rewards_batch_shared", "done_flags_batch",
             "processed_observations_batch_shared"]
    for _ in range(3):
        a.engine.rollout(epsilon=1.0)
        b.engine.rollout(epsilon=1.0)
        for n in names:
            assert torch.equal(a.engine._tensor(n), b.engine._tensor(n)), n
    for tr in (a, b):                      # an optimizer step, then a changed advantage stream
        tr._update_model_params(1)
        with torch.no_grad():
            torch.manual_seed(3)
            w = tr.q_models["shared"].policy_head.advantage[2].weight
            w.add_(0.5 * torch.randn_like(w))
    for x, y in zip(a.q_models["shared"].parameters(), b.q_models["shared"].parameters()):
        assert torch.equal(x, y)
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
        clean &= (want[:, 0] - want[:, 1]).abs() > 3e-4
        ea = a.engine._tensor("sampled_actions")[:, 0, 0]
        eb = b.engine._tensor("sampled_actions")[:, 0, 0]
        assert torch.equal(ea[clean], eb[clean])
        assert torch.equal(ea[clean], want[clean].argmax(dim=-1).to(torch.int32))
    assert float(clean.float().mean()) > 0.8


def test_outside_the_envelope_falls_back_and_trains(tmp_path):
    tr = _trainer(tmp_path, E=16, model=_dueling_model("fully_connected_q", S=48))  # 2S = 96
    assert "shared" not in tr.fused_updates and tr.engine.sa is None
    before = [p.detach().clone() for p in tr.q_models["shared"].parameters()]
    for it in range(6):
        tr._generate_rollout_batch()
        m = tr._update_model_params(0 if it == 5 else 1)
    assert {"Q loss", "Mean Q value", "Mean return", "Epsilon"} <= set(m["shared"])
    after = list(tr.q_models["shared"].parameters())
    assert all(torch.isfinite(p).all() for p in after)
    assert any(not torch.equal(x, y) for x, y in zip(before, after))


def test_prioritized_dueling_c51_trains_and_round_trips_a_checkpoint(tmp_path):
    from warp_drive_b200.training.algorithms.fused_dqn import FusedDuelingUpdate

    per = {"prioritized_replay": True, "priority_beta": [[0, 0.4], [10 ** 5, 1.0]]}
    model = _dueling_model("fully_connected_categorical_q")
    tr = _trainer(tmp_path, E=16, trainer=per, model=model)
    assert isinstance(tr.fused_updates["shared"], FusedDuelingUpdate)
    st = tr.priority_stores["shared"]
    for it in range(30):                                # 240 slots > 203: wraps
        tr._generate_rollout_batch()
        m = tr._update_model_params(0 if it == 29 else 1)
    want = {"Q loss", "Mean Q value", "Mean return", "Priority beta", "Mean IS weight",
            "Max priority"}
    assert want <= set(m["shared"]) and all(np.isfinite(m["shared"][k]) for k in want)
    w = tr.replay_windows["shared"].long()
    leaves = st.leaves[w[:, 0] * 16 + w[:, 1]]
    assert bool(torch.isfinite(leaves).all()) and bool((leaves > 0).all())
    q = tr.q_models["shared"]
    assert all(torch.isfinite(p).all() for p in q.parameters())
    path = str(tmp_path / "shared_q_240.state_dict")
    torch.save(q.state_dict(), path)
    fresh = _trainer(tmp_path, E=16, name="fresh", trainer=per, model=model)
    fresh._load_policy_checkpoint("shared", path)
    obs = torch.randn(32, 4, device=DEV)
    with torch.no_grad():
        assert torch.equal(fresh.q_models["shared"].q_values(obs), q.q_values(obs))
        assert torch.equal(fresh.target_q_models["shared"].q_values(obs), q.q_values(obs))
    fresh._generate_rollout_batch()
    fresh._update_model_params(1)                       # the loaded network trains natively
    assert all(torch.isfinite(p).all() for p in fresh.q_models["shared"].parameters())
