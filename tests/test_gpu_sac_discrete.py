"""Discrete-action SAC on the GPU: both native passes
(wdb_sac_discrete_{critic,actor}_update_sampled) against the float64 reference
(tests/sac_discrete_reference.py) across their shape envelope, with per-row outputs, sums, guard
regions and a bit-identical relaunch; TrainerDiscreteSAC on CartPole -- the fused update against
the torch update from identical state, a non-logging iteration's launches without a host wait,
the one-launch softmax rollout against the per-step path across the ring's wrap, a checkpoint
round trip and the torch fall-back of a shape outside the envelope."""
import copy
import math
import os

import numpy as np
import pytest
import torch

import dqn_update_reference as dref
import sac_discrete_reference as ref
from test_gpu_ddpg_update_exact import GUARD, SENTINEL, _guarded

pytestmark = pytest.mark.gpu

DEV = "cuda"
# norm-wise bound of a float32 evaluation against float64, as tests/test_gpu_dqn.py
REL = 2e-4


# ------------------------------------------------------------------------ the passes
def _net(F, A, dims, seed):
    """An F -> A MLP (a FullyConnectedQ: the shape of the actor and of each Q network; unlike
    fully_connected_actor it takes no hidden layer too), float32."""
    return dref.make_q_models(F, A, dims, seed=seed)[0].float()


def _layers(model):
    from warp_drive_b200.training.algorithms.fused_sac_discrete import _layers as fl

    return [(w.detach().double().cpu().numpy(), b.detach().double().cpu().numpy())
            for w, b in fl(model)]


def _pick_windows(Ls, ring, B, n_step, seed):
    """B windows (one wrapping the physical end of the ring, one duplicate) whose hidden
    pre-activations in every forward lie off the ReLU kink, so float32 cannot flip one."""
    La, L1, L2, T1, T2 = Ls
    g = np.random.default_rng(seed)
    C, E, Np = ring[0].shape[:3]
    w = np.stack([g.integers(0, C, 8 * B + 8), g.integers(0, E * Np, 8 * B + 8)],
                 axis=1).astype(np.int32)
    w[0] = (C - 1, E * Np - 1)
    obs, _, _, _, boot = dref.gather(ring, w, n_step, Np)
    margin = np.full(len(w), np.inf)
    for L, x in ((La, obs), (La, boot), (L1, obs), (L2, obs), (T1, boot), (T2, boot)):
        margin = np.minimum(margin, dref.relu_margin(L, x))
    w = w[margin > 1e-4][:B].copy()
    if B > 2:
        w[2] = w[1]
    assert len(w) == B
    return w


def _rel(got, want):
    got = got.detach().double().cpu().numpy()
    return float(np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30))


def _guard_grads(model):
    guards = []
    for p in model.parameters():
        buf, view = _guarded(p.shape, DEV)
        p.grad = view
        guards.append(buf)
    return guards


def _untouched(guards):
    return all(bool((b[:GUARD] == SENTINEL).all()) and bool((b[-GUARD:] == SENTINEL).all())
               for b in guards)


# (B, n_step, C, E, Np, F, A, actor dims, critic dims, gamma)
SHAPES = [
    (1, 3, 9, 4, 1, 4, 2, [], [], 0.99),
    (17, 1, 6, 3, 3, 6, 3, [16], [64, 64], 0.0),
    (2113, 3, 40, 8, 1, 4, 2, [64, 64], [64, 64], 1.0),        # more than 132 x 16 rows
    (300, 2, 11, 5, 2, 63, 2, [32, 32], [32, 32], 0.9),        # F = 63
    (64, 2, 9, 4, 1, 5, 64, [32], [32, 32], 0.95),             # A = 64
    (200, 3, 12, 6, 1, 4, 3, [64, 64, 64], [64, 64, 64], 0.97),  # the actor pass only
]


@pytest.mark.parametrize("shape", SHAPES, ids=[f"B{s[0]}_A{s[6]}" for s in SHAPES])
def test_passes_match_the_float64_reference(shape):
    from warp_drive_b200.training.algorithms.fused_sac_discrete import FusedDiscreteSACUpdate

    B, ns, C, E, Np, F, A, ad, cd, gamma = shape
    alpha = 0.3
    models = [_net(F, A, ad, B)] + [_net(F, A, cd, B + k) for k in range(1, 5)]
    Ls = [_layers(m) for m in models]
    obs, actions, rewards, done = dref.make_q_ring(C, E, Np, F, A, seed=B)
    ring = [obs.astype(np.float32), actions, rewards.astype(np.float32), done]
    ring64 = [obs.astype(np.float32).astype(np.float64), actions,
              rewards.astype(np.float32).astype(np.float64), done]
    windows = _pick_windows(Ls, ring64, B, ns, B)
    models = [m.to(DEV) for m in models]
    actor, critic, critic2, t1, t2 = models
    log_alpha = torch.tensor([math.log(alpha)], device=DEV)
    critic_fits = FusedDiscreteSACUpdate.supported(actor, critic, critic2, E, Np, C, ns, B)
    fused = FusedDiscreteSACUpdate(actor, critic, critic2, t1, t2, log_alpha, E, Np, C, ns,
                                   gamma, B) if critic_fits else None
    assert critic_fits == (cd != [64, 64, 64])
    if not critic_fits:
        fused = FusedDiscreteSACUpdate.__new__(FusedDiscreteSACUpdate)
        _init_actor_only(fused, models, log_alpha, E, Np, C, ns, gamma, B)
    dev_ring = [torch.from_numpy(np.ascontiguousarray(r)).to(DEV) for r in ring]
    w = torch.from_numpy(windows).to(DEV)
    te = 0.98 * math.log(A)
    if critic_fits:
        want = ref.critic_pass(*Ls, ring64, windows, ns, gamma, alpha)
        guards = _guard_grads(critic) + _guard_grads(critic2)
        outs = [_guarded((B,), DEV) for _ in range(3)]
        guards += [b for b, _ in outs]
        sums = fused.critic_launch(*dev_ring, w, tuple(v for _, v in outs))[:2].clone()
        first = [p.grad.clone() for m in (critic, critic2) for p in m.parameters()]
        for got, key in zip(first, want["grads1"] + want["grads2"]):
            assert _rel(got, key) <= REL
        for (_, v), k in zip(outs, ("q1", "q2", "returns")):
            assert _rel(v, want[k]) <= REL, k
        assert float(sums[0]) == pytest.approx(want["sum_e1"], rel=REL)
        assert float(sums[1]) == pytest.approx(want["sum_e2"], rel=REL)
        assert _untouched(guards)
        again = fused.critic_launch(*dev_ring, w, tuple(v for _, v in outs))[:2]
        assert all(torch.equal(a, p.grad) for a, p in
                   zip(first, [p for m in (critic, critic2) for p in m.parameters()]))
        assert torch.equal(sums, again)
    want = ref.actor_pass(Ls[0], Ls[1], Ls[2], ring64, windows, ns, alpha, te)
    guards = _guard_grads(actor)
    ent_buf, ent = _guarded((B,), DEV)
    sums = fused.actor_launch(dev_ring[0], w, ent)[2:].clone()
    first = [p.grad.clone() for p in actor.parameters()]
    for got, key in zip(first, want["grads"]):
        assert _rel(got, key) <= REL
    assert _rel(ent, want["entropies"]) <= REL
    assert float(sums[0]) == pytest.approx(want["sum_m"], rel=REL, abs=REL * B)
    assert float(sums[1]) == pytest.approx(want["sum_log_pi"], rel=REL, abs=REL * B)
    assert _untouched(guards + [ent_buf])
    again = fused.actor_launch(dev_ring[0], w, ent)[2:]
    assert all(torch.equal(a, p.grad) for a, p in zip(first, actor.parameters()))
    assert torch.equal(sums, again)


def _init_actor_only(fused, models, log_alpha, E, Np, C, ns, gamma, B):
    """A FusedDiscreteSACUpdate for a shape whose critic pass does not fit: the actor pass's
    workspace only."""
    import ctypes

    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.fused_sac_discrete import _shape_struct

    fused.models = tuple(models)
    fused.log_alpha = log_alpha
    fused.u = _shape_struct(models[0], models[1], E, Np, C, ns)
    fused.u.gamma = gamma
    fused.lib = wlib.load()
    fused.rows = B
    n = int(fused.lib.wdb_sac_discrete_actor_update_sampled_workspace_bytes(
        ctypes.byref(fused.u), B))
    assert n > 0
    fused.workspace = torch.empty(n, dtype=torch.uint8, device=DEV)
    fused.sums = torch.zeros(4, dtype=torch.float64, device=DEV)


# ------------------------------------------------------------------------ the trainer
_NETS = ("actor_models", "critic_models", "critic2_models", "target_critic_models",
         "target_critic2_models", "temperatures")


def _trainer(tmp_path, E=64, T=8, name="r", pool=64, slots=203, model=None, **over):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.cartpole import CUDAClassicControlCartPoleEnv
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_sac_discrete import TrainerDiscreteSAC

    cfg = load_run_config("single_cartpole_sac_discrete")
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, num_episodes=E * 40, seed=11,
                          replay_slots_per_env=slots, replay_batch_rows=333,
                          updates_per_iteration=3, replay_warmup_slots=20)
    cfg["trainer"]["evaluator"] = False
    pol = cfg["policy"]["shared"]
    for kind in ("actor", "critic"):
        pol["model"][kind].update((model or {}).get(kind, {}))
    pol.update(over)
    cfg["env"].update(episode_length=32, reset_pool_size=pool)
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1000,
                         model_params_save_freq=100000)
    # a fixed env seed: identically built trainers start from the same states and pool
    env = CUDAClassicControlCartPoleEnv(**cfg["env"], seed=17)
    w = EnvWrapper(env, num_envs=E, env_backend="numba")
    return TrainerDiscreteSAC(env_wrapper=w, config=cfg,
                              policy_tag_to_agent_id_map={"shared": [0]}, results_dir=name,
                              verbose=False)


def _params(tr):
    return [t.detach().clone() for n in _NETS for t in getattr(tr, n)["shared"].parameters()]


def _opts(tr):
    p = "shared"
    return (tr.actor_optimizers[p], tr.critic_optimizers[p], tr.alpha_optimizers[p])


def _filled(tmp_path, **kw):
    tr = _trainer(tmp_path, **kw)
    for _ in range(3):                         # 24 slots: past the warm-up of 20
        tr._generate_rollout_batch()
    return tr


def _trel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def test_fused_update_matches_the_torch_update_and_launches_without_a_host_wait(tmp_path):
    from warp_drive_b200 import lib as wlib

    tr = _filled(tmp_path)
    assert "shared" in tr.fused_updates and tr.engine.sa is not None
    assert not tr.target_actor_models
    algo = tr.trainers["shared"]
    assert algo.target_entropy == pytest.approx(0.98 * math.log(2))
    start = (_params(tr), [copy.deepcopy(o.state_dict()) for o in _opts(tr)],
             dict(tr.current_timestep), tr.replay_draws)
    results = {}
    for fused in (True, False):
        params, opts, ts, draws = start
        with torch.no_grad():
            for t, v in zip([t for n in _NETS for t in getattr(tr, n)["shared"].parameters()],
                            params):
                t.copy_(v)
        for o, s in zip(_opts(tr), opts):
            o.load_state_dict(s)
        tr.current_timestep.update(ts)
        tr.replay_draws = draws
        algo.use_fused_update = fused
        m = tr._update_model_params(0)["shared"]               # a logging iteration
        results[fused] = (m, tr._arena_grads.clone(), _params(tr))
    algo.use_fused_update = True
    (mf, gf, pf), (mt, gt, pt) = results[True], results[False]
    assert _trel(gf, gt) <= 1e-4                               # every gradient, log_alpha's too
    assert tr.alpha_optimizers["shared"].grads[0].abs() > 0
    for a, b in zip(pf, pt):
        assert torch.isfinite(a).all() and _trel(a, b) <= 1e-5
    assert mf.keys() == mt.keys()
    for k in ("Alpha", "Alpha loss", "Entropy", "Actor loss", "Critic loss", "Mean Q value",
              "Mean return", "Replay buffer fill"):
        assert k in mt, k
    for k in mt:
        if isinstance(mt[k], float) and not k.startswith("Mean episodic"):
            assert mf[k] == pytest.approx(mt[k], rel=1e-4, abs=1e-5), k
    # a non-logging iteration: a fixed number of launches and no host wait
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
    # per update: windows (1), critic pass (2), twin-critic norm and Adam (2), actor pass (2),
    # actor norm and Adam (2), alpha Adam (1)
    assert counts == [3 * 10] * 2


def test_one_launch_rollout_matches_the_per_step_path_across_the_ring_wrap(tmp_path):
    """A uniform policy (the actor's head zeroed: pi = 1/2 exactly on both paths), so the
    actions depend on the sampler's draws alone; a ring of 20 slots filled 8 at a time wraps
    mid-rollout, so the one-launch path runs at t0 > 0 and splits at the wrap."""
    a = _trainer(tmp_path, name="a", pool=0, slots=20)
    b = _trainer(tmp_path, name="b", pool=0, slots=20)
    assert a.engine.sa is not None
    b.engine.sa = None
    for tr in (a, b):
        with torch.no_grad():
            head = tr.actor_models["shared"].policy_head[0]
            head.weight.zero_()
            head.bias.zero_()
    names = ["sampled_actions_batch_shared", "rewards_batch_shared", "done_flags_batch",
             "processed_observations_batch_shared"]
    for it in range(6):                        # cursors 0, 8, 16, 4, 12, 0
        assert a.engine.ring_cursor == b.engine.ring_cursor == (8 * it) % 20
        a._generate_rollout_batch()
        b._generate_rollout_batch()
        for n in names:
            assert torch.equal(a.engine._tensor(n), b.engine._tensor(n)), (it, n)
    acts = a.engine._tensor(names[0])
    assert int(acts.min()) == 0 and int(acts.max()) == 1
    assert torch.equal(a.cuda_sample_controller.rng_state, b.cuda_sample_controller.rng_state)


def test_checkpoint_round_trip(tmp_path):
    tr = _filled(tmp_path)
    for it in range(2):
        tr._update_model_params(it + 1)
    tr.save_model_checkpoint(0)
    ts = tr.current_timestep["shared"]
    kinds = ("actor", "critic", "critic2", "alpha")
    paths = {k: os.path.join(tr.save_dir, f"shared_{k}_{ts}.state_dict") for k in kinds}
    assert all(os.path.isfile(v) for v in paths.values())
    nets = dict(zip(kinds, (tr.actor_models, tr.critic_models, tr.critic2_models,
                            tr.temperatures)))
    saved = {k: [t.detach().clone() for t in nets[k]["shared"].parameters()] for k in kinds}
    fresh = _trainer(tmp_path / "b")
    fresh.load_model_checkpoint({"shared": paths})
    assert fresh.current_timestep["shared"] == ts
    fnets = dict(zip(kinds, (fresh.actor_models, fresh.critic_models, fresh.critic2_models,
                             fresh.temperatures)))
    for k in kinds:
        got = list(fnets[k]["shared"].parameters())
        assert all(torch.equal(a, b) for a, b in zip(got, saved[k])), k
    for target, k in ((fresh.target_critic_models, "critic"),
                      (fresh.target_critic2_models, "critic2")):
        got = list(target["shared"].parameters())
        assert all(torch.equal(a, b) for a, b in zip(got, saved[k])), k
    _, step_sum = fresh.evaluate_episodes(use_argmax=True)     # the greedy policy plays
    assert (step_sum["shared"] >= 1).all()


def test_a_shape_outside_the_envelope_trains_through_torch(tmp_path):
    tr = _filled(tmp_path, model={"critic": {"fc_dims": [64, 64, 64]}})
    assert tr.fused_updates == {}
    before = tr.temperatures["shared"].log_alpha.detach().clone()
    for it in range(3):
        tr._update_model_params(it + 1)
    for n in _NETS:
        assert all(torch.isfinite(p).all() for p in getattr(tr, n)["shared"].parameters())
    assert not torch.equal(before, tr.temperatures["shared"].log_alpha.detach())
