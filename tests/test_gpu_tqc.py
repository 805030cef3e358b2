"""TQC on the GPU: both native passes (wdb_tqc_{critic,actor}_update_sampled) against the float64
reference (tests/tqc_reference.py) across their shape envelope, with per-row outputs, sums, guard
regions and a bit-identical relaunch; TrainerTQC on Pendulum -- the fused update against the
torch update from identical state, a non-logging iteration's launches without a host wait, the
run config's shape on the native pass and the one-launch rollout, a checkpoint round trip and
the torch fall-back of shapes outside the envelope."""
import copy
import math
import os

import numpy as np
import pytest
import torch
from torch import nn

import dqn_update_reference as dref
import tqc_reference as ref
from ddpg_update_reference import _forward
from sac_update_reference import squashed
from test_gpu_ddpg_update_exact import GUARD, SENTINEL, _guarded

pytestmark = pytest.mark.gpu

DEV = "cuda"
# norm-wise bound of a float32 evaluation against float64, as tests/test_gpu_sac_discrete.py
REL = 2e-4
LO, HI, SCALE = -5.0, 1.0, 2.0


# ------------------------------------------------------------------------ the passes
class _Net(nn.Module):
    """An MLP with what the fused wrapper reads: `fc.{i}.0` hidden layers (none allowed, unlike
    the model classes), a head `head_name` and the shape attributes of the actor or critic."""

    def __init__(self, inp, dims, out, head_name, **attrs):
        super().__init__()
        sizes = [inp] + list(dims)
        self.fc = nn.ModuleDict({str(i): nn.Sequential(nn.Linear(sizes[i], sizes[i + 1]),
                                                       nn.ReLU()) for i in range(len(dims))})
        setattr(self, head_name, nn.Linear(sizes[-1], out))
        self.fc_dims = list(dims)
        for k, v in attrs.items():
            setattr(self, k, v)


def _models(F, A, ad, cd, N, seed, tied):
    torch.manual_seed(seed)
    actor = _Net(F, ad, 2 * A, "policy_head", flattened_obs_size=F, output_dims=[A],
                 log_std_min=LO, log_std_max=HI, action_scale=SCALE, action_bias=0.0)
    critics = [_Net(F + A, cd, N, "vf_head", num_quantiles=N) for _ in range(4)]
    if tied:
        with torch.no_grad():
            for t in critics[2:]:
                t.vf_head.weight.zero_()
                t.vf_head.bias.fill_(0.5)
    return [m.float() for m in [actor] + critics]


def _layers(model):
    from warp_drive_b200.training.algorithms.fused_ddpg import _layers as fl

    return [(w.detach().double().cpu().numpy(), b.detach().double().cpu().numpy())
            for w, b in fl(model)]


def _pick_windows(Ls, ring, B, n_step, noise, seed):
    """B windows (one wrapping the physical end of the ring, one duplicate) whose hidden
    pre-activations in every forward lie off the ReLU kink, so float32 cannot flip one.  noise:
    (eps', eps) per candidate."""
    La, L1, L2, T1, T2 = Ls
    g = np.random.default_rng(seed)
    C, E, Np = ring[0].shape[:3]
    n = 8 * B + 8
    w = np.stack([g.integers(0, C, n), g.integers(0, E * Np, n)], axis=1).astype(np.int32)
    w[0] = (C - 1, E * Np - 1)
    obs, actions, _, _, boot = ref.gather(ring, w, n_step, Np)
    A = actions.shape[1]
    margin = np.full(n, np.inf)
    for L, x in ((La, obs), (La, boot)):
        margin = np.minimum(margin, dref.relu_margin(L, x))
    x = np.concatenate([obs, actions], axis=1)
    xb = np.concatenate([boot, SCALE * squashed(_forward(La, boot)[0][-1], noise[0], A, LO,
                                                HI)["y"]], axis=1)
    xa = np.concatenate([obs, SCALE * squashed(_forward(La, obs)[0][-1], noise[1], A, LO,
                                               HI)["y"]], axis=1)
    for L in (L1, L2):
        margin = np.minimum(margin, np.minimum(dref.relu_margin(L, x), dref.relu_margin(L, xa)))
    for L in (T1, T2):
        margin = np.minimum(margin, dref.relu_margin(L, xb))
    keep = np.flatnonzero(margin > 1e-4)[:B]
    assert len(keep) == B
    keep[2 % B] = keep[1 % B]
    return w[keep].copy(), noise[0][keep].copy(), noise[1][keep].copy()


def _rel(got, want):
    got = got.detach().double().cpu().numpy()
    return float(np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30))


def _elem(got, want):
    """Per-element error against float64, relative to max(1, |want|)."""
    got = got.detach().double().cpu().numpy()
    return float((np.abs(got - want) / np.maximum(np.abs(want), 1.0)).max())


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


# (B, n_step, C, E, Np, F, A, actor dims, critic dims, N, d, gamma, tied)
SHAPES = [
    (1, 3, 9, 4, 1, 3, 1, [], [], 2, 1, 0.99, False),
    (17, 1, 6, 3, 3, 4, 3, [16], [64], 25, 0, 0.0, False),
    (1024, 5, 40, 8, 1, 3, 1, [64, 64], [64, 64], 25, 2, 0.99, False),   # the run config's
    (2113, 3, 40, 8, 1, 3, 1, [64, 64], [64, 64], 25, 24, 1.0, False),   # > 132 x 16 rows
    (300, 2, 11, 5, 2, 2, 3, [32, 32], [32, 32], 32, 3, 0.9, False),
    (64, 2, 9, 4, 1, 3, 1, [32, 32, 32], [32, 32, 32], 32, 31, 0.95, True),
    (200, 3, 12, 6, 1, 3, 3, [64, 64, 64], [16, 16, 16], 2, 0, 0.97, True),
]


@pytest.mark.parametrize("shape", SHAPES, ids=[f"B{s[0]}_N{s[9]}_d{s[10]}_L{len(s[8])}"
                                               for s in SHAPES])
def test_passes_match_the_float64_reference(shape):
    from warp_drive_b200.training.algorithms.fused_tqc import FusedTQCUpdate
    from warp_drive_b200.training.algorithms.tqc import TQC

    B, ns, C, E, Np, F, A, ad, cd, N, d, gamma, tied = shape
    alpha = 0.3
    models = _models(F, A, ad, cd, N, B, tied)
    Ls = [_layers(m) for m in models]
    obs, actions, rewards, done = ref.make_ring(C, E, Np, F, A, seed=B)
    ring = [obs.astype(np.float32), actions.astype(np.float32), rewards.astype(np.float32),
            done]
    ring64 = [r.astype(np.float64) if r.dtype == np.float32 else r for r in ring]
    noise = np.random.default_rng(B + 1).standard_normal((2, 8 * B + 8, A)).astype(np.float32)
    windows, eps_c, eps_a = _pick_windows(Ls, ring64, B, ns, noise.astype(np.float64), B)
    models = [m.to(DEV) for m in models]
    actor, c1, c2, t1, t2 = models
    algo = TQC(discount_factor_gamma=gamma, n_step=ns, alpha=alpha, action_dim=A,
               n_critics=2, n_quantiles=N, drop_per_net=d)
    log_alpha = torch.tensor([math.log(alpha)], device=DEV)
    assert FusedTQCUpdate.supported(algo, actor, [c1, c2], E, Np, C, ns, B)
    fused = FusedTQCUpdate(algo, actor, [c1, c2], [t1, t2], log_alpha, E, Np, C, ns, B)
    dev_ring = [torch.from_numpy(np.ascontiguousarray(r)).to(DEV) for r in ring]
    w = torch.from_numpy(windows).to(DEV)
    ec, ea = (torch.from_numpy(e.astype(np.float32)).to(DEV) for e in (eps_c, eps_a))
    kw = dict(scale=SCALE, bias=0.0, lo=LO, hi=HI)
    e64c, e64a = eps_c, eps_a                  # float32 values, in float64
    # ---- critic pass
    want = ref.critic_pass(Ls[0], Ls[1:3], Ls[3:], ring64, windows, ns, gamma, alpha,
                           noise=e64c, n_drop=d, **kw)
    guards = _guard_grads(c1) + _guard_grads(c2)
    outs = [_guarded((B,), DEV) for _ in range(2)]
    guards += [b for b, _ in outs]
    sums = fused.critic_launch(*dev_ring, ec, w, tuple(v for _, v in outs))[:2].clone()
    first = [p.grad.clone() for m in (c1, c2) for p in m.parameters()]
    want_grads = [g for m in range(2) for g in want["grads"][m]]
    for got, key in zip(first, want_grads):
        assert _rel(got, key) <= REL
    assert _elem(outs[0][1], want["q_means"]) <= REL
    assert _elem(outs[1][1], want["target_means"]) <= REL
    assert float(sums[0]) == pytest.approx(want["sum_loss"], rel=REL)
    assert float(sums[1]) == pytest.approx(want["sum_q"], rel=REL, abs=REL * B)
    assert _untouched(guards)
    again = fused.critic_launch(*dev_ring, ec, w, tuple(v for _, v in outs))[:2]
    assert all(torch.equal(a, p.grad) for a, p in
               zip(first, [p for m in (c1, c2) for p in m.parameters()]))
    assert torch.equal(sums, again)
    # ---- actor pass
    want = ref.actor_pass(Ls[0], Ls[1:3], ring64, windows, ns, alpha, noise=e64a,
                          target_entropy=-A, **kw)
    guards = _guard_grads(actor)
    lp_buf, lp = _guarded((B,), DEV)
    sums = fused.actor_launch(dev_ring[0], ea, w, lp)[2:].clone()
    first = [p.grad.clone() for p in actor.parameters()]
    for got, key in zip(first, want["grads"]):
        assert _rel(got, key) <= REL
    assert _elem(lp, want["log_probs"]) <= REL
    assert float(sums[0]) == pytest.approx(want["sum_q"], rel=REL, abs=REL * B)
    assert float(sums[1]) == pytest.approx(want["sum_log_pi"], rel=REL, abs=REL * B)
    assert _untouched(guards + [lp_buf])
    again = fused.actor_launch(dev_ring[0], ea, w, lp)[2:]
    assert all(torch.equal(a, p.grad) for a, p in zip(first, actor.parameters()))
    assert torch.equal(sums, again)


# ------------------------------------------------------------------------ the trainer
_NETS = ("actor_models", "critic_models", "target_critic_models", "temperatures")


def _trainer(tmp_path, E=64, T=8, name="r", slots=203, rows=333, model=None, **over):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent import classic_control as cc
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_tqc import TrainerTQC

    cfg = load_run_config("single_pendulum_tqc_replay")
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, num_episodes=E * 40, seed=11,
                          replay_slots_per_env=slots, replay_batch_rows=rows,
                          updates_per_iteration=3, replay_warmup_slots=20)
    cfg["trainer"]["evaluator"] = False
    pol = cfg["policy"]["shared"]
    for kind in ("actor", "critic"):
        pol["model"][kind].update((model or {}).get(kind, {}))
    pol.update(over)
    cfg["env"].update(episode_length=32, reset_pool_size=64)
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1000,
                         model_params_save_freq=100000)
    env = cc.CUDAClassicControlPendulumEnv(**cfg["env"], seed=17)
    w = EnvWrapper(env, num_envs=E, env_backend="numba")
    return TrainerTQC(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                      results_dir=name, verbose=False)


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
    assert not tr.target_actor_models and not tr.critic2_models
    algo = tr.trainers["shared"]
    assert (algo.n_critics, algo.n_quantiles, algo.drop_per_net, algo.target_entropy) == (
        2, 25, 2, -1.0)
    start = (_params(tr), [copy.deepcopy(o.state_dict()) for o in _opts(tr)],
             dict(tr.current_timestep), tr.replay_draws, tr._noise_generator.get_state())
    results = {}
    for fused in (True, False):
        params, opts, ts, draws, gen = start
        with torch.no_grad():
            for t, v in zip([t for n in _NETS for t in getattr(tr, n)["shared"].parameters()],
                            params):
                t.copy_(v)
        for o, s in zip(_opts(tr), opts):
            o.load_state_dict(s)
        tr.current_timestep.update(ts)
        tr.replay_draws = draws
        tr._noise_generator.set_state(gen)
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
    # per update: windows (1), critic pass (2), critics' norm and Adam (2), actor pass (2),
    # actor norm and Adam (2), alpha Adam (1)
    assert counts == [3 * 10] * 2


def test_run_config_shape_takes_the_native_pass_and_the_one_launch_rollout(tmp_path):
    from warp_drive_b200.training.trainer import load_run_config

    cfg = load_run_config("single_pendulum_tqc_replay")["trainer"]
    tr = _trainer(tmp_path, E=cfg["num_envs"], T=cfg["train_batch_size"] // cfg["num_envs"],
                  slots=cfg["replay_slots_per_env"], rows=cfg["replay_batch_rows"])
    assert "shared" in tr.fused_updates and tr.engine.sa is not None
    assert tr.fused_updates["shared"].rows == 1024
    for _ in range(6):                         # 24 slots: past the warm-up of 20
        tr._generate_rollout_batch()
    tr._update_model_params(0)
    for n in _NETS:
        assert all(torch.isfinite(p).all() for p in getattr(tr, n)["shared"].parameters())


def test_checkpoint_round_trip(tmp_path):
    tr = _filled(tmp_path)
    for it in range(2):
        tr._update_model_params(it + 1)
    tr.save_model_checkpoint(0)
    ts = tr.current_timestep["shared"]
    kinds = ("actor", "critic", "alpha")
    paths = {k: os.path.join(tr.save_dir, f"shared_{k}_{ts}.state_dict") for k in kinds}
    assert all(os.path.isfile(v) for v in paths.values())
    assert not os.path.exists(os.path.join(tr.save_dir, f"shared_critic2_{ts}.state_dict"))
    nets = dict(zip(kinds, (tr.actor_models, tr.critic_models, tr.temperatures)))
    saved = {k: [t.detach().clone() for t in nets[k]["shared"].parameters()] for k in kinds}
    assert len(saved["critic"]) == 2 * 6                       # both critics' three layers
    fresh = _trainer(tmp_path / "b")
    fresh.load_model_checkpoint({"shared": paths})
    assert fresh.current_timestep["shared"] == ts
    fnets = dict(zip(kinds, (fresh.actor_models, fresh.critic_models, fresh.temperatures)))
    for k in kinds:
        got = list(fnets[k]["shared"].parameters())
        assert all(torch.equal(a, b) for a, b in zip(got, saved[k])), k
    got = list(fresh.target_critic_models["shared"].parameters())
    assert all(torch.equal(a, b) for a, b in zip(got, saved["critic"]))
    _, step_sum = fresh.evaluate_episodes(use_argmax=True)
    assert (step_sum["shared"] >= 1).all()


@pytest.mark.parametrize("over", [{"n_critics": 3},
                                  {"model": {"critic": {"fc_dims": [128, 128]}}}],
                         ids=["three_critics", "wide_critics"])
def test_a_shape_outside_the_envelope_trains_through_torch(tmp_path, over):
    tr = _filled(tmp_path, **over)
    assert tr.fused_updates == {}
    assert len(tr.critic_models["shared"]) == over.get("n_critics", 2)
    before = tr.temperatures["shared"].log_alpha.detach().clone()
    crit = [p.detach().clone() for p in tr.critic_models["shared"].parameters()]
    for it in (1, 2, 0):                       # the last a logging iteration
        m = tr._update_model_params(it)
    assert "Critic loss" in m["shared"] and math.isfinite(m["shared"]["Critic loss"])
    for n in _NETS:
        assert all(torch.isfinite(p).all() for p in getattr(tr, n)["shared"].parameters())
    assert not torch.equal(before, tr.temperatures["shared"].log_alpha.detach())
    assert not all(torch.equal(a, b) for a, b in zip(crit,
                                                      tr.critic_models["shared"].parameters()))
