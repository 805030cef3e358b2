"""Branching DQN on the GPU: the per-head epsilon-greedy sampler
(wdb_sample_epsilon_greedy_branching) against wdb_sample_epsilon_greedy and a NumPy rule, the
branching pass (wdb_branching_dqn_update_sampled / _prioritized) bit for bit against DQN's at
D = 1 and within per-element float64 bars (tests/branching_q_reference.py) at D > 1, and
TrainerDQN with fully_connected_branching_q on CartPole, GridReachEnv and TagContinuous."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
from scipy import stats

import branching_q_reference as bref
from test_gpu_ddpg_update_exact import _guarded
from test_gpu_dqn import _dev, _guard_grads, _offsets, _rng, _trainer, _untouched
from test_q_update_bounds_cpu import _f64_layers, within

pytestmark = pytest.mark.gpu

DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))


def _branches(sizes):
    from warp_drive_b200 import lib as wlib

    b = wlib.QBranches()
    b.n_heads = len(sizes)
    for d, a in enumerate(sizes):
        b.sizes[d] = a
    return b


def _sample_branching(q, sizes, eps, state=None, words=None):
    from warp_drive_b200 import lib as wlib

    R = q.shape[0]
    out = torch.full((R, len(sizes)), -1, dtype=torch.int32, device=DEV)
    wlib.check(wlib.load().wdb_sample_epsilon_greedy_branching(
        wlib.stream_ptr(), wlib.ptr(state), wlib.ptr(q), ctypes.byref(_branches(sizes)),
        wlib.ptr(out), R, float(eps), wlib.ptr(words)), "sample_epsilon_greedy_branching")
    return out.cpu().numpy()


def _sample_plain(q, eps, state):
    from warp_drive_b200 import lib as wlib

    R, A = q.shape
    out = torch.full((R,), -1, dtype=torch.int32, device=DEV)
    wlib.check(wlib.load().wdb_sample_epsilon_greedy(
        wlib.stream_ptr(), wlib.ptr(state), wlib.ptr(q), wlib.ptr(out), R, A, float(eps), None))
    return out.cpu().numpy()


# ------------------------------------------------------------------------ the sampler
@pytest.mark.parametrize("eps", [0.0, 0.3, 1.0])
def test_one_head_is_the_plain_sampler_bit_for_bit(eps):
    R, A = 5000, 7
    q = torch.randn(R, A, device=DEV)
    a, b = _rng(R, 9), _rng(R, 9)
    for _ in range(3):
        got = _sample_branching(q, [A], eps, a)[:, 0]
        want = _sample_plain(q, eps, b)
        assert np.array_equal(got, want)
        assert np.array_equal(_offsets(a), _offsets(b))


def test_epsilon_zero_is_each_heads_first_argmax_including_ties():
    sizes = [5, 3, 1, 4]
    R = 4096
    g = torch.Generator(device="cpu").manual_seed(3)
    q = torch.randint(0, 3, (R, sum(sizes)), generator=g).float().to(DEV)   # many ties
    got = _sample_branching(q, sizes, 0.0, _rng(R, 1))
    qn = q.cpu().numpy()
    for d, (o, a) in enumerate(zip(bref.offsets(sizes), sizes)):
        assert np.array_equal(got[:, d], np.argmax(qn[:, o:o + a], axis=1))


def test_epsilon_one_is_uniform_per_head():
    sizes = [5, 3, 21]
    R = 60000
    q = torch.randn(R, sum(sizes), device=DEV)
    got = _sample_branching(q, sizes, 1.0, _rng(R, 4))
    for d, a in enumerate(sizes):
        counts = np.bincount(got[:, d], minlength=a)
        assert len(counts) == a
        assert stats.chisquare(counts).pvalue > 1e-4, (d, counts)
    # the heads explore independently: the pair (head 0, head 1) is uniform over 15 cells
    pair = np.bincount(got[:, 0] * 3 + got[:, 1], minlength=15)
    assert stats.chisquare(pair).pvalue > 1e-4


@pytest.mark.parametrize("eps", [0.25, 0.8])
def test_words_hook_predicts_every_action_and_offsets_advance_by_d(eps):
    sizes = [5, 3, 2]
    D, R = len(sizes), 3000
    g = np.random.default_rng(8)
    q = torch.from_numpy(g.standard_normal((R, sum(sizes))).astype(np.float32)).to(DEV)
    wn = g.integers(0, 2 ** 32, (R, D, 2), dtype=np.uint64)
    words = torch.from_numpy(wn.astype(np.uint32).view(np.int32)).to(DEV).contiguous()
    got = _sample_branching(q, sizes, eps, None, words)
    u = wn[..., 0].astype(np.float64) * 2.0 ** -32 + 2.0 ** -33
    keep = np.abs(u - eps) > 1e-6                      # float32 rounding cannot flip these
    assert keep.mean() > 0.999
    qn = q.cpu().numpy()
    for d, (o, a) in enumerate(zip(bref.offsets(sizes), sizes)):
        explore = (wn[:, d, 1] * np.uint64(a)) >> np.uint64(32)
        want = np.where(u[:, d] <= eps, explore, np.argmax(qn[:, o:o + a], axis=1))
        assert np.array_equal(got[keep[:, d], d], want[keep[:, d]]), d
    state = _rng(R, 5)
    before = _offsets(state).copy()
    _sample_branching(q, sizes, eps, state)
    assert np.array_equal(_offsets(state), before + D)


# ------------------------------------------------------------------------ the pass
GAMMA = np.float32(0.97)


def _models32(F, sizes, dims, seed):
    return [m.float() for m in bref.make_branching_models(F, sizes, dims, seed=seed)]


def _case(B, n_step, C, E, Np, F, sizes, dims, double_q, seed):
    """(models, ring float32, windows [B, 2] whose every premise holds, weights)."""
    models = _models32(F, sizes, dims, seed)
    obs, actions, rewards, done = bref.make_branching_ring(C, E, Np, F, sizes, seed)
    ring = [obs.astype(np.float32), actions, rewards.astype(np.float32), done]
    g = np.random.default_rng(seed + 1)
    n = 4 * B + 64
    w = np.stack([g.integers(0, C, n), g.integers(0, E * Np, n)], 1).astype(np.int32)
    ok = _reference(models, ring, w, n_step, double_q, sizes)["ok"]
    keep = np.flatnonzero(ok)
    assert len(keep) >= B
    weights = g.uniform(0.1, 1.0, B).astype(np.float32)
    return models, ring, w[keep[:B]].copy(), weights


def _reference(models, ring, windows, n_step, double_q, sizes, weights=None):
    Np = ring[0].shape[2]
    rows = bref.gather_branching(ring, windows, n_step, Np)
    q, t = (_f64_layers(m) for m in models)
    return bref.branching_pass(q, t, rows, GAMMA, 1.0, double_q, sizes, weights)


def _fused(models, sizes, E, Np, C, B, n_step, double_q, kind="branching"):
    from warp_drive_b200.training.algorithms import dqn as algos
    from warp_drive_b200.training.algorithms import fused_dqn as fd

    q, t = (m.to(DEV) for m in models)
    if kind == "branching":
        algo = algos.BranchingDQN(float(GAMMA), n_step=n_step, double_q=double_q)
        return q, fd.FusedBranchingDQNUpdate(algo, q, t, E, Np, C, B)
    algo = algos.DQN(float(GAMMA), n_step=n_step, double_q=double_q)
    return q, fd.FusedDQNUpdate(algo, q, t, E, Np, C, B)


# (B, n_step, C, E, Np, F, sizes, dims)
PASSES = [(37, 1, 9, 3, 2, 5, [5, 3], []),
          (256, 3, 20, 8, 2, 57, [21, 21], [64, 64]),
          (1000, 3, 24, 16, 3, 63, [2, 7, 4], [64]),
          (531, 2, 12, 8, 1, 12, [32, 32], [48, 64, 32]),
          (4099, 3, 40, 16, 2, 33, [4] * 16, [64, 64])]


def _pid(c):
    return f"B{c[0]}_D{len(c[6])}_A{sum(c[6])}_L{len(c[7])}"


@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("c", PASSES, ids=[_pid(c) for c in PASSES])
def test_branching_pass_within_its_float64_bars(c, double_q):
    B, n_step, C, E, Np, F, sizes, dims = c
    models, ring, windows, weights = _case(B, n_step, C, E, Np, F, sizes, dims, double_q, B)
    refs = [_reference(models, ring, windows, n_step, double_q, sizes, wt)
            for wt in (None, weights)]
    assert all(r["ok"].all() for r in refs)
    q, fused = _fused(models, sizes, E, Np, C, B, n_step, double_q)
    rd = _dev(ring)
    w = torch.from_numpy(windows).to(DEV)
    names = [n for n, _ in q.named_parameters()]
    for weighted, ref in zip((False, True), refs):
        wt = torch.from_numpy(weights).to(DEV) if weighted else None
        guards = _guard_grads(q)
        outs = [_guarded((B,), DEV) for _ in range(2)]
        guards += [b for b, _ in outs]
        sums = fused.launch(*rd, w, tuple(v for _, v in outs), wt).clone()
        first = [p.grad.clone() for p in q.parameters()]
        for name, got, want in zip(names, first, ref["grads"]):
            within(got.double().cpu().numpy(), want, name)
        within(outs[0][1].double().cpu().numpy(), ref["q_values"], "q_values")
        within(outs[1][1].double().cpu().numpy(), ref["returns"], "returns")
        for i in range(2):
            v, b = ref["sums"][i]
            assert abs(float(sums[i]) - v) <= b, (f"sums[{i}]", float(sums[i]), v, b)
        assert _untouched(guards)
        first_outs = [v.clone() for _, v in outs]
        again = fused.launch(*rd, w, tuple(v for _, v in outs), wt)     # a relaunch: same bits
        assert all(torch.equal(a, p.grad) for a, p in zip(first, q.parameters()))
        assert torch.equal(sums, again)
        assert all(torch.equal(a, v) for a, (_, v) in zip(first_outs, outs))


@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("shape", [(37, 1, 9, 3, 2, 5, 5, []), (2113, 3, 40, 16, 2, 57, 42,
                                                                  [64, 64]),
                                   (300, 2, 16, 4, 1, 63, 64, [32, 16, 8])])
def test_one_head_is_the_dqn_pass_bit_for_bit(shape, double_q):
    B, n_step, C, E, Np, F, A, dims = shape
    models, ring, windows, weights = _case(B, n_step, C, E, Np, F, [A], dims, double_q, B)
    q, branching = _fused(models, [A], E, Np, C, B, n_step, double_q)
    _, plain = _fused(models, [A], E, Np, C, B, n_step, double_q, kind="dqn")
    rd = _dev(ring)
    w = torch.from_numpy(windows).to(DEV)
    for wt in (None, torch.from_numpy(weights).to(DEV)):
        got = []
        for fused in (branching, plain):
            for p in q.parameters():
                p.grad = torch.zeros_like(p)
            outs = (torch.empty(B, device=DEV), torch.empty(B, device=DEV))
            sums = fused.launch(*rd, w, outs, wt).clone()
            got.append(([p.grad.clone() for p in q.parameters()], outs, sums))
        (ga, oa, sa), (gb, ob, sb) = got
        assert all(torch.equal(a, b) for a, b in zip(ga, gb))
        assert all(torch.equal(a, b) for a, b in zip(oa, ob)) and torch.equal(sa, sb)


# ------------------------------------------------------------------------ TrainerDQN
def _branching_model(dims=(64, 64)):
    return {"type": "fully_connected_branching_q", "fc_dims": list(dims),
            "model_ckpt_filepath": ""}


@pytest.mark.parametrize("one_launch", [True, False], ids=["one_launch", "per_step"])
def test_cartpole_branching_equals_fully_connected_q(one_launch, tmp_path):
    """D = 1: the same seed gives identical parameters after several iterations, on the
    one-launch rollout and on the per-step path, and the checkpoint round-trips."""
    from warp_drive_b200.training.algorithms import fused_dqn as fd

    a = _trainer(tmp_path, E=32, name="fq")
    b = _trainer(tmp_path, E=32, name="bq", model=_branching_model())
    assert type(b.fused_updates["shared"]) is fd.FusedBranchingDQNUpdate
    assert a.engine.sa is not None and b.engine.sa is not None
    if not one_launch:
        a.engine.sa = b.engine.sa = None
    for x, y in zip(a.q_models["shared"].parameters(), b.q_models["shared"].parameters()):
        assert torch.equal(x, y)
    for it in range(6):
        for tr in (a, b):
            tr._generate_rollout_batch()
            tr._update_model_params(it + 1)
    assert b.replay_draws > 0
    for x, y in zip(a.q_models["shared"].parameters(), b.q_models["shared"].parameters()):
        assert torch.equal(x, y)
    b.save_model_checkpoint(0)
    path = os.path.join(b.save_dir, f"shared_q_{b.current_timestep['shared']}.state_dict")
    assert os.path.isfile(path)
    c = _trainer(tmp_path, E=32, name="bq2", model=dict(_branching_model(),
                                                         model_ckpt_filepath=path))
    assert c.current_timestep["shared"] == b.current_timestep["shared"]
    for x, y, z in zip(b.q_models["shared"].parameters(), c.q_models["shared"].parameters(),
                       c.target_q_models["shared"].parameters()):
        assert torch.equal(x, y) and torch.equal(y, z)


def _grid_trainer(tmp_path, name, E=64, seed=4):
    sys.path.insert(0, os.path.join(HERE, "custom_env"))
    from grid_reach_env import CUDAGridReachEnv

    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import TrainerDQN
    from warp_drive_b200.utils.env_registrar import EnvironmentRegistrar

    reg = EnvironmentRegistrar()
    reg.add_cuda_env_src_path("GridReachEnv",
                              os.path.join(HERE, "custom_env", "grid_reach_env_step.cu"))
    env = CUDAGridReachEnv(num_agents=4, episode_length=16, env_backend="pycuda")
    w = EnvWrapper(env, num_envs=E, env_backend="pycuda", env_registrar=reg)
    cfg = load_run_config("single_cartpole_dqn")
    cfg["trainer"].update(num_envs=E, train_batch_size=E * 6, num_episodes=E * 10000, seed=seed,
                          n_step=3, replay_slots_per_env=240, replay_batch_rows=512,
                          updates_per_iteration=4, replay_warmup_slots=24)
    cfg["trainer"]["evaluator"] = False
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1000,
                         model_params_save_freq=100000)
    pol = cfg["policy"].pop("shared")
    pol.update(gamma=0.9, lr=0.001, tau=0.01, model=_branching_model((32, 32)))
    pm = env.policy_tag_to_agent_id_map()
    cfg["policy"] = {p: dict(pol, model=dict(pol["model"])) for p in pm}
    cfg["sampler"]["params"]["epsilon"] = [[0, 1.0], [20000, 0.05]]
    return TrainerDQN(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map=pm,
                      results_dir=name, verbose=False)


def test_grid_reach_env_learns_the_shortest_paths(tmp_path):
    """Two policies sharing the placeholders (Np = 2), MultiDiscrete((5, 3)) actions with heads
    of unequal size.  Budget: seed 4, 1000 iterations of 6 steps of 64 envs (epsilon annealed
    from 1 to 0.05 over the first 20 000 steps of each policy) with 4 updates of 512 windows
    each.  Then one greedy episode per env: at least 90 % of (env, agent) episodes reach the
    goal within optimal + 2 steps."""
    from warp_drive_b200.training.algorithms import fused_dqn as fd

    tr = _grid_trainer(tmp_path, "grid", seed=4)
    from grid_reach_env import optimal_steps             # (on the path _grid_trainer set)

    eng = tr.engine
    assert eng.sa is None and eng.fused is None and eng.q_network
    assert all(type(f) is fd.FusedBranchingDQNUpdate for f in tr.fused_updates.values())
    assert set(tr.fused_updates) == {"a", "b"}
    for it in range(1000):
        tr._generate_rollout_batch()
        tr._update_model_params(it + 1)
    acts = eng._tensor("sampled_actions_batch_a")
    assert acts.shape[-1] == 2 and int(acts[..., 0].max()) == 4 and int(acts[..., 1].max()) == 2
    rewards, _ = tr.evaluate_episodes(epsilon=0)
    best = optimal_steps(4)
    ok = []
    for p, ids in tr.policy_tag_to_agent_id_map.items():
        steps = -rewards[p].cpu().numpy()                       # [E, Np]
        ok.append(steps <= best[ids][None, :] + 2)
    frac = float(np.concatenate(ok, axis=1).mean())
    print(f"\nGRID greedy episodes within optimal + 2: {frac:.3f}")
    assert frac >= 0.9


def _tag_trainer(tmp_path, name, K=8, dims=(64, 64), E=4, runners=6):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.tag_continuous import TagContinuous
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import TrainerDQN

    cfg = load_run_config("tag_continuous_dqn")
    cfg["env"].update(num_taggers=2, num_runners=runners, num_other_agents_observed=K,
                      episode_length=40)
    cfg["trainer"].update(num_envs=E, train_batch_size=E * 8, num_episodes=E * 100, seed=7,
                          replay_slots_per_env=64, replay_batch_rows=256,
                          replay_warmup_slots=16)
    cfg["trainer"]["evaluator"] = False
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1000,
                         model_params_save_freq=100000)
    for pol in cfg["policy"].values():
        pol["model"]["fc_dims"] = list(dims)
    env = TagContinuous(**cfg["env"])
    w = EnvWrapper(env, num_envs=E, env_backend="b200")
    n_t = cfg["env"]["num_taggers"]
    pm = {"tagger": list(range(n_t)),
          "runner": list(range(n_t, n_t + cfg["env"]["num_runners"]))}
    return TrainerDQN(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map=pm,
                      results_dir=name, verbose=False)


def test_tag_continuous_trains_natively_at_k8(tmp_path):
    from warp_drive_b200.training.algorithms import fused_dqn as fd

    tr = _tag_trainer(tmp_path, "tag8")
    eng = tr.engine
    assert eng.fused is None and eng.sa is None
    assert all(type(tr.fused_updates[p]) is fd.FusedBranchingDQNUpdate
               for p in ("tagger", "runner"))
    for it in range(3):
        tr._generate_rollout_batch()
        tr._update_model_params(it + 1)
    assert tr.replay_draws > 0
    # greedy actions: each head's first argmax on rows with a clear margin
    slots = (eng.ring_cursor + torch.arange(8, device=DEV)) % tr.ring_capacity
    eng.rollout(epsilon=0.0)
    for p in ("tagger", "runner"):
        obs = eng._tensor(f"processed_observations_batch_{p}")[slots]
        acts = eng._tensor(f"sampled_actions_batch_{p}")[slots]
        with torch.no_grad():
            heads = tr.q_models[p].branches(tr.q_models[p].q_values(obs))
        for d, h in enumerate(heads):
            top = h.topk(2, dim=-1).values
            ok = (top[..., 0] - top[..., 1]) > 1e-4
            assert float(ok.float().mean()) > 0.9
            assert torch.equal(acts[..., d][ok], h.argmax(dim=-1).to(torch.int32)[ok]), (p, d)
    # fused and torch gradients of the same windows agree
    for p in ("tagger", "runner"):
        tr._sample_replay_windows(p)
        grads = {}
        for use in (True, False):
            tr.trainers[p].use_fused_update = use
            if use:
                tr._fused_q_gradients(p, tr.fused_updates[p], False)
            else:
                tr._torch_q_gradients(p, False)
            grads[use] = [x.grad.clone() for x in tr.q_models[p].parameters()]
        tr.trainers[p].use_fused_update = True
        for a, b in zip(grads[True], grads[False]):
            assert float((a - b).norm() / b.norm().clamp_min(1e-30)) <= 1e-4, p


def test_tag_continuous_a2c_shape_trains_through_the_torch_loss(tmp_path):
    tr = _tag_trainer(tmp_path, "tag10", K=10, dims=(256, 256), runners=9)
    assert not tr.fused_updates
    before = [p.detach().clone() for p in tr.q_models["runner"].parameters()]
    for it in range(3):
        tr._generate_rollout_batch()
        tr._update_model_params(it + 1)
    assert tr.replay_draws > 0
    assert any(not torch.equal(a, b) for a, b in
               zip(before, tr.q_models["runner"].parameters()))
