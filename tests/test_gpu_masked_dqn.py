"""Action-masked DQN on the GPU: the masked epsilon-greedy sampler
(wdb_sample_epsilon_greedy_masked) against a NumPy reference and against the unmasked sampler,
the masked DQN and C51 passes (wdb_dqn_update_masked, wdb_c51_update_masked) against the float64
reference with error bars (tests/masked_q_reference.py) and against the unmasked passes, the
native updates of masked plain, dueling, noisy and Rainbow-head networks against the masked
torch losses, and TrainerDQN on MaskedCounterEnv."""
import os
import sys

import numpy as np
import pytest
import torch

import masked_q_reference as mref
from test_gpu_ddpg_update_exact import _guarded
from test_gpu_dqn import _dev, _guard_grads, _offsets, _rng, _untouched
from test_q_update_bounds_cpu import Case, _f64_layers, within

pytestmark = pytest.mark.gpu

DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))


# ------------------------------------------------------------------------ the sampler
def _sample(q, mask, eps, state=None, words=None):
    from warp_drive_b200 import lib as wlib

    R, A = q.shape
    out = torch.full((R,), -1, dtype=torch.int32, device=DEV)
    if mask is None:
        rc = wlib.load().wdb_sample_epsilon_greedy(
            wlib.stream_ptr(), wlib.ptr(state), wlib.ptr(q), wlib.ptr(out), R, A, float(eps),
            wlib.ptr(words))
    else:
        rc = wlib.load().wdb_sample_epsilon_greedy_masked(
            wlib.stream_ptr(), wlib.ptr(state), wlib.ptr(q), wlib.ptr(mask), wlib.ptr(out), R,
            A, float(eps), wlib.ptr(words))
    wlib.check(rc, "sample_epsilon_greedy")
    return out.cpu().numpy()


def _random_masks(g, R, A, empty=0.1, single=0.2):
    """Random rows, a `single` share with one valid action and an `empty` share with none."""
    m = (g.random((R, A)) < 0.5).astype(np.float32)
    s = g.random(R) < single
    none = ~m.any(axis=1)
    s |= none                                          # (every other row has a valid action)
    m[s] = 0.0
    m[np.flatnonzero(s), g.integers(0, A, int(s.sum()))] = 1.0
    m[g.random(R) < empty] = 0.0
    return m


def _numpy_sampler(q, mask, words, eps):
    """The rule of include/wdb200.h in NumPy (the float32 uniform within 1e-6 of eps excluded by
    the caller)."""
    valid = mref.valid(mask)
    n = valid.sum(axis=1).astype(np.uint64)
    k = (words[:, 1] * n) >> np.uint64(32)
    explore = np.argmax(np.cumsum(valid, axis=1) > k[:, None].astype(np.int64), axis=1)
    greedy = mref.masked_argmax(q, mask)
    u = words[:, 0].astype(np.float64) * 2.0 ** -32 + 2.0 ** -33
    return np.where(u <= eps, explore, greedy), np.abs(u - eps) > 1e-6


@pytest.mark.parametrize("eps", [0.0, 0.3, 1.0])
def test_masked_sampler_is_the_numpy_rule_on_the_words_hook(eps):
    g = np.random.default_rng(int(eps * 10) + 1)
    R, A = 50000, 6
    q = g.standard_normal((R, A)).astype(np.float32)
    q[:500, 1:4] = 2.0                                 # tied maxima: the first valid one
    mask = _random_masks(g, R, A)
    words = g.integers(0, 2 ** 32, (R, 2), dtype=np.uint64)
    want, keep = _numpy_sampler(q, mask, words, eps)
    w32 = torch.from_numpy(words.astype(np.uint32).view(np.int32)).to(DEV).contiguous()
    state = _rng(R, 3)
    got = _sample(torch.from_numpy(q).to(DEV), torch.from_numpy(mask).to(DEV), eps, state, w32)
    assert (got[keep] == want[keep]).all() and keep.mean() > 0.999
    assert (_offsets(state) == 0).all()               # the hook reads no RNG state
    none = ~(mask != 0).any(axis=1)
    assert none.any() and (mask.sum(axis=1) == 1).any()
    ok = (mask[np.arange(R), got] != 0) | none
    assert ok.all()


def test_all_ones_mask_is_the_unmasked_sampler_bit_for_bit():
    g = np.random.default_rng(5)
    R, A = 100000, 5
    q = torch.from_numpy(g.standard_normal((R, A)).astype(np.float32)).to(DEV)
    ones = torch.ones((R, A), device=DEV)
    a, b = _rng(R, 21), _rng(R, 21)
    for eps in (0.0, 0.3, 1.0, 0.3):
        assert (_sample(q, ones, eps, a) == _sample(q, None, eps, b)).all(), eps
    assert (_offsets(a) == _offsets(b)).all() and (_offsets(a) == 4).all()


def test_epsilon_one_never_returns_an_invalid_action():
    g = np.random.default_rng(7)
    R, A = 1000000, 7
    mask = _random_masks(g, R, A, empty=0.0)
    md = torch.from_numpy(mask).to(DEV)
    q = torch.zeros((R, A), device=DEV)
    state = _rng(R, 8)
    counts = np.zeros(A, dtype=np.int64)
    for _ in range(4):
        got = _sample(q, md, 1.0, state)
        assert (mask[np.arange(R), got] != 0).all()
        counts += np.bincount(got, minlength=A)
    assert (counts > 0).all()                          # every action explored somewhere


def test_masked_sampler_refuses_a_missing_mask_and_a_bad_epsilon():
    from warp_drive_b200 import lib as wlib

    q, m = torch.zeros((4, 3), device=DEV), torch.ones((4, 3), device=DEV)
    out = torch.zeros(4, dtype=torch.int32, device=DEV)
    state = _rng(4, 1)
    L, before = wlib.load(), wlib.launch_count()
    for mask, eps in ((None, 0.5), (m, -0.1), (m, 1.5), (m, float("nan"))):
        assert L.wdb_sample_epsilon_greedy_masked(
            wlib.stream_ptr(), wlib.ptr(state), wlib.ptr(q), wlib.ptr(mask), wlib.ptr(out), 4,
            3, eps, None) == 1
    assert wlib.launch_count() == before


# ------------------------------------------------------------------------ the update passes
# (kind, B, n_step, C, E, Np, F, A, hidden dims, N, gamma)
PASSES = [("dqn", 17, 3, 12, 4, 3, 6, 3, [64, 64], 1, 0.97),
          ("dqn", 2113, 3, 40, 16, 1, 4, 4, [16, 16], 1, 0.97),
          ("c51", 17, 3, 12, 4, 1, 4, 3, [64], 51, 0.97),
          ("c51", 2113, 2, 40, 16, 1, 4, 2, [64, 64], 51, 0.97)]


def _pass_id(c):
    return f"{c[0]}_B{c[1]}_A{c[7]}_L{len(c[8])}_N{c[9]}"


def _masked_case(c, double_q):
    """A Case whose windows satisfy every premise of the masked reference, and a ring mask
    [C, E, Np, A] with random rows, single-valid rows and rows with no valid action."""
    kind, B, n_step, C, E, Np, F, A, dims, N, gamma = c
    case = Case(kind, B, n_step, C, E, Np, F, A, dims, N, None, gamma, double_q)
    g = np.random.default_rng(B + 101)
    mask = _random_masks(g, C * E * Np, A, empty=0.1).reshape(C, E, Np, A)
    n = 4 * B + 64
    w = np.stack([g.integers(0, C, n), g.integers(0, E * Np, n)], axis=1).astype(np.int32)
    ok = _reference(case, mask, w)["ok"]
    keep = np.flatnonzero(ok)
    assert len(keep) >= B
    case.windows = w[keep[:B]].copy()
    return case, mask


def _reference(case, mask, w=None, weights=None):
    w = case.windows if w is None else w
    q, t = (_f64_layers(m) for m in case.models)
    rows, bm = case.rows(w), mref.boot_mask(mask, w, case.n_step)
    if case.kind == "dqn":
        return mref.dqn_masked_pass(q, t, rows, bm, case.gamma, case.kappa, case.double_q,
                                    weights)
    z, dz = case.support()
    return mref.c51_masked_pass(q, t, rows, bm, case.gamma, case.double_q, z, dz, weights)


def _fused_pair(case):
    """(online network on the device, the masked pass, the unmasked pass)."""
    from warp_drive_b200.training.algorithms import dqn as algos
    from warp_drive_b200.training.algorithms import fused_dqn as fd

    q, t = (m.to(DEV) for m in case.models)
    kw = dict(n_step=case.n_step, double_q=case.double_q)
    if case.kind == "c51":
        algo, masked, plain = algos.CategoricalDQN(case.gamma, **kw), fd.FusedMaskedC51Update, \
            fd.FusedC51Update
    else:
        algo = algos.DQN(case.gamma, huber_delta=case.kappa, **kw)
        masked, plain = fd.FusedMaskedDQNUpdate, fd.FusedDQNUpdate
    args = (algo, q, t, case.E, case.Np, case.C, case.B)
    return q, masked(*args), plain(*args)


@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("c", PASSES, ids=[_pass_id(c) for c in PASSES])
def test_masked_pass_within_its_float64_bars(c, double_q):
    case, mask = _masked_case(c, double_q)
    B = case.B
    refs = [_reference(case, mask, weights=wt) for wt in (None, case.weights)]
    assert all(ref["ok"].all() for ref in refs)
    # the mask changes the bootstrap of some of the windows
    unmasked = case.reference()
    assert (refs[0]["returns"][0] != unmasked["returns"][0]).any()
    q, fused, _ = _fused_pair(case)
    ring = _dev(case.ring)
    md = torch.from_numpy(mask).to(DEV)
    w = torch.from_numpy(case.windows).to(DEV)
    names = [n for n, _ in q.named_parameters()]
    for weighted, ref in zip((False, True), refs):
        wt = torch.from_numpy(case.weights).to(DEV) if weighted else None
        guards = _guard_grads(q)
        outs = [_guarded((B,), DEV) for _ in range(2)]
        guards += [b for b, _ in outs]
        sums = fused.launch(*ring, w, tuple(v for _, v in outs), wt, action_mask=md).clone()
        first = [p.grad.clone() for p in q.parameters()]
        ratios = {}
        for name, got, want in zip(names, first, ref["grads"]):
            ratios[name] = within(got.double().cpu().numpy(), want, name)
        ratios["q_values"] = within(outs[0][1].double().cpu().numpy(), ref["q_values"], "q")
        ratios["returns"] = within(outs[1][1].double().cpu().numpy(), ref["returns"], "R")
        for i in range(2):
            v, b = ref["sums"][i]
            assert abs(float(sums[i]) - v) <= b, (f"sums[{i}]", float(sums[i]), v, b)
        assert _untouched(guards)
        first_outs = [v.clone() for _, v in outs]
        again = fused.launch(*ring, w, tuple(v for _, v in outs), wt, action_mask=md)
        assert all(torch.equal(a, p.grad) for a, p in zip(first, q.parameters()))
        assert torch.equal(sums, again)
        assert all(torch.equal(a, v) for a, (_, v) in zip(first_outs, outs))
        worst = max(ratios, key=ratios.get)
        print(f"\nRATIO masked {_pass_id(c)} {'double_q' if double_q else 'max_target'} "
              f"{'weighted' if weighted else 'uniform'}: max |err|/bar {ratios[worst]:.3g} "
              f"({worst})")


@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("c", PASSES, ids=[_pass_id(c) for c in PASSES])
def test_all_ones_mask_is_the_unmasked_pass_bit_for_bit(c, double_q):
    case, mask = _masked_case(c, double_q)
    q, masked, plain = _fused_pair(case)
    for p in q.parameters():
        p.grad = torch.zeros_like(p)
    ring = _dev(case.ring)
    ones = torch.ones(mask.shape, device=DEV)
    w = torch.from_numpy(case.windows).to(DEV)
    for weights in (None, torch.from_numpy(case.weights).to(DEV)):
        got = []
        for run in (lambda o: masked.launch(*ring, w, o, weights, action_mask=ones),
                    lambda o: plain.launch(*ring, w, o, weights)):
            outs = (torch.empty(case.B, device=DEV), torch.empty(case.B, device=DEV))
            sums = run(outs).clone()
            got.append(([p.grad.clone() for p in q.parameters()], outs, sums))
        (ga, oa, sa), (gb, ob, sb) = got
        assert all(torch.equal(a, b) for a, b in zip(ga, gb))
        assert all(torch.equal(a, b) for a, b in zip(oa, ob)) and torch.equal(sa, sb)


# ------------------------------------------------------------------------ TrainerDQN
def _masked_model(kind):
    return dict(_model(kind), masked=True)


def _model(kind):
    if kind == "dqn":
        return {"type": "fully_connected_q", "fc_dims": [32, 32]}
    if kind == "c51":
        return {"type": "fully_connected_categorical_q", "fc_dims": [32], "num_atoms": 21,
                "v_min": 0.0, "v_max": 12.0}
    if kind == "dueling_dqn":
        return {"type": "fully_connected_q", "fc_dims": [32], "dueling": True,
                "stream_fc_dims": [16]}
    if kind == "noisy_dqn":
        return {"type": "fully_connected_q", "fc_dims": [32], "noisy": True}
    if kind == "qr":
        return {"type": "fully_connected_quantile_q", "fc_dims": [32], "num_quantiles": 8}
    # the Rainbow head: dueling noisy C51
    return {"type": "fully_connected_categorical_q", "fc_dims": [32], "num_atoms": 21,
            "v_min": 0.0, "v_max": 12.0, "dueling": True, "stream_fc_dims": [16], "noisy": True}


def masked_counter_trainer(tmp_path, kind, name, prioritized=False, epsilon=1.0, E=64,
                           evaluator=False, seed=5):
    """TrainerDQN on MaskedCounterEnv: 6 agents per env, one shared policy, 3-step returns."""
    sys.path.insert(0, os.path.join(HERE, "custom_env"))
    from masked_counter_env import STEP_TABLE, CUDAMaskedCounterEnv

    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import TrainerDQN
    from warp_drive_b200.utils.env_registrar import EnvironmentRegistrar

    N = 6
    reg = EnvironmentRegistrar()
    reg.add_cuda_env_src_path("MaskedCounterEnv",
                              os.path.join(HERE, "custom_env", "masked_counter_env_step.cu"))
    env = CUDAMaskedCounterEnv(num_agents=N, episode_length=10, env_backend="pycuda")
    w = EnvWrapper(env, num_envs=E, env_backend="pycuda", env_registrar=reg)
    dm, fm = w.cuda_data_manager, w.cuda_function_manager
    dm.add_shared_constants({"kMaskedStepTable": STEP_TABLE})
    fm.initialize_shared_constants(dm, ["kMaskedStepTable"])
    cfg = load_run_config("single_cartpole_dqn")
    cfg["trainer"].update(num_envs=E, train_batch_size=E * 8, num_episodes=E * 200, seed=seed,
                          n_step=3, replay_slots_per_env=64, replay_batch_rows=256,
                          updates_per_iteration=2, replay_warmup_slots=16,
                          prioritized_replay=prioritized)
    if prioritized:
        cfg["trainer"].update(priority_alpha=0.6, priority_beta=0.4, priority_epsilon=1e-6)
    cfg["trainer"]["evaluator"] = evaluator
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1000,
                         model_params_save_freq=100000)
    pol = cfg["policy"]["shared"]
    pol.update(model=_masked_model(kind), gamma=0.9)
    if "categorical" in pol["model"]["type"]:
        pol.pop("huber_delta", None)
    cfg["sampler"]["params"]["epsilon"] = epsilon
    return TrainerDQN(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": list(
        range(N))}, results_dir=name, verbose=False)


TRAINERS = [("dqn", False), ("c51", False), ("dueling_dqn", False), ("noisy_dqn", False),
            ("rainbow", True), ("dqn", True)]


@pytest.mark.parametrize("kind,prioritized", TRAINERS,
                         ids=[f"{k}{'_per' if p else ''}" for k, p in TRAINERS])
def test_trainer_masked_fused_and_torch_gradients_agree(kind, prioritized, tmp_path):
    from warp_drive_b200.training.algorithms import fused_dqn as fd

    tr = masked_counter_trainer(tmp_path, kind, f"g{kind}{prioritized}", prioritized)
    q = tr.q_models["shared"]
    assert q.masked and tr.engine.masked and tr.engine.sa is None
    fused = tr.fused_updates["shared"]
    want = {"dqn": fd.FusedMaskedDQNUpdate, "c51": fd.FusedMaskedC51Update,
            "dueling_dqn": fd.FusedDuelingUpdate}.get(kind, fd.FusedNoisyUpdate)
    assert type(fused) is want
    plain = getattr(fused, "plain", fused)
    assert plain.masked
    for _ in range(3):
        tr._generate_rollout_batch()
    tr._sample_replay_windows("shared")
    grads, metrics = {}, {}
    for use in (True, False):
        tr.trainers["shared"].use_fused_update = use
        if use:
            metrics[use] = tr._fused_q_gradients("shared", fused, True)
        else:
            metrics[use] = tr._torch_q_gradients("shared", True)
        grads[use] = [p.grad.clone() for p in q.parameters()]
    tr.trainers["shared"].use_fused_update = True
    names = [n for n, _ in q.named_parameters()]
    for name, a, b in zip(names, grads[True], grads[False]):
        assert float((a - b).norm() / b.norm().clamp_min(1e-30)) <= 1e-5, name
    for k in metrics[True]:
        assert metrics[True][k] == pytest.approx(metrics[False][k], rel=1e-5, abs=1e-6), k


def test_masked_qr_dqn_trains_through_the_torch_loss(tmp_path):
    tr = masked_counter_trainer(tmp_path, "qr", "gqr")
    assert "shared" not in tr.fused_updates
    for it in range(4):
        tr._generate_rollout_batch()
        tr._update_model_params(it + 1)
    assert tr.replay_draws > 0
    dm = tr.cuda_envs.cuda_data_manager
    assert int(dm.pull_data_from_device("invalid_actions")[0]) == 0


@pytest.mark.parametrize("kind,prioritized", [("dqn", False), ("dqn", True), ("rainbow", True)],
                         ids=["dqn", "dqn_per", "rainbow"])
def test_train_masked_counter_env_end_to_end(kind, prioritized, tmp_path):
    """Several iterations at epsilon 1 (the masked sampler explores over the valid actions
    only), then on a schedule down to 0: no invalid action reaches the env, in training or in
    the evaluator's greedy episodes."""
    eps = 0.0 if kind == "rainbow" else [[0, 1.0], [3000, 1.0], [12000, 0.05]]
    tr = masked_counter_trainer(tmp_path, kind, f"e{kind}{prioritized}", prioritized, eps,
                                evaluator=True)
    dm = tr.cuda_envs.cuda_data_manager
    before = [p.detach().clone() for p in tr.q_models["shared"].parameters()]
    for it in range(12):
        tr._generate_rollout_batch()
        tr._update_model_params(it + 1)
    assert tr.replay_draws > 0
    assert any(not torch.equal(a, b) for a, b in
               zip(before, tr.q_models["shared"].parameters()))
    assert all(torch.isfinite(p).all() for p in tr.q_models["shared"].parameters())
    mask = tr.engine._tensor("action_mask_batch_shared")
    acts = tr.engine._tensor("sampled_actions_batch_shared").long()
    assert (mask == 0).any() and (mask.gather(-1, acts) != 0).all()
    assert int(dm.pull_data_from_device("invalid_actions")[0]) == 0
    rewards, _ = tr.evaluate_episodes()
    assert all(bool((r >= 0).all()) for r in rewards.values())
    assert int(dm.pull_data_from_device("invalid_actions")[0]) == 0
    tr.graceful_close()
