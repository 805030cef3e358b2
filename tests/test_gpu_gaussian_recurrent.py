"""Recurrent Gaussian A2C / PPO on the GPU: the mean head kind of wdb_gru_policy_forward within
its a-priori float64 bound (tests/gaussian_recurrent_reference.py) across its envelope, with h'
the same bits as the softmax kind's; the rollout engine on ReachEnv (two policies, shared and
separate placeholders) and ContinuousRecallEnv: the hidden state against a replay of the recorded batch,
graph against eager rollouts, the native against the torch-step forward, the sampled actions
against wdb_sample_gaussian on the kernel's mean, greedy play of the mean, evaluate_episodes and
fetch_episode_states; one A2C and one PPO update through either rollout path on the fused
Gaussian loss kernels; Pendulum's run config; and learning to recall a continuous cue."""
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "custom_env"))

import gaussian_recurrent_reference as gru_ref  # noqa: E402
import recurrent_reference as ref  # noqa: E402
from test_gaussian_recurrent_cpu import _gmodel  # noqa: E402
from test_recurrent_cpu import _model  # noqa: E402

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------ the step kernel
@pytest.mark.parametrize("fc_dims,H,A,F,R", [
    ((64, 64), 64, 1, 3, 10000 + 7),                 # Pendulum-like: F = 3, A = 1
    ((64, 64), 64, 2, 4, 128 * 4 + 3),               # ReachEnv's shape
    ((48,), 96, 6, 13, 37),                          # one trunk layer; 37 rows: 2 tiles + 5
    ((), 112, 6, 3, 37),                             # the widest GRU shared memory holds
    ((), 24, 2, 3, 1),                               # no trunk, a single row
    ((96,), 64, 64, 33, 1001),                       # A = 64
    ((64, 32), 64, 6, 250, 333),                      # F = 250, near 227 KB of shared memory
])
def test_mean_kernel_within_its_float64_bound(fc_dims, H, A, F, R):
    from warp_drive_b200.training.models.fully_connected_gru import NativeGruStep

    m = _gmodel(fc_dims=fc_dims, gru_dim=H, A=A, F=F, seed=R % 89).cuda()
    with torch.no_grad():                         # spread the weights to exercise the gates
        for p in m.parameters():
            p.mul_(2.0)
    assert NativeGruStep.supported(m)
    g = torch.Generator(device="cuda").manual_seed(R)
    obs = torch.randn(R, F, device="cuda", generator=g)
    h0 = torch.randn(R, H, device="cuda", generator=g)
    guard = 64
    hbuf = torch.full((R * H + 2 * guard,), float("nan"), device="cuda")
    hbuf[guard:guard + R * H] = h0.reshape(-1)
    mbuf = torch.full((R * A + 2 * guard,), float("nan"), device="cuda")
    step = NativeGruStep(m)
    step(obs, hbuf[guard:guard + R * H], [mbuf[guard:guard + R * A]])
    torch.cuda.synchronize()
    P = ref.params_of(m)
    mean, hn, emean, ehn = gru_ref.gaussian_step_with_bounds(P, obs.double().cpu().numpy(),
                                                         h0.double().cpu().numpy())
    got_h = hbuf[guard:guard + R * H].view(R, H).double().cpu().numpy()
    assert (np.abs(got_h - hn) <= ehn).all(), (np.abs(got_h - hn) / ehn).max()
    got = mbuf[guard:guard + R * A].view(R, A).double().cpu().numpy()
    assert (np.abs(got - mean) <= emean).all(), (np.abs(got - mean) / emean).max()
    assert torch.isnan(mbuf[:guard]).all() and torch.isnan(mbuf[guard + R * A:]).all()
    assert torch.isnan(hbuf[:guard]).all() and torch.isnan(hbuf[guard + R * H:]).all()
    # relaunch from the same state: the same bits
    first = mbuf.clone(), hbuf.clone()
    hbuf[guard:guard + R * H] = h0.reshape(-1)
    step(obs, hbuf[guard:guard + R * H], [mbuf[guard:guard + R * A]])
    assert torch.equal(mbuf.nan_to_num(7.0), first[0].nan_to_num(7.0))
    assert torch.equal(hbuf.nan_to_num(7.0), first[1].nan_to_num(7.0))
    # the softmax kind on the same trunk and cell (one head of A): h' is the same bits
    cat = _model(fc_dims=fc_dims, gru_dim=H, heads=(A,), F=F).cuda()
    with torch.no_grad():
        for name, p in cat.named_parameters():
            src = name.replace("policy_head.0.", "policy_head.")
            p.copy_(dict(m.named_parameters())[src])
    h_cat = h0.clone()
    probs = torch.empty(R, A, device="cuda")
    NativeGruStep(cat)(obs, h_cat, [probs])
    assert torch.equal(h_cat.reshape(-1), first[1][guard:guard + R * H])
    if A > 1:       # the softmax kind writes probabilities, the mean kind the raw logits
        torch.testing.assert_close(probs, torch.softmax(first[0][guard:guard + R * A].view(R, A),
                                                        -1), rtol=0, atol=1e-6)


def test_mean_kind_refuses_two_heads_and_unknown_kinds():
    import ctypes

    from warp_drive_b200 import lib as wlib

    m = _model(fc_dims=(8,), gru_dim=8, heads=(3, 4), F=5).cuda()
    obs, h = torch.zeros(4, 5, device="cuda"), torch.zeros(4, 8, device="cuda")
    out = [torch.full((4, a), 5.0, device="cuda") for a in (3, 4)]
    a = wlib.GruForward()
    a.n_rows, a.in_dim, a.n_layers, a.hidden_size, a.n_heads = 4, 5, 1, 8, 2
    a.dims[0], a.heads[0], a.heads[1] = 8, 3, 4
    a.obs, a.hidden = wlib.ptr(obs), wlib.ptr(h)
    a.fc_weight[0], a.fc_bias[0] = wlib.ptr(m.fc["0"][0].weight), wlib.ptr(m.fc["0"][0].bias)
    g = m.gru
    a.weight_ih, a.weight_hh = wlib.ptr(g.weight_ih), wlib.ptr(g.weight_hh)
    a.bias_ih, a.bias_hh = wlib.ptr(g.bias_ih), wlib.ptr(g.bias_hh)
    for k, head in enumerate(m.policy_head):
        a.head_weight[k], a.head_bias[k], a.probs[k] = (
            wlib.ptr(head.weight), wlib.ptr(head.bias), wlib.ptr(out[k]))
    L = wlib.load()
    invalid = 1                                          # cudaErrorInvalidValue
    for kind in (1, 2, -1):
        a.head_kind = kind
        assert L.wdb_gru_policy_forward(wlib.stream_ptr(), ctypes.byref(a)) == invalid
    torch.cuda.synchronize()
    assert all(bool((o == 5.0).all()) for o in out)      # nothing launched
    a.head_kind = 0
    assert L.wdb_gru_policy_forward(wlib.stream_ptr(), ctypes.byref(a)) == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------ engines
GGRU = {"type": "fully_connected_gaussian_gru", "fc_dims": [32, 32], "gru_dim": 32,
        "log_std_init": -0.5}


def _reach(tmp_path, name, separate, algo="PPO", E=64, T=10, L=5, iters=3, seed=11,
           use_cuda_graph=True, **policy_keys):
    """Two Gaussian GRU policies ("near", "far") on ReachEnv, episodes of L steps."""
    from reach_env import CUDAReachEnv

    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.training.trainer import Trainer, load_run_config
    from warp_drive_b200.utils.env_registrar import EnvironmentRegistrar

    reg = EnvironmentRegistrar()
    reg.add_cuda_env_src_path("ReachEnv", os.path.join(HERE, "custom_env", "reach_env_step.cu"))
    env = CUDAReachEnv(num_agents=4, episode_length=L, separate=separate, env_backend="pycuda")
    wrapper = EnvWrapper(env, num_envs=E, env_backend="pycuda", env_registrar=reg)
    cfg = load_run_config("tag_gridworld")
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, num_episodes=E * T * iters // L,
                          seed=seed)
    cfg["saving"].update(metrics_log_freq=1, model_params_save_freq=1000, basedir=str(tmp_path))
    pol = cfg["policy"].pop("shared")
    pol.update(algorithm=algo, lr=0.003, entropy_coeff=0.0, vf_loss_coeff=0.5, gamma=0.95,
               clip_param=0.2, **policy_keys)
    pol["model"] = dict(GGRU, model_ckpt_filepath="")
    pm = env.policy_tag_to_agent_id_map()
    cfg["policy"] = {p: json.loads(json.dumps(pol)) for p in pm}
    return Trainer(env_wrapper=wrapper, config=cfg, policy_tag_to_agent_id_map=pm,
                   create_separate_placeholders_for_each_policy=separate, results_dir=name,
                   verbose=False, use_cuda_graph=use_cuda_graph)


def _recall(tmp_path, name, **kw):
    from continuous_recall_env import make_trainer

    kw.setdefault("num_envs", 64)
    kw.setdefault("steps_per_env", 10)            # episodes of 4 steps end inside the batch
    return make_trainer(dict(GGRU), name, str(tmp_path), **kw)


ENGINES = {"reach_shared": lambda tmp, name, **kw: _reach(tmp, name, False, **kw),
           "reach_separate": lambda tmp, name, **kw: _reach(tmp, name, True, **kw),
           "recall": _recall}


def _actions(tr, p):
    """Policy p's current sampled actions [E, Np, A]."""
    dm = tr.cuda_envs.cuda_data_manager
    if tr.engine.separate:
        return dm.data_on_device_via_torch(f"sampled_actions_{p}")
    return dm.data_on_device_via_torch("sampled_actions")[:, tr.engine.policy_map[p]]


@pytest.mark.parametrize("kind", list(ENGINES))
def test_hidden_state_equals_forward_sequence_over_the_recorded_batch(tmp_path, kind):
    tr = ENGINES[kind](tmp_path, "seq")
    eng = tr.engine
    assert eng.recurrent and all(eng.gaussian_of.values())
    assert set(eng.native_gru) == set(eng.policies) and eng.fused is None and eng.sa is None
    dm = tr.cuda_envs.cuda_data_manager
    for _ in range(3):                              # the state carries over between rollouts
        eng.rollout()
    torch.cuda.synchronize()
    done = dm.data_on_device_via_torch("done_flags_batch")
    assert (done > 0).any()
    for p in eng.policies:
        assert (eng.hidden_start[p] != 0).any()
        obs = dm.data_on_device_via_torch(f"processed_observations_batch_{p}")
        m = tr.models[p]
        with torch.no_grad():
            h = eng.hidden_start[p].reshape(-1, m.hidden_size)
            x = m.trunk(obs)
            E, Np = done.shape[1], obs.shape[2]
            for t in range(obs.shape[0]):
                if t > 0:
                    h = m.reset_hidden(h.view(E, Np, -1), done[t - 1]).view(E * Np, -1)
                h = m.gru(x[t].reshape(E * Np, -1), h)
            h = m.reset_hidden(h.view(E, Np, -1), done[-1])
        torch.testing.assert_close(eng.hidden[p], h, rtol=0, atol=1e-5)


@pytest.mark.parametrize("kind", list(ENGINES))
def test_graph_and_eager_rollouts_agree_bit_for_bit(tmp_path, kind):
    outs = []
    for graph in (True, False):
        tr = ENGINES[kind](tmp_path, f"g{graph}", use_cuda_graph=graph)
        eng = tr.engine
        tr._reset_all_envs()
        eng.resync_observations()
        if not graph:                 # the graph's capture is preceded by one evaluation step
            eng.step(-1)
        eng.rollout()
        tr._reset_all_envs()
        eng.resync_observations()
        eng.rollout()
        torch.cuda.synchronize()
        dm = tr.cuda_envs.cuda_data_manager
        got = [dm.data_on_device_via_torch("done_flags_batch").clone(),
               tr.cuda_sample_controller.rng_state.clone()]
        for p in eng.policies:
            got += [dm.data_on_device_via_torch(f"{n}_{p}").clone() for n in (
                "processed_observations_batch", "sampled_actions_batch", "rewards_batch")]
            got += [eng.hidden[p].clone(), eng.hidden_start[p].clone()]
        outs.append(got)
    for a, b in zip(*outs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("kind", list(ENGINES))
def test_native_and_torch_step_agree_and_actions_are_the_samplers_draw(tmp_path, kind):
    """Teacher-forced over 12 steps: from the same observations and state, the native and
    torch-step forwards agree on the mean and h' to 1e-5; the actions the step samples are
    wdb_sample_gaussian's draw from the kernel's mean under the same RNG state, bit for bit; a
    greedy step plays the mean and draws nothing."""
    tr = ENGINES[kind](tmp_path, "nat", use_cuda_graph=False)
    eng = tr.engine
    sampler = tr.cuda_sample_controller
    tr._reset_all_envs()
    eng.resync_observations()
    for t in range(12):
        h_t = {p: eng.hidden[p].clone() for p in eng.policies}
        rng0 = sampler.rng_state.clone()
        out = eng.evaluate_policies(-1)
        means = ({p: out[p][0].clone() for p in eng.policies} if isinstance(out, dict)
                 else {eng.policies[0]: out[0].clone()})
        # the same rows through the torch step
        obs_rows = {p: _eval_rows(eng, p) for p in eng.policies}
        for p in eng.policies:
            h_nat = eng.hidden[p].clone()
            eng.hidden[p].copy_(h_t[p])
            native = eng.native_gru.pop(p)
            (mean_t,) = eng._recurrent_forward(p, obs_rows[p])
            eng.native_gru[p] = native
            torch.testing.assert_close(means[p], mean_t, rtol=0, atol=1e-5)
            torch.testing.assert_close(h_nat, eng.hidden[p], rtol=0, atol=1e-5)
            eng.hidden[p].copy_(h_t[p])
        greedy = t % 3 == 2
        eng.step(-1, use_argmax=True) if greedy else eng.step(-1)
        torch.cuda.synchronize()
        if greedy:
            assert torch.equal(sampler.rng_state, rng0)
            for p in eng.policies:
                assert torch.equal(_actions(tr, p), means[p]), (t, p)
            continue
        drawn = sampler.rng_state.clone()
        sampler.rng_state.copy_(rng0)
        for p in eng.policies:                    # the engine's draws, in its order
            want = torch.empty_like(means[p])
            sampler.sample_gaussian(means[p], tr.models[p].log_std, want)
            assert torch.equal(_actions(tr, p), want), (t, p)
        assert torch.equal(sampler.rng_state, drawn)


def _eval_rows(eng, p):
    """Policy p's observation rows of an evaluation step, as evaluate_policies gathered them."""
    if eng.gather_fields:
        return eng._field_scratch[0][p].clone()
    obs = eng._tensor("observations").view(eng.E, eng.N, -1)
    return obs[:, eng.policy_map[p]].contiguous()


@pytest.mark.parametrize("kind", ["reach_shared", "reach_separate"])
def test_evaluate_episodes_and_fetch_episode_states_play_the_mean(tmp_path, kind):
    tr = ENGINES[kind](tmp_path, "ev", use_cuda_graph=False)
    tr._reset_all_envs()
    tr.engine.resync_observations()
    tr.engine.rollout()
    rng0 = tr.cuda_sample_controller.rng_state.clone()
    r1, s1 = tr.evaluate_episodes(use_argmax=True)
    r2, s2 = tr.evaluate_episodes(use_argmax=True)
    assert torch.equal(tr.cuda_sample_controller.rng_state, rng0)
    for p in tr.policies:
        assert torch.equal(r1[p], r2[p]) and torch.equal(s1[p], s2[p])
        assert float(r1[p].sum()) != 0.0
    out = tr.fetch_episode_states(["pos"], include_probabilities=True, policy="near")
    assert len(out["probabilities"]) == 5
    assert out["probabilities"][0][0].shape == (2, 2)
    assert all(np.isfinite(np.asarray(q[0])).all() for q in out["probabilities"])


# ------------------------------------------------------------------------ updates
@pytest.mark.parametrize("kind", ["reach_separate", "recall"])
@pytest.mark.parametrize("algorithm", ["A2C", "PPO"])
def test_one_update_agrees_between_the_rollout_paths_on_the_fused_loss(tmp_path, algorithm,
                                                                      kind, monkeypatch):
    from warp_drive_b200.training.algorithms import policygradient as pg

    calls = {"pg": 0, "ppo": 0}
    real_pg, real_ppo = pg.fused_gaussian_pg_loss, pg.fused_ppo_loss

    def spy_pg(*a, **k):
        calls["pg"] += 1
        return real_pg(*a, **k)

    def spy_ppo(*a, **k):
        assert k.get("log_std") is not None
        calls["ppo"] += 1
        return real_ppo(*a, **k)
    monkeypatch.setattr(pg, "fused_gaussian_pg_loss", spy_pg)
    monkeypatch.setattr(pg, "fused_ppo_loss", spy_ppo)
    keys = (dict(num_epochs=2, num_mini_batches=4, gae_lambda=0.95) if algorithm == "PPO"
            else {})
    params = []
    for native in (True, False):
        if kind == "recall":
            tr = _recall(tmp_path, f"u{algorithm}{native}", algorithm=algorithm, seed=11,
                         ppo_steps=(2, 4))
        else:
            tr = _reach(tmp_path, f"u{algorithm}{native}", True, algo=algorithm, **keys)
        if not native:
            tr.engine.native_gru.clear()
        tr._reset_all_envs()
        tr.engine.resync_observations()
        tr._generate_rollout_batch()
        tr._update_model_params(0)
        torch.cuda.synchronize()
        params.append([q.detach().clone() for p in tr.policies
                       for q in tr.models[p].parameters()])
    for a, b in zip(*params):
        torch.testing.assert_close(a, b, rtol=0, atol=1e-5)
    if algorithm == "PPO":
        assert calls["ppo"] > 0 and calls["pg"] == 0
    else:
        assert calls["pg"] > 0 and calls["ppo"] == 0


def test_checkpoints_hold_weights_and_log_std_only(tmp_path):
    tr = _reach(tmp_path, "ck", True, use_cuda_graph=False)
    tr.engine.rollout()
    for p, m in tr.models.items():
        names = set(m.state_dict())
        assert "log_std" in names and not any("hidden" in n for n in names)


# ------------------------------------------------------------------------ Pendulum
def test_pendulum_run_config_trains_an_iteration_on_the_generic_path(tmp_path):
    from test_gpu_ppo import _pendulum_trainer

    tr = _pendulum_trainer(tmp_path, "pend", config="single_pendulum_ppo_gru", E=256, T=16,
                           L=32, iters=2)
    eng = tr.engine
    assert eng.sa is None and eng.fused is None and eng.recurrent
    assert "shared" in eng.native_gru                 # 256 rows: under the routing cut
    assert tr.models["shared"].is_gaussian and tr._minibatch_steps == 16
    tr.train()
    m = tr.models["shared"]
    assert all(torch.isfinite(q).all() for q in m.parameters())
    recs = [json.loads(l) for l in open(os.path.join(tr.save_dir, "results.json"))]
    assert len(recs) == tr.num_iters and np.isfinite(recs[-1]["shared"]["Mean episodic reward"])


# ------------------------------------------------------------------------ learning
# Measured on an H100 80GB HBM3 (700 W power limit) with scripts/continuous_recall_gru_learning.py
# (seed 7, E = 256, 2 agents, T = 8, PPO 4 x 4, lr 3e-3, 300 iterations): a mean last-step
# reward of -0.188 for the recurrent policy and -0.801 for the feed-forward one, against the
# memoryless bound of -0.8.  The test asks the recurrent policy for better than -0.5 (over half
# its measured gain on the bound) and the feed-forward one for no more than -0.75.
LEARN_ITERS = 300
RECURRENT_THRESHOLD = -0.5
MEMORYLESS_NOISE = 0.05


def test_recurrent_gaussian_policy_learns_to_recall_the_cue(tmp_path):
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "scripts"))
    from continuous_recall_env import MEMORYLESS_BOUND, make_trainer
    from continuous_recall_gru_learning import MODELS, last_step_reward

    got = {}
    for name, model in MODELS.items():
        tr = make_trainer(model, name, str(tmp_path), seed=7, iterations=LEARN_ITERS)
        tr.train()
        got[name] = last_step_reward(tr)
    print(f"continuous recall: {got}")
    assert got["fully_connected_gaussian_gru"] > RECURRENT_THRESHOLD, got
    assert got["fully_connected_gaussian"] < MEMORYLESS_BOUND + MEMORYLESS_NOISE, got
