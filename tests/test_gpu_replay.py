"""The replay buffer on the GPU: wdb_replay_sample_windows, the five sampled-row passes against
the float64 reference (tests/replay_update_reference.py) and, bit for bit, against the ring
kernels on the ring's regular windows, and the three trainers from a buffer much longer than a
rollout."""
import copy
import math

import numpy as np
import pytest
import torch

import replay_update_reference as ref
from test_ddpg_update_reference_cpu import make_models, make_ring
from test_gpu_ddpg_update_exact import GUARD, SENTINEL, _guarded
from test_sac_cpu import make_sac_models

pytestmark = pytest.mark.gpu

# norm-wise bound of a float32 evaluation against float64, as tests/test_gpu_sac_update_exact.py
REL = 2e-4
DEV = "cuda"


def _rel(got, want):
    got = got.detach().double().cpu().numpy() if torch.is_tensor(got) else np.asarray(got)
    return float(np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30))


def _sample(B, seed, counter, oldest, filled, capacity, n_step, rows):
    from warp_drive_b200 import lib as wlib

    out = torch.full((B, 2), -1, dtype=torch.int32, device=DEV)
    wlib.check(wlib.load().wdb_replay_sample_windows(
        wlib.stream_ptr(), wlib.ptr(out), B, seed, counter, oldest, filled, capacity, n_step,
        rows))
    return out.cpu().numpy().astype(np.int64)


# ------------------------------------------------------------------------ window sampling
@pytest.mark.parametrize("oldest,filled,capacity", [(0, 40, 1000), (777, 1000, 1000),
                                                    (0, 6, 6)])
def test_sampled_windows_stay_inside_the_filled_ring(oldest, filled, capacity):
    n_step, rows = 5, 12
    w = _sample(100000, 3, 1, oldest, filled, capacity, n_step, rows)
    k = (w[:, 0] - oldest) % capacity                  # logical start
    assert k.min() >= 0 and k.max() <= filled - n_step - 1
    assert w[:, 0].min() >= 0 and w[:, 0].max() < capacity
    assert w[:, 1].min() == 0 and w[:, 1].max() == rows - 1
    assert set(k) == set(range(filled - n_step))       # every start is drawn
    assert (w == _sample(100000, 3, 1, oldest, filled, capacity, n_step, rows)).all()
    assert (w != _sample(100000, 3, 2, oldest, filled, capacity, n_step, rows)).any(axis=1).mean() > 0.9
    assert (w != _sample(100000, 4, 1, oldest, filled, capacity, n_step, rows)).any(axis=1).mean() > 0.9


def test_sampled_windows_are_uniform_and_bad_arguments_are_refused():
    from warp_drive_b200 import lib as wlib

    n, starts, rows = 1000000, 50, 20
    w = _sample(n, 11, 7, 30, 64, 64, 14, rows)
    k = (w[:, 0] - 30) % 64
    # binomial counts: 6 standard deviations around n / bins
    for counts, bins in ((np.bincount(k, minlength=starts), starts),
                         (np.bincount(w[:, 1], minlength=rows), rows)):
        p = 1.0 / bins
        assert len(counts) == bins
        assert np.abs(counts - n * p).max() <= 6 * math.sqrt(n * p * (1 - p))
    joint = np.bincount(k * rows + w[:, 1], minlength=starts * rows)
    p = 1.0 / (starts * rows)
    assert np.abs(joint - n * p).max() <= 6 * math.sqrt(n * p * (1 - p))
    out = torch.zeros((8, 2), dtype=torch.int32, device=DEV)
    L, before = wlib.load(), wlib.launch_count()
    for args in ((8, 1, 1, 0, 5, 10, 5, 4),            # filled < n_step + 1
                 (8, 1, 1, 10, 10, 10, 5, 4),          # oldest outside the ring
                 (8, 1, 1, 0, 11, 10, 5, 4),           # filled > capacity
                 (0, 1, 1, 0, 10, 10, 5, 4), (8, 1, 1, 0, 10, 10, 0, 4),
                 (8, 1, 1, 0, 10, 10, 5, 0)):
        assert L.wdb_replay_sample_windows(wlib.stream_ptr(), wlib.ptr(out), *args) == 1
    assert wlib.launch_count() == before


# ------------------------------------------------------------------------ the sampled passes
def _ring32(C, E, Np, F, A, seed):
    ring = make_ring(C, E, Np, F, A, done_slots=(C // 2,), seed=seed)
    return [r.astype(np.float32) if r.dtype != np.int32 else r for r in ring]


def _windows(B, C, EN, seed):
    g = np.random.default_rng(seed)
    w = np.stack([g.integers(0, C, B), g.integers(0, EN, B)], axis=1).astype(np.int32)
    w[0] = (C - 1, EN - 1)                             # wraps the physical end of the ring
    if B > 2:
        w[2] = w[1]                                    # a duplicate
    assert (w[:, 0] >= 0).all() and (w[:, 0] < C).all() and (w[:, 1] < EN).all()
    return w


def _guard_grads(models):
    guards = []
    for m in models:
        for p in m.parameters():
            buf, view = _guarded(p.shape, DEV)
            p.grad = view
            guards.append(buf)
    return guards


def _untouched(guards):
    return all(bool((b[:GUARD] == SENTINEL).all()) and bool((b[-GUARD:] == SENTINEL).all())
               for b in guards)


def _dev(ring):
    return [torch.from_numpy(np.ascontiguousarray(r)).to(DEV) for r in ring]


def _grads(model):
    return [p.grad.clone() for p in model.parameters()]


# (B, n_step, C, E, Np, F, A, actor dims, critic dims): B = 1, B not a multiple of the 16-row
# tile, more rows than CTAs * tile, and more rows than there are distinct windows
SHAPES = [(1, 5, 9, 4, 1, 3, 1, [64, 64], [64, 64]), (37, 5, 40, 6, 1, 3, 1, [64, 64], [64, 64]),
          (4099, 3, 7, 5, 3, 4, 2, [5, 7, 9], [3, 4, 5]), (300, 1, 2, 3, 2, 2, 1, [16], [16])]


@pytest.mark.parametrize("shape", SHAPES, ids=[f"B{s[0]}" for s in SHAPES])
def test_ddpg_sampled_pass_matches_the_float64_reference(shape):
    from warp_drive_b200.training.algorithms.fused_ddpg import FusedDDPGUpdate

    B, n_step, C, E, Np, F, A, ad, cd = shape
    gamma = 0.97
    models = [m.float() for m in make_models(F, A, ad, cd, scale=2.0, bias=0.25, seed=B)]
    ring, windows = _ring32(C, E, Np, F, A, B), _windows(B, C, E * Np, B)
    want = ref.ddpg_sampled(models, ring, windows, n_step, gamma)
    actor, critic, t_actor, t_critic = models = [m.to(DEV) for m in models]
    guards = _guard_grads((actor, critic))
    outs = [_guarded((B,), DEV) for _ in range(3)]
    guards += [b for b, _ in outs]
    fused = FusedDDPGUpdate(*models, E, Np, C, n_step, gamma, replay_rows=B)
    w = torch.from_numpy(windows).to(DEV)
    # the cursor is not read: any value gives the same result
    sums = fused.launch(*_dev(ring), 0, tuple(v for _, v in outs), windows=w).clone()
    first = _grads(actor) + _grads(critic)
    for got, key in zip(first, want["actor_grads"] + want["critic_grads"]):
        assert _rel(got, key) <= REL
    for (_, v), key in zip(outs, ("values", "j_values", "returns")):
        assert _rel(v, want[key]) <= REL, key
    assert float(sums[0]) == pytest.approx(want["sum_sq_err"], rel=REL)
    assert float(sums[1]) == pytest.approx(want["sum_j"], rel=REL, abs=REL * B)
    assert _untouched(guards)
    again = fused.launch(*_dev(ring), C - 1, tuple(v for _, v in outs), windows=w)
    assert all(torch.equal(a, b) for a, b in zip(first, _grads(actor) + _grads(critic)))
    assert torch.equal(sums, again)


def _td3_models(F, A, ad, cd, seed):
    actor, critic, t_actor, t_critic = make_models(F, A, ad, cd, scale=2.0, bias=0.25, seed=seed)
    _, critic2, _, t_critic2 = make_models(F, A, ad, cd, scale=2.0, bias=0.25, seed=seed + 1000)
    return [m.float() for m in (actor, critic, critic2, t_actor, t_critic, t_critic2)]


@pytest.mark.parametrize("shape", SHAPES, ids=[f"B{s[0]}" for s in SHAPES])
def test_td3_sampled_passes_match_the_float64_reference(shape):
    from warp_drive_b200.training.algorithms.fused_td3 import FusedTD3Update
    from warp_drive_b200.training.algorithms.td3 import TD3

    B, n_step, C, E, Np, F, A, ad, cd = shape
    gamma = 0.97
    algo = TD3(gamma, n_step=n_step, target_noise=0.2, target_noise_clip=0.5)
    models = _td3_models(F, A, ad, cd, B)
    actor, critic, critic2, t_actor, t_critic, t_critic2 = models
    ring, windows = _ring32(C, E, Np, F, A, B), _windows(B, C, E * Np, B)
    noise = np.random.default_rng(B).standard_normal((B, A)).astype(np.float32)
    want = ref.td3_critic_sampled(algo, (t_actor, t_critic, t_critic2, critic, critic2), ring,
                                  windows, noise, n_step, gamma)
    awant = ref.td3_actor_sampled((actor, critic), ring, windows, n_step)
    models = [m.to(DEV) for m in models]
    actor, critic, critic2 = models[:3]
    guards = _guard_grads((actor, critic, critic2))
    outs = [_guarded((B,), DEV) for _ in range(4)]
    guards += [b for b, _ in outs]
    fused = FusedTD3Update(algo, *models, E, Np, C, n_step, gamma, replay_rows=B)
    w, eps = torch.from_numpy(windows).to(DEV), torch.from_numpy(noise).to(DEV)
    obs, actions, rewards, done = _dev(ring)

    def launch():
        fused.critic_launch(obs, actions, rewards, done, 0, eps,
                            tuple(v for _, v in outs[:3]), windows=w)
        critics = _grads(critic) + _grads(critic2)
        sums = fused.actor_launch(obs, 0, outs[3][1], windows=w).clone()
        return critics + _grads(actor), sums

    first, sums = launch()
    for got, key in zip(first, want["critic_grads"] + want["critic2_grads"]
                        + awant["actor_grads"]):
        assert _rel(got, key) <= REL
    for (_, v), key in zip(outs[:3], ("q1", "q2", "returns")):
        assert _rel(v, want[key]) <= REL, key
    assert _rel(outs[3][1], awant["j_values"]) <= REL
    assert float(sums[0]) == pytest.approx(want["sums"][0], rel=REL)
    assert float(sums[1]) == pytest.approx(want["sums"][1], rel=REL)
    assert float(sums[2]) == pytest.approx(awant["sum_j"], rel=REL, abs=REL * B)
    assert _untouched(guards)
    again, sums2 = launch()
    assert all(torch.equal(a, b) for a, b in zip(first, again)) and torch.equal(sums, sums2)


@pytest.mark.parametrize("shape", SHAPES, ids=[f"B{s[0]}" for s in SHAPES])
def test_sac_sampled_passes_match_the_float64_reference(shape):
    from warp_drive_b200.training.algorithms.fused_sac import FusedSACUpdate

    B, n_step, C, E, Np, F, A, ad, cd = shape
    gamma, lo, hi = 0.97, -2.0, 1.0
    la32 = np.float32(math.log(0.3))
    models = [m.float() for m in make_sac_models(F, A, ad, cd, seed=B, lo=lo, hi=hi)]
    actor, critic, critic2, t_critic, t_critic2 = models
    ring, windows = _ring32(C, E, Np, F, A, B), _windows(B, C, E * Np, B)
    g = np.random.default_rng(B)
    cn = g.standard_normal((B, A)).astype(np.float32)
    an = g.standard_normal((B, A)).astype(np.float32)
    want = ref.sac_critic_sampled((actor, t_critic, t_critic2, critic, critic2), float(la32),
                                  ring, windows, cn, n_step, gamma)
    awant = ref.sac_actor_sampled((actor, critic, critic2), float(la32), ring, windows, an,
                                  n_step)
    models = [m.to(DEV) for m in models]
    actor, critic, critic2 = models[:3]
    guards = _guard_grads((actor, critic, critic2))
    outs = [_guarded((B,), DEV) for _ in range(4)]
    guards += [b for b, _ in outs]
    log_alpha = torch.tensor([float(la32)], device=DEV)
    fused = FusedSACUpdate(*models, log_alpha, E, Np, C, n_step, gamma, replay_rows=B)
    w = torch.from_numpy(windows).to(DEV)
    eps_c, eps_a = torch.from_numpy(cn).to(DEV), torch.from_numpy(an).to(DEV)
    obs, actions, rewards, done = _dev(ring)

    def launch():
        fused.critic_launch(obs, actions, rewards, done, 0, eps_c,
                            tuple(v for _, v in outs[:3]), windows=w)
        critics = _grads(critic) + _grads(critic2)
        sums = fused.actor_launch(obs, 0, eps_a, outs[3][1], windows=w).clone()
        return critics + _grads(actor), sums

    first, sums = launch()
    for got, key in zip(first, want["critic_grads"] + want["critic2_grads"]
                        + awant["actor_grads"]):
        assert _rel(got, key) <= REL
    for (_, v), key in zip(outs[:3], ("q1", "q2", "returns")):
        assert _rel(v, want[key]) <= REL, key
    assert _rel(outs[3][1], awant["log_probs"]) <= REL
    for i, v in enumerate(want["sums"] + awant["sums"]):
        assert float(sums[i]) == pytest.approx(v, rel=REL, abs=REL * B), i
    assert _untouched(guards)
    again, sums2 = launch()
    assert all(torch.equal(a, b) for a, b in zip(first, again)) and torch.equal(sums, sums2)


def test_sampled_rows_equal_the_ring_kernels_regular_windows_bit_for_bit():
    """windows = every regular window of a short ring in order: the sampled passes' per-row
    outputs are the ring kernels' rows i < valid - 1."""
    from warp_drive_b200.training.algorithms.fused_ddpg import FusedDDPGUpdate
    from warp_drive_b200.training.algorithms.fused_sac import FusedSACUpdate
    from warp_drive_b200.training.algorithms.fused_td3 import FusedTD3Update
    from warp_drive_b200.training.algorithms.td3 import TD3

    n_step, C, cursor, E, Np, F, A, gamma = 5, 12, 7, 6, 2, 3, 1, 0.99
    EN, valid = E * Np, C - n_step + 1
    B = (valid - 1) * EN
    windows = np.array([((cursor + i) % C, n) for i in range(valid - 1) for n in range(EN)],
                       dtype=np.int32)
    w = torch.from_numpy(windows).to(DEV)
    ring = _dev(_ring32(C, E, Np, F, A, 5))
    noise = torch.randn(valid, E, Np, A, device=DEV)
    noise2 = torch.randn(valid, E, Np, A, device=DEV)
    flat = lambda t: t.reshape(valid * EN, -1)[:B].contiguous()  # noqa: E731

    def outs(n, rows):
        return tuple(torch.zeros(rows, device=DEV) for _ in range(n))

    def grads_on(models):
        for m in models:
            for p in m.parameters():
                p.grad = torch.zeros_like(p)

    # DDPG
    models = [m.float().to(DEV) for m in make_models(F, A, [64, 64], [64, 64], 2.0, 0.25, 3)]
    grads_on(models[:2])
    a, b = outs(3, (valid, E, Np)), outs(3, (B,))
    FusedDDPGUpdate(*models, E, Np, C, n_step, gamma).launch(*ring, cursor, a)
    FusedDDPGUpdate(*models, E, Np, C, n_step, gamma, replay_rows=B).launch(
        *ring, 0, b, windows=w)
    for x, y in zip(a, b):
        assert torch.equal(x.reshape(-1)[:B], y)
    # TD3
    algo = TD3(gamma, n_step=n_step)
    models = [m.to(DEV) for m in _td3_models(F, A, [64, 64], [64, 64], 4)]
    grads_on(models[:3])
    a, b = outs(4, (valid, E, Np)), outs(4, (B,))
    fr = FusedTD3Update(algo, *models, E, Np, C, n_step, gamma)
    fs = FusedTD3Update(algo, *models, E, Np, C, n_step, gamma, replay_rows=B)
    fr.critic_launch(*ring, cursor, noise, a[:3])
    fr.actor_launch(ring[0], cursor, a[3])
    fs.critic_launch(*ring, 0, flat(noise), b[:3], windows=w)
    fs.actor_launch(ring[0], 0, b[3], windows=w)
    for x, y in zip(a, b):
        assert torch.equal(x.reshape(-1)[:B], y)
    # SAC
    models = [m.float().to(DEV) for m in make_sac_models(F, A, [64, 64], [64, 64], seed=5,
                                                         lo=-20.0, hi=2.0)]
    grads_on(models[:3])
    la = torch.tensor([math.log(0.2)], device=DEV)
    a, b = outs(4, (valid, E, Np)), outs(4, (B,))
    fr = FusedSACUpdate(*models, la, E, Np, C, n_step, gamma)
    fs = FusedSACUpdate(*models, la, E, Np, C, n_step, gamma, replay_rows=B)
    fr.critic_launch(*ring, cursor, noise, a[:3])
    fr.actor_launch(ring[0], cursor, noise2, a[3])
    fs.critic_launch(*ring, 0, flat(noise), b[:3], windows=w)
    fs.actor_launch(ring[0], 0, flat(noise2), b[3], windows=w)
    for x, y in zip(a, b):
        assert torch.equal(x.reshape(-1)[:B], y)


# ------------------------------------------------------------------------ trainers
_ALGOS = {"DDPG": "single_pendulum", "TD3": "single_pendulum_td3", "SAC": "single_pendulum_sac"}


def _trainer(tmp_path, algo, E=64, T=8, one_launch=True, **replay):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent import classic_control as cc
    from warp_drive_b200.training import trainer_ddpg, trainer_sac, trainer_td3
    from warp_drive_b200.training.trainer import load_run_config

    cfg = load_run_config(_ALGOS[algo])
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, num_episodes=E * 40, seed=11,
                          replay_slots_per_env=203, replay_batch_rows=333,
                          updates_per_iteration=3, replay_warmup_slots=20)
    cfg["trainer"].update(replay)
    cfg["trainer"]["evaluator"] = False
    cfg["env"].update(episode_length=32, reset_pool_size=64)
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1000,
                         model_params_save_freq=100000)
    if not one_launch:       # four hidden layers: the one-launch rollout does not take the actor
        cfg["policy"]["shared"]["model"]["actor"]["fc_dims"] = [16, 16, 16, 16]
    env = cc.CUDAClassicControlPendulumEnv(**cfg["env"])
    w = EnvWrapper(env, num_envs=E, env_backend="numba")
    cls = {"DDPG": trainer_ddpg.TrainerDDPG, "TD3": trainer_td3.TrainerTD3,
           "SAC": trainer_sac.TrainerSAC}[algo]
    return cls(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
               results_dir="r", verbose=False)


def _nets(tr):
    return tr._all_networks("shared")


def _state(tr):
    return ([p.detach().clone() for m in _nets(tr) for p in m.parameters()],
            [copy.deepcopy(o.state_dict()) for _, o, _ in tr._optimizers_of("shared")],
            dict(tr.current_timestep), dict(getattr(tr, "update_count", {})), tr.replay_draws,
            tr._noise_generator.get_state() if getattr(tr, "_noise_generator", None) else None)


def _restore(tr, state):
    params, opts, ts, counts, draws, gen = state
    with torch.no_grad():
        for p, v in zip([p for m in _nets(tr) for p in m.parameters()], params):
            p.copy_(v)
    for (_, o, _), s in zip(tr._optimizers_of("shared"), opts):
        o.load_state_dict(s)
    tr.current_timestep.update(ts)
    if counts:
        tr.update_count.update(counts)
    tr.replay_draws = draws
    if gen is not None:
        tr._noise_generator.set_state(gen)


@pytest.mark.parametrize("algo", list(_ALGOS))
def test_trainer_fused_and_torch_updates_agree_from_the_buffer(algo, tmp_path):
    from warp_drive_b200 import lib as wlib

    tr = _trainer(tmp_path, algo)
    assert tr.ring_capacity == 203 and "shared" in tr.fused_updates
    assert tr.fused_updates["shared"].rows == 333
    before = [p.detach().clone() for m in _nets(tr) for p in m.parameters()]
    for it in (1, 2):                                   # 16 slots < warm-up of 20: no update
        tr._generate_rollout_batch()
        tr._update_model_params(it)
    assert tr.replay_draws == 0
    assert all(torch.equal(a, b) for a, b in
               zip(before, [p for m in _nets(tr) for p in m.parameters()]))
    tr._generate_rollout_batch()
    state = _state(tr)
    results = {}
    for fused in (True, False):
        _restore(tr, state)
        tr.trainers["shared"].use_fused_update = fused
        first = tr._update_model_params(0)["shared"]    # a logging iteration
        for it in range(1, 4):
            tr._update_model_params(it)
        results[fused] = (first, [p.detach().clone() for m in _nets(tr) for p in m.parameters()])
    tr.trainers["shared"].use_fused_update = True
    assert tr.replay_draws == 4 * 3                     # updates_per_iteration = 3
    if algo != "DDPG":
        assert tr.update_count["shared"] == 12          # the delay counts updates
    (mf, pf), (mt, pt) = results[True], results[False]
    for a, b in zip(pf, pt):
        assert torch.isfinite(a).all()
        assert float((a - b).norm() / b.norm().clamp_min(1e-30)) <= 1e-3
    assert mf.keys() == mt.keys() and mf["Replay buffer fill"] == pytest.approx(24 / 203)
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
    # per update: 1 window draw + 2 per pass + clipping norm and Adam (2) per stepped network
    # (SAC's temperature: Adam only)
    per_update = {"DDPG": 1 + 2 + 4, "TD3": None, "SAC": 1 + 4 + 5}[algo]
    if algo == "TD3":          # the actor steps on every second of the 3 updates: 1 or 2 of them
        assert sorted(counts) == [3 * (1 + 2 + 2) + 4, 3 * (1 + 2 + 2) + 8]
    else:
        assert counts == [3 * per_update] * 2


@pytest.mark.parametrize("one_launch", [True, False], ids=["one_launch", "per_step"])
def test_ring_wraps_at_a_capacity_far_above_the_rollout(one_launch, tmp_path):
    """Capacity 203 is no multiple of T = 8: the 26th rollout wraps.  Every slot then holds what
    a trainer with a ring of exactly one rollout recorded for the same timestep."""
    tr = _trainer(tmp_path, "DDPG", E=16, one_launch=one_launch, replay_warmup_slots=203)
    assert (tr.engine.sa is not None) == one_launch
    name = "rewards_batch_shared"
    seen = []
    for it in range(27):
        cursor = tr.engine.ring_cursor
        tr._generate_rollout_batch()
        t = tr.engine._tensor(name)
        seen.append(torch.stack([t[(cursor + k) % 203] for k in range(8)]).clone())
        assert tr.engine.ring_filled == min(203, 8 * (it + 1))
    assert tr.engine.ring_cursor == (27 * 8) % 203
    t = tr.engine._tensor(name)
    flat = torch.cat(seen)                              # timesteps 0 .. 215 in time order
    for step in range(216 - 203, 216):                  # the newest 203 timesteps
        assert torch.equal(t[step % 203], flat[step]), step
    obs = tr.engine._tensor("processed_observations_batch_shared")
    assert torch.isfinite(obs).all() and bool((obs.abs().amax(dim=(1, 2, 3)) > 0).all())
    # the sampler is handed the seam: oldest = cursor once the ring is full
    tr._update_model_params(1)
    w = tr.replay_windows["shared"].cpu().numpy().astype(np.int64)
    k = (w[:, 0] - tr.engine.ring_cursor) % 203
    assert k.max() <= 203 - tr.n_step - 1


def test_more_than_one_agent_per_env(tmp_path):
    """Np = 3 at the trainer's interface: sampled agent rows map to env = row // Np in the
    gather and in the kernels alike (fused and torch gradients of one update agree)."""
    from warp_drive_b200.training.algorithms.ddpg import DDPG
    from warp_drive_b200.training.algorithms.fused_ddpg import FusedDDPGUpdate

    n_step, C, E, Np, F, A, B, gamma = 3, 50, 7, 3, 4, 2, 500, 0.95
    models = [m.float().to(DEV) for m in make_models(F, A, [32, 32], [32, 32], 2.0, 0.0, 9)]
    actor, critic, t_actor, t_critic = models
    ring = _dev(_ring32(C, E, Np, F, A, 9))
    windows = torch.from_numpy(_windows(B, C, E * Np, 9)).to(DEV)
    for m in (actor, critic):
        for p in m.parameters():
            p.grad = torch.zeros_like(p)
    FusedDDPGUpdate(*models, E, Np, C, n_step, gamma, replay_rows=B).launch(
        *ring, 0, windows=windows)
    fused = _grads(actor) + _grads(critic)
    s, n = windows[:, 0].long(), windows[:, 1].long()
    steps = (s[None] + torch.arange(n_step + 1, device=DEV)[:, None]) % C
    obs, actions, rewards, done = ring
    o, bo = obs.reshape(C, -1, F)[s, n], obs.reshape(C, -1, F)[steps[-1], n]
    with torch.no_grad():
        boot = t_critic(obs=bo, action=t_actor(obs=bo))
        returns = DDPG(gamma, n_step=n_step).sampled_returns(
            rewards.reshape(C, -1)[steps[:-1], n], done[steps[:-1], n // Np].float(), boot)
    for m in (actor, critic):
        m.zero_grad()
    values = critic(obs=o, action=actions.reshape(C, -1, A)[s, n])
    j = critic(obs=o, action=actor(obs=o))
    (-j.mean()).backward()
    torch.nn.functional.mse_loss(values, returns).backward()
    for a, b in zip(fused, _grads(actor) + _grads(critic)):
        assert float((a - b).norm() / b.norm().clamp_min(1e-30)) <= 1e-4
