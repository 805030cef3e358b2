"""GPU tests of multi-epoch PPO over shuffled minibatches.

Kernels: wdb_gae, wdb_ppo_loss_and_grads and wdb_ppo_gaussian_loss_and_grads within the
float32 running-error bars of the float64 reference (ppo_reference.py) across their shape
envelope -- 1-4 heads, widths up to 399, A up to 8, B not a multiple of 32, row lists in random
order, done = 0 / 1 / 2 -- with a guard region around every output, the log_std gradient
bit-identical on relaunch, and the *_supported checks refusing what the launches refuse.
Trainer: the 1 x 1, lambda = 1 step equals the existing fused update; a policy without the new
keys never reaches the new code; each epoch's minibatches cover every row once, reproducibly;
runs on every rollout path end with finite parameters and metrics; PPO with GAE learns
Pendulum; two ranks stay identical."""
import ctypes
import json
import os
import socket
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "custom_env"))

import ppo_reference as ref  # noqa: E402
from update_reference import within  # noqa: E402

GUARD = 64
SENTINEL = 12345.0


def _wlib():
    from warp_drive_b200 import lib as wlib

    return wlib


def _guarded(shape, dtype=torch.float32):
    n = int(np.prod(shape))
    buf = torch.full((2 * GUARD + n,), SENTINEL, dtype=dtype, device="cuda")
    return buf, buf[GUARD:GUARD + n].view(*shape)


def _intact(buf):
    return bool((buf[:GUARD] == SENTINEL).all() and (buf[-GUARD:] == SENTINEL).all())


def _check(name, got, want, mask=None):
    k = got.double().cpu().numpy()
    v, b = want
    if mask is not None:
        k, v, b = k[mask], v[mask], b[mask]
    worst, i = within(k, (v, b))
    assert worst <= 0, (name, worst, i)


# ---------------------------------------------------------------------------------- GAE
@pytest.mark.parametrize("T,E,Np,lam,p_done", [
    (1, 33, 1, 0.95, 0.5), (7, 100, 3, 0.0, 0.2), (16, 1000, 1, 0.95, 0.1),
    (5, 31, 4, 1.0, 1.0), (40, 257, 2, 0.8, 0.05), (12, 10000, 1, 0.95, 0.0)])
def test_gae_is_within_running_error_bars_of_float64(T, E, Np, lam, p_done):
    wl = _wlib()
    g = torch.Generator(device="cuda").manual_seed(T * 1000 + E)
    rewards = torch.randn((T, E, Np), device="cuda", generator=g)
    values = torch.randn((T, E, Np), device="cuda", generator=g)
    done = ((torch.rand((T, E), device="cuda", generator=g) < p_done).int()
            * torch.randint(1, 3, (T, E), device="cuda", generator=g, dtype=torch.int32))
    ab, adv = _guarded((T, E, Np))
    vb, vt = _guarded((T, E, Np))
    G = wl.GaeArgs()
    G.T, G.n_envs, G.n_agents = T, E, Np
    G.rewards, G.values, G.done = wl.ptr(rewards), wl.ptr(values), wl.ptr(done)
    G.gamma, G.gae_lambda = 0.97, lam
    G.advantages, G.value_targets = wl.ptr(adv), wl.ptr(vt)
    wl.check(wl.load().wdb_gae(wl.stream_ptr(), ctypes.byref(G)), "gae")
    torch.cuda.synchronize()
    ra, rv = ref.gae(rewards.cpu().numpy(), values.cpu().numpy(), done.cpu().numpy(), 0.97, lam)
    _check("advantages", adv, ra)
    _check("value_targets", vt, rv)
    assert _intact(ab) and _intact(vb)
    # the trainer's wrapper gives the same bits
    from warp_drive_b200.training.algorithms.policygradient import gae

    a2, v2 = gae(rewards, done, values, 0.97, lam)
    assert torch.equal(a2, adv) and torch.equal(v2, vt)


# ------------------------------------------------------------------------- minibatch loss
def _flat_inputs(R, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    adv = torch.randn(R, device="cuda", generator=g)
    adv[::11] = 0.0
    vt = torch.randn(R, device="cuda", generator=g)
    return g, adv, vt


class _Batch:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def _cat_probs(B, widths, g):
    probs = []
    for A in widths:
        p = torch.softmax(2.0 * torch.randn((B, A), device="cuda", generator=g), -1)
        if A > 1:
            p[::7, 0] = 0.0                           # masked action
        probs.append(p.contiguous())
    return probs


def _launch_cat(probs, values, rows, actions, batch, ppo, clip, vf, ent, with_grads=True,
                old=True):
    wl = _wlib()
    B = int(probs[0].shape[0])
    L = wl.PpoLoss()
    L.B, L.n_heads = B, len(probs)
    out = {"g": [], "gb": []}
    for k, p in enumerate(probs):
        L.n_actions[k] = int(p.shape[-1])
        L.probs[k] = wl.ptr(p)
        if with_grads:
            buf, gp = _guarded(tuple(p.shape))
            out["g"].append(gp)
            out["gb"].append(buf)
            L.grad_probs[k] = wl.ptr(gp)
    lb, lp = _guarded((B,))
    out["log_prob"], out["lb"] = lp, lb
    L.log_prob = wl.ptr(lp)
    L.rows, L.actions = wl.ptr(rows), wl.ptr(actions)
    if old:
        vb, gv = _guarded((B,))
        out["gv"], out["vb"] = gv, vb
        sums = torch.zeros(5, dtype=torch.float64, device="cuda")
        out["sums"] = sums
        L.values, L.advantages, L.value_targets = (wl.ptr(values), wl.ptr(batch.advantages),
                                                   wl.ptr(batch.value_targets))
        L.old_log_prob, L.sums = wl.ptr(batch.old_log_prob), wl.ptr(sums)
        if with_grads:
            L.grad_values = wl.ptr(gv)
    L.ppo, L.clip_param, L.vf_coeff, L.entropy_coeff = int(ppo), clip, vf, ent
    rc = wl.load().wdb_ppo_loss_and_grads(wl.stream_ptr(), ctypes.byref(L))
    torch.cuda.synchronize()
    return rc, out


CAT_CASES = [([3], 100), ([2, 5], 257), ([399], 45), ([21, 21, 1, 7], 1000), ([4, 399, 2], 63),
             ([1], 31)]


@pytest.mark.parametrize("widths,B", CAT_CASES)
@pytest.mark.parametrize("ppo", [True, False])
def test_categorical_ppo_loss_is_within_running_error_bars(widths, B, ppo):
    R = 3 * B + 5
    g, adv, vt = _flat_inputs(R, seed=B + len(widths))
    H = len(widths)
    actions = torch.stack([torch.randint(0, A, (R,), device="cuda", generator=g,
                                         dtype=torch.int32) for A in widths], -1).contiguous()
    rows = torch.randperm(R, device="cuda", generator=g)[:B].to(torch.int32)
    probs = _cat_probs(B, widths, g)
    for k, A in enumerate(widths):                     # never take a masked action
        if A > 1:
            a = actions[rows.long(), k]
            actions[rows.long()[::7], k] = torch.where(a[::7] == 0, 1, a[::7])
    values = torch.randn(B, device="cuda", generator=g)
    # old log-probs: the kernel's own pre-pass on the same rows (rho == 1 exactly) on a third,
    # shifted elsewhere so that rho spreads across and beyond the clip interval
    rc, pre = _launch_cat(probs, None, rows, actions, None, ppo, 0.2, 0.5, 0.01,
                          with_grads=False, old=False)
    assert rc == 0 and _intact(pre["lb"])
    old = torch.randn(R, device="cuda", generator=g)
    shift = 0.4 * torch.randn(B, device="cuda", generator=g)
    shift[::3] = 0.0
    old[rows.long()] = pre["log_prob"] + shift
    batch = _Batch(advantages=adv, value_targets=vt, old_log_prob=old)
    rc, out = _launch_cat(probs, values, rows, actions, batch, ppo, 0.2, 0.5, 0.01)
    assert rc == 0
    assert torch.equal(out["log_prob"], pre["log_prob"])
    idx = rows.long().cpu().numpy()
    r = ref.ppo_loss([p.cpu().numpy() for p in probs], values.cpu().numpy(),
                     actions.cpu().numpy()[idx], adv.cpu().numpy()[idx], vt.cpu().numpy()[idx],
                     old.cpu().numpy()[idx], ppo, 0.2, 0.5, 0.01)
    dec = r["decided"]
    assert dec.mean() > 0.9, dec.mean()
    _check("log_prob", out["log_prob"], r["logp"])
    _check("grad_values", out["gv"], r["grad_values"])
    for k in range(H):
        _check(f"grad_probs[{k}]", out["g"][k], r["grad_probs"][k], dec)
        assert _intact(out["gb"][k])
    assert _intact(out["vb"]) and _intact(out["lb"])
    sums = out["sums"].cpu().numpy()
    for k in range(4):
        v, b = r["sums"][k]
        assert abs(sums[k] - v) <= b, (k, sums[k], v, b)
    count, unsure = r["sums"][4]
    assert abs(sums[4] - count) <= unsure
    if ppo:
        assert (out["log_prob"][::3] - old[rows.long()][::3] == 0).all()


def _launch_gauss(mean, log_std, values, rows, actions, batch, ppo, clip, vf, ent, old=True):
    wl = _wlib()
    B, A = mean.shape
    L = wl.PpoGaussianLoss()
    L.B, L.action_dim = B, A
    L.mean, L.log_std, L.rows, L.actions = (wl.ptr(mean), wl.ptr(log_std), wl.ptr(rows),
                                            wl.ptr(actions))
    out = {}
    lb, lp = _guarded((B,))
    out["log_prob"], out["lb"] = lp, lb
    L.log_prob = wl.ptr(lp)
    if old:
        mb, gm = _guarded((B, A))
        sb, gs = _guarded((A,))
        vb, gv = _guarded((B,))
        sums = torch.zeros(5, dtype=torch.float64, device="cuda")
        partials = torch.empty((-(-B // wl.PG_GAUSSIAN_ROWS_PER_CTA), A), dtype=torch.float64,
                               device="cuda")
        out.update(gm=gm, mb=mb, gs=gs, sb=sb, gv=gv, vb=vb, sums=sums)
        L.values, L.advantages, L.value_targets = (wl.ptr(values), wl.ptr(batch.advantages),
                                                   wl.ptr(batch.value_targets))
        L.old_log_prob, L.sums, L.partials = wl.ptr(batch.old_log_prob), wl.ptr(sums), wl.ptr(
            partials)
        L.grad_mean, L.grad_log_std, L.grad_values = wl.ptr(gm), wl.ptr(gs), wl.ptr(gv)
    L.ppo, L.clip_param, L.vf_coeff, L.entropy_coeff = int(ppo), clip, vf, ent
    rc = wl.load().wdb_ppo_gaussian_loss_and_grads(wl.stream_ptr(), ctypes.byref(L))
    torch.cuda.synchronize()
    return rc, out


def _gauss_setup(B, A, seed):
    R = 2 * B + 3
    g, adv, vt = _flat_inputs(R, seed)
    mean = torch.randn((B, A), device="cuda", generator=g)
    log_std = (0.5 * torch.randn(A, device="cuda", generator=g)).contiguous()
    actions = torch.randn((R, A), device="cuda", generator=g)
    rows = torch.randperm(R, device="cuda", generator=g)[:B].to(torch.int32)
    actions[rows.long()] = mean + log_std.exp() * torch.randn((B, A), device="cuda", generator=g)
    values = torch.randn(B, device="cuda", generator=g)
    rc, pre = _launch_gauss(mean, log_std, None, rows, actions, None, True, 0.2, 0.5, 0.01,
                            old=False)
    assert rc == 0 and _intact(pre["lb"])
    old = torch.randn(R, device="cuda", generator=g)
    shift = 0.3 * torch.randn(B, device="cuda", generator=g)
    shift[::3] = 0.0
    old[rows.long()] = pre["log_prob"] + shift
    return mean, log_std, values, rows, actions, _Batch(advantages=adv, value_targets=vt,
                                                        old_log_prob=old)


@pytest.mark.parametrize("B,A", [(100, 1), (257, 2), (33, 8), (1000, 3), (4097, 1)])
@pytest.mark.parametrize("ppo", [True, False])
def test_gaussian_ppo_loss_is_within_running_error_bars(B, A, ppo):
    mean, log_std, values, rows, actions, batch = _gauss_setup(B, A, seed=B + A)
    rc, out = _launch_gauss(mean, log_std, values, rows, actions, batch, ppo, 0.2, 0.5, 0.01)
    assert rc == 0
    idx = rows.long().cpu().numpy()
    r = ref.ppo_gaussian_loss(mean.cpu().numpy(), log_std.cpu().numpy(), values.cpu().numpy(),
                              actions.cpu().numpy()[idx], batch.advantages.cpu().numpy()[idx],
                              batch.value_targets.cpu().numpy()[idx],
                              batch.old_log_prob.cpu().numpy()[idx], ppo, 0.2, 0.5, 0.01)
    dec = r["decided"]
    assert dec.mean() > 0.9
    _check("log_prob", out["log_prob"], r["logp"])
    _check("grad_values", out["gv"], r["grad_values"])
    _check("grad_mean", out["gm"], r["grad_mean"], dec)
    # an undecided row's weight lies between 0 and |A| rho whichever branch the kernel took:
    # widen the log_std bar by that row's largest possible contribution
    a_np = actions.cpu().numpy()[idx].astype(np.float64)
    z = (a_np - mean.cpu().numpy()) * np.exp(-log_std.cpu().numpy().astype(np.float64))
    w_max = np.abs(batch.advantages.cpu().numpy()[idx]) * r["rho"][0] * (1 + 1e-5)
    extra = (w_max[:, None] * np.abs(z * z - 1.0))[~dec].sum(0) / B
    v, b = r["grad_log_std"]
    _check("grad_log_std", out["gs"], (v, b + extra))
    for k in ("lb", "mb", "sb", "vb"):
        assert _intact(out[k]), k
    sums = out["sums"].cpu().numpy()
    for k in range(4):
        v, b = r["sums"][k]
        assert abs(sums[k] - v) <= b, (k, sums[k], v, b)
    assert abs(sums[4] - r["sums"][4][0]) <= r["sums"][4][1]


def test_gaussian_log_std_gradient_is_bit_identical_on_relaunch():
    mean, log_std, values, rows, actions, batch = _gauss_setup(20000, 3, seed=5)
    first = _launch_gauss(mean, log_std, values, rows, actions, batch, True, 0.2, 0.5, 0.01)[1]
    for _ in range(3):
        again = _launch_gauss(mean, log_std, values, rows, actions, batch, True, 0.2, 0.5,
                              0.01)[1]
        assert torch.equal(first["gs"], again["gs"])
        assert torch.equal(first["gm"], again["gm"]) and torch.equal(first["gv"], again["gv"])


def test_supported_and_the_launches_refuse_the_same_shapes():
    wl = _wlib()
    L = wl.load()
    g = torch.Generator(device="cuda").manual_seed(0)
    for widths in ([0], [400], [3, 400], [1, 2, 3, 4, 5], [399], [1, 2, 3, 4]):
        arr = (ctypes.c_int * len(widths))(*widths)
        sup = bool(L.wdb_ppo_loss_supported(len(widths), arr))
        assert sup == bool(L.wdb_pg_loss_supported(len(widths), arr))
        heads = widths[:4]
        probs = [torch.full((40, max(a, 1)), 1.0 / max(a, 1), device="cuda") for a in heads]
        actions = torch.zeros((40, len(heads)), dtype=torch.int32, device="cuda")
        P = wl.PpoLoss()
        P.B, P.n_heads = 40, len(widths)
        for k, a in enumerate(heads):
            P.n_actions[k], P.probs[k] = a, wl.ptr(probs[k])
        lp = torch.empty(40, device="cuda")
        P.actions, P.log_prob = wl.ptr(actions), wl.ptr(lp)
        rc = L.wdb_ppo_loss_and_grads(wl.stream_ptr(), ctypes.byref(P))
        assert (rc == 0) == sup, (widths, rc)
    for A in (0, 1, 8, 9):
        sup = bool(L.wdb_ppo_gaussian_loss_supported(A))
        mean = torch.zeros((40, max(A, 1)), device="cuda")
        ls = torch.zeros(max(A, 1), device="cuda")
        lp = torch.empty(40, device="cuda")
        P = wl.PpoGaussianLoss()
        P.B, P.action_dim = 40, A
        P.mean, P.log_std, P.actions, P.log_prob = wl.ptr(mean), wl.ptr(ls), wl.ptr(mean), wl.ptr(
            lp)
        rc = L.wdb_ppo_gaussian_loss_and_grads(wl.stream_ptr(), ctypes.byref(P))
        assert (rc == 0) == sup == (1 <= A <= 8), (A, rc)
    # a loss launch missing an input, and a pre-pass asking for gradients, are refused
    probs = [torch.full((40, 3), 1 / 3, device="cuda")]
    P = wl.PpoLoss()
    P.B, P.n_heads, P.n_actions[0], P.probs[0] = 40, 1, 3, wl.ptr(probs[0])
    P.actions = wl.ptr(torch.zeros((40, 1), dtype=torch.int32, device="cuda"))
    P.old_log_prob = wl.ptr(torch.zeros(40, device="cuda"))
    assert L.wdb_ppo_loss_and_grads(wl.stream_ptr(), ctypes.byref(P)) != 0
    P.old_log_prob = None
    P.log_prob = wl.ptr(torch.zeros(40, device="cuda"))
    P.grad_probs[0] = wl.ptr(torch.zeros((40, 3), device="cuda"))
    assert L.wdb_ppo_loss_and_grads(wl.stream_ptr(), ctypes.byref(P)) != 0
    del g


def test_fused_minibatch_loss_agrees_with_the_torch_expression():
    from warp_drive_b200.training.algorithms.fused_loss import fused_ppo_loss
    from warp_drive_b200.training.algorithms.policygradient import ppo_minibatch_loss

    R, B = 999, 250
    g, adv, vt = _flat_inputs(R, seed=3)
    actions = torch.stack([torch.randint(0, A, (R,), device="cuda", generator=g,
                                         dtype=torch.int32) for A in (5, 3)], -1).contiguous()
    rows = torch.randperm(R, device="cuda", generator=g)[:B].to(torch.int32)
    probs = [torch.softmax(torch.randn((B, A), device="cuda", generator=g), -1) for A in (5, 3)]
    values = torch.randn(B, device="cuda", generator=g)
    old = torch.randn(R, device="cuda", generator=g) - 2.0
    batch = _Batch(actions=actions, advantages=adv, value_targets=vt, old_log_prob=old)
    out = []
    for fused in (True, False):
        P = [p.clone().requires_grad_() for p in probs]
        V = values.clone().requires_grad_()
        if fused:
            loss, sums = fused_ppo_loss(V, P, rows, batch, True, 0.2, 0.5, 0.01)
        else:
            i = rows.long()
            loss, sums = ppo_minibatch_loss(P, V, actions[i], adv[i], vt[i], old[i], True, 0.2,
                                            0.5, 0.01)
        loss.backward()
        out.append((loss.detach(), sums, [p.grad for p in P], V.grad))
    (la, sa, pa, va), (lb, sb, pb, vb) = out
    assert torch.allclose(la, lb, rtol=1e-5, atol=1e-6)
    assert torch.allclose(sa[:4], sb[:4], rtol=1e-5, atol=1e-4)
    assert torch.allclose(va, vb, rtol=1e-5, atol=1e-7)
    for a, b in zip(pa, pb):
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6), float((a - b).abs().max())


# ---------------------------------------------------------------------------------- trainer
def _policy_keys(cfg, **keys):
    for p in cfg["policy"].values():
        p.update(keys)
    return cfg


def _cartpole_trainer(tmp_path, name, iters=3, E=256, T=16, **keys):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.cartpole import CUDAClassicControlCartPoleEnv
    from warp_drive_b200.training.trainer import Trainer, load_run_config

    cfg = load_run_config("single_cartpole")
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T,
                          num_episodes=-(-E * T * iters // 100), seed=3)
    cfg["env"].update(episode_length=100, reset_pool_size=64)
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1, model_params_save_freq=100)
    _policy_keys(cfg, algorithm="PPO", **keys)
    env = CUDAClassicControlCartPoleEnv(**cfg["env"])
    wrapper = EnvWrapper(env, num_envs=E, env_backend="numba")
    return Trainer(env_wrapper=wrapper, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                   results_dir=name, verbose=False)


def _pendulum_trainer(tmp_path, name, config="single_pendulum_ppo", E=256, T=16, L=32, iters=3,
                      seed=7, **keys):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent import classic_control as cc
    from warp_drive_b200.training.trainer import Trainer, load_run_config

    cfg = load_run_config(config)
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, num_episodes=E * T * iters // L,
                          seed=seed)
    cfg["env"].update(episode_length=L, reset_pool_size=64)
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1, model_params_save_freq=1000)
    _policy_keys(cfg, **keys)
    env = cc.CUDAClassicControlPendulumEnv(**cfg["env"])
    wrapper = EnvWrapper(env, num_envs=E, env_backend="numba")
    return Trainer(env_wrapper=wrapper, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                   results_dir=name, verbose=False)


def _records(trainer):
    return [json.loads(l) for l in open(os.path.join(trainer.save_dir, "results.json"))]


def _check_finite_run(trainer, ppo=True):
    trainer.train()
    for p in trainer.policies_to_train:
        assert all(torch.isfinite(q).all() for q in trainer.models[p].parameters()), p
    recs = _records(trainer)
    assert len(recs) == trainer.num_iters
    keys = ["Total loss", "Policy loss", "Value function loss", "Mean entropy", "Approx. KL",
            "Mean episodic reward"] + (["Clip fraction"] if ppo else [])
    for rec in recs:
        for p in trainer.policies_to_train:
            for k in keys:
                assert np.isfinite(rec[p][k]), (p, k, rec[p])
    return recs


def _capture_adam(trainer, captured):
    """Replace each policy's Adam step by a capture of its gradient arena (parameters stay)."""
    for p in trainer.policies_to_train:
        opt = trainer.optimizers[p]

        def fake_step(max_grad_norm=None, _opt=opt, _p=p):
            captured[_p] = _opt.grads.clone()
        opt.step = fake_step


def test_one_epoch_one_minibatch_at_lambda_one_equals_the_existing_update(tmp_path):
    """On one rollout batch, from identical parameters: the existing fused update and PPO with
    1 x 1 and gae_lambda = 1 on the new path give the same parameter gradient (the value
    targets are the discounted returns, and the old log-probs come from the same fused training
    forward as the step's, so rho is 1 up to the order of the permuted rows)."""
    from warp_drive_b200.training.algorithms import policygradient as pg

    t = _cartpole_trainer(tmp_path, "eq")
    assert t._minibatch_steps is None
    grads = {}
    _capture_adam(t, grads)
    t.cuda_envs.reset_all_envs()
    t.engine.resync_observations()
    t._generate_rollout_batch()
    t._update_model_params(0)
    old = grads["shared"]
    obj = t.trainers["shared"]
    obj.gae_lambda, obj.minibatch_path = 1.0, True
    t._minibatch_steps = t._minibatch_schedule()
    assert t._minibatch_steps == 1
    rhos = []
    real = pg.fused_ppo_loss

    def spy(values, probs, rows, batch, *a, **kw):
        logp = pg.fused_log_prob(probs, batch.actions[rows.long()].contiguous())
        rhos.append(float((torch.exp(logp - batch.old_log_prob[rows.long()]) - 1).abs().max()))
        return real(values, probs, rows, batch, *a, **kw)
    pg.fused_ppo_loss = spy
    try:
        t._update_model_params(1)
    finally:
        pg.fused_ppo_loss = real
    new = grads["shared"]
    assert float((old - new).norm() / old.norm()) <= 1e-5, float((old - new).norm() / old.norm())
    assert len(rhos) == 1 and rhos[0] <= 1e-5, rhos


def test_a_policy_without_the_new_keys_never_reaches_the_new_code(tmp_path, monkeypatch):
    from warp_drive_b200.training.algorithms import policygradient as pg

    def boom(*a, **kw):
        raise AssertionError("the minibatch update ran")
    monkeypatch.setattr(pg._PolicyGradient, "prepare_batch", boom)
    monkeypatch.setattr(pg._PolicyGradient, "minibatch_loss", boom)
    trainer = _cartpole_trainer(tmp_path, "plain", iters=2)
    assert trainer._minibatch_steps is None
    trainer.train()
    assert trainer.num_iters == 2


def test_each_epoch_covers_every_row_once_and_the_seed_fixes_the_order(tmp_path):
    from warp_drive_b200.training.algorithms import policygradient as pg

    seen = []
    real = pg._PolicyGradient.minibatch_loss

    def spy(self, model, batch, rows, timestep):
        seen.append(rows.clone())
        return real(self, model, batch, rows, timestep)
    pg._PolicyGradient.minibatch_loss = spy
    try:
        orders = []
        for name in ("a", "b"):
            seen.clear()
            t = _cartpole_trainer(tmp_path, name, iters=1, E=100, T=10, num_epochs=3,
                                  num_mini_batches=4, gae_lambda=0.95)
            t.train()
            orders.append([s.cpu() for s in seen])
    finally:
        pg._PolicyGradient.minibatch_loss = real
    R = 100 * 10
    for order in orders:
        assert len(order) == 12
        for e in range(3):
            chunk = order[4 * e:4 * e + 4]
            assert sorted(len(c) for c in chunk) == [250] * 4
            assert torch.equal(torch.sort(torch.cat(chunk).long()).values, torch.arange(R))
        assert not torch.equal(order[0], order[4])      # each epoch draws its own order
    for x, y in zip(*orders):
        assert torch.equal(x, y)


def test_neg_pos_env_ratio_is_refused_on_the_new_path(tmp_path):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.cartpole import CUDAClassicControlCartPoleEnv
    from warp_drive_b200.training.trainer import Trainer, load_run_config

    cfg = load_run_config("single_cartpole")
    cfg["trainer"].update(num_envs=64, train_batch_size=64 * 10, num_episodes=20, seed=3,
                          neg_pos_env_ratio=2)
    cfg["saving"].update(basedir=str(tmp_path))
    _policy_keys(cfg, algorithm="PPO", num_epochs=2)
    env = CUDAClassicControlCartPoleEnv(**cfg["env"])
    with pytest.raises(ValueError, match="neg_pos_env_ratio"):
        Trainer(env_wrapper=EnvWrapper(env, num_envs=64, env_backend="numba"), config=cfg,
                policy_tag_to_agent_id_map={"shared": [0]}, results_dir="n", verbose=False)


NEW = dict(num_epochs=2, num_mini_batches=3, gae_lambda=0.95, normalize_advantage=True)


def test_train_cartpole_one_launch_rollout_on_the_new_path(tmp_path):
    t = _cartpole_trainer(tmp_path, "cp", **NEW)
    assert t.engine.sa is not None
    _check_finite_run(t)


def test_train_pendulum_one_launch_gaussian_rollout_on_the_new_path(tmp_path):
    t = _pendulum_trainer(tmp_path, "pd", **NEW)
    assert t.engine.sa is not None and t.engine.sa.gaussian
    ls0 = t.models["shared"].log_std.detach().clone()
    _check_finite_run(t)
    assert not torch.equal(t.models["shared"].log_std.detach(), ls0)


def test_train_tag_continuous_fused_step_two_policies_on_the_new_path(tmp_path):
    """Runner 2 epochs x 3 minibatches, tagger 3 x 2: six optimizer steps each, and every
    policy's own epochs of its own minibatches each cover that policy's rows exactly once."""
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.tag_continuous import TagContinuous
    from warp_drive_b200.training.algorithms import policygradient as pg
    from warp_drive_b200.training.trainer import Trainer, load_run_config

    cfg = load_run_config("tag_continuous")
    cfg["trainer"].update(num_envs=32, train_batch_size=32 * 25, num_episodes=96, seed=5)
    cfg["env"].update(num_taggers=2, num_runners=10, episode_length=50)
    cfg["saving"].update(basedir=str(tmp_path), metrics_log_freq=1, model_params_save_freq=100)
    _policy_keys(cfg, algorithm="PPO", **NEW)
    cfg["policy"]["tagger"].update(num_epochs=3, num_mini_batches=2)
    env = TagContinuous(**cfg["env"])
    wrapper = EnvWrapper(env, num_envs=32, env_backend="pycuda")
    pm = {"runner": sorted(env.runners), "tagger": sorted(env.taggers)}
    t = Trainer(env_wrapper=wrapper, config=cfg, policy_tag_to_agent_id_map=pm, results_dir="tc",
                verbose=False)
    assert t.engine.fused is not None and t._minibatch_steps == 6
    owner = {id(t.trainers[p]): p for p in t.policies_to_train}
    seen = {p: [] for p in t.policies_to_train}
    real = pg._PolicyGradient.minibatch_loss

    def spy(self, model, batch, rows, timestep):
        seen[owner[id(self)]].append((batch.R, rows.cpu().long()))
        return real(self, model, batch, rows, timestep)
    pg._PolicyGradient.minibatch_loss = spy
    try:
        _check_finite_run(t)
    finally:
        pg._PolicyGradient.minibatch_loss = real
    for p, (epochs, minis) in (("runner", (2, 3)), ("tagger", (3, 2))):
        steps = seen[p]
        assert len(steps) == 6 * t.num_iters, (p, len(steps))
        for it in range(t.num_iters):
            for e in range(epochs):
                chunk = steps[6 * it + minis * e:6 * it + minis * (e + 1)]
                R = chunk[0][0]
                assert len(chunk) == minis
                assert sorted(len(c) for _, c in chunk) == sorted(
                    len(x) for x in torch.tensor_split(torch.arange(R), minis))
                assert torch.equal(torch.sort(torch.cat([c for _, c in chunk])).values,
                                   torch.arange(R)), (p, it, e)


def _with_policy_keys(monkeypatch, **keys):
    """Make the trainer module's load_run_config add `keys` to every policy of the config it
    returns, so that helpers that build their own config take the new path through the real
    config keys and their validation."""
    from warp_drive_b200.training import trainer as trainer_mod

    real = trainer_mod.load_run_config

    def load(name):
        cfg = real(name)
        return _policy_keys(cfg, **keys)
    monkeypatch.setattr(trainer_mod, "load_run_config", load)


def test_train_the_masked_counter_env_on_the_new_path(tmp_path, monkeypatch):
    from test_gpu_masked import _masked_trainer

    from warp_drive_b200.training.algorithms import policygradient as pg

    masks = []
    real = pg._PolicyGradient.prepare_batch

    def spy(self, model, obs, actions, rewards, done, action_mask=None):
        masks.append(action_mask is not None)
        return real(self, model, obs, actions, rewards, done, action_mask)
    pg._PolicyGradient.prepare_batch = spy
    try:
        _with_policy_keys(monkeypatch, num_epochs=2, num_mini_batches=2, gae_lambda=0.9)
        t, _, cfg, _ = _masked_trainer(tmp_path, "PPO", name="mask")
        assert t._minibatch_steps == 4
        _check_finite_run(t)
    finally:
        pg._PolicyGradient.prepare_batch = real
    assert masks and all(masks)
    # no taken action was masked: the old log-probs were finite
    dm = t.cuda_envs.cuda_data_manager
    assert torch.isfinite(dm.data_on_device_via_torch("sampled_actions_batch_even").float()).all()


@pytest.mark.parametrize("layout", ["first", "last"])
def test_train_the_hetero_env_with_separate_placeholders_on_the_new_path(tmp_path, layout,
                                                                         monkeypatch):
    from test_gpu_hetero import _trainer

    _with_policy_keys(monkeypatch, num_epochs=2, num_mini_batches=2, gae_lambda=0.95)
    t, _, pm = _trainer(tmp_path, "PPO", layout=layout, iters=2, name=f"h{layout}")
    assert t._minibatch_steps == 4 and len(t.policies_to_train) == 2
    _check_finite_run(t)


# Measured on an H100 80GB HBM3 (700 W power limit): Pendulum, E = 1024, T = L = 50, seed 7,
# K = 60 iterations; gain = mean episodic reward of the last three iterations minus that of the
# first three.  single_pendulum_ppo_gae.yaml as written (4 epochs x 4 minibatches, GAE(0.95),
# normalised advantages, lr 1e-3): -311.6 -> -229.7, a gain of 81.9.  Today's PPO
# (single_pendulum_ppo.yaml, one step per batch) in the same run: a gain of 1.9 at its own lr
# 3e-4 (-316.2 -> -314.3) and of 8.4 at lr 1e-3 (-309.5 -> -301.1).  Runs of the same seed differ
# (the gradient-norm reduction accumulates with atomics): two more runs of the new config gained
# 45.3 (seed 7) and 43.5 (seed 11).  The test asks for half of the smallest of these gains.
K_ITERS = 60
GAIN_NEW = 43.5


def _pendulum_gain(tmp_path, config, name, **keys):
    t = _pendulum_trainer(tmp_path, name, config=config, E=1024, T=50, L=50, iters=K_ITERS,
                          **keys)
    t.train()
    rewards = [rec["shared"]["Mean episodic reward"] for rec in _records(t)]
    return float(np.mean(rewards[:3])), float(np.mean(rewards[-3:]))


def test_ppo_with_gae_and_minibatches_learns_pendulum(tmp_path):
    first, last = _pendulum_gain(tmp_path, "single_pendulum_ppo_gae", "learn_new")
    print(f"pendulum PPO+GAE (4x4): first {first:.2f} last {last:.2f} gain {last - first:.2f}")
    if os.environ.get("WDB_PPO_MEASURE_BASELINE"):
        for lr in (None, 0.001):
            keys = {} if lr is None else {"lr": lr}
            f0, l0 = _pendulum_gain(tmp_path, "single_pendulum_ppo", f"learn_old{lr}", **keys)
            print(f"pendulum PPO (1x1, lr {lr or 'config'}): first {f0:.2f} last {l0:.2f} "
                  f"gain {l0 - f0:.2f}")
    assert last - first >= 0.5 * GAIN_NEW, (first, last)


# ---------------------------------------------------------------------------------- 2 GPUs
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import copy

    import torch.distributed as dist

    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.tag_continuous import TagContinuous
    from warp_drive_b200.training.trainer import Trainer, load_run_config
    from warp_drive_b200.training.utils.distributed import init_process_group

    torch.cuda.set_device(rank)
    init_process_group("nccl", device_id=rank)
    cfg = load_run_config("tag_continuous")
    cfg["env"].update(num_taggers=2, num_runners=8, episode_length=20)
    cfg["trainer"].update(num_envs=16, train_batch_size=16 * 5, num_episodes=4, seed=7)
    for p in cfg["policy"].values():
        p["model"]["fc_dims"] = [32, 32]
        p.update(algorithm="PPO", num_epochs=2, num_mini_batches=2, gae_lambda=0.95)
    cfg["saving"].update(basedir="/tmp", name="ppo_nccl_test", tag=f"rank{rank}",
                         metrics_log_freq=1000, model_params_save_freq=1000)
    env = TagContinuous(**cfg["env"])
    w = EnvWrapper(env, num_envs=16, env_backend="b200")
    pm = {"runner": sorted(env.runners), "tagger": sorted(env.taggers)}
    tr = Trainer(w, copy.deepcopy(cfg), pm, num_devices=world, device_id=rank, verbose=False)
    tr.train()
    flat = torch.cat([p.detach().reshape(-1) for pol in tr.policies
                      for p in tr.models[pol].parameters()])
    both = [torch.zeros_like(flat) for _ in range(world)]
    dist.all_gather(both, flat)
    out.put((rank, bool(torch.equal(both[0], both[1])), bool(torch.isfinite(flat).all())))
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_hold_identical_parameters_after_minibatch_epochs():
    import torch.multiprocessing as mp

    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, out)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(out.get(timeout=600) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert all(r[1] for r in res) and all(r[2] for r in res)
