"""Noisy Q networks on the GPU: wdb_noisy_draw against the float64 noise (tests/noisy_reference.py),
wdb_noisy_materialize and wdb_noisy_grads against float64 with guard regions, the native noisy
DQN and C51 updates (plain and dueling) against the float64 reference of the plain pass on their
materialized twin, the sigma = 0 identity, reproducibility, and TrainerDQN with noisy heads on
CartPole -- fused against torch gradients, the launches of a non-logging update, per-env acting
noise and the mean network under use_argmax, the fallback outside the envelope and the Rainbow
config with a checkpoint round-trip."""
import numpy as np
import pytest
import torch

import c51_reference as cref
import dqn_update_reference as dref
import dueling_reference as duel
import noisy_reference as ref
import per_reference as pref
from test_gpu_c51 import _pick as _pick_c51
from test_gpu_c51 import _trainer
from test_gpu_ddpg_update_exact import _guarded
from test_gpu_dqn import _delta_off_the_kink, _dev, _guard_grads, _pick_windows, _rel, _ring32
from test_gpu_dqn import _untouched
from test_noisy_cpu import make_noisy

pytestmark = pytest.mark.gpu

DEV = "cuda"
REL = 2e-4                                 # norm-wise float32 against float64, as C51's tests
SEED = 0x1234567890AB


def _np(t):
    return t.detach().double().cpu().numpy()


def _close(got, want, rel=1e-3, floor=REL):
    """Per element: |got - want| <= rel |want| + floor max |want|."""
    got = _np(got) if torch.is_tensor(got) else got
    bound = rel * np.abs(want) + floor * max(float(np.abs(want).max()), 1e-30)
    return bool((np.abs(got - want) <= bound).all())


def _guard_head(head):
    """Guarded views for a NoisyHead's effective layers and scratch and its layers' noise
    buffers."""
    guards = []
    for group in (head.layers, head.grads or []):
        for i, (w, b) in enumerate(group):
            (gw, vw), (gb, vb) = _guarded(tuple(w.shape), DEV), _guarded(tuple(b.shape), DEV)
            group[i] = (vw, vb)
            guards += [gw, gb]
    for L in head.noisy:
        (gi, vi), (go, vo) = _guarded((L.in_features,), DEV), _guarded((L.out_features,), DEV)
        L.noise_in, L.noise_out = vi, vo
        guards += [gi, go]
    return guards


# ------------------------------------------------------------------------ noise, materialize, grads
def test_draw_matches_the_float64_noise_and_materialize_draws_the_same():
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.fused_dqn import (
        NOISY_ACTING, NOISY_UPDATE, NoisyHead, draw_noise, materialize)

    q = make_noisy(4, 3, 13, [16], 8).float().to(DEV)          # 4 noisy layers
    layers = q.noisy_layers()
    R = 37
    rows = [(_guarded((R, L.in_features), DEV), _guarded((R, L.out_features), DEV))
            for L in layers]
    guards = [g for pair in rows for g, _ in pair]
    count = (5 << 32) + 77                                     # the count's high word is used
    draw_noise(q, SEED, NOISY_ACTING, count, row0=3, rows=[(i, o) for (_, i), (_, o) in rows])
    for l, (L, ((_, fi), (_, fo))) in enumerate(zip(layers, rows)):
        got = np.concatenate([_np(fi), _np(fo)], axis=1)
        for r in (0, 1, R - 1):
            want, bar = ref.noise(SEED, ref.ACTING, count, 3 + r, l, got.shape[1])
            assert (np.abs(got[r] - want) <= bar).all(), (l, r)
        assert len({got[r].tobytes() for r in range(R)}) == R      # every row its own sample
    assert _untouched(guards)
    again = [(torch.empty_like(i), torch.empty_like(o)) for (_, i), (_, o) in rows]
    draw_noise(q, SEED, NOISY_ACTING, count, row0=3, rows=again)
    assert all(torch.equal(a, i) and torch.equal(b, o)
               for (a, b), ((_, i), (_, o)) in zip(again, rows))
    # the update's samples: materialize writes what wdb_noisy_draw draws, bit for bit
    t = make_noisy(4, 3, 13, [16], 8, seed=5).float().to(DEV)
    on, tg = NoisyHead(q, grads=True), NoisyHead(t)
    materialize(on, tg, SEED, 9)
    for row, model in enumerate((q, t)):
        drawn = [(torch.empty_like(L.noise_in), torch.empty_like(L.noise_out))
                 for L in model.noisy_layers()]
        draw_noise(model, SEED, NOISY_UPDATE, 9, row0=row, rows=drawn)
        for L, (i, o) in zip(model.noisy_layers(), drawn):
            assert torch.equal(L.noise_in, i) and torch.equal(L.noise_out, o)
    n0 = wlib.launch_count()
    materialize(on, None, SEED, 9)
    assert wlib.launch_count() - n0 == 1


SHAPES = [(2, 1, None, 64), (3, 51, None, 16), (2, 1, 32, 64), (3, 13, 0, 7), (1, 1, 4, 4)]


@pytest.mark.parametrize("shape", SHAPES, ids=[f"A{a}_N{n}_S{'-' if s is None else s}_H{h}"
                                               for a, n, s, h in SHAPES])
def test_materialize_and_grads_match_float64(shape):
    from warp_drive_b200.training.algorithms.fused_dqn import NoisyHead, materialize, noisy_grads

    A, N, S, H = shape
    q = make_noisy(4, A, N, [H], S, seed=A + N + H).float().to(DEV)
    t = make_noisy(4, A, N, [H], S, seed=99).float().to(DEV)
    with torch.no_grad():                      # sigma of both signs and sizes
        for L in q.noisy_layers() + t.noisy_layers():
            L.weight_sigma.normal_()
            L.bias_sigma.normal_()
    on, tg = NoisyHead(q, grads=True), NoisyHead(t)
    guards = _guard_head(on) + _guard_head(tg) + _guard_grads(q)
    materialize(on, tg, SEED, 3)
    for head in (on, tg):
        for L, (w, b) in zip(head.noisy, head.layers):
            fi, fo = _np(L.noise_in), _np(L.noise_out)
            mw, sw, mb, sb = (_np(p) for p in (L.weight_mu, L.weight_sigma, L.bias_mu,
                                                L.bias_sigma))
            rw, rb = ref.materialize(mw, sw, mb, sb, fi, fo)
            bar_w = 1.2e-7 * (np.abs(sw * np.outer(fo, fi)) + np.abs(rw)) * 1.01
            bar_b = 1.2e-7 * np.abs(rb)
            assert (np.abs(_np(w) - rw) <= bar_w).all() and (np.abs(_np(b) - rb) <= bar_b).all()
    first = [(w.clone(), b.clone()) for w, b in on.layers]
    materialize(on, tg, SEED, 3)
    assert all(torch.equal(a, w) and torch.equal(c, b) for (a, c), (w, b) in zip(first, on.layers))
    g = torch.Generator(device=DEV).manual_seed(A * N + H)
    for w, b in on.grads:
        w.copy_(torch.randn(w.shape, generator=g, device=DEV))
        b.copy_(torch.randn(b.shape, generator=g, device=DEV))
    noisy_grads(on)
    for L, (gw, gb) in zip(on.noisy, on.grads):
        want = ref.grads(_np(gw), _np(gb), _np(L.noise_in), _np(L.noise_out))
        assert torch.equal(L.weight_mu.grad, gw) and torch.equal(L.bias_mu.grad, gb)
        for p, w in ((L.weight_sigma, want[1]), (L.bias_sigma, want[3])):
            assert (np.abs(_np(p.grad) - w) <= 2.5e-7 * np.abs(w)).all()
    assert _untouched(guards)


# ------------------------------------------------------------------------ the update
def _stream_params(layers, S):
    """dueling_reference.stream_params of materialized stream layers (module order)."""
    names = (["value_h", "value_o", "adv_h", "adv_o"] if S else ["value_o", "adv_o"])
    out = {}
    for name, (w, b) in zip(names, layers):
        out[name + "w"], out[name + "b"] = w, b
    return out


def _twins(fused, q_net, dims, F, A, N, categorical):
    """Plain float64 networks holding the trunk and the materialized (folded) head the pass
    runs, read back from the device."""
    from warp_drive_b200.training.algorithms.fused_dqn import folded_widths

    widths = folded_widths(q_net) if q_net.dueling else list(dims)
    pair = (cref.make_c51_models(F, A, widths, N=N, v_min=-3.0, v_max=4.0) if categorical
            else dref.make_q_models(F, A, widths))
    for head, twin in zip((fused.online, fused.target), pair):
        src = head.model
        layers = [(_np(src.fc[str(i)][0].weight), _np(src.fc[str(i)][0].bias))
                  for i in range(len(dims))]
        eff = [(_np(w), _np(b)) for w, b in head.layers]
        if q_net.dueling:
            S = src.policy_head.stream_dim
            eff = duel.fold(_stream_params(eff, S), A, N, S)
        dst = [(twin.fc[str(i)][0].weight, twin.fc[str(i)][0].bias)
               for i in range(len(twin.fc))] + [(twin.policy_head.weight, twin.policy_head.bias)]
        with torch.no_grad():
            for (w, b), (dw, db) in zip(layers + eff, dst):
                dw.copy_(torch.from_numpy(w))
                db.copy_(torch.from_numpy(b))
    return pair


def _noisy_wants(grads, fused, q_net, n_trunk, A, N):
    """The reference gradients of the noisy network's parameters, in parameter order."""
    trunk, head = grads[:2 * n_trunk], grads[2 * n_trunk:]
    head = list(zip(head[0::2], head[1::2]))
    if q_net.dueling:
        S = q_net.policy_head.stream_dim
        u = duel.unfold(head, A, N, S)
        names = ["value_h", "value_o", "adv_h", "adv_o"] if S else ["value_o", "adv_o"]
        head = [(u[n + "w"], u[n + "b"]) for n in names]
    out = list(trunk)
    for L, (gw, gb) in zip(fused.online.noisy, head):
        out += list(ref.grads(gw, gb, _np(L.noise_in), _np(L.noise_out)))
    return out


# (B, n_step, C, E, Np, F, A, N, trunk dims, S); N = 1: DQN; S None: a plain head
GRAD_SHAPES = [(333, 3, 40, 6, 1, 4, 2, 1, [64, 64], None),
               (300, 1, 5, 3, 2, 6, 3, 1, [16], 8),
               (129, 3, 30, 4, 1, 3, 4, 1, [8], 0),
               (333, 3, 40, 6, 1, 4, 2, 51, [64], None),
               (333, 3, 40, 6, 1, 4, 2, 51, [64], 32),
               (200, 1, 12, 4, 1, 4, 3, 13, [16], 0)]


def _setup(shape, weighted, double_q, sigma=True):
    from warp_drive_b200.training.algorithms.dqn import DQN, CategoricalDQN
    from warp_drive_b200.training.algorithms.fused_dqn import (
        FusedNoisyUpdate, fused_noisy_supported, materialize)

    B, n_step, C, E, Np, F, A, N, dims, S = shape
    categorical, gamma = N > 1, 0.97
    extra = {"v_min": -3.0, "v_max": 4.0} if categorical else {}
    q_net = make_noisy(F, A, N, dims, S, seed=B, **extra)
    target = make_noisy(F, A, N, dims, S, seed=B, **extra)
    with torch.no_grad():
        for p in target.parameters():
            p.add_(0.3 * torch.randn_like(p))
        if not sigma:
            for L in q_net.noisy_layers() + target.noisy_layers():
                L.weight_sigma.zero_()
                L.bias_sigma.zero_()
    q_net, target = q_net.float().to(DEV), target.float().to(DEV)
    algo0 = CategoricalDQN(gamma, n_step=n_step) if categorical else DQN(gamma, n_step=n_step)
    assert fused_noisy_supported(algo0, q_net, E, Np, C, B)
    fused = FusedNoisyUpdate(algo0, q_net, target, E, Np, C, B, SEED)
    materialize(fused.online, fused.target, SEED, 7)
    twins = _twins(fused, q_net, dims, F, A, N, categorical)
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
    # the fused update of the algorithm the windows were picked for
    fused = FusedNoisyUpdate(algo, q_net, target, E, Np, C, B, SEED)
    w = torch.from_numpy(windows).to(DEV)
    weights = torch.from_numpy(wts).to(DEV) if weighted else None
    return q_net, target, algo, fused, ring, w, weights, want, want_q


@pytest.mark.parametrize("weighted", [False, True], ids=["uniform", "weighted"])
@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("shape", GRAD_SHAPES, ids=[
    f"{'dqn' if s[7] == 1 else 'c51'}_B{s[0]}_n{s[1]}_A{s[6]}_N{s[7]}_L{len(s[8])}_"
    f"S{'-' if s[9] is None else s[9]}" for s in GRAD_SHAPES])
def test_noisy_update_matches_the_float64_reference(shape, double_q, weighted):
    B, dims, A, N = shape[0], shape[8], shape[6], shape[7]
    q_net, target, algo, fused, ring, w, weights, want, want_q = _setup(shape, weighted, double_q)
    guards = _guard_grads(q_net) + _guard_head(fused.online) + _guard_head(fused.target)
    if q_net.dueling:
        from test_gpu_dueling import _guard_fold
        guards += _guard_fold(fused.fold_online) + _guard_fold(fused.fold_target)
    outs = [_guarded((B,), DEV) for _ in range(2)]
    guards += [b for b, _ in outs]
    sums = fused.launch(*_dev(ring), w, tuple(v for _, v in outs), weights, update=7).clone()
    wants = _noisy_wants(want["grads"], fused, q_net, len(dims), A, N)
    first = [p.grad.clone() for p in q_net.parameters()]
    names = [n for n, _ in q_net.named_parameters()]
    assert len(names) == len(wants)
    for name, got, key in zip(names, first, wants):
        assert _rel(got, key) <= REL, name
        assert _close(got, key), name
    assert _rel(outs[0][1], want_q) <= REL
    assert _untouched(guards)
    again = fused.launch(*_dev(ring), w, tuple(v for _, v in outs), weights, update=7)
    assert all(torch.equal(a, p.grad) for a, p in zip(first, q_net.parameters()))
    assert torch.equal(sums, again)
    if not weighted:                           # unit weights: the unweighted pass bit for bit
        outs2 = [torch.empty(B, device=DEV) for _ in range(2)]
        sums2 = fused.launch(*_dev(ring), w, tuple(outs2), torch.ones(B, device=DEV), update=7)
        assert all(torch.equal(a, p.grad) for a, p in zip(first, q_net.parameters()))
        assert torch.equal(sums2, sums)
        assert torch.equal(outs2[0], outs[0][1]) and torch.equal(outs2[1], outs[1][1])
    # another update draws another sample
    fused.launch(*_dev(ring), w, None, weights, update=8)
    assert not all(torch.equal(a, p.grad) for a, p in zip(first, q_net.parameters()))


def _mean_twin(q_net, S, N):
    """A plain (or plain dueling) float32 network on the device with q_net's trunk and its
    noisy layers' mu."""
    from warp_drive_b200.training.models.fully_connected import ModelFactory

    kind = "fully_connected_q" if N == 1 else "fully_connected_categorical_q"
    cfg = {"type": kind, "fc_dims": list(q_net.fc_dims)}
    if S is not None:
        cfg.update(dueling=True, stream_fc_dims=[S] if S else [])
    if N > 1:
        cfg.update(num_atoms=N, v_min=-3.0, v_max=4.0)
    from test_dueling_cpu import _env
    twin = ModelFactory.create(kind)(env=_env(q_net.flattened_obs_size, q_net.output_dims[0]),
                                     model_config=cfg, policy="shared",
                                     policy_tag_to_agent_id_map={"shared": [0]}).to(DEV)
    plain = [m for m in twin.policy_head.modules() if isinstance(m, torch.nn.Linear)]
    with torch.no_grad():
        for i in range(len(q_net.fc)):
            twin.fc[str(i)][0].weight.copy_(q_net.fc[str(i)][0].weight)
            twin.fc[str(i)][0].bias.copy_(q_net.fc[str(i)][0].bias)
        for dst, L in zip(plain, q_net.noisy_layers()):
            dst.weight.copy_(L.weight_mu)
            dst.bias.copy_(L.bias_mu)
    return twin, plain


@pytest.mark.parametrize("weighted", [False, True], ids=["uniform", "weighted"])
@pytest.mark.parametrize("shape", [GRAD_SHAPES[i] for i in (0, 1, 3, 4)], ids=[
    "dqn", "dueling_dqn", "c51", "dueling_c51"])
def test_sigma_zero_gives_the_plain_pass_on_mu(shape, weighted):
    from warp_drive_b200.training.algorithms.fused_dqn import (
        FusedDuelingUpdate, FusedDQNUpdate, FusedC51Update)

    B, n_step, C, E, Np, F, A, N, dims, S = shape
    q_net, target, algo, fused, ring, w, weights, _, _ = _setup(shape, weighted, True,
                                                                 sigma=False)
    twin, plain = _mean_twin(q_net, S, N)
    ttwin, _ = _mean_twin(target, S, N)
    for p in list(q_net.parameters()) + list(twin.parameters()):
        p.grad = torch.zeros_like(p)
    sums = fused.launch(*_dev(ring), w, None, weights, update=7).clone()
    noisy_grads = {n: p.grad.clone() for n, p in q_net.named_parameters()}
    cls = (FusedDuelingUpdate if S is not None else FusedC51Update if N > 1 else FusedDQNUpdate)
    ref_update = cls(algo, twin, ttwin, E, Np, C, B)
    ref_sums = ref_update.launch(*_dev(ring), w, None, weights)
    assert torch.equal(sums, ref_sums)
    for i in range(len(dims)):
        for s in ("weight", "bias"):
            assert torch.equal(noisy_grads[f"fc.{i}.0.{s}"],
                               getattr(twin.fc[str(i)][0], s).grad)
    for L, dst in zip(q_net.noisy_layers(), plain):
        assert torch.equal(L.weight_mu.grad, dst.weight.grad)
        assert torch.equal(L.bias_mu.grad, dst.bias.grad)
        want = ref.grads(_np(dst.weight.grad), _np(dst.bias.grad), _np(L.noise_in),
                         _np(L.noise_out))
        assert (np.abs(_np(L.weight_sigma.grad) - want[1]) <= 2.5e-7 * np.abs(want[1])).all()
        assert (np.abs(_np(L.bias_sigma.grad) - want[3]) <= 1.2e-7 * np.abs(want[3])).all()


# ------------------------------------------------------------------------ the trainer
def _noisy_model(kind, dims=(64, 64), S=None, **extra):
    m = {"type": kind, "fc_dims": list(dims), "noisy": True, "model_ckpt_filepath": "", **extra}
    if S is not None:
        m.update(dueling=True, stream_fc_dims=[S] if S else [])
    if kind == "fully_connected_categorical_q":
        m.update(num_atoms=51, v_min=0.0, v_max=100.0)
    return m


CASES = [("fully_connected_q", (64, 64), None), ("fully_connected_categorical_q", (64,), None),
         ("fully_connected_q", (64,), 32), ("fully_connected_categorical_q", (64,), 32)]
CASE_IDS = ["dqn", "c51", "dueling_dqn", "dueling_c51"]


@pytest.mark.parametrize("kind,dims,S", CASES, ids=CASE_IDS)
def test_trainer_fused_and_torch_gradients_agree(kind, dims, S, tmp_path):
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.fused_dqn import FusedNoisyUpdate

    tr = _trainer(tmp_path, model=_noisy_model(kind, dims, S))
    assert isinstance(tr.fused_updates["shared"], FusedNoisyUpdate)
    # a plain noisy DQN head acts through the one-launch rollout's noisy kind, the others per step
    assert tr.engine.noisy
    assert (tr.engine.sa is not None) == (kind == "fully_connected_q" and S is None)
    for it in range(3):
        steps = tr.engine.acting_steps["shared"]
        tr._generate_rollout_batch()
        assert tr.engine.acting_steps["shared"] == steps + 8     # one draw per env step
    tr._sample_replay_windows("shared")
    tr.update_count["shared"] = 41
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
    assert any(n.endswith("weight_sigma") for n in names)
    for name, a, b in zip(names, grads[True], grads[False]):
        assert float((a - b).norm() / b.norm().clamp_min(1e-30)) <= 1e-5, name
    for k in metrics[True]:
        assert metrics[True][k] == pytest.approx(metrics[False][k], rel=1e-5, abs=1e-6), k
    assert all(L.noise is None for L in tr.q_models["shared"].noisy_layers())
    # a non-logging update: windows, materialize, [fold,] the pass, [unfold,] grads, clipping
    # + Adam; no host wait
    tr._update_model_params(1)
    torch.cuda.synchronize()
    per_update = 9 if S is not None else 7
    for _ in range(2):
        n0 = wlib.launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            tr._update_model_params(1)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert wlib.launch_count() - n0 == 3 * per_update
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        tr._update_model_params(1)
        torch.cuda.synchronize()
    kernels = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    for k in ("noisy_materialize_kernel", "noisy_grads_kernel",
              "c51_kernel" if "categorical" in kind else "dqn_pass_kernel"):
        assert any(k in n for n in kernels), (k, kernels)
    m = tr._update_model_params(0)["shared"]
    layers = tr.q_models["shared"].noisy_layers()
    want = float(sum(L.weight_sigma.detach().abs().double().sum() for L in layers)
                 / sum(L.weight_sigma.numel() for L in layers))
    assert m["Noisy sigma"] == pytest.approx(want, rel=1e-12)


def test_acting_noise_per_env_and_the_mean_network_under_use_argmax(tmp_path):
    from warp_drive_b200.training.algorithms.fused_dqn import NOISY_ACTING, draw_noise

    tr = _trainer(tmp_path, E=64, pool=0, model=_noisy_model("fully_connected_q", (64, 64),
                                                             noisy_sigma0=4.0))
    eng, q = tr.engine, tr.q_models["shared"]
    eng.sa = None                                  # the per-step path
    L = q.noisy_layers()[0]
    step0 = eng.acting_steps["shared"]
    for step in range(step0, step0 + 3):
        obs = eng._tensor("observations")[:, 0].clone()
        eng.step(-1, epsilon=0.0)
        assert eng.acting_steps["shared"] == step + 1
        fi, fo = eng._acting_noise["shared"][0]
        # the documented noise of env row r at this step
        for r in (0, 1, 63):
            got = np.concatenate([_np(fi[r]), _np(fo[r])])
            want, bar = ref.noise(tr.seed, ref.ACTING, step, r, 0, got.size)
            assert (np.abs(got - want) <= bar).all()
        assert len({_np(fi[r]).tobytes() for r in range(64)}) == 64
        # the same (seed, counter, row) draws the same noise
        again = [(torch.empty_like(fi), torch.empty_like(fo))]
        draw_noise(q, tr.seed, NOISY_ACTING, step, rows=again)
        assert torch.equal(again[0][0], fi) and torch.equal(again[0][1], fo)
        # the actions are the first argmax of the noisy Q values where the top two are apart
        with torch.no_grad():
            L.noise = (fi, fo)
            qv = q.q_values(obs)
            L.noise = None
            mean = q.q_values(obs)
        acts = eng._tensor("sampled_actions")[:, 0, 0]
        clean = (qv[:, 0] - qv[:, 1]).abs() > 1e-4
        assert torch.equal(acts[clean], qv[clean].argmax(-1).to(torch.int32))
        assert float((qv - mean).abs().max()) > 1e-3             # the noise is on
    # use_argmax: the mean network, epsilon 0, no draw
    obs = eng._tensor("observations")[:, 0].clone()
    eng.step(-1, use_argmax=True)
    assert eng.acting_steps["shared"] == step0 + 3
    with torch.no_grad():
        mean = q.q_values(obs)
    clean = (mean[:, 0] - mean[:, 1]).abs() > 1e-4
    acts = eng._tensor("sampled_actions")[:, 0, 0]
    assert torch.equal(acts[clean], mean[clean].argmax(-1).to(torch.int32))
    assert all(L.noise is None for L in q.noisy_layers())


def test_outside_the_envelope_falls_back_and_trains(tmp_path):
    tr = _trainer(tmp_path, E=16, model=_noisy_model("fully_connected_q", (16, 16, 16, 16)))
    assert "shared" not in tr.fused_updates and tr.engine.sa is None
    before = [p.detach().clone() for p in tr.q_models["shared"].parameters()]
    for it in range(6):
        tr._generate_rollout_batch()
        m = tr._update_model_params(0 if it == 5 else 1)
    assert {"Q loss", "Mean Q value", "Mean return", "Epsilon", "Noisy sigma"} <= set(m["shared"])
    after = list(tr.q_models["shared"].parameters())
    assert all(torch.isfinite(p).all() for p in after)
    assert any(not torch.equal(x, y) for x, y in zip(before, after))
    sigma = tr.q_models["shared"].policy_head.weight_sigma
    assert not torch.equal(sigma, before[-3])               # sigma trains too


def test_rainbow_trains_and_round_trips_a_checkpoint(tmp_path):
    from warp_drive_b200.training.algorithms.fused_dqn import FusedNoisyUpdate
    from warp_drive_b200.training.trainer import load_run_config

    cfg = load_run_config("single_cartpole_rainbow")
    per = {k: cfg["trainer"][k] for k in cfg["trainer"] if k.startswith("prior")}
    model = dict(cfg["policy"]["shared"]["model"])
    tr = _trainer(tmp_path, E=16, trainer=per, model=model)
    assert isinstance(tr.fused_updates["shared"], FusedNoisyUpdate)
    assert tr.fused_updates["shared"].dueling
    for it in range(30):                                # 240 slots > 203: wraps
        tr._generate_rollout_batch()
        m = tr._update_model_params(0 if it == 29 else 1)
    want = {"Q loss", "Mean Q value", "Mean return", "Priority beta", "Mean IS weight",
            "Max priority", "Noisy sigma"}
    assert want <= set(m["shared"]) and all(np.isfinite(m["shared"][k]) for k in want)
    q = tr.q_models["shared"]
    assert all(torch.isfinite(p).all() for p in q.parameters())
    state = q.state_dict()
    assert not any("noise" in k for k in state)
    assert sum(k.endswith("weight_sigma") for k in state) == 4
    path = str(tmp_path / "shared_q_240.state_dict")
    torch.save(state, path)
    fresh = _trainer(tmp_path, E=16, name="fresh", trainer=per, model=model)
    fresh._load_policy_checkpoint("shared", path)
    for net in (fresh.q_models["shared"], fresh.target_q_models["shared"]):
        for (n, a), b in zip(net.named_parameters(), q.parameters()):
            assert torch.equal(a, b), n
    obs = torch.randn(32, 4, device=DEV)
    with torch.no_grad():                               # the mean networks agree
        assert torch.equal(fresh.q_models["shared"].q_values(obs), q.q_values(obs))
    fresh._generate_rollout_batch()
    fresh._update_model_params(1)                       # the loaded network trains natively
    assert all(torch.isfinite(p).all() for p in fresh.q_models["shared"].parameters())


# ------------------------------------------------------------------------ the one-launch noisy kind
def test_one_launch_noisy_kind_agrees_with_the_per_step_path(tmp_path):
    """epsilon = 1: identical sequences and acting steps.  epsilon = 0 with large sigma: at the
    same acting step, the kernel's Q values agree with the per-step path's factored forward on
    the same noise to 1e-4, and both paths take its first argmax where the margin exceeds 3e-4."""
    model = _noisy_model("fully_connected_q", (64, 64), noisy_sigma0=2.0)
    a = _trainer(tmp_path, E=64, name="a", pool=0, model=model)
    b = _trainer(tmp_path, E=64, name="b", pool=0, model=model)
    assert a.engine.sa is not None and a.engine.sa.noisy
    b.engine.sa = None
    names = ["sampled_actions_batch_shared", "rewards_batch_shared", "done_flags_batch",
             "processed_observations_batch_shared"]
    for _ in range(3):
        a.engine.rollout(epsilon=1.0)
        b.engine.rollout(epsilon=1.0)
        for n in names:
            assert torch.equal(a.engine._tensor(n), b.engine._tensor(n)), n
    assert a.engine.acting_steps == b.engine.acting_steps == {"shared": 3 * 8}
    for tr in (a, b):                      # an optimizer step, then a changed head
        tr._update_model_params(1)
        with torch.no_grad():
            torch.manual_seed(3)
            w = tr.q_models["shared"].policy_head.weight_mu
            w.add_(0.5 * torch.randn_like(w))
    for x, y in zip(a.q_models["shared"].parameters(), b.q_models["shared"].parameters()):
        assert torch.equal(x, y)
    E = 64
    q = torch.empty((1, E, 2), device=DEV)
    clean = torch.ones(E, dtype=torch.bool, device=DEV)
    head = a.q_models["shared"].policy_head
    moved = 0.0
    for _ in range(40):
        obs = a.engine._tensor("observations")[:, 0].clone()
        assert a.engine.acting_steps == b.engine.acting_steps
        a.engine.sa.launch(1, record=False, probs_out=q, epsilon=0.0)
        b.engine.step(-1, epsilon=0.0)
        fi, fo = b.engine._acting_noise["shared"][0]
        with torch.no_grad():
            head.noise = (fi, fo)
            want = a.q_models["shared"].q_values(obs)
            head.noise = None
            mean = a.q_models["shared"].q_values(obs)
        assert float((q[0] - want).abs().max()) <= 1e-4
        moved = max(moved, float((want - mean).abs().max()))
        clean &= (want[:, 0] - want[:, 1]).abs() > 3e-4
        ea = a.engine._tensor("sampled_actions")[:, 0, 0]
        eb = b.engine._tensor("sampled_actions")[:, 0, 0]
        assert torch.equal(ea[clean], eb[clean])
        assert torch.equal(ea[clean], want[clean].argmax(dim=-1).to(torch.int32))
    assert moved > 1e-2                    # the noise is on
    assert float(clean.float().mean()) > 0.8


def test_one_launch_noisy_kind_under_use_argmax_is_the_q_kind_on_mu(tmp_path):
    """use_argmax: the noisy kind's Q values, actions and trajectories equal the Q kind's on a
    plain network holding mu, bit for bit, and the acting step does not move."""
    a = _trainer(tmp_path, E=64, name="a", pool=0,
                 model=_noisy_model("fully_connected_q", (64, 64), noisy_sigma0=2.0))
    c = _trainer(tmp_path, E=64, name="c", pool=0,
                 model={"type": "fully_connected_q", "fc_dims": [64, 64],
                        "model_ckpt_filepath": ""})
    assert a.engine.sa.noisy and not c.engine.sa.noisy
    qa, qc = a.q_models["shared"], c.q_models["shared"]
    with torch.no_grad():
        for i in range(2):
            qc.fc[str(i)][0].weight.copy_(qa.fc[str(i)][0].weight)
            qc.fc[str(i)][0].bias.copy_(qa.fc[str(i)][0].bias)
        qc.policy_head.weight.copy_(qa.policy_head.weight_mu)
        qc.policy_head.bias.copy_(qa.policy_head.bias_mu)
    steps = dict(a.engine.acting_steps)
    T, E = 40, 64
    pa, pc = (torch.empty((T, E, 2), device=DEV) for _ in range(2))
    a.engine.sa.launch(T, record=False, probs_out=pa, use_argmax=True)
    c.engine.sa.launch(T, record=False, probs_out=pc, use_argmax=True)
    assert torch.equal(pa, pc)
    for n in ("observations", "sampled_actions", "rewards", "_done_"):
        assert torch.equal(a.engine._tensor(n), c.engine._tensor(n)), n
    assert a.engine.acting_steps == steps
