"""CPU tests of tests/update_reference.py (the float64 reference of csrc/wdb_update.cu) and of
the update kernels' support queries: the reference against torch autograd in float64, against
torch float32 Categorical at the clamp boundary, its Adam against torch.optim.Adam +
clip_grad_norm_, and wdb_pg_loss_supported / wdb_heads_softmax_supported against the refusals
of the launches they describe."""
import ctypes
import types

import numpy as np
import pytest
import torch

import update_reference as R

EPS = 2.0 ** -23


def _batch(rng, T, E, Np, heads, zeros=False, unnormalised=True):
    probs = []
    for a in heads:
        p = rng.uniform(0.05, 1.0, (T, E, Np, a))
        if zeros and a > 1:
            p[..., 0] = 0.0                                   # an impossible action
        if not unnormalised:
            p /= p.sum(-1, keepdims=True)
        probs.append(p.astype(np.float32))
    actions = np.stack([rng.integers(1 if zeros and a > 1 else 0, a, (T, E, Np)) for a in heads], -1)
    values = rng.standard_normal((T, E, Np)).astype(np.float32)
    rewards = rng.standard_normal((T, E, Np)).astype(np.float32)
    done = (rng.random((T, E)) < 0.2).astype(np.int32)
    done[0, 0] = 2                                            # "goal reached" counts as done
    return probs, values, actions, rewards, done


def _torch_loss(probs, values, actions, rewards, done, gamma, vf, c, dtype):
    """The A2C loss written out in torch with float32's eps explicitly (Categorical on float64
    tensors would clamp at float64's eps)."""
    T = rewards.shape[0]
    P = [torch.tensor(p, dtype=dtype, requires_grad=True) for p in probs]
    V = torch.tensor(values, dtype=dtype, requires_grad=True)
    r = torch.tensor(rewards, dtype=dtype)
    d = torch.tensor(done > 0, dtype=dtype)[:, :, None]
    g = float(np.float32(gamma))
    Vd = V.detach()
    ret = torch.zeros_like(r)
    ret[T - 1] = d[T - 1] * r[T - 1] + (1 - d[T - 1]) * Vd[T - 1]
    for t in range(T - 2, -1, -1):
        ret[t] = r[t] + (1 - d[t]) * g * ret[t + 1]
    adv = ret - Vd
    logp, ent = 0.0, 0.0
    for k, p in enumerate(P):
        q = p / p.sum(-1, keepdim=True)
        lg = torch.log(torch.clamp(q, EPS, 1 - EPS))
        logp = logp + lg.gather(-1, torch.tensor(actions[..., k:k + 1], dtype=torch.long))[..., 0]
        ent = ent + (-(lg * q).sum(-1)).mean()
    loss = (-logp * adv).mean() + vf * ((V - ret) ** 2).mean() - c * ent
    loss.backward()
    return loss, ret, adv, [p.grad for p in P], V.grad


@pytest.mark.parametrize("seed,shape,heads,zeros", [
    (0, (4, 3, 5), (6,), False), (1, (7, 2, 3), (5, 3, 4), True), (2, (1, 5, 2), (2, 9), True),
    (3, (6, 4, 1), (7, 1, 40, 2), False), (4, (3, 2, 2), (1,), False)])
def test_pg_loss_reference_is_torch_autograd_in_float64(seed, shape, heads, zeros):
    rng = np.random.default_rng(seed)
    probs, values, actions, rewards, done = _batch(rng, *shape, heads, zeros=zeros)
    gamma, vf, c = 0.97, 0.75, 0.03125
    ref = R.pg_loss(probs, values, actions, rewards, done, gamma, vf, c)
    loss, ret, adv, gp, gv = _torch_loss(probs, values, actions, rewards, done, gamma, vf, c,
                                         torch.float64)
    close = lambda a, b: np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-15)  # noqa: E731
    close(ref["returns"][0], ret.numpy())
    close(ref["adv"][0], adv.numpy())
    close(ref["grad_values"][0], gv.numpy())
    for a, b in zip(ref["grad_probs"], gp):
        close(a[0], b.numpy())
    close(R.pg_loss_value(ref["sums"], ref["M"], vf, c)[0], loss.item())
    # the bars are bars of float32 evaluation: a few hundred u at most, relative to the terms
    assert all(np.all(b[1] <= 1e-4 * (np.abs(b[0]) + 1e-3)) for b in ref["grad_probs"])


def test_pg_loss_reference_matches_torch_float32_categorical_at_the_clamp_boundary():
    """Rows whose float32 sum is exactly 1 in every order put q exactly on eps and 1 - eps:
    torch.clamp passes the gradient there (both ends inclusive), and so does the reference."""
    rows = np.array([[EPS, 0.5, 0.5 - EPS], [1 - EPS, EPS, 0.0], [0.5 - EPS, EPS, 0.5],
                     [0.0, 1 - EPS, EPS], [EPS, 1 - EPS, 0.0]], dtype=np.float32)
    assert all(float(np.float32(r[0]) + r[1] + r[2]) == 1.0 == float(r[2] + r[1] + r[0])
               for r in rows)
    probs = rows.reshape(1, 5, 1, 3)
    actions = np.array([0, 0, 1, 1, 1]).reshape(1, 5, 1, 1)
    values = np.array([0.5, -1.0, 2.0, 0.25, 3.0], dtype=np.float32).reshape(1, 5, 1)
    rewards = np.array([1.5, 2.0, -1.0, 1.0, -2.0], dtype=np.float32).reshape(1, 5, 1)
    done = np.ones((1, 5), dtype=np.int32)
    gamma, vf, c = 0.9, 0.5, 0.0625
    ref = R.pg_loss([probs], values, actions, rewards, done, gamma, vf, c)
    P = torch.tensor(probs, requires_grad=True)
    dist = torch.distributions.Categorical(probs=P)
    adv = torch.tensor(rewards - values)
    loss = (-dist.log_prob(torch.tensor(actions[..., 0])) * adv).mean() - c * dist.entropy().mean()
    loss.backward()
    v, b = ref["grad_probs"][0]
    assert np.all(np.abs(P.grad.numpy() - v) <= 4 * b + 1e-30), (P.grad.numpy(), v, b)
    # the taken action at q == eps carries -adv / (M q): the strict test would drop it
    assert abs(v[0, 0, 0, 0]) > 1e5 and abs(v[0, 2, 0, 1]) > 1e5
    # torch's own example: d log_prob(0) / dp at [2^-23, 1 - 2^-23]
    p = torch.tensor([EPS, 1 - EPS], requires_grad=True)
    torch.distributions.Categorical(probs=p).log_prob(torch.tensor(0)).backward()
    assert p.grad.tolist() == [8388607.0, -1.0]


def test_heads_softmax_reference_is_float64_softmax():
    rng = np.random.default_rng(5)
    A0, A1, pitch = 7, 3, 12
    z = rng.uniform(-80, 80, (64, pitch)).astype(np.float32)
    p0, p1, values = R.heads_softmax(z, A0, A1)
    t = torch.tensor(z, dtype=torch.float64)
    np.testing.assert_allclose(p0[0], torch.softmax(t[:, :A0], -1).numpy(), rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(p1[0], torch.softmax(t[:, A0:A0 + A1], -1).numpy(), rtol=1e-12,
                               atol=1e-300)
    assert np.array_equal(values, z[:, A0 + A1])
    g0 = rng.standard_normal((64, A0)).astype(np.float32)
    pf0 = p0[0].astype(np.float32)
    pf1 = p1[0].astype(np.float32)
    dz, bar = R.heads_softmax_backward(pf0, pf1, g0, None, None, A0, A1, pitch)
    P = torch.tensor(pf0, dtype=torch.float64)
    want = P * (torch.tensor(g0, dtype=torch.float64) - (torch.tensor(g0, dtype=torch.float64) * P).sum(-1, keepdim=True))
    np.testing.assert_allclose(dz[:, :A0], want.numpy(), rtol=1e-12, atol=1e-15)
    assert not dz[:, A0:].any() and not bar[:, A0:].any()
    assert not np.signbit(dz[:, A0:]).any()


@pytest.mark.parametrize("step", [1, 2, 10, 1000, 100000])
@pytest.mark.parametrize("clip", [0.0, 0.5, 1e6])
def test_adam_reference_matches_torch_adam_with_clipping(step, clip):
    """One step from the same state at any step count: the reference (float32 betas, powf bias
    corrections) against torch.optim.Adam + clip_grad_norm_ on CPU, to the float32 bars plus
    the derived torch deviation (update_reference.adam_torch_deviation).  At step 1 the
    bias-correction difference is largest: sqrt(bias2) differs by 6.4e-6 relative."""
    rng = np.random.default_rng(step)
    n = 1000
    p = rng.standard_normal(n).astype(np.float32)
    g = (rng.standard_normal(n) * 0.1).astype(np.float32)
    m = np.zeros(n, np.float32) if step == 1 else (rng.standard_normal(n) * 0.05).astype(np.float32)
    v = np.zeros(n, np.float32) if step == 1 else (rng.random(n) * 0.01).astype(np.float32)
    lr, b1, b2, eps = 3e-3, 0.9, 0.999, 1e-8
    sumsq = float(np.sum(g.astype(np.float64) ** 2))
    ref = R.adam_step(p, g, m, v, lr, b1, b2, eps, step, clip, sumsq)
    tp = torch.nn.Parameter(torch.tensor(p))
    tp.grad = torch.tensor(g)
    opt = torch.optim.Adam([tp], lr=lr, betas=(b1, b2), eps=eps, foreach=False)
    if step > 1:
        opt.state[tp] = {"step": torch.tensor(float(step - 1)), "exp_avg": torch.tensor(m),
                         "exp_avg_sq": torch.tensor(v)}
    if clip > 0:
        torch.nn.utils.clip_grad_norm_([tp], clip)
    opt.step()
    dev = R.adam_torch_deviation(ref, g, m, v, lr, b1, b2, eps, step,
                                 clipped_n=n if clip > 0 and ref["clip"][0] < 1 else 0)
    got = tp.detach().numpy().astype(np.float64)
    err = np.abs(got - ref["params"][0]) - (2 * ref["params"][1] + dev)
    assert err.max() <= 0, (step, clip, float(err.max()), float(np.max(dev)))
    if step == 1:
        bias2_t, bias2_k = 1 - b2, 1 - float(np.float32(b2))
        assert abs(np.sqrt(bias2_k / bias2_t) - 1) < 6.5e-6


def test_sumsq_and_relu_references():
    rng = np.random.default_rng(9)
    g = rng.standard_normal(5001).astype(np.float32)
    v, b = R.grad_sumsq(g, 2.5)
    assert abs(v - (2.5 + float(torch.tensor(g, dtype=torch.float64).square().sum()))) <= b
    h = rng.standard_normal((130, 12)).astype(np.float32)
    h[0, :3] = [0.0, -0.0, np.nan]
    dh = rng.standard_normal((130, 12)).astype(np.float32)
    dh[h <= 0] = np.nan
    masked, (pv, pb) = R.relu_backward_bias(dh, h, 64)
    assert masked[0, :3].tolist() == [0.0, 0.0, 0.0] and not np.isnan(masked).any()
    assert pv.shape == (3, 12)
    np.testing.assert_allclose(pv.sum(0), masked.astype(np.float64).sum(0), rtol=1e-12)


# ---------------------------------------------------------------- support queries
def _pg_request(wlib, heads):
    L = wlib.PgLoss()
    L.T, L.n_envs, L.n_agents, L.n_heads = 3, 5, 7, len(heads)
    base = 1 << 24
    for k, a in enumerate(heads[:4]):
        L.n_actions[k] = a
        L.probs[k] = base + 0x100000 * (k + 1)
        L.grad_probs[k] = base + 0x100000 * (k + 5)
    L.values, L.actions, L.rewards, L.done = (base + 0x100000 * k for k in range(10, 14))
    L.sums = base + 0x100000 * 14
    return L


def _pg_supported(lib, heads):
    arr = (ctypes.c_int * max(1, len(heads)))(*heads)
    return lib.wdb_pg_loss_supported(len(heads), arr)


@pytest.mark.skipif(
    torch.cuda.is_available(),
    reason="calls the launches with dummy pointers: only where no CUDA device can run them")
def test_update_support_queries_agree_with_the_launches(wdb_lib):
    """wdb_pg_loss_supported / wdb_heads_softmax_supported run the launches' own checks:
    where a query refuses, the launch returns cudaErrorInvalidValue (1); where it accepts, the
    launch reaches the CUDA runtime, which without a GPU returns 35."""
    from warp_drive_b200 import lib as wlib

    checked = 0
    for n_heads in range(1, 6):
        for a in (1, 2, 21, 96, 97, 200, 398, 399, 400, 401, 1000):
            for heads in ([a] * n_heads, [3] * (n_heads - 1) + [a]):
                q = _pg_supported(wdb_lib, heads)
                # the struct holds four heads: a fifth is refused on n_heads alone
                L = _pg_request(wlib, heads)
                rc = wdb_lib.wdb_pg_loss_and_grads(None, ctypes.byref(L))
                assert rc == (35 if q else 1), (heads, q, rc)
                checked += 1
    assert _pg_supported(wdb_lib, [399]) == 1 and _pg_supported(wdb_lib, [400]) == 0
    assert _pg_supported(wdb_lib, [7, 1, 40, 399]) == 1
    assert _pg_supported(wdb_lib, [2] * 4) == 1 and _pg_supported(wdb_lib, [2] * 5) == 0
    assert _pg_supported(wdb_lib, [5, 0]) == 0 and _pg_supported(wdb_lib, []) == 0
    p = 1 << 24
    fwd_max = bwd_max = 0
    for A0 in (1, 2, 21, 98, 197, 300):
        for A1 in (0, 1, 21, 98):
            for pitch in range(A0 + A1 - 1, 410):
                q = wdb_lib.wdb_heads_softmax_supported(A0, A1, pitch)
                f = wdb_lib.wdb_heads_softmax(None, p, 10, A0, A1, pitch, p + 0x100000,
                                              p + 0x200000, p + 0x300000)
                b = wdb_lib.wdb_heads_softmax_backward(None, p, p + 0x100000, p + 0x200000,
                                                       p + 0x300000, p + 0x400000, 10, A0, A1,
                                                       pitch, p + 0x500000)
                assert f in (1, 35) and b in (1, 35), (A0, A1, pitch, f, b)
                assert q == (f == 35 and b == 35), (A0, A1, pitch, q, f, b)
                fwd_max = max(fwd_max, pitch if f == 35 else 0)
                bwd_max = max(bwd_max, pitch if b == 35 else 0)
                checked += 1
    assert fwd_max == 399 and bwd_max == 199
    assert wdb_lib.wdb_heads_softmax_supported(97, 98, 196) == 1
    assert wdb_lib.wdb_heads_softmax_supported(98, 98, 200) == 0        # two 98-action heads
    assert checked > 1000


def test_fused_paths_ask_the_support_queries(wdb_lib):
    """fused_mlp_train.supported() and the fused-loss selection follow the library's answer."""
    from warp_drive_b200.training.algorithms.fused_loss import fused_pg_loss_supported
    from warp_drive_b200.training.models import fused_mlp_train

    obs = types.SimpleNamespace(is_cuda=True, dtype=torch.float32, requires_grad=False)
    for heads in ((21, 21), (3,), (98, 98), (97, 98), (40, 30), (196,), (197,), (1, 1)):
        model = types.SimpleNamespace(is_deterministic=False, fc=[0, 0], output_dims=list(heads),
                                      action_mask=None, parameters=lambda: [])
        a0, a1 = heads[0], heads[1] if len(heads) > 1 else 0
        pitch = -(-(a0 + a1 + 1) // 4) * 4
        assert fused_mlp_train.supported(model, obs) == bool(
            wdb_lib.wdb_heads_softmax_supported(a0, a1, pitch)), heads
    assert fused_mlp_train.supported(
        types.SimpleNamespace(is_deterministic=False, fc=[0, 0], output_dims=[98, 98],
                              action_mask=None, parameters=lambda: []), obs) is False
    for heads in ((21, 21), (2,) * 4, (2,) * 5, (399,), (400,), (7, 1, 40, 2)):
        probs = [torch.empty((1, 1, 1, a)) for a in heads]
        assert fused_pg_loss_supported(probs) == bool(_pg_supported(wdb_lib, list(heads)))
    assert fused_pg_loss_supported([torch.empty((1, 1, 1, 2))] * 5) is False
