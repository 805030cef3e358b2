"""The fused update kernels (csrc/wdb_update.cu) held to the float64 reference of
tests/update_reference.py across their shape envelope: every float output within the bar the
reference derives for it, the bit-exact outputs bit for bit.  Every output is filled with a
NaN sentinel first and followed by a guard region that must come back untouched."""
import ctypes

import numpy as np
import pytest
import torch

import update_reference as R

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FA5A5A5                       # a NaN no kernel computes
GUARD = 67


def _lib():
    from warp_drive_b200 import lib as wlib

    return wlib, wlib.load()


def _out(n, dtype=torch.float32):
    """n elements filled with the sentinel, followed by a guarded tail: (full, view)."""
    if dtype == torch.float64:
        full = torch.full((n + GUARD,), -1.25e300, dtype=dtype, device="cuda")
    else:
        full = torch.full((n + GUARD,), SENTINEL, dtype=torch.int32, device="cuda").view(dtype)
    return full, full[:n]


def _guard_intact(full, n):
    tail = full[n:]
    if tail.dtype == torch.float64:
        assert bool((tail == -1.25e300).all()), "write past the output"
    else:
        assert bool((tail.view(torch.int32) == SENTINEL).all()), "write past the output"


def _check(kernel, ref, what):
    excess, i = R.within(kernel.detach().cpu().numpy() if torch.is_tensor(kernel) else kernel, ref)
    v, b = ref
    k = np.asarray(kernel.detach().cpu().numpy() if torch.is_tensor(kernel) else kernel)
    assert excess <= 0, (what, i, float(k.flat[i]), float(np.ravel(v)[i]), float(np.ravel(b)[i]))


def _bits_equal(a, b, what):
    a = np.ascontiguousarray(a, dtype=np.float32).view(np.int32)
    b = np.ascontiguousarray(b, dtype=np.float32).view(np.int32)
    bad = np.flatnonzero(a.ravel() != b.ravel())
    assert bad.size == 0, (what, bad[:5], a.ravel()[bad[:5]], b.ravel()[bad[:5]])


# ---------------------------------------------------------------- pg_loss
def _pg_inputs(T, E, Np, heads, done_mode, seed, boundary=False):
    rng = np.random.default_rng(seed)
    probs = []
    for a in heads:
        p = rng.uniform(0.05, 1.0, (T, E, Np, a))
        if a > 2:
            p[..., 1] = 0.0                                    # zero probabilities
        probs.append(p.astype(np.float32))
    actions = np.stack([rng.integers(0, a, (T, E, Np)) for a in heads], -1).astype(np.int32)
    if boundary:
        # rows whose float32 sum is 1 in every order: q == p exactly, on 0, eps and 1 - eps,
        # with the taken action on the boundary value
        eps = np.float32(2.0 ** -23)
        rows = np.array([[eps, 0.5, 0.5 - eps], [1 - eps, eps, 0.0], [0.0, 1 - eps, eps],
                         [0.5 - eps, eps, 0.5]], dtype=np.float32)
        take = [0, 0, 1, 1]
        flat = probs[0].reshape(-1, heads[0])
        acts = actions[..., 0].reshape(-1)
        for i in range(0, len(flat), 2):
            r = (i // 2) % 4
            flat[i, :] = 0.0
            flat[i, :3] = rows[r]
            acts[i] = take[r] if (i // 8) % 2 == 0 else 2 - (r == 3)
    values = (rng.standard_normal((T, E, Np)) * 2).astype(np.float32)
    rewards = rng.standard_normal((T, E, Np)).astype(np.float32)
    if done_mode == "all0":
        done = np.zeros((T, E), np.int32)
    elif done_mode == "all1":
        done = np.ones((T, E), np.int32)
    else:
        done = (rng.random((T, E)) < 0.2).astype(np.int32)
        done[rng.random((T, E)) < 0.05] = 2
    return probs, values, actions, rewards, done


def _pg_launch(probs, values, actions, rewards, done, gamma, vf, c, null=()):
    wlib, L = _lib()
    T, E, Np = rewards.shape
    n = T * E * Np
    S = wlib.PgLoss()
    S.T, S.n_envs, S.n_agents, S.n_heads = T, E, Np, len(probs)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()   # noqa: E731
    keep = [dev(p) for p in probs] + [dev(values), dev(actions), dev(rewards), dev(done)]
    outs = {}
    for k, p in enumerate(probs):
        S.n_actions[k] = p.shape[-1]
        S.probs[k] = wlib.ptr(keep[k])
        if f"grad_probs{k}" not in null:
            outs[f"grad_probs{k}"] = _out(p.size)
            S.grad_probs[k] = wlib.ptr(outs[f"grad_probs{k}"][1])
    S.values, S.actions, S.rewards, S.done = (wlib.ptr(t) for t in keep[len(probs):])
    S.gamma, S.vf_coeff, S.entropy_coeff = gamma, vf, c
    for name in ("grad_values", "returns"):
        if name not in null:
            outs[name] = _out(n)
            setattr(S, name, wlib.ptr(outs[name][1]))
    sums = torch.zeros(4 + GUARD, dtype=torch.float64, device="cuda")
    sums[4:] = -1.25e300
    S.sums = wlib.ptr(sums)
    wlib.check(L.wdb_pg_loss_and_grads(wlib.stream_ptr(), ctypes.byref(S)), "pg_loss")
    torch.cuda.synchronize()
    _guard_intact(sums, 4)
    res = {"sums": sums[:4].cpu().numpy()}
    for name, (full, view) in outs.items():
        _guard_intact(full, view.numel())
        res[name] = view.cpu().numpy()
    return res


def _pg_compare(got, ref, heads, shape, null=()):
    T, E, Np = shape
    for k, a in enumerate(heads):
        if f"grad_probs{k}" not in null:
            _check(got[f"grad_probs{k}"].reshape(T, E, Np, a), ref["grad_probs"][k], f"grad_probs{k}")
    if "grad_values" not in null:
        _check(got["grad_values"].reshape(T, E, Np), ref["grad_values"], "grad_values")
    if "returns" not in null:
        _check(got["returns"].reshape(T, E, Np), ref["returns"], "returns")
    for i in range(4):
        _check(got["sums"][i:i + 1], (np.array([ref["sums"][i][0]]), np.array([ref["sums"][i][1]])),
               f"sums[{i}]")


PG_CASES = [
    # T, E, Np (per_t = E * Np), heads, gamma, done, NULL outputs
    (1, 1, 1, (2,), 0.97, "random", ()),
    (4, 31, 1, (1,), 1.0, "all0", ()),
    (3, 8, 4, (32,), 0.0, "all1", ()),
    (3, 11, 3, (33,), 0.97, "random", ()),
    (2, 127, 1, (5, 3, 4), 0.97, "random", ("grad_probs1",)),
    (2, 32, 4, (7, 1, 40, 2), 1.0, "random", ("grad_values", "returns")),
    (2, 43, 3, (96,), 0.97, "random", ()),
    (2, 4129, 1, (97,), 0.97, "random", ("grad_probs0",)),
    (1, 129, 1, (399,), 1.0, "all0", ()),
    (3, 129, 1, (3, 399), 0.97, "random", ()),
    (50, 400, 21, (21, 21), 0.97, "random", ()),               # config 2: 66 CTAs
]


@pytest.mark.parametrize("case", PG_CASES, ids=lambda c: f"T{c[0]}-pt{c[1] * c[2]}-h{'x'.join(map(str, c[3]))}")
def test_pg_loss_matches_float64_reference(case):
    T, E, Np, heads, gamma, done_mode, null = case
    inputs = _pg_inputs(T, E, Np, heads, done_mode, seed=T * 1000 + E)
    vf, c = 0.75, 0.03125
    got = _pg_launch(*inputs, gamma, vf, c, null)
    ref = R.pg_loss(*inputs, gamma, vf, c)
    _pg_compare(got, ref, heads, (T, E, Np), null)


@pytest.mark.parametrize("heads", [(3,), (3, 33)])
def test_pg_loss_at_the_clamp_boundary(heads):
    """q exactly 0, eps and 1 - eps with the taken action on them: torch.clamp's backward is
    inclusive at both ends, so the -adv / q term and the entropy's +1 stay."""
    T, E, Np = 2, 40, 3
    inputs = _pg_inputs(T, E, Np, heads, "random", seed=77, boundary=True)
    got = _pg_launch(*inputs, 0.97, 0.5, 0.0625)
    ref = R.pg_loss(*inputs, 0.97, 0.5, 0.0625)
    _pg_compare(got, ref, heads, (T, E, Np))


@pytest.mark.parametrize("algo,clip", [("A2C", None), ("PPO", 0.0), ("PPO", 0.1), ("PPO", 1.0)])
def test_fused_pg_loss_wrapper_matches_float64_reference(algo, clip):
    """Through compute_loss_and_metrics and fused_pg_loss: loss, metrics and the gradients
    autograd hands to the model outputs; done takes the values 0, 1 and 2."""
    from warp_drive_b200.training.algorithms.fused_loss import fused_pg_loss
    from warp_drive_b200.training.algorithms.policygradient import A2C, PPO

    T, E, Np, heads = 6, 37, 5, (21, 9)
    probs, values, actions, rewards, done = _pg_inputs(T, E, Np, heads, "random", seed=3)
    vf, c, gamma = 0.75, 0.03125, 0.97
    ref = R.pg_loss(probs, values, actions, rewards, done, gamma, vf, c)
    P = [torch.from_numpy(p).cuda().requires_grad_() for p in probs]
    V = torch.from_numpy(values).cuda().requires_grad_()
    kw = dict(discount_factor_gamma=gamma, vf_loss_coeff=vf, entropy_coeff=c)
    tr = A2C(**kw) if algo == "A2C" else PPO(clip_param=clip, **kw)
    assert tr.use_fused_loss
    loss, metrics = tr.compute_loss_and_metrics(
        100, torch.from_numpy(actions).cuda().long(), torch.from_numpy(rewards).cuda(),
        torch.from_numpy(done).cuda(), P, V, perform_logging=True)
    loss.backward()
    lv, lb = R.pg_loss_value(ref["sums"], ref["M"], vf, c, ppo=algo == "PPO")
    assert abs(loss.item() - lv) <= lb, (loss.item(), lv, lb)
    for k in range(len(heads)):
        _check(P[k].grad, ref["grad_probs"][k], f"grad_probs{k}")
    _check(V.grad, ref["grad_values"], "grad_values")
    pol, pol_bar = ((-ref["sums"][3][0], ref["sums"][3][1]) if algo == "PPO" else ref["sums"][0])
    pol, pol_bar = pol / ref["M"], pol_bar / ref["M"]
    # reported as float32: one more rounding
    assert abs(metrics["Policy loss"] - pol) <= pol_bar + 2 * R.U * (abs(pol) + pol_bar)
    # fused_pg_loss itself, with the returns
    _, parts, returns = fused_pg_loss(V.detach(), [p.detach() for p in P],
                                      torch.from_numpy(actions).cuda(),
                                      torch.from_numpy(rewards).cuda(),
                                      torch.from_numpy(done).cuda(), gamma, vf, c,
                                      ppo=algo == "PPO", want_returns=True)
    _check(returns, ref["returns"], "returns")


# ---------------------------------------------------------------- heads softmax
def _softmax_case(A0, A1, rows, pitch, null, seed):
    wlib, L = _lib()
    rng = np.random.default_rng(seed)
    z = rng.uniform(-80, 80, (rows, pitch)).astype(np.float32)
    zd = torch.from_numpy(z).cuda()
    f0, p0 = _out(rows * A0)
    f1, p1 = _out(rows * A1) if A1 else (None, None)
    fv, vals = _out(rows)
    wlib.check(L.wdb_heads_softmax(wlib.stream_ptr(), wlib.ptr(zd), rows, A0, A1, pitch,
                                   wlib.ptr(p0), wlib.ptr(p1), wlib.ptr(vals)), "heads_softmax")
    torch.cuda.synchronize()
    r0, r1, rv = R.heads_softmax(z, A0, A1)
    for full, view in ((f0, p0), (f1, p1), (fv, vals)):
        if full is not None:
            _guard_intact(full, view.numel())
    _check(p0.view(rows, A0), r0, "probs0")
    if A1:
        _check(p1.view(rows, A1), r1, "probs1")
    _bits_equal(vals.cpu().numpy(), rv, "values")
    if pitch > 200:
        return
    # backward from the kernel's own probabilities
    g0 = None if null == "g0" else rng.standard_normal((rows, A0)).astype(np.float32)
    g1 = None if (null == "g1" or not A1) else rng.standard_normal((rows, A1)).astype(np.float32)
    gv = None if null == "gv" else rng.standard_normal(rows).astype(np.float32)
    dev = lambda x: None if x is None else torch.from_numpy(x).cuda()   # noqa: E731
    g0d, g1d, gvd = dev(g0), dev(g1), dev(gv)
    fz, dz = _out(rows * pitch)
    wlib.check(L.wdb_heads_softmax_backward(
        wlib.stream_ptr(), wlib.ptr(p0), wlib.ptr(p1), wlib.ptr(g0d), wlib.ptr(g1d),
        wlib.ptr(gvd), rows, A0, A1, pitch, wlib.ptr(dz)), "heads_softmax_backward")
    torch.cuda.synchronize()
    _guard_intact(fz, dz.numel())
    got = dz.view(rows, pitch).cpu().numpy()
    p1h = p1.view(rows, A1).cpu().numpy() if A1 else None
    v, b = R.heads_softmax_backward(p0.view(rows, A0).cpu().numpy(), p1h, g0, g1, gv, A0, A1,
                                    pitch)
    _check(got, (v, b), "dz")
    fixed = np.zeros(pitch, bool)
    fixed[A0 + A1:] = True                                   # value column and padding
    if g0 is None:
        fixed[:A0] = True
    if g1 is None:
        fixed[A0:A0 + A1] = True
    _bits_equal(got[:, fixed], v[:, fixed].astype(np.float32), "dz exact columns")


SOFTMAX_CASES = [(A0, A1) for A0 in (1, 2, 21, 32, 33, 97) for A1 in (0, 1, 21, 40)]


@pytest.mark.parametrize("A0,A1", SOFTMAX_CASES)
def test_heads_softmax_forward_and_backward_match_float64_reference(A0, A1):
    i = SOFTMAX_CASES.index((A0, A1))
    a = A0 + A1 + 1
    pitch = (a, -(-a // 4) * 4, (-(-a // 4) * 4) | 1)[i % 3]          # exact, padded, odd
    rows = (1, 31, 33, 128, 129)[i % 5]
    _softmax_case(A0, A1, rows, pitch, (None, "g0", "g1", "gv")[i % 4], seed=i)


@pytest.mark.parametrize("A0,A1,pitch", [(97, 40, 399), (97, 40, 199)])
def test_heads_softmax_at_the_largest_pitches_on_200003_rows(A0, A1, pitch):
    _softmax_case(A0, A1, 200003, pitch, None, seed=pitch)


# ---------------------------------------------------------------- relu backward + bias
def _relu_case(rows, width, offset=0, seed=0):
    wlib, L = _lib()
    rng = np.random.default_rng(seed)
    h = rng.standard_normal((rows, width)).astype(np.float32)
    h.ravel()[::7] = 0.0
    h.ravel()[3::11] = -0.0
    h.ravel()[5::13] = np.nan
    dh = rng.standard_normal((rows, width)).astype(np.float32)
    dh[~(h > 0)] = np.nan                                    # masked: must come out 0
    per = int(L.wdb_relu_backward_bias_rows(rows))
    ctas = -(-rows // per)
    n = rows * width
    # `offset` floats in front of both buffers: a 4-byte offset forces the scalar kernel
    hfull = torch.zeros(offset + n, device="cuda")
    hfull[offset:] = torch.from_numpy(h.ravel()).cuda()
    dfull, _ = _out(offset + n)
    dfull[offset:offset + n] = torch.from_numpy(dh.ravel()).cuda()
    pfull, part = _out(ctas * width)
    wlib.check(L.wdb_relu_backward_bias(wlib.stream_ptr(), wlib.ptr(dfull[offset:offset + n]),
                                        wlib.ptr(hfull[offset:]), rows, width, wlib.ptr(part)),
               "relu_backward_bias")
    torch.cuda.synchronize()
    _guard_intact(dfull, offset + n)
    _guard_intact(pfull, part.numel())
    masked, ref = R.relu_backward_bias(dh, h, per)
    _bits_equal(dfull[offset:offset + n].cpu().numpy(), masked.ravel(), "masked dh")
    _check(part.view(ctas, width), ref, "partial bias gradient")


@pytest.mark.parametrize("width", [1, 3, 4, 12, 64, 70, 256, 1024, 1028])
def test_relu_backward_bias_matches_float64_reference(width):
    from warp_drive_b200 import lib as wlib

    per = int(wlib.load().wdb_relu_backward_bias_rows(200))
    for rows in (1, 63, 64, 65, 3 * per + 1, 1000):
        _relu_case(rows, width, seed=rows * 7 + width)


@pytest.mark.parametrize("rows,width,offset", [(2_000_000, 12, 0), (2_000_000, 1, 0),
                                               (300_001, 64, 0), (5000, 64, 1), (20_001, 1024, 0)])
def test_relu_backward_bias_large_and_unaligned(rows, width, offset):
    _relu_case(rows, width, offset, seed=rows % 1000 + width)


# ---------------------------------------------------------------- pad_rows, sumsq
@pytest.mark.parametrize("rows,width,pitch", [(1000, 1, 4), (333, 5, 5), (300_001, 3, 4),
                                              (70_000, 71, 72)])
def test_pad_rows_is_exact(rows, width, pitch):
    wlib, L = _lib()
    src = np.random.default_rng(rows).standard_normal((rows, width)).astype(np.float32)
    full, dst = _out(rows * pitch)
    wlib.check(L.wdb_pad_rows(wlib.stream_ptr(), wlib.ptr(torch.from_numpy(src).cuda()), rows,
                              width, pitch, wlib.ptr(dst)), "pad_rows")
    torch.cuda.synchronize()
    _guard_intact(full, dst.numel())
    _bits_equal(dst.cpu().numpy(), R.pad_rows(src, pitch).ravel(), "pad_rows")


@pytest.mark.parametrize("n", [1, 2047, 2048 * 528 + 5, 10 ** 7])
def test_grad_sumsq_adds_the_exact_sum(n):
    wlib, L = _lib()
    g = (np.random.default_rng(n).standard_normal(n) * 3).astype(np.float32)
    out = torch.full((1 + GUARD,), -1.25e300, dtype=torch.float64, device="cuda")
    out[0] = 1.25
    wlib.check(L.wdb_grad_sumsq(wlib.stream_ptr(), wlib.ptr(torch.from_numpy(g).cuda()), n,
                                wlib.ptr(out)), "grad_sumsq")
    torch.cuda.synchronize()
    _guard_intact(out, 1)
    v, b = R.grad_sumsq(g, 1.25)
    assert abs(float(out[0]) - v) <= b, (float(out[0]), v, b)


# ---------------------------------------------------------------- Adam
ADAM_CASES = [(s, mode) for s in (1, 2, 10, 1000, 100_000)
              for mode in ("off", "below", "above", "zero")]


@pytest.mark.parametrize("step,mode", ADAM_CASES)
def test_adam_step_matches_float64_reference(step, mode):
    wlib, L = _lib()
    i = ADAM_CASES.index((step, mode))
    n = (1, 255, 257, 10 ** 6 + 3)[i % 4]
    rng = np.random.default_rng(i)
    p = rng.standard_normal(n).astype(np.float32)
    g = np.zeros(n, np.float32) if mode == "zero" else (rng.standard_normal(n) * 0.1).astype(np.float32)
    m = (rng.standard_normal(n) * 0.05).astype(np.float32)
    v = (rng.random(n) * 0.01).astype(np.float32)
    if step == 1:
        m[:] = 0.0
        v[:] = 0.0
    sumsq = float(np.sum(g.astype(np.float64) ** 2))
    norm = np.sqrt(sumsq)
    max_norm = {"off": 0.0, "below": 2.0 * norm + 1.0, "above": 0.25 * norm, "zero": 0.5}[mode]
    lr, b1, b2, eps = 3e-3, 0.9, 0.999, 1e-8
    bufs = []
    for x in (p, g, m, v):
        full, view = _out(n)
        view.copy_(torch.from_numpy(x))
        bufs.append((full, view))
    s = torch.tensor([sumsq], dtype=torch.float64, device="cuda")
    wlib.check(L.wdb_adam_step(wlib.stream_ptr(), *(wlib.ptr(b[1]) for b in bufs), n, lr, b1, b2,
                               eps, step, max_norm, wlib.ptr(s) if max_norm > 0 else None),
               "adam_step")
    torch.cuda.synchronize()
    ref = R.adam_step(p, g, m, v, lr, b1, b2, eps, step, max_norm, sumsq)
    if mode == "above":
        assert ref["clip"][0] < 0.3
    for (full, view), name in zip(bufs, ("params", "grads", "exp_avg", "exp_avg_sq")):
        _guard_intact(full, n)
        _check(view, ref[name], name)
    if mode in ("off", "below", "zero"):                    # clip == 1: the gradient is untouched
        _bits_equal(bufs[1][1].cpu().numpy(), g, "grads")


# ---------------------------------------------------------------- end to end
@pytest.mark.parametrize("H", [70, 1024])
def test_fused_train_node_at_unaligned_and_widest_hidden_layers(H):
    """H = 70 takes the scalar ReLU-backward kernel, H = 1024 the vector kernel's one row per
    iteration; same outputs and gradients as the plain module (float32 bars of
    tests/test_gpu_update.py)."""
    from test_gpu_mlp import _Model
    from warp_drive_b200.training.models import fused_mlp_train

    torch.manual_seed(H)
    m = _Model(23, H, 21, 9).cuda()
    m.action_mask = None
    obs = torch.randn(7, 37, 23, device="cuda")
    assert fused_mlp_train.supported(m, obs)
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        probs_f, values_f = fused_mlp_train.fused_train_forward(m, obs)
        w = [torch.randn(p.shape, device="cuda") for p in probs_f] + [torch.randn(values_f.shape, device="cuda")]
        sum((o * wi).sum() for o, wi in zip(probs_f + [values_f], w)).backward()
        grads = {k: p.grad.clone() for k, p in m.named_parameters()}
        m.zero_grad()
        probs_t, values_t = m(obs)
        sum((o * wi).sum() for o, wi in zip(probs_t + [values_t], w)).backward()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    for a, b in zip(probs_f, probs_t):
        assert torch.allclose(a, b, atol=1e-6, rtol=1e-5)
    for k, p in m.named_parameters():
        assert torch.allclose(grads[k], p.grad, atol=2e-4, rtol=1e-4), (k, float((grads[k] - p.grad).abs().max()))


@pytest.mark.parametrize("heads", [(98, 98), (3, 2, 4, 2, 5)])
def test_policies_outside_the_fused_envelope_train_on_the_torch_paths(heads):
    """Two 98-action heads (head GEMM pitch 200: the softmax backward's two tiles do not fit)
    and five heads (the loss kernel takes four): one update runs on the torch paths."""
    from test_gpu_mlp import _Model
    from warp_drive_b200.training.algorithms.fused_loss import fused_pg_loss_supported
    from warp_drive_b200.training.algorithms.policygradient import A2C
    from warp_drive_b200.training.models import fused_mlp_train
    from warp_drive_b200.training.utils.flat_adam import FlatAdam

    torch.manual_seed(1)
    m = _Model(11, 32, heads[0], heads[1]).cuda()
    m.policy_head = torch.nn.ModuleList([torch.nn.Linear(32, a) for a in heads]).cuda()
    m.output_dims = list(heads)
    m.action_mask = None
    T, E, Np = 5, 8, 3
    obs = torch.randn(T, E, Np, 11, device="cuda")
    assert not fused_mlp_train.supported(m, obs)
    opt = FlatAdam(m.parameters(), lr=1e-3)
    before = opt.params.clone()
    probs, values = m(obs)
    assert fused_pg_loss_supported(probs) == (len(heads) <= 4)
    actions = torch.stack([torch.randint(0, a, (T, E, Np), device="cuda") for a in heads], -1)
    tr = A2C(discount_factor_gamma=0.9, vf_loss_coeff=0.5, entropy_coeff=0.01)
    loss, _ = tr.compute_loss_and_metrics(1, actions, torch.randn(T, E, Np, device="cuda"),
                                          torch.zeros(T, E, dtype=torch.int32, device="cuda"),
                                          probs, values)
    opt.zero_grad()
    loss.backward()
    opt.step(max_grad_norm=0.5)
    torch.cuda.synchronize()
    assert torch.isfinite(opt.params).all() and not torch.equal(opt.params, before)
