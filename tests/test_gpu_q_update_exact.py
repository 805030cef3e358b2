"""The DQN-family replay update passes -- wdb_dqn_update_sampled / _prioritized,
wdb_qr_dqn_update_sampled, wdb_c51_update_sampled and wdb_iqn_update_sampled -- against the float64
reference with error bars (tests/q_update_bounds.py), element by element: every gradient, the
per-row outputs and both loss sums within their bars (exactly the value where the bar is 0), the
guard regions untouched and a second launch bit-identical.  The shapes cover one row, a partial
tile, exactly 132 full tiles, CTAs that run several tiles with a tail tile after full ones, the
hidden widths [] to [64, 64, 64], F + A = 64, several agents per env, gamma 0 and 1, QR-DQN at one
and 64 quantiles, C51 at 2, 51 and 64 atoms (MountainCar's 3 x 51 head included) and IQN's
counts at 1 and 64 (K at 1 and 256).  A dueling DQN or C51 update is pinned stage by stage, each
stage on the previous stage's device output: the fold, the plain pass on the folded layers read
back from the device, and the unfold of the folded gradients the pass wrote."""
import pytest
import torch

import dueling_reference as dueling
import q_update_bounds as qb

from test_gpu_ddpg_update_exact import _guarded
from test_dueling_cpu import make_dueling
from test_gpu_dqn import _dev, _guard_grads, _untouched
from test_gpu_dueling import _guard_fold, _param_keys
from test_q_update_bounds_cpu import Case, _case_id, within

pytestmark = pytest.mark.gpu

DEV = "cuda"

# (kind, B, n_step, C, E, Np, F, A, hidden dims, N, iqn (n_cos, N, N', K), gamma)
CASES = [
    ("dqn", 1, 3, 9, 4, 1, 4, 2, [64, 64], 1, None, 0.97),
    ("dqn", 17, 1, 5, 3, 3, 6, 3, [1], 1, None, 0.0),
    ("dqn", 333, 3, 40, 6, 1, 4, 2, [], 1, None, 0.97),
    ("dqn", 2112, 3, 40, 16, 1, 63, 1, [5, 7, 9], 1, None, 1.0),
    ("dqn", 4099, 4, 11, 16, 3, 4, 3, [64, 64, 64], 1, None, 0.97),
    ("qr", 2113, 3, 40, 16, 1, 4, 2, [64, 64], 1, None, 0.97),
    ("qr", 17, 3, 12, 4, 1, 4, 1, [64, 64, 64], 64, None, 1.0),
    ("qr", 333, 2, 40, 6, 3, 4, 2, [64, 64], 32, None, 0.97),
    ("qr", 1, 3, 9, 4, 1, 4, 2, [], 8, None, 0.97),
    ("qr", 17, 1, 5, 3, 3, 6, 2, [1], 4, None, 0.0),
    ("qr", 2112, 2, 12, 8, 1, 63, 1, [5, 7, 9], 64, None, 0.97),
    ("c51", 1, 3, 9, 4, 1, 4, 2, [64, 64], 51, None, 0.97),
    ("c51", 17, 3, 12, 4, 1, 63, 1, [], 64, None, 0.97),
    ("c51", 40, 3, 12, 4, 1, 4, 3, [64, 64], 51, None, 1.0),
    ("c51", 2112, 2, 12, 8, 3, 4, 3, [5, 7, 9], 2, None, 0.0),
    ("c51", 2113, 3, 40, 16, 1, 4, 2, [64, 64], 51, None, 0.97),
    ("c51", 17, 3, 12, 4, 1, 4, 1, [64, 64, 64], 64, None, 0.97),
    ("iqn", 1, 3, 9, 4, 1, 4, 2, [64, 64], 1, (64, 1, 64, 256), 0.97),
    ("iqn", 17, 3, 12, 4, 1, 4, 2, [64, 64], 1, (64, 64, 1, 1), 0.97),
    ("iqn", 17, 2, 12, 4, 3, 63, 1, [5, 7, 9], 1, (1, 1, 64, 1), 0.0),
    ("iqn", 40, 3, 12, 4, 1, 4, 3, [16, 16, 16], 1, (16, 16, 16, 32), 1.0),
    ("iqn", 2113, 3, 40, 16, 1, 4, 2, [16], 1, (4, 2, 3, 8), 0.97),
    ("iqn", 17, 3, 12, 4, 1, 4, 3, [64, 64, 64], 1, (64, 16, 16, 32), 0.97),
    ("iqn", 17, 3, 12, 4, 1, 4, 2, [1], 1, (8, 4, 4, 8), 0.97),
]
# The plans refuse, and so are not here: C51 with [64, 64, 64] beside a head wider than one
# block of 64 atoms (A N = 2 x 51: the weights overflow shared memory; A = 1, N = 64 runs), and
# IQN without hidden layers (the model refuses it: the tau embedding multiplies the trunk's
# output).


def _fused(case):
    from warp_drive_b200.training.algorithms import dqn as algos
    from warp_drive_b200.training.algorithms import fused_dqn as fd

    q, t = (m.to(DEV) for m in case.models)
    kw = dict(n_step=case.n_step, double_q=case.double_q)
    if case.kind == "c51":
        algo, cls = algos.CategoricalDQN(case.gamma, **kw), fd.FusedC51Update
    elif case.kind == "iqn":
        algo = algos.ImplicitQuantileDQN(case.gamma, huber_delta=case.kappa, **kw)
        cls = fd.FusedIQNUpdate
    elif case.kind == "qr":
        algo = algos.QuantileDQN(case.gamma, huber_delta=case.kappa, **kw)
        cls = fd.FusedQRDQNUpdate
    else:
        algo = algos.DQN(case.gamma, huber_delta=case.kappa, **kw)
        cls = fd.FusedDQNUpdate
    return q, cls(algo, q, t, case.E, case.Np, case.C, case.B)


@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("c", CASES, ids=[_case_id(c) for c in CASES])
def test_q_pass_within_its_float64_bars(c, double_q):
    kind, B, n_step, C, E, Np, F, A, dims, N, iqn, gamma = c
    case = Case(kind, B, n_step, C, E, Np, F, A, dims, N, iqn, gamma, double_q)
    if kind == "c51" and B > 2112:              # atom targets clamp at both support ends
        tz = case.existing()["tz"]
        z = case.support()[0]
        assert (tz == z[0]).any() and (tz == z[-1]).any()
    refs = [case.reference(weights=wt) for wt in (None, case.weights)]
    q, fused = _fused(case)
    ring = _dev(case.ring)
    w = torch.from_numpy(case.windows).to(DEV)
    kw = {} if case.taus is None else {"taus": torch.from_numpy(case.taus).to(DEV)}
    names = [n for n, _ in q.named_parameters()]
    assert all(ref["ok"].all() for ref in refs)      # no kept row sits on a branch
    for weighted, ref in zip((False, True), refs):
        wt = torch.from_numpy(case.weights).to(DEV) if weighted else None
        guards = _guard_grads(q)
        outs = [_guarded((B,), DEV) for _ in range(2)]
        guards += [b for b, _ in outs]
        sums = fused.launch(*ring, w, tuple(v for _, v in outs), wt, **kw).clone()
        first = [p.grad.clone() for p in q.parameters()]
        ratios = {}
        for name, got, want in zip(names, first, ref["grads"]):
            ratios[name] = within(got.double().cpu().numpy(), want, name)
        ratios["q_values"] = within(outs[0][1].double().cpu().numpy(), ref["q_values"], "q_values")
        ratios["returns"] = within(outs[1][1].double().cpu().numpy(), ref["returns"], "returns")
        for i in range(2):
            v, b = ref["sums"][i]
            err = abs(float(sums[i]) - v)
            assert err <= b, (f"sums[{i}]", float(sums[i]), v, b)
            ratios[f"sums[{i}]"] = err / b if b > 0 else 0.0
        assert _untouched(guards)
        first_outs = [v.clone() for _, v in outs]
        again = fused.launch(*ring, w, tuple(v for _, v in outs), wt, **kw)
        assert all(torch.equal(a, p.grad) for a, p in zip(first, q.parameters()))
        assert torch.equal(sums, again)
        assert all(torch.equal(a, v) for a, (_, v) in zip(first_outs, outs))
        worst = max(ratios, key=ratios.get)
        print(f"\nRATIO {_case_id(c)} {'double_q' if double_q else 'max_target'} "
              f"{'weighted' if weighted else 'uniform'}: max |err|/bar {ratios[worst]:.3g} "
              f"({worst})")


# ------------------------------------------------------------------------ dueling
def _report(what, ratios):
    worst = max(ratios, key=ratios.get)
    print(f"\nRATIO {what}: max |err|/bar {ratios[worst]:.3g} ({worst})")


def _plain_twins(q_net, target, folds, categorical, F, A, N):
    """Float32 plain networks holding each dueling network's trunk and the folded layers read
    back from the device: the networks the pass runs."""
    import c51_reference as cref
    import dqn_update_reference as dref
    from warp_drive_b200.training.algorithms.fused_dqn import folded_widths

    widths = folded_widths(q_net)
    pair = (cref.make_c51_models(F, A, widths, N=N, v_min=-3.0, v_max=4.0) if categorical
            else dref.make_q_models(F, A, widths))
    pair = [m.float() for m in pair]
    for src, f, twin in zip((q_net, target), folds, pair):
        layers = [(src.fc[str(i)][0].weight, src.fc[str(i)][0].bias) for i in range(len(src.fc))]
        layers += f.layers
        dst = [(twin.fc[str(i)][0].weight, twin.fc[str(i)][0].bias)
               for i in range(len(twin.fc))] + [(twin.policy_head.weight, twin.policy_head.bias)]
        with torch.no_grad():
            for (w, b), (dw, db) in zip(layers, dst):
                dw.copy_(w.detach().cpu())
                db.copy_(b.detach().cpu())
    return pair


# (B, n_step, C, E, Np, F, A, N, trunk dims, S); N = 1: dueling DQN, else dueling C51
DUELING = [(1, 3, 9, 4, 1, 4, 2, 1, [64], 32),
           (17, 3, 12, 4, 1, 4, 3, 51, [], 0),
           (17, 1, 5, 3, 3, 6, 3, 13, [16], 8),
           (2113, 3, 40, 16, 1, 4, 2, 1, [16, 16], 8),
           (2113, 3, 40, 16, 1, 4, 2, 51, [64], 32)]


@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("shape", DUELING, ids=[
    f"{'dqn' if s[7] == 1 else 'c51'}_B{s[0]}_A{s[6]}_N{s[7]}_L{len(s[8])}_S{s[9]}"
    for s in DUELING])
def test_dueling_stages_within_their_float64_bars(shape, double_q):
    from warp_drive_b200.training.algorithms import dqn as algos
    from warp_drive_b200.training.algorithms.fused_dqn import (
        DuelingFold, FusedDuelingUpdate, fold, folded_widths)

    B, n_step, C, E, Np, F, A, N, dims, S = shape
    categorical = N > 1
    tag = f"dueling_{'c51' if categorical else 'dqn'}_B{B}_A{A}_N{N}_S{S}_" + \
        ("double_q" if double_q else "max_target")
    extra = {"v_min": -3.0, "v_max": 4.0} if categorical else {}
    q_net = make_dueling(F, A, N, dims, S, seed=B, **extra)
    target = make_dueling(F, A, N, dims, S, seed=B, **extra)
    with torch.no_grad():
        for p in target.parameters():
            p.add_(0.3 * torch.randn_like(p))
    q_net, target = q_net.float().to(DEV), target.float().to(DEV)
    # 1. the fold, against the float64 fold of the float32 stream parameters
    folds = DuelingFold(q_net), DuelingFold(target)
    fold(*folds)
    ratios = {}
    for net, f, name in ((q_net, folds[0], "online"), (target, folds[1], "target")):
        want = qb.fold(dueling.stream_params(net.policy_head), A, N, S)
        for i, ((w, b), (rw, rb)) in enumerate(zip(f.layers, want)):
            ratios[f"{name} W{i}"] = within(w.double().cpu().numpy(), rw, f"fold {name} W{i}")
            ratios[f"{name} b{i}"] = within(b.double().cpu().numpy(), rb, f"fold {name} b{i}")
    _report(f"{tag} fold", ratios)
    # 2. the plain pass on the folded layers read back from the device
    twins = _plain_twins(q_net, target, folds, categorical, F, A, N)
    case = Case("c51" if categorical else "dqn", B, n_step, C, E, Np, F, A,
                folded_widths(q_net), N, None, 0.97, double_q, models=twins)
    refs = [case.reference(weights=wt) for wt in (None, case.weights)]
    assert all(ref["ok"].all() for ref in refs)
    kw = dict(n_step=n_step, double_q=double_q)
    algo = (algos.CategoricalDQN(case.gamma, **kw) if categorical
            else algos.DQN(case.gamma, huber_delta=case.kappa, **kw))
    fused = FusedDuelingUpdate(algo, q_net, target, E, Np, C, B)
    guards = _guard_grads(q_net) + _guard_fold(fused.online) + _guard_fold(fused.target)
    ring = _dev(case.ring)
    w = torch.from_numpy(case.windows).to(DEV)
    n_trunk = 2 * len(dims)
    params = list(q_net.parameters())
    for weighted, ref in zip((False, True), refs):
        wt = torch.from_numpy(case.weights).to(DEV) if weighted else None
        outs = [_guarded((B,), DEV) for _ in range(2)]
        sums = fused.launch(*ring, w, tuple(v for _, v in outs), wt).clone()
        # the pass ran on the layers the reference holds
        for (a, b), (c, d) in zip(fused.online.layers + fused.target.layers,
                                  folds[0].layers + folds[1].layers):
            assert torch.equal(a, c) and torch.equal(b, d)
        got = [p.grad for p in params[:n_trunk]] + [g for pair in fused.online.grads for g in pair]
        ratios = {}
        for i, (g, want) in enumerate(zip(got, ref["grads"])):
            ratios[f"grad{i}"] = within(g.double().cpu().numpy(), want, f"pass grad {i}")
        ratios["q_values"] = within(outs[0][1].double().cpu().numpy(), ref["q_values"], "q_values")
        ratios["returns"] = within(outs[1][1].double().cpu().numpy(), ref["returns"], "returns")
        for i in range(2):
            v, b = ref["sums"][i]
            assert abs(float(sums[i]) - v) <= b, (f"sums[{i}]", float(sums[i]), v, b)
        _report(f"{tag} {'weighted' if weighted else 'uniform'} pass", ratios)
        # 3. the unfold of the folded gradients the pass wrote
        folded = [(gw.double().cpu().numpy(), gb.double().cpu().numpy())
                  for gw, gb in fused.online.grads]
        want = qb.unfold(folded, A, N, S)
        ratios = {}
        for p, key in zip(params[n_trunk:], _param_keys(q_net.policy_head)):
            ratios[key] = within(p.grad.double().cpu().numpy(), want[key], f"unfold {key}")
        _report(f"{tag} {'weighted' if weighted else 'uniform'} unfold", ratios)
        assert _untouched(guards + [b for b, _ in outs])
        first = [p.grad.clone() for p in params]
        first_outs = [v.clone() for _, v in outs]
        again = fused.launch(*ring, w, tuple(v for _, v in outs), wt)
        assert all(torch.equal(a, p.grad) for a, p in zip(first, params))
        assert torch.equal(sums, again)
        assert all(torch.equal(a, v) for a, (_, v) in zip(first_outs, outs))
