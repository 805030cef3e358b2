"""The SAC-family replay update passes -- wdb_sac_{critic,actor}_update_sampled,
wdb_sac_discrete_{critic,actor}_update_sampled and wdb_tqc_{critic,actor}_update_sampled --
against the float64 reference with error bars (tests/sac_update_bounds.py), element by element:
every gradient, every per-row output and the four loss sums within their bars (exactly the value
where the bar is 0), outputs filled with NaN before the launch, the guard regions untouched and a
second launch bit-identical.  The shapes cover one row, a partial tile, exactly 132 full tiles,
a tail tile after full ones and CTAs that run several tiles; a window that wraps the ring's end
and a duplicate; hidden widths [] to [64, 64, 64]; F + A = 64 (SAC, TQC with A = 32) and F = 63
with A = 64 (discrete SAC); several agents per env; gamma 0 and 1 with done flags 0, 1 and 2
inside windows; TQC at N = 2 and N = 32 with d = 0 and d = N - 1, with exact, few-ulp and
interleaved ties among the target atoms; SAC's raw log-std on both sides of its clamp and pinned
to it, |u| > 10 and log alpha at -10 and +2."""
import ctypes

import numpy as np
import pytest
import torch

from test_gpu_ddpg_update_exact import GUARD, SENTINEL
from test_q_update_bounds_cpu import within
from test_sac_update_bounds_cpu import Case, make_models

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _guarded(shape):
    """A NaN-filled view inside a buffer whose GUARD floats on each side hold SENTINEL."""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * GUARD,), SENTINEL, device=DEV)
    buf[GUARD:GUARD + n] = float("nan")
    return buf, buf[GUARD:GUARD + n].view(shape)


def _guard_grads(models):
    guards = []
    for m in models:
        for p in m.parameters():
            buf, view = _guarded(p.shape)
            p.grad = view
            guards.append(buf)
    return guards


def _untouched(guards):
    return all(bool((b[:GUARD] == SENTINEL).all()) and bool((b[-GUARD:] == SENTINEL).all())
               for b in guards)


def _np(t):
    return t.detach().double().cpu().numpy()


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _fused(case, models):
    """The fused update of the case's kind, the names of its per-row outputs and launch(outs),
    which runs the critic pass, then the actor pass, writing those outputs."""
    actor, c1, c2, t1, t2 = models
    la = torch.tensor([case.log_alpha], device=DEV)
    E, Np, C, ns, B = case.E, case.Np, case.C, case.n_step, case.B
    ring = [_dev(r) for r in case.ring]
    w = _dev(case.windows)
    nc, na = _dev(case.noise_c), _dev(case.noise_a)
    if case.kind == "sac":
        from warp_drive_b200.training.algorithms.fused_sac import FusedSACUpdate

        fused = FusedSACUpdate(actor, c1, c2, t1, t2, la, E, Np, C, ns, case.gamma,
                               replay_rows=B)
        names = ("q1", "q2", "returns", "log_probs")

        def launch(outs):
            fused.critic_launch(*ring, 0, nc, outs[:3], windows=w)
            fused.actor_launch(ring[0], 0, na, outs[3], windows=w)
    elif case.kind == "discrete":
        from warp_drive_b200.training.algorithms.fused_sac_discrete import (
            FusedDiscreteSACUpdate)

        assert FusedDiscreteSACUpdate.supported(actor, c1, c2, E, Np, C, ns, B)
        fused = FusedDiscreteSACUpdate(actor, c1, c2, t1, t2, la, E, Np, C, ns, case.gamma, B)
        names = ("q1", "q2", "returns", "entropies")

        def launch(outs):
            fused.critic_launch(*ring, w, outs[:3])
            fused.actor_launch(ring[0], w, outs[3])
    else:
        from warp_drive_b200.training.algorithms.fused_tqc import FusedTQCUpdate
        from warp_drive_b200.training.algorithms.tqc import TQC

        algo = TQC(discount_factor_gamma=case.gamma, n_step=ns, action_dim=case.A, n_critics=2,
                   n_quantiles=case.N, drop_per_net=case.d)
        assert FusedTQCUpdate.supported(algo, actor, [c1, c2], E, Np, C, ns, B)
        fused = FusedTQCUpdate(algo, actor, [c1, c2], [t1, t2], la, E, Np, C, ns, B)
        names = ("q_means", "target_means", "log_probs")

        def launch(outs):
            fused.critic_launch(*ring, nc, w, outs[:2])
            fused.actor_launch(ring[0], na, w, outs[2])
    return fused, names, launch


# (kind, B, n_step, C, E, Np, F, A, actor dims, critic dims, extra)
CASES = [
    ("sac", 1, 3, 9, 4, 1, 4, 2, [64, 64], [64, 64], {}),
    ("sac", 17, 1, 6, 3, 3, 4, 3, [1], [1], dict(gamma=0.0)),
    ("sac", 2112, 3, 40, 16, 1, 3, 1, [5, 7, 9], [5, 7, 9], dict(gamma=1.0,
                                                                 done_vals=(0, 1, 2))),
    ("sac", 2113, 3, 40, 16, 1, 32, 32, [], [16], dict(noise_scale=12.0, log_alpha=-10.0)),
    ("sac", 4099, 2, 11, 16, 3, 3, 2, [64, 64, 64], [16, 16],
     dict(lo=-0.3, hi=0.2, log_alpha=2.0, pin=[(0, -0.3), (1, 0.2)])),
    ("sac", 333, 3, 12, 8, 1, 4, 3, [16], [64, 64],
     dict(lo=-0.5, hi=0.5, log_std_bias=0.4, pin=[(0, -3.0), (2, 1.5)])),
    ("discrete", 1, 3, 9, 4, 1, 4, 2, [], [], {}),
    ("discrete", 17, 1, 6, 3, 3, 4, 3, [1], [1], dict(gamma=0.0, done_vals=(0, 1, 2))),
    ("discrete", 2112, 3, 40, 16, 1, 4, 3, [5, 7, 9], [5, 7, 9], dict(gamma=1.0,
                                                                      done_vals=(0, 1, 2))),
    ("discrete", 2113, 2, 12, 16, 1, 63, 64, [32], [32, 32], dict(log_alpha=2.0)),
    ("discrete", 4099, 2, 11, 16, 3, 4, 2, [64, 64, 64], [16, 16], dict(log_alpha=-10.0)),
    ("tqc", 1, 3, 9, 4, 1, 3, 1, [], [], dict(N=2, d=0)),
    ("tqc", 17, 1, 6, 3, 3, 4, 3, [1], [1], dict(N=2, d=1, gamma=0.0)),
    ("tqc", 2112, 3, 40, 16, 1, 3, 1, [5, 7, 9], [5, 7, 9],
     dict(N=32, d=0, gamma=1.0, ties="straddle", done_vals=(0, 1, 2))),
    ("tqc", 2113, 3, 40, 16, 1, 3, 2, [64, 64], [48, 48], dict(N=32, d=31, ties="ulp")),
    ("tqc", 4099, 2, 11, 16, 3, 32, 32, [64, 64, 64], [16], dict(N=8, d=3, ties="exact")),
    ("tqc", 333, 3, 12, 8, 1, 3, 1, [64, 64], [64, 64],
     dict(N=25, d=2, noise_scale=12.0, log_alpha=-10.0, lo=-2.0, hi=0.5, log_std_bias=0.3)),
]


def _case_id(c):
    kind, B, _, _, _, _, F, A, ad, cd, extra = c
    tag = "".join(f"_{k}{v}" for k, v in extra.items() if k in ("N", "d", "ties"))
    return f"{kind}_B{B}_F{F}_A{A}_L{len(ad)}{len(cd)}{tag}"


@pytest.mark.parametrize("c", CASES, ids=[_case_id(c) for c in CASES])
def test_sac_family_passes_within_their_float64_bars(c):
    kind, B, n_step, C, E, Np, F, A, ad, cd, extra = c
    case = Case(kind, B, n_step, C, E, Np, F, A, ad, cd, **extra)
    ref_c, ref_a = case.reference()
    assert ref_c["ok"].all() and ref_a["ok"].all()       # no kept row sits on a branch
    models = [m.to(DEV) for m in case.models]
    fused, names, launch = _fused(case, models)
    trained = models[:3]
    guards = _guard_grads(trained)
    outs = [_guarded((B,)) for _ in names]
    guards += [b for b, _ in outs]
    fused.sums.fill_(float("nan"))
    launch(tuple(v for _, v in outs))
    torch.cuda.synchronize()
    first = [p.grad.clone() for m in trained for p in m.parameters()]
    first_outs = [v.clone() for _, v in outs]
    sums = fused.sums.clone()
    want = ref_a["grads"] + ref_c["grads1"] + ref_c["grads2"]
    labels = [f"actor {n}" for n, _ in models[0].named_parameters()] + \
        [f"critic{k} {n}" for k in (1, 2) for n, _ in models[k].named_parameters()]
    got = [p.grad for p in models[0].parameters()] + \
        [p.grad for k in (1, 2) for p in models[k].parameters()]
    ratios = {}
    for label, g, wv in zip(labels, got, want):
        ratios[label] = within(_np(g), wv, label)
    per_row = {**{k: ref_c[k] for k in ref_c if k in names}, **{k: ref_a[k] for k in ref_a
                                                                 if k in names}}
    for (_, v), name in zip(outs, names):
        ratios[name] = within(_np(v), per_row[name], name)
    for i, (v, b) in enumerate(ref_c["sums"] + ref_a["sums"]):
        err = abs(float(sums[i]) - v)
        assert err <= b, (f"sums[{i}]", float(sums[i]), v, b)
        ratios[f"sums[{i}]"] = err / b if b > 0 else 0.0
    assert _untouched(guards)
    launch(tuple(v for _, v in outs))
    torch.cuda.synchronize()
    assert all(torch.equal(a, p.grad) for a, p in
               zip(first, [p for m in trained for p in m.parameters()]))
    assert all(torch.equal(a, v) for a, (_, v) in zip(first_outs, outs))
    assert torch.equal(sums, fused.sums)
    worst = max(ratios, key=ratios.get)
    print(f"\nRATIO {_case_id(c)}: max |err|/bar {ratios[worst]:.3g} ({worst})")
    for pass_name, keys in (("critic", [k for k in ratios if k.startswith("critic")]
                             + ["sums[0]", "sums[1]"]),
                            ("actor", [k for k in ratios if k.startswith("actor")]
                             + ["sums[2]", "sums[3]"])):
        k = max(keys, key=ratios.get)
        print(f"RATIO {_case_id(c)} {pass_name}: {ratios[k]:.3g} ({k})")


def test_tqc_passes_refuse_one_quantile():
    """The TQC passes take N >= 2 (TQC itself refuses N = 1), so N = 1 is not in CASES: its
    struct is refused, and N = 2 of the same shape is taken."""
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.fused_tqc import _shape_struct

    lib = wlib.load()
    for N, want in ((1, 0), (2, 1)):
        actor, c1 = make_models("tqc", 3, 1, [8], [8], N=N)[:2]
        u = _shape_struct(actor, c1, 4, 1, 9, 2, 0)
        assert lib.wdb_tqc_critic_update_sampled_supported(ctypes.byref(u), 17) == want
        assert lib.wdb_tqc_actor_update_sampled_supported(ctypes.byref(u), 17) == want
