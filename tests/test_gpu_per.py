"""Prioritized replay on the GPU: the sampler (wdb_per_sample_windows) and the tree writes
(wdb_per_admit, wdb_per_set_priorities) against the float64 reference (tests/per_reference.py),
the importance-weighted DQN pass (wdb_dqn_update_prioritized) against the reference and against
the unweighted pass, and TrainerDQN with `prioritized_replay`."""
import numpy as np
import pytest
import torch

import dqn_update_reference as dqn_ref
import per_reference as ref
from test_gpu_ddpg_update_exact import _guarded
from test_gpu_dqn import (REL, SHAPES, _delta_off_the_kink, _dev, _guard_grads, _pick_windows,
                          _rel, _ring32, _trainer, _untouched)

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _store(C, n_rows, n_step, rows, alpha=0.6, eps=1e-6):
    from warp_drive_b200.training.utils.prioritized_replay import PrioritizedReplay

    return PrioritizedReplay(C, n_rows, n_step, rows, alpha, eps, DEV)


def _load(st, leaves):
    """A store holding `leaves` and the reference's fresh tree over them."""
    st.leaves.copy_(torch.from_numpy(np.asarray(leaves, np.float32)))
    st.nodes.copy_(torch.from_numpy(ref.flat_nodes(ref.build_tree(leaves))))


def _sample(st, B, seed, counter, beta=0.4):
    windows = torch.zeros((B, 2), dtype=torch.int32, device=DEV)
    st.set_beta(beta)
    st.sample(windows, seed, counter)
    return windows.cpu().numpy(), st.priorities.cpu().numpy(), st.weights.cpu().numpy()


def _tree_is_fresh(st):
    leaves = st.leaves.cpu().numpy()
    return np.array_equal(st.nodes.cpu().numpy(), ref.flat_nodes(ref.build_tree(leaves)))


def _leaves(n, seed, zero_share=0.5, decades=12):
    g = np.random.default_rng(seed)
    p = (10.0 ** g.uniform(-decades / 2, decades / 2, n)).astype(np.float32)
    p[g.random(n) < zero_share] = 0
    return p


# ------------------------------------------------------------------------ the sampler
@pytest.mark.parametrize("C,n_rows,B", [(40, 1000, 256), (1000, 1000, 4096), (50, 7, 50000)])
def test_sampler_matches_the_reference_on_fixed_trees(C, n_rows, B):
    leaves = _leaves(C * n_rows, C, zero_share=0.3)
    st = _store(C, n_rows, 3, B)
    _load(st, leaves)
    w, p, wt = _sample(st, B, 1234, 77)
    want_w, want_p, u = ref.sample(leaves, n_rows, B, 1234, 77)
    assert np.array_equal(w, want_w)
    assert np.array_equal(p, want_p)
    assert np.abs(wt / ref.weights(want_p, 0.4) - 1).max() <= 1e-5
    assert wt.max() == 1.0 and (p > 0).all()
    # each row in its own stratum: the leaf's cumulative interval meets [lo, hi]
    S = ref.build_tree(leaves)[-1][0]
    _, lo, hi = ref.segment_points(S, np.zeros(B))
    leaf = w[:, 0].astype(np.int64) * n_rows + w[:, 1]
    ends = np.cumsum(leaves.astype(np.float64))
    starts = ends - leaves
    tol = 1e-9 * S
    assert ((starts[leaf] <= hi + tol) & (ends[leaf] >= lo - tol)).all()
    # the same (seed, counter) gives the same windows; another counter others
    assert np.array_equal(_sample(st, B, 1234, 77)[0], w)
    assert not np.array_equal(_sample(st, B, 1234, 78)[0], w)


def test_sampler_never_returns_a_zero_leaf():
    C, n_rows, B = 100, 333, 4096
    n = C * n_rows
    st = _store(C, n_rows, 3, B)
    for at in (0, n // 2 + 17, n - 1):
        leaves = np.zeros(n, np.float32)
        leaves[at] = 1e-38
        _load(st, leaves)
        w, p, wt = _sample(st, B, 5, at)
        assert ((w[:, 0].astype(np.int64) * n_rows + w[:, 1]) == at).all(), at
        assert (p == np.float32(1e-38)).all() and (wt == 1).all()
    leaves = _leaves(n, 9, zero_share=0.95, decades=70)       # 1e-35 .. 1e35
    _load(st, leaves)
    for counter in range(5):
        w, p, _ = _sample(st, B, 6, counter)
        assert (leaves[w[:, 0].astype(np.int64) * n_rows + w[:, 1]] > 0).all()
        assert np.array_equal(w, ref.sample(leaves, n_rows, B, 6, counter)[0])


def test_alpha_zero_reaches_every_valid_window_and_no_other():
    """alpha = 0 over a partly filled, then wrapped store: every valid window has priority 1,
    and B = 3 x (valid windows) stratified draws hit each of them and nothing else."""
    C, E, T, n_step = 37, 5, 8, 3
    st = _store(C, E, n_step, 1, alpha=0.0)
    cursor, filled = 0, 0
    for r in range(7):                                  # 56 slots: the ring wraps
        before = (cursor, filled)
        cursor, filled = (cursor + T) % C, min(C, filled + T)
        st.admit(before, (cursor, filled))
        if r in (2, 6):
            oldest = cursor if filled == C else 0
            ok = ref.valid_starts(C, oldest, filled, n_step)
            valid = {(s, n) for s in np.flatnonzero(ok) for n in range(E)}
            st.priorities = torch.zeros(3 * len(valid), device=DEV)
            st.weights = torch.zeros(3 * len(valid), device=DEV)
            w, p, wt = _sample(st, 3 * len(valid), 3, r)
            assert {(int(s), int(n)) for s, n in w} == valid
            assert (p == 1).all() and (wt == 1).all()


# ------------------------------------------------------------------------ the tree
def test_set_priorities_keeps_the_tree_fresh_and_duplicates_order_free():
    C, n_rows, n_step, B = 300, 200, 3, 4096
    st, twin = _store(C, n_rows, n_step, B), _store(C, n_rows, n_step, B)
    leaves = _leaves(C * n_rows, 1, zero_share=0.0, decades=4)
    oldest, filled = 17, C
    ok = np.repeat(ref.valid_starts(C, oldest, filled, n_step), n_rows)
    leaves[~ok] = 0
    _load(st, leaves)
    _load(twin, leaves)
    g = np.random.default_rng(2)
    p_max = np.float32(1.0)
    for batch in range(6):
        w = np.stack([g.integers(0, C, B), g.integers(0, n_rows, B)], axis=1).astype(np.int32)
        w[B // 2:B // 2 + 300] = w[:300]                 # forced duplicates
        q = g.standard_normal(B).astype(np.float32) * 10 ** (batch - 2)
        r = g.standard_normal(B).astype(np.float32)
        want, p_max = ref.set_priorities(st.leaves.cpu().numpy(), p_max, w, q, r, 0.6, 1e-6, C,
                                         n_rows, n_step, oldest, filled)
        dw = torch.from_numpy(w).to(DEV)
        st.set_priorities(dw, torch.from_numpy(q).to(DEV), torch.from_numpy(r).to(DEV), oldest,
                          filled)
        got = st.leaves.cpu().numpy()
        assert np.allclose(got, want, rtol=1e-6, atol=0)   # powf against NumPy's
        assert ((got > 0) == ok).all()
        assert _tree_is_fresh(st)
        assert st.p_max.item() == p_max                    # |Q - R| + eps in float32: exact
        perm = g.permutation(B)                            # the same batch in another order
        twin.set_priorities(dw[perm].contiguous(), torch.from_numpy(q[perm]).to(DEV),
                            torch.from_numpy(r[perm]).to(DEV), oldest, filled)
        assert torch.equal(twin.leaves, st.leaves) and torch.equal(twin.nodes, st.nodes)
        assert torch.equal(twin.p_max, st.p_max)


@pytest.mark.parametrize("C,T,n_step,E", [(11, 8, 3, 4), (5000, 4, 3, 256), (13, 1, 5, 3)])
def test_admit_keeps_the_invariant_and_the_tree_across_wraps(C, T, n_step, E):
    """C = T + n_step wraps on every rollout; priorities written between rollouts survive
    until their slots are rewritten."""
    st = _store(C, E, n_step, 64)
    g = np.random.default_rng(C)
    cursor, filled, p_max = 0, 0, np.float32(1.0)
    leaves = np.zeros(C * E, np.float32)
    rounds = 3 * -(-C // T) if C < 100 else 40
    for r in range(rounds):
        before = (cursor, filled)
        cursor, filled = (cursor + T) % C, min(C, filled + T)
        st.admit(before, (cursor, filled))
        leaves = ref.admit(leaves, p_max, 0.6, C, E, n_step, before, (cursor, filled))
        oldest = cursor if filled == C else 0
        ok = np.repeat(ref.valid_starts(C, oldest, filled, n_step), E)
        got = st.leaves.cpu().numpy()
        assert ((got > 0) == ok).all(), r
        assert np.allclose(got, leaves, rtol=1e-6, atol=0)
        assert _tree_is_fresh(st), r
        if filled >= n_step + 1:                          # new priorities, p_max moves
            w = np.stack([g.integers(0, C, 64), g.integers(0, E, 64)], axis=1).astype(np.int32)
            q = (g.standard_normal(64) * (r + 1)).astype(np.float32)
            rr = np.zeros(64, np.float32)
            leaves, p_max = ref.set_priorities(got, p_max, w, q, rr, 0.6, 1e-6, C, E, n_step,
                                               oldest, filled)
            st.set_priorities(torch.from_numpy(w).to(DEV), torch.from_numpy(q).to(DEV),
                              torch.from_numpy(rr).to(DEV), oldest, filled)
            assert st.p_max.item() == p_max and _tree_is_fresh(st)
            leaves = st.leaves.cpu().numpy()


# ------------------------------------------------------------------------ the weighted pass
@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max_target"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"B{s[0]}" for s in SHAPES])
def test_weighted_pass_matches_the_float64_reference(shape, double_q):
    from warp_drive_b200.training.algorithms.dqn import DQN
    from warp_drive_b200.training.algorithms.fused_dqn import FusedDQNUpdate

    B, n_step, C, E, Np, F, A, dims = shape
    gamma = 0.97
    q_net, target = dqn_ref.make_q_models(F, A, dims, seed=B)
    with torch.no_grad():
        for p in target.parameters():
            p.add_(0.3 * torch.randn_like(p))
    q_net, target = q_net.float(), target.float()
    ring = _ring32(C, E, Np, F, A, B)
    windows = _pick_windows((q_net, target), ring, B, n_step, B, double_q)
    wts = np.random.default_rng(B).uniform(0.01, 1.0, B).astype(np.float32)
    probe = dqn_ref.dqn_sampled((q_net, target), ring, windows, n_step, gamma, 1e9, double_q)
    delta = _delta_off_the_kink(probe["diff"])
    want = ref.dqn_weighted((q_net, target), ring, windows, wts.astype(np.float64), n_step,
                            gamma, delta, double_q)
    q_net, target = q_net.to(DEV), target.to(DEV)
    guards = _guard_grads(q_net)
    outs = [_guarded((B,), DEV) for _ in range(3)]
    guards += [b for b, _ in outs]
    outs[2][1].copy_(torch.from_numpy(wts))
    algo = DQN(gamma, n_step=n_step, double_q=double_q, huber_delta=delta)
    fused = FusedDQNUpdate(algo, q_net, target, E, Np, C, B)
    w = torch.from_numpy(windows).to(DEV)
    ring_d = _dev(ring)
    sums = fused.launch(*ring_d, w, (outs[0][1], outs[1][1]), outs[2][1]).clone()
    first = [p.grad.clone() for p in q_net.parameters()]
    for got, key in zip(first, want["grads"]):
        assert _rel(got, key) <= REL
    assert _rel(outs[0][1], want["q"]) <= REL and _rel(outs[1][1], want["returns"]) <= REL
    assert float(sums[0]) == pytest.approx(want["sum_huber"], rel=REL)
    assert float(sums[1]) == pytest.approx(want["sum_q"], rel=REL, abs=REL * B)
    assert _untouched(guards)
    again = fused.launch(*ring_d, w, (outs[0][1], outs[1][1]), outs[2][1])
    assert all(torch.equal(a, p.grad) for a, p in zip(first, q_net.parameters()))
    assert torch.equal(sums, again)
    # unit weights: the unweighted pass, bit for bit
    ones = torch.ones(B, device=DEV)
    s1 = fused.launch(*ring_d, w, None, ones).clone()
    g1 = [p.grad.clone() for p in q_net.parameters()]
    s0 = fused.launch(*ring_d, w).clone()
    assert torch.equal(s1, s0)
    assert all(torch.equal(a, p.grad) for a, p in zip(g1, q_net.parameters()))


# ------------------------------------------------------------------------ the trainer
_PER = {"prioritized_replay": True, "priority_beta": [[0, 0.4], [10 ** 5, 1.0]]}


def _store_state(st):
    return [t.clone() for t in (st.leaves, st.nodes, st.p_max)]


def test_trainer_fused_and_torch_prioritized_updates_agree(tmp_path):
    import copy

    from warp_drive_b200 import lib as wlib

    tr = _trainer(tmp_path, trainer=dict(_PER))
    st = tr.priority_stores["shared"]
    for it in range(3):
        tr._generate_rollout_batch()
    assert tr.engine.ring_filled == 24
    assert float(st.leaves.max()) == 1.0                # every window entered at p_max = 1
    tr._one_update(False, {})                           # priorities that differ: weights < 1
    assert float(st.p_max) > 1.0
    opt = tr.optimizers["shared"]
    nets = [p for m in tr._all_networks("shared") for p in m.parameters()]
    state = ([p.detach().clone() for p in nets], copy.deepcopy(opt.state_dict()),
             dict(tr.current_timestep), dict(tr.update_count), tr.replay_draws, _store_state(st))
    results = {}
    for fused in (True, False):
        params, o, ts, counts, draws, store = state
        with torch.no_grad():
            for p, v in zip(nets, params):
                p.copy_(v)
        opt.load_state_dict(o)
        tr.current_timestep.update(ts)
        tr.update_count.update(counts)
        tr.replay_draws = draws
        for t, v in zip((st.leaves, st.nodes, st.p_max), store):
            t.copy_(v)
        tr.trainers["shared"].use_fused_update = fused
        step_info = {"shared": ({}, {})}
        tr._one_update(True, step_info)                 # one update from identical state
        results[fused] = ([p.detach().clone() for p in nets], st.leaves.clone(),
                          st.weights.clone(), tr.replay_windows["shared"].clone())
    tr.trainers["shared"].use_fused_update = True
    (pf, lf, wf, winf), (pt, lt, wt, wint) = results[True], results[False]
    assert torch.equal(winf, wint) and torch.equal(wf, wt)     # the same draw and weights
    assert float(wf.min()) < 1 and float(wf.max()) == 1
    for a, b in zip(pf, pt):
        assert float((a - b).norm() / b.norm().clamp_min(1e-30)) <= 1e-5
    assert float((lf - lt).abs().max()) <= 1e-5 * float(lt.max())
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
    # sample (2), the weighted pass (2), the priorities (2 + levels), clipping + Adam (2)
    assert counts == [3 * (2 + 2 + 2 + st.levels + 2)] * 2


def test_trainer_trains_through_wrap_around_with_finite_metrics(tmp_path):
    tr = _trainer(tmp_path, E=16, trainer=dict(_PER))
    st = tr.priority_stores["shared"]
    C = tr.ring_capacity
    for it in range(30):                                # 240 slots > 203: wraps
        tr._generate_rollout_batch()
        m = tr._update_model_params(0 if it in (5, 29) else 1)
        eng = tr.engine
        oldest = eng.ring_cursor if eng.ring_filled == C else 0
        ok = np.repeat(ref.valid_starts(C, oldest, eng.ring_filled, tr.n_step), 16)
        assert ((st.leaves.cpu().numpy() > 0) == ok).all(), it
        if it in (5, 29):
            s = m["shared"]
            for k in ("Q loss", "Mean Q value", "Priority beta", "Mean IS weight",
                      "Max priority"):
                assert np.isfinite(s[k]), k
            assert 0.4 <= s["Priority beta"] <= 1 and 0 < s["Mean IS weight"] <= 1
            assert s["Max priority"] >= 1
    assert _tree_is_fresh(st)
    assert all(torch.isfinite(p).all() for p in tr.q_models["shared"].parameters())


@pytest.mark.parametrize("one_launch", [True, False], ids=["one_launch", "per_step"])
def test_both_rollout_paths_feed_admit_and_plain_configs_launch_as_before(one_launch,
                                                                         tmp_path):
    from warp_drive_b200 import lib as wlib

    plain, per = _trainer(tmp_path, name="a"), _trainer(tmp_path, name="b", trainer=dict(_PER))
    assert plain.prioritized is None and plain.priority_stores == {}
    if not one_launch:
        plain.engine.sa = per.engine.sa = None
    st = per.priority_stores["shared"]
    launches = {}
    for name, tr in (("plain", plain), ("per", per)):
        counts = []
        for it in range(30):
            n0 = wlib.launch_count()
            tr._generate_rollout_batch()
            counts.append(wlib.launch_count() - n0)
        launches[name] = counts
    assert [b - a for a, b in zip(launches["plain"], launches["per"])] == [1 + st.levels] * 30
    eng = per.engine
    oldest = eng.ring_cursor if eng.ring_filled == per.ring_capacity else 0
    ok = np.repeat(ref.valid_starts(per.ring_capacity, oldest, eng.ring_filled, per.n_step),
                   per.num_envs)
    assert ((st.leaves.cpu().numpy() > 0) == ok).all() and _tree_is_fresh(st)
