"""Heterogeneous agents on the GPU: the fields gather with per-policy and agent-last sources
against torch, the bookkeeping with per-policy reward / action sources against a torch
restatement, a rollout of the example env (tests/custom_env/hetero_env*) replayed on its NumPy
twin, graph against eager, and A2C / PPO end to end with separate placeholders in both
observation layouts and with shared agent-last placeholders."""
import ctypes
import glob
import json
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "custom_env"))
SENTINEL = -7.25
GUARD = 97


# ---------------------------------------------------------------- fields gather
def _dest(E, Np, W):
    buf = torch.full((E * Np * W + GUARD,), SENTINEL, device="cuda")
    return buf, buf[:E * Np * W].view(E, Np, W)


def _random(g, shape, is_int):
    if is_int:
        return torch.randint(-1000, 1000, shape, device="cuda", generator=g, dtype=torch.int32)
    return torch.randn(shape, device="cuda", generator=g)


def _gather_case(E, nps, keys_of, mask_of, separate, last, seed):
    """nps: agents per policy; keys_of[i]: [(feature shape, is_int32)] of policy i (shared:
    every policy has keys_of[0]); mask_of[i]: mask width or 0.  Shared sources interleave the
    policies' agents.  Returns (descriptor, sources kept alive, destinations, expected)."""
    from warp_drive_b200 import lib as wlib

    g = torch.Generator(device="cuda").manual_seed(seed)
    P, N = len(nps), sum(nps)
    if separate:
        ids = [list(range(n)) for n in nps]
    else:
        order = [i for r in range(max(nps)) for i in range(P) if r < nps[i]]
        ids = [[a for a, q in enumerate(order) if q == i] for i in range(P)]
    a = wlib.GatherFields()
    a.n_envs, a.n_agents, a.n_policies = E, N, P
    keep, fields = [], []
    want_obs, want_mask = [[] for _ in range(P)], [None] * P
    owners = list(range(P)) if separate else [None]
    for i in owners:
        k = 0 if i is None else i
        ns = N if i is None else nps[i]
        specs = [(shape, is_int, False) for shape, is_int in keys_of[k]]
        if mask_of[k]:
            specs.append(((mask_of[k],), True, True))
        col = 0
        for shape, is_int, is_mask in specs:
            canon = _random(g, (E, ns) + tuple(shape), is_int)
            if is_mask:
                canon = canon.abs() % 2
            src = canon.movedim(1, -1).contiguous() if last else canon
            keep.append(src)
            width = int(np.prod(shape))
            fields.append((src, width, int(is_mask), 0 if is_mask else col, i, is_int))
            flat = canon.reshape(E, ns, width).float()
            for p in (range(P) if i is None else [i]):
                rows = flat if i is not None else flat.index_select(
                    1, torch.tensor(ids[p], device="cuda"))
                if is_mask:
                    want_mask[p] = rows
                else:
                    want_obs[p].append(rows)
            if not is_mask:
                col += width
    a.n_fields = len(fields)
    for j, (src, width, dst, col, i, is_int) in enumerate(fields):
        f = a.field[j]
        f.src, f.width, f.is_int32, f.dst, f.col = wlib.ptr(src), width, int(is_int), dst, col
        f.policy_mask, f.own_rows = (0, 0) if i is None else (1 << i, 1)
        f.agents_last = int(last)
    want_obs = [torch.cat(w, -1) for w in want_obs]
    dests = []
    ids32 = [torch.tensor(x, dtype=torch.int32, device="cuda") for x in ids]
    keep += ids32
    for p in range(P):
        io = a.policy[p]
        io.n_agents = nps[p]
        io.agent_ids = None if separate else wlib.ptr(ids32[p])
        ob, ov = _dest(E, nps[p], want_obs[p].shape[-1])
        mb, mv = (_dest(E, nps[p], want_mask[p].shape[-1]) if want_mask[p] is not None
                  else (None, None))
        io.rows[0], io.rows[1] = wlib.ptr(ov), (wlib.ptr(mv) if mv is not None else None)
        io.dst_width[0] = want_obs[p].shape[-1]
        io.dst_width[1] = want_mask[p].shape[-1] if want_mask[p] is not None else 0
        dests.append((ob, ov, mb, mv))
    a.dst_width[0], a.dst_width[1] = a.policy[0].dst_width[0], a.policy[0].dst_width[1]
    return a, keep, dests, (want_obs, want_mask)


KEYS_A = [((2, 3), False)]
KEYS_B = [((5,), False), ((3,), True), ((2, 2), False)]
KEYS_C = [((40,), False), ((3, 11), True)]
KEYS_D = [((33,), False), ((1,), True)]
GATHER_CASES = [
    # E, nps, keys per policy, mask widths, separate, agent-last
    (37, [45], [KEYS_A], [0], False, True),
    (50, [17, 16], [KEYS_B], [7], False, True),
    (9, [22, 21, 21], [KEYS_D], [0], False, True),
    (11, [3, 4, 2, 1], [KEYS_B], [5], False, False),
    (20, [1, 5, 33, 70], [KEYS_B, KEYS_A, KEYS_C, KEYS_D], [8, 0, 3, 0], True, False),
    (23, [1, 31, 100], [[((3,), False)], KEYS_C, KEYS_B], [8, 0, 4], True, True),
    (13, [2, 64], [KEYS_D, KEYS_A], [0, 0], True, True),
    (4000, [1, 100], [[((3,), False)], KEYS_A], [8, 0], True, True),   # several waves
]


def _case_id(c):
    return f"E{c[0]}-np{c[1]}-sep{int(c[4])}-last{int(c[5])}"


@pytest.mark.parametrize("case", GATHER_CASES, ids=_case_id)
def test_gather_fields_matches_torch(case):
    """Bit-exact against torch movedim / index_select / cat, guard regions untouched."""
    from warp_drive_b200 import lib as wlib

    E, nps, keys_of, mask_of, separate, last = case
    a, keep, dests, (want_obs, want_mask) = _gather_case(E, nps, keys_of, mask_of, separate,
                                                         last, seed=E + len(nps))
    wlib.check(wlib.load().wdb_gather_policy_fields(wlib.stream_ptr(), ctypes.byref(a)),
               "gather_policy_fields")
    torch.cuda.synchronize()
    for p, (ob, ov, mb, mv) in enumerate(dests):
        assert torch.equal(ov, want_obs[p]), (case, p)
        assert (ob[ov.numel():] == SENTINEL).all(), (case, p, "guard written")
        if mv is not None:
            assert torch.equal(mv, want_mask[p]), (case, p)
            assert (mb[mv.numel():] == SENTINEL).all(), (case, p, "mask guard written")
    del keep


def test_gather_fields_refuses_malformed_descriptors():
    from warp_drive_b200 import lib as wlib

    a, keep, _, _ = _gather_case(5, [2, 3], [KEYS_A, KEYS_A], [0, 0], True, True, seed=3)
    L = wlib.load()
    a.field[0].policy_mask = 3                       # own rows of two policies
    assert L.wdb_gather_policy_fields(wlib.stream_ptr(), ctypes.byref(a)) != 0
    a.field[0].policy_mask = 1 << 2                  # a policy the descriptor does not have
    assert L.wdb_gather_policy_fields(wlib.stream_ptr(), ctypes.byref(a)) != 0
    a.field[0].policy_mask, a.policy[0].dst_width[0] = 1, 5       # narrower than the field
    assert L.wdb_gather_policy_fields(wlib.stream_ptr(), ctypes.byref(a)) != 0
    del keep


# ---------------------------------------------------------------- bookkeeping
def test_bookkeep_per_policy_sources_match_torch():
    """Per-policy rewards [E, Np] and actions [E, Np, n_heads_p], six steps with raw done flags
    0 / 1 / 2: every batch slot bit-exact, the sums exact (integer rewards)."""
    from warp_drive_b200 import lib as wlib

    L = wlib.load()
    E, nps, heads = 300, [1, 7, 130], [2, 1, 3]
    g = torch.Generator(device="cuda").manual_seed(9)
    dev = "cuda"
    run = [torch.zeros(E, n, device=dev) for n in nps]
    epi = [torch.zeros((), device=dev) for _ in nps]
    steps = torch.zeros(E, dtype=torch.int32, device=dev)
    epi_steps = torch.zeros((), dtype=torch.int64, device=dev)
    n_done = torch.zeros((), dtype=torch.int64, device=dev)
    ref_run = [r.clone() for r in run]
    ref_epi = [0.0 for _ in nps]
    ref_steps, ref_epi_steps, ref_done = steps.clone(), 0, 0
    for t in range(6):
        rewards = [torch.randint(-3, 4, (E, n), device=dev, generator=g).float() for n in nps]
        actions = [torch.randint(0, 9, (E, n, h), device=dev, generator=g, dtype=torch.int32)
                   for n, h in zip(nps, heads)]
        done = (torch.rand(E, device=dev, generator=g) < 0.3).int() * torch.randint(
            1, 3, (E,), device=dev, generator=g, dtype=torch.int32)
        rb = [torch.full((E, n), SENTINEL, device=dev) for n in nps]
        ab = [torch.full((E, n, h), -5, dtype=torch.int32, device=dev)
              for n, h in zip(nps, heads)]
        db = torch.full((E,), -5, dtype=torch.int32, device=dev)
        k = wlib.Bookkeep()
        k.n_envs, k.n_agents, k.n_policies = E, sum(nps), len(nps)
        k.done, k.done_batch = wlib.ptr(done), wlib.ptr(db)
        k.step_running_sum, k.episodic_step_sum = wlib.ptr(steps), wlib.ptr(epi_steps)
        k.num_completed_episodes = wlib.ptr(n_done)
        for i in range(len(nps)):
            io = k.policy[i]
            io.n_agents = nps[i]
            io.rewards, io.actions = wlib.ptr(rewards[i]), wlib.ptr(actions[i])
            io.n_heads = heads[i]
            io.rewards_batch, io.actions_batch = wlib.ptr(rb[i]), wlib.ptr(ab[i])
            io.reward_running_sum, io.episodic_reward_sum = wlib.ptr(run[i]), wlib.ptr(epi[i])
        wlib.check(L.wdb_rollout_bookkeep(wlib.stream_ptr(), ctypes.byref(k)), "bookkeep")
        torch.cuda.synchronize()
        d = (done > 0)
        assert torch.equal(db, done)
        for i in range(len(nps)):
            assert torch.equal(rb[i], rewards[i]) and torch.equal(ab[i], actions[i])
            ref_run[i] += rewards[i]
            ref_epi[i] += float(ref_run[i][d].sum())
            ref_run[i][d] = 0
            assert torch.equal(run[i], ref_run[i])
        ref_steps += 1
        ref_epi_steps += int(ref_steps[d].sum())
        ref_steps[d] = 0
        ref_done += int(d.sum())
        assert torch.equal(steps, ref_steps)
    assert [float(e) for e in epi] == ref_epi
    assert int(epi_steps) == ref_epi_steps and int(n_done) == ref_done


# ---------------------------------------------------------------- the example env
def _trainer(tmp_path, algo="A2C", layout="first", with_planner=True, use_cuda_graph=True,
             E=64, N=6, L=10, T=10, iters=1, name="h", lr=0.001, seed=11):
    from hetero_env import CUDAHeteroEnv

    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.training.trainer import Trainer, load_run_config
    from warp_drive_b200.utils.env_registrar import EnvironmentRegistrar

    reg = EnvironmentRegistrar()
    reg.add_cuda_env_src_path("HeteroEnv", os.path.join(HERE, "custom_env", "hetero_env_step.cu"))
    env = CUDAHeteroEnv(num_agents=N, episode_length=L, with_planner=with_planner,
                        worker_obs_layout=layout, env_backend="pycuda")
    wrapper = EnvWrapper(env, num_envs=E, env_backend="pycuda", env_registrar=reg)
    cfg = load_run_config("tag_gridworld")
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, num_episodes=E * T * iters // L,
                          seed=seed)
    cfg["saving"].update(metrics_log_freq=1, model_params_save_freq=5, basedir=str(tmp_path))
    pol = cfg["policy"].pop("shared")
    pol.update(algorithm=algo, lr=lr, entropy_coeff=0.01)
    pol["model"]["fc_dims"] = [64, 64]
    pm = env.policy_tag_to_agent_id_map()
    cfg["policy"] = {p: json.loads(json.dumps(pol)) for p in pm}
    trainer = Trainer(env_wrapper=wrapper, config=cfg, policy_tag_to_agent_id_map=pm,
                      create_separate_placeholders_for_each_policy=with_planner,
                      obs_dim_corresponding_to_num_agents=layout, results_dir=name,
                      verbose=False, use_cuda_graph=use_cuda_graph)
    return trainer, wrapper, pm


def _batches(trainer):
    dm = trainer.cuda_envs.cuda_data_manager
    names = [n for n in dm._device_data_via_torch if "_batch" in n]
    return {n: dm.pull_data_from_device(n) for n in names}


ROLLOUT_CASES = [("first", True), ("last", True), ("last", False)]


@pytest.mark.parametrize("layout,with_planner", ROLLOUT_CASES)
def test_hetero_rollout_replays_on_the_cpu_twin(tmp_path, layout, with_planner):
    """A T-step engine rollout (episodes end and restart inside it), replayed on the NumPy twin
    with the actions the batches recorded: observations, masks, rewards and done flags are
    exactly the twin's; graph and eager rollouts are bit-identical."""
    from hetero_env import HeteroTwin

    E, N, L, T = 16, 6, 4, 10
    out = {}
    for graph in (True, False):
        tr, w, pm = _trainer(tmp_path, layout=layout, with_planner=with_planner,
                             use_cuda_graph=graph, E=E, N=N, L=L, T=T, name=f"r{graph}")
        eng = tr.engine
        assert eng.separate == with_planner and eng.agents_last == (layout == "last")
        assert eng.fused is None and eng.sa is None and eng.gather_fields
        if not graph:
            eng.step(-1)            # the graph path's warm-up step: same random draws after it
        eng.rollout()
        w.reset_all_envs()
        eng.resync_observations()
        eng.rollout()
        torch.cuda.synchronize()
        out[graph] = (_batches(tr), w.cuda_data_manager)
    (bg, dm), (be, _) = out[True], out[False]
    assert bg.keys() == be.keys()
    for n in bg:
        assert np.array_equal(bg[n], be[n]), f"graph and eager rollouts differ in {n}"
    nw = N - int(with_planner)
    twin = HeteroTwin(E, N, L, with_planner=with_planner)
    done = bg["done_flags_batch"]
    assert done.any() and not done.all()
    for t in range(T):
        o = twin.observe()
        assert np.array_equal(bg["processed_observations_batch_workers"][t],
                              o["workers"].reshape(E, nw, 6)), t
        planner = None
        if with_planner:
            assert np.array_equal(bg["processed_observations_batch_planner"][t][:, 0],
                                  o["planner_state"]), t
            mask = bg["action_mask_batch_planner"][t][:, 0]
            assert np.array_equal(mask, o["planner_mask"].astype(np.float32)), t
            planner = bg["sampled_actions_batch_planner"][t][:, 0]
        rew, d = twin.step(bg["sampled_actions_batch_workers"][t][..., 0], planner)
        assert np.array_equal(bg["rewards_batch_workers"][t], rew["workers"]), t
        if with_planner:
            assert np.array_equal(bg["rewards_batch_planner"][t][:, 0], rew["planner"]), t
        assert np.array_equal(done[t], d), t
    assert twin.invalid == 0 and int(dm.pull_data_from_device("invalid_actions")[0]) == 0
    # the step arrays hold the state after the last step, in the env's own layout
    o = twin.observe()["workers"]
    name = "observations_workers" if with_planner else "observations"
    raw = dm.pull_data_from_device(name)
    assert np.array_equal(raw, np.moveaxis(o, 1, -1) if layout == "last" else o)


def _episodic_rewards(trainer, pm):
    lines = [json.loads(l) for l in open(os.path.join(trainer.save_dir, "results.json"))]
    assert len(lines) == trainer.num_iters
    return {p: np.array([rec[p]["Mean episodic reward"] for rec in lines]) for p in pm}


TRAIN_CASES = [("A2C", "first", True), ("PPO", "first", True), ("A2C", "last", True),
               ("PPO", "last", True), ("A2C", "last", False), ("PPO", "last", False)]


@pytest.mark.parametrize("algo,layout,with_planner", TRAIN_CASES)
def test_train_hetero_env_end_to_end(tmp_path, algo, layout, with_planner):
    tr, w, pm = _trainer(tmp_path, algo, layout, with_planner, iters=60, lr=0.003)
    dm = w.cuda_data_manager
    tr.train()
    rewards = _episodic_rewards(tr, pm)
    for p, r in rewards.items():
        assert np.isfinite(r).all()
        assert r[-5:].mean() > 1.2 * r[:5].mean() + 1, (p, r[:5], r[-5:])
    assert int(dm.pull_data_from_device("invalid_actions")[0]) == 0
    # per-policy checkpoints, loadable into a fresh trainer
    for p in pm:
        files = glob.glob(os.path.join(tr.save_dir, f"{p}_*.state_dict"))
        assert files, p
        step_of = lambda f: int(  # noqa: E731
            os.path.basename(f).split(".state_dict")[0].split("_")[-1])
        last = max(files, key=step_of)
        assert step_of(last) == tr.current_timestep[p]
    t2, w2, _ = _trainer(tmp_path, algo, layout, with_planner, name="h2")
    t2.load_model_checkpoint({p: max(glob.glob(os.path.join(tr.save_dir, f"{p}_*.state_dict")),
                                     key=step_of) for p in pm})
    for p in pm:
        for a, b in zip(tr.models[p].parameters(), t2.models[p].parameters()):
            assert torch.equal(a.cpu(), b.cpu())
    # evaluation and the episode log, per policy
    rs, steps = t2.evaluate_episodes()
    assert set(rs) == set(pm)
    for p, ids in pm.items():
        assert rs[p].shape == (64, len(ids))
        assert torch.equal(steps[p], steps[next(iter(pm))]) and (steps[p] > 0).all()
    assert float(rs["workers"].sum(1).mean()) > 1.2 * rewards["workers"][0]
    if with_planner:
        assert float(rs["planner"].min()) >= 0
        states = t2.fetch_episode_states(["level", "announced"], env_id=3,
                                         include_rewards_actions=True, policy="planner",
                                         include_probabilities=True)
        assert states["level"].shape == (11,)
        assert states["sampled_actions_planner"].shape == (10, 1, 2)
        assert states["rewards_planner"].shape == (10, 1)
        assert np.array_equal(states["rewards_planner"][:, 0], states["announced"][1:])
        assert len(states["probabilities"]) == 10 and len(states["probabilities"][0]) == 2
        ws = t2.fetch_episode_states(["phase"], env_id=0, include_rewards_actions=True,
                                     policy="workers")
        assert ws["sampled_actions_workers"].shape == (10, N_WORKERS, 1)
        assert ws["rewards_workers"].shape == (10, N_WORKERS)
    assert int(w2.cuda_data_manager.pull_data_from_device("invalid_actions")[0]) == 0
    tr.graceful_close()


N_WORKERS = 5
