"""GPU tests of the fused rollout timestep (wdb_tag_continuous_rollout_step) and of the
RolloutEngine: the single-launch path must produce exactly what the separate
sample / step / bookkeeping / reset calls produce (which are themselves pinned to the
oracle and to the reference kernels in test_gpu_envs.py / test_gpu_core.py)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ENV_KW = dict(num_taggers=3, num_runners=20, grid_length=10.0, episode_length=40,
              max_acceleration=0.1, min_acceleration=-0.1, max_turn=2.356, min_turn=-2.356,
              num_acceleration_levels=20, num_turn_levels=20, seed=274880,
              use_full_observation=False, num_other_agents_observed=5,
              tag_reward_for_tagger=10.0, tag_penalty_for_runner=-10.0,
              edge_hit_penalty=-0.5, tagging_distance=0.08, step_reward_for_runner=0.01)


_BPE = 1     # blocks_per_env of the wrappers built here (tests/test_gpu_wide.py re-runs with 2)


def _setup(E, T, full_obs=False, seed=11, **env_kw):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.tag_continuous import TagContinuous
    from warp_drive_b200.managers.function_manager import CUDASampler
    from warp_drive_b200.training.utils.data_loader import create_and_push_data_placeholders

    kw = dict(ENV_KW, use_full_observation=full_obs, **env_kw)
    env = TagContinuous(**kw)
    wrapper = EnvWrapper(env, num_envs=E, env_backend="b200", blocks_per_env=_BPE)
    wrapper.reset_all_envs()
    policy_map = {"runner": sorted(env.runners), "tagger": sorted(env.taggers)}
    sampler = CUDASampler(wrapper.cuda_function_manager)
    create_and_push_data_placeholders(env_wrapper=wrapper, action_sampler=sampler,
                                      policy_tag_to_agent_id_map=policy_map,
                                      training_batch_size_per_env=T)
    sampler.init_random(seed)
    return wrapper, sampler, policy_map


STATE = ("loc_x", "loc_y", "speed", "direction", "acceleration", "edge_hit_reward_penalty",
         "still_in_the_game", "num_runners", "nearest_neighbor_ids", "_done_", "_timestep_",
         "observations", "rewards", "sampled_actions")


def _process_tc_variant():
    """tc_variant as the library set it when it loaded: from WDB_OPTIONS, else 1."""
    for item in os.environ.get("WDB_OPTIONS", "").split(","):
        key, _, val = item.partition("=")
        if key.strip() == "tc_variant":
            return int(val)
    return 1


@pytest.fixture
def tc_variant(request, wdb_lib):
    """The kernel of a small-env step: 1 = packed, 2 = second-generation (tc_v2_eligible
    accepts this file's 23-agent, K = 5, partial-observation shape)."""
    assert wdb_lib.wdb_set_option(b"tc_variant", request.param) == 0
    try:
        yield request.param
    finally:
        wdb_lib.wdb_set_option(b"tc_variant", _process_tc_variant())


@pytest.mark.parametrize("full_obs, tc_variant", [
    pytest.param(False, 1, id="False"), pytest.param(True, 1, id="True"),
    pytest.param(False, 2, id="False-v2")], indirect=["tc_variant"])
def test_fused_step_equals_separate_calls(full_obs, tc_variant):
    from warp_drive_b200.training.fused_tag_continuous import FusedTagContinuousStep

    E, T = 10, 4
    wa, sa, pm = _setup(E, T, full_obs)
    wb, sb, _ = _setup(E, T, full_obs)
    dma, dmb = wa.cuda_data_manager, wb.cuda_data_manager
    N = wa.n_agents
    ids = {p: torch.as_tensor(v, device="cuda") for p, v in pm.items()}
    fused = FusedTagContinuousStep(wb, pm, sb)
    run = {p: torch.zeros((E, len(v)), device="cuda") for p, v in pm.items()}
    ep_sum = {p: torch.zeros((), device="cuda") for p in pm}
    steps = torch.zeros(E, dtype=torch.int32, device="cuda")
    ep_steps = torch.zeros((), dtype=torch.int64, device="cuda")
    n_done = torch.zeros((), dtype=torch.int64, device="cuda")
    fused.set_bookkeeping(run, ep_sum, steps, ep_steps, n_done)
    ref_run = {p: torch.zeros((E, len(v)), device="cuda") for p, v in pm.items()}
    ref_ep = {p: 0.0 for p in pm}
    ref_steps = torch.zeros(E, dtype=torch.int64, device="cuda")
    ref_ep_steps, ref_n_done = 0, 0
    g = torch.Generator(device="cuda").manual_seed(5)
    F = dma.get_shape("observations")[2]
    total_done = 0
    for t in range(100):
        probs = {p: [torch.softmax(2 * torch.randn((E, len(v), 21), device="cuda", generator=g), -1)
                     for _ in range(2)] for p, v in pm.items()}
        u = torch.rand((E, N, 2), device="cuda", generator=g).clamp_min(1e-7)
        # ---- A: separate calls (combined probs -> sampler x2 -> step -> reset)
        acts = dma.data_on_device_via_torch("sampled_actions")
        for k in range(2):
            comb = torch.zeros((E, N, 21), device="cuda")
            for p in pm:
                comb[:, ids[p]] = probs[p][k]
            sa.sample(dma, comb, f"sampled_actions_{k}", combined=(acts, 2, k),
                      uniforms=u[:, :, k].contiguous())
        wa.step_all_envs()
        done_a = dma.data_on_device_via_torch("_done_").clone()
        rew_a = dma.data_on_device_via_torch("rewards").clone()
        acts_a = acts.clone()
        for p in pm:
            ref_run[p] += rew_a[:, ids[p]]
            ref_ep[p] += float((ref_run[p] * done_a[:, None]).sum())
            ref_run[p] *= (1 - done_a[:, None])
        ref_steps += 1
        ref_ep_steps += int((ref_steps * done_a).sum())
        ref_steps *= (1 - done_a)
        ref_n_done += int(done_a.sum())
        wa.reset_only_done_envs()
        # ---- B: one fused launch
        slot = t % T
        ab = {p: dmb.data_on_device_via_torch(f"sampled_actions_batch_{p}")[slot] for p in pm}
        # one step with the first policy's action slot NULL: that disables the action push for
        # every policy, so the second policy's slot must stay untouched
        null_push = t == 1
        if null_push:
            ab = {p: None if i == 0 else torch.full_like(ab[p], -3) for i, p in enumerate(pm)}
        rb = {p: dmb.data_on_device_via_torch(f"rewards_batch_{p}")[slot] for p in pm}
        ob = {p: torch.full((E, len(v), F), -7.0, device="cuda") for p, v in pm.items()}
        db = dmb.data_on_device_via_torch("done_flags_batch")[slot]
        fused.launch(probs, actions_batch=ab, rewards_batch=rb, obs_next=ob, done_batch=db,
                     uniforms=u)
        torch.cuda.synchronize()
        for k in STATE:
            ta, tb = dma.data_on_device_via_torch(k), dmb.data_on_device_via_torch(k)
            if k == "rewards":
                ta = rew_a
            if k == "nearest_neighbor_ids":
                continue   # stale tails differ only where invalid; covered via observations
            assert torch.equal(ta, tb), (t, k)
        assert torch.equal(dmb.data_on_device_via_torch("sampled_actions_0")[..., 0], acts_a[..., 0])
        assert torch.equal(dmb.data_on_device_via_torch("sampled_actions_1")[..., 0], acts_a[..., 1])
        assert torch.equal(db, done_a)
        obs_post = dma.data_on_device_via_torch("observations").view(E, N, -1)
        for p in pm:
            if null_push:
                assert ab[p] is None or bool((ab[p] == -3).all()), (t, p)
            else:
                assert torch.equal(ab[p], acts_a[:, ids[p]]), (t, p)
            assert torch.equal(rb[p], rew_a[:, ids[p]]), (t, p)
            assert torch.equal(ob[p], obs_post[:, ids[p]]), (t, p)      # post-reset obs
            assert torch.allclose(run[p], ref_run[p], atol=1e-5)
            assert abs(float(ep_sum[p]) - ref_ep[p]) < 1e-2 + 1e-5 * abs(ref_ep[p])
        assert torch.equal(steps.long(), ref_steps)
        assert int(ep_steps) == ref_ep_steps and int(n_done) == ref_n_done
        total_done += int(done_a.sum())
    assert total_done >= 2 * E       # episodes ended and were reset on both paths


def test_fused_step_without_reset_keeps_done_set():
    from warp_drive_b200.training.fused_tag_continuous import FusedTagContinuousStep

    E, T = 4, 2
    w, s, pm = _setup(E, T)
    dm = w.cuda_data_manager
    fused = FusedTagContinuousStep(w, pm, s)
    probs = {p: [torch.full((E, len(v), 21), 1 / 21.0, device="cuda") for _ in range(2)]
             for p, v in pm.items()}
    for t in range(ENV_KW["episode_length"]):
        fused.launch(probs, reset_done_envs=False)
    assert bool((dm.data_on_device_via_torch("_done_") == 1).all())
    assert bool((dm.data_on_device_via_torch("_timestep_") == ENV_KW["episode_length"]).all())
    w.reset_only_done_envs()
    assert int(dm.data_on_device_via_torch("_done_").sum()) == 0
    assert torch.equal(dm.data_on_device_via_torch("loc_x"),
                       dm.data_on_device_via_torch("loc_x_at_reset"))


@pytest.mark.parametrize("tc_variant", [2], ids=["v2"], indirect=True)
def test_fused_step_without_reset_keeps_done_set_second_generation(tc_variant):
    test_fused_step_without_reset_keeps_done_set()


def _engine(E, T, use_graph, fused, seed=3, env_kw=None, **engine_kw):
    from warp_drive_b200.training.models.fully_connected import FullyConnected
    from warp_drive_b200.training.rollout import RolloutEngine

    w, s, pm = _setup(E, T, seed=seed, **(env_kw or {}))
    torch.manual_seed(0)
    cfg = {"type": "fully_connected", "fc_dims": [32, 32], "model_ckpt_filepath": ""}
    models = {p: FullyConnected(w, cfg, p, pm).cuda().eval() for p in pm}
    w.reset_all_envs()
    eng = RolloutEngine(w, models, pm, s, T, use_cuda_graph=use_graph, use_fused_step=fused,
                        **engine_kw)
    return w, eng, pm


@pytest.mark.parametrize("fused", [True, False])
def test_engine_cuda_graph_matches_eager(fused):
    """Same seeds -> the CUDA-graph replayed rollout fills the training batch exactly like
    the eager loop (the warm-up step of the capture is replicated on the eager side)."""
    E, T = 6, 8
    wa, ea, pm = _engine(E, T, True, fused)
    wb, eb, _ = _engine(E, T, False, fused)
    ea.rollout()
    ea.rollout()
    eb.step(-1)             # the graph path ran one eager warm-up step before capturing
    if fused:
        # ... which must leave the engine's current observations in step with the env state
        # (a recording step(0) as warm-up left cur_obs one state behind: ADVICE r1)
        obs = wb.cuda_data_manager.data_on_device_via_torch("observations")
        for p_, ids in pm.items():
            assert torch.equal(eb.cur_obs[p_], obs[:, sorted(ids)]), p_
    eb.rollout()
    eb.rollout()
    torch.cuda.synchronize()
    for p in pm:
        for name in (f"processed_observations_batch_{p}", f"sampled_actions_batch_{p}",
                     f"rewards_batch_{p}"):
            ta = wa.cuda_data_manager.data_on_device_via_torch(name)
            tb = wb.cuda_data_manager.data_on_device_via_torch(name)
            assert torch.equal(ta, tb), name
    assert torch.equal(wa.cuda_data_manager.data_on_device_via_torch("done_flags_batch"),
                       wb.cuda_data_manager.data_on_device_via_torch("done_flags_batch"))
    assert int(ea.num_completed_episodes) == int(eb.num_completed_episodes)


@pytest.mark.parametrize("use_graph", [True, False])
def test_pair_forward_and_programmatic_launches_change_nothing(use_graph):
    """The optional launch mode (both policies' forwards in ONE launch, forward and env step
    chained by programmatic dependent launches that overlap each other's head and tail) must
    fill the batch exactly like the default plain serialised launches with one forward per
    policy: enough envs that every SM is busy, several rollouts with episode resets in between."""
    from warp_drive_b200 import lib as wlib

    L = wlib.load()
    E, T = 3000, 6
    assert L.wdb_set_option(b"pdl", 1) == 0
    try:
        wa, ea, pm = _engine(E, T, use_graph, True, use_pair_forward=True)
        for _ in range(8):
            ea.rollout()
        torch.cuda.synchronize()
    finally:
        L.wdb_set_option(b"pdl", 0)
    wb, eb, _ = _engine(E, T, use_graph, True, use_pair_forward=False)
    for _ in range(8):
        eb.rollout()
    torch.cuda.synchronize()
    names = ["done_flags_batch"]
    for p in pm:
        names += [f"processed_observations_batch_{p}", f"sampled_actions_batch_{p}",
                  f"rewards_batch_{p}"]
    names += list(STATE)
    for name in names:
        ta = wa.cuda_data_manager.data_on_device_via_torch(name)
        tb = wb.cuda_data_manager.data_on_device_via_torch(name)
        assert torch.equal(ta, tb), name
    assert int(ea.num_completed_episodes) == int(eb.num_completed_episodes) > 0


def test_engine_fused_matches_unfused_batches():
    """Fused single-launch timestep vs the generic multi-launch path, same models, same
    RNG seed: identical training batches (both draw u from the same Philox streams:
    generic = one draw per head call, fused = one draw for both heads, so compare through
    the injected-uniform test above; here only structural equivalence of the first step,
    where both consume draw #0.x / #0.x+#1.x differently, is NOT expected) -- instead check
    the batch invariants of the fused engine against its own state arrays."""
    E, T = 8, 16
    w, e, pm = _engine(E, T, True, True)
    dm = w.cuda_data_manager
    for _ in range(4):
        e.rollout()
    torch.cuda.synchronize()
    obs = dm.data_on_device_via_torch("observations")
    N = w.n_agents
    for p, ids in pm.items():
        i = torch.as_tensor(ids, device="cuda")
        # the observation the next forward pass will read == observations[:, ids]
        assert torch.equal(e.cur_obs[p], obs.view(E, N, -1)[:, i])
        acts = dm.data_on_device_via_torch(f"sampled_actions_batch_{p}")
        assert int(acts.min()) >= 0 and int(acts.max()) <= 20
        assert torch.equal(acts[T - 1], dm.data_on_device_via_torch("sampled_actions")[:, i])
        assert torch.equal(dm.data_on_device_via_torch(f"rewards_batch_{p}")[T - 1],
                           dm.data_on_device_via_torch("rewards")[:, i])
    assert int(e.num_completed_episodes) >= E      # 64 steps > one 40-step episode
    assert float(e.episodic_step_sum) / float(e.num_completed_episodes) <= 40


def test_engine_takes_the_generic_path_where_the_fused_step_has_no_plan():
    """23 agents observing K = 11 neighbours, 16 envs: the packed kernel cannot stage the
    observation tile the fused step pushes from, and the library refuses the fused step for
    that shape.  The engine asks the library, so it builds the generic multi-launch timestep
    instead, and its rollouts fill the batch from the env arrays."""
    E, T = 16, 8
    w, e, pm = _engine(E, T, True, True, env_kw=dict(num_other_agents_observed=11))
    assert e.fused is None
    dm = w.cuda_data_manager
    for _ in range(3):
        e.rollout()
    torch.cuda.synchronize()
    for p, ids in pm.items():
        i = torch.as_tensor(ids, device="cuda")
        assert torch.equal(dm.data_on_device_via_torch(f"sampled_actions_batch_{p}")[T - 1],
                           dm.data_on_device_via_torch("sampled_actions")[:, i])
        assert torch.equal(dm.data_on_device_via_torch(f"rewards_batch_{p}")[T - 1],
                           dm.data_on_device_via_torch("rewards")[:, i])


def test_step_with_host_buffers_matches_pull():
    """EnvWrapper.step_with_host_buffers (pinned host actions in; observations / rewards /
    done out over several copy streams) returns exactly what step_all_envs followed by
    pull_data_from_device returns."""
    E = 64
    wa, _, _ = _setup(E, 2)
    wb, _, _ = _setup(E, 2)
    rs = np.random.RandomState(5)
    dma, dmb = wa.cuda_data_manager, wb.cuda_data_manager
    names = ("observations", "rewards", "_done_")
    host_out = {k: torch.empty(dma.data_on_device_via_torch(k).shape,
                               dtype=dma.data_on_device_via_torch(k).dtype).pin_memory()
                for k in names}
    for _ in range(4):
        acts = rs.randint(0, 21, tuple(dma.get_shape("sampled_actions"))).astype(np.int32)
        wa.step_with_host_buffers(torch.from_numpy(acts).pin_memory(), host_out, n_copy_streams=3,
                                  min_split_bytes=1024,    # force the split-copy path
                                  pipeline_env_groups=bool(_ % 2))   # and the grouped pipeline
        dmb.data_on_device_via_torch("sampled_actions").copy_(torch.from_numpy(acts))
        wb.step_all_envs()
        for k in names:
            assert np.array_equal(host_out[k].numpy(), dmb.pull_data_from_device(k)), k


def test_engine_obs_tiles_matches_fp32_forward():
    """use_obs_tiles=True: the fused env step also emits the bf16 MMA-ready copy of the next
    observations (incl. the rows of envs that reset) and the forward reads that copy through
    the TMA.  The A operand is the same bf16 data either way, so whole rollouts -- several
    episodes, with resets -- fill identical training batches."""
    E, T = 40, 16                                   # 40 x 20 runners = 800 rows: partial last tile
    wa, ea, pm = _engine(E, T, True, True, use_obs_tiles=True)
    wb, eb, _ = _engine(E, T, True, True, use_obs_tiles=False)
    assert ea.obs_tiles and not eb.obs_tiles
    for _ in range(6):                              # 96 steps > 2 episodes of 40 steps
        ea.rollout()
        eb.rollout()
    torch.cuda.synchronize()
    for p in pm:
        for name in (f"processed_observations_batch_{p}", f"sampled_actions_batch_{p}",
                     f"rewards_batch_{p}"):
            ta = wa.cuda_data_manager.data_on_device_via_torch(name)
            tb = wb.cuda_data_manager.data_on_device_via_torch(name)
            assert torch.equal(ta, tb), name
    assert int(ea.num_completed_episodes) == int(eb.num_completed_episodes) > 0
    # the tiles the env step wrote (store_obs_chunk, incl. the rows of envs that reset) are
    # byte for byte what pack_obs makes of the same observations, K padding and the zero rows
    # of the last tile included: that padding must be finite, since 0 * NaN in the MMA would
    # poison every row
    for p in pm:
        fwd = ea.fused_forward[p]
        rows = ea.cur_obs[p].numel() // fwd.F
        ref = torch.full((fwd.tiles_bytes(rows),), 0xFF, dtype=torch.uint8, device="cuda")
        fwd.pack_obs(ea.cur_obs[p], ref)
        torch.cuda.synchronize()
        assert torch.equal(ea.obs_tiles[p], ref), p



def test_config4_agent_count_through_wrapper_and_engine():
    """BASELINE config 4 territory (1024 agents per env) with blocks_per_env = 1 and the
    first-generation single-CTA kernel forced (wdb_set_option tc_wide_single = 0): EnvWrapper
    allocates the reference's global neighbour scratch when asked to, the env steps through
    the managers, and the RolloutEngine runs the generic multi-launch timestep."""
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.tag_continuous import TagContinuous
    from warp_drive_b200.managers.function_manager import CUDASampler
    from warp_drive_b200.training.models.fully_connected import FullyConnected
    from warp_drive_b200.training.rollout import RolloutEngine
    from warp_drive_b200.training.utils.data_loader import create_and_push_data_placeholders

    from warp_drive_b200 import lib as wlib

    kw = dict(ENV_KW, num_taggers=24, num_runners=1000, grid_length=64.0,
              num_other_agents_observed=10, tagging_distance=0.3)
    env = TagContinuous(**kw)
    env.allocate_reference_scratch = True          # the [E, N, N-1] arrays of the reference
    E, T = 2, 4
    wlib.check(wlib.load().wdb_set_option(b"tc_wide_single", 0))
    w = EnvWrapper(env, num_envs=E, env_backend="b200")
    w.reset_all_envs()
    pm = {"runner": sorted(env.runners), "tagger": sorted(env.taggers)}
    s = CUDASampler(w.cuda_function_manager)
    create_and_push_data_placeholders(env_wrapper=w, action_sampler=s,
                                      policy_tag_to_agent_id_map=pm,
                                      training_batch_size_per_env=T)
    s.init_random(3)
    torch.manual_seed(0)
    cfg = {"type": "fully_connected", "fc_dims": [32, 32], "model_ckpt_filepath": ""}
    models = {p: FullyConnected(w, cfg, p, pm).cuda().eval() for p in pm}
    eng = RolloutEngine(w, models, pm, s, T, use_cuda_graph=False)
    assert eng.fused is None
    try:
        for _ in range(3):
            eng.rollout()
        torch.cuda.synchronize()
    finally:
        wlib.load().wdb_set_option(b"tc_wide_single", 1)
    dm = w.cuda_data_manager
    x, y = dm.pull_data_from_device("loc_x"), dm.pull_data_from_device("loc_y")
    assert ((x >= 0) & (x <= 64.0) & (y >= 0) & (y <= 64.0)).all()
    assert (dm.pull_data_from_device("_timestep_") == 12).all()
    nn = dm.pull_data_from_device("nearest_neighbor_ids")
    alive = dm.pull_data_from_device("still_in_the_game")
    assert nn.min() >= 0 and nn.max() < 1024
    obs = dm.pull_data_from_device("observations")
    assert np.isfinite(obs).all() and (obs[alive == 0] == 0).all()


def test_generic_path_native_moves_equal_torch_indexing():
    """wdb_gather_policy_rows (both directions) and wdb_rollout_bookkeep against the plain torch
    ops they replace on the generic multi-launch path: 2 policies with interleaved agent ids,
    2 action heads, several steps with resets so that done envs fold their running sums."""
    E, T = 37, 5
    wa, ea, pm = _engine(E, T, False, False)
    wb, eb, _ = _engine(E, T, False, False)
    assert ea.fused is None and ea.sa is None
    dma, dmb = wa.cuda_data_manager, wb.cuda_data_manager
    # gather / scatter
    obs = dma.data_on_device_via_torch("observations").view(E, wa.n_agents, -1)
    rows = {p: torch.zeros((E, len(ids), obs.shape[-1]), device="cuda") for p, ids in pm.items()}
    ea._move_rows(obs, rows)
    for p, ids in pm.items():
        assert torch.equal(rows[p], obs[:, ids]), p
    back = torch.full_like(obs, -7.0)
    ea._move_rows(back, rows, scatter=True)
    assert torch.equal(back, obs)
    # bookkeeping: identical env trajectories (same seeds), native vs torch bookkeeping
    n_done = 0
    for it in range(12):                      # 60 steps > one 40-step episode
        for t in range(T):
            for e, book in ((ea, ea.bookkeep), (eb, eb.bookkeep_torch)):
                with torch.no_grad():
                    probs = e.evaluate_policies(t)
                    e.sample_actions(probs, t)
                    e.env_wrapper.step_all_envs()
                    book(t)
                    e.env_wrapper.reset_only_done_envs()
            n_done += int((dma.data_on_device_via_torch("done_flags_batch")[t] > 0).sum())
        names = ["done_flags_batch"]
        for p in pm:
            names += [f"processed_observations_batch_{p}", f"sampled_actions_batch_{p}",
                      f"rewards_batch_{p}"]
        for name in names:
            assert torch.equal(dma.data_on_device_via_torch(name),
                               dmb.data_on_device_via_torch(name)), (it, name)
        assert torch.equal(ea.step_running_sum, eb.step_running_sum)
        for p in pm:
            assert torch.equal(ea.reward_running_sum[p], eb.reward_running_sum[p]), p
    assert n_done >= E
    assert int(ea.num_completed_episodes) == int(eb.num_completed_episodes) == n_done
    assert int(ea.episodic_step_sum) == int(eb.episodic_step_sum)
    for p in pm:
        a, b = float(ea.episodic_reward_sum[p]), float(eb.episodic_reward_sum[p])
        assert abs(a - b) <= 1e-4 * max(1.0, abs(b)), (p, a, b)


def test_bookkeep_treats_any_nonzero_done_flag_as_done():
    """MountainCar writes done == 2 at the goal: the batch keeps the raw flag (neg / pos env
    sampling tests for == 2) while the episodic sums count the env ONCE and the running sums
    are cleared, not sign-flipped (ADVICE r1)."""
    E, T = 6, 2
    w, e, pm = _engine(E, T, False, False)
    dm = w.cuda_data_manager
    done = dm.data_on_device_via_torch("_done_")
    done.copy_(torch.tensor([0, 1, 2, 0, 2, 0], dtype=done.dtype, device="cuda"))
    rewards = dm.data_on_device_via_torch("rewards")
    rewards.copy_(torch.arange(rewards.numel(), device="cuda").view_as(rewards).float() * 0.25)
    for p in pm:
        e.reward_running_sum[p].fill_(1.0)
    e.step_running_sum.fill_(4)
    before = {p: e.reward_running_sum[p].clone() for p in pm}
    e.bookkeep(1)
    torch.cuda.synchronize()
    assert dm.data_on_device_via_torch("done_flags_batch")[1].tolist() == [0, 1, 2, 0, 2, 0]
    is_done = torch.tensor([False, True, True, False, True, False], device="cuda")
    assert e.step_running_sum.tolist() == [5, 0, 0, 5, 0, 5]
    assert int(e.num_completed_episodes) == 3 and int(e.episodic_step_sum) == 15
    for p, ids in pm.items():
        r_p = rewards[:, ids]
        assert torch.equal(dm.data_on_device_via_torch(f"rewards_batch_{p}")[1], r_p)
        run = before[p] + r_p
        assert torch.equal(e.reward_running_sum[p], torch.where(is_done[:, None], 0.0 * run, run))
        want = float(run[is_done].sum())
        assert abs(float(e.episodic_reward_sum[p]) - want) <= 1e-4 * max(1.0, abs(want))
