"""Sampling in the policy forward (wdb_mlp_policy_forward_sampled) and the fused TagContinuous
step's actions-in mode.  At the config-2 policy shape (F = 71, [256, 256], two 21-way heads)
the RolloutEngine lets the forwards draw both heads' actions straight into the batch slot, and
the env step reads them instead of sampling from the probabilities.  That must change nothing:
the same Philox draws, the same float32 CDF and the same search, so the same actions and
everything that follows from them, bit for bit."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# config 2's observation and policy shape, with fewer agents and envs (row counts that are not
# multiples of 64 or 128: 37 envs x 3 taggers = 111 rows, 37 x 40 runners = 1480 rows) and
# short episodes, so that a run crosses several done-masked resets
ENV_KW = dict(num_taggers=3, num_runners=40, grid_length=10.0, episode_length=25,
              max_acceleration=0.1, min_acceleration=-0.1, max_turn=2.356, min_turn=-2.356,
              num_acceleration_levels=20, num_turn_levels=20, seed=274880,
              use_full_observation=False, num_other_agents_observed=10,
              tag_reward_for_tagger=10.0, tag_penalty_for_runner=-10.0,
              edge_hit_penalty=-0.5, tagging_distance=0.08, step_reward_for_runner=0.01)
MODEL = {"type": "fully_connected", "fc_dims": [256, 256], "model_ckpt_filepath": ""}


def _engine(E, T, seed=5, **engine_kw):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.tag_continuous import TagContinuous
    from warp_drive_b200.managers.function_manager import CUDASampler
    from warp_drive_b200.training.models.fully_connected import FullyConnected
    from warp_drive_b200.training.rollout import RolloutEngine
    from warp_drive_b200.training.utils.data_loader import create_and_push_data_placeholders

    env = TagContinuous(**ENV_KW)
    w = EnvWrapper(env, num_envs=E, env_backend="b200")
    w.reset_all_envs()
    pm = {"runner": sorted(env.runners), "tagger": sorted(env.taggers)}
    s = CUDASampler(w.cuda_function_manager)
    create_and_push_data_placeholders(env_wrapper=w, action_sampler=s, policy_tag_to_agent_id_map=pm,
                                      training_batch_size_per_env=T)
    s.init_random(seed)
    torch.manual_seed(0)
    models = {p: FullyConnected(w, MODEL, p, pm).cuda().eval() for p in pm}
    w.reset_all_envs()
    eng = RolloutEngine(w, models, pm, s, T, use_cuda_graph=False, **engine_kw)
    eng.resync_observations()
    return w, eng, pm, s


STATE = ("loc_x", "loc_y", "speed", "direction", "acceleration", "edge_hit_reward_penalty",
         "still_in_the_game", "num_runners", "nearest_neighbor_ids", "_done_", "_timestep_",
         "rewards", "sampled_actions", "sampled_actions_0", "sampled_actions_1")


def _same(wa, wb, names):
    for name in names:
        ta = wa.cuda_data_manager.data_on_device_via_torch(name)
        tb = wb.cuda_data_manager.data_on_device_via_torch(name)
        assert torch.equal(ta, tb), name


@pytest.mark.parametrize("obs_tiles", [False, True])
@pytest.mark.parametrize("given_uniforms", [False, True])
def test_sampling_in_the_forward_changes_nothing(obs_tiles, given_uniforms):
    """Two engines built from the same seeds; one samples in the forward (the engine's choice
    at this shape), the other is switched back to sampling in the env step.  Every step of 68
    -- a t < 0 step, then 4 rollouts of 16 steps over several episodes -- must leave the same
    actions, rewards, observations, done flags and RNG offsets."""
    E, T = 37, 16
    wa, ea, pm, sa = _engine(E, T, use_obs_tiles=obs_tiles)
    wb, eb, _, sb = _engine(E, T, use_obs_tiles=obs_tiles)
    assert ea.sample_in_forward and bool(ea.obs_tiles) == obs_tiles
    eb.sample_in_forward = False
    assert torch.equal(sa.rng_state, sb.rng_state)
    gen = torch.Generator(device="cuda").manual_seed(9)
    batch = [f"{k}_batch_{p}" for p in pm
             for k in ("sampled_actions", "rewards", "processed_observations")]
    off0 = sa.rng_state[16:].view(torch.int64).clone()    # per-stream draw offsets
    n = 0
    for t in [-1] + list(range(T)) * 4:
        u = None
        if given_uniforms:
            u = torch.rand((E, wa.n_agents, 2), generator=gen, device="cuda")
        ea.step_fused(t, uniforms=u)
        eb.step_fused(t, uniforms=u)
        torch.cuda.synchronize()
        _same(wa, wb, STATE)
        _same(wa, wb, batch + ["done_flags_batch"])
        for p in pm:
            assert torch.equal(ea.cur_obs[p], eb.cur_obs[p]), p
        assert torch.equal(sa.rng_state, sb.rng_state), t
        n += 1
    assert n == 65
    assert int(ea.num_completed_episodes) == int(eb.num_completed_episodes) >= 2 * E
    assert torch.equal(ea.episodic_step_sum, eb.episodic_step_sum)
    for p in pm:
        # (a float sum accumulated by atomicAdd over agents: its order, and so its last bits,
        #  differ from run to run in either mode)
        assert torch.allclose(ea.episodic_reward_sum[p], eb.episodic_reward_sum[p], rtol=1e-5)
    # the Philox offsets moved once per step (the t < 0 step included), or not at all with
    # given uniforms
    moved = sa.rng_state[16:].view(torch.int64) - off0
    assert int(moved.min()) == int(moved.max()) == (0 if given_uniforms else 65)


def _cdf32(p):
    """Float32 prefix sums of the rows of p [rows, A], left to right."""
    c = np.empty_like(p)
    c[:, 0] = p[:, 0]
    for i in range(1, p.shape[1]):
        c[:, i] = p[:, i] + c[:, i - 1]
    return c


def _search_index(cdf, u):
    """The reference's binary search (core/random.cu:33-49), one row at a time."""
    out = np.empty(len(u), np.int64)
    r = cdf.shape[1] - 1
    for i in range(len(u)):
        left, right, res = 0, r, None
        while left <= right:
            mid = left + (right - left) // 2
            v = cdf[i, mid]
            if abs(np.float32(v - u[i])) < np.float32(1e-8):
                res = mid
                break
            if v < u[i]:
                left = mid + 1
            else:
                right = mid - 1
        out[i] = res if res is not None else min(left, r)
    return out


@pytest.mark.parametrize("tiles", [False, True])
@pytest.mark.parametrize("E", [1, 37, 64])
def test_forward_samples_what_the_reference_search_picks(E, tiles):
    """The sampled forward on its own, with given uniforms, at row counts that are and are not
    multiples of the 64-row warpgroup and the 128-row tile: the probabilities are the plain
    forward's, bit for bit, and the actions are what the reference's search picks on the float32
    CDF of those probabilities.  A third of the uniforms sit exactly on a CDF entry (the
    |cdf - u| < 1e-8 branch) and some are 1.0 (above the float32 total: the clamp)."""
    from warp_drive_b200.training.models.fused_forward import FusedPolicyForward

    _, eng, pm, _ = _engine(E, 2)
    N = eng.N
    gen = torch.Generator(device="cuda").manual_seed(3)
    for p, ids in pm.items():
        fwd = eng.fused_forward[p]
        assert isinstance(fwd, FusedPolicyForward) and fwd.samples
        Np = len(ids)
        obs = torch.randn((E, Np, fwd.F), generator=gen, device="cuda")
        ref = [torch.empty((E, Np, 21), device="cuda") for _ in range(2)]
        fwd(obs, ref[0], ref[1])
        probs = [torch.full_like(ref[0], float("nan")) for _ in range(2)]
        acts = torch.full((E, Np, 2), -1, dtype=torch.int32, device="cuda")
        u = torch.rand((E, N, 2), generator=gen, device="cuda")
        slot = torch.arange(Np, device="cuda")
        agent = torch.as_tensor(ids, device="cuda")
        k = torch.randint(0, 21, (E, Np), generator=gen, device="cuda")
        hit = (slot % 3 == 0).expand(E, Np)
        for h in range(2):
            exact = torch.from_numpy(_cdf32(ref[h].reshape(-1, 21).cpu().numpy())).cuda()
            uh = u[:, agent, h]
            uh = torch.where(hit, exact.view(E, Np, 21).gather(2, k[..., None])[..., 0], uh)
            uh[:, -1] = 1.0
            u[:, agent, h] = uh
        agent_of_slot = torch.as_tensor(ids, dtype=torch.int32, device="cuda")
        smp = fwd.sampling(acts, agent_of_slot, N, uniforms=u)
        if tiles:
            t = torch.zeros(fwd.tiles_bytes(E * Np), dtype=torch.uint8, device="cuda")
            fwd.pack_obs(obs, t)
            fwd.forward_tiles(t, E * Np, probs[0], probs[1], sampling=smp)
        else:
            fwd(obs, probs[0], probs[1], sampling=smp)
        torch.cuda.synchronize()
        for h in range(2):
            assert torch.equal(probs[h], ref[h]), (p, h)
            c = _cdf32(ref[h].reshape(-1, 21).cpu().numpy())
            want = _search_index(c, u[:, agent, h].reshape(-1).cpu().numpy())
            got = acts[..., h].reshape(-1).cpu().numpy()
            assert np.array_equal(got, want), (p, h, int((got != want).sum()))


def test_actions_in_mode_is_the_packed_kernels(wdb_lib):
    """The packed kernel takes the mode; the cluster kernel (blocks_per_env > 1) does not, and
    the engine then samples in the env step."""
    import ctypes

    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.fused_tag_continuous import FusedTagContinuousStep

    w, eng, pm, _ = _engine(4, 2)
    assert FusedTagContinuousStep.eligible(w, pm, actions_in=True) and eng.sample_in_forward
    env = eng.fused.env
    ro = wlib.TcRollout()
    ro.n_policies, ro.n_actions0, ro.n_actions1 = 2, 21, 21
    for k, p in enumerate(pm):
        ro.policy[k].n_agents = len(pm[p])
    ro.actions_in = 1
    assert wdb_lib.wdb_tag_continuous_rollout_supported(ctypes.byref(env), ctypes.byref(ro), 0) == 0
    env.blocks_per_env = 2
    assert wdb_lib.wdb_tag_continuous_rollout_supported(ctypes.byref(env), ctypes.byref(ro), 0) != 0
