"""The config-2 rollout as two env groups (each half of the envs runs its own chain of sampling
forwards and env steps on its own streams) computes exactly what it computes as one group:
two engines from the same seeds, one forced to a single group, run the same rollouts (CUDA
graph replays) and must leave every per-env array bit-identical."""
import pytest
import torch

from test_gpu_forward_sampling import _engine

pytestmark = pytest.mark.gpu

PER_ENV = ("loc_x", "loc_y", "speed", "direction", "acceleration", "edge_hit_reward_penalty",
           "still_in_the_game", "num_runners", "nearest_neighbor_ids", "_done_", "_timestep_",
           "rewards", "sampled_actions", "sampled_actions_0", "sampled_actions_1",
           "done_flags_batch")


@pytest.mark.parametrize("E", [7, 667, 2000, 2001])
def test_two_env_groups_compute_what_one_group_computes(E):
    T = 8
    wa, ea, pm, sa = _engine(E, T)
    wb, eb, _, sb = _engine(E, T)
    ea.use_cuda_graph = eb.use_cuda_graph = True
    eb._set_env_groups(1)
    assert len(eb._groups) == 1
    assert len(ea._groups) == (2 if E >= 4 * (320 // ea.N) else 1)
    names = PER_ENV + tuple(f"{k}_batch_{p}" for p in pm
                            for k in ("sampled_actions", "rewards", "processed_observations"))
    for _ in range(2):
        ea.rollout()
        eb.rollout()
        torch.cuda.synchronize()
        for name in names:
            ta = wa.cuda_data_manager.data_on_device_via_torch(name)
            tb = wb.cuda_data_manager.data_on_device_via_torch(name)
            assert torch.equal(ta, tb), name
        for p in pm:
            assert torch.equal(ea.cur_obs[p], eb.cur_obs[p]), p
            assert torch.equal(ea.reward_running_sum[p], eb.reward_running_sum[p]), p
            # (float sums accumulated by atomicAdd: their order differs from run to run)
            assert torch.allclose(ea.episodic_reward_sum[p], eb.episodic_reward_sum[p],
                                  rtol=1e-5)
        assert torch.equal(ea.step_running_sum, eb.step_running_sum)
        assert torch.equal(ea.episodic_step_sum, eb.episodic_step_sum)
        assert torch.equal(ea.num_completed_episodes, eb.num_completed_episodes)
        assert torch.equal(sa.rng_state, sb.rng_state)
