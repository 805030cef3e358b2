"""GridReachEnv: the host side of tests/custom_env/grid_reach_env_step.cu, written like
reach_env.py, with MultiDiscrete((5, 3)) actions: every agent moves on an integer grid toward
the goal (0, 0) by dx = a_0 - 2 in {-2 .. 2} and dy = a_1 - 1 in {-1, 0, 1} per step.  The
reward is -1 per step until the agent stands on the goal, 0 from then on (it stays there), so an
episode's return is minus the steps the agent took to reach it.  Agent a starts at START[a]; the
fewest steps from there are max(ceil(|x| / 2), |y|) (`optimal_steps`).  Two policies, "a"
(agents 0..N/2-1) and "b" (the rest), step through the shared placeholders."""
import numpy as np

from warp_drive_b200.utils import spaces
from warp_drive_b200.utils.data_feed import DataFeed
from warp_drive_b200.utils.gpu_environment_context import CUDAEnvironmentContext

# the start of agent a (the kernel holds the same table); the goal is (0, 0)
START = np.array([[-4, 2], [3, -1], [-2, -2], [2, 1], [4, 0], [-3, 1], [0, 2], [-1, 0]],
                 np.int32)
SCALE = np.array([6.0, 3.0], np.float32)       # observation = (goal - position) / SCALE


def optimal_steps(num_agents):
    """int [N]: the fewest steps from each agent's start to the goal."""
    s = np.abs(START[:num_agents])
    return np.maximum((s[:, 0] + 1) // 2, s[:, 1])


class GridReachEnv:
    name = "GridReachEnv"

    def __init__(self, num_agents=4, episode_length=16, env_backend="cpu"):
        assert 2 <= num_agents <= len(START) and num_agents % 2 == 0
        self.num_agents = num_agents
        self.episode_length = episode_length
        self.env_backend = env_backend
        self.action_space = {a: spaces.MultiDiscrete([5, 3]) for a in range(num_agents)}
        self.observation_space = None
        self.timestep = 0

    def policy_tag_to_agent_id_map(self):
        n = self.num_agents // 2
        return {"a": list(range(n)), "b": list(range(n, self.num_agents))}

    def reset(self):
        self.timestep = 0
        return {a: (-START[a] / SCALE).astype(np.float32) for a in range(self.num_agents)}


class CUDAGridReachEnv(GridReachEnv, CUDAEnvironmentContext):
    def __init__(self, *args, **kwargs):
        GridReachEnv.__init__(self, *args, **kwargs)
        CUDAEnvironmentContext.__init__(self)
        self._args = None

    def get_data_dictionary(self):
        d = DataFeed()
        d.add_data(name="grid_pos", data=START[:self.num_agents].copy(),
                   save_copy_and_apply_at_reset=True)                      # -> [E, N, 2]
        return d

    def step(self, actions=None):
        self.timestep += 1
        if self._args is None:
            dm = self.cuda_data_manager
            self._args = [dm.device_data(n) for n in (
                "grid_pos", "sampled_actions", "rewards", "observations", "_done_",
                "_timestep_")] + [np.int32(self.episode_length)]
        self.cuda_step(*self._args, block=self.cuda_function_manager.block,
                       grid=self.cuda_function_manager.grid)
