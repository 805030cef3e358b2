"""HeteroEnv: the host side of tests/custom_env/hetero_env_step.cu, written like
masked_counter_env.py.  Agent 0 is a planner (MultiDiscrete([3, 5]) actions, Dict observation
{"state", "action_mask"} whose mask depends on the planner's level); agents 1..N-1 are workers
(Discrete(4) actions, Box observation of shape (2, 3)).  with_planner=False leaves only workers,
a homogeneous env.

With the planner, the env steps through separate per-policy placeholders of the policies
"planner" (agent 0) and "workers" (agents 1..N-1): observations_planner_{state,action_mask},
sampled_actions_planner, rewards_planner, observations_workers, sampled_actions_workers,
rewards_workers.  Without it, through the shared observations / sampled_actions / rewards.
`worker_obs_layout` says how the env writes worker observations: "first" [E, Nw, 2, 3] or
"last" [E, 2, 3, Nw]; it must match the trainer's obs_dim_corresponding_to_num_agents.

`HeteroTwin` is the same env for E replicas in NumPy, for replaying a device rollout."""
import numpy as np

from warp_drive_b200.utils import spaces
from warp_drive_b200.utils.constants import Constants
from warp_drive_b200.utils.data_feed import DataFeed
from warp_drive_b200.utils.gpu_environment_context import CUDAEnvironmentContext

PLANNER_HEADS = (3, 5)
MAX_LEVEL = 4


def planner_mask(level):
    """int32 [..., 8] valid planner actions of `level` (int array [...])."""
    level = np.asarray(level)[..., None]
    move = np.concatenate([level > 0, np.ones_like(level, bool), level < MAX_LEVEL], -1)
    say = np.arange(PLANNER_HEADS[1]) <= level
    return np.concatenate([move, say], -1).astype(np.int32)


def worker_obs(phase, level, announced, n_workers):
    """float32 [..., Nw, 2, 3] worker observations (phase [..., Nw]; level, announced [...])."""
    phase = np.asarray(phase)
    lv = np.broadcast_to(np.asarray(level)[..., None], phase.shape)
    an = np.broadcast_to(np.asarray(announced)[..., None], phase.shape)
    wid = np.broadcast_to(np.arange(n_workers) % 3, phase.shape)
    rows = [phase & 1, phase >> 1, np.ones_like(phase), lv, an, wid]
    return np.stack(rows, -1).astype(np.float32).reshape(phase.shape + (2, 3))


class HeteroEnv:
    name = "HeteroEnv"

    def __init__(self, num_agents=5, episode_length=10, with_planner=True,
                 worker_obs_layout="first", env_backend="cpu"):
        assert worker_obs_layout in ("first", "last")
        self.num_agents = num_agents
        self.episode_length = episode_length
        self.with_planner = bool(with_planner)
        self.worker_obs_layout = worker_obs_layout
        self.env_backend = env_backend
        self.n_workers = num_agents - int(self.with_planner)
        assert self.n_workers >= 1
        self.workers = list(range(int(self.with_planner), num_agents))
        self.action_space = {a: spaces.Discrete(4) for a in self.workers}
        if self.with_planner:
            self.action_space[0] = spaces.MultiDiscrete(list(PLANNER_HEADS))
        self.observation_space = None
        self.timestep = 0

    def policy_tag_to_agent_id_map(self):
        if self.with_planner:
            return {"planner": [0], "workers": self.workers}
        return {"workers": self.workers}

    def initial_phase(self):
        return (np.arange(self.n_workers) % 4).astype(np.int32)

    def reset(self):
        self.timestep = 0
        obs = {}
        wo = worker_obs(self.initial_phase(), 0, 0, self.n_workers)
        for w, a in enumerate(self.workers):
            obs[a] = wo[w]
        if self.with_planner:
            obs[0] = {"state": np.array([0, 0, self.episode_length], np.float32),
                      Constants.ACTION_MASK: planner_mask(0)}
        return obs


class CUDAHeteroEnv(HeteroEnv, CUDAEnvironmentContext):
    def __init__(self, *args, **kwargs):
        HeteroEnv.__init__(self, *args, **kwargs)
        CUDAEnvironmentContext.__init__(self)
        self._args = None

    def get_data_dictionary(self):
        d = DataFeed()
        d.add_data(name="level", data=0, save_copy_and_apply_at_reset=True)       # -> [E]
        d.add_data(name="announced", data=0, save_copy_and_apply_at_reset=True)   # -> [E]
        d.add_data(name="phase", data=self.initial_phase(), save_copy_and_apply_at_reset=True)
        d.add_data(name="invalid_actions", data=np.zeros(1, np.int32))
        return d

    def step(self, actions=None):
        self.timestep += 1
        if self._args is None:
            dm = self.cuda_data_manager
            obs, act, rew = Constants.OBSERVATIONS, Constants.ACTIONS, Constants.REWARDS
            if self.with_planner:
                names = ["level", "announced", "phase", f"{act}_planner", f"{act}_workers",
                         "_done_", f"{rew}_planner", f"{rew}_workers", f"{obs}_planner_state",
                         f"{obs}_planner_{Constants.ACTION_MASK}", f"{obs}_workers"]
            else:
                names = ["level", "announced", "phase", None, act, "_done_", None, rew, None,
                         None, obs]
            self._args = [dm.device_data(n) if n else None for n in names] + [
                dm.device_data("invalid_actions"), dm.device_data("_timestep_"),
                np.int32(self.episode_length), np.int32(self.with_planner),
                np.int32(self.worker_obs_layout == "last")]
        self.cuda_step(*self._args, block=self.cuda_function_manager.block,
                       grid=self.cuda_function_manager.grid)


class HeteroTwin:
    """E replicas of the env in NumPy, reset when done like the device's done-masked reset.
    Observations come in the agent-first layout ([E, Nw, 2, 3] workers)."""

    def __init__(self, n_envs, num_agents, episode_length, with_planner=True):
        self.E, self.L = n_envs, episode_length
        self.with_planner = bool(with_planner)
        self.nw = num_agents - int(self.with_planner)
        self.invalid = 0
        self.reset()

    def reset(self, envs=None):
        envs = slice(None) if envs is None else envs
        if not hasattr(self, "t"):
            self.t = np.zeros(self.E, np.int64)
            self.level = np.zeros(self.E, np.int64)
            self.announced = np.zeros(self.E, np.int64)
            self.phase = np.zeros((self.E, self.nw), np.int64)
        self.t[envs] = 0
        self.level[envs] = 0
        self.announced[envs] = 0
        self.phase[envs] = np.arange(self.nw) % 4

    def observe(self):
        out = {"workers": worker_obs(self.phase, self.level, self.announced, self.nw)}
        if self.with_planner:
            out["planner_state"] = np.stack(
                [self.level, self.announced, self.L - self.t], -1).astype(np.float32)
            out["planner_mask"] = planner_mask(self.level)
        return out

    def step(self, worker_actions, planner_actions=None):
        """worker_actions int [E, Nw], planner_actions int [E, 2] -> (rewards {"workers"
        [E, Nw], "planner" [E]}, done int [E]); done envs are reset afterwards."""
        rewards = {}
        if self.with_planner:
            move, say = planner_actions[:, 0], planner_actions[:, 1]
            nxt = self.level + move - 1
            bad_move = (nxt < 0) | (nxt > MAX_LEVEL)
            bad_say = say > self.level
            self.invalid += int(bad_move.sum() + bad_say.sum())
            self.level = np.where(bad_move, self.level, nxt)
            self.announced = np.where(bad_say, 0, say)
            rewards["planner"] = self.announced.astype(np.float32)
        rewards["workers"] = (worker_actions == self.phase).astype(np.float32)
        self.phase = (self.phase + 1 + self.announced[:, None]) % 4
        self.t += 1
        done = (self.t == self.L).astype(np.int32)
        if done.any():
            self.reset(np.nonzero(done)[0])
        return rewards, done
