"""ContinuousRecallEnv: the host side of tests/custom_env/continuous_recall_env_step.cu, written
like recall_env.py.  Every agent sees a cue c, drawn uniformly on the circle of radius
RADIUS = 0.8, once, after the first step ([c_x, c_y, 1]), and blank observations [0, 0, 0]
otherwise; with Box(-1, 1, (2,)) actions, the last step of the episode pays -|clip(a, -1, 1) - c|
and every other step 0.

A memoryless policy sees the same blank observation at the last step whatever c was, so its
expected last-step reward is at most -RADIUS = -0.8, reached at a = 0: for points on a circle,
the circle's centre minimises the expected distance.  A policy that remembers the cue can reach
0."""
import numpy as np

from warp_drive_b200.utils import spaces
from warp_drive_b200.utils.data_feed import DataFeed
from warp_drive_b200.utils.gpu_environment_context import CUDAEnvironmentContext

RADIUS = 0.8
MEMORYLESS_BOUND = -RADIUS


class ContinuousRecallEnv:
    name = "ContinuousRecallEnv"

    def __init__(self, num_agents=2, episode_length=4, env_backend="cpu"):
        assert episode_length >= 3
        self.num_agents = num_agents
        self.episode_length = episode_length
        self.env_backend = env_backend
        self.action_space = {a: spaces.Box(-1.0, 1.0, shape=(2,)) for a in range(num_agents)}
        self.observation_space = None
        self.timestep = 0

    def reset(self):
        self.timestep = 0
        return {a: np.zeros(3, np.float32) for a in range(self.num_agents)}


class CUDAContinuousRecallEnv(ContinuousRecallEnv, CUDAEnvironmentContext):
    def __init__(self, *args, **kwargs):
        ContinuousRecallEnv.__init__(self, *args, **kwargs)
        CUDAEnvironmentContext.__init__(self)
        self._args = None

    def get_data_dictionary(self):
        # (neither is restored at reset, so both are laid out per env here)
        E = int(self.cuda_data_manager.meta_info("n_envs"))
        d = DataFeed()
        d.add_data(name="cue", data=np.zeros((E, self.num_agents, 2), np.float32))
        d.add_data(name="draws", data=np.zeros(E, np.int32))
        return d

    def step(self, actions=None):
        self.timestep += 1
        if self._args is None:
            dm = self.cuda_data_manager
            self._args = [dm.device_data(n) for n in (
                "cue", "draws", "sampled_actions", "rewards", "observations", "_done_",
                "_timestep_")] + [np.int32(self.episode_length)]
        self.cuda_step(*self._args, block=self.cuda_function_manager.block,
                       grid=self.cuda_function_manager.grid)


def make_trainer(model, results_dir, basedir, num_envs=256, steps_per_env=8, num_agents=2,
                 episode_length=4, seed=7, algorithm="PPO", ppo_steps=(4, 4), iterations=1000,
                 lr=0.003, use_cuda_graph=True):
    """A Trainer of one shared policy on ContinuousRecallEnv.  model: a model config dict (type,
    fc_dims, ...); PPO with ppo_steps = (num_epochs, num_mini_batches) and GAE, or A2C."""
    import os

    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.training.trainer import Trainer, load_run_config
    from warp_drive_b200.utils.env_registrar import EnvironmentRegistrar

    reg = EnvironmentRegistrar()
    reg.add_cuda_env_src_path("ContinuousRecallEnv", os.path.join(os.path.dirname(
        os.path.abspath(__file__)), "continuous_recall_env_step.cu"))
    env = CUDAContinuousRecallEnv(num_agents=num_agents, episode_length=episode_length,
                                  env_backend="pycuda")
    w = EnvWrapper(env, num_envs=num_envs, env_backend="pycuda", env_registrar=reg)
    cfg = load_run_config("tag_gridworld")
    cfg.pop("env")
    cfg["name"] = "continuous_recall"
    cfg["trainer"].update(num_envs=num_envs, train_batch_size=num_envs * steps_per_env,
                          num_episodes=iterations * num_envs * steps_per_env // episode_length,
                          seed=seed)
    pol = cfg["policy"]["shared"]
    pol.update(algorithm=algorithm, gamma=0.99, lr=lr, entropy_coeff=0.0, vf_loss_coeff=0.5,
               max_grad_norm=0.5, model=dict(model, model_ckpt_filepath=""))
    if algorithm == "PPO":
        pol.update(clip_param=0.2, num_epochs=ppo_steps[0], num_mini_batches=ppo_steps[1],
                   gae_lambda=0.95)
    cfg["saving"].update(basedir=basedir, name="continuous_recall", metrics_log_freq=10 ** 9,
                         model_params_save_freq=10 ** 9)
    return Trainer(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={
        "shared": list(range(num_agents))}, results_dir=results_dir, verbose=False,
        use_cuda_graph=use_cuda_graph)
