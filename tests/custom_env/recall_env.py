"""RecallEnv: the host side of tests/custom_env/recall_env_step.cu, written like
grid_reach_env.py.  Every agent sees a cue c in {0, 1} once, after the first step ([2c - 1, 1]),
and blank observations [0, 0] otherwise; the last step of the episode pays 1 when the agent's
action equals c.  A memoryless policy earns at most 1/2 per episode on average, a policy that
remembers the cue 1."""
import numpy as np

from warp_drive_b200.utils import spaces
from warp_drive_b200.utils.data_feed import DataFeed
from warp_drive_b200.utils.gpu_environment_context import CUDAEnvironmentContext


class RecallEnv:
    name = "RecallEnv"

    def __init__(self, num_agents=2, episode_length=4, env_backend="cpu"):
        assert episode_length >= 3
        self.num_agents = num_agents
        self.episode_length = episode_length
        self.env_backend = env_backend
        self.action_space = {a: spaces.Discrete(2) for a in range(num_agents)}
        self.observation_space = None
        self.timestep = 0

    def reset(self):
        self.timestep = 0
        return {a: np.zeros(2, np.float32) for a in range(self.num_agents)}


class CUDARecallEnv(RecallEnv, CUDAEnvironmentContext):
    def __init__(self, *args, **kwargs):
        RecallEnv.__init__(self, *args, **kwargs)
        CUDAEnvironmentContext.__init__(self)
        self._args = None

    def get_data_dictionary(self):
        # (neither is restored at reset, so both are laid out per env here)
        E = int(self.cuda_data_manager.meta_info("n_envs"))
        d = DataFeed()
        d.add_data(name="cue", data=np.zeros((E, self.num_agents), np.int32))
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
    """A Trainer of one shared policy on RecallEnv.  model: a model config dict (type, fc_dims,
    ...); PPO with ppo_steps = (num_epochs, num_mini_batches) and GAE, or A2C."""
    import os

    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.training.trainer import Trainer, load_run_config
    from warp_drive_b200.utils.env_registrar import EnvironmentRegistrar

    reg = EnvironmentRegistrar()
    reg.add_cuda_env_src_path("RecallEnv", os.path.join(os.path.dirname(
        os.path.abspath(__file__)), "recall_env_step.cu"))
    env = CUDARecallEnv(num_agents=num_agents, episode_length=episode_length,
                        env_backend="pycuda")
    w = EnvWrapper(env, num_envs=num_envs, env_backend="pycuda", env_registrar=reg)
    cfg = load_run_config("tag_gridworld")
    cfg.pop("env")
    cfg["name"] = "recall"
    cfg["trainer"].update(num_envs=num_envs, train_batch_size=num_envs * steps_per_env,
                          num_episodes=iterations * num_envs * steps_per_env // episode_length,
                          seed=seed)
    pol = cfg["policy"]["shared"]
    pol.update(algorithm=algorithm, gamma=0.99, lr=lr, entropy_coeff=0.01, vf_loss_coeff=0.5,
               max_grad_norm=0.5, model=dict(model, model_ckpt_filepath=""))
    if algorithm == "PPO":
        pol.update(clip_param=0.2, num_epochs=ppo_steps[0], num_mini_batches=ppo_steps[1],
                   gae_lambda=0.95)
    cfg["saving"].update(basedir=basedir, name="recall", metrics_log_freq=10 ** 9,
                         model_params_save_freq=10 ** 9)
    return Trainer(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={
        "shared": list(range(num_agents))}, results_dir=results_dir, verbose=False,
        use_cuda_graph=use_cuda_graph)
