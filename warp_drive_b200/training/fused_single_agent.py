"""The whole T-step rollout of a single-agent classic-control env in ONE launch
(`wdb_single_agent_rollout`, csrc/wdb_sa_rollout.cu): forward -> sample -> step ->
bookkeeping -> done-masked reset -> push to batch, one thread per env replica.

H100 re-design of TrainerBase._generate_rollout_batch (warp_drive/training/trainers/
trainer_base.py:383-428) for ClassicControl{CartPole,MountainCar,Acrobot}Env with a small
FullyConnected policy (BASELINE config 3), and of the DDPG rollout of
ClassicControl{ContinuousMountainCar,Pendulum}Env with a small FullyConnectedActor (tanh head
+ Ornstein-Uhlenbeck exploration noise), and of the A2C / PPO rollout of those two envs with a
small FullyConnectedGaussian policy (raw mean + state-independent log_std), and of the SAC
rollout of those two envs with a small FullyConnectedSACActor (squashed Gaussian head [mu,
log-std]): the reference issues ~50 launches and >= 5 host
synchronisations per timestep, this path one launch per T timesteps and no synchronisation.
"""
import ctypes

import torch

from warp_drive_b200 import lib as _lib
from warp_drive_b200.envs.single_agent.base import SINGLE_AGENT_ENVS
from warp_drive_b200.utils.constants import Constants

_OBSERVATIONS = Constants.OBSERVATIONS
_ACTIONS = Constants.ACTIONS
_REWARDS = Constants.REWARDS
_DONE_FLAGS = Constants.DONE_FLAGS
_PROCESSED_OBSERVATIONS = Constants.PROCESSED_OBSERVATIONS


def _p(t):
    return _lib.ptr(t)


def _unwrap(model):
    """The FullyConnected / FullyConnectedActor behind the rollout engine's ActorAsPolicy."""
    return getattr(model, "actor", model)


def _layers(model):
    """[(weight, bias)] of the hidden layers followed by the (single) action head.  A dueling head
    has no one output layer: its rollout runs the folded layers of a DuelingFold instead."""
    model = _unwrap(model)
    out = [(model.fc[str(i)][0].weight, model.fc[str(i)][0].bias) for i in range(len(model.fc))]
    if getattr(model, "dueling", False):
        raise TypeError("a dueling head runs as its folded layers (DuelingFold)")
    if getattr(model, "noisy", False):
        raise TypeError("a noisy head has no one weight: it acts through the per-step path")
    # the discrete heads are an nn.ModuleList, the deterministic (tanh) head and a Q network's
    # head one nn.Linear
    single = model.is_deterministic or getattr(model, "is_q_network", False)
    head = model.policy_head if single else model.policy_head[0]
    out.append((head.weight, head.bias))
    return out


class FusedSingleAgentRollout:
    @staticmethod
    def eligible(env_wrapper, models, policy_map):
        env = env_wrapper.env
        if getattr(env, "name", "") not in SINGLE_AGENT_ENVS or env_wrapper.n_agents != 1:
            return False
        if len(policy_map) != 1 or len(models) != 1:
            return False
        model = _unwrap(next(iter(models.values())))
        if getattr(model, "is_recurrent", False):     # (its forward keeps no state)
            return False
        continuous = SINGLE_AGENT_ENVS[env.name].continuous
        try:
            # discrete kinds: one softmax head; continuous kinds: one tanh head or one Gaussian
            # head (is_gaussian), of width 1, or one squashed Gaussian head
            # (is_squashed_gaussian) of width 2: [mu, log-std] of the one action
            if getattr(model, "is_deterministic", not continuous) != continuous:
                return False
            if len(model.output_dims) != 1 or (continuous and model.output_dims[0] != 1):
                return False
            if getattr(model, "action_mask", None) is not None or getattr(model, "masked", False):
                return False
            # normalized observations: the softmax and Gaussian heads have kinds that normalize
            if getattr(model, "normalize_observations", False) and continuous and not getattr(
                    model, "is_gaussian", False):
                return False
            # a noisy head draws fresh noise per env and step: the noisy Q kind takes a plain
            # head of one NoisyLinear; noisy C51 and noisy dueling heads act per step
            noisy = getattr(model, "noisy", False)
            if noisy and (model.dueling or getattr(model, "is_categorical_q", False)):
                return False
            # a dueling head runs as its folded layers: the stacked 2S stream layer, if any,
            # then the A * N outputs
            widths = [int(d) for d in model.fc_dims]
            if getattr(model, "dueling", False):
                from warp_drive_b200.training.algorithms.fused_dqn import folded_widths
                widths = folded_widths(model)
            if not 0 <= len(widths) <= 3:
                return False
            head = int(model.policy_head.out_features if continuous else model.output_dims[0])
            categorical = getattr(model, "is_categorical_q", False)
            if categorical:                    # C51: A blocks of N atom logits
                head = int(model.policy_head.out_features)
            dims = [int(model.flattened_obs_size)] + widths + [head]
            arr = (ctypes.c_int * 5)(*(dims + [0] * (5 - len(dims))))
            if categorical:
                return bool(_lib.load().wdb_single_agent_rollout_categorical_supported(
                    len(widths), arr, int(model.num_atoms)))
            if noisy:
                return bool(_lib.load().wdb_single_agent_rollout_noisy_supported(len(widths), arr))
            return bool(_lib.load().wdb_single_agent_rollout_supported(len(widths), arr))
        except Exception:  # noqa: BLE001
            return False

    def __init__(self, env_wrapper, model, policy, sampler, engine=None):
        self.dm = dm = env_wrapper.cuda_data_manager
        self.env_wrapper = env_wrapper
        self.model = model
        self.policy = policy
        self.sampler = sampler
        self.lib = _lib.load()
        self.E = env_wrapper.n_envs
        spec = SINGLE_AGENT_ENVS[env_wrapper.env.name]
        r = self.r = _lib.SaRollout()
        r.env_kind, r.n_envs, r.state_dim = spec.kind, self.E, spec.state_dim
        r.episode_length = int(dm.meta_info("episode_length"))
        for i, name in enumerate(spec.constants):
            r.env_params[i] = float(dm.device_data(name))
        r.state = _p(dm.device_data("state"))
        r.observations = _p(dm.device_data(_OBSERVATIONS))
        r.done = _p(dm.device_data("_done_"))
        r.env_timestep = _p(dm.device_data("_timestep_"))
        r.rewards = _p(dm.device_data(_REWARDS))
        r.sampled_actions = _p(dm.device_data(_ACTIONS))
        # a dueling Q network: the kernel runs its folded layers, kept in buffers of their own
        # and refreshed from the live parameters by one wdb_dueling_fold launch per rollout
        self._dueling = None
        if getattr(_unwrap(model), "dueling", False):
            from warp_drive_b200.training.algorithms.fused_dqn import DuelingFold
            m = _unwrap(model)
            self._dueling = DuelingFold(m)
            layers = [(m.fc[str(i)][0].weight, m.fc[str(i)][0].bias)
                      for i in range(len(m.fc))] + self._dueling.layers
        elif getattr(_unwrap(model), "noisy", False):
            # a noisy Q head: the kernel runs mu as the head's layer and reads sigma from the
            # device buffer below
            m = _unwrap(model)
            layers = [(m.fc[str(i)][0].weight, m.fc[str(i)][0].bias) for i in range(len(m.fc))]
            layers.append((m.policy_head.weight_mu, m.policy_head.bias_mu))
        else:
            layers = _layers(model)
        # a distributional Q network (QR-DQN's, IQN's): the kernel runs epsilon-greedy over its
        # mean, the head collapsed to one Linear(H, A) (collapsed_head), kept in buffers of its
        # own and recomputed from the live parameters at every launch
        self._quantile = model if hasattr(_unwrap(model), "collapsed_head") else None
        if self._quantile is not None:
            with torch.no_grad():
                w, b = _unwrap(model).collapsed_head()
            layers[-1] = self._collapsed = (w.contiguous(), b.contiguous())
        r.n_hidden = len(layers) - 1
        dims = [int(_unwrap(model).flattened_obs_size)] + [int(w.shape[0]) for w, _ in layers]
        for i, d in enumerate(dims):
            r.dims[i] = d
        self.F, self.A = dims[0], dims[-1]
        self._params = layers            # live nn.Parameters: optimizer steps update in place
        for i, (w, b) in enumerate(layers):
            assert w.is_cuda and w.dtype == torch.float32 and w.is_contiguous()
            r.w[i], r.b[i] = _p(w.data), _p(b.data)
        r.rng_state = _p(sampler.rng_state)
        r.reset_done_envs = 1
        self.continuous = spec.continuous
        self.gaussian = bool(getattr(_unwrap(model), "is_gaussian", False))
        self.squashed = bool(getattr(_unwrap(model), "is_squashed_gaussian", False))
        # DQN's Q network: epsilon-greedy over the raw head (sampler param `epsilon`)
        self.q_network = bool(getattr(_unwrap(model), "is_q_network", False))
        # C51's categorical Q network: the kernel reduces each action's atoms to their
        # expectation, and reads [epsilon, z_0 .. z_{N-1}] from the device (refreshed at every
        # launch); the categorical head is 4
        self.categorical = bool(getattr(_unwrap(model), "is_categorical_q", False))
        if self.categorical:
            self.A = int(_unwrap(model).output_dims[0])
        # a noisy Q head (5): the kernel reads [epsilon, the noise key's four words, sigma_W,
        # sigma_b] from the device, refreshed at every launch; the key is the engine's
        # (`noise_seed`, `acting_steps`), so both rollout paths draw the same noise at the same
        # acting step
        self.noisy = bool(getattr(_unwrap(model), "noisy", False))
        self.engine = engine
        if self.q_network:
            # the kernel reads epsilon from the device (the log_std field; the Q head is 3)
            r.gaussian_head = 5 if self.noisy else 4 if self.categorical else 3
            head = _unwrap(model).policy_head
            n = (1 + (int(_unwrap(model).num_atoms) if self.categorical else 0)
                 + (4 + head.weight_sigma.numel() + head.bias_sigma.numel() if self.noisy else 0))
            self._epsilon = torch.zeros(n, dtype=torch.float32, device=dm.device)
            r.log_std = _p(self._epsilon)
        if self.squashed:
            actor = _unwrap(model)
            r.gaussian_head = 2
            r.action_scale = float(actor.action_scale)
            r.action_bias = float(actor.action_bias)
            # the kernel reads the log-std's clamp bounds from the device
            self._log_std_bounds = torch.tensor([actor.log_std_min, actor.log_std_max],
                                                dtype=torch.float32, device=dm.device)
            r.log_std = _p(self._log_std_bounds)
        elif self.gaussian:
            r.gaussian_head = 1
            self._log_std = _unwrap(model).log_std
        # normalized observations: the softmax (6) or Gaussian (3) kind that normalizes, reading
        # [log_std (Gaussian) | shift F | scale F | clip] from a device buffer refreshed from the
        # model's statistics at every launch
        self.normalizing = bool(getattr(_unwrap(model), "normalize_observations", False))
        if self.normalizing:
            r.gaussian_head = 3 if self.gaussian else 6
            self._norm_args = torch.empty(int(self.gaussian) + 2 * self.F + 1,
                                          dtype=torch.float32, device=dm.device)
            self._norm_args[-1] = float(_unwrap(model).observation_clip)
        elif self.continuous:
            actor = _unwrap(model)
            r.action_scale = float(actor.action_scale)
            r.action_bias = float(actor.action_bias)
            r.ou_state = _p(dm.device_data(f"{_ACTIONS}_ou_state"))
        self._table = None

    def set_bookkeeping(self, reward_running_sum, episodic_reward_sum, step_running_sum,
                        episodic_step_sum, num_completed_episodes):
        r = self.r
        r.reward_running_sum = _p(reward_running_sum[self.policy])
        r.episodic_reward_sum = _p(episodic_reward_sum[self.policy])
        r.step_running_sum = _p(step_running_sum)
        r.episodic_step_sum = _p(episodic_step_sum)
        r.num_completed = _p(num_completed_episodes)
        self._keep = (reward_running_sum, episodic_reward_sum, step_running_sum,
                      episodic_step_sum, num_completed_episodes)

    def _reset_table(self):
        resetter = self.env_wrapper.env_resetter
        table, n = resetter.build_table(self.dm)
        if self.dm.reset_target_to_pool:
            assert resetter._random_initialized, (
                "reset pools need init_reset_pool(data_manager, seed) first")
        return table, n, resetter._pool_rng

    def _noise_words(self, eps, use_argmax, n_steps):
        """[epsilon, seed low, seed high, step low, step high] into the device buffer (one copy),
        sigma_W and sigma_b after them; the policy's acting step advances by n_steps unless the
        rollout is greedy (the mean network draws no noise)."""
        import numpy as np

        assert self.engine is not None, "a noisy head's rollout takes its noise key from the engine"
        seed, step = int(self.engine.noise_seed), int(self.engine.acting_steps[self.policy])
        words = np.array([0, seed, seed >> 32, step, step >> 32], dtype=np.uint64)
        words = (words & 0xFFFFFFFF).astype(np.uint32)
        words[0] = np.float32(eps).view(np.uint32)
        self._epsilon.view(torch.int32)[:5].copy_(torch.from_numpy(words.view(np.int32)))
        head = _unwrap(self.model).policy_head
        n_w = head.weight_sigma.numel()
        self._epsilon[5:5 + n_w].copy_(head.weight_sigma.detach().reshape(-1))
        self._epsilon[5 + n_w:].copy_(head.bias_sigma.detach())
        if not use_argmax:
            self.engine.acting_steps[self.policy] += int(n_steps)

    def launch(self, n_steps, t0=0, record=True, uniforms=None, probs_out=None,
               use_argmax=False, reset_done_envs=True, damping=None, stddev=None, scale=None,
               normals=None, epsilon=None):
        """Run `n_steps` timesteps.  record=True pushes them into batch slots t0 .. t0+n_steps-1
        of the policy's training batch.  Discrete kinds sample the softmax head (`uniforms`
        [n_steps, E] replaces the RNG draw, `probs_out` [n_steps, E, A] records the
        probabilities); continuous kinds add OU noise to the actor's mean with the parameters
        of CUDASampler.sample, or sample a Gaussian policy as CUDASampler.sample_gaussian
        (use_argmax: the mean), or a squashed Gaussian as CUDASampler.sample_squashed_gaussian
        (use_argmax: scale * tanh(mu) + bias) (`normals` [n_steps, E] replaces the RNG draw,
        `probs_out` [n_steps, E] records the mean, raw mu for the squashed head).  A Q network
        samples epsilon-greedily as CUDASampler.sample_epsilon_greedy with `epsilon` (default 0;
        use_argmax: 0), one draw per step; `probs_out` [n_steps, E, A] records the Q values (a
        categorical Q network's expectations)."""
        dm, r, p = self.dm, self.r, self.policy
        if self._dueling is not None:
            from warp_drive_b200.training.algorithms.fused_dqn import fold
            fold(self._dueling)
        if self._quantile is not None:
            with torch.no_grad():
                for buf, v in zip(self._collapsed, _unwrap(self._quantile).collapsed_head()):
                    buf.copy_(v)
        # parameters may have been re-allocated (load_state_dict keeps storage; .to() does not)
        for i, (w, b) in enumerate(self._params):
            r.w[i], r.b[i] = _p(w.data), _p(b.data)
        if self.gaussian:
            r.log_std = _p(self._log_std.data)
        if self.normalizing:
            m = _unwrap(self.model)
            parts = ([m.log_std.detach()] if self.gaussian else []) + [m.obs_shift, m.obs_scale]
            torch.cat(parts, out=self._norm_args[:-1])
            r.log_std = _p(self._norm_args)
        r.n_steps = int(n_steps)
        r.use_argmax = int(bool(use_argmax))
        r.uniforms = _p(uniforms)
        r.probs_batch = _p(probs_out)
        r.ou_damping = float(0.15 if damping is None else damping)
        r.ou_stddev = float(0.2 if stddev is None else stddev)
        r.ou_scale = float(1.0 if scale is None else scale)
        r.normals = _p(normals)
        if self.q_network:
            eps = float(0.0 if epsilon is None else epsilon)
            if not 0.0 <= eps <= 1.0:
                raise ValueError(f"epsilon must be in [0, 1], got {epsilon}")
            if self.noisy:
                self._noise_words(eps, use_argmax, n_steps)
            else:
                self._epsilon[0] = eps
            if self.categorical:
                self._epsilon[1:].copy_(_unwrap(self.model).support)
        if record:
            obs_b = dm.data_on_device_via_torch(f"{_PROCESSED_OBSERVATIONS}_batch_{p}")
            assert t0 + n_steps <= obs_b.shape[0]
            r.obs_batch = _p(obs_b[t0])
            r.actions_batch = _p(dm.data_on_device_via_torch(f"{_ACTIONS}_batch_{p}")[t0])
            r.rewards_batch = _p(dm.data_on_device_via_torch(f"{_REWARDS}_batch_{p}")[t0])
            r.done_batch = _p(dm.data_on_device_via_torch(f"{_DONE_FLAGS}_batch")[t0])
        else:
            r.obs_batch = r.actions_batch = r.rewards_batch = r.done_batch = None
        table, n, pool_rng = self._reset_table()
        self._table = table
        r.reset_table = _p(table) if n > 0 else None
        r.n_reset_arrays = n
        r.pool_rng = _p(pool_rng)
        r.reset_done_envs = int(bool(reset_done_envs))
        _lib.check(self.lib.wdb_single_agent_rollout(_lib.stream_ptr(), ctypes.byref(r)),
                   "single_agent_rollout")
