"""ctypes binding of libwdb200.so (the C ABI declared in include/wdb200.h).

This is the ONLY compute backend of the package: if the shared library is missing the
import of any kernel-facing module fails loudly -- there is no Python / CPU fallback.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libwdb200.so")

_vp = ctypes.c_void_p
_i = ctypes.c_int
_f = ctypes.c_float
_ll = ctypes.c_longlong
_ull = ctypes.c_ulonglong


class ResetDesc(ctypes.Structure):
    """struct wdb_reset_desc (include/wdb200.h)."""

    _fields_ = [("dst", _vp), ("ref", _vp), ("bytes_per_env", _ll), ("pool_rows", _ll)]


_fp = ctypes.c_void_p  # device pointers travel as integers


class TcEnv(ctypes.Structure):
    """struct wdb_tc_env (include/wdb200.h)."""

    _fields_ = [
        ("n_envs", _i), ("n_agents", _i),
        ("loc_x", _fp), ("loc_y", _fp), ("speed", _fp), ("direction", _fp),
        ("acceleration", _fp), ("agent_types", _fp), ("edge_hit_reward_penalty", _fp),
        ("edge_hit_penalty", _f), ("grid_length", _f),
        ("acceleration_actions", _fp), ("turn_actions", _fp),
        ("max_speed", _f), ("num_other_agents_observed", _i), ("skill_levels", _fp),
        ("runner_exits_game_after_tagged", _i), ("still_in_the_game", _fp),
        ("use_full_observation", _i), ("obs", _fp), ("neighbor_distances", _fp),
        ("neighbor_ids_sorted_by_distance", _fp), ("nearest_neighbor_ids", _fp),
        ("rewards", _fp), ("step_rewards", _fp), ("num_runners", _fp),
        ("distance_margin_for_reward", _f), ("tag_reward_for_tagger", _f),
        ("tag_penalty_for_runner", _f), ("end_of_game_reward_for_runner", _f),
        ("done", _fp), ("env_timestep", _fp), ("episode_length", _i), ("stats", _fp),
        ("blocks_per_env", _i),
    ]


class TcPolicyIO(ctypes.Structure):
    """struct wdb_tc_policy_io."""

    _fields_ = [
        ("n_agents", _i), ("probs0", _fp), ("probs1", _fp), ("actions_batch", _fp),
        ("rewards_batch", _fp), ("obs_next", _fp), ("reward_running_sum", _fp),
        ("episodic_reward_sum", _fp), ("obs_next_tiles", _fp),
    ]


class TcRollout(ctypes.Structure):
    """struct wdb_tc_rollout."""

    _fields_ = [
        ("rng_state", _fp), ("uniforms", _fp),
        ("n_policies", _i), ("n_actions0", _i), ("n_actions1", _i),
        ("agent_policy", _fp), ("agent_slot", _fp),
        ("policy", TcPolicyIO * 4),
        ("sampled_actions", _fp), ("sampled_actions_0", _fp), ("sampled_actions_1", _fp),
        ("done_batch", _fp), ("step_running_sum", _fp),
        ("episodic_step_sum", _fp), ("num_completed_episodes", _fp),
        ("reset_table", _fp), ("n_reset_arrays", _i), ("obs_at_reset", _fp),
        ("reset_done_envs", _i), ("launch_after_forward", _i), ("actions_in", _i),
        ("env_begin", _i), ("env_count", _i),
    ]


class GatherPolicy(ctypes.Structure):
    _fields_ = [("n_agents", _i), ("agent_ids", _fp), ("rows", _fp)]


class Gather(ctypes.Structure):
    """struct wdb_gather (include/wdb200.h)."""

    _fields_ = [
        ("n_envs", _i), ("n_agents", _i), ("width", _i), ("n_policies", _i), ("scatter", _i),
        ("full", _fp), ("policy", GatherPolicy * 4),
    ]


GATHER_MAX_FIELDS = 16


class GatherField(ctypes.Structure):
    _fields_ = [("src", _fp), ("width", _i), ("is_int32", _i), ("dst", _i), ("col", _i),
                ("policy_mask", _i), ("own_rows", _i), ("agents_last", _i)]


class GatherFieldsPolicy(ctypes.Structure):
    _fields_ = [("n_agents", _i), ("agent_ids", _fp), ("rows", _fp * 2), ("dst_width", _i * 2)]


class GatherFields(ctypes.Structure):
    """struct wdb_gather_fields (include/wdb200.h)."""

    _fields_ = [
        ("n_envs", _i), ("n_agents", _i), ("n_policies", _i), ("n_fields", _i),
        ("dst_width", _i * 2), ("field", GatherField * GATHER_MAX_FIELDS),
        ("policy", GatherFieldsPolicy * 4),
    ]


class BookkeepPolicy(ctypes.Structure):
    _fields_ = [
        ("n_agents", _i), ("agent_ids", _fp), ("rewards_batch", _fp), ("actions_batch", _fp),
        ("reward_running_sum", _fp), ("episodic_reward_sum", _fp),
        ("rewards", _fp), ("actions", _fp), ("n_heads", _i),
    ]


class Bookkeep(ctypes.Structure):
    """struct wdb_bookkeep (include/wdb200.h)."""

    _fields_ = [
        ("n_envs", _i), ("n_agents", _i), ("n_policies", _i), ("n_heads", _i),
        ("done", _fp), ("rewards", _fp), ("actions", _fp), ("done_batch", _fp),
        ("step_running_sum", _fp), ("episodic_step_sum", _fp), ("num_completed_episodes", _fp),
        ("policy", BookkeepPolicy * 4),
    ]


class MlpPair(ctypes.Structure):
    """struct wdb_mlp_pair (include/wdb200.h)."""

    _fields_ = [
        ("blob", _fp * 2), ("F", _i * 2), ("H", _i * 2), ("A0", _i * 2), ("A1", _i * 2),
        ("obs", _fp * 2), ("rows", ctypes.c_longlong * 2),
        ("probs0", _fp * 2), ("probs1", _fp * 2), ("values", _fp * 2),
        ("ctas_b", _i), ("flags", _i),
    ]


MLP_WEIGHTS_STABLE = 1


class MlpSampling(ctypes.Structure):
    """struct wdb_mlp_sampling (include/wdb200.h)."""

    _fields_ = [
        ("actions", _fp), ("rng_state", _fp), ("uniforms", _fp), ("agent_of_slot", _fp),
        ("n_agents", _i), ("n_policy_agents", _i), ("row_offset", ctypes.c_longlong),
    ]


class SaRollout(ctypes.Structure):
    """struct wdb_sa_rollout (include/wdb200.h)."""

    _fields_ = [
        ("env_kind", _i), ("n_envs", _i), ("n_steps", _i), ("episode_length", _i),
        ("state_dim", _i), ("use_argmax", _i), ("env_params", _f * 12),
        ("state", _fp), ("observations", _fp), ("done", _fp), ("env_timestep", _fp),
        ("rewards", _fp), ("sampled_actions", _fp),
        ("n_hidden", _i), ("dims", _i * 5), ("w", _fp * 4), ("b", _fp * 4),
        ("rng_state", _fp), ("uniforms", _fp),
        ("obs_batch", _fp), ("actions_batch", _fp), ("rewards_batch", _fp),
        ("done_batch", _fp), ("probs_batch", _fp),
        ("reward_running_sum", _fp), ("step_running_sum", _fp), ("episodic_reward_sum", _fp),
        ("episodic_step_sum", _fp), ("num_completed", _fp),
        ("reset_table", _fp), ("n_reset_arrays", _i), ("pool_rng", _fp),
        ("reset_done_envs", _i),
        ("ou_damping", _f), ("ou_stddev", _f), ("ou_scale", _f), ("ou_state", _fp),
        ("action_scale", _f), ("action_bias", _f), ("normals", _fp),
        ("log_std", _fp), ("gaussian_head", _i),
    ]


class PgLoss(ctypes.Structure):
    """struct wdb_pg_loss (include/wdb200.h)."""

    _fields_ = [
        ("T", _i), ("n_envs", _i), ("n_agents", _i), ("n_heads", _i), ("n_actions", _i * 4),
        ("probs", _fp * 4), ("values", _fp), ("actions", _fp), ("rewards", _fp), ("done", _fp),
        ("gamma", _f), ("vf_coeff", _f), ("entropy_coeff", _f),
        ("grad_probs", _fp * 4), ("grad_values", _fp), ("returns", _fp), ("sums", _fp),
    ]


PG_GAUSSIAN_MAX_DIM = 8
PG_GAUSSIAN_ROWS_PER_CTA = 128


class PgGaussianLoss(ctypes.Structure):
    """struct wdb_pg_gaussian_loss (include/wdb200.h)."""

    _fields_ = [
        ("T", _i), ("n_envs", _i), ("n_agents", _i), ("action_dim", _i),
        ("mean", _fp), ("log_std", _fp), ("values", _fp), ("actions", _fp), ("rewards", _fp),
        ("done", _fp), ("gamma", _f), ("vf_coeff", _f), ("entropy_coeff", _f),
        ("grad_mean", _fp), ("grad_log_std", _fp), ("grad_values", _fp), ("returns", _fp),
        ("sums", _fp), ("partials", _fp),
    ]


class GaeArgs(ctypes.Structure):
    """struct wdb_gae_args (include/wdb200.h)."""

    _fields_ = [
        ("T", _i), ("n_envs", _i), ("n_agents", _i), ("rewards", _fp), ("values", _fp),
        ("done", _fp), ("gamma", _f), ("gae_lambda", _f), ("advantages", _fp),
        ("value_targets", _fp),
    ]


class PpoLoss(ctypes.Structure):
    """struct wdb_ppo_loss (include/wdb200.h)."""

    _fields_ = [
        ("B", _i), ("n_heads", _i), ("n_actions", _i * 4), ("probs", _fp * 4), ("values", _fp),
        ("rows", _fp), ("actions", _fp), ("advantages", _fp), ("value_targets", _fp),
        ("old_log_prob", _fp), ("ppo", _i), ("clip_param", _f), ("vf_coeff", _f),
        ("entropy_coeff", _f), ("grad_probs", _fp * 4), ("grad_values", _fp),
        ("log_prob", _fp), ("sums", _fp),
    ]


class PpoGaussianLoss(ctypes.Structure):
    """struct wdb_ppo_gaussian_loss (include/wdb200.h)."""

    _fields_ = [
        ("B", _i), ("action_dim", _i), ("mean", _fp), ("log_std", _fp), ("values", _fp),
        ("rows", _fp), ("actions", _fp), ("advantages", _fp), ("value_targets", _fp),
        ("old_log_prob", _fp), ("ppo", _i), ("clip_param", _f), ("vf_coeff", _f),
        ("entropy_coeff", _f), ("grad_mean", _fp), ("grad_log_std", _fp),
        ("grad_values", _fp), ("log_prob", _fp), ("sums", _fp), ("partials", _fp),
    ]


class DdpgNet(ctypes.Structure):
    """struct wdb_ddpg_net (include/wdb200.h)."""

    _fields_ = [("n_hidden", _i), ("widths", _i * 3), ("w", _fp * 4), ("b", _fp * 4),
                ("gw", _fp * 4), ("gb", _fp * 4)]


class DdpgUpdate(ctypes.Structure):
    """struct wdb_ddpg_update_args (include/wdb200.h)."""

    _fields_ = [
        ("n_envs", _i), ("n_agents", _i), ("obs_dim", _i), ("action_dim", _i),
        ("capacity", _i), ("cursor", _i), ("n_step", _i),
        ("gamma", _f), ("action_scale", _f), ("action_bias", _f),
        ("obs", _fp), ("actions", _fp), ("rewards", _fp), ("done", _fp),
        ("actor", DdpgNet), ("critic", DdpgNet), ("target_actor", DdpgNet),
        ("target_critic", DdpgNet),
        ("values", _fp), ("j_values", _fp), ("returns", _fp), ("sums", _fp),
        ("workspace", _fp),
    ]


class Td3Update(ctypes.Structure):
    """struct wdb_td3_update_args (include/wdb200.h)."""

    _fields_ = [
        ("n_envs", _i), ("n_agents", _i), ("obs_dim", _i), ("action_dim", _i),
        ("capacity", _i), ("cursor", _i), ("n_step", _i),
        ("gamma", _f), ("action_scale", _f), ("action_bias", _f),
        ("target_noise", _f), ("target_noise_clip", _f),
        ("obs", _fp), ("actions", _fp), ("rewards", _fp), ("done", _fp), ("noise", _fp),
        ("actor", DdpgNet), ("critic", DdpgNet), ("critic2", DdpgNet),
        ("target_actor", DdpgNet), ("target_critic", DdpgNet), ("target_critic2", DdpgNet),
        ("q1_values", _fp), ("q2_values", _fp), ("returns", _fp), ("j_values", _fp),
        ("sums", _fp), ("workspace", _fp),
    ]


class SacUpdate(ctypes.Structure):
    """struct wdb_sac_update_args (include/wdb200.h)."""

    _fields_ = [
        ("n_envs", _i), ("n_agents", _i), ("obs_dim", _i), ("action_dim", _i),
        ("capacity", _i), ("cursor", _i), ("n_step", _i),
        ("gamma", _f), ("action_scale", _f), ("action_bias", _f),
        ("log_std_min", _f), ("log_std_max", _f), ("log_alpha", _fp),
        ("obs", _fp), ("actions", _fp), ("rewards", _fp), ("done", _fp),
        ("critic_noise", _fp), ("actor_noise", _fp),
        ("actor", DdpgNet), ("critic", DdpgNet), ("critic2", DdpgNet),
        ("target_critic", DdpgNet), ("target_critic2", DdpgNet),
        ("q1_values", _fp), ("q2_values", _fp), ("returns", _fp), ("log_probs", _fp),
        ("sums", _fp), ("workspace", _fp),
    ]


class SacDiscreteUpdate(ctypes.Structure):
    """struct wdb_sac_discrete_update_args (include/wdb200.h)."""

    _fields_ = [
        ("n_envs", _i), ("n_agents", _i), ("obs_dim", _i), ("n_actions", _i),
        ("capacity", _i), ("n_step", _i), ("gamma", _f),
        ("obs", _fp), ("actions", _fp), ("rewards", _fp), ("done", _fp), ("log_alpha", _fp),
        ("actor", DdpgNet), ("critic", DdpgNet), ("critic2", DdpgNet),
        ("target_critic", DdpgNet), ("target_critic2", DdpgNet),
        ("q1_values", _fp), ("q2_values", _fp), ("returns", _fp), ("entropies", _fp),
        ("sums", _fp), ("workspace", _fp),
    ]


class TqcUpdate(ctypes.Structure):
    """struct wdb_tqc_update_args (include/wdb200.h)."""

    _fields_ = [
        ("n_envs", _i), ("n_agents", _i), ("obs_dim", _i), ("action_dim", _i),
        ("capacity", _i), ("n_step", _i), ("n_quantiles", _i), ("n_drop", _i),
        ("gamma", _f), ("action_scale", _f), ("action_bias", _f),
        ("log_std_min", _f), ("log_std_max", _f), ("log_alpha", _fp),
        ("obs", _fp), ("actions", _fp), ("rewards", _fp), ("done", _fp),
        ("critic_noise", _fp), ("actor_noise", _fp),
        ("actor", DdpgNet), ("critic", DdpgNet), ("critic2", DdpgNet),
        ("target_critic", DdpgNet), ("target_critic2", DdpgNet),
        ("q_means", _fp), ("target_means", _fp), ("log_probs", _fp),
        ("sums", _fp), ("workspace", _fp),
    ]


class ReplayWindows(ctypes.Structure):
    """struct wdb_replay_windows (include/wdb200.h)."""

    _fields_ = [("windows", _fp), ("n_windows", _i)]


class DqnUpdate(ctypes.Structure):
    """struct wdb_dqn_update_args (include/wdb200.h)."""

    _fields_ = [
        ("n_envs", _i), ("n_agents", _i), ("obs_dim", _i), ("n_actions", _i),
        ("capacity", _i), ("n_step", _i), ("gamma", _f), ("huber_delta", _f), ("double_q", _i),
        ("obs", _fp), ("actions", _fp), ("rewards", _fp), ("done", _fp),
        ("q", DdpgNet), ("target_q", DdpgNet),
        ("q_values", _fp), ("returns", _fp), ("sums", _fp), ("workspace", _fp),
    ]


class IqnArgs(ctypes.Structure):
    """struct wdb_iqn_args (include/wdb200.h)."""

    _fields_ = [
        ("n_cos", _i), ("n_tau", _i), ("n_tau_prime", _i), ("n_quantile_samples", _i),
        ("taus", _fp), ("embed", DdpgNet), ("target_embed", DdpgNet),
    ]


Q_MAX_BRANCHES = 16                          # wdb_q_branches.sizes


class QBranches(ctypes.Structure):
    """struct wdb_q_branches (include/wdb200.h)."""

    _fields_ = [("n_heads", _i), ("sizes", _i * Q_MAX_BRANCHES)]


class DuelingHead(ctypes.Structure):
    """struct wdb_dueling_head (include/wdb200.h)."""

    _fields_ = [
        ("n_actions", _i), ("n_atoms", _i), ("in_dim", _i), ("stream_dim", _i),
        ("value_hw", _fp), ("value_hb", _fp), ("value_ow", _fp), ("value_ob", _fp),
        ("adv_hw", _fp), ("adv_hb", _fp), ("adv_ow", _fp), ("adv_ob", _fp),
        ("value_ghw", _fp), ("value_ghb", _fp), ("value_gow", _fp), ("value_gob", _fp),
        ("adv_ghw", _fp), ("adv_ghb", _fp), ("adv_gow", _fp), ("adv_gob", _fp),
        ("hw", _fp), ("hb", _fp), ("ow", _fp), ("ob", _fp),
        ("ghw", _fp), ("ghb", _fp), ("gow", _fp), ("gob", _fp),
    ]


NOISY_MAX_LAYERS = 4


class NoisyLayer(ctypes.Structure):
    """struct wdb_noisy_layer (include/wdb200.h)."""

    _fields_ = [
        ("in_dim", _i), ("out_dim", _i),
        ("weight_mu", _fp), ("weight_sigma", _fp), ("bias_mu", _fp), ("bias_sigma", _fp),
        ("noise_in", _fp), ("noise_out", _fp), ("weight", _fp), ("bias", _fp),
        ("grad_weight", _fp), ("grad_bias", _fp),
        ("grad_weight_mu", _fp), ("grad_weight_sigma", _fp), ("grad_bias_mu", _fp),
        ("grad_bias_sigma", _fp),
    ]


class NoisyNet(ctypes.Structure):
    """struct wdb_noisy_net (include/wdb200.h)."""

    _fields_ = [("n_layers", _i), ("layer", NoisyLayer * NOISY_MAX_LAYERS)]


class PerStore(ctypes.Structure):
    """struct wdb_per_store (include/wdb200.h)."""

    _fields_ = [
        ("capacity", _i), ("n_rows", _i), ("n_step", _i), ("alpha", _f), ("epsilon", _f),
        ("leaves", _fp), ("nodes", _fp), ("p_max", _fp),
    ]


GRU_HEAD_SOFTMAX, GRU_HEAD_MEAN = 0, 1     # wdb_gru_forward.head_kind


class GruForward(ctypes.Structure):
    """struct wdb_gru_forward (include/wdb200.h)."""

    _fields_ = [
        ("n_rows", _ll), ("in_dim", _i), ("n_layers", _i), ("dims", _i * 2),
        ("hidden_size", _i), ("n_heads", _i), ("heads", _i * 2),
        ("obs", _fp), ("hidden", _fp), ("fc_weight", _fp * 2), ("fc_bias", _fp * 2),
        ("weight_ih", _fp), ("weight_hh", _fp), ("bias_ih", _fp), ("bias_hh", _fp),
        ("head_weight", _fp * 2), ("head_bias", _fp * 2), ("probs", _fp * 2),
        ("head_kind", _i),
    ]


RECURRENT_MAX_POLICIES = 8


class RecurrentState(ctypes.Structure):
    """struct wdb_recurrent_state (include/wdb200.h)."""

    _fields_ = [("hidden", _fp), ("n_agents", _i), ("hidden_size", _i)]


class RecurrentReset(ctypes.Structure):
    """struct wdb_recurrent_reset (include/wdb200.h)."""

    _fields_ = [("done", _vp), ("n_envs", _i), ("n_policies", _i),
                ("policy", RecurrentState * RECURRENT_MAX_POLICIES)]


_SIGNATURES = {
    "wdb_abi_version": (_i, []),
    "wdb_error_string": (ctypes.c_char_p, [_i]),
    "wdb_launch_count": (_ll, []),
    "wdb_set_option": (_i, [ctypes.c_char_p, _i]),
    "wdb_rng_state_bytes": (_ll, [_ll]),
    "wdb_rng_init": (_i, [_vp, _vp, _ll, _ull]),
    "wdb_rng_draw_u32x4": (_i, [_vp, _vp, _vp, _ll]),
    "wdb_sample_actions": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _i, _i, _vp]),
    "wdb_sample_actions_nonzero": (
        _i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _i, _i, _vp]),
    "wdb_sample_ou_process": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _f, _f, _f, _vp]),
    "wdb_sample_gaussian": (_i, [_vp, _vp, _vp, _vp, _vp, _ll, _i, _i, _vp]),
    "wdb_sample_squashed_gaussian": (
        _i, [_vp, _vp, _vp, _vp, _ll, _i, _f, _f, _f, _f, _i, _vp]),
    "wdb_sample_epsilon_greedy": (_i, [_vp, _vp, _vp, _vp, _ll, _i, _f, _vp]),
    "wdb_sample_epsilon_greedy_masked": (_i, [_vp, _vp, _vp, _vp, _vp, _ll, _i, _f, _vp]),
    "wdb_reset_when_done": (_i, [_vp, _vp, _i, _vp, _vp, _i, _i, _i, _vp]),
    "wdb_reset_log_mask": (_i, [_vp, _vp, _i]),
    "wdb_update_log_mask": (_i, [_vp, _vp, _i, _i]),
    "wdb_log_one_step": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i]),
    "wdb_testkernel": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _f, _i, _i, _i]),
    "wdb_tag_gridworld_step": (
        _i,
        [_vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _i, _i, _vp, _i, _vp],
    ),
    "wdb_tag_continuous_step": (
        _i,
        [_vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _f, _f, _vp, _vp, _f, _i,
         _vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _vp,
         _vp, _i, _vp],
    ),
    "wdb_tag_continuous_rollout_step": (
        _i, [_vp, ctypes.POINTER(TcEnv), ctypes.POINTER(TcRollout)]),
    "wdb_tag_continuous_rollout_supported": (
        _i, [ctypes.POINTER(TcEnv), ctypes.POINTER(TcRollout), _i]),
    "wdb_mlp_blob_bytes": (_ll, [_i, _i, _i, _i]),
    "wdb_mlp_pack_weights": (_i, [_vp] * 12 + [_i, _i, _i, _i]),
    "wdb_mlp_policy_forward": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _ll, _vp, _vp, _vp]),
    "wdb_mlp_policy_forward_masked": (
        _i, [_vp, _vp, _i, _i, _i, _i, _vp, _ll, _vp, _vp, _vp, _vp]),
    "wdb_mlp_policy_forward_pair": (_i, [_vp, ctypes.POINTER(MlpPair)]),
    "wdb_mlp_forward_samples": (_i, [_i, _i, _i, _i]),
    "wdb_mlp_policy_forward_sampled": (
        _i, [_vp, _vp, _i, _i, _i, _i, _vp, _i, _ll, _vp, _vp, _vp, ctypes.POINTER(MlpSampling)]),
    "wdb_gather_policy_rows": (_i, [_vp, ctypes.POINTER(Gather)]),
    "wdb_gather_policy_fields": (_i, [_vp, ctypes.POINTER(GatherFields)]),
    "wdb_rollout_bookkeep": (_i, [_vp, ctypes.POINTER(Bookkeep)]),
    "wdb_mlp_obs_tiles_bytes": (_ll, [_i, _ll]),
    "wdb_mlp_pack_obs": (_i, [_vp, _vp, _ll, _i, _vp]),
    "wdb_mlp_policy_forward_tiles": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _ll, _vp, _vp, _vp]),
    "wdb_discounted_returns": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _f]),
    "wdb_pg_loss_and_grads": (_i, [_vp, ctypes.POINTER(PgLoss)]),
    "wdb_pg_loss_supported": (_i, [_i, ctypes.POINTER(_i)]),
    "wdb_pg_gaussian_loss_and_grads": (_i, [_vp, ctypes.POINTER(PgGaussianLoss)]),
    "wdb_pg_gaussian_loss_supported": (_i, [_i]),
    "wdb_gae": (_i, [_vp, ctypes.POINTER(GaeArgs)]),
    "wdb_ppo_loss_and_grads": (_i, [_vp, ctypes.POINTER(PpoLoss)]),
    "wdb_ppo_loss_supported": (_i, [_i, ctypes.POINTER(_i)]),
    "wdb_ppo_gaussian_loss_and_grads": (_i, [_vp, ctypes.POINTER(PpoGaussianLoss)]),
    "wdb_ppo_gaussian_loss_supported": (_i, [_i]),
    "wdb_heads_softmax": (_i, [_vp, _vp, _ll, _i, _i, _i, _vp, _vp, _vp]),
    "wdb_heads_softmax_masked": (_i, [_vp, _vp, _ll, _i, _i, _i, _vp, _i, _vp, _vp, _vp]),
    "wdb_heads_softmax_backward": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _ll, _i, _i, _i, _vp]),
    "wdb_heads_softmax_supported": (_i, [_i, _i, _i]),
    "wdb_pad_rows": (_i, [_vp, _vp, _ll, _i, _i, _vp]),
    "wdb_relu_backward_bias_rows": (_i, [_ll]),
    "wdb_relu_backward_bias": (_i, [_vp, _vp, _vp, _ll, _i, _vp]),
    "wdb_grad_sumsq": (_i, [_vp, _vp, _ll, _vp]),
    "wdb_adam_step": (_i, [_vp, _vp, _vp, _vp, _vp, _ll, _f, _f, _f, _f, _i, _f, _vp]),
    "wdb_ddpg_update_supported": (_i, [ctypes.POINTER(DdpgUpdate)]),
    "wdb_ddpg_update_workspace_bytes": (_ll, [ctypes.POINTER(DdpgUpdate)]),
    "wdb_ddpg_update": (_i, [_vp, ctypes.POINTER(DdpgUpdate)]),
    "wdb_td3_critic_update_supported": (_i, [ctypes.POINTER(Td3Update)]),
    "wdb_td3_critic_update_workspace_bytes": (_ll, [ctypes.POINTER(Td3Update)]),
    "wdb_td3_critic_update": (_i, [_vp, ctypes.POINTER(Td3Update)]),
    "wdb_td3_actor_update_supported": (_i, [ctypes.POINTER(Td3Update)]),
    "wdb_td3_actor_update_workspace_bytes": (_ll, [ctypes.POINTER(Td3Update)]),
    "wdb_td3_actor_update": (_i, [_vp, ctypes.POINTER(Td3Update)]),
    "wdb_sac_critic_update_supported": (_i, [ctypes.POINTER(SacUpdate)]),
    "wdb_sac_critic_update_workspace_bytes": (_ll, [ctypes.POINTER(SacUpdate)]),
    "wdb_sac_critic_update": (_i, [_vp, ctypes.POINTER(SacUpdate)]),
    "wdb_sac_actor_update_supported": (_i, [ctypes.POINTER(SacUpdate)]),
    "wdb_sac_actor_update_workspace_bytes": (_ll, [ctypes.POINTER(SacUpdate)]),
    "wdb_sac_actor_update": (_i, [_vp, ctypes.POINTER(SacUpdate)]),
    "wdb_ddpg_update_sampled_supported": (_i, [ctypes.POINTER(DdpgUpdate), _i]),
    "wdb_ddpg_update_sampled_workspace_bytes": (_ll, [ctypes.POINTER(DdpgUpdate), _i]),
    "wdb_ddpg_update_sampled": (
        _i, [_vp, ctypes.POINTER(DdpgUpdate), ctypes.POINTER(ReplayWindows)]),
    "wdb_td3_critic_update_sampled_supported": (_i, [ctypes.POINTER(Td3Update), _i]),
    "wdb_td3_critic_update_sampled_workspace_bytes": (_ll, [ctypes.POINTER(Td3Update), _i]),
    "wdb_td3_critic_update_sampled": (
        _i, [_vp, ctypes.POINTER(Td3Update), ctypes.POINTER(ReplayWindows)]),
    "wdb_td3_actor_update_sampled_supported": (_i, [ctypes.POINTER(Td3Update), _i]),
    "wdb_td3_actor_update_sampled_workspace_bytes": (_ll, [ctypes.POINTER(Td3Update), _i]),
    "wdb_td3_actor_update_sampled": (
        _i, [_vp, ctypes.POINTER(Td3Update), ctypes.POINTER(ReplayWindows)]),
    "wdb_sac_critic_update_sampled_supported": (_i, [ctypes.POINTER(SacUpdate), _i]),
    "wdb_sac_critic_update_sampled_workspace_bytes": (_ll, [ctypes.POINTER(SacUpdate), _i]),
    "wdb_sac_critic_update_sampled": (
        _i, [_vp, ctypes.POINTER(SacUpdate), ctypes.POINTER(ReplayWindows)]),
    "wdb_sac_actor_update_sampled_supported": (_i, [ctypes.POINTER(SacUpdate), _i]),
    "wdb_sac_actor_update_sampled_workspace_bytes": (_ll, [ctypes.POINTER(SacUpdate), _i]),
    "wdb_sac_actor_update_sampled": (
        _i, [_vp, ctypes.POINTER(SacUpdate), ctypes.POINTER(ReplayWindows)]),
    "wdb_dqn_update_sampled_supported": (_i, [ctypes.POINTER(DqnUpdate), _i]),
    "wdb_dqn_update_sampled_workspace_bytes": (_ll, [ctypes.POINTER(DqnUpdate), _i]),
    "wdb_dqn_update_sampled": (
        _i, [_vp, ctypes.POINTER(DqnUpdate), ctypes.POINTER(ReplayWindows)]),
    "wdb_dqn_update_prioritized_supported": (_i, [ctypes.POINTER(DqnUpdate), _i]),
    "wdb_dqn_update_prioritized_workspace_bytes": (_ll, [ctypes.POINTER(DqnUpdate), _i]),
    "wdb_dqn_update_prioritized": (
        _i, [_vp, ctypes.POINTER(DqnUpdate), ctypes.POINTER(ReplayWindows), _vp]),
    "wdb_qr_dqn_update_sampled_supported": (_i, [ctypes.POINTER(DqnUpdate), _i, _i]),
    "wdb_qr_dqn_update_sampled_workspace_bytes": (_ll, [ctypes.POINTER(DqnUpdate), _i, _i]),
    "wdb_qr_dqn_update_sampled": (
        _i, [_vp, ctypes.POINTER(DqnUpdate), _i, ctypes.POINTER(ReplayWindows), _vp]),
    "wdb_iqn_update_sampled_supported": (
        _i, [ctypes.POINTER(DqnUpdate), ctypes.POINTER(IqnArgs), _i]),
    "wdb_iqn_update_sampled_workspace_bytes": (
        _ll, [ctypes.POINTER(DqnUpdate), ctypes.POINTER(IqnArgs), _i]),
    "wdb_iqn_update_sampled": (
        _i, [_vp, ctypes.POINTER(DqnUpdate), ctypes.POINTER(IqnArgs),
             ctypes.POINTER(ReplayWindows), _vp]),
    "wdb_c51_update_sampled_supported": (_i, [ctypes.POINTER(DqnUpdate), _i, _i]),
    "wdb_c51_update_sampled_workspace_bytes": (_ll, [ctypes.POINTER(DqnUpdate), _i, _i]),
    "wdb_c51_update_sampled": (
        _i, [_vp, ctypes.POINTER(DqnUpdate), _i, _vp, _f, ctypes.POINTER(ReplayWindows), _vp]),
    "wdb_dqn_update_masked_supported": (_i, [ctypes.POINTER(DqnUpdate), _i]),
    "wdb_dqn_update_masked_workspace_bytes": (_ll, [ctypes.POINTER(DqnUpdate), _i]),
    "wdb_dqn_update_masked": (
        _i, [_vp, ctypes.POINTER(DqnUpdate), ctypes.POINTER(ReplayWindows), _vp, _vp]),
    "wdb_c51_update_masked_supported": (_i, [ctypes.POINTER(DqnUpdate), _i, _i]),
    "wdb_c51_update_masked_workspace_bytes": (_ll, [ctypes.POINTER(DqnUpdate), _i, _i]),
    "wdb_c51_update_masked": (
        _i, [_vp, ctypes.POINTER(DqnUpdate), _i, _vp, _f, ctypes.POINTER(ReplayWindows), _vp,
             _vp]),
    "wdb_sample_epsilon_greedy_branching": (
        _i, [_vp, _vp, _vp, ctypes.POINTER(QBranches), _vp, _ll, _f, _vp]),
    "wdb_branching_dqn_update_sampled_supported": (
        _i, [ctypes.POINTER(DqnUpdate), ctypes.POINTER(QBranches), _i]),
    "wdb_branching_dqn_update_sampled_workspace_bytes": (
        _ll, [ctypes.POINTER(DqnUpdate), ctypes.POINTER(QBranches), _i]),
    "wdb_branching_dqn_update_sampled": (
        _i, [_vp, ctypes.POINTER(DqnUpdate), ctypes.POINTER(QBranches),
             ctypes.POINTER(ReplayWindows)]),
    "wdb_branching_dqn_update_prioritized_supported": (
        _i, [ctypes.POINTER(DqnUpdate), ctypes.POINTER(QBranches), _i]),
    "wdb_branching_dqn_update_prioritized_workspace_bytes": (
        _ll, [ctypes.POINTER(DqnUpdate), ctypes.POINTER(QBranches), _i]),
    "wdb_branching_dqn_update_prioritized": (
        _i, [_vp, ctypes.POINTER(DqnUpdate), ctypes.POINTER(QBranches),
             ctypes.POINTER(ReplayWindows), _vp]),
    "wdb_sac_discrete_critic_update_sampled_supported": (
        _i, [ctypes.POINTER(SacDiscreteUpdate), _i]),
    "wdb_sac_discrete_critic_update_sampled_workspace_bytes": (
        _ll, [ctypes.POINTER(SacDiscreteUpdate), _i]),
    "wdb_sac_discrete_critic_update_sampled": (
        _i, [_vp, ctypes.POINTER(SacDiscreteUpdate), ctypes.POINTER(ReplayWindows)]),
    "wdb_sac_discrete_actor_update_sampled_supported": (
        _i, [ctypes.POINTER(SacDiscreteUpdate), _i]),
    "wdb_sac_discrete_actor_update_sampled_workspace_bytes": (
        _ll, [ctypes.POINTER(SacDiscreteUpdate), _i]),
    "wdb_sac_discrete_actor_update_sampled": (
        _i, [_vp, ctypes.POINTER(SacDiscreteUpdate), ctypes.POINTER(ReplayWindows)]),
    "wdb_tqc_critic_update_sampled_supported": (_i, [ctypes.POINTER(TqcUpdate), _i]),
    "wdb_tqc_critic_update_sampled_workspace_bytes": (_ll, [ctypes.POINTER(TqcUpdate), _i]),
    "wdb_tqc_critic_update_sampled": (
        _i, [_vp, ctypes.POINTER(TqcUpdate), ctypes.POINTER(ReplayWindows)]),
    "wdb_tqc_actor_update_sampled_supported": (_i, [ctypes.POINTER(TqcUpdate), _i]),
    "wdb_tqc_actor_update_sampled_workspace_bytes": (_ll, [ctypes.POINTER(TqcUpdate), _i]),
    "wdb_tqc_actor_update_sampled": (
        _i, [_vp, ctypes.POINTER(TqcUpdate), ctypes.POINTER(ReplayWindows)]),
    "wdb_dueling_fold_supported": (_i, [ctypes.POINTER(DuelingHead)]),
    "wdb_dueling_unfold_grads_supported": (_i, [ctypes.POINTER(DuelingHead)]),
    "wdb_dueling_fold": (
        _i, [_vp, ctypes.POINTER(DuelingHead), ctypes.POINTER(DuelingHead)]),
    "wdb_dueling_unfold_grads": (_i, [_vp, ctypes.POINTER(DuelingHead)]),
    "wdb_noisy_supported": (_i, [ctypes.POINTER(NoisyNet)]),
    "wdb_noisy_draw": (_i, [_vp, ctypes.POINTER(NoisyNet), _ull, _i, _ull, _i, _i]),
    "wdb_noisy_materialize": (
        _i, [_vp, ctypes.POINTER(NoisyNet), ctypes.POINTER(NoisyNet), _ull, _ull]),
    "wdb_noisy_grads": (_i, [_vp, ctypes.POINTER(NoisyNet)]),
    "wdb_replay_sample_windows": (_i, [_vp, _vp, _i, _ull, _ull, _i, _i, _i, _i, _i]),
    "wdb_per_nodes": (_ll, [_ll]),
    "wdb_per_levels": (_i, [_ll]),
    "wdb_per_admit": (_i, [_vp, ctypes.POINTER(PerStore), _i, _i, _i, _i]),
    "wdb_per_sample_windows": (
        _i, [_vp, ctypes.POINTER(PerStore), _vp, _vp, _vp, _i, _ull, _ull, _vp]),
    "wdb_per_set_priorities": (
        _i, [_vp, ctypes.POINTER(PerStore), _vp, _i, _vp, _vp, _i, _i]),
    "wdb_single_agent_rollout_supported": (_i, [_i, ctypes.POINTER(_i)]),
    "wdb_single_agent_rollout_categorical_supported": (_i, [_i, ctypes.POINTER(_i), _i]),
    "wdb_single_agent_rollout_noisy_supported": (_i, [_i, ctypes.POINTER(_i)]),
    "wdb_single_agent_rollout": (_i, [_vp, ctypes.POINTER(SaRollout)]),
    "wdb_obs_moments_scratch_doubles": (_ll, [_ll, _i]),
    "wdb_obs_moments_update": (_i, [_vp, _vp, _ll, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "wdb_obs_moments_batch": (_i, [_vp, _vp, _ll, _i, _vp, _vp]),
    "wdb_obs_moments_merge": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "wdb_obs_normalize": (_i, [_vp, _vp, _vp, _ll, _i, _vp, _vp, _f]),
    "wdb_discounted_return_scan": (_i, [_vp, _vp, _vp, _i, _i, _i, _f, _vp, _vp]),
    "wdb_mountain_car_step": (
        _i, [_vp, _i, _vp, _vp, _vp, _vp, _vp] + [_f] * 7 + [_vp, _i]),
    "wdb_continuous_mountain_car_step": (
        _i, [_vp, _i, _vp, _vp, _vp, _vp, _vp] + [_f] * 8 + [_vp, _i]),
    "wdb_pendulum_step": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i]),
    "wdb_acrobot_step": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i]),
    "wdb_gru_forward_bytes": (_ll, [_i, _i, _i, _i, _i, _i, _i, _i]),
    "wdb_gru_policy_forward": (_i, [_vp, ctypes.POINTER(GruForward)]),
    "wdb_recurrent_reset_done": (_i, [_vp, ctypes.POINTER(RecurrentReset)]),
    "wdb_cartpole_step": (
        _i,
        [_vp, _i, _vp, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _f, _f, _f, _f, _f, _vp, _i],
    ),
}

_lib = None


def exported_symbols():
    """Names every build must export (== the functions include/wdb200.h declares)."""
    return sorted(_SIGNATURES)


def load():
    """dlopen libwdb200.so and type its entry points.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -m warp_drive_b200.build` "
            "(or __graft_entry__.build()).  warp_drive_b200 has no CPU fallback."
        )
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the build lost a symbol
        fn.restype = restype
        fn.argtypes = argtypes
    assert lib.wdb_abi_version() == 1
    _lib = lib
    # A/B switches for whole test / bench runs: WDB_OPTIONS="tc_variant=2,tc_v2_threads=224"
    for item in filter(None, os.environ.get("WDB_OPTIONS", "").split(",")):
        key, _, val = item.partition("=")
        rc = lib.wdb_set_option(key.strip().encode(), int(val))
        if rc != 0:
            raise RuntimeError(f"WDB_OPTIONS: wdb_set_option({key!r}, {val}) failed ({rc})")
    return lib


def check(err, what=""):
    if err != 0:
        msg = load().wdb_error_string(err).decode()
        raise RuntimeError(f"libwdb200 {what} failed: cudaError {err} ({msg})")


def ptr(t):
    """Device pointer of a torch CUDA tensor / DeviceArray handle (None -> NULL)."""
    if t is None:
        return None
    if hasattr(t, "tensor"):
        t = t.tensor
    if torch.is_tensor(t):
        if not t.is_cuda:
            raise RuntimeError(
                "libwdb200 kernels need CUDA tensors; got a CPU tensor "
                "(warp_drive_b200 has no CPU fallback on the kernel path)"
            )
        if not t.is_contiguous():
            raise RuntimeError("libwdb200 kernels need C-contiguous tensors")
        return t.data_ptr()
    if hasattr(t, "gpudata"):  # pycuda-style pointer holder
        return int(t.gpudata)
    if hasattr(t, "data_ptr"):
        return int(t.data_ptr())
    if isinstance(t, int):
        return t
    raise TypeError(f"cannot take a device pointer of {type(t)}")


def stream_ptr(stream=None):
    """cudaStream_t of torch's current stream, so launches order with torch work."""
    if stream is None:
        stream = torch.cuda.current_stream()
    return stream.cuda_stream


def launch_count():
    return int(load().wdb_launch_count())
