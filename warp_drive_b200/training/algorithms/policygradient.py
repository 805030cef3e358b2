"""A2C and PPO objectives for the on-policy update that consumes the rollout batch.

Same mathematics as the reference (warp_drive/training/algorithms/policygradient/
a2c.py:40-194, ppo.py:42-204): bootstrapped discounted returns computed backwards in time
with done masking, optional per-timestep normalisation of returns / advantages over
(env, agent), categorical log-prob + entropy over every action head, MSE value loss.  A
diagonal Gaussian policy (FullyConnectedGaussian: per-row mean, state-independent log_std)
takes the Normal log-prob and entropy summed over the action dimensions instead.
The backward-time recursion runs as ONE kernel (wdb_discounted_returns) instead of
~6 elementwise launches per timestep.

PPO as people use it -- several epochs over shuffled minibatches, the ratio taken against the
policy that generated the batch, GAE(lambda) advantages -- is opt-in per policy (`num_epochs`,
`num_mini_batches`, `gae_lambda`; no reference counterpart): `prepare_batch` runs once per
training batch, `minibatch_loss` once per optimizer step.
"""
import ctypes

import torch
from torch import nn
from torch.distributions import Categorical, Normal

from warp_drive_b200.training.algorithms.fused_loss import (
    fused_gaussian_pg_loss, fused_gaussian_pg_loss_supported, fused_log_prob, fused_pg_loss,
    fused_pg_loss_supported, fused_ppo_loss, fused_ppo_loss_supported)
from warp_drive_b200.training.utils.param_scheduler import ParamScheduler

_EPSILON = 1e-10


def discounted_returns(rewards, done_flags, values, gamma):
    """returns[T-1] = done*r + (1-done)*V ; returns[t] = r[t] + (1-done[t])*gamma*returns[t+1]
    (a2c.py:80-93).  rewards/values [T, E, Np] float32, done_flags [T, E] int."""
    if rewards.is_cuda:
        from warp_drive_b200 import lib as _lib

        rewards = rewards.contiguous()
        values = values.contiguous().float()
        done = (done_flags > 0).to(torch.int32).contiguous()
        out = torch.empty_like(rewards)
        T, E, Np = rewards.shape
        _lib.check(_lib.load().wdb_discounted_returns(
            _lib.stream_ptr(), _lib.ptr(rewards), _lib.ptr(done), _lib.ptr(values),
            _lib.ptr(out), T, E, Np, float(gamma)), "discounted_returns")
        return out
    # host tensors (unit tests of the loss math)
    done = (done_flags > 0).to(rewards.dtype)[:, :, None]
    out = torch.zeros_like(rewards)
    out[-1] = done[-1] * rewards[-1] + (1 - done[-1]) * values[-1]
    for t in range(rewards.shape[0] - 2, -1, -1):
        out[t] = rewards[t] + (1 - done[t]) * gamma * out[t + 1]
    return out


def gae(rewards, done_flags, values, gamma, lam):
    """(advantages, value_targets) of GAE(lambda), with d = done > 0:
    A[T-1] = d ? r - V : 0 ; A[t] = r + (d ? 0 : gamma V[t+1]) - V + (d ? 0 : gamma lam A[t+1]);
    value_targets = A + V (lam = 1: discounted_returns).  Shapes as discounted_returns."""
    if rewards.is_cuda:
        from warp_drive_b200 import lib as _lib

        rewards = rewards.contiguous().float()
        values = values.contiguous().float()
        done = (done_flags > 0).to(torch.int32).contiguous()
        adv, vt = torch.empty_like(rewards), torch.empty_like(rewards)
        G = _lib.GaeArgs()
        G.T, G.n_envs, G.n_agents = rewards.shape
        G.rewards, G.values, G.done = _lib.ptr(rewards), _lib.ptr(values), _lib.ptr(done)
        G.gamma, G.gae_lambda = float(gamma), float(lam)
        G.advantages, G.value_targets = _lib.ptr(adv), _lib.ptr(vt)
        _lib.check(_lib.load().wdb_gae(_lib.stream_ptr(), ctypes.byref(G)), "gae")
        return adv, vt
    done = (done_flags > 0)[:, :, None]
    adv = torch.zeros_like(rewards)
    adv[-1] = torch.where(done[-1], rewards[-1] - values[-1], torch.zeros_like(rewards[-1]))
    for t in range(rewards.shape[0] - 2, -1, -1):
        boot = torch.where(done[t], torch.zeros_like(values[t]), gamma * values[t + 1])
        carry = torch.where(done[t], torch.zeros_like(adv[t]), gamma * lam * adv[t + 1])
        adv[t] = rewards[t] + boot - values[t] + carry
    return adv, adv + values


def _categorical_terms(probs, actions):
    """Summed over the heads: (log-prob of the taken actions, entropy), torch Categorical."""
    log_prob, entropy = 0.0, 0.0
    for k, p in enumerate(probs):
        dist = Categorical(p)
        log_prob = log_prob + dist.log_prob(actions[..., k])
        entropy = entropy + dist.entropy()
    return log_prob, entropy


def _gaussian_terms(mean, log_std, actions):
    dist = Normal(mean, log_std.exp())
    return dist.log_prob(actions).sum(-1), dist.entropy().sum(-1)


def _training_forward(model, obs, action_mask=None):
    """The forward the minibatch steps run -- the fused training node (models/fused_mlp_train.py)
    where it applies, the module otherwise -- so that the old log-probs of prepare_batch and the
    log-probs of the steps come from the same arithmetic.  Under torch.no_grad the fused node
    runs its forward without recording a graph (FullyConnected.forward takes its plain torch
    path there)."""
    if getattr(model, "use_fused_train_forward", False) and obs.is_cuda:
        from warp_drive_b200.training.models import fused_mlp_train

        if fused_mlp_train.supported(model, obs, action_mask):
            return fused_mlp_train.fused_train_forward(model, obs, action_mask)
    kw = {} if action_mask is None else {"action_mask": action_mask}
    return model(obs=obs, **kw)


def ppo_minibatch_loss(probs, values, actions, advantages, value_targets, old_log_prob, ppo,
                       clip_param, vf_coeff, entropy_coeff, log_std=None):
    """The minibatch loss of wdb_ppo_loss_and_grads / wdb_ppo_gaussian_loss_and_grads as a
    float32 torch expression (the fall-back for shapes the kernels refuse, and the reference
    the GPU tests compare them with).  Every argument holds the minibatch's B rows: probs a
    list of [B, A_k] (or [mean [B, A]] with log_std [A]), values / advantages / value_targets /
    old_log_prob [B], actions [B, n_heads] (or float [B, A]).  Returns (loss, float64 sums [5]:
    policy, value, entropy, KL, clip count)."""
    if log_std is not None:
        log_prob, entropy = _gaussian_terms(probs[0], log_std, actions)
    else:
        log_prob, entropy = _categorical_terms(probs, actions.long())
    ratio = torch.exp(log_prob - old_log_prob)
    clip_param = float(clip_param or 0.0)
    if ppo:
        clipped = torch.clamp(ratio, 1.0 - clip_param, 1.0 + clip_param)
        terms = -torch.minimum(ratio * advantages, clipped * advantages)
    else:
        terms = -log_prob * advantages
    sq = (values - value_targets) ** 2
    loss = terms.mean() + vf_coeff * sq.mean() - entropy_coeff * entropy.mean()
    with torch.no_grad():
        sums = torch.stack([
            terms.double().sum(), sq.double().sum(), entropy.double().sum(),
            (old_log_prob - log_prob).double().sum(),
            ((ratio - 1.0).abs() > clip_param).double().sum()])
    return loss, sums


class PPOBatch:
    """One training batch flattened to R = T * E * Np rows for the minibatch loop: the inputs
    of the training forward (obs [R, F], mask [R, sum A_k] or None), the flat actions
    (int32 [R, n_heads] or float [R, A]), and what prepare_batch computed at the rollout's
    parameters (advantages -- normalised if asked --, value_targets, old_log_prob [R]),
    plus the [T, E, Np] tensors the metrics report."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


class _PolicyGradient:
    def __init__(self, discount_factor_gamma=1.0, normalize_advantage=False,
                 normalize_return=False, vf_loss_coeff=0.01, entropy_coeff=0.01,
                 clip_param=None, num_epochs=1, num_mini_batches=1, gae_lambda=None):
        assert 0 <= discount_factor_gamma <= 1
        self.discount_factor_gamma = discount_factor_gamma
        self.normalize_advantage = normalize_advantage
        self.normalize_return = normalize_return
        self.vf_loss_coeff_schedule = ParamScheduler(vf_loss_coeff)
        self.entropy_coeff_schedule = ParamScheduler(entropy_coeff)
        self.clip_param = clip_param
        # several epochs over shuffled minibatches and / or GAE: prepare_batch + minibatch_loss
        # instead of compute_loss_and_metrics
        self.num_epochs, self.num_mini_batches = int(num_epochs), int(num_mini_batches)
        self.gae_lambda = None if gae_lambda is None else float(gae_lambda)
        if self.num_epochs < 1 or self.num_mini_batches < 1:
            raise ValueError("num_epochs and num_mini_batches must be at least 1")
        if self.gae_lambda is not None and not 0.0 <= self.gae_lambda <= 1.0:
            raise ValueError(f"gae_lambda must lie in [0, 1], got {self.gae_lambda}")
        self.minibatch_path = (self.num_epochs > 1 or self.num_mini_batches > 1
                               or self.gae_lambda is not None)
        if self.minibatch_path and clip_param is None and (
                self.num_epochs > 1 or self.num_mini_batches > 1):
            raise ValueError("A2C takes one gradient step per batch: num_epochs and "
                             "num_mini_batches > 1 need PPO (A2C may set gae_lambda)")
        if self.minibatch_path and normalize_return:
            raise ValueError("normalize_return is not supported with num_epochs, "
                             "num_mini_batches or gae_lambda")
        # CUDA: returns / advantages / log-prob / entropy / loss AND the gradient with respect
        # to the model outputs in one kernel (fused_loss.py); the torch expression below stays
        # as the float32 reference the GPU tests compare against (and for the normalised /
        # env-subsampled variants)
        self.use_fused_loss = True

    @staticmethod
    def _normalize(x):
        return (x - x.mean(dim=(1, 2), keepdim=True)) / (x.std(dim=(1, 2), keepdim=True) + _EPSILON)

    def _policy_loss(self, log_prob, advantages):
        raise NotImplementedError

    def compute_loss_and_metrics(self, timestep=None, actions_batch=None, rewards_batch=None,
                                 done_flags_batch=None, action_probabilities_batch=None,
                                 value_functions_batch=None, perform_logging=False,
                                 negative_positive_ratio=-1, log_std=None):
        """log_std [A] given: a Gaussian policy, action_probabilities_batch = [mean
        [T, E, Np, A]] and actions_batch the float actions [T, E, Np, A]."""
        assert timestep is not None
        n_pos = n_neg = None
        if negative_positive_ratio > 0:
            # sparse-goal envs (MountainCar: done == 2 marks "goal reached",
            # mountain_car_step_numba.py:66-70): keep every env that reached the goal in this
            # batch and at most ratio x as many of the others (a2c.py:58-69, 196-220)
            keep, n_pos, n_neg = self._sample_positive_negative_env_ids(
                done_flags_batch, negative_positive_ratio)
            if keep is not None:
                actions_batch = actions_batch[:, keep]
                rewards_batch = rewards_batch[:, keep]
                done_flags_batch = done_flags_batch[:, keep]
                action_probabilities_batch = [p[:, keep] for p in action_probabilities_batch]
                value_functions_batch = value_functions_batch[:, keep]
        if (self.use_fused_loss and value_functions_batch.is_cuda and n_pos is None
                and not self.normalize_return and not self.normalize_advantage
                and (fused_pg_loss_supported(action_probabilities_batch) if log_std is None
                     else fused_gaussian_pg_loss_supported(action_probabilities_batch[0]))):
            return self._fused_loss_and_metrics(
                timestep, actions_batch, rewards_batch, done_flags_batch,
                action_probabilities_batch, value_functions_batch, perform_logging, log_std)
        values_detached = value_functions_batch.detach()
        returns = discounted_returns(rewards_batch, done_flags_batch, values_detached,
                                     self.discount_factor_gamma)
        norm_returns = self._normalize(returns) if self.normalize_return else returns
        vf_loss = nn.functional.mse_loss(value_functions_batch, norm_returns)
        advantages = norm_returns - values_detached
        norm_adv = self._normalize(advantages) if self.normalize_advantage else advantages

        log_prob, mean_entropy = 0.0, 0.0
        if log_std is not None:
            dist = Normal(action_probabilities_batch[0], log_std.exp())
            mean_entropy = dist.entropy().sum(-1).mean()
            log_prob = dist.log_prob(actions_batch).sum(-1)
        else:
            for k in range(actions_batch.shape[-1]):
                dist = Categorical(action_probabilities_batch[k])
                mean_entropy = mean_entropy + dist.entropy().mean()
                log_prob = log_prob + dist.log_prob(actions_batch[..., k])
        policy_loss = self._policy_loss(log_prob, norm_adv)
        vf_c = self.vf_loss_coeff_schedule.get_param_value(timestep)
        ent_c = self.entropy_coeff_schedule.get_param_value(timestep)
        loss = policy_loss + vf_c * vf_loss - ent_c * mean_entropy
        metrics = {}
        if perform_logging:
            var_expl = 1 - norm_adv.detach().var() / (norm_returns.detach().var() + _EPSILON)
            metrics = {
                "VF loss coefficient": vf_c, "Entropy coefficient": ent_c,
                "Total loss": loss.item(), "Policy loss": policy_loss.item(),
                "Value function loss": vf_loss.item(),
                "Mean rewards": rewards_batch.mean().item(),
                "Max. rewards": rewards_batch.max().item(),
                "Min. rewards": rewards_batch.min().item(),
                "Mean value function": value_functions_batch.mean().item(),
                "Mean advantages": advantages.mean().item(),
                "Mean (norm.) advantages": norm_adv.mean().item(),
                "Mean (discounted) returns": returns.mean().item(),
                "Mean normalized returns": norm_returns.mean().item(),
                "Mean entropy": mean_entropy.item(),
                "Variance explained by the value function": max(-1.0, var_expl.item()),
            }
            a = actions_batch.float()
            for k in range(a.shape[-1]):
                metrics[f"Std. of action_{k} over agents"] = a[..., k].std(dim=2).mean().item()
                metrics[f"Std. of action_{k} over envs"] = a[..., k].std(dim=1).mean().item()
                metrics[f"Std. of action_{k} over time"] = a[..., k].std(dim=0).mean().item()
            if n_pos is not None:
                metrics["Num of Positive Sampled Envs"] = n_pos
                metrics["Num of Negative Sampled Envs"] = n_neg
        return loss, metrics

    def _fused_loss_and_metrics(self, timestep, actions_batch, rewards_batch, done_flags_batch,
                                action_probabilities_batch, value_functions_batch,
                                perform_logging, log_std=None):
        vf_c = self.vf_loss_coeff_schedule.get_param_value(timestep)
        ent_c = self.entropy_coeff_schedule.get_param_value(timestep)
        if log_std is None:
            loss, parts, returns = fused_pg_loss(
                value_functions_batch, list(action_probabilities_batch), actions_batch,
                rewards_batch, done_flags_batch, self.discount_factor_gamma, vf_c, ent_c,
                ppo=self.clip_param is not None, want_returns=perform_logging)
        else:
            loss, parts, returns = fused_gaussian_pg_loss(
                value_functions_batch, action_probabilities_batch[0], log_std, actions_batch,
                rewards_batch, done_flags_batch, self.discount_factor_gamma, vf_c, ent_c,
                ppo=self.clip_param is not None, want_returns=perform_logging)
        metrics = {}
        if perform_logging:
            values = value_functions_batch.detach()
            advantages = returns - values
            var_expl = 1 - advantages.var() / (returns.var() + _EPSILON)
            policy_loss, vf_loss, mean_entropy = (float(x) for x in parts)
            metrics = {
                "VF loss coefficient": vf_c, "Entropy coefficient": ent_c,
                "Total loss": loss.item(), "Policy loss": policy_loss,
                "Value function loss": vf_loss,
                "Mean rewards": rewards_batch.mean().item(),
                "Max. rewards": rewards_batch.max().item(),
                "Min. rewards": rewards_batch.min().item(),
                "Mean value function": values.mean().item(),
                "Mean advantages": advantages.mean().item(),
                "Mean (norm.) advantages": advantages.mean().item(),
                "Mean (discounted) returns": returns.mean().item(),
                "Mean normalized returns": returns.mean().item(),
                "Mean entropy": mean_entropy,
                "Variance explained by the value function": max(-1.0, var_expl.item()),
            }
            a = actions_batch.float()
            for k in range(a.shape[-1]):
                metrics[f"Std. of action_{k} over agents"] = a[..., k].std(dim=2).mean().item()
                metrics[f"Std. of action_{k} over envs"] = a[..., k].std(dim=1).mean().item()
                metrics[f"Std. of action_{k} over time"] = a[..., k].std(dim=0).mean().item()
        return loss, metrics

    # ---- several epochs over shuffled minibatches
    def prepare_batch(self, model, obs, actions, rewards, done_flags, action_mask=None,
                      hidden_start=None):
        """Once per training batch, at the parameters the rollout used: one forward of the
        training network without gradients (each timestep under its own action mask), the
        values for GAE and old_log_prob of every row by the loss kernel's own formula, then
        advantages / value targets (gae_lambda absent: the discounted returns) and the
        optional per-timestep advantage normalisation over (env, agent).  obs [T, E, Np, F],
        actions [T, E, Np, n_heads] (float [T, E, Np, A] for a Gaussian policy), rewards
        [T, E, Np], done_flags [T, E].  A recurrent model (FullyConnectedGRU) runs
        forward_sequence from hidden_start [E, Np, H], and its minibatches are sets of whole
        sequences (one (env, agent) pair over the T steps) instead of rows."""
        T, E, Np = rewards.shape
        R = T * E * Np
        recurrent = bool(getattr(model, "is_recurrent", False))
        if R >= 2 ** 31:
            raise ValueError(f"a training batch of {R} rows (T x E x agents) is too large for "
                             "the minibatch update: it indexes rows with int32")
        if recurrent and self.num_mini_batches > E * Np:
            raise ValueError(f"num_mini_batches = {self.num_mini_batches} exceeds the {E * Np} "
                             "sequences (E x agents) of a training batch: a minibatch of a "
                             "recurrent policy would be empty")
        if self.num_mini_batches > R:
            raise ValueError(f"num_mini_batches = {self.num_mini_batches} exceeds the {R} rows "
                             "(T x E x agents) of a training batch: a minibatch would be empty")
        log_std = model.log_std if getattr(model, "is_gaussian", False) else None
        seq = None
        if recurrent:
            assert hidden_start is not None and action_mask is None
            seq = dict(obs=obs.reshape(T, E * Np, -1), h0=hidden_start.reshape(E * Np, -1),
                       done=done_flags, T=T, Np=Np)
        obs = obs.reshape(R, -1)
        if action_mask is not None:
            action_mask = action_mask.reshape(R, -1).float()
        if log_std is not None:
            flat_actions = actions.reshape(R, -1).float().contiguous()
        else:
            flat_actions = actions.reshape(R, -1).to(torch.int32).contiguous()
        with torch.no_grad():
            if recurrent:
                probs, values = model.forward_sequence(
                    seq["obs"].view(T, E, Np, -1), hidden_start, done_flags)
                probs = [p.reshape(R, -1) for p in probs]
            else:
                probs, values = _training_forward(model, obs, action_mask)
            values = values.reshape(T, E, Np)
            if self.use_fused_loss and obs.is_cuda and fused_ppo_loss_supported(probs, log_std):
                old_log_prob = fused_log_prob(probs, flat_actions, log_std)
            elif log_std is not None:
                old_log_prob = _gaussian_terms(probs[0], log_std, flat_actions)[0]
            else:
                old_log_prob = _categorical_terms(probs, flat_actions.long())[0]
            if self.gae_lambda is None:
                value_targets = discounted_returns(rewards, done_flags, values,
                                                   self.discount_factor_gamma)
                advantages = value_targets - values
            else:
                advantages, value_targets = gae(rewards, done_flags, values,
                                                self.discount_factor_gamma, self.gae_lambda)
            norm_adv = self._normalize(advantages) if self.normalize_advantage else advantages
        return PPOBatch(
            R=R, units=E * Np if recurrent else R, rows_per_unit=T if recurrent else 1, seq=seq,
            obs=obs, mask=action_mask, actions=flat_actions, log_std=log_std,
            advantages=norm_adv.reshape(R).contiguous(),
            value_targets=value_targets.reshape(R).contiguous(),
            old_log_prob=old_log_prob.reshape(R).float().contiguous(),
            rewards=rewards, values=values, raw_advantages=advantages, norm_advantages=norm_adv,
            returns=value_targets, actions_batch=actions)

    def minibatch_loss(self, model, batch, rows, timestep):
        """The loss of one minibatch (rows: int32 [B] into the batch's R rows; for a recurrent
        model, `units` of the batch's sequences: see sequence_rows) with the training forward
        under autograd; returns (loss, float64 sums [5] on the device)."""
        if batch.seq is not None:
            probs, values, rows = self._sequence_forward(model, batch, rows)
        else:
            obs = batch.obs.index_select(0, rows)
            kw = {} if batch.mask is None else {"action_mask": batch.mask.index_select(0, rows)}
            probs, values = model(obs=obs, **kw)
        vf_c = self.vf_loss_coeff_schedule.get_param_value(timestep)
        ent_c = self.entropy_coeff_schedule.get_param_value(timestep)
        ppo = self.clip_param is not None
        clip = self.clip_param if ppo else 0.0
        if self.use_fused_loss and values.is_cuda and fused_ppo_loss_supported(probs,
                                                                               batch.log_std):
            return fused_ppo_loss(values, list(probs), rows, batch, ppo, clip, vf_c, ent_c,
                                  log_std=batch.log_std)
        idx = rows.long()
        return ppo_minibatch_loss(
            list(probs), values, batch.actions[idx], batch.advantages[idx],
            batch.value_targets[idx], batch.old_log_prob[idx], ppo, clip, vf_c, ent_c,
            log_std=batch.log_std)

    @staticmethod
    def sequence_rows(seqs, T, S):
        """The flat batch rows of sequences `seqs` (int [B_s] of S = E x Np): t * S + s, in
        (t, chunk) order -- the row order of forward_sequence over [T, B_s].  int32 [T * B_s]."""
        t = torch.arange(T, dtype=torch.int64, device=seqs.device)[:, None] * S
        return (t + seqs.to(torch.int64)[None, :]).reshape(-1).to(torch.int32)

    @staticmethod
    def _sequence_forward(model, batch, seqs):
        """forward_sequence over the sequences `seqs` of a recurrent batch, from their start
        states: ([probs per head] [T * B_s, A_k], values [T * B_s], rows int32 [T * B_s])."""
        sq = batch.seq
        T, S = sq["obs"].shape[0], sq["obs"].shape[1]
        idx = seqs.long()
        obs = sq["obs"].index_select(1, idx)[:, :, None]             # [T, B_s, 1, F]
        h0 = sq["h0"].index_select(0, idx)[:, None]                  # [B_s, 1, H]
        done = sq["done"].index_select(1, torch.div(idx, sq["Np"], rounding_mode="floor"))
        probs, values = model.forward_sequence(obs, h0, done)
        B = T * idx.numel()
        return ([p.reshape(B, -1) for p in probs], values.reshape(B),
                _PolicyGradient.sequence_rows(seqs, T, S))

    def minibatch_metrics(self, batch, mean_sums, timestep):
        """The metrics of a logging iteration: the loss terms from `mean_sums` (the per-step
        sums over B, averaged over the iteration's steps), the rest from the batch."""
        vf_c = self.vf_loss_coeff_schedule.get_param_value(timestep)
        ent_c = self.entropy_coeff_schedule.get_param_value(timestep)
        policy_loss, vf_loss, mean_entropy, kl, clip_frac = (float(x) for x in mean_sums.cpu())
        rewards, adv, ret = batch.rewards, batch.raw_advantages, batch.returns
        var_expl = 1 - adv.var() / (ret.var() + _EPSILON)
        metrics = {
            "VF loss coefficient": vf_c, "Entropy coefficient": ent_c,
            "Total loss": policy_loss + vf_c * vf_loss - ent_c * mean_entropy,
            "Policy loss": policy_loss, "Value function loss": vf_loss,
            "Mean rewards": rewards.mean().item(), "Max. rewards": rewards.max().item(),
            "Min. rewards": rewards.min().item(),
            "Mean value function": batch.values.mean().item(),
            "Mean advantages": adv.mean().item(),
            "Mean (norm.) advantages": batch.norm_advantages.mean().item(),
            "Mean (discounted) returns": ret.mean().item(),
            "Mean normalized returns": ret.mean().item(),
            "Mean entropy": mean_entropy,
            "Variance explained by the value function": max(-1.0, var_expl.item()),
            "Approx. KL": kl,
        }
        if self.clip_param is not None:
            metrics["Clip fraction"] = clip_frac
        a = batch.actions_batch.float()
        for k in range(a.shape[-1]):
            metrics[f"Std. of action_{k} over agents"] = a[..., k].std(dim=2).mean().item()
            metrics[f"Std. of action_{k} over envs"] = a[..., k].std(dim=1).mean().item()
            metrics[f"Std. of action_{k} over time"] = a[..., k].std(dim=0).mean().item()
        return metrics

    @staticmethod
    def _sample_positive_negative_env_ids(done_flags_batch, negative_positive_ratio):
        """(env index tensor or None when nothing is dropped, #positive, #negative kept)."""
        positives = (done_flags_batch == 2).any(dim=0)
        pos_ids = positives.nonzero(as_tuple=True)[0]
        neg_ids = (~positives).nonzero(as_tuple=True)[0]
        n_pos, total = int(pos_ids.numel()), int(done_flags_batch.shape[1])
        n_neg = int(n_pos * negative_positive_ratio)
        if n_pos == 0 or n_pos + n_neg >= total:
            return None, n_pos, int(neg_ids.numel())
        pick = torch.randperm(int(neg_ids.numel()), device=neg_ids.device)[:n_neg]
        return torch.cat((pos_ids, neg_ids[pick])), n_pos, n_neg


class A2C(_PolicyGradient):
    """Advantage actor-critic (a2c.py:123-130)."""

    def _policy_loss(self, log_prob, advantages):
        return (-log_prob * advantages).mean()


class PPO(_PolicyGradient):
    """Clipped-surrogate PPO exactly as the reference states it (ppo.py:127-136): the
    'old' log-prob is the detached current one (single epoch over the fresh batch).  With
    num_epochs / num_mini_batches / gae_lambda set, the ratio is taken against the rollout
    policy's log-prob instead (prepare_batch, minibatch_loss)."""

    def __init__(self, clip_param=0.1, **kw):
        super().__init__(clip_param=clip_param, **kw)
        assert 0 <= clip_param <= 1

    def _policy_loss(self, log_prob, advantages):
        ratio = torch.exp(log_prob - log_prob.detach())
        clipped = torch.clamp(ratio, 1.0 - self.clip_param, 1.0 + self.clip_param)
        return -torch.minimum(ratio * advantages, clipped * advantages).mean()
