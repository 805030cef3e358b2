"""Running mean / variance normalization of a policy's observations (model keys
`normalize_observations` and `observation_clip`, FullyConnected and FullyConnectedGaussian).

The statistics live in the model as buffers, so checkpoints carry them: float64 `obs_count`,
`obs_mean` [F], `obs_m2` [F] and the float32 `obs_shift` [F], `obs_scale` [F] that every
forward reads.  They are updated in place (the CUDA-graph rollout and the one-launch kernel hold
their pointers) once per training iteration, after the last optimizer step, from that
rollout's raw observation batch; the rollout and the update of an iteration both see the
statistics of the iteration before.  Native code: csrc/wdb_obs_norm.cu.
"""
import ctypes
import math

import torch

from warp_drive_b200 import lib as _lib

DEFAULT_CLIP = 10.0


def obs_norm_settings(model_config, model_type):
    """(enabled, clip) of a model config, validated; `model_type` names the model in the
    messages."""
    on = model_config.get("normalize_observations", False)
    if not isinstance(on, bool):
        raise ValueError(f"{model_type}'s model.normalize_observations is true or false, got "
                         f"{on!r}")
    if "observation_clip" not in model_config:
        return on, DEFAULT_CLIP
    clip = model_config["observation_clip"]
    if not on:
        raise ValueError(f"{model_type}'s model.observation_clip needs "
                         f"model.normalize_observations: true, got observation_clip {clip!r} "
                         "without it")
    if (isinstance(clip, bool) or not isinstance(clip, (int, float)) or not math.isfinite(clip)
            or clip <= 0):
        raise ValueError(f"{model_type}'s model.observation_clip is a finite number > 0, got "
                         f"{clip!r}")
    return on, float(clip)


def refuse_obs_norm(config, trainer_name):
    """The replay trainers store observations and sample them long after: normalized under
    statistics that have since moved, they would no longer match.  Refuse the keys there."""
    def walk(d):
        if isinstance(d, dict):
            for k, v in d.items():
                if k in ("normalize_observations", "observation_clip") and v not in (None, False):
                    raise ValueError(f"{trainer_name} does not take model.{k}: observation "
                                     "normalization is for A2C / PPO (Trainer)")
                walk(v)

    for policy_config in config.get("policy", {}).values():
        walk(policy_config.get("model", {}))


def register_buffers(model, n_features):
    """The statistics of an F-wide observation: no samples, so the identity."""
    model.register_buffer("obs_count", torch.zeros((), dtype=torch.float64))
    model.register_buffer("obs_mean", torch.zeros(n_features, dtype=torch.float64))
    model.register_buffer("obs_m2", torch.zeros(n_features, dtype=torch.float64))
    model.register_buffer("obs_shift", torch.zeros(n_features, dtype=torch.float32))
    model.register_buffer("obs_scale", torch.ones(n_features, dtype=torch.float32))


def _rows(x, n_features, what):
    if x.dtype != torch.float32 or not x.is_cuda or x.shape[-1] != n_features:
        raise ValueError(f"{what}: a float32 CUDA batch [..., {n_features}] is normalized, got "
                         f"{x.dtype} {tuple(x.shape)} on {x.device}")
    if not x.is_contiguous():
        raise ValueError(f"{what}: the batch must be [rows, F] contiguous")
    return x.numel() // n_features


def normalize(model, obs):
    """clamp((obs - shift) * scale, -clip, clip) per feature: one wdb_obs_normalize launch into
    a new tensor (observations are not parameters: no backward)."""
    F = int(model.obs_shift.numel())
    obs = obs.detach()
    if not obs.is_contiguous():
        obs = obs.contiguous()
    rows = _rows(obs, F, "normalize_observations")
    out = torch.empty_like(obs)
    _lib.check(_lib.load().wdb_obs_normalize(
        _lib.stream_ptr(), _lib.ptr(obs), _lib.ptr(out), rows, F, _lib.ptr(model.obs_shift),
        _lib.ptr(model.obs_scale), ctypes.c_float(model.observation_clip)), "obs_normalize")
    return out


def _state(model, prefix):
    return [_lib.ptr(getattr(model, f"{prefix}_{n}"))
            for n in ("count", "mean", "m2", "shift", "scale")]


def _scratch(model, rows, F, prefix):
    n = int(_lib.load().wdb_obs_moments_scratch_doubles(rows, F))
    name, dev = f"_{prefix}_moments_scratch", getattr(model, f"{prefix}_mean").device
    buf = getattr(model, name, None)
    if buf is None or buf.numel() < n or buf.device != dev:
        buf = torch.empty(n, dtype=torch.float64, device=dev)
        setattr(model, name, buf)
    return buf


def update_moments(model, batch, num_devices=1, prefix="obs"):
    """Merge the raw batch [..., F] (for observations every row of the policy's [T, E, Np, F]
    batch) into the model's running statistics `{prefix}_count`, `_mean`, `_m2` and rewrite
    `{prefix}_shift` and `_scale`, in place, without a host wait.  Several GPUs: each rank's
    batch moments are all-gathered and merged in rank order, so every rank holds the same bits
    (one all-gather of 2F + 1 float64 per policy)."""
    F = int(getattr(model, f"{prefix}_shift").numel())
    rows = _rows(batch, F, f"the {prefix}_* statistics")
    L, s = _lib.load(), _lib.stream_ptr()
    scratch = _scratch(model, rows, F, prefix)
    if num_devices <= 1:
        _lib.check(L.wdb_obs_moments_update(s, _lib.ptr(batch), rows, F, _lib.ptr(scratch),
                                            *_state(model, prefix)), "obs_moments_update")
        return
    import torch.distributed as dist

    record = torch.empty(2 * F + 1, dtype=torch.float64, device=batch.device)
    _lib.check(L.wdb_obs_moments_batch(s, _lib.ptr(batch), rows, F, _lib.ptr(scratch),
                                       _lib.ptr(record)), "obs_moments_batch")
    gathered = torch.empty((num_devices, 2 * F + 1), dtype=torch.float64, device=batch.device)
    dist.all_gather_into_tensor(gathered, record)
    _lib.check(L.wdb_obs_moments_merge(_lib.stream_ptr(), _lib.ptr(gathered), num_devices, F,
                                       *_state(model, prefix)), "obs_moments_merge")
