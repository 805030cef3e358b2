#!/usr/bin/env python
"""PPO over several epochs of shuffled minibatches, in one process, rounds alternated on the
same trainer and buffers:
  * workloads: single_pendulum_ppo.yaml (Pendulum, 10 000 envs, T = 10, [64, 64] Gaussian
    policy, one-launch rollout) and the config-2 TagContinuous sizes (tag_continuous.yaml with
    5 taggers + 100 runners, 100 envs, T = 250, [256, 256] policies, fused step), both PPO;
  * update variants: the existing single-step update, 1 x 1 with GAE(0.95) on the minibatch
    path, and 4 epochs x 4 minibatches with GAE;
  * per variant: ms of the rollout, of the batch preparation and of the minibatch steps of one
    training iteration, and libwdb200 launches per minibatch step (lib.launch_count);
  * on one minibatch: the fused loss forward (wdb_ppo_loss_and_grads / the Gaussian kernel)
    against the torch expression of the same loss, forward + backward each, with the bytes the
    kernel must move (from the shapes) over 3.35 TB/s;
median and min-max over the rounds, and the GPU name and power limit.  Prints one JSON object."""
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from warp_drive_b200 import lib as wlib  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
VARIANTS = {"existing": None, "gae_1x1": (1, 1), "gae_4x4": (4, 4)}


def gpu_info():
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
             f"--id={torch.cuda.current_device()}"],
            capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    return name, power


def build_pendulum(basedir):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.single_agent.classic_control import CUDAClassicControlPendulumEnv
    from warp_drive_b200.training.trainer import Trainer, load_run_config

    cfg = load_run_config("single_pendulum_ppo")
    cfg["trainer"]["seed"] = 7
    cfg["saving"].update(basedir=basedir, metrics_log_freq=10 ** 9)
    E = cfg["trainer"]["num_envs"]
    w = EnvWrapper(CUDAClassicControlPendulumEnv(**cfg["env"]), num_envs=E, env_backend="numba")
    tr = Trainer(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={"shared": [0]},
                 results_dir="pendulum", verbose=False)
    assert tr.engine.sa is not None and tr.engine.sa.gaussian
    return tr, f"single_pendulum_ppo.yaml: Pendulum, {E} envs, T = {tr.engine.T}, PPO"


def build_tag_continuous(basedir):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.tag_continuous import TagContinuous
    from warp_drive_b200.training.trainer import Trainer, load_run_config

    cfg = load_run_config("tag_continuous")
    cfg["env"].update(num_taggers=5, num_runners=100)
    cfg["trainer"]["seed"] = 7
    cfg["saving"].update(basedir=basedir, metrics_log_freq=10 ** 9)
    for p in cfg["policy"].values():
        p["algorithm"] = "PPO"
    env = TagContinuous(**cfg["env"])
    E = cfg["trainer"]["num_envs"]
    w = EnvWrapper(env, num_envs=E, env_backend="pycuda")
    pm = {"runner": sorted(env.runners), "tagger": sorted(env.taggers)}
    tr = Trainer(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map=pm, results_dir="tc",
                 verbose=False)
    assert tr.engine.fused is not None
    return tr, (f"tag_continuous config 2: {E} envs x (5 taggers + 100 runners), "
                f"T = {tr.engine.T}, [256, 256], PPO")


def set_variant(tr, steps):
    for p in tr.policies_to_train:
        t = tr.trainers[p]
        t.minibatch_path = steps is not None
        t.num_epochs, t.num_mini_batches = steps or (1, 1)
        t.gae_lambda = 0.95 if steps is not None else None
    tr._minibatch_steps = None if steps is None else steps[0] * steps[1]


class PrepareTimer:
    """Wraps each policy objective's prepare_batch with CUDA events."""

    def __init__(self, tr):
        self.pairs = []
        for p in tr.policies_to_train:
            obj = tr.trainers[p]
            real = obj.prepare_batch

            def timed_prepare(*a, _real=real, **kw):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = _real(*a, **kw)
                e1.record()
                self.pairs.append((e0, e1))
                return out
            obj.prepare_batch = timed_prepare

    def take(self):
        ms = sum(a.elapsed_time(b) for a, b in self.pairs)
        self.pairs = []
        return ms


def one_iteration(tr, prep):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ev[0].record()
    tr._generate_rollout_batch()
    ev[1].record()
    tr._update_model_params(1)           # never a logging iteration
    ev[2].record()
    torch.cuda.synchronize()
    p = prep.take()
    return ev[0].elapsed_time(ev[1]), p, ev[1].elapsed_time(ev[2]) - p


def launches_per_step(tr):
    """libwdb200 launches of one minibatch step (forward, fused loss, backward, clip + Adam)."""
    dm = tr.cuda_envs.cuda_data_manager
    batches = {}
    for p in tr.policies_to_train:
        mask = f"action_mask_batch_{p}"
        batches[p] = tr.trainers[p].prepare_batch(
            tr.models[p], dm.data_on_device_via_torch(f"processed_observations_batch_{p}"),
            dm.data_on_device_via_torch(f"sampled_actions_batch_{p}"),
            dm.data_on_device_via_torch(f"rewards_batch_{p}"),
            dm.data_on_device_via_torch("done_flags_batch"),
            dm.data_on_device_via_torch(mask) if dm.is_data_on_device_via_torch(mask) else None)
    torch.cuda.synchronize()
    c0 = wlib.launch_count()
    for p in tr.policies_to_train:
        rows = torch.arange(batches[p].R // 4, dtype=torch.int32, device="cuda")
        loss, _ = tr.trainers[p].minibatch_loss(tr.models[p], batches[p], rows, 1)
        tr.optimizers[p].zero_grad()
        loss.backward()
    tr._optimizer_step(tr.policies_to_train, False)
    torch.cuda.synchronize()
    return wlib.launch_count() - c0, batches


def loss_compare(tr, batches, rounds):
    """Fused loss forward vs the torch expression (forward + backward) on a quarter-batch
    minibatch of the first policy, and the fused kernel's compulsory bytes."""
    from warp_drive_b200.training.algorithms.fused_loss import fused_ppo_loss
    from warp_drive_b200.training.algorithms.policygradient import ppo_minibatch_loss

    p = tr.policies_to_train[0]
    b, obj, model = batches[p], tr.trainers[p], tr.models[p]
    B = b.R // 4
    rows = torch.randperm(b.R, device="cuda")[:B].to(torch.int32)
    with torch.no_grad():
        probs, values = model(obs=b.obs.index_select(0, rows))
    probs = [x.detach().contiguous() for x in probs]
    values = values.detach().contiguous()
    log_std = b.log_std

    def fused():
        fused_ppo_loss(values, probs, rows, b, True, obj.clip_param, 0.5, 0.01, log_std=log_std)

    def torch_expr():
        P = [x.clone().requires_grad_() for x in probs]
        V = values.clone().requires_grad_()
        i = rows.long()
        loss, _ = ppo_minibatch_loss(P, V, b.actions[i], b.advantages[i], b.value_targets[i],
                                     b.old_log_prob[i], True, obj.clip_param, 0.5, 0.01,
                                     log_std=log_std)
        loss.backward()

    widths = [int(x.shape[-1]) for x in probs]
    H = len(widths)
    if log_std is None:
        reads = 4 * B * (sum(widths) * (2 if H > 1 else 1) + 1 + 1 + H + 3)
        writes = 4 * B * (sum(widths) + 1)
    else:
        A = widths[0]
        reads = 4 * B * (2 * A + 1 + 1 + 3)
        writes = 4 * B * (A + 1)
    out = {"policy": p, "rows": B, "kernel_bytes": reads + writes}
    for name, fn in (("fused_forward", fused), ("torch_forward_backward", torch_expr)):
        for _ in range(3):
            fn()
        samples = []
        for _ in range(rounds):
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(20):
                fn()
            e.record()
            torch.cuda.synchronize()
            samples.append(a.elapsed_time(e) / 20)
        out[f"{name}_ms"] = sorted(samples)[len(samples) // 2]
        out[f"{name}_ms_spread"] = [min(samples), max(samples)]
    out["fused_forward_bytes_over_3.35TBps_ms"] = 1e3 * out["kernel_bytes"] / HBM_BYTES_PER_S
    return out


def bench(tr, label, rounds):
    prep = PrepareTimer(tr)
    res = {"workload": label}
    for name, steps in VARIANTS.items():       # warm-up every shape
        set_variant(tr, steps)
        for _ in range(2):
            one_iteration(tr, prep)
    samples = {n: {"rollout": [], "prepare": [], "steps": []} for n in VARIANTS}
    for _ in range(rounds):                    # alternate the variants
        for name, steps in VARIANTS.items():
            set_variant(tr, steps)
            r, p, s = one_iteration(tr, prep)
            samples[name]["rollout"].append(r)
            samples[name]["prepare"].append(p)
            samples[name]["steps"].append(s)
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    for name, steps in VARIANTS.items():
        s = samples[name]
        res[name] = {k + "_ms": med(v) for k, v in s.items()}
        res[name].update({k + "_ms_spread": [min(v), max(v)] for k, v in s.items()})
        res[name]["optimizer_steps"] = 1 if steps is None else steps[0] * steps[1]
    set_variant(tr, (4, 4))
    n, batches = launches_per_step(tr)
    res["libwdb200_launches_per_minibatch_step"] = n
    res["minibatch_loss"] = loss_compare(tr, batches, rounds)
    return res


def main():
    rounds = int(os.environ.get("BENCH_ROUNDS", "5"))
    out = {}
    with tempfile.TemporaryDirectory() as basedir:
        for key, build in (("pendulum", build_pendulum), ("tag_continuous", build_tag_continuous)):
            tr, label = build(basedir)
            out[key] = bench(tr, label, rounds)
            del tr
            torch.cuda.empty_cache()
    out["gpu"], out["power_limit"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
