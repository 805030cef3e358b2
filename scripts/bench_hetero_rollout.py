#!/usr/bin/env python
"""Heterogeneous agents on the generic rollout path: the example env
(tests/custom_env/hetero_env*) at 2000 envs x (1 planner + 100 workers), separate per-policy
placeholders, agent-last worker observations ([E, 2, 3, Nw]), T = 10, A2C.  Reports ms per
rollout timestep (CUDA graph), ms per training iteration (rollout + update), and the
observation gather of one timestep: the one wdb_gather_policy_fields launch against the same
step done with torch permute + indexing + cat (the way the reference's model code does it),
alternated in the same process, each timed as a CUDA graph of 50 back-to-back gathers so that
launch overhead is not counted; the gather's achieved bytes/s (bytes read + written) is put
against the H100 SXM's 3.35 TB/s.  Prints one JSON object with the GPU name and power limit;
writes only under a temporary directory."""
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "custom_env"))

import torch  # noqa: E402

E, NW, T, L = 2000, 100, 10, 10
REPS = 50
PEAK = 3.35e12


def build(basedir):
    from hetero_env import CUDAHeteroEnv

    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.training.trainer import Trainer, load_run_config
    from warp_drive_b200.utils.env_registrar import EnvironmentRegistrar

    reg = EnvironmentRegistrar()
    reg.add_cuda_env_src_path("HeteroEnv", os.path.join(
        ROOT, "tests", "custom_env", "hetero_env_step.cu"))
    env = CUDAHeteroEnv(num_agents=NW + 1, episode_length=L, worker_obs_layout="last",
                        env_backend="pycuda")
    w = EnvWrapper(env, num_envs=E, env_backend="pycuda", env_registrar=reg)
    cfg = load_run_config("tag_gridworld")
    cfg["trainer"].update(num_envs=E, train_batch_size=E * T, num_episodes=E * 100, seed=3)
    cfg["saving"].update(basedir=basedir, metrics_log_freq=10 ** 9, model_params_save_freq=10 ** 9)
    pol = cfg["policy"].pop("shared")
    pol["model"]["fc_dims"] = [64, 64]
    cfg["policy"] = {p: json.loads(json.dumps(pol)) for p in ("planner", "workers")}
    tr = Trainer(env_wrapper=w, config=cfg,
                 policy_tag_to_agent_id_map=env.policy_tag_to_agent_id_map(),
                 create_separate_placeholders_for_each_policy=True,
                 obs_dim_corresponding_to_num_agents="last", results_dir="bench", verbose=False)
    return tr


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


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def as_graph(fn):
    """A CUDA graph of REPS calls of fn (warmed up on a side stream first)."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(REPS):
            fn()
    return g


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_hetero_rollout.py needs a GPU")
    with tempfile.TemporaryDirectory() as tmp:
        tr = build(tmp)
        eng = tr.engine
        tr.cuda_envs.reset_all_envs()
        eng.resync_observations()

        def iteration():
            tr._generate_rollout_batch()
            tr._update_model_params(1)

        for _ in range(3):
            iteration()
        torch.cuda.synchronize()
        rollout_ms = timed(tr._generate_rollout_batch, 20) / T
        iteration_ms = timed(iteration, 10)

        # ---- one timestep's observation gather, native against torch
        dm = tr.cuda_envs.cuda_data_manager
        t = dm.data_on_device_via_torch
        obs_p = {p: t(f"processed_observations_batch_{p}")[0] for p in eng.policies}
        mask_p = {"planner": t("action_mask_batch_planner")[0], "workers": None}
        native = lambda: eng._gather_fields(obs_p, mask_p)       # noqa: E731
        state, mask = t("observations_planner_state"), t("observations_planner_action_mask")
        wobs = t("observations_workers")

        def torch_way():
            # model_base.py's reshape_and_flatten_obs: permute the agent axis forward, flatten
            obs_p["workers"].copy_(wobs.permute(0, 3, 1, 2).reshape(E, NW, -1))
            obs_p["planner"].copy_(state.permute(0, 2, 1).reshape(E, 1, -1))
            mask_p["planner"].copy_(mask.permute(0, 2, 1).reshape(E, 1, -1).float())

        gn, gt = as_graph(native), as_graph(torch_way)
        for g in (gn, gt):
            timed(g.replay, 3)
        ms = {"native": [], "torch": []}
        for _ in range(7):
            ms["native"].append(timed(gn.replay, 10) / REPS)
            ms["torch"].append(timed(gt.replay, 10) / REPS)
        native_ms, torch_ms = min(ms["native"]), min(ms["torch"])
        moved = 2 * sum(x.numel() * 4 for x in (wobs, state, mask))    # read + written
        name, power = gpu_info()
        print(json.dumps({
            "gpu": name, "power_limit": power, "n_envs": E, "n_agents": NW + 1,
            "worker_obs_layout": "last", "T": T, "algorithm": "A2C", "fc_dims": [64, 64],
            "rollout_ms_per_timestep": round(rollout_ms, 4),
            "training_iteration_ms": round(iteration_ms, 3),
            "gather_bytes": moved,
            "gather_ms": round(native_ms, 5),
            "gather_tb_per_s": round(moved / (native_ms * 1e-3) / 1e12, 3),
            "gather_fraction_of_3_35_tb_per_s": round(moved / (native_ms * 1e-3) / PEAK, 3),
            "torch_permute_gather_ms": round(torch_ms, 5),
            "native_speedup": round(torch_ms / native_ms, 2),
        }))


if __name__ == "__main__":
    main()
