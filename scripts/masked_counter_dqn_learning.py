"""Does TrainerDQN learn an action-masked env?  MaskedCounterEnv (tests/custom_env): 6 agents per
env, each with a counter and a cap of its own (3, 4, 5, 6, 7, 3); action a adds 0, 1, 2 or 5 and
is valid only while the counter stays within the cap, so the valid actions depend on the state.
The reward is the step taken (an invalid action would cost -10 and leave the counter), so the
best episode return of an agent is its cap, reached in as few steps as its cap allows.

Three configs of one shared policy with 3-step returns: plain double DQN, the same with
prioritized replay, and the Rainbow head (a dueling noisy C51 network, prioritized, epsilon 0).
Printed as one JSON line per config, then the card:
  greedy_return  per agent, the mean greedy episode return (epsilon 0, the mean network) over
                 the envs, beside its cap;
  invalid        the env's count of invalid actions received, over training and evaluation;
  mean_q         the last update's `Mean Q value` (Q(obs, a) over the sampled windows);
  q0 / disc0     the greedy action's Q value at the episode's first observation and the
                 discounted return (gamma 0.9) the greedy episode then earned, means over agents
                 and envs: a Q network that has learned the masked problem has q0 close to disc0.

    python scripts/masked_counter_dqn_learning.py [--iterations 300] [--seed 1]
"""
import argparse
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "custom_env"))

GAMMA = 0.9
N_AGENTS, EPISODE = 6, 10

MODELS = {
    "dqn": {"type": "fully_connected_q", "fc_dims": [64, 64], "masked": True},
    "rainbow": {"type": "fully_connected_categorical_q", "fc_dims": [64], "num_atoms": 51,
                "v_min": 0.0, "v_max": 12.0, "dueling": True, "stream_fc_dims": [32],
                "noisy": True, "masked": True},
}


def make_trainer(model, prioritized=False, epsilon=1.0, E=256, seed=1, slots=512, rows=512,
                 updates=2, name="m", log_every=10 ** 9):
    """A TrainerDQN on E MaskedCounterEnv replicas with one shared policy of `model` (a key of
    MODELS)."""
    from masked_counter_env import STEP_TABLE, CUDAMaskedCounterEnv

    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import TrainerDQN
    from warp_drive_b200.utils.env_registrar import EnvironmentRegistrar

    reg = EnvironmentRegistrar()
    reg.add_cuda_env_src_path("MaskedCounterEnv", os.path.join(
        ROOT, "tests", "custom_env", "masked_counter_env_step.cu"))
    env = CUDAMaskedCounterEnv(num_agents=N_AGENTS, episode_length=EPISODE,
                               env_backend="pycuda")
    w = EnvWrapper(env, num_envs=E, env_backend="pycuda", env_registrar=reg)
    dm, fm = w.cuda_data_manager, w.cuda_function_manager
    dm.add_shared_constants({"kMaskedStepTable": STEP_TABLE})
    fm.initialize_shared_constants(dm, ["kMaskedStepTable"])
    cfg = load_run_config("single_cartpole_dqn")
    cfg["trainer"].update(num_envs=E, train_batch_size=E * 8, num_episodes=E * 10 ** 6,
                          seed=seed, n_step=3, replay_slots_per_env=slots,
                          replay_batch_rows=rows, updates_per_iteration=updates,
                          replay_warmup_slots=32, evaluator=False)
    if prioritized:
        cfg["trainer"].update(prioritized_replay=True, priority_alpha=0.6, priority_beta=0.4,
                              priority_epsilon=1e-6)
    cfg["saving"].update(basedir=tempfile.mkdtemp(), metrics_log_freq=log_every,
                         model_params_save_freq=10 ** 9)
    pol = cfg["policy"]["shared"]
    pol.update(model=dict(MODELS[model]), gamma=GAMMA, lr=0.001)
    if model == "rainbow":
        pol.pop("huber_delta", None)
    cfg["sampler"]["params"]["epsilon"] = epsilon
    return TrainerDQN(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map={
        "shared": list(range(N_AGENTS))}, results_dir=name, verbose=False)


def greedy_episode(tr):
    """One greedy episode (epsilon 0, the mean network) in every env: per agent the mean return,
    and the means of q0 (the chosen action's Q value at the first observation) and of the
    discounted return."""
    eng = tr.engine
    E = tr.num_envs
    tr.cuda_envs.reset_all_envs()
    ret = torch.zeros((E, N_AGENTS), device="cuda")
    disc = torch.zeros((E, N_AGENTS), device="cuda")
    with torch.no_grad():
        for t in range(EPISODE):
            q = eng.evaluate_policies(-1)[0]
            eng.sample_actions([q], -1, epsilon=0.0)
            if t == 0:
                a = eng._tensor("sampled_actions").long().view(E, N_AGENTS, 1)
                q0 = tr.q_models["shared"].q_values(
                    eng._field_scratch[0]["shared"]).gather(-1, a)[..., 0]
            tr.cuda_envs.step_all_envs()
            r = eng.policy_step_arrays("shared")[0]
            ret += r
            disc += GAMMA ** t * r
    tr.cuda_envs.reset_all_envs()
    return ret.mean(0).tolist(), float(q0.mean()), float(disc.mean())


def run(name, model, prioritized, epsilon, iterations, seed):
    from masked_counter_env import agent_caps

    tr = make_trainer(model, prioritized, epsilon, seed=seed, name=name, log_every=1)
    metrics = {}
    for it in range(1, iterations + 1):
        tr._generate_rollout_batch()
        out = tr._update_model_params(it)
        if out.get("shared"):
            metrics = out["shared"]
    ret, q0, disc = greedy_episode(tr)
    invalid = int(tr.cuda_envs.cuda_data_manager.pull_data_from_device("invalid_actions")[0])
    tr.graceful_close()
    return {"config": name, "iterations": iterations, "seed": seed,
            "greedy_return": [round(x, 3) for x in ret],
            "cap": agent_caps(N_AGENTS).tolist(), "invalid": invalid,
            "mean_q": metrics.get("Mean Q value"), "q0": round(q0, 3), "disc0": round(disc, 3)}


def main():
    from bench_dqn import gpu_info

    ap = argparse.ArgumentParser()
    ap.add_argument("--iterations", type=int, default=300)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    n = args.iterations
    decay = [[0, 1.0], [n * 256 * 8 // 2, 0.05]]      # the policy timestep: E * T per update
    for name, model, per, eps in (("dqn", "dqn", False, decay), ("dqn_per", "dqn", True, decay),
                                  ("rainbow", "rainbow", True, 0.0)):
        print(json.dumps(run(name, model, per, eps, n, args.seed)), flush=True)
    print(json.dumps({"gpu": gpu_info()}))


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    main()
