"""Branching DQN timings on one GPU at the shape of tag_continuous_dqn.yaml, printed as one JSON
line (card name and power limit read in the same run):

  sampler    per-head epsilon-greedy over the config's E * N = 50 * 110 rows of two heads of 21
             Q values (epsilon 0.3), wdb_sample_epsilon_greedy_branching against
             wdb_sample_epsilon_greedy over the same rows' 42 columns as one head;
  pass_B*    the runner policy's gradient over B = 256, 4096 and 50 000 sampled windows of a
             store of 1024 slots x 50 envs x 100 runners (F = 57, [64, 64], A = 21 + 21):
             the native branching pass (2 launches) against BranchingDQN's torch loss and
             backward on the gathered windows, and against DQN's native pass on one head of
             the same A = 42;
  iteration  one TrainerDQN iteration of the run config (a 4-step rollout of 50 envs on the
             per-step path, 2 updates of 1024 windows for each of the two policies), the native
             passes against the torch losses.

Every figure is the median over `--rounds` alternated rounds of CUDA-event-timed loops.

    python scripts/bench_branching_dqn.py [--rounds 5]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_dqn import gpu_info, timed  # noqa: E402

C, E, NP, F, SIZES, DIMS = 1024, 50, 100, 57, [21, 21], [64, 64]


def sampler_fns():
    from warp_drive_b200 import lib as wlib

    L = wlib.load()
    R, A = E * 110, sum(SIZES)
    g = torch.Generator(device="cuda").manual_seed(0)
    q = torch.randn((R, A), device="cuda", generator=g)
    out = torch.empty((R, len(SIZES)), dtype=torch.int32, device="cuda")
    state = torch.zeros(int(L.wdb_rng_state_bytes(R)), dtype=torch.uint8, device="cuda")
    wlib.check(L.wdb_rng_init(wlib.stream_ptr(), wlib.ptr(state), R, 1))
    b = wlib.QBranches()
    b.n_heads = len(SIZES)
    for d, a in enumerate(SIZES):
        b.sizes[d] = a

    def branching():
        wlib.check(L.wdb_sample_epsilon_greedy_branching(
            wlib.stream_ptr(), wlib.ptr(state), wlib.ptr(q), ctypes.byref(b), wlib.ptr(out), R,
            0.3, None))

    def plain():
        wlib.check(L.wdb_sample_epsilon_greedy(
            wlib.stream_ptr(), wlib.ptr(state), wlib.ptr(q), wlib.ptr(out), R, A, 0.3, None))
    return branching, plain


def pass_fns(B):
    """(native branching pass, torch loss + backward, DQN's pass at the same A)."""
    from branching_q_reference import make_branching_models
    from dqn_update_reference import make_q_models
    from warp_drive_b200.training.algorithms import dqn as algos
    from warp_drive_b200.training.algorithms import fused_dqn as fd

    A = sum(SIZES)
    q, t = (m.float().cuda() for m in make_branching_models(F, SIZES, DIMS))
    pq, pt = (m.float().cuda() for m in make_q_models(F, A, DIMS))
    for p in list(q.parameters()) + list(pq.parameters()):
        p.grad = torch.zeros_like(p)
    g = torch.Generator(device="cuda").manual_seed(1)
    obs = torch.randn((C, E, NP, F), device="cuda", generator=g)
    actions = torch.stack([torch.randint(0, a, (C, E, NP), device="cuda", generator=g)
                           for a in SIZES], -1).to(torch.int32).contiguous()
    rewards = torch.rand((C, E, NP), device="cuda", generator=g)
    done = (torch.rand((C, E), device="cuda", generator=g) < 0.01).to(torch.int32)
    windows = torch.stack([torch.randint(0, C, (B,), device="cuda", generator=g),
                           torch.randint(0, E * NP, (B,), device="cuda", generator=g)],
                          1).to(torch.int32).contiguous()
    algo = algos.BranchingDQN(0.98, n_step=3)
    native = fd.FusedBranchingDQNUpdate(algo, q, t, E, NP, C, B)
    dqn = fd.FusedDQNUpdate(algos.DQN(0.98, n_step=3), pq, pt, E, NP, C, B)
    ring = (obs, actions, rewards, done, windows)
    plain_ring = (obs, actions[..., :1].contiguous(), rewards, done, windows)

    def torch_loss():
        w = windows.long()
        steps = (w[:, 0][None, :] + torch.arange(4, device="cuda")[:, None]) % C
        o = obs.reshape(C, -1, F)
        loss, _, _ = algo.loss(q, t, o[w[:, 0], w[:, 1]],
                               actions.reshape(C, -1, len(SIZES))[w[:, 0], w[:, 1]],
                               rewards.reshape(C, -1)[steps[:-1], w[:, 1]],
                               done[steps[:-1], w[:, 1] // NP].float(), o[steps[-1], w[:, 1]])
        q.zero_grad()
        loss.backward()
    return (lambda: native.launch(*ring)), torch_loss, (lambda: dqn.launch(*plain_ring))


def make_trainer(name):
    from warp_drive_b200.env_wrapper import EnvWrapper
    from warp_drive_b200.envs.tag_continuous import TagContinuous
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import TrainerDQN

    cfg = load_run_config("tag_continuous_dqn")
    cfg["trainer"]["evaluator"] = False
    cfg["saving"].update(basedir=tempfile.mkdtemp(), metrics_log_freq=10 ** 9,
                         model_params_save_freq=10 ** 9)
    env = TagContinuous(**cfg["env"])
    w = EnvWrapper(env, num_envs=cfg["trainer"]["num_envs"], env_backend="b200")
    n_t, n_r = cfg["env"]["num_taggers"], cfg["env"]["num_runners"]
    pm = {"tagger": list(range(n_t)), "runner": list(range(n_t, n_t + n_r))}
    return TrainerDQN(env_wrapper=w, config=cfg, policy_tag_to_agent_id_map=pm,
                      results_dir=name, verbose=False)


def iteration_fn(tr, fused):
    def run():
        for p in tr.trainers:
            tr.trainers[p].use_fused_update = fused
        tr._generate_rollout_batch()
        tr._update_model_params(1)
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    fns = {"sampler": (sampler_fns(), 200)}
    for B in (256, 4096, 50000):
        fns[f"pass_B{B}"] = (pass_fns(B), 100 if B < 50000 else 20)
    tr = make_trainer("bench")
    assert set(tr.fused_updates) == {"tagger", "runner"}
    for _ in range(20):                       # fill past the warm-up
        iteration_fn(tr, True)()
    fns["iteration"] = ((iteration_fn(tr, True), iteration_fn(tr, False)), 10)
    times = {k: [[] for _ in f] for k, (f, _) in fns.items()}
    for _ in range(args.rounds):
        for k, (f, n) in fns.items():
            for i, fn in enumerate(f):
                times[k][i].append(timed(fn, n))
    names = {"sampler": ("branching_ms", "one_head_ms"),
             "iteration": ("native_ms", "torch_ms")}
    out = {"gpu": gpu_info(), "rounds": args.rounds}
    for k, ts in times.items():
        keys = names.get(k, ("native_ms", "torch_ms", "dqn_pass_ms"))
        out[k] = {n: round(statistics.median(t), 4) for n, t in zip(keys, ts)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
