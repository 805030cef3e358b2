"""Action-masked DQN timings on one GPU, printed as one JSON line (card name and power limit read
in the same run):

  sampler    epsilon-greedy over 1 000 000 rows of 4 Q values (epsilon 0.3):
             wdb_sample_epsilon_greedy_masked with a random mask against
             wdb_sample_epsilon_greedy;
  dqn / c51  the native pass's gradient (2 launches) over B = 512 and 50 000 sampled windows of
             a store of 1024 slots x 256 envs x 6 agents (MaskedCounterEnv's F = 3, A = 4):
             DQN [64, 64] and C51 [64] x 51 atoms, masked (a random ring mask) against unmasked;
  iteration  one TrainerDQN iteration on 256 MaskedCounterEnv replicas (6 agents, an 8-step
             rollout on the per-step path, 2 updates of 512 windows), the masked DQN pass
             against the masked torch loss.

Every figure is the median over `--rounds` alternated rounds of CUDA-event-timed loops.

    python scripts/bench_masked_dqn.py [--rounds 5]
"""
import argparse
import json
import os
import statistics
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_dqn import gpu_info, timed  # noqa: E402

C, E, NP, F, A = 1024, 256, 6, 3, 4


def sampler_fns():
    from warp_drive_b200 import lib as wlib

    L = wlib.load()
    R = 1000000
    g = torch.Generator(device="cuda").manual_seed(0)
    q = torch.randn((R, A), device="cuda", generator=g)
    mask = (torch.rand((R, A), device="cuda", generator=g) < 0.6).float()
    out = torch.empty(R, dtype=torch.int32, device="cuda")
    state = torch.zeros(int(L.wdb_rng_state_bytes(R)), dtype=torch.uint8, device="cuda")
    wlib.check(L.wdb_rng_init(wlib.stream_ptr(), wlib.ptr(state), R, 1))

    def masked():
        wlib.check(L.wdb_sample_epsilon_greedy_masked(
            wlib.stream_ptr(), wlib.ptr(state), wlib.ptr(q), wlib.ptr(mask), wlib.ptr(out), R,
            A, 0.3, None))

    def plain():
        wlib.check(L.wdb_sample_epsilon_greedy(
            wlib.stream_ptr(), wlib.ptr(state), wlib.ptr(q), wlib.ptr(out), R, A, 0.3, None))
    return masked, plain


def pass_fns(kind, B):
    """(masked, unmasked) gradient launches of one network over B random windows."""
    from c51_reference import make_c51_models
    from dqn_update_reference import make_q_models
    from warp_drive_b200.training.algorithms import dqn as algos
    from warp_drive_b200.training.algorithms import fused_dqn as fd

    if kind == "dqn":
        q, t = (m.float().cuda() for m in make_q_models(F, A, [64, 64]))
        algo, classes = algos.DQN(0.9, n_step=3), (fd.FusedMaskedDQNUpdate, fd.FusedDQNUpdate)
    else:
        q, t = (m.float().cuda() for m in make_c51_models(F, A, [64], N=51, v_min=0, v_max=12))
        algo = algos.CategoricalDQN(0.9, n_step=3)
        classes = (fd.FusedMaskedC51Update, fd.FusedC51Update)
    for p in q.parameters():
        p.grad = torch.zeros_like(p)
    g = torch.Generator(device="cuda").manual_seed(1)
    obs = torch.randn((C, E, NP, F), device="cuda", generator=g)
    actions = torch.randint(0, A, (C, E, NP, 1), device="cuda", generator=g, dtype=torch.int32)
    rewards = torch.rand((C, E, NP), device="cuda", generator=g)
    done = (torch.rand((C, E), device="cuda", generator=g) < 0.1).to(torch.int32)
    mask = (torch.rand((C, E, NP, A), device="cuda", generator=g) < 0.6).float()
    windows = torch.stack([torch.randint(0, C, (B,), device="cuda", generator=g),
                           torch.randint(0, E * NP, (B,), device="cuda", generator=g)],
                          1).to(torch.int32).contiguous()
    masked, plain = (cls(algo, q, t, E, NP, C, B) for cls in classes)
    ring = (obs, actions, rewards, done, windows)
    return (lambda: masked.launch(*ring, action_mask=mask)), (lambda: plain.launch(*ring))


def iteration_fn(tr, fused):
    def run():
        tr.trainers["shared"].use_fused_update = fused
        tr._generate_rollout_batch()
        tr._update_model_params(1)
    return run


def main():
    from masked_counter_dqn_learning import make_trainer

    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    pairs = {"sampler": (sampler_fns(), 200)}
    for B in (512, 50000):
        n = 200 if B == 512 else 20
        for kind in ("dqn", "c51"):
            pairs[f"{kind}_B{B}"] = (pass_fns(kind, B), n)
    tr = make_trainer("dqn", E=256, slots=64, name="bench")
    for it in range(8):                       # fill past the warm-up
        iteration_fn(tr, True)()
    pairs["iteration"] = ((iteration_fn(tr, True), iteration_fn(tr, False)), 20)
    times = {k: ([], []) for k in pairs}
    for _ in range(args.rounds):
        for k, ((a, b), n) in pairs.items():
            times[k][0].append(timed(a, n))
            times[k][1].append(timed(b, n))
    out = {"gpu": gpu_info(), "rounds": args.rounds}
    names = {"sampler": ("masked_ms", "unmasked_ms"), "iteration": ("native_ms", "torch_ms")}
    for k, (a, b) in times.items():
        na, nb = names.get(k, ("masked_ms", "unmasked_ms"))
        out[k] = {na: round(statistics.median(a), 4), nb: round(statistics.median(b), 4)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
