"""Implicit quantile network (IQN) timings on one GPU, printed as one JSON line (card name and
power limit read in the same run).  On a full store of 256 CartPole envs x 4096 slots (~10^6
transitions), with the fc_dims [64, 64] network and n_cos = 64 cosine features of
single_cartpole_iqn.yaml, for B = 256, 4096 and 50 000 sampled windows and N = N' = 8 and 32
levels per loss row:

  pass_ms    the native pass alone (wdb_iqn_update_sampled: tile kernel + reduction) against
             QR-DQN's (wdb_qr_dqn_update_sampled, N quantiles) on the same windows;
  update_ms  one whole update (window draw + level draw + gradients + clipping + Adam) with the
             native pass, with the torch autograd loss on the gathered windows, and QR-DQN's
             native update;
  launches   of this library per native IQN update (the level draw is one torch launch more).

Every figure is the median over `--rounds` alternated rounds of CUDA-event-timed loops.

    python scripts/bench_iqn.py [--rounds 5]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_dqn import gpu_info, timed  # noqa: E402
from bench_qr_dqn import E, SLOTS, fill, make_trainer, pass_fn, setup  # noqa: E402


def iqn_setup(tr, B):
    """setup() for IQN: the pass and the levels buffer for B windows."""
    from warp_drive_b200.training.algorithms.fused_dqn import FusedIQNUpdate

    q = tr.q_models["shared"]
    tr.iqn_taus["shared"] = torch.zeros(
        B, q.num_tau_samples + q.num_tau_prime_samples, device="cuda")
    setup(tr, FusedIQNUpdate, B)
    tr.iqn_taus["shared"].uniform_(generator=tr._tau_generator)


def iqn_pass_fn(tr):
    eng, f = tr.engine, tr.fused_updates["shared"]
    args = (eng._tensor("processed_observations_batch_shared"),
            eng._tensor("sampled_actions_batch_shared"), eng._tensor("rewards_batch_shared"),
            eng._tensor("done_flags_batch"), tr.replay_windows["shared"])
    taus = tr.iqn_taus["shared"]
    return lambda: f.launch(*args, taus=taus)


def main():
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.fused_dqn import FusedQRDQNUpdate

    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    iqn = {N: make_trainer(f"iqn{N}", model={
        "type": "fully_connected_iqn", "fc_dims": [64, 64], "num_cosines": 64,
        "num_tau_samples": N, "num_tau_prime_samples": N, "num_quantile_samples": 32,
        "model_ckpt_filepath": ""}) for N in (8, 32)}
    qr = {N: make_trainer(f"qr{N}", model={
        "type": "fully_connected_quantile_q", "fc_dims": [64, 64], "num_quantiles": N,
        "model_ckpt_filepath": ""}) for N in (8, 32)}
    for tr in [*iqn.values(), *qr.values()]:
        fill(tr)
    out = {}
    for B in (256, 4096, 50000):
        for N, tr in iqn.items():
            iqn_setup(tr, B)
            setup(qr[N], FusedQRDQNUpdate, B)
            algo = tr.trainers["shared"]
            t = {k: [] for k in ("pass_iqn", "pass_qr", "update_iqn", "update_torch",
                                 "update_qr")}
            for _ in range(args.rounds):
                t["pass_iqn"].append(timed(iqn_pass_fn(tr), 20))
                t["pass_qr"].append(timed(pass_fn(qr[N]), 20))
                algo.use_fused_update = True
                t["update_iqn"].append(timed(lambda: tr._one_update(False, {}), 20))
                algo.use_fused_update = False
                t["update_torch"].append(timed(lambda: tr._one_update(False, {}), 5))
                t["update_qr"].append(timed(lambda: qr[N]._one_update(False, {}), 20))
            algo.use_fused_update = True
            n0 = wlib.launch_count()
            tr._one_update(False, {})
            torch.cuda.synchronize()
            launches = wlib.launch_count() - n0
            m = {k: statistics.median(v) for k, v in t.items()}
            out[f"B{B}_N{N}"] = {
                "pass_ms": {"iqn": m["pass_iqn"], "qr_dqn": m["pass_qr"]},
                "update_ms": {"iqn_native": m["update_iqn"], "iqn_torch": m["update_torch"],
                              "qr_dqn_native": m["update_qr"]},
                "native_over_torch_speedup": m["update_torch"] / m["update_iqn"],
                "launches_per_native_update": launches}
    print(json.dumps({"gpu": gpu_info(), "rounds": args.rounds, "envs": E, "slots": SLOTS,
                      "fc_dims": [64, 64], "num_cosines": 64, "results": out}))


if __name__ == "__main__":
    main()
