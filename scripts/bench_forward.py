#!/usr/bin/env python
"""Where the config-2 rollout timestep spends its time in the wgmma policy forward
(csrc/wdb_mlp.cu), on the real seeded engine of bench.py (2000 envs x (5 taggers + 100
runners), FullyConnected [256, 256], two 21-way heads).

    python scripts/bench_forward.py [--iters 200] [--json OUT]

Reports, as CUDA-event medians with min-max over `--iters` launches:
  * each policy's forward alone, on the SM share the rollout gives it and on all SMs, with the
    L2 warm (back-to-back launches) and flushed (512 MiB written before every launch);
  * the side-by-side pair exactly as RolloutEngine._forward_side_by_side issues it (fork onto
    a side stream, both forwards, join);
  * eager rollout timesteps with events around the forward pair and the fused env launch, and
    around each forward inside it, splitting the step into forwards, fork/join and env launch;
  * the CUDA-graph rollout's ms per step, as bench.py times it.
Achieved TFLOP/s and GB/s are computed from the shapes (padded MMA work; observation bytes
read + probability bytes written).  The card's name, power limit and max SM clock are read in
the same run.  Prints one JSON object.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, power, clock = [s.strip() for s in out.split(",")]
    except Exception:  # noqa: BLE001
        name, power, clock = torch.cuda.get_device_name(), "unknown", "unknown"
    return {"name": name, "power_limit": power, "sm_clock_max": clock,
            "sms": torch.cuda.get_device_properties(0).multi_processor_count}


def stats(ms):
    ms = sorted(ms)
    return {"ms_median": ms[len(ms) // 2], "ms_min": ms[0], "ms_max": ms[-1], "n": len(ms)}


def work(f, rows):
    """(padded MMA FLOP, algorithmic HBM bytes) of one forward over `rows` rows."""
    k1, n3 = -(-f.F // 16) * 16, -(-(f.A0 + f.A1 + 1) // 16) * 16
    flop = 2 * rows * (k1 * f.H + f.H * f.H + f.H * n3)
    nbytes = rows * 4 * (f.F + f.A0 + f.A1)
    return flop, nbytes


def with_rates(s, flop, nbytes):
    t = s["ms_median"] * 1e-3
    return dict(s, tflops=flop / t / 1e12, gbs=nbytes / t / 1e9)


def time_launches(fn, iters, flush=None):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
          for _ in range(iters)]
    for _ in range(5):
        fn()
    for a, b in ev:
        if flush is not None:
            bench.flush_l2(flush)
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return stats([a.elapsed_time(b) for a, b in ev])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--envs", type=int, default=2000)
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_forward.py measures on the GPU"
    T = 10
    wrapper, engine, _, _ = bench.build_engine(args.envs, seed=1234, graph_steps=T,
                                               use_graph=True)
    assert engine.fused is not None and engine.fused_forward, "config 2 must run the fused path"
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    obs = engine.cur_obs
    probs = engine._probs
    with torch.no_grad():
        engine._forward_side_by_side(obs, probs)      # builds the SM split (_fwd_plan)
    order, share = engine._fwd_plan
    flush = torch.zeros(128 * 1024 * 1024, dtype=torch.float32, device="cuda")
    out = {"card": card(), "envs": args.envs, "iters": args.iters, "policies": {}}

    total_flop = total_bytes = 0
    for p in order:
        f = engine.fused_forward[p]
        rows = obs[p].numel() // f.F
        flop, nbytes = work(f, rows)
        total_flop += flop
        total_bytes += nbytes
        r = {"rows": rows, "tiles": -(-rows // 128), "sm_share": share[p],
             "shape": [f.F, f.H, f.A0, f.A1], "flop": flop, "bytes": nbytes}
        for label, ctas in (("share", share[p]), ("all_sms", 0)):
            def fn(f=f, p=p, ctas=ctas):
                f(obs[p], probs[p][0], probs[p][1], max_ctas=ctas)
            for l2, fl in (("warm", None), ("flushed", flush)):
                r[f"{label}_{l2}"] = with_rates(time_launches(fn, args.iters, fl), flop, nbytes)
        out["policies"][p] = r

    def pair():
        engine._forward_side_by_side(obs, probs)
    with torch.no_grad():
        for l2, fl in (("warm", None), ("flushed", flush)):
            out[f"pair_{l2}"] = with_rates(time_launches(pair, args.iters, fl), total_flop,
                                           total_bytes)

    # ---- the side-by-side pair at every split near the cost model's choice: the constants
    # of RolloutEngine._forward_side_by_side are fitted to this
    small = order[1]
    sweep = {}
    with torch.no_grad():
        for k in range(max(1, share[small] - 4), share[small] + 7):
            engine._fwd_plan = (order, {order[0]: n_sm - k, small: k})
            sweep[k] = time_launches(pair, max(20, args.iters // 4))["ms_median"]
    engine._fwd_plan = (order, share)
    out["pair_split_sweep"] = {"small_policy": small, "chosen": share[small],
                               "ms_median_by_small_share": sweep}

    # ---- eager timesteps, events around the forward pair, each forward and the env launch
    spans = {"step": [], "forwards": [], "env": []}
    per_fwd = {p: [] for p in order}
    orig_pair, orig_one, orig_launch = (engine._forward_side_by_side, engine._one_forward,
                                        engine.fused.launch)

    def ev():
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return e
    cur = {}

    def timed_pair(*a, **k):
        cur["f0"] = ev()
        r = orig_pair(*a, **k)
        cur["f1"] = ev()
        return r

    def timed_one(p, *a, **k):
        s = ev()
        orig_one(p, *a, **k)
        cur[p] = (s, ev())

    def timed_launch(*a, **k):
        cur["e0"] = ev()
        orig_launch(*a, **k)
        cur["e1"] = ev()

    engine._forward_side_by_side, engine._one_forward = timed_pair, timed_one
    engine.fused.launch = timed_launch
    records = []
    try:
        for i in range(args.iters + 10):
            s = ev()
            engine.step(i % T)
            cur["s"] = s
            records.append(dict(cur))
    finally:
        engine._forward_side_by_side, engine._one_forward = orig_pair, orig_one
        engine.fused.launch = orig_launch
    torch.cuda.synchronize()
    for r in records[10:]:
        spans["step"].append(r["s"].elapsed_time(r["e1"]))
        spans["forwards"].append(r["f0"].elapsed_time(r["f1"]))
        spans["env"].append(r["e0"].elapsed_time(r["e1"]))
        for p in order:
            per_fwd[p].append(r[p][0].elapsed_time(r[p][1]))
    eager = {k: stats(v) for k, v in spans.items()}
    eager["forward_in_step"] = {p: stats(v) for p, v in per_fwd.items()}
    slowest = [max(r[p][0].elapsed_time(r[p][1]) for p in order) for r in records[10:]]
    eager["fork_join"] = stats([f - s for f, s in zip(spans["forwards"], slowest)])
    eager["note"] = ("eager steps: the host launches each kernel, so gaps can include host "
                     "launch latency; fork_join = forwards span - slowest forward in it")
    out["eager_step"] = eager

    # ---- the CUDA-graph rollout, as bench.py times it
    for _ in range(5):
        engine.rollout()
    torch.cuda.synchronize()
    reps = []
    for _ in range(max(5, args.iters // 20)):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(5):
            engine.rollout()
        b.record()
        b.synchronize()
        reps.append(a.elapsed_time(b) / (5 * T))
    out["graph_ms_per_step"] = stats(reps)
    text = json.dumps(out, indent=1)
    print(text)
    if args.json:
        with open(args.json, "w") as fp:
            fp.write(text + "\n")


if __name__ == "__main__":
    main()
