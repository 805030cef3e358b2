"""The recurrent policy's costs at TagContinuous's bench shape (2000 envs x 105 agents, F = 71,
trunk [64, 64], GRU 64, two 21-way heads) and at gridworld's (2000 envs x 5 agents, F = 21,
trunk [32, 32], GRU 32, one 5-way head):

* per-step rollout forward: wdb_gru_policy_forward (native), the model's torch `step`
  expression, and the feed-forward FullyConnected policy of the same trunk in torch;
* training: forward_sequence + backward over T = 10 steps of every row (the loop of cuBLAS GEMMs
  and elementwise ops the A2C / PPO update runs).

The Gaussian policy's mean head (fully_connected_gaussian_gru, the kernel's mean head kind) at
three more shapes: Pendulum-like (10 000 envs x 1 agent, F = 3, trunk [64, 64], GRU 64, A = 1),
one just over the 1 GFLOP routing cut (20 000 rows, F = 17, [64, 64], GRU 64, A = 6) and
TagContinuous's rows (2000 x 105, F = 71, [64, 64], GRU 64, A = 2); there the feed-forward
comparison is fully_connected_gaussian of the same trunk.

Alternated rounds; median and min-max of ms per call; FLOPs counted from the shapes; the card's
name and power limit read in the same process.

    python scripts/bench_recurrent.py [--rounds 5] [--iters 50] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SHAPES = {"tag_continuous": dict(R=2000 * 105, F=71, fc=(64, 64), H=64, heads=(21, 21)),
          "gridworld": dict(R=2000 * 5, F=21, fc=(32, 32), H=32, heads=(5,)),
          "pendulum_mean": dict(R=10000, F=3, fc=(64, 64), H=64, heads=(1,), mean=True),
          "over_cut_mean": dict(R=20000, F=17, fc=(64, 64), H=64, heads=(6,), mean=True),
          "tag_continuous_mean": dict(R=2000 * 105, F=71, fc=(64, 64), H=64, heads=(2,),
                                      mean=True)}


def step_flops(F, fc, H, heads, **_):
    dims = [F] + list(fc)
    mac = sum(a * b for a, b in zip(dims[:-1], dims[1:])) + 3 * H * (dims[-1] + H)
    return 2 * (mac + H * sum(heads))


def main():
    import torch

    from test_gaussian_recurrent_cpu import _gmodel
    from test_recurrent_cpu import _built_fc, _model, _stub_env
    from warp_drive_b200.training.models.fully_connected import FullyConnectedGaussian
    from warp_drive_b200.utils.spaces import Box
    from warp_drive_b200.training.models.fully_connected_gru import NativeGruStep

    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--T", type=int, default=10)
    ap.add_argument("--only", default=None, help="comma-separated shape names")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout
    res = {"card": card.strip(), "rounds": a.rounds, "iters": a.iters, "T": a.T}

    def timed(fn, iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    names = a.only.split(",") if a.only else list(SHAPES)
    for name in names:
        s = SHAPES[name]
        R = s["R"]
        if s.get("mean"):
            A = s["heads"][0]
            gru = _gmodel(fc_dims=s["fc"], gru_dim=s["H"], A=A, F=s["F"]).cuda()
            ff = FullyConnectedGaussian(_stub_env(Box(-1, 1, shape=(A,)), s["F"]),
                                        {"fc_dims": list(s["fc"])}, "p", {"p": [0]}).cuda()
        else:
            gru = _model(fc_dims=s["fc"], gru_dim=s["H"], heads=s["heads"], F=s["F"]).cuda()
            ff = _built_fc(s["fc"], s["heads"], F=s["F"]).cuda()
        native = NativeGruStep(gru)
        obs = torch.randn(R, s["F"], device="cuda")
        h = torch.zeros(R, s["H"], device="cuda")
        probs = [torch.empty(R, k, device="cuda") for k in s["heads"]]
        seq_obs = torch.randn(a.T, R, 1, s["F"], device="cuda")
        h0 = torch.zeros(R, 1, s["H"], device="cuda")
        done = torch.zeros(a.T, R, dtype=torch.int32, device="cuda")

        def torch_step():
            with torch.no_grad():
                p, hn = gru.step(obs, h)
                h.copy_(hn)

        def ff_step():
            with torch.no_grad():
                ff.forward(obs)

        def train():
            p, v = gru.forward_sequence(seq_obs, h0, done)
            (sum(q.sum() for q in p) + v.sum()).backward()

        cases = {"native": lambda: native(obs, h, probs), "torch_step": torch_step,
                 "feed_forward_torch": ff_step}
        times = {k: [] for k in cases}
        for fn in cases.values():
            timed(fn, 3)
        for _ in range(a.rounds):
            for k, fn in cases.items():
                times[k].append(timed(fn, a.iters))
        timed(train, 2)
        train_t = [timed(train, 3) for _ in range(a.rounds)]
        fl = step_flops(**s) * R
        out = {"rows": R, "step_gflop": fl / 1e9, "head": "mean" if s.get("mean") else "softmax",
               "routed": NativeGruStep.routed(gru, R)}
        for k, ms in list(times.items()) + [("train_T_steps", train_t)]:
            ss = sorted(ms)
            out[k] = {"median_ms": ss[len(ss) // 2], "min_ms": ss[0], "max_ms": ss[-1]}
        out["native_tflops"] = fl / (out["native"]["median_ms"] * 1e-3) / 1e12
        out["native_speedup_vs_torch_step"] = (out["torch_step"]["median_ms"]
                                               / out["native"]["median_ms"])
        res[name] = out
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_recurrent.json"), "w", encoding="utf8") as fp:
            fp.write(line + "\n")


if __name__ == "__main__":
    main()
