"""Generate tests/golden/mlp_forward_bits.npz: the exact output bytes of the wgmma policy
forward (csrc/wdb_mlp.cu) on two seeded cases.  Run on an H100:

    python tests/golden/make_mlp_forward_golden.py [OUT.npz]

Only the outputs are stored; `inputs(name)` regenerates the weights and observations from
the case's seed.  tests/test_gpu_mlp_bits.py requires the forward to reproduce them byte for
byte through both entries (fp32 observations and bf16 obs tiles), so a change to the kernel's
schedule cannot change a single bit of what the rollout samples from.

  config2      the headline policy shape (F = 71, H = 256, two 21-way heads), 4000 rows on 3
               CTAs: every CTA loops over ~10 tiles and the last tile is partial (its second
               warpgroup has no rows);
  single_head  (144, 224, 32, 0): one head + value, K1 = 144 (more observation chunks per
               thread than the config-2 shape).

Weights follow nn.Linear's default initialisation (uniform +-1/sqrt(fan_in)); observations
look like TagContinuous ones: values in [-1, 1], 0/1 flag columns, and rows whose trailing
neighbour features are zero.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(HERE, "mlp_forward_bits.npz")
CASES = {
    "config2": {"shape": (71, 256, 21, 21), "rows": 4000, "max_ctas": 3, "seed": 20260},
    "single_head": {"shape": (144, 224, 32, 0), "rows": 1000, "max_ctas": 2, "seed": 20261},
}
ENTRIES = ("fp32", "tiles")


def inputs(name):
    """(params, obs) of a case: float32 numpy arrays."""
    c = CASES[name]
    F, H, A0, A1 = c["shape"]
    rs = np.random.RandomState(c["seed"])

    def linear(n_out, n_in):
        bound = 1.0 / np.sqrt(n_in)
        return (rs.uniform(-bound, bound, (n_out, n_in)).astype(np.float32),
                rs.uniform(-bound, bound, n_out).astype(np.float32))

    p = {}
    p["w1"], p["b1"] = linear(H, F)
    p["w2"], p["b2"] = linear(H, H)
    p["wh0"], p["bh0"] = linear(A0, H)
    if A1:
        p["wh1"], p["bh1"] = linear(A1, H)
    p["wv"], p["bv"] = linear(1, H)
    rows = c["rows"]
    obs = rs.uniform(-1.0, 1.0, (rows, F)).astype(np.float32)
    obs[:, ::7] = rs.randint(0, 2, (rows, len(range(0, F, 7))))
    empty = rs.rand(rows) < 0.1
    obs[empty, F - F // 3:] = 0.0
    return p, obs


def run(name, entry):
    """The forward's outputs {probs0, probs1 (two-head shapes), values} as numpy arrays."""
    import torch

    from warp_drive_b200 import lib as wlib

    c = CASES[name]
    F, H, A0, A1 = c["shape"]
    rows = c["rows"]
    p, obs = inputs(name)
    L = wlib.load()
    dev = torch.device("cuda")
    t = {k: torch.from_numpy(v).to(dev).contiguous() for k, v in p.items()}
    x = torch.from_numpy(obs).to(dev)
    blob = torch.zeros(int(L.wdb_mlp_blob_bytes(F, H, A0, A1)), dtype=torch.uint8, device=dev)
    s = wlib.stream_ptr()
    wlib.check(L.wdb_mlp_pack_weights(
        s, wlib.ptr(blob), *[wlib.ptr(t.get(k)) for k in
                             ("w1", "b1", "w2", "b2", "wh0", "bh0", "wh1", "bh1", "wv", "bv")],
        F, H, A0, A1), "mlp_pack_weights")
    p0 = torch.full((rows, A0), -7.0, device=dev)
    p1 = torch.full((rows, A1), -7.0, device=dev) if A1 else None
    v = torch.full((rows,), -7.0, device=dev)
    wlib.check(L.wdb_set_option(b"mlp_max_ctas", c["max_ctas"]), "set_option")
    try:
        if entry == "fp32":
            wlib.check(L.wdb_mlp_policy_forward(s, wlib.ptr(blob), F, H, A0, A1, wlib.ptr(x), rows,
                                                wlib.ptr(p0), wlib.ptr(p1), wlib.ptr(v)),
                       "mlp_policy_forward")
        else:
            tiles = torch.zeros(int(L.wdb_mlp_obs_tiles_bytes(F, rows)), dtype=torch.uint8,
                                device=dev)
            wlib.check(L.wdb_mlp_pack_obs(s, wlib.ptr(x), rows, F, wlib.ptr(tiles)),
                       "mlp_pack_obs")
            wlib.check(L.wdb_mlp_policy_forward_tiles(s, wlib.ptr(blob), F, H, A0, A1,
                                                      wlib.ptr(tiles), rows, wlib.ptr(p0),
                                                      wlib.ptr(p1), wlib.ptr(v)),
                       "mlp_policy_forward_tiles")
    finally:
        wlib.check(L.wdb_set_option(b"mlp_max_ctas", 0), "set_option")
    torch.cuda.synchronize()
    out = {"probs0": p0, "values": v}
    if A1:
        out["probs1"] = p1
    return {k: a.cpu().numpy() for k, a in out.items()}


def main(path=GOLDEN):
    arrays = {}
    for name in CASES:
        ref = run(name, "fp32")
        got = run(name, "tiles")
        for k in ref:   # both entries stage the same bf16 A operand
            assert ref[k].tobytes() == got[k].tobytes(), (name, k)
            assert np.isfinite(ref[k]).all(), (name, k)
            arrays[f"{name}_{k}"] = ref[k]
    np.savez_compressed(path, **arrays)
    print(f"wrote {path}: " + ", ".join(f"{k} {a.shape}" for k, a in arrays.items()))


if __name__ == "__main__":
    main(*sys.argv[1:])
