"""The config-2 policy forward (FastShape schedule of csrc/wdb_mlp.cu) at every tile-ownership
edge, bit for bit against the one-slice-at-a-time schedule (AnyShape) on the same inputs.

The FastShape kernel carries work from one tile of a warpgroup into the next (the next
tile's observations are loaded during layer 2), so the edges where a warpgroup has no next
tile, or no tile at all, are covered here: the empty second half of a last tile
(rows % 128 in (0, 64]), rows < 64, and CTAs with unequal tile counts.  The AnyShape
reference is the pair kernel (wdb_mlp_policy_forward_pair always runs the runtime-shape
schedule).  Both schedules accumulate every output in the same order, layer 3 included (one
m64n48k16 per k-step here, three m64n16k16 there), so their outputs agree byte for byte.
Both FastShape entries are covered: fp32 observations and bf16 obs tiles.  Every launch must
complete and must leave the guard row past `rows` untouched.
"""
import ctypes
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location(
    "make_mlp_forward_golden", os.path.join(HERE, "golden", "make_mlp_forward_golden.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)

SHAPE = (71, 256, 21, 21)        # the config-2 policies: K1 = 80, H = 256, N3 = 48
SENTINEL = -1234.5

# (rows, max_ctas): max_ctas 0 = one CTA per tile up to every SM
CASES = (
    [(r, 0) for r in (1, 37, 63, 64, 65, 100, 127, 128)]
    + [(5 * 128 + d, c) for d in (1, 63, 64, 65, 127) for c in (0, 2)]
    + [(17 * 128 + d, c) for d in (1, 63, 64, 65, 127) for c in (3, 7)]
    + [(300 * 128 + 63, 0), (300 * 128 + 65, 0), (2 * 132 * 128 + 64, 0), (2 * 132 * 128, 5)]
)

_STATE = {}


def _setup():
    """{lib, blob, x (the observations on the device)} for the largest case, built once."""
    if not _STATE:
        import torch

        from warp_drive_b200 import lib as wlib

        F, H, A0, A1 = SHAPE
        p, obs = G.inputs("config2")
        rows = max(r for r, _ in CASES)
        obs = np.resize(obs, (rows, F))
        L = wlib.load()
        dev = torch.device("cuda")
        t = {k: torch.from_numpy(v).to(dev).contiguous() for k, v in p.items()}
        blob = torch.zeros(int(L.wdb_mlp_blob_bytes(F, H, A0, A1)), dtype=torch.uint8,
                           device=dev)
        wlib.check(L.wdb_mlp_pack_weights(
            wlib.stream_ptr(), wlib.ptr(blob),
            *[wlib.ptr(t.get(k)) for k in
              ("w1", "b1", "w2", "b2", "wh0", "bh0", "wh1", "bh1", "wv", "bv")],
            F, H, A0, A1), "mlp_pack_weights")
        _STATE.update(lib=L, blob=blob, x=torch.from_numpy(obs).to(dev))
    return _STATE


def _outputs(rows):
    import torch

    _, _, A0, A1 = SHAPE
    full = lambda *s: torch.full(s, SENTINEL, device="cuda")               # noqa: E731
    return full(rows + 1, A0), full(rows + 1, A1), full(rows + 1)


def _anyshape(rows):
    """The runtime-shape schedule's outputs: policy A of the pair kernel over `rows` rows
    (policy B, one row on one CTA, is a dummy)."""
    from warp_drive_b200 import lib as wlib

    s = _setup()
    F, H, A0, A1 = SHAPE
    out = _outputs(rows)
    dummy = _outputs(1)
    pair = wlib.MlpPair()
    for w, (n, o) in enumerate(((rows, out), (1, dummy))):
        pair.blob[w] = wlib.ptr(s["blob"])
        pair.F[w], pair.H[w], pair.A0[w], pair.A1[w] = F, H, A0, A1
        pair.obs[w] = wlib.ptr(s["x"])
        pair.rows[w] = n
        pair.probs0[w], pair.probs1[w], pair.values[w] = (wlib.ptr(t) for t in o)
    pair.ctas_b = 1
    pair.flags = 0
    wlib.check(s["lib"].wdb_mlp_policy_forward_pair(wlib.stream_ptr(), ctypes.byref(pair)),
               "mlp_policy_forward_pair")
    return out


def _fastshape(rows, max_ctas, entry):
    import torch

    from warp_drive_b200 import lib as wlib

    s = _setup()
    L = s["lib"]
    F, H, A0, A1 = SHAPE
    p0, p1, v = _outputs(rows)
    st = wlib.stream_ptr()
    x = s["x"]
    wlib.check(L.wdb_set_option(b"mlp_max_ctas", max_ctas), "set_option")
    try:
        if entry == "fp32":
            wlib.check(L.wdb_mlp_policy_forward(st, wlib.ptr(s["blob"]), F, H, A0, A1,
                                                wlib.ptr(x), rows, wlib.ptr(p0), wlib.ptr(p1),
                                                wlib.ptr(v)), "mlp_policy_forward")
        else:
            tiles = torch.zeros(int(L.wdb_mlp_obs_tiles_bytes(F, rows)), dtype=torch.uint8,
                                device="cuda")
            wlib.check(L.wdb_mlp_pack_obs(st, wlib.ptr(x), rows, F, wlib.ptr(tiles)),
                       "mlp_pack_obs")
            wlib.check(L.wdb_mlp_policy_forward_tiles(st, wlib.ptr(s["blob"]), F, H, A0, A1,
                                                      wlib.ptr(tiles), rows, wlib.ptr(p0),
                                                      wlib.ptr(p1), wlib.ptr(v)),
                       "mlp_policy_forward_tiles")
    finally:
        wlib.check(L.wdb_set_option(b"mlp_max_ctas", 0), "set_option")
    return p0, p1, v


@pytest.mark.parametrize("entry", ("fp32", "tiles"))
@pytest.mark.parametrize("rows,max_ctas", CASES)
def test_fastshape_matches_anyshape_bits(wdb_lib, rows, max_ctas, entry):
    import torch

    want = _anyshape(rows)
    got = _fastshape(rows, max_ctas, entry)
    torch.cuda.synchronize()        # raises if a launch faulted
    for name, g, w in zip(("probs0", "probs1", "values"), got, want):
        g, w = g.cpu().numpy(), w.cpu().numpy()
        assert (g[rows] == SENTINEL).all(), (rows, max_ctas, entry, name, "guard row written")
        assert np.isfinite(w[:rows]).all(), (rows, name, "reference not written")
        diff = np.flatnonzero(g[:rows].view(np.uint32) != w[:rows].view(np.uint32))
        assert diff.size == 0, (
            f"rows={rows} max_ctas={max_ctas} {entry}/{name}: {diff.size} of {w[:rows].size} "
            f"differ, first at flat index {diff[0]}: {g[:rows].flat[diff[0]]!r} vs "
            f"{w[:rows].flat[diff[0]]!r}")
