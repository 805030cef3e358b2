"""The wgmma policy forward (csrc/wdb_mlp.cu) pinned to the float64 reference of
tests/mlp_reference.py across the shape envelope the library accepts.

Why the bars can be this tight.  The inputs are small integers times per-layer powers of two
(mlp_reference.exact_case), so:
  * every product of every dot product is a multiple of the layer's grid step, and the sum of
    their magnitudes plus the bias is at most 2^20 steps (the "span", asserted for every dot
    product of every row that runs): every partial sum, in any order and with any alignment
    that keeps 24 bits, is exact in fp32, and so is the bias add;
  * the bf16 rounding of a hidden activation is then the round-to-nearest-even of an exactly
    known value (the reference does it on the bit pattern); the cases are checked to contain
    hidden pre-activations off the bf16 grid, exact ties and negatives (ReLU);
  * the logits, and so the value, are exact: the value must match bit for bit.
The only inexact step left is the softmax, with |logit| <= 16 (asserted):
  * x * log2(e) is rounded: half an ulp of |x log2 e| <= 23.1 is 2^-20;
  * lg - max is rounded: half an ulp of a number below 46.2 is 2^-19;
    together <= 3 * 2^-20 in the exponent, i.e. 3 * 2^-20 * ln 2 = 2.0e-6 relative;
  * ex2.approx.ftz: about 2 ulp = 2.4e-7 relative;
  * the sum of at most 32 terms: <= 31 * 2^-24 = 1.8e-6 relative;
  * one IEEE reciprocal and one multiply (the library is built without fast-math): 1.2e-7.
A probability is a term over the sum: <= 2.2e-6 + (2.2e-6 + 1.8e-6) + 1.2e-7 = 6.4e-6
relative.  The bar is 1e-5 relative per probability.  A wrong descriptor, fragment, bias or
column is an O(1) error under it.
"""
import numpy as np
import pytest
import torch

import mlp_reference as R

pytestmark = pytest.mark.gpu

PROB_RTOL = 1e-5
SENTINEL = -1234.5

# rows = 2 full waves of 132 CTAs plus a partial tile
WAVES_ROWS = 2 * 132 * 128 + 77
CONFIG2 = (71, 256, 21, 21)
# the largest F that fits for each (H, heads) edge; F + 1 does not fit
EDGE_SHAPES = [(R.max_supported_F(H, A0, A1), H, A0, A1)
               for H in (192, 224, 256) for A0, A1 in ((21, 21), (32, 31))] + [(144, 224, 32, 0)]
FORWARD_SHAPES = [CONFIG2, (1, 32, 2, 0), (16, 96, 15, 0), (17, 160, 15, 16),
                  (256, 128, 32, 31)] + EDGE_SHAPES
SWEEP_SHAPES = [CONFIG2, (96, 256, 21, 21), (144, 224, 32, 0)]

_CASES = {}


def _case(shape):
    """(obs, params, reference) of `shape`, WAVES_ROWS rows (every test uses a prefix)."""
    if shape not in _CASES:
        _CASES[shape] = R.exact_case(*shape, WAVES_ROWS if shape in SWEEP_SHAPES else 1000)
    return _CASES[shape]


class _Policy(torch.nn.Module):
    """The attributes FusedPolicyForward reads, holding the given parameters."""

    def __init__(self, F, H, A0, A1, params):
        super().__init__()
        self.flattened_obs_size, self.fc_dims = F, [H, H]
        self.output_dims = [A0, A1] if A1 else [A0]
        self.is_deterministic = False
        lin = lambda w, b: self._linear(params[w], params[b])              # noqa: E731
        self.fc = torch.nn.ModuleDict({"0": torch.nn.Sequential(lin("w1", "b1"), torch.nn.ReLU()),
                                       "1": torch.nn.Sequential(lin("w2", "b2"), torch.nn.ReLU())})
        self.policy_head = torch.nn.ModuleList(
            [lin("wh0", "bh0")] + ([lin("wh1", "bh1")] if A1 else []))
        self.vf_head = lin("wv", "bv")

    @staticmethod
    def _linear(w, b):
        w = np.asarray(w, np.float32)
        m = torch.nn.Linear(w.shape[1], w.shape[0])
        with torch.no_grad():
            m.weight.copy_(torch.from_numpy(w))
            m.bias.copy_(torch.from_numpy(np.asarray(b, np.float32).reshape(-1)))
        return m


def _fused(shape, params):
    from warp_drive_b200.training.models.fused_forward import FusedPolicyForward

    model = _Policy(*shape, params).cuda()
    assert FusedPolicyForward.supported(model)
    return FusedPolicyForward(model)


def _outputs(rows, A0, A1):
    """probs0, probs1 (None for a single head), values: one guard row past `rows`."""
    full = lambda *s: torch.full(s, SENTINEL, device="cuda")               # noqa: E731
    return full(rows + 1, A0), (full(rows + 1, A1) if A1 else None), full(rows + 1)


def _check(ref, rows, p0, p1, v, what):
    torch.cuda.synchronize()
    R.check_premise(ref, rows)
    outs = [("probs0", p0), ("probs1", p1)] + ([("value", v)] if v is not None else [])
    for name, t in outs:
        if t is None:
            continue
        assert (t[rows] == SENTINEL).all(), (what, name, "guard row written")
        got = t[:rows].cpu().numpy().astype(np.float64)
        want = ref[name][:rows]
        if name == "value":
            bad = np.flatnonzero(got != want.astype(np.float32))
            assert bad.size == 0, (what, "value", bad[:5], got[bad[:5]], want[bad[:5]])
        else:
            err = np.abs(got - want) / want
            assert err.max() <= PROB_RTOL, (what, name, err.max(),
                                            np.unravel_index(err.argmax(), err.shape))


# ---------------------------------------------------------------- layouts, byte for byte
def _off_grid(rng, *shape):
    """fp32 values that are mostly not bf16-representable: normals, exact ties (both
    parities), -0, subnormals, and finite values that round to +-inf."""
    x = rng.standard_normal(shape).astype(np.float32)
    u = x.reshape(-1).view(np.uint32)
    n = u.size
    pick = rng.random(n)
    u[pick < 0.25] = (u[pick < 0.25] & 0xFFFF0000) | 0x8000                   # ties
    specials = np.array([0x80000000, 0x00000001, 0x00008000, 0x00018000, 0x807FFFFF,
                         0x7F7F8000, 0xFF7FFFFF], dtype=np.uint32)
    u[rng.choice(n, min(n, len(specials)), replace=False)] = specials[:min(n, len(specials))]
    return x


@pytest.mark.parametrize("shape", [CONFIG2, (1, 32, 2, 0), (16, 96, 15, 0), (17, 160, 15, 16),
                                   (256, 128, 32, 31), (9, 32, 5, 0)])
def test_weight_blob_is_byte_exact(shape):
    """refresh() writes the header, the canonical W1 / W2 / W3 with their zero padding and the
    fp32 biases exactly as the reference packs them (bf16 round to nearest even)."""
    F, H, A0, A1 = shape
    rng = np.random.default_rng(sum(shape))
    p = {"w1": _off_grid(rng, H, F), "b1": _off_grid(rng, H), "w2": _off_grid(rng, H, H),
         "b2": _off_grid(rng, H), "wh0": _off_grid(rng, A0, H), "bh0": _off_grid(rng, A0),
         "wh1": _off_grid(rng, A1, H) if A1 else None, "bh1": _off_grid(rng, A1) if A1 else None,
         "wv": _off_grid(rng, 1, H), "bv": _off_grid(rng, 1)}
    fwd = _fused(shape, p)
    fwd.blob.fill_(0xFF)
    fwd.refresh()
    got = fwd.blob.cpu().numpy()
    want = R.pack_blob(F, H, A0, A1, p)
    assert got.size == want.size
    assert np.array_equal(got[:R.HEADER_BYTES], want[:R.HEADER_BYTES])
    bad = np.flatnonzero(got[128:] != want[128:])
    assert bad.size == 0, (bad.size, bad[:8] + 128)


@pytest.mark.parametrize("F", [1, 15, 16, 17, 71, 256])
def test_obs_tiles_are_byte_exact(F):
    """wdb_mlp_pack_obs overwrites every byte of the tiles with the reference's layout: bf16
    RNE of the observations, zero K padding, zero rows past the last observation."""
    from warp_drive_b200 import lib as wlib

    L = wlib.load()
    rng = np.random.default_rng(F)
    for rows in (1, 63, 64, 65, 127, 128, 129, 1000):
        obs = _off_grid(rng, rows, F)
        tiles = torch.full((int(L.wdb_mlp_obs_tiles_bytes(F, rows)),), 0xFF, dtype=torch.uint8,
                           device="cuda")
        wlib.check(L.wdb_mlp_pack_obs(wlib.stream_ptr(), wlib.ptr(torch.from_numpy(obs).cuda()),
                                      rows, F, wlib.ptr(tiles)), "mlp_pack_obs")
        got = tiles.cpu().numpy()
        want = R.pack_obs_tiles(obs, F)
        bad = np.flatnonzero(got != want)
        assert got.size == want.size and bad.size == 0, (rows, bad.size, bad[:8])


# ---------------------------------------------------------------- exact forward
@pytest.mark.parametrize("entry", ["obs", "tiles"])
@pytest.mark.parametrize("shape", FORWARD_SHAPES)
def test_exact_forward(shape, entry):
    """Every shape at 1 row (the second warpgroup idle) and 1000 rows, through the fp32-obs
    entry point or through pack_obs + forward_tiles."""
    F, H, A0, A1 = shape
    obs, params, ref = _case(shape)
    fwd = _fused(shape, params)
    for rows in (1, 1000):
        x = torch.from_numpy(obs[:rows]).cuda()
        p0, p1, v = _outputs(rows, A0, A1)
        if entry == "tiles":
            tiles = torch.full((fwd.tiles_bytes(rows),), 0xFF, dtype=torch.uint8, device="cuda")
            fwd.pack_obs(x, tiles)
            fwd.forward_tiles(tiles, rows, p0, p1, v)
        else:
            fwd(x, p0, p1, v)
        _check(ref, rows, p0, p1, v, (shape, entry, rows))


@pytest.mark.parametrize("shape", SWEEP_SHAPES)
def test_exact_forward_rows_and_ctas(shape):
    """Partial warpgroups and tiles, and persistent CTAs walking many tiles with the same
    staging buffers (max_ctas = 1: one CTA does every tile)."""
    F, H, A0, A1 = shape
    obs, params, ref = _case(shape)
    fwd = _fused(shape, params)
    x_all = torch.from_numpy(obs).cuda()
    for rows in (1, 63, 64, 65, 128, 129, WAVES_ROWS):
        for max_ctas in (0, 1, 5):
            p0, p1, v = _outputs(rows, A0, A1)
            fwd(x_all[:rows], p0, p1, v, max_ctas=max_ctas)
            _check(ref, rows, p0, p1, v, (shape, rows, max_ctas))


def test_exact_forward_200k_rows():
    """Config 2 at 200 000 rows (rows drawn from the exact case's pool, so the reference is a
    gather), through both entry points."""
    F, H, A0, A1 = CONFIG2
    obs, params, ref = _case(CONFIG2)
    rows = 200_000
    idx = np.random.default_rng(5).integers(0, obs.shape[0], rows)
    big = {k: v[idx] for k, v in ref.items()}
    fwd = _fused(CONFIG2, params)
    x = torch.from_numpy(obs[idx]).cuda()
    p0, p1, v = _outputs(rows, A0, A1)
    fwd(x, p0, p1, v)
    _check(big, rows, p0, p1, v, "obs")
    tiles = torch.full((fwd.tiles_bytes(rows),), 0xFF, dtype=torch.uint8, device="cuda")
    fwd.pack_obs(x, tiles)
    p0, p1, v = _outputs(rows, A0, A1)
    fwd.forward_tiles(tiles, rows, p0, p1, v)
    _check(big, rows, p0, p1, v, "tiles")


@pytest.mark.parametrize("stable", [False, True])
def test_exact_pair_forward(stable):
    """Two different exact policies in one grid (config 2 and an H = 96 single-head policy),
    with the CTA split chosen by the library or forced: each side matches the reference."""
    from warp_drive_b200.training.models.fused_forward import forward_pair

    shapes, rows = [CONFIG2, (16, 96, 15, 0)], [WAVES_ROWS, 1000]
    cases = [_case(s) for s in shapes]
    fw = [_fused(s, c[1]) for s, c in zip(shapes, cases)]
    xs = [torch.from_numpy(c[0][:n]).cuda() for c, n in zip(cases, rows)]
    for ctas_b in (0, 1, 40):
        outs = [_outputs(n, s[2], s[3])[:2] for s, n in zip(shapes, rows)]
        forward_pair(fw[0], fw[1], xs[0], xs[1], [o for o in outs[0] if o is not None],
                     [o for o in outs[1] if o is not None], ctas_b=ctas_b, weights_stable=stable)
        for w in range(2):
            _check(cases[w][2], rows[w], outs[w][0], outs[w][1], None, (w, ctas_b, stable))


@pytest.mark.parametrize("shape", EDGE_SHAPES)
def test_just_past_the_envelope_is_refused(shape):
    """F + 1 beyond an edge shape does not fit the shared memory: supported() says so, and
    both forward entry points return an error without launching."""
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.models.fused_forward import FusedPolicyForward

    F, H, A0, A1 = shape
    assert R.shape_supported(F, H, A0, A1) and not R.shape_supported(F + 1, H, A0, A1)
    F += 1
    rng = np.random.default_rng(0)
    g = lambda *s: rng.standard_normal(s).astype(np.float32)              # noqa: E731
    p = {"w1": g(H, F), "b1": g(H), "w2": g(H, H), "b2": g(H), "wh0": g(A0, H), "bh0": g(A0),
         "wh1": g(A1, H) if A1 else None, "bh1": g(A1) if A1 else None, "wv": g(1, H), "bv": g(1)}
    assert not FusedPolicyForward.supported(_Policy(F, H, A0, A1, p))
    L = wlib.load()
    assert L.wdb_mlp_blob_bytes(F, H, A0, A1) == -1
    rows = 256
    blob = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    obs = torch.zeros(rows, F, device="cuda")
    tiles = torch.zeros(int(L.wdb_mlp_obs_tiles_bytes(F, rows)), dtype=torch.uint8, device="cuda")
    p0, p1, v = _outputs(rows, A0, A1)
    torch.cuda.synchronize()
    n0 = wlib.launch_count()
    for fn, inp in ((L.wdb_mlp_policy_forward, obs), (L.wdb_mlp_policy_forward_tiles, tiles)):
        rc = fn(wlib.stream_ptr(), wlib.ptr(blob), F, H, A0, A1, wlib.ptr(inp), rows,
                wlib.ptr(p0), wlib.ptr(p1), wlib.ptr(v))
        assert rc != 0
    assert wlib.launch_count() == n0
    torch.cuda.synchronize()
    assert (p0 == SENTINEL).all() and (v == SENTINEL).all()
