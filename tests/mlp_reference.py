"""Float64 reference of the fused policy forward (csrc/wdb_mlp.cu), in plain numpy.

It restates, independently of the CUDA code:
  * bf16_rne: fp32 -> bf16 round-to-nearest-even on the bit pattern;
  * the weight blob (header, canonical K-major bf16 W1 / W2 / W3 = [head0; head1; value],
    zero padding to K1 and N3, fp32 biases) and the 128-row bf16 obs tiles;
  * the forward with the kernel's quantisation: bf16 operands, exact dot products, fp32 bias,
    ReLU, bf16 rounding of the hidden activations, float64 logits / softmax / value;
  * a generator of "exact" policies and observations: small integers times per-layer powers
    of two, so that every dot product the tensor cores compute in fp32 is exact.  forward()
    records what that premise needs (the span of every dot product, |logit|) and how much
    rounding the hidden layers really did, and `check_premise` asserts it.

Canonical K-major no-swizzle layout (wgmma core matrices of 8 rows x 16 bytes): element
(r, k) of a [R, K] bf16 matrix lives at byte (r / 8) * K * 16 + (k / 8) * 128 + (r % 8) * 16
+ (k % 8) * 2.  The obs tiles use it with K = K1 over rows padded to a multiple of 128.
"""
import numpy as np

SMEM_LIMIT = 227 * 1024          # dynamic shared memory a block may use on an H100
TILE_M = 128
HEADER_BYTES = 48                # struct MlpHeader: 12 int32; the blob's weights start at 128
SPAN_LIMIT = 2 ** 20             # 4 bits of margin below fp32's 24-bit significand
LOGIT_LIMIT = 16.0


def round_up(x, m):
    return (x + m - 1) // m * m


# ---------------------------------------------------------------- bf16 rounding
def bf16_bits(x):
    """float32 array -> uint16 bf16 bit patterns, round to nearest even (NaN -> 0x7FC0)."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(x), np.uint16(0x7FC0), r)


def bf16_to_f32(bits):
    return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def bf16_rne(x):
    """float32 array -> float32 array holding the bf16-rounded values."""
    return bf16_to_f32(bf16_bits(x))


# ---------------------------------------------------------------- layouts
def mlp_shape_ok(F, H, A0, A1):
    return (1 <= F <= 256 and 16 <= H <= 256 and H % 32 == 0 and 1 <= A0 <= 32
            and 0 <= A1 and A1 + 1 <= 32)


def blob_header(F, H, A0, A1):
    """The MlpHeader fields, in order: F, K1, H, A0, A1, N3, off_w1, off_w2, off_w3, off_b,
    total_bytes, pad."""
    K1, N3 = round_up(F, 16), round_up(A0 + A1 + 1, 16)
    off_w1 = 128
    off_w2 = off_w1 + H * K1 * 2
    off_w3 = off_w2 + H * H * 2
    off_b = off_w3 + N3 * H * 2
    total = round_up(off_b + (2 * H + N3) * 4, 16)
    return dict(F=F, K1=K1, H=H, A0=A0, A1=A1, N3=N3, off_w1=off_w1, off_w2=off_w2,
                off_w3=off_w3, off_b=off_b, total_bytes=total, pad=0)


def smem_bytes(F, H, A0, A1):
    """Dynamic shared memory of the forward kernel: weights + biases (rounded to 128 bytes),
    two warpgroup staging buffers (64 rows of the layer-1 A operand or of the N3 logits) and
    the weights' mbarrier."""
    hd = blob_header(F, H, A0, A1)
    w = round_up(hd["total_bytes"] - hd["off_w1"], 128)
    return w + 2 * 64 * max(hd["K1"] * 2, hd["N3"] * 4) + 16


def shape_supported(F, H, A0, A1):
    return mlp_shape_ok(F, H, A0, A1) and smem_bytes(F, H, A0, A1) <= SMEM_LIMIT


def max_supported_F(H, A0, A1):
    return max((F for F in range(1, 257) if shape_supported(F, H, A0, A1)), default=0)


def canonical(bits):
    """[R, K] uint16 (R, K multiples of 8) -> flat uint16 in the canonical K-major layout."""
    R, K = bits.shape
    return bits.reshape(R // 8, 8, K // 8, 8).transpose(0, 2, 1, 3).reshape(-1)


def _pad(a, rows, cols):
    out = np.zeros((rows, cols), dtype=np.float32)
    out[:a.shape[0], :a.shape[1]] = a
    return out


def pack_blob(F, H, A0, A1, params):
    """The weight blob wdb_mlp_pack_weights writes, as uint8.  Bytes HEADER_BYTES..127 are
    not part of the format (left 0 here)."""
    hd = blob_header(F, H, A0, A1)
    K1, N3 = hd["K1"], hd["N3"]
    out = np.zeros(hd["total_bytes"], dtype=np.uint8)
    out[:HEADER_BYTES] = np.array(list(hd.values()), dtype=np.int32).view(np.uint8)
    heads = [params["wh0"]] + ([params["wh1"]] if A1 > 0 else []) + [params["wv"]]
    w3 = np.concatenate([np.asarray(h, np.float32).reshape(-1, H) for h in heads])
    for off, w, rows, cols in ((hd["off_w1"], params["w1"], H, K1),
                               (hd["off_w2"], params["w2"], H, H),
                               (hd["off_w3"], w3, N3, H)):
        packed = canonical(bf16_bits(_pad(np.asarray(w, np.float32), rows, cols)))
        out[off:off + packed.nbytes] = packed.view(np.uint8)
    b3 = np.zeros(N3, np.float32)
    b3[:A0] = params["bh0"]
    if A1 > 0:
        b3[A0:A0 + A1] = params["bh1"]
    b3[A0 + A1] = np.asarray(params["bv"], np.float32).reshape(-1)[0]
    b = np.concatenate([np.asarray(params["b1"], np.float32), np.asarray(params["b2"], np.float32), b3])
    out[hd["off_b"]:hd["off_b"] + b.nbytes] = b.view(np.uint8)
    return out


def pack_obs_tiles(obs, F):
    """fp32 obs [rows, F] -> the bf16 A-operand tiles (uint8): 128-row tiles, K padded to
    K1 = round_up(F, 16) with zeros, rows past `rows` zero."""
    obs = np.asarray(obs, np.float32).reshape(-1, F)
    rows = obs.shape[0]
    return canonical(bf16_bits(_pad(obs, round_up(rows, TILE_M), round_up(F, 16)))).view(np.uint8)


# ---------------------------------------------------------------- forward
def _lowbit(x):
    """Largest power of two dividing every nonzero element of float64 array x (inf if none)."""
    x = np.abs(x[x != 0])
    if x.size == 0:
        return np.inf
    m, e = np.frexp(x)
    mi = (m * 2.0 ** 53).astype(np.int64)
    return float(np.min((mi & -mi).astype(np.float64) * np.exp2(e.astype(np.float64) - 53)))


def _softmax(z):
    z = z - z.max(-1, keepdims=True)
    e = np.exp(z)
    return e / e.sum(-1, keepdims=True)


def _layers(params):
    H = np.asarray(params["w2"]).shape[0]
    A0 = np.asarray(params["wh0"]).reshape(-1, H).shape[0]
    heads = [params["wh0"]] + ([params["wh1"]] if params.get("wh1") is not None else []) + [params["wv"]]
    w3 = np.concatenate([np.asarray(h, np.float32).reshape(-1, H) for h in heads])
    b3 = np.concatenate([np.asarray(params["bh0"], np.float32).reshape(-1)]
                        + ([np.asarray(params["bh1"], np.float32).reshape(-1)]
                           if params.get("wh1") is not None else [])
                        + [np.asarray(params["bv"], np.float32).reshape(-1)])
    q = lambda w: bf16_rne(np.asarray(w, np.float32)).astype(np.float64)   # noqa: E731
    f = lambda b: np.asarray(b, np.float32).astype(np.float64)             # noqa: E731
    return A0, [(q(params["w1"]), f(params["b1"])), (q(params["w2"]), f(params["b2"])),
                (q(w3), f(b3))]


def forward(obs, params, chunk=16384):
    """The kernel's forward in float64.  obs [rows, F] fp32; params: w1 [H, F], b1, w2 [H, H],
    b2, wh0 [A0, H], bh0, wh1 [A1, H] / bh1 (None for a single head), wv [1, H], bv [1].

    Returns probs0 [rows, A0], probs1 [rows, A1], value [rows] (float64) and the per-row
    premise statistics: span (largest over the three layers), max |logit|, and the number of
    positive hidden pre-activations that are not bf16-representable, that are exact RNE ties,
    and of negative hidden pre-activations."""
    obs = np.asarray(obs, np.float32)
    A0, layers = _layers(params)
    x_all = bf16_rne(obs).astype(np.float64)
    # grid step of the products of each layer over all rows: hidden activations after bf16
    # rounding stay multiples of the step of their layer's pre-activations
    steps, a_step = [], _lowbit(x_all)
    for w, b in layers:
        s = a_step * _lowbit(w)
        steps.append(s)
        assert np.all(np.mod(b, s) == 0), "bias off the product grid"
        a_step = s
    out = {k: [] for k in ("probs0", "probs1", "value", "span", "logit_max", "inexact",
                           "ties", "negative")}
    for r0 in range(0, obs.shape[0], chunk):
        a = x_all[r0:r0 + chunk]
        span = np.zeros(a.shape[0])
        inexact = np.zeros(a.shape[0], np.int64)
        ties = np.zeros(a.shape[0], np.int64)
        neg = np.zeros(a.shape[0], np.int64)
        for li, ((w, b), s) in enumerate(zip(layers, steps)):
            z = a @ w.T + b                     # exact: every partial sum is on the grid s
            span = np.maximum(span, ((np.abs(a) @ np.abs(w).T + np.abs(b)) / s).max(-1))
            if li == 2:
                break
            z32 = z.astype(np.float32)
            assert np.array_equal(z32.astype(np.float64), z), "pre-activation not fp32-exact"
            low = z32.view(np.uint32) & 0xFFFF
            pos = z32 > 0
            inexact += (pos & (low != 0)).sum(-1)
            ties += (pos & (low == 0x8000)).sum(-1)
            neg += (z32 < 0).sum(-1)
            a = bf16_rne(np.maximum(z32, np.float32(0))).astype(np.float64)
        nh = w.shape[0] - 1
        out["probs0"].append(_softmax(z[:, :A0]))
        out["probs1"].append(_softmax(z[:, A0:nh]) if nh > A0 else np.zeros((z.shape[0], 0)))
        out["value"].append(z[:, nh])
        out["span"].append(span)
        out["logit_max"].append(np.abs(z[:, :nh]).max(-1))
        out["inexact"].append(inexact)
        out["ties"].append(ties)
        out["negative"].append(neg)
    return {k: np.concatenate(v) for k, v in out.items()}


def check_premise(ref, rows=None):
    """Assert, over the first `rows` rows, what makes the reference exact (span <= 2^20,
    |logit| <= 16) and that the hidden layers really rounded: some positive pre-activations
    off the bf16 grid, at least one exact RNE tie, some ReLU zeros."""
    sl = slice(0, rows)
    span = ref["span"][sl].max()
    assert span <= SPAN_LIMIT, f"span {span} > 2^20"
    assert ref["logit_max"][sl].max() <= LOGIT_LIMIT, ref["logit_max"][sl].max()
    assert ref["inexact"][sl].sum() > 0, "no hidden pre-activation off the bf16 grid"
    assert ref["ties"][sl].sum() > 0, "no RNE tie among the hidden pre-activations"
    assert ref["negative"][sl].sum() > 0, "no negative hidden pre-activation"


# ---------------------------------------------------------------- exact inputs
def _sparse_ints(rng, n_out, n_in, nnz, mag):
    """[n_out, n_in] integers in [-mag, mag] \\ {0}, nnz of them per row."""
    w = np.zeros((n_out, n_in))
    nnz = min(nnz, n_in)
    for i in range(n_out):
        cols = rng.choice(n_in, nnz, replace=False)
        w[i, cols] = rng.integers(1, mag + 1, nnz) * rng.choice([-1, 1], nnz)
    return w


def exact_obs(rows, F, seed):
    """Observations on the grid 2^-4: integers in [-31, 31], and 1 in 16 an odd integer in
    [257, 383] (not bf16-representable; half of them RNE ties) -- the kernel rounds them."""
    rng = np.random.default_rng(seed)
    o = rng.integers(-31, 32, (rows, F)).astype(np.float64)
    big = rng.random((rows, F)) < 1 / 16
    o[big] = (2 * rng.integers(128, 192, int(big.sum())) + 1) * rng.choice([-1, 1], int(big.sum()))
    return (o * 2.0 ** -4).astype(np.float32)


def exact_params(F, H, A0, A1, seed, obs):
    """A policy whose forward on `obs` is exact in fp32 (see check_premise): sparse small
    integer weights, integer biases, per-layer power-of-two scales.  The head / value scale is
    the largest power of two that keeps every logit of `obs` within 16."""
    rng = np.random.default_rng(seed)
    p = {"w1": _sparse_ints(rng, H, F, 12, 7) * 2.0 ** -2,
         "b1": rng.integers(-400, 401, H) * 2.0 ** -6,
         "w2": _sparse_ints(rng, H, H, 10, 3) * 2.0 ** -3,
         "b2": rng.integers(-2000, 2001, H) * 2.0 ** -9}
    n3 = A0 + A1 + 1
    w3 = _sparse_ints(rng, n3, H, 8, 3)
    b3 = rng.integers(-2000, 2001, n3).astype(np.float64)
    p = {k: v.astype(np.float32) for k, v in p.items()}
    # raw integer logits on the layer-2 grid, then the scale
    p.update(wh0=w3[:A0].astype(np.float32), bh0=np.zeros(A0, np.float32),
             wh1=w3[A0:A0 + A1].astype(np.float32) if A1 else None,
             bh1=np.zeros(A1, np.float32) if A1 else None,
             wv=w3[A0 + A1:].astype(np.float32), bv=np.zeros(1, np.float32))
    step2 = 2.0 ** -4 * 2.0 ** -2 * 2.0 ** -3           # grid of the layer-2 pre-activations
    raw = forward(obs, p)
    lmax = max(raw["logit_max"].max(), 1.0)
    shift = int(np.floor(np.log2(LOGIT_LIMIT / (lmax + np.abs(b3).max() * step2))))
    sc = 2.0 ** shift
    p.update(wh0=(w3[:A0] * sc).astype(np.float32), bh0=(b3[:A0] * step2 * sc).astype(np.float32),
             wv=(w3[A0 + A1:] * sc).astype(np.float32),
             bv=(b3[A0 + A1:] * step2 * sc).astype(np.float32))
    if A1:
        p.update(wh1=(w3[A0:A0 + A1] * sc).astype(np.float32),
                 bh1=(b3[A0:A0 + A1] * step2 * sc).astype(np.float32))
    return p


def exact_case(F, H, A0, A1, rows, seed=0):
    """(obs [rows, F], params, reference) with the premise holding on row 0 alone and on
    every prefix of rows; deterministic in `seed`."""
    for s in range(seed, seed + 50):
        obs = exact_obs(rows, F, 1000 + s)
        params = exact_params(F, H, A0, A1, s, obs)
        ref = forward(obs, params)
        try:
            check_premise(ref, 1)
            check_premise(ref)
        except AssertionError:
            continue
        return obs, params, ref
    raise AssertionError(f"no exact case for {(F, H, A0, A1, rows)}")
