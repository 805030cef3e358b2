"""CPU checks of the float64 policy-forward reference (tests/mlp_reference.py) and of the
shape envelope the library accepts: the reference's bf16 rounding against torch, its packers
against the layout's address formula, its forward against a plain float64 MLP, and
wdb_mlp_blob_bytes / FusedPolicyForward.supported() against a restatement of the kernel's
shared-memory budget."""
import numpy as np
import pytest
import torch

import mlp_reference as R


def _torch_bf16_bits(x):
    return torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)


def test_bf16_rne_matches_torch_on_every_upper_half():
    upper = np.arange(1 << 16, dtype=np.uint32) << 16
    lows = np.array([0x0000, 0x7FFF, 0x8000, 0x8001, 0xFFFF], dtype=np.uint32)
    specials = np.array([0x00000000, 0x80000000, 0x00000001, 0x00008000, 0x00018000,
                         0x007FFFFF, 0x807FFFFF, 0x00800000, 0x7F800000, 0xFF800000,
                         0x7F7F7FFF, 0x7F7F8000, 0x7F7FFFFF, 0xFF7F8000, 0xFF7FFFFF],
                        dtype=np.uint32)
    x = np.concatenate([(upper[:, None] | lows[None, :]).reshape(-1), specials]).view(np.float32)
    got, want = R.bf16_bits(x), _torch_bf16_bits(x)
    nan = np.isnan(x)
    assert np.array_equal(got[~nan], want[~nan])
    assert np.isnan(R.bf16_to_f32(got[nan])).all()
    # the edges named explicitly: ties to even, +-0, subnormals, rounding up to inf
    f = lambda b: np.array([b], np.uint32).view(np.float32)          # noqa: E731
    assert R.bf16_bits(f(0x3F808000))[0] == 0x3F80                    # tie, even below
    assert R.bf16_bits(f(0x3F818000))[0] == 0x3F82                    # tie, even above
    assert R.bf16_bits(f(0x80000000))[0] == 0x8000                    # -0 keeps its sign
    assert R.bf16_bits(f(0x00008000))[0] == 0x0000                    # subnormal tie -> 0
    assert R.bf16_bits(f(0x00018000))[0] == 0x0002
    assert R.bf16_bits(f(0x7F7F8000))[0] == 0x7F80                    # finite -> +inf
    assert R.bf16_bits(f(0xFF7FFFFF))[0] == 0xFF80


def _unpack(buf, off, rows, K):
    """Read a [rows, K] bf16 matrix back through the address formula, element by element."""
    u16 = np.frombuffer(buf.tobytes(), dtype=np.uint16)
    out = np.empty((rows, K), np.uint16)
    for r in range(rows):
        for k in range(K):
            byte = off + (r // 8) * K * 16 + (k // 8) * 128 + (r % 8) * 16 + (k % 8) * 2
            out[r, k] = u16[byte // 2]
    return out


def _params(F, H, A0, A1, seed):
    rng = np.random.default_rng(seed)
    g = lambda *s: rng.standard_normal(s).astype(np.float32)         # noqa: E731
    return {"w1": g(H, F), "b1": g(H), "w2": g(H, H), "b2": g(H), "wh0": g(A0, H), "bh0": g(A0),
            "wh1": g(A1, H) if A1 else None, "bh1": g(A1) if A1 else None,
            "wv": g(1, H), "bv": g(1)}


@pytest.mark.parametrize("F,H,A0,A1", [(17, 32, 3, 5), (1, 32, 2, 0), (16, 64, 15, 0),
                                       (9, 32, 32, 31)])
def test_pack_blob_follows_the_address_formula(F, H, A0, A1):
    p = _params(F, H, A0, A1, F + H)
    blob = R.pack_blob(F, H, A0, A1, p)
    hd = R.blob_header(F, H, A0, A1)
    assert blob.size == hd["total_bytes"]
    assert list(blob[:R.HEADER_BYTES].view(np.int32)) == list(hd.values())
    K1, N3 = hd["K1"], hd["N3"]
    bits = lambda w, r, c: R.bf16_bits(np.pad(w, ((0, r - w.shape[0]), (0, c - w.shape[1]))))  # noqa: E731
    assert np.array_equal(_unpack(blob, hd["off_w1"], H, K1), bits(p["w1"], H, K1))
    assert np.array_equal(_unpack(blob, hd["off_w2"], H, H), bits(p["w2"], H, H))
    w3 = np.concatenate([p["wh0"]] + ([p["wh1"]] if A1 else []) + [p["wv"]])
    assert np.array_equal(_unpack(blob, hd["off_w3"], N3, H), bits(w3, N3, H))
    b = blob[hd["off_b"]:hd["off_b"] + (2 * H + N3) * 4].view(np.float32)
    b3 = np.zeros(N3, np.float32)
    b3[:A0 + A1 + 1] = np.concatenate([p["bh0"]] + ([p["bh1"]] if A1 else []) + [p["bv"]])
    assert np.array_equal(b, np.concatenate([p["b1"], p["b2"], b3]))


@pytest.mark.parametrize("F,rows", [(1, 1), (15, 130), (16, 64), (17, 129), (71, 9)])
def test_pack_obs_tiles_follows_the_address_formula(F, rows):
    obs = np.random.default_rng(rows).standard_normal((rows, F)).astype(np.float32)
    tiles = R.pack_obs_tiles(obs, F)
    K1, rp = R.round_up(F, 16), R.round_up(rows, 128)
    assert tiles.size == rp * K1 * 2
    want = np.zeros((rp, K1), np.uint16)
    want[:rows, :F] = R.bf16_bits(obs)
    assert np.array_equal(_unpack(tiles, 0, rp, K1), want)


def test_forward_equals_a_plain_float64_mlp_on_bf16_representable_values():
    """Whenever every input and every hidden value is on the bf16 grid, the quantisation the
    reference emulates is the identity: it must then equal an ordinary float64 MLP."""
    F, H, A0, A1, rows = 13, 64, 6, 5, 300
    rng = np.random.default_rng(3)
    ints = lambda lo, hi, *s: rng.integers(lo, hi + 1, s).astype(np.float32)   # noqa: E731
    obs = ints(-3, 3, rows, F) * 0.5
    p = {"w1": ints(-1, 1, H, F) * 0.25, "b1": ints(-4, 4, H) * 0.125,
         "w2": ints(-1, 1, H, H) * 0.125, "b2": ints(-2, 2, H) * 2.0 ** -6,
         "wh0": ints(-2, 2, A0, H), "bh0": ints(-2, 2, A0) * 0.25,
         "wh1": ints(-2, 2, A1, H), "bh1": ints(-2, 2, A1), "wv": ints(-3, 3, 1, H),
         "bv": ints(-9, 9, 1)}
    ref = R.forward(obs, p)
    assert ref["inexact"].sum() == 0 and ref["negative"].sum() > 0
    t = {k: torch.from_numpy(v).double() for k, v in p.items()}
    x = torch.from_numpy(obs).double()
    h = torch.relu(torch.nn.functional.linear(x, t["w1"], t["b1"]))
    h = torch.relu(torch.nn.functional.linear(h, t["w2"], t["b2"]))
    q0 = torch.softmax(torch.nn.functional.linear(h, t["wh0"], t["bh0"]), -1).numpy()
    q1 = torch.softmax(torch.nn.functional.linear(h, t["wh1"], t["bh1"]), -1).numpy()
    v = torch.nn.functional.linear(h, t["wv"], t["bv"])[:, 0].numpy()
    assert np.array_equal(ref["value"], v)
    np.testing.assert_allclose(ref["probs0"], q0, rtol=1e-13, atol=0)
    np.testing.assert_allclose(ref["probs1"], q1, rtol=1e-13, atol=0)


def test_exact_generator_premise_and_rounding():
    """The generator's cases carry their own proof: spans within 2^20, logits within 16, and
    hidden layers that round (off-grid values, a tie) and clip (negatives) on row 0 alone."""
    for shape in [(71, 256, 21, 21), (1, 32, 2, 0), (256, 128, 32, 31)]:
        obs, p, ref = R.exact_case(*shape, 300)
        R.check_premise(ref, 1)
        R.check_premise(ref)
        # a rounding of the hidden layer changes the result: the emulation is not a no-op
        assert ref["ties"][0] > 0 and ref["inexact"][0] > ref["ties"][0]


_PAIRS = [(32, 31), (33, 0), (1, 32), (21, 21), (32, 0), (1, 0), (15, 16), (0, 3), (2, 31)]


class _Stub:
    def __init__(self, F, H, A0, A1):
        self.is_deterministic = False
        self.fc = {"0": None, "1": None}
        self.fc_dims = [H, H]
        self.output_dims = [A0, A1] if A1 else [A0]
        self.flattened_obs_size = F


def test_envelope_matches_the_shared_memory_budget(wdb_lib):
    """wdb_mlp_blob_bytes accepts a shape exactly when it is valid and its weights plus the
    two staging buffers fit the 227 KB of shared memory a block may use, and then returns the
    blob size of the layout; FusedPolicyForward.supported() agrees."""
    from warp_drive_b200.training.models.fused_forward import FusedPolicyForward

    n_ok = 0
    for H in range(16, 289, 16):
        for A0, A1 in _PAIRS:
            for F in range(1, 258):
                ok = R.shape_supported(F, H, A0, A1)
                got = wdb_lib.wdb_mlp_blob_bytes(F, H, A0, A1)
                want = R.blob_header(F, H, A0, A1)["total_bytes"] if ok else -1
                assert got == want, (F, H, A0, A1, got, want)
                assert FusedPolicyForward.supported(_Stub(F, H, A0, A1)) == ok, (F, H, A0, A1)
                n_ok += ok
    assert n_ok > 0
    # the edges the GPU tests run at
    assert R.smem_bytes(71, 256, 21, 21) == 223504
    assert R.max_supported_F(256, 21, 21) == 96
    assert R.max_supported_F(224, 32, 0) == 144
