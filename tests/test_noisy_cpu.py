"""Noisy Q networks' host side without a GPU: the model's keys, initialisation and refusals, the
numpy noise (tests/noisy_reference.py) against the documented counter layout, NoisyLinear's
materialized() against its factored forward, the float64 gradient map against autograd, the
noisy dueling head's fold, the run configs, the native envelope, the bindings against the
header, the new kernels' resource use and the machine code of every earlier kernel."""
import ctypes
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import dueling_reference as dref
import noisy_reference as ref
from test_dueling_cpu import _env

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")


def make_noisy(F, A, N, dims, S=None, seed=0, **extra):
    """A noisy FullyConnectedQ (N = 1) or FullyConnectedCategoricalQ (N atoms) in float64; S:
    None for a plain head, else the dueling stream width (0: no stream hidden layer)."""
    from warp_drive_b200.training.models.fully_connected import ModelFactory

    torch.manual_seed(seed)
    kind = "fully_connected_q" if N == 1 else "fully_connected_categorical_q"
    cfg = {"type": kind, "fc_dims": list(dims), "noisy": True, **extra}
    if S is not None:
        cfg.update(dueling=True, stream_fc_dims=[S] if S else [])
    if N > 1:
        cfg = {"num_atoms": N, "v_min": -1.0, "v_max": 1.0, **cfg}
    return ModelFactory.create(kind)(env=_env(F, A), model_config=cfg, policy="shared",
                                     policy_tag_to_agent_id_map={"shared": [0]}).double()


def _mk(kind, **extra):
    from warp_drive_b200.training.models.fully_connected import ModelFactory

    cfg = {"type": kind, "fc_dims": [8], **extra}
    if kind == "fully_connected_categorical_q":
        cfg.update(v_min=0, v_max=1)
    if kind == "fully_connected_quantile_q":
        cfg.update(num_quantiles=4)
    return ModelFactory.create(kind)(env=_env(), model_config=cfg, policy="shared",
                                     policy_tag_to_agent_id_map={"shared": [0]})


def _set_noise(q, rng):
    """Random f(eps) vectors in every noisy layer's buffers; returns them."""
    out = []
    for L in q.noisy_layers():
        fi = torch.from_numpy(rng.standard_normal(L.in_features))
        fo = torch.from_numpy(rng.standard_normal(L.out_features))
        L.noise_in, L.noise_out = fi, fo
        out.append((fi.numpy(), fo.numpy()))
    return out


# ------------------------------------------------------------------------ the model
def test_noisy_model_names_init_and_state_dict():
    from warp_drive_b200.training.models.fully_connected_q import NoisyLinear

    q = make_noisy(4, 3, 1, [8])
    assert q.noisy and q.noisy_sigma0 == 0.5 and isinstance(q.policy_head, NoisyLinear)
    names = [n for n, _ in q.named_parameters()]
    assert names == ["fc.0.0.weight", "fc.0.0.bias", "policy_head.weight_mu",
                     "policy_head.weight_sigma", "policy_head.bias_mu", "policy_head.bias_sigma"]
    assert list(q.state_dict()) == names               # no noise buffers in checkpoints
    assert [n for n, _ in q.named_buffers()] == ["policy_head.noise_in", "policy_head.noise_out"]
    # the trunk stays plain
    assert isinstance(q.fc["0"][0], torch.nn.Linear)
    d = make_noisy(4, 3, 51, [8], S=5, noisy_sigma0=0.25)
    assert len(d.noisy_layers()) == 4 and d.noisy_sigma0 == 0.25
    assert [n for n, _ in d.named_parameters()][2:6] == [
        "policy_head.value.0.weight_mu", "policy_head.value.0.weight_sigma",
        "policy_head.value.0.bias_mu", "policy_head.value.0.bias_sigma"]
    assert len(make_noisy(4, 3, 1, [8], S=0).noisy_layers()) == 2
    # initialisation: mu ~ U(+-1/sqrt(in)), sigma = sigma0 / sqrt(in)
    torch.manual_seed(0)
    L = NoisyLinear(400, 300, sigma0=0.4)
    bound = 1 / math.sqrt(400)
    for mu in (L.weight_mu.detach(), L.bias_mu.detach()):
        assert float(mu.abs().max()) <= bound
        assert abs(float(mu.mean())) < 0.05 * bound
    assert abs(float(L.weight_mu.detach().var()) - bound ** 2 / 3) < 0.02 * bound ** 2
    assert torch.all(L.weight_sigma == 0.4 * bound) and torch.all(L.bias_sigma == 0.4 * bound)
    # no noise set: the mean network
    x = torch.randn(5, 400)
    want = torch.nn.functional.linear(x, L.weight_mu, L.bias_mu)
    assert torch.equal(L(x), want)
    L.noise_in.normal_()
    assert torch.equal(L(x), want)          # buffers alone do not switch the noise on


def test_noisy_model_refusals():
    for kind in ("fully_connected_q", "fully_connected_categorical_q"):
        for v in (1, 0, "true", None, [True]):
            with pytest.raises(ValueError, match="model.noisy is true or false"):
                _mk(kind, noisy=v)
        for extra in ({"noisy_sigma0": 0.5}, {"noisy": False, "noisy_sigma0": 0.5}):
            with pytest.raises(ValueError, match="noisy_sigma0 needs model.noisy"):
                _mk(kind, **extra)
        for s in (0, -0.1, float("inf"), float("nan"), True, "0.5", None, [0.5]):
            with pytest.raises(ValueError, match="noisy_sigma0 is a finite number > 0"):
                _mk(kind, noisy=True, noisy_sigma0=s)
        assert _mk(kind, noisy=True, noisy_sigma0=2).noisy_sigma0 == 2.0
        assert not _mk(kind, noisy=False).noisy
    for kind in ("fully_connected_quantile_q", "fully_connected_iqn"):
        for extra in ({"noisy": True}, {"noisy_sigma0": 0.5}):
            with pytest.raises(ValueError, match=f"{kind} does not take model.noisy"):
                _mk(kind, **extra)
        assert not _mk(kind, noisy=False).noisy


# ------------------------------------------------------------------------ the noise
def test_noise_counter_layout_and_statistics():
    import oracle

    # the documented words, and a second word no replay or sampler counter reaches
    assert ref.counter(1, 7, 9, 2, 5) == [7, 0x4E010000, 9, (2 << 16) | 2]
    assert ref.counter(0, (3 << 32) + 4, 0, 0, 0) == [4, 0x4E000003, 0, 0]
    # element e: words (x, y) for even e, (z, w) for odd e of one Philox block
    seed = 12345678901
    f, bar = ref.noise(seed, ref.ACTING, 17, 3, 1, 6)
    key = [seed & 0xFFFFFFFF, seed >> 32]
    for e in range(6):
        w = oracle.philox4x32_10([17, 0x4E010000, 3, (1 << 16) | (e >> 1)], key)
        a, b = (int(w[0]), int(w[1])) if e % 2 == 0 else (int(w[2]), int(w[3]))
        u1, u2 = a * 2.0 ** -32 + 2.0 ** -33, b * 2.0 ** -32 + 2.0 ** -33
        x = math.sqrt(-2 * math.log(u1)) * math.cos(2 * math.pi * u2)
        assert f[e] == pytest.approx(math.copysign(math.sqrt(abs(x)), x), rel=1e-5)
        assert 0 < bar[e] <= 1e-6 * abs(f[e]) + 1e-300
    # domains, counts, rows and layers draw different values
    base = ref.noise(seed, 0, 5, 0, 0, 8)[0]
    for args in ((seed, 1, 5, 0, 0), (seed, 0, 6, 0, 0), (seed, 0, 5, 1, 0), (seed, 0, 5, 0, 1),
                 (seed + 1, 0, 5, 0, 0)):
        assert not np.array_equal(ref.noise(*args, 8)[0], base), args
    # f(eps) of N(0, 1) draws: E f = 0, E f^2 = E|eps| = sqrt(2 / pi)
    big = np.concatenate([ref.noise(7, 0, c, 0, 0, 500)[0] for c in range(4)])
    assert abs(big.mean()) < 0.06
    assert abs((big ** 2).mean() - math.sqrt(2 / math.pi)) < 0.05


# ------------------------------------------------------------------------ materialize / grads
# (A, N, S, H): S None is a plain head
_SHAPES = [(A, N, S, H) for A in (1, 3) for N in (1, 13) for S in (None, 0, 8) for H in (1, 7, 64)]


def _ids(shapes):
    return [f"A{a}_N{n}_S{'-' if s is None else s}_H{h}" for a, n, s, h in shapes]


@pytest.mark.parametrize("A,N,S,H", _SHAPES, ids=_ids(_SHAPES))
def test_materialized_is_the_factored_forward(A, N, S, H):
    q = make_noisy(4, A, N, [H], S, seed=A + N + H)
    rng = np.random.default_rng(A * 1000 + N * 10 + H)
    x = torch.from_numpy(rng.standard_normal((11, H)))
    for L in q.noisy_layers():
        fi = torch.from_numpy(rng.standard_normal((11, L.in_features)))
        fo = torch.from_numpy(rng.standard_normal((11, L.out_features)))
        xin = torch.from_numpy(rng.standard_normal((11, L.in_features)))
        p = [t.detach().numpy() for t in (L.weight_mu, L.weight_sigma, L.bias_mu, L.bias_sigma)]
        with torch.no_grad():
            L.noise = (fi, fo)
            rows = L(xin).numpy()
            L.noise = None
            for r in range(11):                # row r's own effective layer
                w, b = L.materialized(fi[r], fo[r])
                want = xin[r].numpy() @ w.numpy().T + b.numpy()
                np.testing.assert_allclose(rows[r], want, rtol=0, atol=1e-12)
                rw, rb = ref.materialize(*p, fi[r].numpy(), fo[r].numpy())
                np.testing.assert_allclose(w.numpy(), rw, rtol=0, atol=1e-12)
                np.testing.assert_allclose(b.numpy(), rb, rtol=0, atol=1e-12)
        np.testing.assert_allclose(rows, ref.factored(xin.numpy(), *p, fi.numpy(), fo.numpy()),
                                   rtol=0, atol=1e-12)
    # the whole head under one sample (the buffers): the update's forward
    _set_noise(q, rng)
    for L in q.noisy_layers():
        L.noise = (L.noise_in, L.noise_out)
    with torch.no_grad():
        got = q.policy_head(x).numpy()
    for L in q.noisy_layers():
        L.noise = None
    if S is None:
        w, b = q.policy_head.materialized()
        want = x.numpy() @ w.detach().numpy().T + b.detach().numpy()
    else:                                      # materialize, then fold
        p = _materialized_streams(q.policy_head)
        want = dref.mlp(x.numpy(), dref.fold(p, A, N, S))
        for (fw, fb), (rw, rb) in zip(q.policy_head.folded(), dref.fold(p, A, N, S)):
            np.testing.assert_allclose(fw.detach().numpy(), rw, rtol=0, atol=1e-12)
            np.testing.assert_allclose(fb.detach().numpy(), rb, rtol=0, atol=1e-12)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)


def _materialized_streams(head):
    """dueling_reference.stream_params of a noisy DuelingHead's materialized() layers."""
    out = {}
    for prefix, (hidden, output) in zip(("value_", "adv_"), head.streams()):
        for name, layer in (("h", hidden), ("o", output)):
            if layer is not None:
                w, b = layer.materialized()
                out[prefix + name + "w"] = w.detach().numpy()
                out[prefix + name + "b"] = b.detach().numpy()
    return out


@pytest.mark.parametrize("A,N,S,H", _SHAPES[::3], ids=_ids(_SHAPES[::3]))
def test_grads_map_is_autograd_through_materialized(A, N, S, H):
    q = make_noisy(4, A, N, [H], S, seed=3)
    rng = np.random.default_rng(A + N + H)
    noise = _set_noise(q, rng)
    layers = q.noisy_layers()
    eff = [L.materialized() for L in layers]
    g = [(rng.standard_normal(tuple(w.shape)), rng.standard_normal(tuple(b.shape)))
         for w, b in eff]
    loss = sum((w * torch.from_numpy(gw)).sum() + (b * torch.from_numpy(gb)).sum()
               for (w, b), (gw, gb) in zip(eff, g))
    loss.backward()
    for L, (gw, gb), (fi, fo) in zip(layers, g, noise):
        want = ref.grads(gw, gb, fi, fo)
        for p, w in zip((L.weight_mu, L.weight_sigma, L.bias_mu, L.bias_sigma), want):
            np.testing.assert_allclose(p.grad.numpy(), w, rtol=0, atol=1e-12)


# ------------------------------------------------------------------------ configs
def test_noisy_run_configs_load():
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import (
        categorical_policy_settings, dqn_policy_settings, epsilon_schedule)

    for name, base_name, extra in (
            ("single_cartpole_noisy_dqn", "single_cartpole_dqn",
             {"noisy": True, "noisy_sigma0": 0.5}),
            ("single_cartpole_rainbow", "single_cartpole_dueling_c51", {"noisy": True})):
        cfg, base = load_run_config(name), load_run_config(base_name)
        pol, bpol = cfg["policy"]["shared"], base["policy"]["shared"]
        assert pol["model"] == dict(bpol["model"], **extra), name
        assert {k: v for k, v in pol.items() if k != "model"} == {
            k: v for k, v in bpol.items() if k != "model"}
        assert cfg["sampler"] == {"params": {"epsilon": 0}}
        assert cfg["trainer"] == base["trainer"] and cfg["env"] == base["env"]
        assert cfg["saving"]["name"] == name
        (categorical_policy_settings if "rainbow" in name else dqn_policy_settings)(pol)
        assert epsilon_schedule(cfg).get_param_value(10 ** 6) == 0
        q = ModelFactory.create(pol["model"]["type"])(
            env=_env(4, 2), model_config=pol["model"], policy="shared",
            policy_tag_to_agent_id_map={"shared": [0]})
        assert q.noisy and len(q.noisy_layers()) == (4 if "rainbow" in name else 1)


# ------------------------------------------------------------------------ the native envelope
def _lib_or_skip():
    from warp_drive_b200 import lib as wlib

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    return wlib


def test_fused_envelope_and_refusals():
    _lib_or_skip()
    from warp_drive_b200.training import fused_single_agent
    from warp_drive_b200.training.algorithms import fused_ddpg
    from warp_drive_b200.training.algorithms.dqn import DQN, CategoricalDQN
    from warp_drive_b200.training.algorithms.fused_dqn import (
        fused_c51_supported, fused_dqn_supported, fused_dueling_supported,
        fused_noisy_supported)

    dqn, c51 = DQN(0.99, n_step=3), CategoricalDQN(0.99, n_step=3)

    def ok(algo, N, dims, S=None, A=2, F=4):
        q = make_noisy(F, A, N, dims, S).float()
        return fused_noisy_supported(algo, q, 8, 1, 100, 256)

    # the run configs' shapes
    assert ok(dqn, 1, [64, 64]) and ok(c51, 51, [64], 32)
    assert ok(dqn, 1, [64, 64, 64]) and not ok(dqn, 1, [64, 64, 64, 64])
    assert ok(dqn, 1, []) and ok(dqn, 1, [8], F=63) and not ok(dqn, 1, [8], F=64)
    assert ok(dqn, 1, [64], 32) and not ok(dqn, 1, [64], 48) and not ok(dqn, 1, [64, 64, 64], 32)
    assert not ok(c51, 51, [64, 64], 32)                  # C51's shared-memory cap
    # the plain and dueling passes refuse a noisy network: they would run mu alone
    for algo, N, S, supported in ((dqn, 1, None, fused_dqn_supported),
                                  (c51, 51, None, fused_c51_supported),
                                  (dqn, 1, 32, fused_dueling_supported),
                                  (c51, 51, 32, fused_dueling_supported)):
        q = make_noisy(4, 2, N, [64], S).float()
        assert supported(algo, q, 8, 1, 100, 256) is False
    # and the noisy one a plain network
    plain = _mk("fully_connected_q").float()
    assert fused_noisy_supported(dqn, plain, 8, 1, 100, 256) is False
    q = make_noisy(4, 2, 1, [8])
    for layers in (fused_ddpg._layers, fused_single_agent._layers):
        with pytest.raises(TypeError, match="noisy"):
            layers(q)


def test_noisy_struct_shape_and_null_pointers():
    wlib = _lib_or_skip()
    from warp_drive_b200.training.algorithms.fused_dqn import NoisyHead

    q = make_noisy(4, 3, 51, [16], 8)
    n = NoisyHead.shape(q)
    assert n.n_layers == 4
    assert [(n.layer[i].in_dim, n.layer[i].out_dim) for i in range(4)] == [
        (16, 8), (8, 51), (16, 8), (8, 153)]
    L = wlib.load()
    assert L.wdb_noisy_supported(ctypes.byref(n)) == 1
    for field, v in (("n_layers", 0), ("n_layers", 5)):
        bad = NoisyHead.shape(q)
        setattr(bad, field, v)
        assert L.wdb_noisy_supported(ctypes.byref(bad)) == 0, (field, v)
    for in_dim, out_dim in ((0, 4), (4, 0), (1 << 16, 1 << 16 + 1)):
        bad = NoisyHead.shape(q)
        bad.layer[1].in_dim, bad.layer[1].out_dim = in_dim, out_dim
        assert L.wdb_noisy_supported(ctypes.byref(bad)) == 0, (in_dim, out_dim)
    # NULL pointers and bad arguments are refused before any CUDA call
    launches = L.wdb_launch_count()
    assert L.wdb_noisy_draw(None, ctypes.byref(n), 1, 0, 0, 0, 1) == 1
    assert L.wdb_noisy_materialize(None, ctypes.byref(n), None, 1, 0) == 1
    assert L.wdb_noisy_grads(None, ctypes.byref(n)) == 1
    assert L.wdb_launch_count() == launches


# ------------------------------------------------------------------------ bindings
def test_struct_layout_matches_the_header(tmp_path):
    from test_abi_layout_cpu import _c_fields
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    assert "#define WDB_NOISY_MAX_LAYERS 4" in header and wlib.NOISY_MAX_LAYERS == 4
    got = {}
    for struct in ("wdb_noisy_layer", "wdb_noisy_net"):
        fields = _c_fields(header, struct)
        lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "wdb200.h"',
                 "int main(void) {", f'  printf("size %zu\\n", sizeof({struct}));']
        lines += [f'  printf("{f} %zu\\n", offsetof({struct}, {f}));' for f in fields]
        lines += ["  return 0;", "}"]
        (tmp_path / "layout.c").write_text("\n".join(lines))
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o",
                        str(tmp_path / "layout"), str(tmp_path / "layout.c")], check=True)
        out = subprocess.run([str(tmp_path / "layout")], check=True, capture_output=True,
                             text=True).stdout
        got[struct] = (fields, dict((k, int(v)) for k, v in (l.split() for l in out.splitlines())))
    for struct, cls in (("wdb_noisy_layer", wlib.NoisyLayer), ("wdb_noisy_net", wlib.NoisyNet)):
        fields, offsets = got[struct]
        assert [n for n, _ in cls._fields_] == fields
        assert ctypes.sizeof(cls) == offsets["size"]
        for f in fields:
            assert getattr(cls, f).offset == offsets[f], f


def test_bindings_match_the_header():
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    flat = re.sub(r"\s+", " ", header)
    want = {
        "wdb_noisy_supported": r"int wdb_noisy_supported\(const wdb_noisy_net \*net\);",
        "wdb_noisy_draw":
            r"int wdb_noisy_draw\(void \*stream, const wdb_noisy_net \*net, unsigned long long "
            r"seed, int domain, unsigned long long count, int row0, int n_rows\);",
        "wdb_noisy_materialize":
            r"int wdb_noisy_materialize\(void \*stream, const wdb_noisy_net \*online, const "
            r"wdb_noisy_net \*target, unsigned long long seed, unsigned long long update\);",
        "wdb_noisy_grads": r"int wdb_noisy_grads\(void \*stream, const wdb_noisy_net \*net\);",
    }
    for name, pattern in want.items():
        assert re.search(pattern, flat), name
    sig = wlib._SIGNATURES
    net = ctypes.POINTER(wlib.NoisyNet)
    i, vp, ull = ctypes.c_int, ctypes.c_void_p, ctypes.c_ulonglong
    assert sig["wdb_noisy_supported"] == (i, [net])
    assert sig["wdb_noisy_draw"] == (i, [vp, net, ull, i, ull, i, i])
    assert sig["wdb_noisy_materialize"] == (i, [vp, net, net, ull, ull])
    assert sig["wdb_noisy_grads"] == (i, [vp, net])


# ------------------------------------------------------------------------ ptxas / SASS
_SA_NOISY = "17sa_rollout_kernelILi6EEEv14wdb_sa_rollout"
_NOISY_KERNELS = {
    "17noisy_draw_kernelE13wdb_noisy_netyiyii",
    "24noisy_materialize_kernelE13wdb_noisy_netS0_yy",
    "18noisy_grads_kernelE13wdb_noisy_net",
}


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_noisy_kernels_compile_without_spills_and_earlier_kernels_keep_their_code(tmp_path):
    from test_c51_cpu import _IQN_SASS_SHA256, _REDUCE
    from test_dueling_cpu import _C51_SASS_SHA256
    from test_iqn_cpu import _QR_SASS_SHA256
    from test_qr_dqn_cpu import _KEPT_SASS_SHA256, _cubin, _sass_hashes

    stats, _ = _cubin(os.path.join(CSRC, "wdb_noisy.cu"), tmp_path)
    assert set(stats) == _NOISY_KERNELS
    for k in _NOISY_KERNELS:
        assert stats[k]["spill"] == (0, 0), (k, stats[k])
    # the one-launch rollout's noisy Q kind, in a translation unit of its own
    stats, _ = _cubin(os.path.join(CSRC, "wdb_sa_rollout_noisy.cu"), tmp_path)
    assert _SA_NOISY in stats
    for k, v in stats.items():
        assert v["spill"] == (0, 0), (k, v)
    version = subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout
    if "release 12.9" not in version:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    want = dict(_KEPT_SASS_SHA256)
    want["wdb_ddpg_update.cu"] = dict(want["wdb_ddpg_update.cu"], **_QR_SASS_SHA256)
    want["wdb_iqn_update.cu"] = dict(_IQN_SASS_SHA256, **{
        _REDUCE: want["wdb_ddpg_update.cu"][_REDUCE]})
    want.update(_C51_SASS_SHA256)
    for src, kept in want.items():
        _, cubin = _cubin(os.path.join(CSRC, src), tmp_path)
        got = _sass_hashes(cubin)
        assert set(got) == set(kept), src      # no kernel lost or added
        assert got == kept, src


def test_one_launch_noisy_kind_envelope():
    wlib = _lib_or_skip()
    from warp_drive_b200.training.fused_single_agent import FusedSingleAgentRollout

    L = wlib.load()

    def ok(dims):
        arr = (ctypes.c_int * 6)(*(dims + [0] * (6 - len(dims))))
        return L.wdb_single_agent_rollout_noisy_supported(len(dims) - 2, arr)

    # CartPole [64, 64]: 4 610 mu floats + 130 sigma floats
    assert ok([4, 64, 64, 2]) == 1 and ok([6, 64, 64, 64, 3]) == 1 and ok([4, 2]) == 1
    assert ok([4, 64, 64, 64, 8]) == 1 and ok([4, 64, 64, 64, 9]) == 0   # one output per lane
    assert ok([4, 64, 65, 2]) == 0 and ok([4, 64, 64, 64, 64, 2]) == 0
    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    assert re.search(r"int wdb_single_agent_rollout_noisy_supported\(int n_hidden, "
                     r"const int \*dims\);", header)
    assert wlib._SIGNATURES["wdb_single_agent_rollout_noisy_supported"] == (
        ctypes.c_int, [ctypes.c_int, ctypes.POINTER(ctypes.c_int)])

    class _W:                                # the parts of an EnvWrapper eligible() reads
        n_agents = 1

        class env:
            name = "ClassicControlCartPoleEnv"

    def eligible(q):
        return FusedSingleAgentRollout.eligible(_W, {"shared": q}, {"shared": [0]})

    assert eligible(make_noisy(4, 2, 1, [64, 64]).float())
    assert not eligible(make_noisy(4, 2, 51, [64]).float())          # noisy C51: per step
    assert not eligible(make_noisy(4, 2, 1, [64], S=32).float())     # noisy dueling: per step
