"""Dueling Q networks' host side without a GPU: the float64 fold (tests/dueling_reference.py)
against the streamed DuelingHead forward, the unfold against torch autograd through
DuelingHead.folded(), the model's keys and refusals, the run configs, the native envelope, the
bindings against the header, the new kernels' resource use, and the machine code of every
earlier update and rollout kernel."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import dueling_reference as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")


def _env(F=4, A=3):
    from test_ddpg_update_reference_cpu import _Env
    from warp_drive_b200.utils import spaces as sp

    env = _Env(F, 1)
    env.env.action_space = {0: sp.Discrete(A)}
    return env


def make_dueling(F, A, N, dims, S, seed=0, **extra):
    """A dueling FullyConnectedQ (N = 1) or FullyConnectedCategoricalQ (N atoms) in float64."""
    from warp_drive_b200.training.models.fully_connected import ModelFactory

    torch.manual_seed(seed)
    kind = "fully_connected_q" if N == 1 else "fully_connected_categorical_q"
    cfg = {"type": kind, "fc_dims": list(dims), "dueling": True, **extra}
    if S:
        cfg["stream_fc_dims"] = [S]
    if N > 1:
        cfg = {"num_atoms": N, "v_min": -1.0, "v_max": 1.0, **cfg}
    return ModelFactory.create(kind)(env=_env(F, A), model_config=cfg, policy="shared",
                                     policy_tag_to_agent_id_map={"shared": [0]}).double()


def _trunk(q):
    return [(q.fc[str(i)][0].weight.detach().numpy(), q.fc[str(i)][0].bias.detach().numpy())
            for i in range(len(q.fc))]


_SHAPES = [(A, N, S, dims) for A in (1, 2, 3) for N in (1, 2, 51) for S in (0, 8)
           for dims in ([], [7], [6, 5])]


@pytest.mark.parametrize("A,N,S,dims", _SHAPES)
def test_fold_is_the_streamed_forward(A, N, S, dims):
    q = make_dueling(4, A, N, dims, S)
    head = q.policy_head
    obs = torch.randn(13, 4, dtype=torch.float64)
    x = obs
    for i in range(len(q.fc)):
        x = q.fc[str(i)](x)
    want = head(x).detach().numpy()
    assert want.shape == (13, A * N)
    layers = ref.fold(ref.stream_params(head), A, N, S)
    got = ref.mlp(obs.numpy(), _trunk(q) + layers)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
    # folded() is the same map in torch
    for (w, b), (rw, rb) in zip(head.folded(), layers):
        np.testing.assert_allclose(w.detach().numpy(), rw, rtol=0, atol=1e-12)
        np.testing.assert_allclose(b.detach().numpy(), rb, rtol=0, atol=1e-12)
    # the mean combine: the mean over the actions of each output is the value stream's
    np.testing.assert_allclose(want.reshape(13, A, N).mean(1), head.value(x).detach().numpy(),
                               rtol=0, atol=1e-12)


@pytest.mark.parametrize("A,N,S", [(A, N, S) for A in (1, 2, 3) for N in (1, 2, 51)
                                   for S in (0, 8)])
def test_unfold_is_autograd_through_the_fold(A, N, S):
    q = make_dueling(4, A, N, [6], S, seed=1)
    head = q.policy_head
    folded = head.folded()
    rng = np.random.default_rng(A * 100 + N + S)
    grads = [(rng.standard_normal(tuple(w.shape)), rng.standard_normal(tuple(b.shape)))
             for w, b in folded]
    loss = sum((w * torch.from_numpy(gw)).sum() + (b * torch.from_numpy(gb)).sum()
               for (w, b), (gw, gb) in zip(folded, grads))
    loss.backward()
    want = ref.unfold(grads, A, N, S)
    (vh, vo), (ah, ao) = head.streams()
    named = {"value_o": vo, "adv_o": ao}
    if S:
        named.update(value_h=vh, adv_h=ah)
    assert set(want) == {k + s for k in named for s in "wb"}
    for k, layer in named.items():
        np.testing.assert_allclose(layer.weight.grad.numpy(), want[k + "w"], rtol=0, atol=1e-12)
        np.testing.assert_allclose(layer.bias.grad.numpy(), want[k + "b"], rtol=0, atol=1e-12)


def test_dueling_model_names_and_state_dict():
    q = make_dueling(4, 3, 1, [8], 5)
    assert q.dueling and q.stream_fc_dims == [5] and q.output_dims == [3]
    assert q.policy_head.is_dueling and q.policy_head.out_features == 3
    names = [n for n, _ in q.named_parameters()]
    assert names == ["fc.0.0.weight", "fc.0.0.bias",
                     "policy_head.value.0.weight", "policy_head.value.0.bias",
                     "policy_head.value.2.weight", "policy_head.value.2.bias",
                     "policy_head.advantage.0.weight", "policy_head.advantage.0.bias",
                     "policy_head.advantage.2.weight", "policy_head.advantage.2.bias"]
    assert list(q.state_dict()) == names          # parameters only, no folded buffers
    q0 = make_dueling(4, 3, 1, [8], 0)
    assert [n for n, _ in q0.named_parameters()][2:] == [
        "policy_head.value.weight", "policy_head.value.bias",
        "policy_head.advantage.weight", "policy_head.advantage.bias"]
    c = make_dueling(4, 2, 51, [8, 8], 16)
    assert c.policy_head.out_features == 102 and list(c.state_dict()) == [
        n for n, _ in c.named_parameters()]
    assert c.logits(torch.zeros(5, 4, dtype=torch.float64)).shape == (5, 2, 51)
    assert c.q_values(torch.zeros(5, 4, dtype=torch.float64)).shape == (5, 2)
    # a plain config keeps its plain head
    from warp_drive_b200.training.models.fully_connected import ModelFactory

    plain = ModelFactory.create("fully_connected_q")(
        env=_env(), model_config={"type": "fully_connected_q", "fc_dims": [8]}, policy="shared",
        policy_tag_to_agent_id_map={"shared": [0]})
    assert not plain.dueling and isinstance(plain.policy_head, torch.nn.Linear)


def test_dueling_model_refusals():
    from warp_drive_b200.training.models.fully_connected import ModelFactory

    def mk(kind, **extra):
        cfg = {"type": kind, "fc_dims": [8], **extra}
        if kind == "fully_connected_categorical_q":
            cfg.update(v_min=0, v_max=1)
        if kind == "fully_connected_quantile_q":
            cfg.update(num_quantiles=4)
        return ModelFactory.create(kind)(env=_env(), model_config=cfg, policy="shared",
                                         policy_tag_to_agent_id_map={"shared": [0]})

    for kind in ("fully_connected_q", "fully_connected_categorical_q"):
        for v in (1, 0, "true", None, [True]):
            with pytest.raises(ValueError, match="model.dueling"):
                mk(kind, dueling=v)
        for extra in ({"stream_fc_dims": [8]}, {"dueling": False, "stream_fc_dims": []}):
            with pytest.raises(ValueError, match="stream_fc_dims needs model.dueling"):
                mk(kind, **extra)
        for dims in ([8, 8], [0], [-1], [2.0], [True], 8, "8", None, (8,)):
            with pytest.raises(ValueError, match="stream_fc_dims is a list"):
                mk(kind, dueling=True, stream_fc_dims=dims)
        assert mk(kind, dueling=True, stream_fc_dims=[]).policy_head.stream_dim == 0
        assert not mk(kind, dueling=False).dueling
    for kind in ("fully_connected_quantile_q", "fully_connected_iqn"):
        for extra in ({"dueling": True}, {"stream_fc_dims": [8]}):
            with pytest.raises(ValueError, match=f"{kind} does not take model.dueling|"
                                                 f"{kind} does not take model.stream_fc_dims"):
                mk(kind, **extra)
        assert not mk(kind, dueling=False).dueling


def test_dueling_run_configs_load():
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.training.trainer import load_run_config
    from warp_drive_b200.training.trainer_dqn import (
        categorical_policy_settings, dqn_policy_settings, epsilon_schedule)

    for name, base_name in (("single_cartpole_dueling_dqn", "single_cartpole_dqn"),
                            ("single_cartpole_dueling_c51", "single_cartpole_c51")):
        cfg, base = load_run_config(name), load_run_config(base_name)
        pol, bpol = cfg["policy"]["shared"], base["policy"]["shared"]
        want_model = dict(bpol["model"], fc_dims=[64], dueling=True, stream_fc_dims=[32])
        assert pol["model"] == want_model, name
        assert {k: v for k, v in pol.items() if k != "model"} == {
            k: v for k, v in bpol.items() if k != "model"}
        assert cfg["sampler"] == base["sampler"]
        (categorical_policy_settings if "c51" in name else dqn_policy_settings)(pol)
        epsilon_schedule(cfg)
        q = ModelFactory.create(pol["model"]["type"])(
            env=_env(4, 2), model_config=pol["model"], policy="shared",
            policy_tag_to_agent_id_map={"shared": [0]})
        assert q.dueling and q.policy_head.stream_dim == 32
    c51 = load_run_config("single_cartpole_dueling_c51")["trainer"]
    base = load_run_config("single_cartpole_c51")["trainer"]
    assert c51["prioritized_replay"] is True and c51["n_step"] == 3
    assert {k: v for k, v in c51.items() if not k.startswith("prior")} == base
    assert load_run_config("single_cartpole_dueling_dqn")["trainer"] == load_run_config(
        "single_cartpole_dqn")["trainer"]


# ------------------------------------------------------------------------ the native envelope
def test_fused_envelope():
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.dqn import DQN, CategoricalDQN
    from warp_drive_b200.training.algorithms.fused_dqn import (
        fused_c51_supported, fused_dqn_supported, fused_dueling_supported)

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    dqn, c51 = DQN(0.99, n_step=3), CategoricalDQN(0.99, n_step=3)

    def ok(algo, N, dims, S, A=2, F=4):
        q = make_dueling(F, A, N, dims, S).float()
        return fused_dueling_supported(algo, q, 8, 1, 100, 256)

    # the run configs' shapes
    assert ok(dqn, 1, [64], 32) and ok(c51, 51, [64], 32)
    # at most three hidden layers in all, 2S <= 64, F <= 63
    assert ok(dqn, 1, [64, 64], 32) and not ok(dqn, 1, [64, 64, 64], 32)
    assert ok(dqn, 1, [64, 64, 64], 0) and ok(dqn, 1, [], 0) and ok(dqn, 1, [], 8)
    assert not ok(dqn, 1, [64], 48) and not ok(dqn, 1, [64], 33) and ok(dqn, 1, [8], 1)
    assert ok(dqn, 1, [8], 8, F=63) and not ok(dqn, 1, [8], 8, F=64)
    # C51's shared-memory cap applies to the folded network
    assert not ok(c51, 51, [64, 64], 32) and ok(c51, 51, [64], 32, A=3)
    # the plain passes refuse a dueling network (they would run the wrong head)
    for algo, N, supported in ((dqn, 1, fused_dqn_supported), (c51, 51, fused_c51_supported)):
        q = make_dueling(4, 2, N, [64], 32).float()
        assert supported(algo, q, 8, 1, 100, 256) is False
    # and the dueling one a plain network
    from c51_reference import make_c51_models

    plain, _ = make_c51_models(4, 2, [64, 64], N=51)
    assert fused_dueling_supported(c51, plain.float(), 8, 1, 100, 256) is False
    assert fused_c51_supported(c51, plain.float(), 8, 1, 100, 256) is True


def test_native_layers_refuse_a_dueling_head():
    from warp_drive_b200.training import fused_single_agent
    from warp_drive_b200.training.algorithms import fused_ddpg

    q = make_dueling(4, 2, 1, [8], 4)
    for layers in (fused_ddpg._layers, fused_single_agent._layers):
        with pytest.raises(TypeError, match="dueling"):
            layers(q)


def test_fold_supported_and_the_struct_ties_the_parameters():
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.fused_dqn import dueling_shape, folded_widths

    q = make_dueling(4, 3, 51, [16], 8)
    d = dueling_shape(q.policy_head)
    assert (d.n_actions, d.n_atoms, d.in_dim, d.stream_dim) == (3, 51, 16, 8)
    assert folded_widths(q) == [16, 16] and folded_widths(make_dueling(4, 3, 1, [16], 0)) == [16]
    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    L = wlib.load()
    assert L.wdb_dueling_fold_supported(ctypes.byref(d)) == 1
    assert L.wdb_dueling_unfold_grads_supported(ctypes.byref(d)) == 1
    for field, v in (("n_actions", 0), ("n_atoms", 0), ("in_dim", 0), ("stream_dim", -1)):
        bad = dueling_shape(q.policy_head)
        setattr(bad, field, v)
        assert L.wdb_dueling_fold_supported(ctypes.byref(bad)) == 0, field
        assert L.wdb_dueling_unfold_grads_supported(ctypes.byref(bad)) == 0, field
    # a NULL required pointer is refused before any CUDA call
    launches = L.wdb_launch_count()
    assert L.wdb_dueling_fold(None, ctypes.byref(d), None) == 1      # cudaErrorInvalidValue
    assert L.wdb_dueling_unfold_grads(None, ctypes.byref(d)) == 1
    assert L.wdb_launch_count() == launches


# ------------------------------------------------------------------------ bindings
def test_struct_layout_matches_the_header(tmp_path):
    from test_abi_layout_cpu import _c_fields
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    fields = _c_fields(header, "wdb_dueling_head")
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "wdb200.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(wdb_dueling_head));']
    lines += [f'  printf("{f} %zu\\n", offsetof(wdb_dueling_head, {f}));' for f in fields]
    lines += ["  return 0;", "}"]
    (tmp_path / "layout.c").write_text("\n".join(lines))
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(tmp_path / "layout"),
                    str(tmp_path / "layout.c")], check=True)
    out = subprocess.run([str(tmp_path / "layout")], check=True, capture_output=True,
                         text=True).stdout
    got = dict((k, int(v)) for k, v in (line.split() for line in out.splitlines()))
    cls = wlib.DuelingHead
    assert [n for n, _ in cls._fields_] == fields
    assert ctypes.sizeof(cls) == got["size"]
    for f in fields:
        assert getattr(cls, f).offset == got[f], f


def test_bindings_match_the_header():
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    want = {
        "wdb_dueling_fold_supported":
            r"int wdb_dueling_fold_supported\(const wdb_dueling_head \*head\);",
        "wdb_dueling_unfold_grads_supported":
            r"int wdb_dueling_unfold_grads_supported\(const wdb_dueling_head \*head\);",
        "wdb_dueling_fold":
            r"int wdb_dueling_fold\(void \*stream, const wdb_dueling_head \*head, "
            r"const wdb_dueling_head \*target\);",
        "wdb_dueling_unfold_grads":
            r"int wdb_dueling_unfold_grads\(void \*stream, const wdb_dueling_head \*head\);",
    }
    for name, pattern in want.items():
        assert re.search(pattern, header), name
    sig = wlib._SIGNATURES
    head = ctypes.POINTER(wlib.DuelingHead)
    assert sig["wdb_dueling_fold_supported"] == (ctypes.c_int, [head])
    assert sig["wdb_dueling_unfold_grads_supported"] == (ctypes.c_int, [head])
    assert sig["wdb_dueling_fold"] == (ctypes.c_int, [ctypes.c_void_p, head, head])
    assert sig["wdb_dueling_unfold_grads"] == (ctypes.c_int, [ctypes.c_void_p, head])


# ------------------------------------------------------------------------ ptxas / SASS
_DUELING_KERNELS = {
    "19dueling_fold_kernelE16wdb_dueling_headS0_",
    "21dueling_unfold_kernelE16wdb_dueling_head",
}

# The normalised SASS of the C51 update kernels and the categorical rollout kind, recorded at
# the parent commit with nvcc 12.9.
_C51_SASS_SHA256 = {
    "wdb_c51_update.cu": {
        "10c51_kernelE19wdb_dqn_update_argsNS_4PlanEiPKffPfPdPK4int2":
            "4f8d1e1b22fd680afb3d5a02624c7d4cf6a9dacff0681a9bf6243c8f3cbc3016",
        "22c51_prioritized_kernelE19wdb_dqn_update_argsNS_4PlanEiPKffPfPdPK4int2S3_":
            "bf9782964e03f5212aa9ae922a96c1ef155e37eac52c8ab588dbf9014ba84e2b",
        "18ddpg_reduce_kernelENS_6ReduceEPKfPKdPd":
            "bdb2c09a27e603435f6aab684188c6b044308552f7cb68d16c73f53fc4ef2718",
    },
    "wdb_sa_rollout_categorical.cu": {
        "17sa_rollout_kernelILi5EEEv14wdb_sa_rollout":
            "63b1d25c0003c59150d3d24b73ffc357140cc8527f344b1c5e063283ac494f1d",
    },
}


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_dueling_kernels_compile_without_spills_and_earlier_kernels_keep_their_code(tmp_path):
    from test_c51_cpu import _IQN_SASS_SHA256, _REDUCE
    from test_iqn_cpu import _QR_SASS_SHA256
    from test_qr_dqn_cpu import _KEPT_SASS_SHA256, _cubin, _sass_hashes

    stats, _ = _cubin(os.path.join(CSRC, "wdb_dueling.cu"), tmp_path)
    assert set(stats) == _DUELING_KERNELS
    for k in _DUELING_KERNELS:
        assert stats[k]["spill"] == (0, 0), (k, stats[k])
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
