"""CPU tests of the recurrent A2C / PPO policy (FullyConnectedGRU): config keys, refusals and
state_dict names; the cell against nn.GRUCell; forward_sequence against a loop of step with the
reset rule; the float64 reference (tests/recurrent_reference.py) against torch autograd; the
feed-forward eligibility checks; the sequence minibatch rows; the native forward's envelope
query, struct layout and bindings; and what ptxas makes of csrc/wdb_recurrent.cu."""
import ctypes
import os
import re
import shutil
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import recurrent_reference as ref  # noqa: E402
from test_abi_layout_cpu import _c_fields  # noqa: E402

CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")


def _stub_env(action_space, F=5, obs_space=None, T=4):
    from warp_drive_b200.utils.spaces import Box

    inner = SimpleNamespace(observation_space={0: obs_space or Box(-1, 1, shape=(F,))},
                            action_space={0: action_space})
    dm = SimpleNamespace(get_shape=lambda name: (T, 1, 1, F))
    return SimpleNamespace(env=inner, cuda_data_manager=dm, n_agents=1)


def _model(fc_dims=(8, 8), gru_dim=None, heads=(3, 4), F=5, dtype=torch.float32, seed=0):
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils.spaces import Discrete, MultiDiscrete

    space = Discrete(heads[0]) if len(heads) == 1 else MultiDiscrete(list(heads))
    cfg = {"type": "fully_connected_gru", "fc_dims": list(fc_dims)}
    if gru_dim is not None:
        cfg["gru_dim"] = gru_dim
    torch.manual_seed(seed)
    m = ModelFactory.create("fully_connected_gru")(_stub_env(space, F), cfg, "p", {"p": [0]})
    return m.to(dtype)


# ------------------------------------------------------------------------ config and refusals
def test_config_keys_and_state_dict_names():
    m = _model(fc_dims=(8, 6), gru_dim=7)
    assert m.is_recurrent and m.hidden_size == 7
    names = list(m.state_dict())
    assert names == ["fc.0.0.weight", "fc.0.0.bias", "fc.1.0.weight", "fc.1.0.bias",
                     "gru.weight_ih", "gru.weight_hh", "gru.bias_ih", "gru.bias_hh",
                     "policy_head.0.weight", "policy_head.0.bias", "policy_head.1.weight",
                     "policy_head.1.bias", "vf_head.weight", "vf_head.bias"]
    assert tuple(m.gru.weight_ih.shape) == (21, 6) and tuple(m.gru.weight_hh.shape) == (21, 7)
    assert _model(fc_dims=(8, 6)).hidden_size == 6            # gru_dim defaults to fc_dims[-1]
    assert len(_model(fc_dims=(), gru_dim=5).fc) == 0
    with pytest.raises(ValueError):
        _model(fc_dims=())
    with pytest.raises(RuntimeError):
        m(torch.zeros(2, 5))


def test_refusals():
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils.spaces import Box, Dict, Discrete, MultiDiscrete

    cls = ModelFactory.create("fully_connected_gru")
    cfg = {"type": "fully_connected_gru", "fc_dims": [8]}
    with pytest.raises(ValueError, match="Box action"):
        cls(_stub_env(Box(-1, 1, shape=(2,))), cfg, "p", {"p": [0]})
    masked = Dict({"obs": Box(-1, 1, shape=(5,)), "action_mask": Box(0, 1, shape=(3,))})
    with pytest.raises(ValueError, match="action mask"):
        cls(_stub_env(Discrete(3), obs_space=masked), cfg, "p", {"p": [0]})
    with pytest.raises(ValueError, match="normalize_observations"):
        cls(_stub_env(MultiDiscrete([3, 3])), dict(cfg, normalize_observations=True), "p",
            {"p": [0]})
    # algorithms other than A2C / PPO: refused where the trainer builds the model
    from warp_drive_b200.training.trainer import Trainer

    fake = SimpleNamespace(config={"policy": {"p": {"algorithm": "DQN"}}})
    with pytest.raises(ValueError, match="A2C or PPO"):
        Trainer._build_model(fake, "p", cfg)


# ------------------------------------------------------------------------ the torch forwards
def test_cell_equals_nn_grucell_bit_for_bit():
    m = _model(fc_dims=(8,), gru_dim=6)
    cell = torch.nn.GRUCell(8, 6)
    cell.load_state_dict({k[4:]: v for k, v in m.state_dict().items() if k.startswith("gru.")})
    x, h = torch.randn(11, 8), torch.randn(11, 6)
    assert torch.equal(m.gru(x, h), cell(x, h))
    obs = torch.randn(11, 5)
    probs, h_new = m.step(obs, h)
    assert torch.equal(h_new, cell(m.trunk(obs), h))
    for k, head in enumerate(m.policy_head):
        assert torch.equal(probs[k], torch.softmax(head(h_new), -1))


def test_forward_sequence_equals_a_loop_of_step_with_the_reset_rule():
    """(float64: the loop's GEMMs over one step's rows and the sequence's over all T steps may
    order their sums differently)"""
    m = _model(dtype=torch.float64)
    T, E, Np = 7, 3, 2
    obs = torch.randn(T, E, Np, 5, dtype=torch.float64)
    h0 = torch.randn(E, Np, 8, dtype=torch.float64)
    done = torch.tensor(np.random.default_rng(1).integers(0, 3, (T, E)), dtype=torch.int32)
    done[2, 1] = 1
    probs, values = m.forward_sequence(obs, h0, done)
    h = h0
    for t in range(T):
        if t > 0:
            h = m.reset_hidden(h, done[t - 1])
        p, hn = m.step(obs[t].reshape(E * Np, -1), h.reshape(E * Np, -1))
        h = hn.view(E, Np, -1)
        for k in range(2):
            torch.testing.assert_close(p[k].view(E, Np, -1), probs[k][t], rtol=0, atol=1e-12)
        torch.testing.assert_close(m.vf_head(h)[..., 0], values[t], rtol=0, atol=1e-12)


@pytest.mark.parametrize("fc_dims,heads", [((8, 8), (3, 4)), ((6,), (5,)), ((), (2, 3))])
def test_float64_reference_equals_torch_autograd(fc_dims, heads):
    m = _model(fc_dims=fc_dims, gru_dim=7, heads=heads, dtype=torch.float64, seed=3)
    T, E, Np = 6, 3, 2
    rng = np.random.default_rng(5)
    obs = rng.normal(size=(T, E, Np, 5))
    h0 = rng.normal(size=(E, Np, 7))
    done = rng.integers(0, 3, (T, E)) * (rng.random((T, E)) < 0.4)
    cp = [rng.normal(size=(T, E, Np, a)) for a in heads]
    cv = rng.normal(size=(T, E, Np))
    P = ref.params_of(m)
    probs, values, _ = ref.forward_sequence(P, obs, h0, done)
    h0_t = torch.tensor(h0, requires_grad=True)
    tp, tv = m.forward_sequence(torch.tensor(obs), h0_t, torch.tensor(done))
    for a, b in zip(probs, tp):
        np.testing.assert_allclose(a, b.detach().numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(values, tv.detach().numpy(), rtol=0, atol=1e-12)
    loss = sum((torch.tensor(c) * p).sum() for c, p in zip(cp, tp)) + (torch.tensor(cv) * tv).sum()
    loss.backward()
    G = ref.gradients(P, obs, h0, done, cp, cv)
    for name, p in m.named_parameters():
        np.testing.assert_allclose(G[name], p.grad.numpy(), rtol=0, atol=1e-12, err_msg=name)
    assert h0_t.grad is None                     # no gradient flows into the start state


def test_step_bounds_are_positive_and_small():
    m = _model(dtype=torch.float64)
    P = ref.params_of(m)
    rng = np.random.default_rng(0)
    probs, h, eprobs, eh = ref.step_with_bounds(P, rng.normal(size=(9, 5)),
                                                rng.normal(size=(9, 8)))
    assert (eh > 0).all() and eh.max() < 1e-5
    for p, e in zip(probs, eprobs):
        assert (e > 0).all() and (e / np.maximum(p, 1e-30)).max() < 1e-4


# ------------------------------------------------------------------------ eligibility checks
def _built_fc(fc_dims, heads, F=5):
    from warp_drive_b200.training.models.fully_connected import FullyConnected
    from warp_drive_b200.utils.spaces import MultiDiscrete

    return FullyConnected(_stub_env(MultiDiscrete(list(heads)), F),
                          {"type": "fully_connected", "fc_dims": list(fc_dims)}, "p", {"p": [0]})


def test_feed_forward_paths_refuse_a_recurrent_model_and_keep_accepting_the_rest():
    from warp_drive_b200.training.fused_single_agent import FusedSingleAgentRollout
    from warp_drive_b200.training.models import fused_mlp_train
    from warp_drive_b200.training.models.fused_forward import FusedPolicyForward
    from warp_drive_b200.training.rollout import RolloutEngine

    gru = _model(fc_dims=(64, 64), heads=(21, 21))
    ff = _built_fc((64, 64), (21, 21))
    assert FusedPolicyForward.supported(ff) and not FusedPolicyForward.supported(gru)

    # (the fused training node checks the tensors' device: stand-ins that say "cuda")
    obs = SimpleNamespace(is_cuda=True, dtype=torch.float32, requires_grad=False, shape=(4, 5))
    param = SimpleNamespace(is_cuda=True, dtype=torch.float32)
    ff_cuda = SimpleNamespace(is_deterministic=False, fc=ff.fc, output_dims=[21, 21],
                              parameters=lambda: [param])
    gru_cuda = SimpleNamespace(**vars(ff_cuda), is_recurrent=True)
    assert fused_mlp_train.supported(ff_cuda, obs)
    assert not fused_mlp_train.supported(gru_cuda, obs)

    from warp_drive_b200.utils.spaces import Box, Discrete, MultiDiscrete

    env = SimpleNamespace(name="ClassicControlCartPoleEnv", action_space={0: Discrete(2)},
                          observation_space={0: Box(-1, 1, shape=(4,))})
    wrapper = SimpleNamespace(env=env, n_agents=1)
    from warp_drive_b200.training.models.fully_connected import FullyConnected

    ff_sa = FullyConnected(_stub_env(Discrete(2), 4),
                           {"type": "fully_connected", "fc_dims": [32, 32]}, "p", {"p": [0]})
    gru_sa = _model(fc_dims=(32, 32), heads=(2,), F=4)
    assert FusedSingleAgentRollout.eligible(wrapper, {"p": ff_sa}, {"p": [0]})
    assert not FusedSingleAgentRollout.eligible(wrapper, {"p": gru_sa}, {"p": [0]})

    # RolloutEngine._fused_eligible: the recurrent switch comes before the library's plan
    tc_env = SimpleNamespace(name="TagContinuous", action_space={0: MultiDiscrete([21, 21])},
                             observation_space={0: Box(-1, 1, shape=(5,))})
    eng = SimpleNamespace(separate=False, agents_last=False, env_wrapper=SimpleNamespace(
        env=tc_env), policies=["p"], continuous=False, n_heads=2, T=4,
        dm=SimpleNamespace(reset_target_to_pool=False), models={"p": gru}, q_network=False,
        recurrent=True, policy_map={"p": [0]})
    assert RolloutEngine._fused_eligible(eng) is False


# ------------------------------------------------------------------------ sequence minibatches
@pytest.mark.parametrize("T,E,Np,m", [(5, 3, 2, 4), (1, 7, 1, 7), (4, 2, 3, 1)])
def test_sequence_minibatch_rows_cover_every_row_once_per_epoch(T, E, Np, m):
    from warp_drive_b200.training.algorithms.policygradient import _PolicyGradient

    S = E * Np
    gen = torch.Generator().manual_seed(2)
    for _ in range(3):                            # epochs
        perm = torch.randperm(S, generator=gen).to(torch.int32)
        rows = [_PolicyGradient.sequence_rows(c, T, S) for c in torch.tensor_split(perm, m)]
        for c, r in zip(torch.tensor_split(perm, m), rows):
            assert r.dtype == torch.int32
            # (t, chunk) order: row t * B_s + j is step t of the chunk's j-th sequence
            assert torch.equal(r.view(T, -1) % S, c.view(1, -1).expand(T, -1))
            assert torch.equal(r.view(T, -1) // S, torch.arange(T)[:, None].expand_as(r.view(T, -1)).int())
        got = torch.sort(torch.cat(rows)).values
        assert torch.equal(got, torch.arange(T * S, dtype=torch.int32))


def test_too_many_sequence_minibatches_are_refused():
    from warp_drive_b200.training.algorithms.policygradient import PPO

    m = _model()
    T, E, Np = 3, 2, 1
    with pytest.raises(ValueError, match="sequences"):
        PPO(clip_param=0.2, num_epochs=2, num_mini_batches=3).prepare_batch(
            m, torch.zeros(T, E, Np, 5), torch.zeros(T, E, Np, 2, dtype=torch.int32),
            torch.zeros(T, E, Np), torch.zeros(T, E, dtype=torch.int32),
            hidden_start=torch.zeros(E, Np, 8))


# ------------------------------------------------------------------------ native envelope / ABI
def test_envelope_query_answers_without_a_cuda_call():
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.models.fully_connected_gru import NativeGruStep

    L = wlib.load()
    q = L.wdb_gru_forward_bytes
    assert q(71, 2, 64, 64, 64, 2, 21, 21) > 0          # TagContinuous run config (K = 10)
    assert q(57, 2, 64, 64, 64, 2, 21, 21) > 0
    assert q(26, 2, 32, 32, 32, 1, 5, 0) > 0            # gridworld shape
    for n_layers, d0, d1 in ((0, 0, 0), (1, 48, 0), (2, 64, 32)):
        assert q(13, n_layers, d0, d1, 40, 1, 3, 0) > 0
    assert q(71, 3, 64, 64, 64, 2, 21, 21) == 0         # three trunk layers
    assert q(71, 2, 64, 64, 64, 3, 21, 21) == 0         # three heads
    assert q(71, 2, 64, 64, 129, 2, 21, 21) == 0        # H > 128
    assert q(257, 2, 64, 64, 64, 2, 21, 21) == 0        # F > 256
    assert q(71, 2, 64, 64, 64, 2, 65, 21) == 0         # A > 64
    assert q(256, 2, 128, 128, 128, 2, 64, 64) == 0     # over 227 KB of shared memory
    assert NativeGruStep.supported(_model(fc_dims=(64, 64), heads=(21, 21)))
    assert not NativeGruStep.supported(_model(fc_dims=(8, 8, 8), heads=(3,)))
    assert not NativeGruStep.supported(_built_fc((64, 64), (21, 21)))
    # routed only below the measured cross-over: gridworld's step yes, TagContinuous's no
    grid = _model(fc_dims=(32, 32), gru_dim=32, heads=(5,), F=21)
    tc = _model(fc_dims=(64, 64), heads=(21, 21), F=71)
    assert NativeGruStep.routed(grid, 2000 * 5) and not NativeGruStep.routed(tc, 2000 * 105)
    assert NativeGruStep.step_flops(tc, 2000 * 105) == pytest.approx(15.07968e9)


def test_struct_layout_and_prototypes_match_the_header(tmp_path):
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    pairs = {"wdb_gru_forward": wlib.GruForward, "wdb_recurrent_state": wlib.RecurrentState,
             "wdb_recurrent_reset": wlib.RecurrentReset}
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "wdb200.h"', "int main(void) {"]
    fields = {}
    for c_name in pairs:
        fields[c_name] = _c_fields(header, c_name)
        lines.append(f'  printf("{c_name} size %zu\\n", sizeof({c_name}));')
        lines += [f'  printf("{c_name} {f} %zu\\n", offsetof({c_name}, {f}));'
                  for f in fields[c_name]]
    lines += ['  printf("max policies %d\\n", WDB_RECURRENT_MAX_POLICIES);', "  return 0;", "}"]
    (tmp_path / "layout.c").write_text("\n".join(lines))
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(tmp_path / "layout"),
                    str(tmp_path / "layout.c")], check=True)
    out = subprocess.run([str(tmp_path / "layout")], check=True, capture_output=True,
                         text=True).stdout.splitlines()
    got = {}
    for line in out:
        *key, v = line.split()
        got[" ".join(key)] = int(v)
    assert got["max policies"] == wlib.RECURRENT_MAX_POLICIES
    for c_name, py in pairs.items():
        assert ctypes.sizeof(py) == got[f"{c_name} size"], c_name
        assert [n for n, _ in py._fields_] == fields[c_name]
        for f in fields[c_name]:
            assert getattr(py, f).offset == got[f"{c_name} {f}"], (c_name, f)
    flat = re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", header, flags=re.S))
    for name in ("wdb_gru_forward_bytes", "wdb_gru_policy_forward", "wdb_recurrent_reset_done"):
        m = re.search(r"\b" + name + r"\(([^)]*)\);", flat)
        assert m, name
        assert len(m.group(1).split(",")) == len(wlib._SIGNATURES[name][1]), name


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_kernels_compile_for_sm90a_without_spills(tmp_path):
    out = subprocess.run(
        ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler",
         "-fPIC", "-Xptxas", "-v", "-c", os.path.join(CSRC, "wdb_recurrent.cu"), "-o",
         str(tmp_path / "r.o")], check=True, capture_output=True, text=True)
    log = out.stdout + out.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)'", log)
    assert any("gru_policy_forward_kernel" in k for k in kernels)
    assert any("recurrent_reset_done_kernel" in k for k in kernels)
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert spills and all(s == ("0", "0") for s in spills)
    assert "bytes stack frame" in log and not re.search(r"[1-9]\d* bytes stack frame", log)
