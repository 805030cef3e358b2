"""CPU tests of the recurrent Gaussian A2C / PPO policy (FullyConnectedGaussianGRU): config keys,
state_dict names, log_std_init and refusals; step against nn.GRUCell plus Linear; forward_sequence
against a loop of step with the reset rule; the float64 reference
(tests/gaussian_recurrent_reference.py, tests/gaussian_reference.py) against torch autograd
through the A2C and PPO Gaussian losses; the
native forward's shape query and head kind; what ptxas makes of both kernel instantiations; and
PPO's sequence minibatches over a Gaussian batch."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import gaussian_reference as gref  # noqa: E402
import gaussian_recurrent_reference as gru_ref  # noqa: E402
import recurrent_reference as ref  # noqa: E402
from test_recurrent_cpu import _stub_env  # noqa: E402

CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")


def _gmodel(fc_dims=(8, 8), gru_dim=None, A=2, F=5, dtype=torch.float32, seed=0, **keys):
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils.spaces import Box

    cfg = dict({"type": "fully_connected_gaussian_gru", "fc_dims": list(fc_dims)}, **keys)
    if gru_dim is not None:
        cfg["gru_dim"] = gru_dim
    torch.manual_seed(seed)
    m = ModelFactory.create("fully_connected_gaussian_gru")(
        _stub_env(Box(-1, 1, shape=(A,)), F), cfg, "p", {"p": [0]})
    return m.to(dtype)


# ------------------------------------------------------------------------ config and refusals
def test_config_keys_state_dict_names_and_log_std_init():
    from warp_drive_b200.training.models.fully_connected_gru import (
        FullyConnectedGaussianGRU, FullyConnectedGRU)

    m = _gmodel(fc_dims=(8, 6), gru_dim=7, A=3)
    assert isinstance(m, FullyConnectedGaussianGRU) and isinstance(m, FullyConnectedGRU)
    assert m.is_recurrent and m.is_gaussian and m.hidden_size == 7
    assert m.output_dims == [3] and m.flattened_action_size == 3
    # (a module's own parameters come before its children's, as in fully_connected_gaussian)
    assert list(m.state_dict()) == [
        "log_std", "fc.0.0.weight", "fc.0.0.bias", "fc.1.0.weight", "fc.1.0.bias",
        "gru.weight_ih", "gru.weight_hh", "gru.bias_ih", "gru.bias_hh",
        "policy_head.weight", "policy_head.bias", "vf_head.weight", "vf_head.bias"]
    assert tuple(m.policy_head.weight.shape) == (3, 7)
    assert torch.equal(m.log_std.detach(), torch.zeros(3))
    assert torch.equal(_gmodel(log_std_init=-0.5).log_std.detach(), torch.full((2,), -0.5))
    assert _gmodel(fc_dims=(8, 6)).hidden_size == 6           # gru_dim defaults to fc_dims[-1]
    assert len(_gmodel(fc_dims=(), gru_dim=5).fc) == 0
    with pytest.raises(ValueError):
        _gmodel(fc_dims=())
    with pytest.raises(RuntimeError, match="recurrent"):
        m(torch.zeros(2, 5))
    # the parameters fully_connected_gaussian names alike have its shapes
    from warp_drive_b200.training.models.fully_connected import FullyConnectedGaussian
    from warp_drive_b200.utils.spaces import Box

    ff = FullyConnectedGaussian(_stub_env(Box(-1, 1, shape=(3,))), {"fc_dims": [8, 7]}, "p",
                                {"p": [0]})
    assert list(ff.state_dict())[0] == "log_std"
    for name in ("policy_head.weight", "policy_head.bias", "log_std", "vf_head.weight"):
        assert ff.state_dict()[name].shape == m.state_dict()[name].shape, name


def test_refusals():
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.training.trainer import Trainer
    from warp_drive_b200.utils.spaces import Box, Dict, Discrete, MultiDiscrete
    from types import SimpleNamespace

    cls = ModelFactory.create("fully_connected_gaussian_gru")
    cfg = {"type": "fully_connected_gaussian_gru", "fc_dims": [8]}
    for space in (Discrete(3), MultiDiscrete([3, 2])):
        with pytest.raises(ValueError, match="fully_connected_gaussian_gru.*Box"):
            cls(_stub_env(space), cfg, "p", {"p": [0]})
    masked = Dict({"obs": Box(-1, 1, shape=(5,)), "action_mask": Box(0, 1, shape=(2,))})
    with pytest.raises(ValueError, match="action mask"):
        cls(_stub_env(Box(-1, 1, shape=(2,)), obs_space=masked), cfg, "p", {"p": [0]})
    with pytest.raises(ValueError, match="normalize_observations"):
        cls(_stub_env(Box(-1, 1, shape=(2,))), dict(cfg, normalize_observations=True), "p",
            {"p": [0]})
    for algorithm in ("DQN", "SAC", "DDPG"):
        fake = SimpleNamespace(config={"policy": {"p": {"algorithm": algorithm}}})
        with pytest.raises(ValueError, match="A2C or PPO"):
            Trainer._build_model(fake, "p", cfg)
    # the categorical type keeps refusing Box actions, and names the Gaussian type
    gru = ModelFactory.create("fully_connected_gru")
    with pytest.raises(ValueError, match="Box action.*fully_connected_gaussian_gru"):
        gru(_stub_env(Box(-1, 1, shape=(2,))), {"type": "fully_connected_gru", "fc_dims": [8]},
            "p", {"p": [0]})


# ------------------------------------------------------------------------ the torch forwards
def test_step_equals_nn_grucell_plus_linear_bit_for_bit():
    m = _gmodel(fc_dims=(8,), gru_dim=6, A=3)
    cell = torch.nn.GRUCell(8, 6)
    cell.load_state_dict({k[4:]: v for k, v in m.state_dict().items() if k.startswith("gru.")})
    head = torch.nn.Linear(6, 3)
    head.load_state_dict({"weight": m.policy_head.weight, "bias": m.policy_head.bias})
    obs, h = torch.randn(11, 5), torch.randn(11, 6)
    (mean,), h_new = m.step(obs, h)
    assert torch.equal(h_new, cell(m.trunk(obs), h))
    assert torch.equal(mean, head(h_new))


def test_forward_sequence_equals_a_loop_of_step_with_the_reset_rule():
    m = _gmodel(dtype=torch.float64, A=3)
    T, E, Np = 7, 3, 2
    obs = torch.randn(T, E, Np, 5, dtype=torch.float64)
    h0 = torch.randn(E, Np, 8, dtype=torch.float64)
    done = torch.tensor(np.random.default_rng(1).integers(0, 3, (T, E)), dtype=torch.int32)
    done[2, 1] = 1
    (mean,), values = m.forward_sequence(obs, h0, done)
    assert mean.shape == (T, E, Np, 3) and values.shape == (T, E, Np)
    h = h0
    for t in range(T):
        if t > 0:
            h = m.reset_hidden(h, done[t - 1])
        (mu,), hn = m.step(obs[t].reshape(E * Np, -1), h.reshape(E * Np, -1))
        h = hn.view(E, Np, -1)
        torch.testing.assert_close(mu.view(E, Np, -1), mean[t], rtol=0, atol=1e-12)
        torch.testing.assert_close(m.vf_head(h)[..., 0], values[t], rtol=0, atol=1e-12)


@pytest.mark.parametrize("algorithm", ["A2C", "PPO"])
@pytest.mark.parametrize("fc_dims,A", [((8, 8), 3), ((6,), 1), ((), 3), ((7,), 3)])
def test_float64_reference_equals_torch_autograd_through_the_gaussian_loss(algorithm, fc_dims,
                                                                          A):
    from warp_drive_b200.training.algorithms.policygradient import A2C, PPO

    m = _gmodel(fc_dims=fc_dims, gru_dim=7, A=A, dtype=torch.float64, seed=3,
                log_std_init=-0.3)
    T, E, Np = 6, 3, 2
    rng = np.random.default_rng(5 + A)
    obs = rng.normal(size=(T, E, Np, 5))
    h0 = rng.normal(size=(E, Np, 7))
    done = rng.integers(0, 3, (T, E)) * (rng.random((T, E)) < 0.4)
    done[2, 0] = 1                                     # an episode ends mid-sequence
    actions = rng.normal(size=(T, E, Np, A))
    rewards = rng.normal(size=(T, E, Np))
    gamma, vf_c, ent_c = 0.9, 0.5, 0.01
    P = ref.params_of(m)
    mean, values, _ = gru_ref.gaussian_forward_sequence(P, obs, h0, done)
    (tm,), tv = m.forward_sequence(torch.tensor(obs), torch.tensor(h0), torch.tensor(done))
    np.testing.assert_allclose(mean, tm.detach().numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(values, tv.detach().numpy(), rtol=0, atol=1e-12)
    algo = (A2C if algorithm == "A2C" else PPO)(discount_factor_gamma=gamma, vf_loss_coeff=vf_c,
                                                entropy_coeff=ent_c)
    loss, _ = algo.compute_loss_and_metrics(
        0, torch.tensor(actions), torch.tensor(rewards), torch.tensor(done), [tm], tv,
        log_std=m.log_std)
    loss.backward()
    L = gref.gaussian_loss(mean, P["log_std"], values, actions, rewards, done, gamma, vf_c,
                           ent_c, ppo=algorithm == "PPO")
    np.testing.assert_allclose(L["loss"], float(loss.detach()), rtol=0, atol=1e-12)
    G = gru_ref.gaussian_gradients(P, obs, h0, done, L["grad_mean"], L["grad_values"],
                               L["grad_log_std"])
    for name, p in m.named_parameters():
        np.testing.assert_allclose(G[name], p.grad.numpy(), rtol=0, atol=1e-12, err_msg=name)


def test_gaussian_step_bounds_are_positive_and_small():
    m = _gmodel(dtype=torch.float64, A=3)
    P = ref.params_of(m)
    rng = np.random.default_rng(0)
    obs, h = rng.normal(size=(9, 5)), rng.normal(size=(9, 8))
    mean, hn, emean, ehn = gru_ref.gaussian_step_with_bounds(P, obs, h)
    with torch.no_grad():
        (mu,), h_t = m.step(torch.tensor(obs), torch.tensor(h))
    np.testing.assert_allclose(mean, mu.numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(hn, h_t.numpy(), rtol=0, atol=1e-12)
    assert (ehn > 0).all() and ehn.max() < 1e-5
    assert (emean > 0).all() and emean.max() < 1e-4


# ------------------------------------------------------------------------ native step: shape
def test_native_step_takes_the_mean_head_as_one_head_of_a():
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.models.fully_connected_gru import NativeGruStep

    pend = _gmodel(fc_dims=(64, 64), A=1, F=3)
    assert NativeGruStep.shape_args(pend) == (3, 2, 64, 64, 64, 1, 1, 0)
    assert NativeGruStep.supported(pend)
    six = _gmodel(fc_dims=(32,), gru_dim=48, A=6, F=11)
    assert NativeGruStep.shape_args(six) == (11, 1, 32, 0, 48, 1, 6, 0)
    # the query answers as for a softmax head of A actions
    q = wlib.load().wdb_gru_forward_bytes
    assert q(*NativeGruStep.shape_args(six)) == q(11, 1, 32, 0, 48, 1, 6, 0) > 0
    assert not NativeGruStep.supported(_gmodel(fc_dims=(8, 8, 8)))
    assert not NativeGruStep.supported(_gmodel(fc_dims=(8,), A=65))        # A > 64
    # FLOPs: trunk + cell + the mean head's H x A
    rows = 10000
    mac = 3 * 64 + 64 * 64 + 3 * 64 * (64 + 64) + 64 * 1
    assert NativeGruStep.step_flops(pend, rows) == pytest.approx(2.0 * rows * mac)
    assert NativeGruStep.routed(pend, rows)
    big = _gmodel(fc_dims=(128, 128), gru_dim=128, A=8, F=64)
    assert not NativeGruStep.routed(big, 50000)
    assert wlib.GruForward().head_kind == wlib.GRU_HEAD_SOFTMAX == 0
    assert wlib.GRU_HEAD_MEAN == 1
    # head_kind is appended: every earlier field keeps its offset
    assert wlib.GruForward.head_kind.offset == wlib.GruForward.probs.offset + 16


def test_engine_mean_buffer_follows_the_model_output_dims():
    """RolloutEngine sizes a native recurrent policy's buffers by output_dims: [A] for the
    Gaussian model (its action space reads as A heads of size 1)."""
    from warp_drive_b200.training.utils.data_loader import action_head_sizes
    from warp_drive_b200.utils.spaces import Box

    m = _gmodel(A=3)
    assert action_head_sizes(Box(-1, 1, shape=(3,)))[0] == [1, 1, 1]
    assert m.output_dims == [3] and [h.out_features for h in m.head_layers()] == [3]


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_both_kernel_instantiations_compile_for_sm90a_without_spills(tmp_path):
    out = subprocess.run(
        ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler",
         "-fPIC", "-Xptxas", "-v", "-c", os.path.join(CSRC, "wdb_recurrent.cu"), "-o",
         str(tmp_path / "r.o")], check=True, capture_output=True, text=True)
    log = out.stdout + out.stderr
    blocks = re.split(r"Compiling entry function '", log)[1:]
    props = {}
    for b in blocks:
        name = b.split("'")[0]
        props[name] = b
    forwards = [n for n in props if "gru_policy_forward_kernel" in n]
    assert len(forwards) == 2
    assert any("ILi0E" in n for n in forwards) and any("ILi1E" in n for n in forwards)
    for n in forwards:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in props[n], n


# ------------------------------------------------------------------------ sequence minibatches
@pytest.mark.parametrize("T,E,Np,n_mini", [(5, 3, 2, 4), (4, 2, 1, 2)])
def test_ppo_sequence_minibatches_of_a_gaussian_batch_cover_every_row_once(T, E, Np, n_mini):
    from warp_drive_b200.training.algorithms.policygradient import PPO

    m = _gmodel(fc_dims=(6,), A=2, dtype=torch.float64)
    rng = np.random.default_rng(4)
    obs = torch.tensor(rng.normal(size=(T, E, Np, 5)))
    actions = torch.tensor(rng.normal(size=(T, E, Np, 2)))
    rewards = torch.tensor(rng.normal(size=(T, E, Np)))
    done = torch.tensor(rng.integers(0, 2, (T, E)), dtype=torch.int32)
    h0 = torch.tensor(rng.normal(size=(E, Np, 6)))
    algo = PPO(clip_param=0.2, num_epochs=2, num_mini_batches=n_mini, gae_lambda=0.95)
    batch = algo.prepare_batch(m, obs, actions, rewards, done, hidden_start=h0)
    assert batch.log_std is m.log_std and batch.units == E * Np and batch.rows_per_unit == T
    assert batch.actions.shape == (T * E * Np, 2) and batch.actions.is_floating_point()
    with torch.no_grad():
        (full,), _ = m.forward_sequence(obs, h0, done)
    full = full.reshape(T * E * Np, 2)
    gen = torch.Generator().manual_seed(1)
    for _ in range(2):                                  # epochs
        perm = torch.randperm(E * Np, generator=gen).to(torch.int32)
        rows = []
        for seqs in torch.tensor_split(perm, n_mini):
            with torch.no_grad():
                (mean,), values, r = algo._sequence_forward(m, batch, seqs)
            torch.testing.assert_close(mean, full[r.long()], rtol=0, atol=1e-12)
            rows.append(r)
        got = torch.sort(torch.cat(rows)).values
        assert torch.equal(got, torch.arange(T * E * Np, dtype=torch.int32))
    # one minibatch loss takes log_std's gradient
    loss, _ = algo.minibatch_loss(m, batch, torch.tensor([0, 1], dtype=torch.int32), 0)
    loss.backward()
    assert m.log_std.grad is not None and torch.isfinite(m.log_std.grad).all()
