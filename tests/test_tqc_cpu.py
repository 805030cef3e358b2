"""CPU tests of TQC: the float64 restatement of both update passes (tests/tqc_reference.py) pinned
to what TrainerTQC's torch update computes by autograd -- the real TQC class, the real squashed
actor and quantile critics, in float64, for M = 1, 2, 3 critics; the model's and the trainer's
refusals; the ctypes layout of the new ABI struct and its prototypes; the support envelope; what
ptxas makes of the new kernels; the run config."""
import ctypes
import math
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import tqc_reference as ref  # noqa: E402
from test_abi_layout_cpu import _c_fields  # noqa: E402
from test_ddpg_update_reference_cpu import _Env  # noqa: E402

NVCC_SM90A = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC"]
CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")
SCALE = 2.0


def make_models(F, A, ad, cd, M, N, seed=0, zero_target_head=False):
    """actor (FullyConnectedSACActor), critics and target critics (QuantileCritics of M
    FullyConnectedQuantileCritics) in float64; the targets differ from the online critics.
    zero_target_head: every target atom of a row the same value (tied atoms)."""
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.training.models.fully_connected_actor_critic import QuantileCritics

    torch.manual_seed(seed)
    kw = dict(env=_Env(F, A), policy="shared", policy_tag_to_agent_id_map={"shared": [0]})
    actor = ModelFactory.create("fully_connected_sac_actor")(
        model_config={"type": "fully_connected_sac_actor", "fc_dims": ad, "output_w": SCALE,
                      "log_std_min": -2.0, "log_std_max": 0.5}, **kw).double()
    mk = lambda: ModelFactory.create("fully_connected_quantile_critic")(  # noqa: E731
        model_config={"type": "fully_connected_quantile_critic", "fc_dims": cd,
                      "num_quantiles": N}, **kw).double()
    critics = QuantileCritics([mk() for _ in range(M)])
    targets = QuantileCritics([mk() for _ in range(M)])
    if zero_target_head:
        with torch.no_grad():
            for t in targets:
                t.vf_head.weight.zero_()
                t.vf_head.bias.fill_(0.25)
    return actor, critics, targets


def _layers(model):
    from warp_drive_b200.training.algorithms.fused_ddpg import _layers as fl

    return [(w.detach().numpy(), b.detach().numpy()) for w, b in fl(model)]


def _params(model):
    from warp_drive_b200.training.algorithms.fused_ddpg import _layers as fl

    return [t for pair in fl(model) for t in pair]


def torch_update(models, ring, windows, n_step, gamma, alpha, d, critic_noise, actor_noise):
    """TrainerTQC's torch update in float64 on the gathered windows: the critic pass, then the
    actor pass (the actor's gradient only) and the log_alpha gradient."""
    from warp_drive_b200.training.algorithms.tqc import (TQC, torch_actor_loss,
                                                         torch_sampled_critic_loss)

    actor, critics, targets = models
    A = actor.output_dims[0]
    algo = TQC(discount_factor_gamma=gamma, n_step=n_step, alpha=alpha, action_dim=A,
               n_critics=len(critics), n_quantiles=critics[0].num_quantiles, drop_per_net=d)
    log_alpha = torch.tensor([math.log(alpha)], dtype=torch.float64, requires_grad=True)
    Np = ring[0].shape[2]
    batch = [torch.from_numpy(np.asarray(t, dtype=np.float64))
             for t in ref.gather(ring, windows, n_step, Np)]
    for m in (actor, critics, targets):
        m.zero_grad()
    loss, theta, returns = torch_sampled_critic_loss(
        algo, actor, targets, critics, log_alpha, *batch, torch.from_numpy(critic_noise))
    loss.backward()
    assert all(p.grad is None for p in list(actor.parameters()) + list(targets.parameters()))
    aloss, q_bar, log_pi = torch_actor_loss(algo, actor, critics, log_alpha, batch[0],
                                            torch.from_numpy(actor_noise))
    critic_grads = [[p.grad.numpy().copy() for p in _params(c)] for c in critics]
    aloss.backward(inputs=list(actor.parameters()))
    return {"critic_grads": critic_grads, "grads": [p.grad.numpy() for p in _params(actor)],
            "loss": loss.item(), "theta": theta.detach().numpy(), "returns": returns.numpy(),
            "actor_loss": aloss.item(), "q_bar": q_bar.detach().numpy(),
            "log_probs": log_pi.detach().numpy(),
            "alpha_grad": float(algo.alpha_grad(log_pi.detach().sum(), log_pi.numel())),
            "target_entropy": algo.target_entropy}


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-3))


# (F, A, actor dims, critic dims, M, N, d, E, Np, C, n_step, B, gamma, alpha, tied)
CASES = [
    (3, 1, [64, 64], [64, 64], 2, 25, 2, 8, 1, 12, 3, 40, 0.99, 0.2, False),   # the run config
    (2, 1, [16], [8], 1, 5, 0, 5, 2, 9, 1, 17, 0.9, 1.5, False),
    (4, 3, [8, 5], [16], 3, 7, 6, 4, 3, 7, 2, 33, 1.0, 0.05, False),          # d = N - 1
    (3, 2, [16], [16, 8, 4], 2, 4, 2, 6, 1, 10, 3, 25, 0.0, 0.3, True),       # tied atoms
    (5, 3, [32, 32], [32, 32], 3, 6, 0, 3, 2, 6, 2, 19, 0.97, 0.2, True),
    (3, 1, [8], [8], 2, 2, 1, 4, 1, 8, 2, 11, 0.95, 0.7, False),              # N = 2, d = N - 1
]


def _case(case, seed):
    F, A, ad, cd, M, N, d, E, Np, C, ns, B, gamma, alpha, tied = case
    models = make_models(F, A, ad, cd, M, N, seed=seed, zero_target_head=tied)
    ring = ref.make_ring(C, E, Np, F, A, seed=seed)
    g = np.random.default_rng(seed + 100)
    windows = np.stack([g.integers(0, C, B), g.integers(0, E * Np, B)], axis=1).astype(np.int32)
    windows[1] = windows[0]                                       # a duplicated window
    noise = g.standard_normal((2, B, A))
    return models, ring, windows, ns, gamma, alpha, d, noise


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"case{i}" for i in range(len(CASES))])
def test_reference_matches_torch_autograd_in_float64(i):
    models, ring, windows, ns, gamma, alpha, d, noise = _case(CASES[i], seed=i)
    want = torch_update(models, ring, windows, ns, gamma, alpha, d, noise[0], noise[1])
    actor, critics, targets = models
    La, Lcs, Lts = _layers(actor), [_layers(c) for c in critics], [_layers(t) for t in targets]
    kw = dict(scale=SCALE, bias=0.0, lo=actor.log_std_min, hi=actor.log_std_max)
    c = ref.critic_pass(La, Lcs, Lts, ring, windows, ns, gamma, alpha, noise=noise[0],
                        n_drop=d, **kw)
    a = ref.actor_pass(La, Lcs, ring, windows, ns, alpha, noise=noise[1],
                       target_entropy=want["target_entropy"], **kw)
    for got_m, exp_m in zip(c["grads"], want["critic_grads"]):
        for got, exp in zip(got_m, exp_m):
            assert _rel(got, exp) <= 1e-12
    for got, exp in zip(a["grads"], want["grads"]):
        assert _rel(got, exp) <= 1e-12
    assert _rel(c["theta"], want["theta"]) <= 1e-12
    assert _rel(c["returns"], want["returns"]) <= 1e-12
    assert c["loss"] == pytest.approx(want["loss"], rel=1e-12, abs=1e-12)
    assert _rel(a["q_bar"], want["q_bar"]) <= 1e-12
    assert _rel(a["log_probs"], want["log_probs"]) <= 1e-12
    for k in ("actor_loss", "alpha_grad"):
        assert a["loss" if k == "actor_loss" else k] == pytest.approx(want[k], rel=1e-12,
                                                                      abs=1e-12), k


def test_cases_cover_done_flags_tied_atoms_the_drop_range_and_every_n_step():
    seen_flags, tied = set(), False
    for i, case in enumerate(CASES):
        models, ring, windows, ns, *_ = _case(case, seed=i)
        C, Np = ring[0].shape[0], ring[0].shape[2]
        for s, n in windows:
            for j in range(ns):
                seen_flags.add(int(ring[3][(s + j) % C, n // Np]))
        if case[-1]:
            _, _, targets = models
            x = torch.zeros(3, case[0] + case[1], dtype=torch.float64)
            atoms = targets(obs=x[:, :case[0]], action=x[:, case[0]:]).reshape(3, -1)
            tied |= bool((atoms == atoms[:, :1]).all())
    assert seen_flags == {0, 1} and tied
    assert {c[10] for c in CASES} == {1, 2, 3}
    assert {c[4] for c in CASES} == {1, 2, 3}
    assert any(c[6] == 0 for c in CASES) and any(c[6] == 2 for c in CASES)
    assert any(c[6] == c[5] - 1 for c in CASES)


def test_truncation_is_a_stable_sort_of_the_pooled_atoms():
    from warp_drive_b200.training.algorithms.tqc import TQC

    algo = TQC(discount_factor_gamma=0.5, n_step=1, n_critics=2, n_quantiles=3, drop_per_net=1)
    atoms = torch.tensor([[[3.0, 1.0, 2.0], [1.0, 0.0, 3.0]]])        # pooled 3 1 2 1 0 3
    T = algo.truncated_returns(torch.zeros(1, 1), torch.zeros(1, 1), atoms,
                               torch.zeros(1), torch.zeros(1))
    assert T.tolist() == [[0.0, 0.5, 0.5, 1.0]]                        # 0 1 1 2, times gamma
    assert algo.kept_atoms == 4
    assert algo.quantile_fractions().tolist() == [np.float32(v) for v in (1 / 6, 0.5, 5 / 6)]


# ------------------------------------------------------------------------ algorithm and model
@pytest.mark.parametrize("kw", [{"normalize_return": True}, {"alpha": 0.0},
                                {"n_critics": 0}, {"n_critics": 1.5}, {"n_quantiles": 1},
                                {"n_quantiles": 65}, {"drop_per_net": -1},
                                {"drop_per_net": 25}, {"drop_per_net": True}])
def test_tqc_refuses_what_it_does_not_train(kw):
    from warp_drive_b200.training.algorithms.tqc import TQC

    args = dict(n_step=1)
    args.update(kw)
    with pytest.raises(ValueError):
        TQC(**args)


def test_quantile_critic_model():
    from warp_drive_b200.training.models.fully_connected import ModelFactory

    kw = dict(env=_Env(3, 2), policy="shared", policy_tag_to_agent_id_map={"shared": [0]})
    cls = ModelFactory.create("fully_connected_quantile_critic")
    critic = cls(model_config={"type": "fully_connected_quantile_critic", "fc_dims": [8]}, **kw)
    assert critic.num_quantiles == 25
    assert critic(obs=torch.zeros(4, 7, 3), action=torch.zeros(4, 7, 2)).shape == (4, 7, 25)
    for bad in (1, 65, 2.0, True):
        with pytest.raises(ValueError, match="num_quantiles"):
            cls(model_config={"type": "fully_connected_quantile_critic", "fc_dims": [8],
                              "num_quantiles": bad}, **kw)


# ------------------------------------------------------------------------ trainer refusals
def _stub(actor_cfg=None, critic_cfg=None, sampler=None, action_space=None, algorithm="TQC",
          **policy):
    """A TrainerTQC with only what _initialize_policy_model reads."""
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.training.trainer_tqc import TrainerTQC

    env = _Env(3, 1)
    if action_space is not None:
        env.env.action_space = {0: action_space}
    tr = object.__new__(TrainerTQC)
    tr.config = {"policy": {"shared": {"algorithm": algorithm, **policy, "model": {
        "actor": {"type": "fully_connected_sac_actor", "fc_dims": [8], **(actor_cfg or {})},
        "critic": {"type": "fully_connected_quantile_critic", "fc_dims": [8],
                   **(critic_cfg or {})}}}}}
    tr.sample_params_schedules = dict(sampler or {})
    tr._create_network_dicts()
    tr._build_model = lambda policy, cfg: ModelFactory.create(cfg["type"])(
        env=env, model_config=cfg, policy=policy, policy_tag_to_agent_id_map={"shared": [0]})
    return tr


def test_trainer_builds_the_models():
    tr = _stub(n_critics=3, critic_cfg={"num_quantiles": 7})
    tr._initialize_policy_model("shared")
    critics, targets = tr.critic_models["shared"], tr.target_critic_models["shared"]
    assert len(critics) == len(targets) == 3
    assert critics(obs=torch.zeros(5, 3), action=torch.zeros(5, 1)).shape == (5, 3, 7)
    for a, b in zip(critics.parameters(), targets.parameters()):
        assert torch.equal(a, b)
    assert not tr.target_actor_models and not tr.critic2_models
    assert tr._trained_networks("shared")[1] is critics
    assert tr._critic_optimized("shared") is critics
    assert float(tr.temperatures["shared"].log_alpha.detach().exp()) == pytest.approx(0.2)


@pytest.mark.parametrize("kw, match", [
    ({"algorithm": "SAC"}, "TQC"),
    ({"sampler": {"scale": 0.1}}, "sampler params"),
    ({"actor_cfg": {"type": "fully_connected_actor"}}, "fully_connected_sac_actor"),
    ({"critic_cfg": {"type": "fully_connected_action_value_critic"}},
     "fully_connected_quantile_critic"),
    ({"n_critics": 0}, "n_critics"),
    ({"n_critics": 2.0}, "n_critics"),
    ({"critic_cfg": {"num_quantiles": 1}}, "num_quantiles"),
    ({"critic_cfg": {"num_quantiles": 65}}, "num_quantiles"),
    ({"top_quantiles_to_drop_per_net": 25}, "top_quantiles_to_drop_per_net"),
    ({"top_quantiles_to_drop_per_net": -1}, "top_quantiles_to_drop_per_net"),
    ({"critic_cfg": {"num_quantiles": 4}, "top_quantiles_to_drop_per_net": 4},
     "top_quantiles_to_drop_per_net"),
], ids=["algorithm", "sampler", "actor_type", "critic_type", "n_critics_0", "n_critics_float",
        "num_quantiles_1", "num_quantiles_65", "drop_25", "drop_negative", "drop_N"])
def test_trainer_refuses(kw, match):
    tr = _stub(**kw)
    with pytest.raises(ValueError, match=match):
        tr._initialize_policy_model("shared")


def test_trainer_refuses_a_discrete_action_space():
    from warp_drive_b200.utils import spaces

    tr = _stub(action_space=spaces.Discrete(3))
    with pytest.raises(ValueError, match="Box action space"):
        tr._initialize_policy_model("shared")


def _slots_stub(trainer_config):
    from warp_drive_b200.training.trainer_tqc import TrainerTQC

    tr = object.__new__(TrainerTQC)
    tr.training_batch_size_per_env = 4
    return tr._batch_slots_per_env(trainer_config)


def test_trainer_refuses_the_ring_without_a_replay_buffer_and_prioritized_replay():
    assert _slots_stub({"n_step": 3, "replay_slots_per_env": 64}) == 64
    with pytest.raises(ValueError, match="replay_slots_per_env"):
        _slots_stub({"n_step": 3})
    with pytest.raises(ValueError, match="prioritized_replay"):
        _slots_stub({"n_step": 3, "replay_slots_per_env": 64, "prioritized_replay": True})


def test_trainer_refuses_separate_placeholders_obs_norm_and_reward_scaling():
    from warp_drive_b200.training.trainer_tqc import TrainerTQC

    with pytest.raises(AssertionError, match="separate per-policy placeholders"):
        TrainerTQC(env_wrapper=None, config={}, create_separate_placeholders_for_each_policy=True)
    for model, policy in (({"normalize_observations": True}, {}),
                          ({}, {"scale_rewards": True})):
        cfg = {"policy": {"shared": {"algorithm": "TQC", **policy,
                                     "model": {"actor": model, "critic": {}}}}}
        with pytest.raises(ValueError):
            TrainerTQC(env_wrapper=None, config=cfg)


def test_run_config_loads():
    from warp_drive_b200.training.trainer import load_run_config

    cfg = load_run_config("single_pendulum_tqc_replay")
    sac = load_run_config("single_pendulum_sac_replay")
    pol, sac_pol = cfg["policy"]["shared"], sac["policy"]["shared"]
    assert pol["algorithm"] == "TQC"
    assert cfg["trainer"] == sac["trainer"] and cfg["env"] == sac["env"]
    assert pol["model"]["actor"] == sac_pol["model"]["actor"]
    assert pol["model"]["critic"] == {"type": "fully_connected_quantile_critic",
                                      "fc_dims": [64, 64], "num_quantiles": 25}
    assert (pol["n_critics"], pol["top_quantiles_to_drop_per_net"]) == (2, 2)
    assert set(pol["model"]["model_ckpt_filepath"]) == {"actor", "critic", "alpha"}
    for k in ("gamma", "tau", "alpha", "autotune_alpha", "lr", "clip_grad_norm"):
        assert pol[k] == sac_pol[k], k


# ------------------------------------------------------------------------ ABI
def test_struct_layout_and_prototypes_match_the_header(tmp_path):
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    c_name = "wdb_tqc_update_args"
    fields = _c_fields(header, c_name)
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "wdb200.h"', "int main(void) {",
             f'  printf("{c_name} size %zu\\n", sizeof({c_name}));']
    lines += [f'  printf("{c_name} {f} %zu\\n", offsetof({c_name}, {f}));' for f in fields]
    lines += ["  return 0;", "}"]
    (tmp_path / "layout.c").write_text("\n".join(lines))
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(tmp_path / "layout"),
                    str(tmp_path / "layout.c")], check=True)
    out = subprocess.run([str(tmp_path / "layout")], check=True, capture_output=True,
                         text=True).stdout
    got = {f: int(v) for _, f, v in (line.split() for line in out.splitlines())}
    assert ctypes.sizeof(wlib.TqcUpdate) == got["size"]
    assert [n for n, _ in wlib.TqcUpdate._fields_] == fields
    for f in fields:
        assert getattr(wlib.TqcUpdate, f).offset == got[f], f
    flat = re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", header, flags=re.S))
    names = [n for n in wlib.exported_symbols() if n.startswith("wdb_tqc_")]
    assert len(names) == 6
    for name in names:
        m = re.search(r"\b" + name + r"\(([^)]*)\);", flat)
        assert m, name
        assert len(m.group(1).split(",")) == len(wlib._SIGNATURES[name][1]), name


def _struct(F=3, A=1, ad=(64, 64), cd=(64, 64), N=25, d=2, E=256, Np=1, C=4096, n_step=5):
    from warp_drive_b200 import lib as wlib

    u = wlib.TqcUpdate()
    u.n_envs, u.n_agents, u.obs_dim, u.action_dim = E, Np, F, A
    u.capacity, u.n_step, u.n_quantiles, u.n_drop = C, n_step, N, d
    u.log_std_min, u.log_std_max = -20.0, 2.0
    for net, dims in ((u.actor, ad), (u.critic, cd), (u.critic2, cd), (u.target_critic, cd),
                      (u.target_critic2, cd)):
        net.n_hidden = len(dims)
        for i, w in enumerate(dims[:3]):
            net.widths[i] = w
    return u


def _both(u, B=1024):
    from warp_drive_b200 import lib as wlib

    L = wlib.load()
    return (L.wdb_tqc_critic_update_sampled_supported(ctypes.byref(u), B),
            L.wdb_tqc_actor_update_sampled_supported(ctypes.byref(u), B))


def _smem_kb(F, A, ad, cd, N, actor_pass):
    """The pass's dynamic shared memory from plan_layout's padding rules: an independent
    statement of tqc_plan's arithmetic."""
    def net(inp, dims, head):
        w = g = 0
        for out in list(dims) + [head]:
            pw = -(-inp // 4) * 4
            pw += 4 if pw % 8 == 0 else 0
            w += -(-(out * pw + out) // 4) * 4
            g += out * inp + out
            inp = out
        return w, g
    wa, ga = net(F, ad, 2 * A)
    wc, gc = net(F + A, cd, N)
    if actor_pass:
        floats = wa + 2 * wc + -(-ga // 4) * 4 + (6 + 2 * len(cd) + len(ad)) * 16 * 68
    else:
        floats = wa + 4 * wc + -(-2 * gc // 4) * 4 + (8 + 2 * len(cd)) * 16 * 68
    return floats * 4 / 1024


def test_supported_accepts_exactly_the_documented_shapes():
    from warp_drive_b200 import lib as wlib

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    assert _both(_struct()) == (1, 1)                              # the run config's shape
    assert 218 < _smem_kb(3, 1, (64, 64), (64, 64), 25, False) < 220
    assert _both(_struct(F=2)) == (1, 1)                           # ContinuousMountainCar
    assert _both(_struct(ad=(), cd=())) == (1, 1)
    assert _both(_struct(N=2, d=1)) == (1, 1) and _both(_struct(N=32, cd=(32, 32))) == (1, 1)
    assert _both(_struct(N=32, d=31, cd=(32, 32))) == (1, 1)
    assert _both(_struct(F=32, A=32, ad=(32,), cd=(32,))) == (1, 1)
    assert _both(_struct(ad=(64, 64, 64), cd=(32, 32, 32))) == (1, 1)
    assert _both(_struct(n_step=1, C=2)) == (1, 1) and _both(_struct(Np=3)) == (1, 1)
    assert _both(_struct(), B=1) == (1, 1) and _both(_struct(), B=2 ** 31 - 1) == (1, 1)
    # just outside: the critic pass's shared memory, N, d, A, F + A, widths, depth
    assert _both(_struct(cd=(128, 128))) == (0, 0)
    assert _smem_kb(3, 1, (64, 64), (64, 64, 64), 25, False) > 226
    assert _both(_struct(cd=(64, 64, 64))) == (0, 1)
    assert _both(_struct(N=32)) == (0, 1)       # [64, 64] critics of 32 quantiles: 230 KB
    for bad in (_struct(N=33), _struct(N=1, d=0), _struct(d=25), _struct(d=-1),
                _struct(A=33, F=3, ad=(8,), cd=(8,)), _struct(F=33, A=32, ad=(8,), cd=(8,)),
                _struct(ad=(65, 64)), _struct(cd=(64, 0)), _struct(ad=(8, 8, 8, 8)),
                _struct(n_step=3, C=3), _struct(n_step=0), _struct(E=0), _struct(Np=0)):
        assert _both(bad) == (0, 0)
    assert _both(_struct(), B=0) == (0, 0)
    u = _struct()
    u.log_std_min, u.log_std_max = 1.0, 0.0
    assert _both(u) == (0, 0)
    for name in ("critic2", "target_critic", "target_critic2"):
        u = _struct()
        getattr(u, name).widths[1] = 32                            # shaped as the critic
        assert _both(u) == (0, 0), name
    L = wlib.load()
    u = _struct(ad=(65,))
    assert L.wdb_tqc_critic_update_sampled_workspace_bytes(ctypes.byref(u), 8) == -1
    assert L.wdb_tqc_actor_update_sampled_workspace_bytes(ctypes.byref(u), 8) == -1
    # 64 tiles of 16 rows, one CTA each: 16 B of sums and the critics' (or the actor's)
    # gradient block per CTA
    gc = 2 * (4 * 64 + 64 + 64 * 64 + 64 + 64 * 25 + 25)
    ga = 3 * 64 + 64 + 64 * 64 + 64 + 64 * 2 + 2
    assert L.wdb_tqc_critic_update_sampled_workspace_bytes(
        ctypes.byref(_struct()), 1024) == 64 * (16 + 4 * gc)
    assert L.wdb_tqc_actor_update_sampled_workspace_bytes(
        ctypes.byref(_struct()), 1024) == 64 * (16 + 4 * ga)
    assert L.wdb_tqc_critic_update_sampled(None, ctypes.byref(_struct()), None) != 0
    assert L.wdb_tqc_actor_update_sampled(None, ctypes.byref(_struct()), None) != 0


def test_fused_supported_needs_two_critics_of_one_shape():
    from warp_drive_b200 import lib as wlib
    from warp_drive_b200.training.algorithms.fused_tqc import FusedTQCUpdate
    from warp_drive_b200.training.algorithms.tqc import TQC

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    for M, cd, want in ((2, [64, 64], True), (3, [64, 64], False), (1, [64, 64], False),
                        (2, [128, 128], False)):
        actor, critics, _ = make_models(3, 1, [64, 64], cd, M, 25)
        algo = TQC(n_step=5, n_critics=M, n_quantiles=25, drop_per_net=2)
        assert FusedTQCUpdate.supported(algo, actor, critics, 256, 1, 4096, 5, 1024) == want


# ------------------------------------------------------------------------ ptxas
@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_kernels_compile_for_sm90a_without_spills(tmp_path):
    out = str(tmp_path / "tqc.cubin")
    proc = subprocess.run(NVCC_SM90A + ["-Xptxas", "-v", "-cubin", "-I",
                                        os.path.join(ROOT, "include"),
                                        os.path.join(CSRC, "wdb_tqc.cu"), "-o", out],
                          capture_output=True, text=True, check=True)
    stats, regs, name = {}, {}, None
    for line in proc.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            stats[name] = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m and name:
            regs[name] = int(m.group(1))
    for k in ("tqc_critic_kernel", "tqc_actor_kernel", "ddpg_reduce_kernel"):
        hits = [v for n, v in stats.items() if k in n]
        assert hits == [(0, 0)], (k, stats)
    # one CTA of 256 threads per SM: 255 registers a thread is the ceiling; the README records
    # the counts nvcc 12.9 gives (critic 137, actor 130)
    for k in ("tqc_critic_kernel", "tqc_actor_kernel"):
        assert [v for n, v in regs.items() if k in n][0] <= 255
