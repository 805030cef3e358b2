"""CPU tests of discrete-action SAC: the float64 restatement of both update passes
(tests/sac_discrete_reference.py) pinned to what TrainerDiscreteSAC's torch update computes by
autograd -- the real DiscreteSAC class and the real actor and Q modules, in float64; the
trainer's refusals; the ctypes layout of the new ABI struct and its prototypes; the support
envelope; what ptxas makes of the new kernels; the run config."""
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import sac_discrete_reference as ref  # noqa: E402
from dqn_update_reference import forward, gather, make_q_ring  # noqa: E402
from test_abi_layout_cpu import _c_fields  # noqa: E402
from test_ddpg_update_reference_cpu import _Env  # noqa: E402

NVCC_SM90A = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC"]
CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")


def _discrete_env(F, A):
    from warp_drive_b200.utils import spaces

    env = _Env(F, 1)
    env.env.action_space = {0: spaces.Discrete(A)}
    return env


def make_models(F, A, ad, cd, seed=0, gap=0.0):
    """actor (FullyConnectedActor), critic, critic2, target critic, target critic2 in float64;
    the targets differ from the online networks.  gap: added to the actor's head bias of
    action 0, a near-deterministic policy when large."""
    from warp_drive_b200.training.models.fully_connected import ModelFactory

    torch.manual_seed(seed)
    kw = dict(env=_discrete_env(F, A), policy="shared", policy_tag_to_agent_id_map={"shared": [0]})
    actor = ModelFactory.create("fully_connected_actor")(
        model_config={"type": "fully_connected_actor", "fc_dims": ad}, **kw).double()
    with torch.no_grad():
        actor.policy_head[0].bias[0] += gap
    critics = [ModelFactory.create("fully_connected_q")(
        model_config={"type": "fully_connected_q", "fc_dims": cd}, **kw).double()
        for _ in range(4)]
    return [actor] + critics


def _layers(model):
    from warp_drive_b200.training.algorithms.fused_sac_discrete import _layers as fl

    return [(w.detach().numpy(), b.detach().numpy()) for w, b in fl(model)]


def torch_update(models, ring, windows, n_step, gamma, alpha):
    """TrainerDiscreteSAC's torch update in float64 on the gathered windows: the critic pass,
    then the actor pass (the actor's gradient only) and the log_alpha gradient."""
    from warp_drive_b200.training.algorithms.sac_discrete import (
        DiscreteSAC, torch_actor_loss, torch_sampled_critic_loss)

    actor, critic, critic2, t1, t2 = models
    A = actor.output_dims[0]
    algo = DiscreteSAC(discount_factor_gamma=gamma, n_step=n_step, alpha=alpha, n_actions=A)
    log_alpha = torch.tensor([math.log(alpha)], dtype=torch.float64, requires_grad=True)
    Np = ring[0].shape[2]
    obs, actions, rewards, done, boot_obs = gather(ring, windows, n_step, Np)
    batch = (torch.from_numpy(obs), torch.from_numpy(actions.reshape(-1, 1)),
             torch.from_numpy(rewards), torch.from_numpy(done.astype(np.float64)),
             torch.from_numpy(boot_obs))
    for m in models:
        m.zero_grad()
    l1, l2, q1, q2, R = torch_sampled_critic_loss(algo, actor, t1, t2, critic, critic2,
                                                  log_alpha, *batch)
    (l1 + l2).backward()
    loss, pm, plp = torch_actor_loss(algo, actor, critic, critic2, log_alpha, batch[0])
    loss.backward(inputs=list(actor.parameters()))
    grad = lambda m: [p.grad.numpy().copy() for p in _params(m)]  # noqa: E731
    return {"grads1": grad(critic), "grads2": grad(critic2), "grads": grad(actor),
            "q1": q1.detach().numpy(), "q2": q2.detach().numpy(), "returns": R.numpy(),
            "sum_e1": float(((q1.detach() - R) ** 2).sum()),
            "sum_e2": float(((q2.detach() - R) ** 2).sum()),
            "sum_m": float(pm.sum()), "sum_log_pi": float(plp.sum()), "loss": loss.item(),
            "alpha_grad": float(algo.alpha_grad(plp.sum(), plp.numel())),
            "target_entropy": algo.target_entropy}


def _params(model):
    """Parameters in the order of fused_sac_discrete._layers: (W, b) per layer."""
    from warp_drive_b200.training.algorithms.fused_sac_discrete import _layers as fl

    return [t for pair in fl(model) for t in pair]


def _rel(a, b):
    """Norm-wise relative difference, floored at a norm of 1e-3: with a logit gap of 40 the
    actor's gradient is ~1e-18, below the round-off of its O(1) terms in either evaluation."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-3))


# (F, A, actor dims, critic dims, E, Np, C, n_step, B, gamma, alpha, gap)
CASES = [
    (4, 2, [64, 64], [64, 64], 8, 1, 12, 3, 40, 0.99, 0.2, 0.0),     # CartPole's shape
    (2, 3, [8], [], 5, 2, 9, 1, 17, 0.9, 1.5, 0.0),
    (6, 3, [8, 5, 7], [16], 4, 3, 7, 2, 33, 1.0, 0.05, 0.0),
    (3, 5, [16], [16, 8, 4], 6, 1, 10, 3, 25, 0.0, 0.3, 40.0),        # near-deterministic pi
    (5, 4, [32, 32], [32, 32], 3, 2, 6, 2, 19, 0.97, 0.2, 40.0),
]


def _case(case, seed):
    F, A, ad, cd, E, Np, C, ns, B, gamma, alpha, gap = case
    models = make_models(F, A, ad, cd, seed=seed, gap=gap)
    ring = make_q_ring(C, E, Np, F, A, seed=seed)
    g = np.random.default_rng(seed + 100)
    windows = np.stack([g.integers(0, C, B), g.integers(0, E * Np, B)], axis=1).astype(np.int32)
    return models, ring, windows, ns, gamma, alpha


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"case{i}" for i in range(len(CASES))])
def test_reference_matches_torch_autograd_in_float64(i):
    models, ring, windows, ns, gamma, alpha = _case(CASES[i], seed=i)
    want = torch_update(models, ring, windows, ns, gamma, alpha)
    La, L1, L2, T1, T2 = (_layers(m) for m in models)
    c = ref.critic_pass(La, L1, L2, T1, T2, ring, windows, ns, gamma, alpha)
    a = ref.actor_pass(La, L1, L2, ring, windows, ns, alpha, want["target_entropy"])
    for k in ("grads1", "grads2"):
        for got, exp in zip(c[k], want[k]):
            assert _rel(got, exp) <= 1e-12, k
    for got, exp in zip(a["grads"], want["grads"]):
        assert _rel(got, exp) <= 1e-12
    for k in ("q1", "q2", "returns"):
        assert _rel(c[k], want[k]) <= 1e-12, k
    for k in ("sum_e1", "sum_e2"):
        assert c[k] == pytest.approx(want[k], rel=1e-12, abs=1e-12), k
    for k in ("sum_m", "sum_log_pi", "loss", "alpha_grad"):
        assert a[k] == pytest.approx(want[k], rel=1e-12, abs=1e-12), k


def test_cases_cover_every_done_flag_inside_windows_and_a_saturated_policy():
    seen_flags, saturated = set(), False
    for i, case in enumerate(CASES):
        models, ring, windows, ns, _, _ = _case(case, seed=i)
        C = ring[0].shape[0]
        Np = ring[0].shape[2]
        for s, n in windows:
            for j in range(ns):
                seen_flags.add(int(ring[3][(s + j) % C, n // Np]))
        La = _layers(models[0])
        obs = gather(ring, windows, ns, Np)[0]
        lp = ref.log_softmax(forward(La, obs)[0])
        saturated |= bool((np.exp(lp) == 0.0).any() or (lp < -30).any())
    assert seen_flags == {0, 1, 2}
    assert saturated
    assert {c[7] for c in CASES} == {1, 2, 3}


# ------------------------------------------------------------------------ algorithm
def test_discrete_sac_defaults_and_returns():
    from warp_drive_b200.training.algorithms.dqn import DQN
    from warp_drive_b200.training.algorithms.sac_discrete import DiscreteSAC

    algo = DiscreteSAC(n_step=3, n_actions=3)
    assert algo.target_entropy == pytest.approx(0.98 * math.log(3))
    assert (algo.alpha, algo.autotune_alpha) == (0.2, True)
    g = torch.Generator().manual_seed(0)
    rewards, boot = torch.randn(3, 7, generator=g), torch.randn(7, generator=g)
    done = torch.tensor([[0, 2, 0, 1, 0, 0, 0], [0, 0, 0, 0, 2, 0, 1], [1, 0, 0, 0, 0, 2, 0]])
    want = DQN(discount_factor_gamma=0.9, n_step=3).sampled_returns(rewards, done, boot)
    algo.discount_factor_gamma = 0.9
    assert torch.equal(algo.sampled_returns(rewards, done, boot), want)


@pytest.mark.parametrize("kw", [{"normalize_return": True}, {"alpha": 0.0},
                                {"target_entropy": float("nan")}, {"n_actions": 1}])
def test_discrete_sac_refuses_what_it_does_not_train(kw):
    from warp_drive_b200.training.algorithms.sac_discrete import DiscreteSAC

    args = dict(n_step=1, n_actions=2)
    args.update(kw)
    with pytest.raises(ValueError):
        DiscreteSAC(**args)


# ------------------------------------------------------------------------ trainer refusals
def _stub(actor_cfg=None, critic_cfg=None, sampler=None, action_space=None, F=4, mask=False,
          algorithm="DiscreteSAC"):
    """A TrainerDiscreteSAC with only what _initialize_policy_model reads."""
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.training.trainer_sac_discrete import TrainerDiscreteSAC
    from warp_drive_b200.utils import spaces

    env = _discrete_env(F, 2)
    if action_space is not None:
        env.env.action_space = {0: action_space}
    if mask:
        env.env.observation_space = {0: spaces.Dict({
            "obs": spaces.Box(-1.0, 1.0, shape=(F,), dtype=np.float32),
            "action_mask": spaces.Box(0.0, 1.0, shape=(2,), dtype=np.float32)})}
    tr = object.__new__(TrainerDiscreteSAC)
    tr.config = {"policy": {"shared": {"algorithm": algorithm, "model": {
        "actor": {"type": "fully_connected_actor", "fc_dims": [8], **(actor_cfg or {})},
        "critic": {"type": "fully_connected_q", "fc_dims": [8], **(critic_cfg or {})}}}}}
    tr.sample_params_schedules = dict(sampler or {})
    tr._create_network_dicts()
    tr._build_model = lambda policy, cfg: ModelFactory.create(cfg["type"])(
        env=env, model_config=cfg, policy=policy, policy_tag_to_agent_id_map={"shared": [0]})
    return tr


def test_trainer_builds_the_models():
    tr = _stub()
    tr._initialize_policy_model("shared")
    assert tr.actor_models["shared"].output_dims == [2]
    assert not tr.target_actor_models
    for m in (tr.critic_models, tr.critic2_models, tr.target_critic_models,
              tr.target_critic2_models):
        assert m["shared"].output_dims == [2]
    assert float(tr.temperatures["shared"].log_alpha.detach().exp()) == pytest.approx(0.2)


@pytest.mark.parametrize("kw, match", [
    ({"algorithm": "SAC"}, "DiscreteSAC"),
    ({"sampler": {"epsilon": 0.1}}, "sampler params"),
    ({"actor_cfg": {"type": "fully_connected"}}, "fully_connected_actor"),
    ({"critic_cfg": {"dueling": True}}, "dueling"),
    ({"critic_cfg": {"noisy": True}}, "noisy"),
    ({"critic_cfg": {"type": "fully_connected_quantile_q", "num_quantiles": 4}},
     "fully_connected_q"),
    ({"critic_cfg": {"type": "fully_connected_iqn"}}, "fully_connected_q"),
    ({"critic_cfg": {"type": "fully_connected_categorical_q", "num_atoms": 5, "v_min": -1.0,
                     "v_max": 1.0}}, "fully_connected_q"),
    ({"mask": True}, "action_mask"),
    ({"critic_cfg": {"masked": True}}, "masked"),
], ids=["algorithm", "sampler", "actor_type", "dueling", "noisy", "quantile", "iqn",
        "categorical", "mask", "masked_critic"])
def test_trainer_refuses(kw, match):
    tr = _stub(**kw)
    with pytest.raises(ValueError, match=match):
        tr._initialize_policy_model("shared")


def test_trainer_refuses_box_and_multi_head_action_spaces():
    from warp_drive_b200.utils import spaces

    for space in (spaces.Box(-1.0, 1.0, shape=(1,), dtype=np.float32),
                  spaces.MultiDiscrete([2, 3])):
        tr = _stub(action_space=space)
        with pytest.raises(ValueError, match="action space"):
            tr._initialize_policy_model("shared")


def test_trainer_refuses_differing_action_counts():
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils import spaces

    tr = _stub()
    build = tr._build_model

    def three_action_critic(policy, cfg):
        if cfg["type"] != "fully_connected_q":
            return build(policy, cfg)
        env = _discrete_env(4, 2)
        env.env.action_space = {0: spaces.Discrete(3)}
        return ModelFactory.create(cfg["type"])(env=env, model_config=cfg, policy=policy,
                                                policy_tag_to_agent_id_map={"shared": [0]})

    tr._build_model = three_action_critic
    with pytest.raises(ValueError, match="must agree"):
        tr._initialize_policy_model("shared")


def _slots_stub(trainer_config):
    from warp_drive_b200.training.trainer_sac_discrete import TrainerDiscreteSAC

    tr = object.__new__(TrainerDiscreteSAC)
    tr.training_batch_size_per_env = 4
    return tr._batch_slots_per_env(trainer_config)


def test_trainer_refuses_the_ring_without_a_replay_buffer_and_prioritized_replay():
    assert _slots_stub({"n_step": 3, "replay_slots_per_env": 64}) == 64
    with pytest.raises(ValueError, match="replay_slots_per_env"):
        _slots_stub({"n_step": 3})
    with pytest.raises(ValueError, match="prioritized_replay"):
        _slots_stub({"n_step": 3, "replay_slots_per_env": 64, "prioritized_replay": True})


def test_trainer_refuses_separate_placeholders():
    from warp_drive_b200.training.trainer_sac_discrete import TrainerDiscreteSAC

    with pytest.raises(AssertionError, match="separate per-policy placeholders"):
        TrainerDiscreteSAC(env_wrapper=None, config={},
                           create_separate_placeholders_for_each_policy=True)


def test_run_config_loads():
    from warp_drive_b200.training.trainer import load_run_config

    cfg = load_run_config("single_cartpole_sac_discrete")
    dqn = load_run_config("single_cartpole_dqn")
    pol = cfg["policy"]["shared"]
    assert pol["algorithm"] == "DiscreteSAC"
    assert not cfg.get("sampler", {}).get("params")
    assert cfg["trainer"] == dqn["trainer"]
    assert pol["model"]["actor"]["type"] == "fully_connected_actor"
    assert pol["model"]["critic"]["type"] == "fully_connected_q"
    assert set(pol["model"]["model_ckpt_filepath"]) == {"actor", "critic", "critic2", "alpha"}


# ------------------------------------------------------------------------ ABI
def test_struct_layout_and_prototypes_match_the_header(tmp_path):
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    c_name = "wdb_sac_discrete_update_args"
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
    assert ctypes.sizeof(wlib.SacDiscreteUpdate) == got["size"]
    assert [n for n, _ in wlib.SacDiscreteUpdate._fields_] == fields
    for f in fields:
        assert getattr(wlib.SacDiscreteUpdate, f).offset == got[f], f
    # every new entry point is declared with the argument count lib.py types it with
    flat = re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", header, flags=re.S))
    names = [n for n in wlib.exported_symbols() if n.startswith("wdb_sac_discrete_")]
    assert len(names) == 6
    for name in names:
        m = re.search(r"\b" + name + r"\(([^)]*)\);", flat)
        assert m, name
        assert len(m.group(1).split(",")) == len(wlib._SIGNATURES[name][1]), name


def _struct(F=4, A=2, ad=(64, 64), cd=(64, 64), E=256, Np=1, C=4096, n_step=3):
    from warp_drive_b200 import lib as wlib

    u = wlib.SacDiscreteUpdate()
    u.n_envs, u.n_agents, u.obs_dim, u.n_actions = E, Np, F, A
    u.capacity, u.n_step = C, n_step
    for net, dims in ((u.actor, ad), (u.critic, cd), (u.critic2, cd), (u.target_critic, cd),
                      (u.target_critic2, cd)):
        net.n_hidden = len(dims)
        for i, w in enumerate(dims[:3]):
            net.widths[i] = w
    return u


def _both(u, B=512):
    from warp_drive_b200 import lib as wlib

    L = wlib.load()
    return (L.wdb_sac_discrete_critic_update_sampled_supported(ctypes.byref(u), B),
            L.wdb_sac_discrete_actor_update_sampled_supported(ctypes.byref(u), B))


def test_supported_accepts_exactly_the_documented_shapes():
    from warp_drive_b200 import lib as wlib

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    assert _both(_struct()) == (1, 1)                              # CartPole
    assert _both(_struct(F=2, A=3)) == (1, 1)                      # MountainCar
    assert _both(_struct(F=6, A=3)) == (1, 1)                      # Acrobot
    assert _both(_struct(ad=(), cd=())) == (1, 1)
    assert _both(_struct(F=63, A=2, ad=(32, 32), cd=(32, 32))) == (1, 1)
    assert _both(_struct(A=64, ad=(32, 32), cd=(32, 32))) == (1, 1)
    assert _both(_struct(F=63, A=2)) == (0, 1) and _both(_struct(A=64)) == (0, 1)
    assert _both(_struct(ad=(1, 1, 1), cd=(64, 1, 64))) == (1, 1)
    assert _both(_struct(n_step=1, C=2)) == (1, 1) and _both(_struct(Np=3)) == (1, 1)
    assert _both(_struct(), B=1) == (1, 1) and _both(_struct(), B=2 ** 31 - 1) == (1, 1)
    # the actor and four Q networks in shared memory: three hidden layers of 64 fit the actor
    # pass only
    assert _both(_struct(ad=(64, 64, 64), cd=(64, 64, 64))) == (0, 1)
    for bad in (_struct(A=1), _struct(A=65), _struct(F=64), _struct(ad=(65, 64)),
                _struct(cd=(64, 0)), _struct(ad=(8, 8, 8, 8)), _struct(n_step=3, C=3),
                _struct(n_step=0), _struct(E=0), _struct(Np=0)):
        assert _both(bad) == (0, 0)
    assert _both(_struct(), B=0) == (0, 0)
    for name in ("critic2", "target_critic", "target_critic2"):
        u = _struct()
        getattr(u, name).widths[1] = 32                            # shaped as the critic
        assert _both(u) == (0, 0), name
    L = wlib.load()
    u = _struct(ad=(65,))
    assert L.wdb_sac_discrete_critic_update_sampled_workspace_bytes(ctypes.byref(u), 8) == -1
    assert L.wdb_sac_discrete_actor_update_sampled_workspace_bytes(ctypes.byref(u), 8) == -1
    assert L.wdb_sac_discrete_critic_update_sampled_workspace_bytes(
        ctypes.byref(_struct()), 512) > 0
    assert L.wdb_sac_discrete_critic_update_sampled(None, ctypes.byref(_struct()), None) != 0


# ------------------------------------------------------------------------ ptxas
@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_kernels_compile_for_sm90a_without_spills(tmp_path):
    out = str(tmp_path / "sac_discrete.cubin")
    proc = subprocess.run(NVCC_SM90A + ["-Xptxas", "-v", "-cubin", "-I",
                                        os.path.join(ROOT, "include"),
                                        os.path.join(CSRC, "wdb_sac_discrete.cu"), "-o", out],
                          capture_output=True, text=True, check=True)
    stats, name = {}, None
    for line in proc.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            stats[name] = (int(m.group(1)), int(m.group(2)))
    for k in ("sac_discrete_critic_kernel", "sac_discrete_actor_kernel", "ddpg_reduce_kernel"):
        hits = [v for n, v in stats.items() if k in n]
        assert hits == [(0, 0)], (k, stats)
