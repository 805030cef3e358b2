"""CPU tests of SAC: the float64 restatement of both update passes (tests/sac_update_reference.py)
pinned to what TrainerSAC's torch update computes by autograd -- the real SAC class and actor /
critic modules, in float64; the squashed log-prob against torch.distributions; the ctypes layout
of the new ABI struct; the support envelope; the run config and the refusals; what ptxas makes
of the new kernels, and the existing update, rollout and sampler kernels keeping their code."""
import ctypes
import hashlib
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

from sac_update_reference import sac_actor_update, sac_critic_update  # noqa: E402
from test_abi_layout_cpu import _c_fields  # noqa: E402
from test_ddpg_update_reference_cpu import _Env, layers, make_ring, rel  # noqa: E402
from test_td3_cpu import RING  # noqa: E402

NVCC_SM90A = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC"]
CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")


def make_sac_models(F, A, ad, cd, seed, scale=2.0, bias=0.25, lo=-20.0, hi=2.0):
    """actor (FullyConnectedSACActor), critic, critic2, target critic, target critic2 (float64;
    the targets differ from the online networks)."""
    from warp_drive_b200.training.models.fully_connected import ModelFactory

    torch.manual_seed(seed)
    kw = dict(env=_Env(F, A), policy="shared", policy_tag_to_agent_id_map={"shared": [0]})
    mk = lambda kind, dims, **extra: ModelFactory.create(kind)(  # noqa: E731
        model_config={"type": kind, "fc_dims": dims, **extra}, **kw).double()
    actor = mk("fully_connected_sac_actor", ad, output_w=scale, output_b=bias, log_std_min=lo,
               log_std_max=hi)
    critics = [mk("fully_connected_action_value_critic", cd) for _ in range(4)]
    return [actor] + critics


def torch_sac(models, ring, critic_noise, actor_noise, cursor, n_step, gamma, alpha):
    """TrainerSAC's torch update in float64 on the unrolled ring: critic pass, then actor pass
    (the actor's gradient only) and the log_alpha gradient."""
    from warp_drive_b200.training.algorithms.fused_ddpg import _layers
    from warp_drive_b200.training.algorithms.sac import SAC, torch_actor_loss, torch_critic_loss

    actor, critic, critic2, t_critic, t_critic2 = models
    C = ring[0].shape[0]
    order = (cursor + np.arange(C)) % C
    obs, actions, rewards, done = (torch.from_numpy(np.ascontiguousarray(x[order])) for x in ring)
    algo = SAC(discount_factor_gamma=gamma, n_step=n_step, alpha=alpha,
               action_dim=actions.shape[-1])
    log_alpha = torch.tensor([math.log(alpha)], dtype=torch.float64, requires_grad=True)
    for m in models:
        m.zero_grad()
    boot = torch.tensor(algo.bootstrap_slots(C))
    l1, l2, q1, q2, ret = torch_critic_loss(algo, actor, t_critic, t_critic2, critic, critic2,
                                            log_alpha, obs, actions, rewards, done,
                                            torch.from_numpy(critic_noise), boot)
    (l1 + l2).backward()
    assert all(p.grad is None for p in actor.parameters()) and log_alpha.grad is None
    valid = C - n_step + 1
    critic_grads = [(w.grad.clone(), b.grad.clone()) for m in (critic, critic2)
                    for w, b in _layers(m)]
    a_loss, q, log_pi = torch_actor_loss(algo, actor, critic, critic2, log_alpha, obs[:valid],
                                         torch.from_numpy(actor_noise))
    a_loss.backward(inputs=list(actor.parameters()))
    # the actor loss left the critics' gradients (and log_alpha's) alone
    after = [(w.grad, b.grad) for m in (critic, critic2) for w, b in _layers(m)]
    for (w, b), (w0, b0) in zip(after, critic_grads):
        assert torch.equal(w, w0) and torch.equal(b, b0)
    assert log_alpha.grad is None
    # the temperature's loss, by autograd: d/d log_alpha = -mean(log pi + target entropy)
    alpha_loss = -(log_alpha * (log_pi.detach() + algo.target_entropy)).mean()
    alpha_loss.backward()
    grads = lambda m: [(w.grad.numpy(), b.grad.numpy()) for w, b in _layers(m)]  # noqa: E731
    return dict(l1=l1.item(), l2=l2.item(), actor_loss=a_loss.item(), critic=grads(critic),
                critic2=grads(critic2), actor=grads(actor), returns=ret.numpy(),
                alpha_grad=float(log_alpha.grad), log_pi=log_pi.detach().numpy(),
                alpha_grad_algo=float(algo.alpha_grad(log_pi.detach().sum(), log_pi.numel())))


# (n_step, C, cursor, E, Np, F, A, actor dims, critic dims, gamma, done slots, alpha, lo, hi)
CASES = [
    (1, 2, 1, 5, 1, 3, 1, [64, 64], [64, 64], 0.99, (), 0.2, -20.0, 2.0),
    (5, 9, 3, 6, 1, 3, 1, [64, 64], [64, 64], 0.99, (2, 6), 0.2, -20.0, 2.0),   # done inside
    (5, 9, 0, 4, 1, 2, 1, [32, 64, 32], [64, 16, 64], 0.99, (0, 8), 0.5, -0.1, 0.1),  # clamps
    (3, 7, 5, 3, 3, 3, 2, [5, 7, 9], [3, 4, 5], 1.0, (0, 6), 1.5, -0.3, 0.2),
    (2, 10, 9, 4, 1, 5, 3, [1], [2], 0.5, (9,), 0.05, -20.0, 2.0),
    (4, 12, 6, 2, 1, 60, 4, [32, 32], [32, 32], 0.99, (11,), 0.2, -0.2, 0.2),   # F + A = 64
    (2, 5, 2, 3, 1, 1, 32, [2, 64], [64, 3], 0.99, (0,), 0.3, -0.5, 0.5),       # head 2A = 64
]


def _case(case):
    n_step, C, cursor, E, Np, F, A, ad, cd, gamma, done_slots, alpha, lo, hi = case
    models = make_sac_models(F, A, ad, cd, seed=C + A, lo=lo, hi=hi)
    ring = make_ring(C, E, Np, F, A, done_slots, seed=n_step + C)
    ring[0][:] *= 3.0                  # larger observations: clamped log-stds
    g = np.random.default_rng(C)
    valid = C - n_step + 1
    critic_noise = g.standard_normal((valid, E, Np, A))
    actor_noise = g.standard_normal((valid, E, Np, A))
    return models, ring, critic_noise, actor_noise


def _refs(case, models, ring, critic_noise, actor_noise):
    n_step, C, cursor, E, Np, F, A, ad, cd, gamma, done_slots, alpha, lo, hi = case
    lw = [layers(m) for m in models]
    ref = sac_critic_update(*ring, cursor, n_step, gamma, 2.0, 0.25, lo, hi, alpha,
                            critic_noise, *lw)
    aref = sac_actor_update(ring[0], cursor, n_step, 2.0, 0.25, lo, hi, alpha, actor_noise,
                            lw[0], lw[1], lw[2])
    return ref, aref


@pytest.mark.parametrize("case", CASES, ids=[f"case{i}" for i in range(len(CASES))])
def test_reference_matches_torch_autograd_in_float64(case):
    n_step, C, cursor, E, Np, F, A, ad, cd, gamma, done_slots, alpha, lo, hi = case
    models, ring, cn, an = _case(case)
    got = torch_sac(models, ring, cn, an, cursor, n_step, gamma, alpha)
    ref, aref = _refs(case, models, ring, cn, an)
    assert abs(ref["critic1_loss"] - got["l1"]) <= 1e-12 * abs(got["l1"])
    assert abs(ref["critic2_loss"] - got["l2"]) <= 1e-12 * abs(got["l2"])
    assert abs(aref["actor_loss"] - got["actor_loss"]) <= 1e-12 * abs(got["actor_loss"])
    assert rel(ref["returns"], got["returns"]) <= 1e-12
    assert rel(aref["log_probs"], got["log_pi"]) <= 1e-12
    M = aref["log_probs"].size
    target_entropy = -float(A)
    want_alpha_grad = -(aref["sum_log_pi"] / M + target_entropy)
    assert got["alpha_grad"] == pytest.approx(want_alpha_grad, rel=1e-12, abs=1e-12)
    assert got["alpha_grad_algo"] == pytest.approx(want_alpha_grad, rel=1e-12, abs=1e-12)
    for want, have in ((ref["critic_grads"], got["critic"]), (ref["critic2_grads"],
                                                              got["critic2"]),
                       (aref["actor_grads"], got["actor"])):
        for (dw, db), (tw, tb) in zip(want, have):
            assert rel(dw, tw) <= 1e-12 and rel(db, tb) <= 1e-12


def test_cases_reach_both_clamps_both_critics_and_the_window_rules():
    hit = {k: False for k in ("low", "high", "q1", "q2", "actor_q1", "actor_q2", "done_inside",
                              "last_window_done", "last_window_bootstrapped")}
    for case in CASES:
        n_step, C, cursor, E, Np, F, A, ad, cd, gamma, done_slots, alpha, lo, hi = case
        models, ring, cn, an = _case(case)
        ref, aref = _refs(case, models, ring, cn, an)
        for r in (ref, aref):
            hit["low"] |= bool(r["clamped_low"].any())
            hit["high"] |= bool(r["clamped_high"].any())
        hit["q1"] |= bool(ref["min_is_first"].any())
        hit["q2"] |= bool((~ref["min_is_first"]).any())
        hit["actor_q1"] |= bool(aref["min_is_first"].any())
        hit["actor_q2"] |= bool((~aref["min_is_first"]).any())
        order = (cursor + np.arange(C)) % C
        done = ring[3][order]
        valid = C - n_step + 1
        # a done at a window's step before its last cuts the return
        hit["done_inside"] |= bool(n_step > 1 and done[:valid + n_step - 2].any())
        # the last window's rule: its reward alone when its last step (slot C - 1) is done,
        # else reward + the undiscounted bootstrap value -- both branches occur
        hit["last_window_done"] |= bool(done[C - 1].any())
        hit["last_window_bootstrapped"] |= bool((done[C - 1] == 0).any())
    assert all(hit.values()), hit


def test_squashed_log_prob_matches_torch_distributions():
    from torch.distributions import Normal, TransformedDistribution
    from torch.distributions.transforms import TanhTransform

    from warp_drive_b200.training.models.fully_connected_actor_critic import squashed_log_prob

    g = torch.Generator().manual_seed(0)
    mu = torch.randn(200, 3, generator=g, dtype=torch.float64) * 2
    log_std = torch.rand(200, 3, generator=g, dtype=torch.float64) * 3 - 2
    eps = torch.randn(200, 3, generator=g, dtype=torch.float64)
    u = mu + log_std.exp() * eps
    dist = TransformedDistribution(Normal(mu, log_std.exp()), [TanhTransform()])
    want = dist.log_prob(torch.tanh(u)).sum(-1)
    got = squashed_log_prob(u, log_std, eps)
    keep = torch.tanh(u).abs() < 1 - 1e-9      # tanh rounds to +-1 past that: log 0 there
    assert keep.all(dim=-1).sum() > 150
    assert torch.allclose(got[keep.all(dim=-1)], want[keep.all(dim=-1)], rtol=1e-9, atol=1e-9)


def test_actor_forward_is_the_squashed_mean_and_sample_uses_the_clamp():
    models = make_sac_models(3, 2, [8], [8], seed=1, lo=-0.5, hi=0.5)
    actor = models[0]
    assert actor.is_squashed_gaussian and actor.policy_head.out_features == 4
    obs = torch.randn(5, 1, 3, dtype=torch.float64) * 10
    z = actor.head_output(obs)
    mu, log_std = actor.mean_and_log_std(obs)
    assert torch.equal(mu, z[..., :2])
    assert torch.equal(log_std, z[..., 2:].clamp(-0.5, 0.5))
    out = torch.cat(actor(obs), dim=-1)
    assert torch.allclose(out, 2.0 * torch.tanh(mu) + 0.25)
    a, _ = actor.sample(obs, torch.zeros(5, 1, 2, dtype=torch.float64))
    assert torch.allclose(a, out)


def test_sac_update_struct_layout_matches_the_header(tmp_path):
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    c_name = "wdb_sac_update_args"
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
    assert ctypes.sizeof(wlib.SacUpdate) == got["size"]
    assert [n for n, _ in wlib.SacUpdate._fields_] == fields
    for f in fields:
        assert getattr(wlib.SacUpdate, f).offset == got[f], f


def _struct(F=3, A=1, ad=(64, 64), cd=(64, 64), E=10, Np=1, C=9, n_step=5, cursor=0,
            lo=-20.0, hi=2.0):
    from warp_drive_b200 import lib as wlib

    u = wlib.SacUpdate()
    u.n_envs, u.n_agents, u.obs_dim, u.action_dim = E, Np, F, A
    u.capacity, u.cursor, u.n_step = C, cursor, n_step
    u.log_std_min, u.log_std_max = lo, hi
    for net, dims in ((u.actor, ad), (u.critic, cd), (u.critic2, cd), (u.target_critic, cd),
                      (u.target_critic2, cd)):
        net.n_hidden = len(dims)
        for i, w in enumerate(dims[:3]):
            net.widths[i] = w
    return u


def _both(u):
    from warp_drive_b200 import lib as wlib

    L = wlib.load()
    return (L.wdb_sac_critic_update_supported(ctypes.byref(u)),
            L.wdb_sac_actor_update_supported(ctypes.byref(u)))


def test_supported_accepts_exactly_the_documented_shapes():
    from warp_drive_b200 import lib as wlib

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    assert _both(_struct()) == (1, 1)                              # single_pendulum_sac
    assert _both(_struct(F=2)) == (1, 1)                           # continuous mountain car
    assert _both(_struct(ad=(), cd=())) == (1, 1)
    assert _both(_struct(ad=(1, 1, 1), cd=(64, 1, 64))) == (1, 1)
    assert _both(_struct(F=60, A=4, ad=(32, 32), cd=(32, 32))) == (1, 1)
    assert _both(_struct(F=1, A=32, ad=(2, 64), cd=(64, 3))) == (1, 1)   # head 2A = 64
    assert _both(_struct(n_step=1, C=2)) == (1, 1) and _both(_struct(cursor=8, Np=3)) == (1, 1)
    assert _both(_struct(lo=0.5, hi=0.5)) == (1, 1)
    # the actor and four critics in shared memory: three hidden layers of 64 fit the actor
    # pass only
    assert _both(_struct(ad=(64, 64, 64), cd=(64, 64, 64))) == (0, 1)
    for bad in (_struct(F=1, A=33, ad=(8,), cd=(8,)), _struct(F=63, A=2), _struct(ad=(65, 64)),
                _struct(cd=(64, 0)), _struct(ad=(8, 8, 8, 8)), _struct(n_step=6, C=5),
                _struct(cursor=9), _struct(E=0), _struct(A=0), _struct(n_step=1, C=1),
                _struct(lo=1.0, hi=0.0), _struct(lo=float("nan"))):
        assert _both(bad) == (0, 0)
    for name in ("critic2", "target_critic", "target_critic2"):
        u = _struct()
        getattr(u, name).widths[1] = 32                            # shaped as the critic
        assert _both(u) == (0, 0), name
    L = wlib.load()
    assert L.wdb_sac_critic_update_workspace_bytes(ctypes.byref(_struct(ad=(65,)))) == -1
    assert L.wdb_sac_actor_update_workspace_bytes(ctypes.byref(_struct(ad=(65,)))) == -1
    assert L.wdb_sac_critic_update_workspace_bytes(ctypes.byref(_struct())) > 0


def test_run_config_loads_as_sac():
    from warp_drive_b200.training.trainer import load_run_config

    cfg = load_run_config("single_pendulum_sac")
    ddpg = load_run_config("single_pendulum")
    pol = cfg["policy"]["shared"]
    assert pol["algorithm"] == "SAC"
    assert (pol["alpha"], pol["autotune_alpha"]) == (0.2, True)
    assert not cfg.get("sampler", {}).get("params")
    assert cfg["trainer"] == ddpg["trainer"]
    assert pol["model"]["actor"]["type"] == "fully_connected_sac_actor"
    assert pol["model"]["actor"]["fc_dims"] == ddpg["policy"]["shared"]["model"]["actor"][
        "fc_dims"]
    assert pol["model"]["critic"] == ddpg["policy"]["shared"]["model"]["critic"]
    assert set(pol["model"]["model_ckpt_filepath"]) == {"actor", "critic", "critic2", "alpha"}


@pytest.mark.parametrize("kw", [{"normalize_return": True}, {"alpha": 0.0}, {"alpha": -0.1},
                                {"target_entropy": float("nan")},
                                {"target_entropy": float("inf")}])
def test_sac_refuses_what_it_does_not_train(kw):
    from warp_drive_b200.training.algorithms.sac import SAC

    with pytest.raises(ValueError):
        SAC(n_step=5, **kw)


def test_sac_defaults():
    from warp_drive_b200.training.algorithms.sac import SAC

    algo = SAC(n_step=5, action_dim=3)
    assert (algo.alpha, algo.autotune_alpha, algo.target_entropy) == (0.2, True, -3.0)


def test_temperature_refuses_a_non_positive_alpha():
    from warp_drive_b200.training.trainer_sac import Temperature

    assert float(Temperature(0.5).log_alpha.detach().exp()) == pytest.approx(0.5)
    for bad in (0.0, -1.0):
        with pytest.raises(ValueError):
            Temperature(bad)


def test_actor_needs_a_box_action_space():
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils import spaces

    env = _Env(3, 1)
    env.env.action_space = {0: spaces.Discrete(3)}
    with pytest.raises(AssertionError, match="Box action space"):
        ModelFactory.create("fully_connected_sac_actor")(
            env=env, model_config={"type": "fully_connected_sac_actor", "fc_dims": [8]},
            policy="shared", policy_tag_to_agent_id_map={"shared": [0]})


def _policy_model_stub(actor_type, sampler_params):
    """A TrainerSAC with only what _initialize_policy_model reads: the policy config, the
    sampler params and a model builder on a CPU stand-in env."""
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.training.trainer_sac import TrainerSAC

    tr = object.__new__(TrainerSAC)
    tr.config = {"policy": {"shared": {
        "algorithm": "SAC", "model": {"actor": {"type": actor_type, "fc_dims": [8]},
                                      "critic": {"type": "fully_connected_action_value_critic",
                                                 "fc_dims": [8]}}}}}
    tr.sample_params_schedules = dict(sampler_params)
    tr._create_network_dicts()
    tr._build_model = lambda policy, cfg: ModelFactory.create(cfg["type"])(
        env=_Env(3, 1), model_config=cfg, policy=policy,
        policy_tag_to_agent_id_map={"shared": [0]})
    return tr


def test_trainer_builds_the_sac_models():
    tr = _policy_model_stub("fully_connected_sac_actor", {})
    tr._initialize_policy_model("shared")
    assert tr.actor_models["shared"].is_squashed_gaussian
    assert float(tr.temperatures["shared"].log_alpha.detach().exp()) == pytest.approx(0.2)


def test_trainer_refuses_sampler_params():
    tr = _policy_model_stub("fully_connected_sac_actor", {"damping": 1.0, "stddev": 0.2})
    with pytest.raises(ValueError, match="sampler params"):
        tr._initialize_policy_model("shared")


def test_trainer_refuses_another_actor_type():
    tr = _policy_model_stub("fully_connected_actor", {})
    with pytest.raises(ValueError, match="fully_connected_sac_actor"):
        tr._initialize_policy_model("shared")


def test_trainer_refuses_separate_placeholders():
    from warp_drive_b200.training.trainer_sac import TrainerSAC

    with pytest.raises(AssertionError, match="separate per-policy placeholders"):
        TrainerSAC(env_wrapper=None, config={}, create_separate_placeholders_for_each_policy=True)


def test_min_first_sends_ties_to_q1():
    from warp_drive_b200.training.algorithms.sac import min_first

    q1 = torch.tensor([1.0, 2.0, 3.0], requires_grad=True)
    q2 = torch.tensor([1.0, 1.0, 4.0], requires_grad=True)
    min_first(q1, q2).sum().backward()
    assert q1.grad.tolist() == [1.0, 0.0, 1.0] and q2.grad.tolist() == [0.0, 1.0, 0.0]


# ------------------------------------------------------------------------ ptxas
def _cubin(src, tmp_path):
    out = str(tmp_path / (os.path.basename(src) + ".cubin"))
    proc = subprocess.run(NVCC_SM90A + ["-Xptxas", "-v", "-cubin", "-I",
                                        os.path.join(ROOT, "include"), src, "-o", out],
                          capture_output=True, text=True, check=True)
    stats, name = {}, None
    for line in proc.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = m.group(1)
            stats[name] = {}
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name and "spill" not in stats[name]:
            stats[name]["spill"] = (int(m.group(1)), int(m.group(2)))
    return stats, out


def _sass_hashes(cubin, keys):
    """Normalised SASS (addresses and the function's own name dropped) per kernel whose
    mangled name contains one of `keys` (and not "squashed")."""
    sass = subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True,
                          check=True).stdout
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            name = m.group(1)
            cur = next((k for k in keys if k in name and "squashed" not in name), None)
            if cur is not None:
                assert cur not in funcs, (cur, name)
                funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(re.sub(r"/\*[0-9a-f]{4}\*/", "", line).rstrip())
    return {k: hashlib.sha256("\n".join(v).encode()).hexdigest() for k, v in funcs.items()}


# The normalised SASS of the kernels that existed before SAC joined their files, recorded at
# the parent commit with nvcc 12.9.
_KEPT_SASS_SHA256 = {
    "wdb_ddpg_update.cu": {
        "ddpg_update_kernel" + RING:
            "43727eb73fb299e5ca72c15d364be91aa0dc4bb253d8bcd24a5d3ef3d3cdd04f",
        "ddpg_reduce_kernel": "4ad80efbdf62dead0279d0872ad06dadfc625476fb41c2e1bf18b8292e280def",
        "td3_critic_kernel" + RING:
            "9ea51c60bf071869f36de6c0668b280a7dc51dc454cd5abd4af04307c46f3ac4",
        "td3_actor_kernel" + RING:
            "baa1f44c5fde6671d02a45f1973dd31e95d8d52b2cd29ad6f81c106bc5a9b612",
    },
    "wdb_core.cu": {
        "sample_gaussian_kernel":
            "43163a52804c973bfde1ce684bc53e617e752aa4a676ad574ddf64036a004738",
    },
    "wdb_sa_rollout.cu": {
        "sa_rollout_kernelILi0E": "281b4fbcb8b090b3c004a7177d116ce01d9f7eccf7464bf76181381d465fcdc4",
        "sa_rollout_kernelILi1E": "e9440085d721d2e49daea49ee9cadf190d1c7a71770c05d72b8550214242d2d5",
        "sa_rollout_kernelILi2E": "416864e0a61a02291bba8789103b3352cd9a4d1eb33bf5297b197f921bb73080",
    },
}


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_sac_ring_passes_compile_without_spills_and_existing_kernels_keep_their_code(tmp_path):
    stats, _ = _cubin(os.path.join(CSRC, "wdb_ddpg_update.cu"), tmp_path)
    for k in ("sac_critic_kernel" + RING, "sac_actor_kernel" + RING):
        hits = [v for n, v in stats.items() if k in n]
        assert len(hits) == 1, (k, list(stats))
        assert hits[0]["spill"] == (0, 0), (k, hits[0])
    stats, _ = _cubin(os.path.join(CSRC, "wdb_core.cu"), tmp_path)
    hits = [v for n, v in stats.items() if "sample_squashed_gaussian_kernel" in n]
    assert len(hits) == 1 and hits[0]["spill"] == (0, 0), hits
    # the one-launch rollout's squashed-Gaussian instantiation (kSaSquashed = 3)
    stats, _ = _cubin(os.path.join(CSRC, "wdb_sa_rollout.cu"), tmp_path)
    hits = [v for n, v in stats.items() if "sa_rollout_kernelILi3E" in n]
    assert len(hits) == 1 and hits[0]["spill"] == (0, 0), hits
    version = subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout
    if "release 12.9" not in version:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    for src, want in _KEPT_SASS_SHA256.items():
        _, cubin = _cubin(os.path.join(CSRC, src), tmp_path)
        got = _sass_hashes(cubin, list(want))
        assert got == want, src
