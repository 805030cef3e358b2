"""CPU tests of TD3: the float64 restatement of both update passes (tests/td3_update_reference.py)
pinned to what TrainerTD3's torch update computes by autograd -- the real TD3 class and actor /
critic modules, in float64; the ctypes layout of the new ABI struct; the support envelope; the
run config and the refusals; what ptxas makes of the new kernels, and every kernel of the
fused update file keeping its code."""
import ctypes
import hashlib
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

from td3_update_reference import td3_actor_update, td3_critic_update  # noqa: E402
from test_abi_layout_cpu import _c_fields  # noqa: E402
from test_ddpg_update_reference_cpu import layers, make_models, make_ring, rel  # noqa: E402

NVCC_SM90A = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC"]
CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")


def make_td3_models(F, A, ad, cd, seed):
    """actor, critic, critic2, target actor, target critic, target critic2 (float64; the
    targets differ from the online networks)."""
    actor, critic, t_actor, t_critic = make_models(F, A, ad, cd, scale=2.0, bias=0.25, seed=seed)
    _, critic2, _, t_critic2 = make_models(F, A, ad, cd, scale=2.0, bias=0.25, seed=seed + 1000)
    return actor, critic, critic2, t_actor, t_critic, t_critic2


def torch_td3(models, ring, noise, cursor, n_step, gamma, sigma, clip):
    """TrainerTD3's torch update in float64 on the unrolled ring: critic pass, then actor pass
    (the actor's gradient only)."""
    from warp_drive_b200.training.algorithms.fused_ddpg import _layers
    from warp_drive_b200.training.algorithms.td3 import TD3, torch_actor_loss, torch_critic_loss

    actor, critic, critic2, t_actor, t_critic, t_critic2 = models
    C = ring[0].shape[0]
    order = (cursor + np.arange(C)) % C
    obs, actions, rewards, done = (torch.from_numpy(np.ascontiguousarray(x[order])) for x in ring)
    algo = TD3(discount_factor_gamma=gamma, n_step=n_step, target_noise=sigma,
               target_noise_clip=clip)
    for m in models:
        m.zero_grad()
    boot = torch.tensor(algo.bootstrap_slots(C))
    l1, l2, q1, q2, ret = torch_critic_loss(algo, t_actor, t_critic, t_critic2, critic, critic2,
                                            obs, actions, rewards, done,
                                            torch.from_numpy(noise), boot)
    (l1 + l2).backward()
    valid = C - n_step + 1
    a_loss, _ = torch_actor_loss(algo, actor, critic, obs[:valid])
    critic_grads = [(w.grad.clone(), b.grad.clone()) for w, b in _layers(critic)]
    a_loss.backward(inputs=list(actor.parameters()))
    grads = lambda m: [(w.grad.numpy(), b.grad.numpy()) for w, b in _layers(m)]  # noqa: E731
    # the actor loss left the critic's gradient alone
    for (w, b), (w0, b0) in zip(_layers(critic), critic_grads):
        assert torch.equal(w.grad, w0) and torch.equal(b.grad, b0)
    return dict(l1=l1.item(), l2=l2.item(), actor_loss=a_loss.item(), critic=grads(critic),
                critic2=grads(critic2), actor=grads(actor), returns=ret.numpy())


# (n_step, C, cursor, E, Np, F, A, actor dims, critic dims, gamma, done slots, sigma, clip)
CASES = [
    (1, 2, 1, 5, 1, 3, 1, [64, 64], [64, 64], 0.99, (), 0.2, 0.5),
    (5, 9, 3, 6, 1, 3, 1, [64, 64], [64, 64], 0.99, (2, 6), 0.2, 0.5),   # done inside windows
    (5, 9, 0, 4, 1, 2, 1, [32, 64, 32], [64, 16, 64], 0.99, (0, 8), 1.5, 0.5),  # both clamps
    (3, 7, 5, 3, 3, 3, 2, [5, 7, 9], [3, 4, 5], 1.0, (0, 6), 2.0, 0.3),
    (2, 10, 9, 4, 1, 5, 3, [1], [2], 0.5, (9,), 0.0, 0.0),              # no noise
    (4, 12, 6, 2, 1, 63, 1, [32, 32], [32, 32], 0.99, (11,), 0.2, 0.5),  # F + A = 64
    (2, 5, 2, 3, 1, 1, 63, [2, 64], [64, 3], 0.99, (0,), 3.0, 1.0),
]


def _case(case):
    n_step, C, cursor, E, Np, F, A, ad, cd, gamma, done_slots, sigma, clip = case
    models = make_td3_models(F, A, ad, cd, seed=C + A)
    ring = make_ring(C, E, Np, F, A, done_slots, seed=n_step + C)
    ring[0][:] *= 3.0                  # larger observations: saturated target actions
    noise = np.random.default_rng(C).standard_normal((C - n_step + 1, E, Np, A))
    return models, ring, noise


@pytest.mark.parametrize("case", CASES, ids=[f"case{i}" for i in range(len(CASES))])
def test_reference_matches_torch_autograd_in_float64(case):
    n_step, C, cursor, E, Np, F, A, ad, cd, gamma, done_slots, sigma, clip = case
    models, ring, noise = _case(case)
    got = torch_td3(models, ring, noise, cursor, n_step, gamma, sigma, clip)
    lw = [layers(m) for m in models]
    ref = td3_critic_update(*ring, cursor, n_step, gamma, 2.0, 0.25, sigma, clip, noise,
                            *lw[1:])
    aref = td3_actor_update(ring[0], cursor, n_step, 2.0, 0.25, lw[0], lw[1])
    assert abs(ref["critic1_loss"] - got["l1"]) <= 1e-12 * abs(got["l1"])
    assert abs(ref["critic2_loss"] - got["l2"]) <= 1e-12 * abs(got["l2"])
    assert abs(aref["actor_loss"] - got["actor_loss"]) <= 1e-12 * abs(got["actor_loss"])
    assert rel(ref["returns"], got["returns"]) <= 1e-12
    for want, have in ((ref["critic_grads"], got["critic"]), (ref["critic2_grads"],
                                                              got["critic2"]),
                       (aref["actor_grads"], got["actor"])):
        for (dw, db), (tw, tb) in zip(want, have):
            assert rel(dw, tw) <= 1e-12 and rel(db, tb) <= 1e-12


def test_cases_reach_both_clamps_and_both_critics_in_the_minimum():
    hit = {"noise": False, "low": False, "high": False, "q1": False, "q2": False}
    for case in CASES:
        n_step, C, cursor, E, Np, F, A, ad, cd, gamma, done_slots, sigma, clip = case
        models, ring, noise = _case(case)
        lw = [layers(m) for m in models]
        ref = td3_critic_update(*ring, cursor, n_step, gamma, 2.0, 0.25, sigma, clip, noise,
                                *lw[1:])
        hit["noise"] |= bool(ref["noise_clamped"].any())
        hit["q1"] |= bool(ref["min_is_first"].any())
        hit["q2"] |= bool((~ref["min_is_first"]).any())
        # which side of the action range clamped: recompute the unclamped action's sign
        if ref["action_clamped"].any():
            _, _, _, t_actor, _, _ = models
            C_ = ring[0].shape[0]
            order = (cursor + np.arange(C_)) % C_
            valid = C_ - n_step + 1
            tslot = [i + n_step if i < valid - 1 else C_ - 1 for i in range(valid)]
            ot = torch.from_numpy(ring[0][order][tslot])
            with torch.no_grad():
                pi = torch.cat(list(t_actor(obs=ot)), dim=-1).numpy().reshape(-1, A)
            raw = np.clip(sigma * 2.0 * noise.reshape(-1, A), -clip * 2.0, clip * 2.0)
            a = pi + raw
            hit["low"] |= bool((a < 0.25 - 2.0).any())
            hit["high"] |= bool((a > 0.25 + 2.0).any())
    assert all(hit.values()), hit


def test_done_inside_the_window_cuts_the_return():
    from warp_drive_b200.training.algorithms.td3 import TD3

    algo = TD3(discount_factor_gamma=0.5, n_step=3)
    rewards = torch.ones(5, 1, 1, dtype=torch.float64)
    done = torch.zeros(5, 1, dtype=torch.int32)
    done[1] = 1
    boot = torch.full((3, 1, 1), 10.0, dtype=torch.float64)
    r = algo.returns(rewards, done, boot)
    assert float(r[0]) == 1.5                         # 1 + 0.5 * 1, cut at slot 1
    assert float(r[1]) == 1.0                         # done at its first step
    assert float(r[2]) == pytest.approx(1 + 0.5 * 1 + 0.25 * 10.0)   # last window: undiscounted
    assert algo.bootstrap_slots(5) == [3, 4, 4]


def test_td3_update_struct_layout_matches_the_header(tmp_path):
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    c_name = "wdb_td3_update_args"
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
    assert ctypes.sizeof(wlib.Td3Update) == got["size"]
    assert [n for n, _ in wlib.Td3Update._fields_] == fields
    for f in fields:
        assert getattr(wlib.Td3Update, f).offset == got[f], f


def _struct(F=3, A=1, ad=(64, 64), cd=(64, 64), E=10, Np=1, C=9, n_step=5, cursor=0,
            sigma=0.2, clip=0.5):
    from warp_drive_b200 import lib as wlib

    u = wlib.Td3Update()
    u.n_envs, u.n_agents, u.obs_dim, u.action_dim = E, Np, F, A
    u.capacity, u.cursor, u.n_step = C, cursor, n_step
    u.target_noise, u.target_noise_clip = sigma, clip
    for net, dims in ((u.actor, ad), (u.critic, cd), (u.critic2, cd), (u.target_actor, ad),
                      (u.target_critic, cd), (u.target_critic2, cd)):
        net.n_hidden = len(dims)
        for i, w in enumerate(dims[:3]):
            net.widths[i] = w
    return u


def _both(u):
    from warp_drive_b200 import lib as wlib

    L = wlib.load()
    return (L.wdb_td3_critic_update_supported(ctypes.byref(u)),
            L.wdb_td3_actor_update_supported(ctypes.byref(u)))


def test_supported_accepts_exactly_the_documented_shapes():
    from warp_drive_b200 import lib as wlib

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    assert _both(_struct()) == (1, 1)                              # single_pendulum_td3
    assert _both(_struct(F=2)) == (1, 1)                           # continuous mountain car
    assert _both(_struct(ad=(), cd=())) == (1, 1)
    assert _both(_struct(ad=(1, 1, 1), cd=(64, 1, 64))) == (1, 1)
    assert _both(_struct(F=63, A=1, ad=(32, 32), cd=(32, 32))) == (1, 1)
    assert _both(_struct(F=1, A=63, ad=(2, 64), cd=(64, 3))) == (1, 1)
    assert _both(_struct(n_step=1, C=2)) == (1, 1) and _both(_struct(cursor=8, Np=3)) == (1, 1)
    assert _both(_struct(sigma=0.0, clip=0.0)) == (1, 1)
    # five networks in shared memory: three hidden layers of 64 fit the actor pass only
    assert _both(_struct(ad=(64, 64, 64), cd=(64, 64, 64))) == (0, 1)
    assert _both(_struct(F=63, A=1)) == (0, 1)
    for bad in (_struct(F=63, A=2), _struct(ad=(65, 64)), _struct(cd=(64, 0)),
                _struct(ad=(8, 8, 8, 8)), _struct(n_step=6, C=5), _struct(cursor=9),
                _struct(E=0), _struct(A=0), _struct(n_step=1, C=1), _struct(sigma=-0.1),
                _struct(clip=-1.0)):
        assert _both(bad) == (0, 0)
    for name in ("critic2", "target_critic2", "target_actor"):
        u = _struct()
        getattr(u, name).widths[1] = 32                            # shaped as online
        assert _both(u) == (0, 0), name
    L = wlib.load()
    assert L.wdb_td3_critic_update_workspace_bytes(ctypes.byref(_struct(ad=(65,)))) == -1
    assert L.wdb_td3_actor_update_workspace_bytes(ctypes.byref(_struct(ad=(65,)))) == -1
    assert L.wdb_td3_critic_update_workspace_bytes(ctypes.byref(_struct())) > 0


def test_run_config_loads_as_td3():
    from warp_drive_b200.training.trainer import load_run_config

    cfg = load_run_config("single_pendulum_td3")
    ddpg = load_run_config("single_pendulum")
    pol = cfg["policy"]["shared"]
    assert pol["algorithm"] == "TD3"
    assert (pol["target_noise"], pol["target_noise_clip"], pol["policy_delay"]) == (0.2, 0.5, 2)
    assert cfg["sampler"]["params"]["damping"] == 1.0
    assert cfg["trainer"] == ddpg["trainer"]
    assert pol["model"]["actor"] == ddpg["policy"]["shared"]["model"]["actor"]
    assert pol["model"]["critic"] == ddpg["policy"]["shared"]["model"]["critic"]
    assert set(pol["model"]["model_ckpt_filepath"]) == {"actor", "critic", "critic2"}


@pytest.mark.parametrize("kw", [{"normalize_return": True}, {"policy_delay": 0},
                                {"policy_delay": 1.5}, {"target_noise": -0.1},
                                {"target_noise_clip": -0.5}])
def test_td3_refuses_what_it_does_not_train(kw):
    from warp_drive_b200.training.algorithms.td3 import TD3

    with pytest.raises(ValueError):
        TD3(n_step=5, **kw)


def test_trainer_refuses_separate_placeholders():
    from warp_drive_b200.training.trainer_td3 import TrainerTD3

    with pytest.raises(AssertionError, match="separate per-policy placeholders"):
        TrainerTD3(env_wrapper=None, config={}, create_separate_placeholders_for_each_policy=True)


def test_target_actions_clip_noise_then_action():
    from warp_drive_b200.training.algorithms.td3 import TD3

    algo = TD3(target_noise=0.2, target_noise_clip=0.5)
    pi = torch.tensor([0.0, 1.9, -1.9, 0.0])
    eps = torch.tensor([1.0, 1.0, -1.0, 10.0])
    a = algo.target_actions(pi, eps, 2.0, 0.0)
    assert torch.allclose(a, torch.tensor([0.4, 2.0, -2.0, 1.0]))


# ------------------------------------------------------------------------ ptxas
def _cubin(tmp_path):
    proc = subprocess.run(NVCC_SM90A + ["-Xptxas", "-v", "-cubin",
                                        os.path.join(CSRC, "wdb_ddpg_update.cu"), "-o",
                                        str(tmp_path / "k.cubin")],
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
    return stats, str(tmp_path / "k.cubin")


# Each update pass kernel is a template over its row source; these mangled-name fragments
# select its instantiation over every window of the ring and over sampled windows.
RING = "INS_9NoWindowsE"
SAMPLED = "IPK4int2E"

# The normalised SASS (addresses and the kernel's own name dropped) of every kernel of
# wdb_ddpg_update.cu with nvcc 12.9: both instantiations of each pass, the reduction and DQN's
# pass.
_DDPG_SASS_SHA256 = {
    "ddpg_update_kernel" + RING:
        "43727eb73fb299e5ca72c15d364be91aa0dc4bb253d8bcd24a5d3ef3d3cdd04f",
    "td3_critic_kernel" + RING:
        "9ea51c60bf071869f36de6c0668b280a7dc51dc454cd5abd4af04307c46f3ac4",
    "td3_actor_kernel" + RING:
        "baa1f44c5fde6671d02a45f1973dd31e95d8d52b2cd29ad6f81c106bc5a9b612",
    "sac_critic_kernel" + RING:
        "e963a0aa5bfe088ed0ac0b725bf126499d2386a18edfda269dd6c9078dbb4266",
    "sac_actor_kernel" + RING:
        "5e3dddfb3ee486667e1c9cc52d3fe31e7c70a2445be11b4e0f8cf8ecd3766537",
    "ddpg_update_kernel" + SAMPLED:
        "3c1bc0aad87b8df9296a4e1b260f6561df0e407bc08c6a97ac4f681cd717437e",
    "td3_critic_kernel" + SAMPLED:
        "bdb79e4a2a1926b5d2a56d689ceae355645d294d6a67bbf9c564d66a1b5a73bb",
    "td3_actor_kernel" + SAMPLED:
        "785909197a2abef31f4c2f8fdaf922101bf73d455fe421dbc2377bea8ab4a388",
    "sac_critic_kernel" + SAMPLED:
        "cc8270109477b67b20fd7165e43fee4063342aa9dc811c221db428abad943258",
    "sac_actor_kernel" + SAMPLED:
        "86bea485eed4957d8e592ffcd6888de1976c8e612d9d2266a7242acea2184237",
    "ddpg_reduce_kernel": "4ad80efbdf62dead0279d0872ad06dadfc625476fb41c2e1bf18b8292e280def",
    "dqn_pass_kernel": "6ddc90ace4fb4f4e215234478611c5493c6e854d826da4ab2c899380da37d283",
}


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_td3_ring_passes_compile_without_spills_and_every_update_kernel_keeps_its_code(tmp_path):
    stats, cubin = _cubin(tmp_path)
    for k in ("td3_critic_kernel" + RING, "td3_actor_kernel" + RING):
        hits = [v for n, v in stats.items() if k in n]
        assert len(hits) == 1, (k, list(stats))
        assert hits[0]["spill"] == (0, 0), (k, hits[0])
    version = subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout
    if "release 12.9" not in version:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    sass = subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True,
                          check=True).stdout
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = next((k for k in _DDPG_SASS_SHA256 if k in m.group(1)), None)
            if cur is not None:
                assert cur not in funcs, (cur, m.group(1))
                funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(re.sub(r"/\*[0-9a-f]{4}\*/", "", line).rstrip())
    for k, want in _DDPG_SASS_SHA256.items():
        assert hashlib.sha256("\n".join(funcs[k]).encode()).hexdigest() == want, k
