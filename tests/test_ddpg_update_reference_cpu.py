"""The float64 restatement of the DDPG update (tests/ddpg_update_reference.py), which the GPU
tests hold `wdb_ddpg_update` to, pinned on the CPU to what TrainerDDPG's torch update computes
by autograd -- the real DDPG class and actor / critic modules, in float64 -- across the shapes
the kernel takes; plus the layout of the new ABI struct and the support check."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import load_golden
from ddpg_update_reference import ddpg_update, n_step_returns

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class _Env:
    """What the model classes read from an EnvWrapper (no device needed)."""

    class _DM:
        def get_shape(self, name=None):
            return (8, 4, 1, 3)

    def __init__(self, F, A):
        from warp_drive_b200.utils import spaces

        class _E:
            observation_space = {0: spaces.Box(-1.0, 1.0, shape=(F,), dtype=np.float32)}
            action_space = {0: spaces.Box(-2.0, 2.0, shape=(A,), dtype=np.float32)}

        self.env = _E()
        self.n_agents = 1
        self.cuda_data_manager = self._DM()


def make_models(F, A, actor_dims, critic_dims, scale=2.0, bias=0.0, seed=0):
    from warp_drive_b200.training.models.fully_connected import ModelFactory

    torch.manual_seed(seed)
    kw = dict(env=_Env(F, A), policy="shared", policy_tag_to_agent_id_map={"shared": [0]})
    mk = lambda kind, dims, **extra: ModelFactory.create(kind)(  # noqa: E731
        model_config={"type": kind, "fc_dims": dims, **extra}, **kw).double()
    actor = mk("fully_connected_actor", actor_dims, output_w=scale, output_b=bias)
    critic = mk("fully_connected_action_value_critic", critic_dims)
    t_actor = mk("fully_connected_actor", actor_dims, output_w=scale, output_b=bias)
    t_critic = mk("fully_connected_action_value_critic", critic_dims)
    return actor, critic, t_actor, t_critic


def layers(model):
    from warp_drive_b200.training.algorithms.fused_ddpg import _layers

    return [(w.detach().numpy(), b.detach().numpy()) for w, b in _layers(model)]


def make_ring(C, E, Np, F, A, done_slots=(), seed=0):
    g = np.random.default_rng(seed)
    obs = g.standard_normal((C, E, Np, F))
    actions = g.uniform(-2, 2, (C, E, Np, A))
    rewards = g.standard_normal((C, E, Np))
    done = (g.random((C, E)) < 0.2).astype(np.int32)
    for s in done_slots:
        done[s] = 1
    return obs, actions, rewards, done


def torch_update(models, ring, cursor, n_step, gamma):
    """TrainerDDPG._torch_gradients in float64 on the unrolled ring."""
    from warp_drive_b200.training.algorithms.ddpg import DDPG

    actor, critic, t_actor, t_critic = models
    C = ring[0].shape[0]
    order = (cursor + np.arange(C)) % C
    obs, actions, rewards, done = (torch.from_numpy(np.ascontiguousarray(x[order])) for x in ring)
    for m in (actor, critic):
        m.zero_grad()
    probs = actor(obs=obs)
    with torch.no_grad():
        target_probs = t_actor(obs=obs)
        next_values = t_critic(obs=obs[1:], action=[p[1:] for p in target_probs])
    values = critic(obs=obs, action=actions)
    j_values = critic(obs=obs, action=probs)
    algo = DDPG(discount_factor_gamma=gamma, n_step=n_step)
    actor_loss, critic_loss, _ = algo.compute_loss_and_metrics(
        1, actions, rewards, done, values, next_values, j_values)
    actor_loss.backward()
    critic_loss.backward()
    from warp_drive_b200.training.algorithms.fused_ddpg import _layers

    grads = lambda m: [(w.grad.numpy(), b.grad.numpy()) for w, b in _layers(m)]  # noqa: E731
    return float(actor_loss), float(critic_loss), grads(actor), grads(critic)


def rel(a, b):
    return np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(np.asarray(b)),
                                                                1e-300)


# (n_step, C, cursor, E, Np, F, A, actor dims, critic dims, gamma, done slots)
CASES = [
    (1, 2, 1, 5, 1, 3, 1, [64, 64], [64, 64], 0.99, ()),
    (1, 9, 4, 4, 2, 3, 1, [8], [8], 0.99, (0,)),
    (2, 2, 1, 3, 1, 2, 1, [16, 16], [16, 16], 1.0, (1,)),
    (3, 7, 0, 3, 3, 3, 1, [5, 7, 9], [3, 4, 5], 0.99, (0, 6)),
    (4, 12, 6, 2, 1, 4, 2, [1], [1], 0.0, (11,)),
    (5, 5, 2, 6, 1, 3, 1, [64, 64], [64, 64], 0.99, (2,)),
    (5, 9, 0, 4, 1, 2, 1, [32, 64, 32], [64, 16, 64], 0.99, (0, 8)),
    (5, 13, 12, 2, 2, 3, 1, [64], [64], 1.0, ()),
    (2, 6, 3, 2, 1, 63, 1, [64, 64], [64, 64], 0.99, (5,)),
    (3, 5, 4, 2, 1, 1, 63, [2, 64], [64, 3], 0.5, (0,)),
    (2, 4, 0, 3, 1, 32, 32, [33, 17], [64], 0.99, (3,)),
]


@pytest.mark.parametrize("case", CASES, ids=[f"case{i}" for i in range(len(CASES))])
def test_reference_matches_torch_autograd_in_float64(case):
    n_step, C, cursor, E, Np, F, A, ad, cd, gamma, done_slots = case
    models = make_models(F, A, ad, cd, scale=2.0, bias=0.25, seed=C)   # targets differ
    ring = make_ring(C, E, Np, F, A, done_slots, seed=n_step + C)
    a_loss, c_loss, ga, gc = torch_update(models, ring, cursor, n_step, gamma)
    ref = ddpg_update(*ring, cursor, n_step, gamma, 2.0, 0.25, *[layers(m) for m in models])
    assert abs(ref["actor_loss"] - a_loss) <= 1e-12 * abs(a_loss)
    assert abs(ref["critic_loss"] - c_loss) <= 1e-12 * abs(c_loss)
    for got, want in ((ref["actor_grads"], ga), (ref["critic_grads"], gc)):
        for (dw, db), (tw, tb) in zip(got, want):
            assert rel(dw, tw) <= 1e-12 and rel(db, tb) <= 1e-12


def test_reference_returns_and_losses_match_the_reference_class_vectors():
    g = load_golden("ddpg_reference.npz")
    for c in range(int(g["n_cases"])):
        T, E, Np, n, gamma, nr, na = g[f"case{c}__cfg"]
        if nr:
            continue
        T, n = int(T), int(n)
        valid = T - n + 1
        nv = g[f"case{c}__next_values"].astype(np.float64)
        qt = np.stack([nv[i + n - 1] if i < valid - 1 else nv[-1] for i in range(valid)])
        ret = n_step_returns(g[f"case{c}__rewards"].astype(np.float64), g[f"case{c}__done"],
                             qt, n, float(gamma))
        values = g[f"case{c}__values"].astype(np.float64)[:valid]
        critic_loss = float(((values - ret) ** 2).mean())
        actor_loss = -float(g[f"case{c}__j_values"].astype(np.float64)[:valid].mean())
        assert critic_loss == pytest.approx(float(g[f"case{c}__critic_loss"]), rel=1e-5, abs=1e-6)
        assert actor_loss == pytest.approx(float(g[f"case{c}__actor_loss"]), rel=1e-5, abs=1e-6)
        assert ret.mean() == pytest.approx(float(g[f"case{c}__mean_returns"]), rel=1e-5, abs=1e-6)


def test_ddpg_update_struct_layout_matches_the_header(tmp_path):
    from test_abi_layout_cpu import _c_fields
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    pairs = {"wdb_ddpg_net": "DdpgNet", "wdb_ddpg_update_args": "DdpgUpdate"}
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "wdb200.h"', "int main(void) {"]
    fields = {}
    for c_name in pairs:
        fields[c_name] = _c_fields(header, c_name)
        lines.append(f'  printf("{c_name} size %zu\\n", sizeof({c_name}));')
        for f in fields[c_name]:
            lines.append(f'  printf("{c_name} {f} %zu\\n", offsetof({c_name}, {f}));')
    lines += ["  return 0;", "}"]
    (tmp_path / "layout.c").write_text("\n".join(lines))
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(tmp_path / "layout"),
                    str(tmp_path / "layout.c")], check=True)
    out = subprocess.run([str(tmp_path / "layout")], check=True, capture_output=True,
                         text=True).stdout
    got = {(s, f): int(v) for s, f, v in (line.split() for line in out.splitlines())}
    for c_name, py_name in pairs.items():
        cls = getattr(wlib, py_name)
        assert ctypes.sizeof(cls) == got[(c_name, "size")]
        assert [n for n, _ in cls._fields_] == fields[c_name]
        for f in fields[c_name]:
            assert getattr(cls, f).offset == got[(c_name, f)], (c_name, f)


def _struct(F=3, A=1, ad=(64, 64), cd=(64, 64), E=10, Np=1, C=9, n_step=5, cursor=0):
    from warp_drive_b200 import lib as wlib

    u = wlib.DdpgUpdate()
    u.n_envs, u.n_agents, u.obs_dim, u.action_dim = E, Np, F, A
    u.capacity, u.cursor, u.n_step = C, cursor, n_step
    for net, dims in ((u.actor, ad), (u.critic, cd), (u.target_actor, ad), (u.target_critic, cd)):
        net.n_hidden = len(dims)
        for i, w in enumerate(dims[:3]):
            net.widths[i] = w
    return u


def _supported(u):
    from warp_drive_b200 import lib as wlib

    return wlib.load().wdb_ddpg_update_supported(ctypes.byref(u)) == 1


def test_supported_accepts_exactly_the_documented_shapes():
    from warp_drive_b200 import lib as wlib

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    assert _supported(_struct())                                   # both reference configs
    assert _supported(_struct(F=2))
    assert _supported(_struct(ad=(), cd=()))                       # no hidden layer
    assert _supported(_struct(ad=(1, 1, 1), cd=(64, 1, 64)))
    assert _supported(_struct(F=63, A=1, ad=(32, 32), cd=(32, 32)))
    assert _supported(_struct(F=1, A=63, ad=(2, 64), cd=(64, 3)))
    # every network in shared memory: [64, 64] with F + A = 64 does not fit
    assert not _supported(_struct(F=63, A=1))
    assert _supported(_struct(n_step=1, C=2)) and _supported(_struct(cursor=8, Np=3))
    assert _supported(_struct(n_step=2, C=2)) and not _supported(_struct(n_step=1, C=1))
    assert not _supported(_struct(F=63, A=2))                      # F + A > 64
    assert not _supported(_struct(ad=(65, 64)))                    # width 65
    assert not _supported(_struct(cd=(64, 0)))                     # width 0
    assert not _supported(_struct(ad=(8, 8, 8, 8)))                # 4 hidden layers
    assert not _supported(_struct(ad=(64, 64, 64), cd=(64, 64, 64), F=60, A=4))   # smem
    assert not _supported(_struct(n_step=6, C=5)) and not _supported(_struct(cursor=9))
    assert not _supported(_struct(E=0)) and not _supported(_struct(A=0))
    u = _struct()
    u.target_actor.widths[1] = 32                                  # targets shaped as online
    assert not _supported(u)
    assert wlib.load().wdb_ddpg_update_workspace_bytes(ctypes.byref(_struct(ad=(65,)))) == -1
