"""`wdb_td3_critic_update` and `wdb_td3_actor_update` against the float64 restatement of the
TD3 update (tests/td3_update_reference.py): every gradient, per-row output and loss sum within
an a-priori float32 bound, bit-identical on two launches, nothing written outside the outputs;
an unsupported struct is refused without a launch."""
import ctypes

import numpy as np
import pytest
import torch

from td3_update_reference import td3_actor_update, td3_critic_update
from test_ddpg_update_reference_cpu import layers, make_models, make_ring
from test_gpu_ddpg_update_exact import GUARD, SENTINEL, U, _chain, _chain_forward, _guarded

pytestmark = pytest.mark.gpu


def _models(F, A, ad, cd, seed):
    actor, critic, t_actor, t_critic = make_models(F, A, ad, cd, scale=2.0, bias=0.25, seed=seed)
    _, critic2, _, t_critic2 = make_models(F, A, ad, cd, scale=2.0, bias=0.25,
                                           seed=seed + 1000)
    return [m.float() for m in (actor, critic, critic2, t_actor, t_critic, t_critic2)]


def _run(case, seed):
    n_step, C, cursor, E, Np, F, A, ad, cd, gamma, done_slots, sigma, clip = case
    models = _models(F, A, ad, cd, seed)
    # wide rings repeat 8 distinct envs: many rows and CTAs, few distinct ReLU pre-activations
    E0 = 8 if E > 16 else E
    ring = make_ring(C, E0, Np, F, A, done_slots, seed=seed)
    ring = [np.concatenate([r] * (E // E0), axis=1) for r in ring]
    ring32 = [r.astype(np.float32) if r.dtype != np.int32 else r for r in ring]
    valid = C - n_step + 1
    noise = np.random.default_rng(seed).standard_normal((valid, E0, Np, A))
    noise = np.concatenate([noise] * (E // E0), axis=1).astype(np.float32)
    lw = [[(w.astype(np.float64), b.astype(np.float64)) for w, b in layers(m)] for m in models]
    args = (*ring32, cursor, n_step, gamma, 2.0, 0.25, sigma, clip, noise, *lw[1:])
    ref = td3_critic_update(*args)
    absr = td3_critic_update(*args, absolute=True)
    aargs = (ring32[0], cursor, n_step, 2.0, 0.25, lw[0], lw[1])
    aref, aabs = td3_actor_update(*aargs), td3_actor_update(*aargs, absolute=True)
    return [m.cuda() for m in models], ring32, noise, (ref, absr), (aref, aabs)


def _accept(pairs, N):
    """Every ReLU pre-activation lies outside its rounding bound of zero (N: _chain_forward)."""
    for ref, absr in pairs:
        for name, pres in ref["pre"].items():
            for z, za in zip(pres, absr["pre"][name]):
                if (np.abs(z) <= (N + 2) * U * za).any():
                    return False
    return True


CASES = [
    # (n_step, C, cursor, E, Np, F, A, actor dims, critic dims, gamma, done slots, sigma, clip)
    (5, 9, 0, 40, 1, 3, 1, [64, 64], [64, 64], 0.99, (0, 8), 0.2, 0.5),     # single_pendulum_td3
    (5, 9, 4, 40, 1, 2, 1, [64, 64], [64, 64], 0.99, (), 0.2, 0.5),         # continuous mountain car
    (5, 9, 7, 440, 1, 3, 1, [64, 64], [64, 64], 0.99, (3,), 0.2, 0.5),      # > 132 tiles
    (1, 2, 1, 32, 2, 3, 1, [16], [16], 0.0, (1,), 1.0, 0.5),
    (3, 7, 5, 12, 3, 4, 2, [5, 7, 9], [3, 4, 5], 1.0, (0, 6), 2.0, 0.3),   # clamps
    (2, 10, 9, 9, 1, 5, 3, [1], [2], 0.99, (9,), 0.2, 0.5),                 # width 1 and 2
    (4, 12, 6, 4, 1, 63, 1, [32, 32], [32, 32], 0.5, (11,), 0.2, 0.5),      # F + A = 64
    (2, 5, 2, 8, 1, 1, 63, [2, 64], [64, 3], 0.99, (0,), 0.2, 0.5),
]


@pytest.mark.parametrize("case", CASES, ids=[f"case{i}" for i in range(len(CASES))])
def test_td3_update_within_float32_bound_of_float64_reference(case):
    from warp_drive_b200.training.algorithms.fused_ddpg import _layers
    from warp_drive_b200.training.algorithms.td3 import TD3
    from warp_drive_b200.training.algorithms.fused_td3 import FusedTD3Update

    n_step, C, cursor, E, Np, F, A, ad, cd, gamma, done_slots, sigma, clip = case
    valid = C - n_step + 1
    M = valid * E * Np
    # the critic pass chains the target actor, the noise / clamps and a target critic into the
    # return: no longer than the DDPG update's chain, which also adds the actor path's
    N = _chain(F, A, ad, cd, n_step, M) + 8
    for seed in range(200):
        models, ring, noise, (ref, absr), (aref, aabs) = _run(case, seed)
        if _accept(((ref, absr), (aref, aabs)), _chain_forward(F, A, ad, cd) + 4):
            break
    else:
        pytest.fail("no input draw kept every ReLU pre-activation off its bound of zero")
    dev = torch.device("cuda")
    actor, critic, critic2 = models[:3]
    guards = []
    for m in (actor, critic, critic2):
        for p in m.parameters():
            buf, view = _guarded(p.shape, dev)
            p.grad = view
            guards.append(buf)
    outs = [_guarded((valid, E, Np), dev) for _ in range(4)]
    guards += [b for b, _ in outs]
    algo = TD3(discount_factor_gamma=gamma, n_step=n_step, target_noise=sigma,
               target_noise_clip=clip)
    fused = FusedTD3Update(algo, *models, E, Np, C, n_step, gamma)
    obs, actions, rewards, done = (torch.from_numpy(np.ascontiguousarray(r)).to(dev)
                                   for r in ring)
    eps = torch.from_numpy(noise).to(dev)

    def launch():
        fused.critic_launch(obs, actions, rewards, done, cursor, eps,
                            tuple(v for _, v in outs[:3]))
        fused.actor_launch(obs, cursor, outs[3][1])
        torch.cuda.synchronize()
        return ([p.grad.clone() for m in (actor, critic, critic2) for p in m.parameters()],
                fused.sums.clone())

    first, sums = launch()

    def check(got, want, bound, what):
        got = got.detach().double().cpu().numpy()
        err = np.abs(got - want)
        lim = (N + 2) * U * bound
        assert (err <= lim).all(), (what, float((err - lim).max()), float(err.max()))

    for m, want, wabs, kind in ((actor, aref["actor_grads"], aabs["actor_grads"], "actor"),
                                (critic, ref["critic_grads"], absr["critic_grads"], "critic"),
                                (critic2, ref["critic2_grads"], absr["critic2_grads"],
                                 "critic2")):
        for l, (w, b) in enumerate(_layers(m)):
            check(w.grad, want[l][0], wabs[l][0], f"{kind} W{l}")
            check(b.grad, want[l][1], wabs[l][1], f"{kind} b{l}")
    for (_, v), (r, a, key) in zip(outs, ((ref, absr, "q1"), (ref, absr, "q2"),
                                          (ref, absr, "returns"), (aref, aabs, "j_values"))):
        check(v, r[key], a[key], key)
    for k, q in ((0, "q1"), (1, "q2")):
        diff = np.abs(ref[q] - ref["returns"])
        dabs = absr[q] + absr["returns"]
        bound = float((2 * diff * dabs + dabs ** 2 * (N + 2) * U).sum())
        assert abs(float(sums[k]) - ref[f"sum_sq_err{k + 1}"]) <= (N + 2) * U * bound
    assert abs(float(sums[2]) - aref["sum_j"]) <= (N + 2) * U * float(aabs["j_values"].sum())
    assert float(sums[3]) == 0.0
    for buf in guards:
        assert bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[-GUARD:] == SENTINEL).all())
    again, sums2 = launch()
    assert all(torch.equal(a, b) for a, b in zip(first, again))
    assert torch.equal(sums, sums2)


def test_unsupported_struct_is_refused_without_a_launch():
    from warp_drive_b200 import lib as wlib

    lib = wlib.load()
    u = wlib.Td3Update()
    u.n_envs, u.n_agents, u.obs_dim, u.action_dim = 4, 1, 3, 1
    u.capacity, u.cursor, u.n_step = 9, 0, 5
    u.target_noise, u.target_noise_clip = 0.2, 0.5
    nets = (u.actor, u.critic, u.critic2, u.target_actor, u.target_critic, u.target_critic2)
    for net in nets:
        net.n_hidden = 2
        net.widths[0], net.widths[1] = 65, 64              # width 65
    before = wlib.launch_count()
    stream = wlib.stream_ptr()
    assert lib.wdb_td3_critic_update(stream, ctypes.byref(u)) == 1   # cudaErrorInvalidValue
    assert lib.wdb_td3_actor_update(stream, ctypes.byref(u)) == 1
    for net in nets:
        net.widths[0] = 64                                  # supported shapes, NULL pointers
    assert lib.wdb_td3_critic_update_supported(ctypes.byref(u)) == 1
    assert lib.wdb_td3_actor_update_supported(ctypes.byref(u)) == 1
    assert lib.wdb_td3_critic_update(stream, ctypes.byref(u)) == 1
    assert lib.wdb_td3_actor_update(stream, ctypes.byref(u)) == 1
    u.target_noise = -0.2                                   # negative noise
    assert lib.wdb_td3_critic_update_supported(ctypes.byref(u)) == 0
    assert wlib.launch_count() == before
