"""`wdb_ddpg_update` against the float64 restatement of the DDPG update
(tests/ddpg_update_reference.py): every gradient, per-row output and loss sum within an a-priori
float32 bound, bit-identical on two launches, nothing written outside its outputs."""
import numpy as np
import pytest
import torch

from ddpg_update_reference import ddpg_update
from test_ddpg_update_reference_cpu import layers, make_models, make_ring

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
GUARD = 64
SENTINEL = 12345.0


def _chain(F, A, ad, cd, n_step, M):
    """Roundings on the longest accumulation chain of any output: every fan-in sum of the five
    forwards and the three backward passes (each sum counted with its bias add), the head,
    return and loss-gradient arithmetic, and the sum over at most M rows plus the fixed-order
    reduction over at most 132 CTA partials."""
    def fans(ins, dims, out):
        widths = list(dims) + [out]
        fan_in = [ins] + list(dims)
        return sum(k + 1 for k in fan_in) + sum(w + 1 for w in widths)

    per_net = fans(F, ad, A) + fans(F + A, cd, 1)
    return 3 * per_net + 3 * n_step + 24 + M + 132


def _chain_forward(F, A, ad, cd):
    """Roundings on the longest chain into any ReLU pre-activation: the actor, its head and the
    critic's forward (each fan-in sum with its bias add)."""
    return sum(k + 1 for k in [F] + list(ad)) + 4 + sum(k + 1 for k in [F + A] + list(cd))


def _guarded(shape, dev):
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * GUARD,), SENTINEL, device=dev)
    return buf, buf[GUARD:GUARD + n].view(shape)


def _run(case, seed):
    n_step, C, cursor, E, Np, F, A, ad, cd, gamma, done_slots = case
    models = [m.float() for m in make_models(F, A, ad, cd, scale=2.0, bias=0.25, seed=seed)]
    # wide rings repeat 8 distinct envs: many rows and CTAs, few distinct ReLU pre-activations
    E0 = 8 if E > 16 else E
    ring = make_ring(C, E0, Np, F, A, done_slots, seed=seed)
    ring = [np.concatenate([r] * (E // E0), axis=1) for r in ring]
    ring32 = [r.astype(np.float32) if r.dtype != np.int32 else r for r in ring]
    lw = [[(w.astype(np.float64), b.astype(np.float64)) for w, b in layers(m)] for m in models]
    models = [m.cuda() for m in models]
    ref = ddpg_update(*ring32, cursor, n_step, gamma, 2.0, 0.25, *lw)
    absr = ddpg_update(*ring32, cursor, n_step, gamma, 2.0, 0.25, *lw, absolute=True)
    return models, ring32, ref, absr


def _accept(ref, absr, N):
    """Every ReLU pre-activation lies outside its rounding bound of zero (N: _chain_forward)."""
    for name, pres in ref["pre"].items():
        for z, za in zip(pres, absr["pre"][name]):
            if (np.abs(z) <= (N + 2) * U * za).any():
                return False
    return True


CASES = [
    # (n_step, C, cursor, E, Np, F, A, actor dims, critic dims, gamma, done slots)
    (5, 9, 0, 40, 1, 3, 1, [64, 64], [64, 64], 0.99, (0, 8)),        # single_pendulum shapes
    (5, 9, 4, 40, 1, 2, 1, [64, 64], [64, 64], 0.99, ()),            # continuous mountain car
    (5, 9, 7, 440, 1, 3, 1, [64, 64], [64, 64], 0.99, (3,)),         # > 132 tiles
    (1, 2, 1, 32, 2, 3, 1, [16], [16], 0.0, (1,)),
    (3, 7, 5, 12, 3, 4, 2, [5, 7, 9], [3, 4, 5], 1.0, (0, 6)),
    (2, 10, 9, 9, 1, 5, 3, [1], [2], 0.99, (9,)),                    # width 1 and 2
    (4, 12, 6, 4, 1, 63, 1, [32, 32], [32, 32], 0.5, (11,)),         # F + A = 64
    (2, 5, 2, 8, 1, 1, 63, [2, 64], [64, 3], 0.99, (0,)),
]


@pytest.mark.parametrize("case", CASES, ids=[f"case{i}" for i in range(len(CASES))])
def test_ddpg_update_within_float32_bound_of_float64_reference(case):
    from warp_drive_b200.training.algorithms.fused_ddpg import FusedDDPGUpdate, _layers

    n_step, C, cursor, E, Np, F, A, ad, cd, gamma, done_slots = case
    valid = C - n_step + 1
    M = valid * E * Np
    N = _chain(F, A, ad, cd, n_step, M)
    for seed in range(200):
        models, ring, ref, absr = _run(case, seed)
        if _accept(ref, absr, _chain_forward(F, A, ad, cd)):
            break
    else:
        pytest.fail("no input draw kept every ReLU pre-activation off its bound of zero")
    dev = torch.device("cuda")
    actor, critic, t_actor, t_critic = models
    guards = []
    for m in (actor, critic):
        for p in m.parameters():
            buf, view = _guarded(p.shape, dev)
            p.grad = view
            guards.append(buf)
    outs = [_guarded((valid, E, Np), dev) for _ in range(3)]
    guards += [b for b, _ in outs]
    fused = FusedDDPGUpdate(actor, critic, t_actor, t_critic, E, Np, C, n_step, gamma)
    obs, actions, rewards, done = (torch.from_numpy(np.ascontiguousarray(r)).to(dev)
                                   for r in ring)
    sums = fused.launch(obs, actions, rewards, done, cursor, tuple(v for _, v in outs))
    torch.cuda.synchronize()
    first = [p.grad.clone() for m in (actor, critic) for p in m.parameters()]
    first_sums = sums.clone()

    def check(got, want, bound, what):
        got = got.detach().double().cpu().numpy()
        err = np.abs(got - want)
        lim = (N + 2) * U * bound
        assert (err <= lim).all(), (what, float((err - lim).max()), float(err.max()))

    for m, want, wabs, kind in ((actor, ref["actor_grads"], absr["actor_grads"], "actor"),
                                (critic, ref["critic_grads"], absr["critic_grads"], "critic")):
        for l, (w, b) in enumerate(_layers(m)):
            check(w.grad, want[l][0], wabs[l][0], f"{kind} W{l}")
            check(b.grad, want[l][1], wabs[l][1], f"{kind} b{l}")
    for (_, v), key in zip(outs, ("values", "j_values", "returns")):
        check(v, ref[key], absr[key], key)
    diff = np.abs(ref["values"] - ref["returns"])
    dabs = absr["values"] + absr["returns"]
    err_bound = float((2 * diff * dabs + dabs ** 2 * (N + 2) * U).sum())
    assert abs(float(sums[0]) - ref["sum_sq_err"]) <= (N + 2) * U * err_bound
    assert abs(float(sums[1]) - ref["sum_j"]) <= (N + 2) * U * float(absr["j_values"].sum())
    # guard regions untouched
    for buf in guards:
        assert bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[-GUARD:] == SENTINEL).all())
    # bit-identical on a second launch
    fused.launch(obs, actions, rewards, done, cursor, tuple(v for _, v in outs))
    torch.cuda.synchronize()
    again = [p.grad for m in (actor, critic) for p in m.parameters()]
    assert all(torch.equal(a, b) for a, b in zip(first, again))
    assert torch.equal(first_sums, sums)


def test_unsupported_struct_is_refused_without_a_launch():
    import ctypes

    from warp_drive_b200 import lib as wlib

    lib = wlib.load()
    u = wlib.DdpgUpdate()
    u.n_envs, u.n_agents, u.obs_dim, u.action_dim = 4, 1, 3, 1
    u.capacity, u.cursor, u.n_step = 9, 0, 5
    for net in (u.actor, u.critic, u.target_actor, u.target_critic):
        net.n_hidden = 2
        net.widths[0], net.widths[1] = 65, 64              # width 65
    before = wlib.launch_count()
    assert lib.wdb_ddpg_update(wlib.stream_ptr(), ctypes.byref(u)) == 1   # cudaErrorInvalidValue
    for net in (u.actor, u.critic, u.target_actor, u.target_critic):
        net.widths[0] = 64                                  # supported shapes, NULL pointers
    assert lib.wdb_ddpg_update_supported(ctypes.byref(u)) == 1
    assert lib.wdb_ddpg_update(wlib.stream_ptr(), ctypes.byref(u)) == 1
    assert wlib.launch_count() == before
