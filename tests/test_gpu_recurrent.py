"""Recurrent A2C / PPO on the GPU: wdb_gru_policy_forward within its a-priori float64 bound
(tests/recurrent_reference.py) across its envelope, wdb_recurrent_reset_done against its torch
expression, the rollout's hidden state against forward_sequence replayed over the recorded batch,
graph against eager rollouts, the native against the torch-step rollout path, one A2C and one PPO
update through either path, and the launch count of a feed-forward rollout."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "custom_env"))

import recurrent_reference as ref  # noqa: E402
from test_recurrent_cpu import _model  # noqa: E402

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------ the step kernel
@pytest.mark.parametrize("fc_dims,H,heads,F,R", [
    ((64, 64), 64, (21, 21), 71, 2000 * 7 + 5),      # TagContinuous run config's shape
    ((32, 32), 32, (5,), 26, 1),                      # gridworld's shape, a single row
    ((48,), 40, (3, 7), 13, 37),                      # one trunk layer; 37 rows: 2 tiles + 5
    ((), 24, (2,), 9, 16),                            # no trunk
    ((96,), 64, (64,), 33, 1000),
])
def test_step_kernel_within_its_float64_bound(fc_dims, H, heads, F, R):
    from warp_drive_b200.training.models.fully_connected_gru import NativeGruStep

    m = _model(fc_dims=fc_dims, gru_dim=H, heads=heads, F=F, seed=R % 97).cuda()
    with torch.no_grad():                         # spread the weights to exercise the gates
        for p in m.parameters():
            p.mul_(2.0)
    assert NativeGruStep.supported(m)
    g = torch.Generator(device="cuda").manual_seed(R)
    obs = torch.randn(R, F, device="cuda", generator=g)
    h0 = torch.randn(R, H, device="cuda", generator=g)
    guard = 64
    hbuf = torch.full((R * H + 2 * guard,), float("nan"), device="cuda")
    hbuf[guard:guard + R * H] = h0.reshape(-1)
    pbufs = [torch.full((R * a + 2 * guard,), float("nan"), device="cuda") for a in heads]
    step = NativeGruStep(m)
    step(obs, hbuf[guard:guard + R * H], [b[guard:guard + R * a] for b, a in zip(pbufs, heads)])
    torch.cuda.synchronize()
    P = ref.params_of(m)
    probs, hn, eprobs, ehn = ref.step_with_bounds(P, obs.double().cpu().numpy(),
                                                  h0.double().cpu().numpy())
    got_h = hbuf[guard:guard + R * H].view(R, H).double().cpu().numpy()
    assert np.abs(got_h - hn).max() >= 0 and (np.abs(got_h - hn) <= ehn).all(), (
        np.abs(got_h - hn) / ehn).max()
    for b, a, p, e in zip(pbufs, heads, probs, eprobs):
        got = b[guard:guard + R * a].view(R, a).double().cpu().numpy()
        assert (np.abs(got - p) <= e).all(), (np.abs(got - p) / e).max()
        assert torch.isnan(b[:guard]).all() and torch.isnan(b[guard + R * a:]).all()
    assert torch.isnan(hbuf[:guard]).all() and torch.isnan(hbuf[guard + R * H:]).all()
    # relaunch from the same state: the same bits
    first = [b.clone() for b in pbufs], hbuf.clone()
    hbuf[guard:guard + R * H] = h0.reshape(-1)
    step(obs, hbuf[guard:guard + R * H], [b[guard:guard + R * a] for b, a in zip(pbufs, heads)])
    assert torch.equal(hbuf.nan_to_num(7.0), first[1].nan_to_num(7.0))
    for b, c in zip(pbufs, first[0]):
        assert torch.equal(b.nan_to_num(7.0), c.nan_to_num(7.0))


def test_reset_done_kernel_equals_its_torch_expression():
    from warp_drive_b200 import lib as wlib

    E = 1001
    g = torch.Generator(device="cuda").manual_seed(3)
    hs = [torch.randn(E, n, h, device="cuda", generator=g) for n, h in ((3, 64), (1, 5), (7, 9))]
    done = torch.randint(0, 3, (E,), device="cuda", dtype=torch.int32, generator=g)
    done[::5] = -1                                  # only done > 0 resets
    want = [h * (done <= 0).float()[:, None, None] for h in hs]
    k = wlib.RecurrentReset()
    k.done, k.n_envs, k.n_policies = wlib.ptr(done), E, len(hs)
    for i, h in enumerate(hs):
        k.policy[i].hidden, k.policy[i].n_agents, k.policy[i].hidden_size = (
            wlib.ptr(h), h.shape[1], h.shape[2])
    wlib.check(wlib.load().wdb_recurrent_reset_done(wlib.stream_ptr(), ctypes.byref(k)))
    for h, w in zip(hs, want):
        assert torch.equal(h, w)


# ------------------------------------------------------------------------ rollouts
GRU = {"type": "fully_connected_gru", "fc_dims": [32, 32], "gru_dim": 32}


def _trainer(tmp_path, name, model=GRU, **kw):
    from recall_env import make_trainer

    kw.setdefault("num_envs", 64)
    kw.setdefault("steps_per_env", 10)            # episodes of 4 steps end inside the batch
    return make_trainer(model, name, str(tmp_path), **kw)


def _rollout(tr):
    tr._reset_all_envs()
    tr.engine.resync_observations()
    tr.engine.rollout()
    torch.cuda.synchronize()


def test_hidden_state_equals_forward_sequence_over_the_recorded_batch(tmp_path):
    tr = _trainer(tmp_path, "seq")
    eng = tr.engine
    assert eng.recurrent and "shared" in eng.native_gru and eng.fused is None and eng.sa is None
    dm = tr.cuda_envs.cuda_data_manager
    for _ in range(3):                              # the state carries over between rollouts
        eng.rollout()
    torch.cuda.synchronize()
    obs = dm.data_on_device_via_torch("processed_observations_batch_shared")
    done = dm.data_on_device_via_torch("done_flags_batch")
    assert (done > 0).any()
    assert (eng.hidden_start["shared"] != 0).any()
    m = tr.models["shared"]
    with torch.no_grad():
        h = eng.hidden_start["shared"].reshape(-1, m.hidden_size)
        x = m.trunk(obs)
        E, Np = done.shape[1], obs.shape[2]
        for t in range(obs.shape[0]):
            if t > 0:
                h = m.reset_hidden(h.view(E, Np, -1), done[t - 1]).view(E * Np, -1)
            h = m.gru(x[t].reshape(E * Np, -1), h)
        h = m.reset_hidden(h.view(E, Np, -1), done[-1])
    torch.testing.assert_close(eng.hidden["shared"], h, rtol=0, atol=1e-5)


def test_graph_and_eager_rollouts_agree_bit_for_bit(tmp_path):
    outs = []
    for graph in (True, False):
        tr = _trainer(tmp_path, f"g{graph}", use_cuda_graph=graph)
        tr._reset_all_envs()
        tr.engine.resync_observations()
        if not graph:                 # the graph's capture is preceded by one evaluation step
            tr.engine.step(-1)
        tr.engine.rollout()
        _rollout(tr)
        dm = tr.cuda_envs.cuda_data_manager
        outs.append([dm.data_on_device_via_torch(n).clone() for n in (
            "processed_observations_batch_shared", "sampled_actions_batch_shared",
            "rewards_batch_shared", "done_flags_batch")] + [
            tr.engine.hidden["shared"].clone(), tr.engine.hidden_start["shared"].clone()])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_native_and_torch_step_rollouts_agree(tmp_path):
    """Teacher-forced over 12 steps (three episodes): from the same observations and state, the
    native and torch-step forwards agree on the probabilities and h' to 1e-5."""
    tr = _trainer(tmp_path, "nat", use_cuda_graph=False)
    eng = tr.engine
    tr._reset_all_envs()
    eng.resync_observations()
    native = eng.native_gru["shared"]
    observations = tr.cuda_envs.cuda_data_manager.data_on_device_via_torch("observations")
    for t in range(12):
        obs = observations.reshape(-1, 2).clone()
        h_t = eng.hidden["shared"].clone()
        p_nat = [q.clone() for q in eng._recurrent_forward("shared", obs)]
        h_nat = eng.hidden["shared"].clone()
        eng.hidden["shared"].copy_(h_t)
        del eng.native_gru["shared"]
        p_torch = eng._recurrent_forward("shared", obs)
        for a, b in zip(p_nat, p_torch):
            torch.testing.assert_close(a, b, rtol=0, atol=1e-5)
        torch.testing.assert_close(h_nat, eng.hidden["shared"], rtol=0, atol=1e-5)
        eng.hidden["shared"].copy_(h_t)
        eng.native_gru["shared"] = native
        eng.step(-1)                              # the native path advances the env
    torch.cuda.synchronize()


@pytest.mark.parametrize("algorithm", ["A2C", "PPO"])
def test_one_update_agrees_between_the_native_and_torch_rollout_paths(tmp_path, algorithm):
    params = []
    for native in (True, False):
        tr = _trainer(tmp_path, f"u{algorithm}{native}", algorithm=algorithm, seed=11,
                      ppo_steps=(2, 4))
        if not native:
            tr.engine.native_gru.clear()
        tr._reset_all_envs()
        tr.engine.resync_observations()
        tr._generate_rollout_batch()
        tr._update_model_params(0)
        torch.cuda.synchronize()
        params.append([p.detach().clone() for p in tr.models["shared"].parameters()])
    for a, b in zip(*params):
        torch.testing.assert_close(a, b, rtol=0, atol=1e-5)


def test_feed_forward_rollouts_keep_their_launches_and_path(tmp_path):
    from warp_drive_b200 import lib as wlib

    counts = {}
    for name, model, native in (("ff", {"type": "fully_connected", "fc_dims": [32, 32]}, True),
                                ("rn", GRU, True), ("rt", GRU, False)):
        tr = _trainer(tmp_path, name, model=model, use_cuda_graph=False)
        if not native:
            tr.engine.native_gru.clear()
        tr.engine.step(0)
        torch.cuda.synchronize()
        n0 = wlib.launch_count()
        tr.engine.step(1)
        torch.cuda.synchronize()
        counts[name] = wlib.launch_count() - n0
        if name == "ff":
            assert not tr.engine.recurrent and tr.engine.hidden == {}
            ff_forward = len(tr.engine.fused_forward)       # the wgmma forward, one launch
    assert counts["rn"] == counts["rt"] + 1          # the native forward
    # the feed-forward step: no reset launch, its forward on its own path
    assert counts["ff"] == counts["rt"] - 1 + ff_forward
