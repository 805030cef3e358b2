"""Action-masked DQN without a GPU: the masked bootstraps of the four torch objectives against
the float64 reference (tests/masked_q_reference.py), the Q models' masked Dict spaces, the
native pass selection, the bindings against the header, the new translation unit's kernels and
resources, and the machine code of the DQN and C51 kernels whose tile bodies it shares."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import masked_q_reference as mref
from c51_reference import make_c51_models
from dqn_update_reference import forward, make_q_models
from iqn_reference import make_iqn_models
from qr_dqn_reference import make_qr_models
from test_ddpg_update_reference_cpu import layers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "warp_drive_b200", "csrc")


def _masks(scores, seed):
    """Masks [B, A] over rows whose unmasked choice is argmax(scores): random rows, rows that
    exclude that choice, single-valid rows and all-invalid rows (the unmasked rule)."""
    g = np.random.default_rng(seed)
    B, A = scores.shape
    m = (g.random((B, A)) < 0.6).astype(np.float32)
    best = np.argmax(scores, axis=1)
    q = B // 4
    m[:q] = 1.0
    m[np.arange(q), best[:q]] = 0.0                           # the unmasked argmax excluded
    m[q:2 * q] = 0.0
    m[np.arange(q, 2 * q), g.integers(0, A, q)] = 1.0          # one valid action
    m[2 * q:2 * q + 3] = 0.0                                    # none valid
    return m


def _windows(B, F, seed):
    g = np.random.default_rng(seed)
    return g.standard_normal((B, F))


# ------------------------------------------------------------------------ torch bootstraps
@pytest.mark.parametrize("double_q", [True, False])
@pytest.mark.parametrize("kind", ["dqn", "qr", "iqn", "c51"])
def test_masked_bootstraps_equal_the_reference(kind, double_q):
    from warp_drive_b200.training.algorithms.dqn import (
        DQN, CategoricalDQN, ImplicitQuantileDQN, QuantileDQN)

    F, A, B = 5, 4, 64
    x = _windows(B, F, 1)
    xt = torch.from_numpy(x)
    if kind == "dqn":
        models = make_q_models(F, A, [16], seed=2)
        algo = DQN(0.9, n_step=2, double_q=double_q)
        Lq, Lt = layers(models[0]), layers(models[1])
        scores = forward(Lq if double_q else Lt, x)[0]

        def torch_boot(mask):
            return algo.bootstrap(*models, xt, mask)

        def ref_boot(mask):
            return mref.dqn_boot(Lq, Lt, x, mask, double_q)
    elif kind == "qr":
        N = 3
        models = make_qr_models(F, A, N, [16], seed=2)
        algo = QuantileDQN(0.9, n_step=2, double_q=double_q)
        Lq, Lt = layers(models[0]), layers(models[1])
        scores = forward(Lq if double_q else Lt, x)[0].reshape(B, A, N).mean(axis=2)

        def torch_boot(mask):
            return algo.bootstrap_quantiles(*models, xt, mask)

        def ref_boot(mask):
            return mref.qr_boot(Lq, Lt, x, mask, double_q, N)
    elif kind == "iqn":
        models = make_iqn_models(F, A, [16], seed=2)
        algo = ImplicitQuantileDQN(0.9, n_step=2, double_q=double_q)
        taus = torch.from_numpy(np.random.default_rng(3).random((B, models[0].num_tau_prime_samples)))
        with torch.no_grad():
            scores = (models[0] if double_q else models[1]).q_values(xt).numpy()

        def torch_boot(mask):
            return algo.bootstrap_quantiles(*models, xt, taus, mask)

        def ref_boot(mask):
            return mref.iqn_boot(models, x, taus.numpy(), mask, double_q)
    else:
        models = make_c51_models(F, A, [16], N=11, seed=2)
        algo = CategoricalDQN(0.9, n_step=2, double_q=double_q)
        Lq, Lt = layers(models[0]), layers(models[1])
        z = models[0].support.double().numpy()
        with torch.no_grad():
            scores = (models[0] if double_q else models[1]).q_values(xt).numpy()

        def torch_boot(mask):
            return algo.bootstrap_distribution(*models, xt, mask)

        def ref_boot(mask):
            return mref.c51_boot(Lq, Lt, x, mask, double_q, z)

    mask = _masks(scores, 4)
    got = torch_boot(torch.from_numpy(mask)).numpy()
    np.testing.assert_allclose(got, ref_boot(mask), rtol=1e-12, atol=1e-12)
    # the masks changed the bootstrap of the rows that excluded the unmasked choice
    unmasked = torch_boot(None).numpy()
    assert not np.allclose(got[:B // 4], unmasked[:B // 4])
    # all-invalid rows take the unmasked rule; an all-ones mask and None are the unmasked ops
    np.testing.assert_array_equal(got[B // 2:B // 2 + 3], unmasked[B // 2:B // 2 + 3])
    assert torch.equal(torch_boot(torch.ones(B, A, dtype=torch.float64)), torch_boot(None))


def test_masked_dqn_loss_takes_the_masked_bootstrap():
    from warp_drive_b200.training.algorithms.dqn import DQN

    F, A, B, ns = 5, 4, 32, 3
    models = make_q_models(F, A, [16], seed=5)
    g = np.random.default_rng(6)
    obs, boot_obs = torch.from_numpy(g.standard_normal((B, F))), torch.from_numpy(
        g.standard_normal((B, F)))
    actions = torch.from_numpy(g.integers(0, A, (B, 1)))
    rewards = torch.from_numpy(g.standard_normal((ns, B)))
    done = torch.from_numpy((g.random((ns, B)) < 0.2).astype(np.float64))
    mask = torch.from_numpy((g.random((B, A)) < 0.5).astype(np.float32))
    algo = DQN(0.9, n_step=ns)
    _, q, returns = algo.loss(*models, obs, actions, rewards, done, boot_obs, boot_mask=mask)
    boot = mref.dqn_boot(layers(models[0]), layers(models[1]), boot_obs.numpy(), mask.numpy(),
                         True)
    np.testing.assert_allclose(returns.numpy(), algo.sampled_returns(
        rewards, done, torch.from_numpy(boot)).numpy(), rtol=1e-12, atol=1e-12)
    base = algo.loss(*models, obs, actions, rewards, done, boot_obs)
    masked_none = algo.loss(*models, obs, actions, rewards, done, boot_obs, boot_mask=None)
    for a, b in zip(base, masked_none):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------ models
def _masked_env(F=3, A=4, mask_width=None):
    from test_ddpg_update_reference_cpu import _Env
    from warp_drive_b200.utils import spaces as sp

    env = _Env(F, 1)
    env.env.action_space = {0: sp.Discrete(A)}
    env.env.observation_space = {0: sp.Dict({
        "state": sp.Box(-1.0, 1.0, shape=(F,), dtype=np.float32),
        "action_mask": sp.Box(0, 1, shape=(A if mask_width is None else mask_width,),
                              dtype=np.int32)})}
    return env


_KINDS = {
    "fully_connected_q": {},
    "fully_connected_categorical_q": {"num_atoms": 11, "v_min": -1.0, "v_max": 1.0},
    "fully_connected_quantile_q": {"num_quantiles": 4},
    "fully_connected_iqn": {},
}


def make_masked(kind, F=3, A=4, dims=(16,), mask_width=None, seed=0, **extra):
    from warp_drive_b200.training.models.fully_connected import ModelFactory

    torch.manual_seed(seed)
    cfg = {"type": kind, "fc_dims": list(dims), "masked": True, **_KINDS[kind], **extra}
    return ModelFactory.create(kind)(env=_masked_env(F, A, mask_width), model_config=cfg,
                                     policy="shared", policy_tag_to_agent_id_map={"shared": [0]})


@pytest.mark.parametrize("kind", sorted(_KINDS))
def test_masked_is_opt_in_and_checked(kind):
    """An action_mask is refused as before unless model.masked is true; masked: true needs an
    action_mask of one entry per action, and is a bool."""
    from test_dqn_cpu import _mk_env
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils import spaces as sp

    cls = ModelFactory.create(kind)

    def mk(env, **extra):
        cfg = {"type": kind, "fc_dims": [8], **_KINDS[kind], **extra}
        return cls(env=env, model_config=cfg, policy="shared",
                   policy_tag_to_agent_id_map={"shared": [0]})

    with pytest.raises(ValueError, match="does not take observations with an action_mask"):
        mk(_masked_env(4, 3))
    assert mk(_masked_env(4, 3), masked=True).masked is True
    assert mk(_mk_env(sp.Discrete(3))).masked is False
    with pytest.raises(ValueError, match="needs a Dict observation space"):
        mk(_mk_env(sp.Discrete(3)), masked=True)
    with pytest.raises(ValueError, match="one entry per action"):
        mk(_masked_env(4, 3, mask_width=2), masked=True)
    for v in (1, "true", None):
        with pytest.raises(ValueError, match="model.masked is true or false"):
            mk(_masked_env(4, 3), masked=v)


@pytest.mark.parametrize("kind", sorted(_KINDS))
def test_q_models_take_a_masked_dict_space(kind):
    q = make_masked(kind)
    assert q.masked is True and q.flattened_obs_size == 3 and q.output_dims == [4]
    # the Q values stay raw: forward ignores a mask
    x = torch.randn(2, 3)
    with torch.no_grad():
        assert torch.equal(q(x)[0][0], q(x, action_mask=torch.zeros(2, 4))[0][0])
    with pytest.raises(ValueError, match="one entry per action"):
        make_masked(kind, mask_width=5)


# ------------------------------------------------------------------------ pass selection
def _lib_or_skip():
    from warp_drive_b200 import lib as wlib

    if not os.path.exists(wlib.LIB_PATH):
        pytest.skip("libwdb200.so is not built")
    return wlib


def test_pass_selection():
    _lib_or_skip()
    from warp_drive_b200.training.algorithms import fused_dqn as fd
    from warp_drive_b200.training.algorithms.dqn import (
        DQN, CategoricalDQN, ImplicitQuantileDQN, QuantileDQN)

    dqn, c51 = DQN(0.99, n_step=3), CategoricalDQN(0.99, n_step=3)
    qr, iqn = QuantileDQN(0.99, n_step=3), ImplicitQuantileDQN(0.99, n_step=3)
    classes = (fd.FusedDQNUpdate, fd.FusedQRDQNUpdate, fd.FusedIQNUpdate, fd.FusedC51Update,
               fd.FusedMaskedDQNUpdate, fd.FusedMaskedC51Update, fd.FusedDuelingUpdate,
               fd.FusedNoisyUpdate)

    def takers(algo, q):
        return {c.__name__ for c in classes if c.supported(algo, q, 8, 6, 100, 256)}

    # masked plain networks: the masked passes only
    assert takers(dqn, make_masked("fully_connected_q")) == {"FusedMaskedDQNUpdate"}
    assert takers(c51, make_masked("fully_connected_categorical_q")) == {"FusedMaskedC51Update"}
    # masked QR-DQN and IQN: none (the torch losses)
    assert takers(qr, make_masked("fully_connected_quantile_q")) == set()
    assert takers(iqn, make_masked("fully_connected_iqn")) == set()
    # masked dueling and noisy heads: their wrappers, over the masked plain passes
    for kind, algo in (("fully_connected_q", dqn), ("fully_connected_categorical_q", c51)):
        for extra, wrapper in (({"dueling": True, "stream_fc_dims": [8]}, "FusedDuelingUpdate"),
                               ({"noisy": True}, "FusedNoisyUpdate"),
                               ({"noisy": True, "dueling": True}, "FusedNoisyUpdate")):
            q = make_masked(kind, **extra)
            assert takers(algo, q) == {wrapper}, (kind, extra)
            assert getattr(fd, wrapper).plain_type(q).masked is True
    # masked: F <= 63 as before
    assert takers(dqn, make_masked("fully_connected_q", F=63)) == {"FusedMaskedDQNUpdate"}
    assert takers(dqn, make_masked("fully_connected_q", F=64)) == set()
    # unmasked Box networks: exactly the classes of before
    plain = make_q_models(4, 3, [16])[0].float()
    assert takers(dqn, plain) == {"FusedDQNUpdate"}
    cat = make_c51_models(4, 3, [16], N=11)[0].float()
    assert takers(c51, cat) == {"FusedC51Update"}
    assert takers(qr, make_qr_models(4, 3, 4, [16])[0].float()) == {"FusedQRDQNUpdate"}
    assert takers(iqn, make_iqn_models(4, 3, [16])[0].float()) == {"FusedIQNUpdate"}
    assert fd.FusedDuelingUpdate.plain_type(plain) is fd.FusedDQNUpdate
    assert fd.FusedNoisyUpdate.plain_type(cat) is fd.FusedC51Update


def test_unmasked_dict_networks_keep_the_torch_path():
    _lib_or_skip()
    from test_ddpg_update_reference_cpu import _Env
    from warp_drive_b200.training.algorithms import fused_dqn as fd
    from warp_drive_b200.training.algorithms.dqn import DQN
    from warp_drive_b200.training.models.fully_connected import ModelFactory
    from warp_drive_b200.utils import spaces as sp

    env = _Env(3, 1)
    env.env.action_space = {0: sp.Discrete(4)}
    env.env.observation_space = {0: sp.Dict({
        "state": sp.Box(-1.0, 1.0, shape=(3,), dtype=np.float32)})}
    q = ModelFactory.create("fully_connected_q")(
        env=env, model_config={"type": "fully_connected_q", "fc_dims": [8]}, policy="shared",
        policy_tag_to_agent_id_map={"shared": [0]})
    assert q.masked is False
    for cls in (fd.FusedDQNUpdate, fd.FusedMaskedDQNUpdate):
        assert cls.supported(DQN(0.99, n_step=3), q, 8, 6, 100, 256) is False


def test_one_launch_rollout_refuses_a_masked_q_network():
    from warp_drive_b200.training.fused_single_agent import FusedSingleAgentRollout

    class _W:
        n_agents = 1

        class env:
            name = "ClassicControlCartPoleEnv"

    q = make_masked("fully_connected_q", F=4, A=2)
    assert not FusedSingleAgentRollout.eligible(_W, {"shared": q}, {"shared": [0]})


# ------------------------------------------------------------------------ bindings
def test_bindings_match_the_header():
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    squash = re.sub(r"\s+", " ", header)
    want = [
        "int wdb_sample_epsilon_greedy_masked(void *stream, void *rng_state, const float "
        "*q_values, const float *action_mask, int *actions, long long n_rows, int n_actions, "
        "float epsilon, const unsigned int *words);",
        "int wdb_dqn_update_masked_supported(const wdb_dqn_update_args *update, int n_windows);",
        "long long wdb_dqn_update_masked_workspace_bytes(const wdb_dqn_update_args *update, "
        "int n_windows);",
        "int wdb_dqn_update_masked(void *stream, const wdb_dqn_update_args *update, const "
        "wdb_replay_windows *windows, const float *weights, const float *action_mask);",
        "int wdb_c51_update_masked_supported(const wdb_dqn_update_args *update, int n_atoms, "
        "int n_windows);",
        "long long wdb_c51_update_masked_workspace_bytes(const wdb_dqn_update_args *update, "
        "int n_atoms, int n_windows);",
        "int wdb_c51_update_masked(void *stream, const wdb_dqn_update_args *update, int n_atoms, "
        "const float *support, float delta_z, const wdb_replay_windows *windows, const float "
        "*weights, const float *action_mask);",
    ]
    for proto in want:
        assert proto in squash, proto
    sig = wlib._SIGNATURES
    i, ll, f, vp = ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_void_p
    u, w = ctypes.POINTER(wlib.DqnUpdate), ctypes.POINTER(wlib.ReplayWindows)
    assert sig["wdb_sample_epsilon_greedy_masked"] == (i, [vp, vp, vp, vp, vp, ll, i, f, vp])
    assert sig["wdb_dqn_update_masked_supported"] == (i, [u, i])
    assert sig["wdb_dqn_update_masked_workspace_bytes"] == (ll, [u, i])
    assert sig["wdb_dqn_update_masked"] == (i, [vp, u, w, vp, vp])
    assert sig["wdb_c51_update_masked_supported"] == (i, [u, i, i])
    assert sig["wdb_c51_update_masked_workspace_bytes"] == (ll, [u, i, i])
    assert sig["wdb_c51_update_masked"] == (i, [vp, u, i, vp, f, w, vp, vp])


def test_masked_entries_share_the_unmasked_envelope_and_refuse_a_missing_mask():
    wlib = _lib_or_skip()
    from warp_drive_b200.training.algorithms.fused_dqn import _shape_struct
    from warp_drive_b200.training.algorithms.dqn import DQN

    L = wlib.load()
    q = make_q_models(4, 3, [16])[0].float()
    for B in (1, 256, 50000):
        u = _shape_struct(DQN(0.99, n_step=3), q, 8, 6, 100)
        assert L.wdb_dqn_update_masked_supported(u, B) == L.wdb_dqn_update_sampled_supported(u, B)
        assert (L.wdb_dqn_update_masked_workspace_bytes(u, B)
                == L.wdb_dqn_update_sampled_workspace_bytes(u, B))
        for N in (2, 51, 65):
            assert (L.wdb_c51_update_masked_supported(u, N, B)
                    == L.wdb_c51_update_sampled_supported(u, N, B))
            assert (L.wdb_c51_update_masked_workspace_bytes(u, N, B)
                    == L.wdb_c51_update_sampled_workspace_bytes(u, N, B))
    # no launch without a mask (or with a bad epsilon)
    w = wlib.ReplayWindows()
    w.n_windows = 8
    assert L.wdb_dqn_update_masked(None, u, ctypes.byref(w), None, None) == 1
    assert L.wdb_c51_update_masked(None, u, 51, None, 0.1, ctypes.byref(w), None, None) == 1
    assert L.wdb_sample_epsilon_greedy_masked(None, None, None, None, None, 4, 3, 0.5, None) == 1


# ------------------------------------------------------------------------ ptxas / SASS
_MASKED_KERNELS = {
    "28epsilon_greedy_masked_kernelEPvPKfS2_PixifPKj",
    "17dqn_masked_kernelEPKf19wdb_dqn_update_argsNS_4PlanEPfPdPK4int2",
    "26dqn_masked_weighted_kernelEPKf19wdb_dqn_update_argsNS_4PlanEPfPdPK4int2S1_",
    "17c51_masked_kernelEPKf19wdb_dqn_update_argsNS_4PlanEiS1_fPfPdPK4int2",
    "29c51_masked_prioritized_kernelEPKf19wdb_dqn_update_argsNS_4PlanEiS1_fPfPdPK4int2S1_",
    "18ddpg_reduce_kernelENS_6ReduceEPKfPKdPd",           # the passes' second launch
}


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_masked_kernels_compile_without_spills_and_the_shared_bodies_keep_their_code(tmp_path):
    from test_dueling_cpu import _C51_SASS_SHA256
    from test_iqn_cpu import _QR_SASS_SHA256
    from test_qr_dqn_cpu import _KEPT_SASS_SHA256, _cubin, _sass_hashes

    stats, _ = _cubin(os.path.join(CSRC, "wdb_masked_q.cu"), tmp_path)
    assert set(stats) == _MASKED_KERNELS
    for k, v in stats.items():
        assert v["spill"] == (0, 0), (k, v)
    version = subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout
    if "release 12.9" not in version:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    want = {"wdb_ddpg_update.cu": dict(_KEPT_SASS_SHA256["wdb_ddpg_update.cu"],
                                       **_QR_SASS_SHA256),
            "wdb_c51_update.cu": _C51_SASS_SHA256["wdb_c51_update.cu"]}
    for src, kept in want.items():
        _, cubin = _cubin(os.path.join(CSRC, src), tmp_path)
        got = _sass_hashes(cubin)
        assert got == kept, src                # no kernel lost, added or changed
