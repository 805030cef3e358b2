"""Multi-epoch PPO without a GPU: the new argument structs match include/wdb200.h field by
field, the prototypes match the ctypes signatures, and the config keys select and refuse what
they should."""
import ctypes
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from test_abi_layout_cpu import _c_fields  # noqa: E402

PAIRS = {"wdb_gae_args": "GaeArgs", "wdb_ppo_loss": "PpoLoss",
         "wdb_ppo_gaussian_loss": "PpoGaussianLoss"}
PROTOS = {"wdb_gae": 2, "wdb_ppo_loss_and_grads": 2, "wdb_ppo_loss_supported": 2,
          "wdb_ppo_gaussian_loss_and_grads": 2, "wdb_ppo_gaussian_loss_supported": 1}


def test_new_structs_match_the_header(tmp_path):
    from warp_drive_b200 import lib as wlib

    header = open(os.path.join(ROOT, "include", "wdb200.h"), encoding="utf8").read()
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "wdb200.h"', "int main(void) {"]
    fields = {}
    for c_name in PAIRS:
        fields[c_name] = _c_fields(header, c_name)
        lines.append(f'  printf("{c_name} size %zu\\n", sizeof({c_name}));')
        for f in fields[c_name]:
            lines.append(f'  printf("{c_name} {f} %zu\\n", offsetof({c_name}, {f}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)],
                   check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    got = {}
    for line in out.splitlines():
        s, f, v = line.split()
        got[(s, f)] = int(v)
    for c_name, py_name in PAIRS.items():
        cls = getattr(wlib, py_name)
        assert ctypes.sizeof(cls) == got[(c_name, "size")], c_name
        assert [n for n, _ in cls._fields_] == fields[c_name], c_name
        for f in fields[c_name]:
            assert getattr(cls, f).offset == got[(c_name, f)], (c_name, f)


def test_new_prototypes_are_bound_with_their_arity():
    from warp_drive_b200 import lib as wlib

    for name, n in PROTOS.items():
        assert name in wlib._SIGNATURES and len(wlib._SIGNATURES[name][1]) == n, name
    # every argument type agrees with the header (the generic prototype check covers them all)
    from test_abi_layout_cpu import test_ctypes_signatures_match_the_header_prototypes

    test_ctypes_signatures_match_the_header_prototypes()


def _pg(algo="PPO", **kw):
    from warp_drive_b200.training.algorithms.policygradient import A2C, PPO

    return PPO(clip_param=0.2, **kw) if algo == "PPO" else A2C(**kw)


def test_defaults_select_the_single_step_update():
    from warp_drive_b200.training.trainer import load_run_config

    for algo in ("A2C", "PPO"):
        assert not _pg(algo).minibatch_path
        assert not _pg(algo, num_epochs=1, num_mini_batches=1, gae_lambda=None).minibatch_path
    cfg = load_run_config("single_pendulum_ppo")["policy"]["shared"]
    assert "num_epochs" not in cfg and "gae_lambda" not in cfg
    assert _pg(num_epochs=2).minibatch_path and _pg(num_mini_batches=3).minibatch_path
    assert _pg(gae_lambda=1.0).minibatch_path and _pg("A2C", gae_lambda=0.9).minibatch_path


def test_the_gae_run_config_takes_the_minibatch_update():
    from warp_drive_b200.training.trainer import load_run_config

    c = load_run_config("single_pendulum_ppo_gae")["policy"]["shared"]
    base = load_run_config("single_pendulum_ppo")["policy"]["shared"]
    assert c["gae_lambda"] == 0.95 and c["normalize_advantage"] is True
    assert c["num_epochs"] > 1 and c["num_mini_batches"] > 1
    assert c["model"] == base["model"] and c["lr"] == 0.001
    for k in ("num_envs", "train_batch_size", "num_episodes"):
        assert load_run_config("single_pendulum_ppo_gae")["trainer"][k] == \
            load_run_config("single_pendulum_ppo")["trainer"][k]


@pytest.mark.parametrize("algo,kw", [
    ("A2C", dict(num_epochs=2)), ("A2C", dict(num_mini_batches=4)),
    ("PPO", dict(num_epochs=2, normalize_return=True)),
    ("PPO", dict(gae_lambda=0.9, normalize_return=True)),
    ("PPO", dict(num_epochs=0)), ("PPO", dict(num_mini_batches=0)),
    ("PPO", dict(gae_lambda=1.5)), ("PPO", dict(gae_lambda=-0.1))])
def test_refused_combinations_raise(algo, kw):
    with pytest.raises(ValueError):
        _pg(algo, **kw)


class _FakeTrainer:
    """Just what Trainer._minibatch_schedule reads."""

    def __init__(self, objectives):
        self.trainers = objectives
        self.policies_to_train = list(objectives)


def test_policies_must_agree_on_the_number_of_steps():
    """The schedule is the number of optimizer steps per iteration; policies may split it
    differently (each keeps its own epochs and minibatches) but must agree on the product."""
    from warp_drive_b200.training.trainer import Trainer

    sched = Trainer._minibatch_schedule
    assert sched(_FakeTrainer({"a": _pg(), "b": _pg()})) is None
    assert sched(_FakeTrainer({"a": _pg(num_epochs=2, num_mini_batches=3),
                               "b": _pg(num_epochs=3, num_mini_batches=2)})) == 6
    assert sched(_FakeTrainer({"a": _pg(gae_lambda=0.9)})) == 1
    with pytest.raises(ValueError):
        sched(_FakeTrainer({"a": _pg(num_epochs=2), "b": _pg(num_epochs=3)}))
    with pytest.raises(ValueError):
        sched(_FakeTrainer({"a": _pg(num_epochs=2), "b": _pg()}))


def test_batches_of_two_to_the_31_rows_are_refused():
    import torch

    from warp_drive_b200.training.algorithms.policygradient import PPO

    class _Huge:
        shape = (2 ** 16, 2 ** 15, 1)

    with pytest.raises(ValueError, match="int32"):
        PPO(clip_param=0.2, num_epochs=2).prepare_batch(None, None, None, _Huge(),
                                                        torch.zeros(1))


def test_more_minibatches_than_rows_are_refused():
    import torch

    from warp_drive_b200.training.algorithms.policygradient import PPO

    class _Small:
        shape = (2, 3, 1)

    with pytest.raises(ValueError, match="empty"):
        PPO(clip_param=0.2, num_mini_batches=7).prepare_batch(None, None, None, _Small(),
                                                              torch.zeros(1))
