"""The wgmma policy forward reproduces tests/golden/mlp_forward_bits.npz byte for byte.

test_gpu_mlp_exact.py pins the forward to a float64 reference within 1e-5 on inputs built to
be exact; this file pins the bits on realistic inputs (nn.Linear-initialised weights,
observation-like rows) so that rescheduling the kernel -- the order its MMAs issue in, how
its epilogues overlap, how it stages observations -- cannot move the probabilities or values
by even one ulp.  The fixture and how it was made: tests/golden/make_mlp_forward_golden.py.
"""
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location(
    "make_mlp_forward_golden", os.path.join(HERE, "golden", "make_mlp_forward_golden.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)


@pytest.mark.parametrize("entry", G.ENTRIES)
@pytest.mark.parametrize("name", sorted(G.CASES))
def test_forward_bits_match_golden(wdb_lib, name, entry):
    golden = np.load(G.GOLDEN)
    got = G.run(name, entry)
    keys = sorted(k[len(name) + 1:] for k in golden.files if k.startswith(name + "_"))
    assert keys == sorted(got), (keys, sorted(got))
    for k in keys:
        want = golden[f"{name}_{k}"]
        assert got[k].shape == want.shape, (name, entry, k)
        diff = np.flatnonzero(got[k].view(np.uint32) != want.view(np.uint32))
        assert diff.size == 0, (
            f"{name}/{entry}/{k}: {diff.size} of {want.size} elements differ, first at flat "
            f"index {diff[0]}: {got[k].flat[diff[0]]!r} vs {want.flat[diff[0]]!r}")
