"""Host side of the sampling policy forward: the ctypes mirror of wdb_mlp_sampling has the
header's layout, and the library says which policy shapes sample (only the config-2 shape
whose forward is compiled with constant bounds) without a GPU."""
import ctypes
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_mlp_sampling_struct_matches_the_header(tmp_path):
    from warp_drive_b200 import lib as wlib

    names = [n for n, _ in wlib.MlpSampling._fields_]
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "wdb200.h"',
             "int main(void) {", '  printf("size %zu\\n", sizeof(wdb_mlp_sampling));']
    lines += [f'  printf("{n} %zu\\n", offsetof(wdb_mlp_sampling, {n}));' for n in names]
    lines += ["  return 0;", "}"]
    src = tmp_path / "sampling.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "sampling"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)],
                   check=True)
    out = dict(line.split() for line in subprocess.run(
        [str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["size"]) == ctypes.sizeof(wlib.MlpSampling)
    for n in names:
        assert int(out[n]) == getattr(wlib.MlpSampling, n).offset, n


def test_only_the_config2_shape_samples(wdb_lib):
    assert wdb_lib.wdb_mlp_forward_samples(71, 256, 21, 21) == 1
    assert wdb_lib.wdb_mlp_forward_samples(80, 256, 16, 16) == 1
    assert wdb_lib.wdb_mlp_forward_samples(71, 128, 21, 21) == 0    # another width
    assert wdb_lib.wdb_mlp_forward_samples(36, 256, 21, 21) == 0    # another K1
    assert wdb_lib.wdb_mlp_forward_samples(71, 256, 21, 0) == 0     # one head
    assert wdb_lib.wdb_mlp_forward_samples(71, 256, 8, 8) == 0      # N3 = 32
