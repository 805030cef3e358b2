"""The sampling policy forward's three-warpgroup kernel, checked from its compiled code: the
register split between the MMA warpgroups and the epilogue warpgroup (setmaxnreg) spills
nothing and keeps every wgmma of the MMA schedule unserialised, and every other kernel of
csrc/wdb_mlp.cu (the AnyShape, pair and masked kernels and the unsampled FastShape entries)
keeps the machine code it had before the sampling forward got its epilogue warpgroup."""
import os
import re
import shutil
import subprocess

import pytest

from test_qr_dqn_cpu import NVCC_SM90A, ROOT, _sass_hashes, _strip

SRC = os.path.join(ROOT, "warp_drive_b200", "csrc", "wdb_mlp.cu")

# recorded with nvcc 12.9 at the commit before the epilogue warpgroup
_KEPT_SASS_SHA256 = {
    "15pack_obs_kernelEPKfxiiPh":
        "d98068a30273555ed28f67f3bec9ca1d07e6e8986caa6901307ceb9c59f013b7",
    "16pack_misc_kernelENS_9MlpHeaderEPhPKfS3_S3_S3_S3_":
        "cbac5b223eb4495d6455d4a9e3eb67976ffb661f9e29d325f04af0a5a71e08ce",
    "16pack_rows_kernelEPKfiiiiP13__nv_bfloat16":
        "e084355670b217025c14ee8ecbc4c5f50bedd3936f0b3b2b1ed8c20bc4d7c31d",
    "18mlp_forward_kernelILb0ENS_8MlpShapeILi0ELi0ELi0EEEEEvPKhPKvxPfS7_S7_i":
        "2c9b76015c12c229d19c462c23f31e680e76910d14686218e49f985a9e23b427",
    "18mlp_forward_kernelILb0ENS_8MlpShapeILi80ELi256ELi48EEEEEvPKhPKvxPfS7_S7_i":
        "afb26e76f16d4cad4c5bb289b0d8d81f68df2e922697a909b8bcaa95cb5cf178",
    "18mlp_forward_kernelILb1ENS_8MlpShapeILi0ELi0ELi0EEEEEvPKhPKvxPfS7_S7_i":
        "f6751d94f21886e7dc44294d51966ef2e8c5fa41e30d0ad728abbfb14ea84260",
    "18mlp_forward_kernelILb1ENS_8MlpShapeILi80ELi256ELi48EEEEEvPKhPKvxPfS7_S7_i":
        "7baa2af1e910b8f201e609e1a8f1a916611d8abad834c5594e73cd41f21a63b6",
    "18pack_matrix_kernelEPKfiiiiP13__nv_bfloat16":
        "dfd7d2e760a1ce6d7e8002712210dafb8fa91e6ec2fff5a5ce5b2efb7395b112",
    "23mlp_forward_pair_kernelENS_11MlpPairArgsE":
        "0c60912ae1b1225305c708d301b46510d22dc51bcef5a87be96173ee58b6cb3d",
    "25mlp_forward_masked_kernelINS_8MlpShapeILi0ELi0ELi0EEEEEvPKhPKfxS6_PfS7_S7_":
        "3131e81a515acfe0011226196a28ba0888c6cb4943cf039d25c03f14231d3b9b",
    "25mlp_forward_masked_kernelINS_8MlpShapeILi80ELi256ELi48EEEEEvPKhPKfxS6_PfS7_S7_":
        "fcb286b2bd044aec744ee88f66ff2bf578515a658721bc9ca44e34d89eb9b330",
}
_SAMPLED = ("26mlp_forward_sampled_kernelILb0EEEvPKhPKvxPfS5_S5_NS_11MlpSamplingE",
            "26mlp_forward_sampled_kernelILb1EEEvPKhPKvxPfS5_S5_NS_11MlpSamplingE")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.skip("needs nvcc")
    out = str(tmp_path_factory.mktemp("mlp") / "wdb_mlp.cubin")
    proc = subprocess.run(NVCC_SM90A + ["-Xptxas", "-v", "-cubin", "-I",
                                        os.path.join(ROOT, "include"), SRC, "-o", out],
                          capture_output=True, text=True, check=True)
    version = subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout
    return proc.stderr, out, "release 12.9" in version


def test_sampled_kernel_roles_fit_without_spills_or_serialised_wgmma(compiled):
    log, cubin, _ = compiled
    spills, name = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = _strip(m.group(1))
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name in _SAMPLED:
            spills[name] = (int(m.group(1)), int(m.group(2)))
        if re.search(r"C75(14|19)", line):
            assert "mlp_forward_sampled_kernel" not in line, line
    assert spills == {k: (0, 0) for k in _SAMPLED}, spills
    sass = subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True,
                          check=True).stdout
    for k in _SAMPLED:
        body = sass.split(k, 1)[1].split("Function :", 1)[0]
        # the epilogue warpgroup gives registers up (56 each), the MMA warpgroups take them
        # (224); 2 x 224 + 56 is the 3 x 168 the CTA is launched with
        assert re.search(r"USETMAXREG\.DEALLOC\.CTAPOOL 0x38\b", body), k
        mma = re.split(r"USETMAXREG\.TRY_ALLOC\.CTAPOOL \w+, 0xe0\b", body)
        assert len(mma) == 2, k
        assert not re.search(r"\b(STL|LDL)\b", body), k


def test_other_forward_kernels_keep_their_machine_code(compiled):
    _, cubin, is_129 = compiled
    if not is_129:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    got = _sass_hashes(cubin)
    assert {k: got.get(k) for k in _KEPT_SASS_SHA256} == _KEPT_SASS_SHA256
    assert set(got) == set(_KEPT_SASS_SHA256) | set(_SAMPLED)
