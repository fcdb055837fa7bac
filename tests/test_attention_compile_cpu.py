"""Compile-time check of the sm_90a flash-attention kernels (no GPU needed): every kernel in attention_sm90.cu compiles
with no stack frame and no spills, and ptxas never serialises its wgmma chains (note C7520, "wgmma.mma_async instructions
are serialized").  Both were once true of the 64-wide-head kernels and cost them most of their speed."""
import os
import re
import shutil
import subprocess

import pytest

from tepdist_b200 import build_native

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    src = os.path.join(build_native.OPS_SRC, "attention_sm90.cu")
    obj = tmp_path_factory.mktemp("attn") / "attention_sm90.o"
    r = subprocess.run([NVCC, *build_native.NVCC_FLAGS, "-I", build_native.OPS_SRC, "-c", src, "-o", str(obj)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


def test_attention_kernels_do_not_spill(ptxas_log):
    props = re.findall(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", ptxas_log)
    kernels = {name: tuple(map(int, v)) for name, *v in props}
    for kind in ("attn_fwd_kernelILi64ELb0", "attn_fwd_kernelILi64ELb1", "attn_bwd_kernelILi64ELb0",
                 "attn_bwd_kernelILi64ELb1", "attn_fwd_kernelILi128", "attn_bwd_kernelILi128"):
        assert any(kind in n for n in kernels), f"{kind} not compiled"
    spilling = {n: v for n, v in kernels.items() if v != (0, 0, 0)}
    assert not spilling, spilling


def test_attention_wgmma_is_not_serialized(ptxas_log):
    assert "C7520" not in ptxas_log, [l for l in ptxas_log.splitlines() if "C7520" in l]
