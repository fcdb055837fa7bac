"""The multi-tensor optimizer kernels without a GPU: every kernel of optim_sm90.cu compiles for sm_90a with no stack frame and
no spills, and the host-built work table (ops.optim_tables) covers every element of the GPT-2 345M and GPT-MoE variable
sets exactly once, with row chunks of whole rows."""
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from tepdist_b200 import build_native, ops

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
KERNELS = ("optim_momentum_kernel", "optim_lamb_moments_kernel", "optim_lamb_apply_kernel", "optim_af_stats_kernel",
           "optim_af_cols_kernel", "optim_af_usq_kernel", "optim_af_apply_kernel", "optim_sm3_kernel", "optim_sm3_finish_kernel")


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")
def test_optimizer_kernels_do_not_spill(tmp_path):
    src = os.path.join(build_native.OPS_SRC, "optim_sm90.cu")
    r = subprocess.run([NVCC, *build_native.NVCC_FLAGS, "-I", build_native.OPS_SRC, "-c", src, "-o", str(tmp_path / "o.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    props = re.findall(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stdout + r.stderr)
    kernels = {name: tuple(map(int, v)) for name, *v in props}
    for k in KERNELS:
        assert any(k in n for n in kernels), f"{k} not compiled"
    spilling = {n: v for n, v in kernels.items() if v != (0, 0, 0)}
    assert not spilling, spilling


def variable_sets():
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    from tepdist_b200.models.gpt_moe import MoEConfig, build_gpt_moe_graph
    g2 = build_gpt2_graph(CONFIGS["345M"])
    moe = build_gpt_moe_graph(MoEConfig())
    return {"gpt2-345M": [tuple(n.outputs[0].shape) for n in g2.params()],
            "gpt-moe": [tuple(n.outputs[0].shape) for n in moe.params()]}


@pytest.mark.parametrize("op,opt", [("apply_momentum", {}), ("apply_lamb", {}), ("apply_adafactor", {}),
                                    ("apply_adafactor", {"factored": False}), ("apply_sm3", {"momentum": 0.9})])
def test_work_table_covers_every_element_once(op, opt):
    for label, shapes in variable_sets().items():
        offs, off = [], 0
        for s in shapes:
            offs.append(off)
            off += -(-math.prod(s) // 128) * 128
        decays = [len(s) >= 2 for s in shapes]
        vars_, chunks, ws, col_blocks = ops.optim_tables(op, shapes, offs, decays, opt)
        assert len(vars_) == len(shapes) and 1 <= col_blocks <= 1024
        if label == "gpt-moe":
            assert any(len(s) == 3 for s in shapes)
        extent = 4 * len(chunks)
        for i, s in enumerate(shapes):
            n = math.prod(s)
            off_, n_, B, R, C, flags, c0, nc, sc, rank = (int(x) for x in vars_[i, :10])
            assert (off_, n_, rank, B * R * C) == (offs[i], n, len(s), n)
            mine = chunks[c0:c0 + nc]
            assert (mine[:, 0] == i).all() and nc >= 1
            order = np.argsort(mine[:, 4], kind="stable")
            e0, ne = mine[order, 4], mine[order, 5]
            assert e0[0] == 0 and (ne > 0).all() and (e0[1:] == (e0 + ne)[:-1]).all() and int(e0[-1] + ne[-1]) == n, (label, s)
            if flags & 2:                  # row chunks: whole rows of the [B * R, C] view, at most 32 per chunk
                assert len(s) >= 2 and C == s[-1] and R == s[-2]
                assert (mine[:, 3] <= ops.OPTIM_ROW_CHUNK).all() and (mine[:, 4] == (mine[:, 1] * R + mine[:, 2]) * C).all()
                assert (mine[:, 5] == mine[:, 3] * C).all() and int(vars_[i, 14]) * B == nc
                need = nc * C if op == "apply_adafactor" else B + R + C
                assert sc >= 4 * len(chunks) and sc + need <= ws
                extent = max(extent, sc + need)
            else:
                assert (mine[:, 4] % 4 == 0).all() and (mine[:, 5] <= ops.OPTIM_FLAT_CHUNK).all()
        assert extent == ws
        assert (chunks[:, 0] == np.repeat(np.arange(len(shapes)), [int(v[7]) for v in vars_])).all()
