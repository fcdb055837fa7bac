"""Needs >= 2 GPUs: fused peer-memory optimizer path == NCCL path == single GPU (loss trajectories)."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_fused_dp_matches_nccl_and_single(tmp_path):
    out = str(tmp_path / "o.json")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29741", os.path.join(HERE, "multi_gpu_worker.py"), out]
    pr = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert pr.returncode == 0, pr.stderr[-3000:]
    r = json.load(open(out))
    assert r["fused_fused_active"] and not r["nccl_fused_active"]
    for a, b, c in zip(r["fused"], r["nccl"], r["single"]):
        assert abs(a - b) < 2e-2 * abs(b) and abs(a - c) < 2e-2 * abs(c), r
    assert r["fused"][-1] < r["fused"][0]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_tp_plan_fused_all_reduce_matches_nccl(tmp_path):
    out = str(tmp_path / "tpplan.json")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29744", os.path.join(HERE, "tp_plan_worker.py"), out]
    pr = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert pr.returncode == 0, pr.stderr[-3000:]
    r = json.load(open(out))
    assert r["fused_chains"] > 0 and r["nccl_chains"] == 0, r
    for a, b, c in zip(r["fused"], r["nccl"], r["single"]):
        assert abs(a - b) < 2e-2 * abs(b) and abs(a - c) < 2e-2 * abs(c), r


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_nvls_multicast_substrate_and_multimem_kernels(tmp_path):
    """VMM symmetric memory bound to an NVSwitch multicast object; multimem all-reduce (+ bias + residual) and the NVLS
    optimizer step (fp32 and bf16 gradient wire) against plain references."""
    out = str(tmp_path / "mc.json")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29745", os.path.join(HERE, "mc_worker.py"), out]
    pr = subprocess.run(cmd, capture_output=True, text=True, timeout=400)
    assert pr.returncode == 0, (pr.stdout[-2000:], pr.stderr[-3000:])
    r = json.load(open(out))
    if r["backend"] != "vmm":
        pytest.skip("no multicast support on this box")
    assert r["barrier_ok"] and r["peer_read_ok"], r
    assert r["ar_relerr"] < 1e-2 and r["ar_epi_relerr"] < 1e-2, r
    assert r["opt_f32_relerr"] < 1e-2 and r["opt_bf16_relerr"] < 1e-2 and r["opt_f32_master_relerr"] < 1e-5, r
