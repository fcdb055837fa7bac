"""Plans x GPUs: the same worker cases as the gloo tests (tests/dist_worker.py), on real GPUs over NCCL, against one GPU.

Covers what only ran on CPU before: tensor-parallel, pipeline (1F1B over NCCL p2p), pipeline x SPMD, a two-dimensional SPMD
mesh and expert parallelism (all-to-all) -- each must reproduce the single-GPU loss trajectory of the same model
(reference: xla/tests/dapple_*_test.cc run their collectives on real devices, SURVEY §4)."""
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run(case, world, tmp_path, extra_env=None):
    out = str(tmp_path / f"out{world}.json")
    env = dict(os.environ, TEPDIST_TEST_DEVICE="cuda", OMP_NUM_THREADS="2", **(extra_env or {}))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(HERE, "dist_worker.py"), case, out]
    if world == 1:
        cmd = [sys.executable, os.path.join(HERE, "dist_worker.py"), case, out]
    pr = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    assert pr.returncode == 0, (pr.stdout[-1500:], pr.stderr[-3000:])
    return json.load(open(out))


def _close(got, ref, tol=3e-2):
    for a, b in zip(got["losses"], ref["losses"]):
        assert abs(a - b) <= tol * max(1.0, abs(b)), (got, ref)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_plans_on_two_gpus_match_one_gpu(tmp_path):
    cases = ["gpt2:auto", "gpt2:tp", "gpt2:pp2m2", "moe:ep", "mlp:dp", "conv:dp"]     # conv:dp = synchronised BatchNorm; its f32 graph takes the torch path (the native split phases need bf16 and are checked on one GPU in test_conv_numerics_gpu.py)
    ref = _run("gpt2:auto+moe:auto+mlp:auto+conv:auto", 1, tmp_path)
    got = _run("+".join(cases), 2, tmp_path)
    for c in cases:
        _close(got[c], ref[c.split(":")[0] + ":auto"])
    assert got["gpt2:tp"]["parallelism"].startswith("tp"), got["gpt2:tp"]
    assert got["gpt2:pp2m2"]["parallelism"].startswith("pp2"), got["gpt2:pp2m2"]
    assert got["moe:ep"]["collectives"].get("all_to_all", 0) >= 2, got["moe:ep"]


@pytest.mark.skipif(torch.cuda.device_count() < 4, reason="needs 4 GPUs")
def test_pipeline_x_spmd_and_2d_mesh_on_four_gpus_match_one_gpu(tmp_path):
    ref = _run("gpt2:auto", 1, tmp_path)
    got = _run("gpt2:pp2m2+gpt2:dp2tp2", 4, tmp_path)
    assert got["gpt2:pp2m2"]["parallelism"] == "pp2xspmd2/micro2", got["gpt2:pp2m2"]
    _close(got["gpt2:pp2m2"], ref)
    _close(got["gpt2:dp2tp2"], ref)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_context_parallel_ring_attention_on_two_gpus_matches_one_gpu(tmp_path):
    """`cp`: the sequence (256 tokens) is cut in two blocks of 128, every token-wise op runs on its block, attention keeps its
    queries and passes K / V (forward) and K / V + the fp32 dK / dV accumulators (backward) around the ring over NCCL; the
    diagonal block runs the causal attention kernel, the off-diagonal one the unmasked kernel, partial outputs merge by
    log-sum-exp (parallel/ring_attention.py)."""
    env = {"TEPDIST_TEST_NCTX": "256"}
    ref = _run("gpt2:auto", 1, tmp_path, env)
    got = _run("gpt2:cp", 2, tmp_path, env)
    assert got["parallelism"] == "cp2", got
    _close(got, ref)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_context_parallel_zigzag_on_two_gpus_matches_one_gpu(tmp_path):
    """Load-balanced (zig-zag) ring: 512 tokens = 4 chunks of 128; rank 0 computes for chunks (0, 3), rank 1 for (1, 2); the
    half-block products run the same attention block kernels as the contiguous ring."""
    env = {"TEPDIST_TEST_NCTX": "512", "TEPDIST_CP_ZIGZAG": "1"}
    ref = _run("gpt2:auto", 1, tmp_path, env)
    got = _run("gpt2:cp", 2, tmp_path, env)
    assert got["parallelism"] == "cp2", got
    _close(got, ref)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_collective_lowering_on_gpus_over_nccl(tmp_path):
    """Every collective op of the IR on every dim of a rank-3 tensor over NCCL (the reference's dapple_*_test.cc run on real
    devices): 1-D mesh over all visible GPUs, and a 2 x (n/2) mesh when there are at least 4."""
    n = 8 if torch.cuda.device_count() >= 8 else (4 if torch.cuda.device_count() >= 4 else 2)
    got = _run("collectives:1d", n, tmp_path)
    assert got["checks"] == 16 and not got["fails"], got
    if n >= 4:
        got = _run("collectives:2d", n, tmp_path)
        assert got["checks"] == 32 and not got["fails"], got


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sequence_parallel_tensor_parallelism_on_two_gpus_matches_one_gpu(tmp_path):
    """`tpsp`: row-parallel GEMM -> NCCL reduce-scatter over tokens -> bias + residual shard; all-gather before the next
    column-parallel GEMM."""
    ref = _run("gpt2:auto", 1, tmp_path)
    got = _run("gpt2:tpsp", 2, tmp_path)
    assert got["parallelism"].startswith("tp") and got["collectives"].get("reduce_scatter", 0) >= 4, got
    _close(got, ref)
