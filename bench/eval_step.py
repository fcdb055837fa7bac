#!/usr/bin/env python
"""Evaluation step of GPT-2 345M on one GPU, and the two kernels it adds, timed with CUDA events after warm-up:

  * Executor.evaluate (forward only, dropout off, CUDA graph) against Executor.step, both at the 345M step shape (4 x 1024
    tokens) and on the same weights;
  * ops.xent_fwd (one read of the logits, nothing written) against ops.xent_fwd_bwd at [4096, 50304] bf16, with the HBM
    floor of each computed from bytes at 3.35 TB/s (H100 SXM data sheet);
  * the mlp/c_fc GEMM (4096 x 4096 x 1024, bias + GELU) through EPI_BIAS_GELU, EPI_GELU_DUAL (which also writes the
    pre-activation) and EPI_DIRECT (fragment stores, forced by a padded output row pitch).

    python bench/eval_step.py [--steps 20] [--warmup 5] [--out results.json]

Prints one JSON line with every time in ms, the card's name and its power limit.  Writes nothing into the repository.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench/eval_step.py needs a GPU")
    from tepdist_b200 import ops
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    from tepdist_b200.runtime.executor import Executor
    res = {"card": card()}

    # kernels first, on an otherwise idle device
    T, Vp, V = 4096, 50304, 50257
    logits = (torch.randn(T, Vp, device="cuda") * 3).to(torch.bfloat16)
    labels = torch.randint(0, V, (T,), device="cuda", dtype=torch.int32)
    work = logits.clone()
    row_bytes = T * Vp * 2
    res["xent_fwd_ms"] = timed(lambda: ops.xent_fwd(logits, labels, V), 50, 10)
    res["xent_fwd_bwd_ms"] = timed(lambda: ops.xent_fwd_bwd(work, labels, V, 1.0), 50, 10)   # (overwrites `work`: timing only)
    res["xent_fwd_floor_ms"] = row_bytes / HBM_BYTES_PER_S * 1e3
    res["xent_fwd_bwd_floor_ms"] = 4 * row_bytes / HBM_BYTES_PER_S * 1e3
    del logits, work

    M, N, K = 4096, 4096, 1024
    a = (torch.randn(M, K, device="cuda") * 0.5).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda") * 0.03).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda") * 0.1
    out, pre, act = (torch.empty(M, N, device="cuda", dtype=torch.bfloat16) for _ in range(3))
    padded = torch.empty(M, N + 4, device="cuda", dtype=torch.bfloat16)[:, :N]
    gemm_flop = 2.0 * M * N * K
    kinds = {"EPI_BIAS_GELU": lambda: ops.gemm(a, w, bias=bias, act="gelu", out=out),
             "EPI_GELU_DUAL": lambda: ops.gemm(a, w, bias=bias, act="gelu", out=pre, out2=act),
             "EPI_DIRECT": lambda: ops.gemm(a, w, bias=bias, act="gelu", out=padded)}
    res["c_fc_gemm"] = {}
    for name, fn in kinds.items():
        ms = timed(fn, 100, 20)
        res["c_fc_gemm"][name] = {"ms": ms, "tflops": gemm_flop / ms / 1e9}
    del a, w, out, pre, act, padded

    cfg = CONFIGS["345M"]
    ex = Executor(build_gpt2_graph(cfg), torch.device("cuda", 0), seed=0, use_cuda_graph=True)
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (cfg.batch, cfg.n_ctx), dtype=torch.int32, device="cuda")
    feeds = {"tokens": tok, "labels": torch.roll(tok, -1, 1)}
    res["train_step_ms"] = timed(lambda: ex.step(feeds), args.steps, args.warmup)
    res["eval_step_ms"] = timed(lambda: ex.evaluate(feeds), args.steps, args.warmup)
    torch.cuda.synchronize()
    ex2 = Executor(build_gpt2_graph(cfg), torch.device("cuda", 0), seed=0)     # eager: peak memory of each call
    for fn in (lambda: ex2.step(feeds), lambda: ex2.evaluate(feeds)):
        fn()
    peaks = {}
    for name, fn in (("train_step", lambda: ex2.step(feeds)), ("eval_step", lambda: ex2.evaluate(feeds))):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fn()
        torch.cuda.synchronize()
        peaks[name] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    res["peak_mib_above_resident"] = peaks
    res["shape"] = {"model": cfg.name, "batch": cfg.batch, "n_ctx": cfg.n_ctx}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
