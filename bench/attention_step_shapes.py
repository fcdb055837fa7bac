"""Flash-attention calls at the shapes the GPT-2 training steps run them: 345M (B 4, H 16, S 1024, D 64, causal) and 1.3B
(B 2, H 16, S 2048, D 128, causal), q / k / v as views of one fused [B, S, H, 3, D] buffer as the executor passes them.

Per shape: the forward and backward call times (CUDA-event means over `--iters` calls after warm-up), then a torch.profiler
pass in which each kernel of the calls (forward, delta, backward, dQ cast) gets its own time.  TFLOP/s counts
4 * B * H * S^2 * D / 2 for the causal forward and 2.5 x that for the backward.  The card name, power limit and max SM clock
are read (read-only nvidia-smi query) in the same run.

    python bench/attention_step_shapes.py [--iters 50] [--json out.json]
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from attention_heads import _card, _time_ms  # noqa: E402

SHAPES = {"345M": (4, 16, 1024, 64), "1.3B": (2, 16, 2048, 128)}


def run(name: str, iters: int) -> dict:
    from tepdist_b200 import ops
    B, H, S, D = SHAPES[name]
    torch.manual_seed(0)
    qkv = torch.randn(B, S, H, 3, D, device="cuda", dtype=torch.bfloat16)
    q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    do = torch.randn(B, S, H, D, device="cuda", dtype=torch.bfloat16)
    dqkv = torch.empty_like(qkv)
    fl = 4.0 * B * H * S * S * D * 0.5
    n0 = ops.launch_count()
    o, lse = ops.attention_fwd(q, k, v, causal=True)
    ops.attention_bwd(do, q, k, v, o, lse, causal=True, dqkv_out=dqkv)
    assert ops.launch_count() >= n0 + 4, "attention kernels did not run"
    fwd = lambda: ops.attention_fwd(q, k, v, causal=True)  # noqa: E731
    bwd = lambda: ops.attention_bwd(do, q, k, v, o, lse, causal=True, dqkv_out=dqkv)  # noqa: E731
    r = {"shape": name, "B": B, "H": H, "S": S, "D": D, "fwd_ms": _time_ms(fwd, iters), "bwd_ms": _time_ms(bwd, iters)}
    r["fwd_tflops"] = fl / r["fwd_ms"] / 1e9
    r["bwd_tflops"] = 2.5 * fl / r["bwd_ms"] / 1e9
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fwd()
            bwd()
        torch.cuda.synchronize()
    kern = collections.defaultdict(float)
    for ka in prof.key_averages():
        us = getattr(ka, "self_device_time_total", None) or getattr(ka, "self_cuda_time_total", 0.0)
        m = re.search(r"attn_\w+<[^>]*>", ka.key)
        if us and m:
            kern[m.group(0)] += us / iters / 1e3
    r["kernels_ms"] = dict(kern)
    return r


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("attention_step_shapes.py: no CUDA GPU; the timings are only meaningful on the H100")
    from tepdist_b200 import ops
    ops.lib()
    card = _card()
    print(f"# card: {card}  (name, power limit, max SM clock)")
    rows = []
    for name in SHAPES:
        r = run(name, a.iters)
        rows.append(r)
        print(f"{name:5s} B {r['B']} H {r['H']} S {r['S']} D {r['D']} causal | fwd {r['fwd_ms']:.4f} ms {r['fwd_tflops']:6.1f} TFLOP/s"
              f" | bwd {r['bwd_ms']:.4f} ms {r['bwd_tflops']:6.1f} TFLOP/s", flush=True)
        for kname, ms in sorted(r["kernels_ms"].items(), key=lambda kv: -kv[1]):
            print(f"      {kname:32s} {ms:.4f} ms")
    if a.json:
        with open(a.json, "w") as fh:
            json.dump({"card": card, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
