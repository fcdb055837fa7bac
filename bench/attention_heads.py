"""Attention forward / backward time for 64- and 128-wide heads: our kernels vs PyTorch SDPA (flash backend) and vs the
fp32 torch-math path that shapes without a kernel run (materialised [B, H, S, S] scores).

B * H * D is held at 4 * 2048 (B = 4, H = 2048 / D), as for a 2048-wide model, over S = 1024 .. 8192, causal and not.
TFLOP/s counts 4 * B * H * S^2 * D for the forward (halved when causal) and 2.5 x that for the backward.  Times are
CUDA-event means over `--iters` calls after warm-up.  The card name, power limit and max SM clock are read (read-only
nvidia-smi query) in the same run and printed with the table.

    python bench/attention_heads.py [--iters 10] [--json out.json]
"""
from __future__ import annotations

import argparse
import contextlib
import json
import os
import subprocess
import sys
import warnings

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402


def _card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name()


def _time_ms(fn, iters: int, warmup: int = 3) -> float:
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


@contextlib.contextmanager
def _torch_math():
    """Route ops.attention_* through the torch-math path (what shapes without a kernel run)."""
    from tepdist_b200.ops import attention as A
    saved = A._KERNEL_WIDTHS
    A._KERNEL_WIDTHS = ()
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            yield
    finally:
        A._KERNEL_WIDTHS = saved


def run(D: int, S: int, causal: bool, iters: int) -> dict:
    from tepdist_b200 import ops
    B, H = 4, 2048 // D
    torch.manual_seed(0)
    qkv = torch.randn(B, S, H, 3, D, device="cuda", dtype=torch.bfloat16)
    q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    do = torch.randn(B, S, H, D, device="cuda", dtype=torch.bfloat16)
    fl = 4.0 * B * H * S * S * D * (0.5 if causal else 1.0)
    r = {"D": D, "S": S, "B": B, "H": H, "causal": causal}

    n0 = ops.launch_count()
    o, lse = ops.attention_fwd(q, k, v, causal=causal)
    assert ops.launch_count() > n0, "attention kernel did not run"
    r["ours_fwd_ms"] = _time_ms(lambda: ops.attention_fwd(q, k, v, causal=causal), iters)
    r["ours_bwd_ms"] = _time_ms(lambda: ops.attention_bwd(do, q, k, v, o, lse, causal=causal), iters)

    qs, ks, vs = (t.permute(0, 2, 1, 3).contiguous().requires_grad_(True) for t in (q, k, v))
    dos = do.permute(0, 2, 1, 3).contiguous()
    with torch.nn.attention.sdpa_kernel(torch.nn.attention.SDPBackend.FLASH_ATTENTION):
        r["sdpa_fwd_ms"] = _time_ms(lambda: F.scaled_dot_product_attention(qs, ks, vs, is_causal=causal), iters)
        out = F.scaled_dot_product_attention(qs, ks, vs, is_causal=causal)
        r["sdpa_bwd_ms"] = _time_ms(lambda: torch.autograd.grad(out, (qs, ks, vs), dos, retain_graph=True), iters)
    del qs, ks, vs, dos, out

    # the torch-math backward holds ~6 fp32 [B, H, S, S] tensors at once
    torch.cuda.empty_cache()
    if 6 * B * H * S * S * 4 < 0.9 * torch.cuda.mem_get_info()[0]:
        with _torch_math():
            r["math_fwd_ms"] = _time_ms(lambda: ops.attention_fwd(q, k, v, causal=causal), max(2, iters // 4), warmup=1)
            r["math_bwd_ms"] = _time_ms(lambda: ops.attention_bwd(do, q, k, v, o, lse, causal=causal), max(2, iters // 4),
                                        warmup=1)
        torch.cuda.empty_cache()
    for k_ in [k_ for k_ in r if k_.endswith("_ms")]:
        r[k_.replace("_ms", "_tflops")] = (fl if "fwd" in k_ else 2.5 * fl) / r[k_] / 1e9
    return r


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", default=None, help="also write the rows (and the card) to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("attention_heads.py: no CUDA GPU; the timings are only meaningful on the H100")
    from tepdist_b200 import ops
    ops.lib()
    card = _card()
    print(f"# card: {card}  (name, power limit, max SM clock)")
    hdr = f"{'D':>4} {'S':>5} {'causal':>6} | {'ours fwd':>9} {'sdpa fwd':>9} {'math fwd':>9} | {'ours bwd':>9} {'sdpa bwd':>9} " \
          f"{'math bwd':>9} | fwd/sdpa bwd/sdpa  (TFLOP/s; ratio = sdpa time / ours time)"
    print(hdr)
    rows = []
    for D in (64, 128):
        for causal in (True, False):
            for S in (1024, 2048, 4096, 8192):
                r = run(D, S, causal, a.iters)
                rows.append(r)
                f = lambda k: f"{r[k]:9.1f}" if k in r else f"{'-':>9}"
                print(f"{D:>4} {S:>5} {str(causal):>6} | {f('ours_fwd_tflops')} {f('sdpa_fwd_tflops')} {f('math_fwd_tflops')} | "
                      f"{f('ours_bwd_tflops')} {f('sdpa_bwd_tflops')} {f('math_bwd_tflops')} | "
                      f"{r['sdpa_fwd_ms'] / r['ours_fwd_ms']:8.2f} {r['sdpa_bwd_ms'] / r['ours_bwd_ms']:8.2f}", flush=True)
    if a.json:
        with open(a.json, "w") as fh:
            json.dump({"card": card, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
