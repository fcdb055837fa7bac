"""Document-masked causal attention (packed rows, `doc_start`) against our plain causal kernel and PyTorch SDPA with a dense
boolean mask, and the GPT-2 345M training step with and without `eot_token`.

Attention table: D in {64, 128} with B * H * D = 4 * 2048 (B = 4, H = 2048 / D), causal, S in {1024, 2048, 4096, 8192}, and
document lengths drawn per row from a seeded geometric distribution with mean S (one document per row), 1024 or 256.
TFLOP/s counts 4 * D * H * (unmasked (query, key) pairs, counted from doc_start) for the forward and 2.5 x that for the
backward, so the masked and the plain kernel are rated on the work each must do.  SDPA gets the same mask as a dense
[B, 1, S, S] boolean tensor; the backend torch picks for it (torch._fused_sdp_choice) is named, and the math backend is skipped
when its [B, H, S, S] fp32 scores would not fit.  Times are CUDA-event means over --iters calls after warm-up.

Whole step: GPT-2 345M, batch 4, CUDA-graph steps, synthetic tokens with EOT (50256) at a seeded rate of 1 / 256 (mean
document 256 tokens); the plain and the eot_token model alternate --rounds times in this process on the same tokens.

The card name, power limit and max SM clock are read (read-only nvidia-smi query) in the same run.

    python bench/doc_mask_attention.py [--iters 10] [--rounds 5] [--steps 20] [--json out.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

EOT = 50256


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


def packed_tokens(B: int, S: int, mean: int, gen: torch.Generator, vocab: int = EOT) -> torch.Tensor:
    """int32 [B, S]: random tokens with EOT ending documents of geometric length (mean `mean`; mean >= S: no EOT)."""
    tok = torch.randint(0, vocab, (B, S), generator=gen, dtype=torch.int32)
    if mean < S:
        tok[torch.rand(B, S, generator=gen) < 1.0 / mean] = EOT
    return tok


def _pairs(ds: torch.Tensor) -> int:
    S = ds.shape[1]
    return int((torch.arange(S, device=ds.device) - ds.long() + 1).sum())


def attention_table(iters: int):
    from tepdist_b200 import ops
    rows = []
    gen = torch.Generator().manual_seed(0)
    for D in (64, 128):
        B, H = 4, 2048 // D
        for S in (1024, 2048, 4096, 8192):
            q, k, v = (torch.randn(B, S, H, D, device="cuda", dtype=torch.bfloat16) for _ in range(3))
            do = torch.randn(B, S, H, D, device="cuda", dtype=torch.bfloat16)
            o0, lse0 = ops.attention_fwd(q, k, v, causal=True)
            plain_pairs = B * S * (S + 1) // 2
            t_pf = _time_ms(lambda: ops.attention_fwd(q, k, v, causal=True), iters)
            t_pb = _time_ms(lambda: ops.attention_bwd(do, q, k, v, o0, lse0, causal=True), iters)
            for mean in [S] + [m for m in (1024, 256) if m < S]:
                ds = ops.doc_starts(packed_tokens(B, S, mean, gen).cuda(), EOT)
                pairs = _pairs(ds)
                n0 = ops.launch_count()
                o, lse = ops.attention_fwd(q, k, v, causal=True, doc_start=ds)
                t_f = _time_ms(lambda: ops.attention_fwd(q, k, v, causal=True, doc_start=ds), iters)
                t_b = _time_ms(lambda: ops.attention_bwd(do, q, k, v, o, lse, causal=True, doc_start=ds), iters)
                assert ops.launch_count() > n0, "attention kernels did not run"
                fl = 4.0 * D * H * pairs
                row = {"D": D, "S": S, "B": B, "H": H, "mean_doc": mean, "docs_per_row": float((ds[:, 1:] != ds[:, :-1]).sum()) / B + 1,
                       "unmasked_pairs_frac": pairs / plain_pairs,
                       "doc_fwd_ms": t_f, "doc_bwd_ms": t_b, "doc_fwd_tflops": fl / t_f / 1e9, "doc_bwd_tflops": 2.5 * fl / t_b / 1e9,
                       "causal_fwd_ms": t_pf, "causal_bwd_ms": t_pb,
                       "causal_fwd_tflops": 4.0 * D * H * plain_pairs / t_pf / 1e9,
                       "causal_bwd_tflops": 10.0 * D * H * plain_pairs / t_pb / 1e9}
                row.update(_sdpa(q, k, v, do, ds, iters))
                rows.append(row)
                print(json.dumps(row), flush=True)
            del q, k, v, do, o0, lse0
            torch.cuda.empty_cache()
    return rows


def _sdpa(q, k, v, do, ds, iters: int):
    B, S, H, D = q.shape
    keys = torch.arange(S, device="cuda")
    mask = (torch.ones(S, S, dtype=torch.bool, device="cuda").tril()
            & (keys.view(1, 1, S) >= ds.long().unsqueeze(-1))).unsqueeze(1)      # [B, 1, S, S], True = attend
    qt, kt, vt = (t.transpose(1, 2).detach().requires_grad_(True) for t in (q, k, v))
    dot = do.transpose(1, 2)
    from torch.nn.attention import SDPBackend
    backend = SDPBackend(torch._fused_sdp_choice(qt, kt, vt, mask, 0.0, False)).name
    if backend == "MATH" and B * H * S * S * 4 * 4 > 40e9:
        return {"sdpa_backend": backend, "sdpa_fwd_ms": None, "sdpa_bwd_ms": None, "sdpa_note": "skipped: [B,H,S,S] fp32 scores"}
    try:
        t_f = _time_ms(lambda: F.scaled_dot_product_attention(qt, kt, vt, attn_mask=mask), iters)
        out = F.scaled_dot_product_attention(qt, kt, vt, attn_mask=mask)
        t_b = _time_ms(lambda: torch.autograd.grad(out, (qt, kt, vt), dot, retain_graph=True), iters)
    except torch.cuda.OutOfMemoryError:
        torch.cuda.empty_cache()
        return {"sdpa_backend": backend, "sdpa_fwd_ms": None, "sdpa_bwd_ms": None, "sdpa_note": "out of memory"}
    return {"sdpa_backend": backend, "sdpa_fwd_ms": t_f, "sdpa_bwd_ms": t_b}


def whole_step(rounds: int, steps: int):
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    cfg = CONFIGS["345M"]
    gen = torch.Generator().manual_seed(1)
    toks = [packed_tokens(cfg.batch, cfg.n_ctx, 256, gen).cuda() for _ in range(4)]
    feeds = [{"tokens": t, "labels": torch.roll(t, -1, 1)} for t in toks]
    arms = {"plain": Trainer(build_gpt2_graph(cfg), use_cuda_graph=True),
            "eot_token": Trainer(build_gpt2_graph(cfg, eot_token=EOT), use_cuda_graph=True)}
    for tr in arms.values():
        for i in range(5):
            tr.step_async(feeds[i % 4])
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    loss = {}
    for _ in range(rounds):
        for name, tr in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(steps):
                l = tr.step_async(feeds[i % 4])
            b.record()
            torch.cuda.synchronize()
            ms[name].append(a.elapsed_time(b) / steps)
            loss[name] = float(l)
    return {"model": cfg.name, "batch": cfg.batch, "n_ctx": cfg.n_ctx, "steps_per_round": steps, "rounds": rounds,
            "ms_per_step": ms, "median_ms": {k: statistics.median(v) for k, v in ms.items()}, "last_loss": loss,
            "docs_per_row": float(sum(int((t == EOT).sum()) for t in toks)) / (4 * cfg.batch) + 1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--no-step", action="store_true")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("doc_mask_attention.py: no CUDA GPU; the timings are only meaningful on the H100")
    card = _card()
    print("card:", card, flush=True)
    res = {"card": card, "attention": attention_table(a.iters)}
    if not a.no_step:
        res["step"] = whole_step(a.rounds, a.steps)
        print(json.dumps(res["step"]), flush=True)
    res["card_after"] = _card()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
