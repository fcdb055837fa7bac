"""GPT-2 training step with and without dropout on one GPU: the cost of the masks in the whole step.

Two executors of the same model (default 345M, batch 4 x 1024 tokens, AdamW, CUDA-graph replay), one without dropout and one
with embd_pdrop = attn_pdrop = resid_pdrop = `--dropout`, warmed up, then timed in alternating rounds of `--steps` steps
(host clock around each round, which ends in a device synchronise).  Prints the median step time of each and their ratio;
the card name, power limit and max SM clock are read (read-only nvidia-smi query) in the same run.

    python bench/dropout_step.py [--model 345M] [--dropout 0.1] [--steps 10] [--rounds 5] [--json out.json]
"""
from __future__ import annotations

import argparse
import dataclasses
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from attention_heads import _card  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--model", default="345M")
    ap.add_argument("--dropout", type=float, default=0.1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("dropout_step.py: no CUDA GPU; the timings are only meaningful on the H100")
    from tepdist_b200 import ops
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    from tepdist_b200.runtime.executor import Executor
    ops.lib()
    card = _card()
    print(f"# card: {card}  (name, power limit, max SM clock)")
    base = CONFIGS[a.model]
    cfgs = {"off": base, f"p{a.dropout:g}": dataclasses.replace(base, embd_pdrop=a.dropout, attn_pdrop=a.dropout,
                                                                 resid_pdrop=a.dropout)}
    torch.manual_seed(0)
    tok = torch.randint(0, base.n_vocab, (base.batch, base.n_ctx), dtype=torch.int32, device="cuda")
    feeds = {"tokens": tok, "labels": torch.roll(tok, -1, 1)}
    exes = {k: Executor(build_gpt2_graph(c), torch.device("cuda", 0), use_cuda_graph=True) for k, c in cfgs.items()}
    for ex in exes.values():
        for _ in range(a.warmup):
            ex.step(feeds)
    torch.cuda.synchronize()
    times = {k: [] for k in exes}
    for _ in range(a.rounds):
        for k, ex in exes.items():
            t0 = time.perf_counter()
            for _ in range(a.steps):
                out = ex.step(feeds)
            float(out[0])
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) / a.steps * 1e3)
    med = {k: statistics.median(v) for k, v in times.items()}
    keys = list(exes)
    for k in keys:
        print(f"{a.model} {k:6s} step {med[k]:.2f} ms (rounds: {', '.join(f'{t:.2f}' for t in times[k])})")
    print(f"dropout / no dropout: {med[keys[1]] / med[keys[0]]:.3f}")
    if a.json:
        with open(a.json, "w") as fh:
            json.dump({"card": card, "model": a.model, "dropout": a.dropout, "step_ms": times, "median_ms": med}, fh, indent=1)


if __name__ == "__main__":
    main()
