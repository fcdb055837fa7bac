#!/usr/bin/env python
"""GPT-2 training (reference examples/GPT2/main.py: "Train loop took X s").  Input: synthetic `fake_input` by default (one fixed
random batch, like the reference's FAKE_INPUT server flag), `--data a.bin,b.bin` for token files through the native prefetching
loader (tepdist_b200/data: memory-mapped uint16 / int32 token streams, windows of n_ctx + 1 tokens, stateless sampling), or
`--data synthetic` for a fresh random batch every step from the same loader."""
import argparse
import dataclasses
import math
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tepdist_b200.api import Trainer  # noqa: E402
from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="345M", choices=list(CONFIGS))
    ap.add_argument("--batch", type=int, default=4, help="sequences per GPU")
    ap.add_argument("--train-steps", type=int, default=10)
    ap.add_argument("--strategy", default="auto")
    ap.add_argument("--comm", default="fused", choices=["fused", "nccl"])
    ap.add_argument("--warmup-steps", type=int, default=0, help='linear warm-up then cosine decay over --train-steps (reference json: "warmup_steps")')
    ap.add_argument("--optimizer", default="adamw", choices=["adam", "adamw", "adafactor", "lamb", "sm3", "momentum", "sgd"],
                    help='reference: "opt_name" adam | adafactor in examples/GPT2/*.json')
    ap.add_argument("--clip-norm", default=None, choices=["global", "local"], help='gradient clipping (reference gpt_moe config: "clip_norm")')
    ap.add_argument("--clip-norm-value", type=float, default=1.0)
    ap.add_argument("--data", default=None, help="comma-separated token files (see tepdist_b200.data.write_token_file) or 'synthetic'")
    ap.add_argument("--data-int32", action="store_true", help="token files hold int32 ids (default uint16)")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--dropout", type=float, default=0.0,
                    help="GPT-2's dropout: this probability on the embedding sum, the attention probabilities and every block output "
                         "(embd_pdrop = attn_pdrop = resid_pdrop; the reference configuration uses 0.1)")
    ap.add_argument("--eot-token", type=int, default=None,
                    help="end-of-text token id (50256 for GPT-2): attention stays inside each packed document")
    ap.add_argument("--reset-position-ids", action="store_true",
                    help="learned positions count from each document's start (needs --eot-token)")
    ap.add_argument("--eval-data", default=None,
                    help="held-out token files (comma-separated) or 'synthetic': evaluation loss and perplexity, dropout off")
    ap.add_argument("--eval-every", type=int, default=0, help="evaluate after every N training steps (0: never)")
    ap.add_argument("--eval-batches", type=int, default=4, help="batches per evaluation")
    a = ap.parse_args()
    clip = {"clip_norm": a.clip_norm, "clip_norm_value": a.clip_norm_value} if a.clip_norm else {}
    cfg = CONFIGS[a.model]
    if a.dropout:
        cfg = dataclasses.replace(cfg, embd_pdrop=a.dropout, attn_pdrop=a.dropout, resid_pdrop=a.dropout)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    g = build_gpt2_graph(cfg, batch=a.batch * world, optimizer=a.optimizer, eot_token=a.eot_token,
                         reset_position_ids=a.reset_position_ids, **clip)
    tr = Trainer(g, strategy=a.strategy, comm_mode=a.comm)
    if a.warmup_steps > 0:
        from tepdist_b200.utils.schedules import warmup_cosine
        tr.set_lr_schedule(warmup_cosine(cfg.lr, a.warmup_steps, a.train_steps))
    if a.data:
        # every rank draws the same GLOBAL batch (sampling is a pure function of seed and step) and the trainer takes the rows /
        # columns its plan assigns to this rank: works unchanged under data, tensor, context and pipeline parallel plans
        from tepdist_b200.data import TokenLoader
        src = {"synthetic_vocab": cfg.n_vocab} if a.data == "synthetic" else {"files": a.data.split(","), "bytes_per_token": 4 if a.data_int32 else 2}
        batches = iter(TokenLoader(batch=a.batch * world, n_ctx=cfg.n_ctx, seed=a.seed, **src))
    else:
        gen = torch.Generator().manual_seed(a.seed)
        tok = torch.randint(0, cfg.n_vocab, (a.batch * world, cfg.n_ctx), generator=gen, dtype=torch.int32)
        fixed = {"tokens": tok, "labels": torch.roll(tok, -1, 1)}
        batches = iter(lambda: fixed, None)
    eval_batches = None
    if a.eval_data and a.eval_every > 0:
        # its own fixed seed and step 0 on every evaluation: every evaluation sees the same held-out batches
        from tepdist_b200.data import TokenLoader
        src = ({"synthetic_vocab": cfg.n_vocab} if a.eval_data == "synthetic" else
               {"files": a.eval_data.split(","), "bytes_per_token": 4 if a.data_int32 else 2})
        eval_batches = [{k: v.clone() for k, v in b.items()} for b, _ in zip(TokenLoader(batch=a.batch * world, n_ctx=cfg.n_ctx, seed=a.seed + 1_000_003, start_step=0,
                                                      **src), range(a.eval_batches))]
    t0 = time.time()
    for i in range(a.train_steps):
        loss = tr.step(next(batches))
        if tr.rank == 0:
            print(f"step {i} loss {loss:.4f}")
        if eval_batches and (i + 1) % a.eval_every == 0:
            total, tokens = 0.0, 0
            for b in eval_batches:
                s, n = tr.evaluate(b)
                total, tokens = total + s, tokens + n
            if tr.rank == 0:
                print(f"step {i} eval loss {total / tokens:.4f} ppl {math.exp(total / tokens):.2f} ({tokens} tokens)")
    if tr.rank == 0:
        dt = time.time() - t0
        print(f"Train loop took {dt:.2f} s  ({a.train_steps * a.batch * world * cfg.n_ctx / dt:.0f} tokens/s incl. planning + warm-up); "
              f"plan: {tr.plan_info.get('parallelism', 'single')}")
    os._exit(0)


if __name__ == "__main__":
    main()
