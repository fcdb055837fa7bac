"""Worker for the document-masking parity test: python tests/doc_mask_worker.py <strategy> <out.json> under torchrun env.
`run("auto")` in a plain process is the single-process reference."""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

EOT = 999   # (GPT-2 tiny has a 1000-token vocabulary)


def packed_tokens(batch: int, n_ctx: int) -> torch.Tensor:
    """Seeded tokens with end-of-text markers placed so that documents straddle the middle of the row (where a sequence split
    would cut) and the row boundaries the batch shards and micro-batches cut at: no EOT, one EOT just before the middle, EOTs
    on both sides of it, and EOTs at positions 0 / 1 / last."""
    g = torch.Generator().manual_seed(0)
    tok = torch.randint(0, EOT, (batch, n_ctx), generator=g, dtype=torch.int32)
    half = n_ctx // 2
    marks = [[], [half - 1], [half // 2, half + 7, n_ctx - 20], [0, 1, n_ctx - 1]]
    for r in range(batch):
        for p in marks[r % len(marks)]:
            tok[r, p] = EOT
    return tok


def run(strategy: str):
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    cfg = CONFIGS["tiny"]
    if strategy.startswith("pp") and int(os.environ.get("WORLD_SIZE", "1")) == 1:
        strategy = "auto"
    g = build_gpt2_graph(cfg, batch=4, eot_token=EOT, reset_position_ids=True)
    tr = Trainer(g, strategy=strategy, device=torch.device("cpu"), use_cuda_graph=False)
    tok = packed_tokens(4, cfg.n_ctx)
    feeds = {"tokens": tok, "labels": torch.roll(tok, -1, 1)}
    losses = [tr.step(feeds) for _ in range(4)]
    return {"losses": losses, "parallelism": tr.plan_info.get("parallelism")}


if __name__ == "__main__":
    cases, out = sys.argv[1], sys.argv[2]
    res = {c: run(c) for c in cases.split("+")}
    if int(os.environ.get("RANK", "0")) == 0:
        json.dump(res, open(out, "w"))
    if dist.is_initialized():
        dist.barrier()
        sys.stdout.flush()
        sys.stderr.flush()
        os._exit(0)   # (like dist_worker.py: leave without tearing down the gloo groups)
