"""Worker for the evaluation-step tests: python tests/eval_worker.py <case>[+<case>...] <out.json> under torchrun (gloo on CPU, or
NCCL with TEPDIST_TEST_DEVICE=cuda).  Without torchrun the same functions give the single-process result."""
import dataclasses
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _dev():
    if os.environ.get("TEPDIST_TEST_DEVICE") == "cuda":
        return torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    return torch.device("cpu")


def _single(strategy):
    return "auto" if int(os.environ.get("WORLD_SIZE", "1")) == 1 else strategy


def batch(cfg, n=4, ignore=True):
    """Seeded tokens and next-token labels; with `ignore` the last 5 labels of sequence 1 are -1 (a padded tail)."""
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (n, cfg.n_ctx), dtype=torch.int32)
    lab = torch.roll(tok, -1, 1)
    if ignore:
        lab[1, -5:] = -1
    return {"tokens": tok, "labels": lab}


def _same_on_every_rank(x):
    if not dist.is_initialized():
        return True
    xs = [None] * dist.get_world_size()
    dist.all_gather_object(xs, x)
    return all(v == xs[0] for v in xs)


def case_eval(strategy):
    """(loss_sum, tokens) of GPT-2 tiny's freshly initialised weights, then after one training step."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    cfg = CONFIGS["tiny"]
    tr = Trainer(build_gpt2_graph(cfg, batch=4), strategy=_single(strategy), device=_dev(), use_cuda_graph=False)
    feeds = batch(cfg)
    ev = [tr.evaluate(feeds)]
    tr.step(batch(cfg, ignore=False))
    ev.append(tr.evaluate(feeds))
    return {"eval": ev, "same_on_every_rank": _same_on_every_rank(ev), "parallelism": tr.plan_info.get("parallelism")}


def case_interleave(strategy):
    """Training losses of 4 steps of GPT-2 tiny with dropout 0.1, without and with evaluate() after steps 1 and 3."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    cfg = dataclasses.replace(CONFIGS["tiny"], embd_pdrop=0.1, attn_pdrop=0.1, resid_pdrop=0.1)
    out = {}
    for interleave in (False, True):
        tr = Trainer(build_gpt2_graph(cfg, batch=4), strategy=_single(strategy), device=_dev(), use_cuda_graph=False)
        losses = []
        for i in range(4):
            losses.append(tr.step(batch(cfg, ignore=False)))
            if interleave and i in (0, 2):
                tr.evaluate(batch(cfg))
        out["interleaved" if interleave else "plain"] = losses
    return out


def case_refuse(strategy):
    """The error each refused graph raises under `strategy` (None: it did not raise)."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.smoke import build_conv_graph, build_mlp_graph
    out = {}
    for name, g in (("batchnorm", build_conv_graph()), ("not_xent", build_mlp_graph())):
        tr = Trainer(g, strategy=_single(strategy), device=_dev(), use_cuda_graph=False)
        feeds = {n.name: torch.randn(tuple(n.attrs.get("full_shape", n.outputs[0].shape))) for n in g.inputs()}
        try:
            tr.evaluate(feeds)
            out[name] = None
        except ValueError as e:
            out[name] = str(e)
    return out


CASES = {"eval": case_eval, "interleave": case_interleave, "refuse": case_refuse}

if __name__ == "__main__":
    case, out = sys.argv[1], sys.argv[2]
    res = {}
    for c in case.split("+"):
        name, _, strat = c.partition(":")
        res[c] = CASES[name](strat or "auto")
    if int(os.environ.get("RANK", "0")) == 0:
        json.dump(res, open(out, "w"))
    if dist.is_initialized():
        dist.barrier()
        sys.stdout.flush()
        sys.stderr.flush()
        os._exit(0)      # (as tests/dist_worker.py: no gloo group teardown while its threads drain)
