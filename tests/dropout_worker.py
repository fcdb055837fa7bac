"""Worker for the dropout plan-invariance tests: python tests/dropout_worker.py <case[+case..]> <out.pt> under torchrun env.
A case is a strategy, optionally with "/attn" (attention dropout only; default: embedding, attention and residual dropout);
`run("auto")` in a plain process is the single-process reference.  GPT-2 tiny, SGD (so a step's parameter change is -lr
times its gradient): the losses of three steps, every variable's gradient of the third step as whole (unsharded) tensors,
and how the plan split each attention node (tag and qkv input shape)."""
import dataclasses
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

LR = 0.1
STEPS = 3


def model(which: str = "all"):
    from tepdist_b200.models.gpt2 import CONFIGS
    if which == "attn":
        return dataclasses.replace(CONFIGS["tiny"], attn_pdrop=0.15)
    return dataclasses.replace(CONFIGS["tiny"], embd_pdrop=0.1, attn_pdrop=0.15, resid_pdrop=0.2)


def feeds(cfg, batch=4):
    g = torch.Generator().manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (batch, cfg.n_ctx), generator=g, dtype=torch.int32)
    return {"tokens": tok, "labels": torch.roll(tok, -1, 1)}


def run(case: str):
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import build_gpt2_graph
    strategy, _, which = case.partition("/")
    if strategy.startswith(("pp", "dp2")) and int(os.environ.get("WORLD_SIZE", "1")) == 1:
        strategy = "auto"
    cfg = model(which or "all")
    tr = Trainer(build_gpt2_graph(cfg, batch=4, optimizer="sgd", lr=LR), strategy=strategy, device=torch.device("cpu"),
                 use_cuda_graph=False, seed=3)
    f = feeds(cfg)
    losses = [tr.step(f) for _ in range(STEPS - 1)]
    before = {k: v.double().clone() for k, v in tr.full_state_dict().items()}
    losses.append(tr.step(f))
    after = tr.full_state_dict()
    grads = {k: (before[k] - after[k].double()) / LR for k in before}
    worker = getattr(tr.exec, "worker", None)
    replayed = worker.graph_stats["replayed"] if worker is not None else None
    g = tr.executor().g
    attn = [(n.op, int(n.attrs["heads"]), tuple(g.type_of(n.inputs[0 if n.op == "attention" else 1]).shape))
            for n in g.nodes if n.op in ("attention", "attention_bwd")]
    return {"losses": losses, "grads": grads, "parallelism": tr.plan_info.get("parallelism"), "replayed": replayed,
            "attention": attn}


def run_pipeline_one_gpu(graphed: bool):
    """One process, one GPU: a one-stage pipeline of two micro-batches (pp1m2 built directly, as a pipeline rank would) for
    four steps.  With `graphed` the stage bodies are captured in CUDA graphs from step 2 on; the schedule keeps one slot in
    flight, so micro-batch 1 replays the bodies captured for micro-batch 0.  -> losses and the slot statistics."""
    import socket
    import types
    from tepdist_b200.models.gpt2 import build_gpt2_graph
    from tepdist_b200.parallel import build_pipeline
    if not dist.is_initialized():
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
        s.close()
        dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    dev = torch.device("cuda", 0)
    cfg = model()
    tr = types.SimpleNamespace(world=1, rank=0, device=dev, plan_info={}, mesh=None)
    runner = build_pipeline(build_gpt2_graph(cfg, batch=4), tr, 1, 2, "nccl", 3, use_cuda_graph=graphed)
    f = {k: v.to(dev) for k, v in feeds(cfg).items()}
    losses = [float(runner.step(f)[0]) for _ in range(4)]
    w = runner.worker
    return {"losses": losses, "graph_stats": dict(w.graph_stats), "slots": w.num_slots, "use_graph": w.use_graph,
            "parallelism": tr.plan_info.get("parallelism")}


if __name__ == "__main__":
    if sys.argv[1] == "--pp1":
        res = {g: run_pipeline_one_gpu(g) for g in (False, True)}
        torch.save(res, sys.argv[2])
        sys.stdout.flush()
        os._exit(0)
    cases, out = sys.argv[1], sys.argv[2]
    res = {c: run(c) for c in cases.split("+")}
    if int(os.environ.get("RANK", "0")) == 0:
        torch.save(res, out)
    if dist.is_initialized():
        dist.barrier()
        sys.stdout.flush()
        sys.stderr.flush()
        os._exit(0)   # (like dist_worker.py: leave without tearing down the gloo groups)
