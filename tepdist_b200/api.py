"""Public user-facing API.

    import tepdist_b200 as td
    graph   = td.models.gpt2.build_gpt2_graph(cfg)          # or td.frontend.trace(module, ...)
    trainer = td.Trainer(graph, strategy="auto")             # plans + builds the runtime on this rank
    loss    = trainer.step({"tokens": tok_cpu, "labels": lab_cpu})

`Trainer` is what a reference user's `session.run(train_op)` becomes: the first call plans and compiles,
later calls execute the cached plan (reference: XlaRunOp -> BuildExecutionPlan / ExecutePlan, SURVEY §3.2-3.3).
Launch with torchrun (one process per GPU); single-process works for 1 GPU / CPU.
"""
from __future__ import annotations

import os
from typing import Any, Dict, Optional, Tuple

import torch
import torch.distributed as dist

from .ir import Graph
from .runtime.executor import Executor


def init_distributed(backend: Optional[str] = None) -> Dict[str, int]:
    """Rendezvous from torchrun env (RANK/LOCAL_RANK/WORLD_SIZE/MASTER_*); idempotent."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
            dist.init_process_group(backend, device_id=torch.device("cuda", local))
        else:
            dist.init_process_group(backend)
    elif torch.cuda.is_available():
        torch.cuda.set_device(local)
    return {"rank": rank, "world": world, "local_rank": local}


class Trainer:
    def __init__(self, graph: Graph, strategy: str = "auto", device: Optional[torch.device] = None,
                 use_cuda_graph: bool = True, seed: int = 0, comm_mode: Optional[str] = None):
        self.ctx = init_distributed()
        self.world, self.rank = self.ctx["world"], self.ctx["rank"]
        if device is None:
            device = torch.device("cuda", self.ctx["local_rank"]) if torch.cuda.is_available() else torch.device("cpu")
        self.device = device
        from . import config
        comm_mode = config.comm_mode(comm_mode)
        self.strategy = strategy
        self._fake_input = config.fake_input()   # FAKE_INPUT: cache the first step's inputs and reuse them
        self._fake_feeds: Optional[Dict[str, torch.Tensor]] = None
        grad_sync = None
        self.plan_info: Dict[str, Any] = {"strategy": strategy, "world": self.world}
        from .parallel import check_context_parallel
        check_context_parallel(graph, config.resolve_strategy(strategy))
        from .planner import liveness_optimize
        graph, copies = liveness_optimize(graph)    # per-user copies of large convert(variable) results (B6)
        if copies:
            self.plan_info["liveness_copies"] = copies
        if self.world > 1:
            from .parallel import plan_and_build
            self.exec = plan_and_build(graph, self, strategy, comm_mode, use_cuda_graph, seed)
        else:
            self.exec = Executor(graph, device, seed=seed, grad_sync=grad_sync, use_cuda_graph=use_cuda_graph)
        self._pinned: Dict[str, torch.Tensor] = {}
        self._loss_host = torch.zeros(1, dtype=torch.float32).pin_memory() if device.type == "cuda" else None

    def step(self, feeds: Dict[str, torch.Tensor]) -> float:
        """One training step on this rank's shard of the batch; returns the (local) loss as a python float.
        Host tensors are copied to the device (async from pinned memory); the loss is read back."""
        if self._fake_input and self._fake_feeds is not None:
            dev_feeds = self._fake_feeds
        else:
            dev_feeds = {}
            for k, t in feeds.items():
                dev_feeds[k] = t if t.device == self.device else t.to(self.device, non_blocking=True)
            if self._fake_input:
                self._fake_feeds = dev_feeds
        out = self.exec.step(dev_feeds)
        loss = out[0]
        if self._loss_host is not None:
            self._loss_host.copy_(loss.reshape(1), non_blocking=True)
            torch.cuda.current_stream().synchronize()
            return float(self._loss_host[0])
        return float(loss)

    def step_async(self, dev_feeds: Dict[str, torch.Tensor]) -> torch.Tensor:
        """Device-resident variant (no host sync): returns the loss tensor."""
        return self.exec.step(dev_feeds)[0]

    def evaluate(self, feeds: Dict[str, torch.Tensor]) -> Tuple[float, int]:
        """Validation loss of one batch: dropout off, forward only, nothing of the training state changes.  Returns
        (loss_sum, tokens) over the GLOBAL batch, the same on every rank; labels < 0 are ignored (padding), so
        loss_sum / tokens is the mean over the real tokens and exp of it the perplexity.  Raises ValueError if a label is
        >= the vocabulary size.  Host tensors are copied to the device as in `step` (never from the FAKE_INPUT cache)."""
        dev_feeds = {k: t if t.device == self.device else t.to(self.device, non_blocking=True) for k, t in feeds.items()}
        s, n, bad = (float(x) for x in self.evaluate_async(dev_feeds).cpu())
        if bad:
            raise ValueError(f"evaluate: {int(bad)} label(s) >= the vocabulary size")
        return s, int(n)

    def evaluate_async(self, dev_feeds: Dict[str, torch.Tensor]) -> torch.Tensor:
        """Device-resident variant of `evaluate` (no host sync): fp64 [3] = (loss_sum, tokens, labels >= vocab).  A tensor of
        its own (a copy of the captured evaluation's output buffer, which the next evaluation overwrites), so triples of
        several batches can be summed without a sync."""
        return self.exec.evaluate(dev_feeds).clone()

    def executor(self):
        """The Executor that owns this rank's variables: the whole (sharded) step graph, or -- under a pipeline plan -- this
        rank's stage."""
        w = getattr(self.exec, "worker", None)
        return w.exec if w is not None else self.exec

    def set_lr_schedule(self, fn) -> None:
        """`fn(step) -> lr` for the 1-based optimizer step (see utils/schedules.py); None = the graph's constant rate."""
        self.executor().set_lr_schedule(fn)

    def full_state_dict(self, moments: bool = False, dst: int = 0):
        """WHOLE variables by name, whatever the plan did to them (ZeRO chunks, tensor-parallel shards, pipeline stages): every
        rank contributes what it stores, rank `dst` assembles (coverage-checked) and returns the dict, the others return {}.
        Collective: every rank must call it.  Meant for fetching / inspection (everything travels through host memory)."""
        import torch.distributed as dist
        ex = self.executor()
        if hasattr(ex, "materialize_full_state"):
            ex.materialize_full_state()
        st, g = ex.store, ex.g
        sd = st.state_dict()
        mine = {}
        for pid in st.order:
            n, name = g.nodes[pid], st.names[pid]
            meta = (list(n.attrs.get("full_shape", st.shape[pid])), list(n.attrs.get("shard_dims", [])), list(n.attrs.get("shard_nums", [])),
                    [int(ex.coords.get(int(l), 0)) for l in n.attrs.get("shard_levels", [])])
            keys = [name] + ([name + "/m", name + "/v"] if moments else [])
            for k in keys:
                if k in sd and tuple(sd[k].shape) == tuple(st.shape[pid]):
                    mine[k] = (meta, sd[k].detach().cpu())
        if moments:      # optimizer slots the execution keeps outside the flat buffers, with their own shard description
            for n in st._state_nodes:
                if st.slot_is_live(n):
                    t = st.state[n.id]
                    mine[n.name] = ((list(n.attrs.get("full_shape", t.shape)), list(n.attrs.get("shard_dims", [])),
                                     list(n.attrs.get("shard_nums", [])),
                                     [int(ex.coords.get(int(l), 0)) for l in n.attrs.get("shard_levels", [])]), t.detach().cpu())
        if self.world == 1:
            return {k: t for k, (_, t) in mine.items()}
        parts = [None] * self.world if self.rank == dst else None
        dist.gather_object(mine, parts, dst=dst)
        if self.rank != dst:
            return {}
        out, covered = {}, {}
        for part in parts:
            for k, ((full_shape, dims, nums, idx), t) in part.items():
                if k not in out:
                    out[k] = torch.zeros(full_shape, dtype=t.dtype)
                    covered[k] = torch.zeros(full_shape, dtype=torch.bool)
                view, cview = out[k], covered[k]
                for d_, n_, i_ in zip(dims, nums, idx):
                    sz = view.shape[d_] // n_
                    view, cview = view.narrow(d_, i_ * sz, sz), cview.narrow(d_, i_ * sz, sz)
                view.copy_(t.reshape(view.shape))
                cview.fill_(True)
        bad = [k for k, c in covered.items() if not bool(c.all())]
        if bad:
            raise RuntimeError(f"full_state_dict: incomplete variables {bad[:4]}")
        return out

    def state_dict(self):
        """Master weights (+ optimizer moments).  Collective under sharded-optimizer plans: every rank must call it."""
        ex = self.executor()
        if hasattr(ex, "materialize_full_state"):
            ex.materialize_full_state()
        return ex.store.state_dict()

    # ------------------------------------------------------------------ sharded checkpoints (reference DoRemoteSave / Restore)
    def _ckpt(self, root: str, max_to_keep: int = 5):
        from .ckpt import CheckpointManager
        key = (os.path.abspath(root), max_to_keep)
        if getattr(self, "_ckpt_mgr", None) is None or self._ckpt_key != key:
            self._ckpt_mgr, self._ckpt_key = CheckpointManager(root, self.rank, self.world, max_to_keep), key
        return self._ckpt_mgr

    def save(self, root: str, global_step: int, max_to_keep: int = 5) -> str:
        """Every rank writes its own shards (master weights + optimizer moments) under root/ckpt_<rank>_of_<world>/."""
        return self._ckpt(root, max_to_keep).save(self.executor(), global_step)

    def restore(self, root: str, global_step: Optional[int] = None) -> int:
        """Load this rank's shards of `global_step` (default: the latest kept step); returns the restored step."""
        return self._ckpt(root).restore(self.executor(), global_step)
