"""Data-parallel gradient synchronisation over the flat gradient buffer.

Baseline ("reference-semantics") mode issues NCCL all-reduces (the reference's DAPPLEAllReduceThunk,
SURVEY K1, but bucketed as its unregistered DAPPLEAllReduceCombiner intended, B7).  The product path is the
peer-memory reduce-scatter fused with scale (parallel/symm.py + ops/csrc/comm_sm90.cu).
"""
from __future__ import annotations

from typing import Callable, Optional

import torch
import torch.distributed as dist


def make_nccl_grad_sync(group: Optional[dist.ProcessGroup] = None, bucket_elems: int = 64 * 1024 * 1024,
                        average: bool = True) -> Callable[[torch.Tensor], None]:
    world = dist.get_world_size(group)

    def sync(flat: torch.Tensor) -> None:
        if world == 1:
            return
        n = flat.numel()
        works = []
        for off in range(0, n, bucket_elems):
            chunk = flat[off:min(n, off + bucket_elems)]
            works.append(dist.all_reduce(chunk, op=dist.ReduceOp.AVG if (average and flat.is_cuda) else dist.ReduceOp.SUM,
                                         group=group, async_op=True))
        for w in works:
            w.wait()
        if average and not flat.is_cuda:
            flat.div_(world)

    return sync
