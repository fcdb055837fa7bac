"""Execution of the collective IR ops inserted by the SPMD transform.

"nccl" mode = reference semantics (SURVEY K1-K3: per-tensor NCCL collectives issued in-stream).  The fused
peer-memory kernels (parallel/symm.py) replace the hot ones in "fused" mode.  The collective lowering that the
reference performs as HLO reshape/transpose sandwiches (CustomCollectiveExpander, B2) happens here on views.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.distributed as dist

from .mesh import DeviceMesh

_REDUCE = {0: dist.ReduceOp.SUM, 1: dist.ReduceOp.MAX, 2: dist.ReduceOp.MIN, 3: dist.ReduceOp.PRODUCT}


class CollectiveRunner:
    def __init__(self, mesh: DeviceMesh, comm_dtype: Optional[torch.dtype] = None):
        self.mesh = mesh
        self.comm_dtype = comm_dtype  # FP16_COMM equivalent (bf16)
        self.bytes_moved = 0
        self.dry = False  # timing-only stand-ins (no communication), see Executor.dry_comm

    def _g(self, n):
        return self.mesh.group(int(n.attrs["level"]))

    def _gloo(self, t: torch.Tensor) -> bool:
        return not t.is_cuda

    def gather_input(self, t: torch.Tensor) -> torch.Tensor:
        """Concatenate every rank's batch shard of a fed input along dim 0 (world rank order)."""
        tc = t.contiguous()
        w = self.mesh.world
        if self.dry:
            return tc.repeat((w,) + (1,) * (tc.dim() - 1))
        if self._gloo(tc):
            parts = [torch.empty_like(tc) for _ in range(w)]
            dist.all_gather(parts, tc)
            return torch.cat(parts, 0)
        buf = torch.empty((w * tc.shape[0],) + tuple(tc.shape[1:]), dtype=tc.dtype, device=tc.device)
        dist.all_gather_into_tensor(buf.view(-1), tc.view(-1))
        return buf

    def run(self, n, ins: List[torch.Tensor], out: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
        op, a = n.op, n.attrs
        x = ins[0]
        num = int(a.get("num", 1))
        lvl = int(a["level"])
        if num == 1 or self.mesh.world == 1:
            return [x]
        pg = self._g(n)
        if self.dry and op != "dynamic_slice":
            if op == "all_reduce":
                return [x if out is None else out.copy_(x)]
            if op == "all_gather":
                d = int(a["dim"])
                return [x.repeat(tuple(num if i == d else 1 for i in range(x.dim())))]
            if op == "reduce_scatter":
                d = int(a["dim"])
                y = x.narrow(d, 0, x.shape[d] // num).contiguous()
                return [y if out is None else out.copy_(y.view(out.shape))]
            if op == "all_to_all":
                sd, cd = int(a["split_dim"]), int(a["concat_dim"])
                return [torch.cat(list(x.split(x.shape[sd] // num, dim=sd)), dim=cd)]
        if op == "dynamic_slice":
            d = int(a["dim"])
            sz = x.shape[d] // num
            return [x.narrow(d, self.mesh.index_in_group(lvl) * sz, sz).contiguous()]
        if op == "all_reduce":
            y = x.contiguous().clone() if out is None else out.copy_(x)
            red = _REDUCE[int(a.get("reduce", 0))]
            if self.comm_dtype is not None and y.dtype == torch.float32 and red == dist.ReduceOp.SUM:
                z = y.to(self.comm_dtype)
                dist.all_reduce(z, op=red, group=pg)
                y.copy_(z)
            else:
                dist.all_reduce(y, op=red, group=pg)
            return [y]
        if op == "all_gather":
            d = int(a["dim"])
            xc = x.contiguous()
            buf = torch.empty((num,) + tuple(xc.shape), dtype=xc.dtype, device=xc.device)
            try:
                dist.all_gather_into_tensor(buf.view(-1), xc.view(-1), group=pg)
            except (RuntimeError, NotImplementedError):
                parts = [torch.empty_like(xc) for _ in range(num)]
                dist.all_gather(parts, xc, group=pg)
                buf = torch.stack(parts, 0)
            if d == 0:
                return [buf.reshape((num * xc.shape[0],) + tuple(xc.shape[1:]))]
            return [torch.cat(list(buf.unbind(0)), dim=d)]
        if op == "reduce_scatter":
            d = int(a["dim"])
            red = _REDUCE[int(a.get("reduce", 0))]
            sz = x.shape[d] // num
            if d != 0:
                xs = torch.stack(list(x.split(sz, dim=d)), 0).contiguous()   # [num, ...shard...]
            else:
                xs = x.contiguous().view((num, sz) + tuple(x.shape[1:]))
            shard_shape = tuple(xs.shape[1:])
            y = out if out is not None else torch.empty(shard_shape, dtype=x.dtype, device=x.device)
            if self._gloo(x):
                t = xs.clone()
                dist.all_reduce(t, op=red, group=pg)
                y.copy_(t[self.mesh.index_in_group(lvl)].reshape(y.shape))
            else:
                dist.reduce_scatter_tensor(y.view(-1), xs.view(-1), op=red, group=pg)
            return [y.view(shard_shape) if y.numel() == xs[0].numel() else y]
        if op == "all_to_all":
            sd, cd = int(a["split_dim"]), int(a["concat_dim"])
            sz = x.shape[sd] // num
            send = torch.stack(list(x.split(sz, dim=sd)), 0).contiguous()
            recv = torch.empty_like(send)
            try:
                dist.all_to_all_single(recv.view(-1), send.view(-1), group=pg)
            except (RuntimeError, NotImplementedError):
                gathered = [torch.empty_like(send) for _ in range(num)]
                dist.all_gather(gathered, send, group=pg)
                me = self.mesh.index_in_group(lvl)
                recv = torch.stack([gathered[r][me] for r in range(num)], 0)
            return [torch.cat(list(recv.unbind(0)), dim=cd)]
        raise NotImplementedError(op)
