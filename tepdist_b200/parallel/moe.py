"""Fused expert-parallel MoE FFN forward over peer memory (kernels: ops/csrc/moe_sm90.cu).

    dispatch (quantise to e4m3 + P2P push into the expert owner's buffer)  ->  barrier
    FC1 in fp8 on wgmma (per-token x per-expert scales, GELU fused)      ->  FC2 (bf16 wgmma, batched over local experts)
    barrier  ->  combine (P2P pull of expert outputs, gate-weighted sum)

Routing follows GShard local groups: every source rank owns `capacity` slots per expert, so slot assignment is a purely
local cumsum (reference: examples/gpt_moe/layers/moe_layers.py top-2 gating + einsum dispatch / combine).
"""
from __future__ import annotations

import ctypes
from typing import Optional, Tuple

import torch
import torch.distributed as dist

from .. import ops
from .symm import SymmBarrier, SymmetricBuffer


def _sig(lib):
    vp, i, ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
    pp = ctypes.POINTER(ctypes.c_void_p)
    for name, args in {
        "tepd_moe_dispatch": [vp, vp, pp, pp, i, i, i, i, i, i, i, vp],
        "tepd_moe_combine": [pp, vp, vp, vp, i, i, i, i, i, i, i, vp],
        "tepd_quant_weight_fp8": [vp, vp, vp, ll, ll, vp],
        "tepd_gemm_fp8": [vp, vp, vp, vp, vp, vp, i, i, i, i, i, i, vp],
    }.items():
        fn = getattr(lib, name)
        fn.restype = ctypes.c_int
        fn.argtypes = args


def route_top_k(gates: torch.Tensor, capacity: int, top_k: int = 2) -> Tuple[torch.Tensor, torch.Tensor]:
    """gates [T, E] (probabilities) -> (route [T, K] int32 = expert << 16 | slot or -1 when dropped, gate [T, K] fp32)."""
    T, E = gates.shape
    remaining = gates.float().clone()
    offset = torch.zeros(E, device=gates.device)
    routes, gvals = [], []
    for _ in range(top_k):
        idx = remaining.argmax(-1)
        mask = torch.nn.functional.one_hot(idx, E).float()
        pos = ((mask.cumsum(0) - 1 + offset) * mask).sum(-1).long()
        keep = pos < capacity
        routes.append(torch.where(keep, (idx << 16) | pos, torch.full_like(idx, -1)).int())
        gvals.append(gates.float().gather(1, idx[:, None]).squeeze(1) * keep)
        offset = offset + mask.sum(0)
        remaining = remaining.masked_fill(mask.bool(), float("-inf"))
    return torch.stack(routes, 1).contiguous(), torch.stack(gvals, 1).contiguous()


class FusedMoE:
    def __init__(self, model_dim: int, hidden: int, num_experts: int, capacity: int, w1: torch.Tensor, b1: Optional[torch.Tensor],
                 w2: torch.Tensor, group=None):
        """w1 [E_local, H, M], w2 [E_local, M, H] (bf16): this rank's experts."""
        self.lib = ops.lib()
        _sig(self.lib)
        self.n = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.M, self.H, self.E, self.C = model_dim, hidden, num_experts, capacity
        self.El = num_experts // self.n
        rows = self.El * self.n * capacity
        self.rows = rows
        self.xin = SymmetricBuffer(rows * model_dim, group)          # e4m3 expert inputs
        self.xscale = SymmetricBuffer(rows * 4, group)               # fp32 per-token scales
        self.y = SymmetricBuffer(rows * model_dim * 2, group)        # bf16 expert outputs
        self.barrier = SymmBarrier(group)
        dev = w1.device
        # per-expert weight quantisation
        amax = w1.float().abs().amax(dim=(1, 2)).clamp_min(1e-12)
        self.w_scale = (amax / 448.0).contiguous()
        self.w1q = torch.empty(w1.shape, dtype=torch.uint8, device=dev)
        inv = (1.0 / self.w_scale).contiguous()
        rc = self.lib.tepd_quant_weight_fp8(w1.contiguous().data_ptr(), self.w1q.data_ptr(), inv.data_ptr(), hidden * model_dim, w1.numel(),
                                            torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        self.b1 = None if b1 is None else b1.float().contiguous()
        self.w2 = w2.contiguous()
        self.h = torch.empty(self.El, self.n * capacity, hidden, dtype=torch.bfloat16, device=dev)

    def forward(self, x: torch.Tensor, route: torch.Tensor, gate: torch.Tensor) -> torch.Tensor:
        T, M = x.shape
        K = route.shape[1]
        s = torch.cuda.current_stream().cuda_stream
        lib = self.lib
        self.xin.tensor(torch.uint8).zero_()
        self.xscale.tensor(torch.float32).zero_()
        self.barrier()
        rc = lib.tepd_moe_dispatch(x.data_ptr(), route.data_ptr(), self.xin.ptr_array, self.xscale.ptr_array, T, M, K, self.El, self.C,
                                   self.n, self.rank, s)
        assert rc == 0, rc
        self.barrier()    # every source has pushed its tokens
        rows_per_e = self.n * self.C
        rc = lib.tepd_gemm_fp8(self.xin.local_ptr, self.w1q.data_ptr(), self.h.data_ptr(), self.xscale.local_ptr, self.w_scale.data_ptr(),
                               None if self.b1 is None else self.b1.data_ptr(), rows_per_e, self.H, M, self.El, 1, ops._sms(), s)
        assert rc == 0, rc
        y = self.y.tensor(torch.bfloat16, self.rows * M).view(self.El, rows_per_e, M)
        ops.gemm(self.h, self.w2, out=y)          # FC2: batched bf16 wgmma GEMM over the local experts
        self.barrier()    # every expert output is in place
        out = torch.empty(T, M, dtype=torch.bfloat16, device=x.device)
        rc = lib.tepd_moe_combine(self.y.ptr_array, route.data_ptr(), gate.data_ptr(), out.data_ptr(), T, M, K, self.El, self.C, self.n,
                                  self.rank, s)
        assert rc == 0, rc
        ops._count(4)
        return out
