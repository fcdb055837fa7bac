"""Fused attention op wrappers (kernels in csrc/attention_sm90.cu).

Tensors use the "bshd" convention: q/k/v are views [B, S, H, D] (arbitrary batch/seq/head strides, D
contiguous) — typically slices of the fused qkv projection output [B, S, H, 3, D] (heads-major); the output is a
contiguous [B, S, H, D] tensor, i.e. already the [tokens, hidden] input of the output projection.

On CUDA tensors the wgmma kernels cover head widths 64 and 128 with S % 128 == 0; narrower heads and a ragged causal
sequence length are zero-padded onto them (see `_can_pad`).  The remaining shapes (D > 128, non-causal ragged S) run
plain torch math, which materialises [B, H, S, S] fp32 scores, and warn once per shape.
"""
from __future__ import annotations

import math

import torch

_KERNEL_WIDTHS = (64, 128)   # head dims of the wgmma kernels (attention_sm90.cu)


def _kernel_width(D: int) -> int | None:
    """The kernel head width a D-wide head runs on (zero-padded up to it), or None when no kernel is wide enough."""
    return next((w for w in _KERNEL_WIDTHS if D <= w), None)


def _can_pad(S: int, D: int, causal: bool) -> bool:
    """Shapes that run on the D = 64 / 128, S % 128 == 0 kernels through zero padding, exactly:
       * narrower heads (D <= 64 -> 64, 64 < D <= 128 -> 128): padded q.k terms are zero, padded V / O columns are
         dropped;
       * a ragged sequence length under a CAUSAL mask: padded keys sit after every real query (masked), padded query rows
         are dropped, and their zero dO makes their contribution to dK / dV vanish."""
    return _kernel_width(D) is not None and (S % 128 == 0 or causal)


def _pad_sd(t: torch.Tensor, S: int, D: int, W: int) -> torch.Tensor:
    """[B, S, H, D] -> zero-padded contiguous [B, ceil128(S), H, W]."""
    Sp = (S + 127) // 128 * 128
    return torch.nn.functional.pad(t, (0, W - D, 0, 0, 0, Sp - S))


def _warn_torch_math(S: int, D: int, causal: bool) -> None:
    from . import _warn_once
    _warn_once(f"attention: no kernel for head dim {D}, seq {S}, causal={causal}; running torch math with "
               f"[B, H, {S}, {S}] fp32 scores")


def _ref_fwd(q, k, v, scale, causal):
    # q,k,v: [B,S,H,D] -> fp32 math in [B,H,S,D]
    qf, kf, vf = (t.float().permute(0, 2, 1, 3) for t in (q, k, v))
    s = torch.matmul(qf, kf.transpose(-1, -2)) * scale
    if causal:
        S = q.shape[1]
        mask = torch.ones(S, S, dtype=torch.bool, device=q.device).tril()
        s = s.masked_fill(~mask, float("-inf"))
    lse = torch.logsumexp(s, -1)  # [B,H,S]
    p = torch.exp(s - lse.unsqueeze(-1))
    o = torch.matmul(p, vf).permute(0, 2, 1, 3).contiguous()
    return o.to(q.dtype), lse, p


def attention_fwd(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float | None = None,
                  causal: bool = True):
    """Returns (o [B,S,H,D], lse [B,H,S])."""
    B, S, H, D = q.shape
    if scale is None:
        scale = 1.0 / math.sqrt(D)
    if not q.is_cuda:
        o, lse, _ = _ref_fwd(q, k, v, scale, causal)
        return o, lse
    if D not in _KERNEL_WIDTHS or S % 128:
        if _can_pad(S, D, causal):
            W = _kernel_width(D)
            qp, kp, vp = (_pad_sd(t, S, D, W) for t in (q, k, v))
            o, lse = attention_fwd(qp, kp, vp, scale, causal)
            return o[:, :S, :, :D].contiguous(), lse[:, :, :S].contiguous()
        _warn_torch_math(S, D, causal)
        o, lse, _ = _ref_fwd(q, k, v, scale, causal)   # shapes the wgmma kernels do not cover: plain torch math
        return o, lse
    from . import lib, _check, _count, _stream
    assert q.dtype == torch.bfloat16 and q.stride(3) == 1
    assert q.stride() == k.stride() == v.stride(), "q/k/v must share strides (slices of one qkv buffer)"
    o = torch.empty(B, S, H, D, dtype=q.dtype, device=q.device)
    lse = torch.empty(B, H, S, dtype=torch.float32, device=q.device)
    _check(lib().tepd_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(), B, H, S, D,
                               float(scale), int(causal), q.stride(0), q.stride(1), q.stride(2), _stream()),
           "attn_fwd")
    _count()
    return o, lse


def attention_bwd(do: torch.Tensor, q, k, v, o, lse, scale: float | None = None, causal: bool = True,
                  dqkv_out: torch.Tensor | None = None):
    """Returns (dq, dk, dv) as [B,S,H,D] views (of ``dqkv_out`` [B,S,H,3,D] when given)."""
    B, S, H, D = q.shape
    if scale is None:
        scale = 1.0 / math.sqrt(D)
    if dqkv_out is None:
        dqkv_out = torch.empty(B, S, H, 3, D, dtype=q.dtype, device=q.device)
    dq, dk, dv = dqkv_out[:, :, :, 0], dqkv_out[:, :, :, 1], dqkv_out[:, :, :, 2]
    if q.is_cuda and (D not in _KERNEL_WIDTHS or S % 128) and _can_pad(S, D, causal):
        Sp = (S + 127) // 128 * 128
        W = _kernel_width(D)
        lse_p = lse if Sp == S else torch.nn.functional.pad(lse, (0, Sp - S))
        gq, gk, gv = attention_bwd(*(_pad_sd(t, S, D, W) for t in (do, q, k, v, o)), lse_p, scale, causal)
        dq.copy_(gq[:, :S, :, :D]); dk.copy_(gk[:, :S, :, :D]); dv.copy_(gv[:, :S, :, :D])
        return dq, dk, dv
    if not q.is_cuda or D not in _KERNEL_WIDTHS or S % 128:
        if q.is_cuda:
            _warn_torch_math(S, D, causal)
        dof = do.float().permute(0, 2, 1, 3)
        qf, kf, vf = (t.float().permute(0, 2, 1, 3) for t in (q, k, v))
        # probabilities from the GIVEN log-sum-exp (like the kernels): a block of a longer key sequence (ring attention) passes
        # the log-sum-exp over ALL keys, and its probabilities must not be re-normalised over the block
        sc = torch.matmul(qf, kf.transpose(-1, -2)) * scale
        if causal:
            mask = torch.ones(S, S, dtype=torch.bool, device=q.device).tril()
            sc = sc.masked_fill(~mask, float("-inf"))
        p = torch.exp(sc - lse.float().unsqueeze(-1))
        dvf = torch.matmul(p.transpose(-1, -2), dof)
        dp = torch.matmul(dof, vf.transpose(-1, -2))
        delta = (dof * o.float().permute(0, 2, 1, 3)).sum(-1, keepdim=True)
        ds = p * (dp - delta) * scale
        dqf = torch.matmul(ds, kf)
        dkf = torch.matmul(ds.transpose(-1, -2), qf)
        dq.copy_(dqf.permute(0, 2, 1, 3).to(q.dtype))
        dk.copy_(dkf.permute(0, 2, 1, 3).to(q.dtype))
        dv.copy_(dvf.permute(0, 2, 1, 3).to(q.dtype))
        return dq, dk, dv
    from . import lib, _check, _count, _stream
    do = do.contiguous()
    assert o.is_contiguous() and do.is_contiguous()
    # dq accumulator: persistent self-clearing fp32 workspace inside the library (no per-call memset)
    _check(lib().tepd_attn_bwd(do.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                               None, dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B, H, S, D,
                               float(scale), int(causal), q.stride(0), q.stride(1), q.stride(2),
                               dq.stride(0), dq.stride(1), dq.stride(2), _stream()), "attn_bwd")
    _count(3)
    return dq, dk, dv


# --------------------------------------------------------------------------------------------- ring (context-parallel) helpers
def _native_ring(*ts: torch.Tensor) -> bool:
    return all(t.is_cuda and t.is_contiguous() for t in ts) and ts[0].shape[-1] % 8 == 0


def attn_merge_(o_acc: torch.Tensor, lse_acc: torch.Tensor, lse_out: torch.Tensor, o_j: torch.Tensor, lse_j: torch.Tensor,
                first: bool) -> torch.Tensor:
    """Log-sum-exp merge of one block's partial attention (o_j [B,L,H,D], lse_j [B,H,L]) into the running fp32 pair
    (o_acc in place; the merged log-sum-exp goes to `lse_out`, which is returned).  One kernel (elementwise_sm90.cu
    attn_merge_kernel); plain torch math on CPU."""
    B, L, H, D = o_j.shape
    if o_j.dtype == torch.bfloat16 and _native_ring(o_j, o_acc, lse_acc, lse_out, lse_j):
        from . import lib, _check, _count, _stream
        _check(lib().tepd_attn_merge(o_acc.data_ptr(), lse_acc.data_ptr(), lse_out.data_ptr(), o_j.data_ptr(), lse_j.data_ptr(),
                                     B, L, H, D, int(first), _stream()), "attn_merge")
        _count()
        return lse_out
    if first:
        o_acc.copy_(o_j)
        lse_out.copy_(lse_j)
        return lse_out
    new = torch.logaddexp(lse_acc, lse_j)
    wa = torch.exp(lse_acc - new).permute(0, 2, 1).unsqueeze(-1)     # [B,L,H,1]
    wj = torch.exp(lse_j - new).permute(0, 2, 1).unsqueeze(-1)
    o_acc.mul_(wa).add_(o_j.float() * wj)
    lse_out.copy_(new)
    return lse_out


def attn_ring_accum_(dq_acc: torch.Tensor, kv_acc: torch.Tensor, part: torch.Tensor) -> None:
    """dq_acc [B,L,H,D] += part[..,0,:]; kv_acc [B,L,H,2,D] += part[..,1:,:] (part [B,L,H,3,D]: one block's dq / dk / dv)."""
    if part.dtype == torch.bfloat16 and _native_ring(part, dq_acc, kv_acc):
        from . import lib, _check, _count, _stream
        _check(lib().tepd_attn_ring_accum(dq_acc.data_ptr(), kv_acc.data_ptr(), part.data_ptr(), dq_acc.numel() // dq_acc.shape[-1],
                                          dq_acc.shape[-1], 0, _stream()), "attn_ring_accum")
        _count()
        return
    dq_acc += part[:, :, :, 0]
    kv_acc += part[:, :, :, 1:]


def attn_ring_pack(dq_acc: torch.Tensor, kv_acc: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out [B,L,H,3,D] (compute dtype) <- the fp32 accumulators at the end of the ring."""
    if out.dtype == torch.bfloat16 and _native_ring(out, dq_acc, kv_acc):
        from . import lib, _check, _count, _stream
        _check(lib().tepd_attn_ring_accum(dq_acc.data_ptr(), kv_acc.data_ptr(), out.data_ptr(), dq_acc.numel() // dq_acc.shape[-1],
                                          dq_acc.shape[-1], 1, _stream()), "attn_ring_pack")
        _count()
        return out
    out[:, :, :, 0].copy_(dq_acc)
    out[:, :, :, 1:].copy_(kv_acc)
    return out
