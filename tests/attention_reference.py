"""The fp64 reference of the flash-attention kernels (ops/csrc/attention_sm90.cu), with a bound on every output element.

Imported by the attention tests, as kernel_checks.py is.  `reference` computes attention and its backward by explicit formulas
in fp64 on the inputs' device; `check` asserts |got - ref| <= bound element by element.

The bound of an element is the sum of the errors of the roundings the kernels make on its way, each at its worst case.
u = 2^-8 is the unit roundoff of bf16 (8 significant bits, round to nearest even: one rounding moves x by at most u |x|).
P are the probabilities, Z the scaled dropout keep mask (1 without dropout), n the number of keys, all products elementwise
unless written as matrix products, and |.| taken elementwise:

    O      (u + n 2^-24) (P Z) |V|        P rounded to bf16 for the P V MMA, fp32 accumulation over the keys
           + u |O|                        the final bf16 rounding of O
    dV     (u + n 2^-24) (P Z)^T |dO|     P Z rounded to bf16 for the P^T dO MMA
           + u |dV|
    e_delta  u sum_d |dO| |O|             delta = rowsum(dO O) is formed from the kernels' own bf16 O: its final rounding, and
                                          its P roundings, a sum of random signs of about the size of u |O| (their worst
                                          case u (P Z)|V| is sqrt(n) times too large to be useful)
    e_S    (1 + u) P e_delta + u |dS|     dS = P (dP Z - delta) carries P e_delta and is rounded to bf16 for the dQ / dK MMAs
    dQ     scale (e_S + n 2^-24 |dS|) |K|  + u |dQ|
    dK     scale (e_S + n 2^-24 |dS|)^T |Q| + u |dK|
    lse    2^-24 D scale sum_k P (|q| . |k|)   the fp32 score error of a D-term dot product, weighted by the probabilities
           + 2^-22 (4 + |lse|)                ex2 / lg2 approximations, the fp32 sum of the probabilities, the base change

A context-parallel ring (``blocks`` > 1) merges the bf16 outputs of up to ``blocks`` key blocks in fp32 and sums their bf16
dQ / dK / dV partials in fp32, which rounds every block result once more: O gains u (P Z)|V| (the merge weights w_j of the
block outputs o_j satisfy sum_j w_j |o_j| <= (P Z)|V|), dV u (P Z)^T|dO|, dQ / dK u scale |dS| |K| / |dS|^T |Q|, and lse
(blocks - 1) (2^-20 + 2^-23 |lse|) for the __expf / __logf of each log-sum-exp merge.

Every bound is C = 2 times the sum of its terms.  The worst elements of the CPU emulation of the kernels' roundings
(tests/test_attention_reference_cpu.py) reach 0.13 - 0.39 of the O, dQ, dK and dV bounds; those of the kernels on an H100
(80 GB HBM3, 700 W power limit) reached 0.14 - 0.47.  The lse bound is the loosest: its worst elements reached 0.02 - 0.08
on the H100, because the score term counts all D roundings of a dot product at their worst, where their signs are random.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np
import torch

U = 2.0 ** -8      # bf16 unit roundoff
C = 2.0            # safety factor over the summed worst-case terms (module docstring)


def kernels_only(monkeypatch):
    """The kernel layer, with the torch-math attention paths on CUDA tensors turned into errors (CPU tensors keep them)."""
    from tepdist_b200 import ops
    from tepdist_b200.ops import attention
    ref_fwd = attention._ref_fwd

    def fail(*a, **k):
        raise AssertionError("attention fell back to torch math instead of our kernel")

    monkeypatch.setattr(attention, "_ref_fwd", lambda q, *a, **k: fail() if q.is_cuda else ref_fwd(q, *a, **k))
    monkeypatch.setattr(attention, "_warn_torch_math", fail)
    ops.lib()
    return ops


def visible(S: int, causal: bool, doc_start: torch.Tensor | None, device) -> torch.Tensor:
    """bool [B or 1, 1, S (query), S (key)]: the (query, key) pairs attention sees."""
    vis = torch.ones(1, 1, S, S, dtype=torch.bool, device=device)
    if causal:
        vis = vis.tril()
    if doc_start is not None:
        keys = torch.arange(S, device=device)
        vis = vis & (keys.view(1, 1, 1, S) >= doc_start.to(device).long().view(-1, 1, S, 1))
    return vis


@dataclass
class Reference:
    """fp64 attention: o, dq, dk, dv [B, S, H, D] and lse [B, H, S], the intermediates p, dp [B, H, S (query), S (key)] and
    delta [B, H, S], and the bound of every output element (``bound[name]``, shaped like the output)."""
    o: torch.Tensor
    lse: torch.Tensor
    dq: torch.Tensor
    dk: torch.Tensor
    dv: torch.Tensor
    p: torch.Tensor
    dp: torch.Tensor
    delta: torch.Tensor
    bound: dict = field(default_factory=dict)

    def check(self, **got) -> dict:
        """check() every output given by name (o=, lse=, dq=, dk=, dv=); returns {name: worst error / bound}."""
        return {name: check(t, getattr(self, name), self.bound[name], name) for name, t in got.items()}


def reference(q, k, v, do, causal: bool = True, doc_start=None, z=None, scale: float | None = None,
              blocks: int = 1) -> Reference:
    """fp64 attention forward and backward of q, k, v, dO [B, S, H, D] on their device, with the module docstring's bounds.
    ``z``: the scaled dropout keep mask [B, H, S, S] (``keep_mask(..) * _drop_scale(p)``) or None; ``doc_start``: int [B, S]
    (causal only); ``scale`` defaults to 1 / sqrt(D); ``blocks``: the most key blocks a ring merges into one row."""
    B, S, H, D = q.shape
    scale = D ** -0.5 if scale is None else scale
    qf, kf, vf, dof = (t.detach().double().permute(0, 2, 1, 3) for t in (q, k, v, do))    # [B, H, S, D]
    s = (qf @ kf.transpose(-1, -2)) * scale
    s = s.masked_fill(~visible(S, causal, doc_start, q.device), float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse.unsqueeze(-1))
    del s
    pz = p if z is None else p * z.to(p.device, torch.float64)
    o = pz @ vf
    dp = dof @ vf.transpose(-1, -2)
    delta = (dof * o).sum(-1)
    ds = p * ((dp if z is None else dp * z.to(p.device, torch.float64)) - delta.unsqueeze(-1))
    dv = pz.transpose(-1, -2) @ dof
    dq = (ds @ kf) * scale
    dk = (ds.transpose(-1, -2) @ qf) * scale

    acc = U + S * 2.0 ** -24                        # one bf16 operand rounding + fp32 accumulation over n = S keys
    extra = U if blocks > 1 else 0.0                # ring: every block result is rounded to bf16 once more
    pz_abs = pz.abs()
    pv = pz_abs @ vf.abs()
    b_o = acc * pv + U * o.abs()
    e_delta = U * (dof.abs() * o.abs()).sum(-1, keepdim=True)
    ds_abs = ds.abs()
    e_s = (1 + U) * p * e_delta + (U + S * 2.0 ** -24 + extra) * ds_abs
    del ds, ds_abs
    b_q = scale * (e_s @ kf.abs()) + U * dq.abs()
    b_k = scale * (e_s.transpose(-1, -2) @ qf.abs()) + U * dk.abs()
    del e_s
    b_v = (acc + extra) * (pz_abs.transpose(-1, -2) @ dof.abs()) + U * dv.abs()
    b_o = b_o + extra * pv
    del pz_abs, pv
    b_lse = 2.0 ** -24 * D * scale * (qf.abs() * (p @ kf.abs())).sum(-1) + 2.0 ** -22 * (4 + lse.abs())
    if blocks > 1:
        b_lse = b_lse + (blocks - 1) * (2.0 ** -20 + 2.0 ** -23 * lse.abs())

    bshd = lambda t: t.permute(0, 2, 1, 3).contiguous()
    bound = {"o": bshd(b_o), "lse": b_lse, "dq": bshd(b_q), "dk": bshd(b_k), "dv": bshd(b_v)}
    return Reference(bshd(o), lse, bshd(dq), bshd(dk), bshd(dv), p, dp, delta, {n: C * b for n, b in bound.items()})


def check(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, what: str) -> float:
    """Every element of ``got`` finite and within ``bound`` of ``ref``; on failure the worst error / bound and its index
    ((b, s, h, d) for [B, S, H, D] outputs, (b, h, s) for lse).  Returns the worst ratio."""
    got = got.detach().to(ref.device, torch.float64)
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)}, reference {tuple(ref.shape)}"
    bad = ~torch.isfinite(got)
    if bad.any():
        idx = np.unravel_index(int(bad.flatten().nonzero()[0]), tuple(got.shape))
        raise AssertionError(f"{what}: {int(bad.sum())} non-finite elements, the first at {tuple(map(int, idx))}")
    err = (got - ref).abs()
    ratio = torch.where(err == 0, 0.0, err / bound)
    worst = int(ratio.flatten().argmax())
    r = ratio.flatten()[worst].item()
    if not r <= 1.0:
        idx = tuple(map(int, np.unravel_index(worst, tuple(got.shape))))
        raise AssertionError(f"{what}: error / bound {r:.3g} at {idx} (got {got.flatten()[worst].item():.6g}, reference "
                             f"{ref.flatten()[worst].item():.6g}, bound {bound.flatten()[worst].item():.3g}); "
                             f"{int((ratio > 1).sum())} elements over the bound")
    return r
