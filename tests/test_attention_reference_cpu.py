"""The attention reference and its per-element bounds (attention_reference.py) on the CPU: an emulation of the flash kernels'
arithmetic -- fp64 with the kernels' bf16 roundings of P, O, dS and the outputs -- stays within the bounds, and each of a set
of plausible kernel bugs breaks the bound of the output it corrupts."""
import math

import pytest
import torch

import attention_reference as ar


def _bf(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.bfloat16).double()


def _inputs(S, D, B=1, H=2, seed=0):
    g = torch.Generator().manual_seed(seed + S + D)
    return [torch.randn(B, S, H, D, generator=g).to(torch.bfloat16) for _ in range(4)]


def _doc_start(B, S):
    """Documents [0, 50), [50, 177), [177, S) in every row."""
    ds = torch.zeros(B, S, dtype=torch.int32)
    for cut in (50, 177):
        ds[:, cut:] = cut
    return ds


def _keep(B, S, H, D, p=0.1):
    from tepdist_b200 import ops
    from tepdist_b200.ops.attention import _drop_scale, keep_mask
    rng = ops.DropoutRng(5, torch.tensor([3, 0]), 2, global_shape=(B, S, H * D))
    return keep_mask(rng, p, B, H, S, D).double() * _drop_scale(p)


def _emulate(q, k, v, do, causal, doc=None, z=None, scale=None, vis=None, lose_dq=None, lose_dk=None, lse_base2=False):
    """The kernels' arithmetic in fp64 plus their bf16 roundings: the unnormalised probabilities exp(s - max) into the P V MMA,
    the final O, delta from that bf16 O, P Z into the P^T dO MMA, dS into the dQ / dK MMAs, and dQ / dK / dV.  The keyword
    arguments after ``scale`` plant bugs: ``vis`` replaces the visible pairs, ``lose_dq`` / ``lose_dk`` = (query slice, key
    slice) drop one block pair's dS from dQ / dK, ``lse_base2`` stores log2 of the softmax denominator."""
    B, S, H, D = q.shape
    scale = D ** -0.5 if scale is None else scale
    qf, kf, vf, dof = (t.double().permute(0, 2, 1, 3) for t in (q, k, v, do))
    vis = ar.visible(S, causal, doc, q.device) if vis is None else vis
    s = (qf @ kf.transpose(-1, -2) * scale).masked_fill(~vis, float("-inf"))
    m = s.amax(-1, keepdim=True)
    pt = torch.exp(s - m)
    den = pt.sum(-1, keepdim=True)
    lse = (m + torch.log(den)).squeeze(-1)
    keep, dscale = (1.0, 1.0) if z is None else ((z != 0).double(), z.max().item())
    zz = 1.0 if z is None else z
    o = _bf((_bf(pt * keep) @ vf) * dscale / den)
    delta = (dof * o).sum(-1, keepdim=True)
    p = torch.exp(s - lse.unsqueeze(-1))
    dv = _bf(_bf(p * zz).transpose(-1, -2) @ dof)
    ds = _bf(p * ((dof @ vf.transpose(-1, -2)) * zz - delta))
    ds_q, ds_k = ds.clone(), ds.clone()
    for t, lost in ((ds_q, lose_dq), (ds_k, lose_dk)):
        if lost is not None:
            t[:, :, lost[0], lost[1]] = 0
    dq = _bf(ds_q @ kf * scale)
    dk = _bf(ds_k.transpose(-1, -2) @ qf * scale)
    if lse_base2:
        lse = lse / math.log(2)
    bshd = lambda t: t.permute(0, 2, 1, 3).float()
    return {"o": bshd(o), "lse": lse.float(), "dq": bshd(dq), "dk": bshd(dk), "dv": bshd(dv)}


CASES = [   # (S, D, causal, doc, drop)
    (256, 64, True, False, False),
    (384, 64, True, False, False),
    (256, 64, False, False, False),
    (384, 48, True, False, False),
    (256, 48, False, False, False),
    (384, 64, True, True, False),
    (256, 64, True, False, True),
    (384, 48, False, False, True),
]


@pytest.mark.parametrize("S,D,causal,doc,drop", CASES)
def test_emulated_kernel_arithmetic_is_within_the_bounds(S, D, causal, doc, drop):
    """The emulation must pass, and not by a wide margin: a bound 20x above the kernels' worst rounding would let a bug of
    that size through."""
    B, H = 2, 3
    q, k, v, do = _inputs(S, D, B, H)
    ds = _doc_start(B, S) if doc else None
    z = _keep(B, S, H, D) if drop else None
    ref = ar.reference(q, k, v, do, causal, ds, z)
    worst = ref.check(**_emulate(q, k, v, do, causal, ds, z))
    for name in ("o", "dq", "dk", "dv"):
        assert worst[name] > 0.05, (name, worst)


def _mutations(S):
    tril = lambda d: torch.ones(S, S, dtype=torch.bool).tril(d).view(1, 1, S, S)
    key = torch.arange(S)
    return {   # name: (causal, dropout, the _emulate keyword arguments (a function of doc_start / Z), the outputs that must fail)
        "diagonal_one_key_later": (True, False, lambda ds, z: dict(vis=tril(1)), ("o", "lse", "dq", "dk", "dv")),
        "diagonal_one_key_earlier": (True, False, lambda ds, z: dict(vis=tril(-1)), ("o", "lse", "dq", "dk", "dv")),
        "one_key_per_block_dropped": (True, False, lambda ds, z: dict(vis=tril(0) & (key % 128 != 37).view(1, 1, 1, S)),
                                      ("o", "lse", "dq", "dk", "dv")),
        "block_pair_lost_from_dq": (True, False, lambda ds, z: dict(lose_dq=(slice(192, 256), slice(0, 128))), ("dq",)),
        "block_pair_lost_from_dk": (True, False, lambda ds, z: dict(lose_dk=(slice(192, 256), slice(0, 128))), ("dk",)),
        "doc_start_one_later": (True, False, lambda ds, z: dict(doc=torch.where(ds > 0, ds + 1, ds)), ("o", "lse", "dq", "dk", "dv")),
        "doc_start_one_earlier": (True, False, lambda ds, z: dict(doc=torch.where(ds > 0, ds - 1, ds)), ("o", "lse", "dq", "dk", "dv")),
        "scale_of_the_padded_width": (False, False, lambda ds, z: dict(scale=64 ** -0.5), ("o", "lse", "dq", "dk", "dv")),
        "dropout_mask_one_key_later": (False, True, lambda ds, z: dict(z=z.roll(1, -1)), ("o", "dq", "dk", "dv")),
        "dropout_mask_transposed": (False, True, lambda ds, z: dict(z=z.transpose(-1, -2)), ("o", "dq", "dk", "dv")),
        "lse_in_base_2": (False, False, lambda ds, z: dict(lse_base2=True), ("lse",)),
    }


MUTATION_CASES = [(m, S, D) for m in _mutations(256) for S, D in ((256, 64), (384, 48))
                  if not (m == "scale_of_the_padded_width" and D == 64)]   # 1 / sqrt(64) is right at D = 64


@pytest.mark.parametrize("mutation,S,D", MUTATION_CASES)
def test_planted_kernel_bug_breaks_the_bound(mutation, S, D):
    causal, drop, kwargs, broken = _mutations(S)[mutation]
    doc = mutation.startswith("doc_start")
    B, H = 1, 2
    q, k, v, do = _inputs(S, D, B, H, seed=1)
    ds = _doc_start(B, S) if doc else None
    z = _keep(B, S, H, D) if drop else None
    ref = ar.reference(q, k, v, do, causal, ds, z)
    args = dict(doc=ds, z=z)
    args.update(kwargs(ds, z))
    got = _emulate(q, k, v, do, causal, **args)
    for name in broken:
        with pytest.raises(AssertionError, match=f"^{name}: "):
            ar.check(got[name], getattr(ref, name), ref.bound[name], name)
