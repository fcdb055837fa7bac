"""GPU numerics of the flash-attention kernels at 64-wide heads (the GPT-2 345M head width), element by element against the
fp64 reference and its per-element bounds (attention_reference.py): the 345M shape with q / k / v as views of one fused
[B, S, H, 3, D] buffer (as the executor passes them), a single tile, a long causal row, a non-causal shape with an odd head
count, the GPT-MoE shape with 48-wide heads (16 x 48 = 768, zero-padded onto the D = 64 kernels), and the dqkv_out path.  A
second call must reproduce O, lse, dK and dV bit for bit; dQ is summed over KV blocks with fp32 reduce-adds whose order may
differ.  Every case checks that our kernels ran: the launch counter grows and the torch-math attention paths are errors."""
import pytest
import torch

import attention_reference as ar

pytestmark = pytest.mark.gpu

D = 64     # (the head width unless a case gives another)


def _inputs(B, S, H, seed, D=D):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.randn(B, S, H, 3, D, device="cuda", generator=g).to(torch.bfloat16)
    do = torch.randn(B, S, H, D, device="cuda", generator=g).to(torch.bfloat16)
    return qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2], do


def _run(ops, q, k, v, do, causal, dqkv_out=None):
    n0 = ops.launch_count()
    o, lse = ops.attention_fwd(q, k, v, causal=causal)
    dq, dk, dv = ops.attention_bwd(do, q, k, v, o, lse, causal=causal, dqkv_out=dqkv_out)
    torch.cuda.synchronize()
    assert ops.launch_count() >= n0 + 4, "attention kernels did not run"
    return [t.clone() for t in (o, lse, dq, dk, dv)]


CASES = [
    (4, 1024, 16, True, 64),    # GPT-2 345M
    (2, 128, 2, True, 64),
    (1, 4096, 2, True, 64),
    (2, 512, 3, False, 64),
    (2, 1024, 16, True, 48),    # GPT-MoE: 16 heads x 48
]


@pytest.mark.parametrize("B,S,H,causal,D", CASES, ids=["-".join(map(str, c[:4])) + ("" if c[4] == D else f"-D{c[4]}") for c in CASES])
def test_hd64_matches_fp64_reference_and_repeats(B, S, H, causal, D, monkeypatch):
    ops = ar.kernels_only(monkeypatch)
    q, k, v, do = _inputs(B, S, H, seed=S + H, D=D)
    first = _run(ops, q, k, v, do, causal)
    o, lse, dq, dk, dv = first
    ref = ar.reference(q, k, v, do, causal)
    ref.check(o=o, lse=lse, dq=dq, dk=dk, dv=dv)
    again = _run(ops, q, k, v, do, causal)
    for name, a, b in zip(("o", "lse", "dk", "dv"), first[:2] + first[3:], again[:2] + again[3:]):
        assert torch.equal(a, b), f"{name} differs between two calls"
    ref.check(dq=again[2])   # dQ: only the fp32 summation order of the per-block partials may differ


def test_hd64_dqkv_out_path(monkeypatch):
    ops = ar.kernels_only(monkeypatch)
    B, S, H = 2, 1024, 4
    q, k, v, do = _inputs(B, S, H, seed=7)
    part = torch.full((B, S, H, 3, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    o, lse, dq, dk, dv = _run(ops, q, k, v, do, True, dqkv_out=part)
    assert torch.equal(part[:, :, :, 0], dq) and torch.equal(part[:, :, :, 1], dk) and torch.equal(part[:, :, :, 2], dv)
    ar.reference(q, k, v, do, True).check(dq=dq, dk=dk, dv=dv)
