"""GPU numerics of the flash-attention kernels at 64-wide heads (the GPT-2 345M head width), element by element against an
fp64 autograd reference: the 345M shape with q / k / v as views of one fused [B, S, H, 3, D] buffer (as the executor passes
them), a single tile, a long causal row, a non-causal shape with an odd head count, the GPT-MoE shape with 48-wide heads
(16 x 48 = 768, zero-padded onto the D = 64 kernels), and the dqkv_out path.  A second call
must reproduce O, lse, dK and dV bit for bit; dQ is summed over KV blocks with fp32 reduce-adds whose order may differ.
Every case checks that our kernels ran: the launch counter grows and the torch-math attention paths are errors."""
import pytest
import torch

pytestmark = pytest.mark.gpu

D = 64     # (the head width unless a case gives another)


def _kernels_only(monkeypatch):
    from tepdist_b200 import ops
    from tepdist_b200.ops import attention
    ref_fwd = attention._ref_fwd

    def fail(*a, **k):
        raise AssertionError("attention fell back to torch math")

    monkeypatch.setattr(attention, "_ref_fwd", lambda q, *a: fail() if q.is_cuda else ref_fwd(q, *a))
    monkeypatch.setattr(attention, "_warn_torch_math", fail)
    ops.lib()
    return ops


def _inputs(B, S, H, seed, D=D):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.randn(B, S, H, 3, D, device="cuda", generator=g).to(torch.bfloat16)
    do = torch.randn(B, S, H, D, device="cuda", generator=g).to(torch.bfloat16)
    return qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2], do


def _ref(q, k, v, do, causal):
    """fp64 autograd attention on [B, S, H, D] -> (o, lse [B, H, S], dq, dk, dv)."""
    S, D = q.shape[1], q.shape[3]
    qf, kf, vf = (t.double().detach().clone().requires_grad_(True) for t in (q, k, v))
    s = torch.einsum("bqhd,bkhd->bhqk", qf, kf) * D ** -0.5
    if causal:
        s = s.masked_fill(~torch.ones(S, S, dtype=torch.bool, device=q.device).tril(), float("-inf"))
    o = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), vf)
    o.backward(do.double())
    return o.detach(), torch.logsumexp(s, -1).detach(), qf.grad, kf.grad, vf.grad


def _close(got, want, rel, what):
    """Norm-relative error under `rel`, and every element within 4 * rel of the reference's largest magnitude."""
    got = got.double()
    assert torch.isfinite(got).all(), f"{what}: non-finite values"
    err_norm = ((got - want).norm() / (want.norm() + 1e-12)).item()
    assert err_norm < rel, (what, err_norm)
    err = (got - want).abs().max().item()
    assert err <= 4 * rel * want.abs().max().item() + 1e-3, (what, err, want.abs().max().item())


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
    ops = _kernels_only(monkeypatch)
    q, k, v, do = _inputs(B, S, H, seed=S + H, D=D)
    first = _run(ops, q, k, v, do, causal)
    o, lse, dq, dk, dv = first
    o_ref, lse_ref, *g_ref = _ref(q, k, v, do, causal)
    _close(o, o_ref, 2e-2, "o")
    _close(lse, lse_ref, 1e-3, "lse")
    for name, got, want in zip(("dq", "dk", "dv"), (dq, dk, dv), g_ref):
        _close(got, want, 3e-2, name)
    again = _run(ops, q, k, v, do, causal)
    for name, a, b in zip(("o", "lse", "dk", "dv"), first[:2] + first[3:], again[:2] + again[3:]):
        assert torch.equal(a, b), f"{name} differs between two calls"
    # dQ: only the fp32 summation order of the per-block partials may differ
    assert (again[2].float() - dq.float()).abs().max().item() <= 1e-2 * dq.float().abs().max().item()


def test_hd64_dqkv_out_path(monkeypatch):
    ops = _kernels_only(monkeypatch)
    B, S, H = 2, 1024, 4
    q, k, v, do = _inputs(B, S, H, seed=7)
    part = torch.full((B, S, H, 3, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    o, lse, dq, dk, dv = _run(ops, q, k, v, do, True, dqkv_out=part)
    assert torch.equal(part[:, :, :, 0], dq) and torch.equal(part[:, :, :, 1], dk) and torch.equal(part[:, :, :, 2], dv)
    _, _, *g_ref = _ref(q, k, v, do, True)
    for name, got, want in zip(("dq", "dk", "dv"), (dq, dk, dv), g_ref):
        _close(got, want, 3e-2, name)
