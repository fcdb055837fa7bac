"""Element-by-element numerics of the kernels one GPT-2 training step launches, and every parameter's gradient of whole steps
against the fp32 CPU executor.

Every kernel case checks that our kernel ran (the launch counter grew, no torch fallback warned) and compares each element
with a reference computed in fp64 from the same bf16 / fp32 inputs.  Where the arithmetic is exact (integer-valued GEMM,
embedding and column-sum operands, casts, the bf16 copy of the optimizer) the comparison is bit for bit; elsewhere the
tolerance is derived per element from the output type and the kernel's arithmetic, as stated beside each case.
"""
import math
import os
import re
import subprocess
import sys
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24          # unit roundoff of fp32 (round to nearest)
FTZ = 2.0 ** -125         # the kernels are built with --use_fast_math: fp32 results below 2^-126 flush to zero
TANH_APPROX = 2.0 ** -10.987   # max error of tanh.approx.f32 (PTX ISA), relative to |tanh|, hence absolute as |tanh| <= 1
_GEN = []


def gen():
    """One seeded CUDA generator for the inputs (created on first use: collecting this file needs no GPU)."""
    if not _GEN:
        _GEN.append(torch.Generator(device="cuda"))
    return _GEN[0]


@pytest.fixture
def ops(monkeypatch):
    """The kernel layer, with every torch-fallback warning turned into a failure."""
    from tepdist_b200 import ops as _ops
    _ops.lib()

    def fallback(msg):
        raise AssertionError(f"torch fallback instead of our kernel: {msg}")

    monkeypatch.setattr(_ops, "_warn_once", fallback)
    return _ops


def launched(ops, fn, *args, **kw):
    """Run fn and assert that it launched at least one of our kernels."""
    n0 = ops.launch_count()
    out = fn(*args, **kw)
    assert ops.launch_count() > n0, f"{getattr(fn, '__name__', fn)} launched no kernel"
    return out


def _seed(s):
    gen().manual_seed(s)
    torch.manual_seed(s)


def ints(*shape, lo=-3, hi=3, dtype=torch.bfloat16):
    return torch.randint(lo, hi + 1, shape, device="cuda", generator=gen()).to(dtype)


def randn(*shape, dtype=torch.bfloat16, scale=1.0):
    return (torch.randn(shape, device="cuda", generator=gen()) * scale).to(dtype)


def ulp_bf16(x):
    """One bf16 ulp at |x| (fp64): |x| = m * 2^e with m in [0.5, 1) -> 2^(e - 8); 2^-133 (the subnormal step) at zero."""
    x = x.double().abs()
    _, e = torch.frexp(x)
    u = torch.ldexp(torch.ones_like(x), e - 8)
    return torch.where(x > 0, u, torch.full_like(x, 2.0 ** -133)).clamp_min(2.0 ** -133)


def bf16_tol(ref, err):
    """Bound for a bf16 output whose fp32 value before the store is within `err` of `ref`: the round-to-nearest store adds
    at most half an ulp of that value; one full ulp of |ref| + err covers it with a factor of two."""
    err = torch.as_tensor(err, dtype=torch.float64, device=ref.device)
    return ulp_bf16(ref.double().abs() + err) + err + FTZ


def close(what, got, ref, tol):
    """Element-wise |got - ref| <= tol (NaN fails).  Returns max(|got - ref| / tol) for reporting."""
    g, r = got.double(), ref.double().to(got.device)
    tol = torch.as_tensor(tol, dtype=torch.float64, device=g.device).expand(r.shape)
    err = (g - r).abs()
    bad = ~(err <= tol)
    if bool(bad.any()):
        excess = torch.where(bad, (err - tol).nan_to_num(float("inf")), torch.full_like(err, -1.0))
        i = int(excess.argmax())
        idx = tuple(int(x) for x in torch.unravel_index(torch.tensor(i), g.shape))
        raise AssertionError(f"{what}: {int(bad.sum())} of {g.numel()} elements off; worst at {idx}: kernel "
                             f"{g.flatten()[i].item()!r}, reference {r.flatten()[i].item()!r}, tolerance {tol.flatten()[i].item():.3g}")
    return float((err / tol.clamp_min(1e-300)).max()) if g.numel() else 0.0


def exact(what, got, ref):
    """Bit-exact equality (bf16 by bit pattern; fp32 by value, so the reference may be fp64 holding exact values)."""
    if got.dtype == torch.bfloat16:
        assert ref.dtype == torch.bfloat16
        g, r = got.view(torch.int16), ref.to(got.device).view(torch.int16)
        bad = g != r
        if bool(bad.any()):
            i = int(bad.flatten().nonzero()[0])
            idx = tuple(int(x) for x in torch.unravel_index(torch.tensor(i), g.shape))
            raise AssertionError(f"{what}: {int(bad.sum())} of {g.numel()} bf16 elements differ; first at {idx}: kernel "
                                 f"{got.flatten()[i].item()!r}, reference {ref.flatten()[i].item()!r}")
    else:
        close(what, got, ref, 0.0)


# ============================================================================================== A. GEMM, exact
# Integer operands in [-3, 3], integer bias / residual / starting `out`, alpha in {0.5, 2}: every product and every partial
# sum is an integer or half-integer below 2^24, so the fp32 accumulator of any schedule holds the exact value whatever the
# summation order.  fp32 outputs must equal the fp64 reference; bf16 outputs must equal its round-to-nearest-even cast.

def gemm_operands(M, N, K, a_mn, b_mn, batch=0):
    lead = (batch,) if batch else ()
    A, B = ints(*lead, M, K), ints(*lead, K, N)
    a = A.transpose(-1, -2).contiguous() if a_mn else A
    b = B if b_mn else B.transpose(-1, -2).contiguous()
    return A, B, a, b


def gemm_ref(A, B, alpha=1.0, bias=None, residual=None, out0=None):
    d = alpha * torch.matmul(A.double(), B.double())
    if bias is not None:
        d = d + bias.double()
    if residual is not None:
        d = d + residual.double()
    if out0 is not None:
        d = d + out0.double()
    return d


def check_gemm_out(what, out, ref):
    if out.dtype == torch.float32:
        exact(what, out, ref)
    else:
        exact(what, out, ref.float().to(torch.bfloat16))


LAYOUTS = [(False, False), (False, True), (True, False), (True, True)]


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (129, 136, 72), (1000, 520, 2056)])
def test_gemm_layouts_exact(ops, M, N, K, a_mn, b_mn, block_n):
    if a_mn:
        M = -(-M // 8) * 8       # an MN-major A needs M % 8 == 0
    _seed(1)
    A, B, a, b = gemm_operands(M, N, K, a_mn, b_mn)
    bias, res = ints(N, dtype=torch.float32), ints(M, N)
    d = launched(ops, ops.gemm, a, b, a_mn=a_mn, b_mn=b_mn, bias=bias, residual=res, alpha=2.0, split_k=1, block_n=block_n)
    check_gemm_out("bf16 out, fp32 bias, residual, alpha 2", d, gemm_ref(A, B, 2.0, bias, res))
    d = launched(ops, ops.gemm, a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32, alpha=0.5, split_k=1, block_n=block_n)
    check_gemm_out("fp32 plain store, alpha 0.5", d, gemm_ref(A, B, 0.5))


# GPT-2 345M at 4096 tokens (C = 1024, 4C = 4096, padded vocab 50304): (kind, M, N, K, with bias, with residual)
STEP_SHAPES = [
    ("fwd", 4096, 3072, 1024, True, False), ("fwd", 4096, 1024, 1024, True, True), ("fwd", 4096, 4096, 1024, True, False),
    ("fwd", 4096, 1024, 4096, True, True), ("fwd", 4096, 50304, 1024, False, False),
    ("dgrad", 4096, 1024, 3072, False, False), ("dgrad", 4096, 1024, 1024, False, False),
    ("dgrad", 4096, 4096, 1024, False, False), ("dgrad", 4096, 1024, 4096, False, False),
    ("dgrad", 4096, 1024, 50304, False, False),
    ("wgrad", 3072, 1024, 4096, False, False), ("wgrad", 1024, 1024, 4096, False, False),
    ("wgrad", 4096, 1024, 4096, False, False), ("wgrad", 1024, 4096, 4096, False, False),
    ("wgrad", 50304, 1024, 4096, False, False),
]


@pytest.mark.parametrize("kind,M,N,K,has_bias,has_res", STEP_SHAPES, ids=[f"{s[0]}-{s[1]}x{s[2]}x{s[3]}" for s in STEP_SHAPES])
def test_gemm_step_shapes_exact(ops, kind, M, N, K, has_bias, has_res):
    """The operand layouts and schedules the executor uses for the 345M step (automatic tile / schedule choice)."""
    _seed(2)
    if kind != "wgrad":
        A, B, a, b = gemm_operands(M, N, K, False, kind == "dgrad")
        bias = ints(N, dtype=torch.float32) if has_bias else None
        res = ints(M, N) if has_res else None
        d = launched(ops, ops.gemm, a, b, b_mn=kind == "dgrad", bias=bias, residual=res)
        check_gemm_out(kind, d, gemm_ref(A, B, 1.0, bias, res))
        return
    A, B, a, b = gemm_operands(M, N, K, True, True)
    out = torch.full((M, N), float("nan"), device="cuda")
    launched(ops, ops.gemm, a, b, a_mn=True, b_mn=True, out=out, accumulate=False, split_k=1)
    check_gemm_out("wgrad plain store", out, gemm_ref(A, B))
    out0 = ints(M, N, lo=-100, hi=100, dtype=torch.float32)
    out = out0.clone()
    launched(ops, ops.gemm, a, b, a_mn=True, b_mn=True, out=out, accumulate=True, split_k=0)
    check_gemm_out("wgrad accumulate (split-K / stream-K red.add)", out, gemm_ref(A, B, out0=out0))


@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
@pytest.mark.parametrize("split", [2, 3, 4])
def test_gemm_split_k_exact(ops, split, a_mn, b_mn):
    """Explicit split-K into a non-zero fp32 `out`: 7 k-blocks (K = 440) split 2 / 3 / 4 ways, bias added once."""
    _seed(3)
    M, N, K = 256, 264, 440
    A, B, a, b = gemm_operands(M, N, K, a_mn, b_mn)
    bias, out0 = ints(N, dtype=torch.float32), ints(M, N, lo=-50, hi=50, dtype=torch.float32)
    out = out0.clone()
    launched(ops, ops.gemm, a, b, a_mn=a_mn, b_mn=b_mn, bias=bias, out=out, accumulate=True, alpha=0.5, split_k=split)
    check_gemm_out(f"split-K {split}", out, gemm_ref(A, B, 0.5, bias, out0=out0))


def sk_ctas_per_tile(ops, M, N, K, block_n):
    """Largest number of CTAs that share one output tile under the stream-K schedule (mirrors tepd_gemm_bf16)."""
    tiles, kb = math.ceil(M / 128) * math.ceil(N / block_n), math.ceil(K / 64)
    per = max(4, math.ceil(tiles * kb / ops._sms()))
    return max(len({it // per for it in range(t * kb, (t + 1) * kb)}) for t in range(tiles))


SK_SHAPES = [(4096, 1024, 1024, 256), (1280, 2048, 1024, 256), (1000, 520, 2056, 256), (1000, 520, 2056, 128),
             (256, 256, 8192, 256), (384, 520, 200, 128)]


@pytest.mark.parametrize("M,N,K,block_n", SK_SHAPES)
def test_gemm_stream_k_exact(ops, M, N, K, block_n):
    """Stream-K: fp32 red.add into a non-zero `out`.  An output that is not accumulated (bf16 with bias + residual, fp32
    plain store) cannot take the partial tiles of units that end mid-tile, so split_k=-1 there is refused before launch."""
    _seed(4)
    spread = sk_ctas_per_tile(ops, M, N, K, block_n)
    if (M, N, K) == (256, 256, 8192):
        assert spread > 16, spread
    A, B, a, b = gemm_operands(M, N, K, False, False)
    bias, res = ints(N, dtype=torch.float32), ints(M, N)
    out0 = ints(M, N, lo=-50, hi=50, dtype=torch.float32)
    out = out0.clone()
    launched(ops, ops.gemm, a, b, bias=bias, out=out, accumulate=True, alpha=2.0, split_k=-1, block_n=block_n)
    check_gemm_out(f"stream-K red.add ({spread} CTAs per tile)", out, gemm_ref(A, B, 2.0, bias, out0=out0))
    n0 = ops.launch_count()
    with pytest.raises(ValueError, match="split_k=-1"):
        ops.gemm(a, b, bias=bias, residual=res, split_k=-1, block_n=block_n)
    with pytest.raises(ValueError, match="split_k=-1"):
        ops.gemm(a, b, out_dtype=torch.float32, alpha=0.5, split_k=-1, block_n=block_n)
    with pytest.raises(ValueError, match="split_k=2"):
        ops.gemm(a, b, out_dtype=torch.float32, split_k=2, block_n=block_n)
    assert ops.launch_count() == n0


@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
def test_gemm_strided_epilogues_exact(ops, a_mn, b_mn):
    """bf16 bias; residual as a column slice of a wider tensor (ld_res != N); `out` as a column slice of a wider buffer
    (ldd != N) with the columns outside the slice untouched, for bf16, fp32 plain-store and fp32 accumulate outputs."""
    _seed(5)
    M, N, K = 264, 136, 200
    A, B, a, b = gemm_operands(M, N, K, a_mn, b_mn)
    bias16 = ints(N)
    res_wide = ints(M, N + 24)
    res = res_wide[:, 8:8 + N]
    assert res.stride(0) == N + 24
    d = launched(ops, ops.gemm, a, b, a_mn=a_mn, b_mn=b_mn, bias=bias16, residual=res, split_k=1)
    check_gemm_out("bf16 bias + strided residual", d, gemm_ref(A, B, 1.0, bias16, res))
    for dt, acc, sched in ((torch.bfloat16, False, 1), (torch.float32, False, 1), (torch.float32, True, 1),
                           (torch.float32, True, -1)):
        wide = torch.full((M, N + 16), -7.0, device="cuda", dtype=dt)
        wide[:, 8:8 + N] = ints(M, N, lo=-20, hi=20, dtype=dt) if acc else 0
        before = wide.clone()
        out = wide[:, 8:8 + N]
        launched(ops, ops.gemm, a, b, a_mn=a_mn, b_mn=b_mn, bias=bias16, residual=res, out=out, accumulate=acc, alpha=2.0,
                 split_k=sched)
        what = f"strided out {dt} accumulate={acc} split_k={sched}"
        check_gemm_out(what, out, gemm_ref(A, B, 2.0, bias16, res, before[:, 8:8 + N] if acc else None))
        assert torch.equal(wide[:, :8], before[:, :8]) and torch.equal(wide[:, 8 + N:], before[:, 8 + N:]), what


@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
def test_gemm_batched_exact(ops, a_mn, b_mn):
    """Batch 3 with ragged M / N / K and one bias shared by the batch, bf16 and fp32 outputs."""
    _seed(6)
    M, N, K = 200, 136, 200
    A, B, a, b = gemm_operands(M, N, K, a_mn, b_mn, batch=3)
    bias = ints(N, dtype=torch.float32)
    d = launched(ops, ops.gemm, a, b, a_mn=a_mn, b_mn=b_mn, bias=bias, alpha=2.0)
    check_gemm_out("batched bf16", d, gemm_ref(A, B, 2.0, bias))
    d = launched(ops, ops.gemm, a, b, a_mn=a_mn, b_mn=b_mn, bias=bias, out_dtype=torch.float32, alpha=0.5)
    check_gemm_out("batched fp32", d, gemm_ref(A, B, 0.5, bias))


def gelu64(x):
    x = x.double()
    return 0.5 * x * (1 + torch.tanh(0.7978845608028654 * (x + 0.044715 * x ** 3)))


def gelu_grad64(x):
    x = x.double()
    t = torch.tanh(0.7978845608028654 * (x + 0.044715 * x ** 3))
    return 0.5 * (1 + t) + 0.5 * x * (1 - t * t) * 0.7978845608028654 * (1 + 3 * 0.044715 * x * x)


def gelu_err(x):
    """Bound on |gelu_k(x) - gelu(x)| in fp32: the tanh.approx error times d gelu / dt = x / 2, plus a few fp32 roundings."""
    x = x.double().abs()
    return 0.5 * x * TANH_APPROX + 8 * U32 * x


def gelu_grad_err(x):
    """Bound on |gelu'_k(x) - gelu'(x)|: the tanh.approx error times |d gelu' / dt| <= 1/2 + |x t| k0 (1 + 3 k1 x^2), plus
    fp32 roundings of terms of that size."""
    x = x.double().abs()
    dgdt = 0.5 + x * 0.7978845608028654 * (1 + 3 * 0.044715 * x * x)
    return dgdt * (TANH_APPROX + 16 * U32)


@pytest.mark.parametrize("split_k,block_n", [(1, 128), (1, 256)])
def test_gemm_gelu_epilogues(ops, split_k, block_n):
    """Dual GELU: the pre-activation output exactly, the activated output to gelu_err; GELU backward (dgrad layout, aux =
    the bf16 pre-activation) to |acc| * gelu_grad_err, both through one bf16 store."""
    _seed(7)
    M, N, K = 1000, 520, 2056
    A, B, a, b = gemm_operands(M, N, K, False, False)
    bias = ints(N, dtype=torch.float32)
    pre = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    act = torch.empty_like(pre)
    launched(ops, ops.gemm, a, b, bias=bias, act="gelu", out=pre, out2=act, split_k=split_k, block_n=block_n)
    ref = gemm_ref(A, B, 1.0, bias)
    check_gemm_out("gelu dual: pre-activation", pre, ref)
    close("gelu dual: activation", act, gelu64(ref), bf16_tol(gelu64(ref), gelu_err(ref)))
    A2, B2, a2, b2 = gemm_operands(M, N, K, False, True)
    f = randn(M, N, scale=3.0)
    d = launched(ops, ops.gemm, a2, b2, b_mn=True, act="gelu_bwd", aux=f, alpha=0.5, split_k=split_k, block_n=block_n)
    acc = gemm_ref(A2, B2, 0.5)
    ref = acc * gelu_grad64(f)
    close("gelu_bwd epilogue", d, ref, bf16_tol(ref, acc.abs() * gelu_grad_err(f) + 2 * U32 * ref.abs()))


def test_gemm_rejects_mismatched_aux_and_out2(ops):
    """aux / out2 are addressed with out's offsets: a layout or dtype that differs is refused before any launch."""
    _seed(8)
    M, N, K = 256, 128, 64
    a, b = randn(M, K), randn(N, K)
    wide = torch.empty(M, N + 8, device="cuda", dtype=torch.bfloat16)
    out = wide[:, :N]
    n0 = ops.launch_count()
    with pytest.raises(ValueError, match="aux"):
        ops.gemm(a, b, act="gelu_bwd", out=out, aux=randn(M, N))
    with pytest.raises(ValueError, match="aux"):
        ops.gemm(a, b, act="gelu_bwd", aux=randn(M, N).float())
    with pytest.raises(ValueError, match="out2"):
        ops.gemm(a, b, act="gelu", out=out, out2=torch.empty(M, N, device="cuda", dtype=torch.bfloat16))
    with pytest.raises(ValueError, match="out2"):
        ops.gemm(a, b, act="gelu", out2=torch.empty(M * N, device="cuda", dtype=torch.bfloat16))
    assert ops.launch_count() == n0


# ============================================================================================== B. LayerNorm
def ln_ref(x, gamma, beta, eps=1e-5):
    xd = x.double()
    mean = xd.mean(-1)
    rstd = ((xd - mean[:, None]).pow(2).mean(-1) + eps).rsqrt()
    return (xd - mean[:, None]) * rstd[:, None] * gamma.double() + beta.double(), mean, rstd


def ln_inputs(rows, C, seed):
    _seed(seed)
    x = (torch.randn(rows, C, device="cuda", generator=gen()) * 2 + 0.5).to(torch.bfloat16)
    gamma = torch.randn(C, device="cuda", generator=gen()) * 0.5 + 1
    beta = torch.randn(C, device="cuda", generator=gen()) * 0.5
    return x, gamma, beta


@pytest.mark.parametrize("C", [8, 1024, 1032, 1600, 2048, 2056, 4096])
def test_layernorm_fwd(ops, C):
    """y, mean and rstd.  One warp sums each row: every lane adds its C/32 values in sequence, then 5 shuffle levels, so a
    sum carries at most n = C/32 + 5 roundings: |d mean| <= n u mean|x|, rstd is off by (n/2 + 4) u relative (rsqrt.approx
    is within 2^-22.9), and y = (x - mean) rstd g + b adds |g| rstd (|x - mean| d rstd / rstd + |d mean|) + 3 u |y|."""
    rows = 123
    x, gamma, beta = ln_inputs(rows, C, C)
    y, mean, rstd = launched(ops, ops.layernorm_fwd, x, gamma, beta)
    y_ref, m_ref, r_ref = ln_ref(x, gamma, beta)
    n = C / 32 + 5
    d_mean = n * U32 * x.double().abs().mean(-1)
    rel_rstd = (n / 2 + 6) * U32
    close("mean", mean, m_ref, 2 * (d_mean + 3 * U32 * m_ref.abs()))
    close("rstd", rstd, r_ref, 2 * rel_rstd * r_ref)
    xc = (x.double() - m_ref[:, None]).abs()
    err = gamma.double().abs() * r_ref[:, None] * (xc * rel_rstd + d_mean[:, None]) + 3 * U32 * y_ref.abs() + U32 * beta.double().abs()
    close("y", y, y_ref, bf16_tol(y_ref, err))


def ln_bwd_case(ops, rows, C, with_dres, seed=0):
    """dx (+ dres) of one case, and dgamma / dbeta added into buffers that start non-zero.

    dx = rstd (g - mean(g) - xh mean(g xh)) with g = dy gamma cancels terms as large as |g|, |mean(g)| and |xh mean(g xh)|:
    each carries a few fp32 roundings and the two row means carry n = C/32 + 5 more, so the fp32 value is within
    rstd (6 u (|g| + |s1| + |xh s2|) + n u (mean|g| + |xh| mean|g xh|)) + u |dres| of the reference.
    dgamma / dbeta: sums over rows in per-warp rows, then over the warps, then fp32 atomics across CTAs; whatever that order,
    the error is at most (chain - 1) u times the sum of |terms| with chain <= min(rows, 450) + 1 (the longest sequential
    path: rows per warp + warps + CTAs), plus the fp32 error of xh (3 u |xh|)."""
    _seed(seed)
    x, gamma, _ = ln_inputs(rows, C, seed + 1)
    _, m_ref, r_ref = ln_ref(x, gamma, torch.zeros_like(gamma))
    mean, rstd = m_ref.float(), r_ref.float()
    dy = randn(rows, C)
    dres = randn(rows, C, scale=3.0) if with_dres else None
    dg0 = torch.randn(C, device="cuda", generator=gen()) * 10
    db0 = torch.randn(C, device="cuda", generator=gen()) * 10
    dg, db = dg0.clone(), db0.clone()
    dx = launched(ops, ops.layernorm_bwd, dy, x, gamma, mean, rstd, dg, db, dres)
    xh = (x.double() - mean.double()[:, None]) * rstd.double()[:, None]
    g = dy.double() * gamma.double()
    s1, s2 = g.mean(-1, keepdim=True), (g * xh).mean(-1, keepdim=True)
    r = rstd.double()[:, None]
    ref = r * (g - s1 - xh * s2)
    n = C / 32 + 5
    err = r * (6 * U32 * (g.abs() + s1.abs() + (xh * s2).abs()) + n * U32 * (g.abs().mean(-1, keepdim=True)
                                                                              + xh.abs() * (g * xh).abs().mean(-1, keepdim=True)))
    if dres is not None:
        ref = ref + dres.double()
        err = err + U32 * dres.double().abs()
    close(f"dx rows={rows} C={C} dres={with_dres}", dx, ref, bf16_tol(ref, err))
    chain = min(rows, 450) + 1
    t_g, t_b = dy.double() * xh, dy.double()
    close("dgamma", dg, dg0.double() + t_g.sum(0),
          chain * U32 * (t_g.abs().sum(0) + dg0.double().abs()) + 3 * U32 * (dy.double() * xh).abs().sum(0) + FTZ)
    close("dbeta", db, db0.double() + t_b.sum(0), chain * U32 * (t_b.abs().sum(0) + db0.double().abs()) + FTZ)


@pytest.mark.parametrize("with_dres", [False, True])
@pytest.mark.parametrize("rows", [1, 7, 9, 4099])
@pytest.mark.parametrize("C", [8, 768, 1024, 1032, 1600, 2048])
def test_layernorm_bwd(ops, C, rows, with_dres):
    ln_bwd_case(ops, rows, C, with_dres, seed=C + rows)


def test_layernorm_bwd_eight_warps():
    """TEPDIST_LN_BWD_WARPS=8 (3 CTAs of 8 warps per SM at C <= 1024; read once per process, hence a fresh process)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys; sys.path[:0] = [sys.argv[1], sys.argv[2]]\n"
            "import test_step_numerics_gpu as t\n"
            "from tepdist_b200 import ops\n"
            "for C in (8, 768, 1024):\n"
            "    for rows in (1, 7, 9, 4099):\n"
            "        for d in (False, True):\n"
            "            t.ln_bwd_case(ops, rows, C, d, seed=C + rows)\n"
            "print('ok')\n")
    env = dict(os.environ, TEPDIST_LN_BWD_WARPS="8")
    p = subprocess.run([sys.executable, "-c", code, root, os.path.join(root, "tests")], env=env, capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0 and p.stdout.strip().endswith("ok"), p.stdout[-3000:] + p.stderr[-3000:]


# ============================================================================================== C. loss
def xent_case(ops, T, V, Vp, gscale, labels_hint, seed):
    _seed(seed)
    scale = torch.linspace(0.5, 25.0, T, device="cuda")[:, None]
    logits = (torch.randn(T, Vp, device="cuda", generator=gen()) * scale).clamp(-60, 60)
    logits[T // 2: T // 2 + 8] = torch.rand(8, Vp, device="cuda", generator=gen()) * 120 - 60   # magnitudes up to 60
    logits[:, V:] = 100.0                      # padding columns: must be ignored, then set to exactly zero
    logits = logits.to(torch.bfloat16)
    labels = torch.randint(0, V, (T,), device="cuda", generator=gen(), dtype=torch.int32)
    labels[:len(labels_hint)] = torch.tensor(labels_hint, device="cuda", dtype=torch.int32)
    lf = logits[:, :V].double()
    lse = torch.logsumexp(lf, -1)
    mx = lf.max(-1).values
    lab = labels.long()
    f_lab = lf.gather(1, lab[:, None])[:, 0]
    rows_ref = lse - f_lab
    p = torch.softmax(lf, -1)
    d_ref = p.clone()
    d_ref[torch.arange(T, device="cuda"), lab] -= 1
    d_ref *= gscale
    buf = logits.clone()
    total, rows = launched(ops, ops.xent_fwd_bwd, buf, labels, V, gscale)
    # per-row loss = -(f - mx - log(se)) with se = sum exp(f - mx) in fp32: __expf is within 2^-21 + |f - mx| 2^-23 relative
    # (its argument is rounded after the scaling by log2 e), a thread adds ~Vp/512 terms in sequence before a 9-level tree,
    # so se is within 3e-5 relative and log(se) within 3e-5 + 2^-21 (lg2.approx) absolute
    tol_rows = 2 * (3e-5 + 2.0 ** -21 + 2 * U32 * ((f_lab - mx).abs() + (lse - mx)))
    close(f"per-row loss V={V} Vp={Vp}", rows, rows_ref, tol_rows)
    # total = sum(rows * gscale) by fp32 atomics in any order
    close("total", total[0], rows.double().sum() * gscale, T * U32 * rows.double().abs().sum() * gscale + 1e-30)
    # dlogits = (exp(f - mx) / se - [c == label]) * gscale, one bf16 store: p is within (2^-21 + |f - mx| 2^-23 + 3e-5) p
    err = gscale * p * (2.0 ** -21 + (lf - mx[:, None]).abs() * 2.0 ** -23 + 3e-5) + FTZ
    close("dlogits", buf[:, :V], d_ref, bf16_tol(d_ref, err))
    assert bool((buf[:, V:].view(torch.int16) == 0).all()), "padding columns of dlogits are not exactly +0"


def test_xent_gpt2_vocab(ops):
    """T = 4096 rows of the padded GPT-2 vocabulary (V = 50257, Vp = 50304), grad scale 1/T; labels V - 1 (the only valid
    column of the last vector) and V - 2 on some rows."""
    xent_case(ops, 4096, 50257, 50304, 1.0 / 4096, [50256, 50255, 50256, 0], seed=10)


def test_xent_unpadded_vocab_and_partial_last_vector(ops):
    xent_case(ops, 512, 50304, 50304, 0.37, list(range(50296, 50304)), seed=11)          # Vp == V, labels in the last vector
    xent_case(ops, 64, 1003, 1008, 1.0, [1000, 1001, 1002, 1002, 999], seed=12)           # last vector holds 3 valid columns


# ============================================================================================== D. embedding / bias gradients
def test_embedding_fwd_exact(ops):
    _seed(20)
    B, S, C, Vp = 4, 1024, 1024, 50304
    wte, wpe = randn(Vp, C, scale=0.5), randn(S, C, scale=0.5)
    tok = torch.randint(0, 50257, (B, S), device="cuda", generator=gen(), dtype=torch.int32)
    out = launched(ops, ops.embedding_fwd, tok, wte, wpe)
    exact("embedding_fwd", out, (wte[tok.long()].float() + wpe.float()).bfloat16())


def test_embedding_bwd_exact(ops):
    """Integer dout, one token id in half of the positions, integer starting dwte / dwpe: every sum is exact in any atomic
    order, so the result must equal index_add exactly."""
    _seed(21)
    B, S, C, Vp = 4, 1024, 1024, 50304
    tok = torch.randint(0, 50257, (B, S), device="cuda", generator=gen(), dtype=torch.int32)
    tok.view(-1)[torch.randperm(B * S, device="cuda", generator=gen())[:B * S // 2]] = 4242
    dout = ints(B, S, C)
    dwte0 = ints(Vp, C, lo=-50, hi=50, dtype=torch.float32)
    dwpe0 = ints(S, C, lo=-50, hi=50, dtype=torch.float32)
    dwte, dwpe = dwte0.clone(), dwpe0.clone()
    launched(ops, ops.embedding_bwd, tok, dout, dwte, dwpe)
    exact("dwte", dwte, dwte0.double().index_add_(0, tok.view(-1).long(), dout.double().view(-1, C)))
    exact("dwpe", dwpe, dwpe0.double() + dout.double().sum(0))


@pytest.mark.parametrize("C", [8, 264, 1024, 4104])
@pytest.mark.parametrize("rows", [1, 63, 64, 65, 4097])
def test_colsum_exact(ops, rows, C):
    _seed(22)
    x = ints(rows, C)
    out0 = ints(C, lo=-1000, hi=1000, dtype=torch.float32)
    out = out0.clone()
    launched(ops, ops.colsum_acc, x, out)
    exact(f"colsum {rows}x{C}", out, out0.double() + x.double().sum(0))


# ============================================================================================== E. optimizer, casts, GELU
def f32(x):
    """A host scalar as the fp32 value the kernel computes with."""
    return float(torch.tensor(x, dtype=torch.float32))


def adamw_ref(p, g, m, v, hyper, n_decay, beta1, beta2, eps, wd):
    """fp64 restatement of adamw_kernel with its fp32 constants; returns (p, m, v, tolerances).

    m = b1 m + (1 - b1) g' (g' = g gscale) is within 3 u (|b1 m| + |(1 - b1) g'|); v (all terms positive) within 4 u v.
    The update u = (m / bc1) / (sqrt(v / bc2) + eps) (fast-math division and sqrt: 2 ulp each) is then within
    dm / bc1 / den + 12 u |u|, and p - lr (u + wd p) within u |p'| + lr (du + 2 u (|u| + wd |p|)).  Tolerances are twice that."""
    lr, bc1, bc2, gs = (float(x) for x in hyper.tolist())
    b1, b2, c1, c2 = f32(beta1), f32(beta2), f32(1 - f32(beta1)), f32(1 - f32(beta2))
    p, g, m, v = (t.double() for t in (p, g, m, v))
    gg = g * gs
    m1 = b1 * m + c1 * gg
    v1 = b2 * v + c2 * gg * gg
    den = (v1 / bc2).sqrt() + f32(eps)
    u = (m1 / bc1) / den
    decay = torch.zeros_like(p)
    decay[:n_decay] = f32(wd)
    p1 = p - lr * (u + decay * p)
    dm = 3 * U32 * ((b1 * m).abs() + (c1 * gg).abs())
    du = dm / bc1 / den + 12 * U32 * u.abs()
    dp = U32 * p1.abs() + lr * (du + 2 * U32 * (u.abs() + decay * p.abs()))
    return p1, m1, v1, (2 * dp + FTZ, 2 * dm + FTZ, 8 * U32 * v1 + FTZ)


def test_adamw_hyper_tail_decay_boundary_and_graph_replay(ops):
    """n = 4k + 3 (scalar tail), n_decay = 4j + 2 (boundary inside a float4), grad scale 0.25, three steps whose lr, bc1, bc2
    and grad scale come only from the device `hyper` tensor (the host scalars passed are wrong on purpose); then the same
    three steps captured once in a CUDA graph and replayed with new `hyper` contents must give the same bits."""
    _seed(30)
    n, n_decay = 4 * 25_000 + 3, 4 * 12_345 + 2
    beta1, beta2, eps, wd = 0.9, 0.95, 1e-8, 0.1
    p0 = torch.randn(n, device="cuda", generator=gen())
    m0 = torch.randn(n, device="cuda", generator=gen()) * 1e-2
    v0 = torch.rand(n, device="cuda", generator=gen()) * 1e-3
    grads = [torch.randn(n, device="cuda", generator=gen()) * 4 for _ in range(3)]
    hypers = [torch.tensor([1e-2 * (s + 1) / 3, 1 - beta1 ** (s + 1), 1 - beta2 ** (s + 1), 0.25], device="cuda")
              for s in range(3)]
    p, m, v = p0.clone(), m0.clone(), v0.clone()
    pb = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    eager = []
    for s in range(3):
        pp, mp, vp = p.clone(), m.clone(), v.clone()
        launched(ops, ops.adamw_step, p, grads[s], m, v, pb, n_decay, 123.0, beta1, beta2, eps, wd, 1000, grad_scale=7.0,
                 hyper=hypers[s])
        p_ref, m_ref, v_ref, (tp, tm, tv) = adamw_ref(pp, grads[s], mp, vp, hypers[s], n_decay, beta1, beta2, eps, wd)
        close(f"adamw p step {s + 1}", p, p_ref, tp)
        close(f"adamw m step {s + 1}", m, m_ref, tm)
        close(f"adamw v step {s + 1}", v, v_ref, tv)
        exact(f"adamw bf16 copy step {s + 1}", pb, p.to(torch.bfloat16))
        eager.append((p.clone(), m.clone(), v.clone(), pb.clone()))

    p.copy_(p0); m.copy_(m0); v.copy_(v0)
    g_in, h_in = grads[0].clone(), hypers[0].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side), torch.cuda.graph(graph):
        ops.adamw_step(p, g_in, m, v, pb, n_decay, 123.0, beta1, beta2, eps, wd, 1000, grad_scale=7.0, hyper=h_in)
    torch.cuda.current_stream().wait_stream(side)
    p.copy_(p0); m.copy_(m0); v.copy_(v0)          # (capture records, it does not run)
    for s in range(3):
        g_in.copy_(grads[s]); h_in.copy_(hypers[s])
        graph.replay()
        torch.cuda.synchronize()
        for name, got, want in zip(("p", "m", "v"), (p, m, v), eager[s][:3]):
            assert torch.equal(got.view(torch.int32), want.view(torch.int32)), f"graph replay {s + 1}: {name} differs from eager"
        assert torch.equal(pb.view(torch.int16), eager[s][3].view(torch.int16)), f"graph replay {s + 1}: bf16 copy differs"


def cast_values():
    """fp32 values for the cast: exact midpoints between bf16 neighbours (even and odd lower neighbour), one fp32 ulp either
    side of them, subnormals (incl. midpoints), values that round up to inf, +-inf, NaN, and random normals."""
    hi16 = torch.arange(0, 1 << 15, 97, dtype=torch.int32)          # bf16 bit patterns (positive, finite and not)
    lo = (hi16 << 16)
    mids = lo | 0x8000                                           # exactly halfway to the next bf16 value
    vals = torch.cat([mids, mids + 1, mids - 1, lo, torch.tensor([1, 2, 0x7FFF, 0x8000, 0x18000, 0x7F7F8000, 0x7F7FFFFF,
                                                                    0x7F800000, 0x7FC00000, 0x7F800001, 0x00800000])])
    vals = torch.cat([vals, vals | torch.tensor(-0x80000000, dtype=torch.int32)]).view(torch.float32)
    rnd = torch.randn(4096) * torch.logspace(-30, 30, 4096)
    return torch.cat([vals, rnd])


def test_cast_f32_bf16_vector_and_scalar_paths(ops):
    """Round to nearest even, bit for bit against torch (NaN compared by isnan), on the 8-wide vector kernel (aligned,
    n % 8 == 0) and on the scalar kernel (a slice that starts 4 bytes into its buffer, n % 8 != 0)."""
    _seed(32)
    vals = cast_values()
    n8 = vals.numel() // 8 * 8
    for what, src in (("vector", vals[:n8].cuda().contiguous()), ("scalar", torch.cat([vals[:1], vals[:n8 - 3]]).cuda()[1:])):
        assert (src.data_ptr() % 32 == 0 and src.numel() % 8 == 0) == (what == "vector")
        dst = torch.empty(src.numel(), device="cuda", dtype=torch.bfloat16)
        launched(ops, ops.cast_f32_bf16, src, dst)
        want = src.cpu().to(torch.bfloat16)
        nan = torch.isnan(want)
        assert torch.equal(torch.isnan(dst.cpu()), nan), what
        exact(f"cast ({what} path)", dst.cpu()[~nan], want[~nan])


def test_gelu_fwd_bwd_dense_sweep(ops):
    """Every bf16 value in [-12, 12].  Bound: one bf16 ulp plus the tanh.approx.f32 error (2^-10.987, PTX ISA) carried
    through (gelu_err, gelu_grad_err).  Measured on an H100: forward max |err| 7.8e-3, at most 0.50 of the bound; backward
    at most 0.47 of the bound (printed on every run)."""
    _seed(31)
    bits = torch.arange(-(1 << 15), 1 << 15, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    x = bits[torch.isfinite(bits.float()) & (bits.float().abs() <= 12)]
    x = torch.cat([x, x[: (-x.numel()) % 8]]).cuda()
    y = launched(ops, ops.gelu_fwd, x)
    ref = gelu64(x)
    worst_f = close("gelu_fwd", y, ref, bf16_tol(ref, gelu_err(x)))
    dy = randn(x.numel(), scale=2.0)
    dx = launched(ops, ops.gelu_bwd, dy, x)
    ref = dy.double() * gelu_grad64(x)
    worst_b = close("gelu_bwd", dx, ref, bf16_tol(ref, dy.double().abs() * gelu_grad_err(x) + 2 * U32 * ref.abs()))
    err_f = (y.double() - gelu64(x)).abs().max().item()
    print(f"\ngelu sweep over {x.numel()} values: fwd max |err| {err_f:.3g} (worst err / bound {worst_f:.3f}); "
          f"bwd worst err / bound {worst_b:.3f}")


# ============================================================================================== F. whole steps
# Bound on each parameter's relative gradient error ||g_gpu - g_cpu|| / ||g_cpu|| against the fp32 CPU executor (names
# without "model/" and "h0/").  The GPU step computes in bf16, so these are measured, not derived: on an H100 80GB HBM3 at
# 700 W the largest value over the three 345M steps and the 1.3B step was 2.6e-3 to 9.5e-3 depending on the parameter, and
# each bound is about twice that parameter's largest value.
GRAD_TOL = {"wte": 2e-2, "wpe": 2e-2, "attn/c_attn/w": 2e-2, "attn/c_proj/w": 1.8e-2, "mlp/c_fc/w": 1.7e-2,
            "mlp/c_proj/w": 1.4e-2, "output": 1.4e-2, "ln_1/g": 1.9e-2, "ln_1/b": 1.5e-2, "attn/c_attn/b": 1.4e-2,
            "attn/c_proj/b": 1.3e-2, "ln_2/g": 1.7e-2, "ln_2/b": 1.3e-2, "mlp/c_fc/b": 1.2e-2, "mlp/c_proj/b": 7e-3,
            "ln_f/g": 1.2e-2, "ln_f/b": 6e-3}


def grad_tol(name):
    return GRAD_TOL[re.sub(r"^model/(h0/)?", "", name)]


def step_checks(gpu, cpu, feeds_gpu, feeds_cpu, label, tol=grad_tol):
    """One GPU step with the CPU oracle run from the same fp32 master / m / v, then the gradient table (bound per parameter
    name from `tol`) and the update."""
    gs, cs = gpu.store, cpu.store
    assert gs.total == cs.total and gs.order == cs.order
    for name in ("master", "m", "v"):
        getattr(cs, name).copy_(getattr(gs, name).cpu())
    pre = {name: getattr(gs, name).clone() for name in ("master", "m", "v")}
    cpu.step_count = gpu.step_count
    t0 = time.perf_counter()
    gpu.step(feeds_gpu)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    cpu.step(feeds_cpu)
    t2 = time.perf_counter()
    print(f"\n{label}: GPU step {t1 - t0:.2f} s, CPU oracle {t2 - t1:.2f} s; lr {gpu.lr_now:.3g}")
    print(f"  {'parameter':<32} {'|g_cpu|':>10} {'rel err':>9} {'bound':>8}")
    worst = {}
    for pid in gs.order:
        name = gs.names[pid]
        g, r = gs.grad_view(pid).double().cpu(), cs.grad_view(pid).double()
        rel = float((g - r).norm() / r.norm().clamp_min(1e-30))
        worst[name] = rel
        print(f"  {name:<32} {float(r.norm()):>10.3e} {rel:>9.2e} {tol(name):>8.1e}")
    for name, rel in worst.items():
        assert rel <= tol(name), f"{label}: gradient of {name} off by {rel:.3e} relative (bound {tol(name)})"
    # the update: fp64 AdamW of the GPU's own gradient, pre-step master / m / v and this step's hyper
    o = gpu.opt
    p_ref, m_ref, v_ref, (tp, tm, tv) = adamw_ref(pre["master"], gs.grad, pre["m"], pre["v"], gpu.hyper[:4], gs.n_decay,
                                                  o.get("beta1", 0.9), o.get("beta2", 0.999), o.get("eps", 1e-8),
                                                  o.get("weight_decay", 0.0))
    close(f"{label}: master", gs.master, p_ref, tp)
    close(f"{label}: m", gs.m, m_ref, tm)
    close(f"{label}: v", gs.v, v_ref, tv)
    exact(f"{label}: bf16 compute copy", gs.compute, gs.master.to(torch.bfloat16))
    return worst


def gpt2_pair(cfg, use_cuda_graph):
    from tepdist_b200.models.gpt2 import build_gpt2_graph
    from tepdist_b200.runtime.executor import Executor
    g = build_gpt2_graph(cfg)
    gpu = Executor(g, torch.device("cuda", 0), seed=0, use_cuda_graph=use_cuda_graph)
    cpu = Executor(g, torch.device("cpu"), seed=0)
    sched = lambda step: cfg.lr * min(1.0, step / 4)      # linear warm-up
    gpu.set_lr_schedule(sched)
    cpu.set_lr_schedule(sched)
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (cfg.batch, cfg.n_ctx), dtype=torch.int32)
    lab = torch.roll(tok, -1, 1)
    return gpu, cpu, {"tokens": tok.cuda(), "labels": lab.cuda()}, {"tokens": tok, "labels": lab}


def test_gpt2_345m_widths_steps_gradient_by_gradient(ops):
    """One layer at the 345M widths and 4096 tokens: the schedule decisions of the benchmarked step.  Step 1 eager, step 2
    CUDA-graph capture + replay, step 3 replay."""
    from tepdist_b200.models.gpt2 import GPT2Config
    cfg = GPT2Config(1, 1024, 16, 1024, 50257, 4)
    gpu, cpu, fg, fc = gpt2_pair(cfg, use_cuda_graph=True)
    wgrads = [n.id for n in gpu.g.nodes if n.op == "linear_wgrad"]
    assert any((i, 0) in gpu._store_init for i in wgrads), "no weight gradient on the plain-store path"
    assert any((i, 0) not in gpu._store_init for i in wgrads), "no weight gradient on the accumulate / split-K path"
    assert gpu._zero_ranges is not None
    assert gpu.ln_fuse and gpu.gelu_dual and gpu.gelu_bwd_fuse
    t0 = time.perf_counter()
    for s, label in enumerate(("345M step 1 (eager)", "345M step 2 (capture + replay)", "345M step 3 (replay)")):
        n0 = ops.launch_count()
        step_checks(gpu, cpu, fg, fc, label)
        assert ops.launch_count() > n0
        assert (gpu._graph is None) == (s == 0)
    print(f"345M steps with oracle: {time.perf_counter() - t0:.1f} s")


def test_gpt2_1p3b_widths_step_gradient_by_gradient(ops):
    """One layer at the 1.3B widths (C = 2048: LayerNorm backward at MAXV = 8, 128-wide heads), one eager step."""
    from tepdist_b200.models.gpt2 import GPT2Config
    cfg = GPT2Config(1, 2048, 16, 2048, 50257, 1)
    gpu, cpu, fg, fc = gpt2_pair(cfg, use_cuda_graph=False)
    assert gpu.ln_fuse and gpu.gelu_dual and gpu.gelu_bwd_fuse
    step_checks(gpu, cpu, fg, fc, "1.3B step 1 (eager)")
