"""The fp32 weight-gradient GEMM (A and B MN-major) gives the same elements on its two store paths.

An fp32 output that TMA can address (16-byte aligned base, row pitch a multiple of 4 elements) is written through the
shared-memory staging buffer with TMA stores, or with TMA reduce-adds when the GEMM accumulates into it (split-K, stream-K,
gradient accumulation); any other fp32 output is stored straight from the accumulator fragments with float2 stores or
red.add.  Operands are integers in [-3, 3], the starting `out` is integer and alpha is 0.5 or 2, so every schedule's fp32
result is exact: it must equal an fp64 reference, and the staged result must be bit-identical to the direct one.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

M, N = 296, 520      # an M tail (M % 8 == 0, as an MN-major A needs) and an N tail at both tile widths
K = 584              # 10 k-blocks, the last one partial: split 3 and 4 give uneven, non-empty splits


def _ops():
    from tepdist_b200 import ops
    ops.lib()
    return ops


def _ints(gen, *shape, lo=-3, hi=3, dtype=torch.bfloat16):
    return torch.randint(lo, hi + 1, shape, generator=gen, device="cuda").to(dtype)


def _operands(seed, batch=0):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    lead = (batch,) if batch else ()
    dy, x = _ints(gen, *lead, K, M), _ints(gen, *lead, K, N)   # dW = dy^T @ x, both stored [K, *]
    return gen, dy, x


def _ref(dy, x, alpha, out0=None):
    d = alpha * torch.matmul(dy.double().transpose(-1, -2), x.double())
    return d if out0 is None else d + out0.double()


def _run(ops, dy, x, out, **kw):
    n0 = ops.launch_count()
    ops.gemm(dy, x, a_mn=True, b_mn=True, out=out, **kw)
    assert ops.launch_count() == n0 + 1, "our GEMM kernel did not run"
    torch.cuda.synchronize()
    return out


def _exact(what, got, ref):
    bad = got.double() != ref
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {got.numel()} elements differ from the fp64 reference"


def _unaligned(pitch_extra):
    """An fp32 [M, N] view whose base is 8 bytes past a 16-byte boundary (pitch_extra = 0) or whose row pitch is N + 2."""
    if pitch_extra:
        return torch.zeros(M, N + pitch_extra, device="cuda")[:, :N]
    return torch.zeros(M * N + 2, device="cuda")[2:].view(M, N)


@pytest.mark.parametrize("block_n", [128, 256])
def test_f32_store_exact(block_n):
    ops = _ops()
    _, dy, x = _operands(11)
    out = _run(ops, dy, x, torch.full((M, N), float("nan"), device="cuda"), alpha=0.5, split_k=1, block_n=block_n)
    _exact("fp32 store", out, _ref(dy, x, 0.5))


@pytest.mark.parametrize("split", [1, 2, 3, 4, -1], ids=["split1", "split2", "split3", "split4", "stream_k"])
@pytest.mark.parametrize("block_n", [128, 256])
def test_f32_accumulate_exact(block_n, split):
    """Reduce-add into a non-zero `out`: one unit per tile, split-K 2 / 3 / 4, and stream-K units that end mid-tile."""
    ops = _ops()
    gen, dy, x = _operands(12)
    out0 = _ints(gen, M, N, lo=-100, hi=100, dtype=torch.float32)
    out = _run(ops, dy, x, out0.clone(), accumulate=True, alpha=2.0, split_k=split, block_n=block_n)
    _exact(f"fp32 accumulate, split_k={split}", out, _ref(dy, x, 2.0, out0))


def test_f32_batched_exact():
    ops = _ops()
    gen, dy, x = _operands(13, batch=3)
    out = _run(ops, dy, x, torch.full((3, M, N), float("nan"), device="cuda"), alpha=0.5, split_k=1)
    _exact("batched fp32 store", out, _ref(dy, x, 0.5))
    out0 = _ints(gen, 3, M, N, lo=-100, hi=100, dtype=torch.float32)
    out = _run(ops, dy, x, out0.clone(), accumulate=True, alpha=2.0, split_k=2)
    _exact("batched fp32 accumulate", out, _ref(dy, x, 2.0, out0))


@pytest.mark.parametrize("pitch_extra", [0, 2])
@pytest.mark.parametrize("split", [0, 1, 3, -1], ids=["store", "accumulate", "split3", "stream_k"])
@pytest.mark.parametrize("block_n", [128, 256])
def test_staged_and_direct_f32_match(block_n, split, pitch_extra):
    """The same call into an aligned `out` (staged) and into an unaligned one (direct): bit-identical results."""
    ops = _ops()
    gen, dy, x = _operands(14)
    acc = split != 0
    out0 = _ints(gen, M, N, lo=-100, hi=100, dtype=torch.float32) if acc else torch.zeros(M, N, device="cuda")
    kw = dict(accumulate=acc, alpha=0.5, split_k=split if acc else 1, block_n=block_n)
    staged = _run(ops, dy, x, out0.clone(), **kw)
    u = _unaligned(pitch_extra)
    u.copy_(out0)
    direct = _run(ops, dy, x, u, **kw)
    assert torch.equal(staged.view(torch.int32), direct.contiguous().view(torch.int32))
    _exact("staged fp32", staged, _ref(dy, x, 0.5, out0 if acc else None))


@pytest.mark.parametrize("acc", [False, True], ids=["store", "accumulate"])
@pytest.mark.parametrize("block_n", [128, 256])
def test_f32_strided_out_leaves_other_columns(block_n, acc):
    """`out` as a column slice of a wider buffer whose pitch TMA can address: the columns outside it stay untouched."""
    ops = _ops()
    gen, dy, x = _operands(15)
    wide = torch.full((M, N + 16), -7.0, device="cuda")
    wide[:, 8:8 + N] = _ints(gen, M, N, lo=-20, hi=20, dtype=torch.float32) if acc else float("nan")
    before = wide.clone()
    out = wide[:, 8:8 + N]
    _run(ops, dy, x, out, accumulate=acc, alpha=2.0, split_k=0 if acc else 1, block_n=block_n)
    _exact("strided fp32 out", out, _ref(dy, x, 2.0, before[:, 8:8 + N] if acc else None))
    assert torch.equal(wide[:, :8], before[:, :8]) and torch.equal(wide[:, 8 + N:], before[:, 8 + N:])
