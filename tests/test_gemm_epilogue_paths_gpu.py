"""The GEMM's two bf16 store paths give the same elements.

An output (and a residual / GELU' aux) that TMA can address is written through the shared-memory staging buffer with TMA
stores; one whose base address or row pitch breaks TMA's 16-byte rules is stored straight from the accumulator fragments.
Each epilogue the training step uses runs once on an aligned output and once on an output 4 elements (8 bytes) into a
larger buffer or with a row pitch that is not a multiple of 8: both results must be bit-identical, and where the arithmetic
is exact (integer-valued operands, no GELU) equal to the round-to-nearest-even bf16 cast of an fp64 reference.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

M, N, K = 300, 520, 200   # M and N tails in both tile widths


def _ints(gen, *shape):
    return torch.randint(-3, 4, shape, generator=gen, device="cuda").to(torch.bfloat16)


def _unaligned(shape, pitch_extra):
    """A bf16 [M, N] view whose base is 8 bytes past a 16-byte boundary (pitch_extra = 0) or whose row pitch is N + 4."""
    if pitch_extra:
        return torch.zeros(shape[0], shape[1] + pitch_extra, dtype=torch.bfloat16, device="cuda")[:, : shape[1]]
    return torch.zeros(shape[0] * shape[1] + 4, dtype=torch.bfloat16, device="cuda")[4:].view(shape)


@pytest.mark.parametrize("pitch_extra", [0, 4])
@pytest.mark.parametrize("kind", ["plain", "bias", "bias_res", "gelu_dual", "gelu_bwd"])
@pytest.mark.parametrize("block_n", [128, 256])
def test_staged_and_direct_stores_match(kind, pitch_extra, block_n):
    from tepdist_b200 import ops
    ops.lib()
    gen = torch.Generator(device="cuda")
    gen.manual_seed(7)
    a = _ints(gen, M, K)
    b_mn = kind == "gelu_bwd"    # the data-gradient layout, as the step runs GELU'
    w = _ints(gen, K, N) if b_mn else _ints(gen, N, K)
    bias = _ints(gen, N) if kind in ("bias", "bias_res", "gelu_dual") else None
    res = _ints(gen, M, N) if kind == "bias_res" else None
    act = {"gelu_dual": "gelu", "gelu_bwd": "gelu_bwd"}.get(kind)

    def run(out, out2, aux, residual):
        n0 = ops.launch_count()
        ops.gemm(a, w, b_mn=b_mn, bias=bias, residual=residual, act=act, out=out, out2=out2, aux=aux, alpha=0.5,
                 block_n=block_n)
        assert ops.launch_count() == n0 + 1
        return out, out2

    aux = _ints(gen, M, N) if kind == "gelu_bwd" else None
    al = run(torch.empty(M, N, dtype=torch.bfloat16, device="cuda"),
             torch.empty(M, N, dtype=torch.bfloat16, device="cuda") if kind == "gelu_dual" else None, aux, res)
    u_out = _unaligned((M, N), pitch_extra)
    u_out2 = _unaligned((M, N), pitch_extra) if kind == "gelu_dual" else None
    u_aux = None
    if aux is not None:       # aux must share out's layout
        u_aux = _unaligned((M, N), pitch_extra)
        u_aux.copy_(aux)
    u_res = None
    if res is not None:
        u_res = _unaligned((M, N), pitch_extra)
        u_res.copy_(res)
    un = run(u_out, u_out2, u_aux, u_res)
    torch.cuda.synchronize()
    assert torch.equal(al[0], un[0])
    if kind == "gelu_dual":
        assert torch.equal(al[1], un[1])
    if act is None:
        ref = 0.5 * (a.double() @ (w.double() if b_mn else w.double().t()))
        if bias is not None:
            ref += bias.double()
        if res is not None:
            ref += res.double()
        assert torch.equal(al[0], ref.to(torch.bfloat16))
