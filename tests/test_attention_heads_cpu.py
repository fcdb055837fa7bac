"""Head-width dispatch of ops/attention.py and the exactness of the zero padding it applies around the kernels, checked
with the fp32 reference math on CPU."""
import warnings

import pytest
import torch

from tepdist_b200.ops import attention as A


def test_head_width_dispatch():
    assert [A._kernel_width(D) for D in (8, 48, 64)] == [64, 64, 64]
    assert [A._kernel_width(D) for D in (65, 80, 96, 112, 128)] == [128] * 5
    assert A._kernel_width(129) is None and A._kernel_width(256) is None
    assert A._can_pad(256, 96, False) and A._can_pad(200, 128, True) and A._can_pad(200, 48, True)
    assert not A._can_pad(256, 192, True)        # wider than every kernel
    assert not A._can_pad(200, 128, False)       # non-causal ragged S: padded keys would be attended to


def test_torch_math_shapes_warn_once_per_shape():
    with pytest.warns(UserWarning, match="head dim 192"):
        A._warn_torch_math(256, 192, True)
    with pytest.warns(UserWarning, match="seq 200"):
        A._warn_torch_math(200, 128, False)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        A._warn_torch_math(256, 192, True)


def _qkv(B, S, H, D, seed=0):
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B, S, H, 3, D, generator=g)
    return qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2], torch.randn(B, S, H, D, generator=g)


@pytest.mark.parametrize("S,D,causal", [(256, 96, True), (256, 96, False), (200, 96, True), (200, 128, True)])
def test_padding_to_kernel_shape_is_exact(S, D, causal):
    B, H = 2, 3
    q, k, v, do = _qkv(B, S, H, D)
    scale = D ** -0.5
    o, lse = A.attention_fwd(q, k, v, scale, causal)
    dq, dk, dv = A.attention_bwd(do, q, k, v, o, lse, scale, causal)
    W = A._kernel_width(D)
    Sp = (S + 127) // 128 * 128
    pq, pk, pv, pdo = (A._pad_sd(t, S, D, W) for t in (q, k, v, do))
    assert pq.shape == (B, Sp, H, W)
    po, plse = A.attention_fwd(pq, pk, pv, scale, causal)
    pg = A.attention_bwd(pdo, pq, pk, pv, po, plse, scale, causal)
    torch.testing.assert_close(po[:, :S, :, :D], o, atol=1e-6, rtol=1e-6)
    assert not po[:, :S, :, D:].any()
    torch.testing.assert_close(plse[:, :, :S], lse, atol=1e-6, rtol=1e-6)
    for got, want in zip(pg, (dq, dk, dv)):
        torch.testing.assert_close(got[:, :S, :, :D], want, atol=1e-6, rtol=1e-6)
