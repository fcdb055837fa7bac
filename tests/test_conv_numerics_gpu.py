"""Element-by-element numerics of the kernels one Wide-ResNet training step launches (convolution, BatchNorm, pooling, the
conv-net elementwise ops, SGD), and every parameter's gradient of whole Wide-ResNet steps against the fp32 CPU executor.

Conventions as in test_step_numerics_gpu.py: every case checks that our kernel ran, and compares each element with a
reference computed in fp64 from the same bf16 / fp32 inputs; bit for bit where the arithmetic is exact, otherwise within a
per-element bound derived from the kernel's arithmetic and stated beside the case.
"""
import math
import time

import pytest
import torch
import torch.nn.functional as F

from test_step_numerics_gpu import (FTZ, U32, adamw_ref, bf16_tol, close, exact, gen, ints, launched, ops, randn,  # noqa: F401
                                    step_checks, _seed)

pytestmark = pytest.mark.gpu

RSQRT_APPROX = 2.0 ** -22.9     # max relative error of rsqrt.approx.f32 (PTX ISA); --use_fast_math maps rsqrtf / 1.f / x to it


class _CountingLib:
    """Wraps the kernel library and counts calls per entry point (which data-movement path a convolution took)."""

    def __init__(self, real):
        self.real, self.calls = real, {}

    def __getattr__(self, name):
        fn = getattr(self.real, name)

        def call(*args):
            self.calls[name] = self.calls.get(name, 0) + 1
            return fn(*args)
        return call


@pytest.fixture
def counted(ops, monkeypatch):
    lib = _CountingLib(ops.lib())
    monkeypatch.setattr(ops, "lib", lambda: lib)
    return lib


# ============================================================================================== A. convolution, exact
# Operands are integers in [-2, 2].  Every product is an integer and every partial sum of every GEMM schedule stays below
# 2^24 (|sum| <= 4 K with K <= 6000), so the fp32 accumulators hold exact integers: the forward must equal bf16(fp64 conv),
# the fp32 weight gradient the fp64 value.  The input gradient rounds twice by design: dcol = dY . Wmat is stored as bf16,
# then col2im adds the bf16 taps in fp32 (at most k*k integers of a bf16, exact) and stores bf16 once.

# N, C, H, W, Cout, k, stride, pad
CONV_CASES = [
    (1, 3, 224, 224, 64, 7, 2, 3),     # the Wide-ResNet stem: generic VEC = 1 path, K = 147 padded to 152
    (2, 3, 29, 22, 64, 7, 2, 3),       # stem geometry on a non-square odd image
    (1, 3, 3, 5, 8, 7, 2, 3),          # stem on an image smaller than the kernel: every output touches the padding
    (2, 64, 13, 21, 128, 1, 1, 0),     # 1x1 s1: direct GEMM, no im2col / col2im
    (2, 32, 13, 21, 40, 3, 1, 1),      # 3x3 s1 p1, non-square, 546 rows (not a multiple of the GEMM tile)
    (2, 32, 25, 25, 48, 3, 2, 1),      # 3x3 s2 p1, 25 -> 13
    (1, 16, 7, 7, 16, 3, 2, 1),        # 3x3 s2 p1, 7 -> 4
    (2, 64, 25, 13, 128, 1, 2, 0),     # 1x1 s2 shortcut on odd sizes: im2col path
    (2, 16, 3, 3, 24, 3, 1, 1),        # 3x3 image: every output touches the padding
    (1, 8, 1, 1, 8, 3, 1, 1),          # 1x1 image, C = 8 (one channel vector), Cout = 8
    (1, 8, 9, 14, 8, 3, 2, 1),         # C = 8, Cout = 8, stride 2 on a non-square image
    (2, 5, 11, 17, 16, 3, 1, 1),       # C % 8 != 0: VEC = 1 im2col and col2im_nhwc_kernel<1>
    (2, 3, 13, 21, 8, 3, 2, 1),        # C = 3 with stride 2
    (2, 64, 14, 10, 320, 3, 1, 1),     # Cout = 320: dcol values up to 1280, so its bf16 rounding is exercised
]


def conv_ids(c):
    return "N{}C{}_{}x{}_Co{}_k{}s{}p{}".format(*c)


def dgrad_ref(dy, w, x_shape, stride, pad):
    """fp64 model of the two roundings: dcol = bf16(dY . Wmat) with columns (tap, cin), then the fp64 gather-sum (F.fold
    after permuting to (cin, tap)), then one round to bf16."""
    N, C, H, W = x_shape
    Cout, _, kh, kw = w.shape
    Ho, Wo = dy.shape[2], dy.shape[3]
    dyn = dy.double().permute(0, 2, 3, 1).reshape(N * Ho * Wo, Cout)
    wmat = w.double().permute(0, 2, 3, 1).reshape(Cout, kh * kw * C)
    dcol = (dyn @ wmat).float().to(torch.bfloat16).double()                  # exact integers before the bf16 round
    cols = dcol.view(N, Ho * Wo, kh * kw, C).permute(0, 3, 2, 1).reshape(N, C * kh * kw, Ho * Wo)
    return F.fold(cols, (H, W), (kh, kw), padding=pad, stride=stride).float().to(torch.bfloat16)


def im2col_ref(x, k, stride, pad, Kpad):
    N, C, H, W = x.shape
    u = F.unfold(x.double(), k, padding=pad, stride=stride)                 # [N, C*k*k, L], rows (c, tap)
    L = u.shape[-1]
    col = u.view(N, C, k * k, L).permute(0, 3, 2, 1).reshape(N * L, k * k * C)
    return F.pad(col, (0, Kpad - k * k * C)).float().to(torch.bfloat16)


@pytest.mark.parametrize("case", CONV_CASES, ids=[conv_ids(c) for c in CONV_CASES])
def test_conv_exact(ops, counted, case):
    N, C, H, W, Cout, k, s, p = case
    _seed(sum(case))
    x, w = ints(N, C, H, W, lo=-2, hi=2), ints(Cout, C, k, k, lo=-2, hi=2)
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    dy = ints(N, Cout, Ho, Wo, lo=-2, hi=2)
    direct = k == 1 and s == 1 and p == 0 and C % 8 == 0
    xc, wc, dyc = x.cpu().double(), w.cpu().double(), dy.cpu().double()

    y = launched(ops, ops.conv2d_fwd, x, w, s, p)
    assert tuple(y.shape) == (N, Cout, Ho, Wo)
    exact("forward", y, F.conv2d(xc, wc, stride=s, padding=p).float().to(torch.bfloat16))
    gw = launched(ops, ops.conv2d_wgrad, dy, x, w.shape, s, p)
    assert tuple(gw.shape) == tuple(w.shape) and gw.dtype == torch.float32       # K-padding columns dropped
    exact("wgrad", gw, torch.nn.grad.conv2d_weight(xc, w.shape, dyc, stride=s, padding=p))
    dx = launched(ops, ops.conv2d_dgrad, dy, w, x.shape, s, p)
    assert tuple(dx.shape) == (N, C, H, W)
    exact("dgrad", dx, dgrad_ref(dyc, wc, x.shape, s, p))

    im2col, col2im = counted.calls.get("tepd_im2col_nhwc", 0), counted.calls.get("tepd_col2im_nhwc", 0)
    assert (im2col, col2im) == ((0, 0) if direct else (2, 1)), counted.calls
    if not direct:
        # the column matrix itself, K padding included, into a buffer full of NaN
        Kpad = (k * k * C + 7) // 8 * 8
        col = torch.full((N * Ho * Wo, Kpad), float("nan"), device="cuda", dtype=torch.bfloat16)
        xn = x.contiguous(memory_format=torch.channels_last)
        rc = counted.tepd_im2col_nhwc(xn.data_ptr(), col.data_ptr(), N, H, W, C, Ho, Wo, k, k, s, p, Kpad, ops._stream())
        assert rc == 0
        exact("im2col", col, im2col_ref(x.cpu(), k, s, p, Kpad))


# ============================================================================================== B. BatchNorm
# Reference: fp64 two-pass statistics of the same bf16 input.  Forward error analysis of the kernels: every per-channel sum
# runs along a chain of at most L = ceil(min(rows, 128) / 8) (one warp's strip of a 128-row block) + 8 (the warps) +
# ceil(rows / 128) (one fp32 atomic per block) + 3 (the all-reduce of up to 3 shards) additions, so it is within
# (L - 1) u sum|terms| whatever the order.  mean = sum * (1/count) adds two roundings of the reciprocal / product (4 u).
# The centred sum of squares of d = x - mean_k (mean_k = mean + dm) equals sum (x - mean)^2 + rows dm^2 exactly; each term
# adds 3 u relative and the chain L u, so var_k is within (L + 6) u (var + dm^2) + dm^2 of var.  rstd = rsqrt(var_k + eps)
# is then within |d var| / (2 (var + eps)) + RSQRT_APPROX + 2 u relative.  All bounds below are twice these.
EPS = 1e-5


def bn_chain(rows):
    return math.ceil(min(rows, 128) / 8) + 8 + math.ceil(rows / 128) + 3


def bn_inputs(rows, C, seed, cancel):
    """[rows, C] bf16: per-channel means in [-1, 1] and std in [0.5, 2.5]; channel 0 constant (variance 0); with `cancel`,
    channel 1 has mean / std = 300 (30 +- 0.1)."""
    _seed(seed)
    m = torch.rand(C, device="cuda", generator=gen()) * 2 - 1
    s = torch.rand(C, device="cuda", generator=gen()) * 2 + 0.5
    x = torch.randn(rows, C, device="cuda", generator=gen()) * s + m
    x[:, 0] = 0.75
    if cancel:
        x[:, 1] = 30 + 0.1 * torch.randn(rows, device="cuda", generator=gen())
    return x.to(torch.bfloat16)


def bn_ref(x2d, gamma, beta, relu):
    xd = x2d.double()
    mean = xd.mean(0)
    var = (xd - mean).pow(2).mean(0)
    rstd = (var + EPS).rsqrt()
    y = (xd - mean) * rstd * gamma.double() + beta.double()
    return (y.clamp_min(0) if relu else y), mean, var, rstd


def bn_fwd_bounds(x2d, gamma, beta, mean, var, rstd, y, L):
    xd = x2d.double()
    d_mean = L * U32 * xd.abs().mean(0) + 4 * U32 * mean.abs()
    d_var = (L + 6) * U32 * (var + d_mean ** 2) + d_mean ** 2
    rel_rstd = d_var / (2 * (var + EPS)) + RSQRT_APPROX + 2 * U32
    xc = (xd - mean).abs()
    err = gamma.double().abs() * rstd * (xc * rel_rstd + d_mean) + 3 * U32 * y.abs() + U32 * beta.double().abs()
    return 2 * d_mean + FTZ, 2 * rel_rstd * rstd, bf16_tol(y, 2 * err)


def check_bn_fwd(what, x2d, gamma, beta, relu, y, mean, rstd):
    y_ref, m_ref, v_ref, r_ref = bn_ref(x2d, gamma, beta, relu)
    t_mean, t_rstd, t_y = bn_fwd_bounds(x2d, gamma, beta, m_ref, v_ref, r_ref, y_ref, bn_chain(x2d.shape[0]))
    close(f"{what}: mean", mean, m_ref, t_mean)
    close(f"{what}: rstd", rstd, r_ref, t_rstd)
    close(f"{what}: y", y, y_ref, t_y)


def bn_bwd_ref(dy2d, x2d, gamma, mean, rstd, L):
    """dx = g rstd (dy - mean(dy) - xh mean(dy xh)) from the fp32 mean / rstd the kernel is given.  xh carries 2 u relative;
    the two sums carry (L + 3) u sum|terms|; the apply's own arithmetic cancels terms as large as |dy|, |mean(dy)| and
    |xh mean(dy xh)| (6 u of each).  dgamma = sum dy xh, dbeta = sum dy within (L + 3) u of their |terms|."""
    n = x2d.shape[0]
    dyd, xh = dy2d.double(), (x2d.double() - mean.double()) * rstd.double()
    m1, m2 = dyd.mean(0), (dyd * xh).mean(0)
    r, g = rstd.double(), gamma.double()
    ref = g * r * (dyd - m1 - xh * m2)
    err = g.abs() * r * (6 * U32 * (dyd.abs() + m1.abs() + (xh * m2).abs())
                         + (L + 4) * U32 * (dyd.abs().mean(0) + xh.abs() * (dyd * xh).abs().mean(0)))
    t_dg = 2 * (L + 3) * U32 * (dyd * xh).abs().sum(0) + FTZ
    t_db = 2 * (L + 3) * U32 * dyd.abs().sum(0) + FTZ
    return ref, bf16_tol(ref, 2 * err), (dyd * xh).sum(0), t_dg, dyd.sum(0), t_db, n


def bn_params(C):
    gamma = torch.rand(C, device="cuda", generator=gen()) + 0.5
    beta = torch.randn(C, device="cuda", generator=gen())
    return gamma, beta


def nchw(x2d, N, H, W):
    """[N*H*W, C] rows -> [N, C, H, W] view of channels_last memory."""
    return x2d.view(N, H, W, -1).permute(0, 3, 1, 2)


BN_ROWS = [(1, 1, 1), (1, 1, 7), (1, 127, 1), (2, 8, 8), (1, 3, 43), (4, 112, 112)]     # N, H, W: 1, 7, 127, 128, 129, 50176 rows


@pytest.mark.parametrize("N,H,W", BN_ROWS, ids=[f"rows{n * h * w}" for n, h, w in BN_ROWS])
@pytest.mark.parametrize("C", [8, 264, 5120])
def test_batchnorm_fwd_bwd(ops, C, N, H, W):
    rows = N * H * W
    x2d = bn_inputs(rows, C, seed=C + rows, cancel=rows == 50176)
    gamma, beta = bn_params(C)
    x = nchw(x2d, N, H, W)
    for relu in (False, True):
        y, mean, rstd = launched(ops, ops.batchnorm_fwd, x, gamma, beta, EPS, relu)
        check_bn_fwd(f"rows={rows} C={C} relu={relu}", x2d, gamma, beta, relu, y.permute(0, 2, 3, 1).reshape(rows, C), mean, rstd)
    _, m_ref, _, r_ref = bn_ref(x2d, gamma, beta, False)
    mean, rstd = m_ref.float(), r_ref.float()
    dy2d = randn(rows, C)
    dx, dg, db = launched(ops, ops.batchnorm_bwd, nchw(dy2d, N, H, W), x, gamma, mean, rstd)
    ref, t_dx, dg_ref, t_dg, db_ref, t_db, _ = bn_bwd_ref(dy2d, x2d, gamma, mean, rstd, bn_chain(rows))
    close(f"dx rows={rows} C={C}", dx.permute(0, 2, 3, 1).reshape(rows, C), ref, t_dx)
    close("dgamma", dg, dg_ref, t_dg)
    close("dbeta", db, db_ref, t_db)


class ShardedAllSum:
    """One-GPU stand-in for the all-reduce of split-phase BatchNorm.  Each shard's call is run once per pass over the shards;
    the j-th `allsum` call of a shard records its local tensor until call j has been seen on every shard, and from the next
    pass on writes the total over the shards into it.  Passes repeat until every call returns totals, so each phase sees
    exactly what a real all-reduce would have given it."""

    def __init__(self, shards):
        self.shards, self.totals, self.seen = shards, [], {}

    def run(self, fn):
        while True:
            self.seen, outs = {}, []
            for s in range(self.shards):
                self.call = 0
                outs.append(fn(s, self))
            j = len(self.totals)
            if j not in self.seen:
                return outs
            self.totals.append(sum(self.seen[j]))

    def __call__(self, t):
        j = self.call
        self.call += 1
        if j < len(self.totals):
            t.copy_(self.totals[j])
        else:
            self.seen.setdefault(j, []).append(t.clone())
        return t


# N (divisible by 2 and 3), H, W: 6, 126 and 18,816 rows over the whole batch
SYNC_ROWS = [(6, 1, 1), (6, 3, 7), (6, 56, 56)]


@pytest.mark.parametrize("shards", [2, 3])
@pytest.mark.parametrize("N,H,W", SYNC_ROWS, ids=[f"rows{n * h * w}" for n, h, w in SYNC_ROWS])
@pytest.mark.parametrize("C", [8, 264, 5120])
def test_batchnorm_split_phases_one_gpu(ops, C, N, H, W, shards):
    """batchnorm_fwd_synced / batchnorm_bwd_synced over k shards of one batch: the concatenated outputs equal BatchNorm of
    the whole batch within the bounds above; the returned dgamma / dbeta are each shard's own partial sums."""
    rows = N * H * W
    x2d = bn_inputs(rows, C, seed=C + rows + shards, cancel=rows > 10000)
    gamma, beta = bn_params(C)
    per = rows // shards
    part = lambda t, s: nchw(t[s * per:(s + 1) * per], N // shards, H, W)
    for relu in (False, True):
        outs = ShardedAllSum(shards).run(
            lambda s, allsum: launched(ops, ops.batchnorm_fwd_synced, part(x2d, s), gamma, beta, EPS, allsum, shards, relu=relu))
        y = torch.cat([o[0].permute(0, 2, 3, 1).reshape(per, C) for o in outs])
        for s, (_, mean, rstd) in enumerate(outs):
            check_bn_fwd(f"{shards} shards, shard {s}, rows={rows} C={C} relu={relu}", x2d, gamma, beta, relu, y, mean, rstd)
    _, m_ref, _, r_ref = bn_ref(x2d, gamma, beta, False)
    mean, rstd = m_ref.float(), r_ref.float()
    dy2d = randn(rows, C)
    outs = ShardedAllSum(shards).run(
        lambda s, allsum: launched(ops, ops.batchnorm_bwd_synced, part(dy2d, s), part(x2d, s), gamma, mean, rstd, allsum, shards))
    dx = torch.cat([o[0].permute(0, 2, 3, 1).reshape(per, C) for o in outs])
    ref, t_dx, *_ = bn_bwd_ref(dy2d, x2d, gamma, mean, rstd, bn_chain(rows))
    close(f"dx {shards} shards rows={rows} C={C}", dx, ref, t_dx)
    for s, (_, dg, db) in enumerate(outs):
        _, _, dg_ref, t_dg, db_ref, t_db, _ = bn_bwd_ref(dy2d[s * per:(s + 1) * per], x2d[s * per:(s + 1) * per], gamma, mean,
                                                         rstd, bn_chain(per))
        close(f"dgamma of shard {s}", dg, dg_ref, t_dg)
        close(f"dbeta of shard {s}", db, db_ref, t_db)


# ============================================================================================== C. pooling, elementwise, SGD
def maxpool_ref(x, dy, k, s, p):
    """fp64 max pool and its gradient with the first maximum of a window (row-major scan) taking dy, on -inf padding."""
    N, C, H, W = x.shape
    xp = F.pad(x.double(), (p, p, p, p), value=float("-inf"))
    u = F.unfold(xp, k, stride=s).view(N, C, k * k, -1)                    # [N, C, taps, L]
    idx = u.argmax(2)                                                       # first maximal tap
    y = u.gather(2, idx.unsqueeze(2)).squeeze(2)
    Ho, Wo = dy.shape[2], dy.shape[3]
    L = Ho * Wo
    lo = torch.arange(L)
    rr = (lo // Wo) * s + idx // k
    cc = (lo % Wo) * s + idx % k
    flat = (rr * (W + 2 * p) + cc).view(N * C, L)
    dxp = torch.zeros(N * C, (H + 2 * p) * (W + 2 * p), dtype=torch.float64)
    dxp.scatter_add_(1, flat, dy.double().reshape(N * C, L))
    dx = dxp.view(N, C, H + 2 * p, W + 2 * p)[:, :, p:p + H, p:p + W]
    return y.view(N, C, Ho, Wo), dx


POOL_CASES = [(13, 9, 3, 2, 1), (14, 10, 3, 2, 1), (7, 9, 2, 2, 0), (8, 5, 3, 1, 1), (11, 7, 2, 3, 0), (2, 3, 3, 2, 1)]


@pytest.mark.parametrize("H,W,k,s,p", POOL_CASES, ids=[f"{h}x{w}_k{k}s{s}p{p}" for h, w, k, s, p in POOL_CASES])
def test_maxpool_exact(ops, H, W, k, s, p):
    """Post-ReLU-like integers in {0, 1, 2} (ties in almost every window), integer dy: both directions bit for bit.  k2 s3
    leaves rows / columns in no window; their gradient must be exactly 0."""
    _seed(H * W + k)
    N, C = 2, 16
    x = ints(N, C, H, W, lo=-2, hi=2).clamp_min(0).contiguous(memory_format=torch.channels_last)
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    dy = ints(N, C, Ho, Wo).contiguous(memory_format=torch.channels_last)
    y = launched(ops, ops.maxpool2d_fwd, x, k, s, p)
    y_ref, dx_ref = maxpool_ref(x.cpu(), dy.cpu(), k, s, p)
    exact("maxpool fwd", y, y_ref.float().to(torch.bfloat16))
    dx = launched(ops, ops.maxpool2d_bwd, dy, x, y, k, s, p)
    exact("maxpool bwd", dx, dx_ref.float().to(torch.bfloat16))
    if s > k:
        covered = torch.zeros(H, W, dtype=torch.bool)
        for ho in range(Ho):
            for wo in range(Wo):
                covered[max(0, ho * s - p):ho * s - p + k, max(0, wo * s - p):wo * s - p + k] = True
        assert not bool(covered.all())
        assert bool((dx.cpu()[:, :, ~covered].view(torch.int16) == 0).all())


@pytest.mark.parametrize("HW", [(1, 1), (7, 7), (56, 56)])
def test_global_avgpool(ops, HW):
    """Forward: one thread adds the HW values of its channel in sequence (HW - 1 roundings) and multiplies by 1/HW
    (2 roundings): within (HW + 2) u mean|x| of the fp64 mean before the bf16 store.  Backward: dy * (1/HW), 3 u relative."""
    H, W = HW
    _seed(H)
    N, C = 3, 264
    x = randn(N, C, H, W, scale=2.0).contiguous(memory_format=torch.channels_last) + 0.5
    y = launched(ops, ops.global_avgpool_fwd, x)
    ref = x.double().mean((2, 3))
    close(f"gap fwd HW={H * W}", y, ref, bf16_tol(ref, 2 * (H * W + 2) * U32 * x.double().abs().mean((2, 3))))
    dy = randn(N, C)
    dx = launched(ops, ops.global_avgpool_bwd, dy, (N, C, H, W))
    ref = (dy.double() / (H * W)).view(N, C, 1, 1).expand(N, C, H, W)
    close(f"gap bwd HW={H * W}", dx, ref, bf16_tol(ref, 6 * U32 * ref.abs()))


def test_ew_native_exact(ops):
    """relu, relu backward (a where the forward output b > 0) and add: bf16 -> fp32 -> one bf16 store; the fp32 sum of two
    bf16 values of these magnitudes is exact, so all three are bit for bit."""
    _seed(40)
    shape = (3, 40, 13, 21)
    a, b = randn(*shape, scale=3.0), randn(*shape, scale=3.0)
    b.view(-1)[::7] = 0
    for layout in (torch.contiguous_format, torch.channels_last):
        aa, bb = a.contiguous(memory_format=layout), b.contiguous(memory_format=layout)
        exact("relu", launched(ops, ops.ew_native, "relu", aa), torch.where(aa > 0, aa, torch.zeros_like(aa)))
        exact("relu_bwd", launched(ops, ops.ew_native, "relu_bwd", aa, bb), torch.where(bb > 0, aa, torch.zeros_like(aa)))
        exact("add", launched(ops, ops.ew_native, "add", aa, bb), (aa.float() + bb.float()).to(torch.bfloat16))


@pytest.mark.parametrize("with_copy", [False, True])
def test_sgd_step(ops, with_copy):
    """p - lr g gscale in fp32 (two products, one subtraction, possibly contracted to an FMA): within u |p'| + 2 u |lr g gs|,
    doubled; n = 4k + 3 leaves a tail.  The bf16 copy equals master.to(bf16) bit for bit."""
    _seed(41)
    n, lr, gs = 4 * 250_000 + 3, 0.0125, 0.37
    p0 = torch.randn(n, device="cuda", generator=gen())
    g = torch.randn(n, device="cuda", generator=gen()) * 3
    p = p0.clone()
    pb = torch.empty(n, device="cuda", dtype=torch.bfloat16) if with_copy else None
    launched(ops, ops.sgd_step, p, g, pb, lr, gs)
    upd = float(torch.tensor(lr, dtype=torch.float32)) * g.double() * float(torch.tensor(gs, dtype=torch.float32))
    ref = p0.double() - upd
    close("sgd", p, ref, 2 * (U32 * ref.abs() + 2 * U32 * upd.abs()) + FTZ)
    if with_copy:
        exact("sgd bf16 copy", pb, p.to(torch.bfloat16))


# ============================================================================================== D. whole Wide-ResNet steps
# Bound on each parameter's relative gradient error ||g_gpu - g_cpu|| / ||g_cpu|| against the fp32 CPU executor, keyed by
# layer kind.  These are measured, not derived: on an H100 80GB HBM3 at 700 W the largest values over the steps at image
# 224 / batch 2 and the step at image 200 / batch 1 were conv w 1.37, bn g 1.65, bn b 1.55, fc w 8.7e-2 and fc b 5.9e-2,
# and each bound is about twice that.  fc b grows from step to step and varies from run to run (the fp32 atomics round
# differently each time): 1.8e-3 to 1.9e-3 in step 1, 6.8e-3 to 8.6e-3 in step 2, 2.2e-2 and 5.9e-2 in step 3.
#
# Below the classifier these bounds only catch gross failures (NaN, a layer's gradient missing or blown up).  The reason is
# the model, not the kernels: at initialisation the Wide-ResNet step is chaotic in its weights.  The fp32 CPU executor
# itself, run once with the fp32 master weights and once with the same weights rounded to bf16 (which is what the GPU
# computes with), gives gradients 1.2 apart in relative norm for every convolution and BatchNorm below the last block
# (model 0, image 64, batch 2).  No bf16 step can agree with the fp32 one more closely than that.  Element-wise precision
# of every kernel the step runs is checked in sections A to C; this section checks that the whole step runs on those
# kernels (no torch fallback), that its loss-side gradients agree, and that the AdamW update of its own gradient is right.
WRN_GRAD_TOL = {"conv/w": 3.0, "bn/g": 3.0, "bn/b": 3.0, "fc/w": 0.2, "fc/b": 0.12}


def wrn_kind(name):
    if name.endswith("/bn/g"):
        return "bn/g"
    if name.endswith("/bn/b"):
        return "bn/b"
    if name.startswith("fc/"):
        return name
    assert name.endswith("/w"), name
    return "conv/w"


def wrn_grad_tol(name):
    return WRN_GRAD_TOL[wrn_kind(name)]


@pytest.fixture
def no_torch_conv_fallback(monkeypatch):
    """Convolution, BatchNorm and max pool have torch fallbacks in the executor; make any of them fail on a CUDA tensor."""
    def guard(mod, name):
        real = getattr(mod, name)

        def fn(*args, **kw):
            if any(isinstance(t, torch.Tensor) and t.is_cuda for t in list(args) + list(kw.values())):
                raise AssertionError(f"torch {name} ran on the GPU instead of our kernel")
            return real(*args, **kw)
        monkeypatch.setattr(mod, name, fn)
    for name in ("conv2d", "batch_norm", "max_pool2d"):
        guard(torch.nn.functional, name)
    for name in ("conv2d_input", "conv2d_weight"):
        guard(torch.nn.grad, name)


def wrn_pair(cfg, use_cuda_graph):
    from tepdist_b200.models.wide_resnet import build_wide_resnet_graph
    from tepdist_b200.runtime.executor import Executor
    g = build_wide_resnet_graph(cfg)
    gpu = Executor(g, torch.device("cuda", 0), seed=0, use_cuda_graph=use_cuda_graph)
    cpu = Executor(g, torch.device("cpu"), seed=0)
    sched = lambda step: 1e-3 * min(1.0, step / 4)
    gpu.set_lr_schedule(sched)
    cpu.set_lr_schedule(sched)
    torch.manual_seed(0)
    img = torch.randn(cfg.batch, 3, cfg.image, cfg.image).to(torch.bfloat16).float()
    lab = torch.randint(0, cfg.classes, (cfg.batch,), dtype=torch.int32)
    return gpu, cpu, {"images": img.cuda(), "labels": lab.cuda()}, {"images": img, "labels": lab}


def wrn_report(worst):
    by_kind = {}
    for name, rel in worst.items():
        k = wrn_kind(name)
        by_kind[k] = max(by_kind.get(k, 0.0), rel)
    print("  largest relative error by kind: " + ", ".join(f"{k} {v:.2e}" for k, v in sorted(by_kind.items())))


def test_wide_resnet_steps_gradient_by_gradient(ops, no_torch_conv_fallback):
    """Model type 0 at image 224, batch 2: step 1 eager, step 2 CUDA-graph capture + replay, step 3 replay."""
    from tepdist_b200.models.wide_resnet import WideResNetConfig
    gpu, cpu, fg, fc = wrn_pair(WideResNetConfig(model_type=0, batch=2, image=224), use_cuda_graph=True)
    t0 = time.perf_counter()
    for s, label in enumerate(("WRN-0 224 step 1 (eager)", "WRN-0 224 step 2 (capture + replay)", "WRN-0 224 step 3 (replay)")):
        n0 = ops.launch_count()
        wrn_report(step_checks(gpu, cpu, fg, fc, label, tol=wrn_grad_tol))
        assert ops.launch_count() > n0
        assert (gpu._graph is None) == (s == 0)
    print(f"WRN-0 224 steps with oracle: {time.perf_counter() - t0:.1f} s")


def test_wide_resnet_odd_sizes_step_gradient_by_gradient(ops, no_torch_conv_fallback):
    """Model type 0 at image 200, batch 1: 100 -> 50 -> 25 -> 13 -> 7, so the stride-2 convolutions and shortcuts run on
    odd sizes inside the real graph.  One eager step."""
    from tepdist_b200.models.wide_resnet import WideResNetConfig
    gpu, cpu, fg, fc = wrn_pair(WideResNetConfig(model_type=0, batch=1, image=200), use_cuda_graph=False)
    wrn_report(step_checks(gpu, cpu, fg, fc, "WRN-0 200 step 1 (eager)", tol=wrn_grad_tol))
