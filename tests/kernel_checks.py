"""Numerics + timing checks for the sm_90a kernels against plain-PyTorch fp32 references.

Used two ways: (1) `python tests/kernel_checks.py [names...]` on a GPU box runs every check in its own
subprocess with a timeout (so one hung kernel cannot take the whole run down) and writes
gpurun_out/kernel_checks.json; (2) tests/test_kernels_gpu.py imports the check functions under pytest.
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def _time_ms(fn, iters=20, warmup=5):
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


# ------------------------------------------------------------------------------------------ GEMM
def check_gemm_layouts():
    from tepdist_b200 import ops
    out = {}
    torch.manual_seed(0)
    for (M, N, K) in [(256, 256, 128), (384, 640, 320), (1024, 1024, 1024), (200, 136, 72)]:
        for a_mn in (False, True):
            for b_mn in (False, True):
                if a_mn and M % 8:
                    continue
                A = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
                B = torch.randn(K, N, device="cuda", dtype=torch.bfloat16)
                a = A.t().contiguous() if a_mn else A
                b = B if b_mn else B.t().contiguous()
                ref = A.float() @ B.float()
                for bn in (128, 256):
                    d = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, block_n=bn)
                    torch.cuda.synchronize()
                    err = _rel_err(d, ref)
                    out[f"{M}x{N}x{K}_a{int(a_mn)}b{int(b_mn)}_bn{bn}"] = err
                    assert err < 1e-2, (M, N, K, a_mn, b_mn, bn, err)
    return out


def check_gemm_epilogues():
    from tepdist_b200 import ops
    out = {}
    torch.manual_seed(1)
    M, N, K = 512, 768, 256
    A = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    W = torch.randn(N, K, device="cuda", dtype=torch.bfloat16) * 0.05
    bias = torch.randn(N, device="cuda", dtype=torch.float32)
    res = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
    ref = A.float() @ W.float().t() + bias
    d = ops.gemm(A, W, bias=bias)
    out["bias"] = _rel_err(d, ref)
    d = ops.gemm(A, W, bias=bias.bfloat16())
    out["bias_bf16"] = _rel_err(d, A.float() @ W.float().t() + bias.bfloat16().float())
    d = ops.gemm(A, W, bias=bias, act="gelu")
    out["gelu"] = _rel_err(d, torch.nn.functional.gelu(ref, approximate="tanh"))
    d = ops.gemm(A, W, bias=bias, residual=res)
    out["residual"] = _rel_err(d, ref + res.float())
    d = ops.gemm(A, W, out_dtype=torch.float32, alpha=0.5)
    out["fp32_alpha"] = _rel_err(d, 0.5 * (A.float() @ W.float().t()))
    acc = torch.ones(M, N, device="cuda", dtype=torch.float32)
    ops.gemm(A, W, out=acc, accumulate=True, split_k=1)
    out["accumulate"] = _rel_err(acc, 1.0 + A.float() @ W.float().t())
    acc = torch.zeros(M, N, device="cuda", dtype=torch.float32)
    ops.gemm(A, W, out=acc, accumulate=True, split_k=4)
    out["splitk4"] = _rel_err(acc, A.float() @ W.float().t())
    # wgrad-style: dW[N,K] += dY[M,N]^T @ X[M,K]   (both operands MN-major, split-K over tokens)
    T = 2048
    dY = torch.randn(T, N, device="cuda", dtype=torch.bfloat16)
    X = torch.randn(T, K, device="cuda", dtype=torch.bfloat16)
    acc = torch.zeros(N, K, device="cuda", dtype=torch.float32)
    ops.gemm(dY, X, a_mn=True, b_mn=True, out=acc, accumulate=True)
    out["wgrad"] = _rel_err(acc, dY.float().t() @ X.float())
    # stream-K scheduling (split_k=-1) on tile counts that do not divide the SM count, incl. ragged edges, + bias on the
    # leading unit only; and the explicit data-parallel schedule for comparison
    for (Ns, Ks, Ts) in [(3072, 1024, 4096), (1024, 1024, 4096), (1000, 520, 1096), (384, 256, 8192)]:
        dYs = torch.randn(Ts, Ns, device="cuda", dtype=torch.bfloat16)
        Xs = torch.randn(Ts, Ks, device="cuda", dtype=torch.bfloat16)
        refs = dYs.float().t() @ Xs.float()
        for sk in (-1, 1):
            acc = torch.ones(Ns, Ks, device="cuda", dtype=torch.float32)
            ops.gemm(dYs, Xs, a_mn=True, b_mn=True, out=acc, accumulate=True, split_k=sk)
            out[f"streamk{sk}_{Ns}x{Ks}x{Ts}"] = _rel_err(acc, 1.0 + refs)
    bs = torch.randn(N, device="cuda", dtype=torch.float32)
    acc = torch.zeros(M, N, device="cuda", dtype=torch.float32)
    ops.gemm(A, W, bias=bs, out=acc, accumulate=True, split_k=-1)
    out["streamk_bias"] = _rel_err(acc, A.float() @ W.float().t() + bs)
    # dual-output GELU (pre-activation + activation in one pass) and fused GELU backward on a dgrad-layout GEMM
    pre, act = torch.empty(M, N, device="cuda", dtype=torch.bfloat16), torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(A, W, bias=bias, act="gelu", out=pre, out2=act)
    out["gelu_dual_pre"] = _rel_err(pre, ref)
    out["gelu_dual_act"] = _rel_err(act, torch.nn.functional.gelu(ref, approximate="tanh"))
    dz = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
    Wd = torch.randn(N, K, device="cuda", dtype=torch.bfloat16) * 0.05     # dgrad: dx[M,K] = dz[M,N] @ Wd[N,K]
    f = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    fr = f.float().requires_grad_(True)
    torch.nn.functional.gelu(fr, approximate="tanh").backward(dz.float() @ Wd.float())
    d = ops.gemm(dz, Wd, b_mn=True, act="gelu_bwd", aux=f)
    out["gelu_bwd_fused"] = _rel_err(d, fr.grad)
    # batched
    Ab = torch.randn(6, 256, 64, device="cuda", dtype=torch.bfloat16)
    Bb = torch.randn(6, 384, 64, device="cuda", dtype=torch.bfloat16)
    d = ops.gemm(Ab, Bb)
    out["batched"] = _rel_err(d, torch.matmul(Ab.float(), Bb.float().transpose(1, 2)))
    torch.cuda.synchronize()
    for k, v in out.items():
        assert v < 1e-2, (k, v)
    return out


def check_gemm_perf():
    from tepdist_b200 import ops
    out = {}
    for (M, N, K) in [(8192, 8192, 8192), (4096, 4096, 1024), (4096, 1024, 4096), (4096, 3072, 1024), (4096, 50304, 1024)]:
        A = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
        W = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
        for bn in (128, 256):
            ms = _time_ms(lambda: ops.gemm(A, W, block_n=bn))
            out[f"ours_{M}x{N}x{K}_bn{bn}_tflops"] = 2.0 * M * N * K / ms / 1e9
        ms = _time_ms(lambda: torch.matmul(A, W.t()))
        out[f"cublas_{M}x{N}x{K}_tflops"] = 2.0 * M * N * K / ms / 1e9
    # wgrad shape with split-K
    T, N, K = 4096, 1024, 4096
    dY = torch.randn(T, N, device="cuda", dtype=torch.bfloat16)
    X = torch.randn(T, K, device="cuda", dtype=torch.bfloat16)
    acc = torch.zeros(N, K, device="cuda", dtype=torch.float32)
    ms = _time_ms(lambda: ops.gemm(dY, X, a_mn=True, b_mn=True, out=acc, accumulate=True))
    out["ours_wgrad_4096tok_1024x4096_tflops"] = 2.0 * T * N * K / ms / 1e9
    ms = _time_ms(lambda: torch.matmul(dY.t(), X))
    out["cublas_wgrad_tflops"] = 2.0 * T * N * K / ms / 1e9
    # the 256-wide tile schedule and cuBLAS on the forward and dgrad shapes
    for (M, N, K, bmn) in [(4096, 3072, 1024, False), (4096, 1024, 1024, False), (4096, 4096, 1024, False), (4096, 1024, 4096, False),
                           (4096, 1024, 3072, True), (4096, 1024, 4096, True), (4096, 4096, 1024, True)]:
        A = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
        W = torch.randn(K, N, device="cuda", dtype=torch.bfloat16) if bmn else torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
        tag = f"{M}x{N}x{K}{'_bmn' if bmn else ''}"
        ms = _time_ms(lambda: ops.gemm(A, W, b_mn=bmn, block_n=256))
        out[f"cta1_{tag}_tflops"] = 2.0 * M * N * K / ms / 1e9
        ms = _time_ms(lambda: torch.matmul(A, W if bmn else W.t()))
        out[f"cublas_{tag}_tflops"] = 2.0 * M * N * K / ms / 1e9
    # wave-quantisation probe: 33 m-blocks x {4, 16} n-blocks = exact multiples of 132 tiles vs the 32 m-block shapes
    for (M, N, K) in [(4224, 1024, 4096), (4224, 4096, 1024), (4224, 3072, 1024)]:
        A = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
        W = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
        ms = _time_ms(lambda: ops.gemm(A, W, block_n=256))
        out[f"probe_cta1_{M}x{N}x{K}_tflops"] = 2.0 * M * N * K / ms / 1e9
        ms = _time_ms(lambda: torch.matmul(A, W.t()))
        out[f"probe_cublas_{M}x{N}x{K}_tflops"] = 2.0 * M * N * K / ms / 1e9
    # stream-K vs the data-parallel / split-K schedule on the four GPT-2 345M weight-gradient shapes (4096 tokens)
    for (N, K) in [(3072, 1024), (1024, 1024), (4096, 1024), (1024, 4096)]:
        dY = torch.randn(T, N, device="cuda", dtype=torch.bfloat16)
        X = torch.randn(T, K, device="cuda", dtype=torch.bfloat16)
        acc = torch.zeros(N, K, device="cuda", dtype=torch.float32)
        ms = _time_ms(lambda: ops.gemm(dY, X, a_mn=True, b_mn=True, out=acc, accumulate=False, split_k=1))
        out[f"wgrad_{N}x{K}_plainstore_tflops"] = 2.0 * T * N * K / ms / 1e9
        for tag, sk in (("streamk", -1), ("dp", 1)):
            ms = _time_ms(lambda: ops.gemm(dY, X, a_mn=True, b_mn=True, out=acc, accumulate=True, split_k=sk))
            out[f"wgrad_{N}x{K}_{tag}_tflops"] = 2.0 * T * N * K / ms / 1e9
        ms = _time_ms(lambda: torch.matmul(dY.t(), X))
        out[f"wgrad_{N}x{K}_cublas_tflops"] = 2.0 * T * N * K / ms / 1e9
    return out


def check_conv():
    """NHWC im2col / col2im kernels + wgmma GEMMs vs torch (cuDNN) convolutions in fp32 on the same bf16 inputs."""
    import torch.nn.functional as F
    from tepdist_b200 import ops
    out = {}
    torch.manual_seed(3)
    cases = [  # N, Cin, H, Cout, k, stride, pad
        (4, 64, 56, 160, 1, 1, 0), (4, 160, 56, 320, 3, 1, 1), (4, 320, 28, 640, 3, 2, 1), (4, 256, 56, 512, 1, 2, 0),
        (4, 3, 224, 64, 7, 2, 3), (4, 640, 7, 1280, 3, 1, 1), (2, 1280, 7, 2560, 1, 1, 0),
    ]
    for (N, C, H, Co, k, st, pd) in cases:
        x = torch.randn(N, C, H, H, device="cuda", dtype=torch.bfloat16)
        w = (torch.randn(Co, C, k, k, device="cuda") * (2.0 / (C * k * k)) ** 0.5).to(torch.bfloat16)
        tag = f"N{N}C{C}H{H}Co{Co}k{k}s{st}"
        y = ops.conv2d_fwd(x, w, st, pd)
        ref = F.conv2d(x.float(), w.float(), stride=st, padding=pd)
        out[f"fwd_{tag}"] = _rel_err(y, ref)
        dy = torch.randn_like(ref).to(torch.bfloat16)
        gw = ops.conv2d_wgrad(dy, x, w.shape, st, pd)
        out[f"wgrad_{tag}"] = _rel_err(gw, torch.nn.grad.conv2d_weight(x.float(), w.shape, dy.float(), stride=st, padding=pd))
        if C % 8 == 0:
            dx = ops.conv2d_dgrad(dy, w, x.shape, st, pd)
            out[f"dgrad_{tag}"] = _rel_err(dx, torch.nn.grad.conv2d_input(x.shape, w.float(), dy.float(), stride=st, padding=pd))
    # BatchNorm (training mode) NHWC kernels vs fp32 torch
    for (N, C, H) in [(4, 320, 28), (4, 64, 112), (2, 1280, 7)]:
        x = (torch.randn(N, C, H, H, device="cuda") * 2.0 + 0.5).to(torch.bfloat16)
        gm, bt = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda")
        y, mean, rstd = ops.batchnorm_fwd(x, gm, bt, 1e-5)
        xf = x.float()
        mu, var = xf.mean((0, 2, 3)), xf.var((0, 2, 3), unbiased=False)
        ref = (xf - mu.view(1, -1, 1, 1)) * torch.rsqrt(var + 1e-5).view(1, -1, 1, 1) * gm.view(1, -1, 1, 1) + bt.view(1, -1, 1, 1)
        out[f"bn_fwd_C{C}H{H}"] = _rel_err(y, ref)
        out[f"bn_mean_C{C}H{H}"] = _rel_err(mean, mu)
        dy = torch.randn_like(ref).to(torch.bfloat16)
        dx, dgm, dbt = ops.batchnorm_bwd(dy, x, gm, mean, rstd)
        xr = xf.clone().requires_grad_(True)
        gr, br = gm.clone().requires_grad_(True), bt.clone().requires_grad_(True)
        F.batch_norm(xr, None, None, gr, br, True, 0.0, 1e-5).backward(dy.float())
        out[f"bn_dx_C{C}H{H}"] = _rel_err(dx, xr.grad)
        out[f"bn_dgamma_C{C}H{H}"] = _rel_err(dgm, gr.grad)
        out[f"bn_dbeta_C{C}H{H}"] = _rel_err(dbt, br.grad)
    for k_, v in out.items():
        assert v < 1.5e-2, (k_, v)
    # timing vs cuDNN (channels_last bf16) on the two dominant Wide-ResNet-250M shapes
    for (N, C, H, Co, k, st, pd) in [(4, 160, 56, 320, 3, 1, 1), (4, 320, 56, 640, 1, 1, 0)]:
        x = torch.randn(N, C, H, H, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
        w = torch.randn(Co, C, k, k, device="cuda", dtype=torch.bfloat16)
        wc = w.contiguous(memory_format=torch.channels_last)
        fl = 2.0 * N * (H // st) ** 2 * Co * C * k * k / 1e9
        out[f"tflops_ours_C{C}k{k}"] = fl / _time_ms(lambda: ops.conv2d_fwd(x, w, st, pd))
        out[f"tflops_cudnn_C{C}k{k}"] = fl / _time_ms(lambda: F.conv2d(x, wc, stride=st, padding=pd))
    return out


# ------------------------------------------------------------------------------------------ elementwise
def check_layernorm():
    from tepdist_b200 import ops
    out = {}
    torch.manual_seed(2)
    for C in (1024, 768, 1600):
        rows = 1000
        x = torch.randn(rows, C, device="cuda", dtype=torch.bfloat16) * 2 + 0.5
        g = torch.randn(C, device="cuda") * 0.1 + 1
        b = torch.randn(C, device="cuda") * 0.1
        y, mean, rstd = ops.layernorm_fwd(x, g, b)
        ref = torch.nn.functional.layer_norm(x.float(), (C,), g, b, 1e-5)
        out[f"fwd_{C}"] = _rel_err(y, ref)
        dy = torch.randn_like(x)
        dg, db = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
        dx = ops.layernorm_bwd(dy, x, g, mean, rstd, dg, db)
        xr = x.float().requires_grad_(True)
        gr, br = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
        torch.nn.functional.layer_norm(xr, (C,), gr, br, 1e-5).backward(dy.float())
        out[f"dx_{C}"] = _rel_err(dx, xr.grad)
        out[f"dgamma_{C}"] = _rel_err(dg, gr.grad)
        out[f"dbeta_{C}"] = _rel_err(db, br.grad)
    for k, v in out.items():
        assert v < 1.5e-2, (k, v)
    return out


def check_gelu_colsum_embed():
    from tepdist_b200 import ops
    out = {}
    torch.manual_seed(3)
    x = torch.randn(512, 4096, device="cuda", dtype=torch.bfloat16)
    out["gelu_fwd"] = _rel_err(ops.gelu_fwd(x), torch.nn.functional.gelu(x.float(), approximate="tanh"))
    dy = torch.randn_like(x)
    xr = x.float().requires_grad_(True)
    torch.nn.functional.gelu(xr, approximate="tanh").backward(dy.float())
    out["gelu_bwd"] = _rel_err(ops.gelu_bwd(dy, x), xr.grad)
    acc = torch.zeros(4096, device="cuda")
    ops.colsum_acc(x, acc)
    out["colsum"] = _rel_err(acc, x.float().sum(0))
    V, C, B, S = 1000, 256, 3, 64
    wte = torch.randn(V, C, device="cuda", dtype=torch.bfloat16)
    wpe = torch.randn(S, C, device="cuda", dtype=torch.bfloat16)
    tok = torch.randint(0, V, (B, S), device="cuda")
    e = ops.embedding_fwd(tok, wte, wpe)
    out["embed_fwd"] = _rel_err(e, wte[tok].float() + wpe.float())
    de = torch.randn(B, S, C, device="cuda", dtype=torch.bfloat16)
    dwte, dwpe = torch.zeros(V, C, device="cuda"), torch.zeros(S, C, device="cuda")
    ops.embedding_bwd(tok, de, dwte, dwpe)
    ref = torch.zeros(V, C, device="cuda").index_add_(0, tok.reshape(-1), de.float().reshape(-1, C))
    out["embed_bwd_wte"] = _rel_err(dwte, ref)
    out["embed_bwd_wpe"] = _rel_err(dwpe, de.float().sum(0))
    for k, v in out.items():
        assert v < 1e-2, (k, v)
    return out


def check_xent_adam():
    from tepdist_b200 import ops
    out = {}
    torch.manual_seed(4)
    T, V, Vp = 256, 50257, 50304
    logits = torch.randn(T, Vp, device="cuda", dtype=torch.bfloat16) * 3
    labels = torch.randint(0, V, (T,), device="cuda")
    lf = logits.float()[:, :V].clone().requires_grad_(True)
    loss_ref = torch.nn.functional.cross_entropy(lf, labels, reduction="sum") / T
    loss_ref.backward()
    total, rows = ops.xent_fwd_bwd(logits, labels, V, 1.0 / T)
    out["loss"] = abs(total.item() - loss_ref.item()) / abs(loss_ref.item())
    out["dlogits"] = _rel_err(logits[:, :V], lf.grad)
    out["dlogits_pad"] = logits[:, V:].float().abs().max().item()
    n = 1 << 20
    p = torch.randn(n, device="cuda")
    g = torch.randn(n, device="cuda")
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    pb = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    pr = p.clone().requires_grad_(True)
    opt = torch.optim.AdamW([pr], lr=1e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    for step in (1, 2, 3):
        pr.grad = g.clone()
        opt.step()
        ops.adamw_step(p, g, m, v, pb, n, 1e-3, 0.9, 0.95, 1e-8, 0.1, step)
    out["adamw"] = _rel_err(p, pr.detach())
    out["adamw_bf16"] = _rel_err(pb, pr.detach())
    assert out["loss"] < 1e-3 and out["dlogits"] < 2e-2 and out["dlogits_pad"] == 0.0, out
    assert out["adamw"] < 1e-5 and out["adamw_bf16"] < 5e-3, out
    return out


# ------------------------------------------------------------------------------------------ attention
def _qkv(B, S, H, D, seed=5):
    torch.manual_seed(seed)
    qkv = torch.randn(B, S, H, 3, D, device="cuda", dtype=torch.bfloat16)  # heads-major fused qkv layout
    return qkv, qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]


def check_attn_fwd():
    from tepdist_b200 import ops
    from tepdist_b200.ops.attention import _ref_fwd
    out = {}
    for (B, S, H, causal) in [(1, 128, 1, True), (2, 256, 3, True), (2, 512, 4, False), (1, 1024, 16, True)]:
        qkv, q, k, v = _qkv(B, S, H, 64)
        o, lse = ops.attention_fwd(q, k, v, causal=causal)
        torch.cuda.synchronize()
        o_ref, lse_ref, _ = _ref_fwd(q, k, v, 1.0 / 8.0, causal)
        tag = f"B{B}S{S}H{H}c{int(causal)}"
        out["o_" + tag] = _rel_err(o, o_ref)
        out["lse_" + tag] = _rel_err(lse, lse_ref)
        assert out["o_" + tag] < 2e-2 and out["lse_" + tag] < 1e-3, out
    return out


def check_attn_d48():
    """Head dims below 64 run on the same kernels through zero padding (ops/attention.py)."""
    from tepdist_b200 import ops
    from tepdist_b200.ops.attention import _ref_fwd
    out = {}
    # 48-wide heads (GPT-MoE): zero-padded to the kernel's head dim, forward and backward
    qkv, q, k, v = _qkv(2, 256, 4, 48)
    o, lse = ops.attention_fwd(q, k, v, causal=True)
    o_ref, lse_ref, _ = _ref_fwd(q, k, v, 48 ** -0.5, True)
    out["o_d48"], out["lse_d48"] = _rel_err(o, o_ref), _rel_err(lse, lse_ref)
    do = torch.randn_like(o)
    dq, dk, dv = ops.attention_bwd(do, q, k, v, o, lse, causal=True)
    qf, kf, vf = (t.float().detach().requires_grad_(True) for t in (q, k, v))
    s = torch.einsum("bshd,bthd->bhst", qf, kf) * 48 ** -0.5
    s = s.masked_fill(~torch.ones(256, 256, dtype=torch.bool, device="cuda").tril(), float("-inf"))
    torch.einsum("bhst,bthd->bshd", torch.softmax(s, -1), vf).backward(do.float())
    out["dq_d48"], out["dk_d48"], out["dv_d48"] = _rel_err(dq, qf.grad), _rel_err(dk, kf.grad), _rel_err(dv, vf.grad)
    assert max(out["o_d48"], out["dq_d48"], out["dk_d48"], out["dv_d48"]) < 3e-2 and out["lse_d48"] < 1e-3, out
    # ragged causal sequence (S = 200) with 64-wide heads: padded to 256 around the kernel
    qkv, q, k, v = _qkv(2, 200, 3, 64)
    o, lse = ops.attention_fwd(q, k, v, causal=True)
    o_ref, lse_ref, _ = _ref_fwd(q, k, v, 0.125, True)
    out["o_s200"], out["lse_s200"] = _rel_err(o, o_ref), _rel_err(lse, lse_ref)
    do = torch.randn_like(o)
    dq, dk, dv = ops.attention_bwd(do, q, k, v, o, lse, causal=True)
    qf, kf, vf = (t.float().detach().requires_grad_(True) for t in (q, k, v))
    s = torch.einsum("bshd,bthd->bhst", qf, kf) * 0.125
    s = s.masked_fill(~torch.ones(200, 200, dtype=torch.bool, device="cuda").tril(), float("-inf"))
    torch.einsum("bhst,bthd->bshd", torch.softmax(s, -1), vf).backward(do.float())
    out["dq_s200"], out["dk_s200"], out["dv_s200"] = _rel_err(dq, qf.grad), _rel_err(dk, kf.grad), _rel_err(dv, vf.grad)
    assert max(out["o_s200"], out["dq_s200"], out["dk_s200"], out["dv_s200"]) < 3e-2 and out["lse_s200"] < 1e-3, out
    return out


def check_attn_bwd():
    from tepdist_b200 import ops
    from tepdist_b200.ops.attention import _ref_fwd
    out = {}
    for (B, S, H, causal) in [(1, 128, 1, True), (2, 256, 3, True), (1, 512, 2, False), (1, 1024, 16, True)]:
        qkv, q, k, v = _qkv(B, S, H, 64)
        o, lse = ops.attention_fwd(q, k, v, causal=causal)
        do = torch.randn_like(o)
        dq, dk, dv = ops.attention_bwd(do, q, k, v, o, lse, causal=causal)
        torch.cuda.synchronize()
        qr, kr, vr = (t.float().detach().clone().requires_grad_(True) for t in (q, k, v))
        s = torch.einsum("bqhd,bkhd->bhqk", qr, kr) / 8.0
        if causal:
            mask = torch.ones(S, S, dtype=torch.bool, device="cuda").tril()
            s = s.masked_fill(~mask, float("-inf"))
        oo = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), vr)
        oo.backward(do.float())
        tag = f"B{B}S{S}H{H}c{int(causal)}"
        out["dq_" + tag] = _rel_err(dq, qr.grad)
        out["dk_" + tag] = _rel_err(dk, kr.grad)
        out["dv_" + tag] = _rel_err(dv, vr.grad)
        for n in ("dq_", "dk_", "dv_"):
            assert out[n + tag] < 3e-2, out
    return out


def check_attn_perf():
    from tepdist_b200 import ops
    out = {}
    B, S, H, D = 4, 1024, 16, 64
    qkv, q, k, v = _qkv(B, S, H, D)
    ms = _time_ms(lambda: ops.attention_fwd(q, k, v))
    fl = 4.0 * B * H * S * S * D / 2
    out["fwd_ms"] = ms
    out["fwd_tflops"] = fl / ms / 1e9
    qc, kc, vc = (t.permute(0, 2, 1, 3).contiguous() for t in (q, k, v))
    ms2 = _time_ms(lambda: torch.nn.functional.scaled_dot_product_attention(qc, kc, vc, is_causal=True))
    out["sdpa_fwd_ms"] = ms2
    try:
        o, lse = ops.attention_fwd(q, k, v)
        do = torch.randn_like(o)
        msb = _time_ms(lambda: ops.attention_bwd(do, q, k, v, o, lse))
        out["bwd_ms"] = msb
        out["bwd_tflops"] = 2.5 * fl / msb / 1e9
    except Exception as e:  # bwd kernel may not be built yet
        out["bwd_error"] = repr(e)
    return out


def check_einsum():
    """ops.einsum (one batched wgmma GEMM per einsum) on the GPT-MoE patterns: forward and gradient equations, both operand
    majors, with and without the layout copies; vs torch.einsum in fp32.  Then throughput of the expert FC vs torch.einsum."""
    from tepdist_b200 import ops
    out = {}
    torch.manual_seed(3)
    G, S, E, C, M, H = 4, 256, 8, 32, 128, 256
    t = {k: (torch.randn(*shape, device="cuda") * 0.5).to(torch.bfloat16) for k, shape in {
        "GSEC": (G, S, E, C), "GSM": (G, S, M), "EGCM": (E, G, C, M), "EMH": (E, M, H), "EGCH": (E, G, C, H), "EHM": (E, H, M)}.items()}
    for eq in ["GSEC,GSM->EGCM", "EGCM,EMH->EGCH", "EGCH,EHM->EGCM", "GSEC,EGCM->GSM", "EGCM,GSM->GSEC", "EGCH,EMH->EGCM",
               "EGCM,EGCH->EMH", "EGCM,EHM->EGCH", "EGCH,EGCM->EHM"]:
        ia, ib = eq.split("->")[0].split(",")
        n0 = ops.launch_count()
        got = ops.einsum(eq, t[ia], t[ib])
        assert ops.launch_count() > n0, eq           # the wgmma GEMM ran, not the torch fallback
        ref = torch.einsum(eq, t[ia].float(), t[ib].float())
        out[eq] = _rel_err(got, ref)
        assert out[eq] < 1e-2, (eq, out[eq])
    # GPT-MoE expert FC1 at the reference shape per GPU under EP-8: 1 local expert x (8 groups x 256 slots) x 768 -> 6144
    x = torch.randn(1, 8, 256, 768, device="cuda", dtype=torch.bfloat16)
    w = torch.randn(1, 768, 6144, device="cuda", dtype=torch.bfloat16)
    fl = 2.0 * 2048 * 768 * 6144
    out["fc1_tflops"] = fl / _time_ms(lambda: ops.einsum("EGCM,EMH->EGCH", x, w)) / 1e9
    out["fc1_torch_tflops"] = fl / _time_ms(lambda: torch.einsum("EGCM,EMH->EGCH", x, w)) / 1e9
    return out


def check_ew():
    """Own elementwise kernels of the conv path (ReLU, ReLU backward, residual add) on contiguous and channels_last tensors."""
    from tepdist_b200 import ops
    out = {}
    torch.manual_seed(5)
    for tag, mk in (("nchw", lambda t: t), ("nhwc", lambda t: t.contiguous(memory_format=torch.channels_last))):
        a = mk(torch.randn(4, 64, 14, 14, device="cuda").to(torch.bfloat16))
        b = mk(torch.randn(4, 64, 14, 14, device="cuda").to(torch.bfloat16))
        n0 = ops.launch_count()
        r = ops.ew_native("relu", a)
        rb = ops.ew_native("relu_bwd", a, r)
        ad = ops.ew_native("add", a, b)
        assert ops.launch_count() - n0 == 3 and r.stride() == a.stride()
        assert torch.equal(r, a.relu()) and torch.equal(rb, a * (r > 0).to(a.dtype))
        out["add_" + tag] = _rel_err(ad, a.float() + b.float())
        assert out["add_" + tag] < 1e-2
    assert ops.ew_native("add", a, b[:, :32]) is None        # shapes differ: caller falls back to the torch op
    return out


def check_moe_routes():
    """Route-table dispatch / combine kernels (ops.moe_gather_scale / moe_combine_sum / moe_route_dots) vs their plain torch
    reference (the CPU branch of the same functions, fp32), with dropped routes; then time vs the dense einsum they replace."""
    from tepdist_b200 import ops
    out = {}
    torch.manual_seed(11)
    G, S, E, C, M, K = 2, 512, 8, 64, 768, 2
    x = torch.randn(G, S, M, device="cuda").to(torch.bfloat16)
    y = torch.randn(E, G, C, M, device="cuda").to(torch.bfloat16)
    re = torch.randint(-1, E, (G, S, K), device="cuda", dtype=torch.int32)
    rc = torch.randint(0, C, (G, S, K), device="cuda", dtype=torch.int32)
    gw = torch.rand(G, S, K, device="cuda") * (re >= 0)
    slot_src = torch.randint(-1, S, (G, E, C), device="cuda", dtype=torch.int32)
    slot_w = torch.rand(G, E, C, device="cuda")
    cpu = lambda t: t.cpu().float() if t.is_floating_point() else t.cpu()
    n0 = ops.launch_count()
    out["gather"] = _rel_err(ops.moe_gather_scale(x, slot_src, slot_w, E, C), ops.moe_gather_scale(cpu(x), cpu(slot_src), cpu(slot_w), E, C).cuda())
    out["combine"] = _rel_err(ops.moe_combine_sum(y, re, rc, gw, S), ops.moe_combine_sum(cpu(y), cpu(re), cpu(rc), cpu(gw), S).cuda())
    out["dots"] = _rel_err(ops.moe_route_dots(x, y, re, rc), ops.moe_route_dots(cpu(x), cpu(y), cpu(re), cpu(rc)).cuda())
    assert ops.launch_count() - n0 == 3
    for k in ("gather", "combine", "dots"):
        assert out[k] < 1e-2, out
    # reference shape per GPU under EP-8 (1 group of 8192 tokens, 8 experts x 256 slots, model 768)
    G, S, E, C, M = 1, 8192, 8, 256, 768
    x = torch.randn(G, S, M, device="cuda").to(torch.bfloat16)
    mask = torch.zeros(G, S, E, C, device="cuda", dtype=torch.bfloat16)
    slot_src = torch.randint(0, S, (G, E, C), device="cuda", dtype=torch.int32)
    slot_w = torch.rand(G, E, C, device="cuda")
    out["gather_us"] = 1e3 * _time_ms(lambda: ops.moe_gather_scale(x, slot_src, slot_w, E, C))
    out["dense_dispatch_einsum_us"] = 1e3 * _time_ms(lambda: ops.einsum("GSEC,GSM->EGCM", mask, x))
    return out


def check_ring_blocks(device="cuda"):
    """Context-parallel attention on ONE device: every virtual rank's ring schedule (parallel/ring_attention.py) run serially
    with the same block kernels and helper kernels -- causal diagonal block, unmasked off-diagonal blocks through the shared-stride
    work buffer, log-sum-exp merge kernel, backward blocks fed the GLOBAL log-sum-exp / output, fp32 dq / dK / dV accumulation and
    pack kernels -- against full-sequence attention (fp32 torch reference)."""
    from tepdist_b200 import ops
    from tepdist_b200.ops.attention import _ref_fwd, attn_merge_, attn_ring_accum_, attn_ring_pack
    out = {}
    torch.manual_seed(3)
    dt = torch.bfloat16 if device == "cuda" else torch.float32
    for (B, S, H, n, causal) in [(2, 512, 3, 4, True), (1, 256, 2, 2, False)]:
        D, L = 64, S // n
        qkv = torch.randn(B, S, H, 3, D, device=device).to(dt)
        do = torch.randn(B, S, H, D, device=device).to(dt)
        q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
        o_ref, lse_ref, _ = _ref_fwd(q.float(), k.float(), v.float(), 1.0 / 8.0, causal)
        g_ref = torch.empty(B, S, H, 3, D, device=device)
        ops.attention_bwd(do.float().cpu(), q.float().cpu(), k.float().cpu(), v.float().cpu(), o_ref.cpu(), lse_ref.cpu(), causal=causal,
                          dqkv_out=(g_cpu := torch.empty(B, S, H, 3, D)))
        g_ref.copy_(g_cpu)
        o_all = torch.empty(B, S, H, D, device=device, dtype=dt)
        lse_all = torch.empty(B, H, S, device=device)
        blk = lambda t, r: t[:, r * L:(r + 1) * L]
        dq_acc = torch.zeros(n, B, L, H, D, device=device)
        kv_acc = torch.zeros(n, B, L, H, 2, D, device=device)
        n0 = ops.launch_count()
        for r in range(n):                              # forward of virtual rank r
            o_acc = torch.empty(B, L, H, D, device=device)
            la, lb = torch.empty(B, H, L, device=device), torch.empty(B, H, L, device=device)
            work = torch.empty(B, L, H, 3, D, device=device, dtype=dt)
            work[:, :, :, 0].copy_(blk(q, r))
            first = True
            for t in range(n):
                j = (r - t) % n
                if causal and j > r:
                    continue
                if t == 0:
                    o_j, lse_j = ops.attention_fwd(blk(q, r), blk(k, r), blk(v, r), causal=causal)
                else:
                    work[:, :, :, 1:].copy_(torch.stack((blk(k, j), blk(v, j)), 3))
                    o_j, lse_j = ops.attention_fwd(work[:, :, :, 0], work[:, :, :, 1], work[:, :, :, 2], causal=False)
                attn_merge_(o_acc, la, lb, o_j.contiguous(), lse_j.contiguous(), first)
                la, lb, first = lb, la, False
            blk(o_all, r).copy_(o_acc)
            lse_all[:, :, r * L:(r + 1) * L].copy_(la)
        for r in range(n):                              # backward of virtual rank r: contributions to dq_r and to dK / dV of block j
            work = torch.empty(B, L, H, 3, D, device=device, dtype=dt)
            work[:, :, :, 0].copy_(blk(q, r))
            part = torch.empty(B, L, H, 3, D, device=device, dtype=dt)
            o_r, lse_r, do_r = blk(o_all, r).contiguous(), lse_all[:, :, r * L:(r + 1) * L].contiguous(), blk(do, r).contiguous()
            for t in range(n):
                j = (r - t) % n
                if causal and j > r:
                    continue
                if t == 0:
                    ops.attention_bwd(do_r, blk(q, r), blk(k, r), blk(v, r), o_r, lse_r, causal=causal, dqkv_out=part)
                else:
                    work[:, :, :, 1:].copy_(torch.stack((blk(k, j), blk(v, j)), 3))
                    ops.attention_bwd(do_r, work[:, :, :, 0], work[:, :, :, 1], work[:, :, :, 2], o_r, lse_r, causal=False, dqkv_out=part)
                attn_ring_accum_(dq_acc[r], kv_acc[j], part)
        g = torch.empty(B, S, H, 3, D, device=device, dtype=dt)
        for r in range(n):
            blk(g, r).copy_(attn_ring_pack(dq_acc[r], kv_acc[r], torch.empty(B, L, H, 3, D, device=device, dtype=dt)))
        if device == "cuda":
            assert ops.launch_count() > n0
        tag = f"S{S}n{n}c{int(causal)}"
        out["o_" + tag] = _rel_err(o_all, o_ref)
        out["lse_" + tag] = _rel_err(lse_all, lse_ref)
        for i, nm in enumerate(("dq", "dk", "dv")):
            out[f"{nm}_{tag}"] = _rel_err(g[:, :, :, i], g_ref[:, :, :, i])
        tol = 3e-2 if device == "cuda" else 1e-5
        for key, e in out.items():
            assert e < tol, (key, e, out)
    return out


def check_pool():
    """Own NHWC pooling kernels vs torch (fp32 math on the same bf16 values, so ties -- plentiful after a ReLU -- must resolve to the
    same element: first maximum in row-major window order)."""
    import torch.nn.functional as F
    from tepdist_b200 import ops
    out = {}
    torch.manual_seed(9)
    for (N, C, H, W, k, s_, p_) in [(4, 64, 56, 56, 3, 2, 1), (2, 32, 15, 17, 2, 2, 0), (2, 16, 9, 9, 3, 1, 1)]:
        x = torch.randn(N, C, H, W, device="cuda").relu().to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        n0 = ops.launch_count()
        y = ops.maxpool2d_fwd(x, k, s_, p_)
        xr = x.float().requires_grad_(True)
        yr = F.max_pool2d(xr, k, s_, p_)
        assert torch.equal(y.float(), yr.detach()), "maxpool fwd"
        dy = torch.randn_like(yr).to(torch.bfloat16)
        dx = ops.maxpool2d_bwd(dy, x, y, k, s_, p_)
        (gr,) = torch.autograd.grad(yr, xr, dy.float())
        assert ops.launch_count() - n0 == 2
        out[f"maxpool_bwd_{H}x{W}k{k}s{s_}"] = _rel_err(dx, gr)
        assert out[f"maxpool_bwd_{H}x{W}k{k}s{s_}"] < 1e-2, out
        assert int(((dx.float() != 0) != (gr != 0)).sum()) == 0, "gradient routed to a different element of a tie"
    x = torch.randn(8, 256, 7, 7, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    g = ops.global_avgpool_fwd(x)
    out["gap"] = _rel_err(g, x.float().mean((2, 3)))
    dyg = torch.randn(8, 256, device="cuda").to(torch.bfloat16)
    dxg = ops.global_avgpool_bwd(dyg, (8, 256, 7, 7))
    out["gap_bwd"] = _rel_err(dxg, (dyg.float() / 49).view(8, 256, 1, 1).expand(8, 256, 7, 7))
    assert out["gap"] < 1e-2 and out["gap_bwd"] < 1e-2, out
    return out


CHECKS = {
    "pool": check_pool,
    "ring_blocks": check_ring_blocks,
    "gemm_layouts": check_gemm_layouts,
    "gemm_epilogues": check_gemm_epilogues,
    "layernorm": check_layernorm,
    "gelu_colsum_embed": check_gelu_colsum_embed,
    "xent_adam": check_xent_adam,
    "attn_fwd": check_attn_fwd,
    "attn_bwd": check_attn_bwd,
    "gemm_perf": check_gemm_perf,
    "conv": check_conv,
    "einsum": check_einsum,
    "moe_routes": check_moe_routes,
    "ew": check_ew,
    "attn_d48": check_attn_d48,
    "attn_perf": check_attn_perf,
}


def _run_one(name: str) -> None:
    res = CHECKS[name]()
    torch.cuda.synchronize()
    print("RESULT " + json.dumps(res))


if __name__ == "__main__":
    if len(sys.argv) >= 3 and sys.argv[1] == "--one":
        _run_one(sys.argv[2])
        sys.exit(0)
    names = [a for a in sys.argv[1:] if a in CHECKS] or list(CHECKS)
    os.makedirs("gpurun_out", exist_ok=True)
    summary = {}
    for n in names:
        t0 = time.time()
        try:
            pr = subprocess.run([sys.executable, __file__, "--one", n], capture_output=True, text=True, timeout=120)
            res = None
            for line in pr.stdout.splitlines():
                if line.startswith("RESULT "):
                    res = json.loads(line[7:])
            summary[n] = {"rc": pr.returncode, "result": res, "secs": round(time.time() - t0, 1),
                          "stderr": pr.stderr[-1500:] if pr.returncode else ""}
        except subprocess.TimeoutExpired:
            summary[n] = {"rc": "timeout", "secs": round(time.time() - t0, 1)}
        print(n, json.dumps(summary[n])[:3000], flush=True)
        with open("gpurun_out/kernel_checks.json", "w") as f:
            json.dump(summary, f, indent=1)
