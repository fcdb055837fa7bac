"""Tiny driver for ncu: launches the flagship GEMM shapes + attention + fused AdamW a few times."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from tepdist_b200 import ops

which = sys.argv[1] if len(sys.argv) > 1 else "gemm"
torch.manual_seed(0)
if which == "gemm":
    M, N, K = 4096, 4096, 1024
    A = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    W = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    for _ in range(12):
        ops.gemm(A, W, block_n=256)
elif which == "attn":
    qkv = torch.randn(4, 1024, 16, 3, 64, device="cuda", dtype=torch.bfloat16)
    q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    for _ in range(6):
        o, lse = ops.attention_fwd(q, k, v)
        ops.attention_bwd(torch.randn_like(o), q, k, v, o, lse)
torch.cuda.synchronize()
if which == "wgrad":
    T, N, K = 4096, 4096, 1024
    dY = torch.randn(T, N, device="cuda", dtype=torch.bfloat16)
    X = torch.randn(T, K, device="cuda", dtype=torch.bfloat16)
    acc = torch.zeros(N, K, device="cuda", dtype=torch.float32)
    for _ in range(12):
        ops.gemm(dY, X, a_mn=True, b_mn=True, out=acc, accumulate=True)
elif which == "adamw":
    n = 64 << 20
    p, g = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    pb = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    for i in range(6):
        ops.adamw_step(p, g, m, v, pb, n, 1e-4, 0.9, 0.999, 1e-8, 0.01, i + 1)
elif which == "ln":
    x = torch.randn(4096, 1024, device="cuda", dtype=torch.bfloat16)
    gmm, bta = torch.ones(1024, device="cuda"), torch.zeros(1024, device="cuda")
    dg, db = torch.zeros(1024, device="cuda"), torch.zeros(1024, device="cuda")
    for _ in range(6):
        y, mean, rstd = ops.layernorm_fwd(x, gmm, bta)
        ops.layernorm_bwd(torch.randn_like(y), x, gmm, mean, rstd, dg, db, dres=x)
torch.cuda.synchronize()
if which == "gemm_step":        # the GEMM kernel's three operand layouts as the GPT-2 step uses them
    M, N, K = 4096, 4096, 1024
    A = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    W = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    Wt = torch.randn(K, N, device="cuda", dtype=torch.bfloat16)
    dY = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
    X = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    acc = torch.empty(N, K, device="cuda", dtype=torch.float32)
    for _ in range(4):
        ops.gemm(A, W)                                                   # forward, bf16 epilogue
        ops.gemm(A, Wt, b_mn=True)                                       # dgrad layout
        ops.gemm(dY, X, a_mn=True, b_mn=True, out=acc, split_k=1)        # weight gradient, fp32 plain stores
    torch.cuda.synchronize()
elif which == "conv":
    x = torch.randn(4, 160, 56, 56, device="cuda", dtype=torch.bfloat16)
    w = torch.randn(320, 160, 3, 3, device="cuda", dtype=torch.bfloat16)
    for _ in range(4):
        y = ops.conv2d_fwd(x, w, 1, 1)
        ops.conv2d_dgrad(y, w, x.shape, 1, 1)
    torch.cuda.synchronize()
if which == "moe":                # GPT-MoE per-GPU shapes under EP-8: route-table gather / combine / dots + the expert FC einsums
    G, S, E, C, M, H = 1, 8192, 8, 256, 768, 6144
    x = torch.randn(G, S, M, device="cuda", dtype=torch.bfloat16)
    y = torch.randn(E, G, C, M, device="cuda", dtype=torch.bfloat16)
    slot_src = torch.randint(0, S, (G, E, C), device="cuda", dtype=torch.int32)
    slot_w = torch.rand(G, E, C, device="cuda")
    re = torch.randint(0, E, (G, S, 2), device="cuda", dtype=torch.int32)
    rc = torch.randint(0, C, (G, S, 2), device="cuda", dtype=torch.int32)
    gw = torch.rand(G, S, 2, device="cuda")
    xe = torch.randn(1, 8, 256, M, device="cuda", dtype=torch.bfloat16)
    wi = torch.randn(1, M, H, device="cuda", dtype=torch.bfloat16)
    for _ in range(4):
        ops.moe_gather_scale(x, slot_src, slot_w, E, C)
        ops.moe_combine_sum(y, re, rc, gw, S)
        ops.moe_route_dots(x, y, re, rc)
        ops.einsum("EGCM,EMH->EGCH", xe, wi)
    torch.cuda.synchronize()
