"""GPU numerics of the 128-wide-head attention kernels and of the paths that reach them: padded head widths 65..128 and a
ragged causal sequence (against the fp64 reference of attention_reference.py), GPT-2 with 128-wide heads, and a traced SDPA
module.  Every case checks that our kernels ran (no torch-math fallback)."""
import pytest
import torch

import attention_reference as ar
import kernel_checks as kc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,S,H,D,causal", [
    (1, 128, 1, 128, True), (2, 256, 3, 128, True), (2, 512, 4, 128, False), (1, 2048, 8, 128, True),
    (2, 256, 2, 80, True), (2, 256, 2, 96, False), (2, 256, 2, 112, True),   # zero-padded to 128
    (2, 200, 3, 128, True),                                                  # ragged causal S, padded to 256
])
def test_attention_fwd_bwd_matches_fp32_reference(B, S, H, D, causal, monkeypatch):
    ops = ar.kernels_only(monkeypatch)
    qkv, q, k, v = kc._qkv(B, S, H, D)
    n0 = ops.launch_count()
    o, lse = ops.attention_fwd(q, k, v, causal=causal)
    do = torch.randn_like(o)
    grads = ops.attention_bwd(do, q, k, v, o, lse, causal=causal)
    buf = torch.full_like(qkv, float("nan"))
    ops.attention_bwd(do, q, k, v, o, lse, causal=causal, dqkv_out=buf)
    torch.cuda.synchronize()
    assert ops.launch_count() >= n0 + 7
    ref = ar.reference(q, k, v, do, causal)
    ref.check(o=o, lse=lse, dq=grads[0], dk=grads[1], dv=grads[2])
    ref.check(dq=buf[:, :, :, 0], dk=buf[:, :, :, 1], dv=buf[:, :, :, 2])


def test_hd128_long_sequence_memory_stays_linear(monkeypatch):
    """S = 8192: one fp32 [H, S, S] score tensor alone would be 2 GB; the kernels need no S x S storage."""
    ops = ar.kernels_only(monkeypatch)
    B, S, H, D = 1, 8192, 8, 128
    qkv, q, k, v = kc._qkv(B, S, H, D)
    do = torch.randn(B, S, H, D, device="cuda", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    o, lse = ops.attention_fwd(q, k, v, causal=True)
    dq, dk, dv = ops.attention_bwd(do, q, k, v, o, lse, causal=True)
    torch.cuda.synchronize()
    outputs = o.numel() * 2 + lse.numel() * 4 + 3 * dq.numel() * 2
    growth = torch.cuda.max_memory_allocated() - base - outputs
    assert growth < 256 * 2 ** 20, growth
    assert torch.isfinite(dq.float()).all() and torch.isfinite(o.float()).all()


def test_gpt2_hd128_trains_and_matches_cpu_reference(monkeypatch):
    ar.kernels_only(monkeypatch)
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    from tepdist_b200.runtime.executor import Executor
    cfg = CONFIGS["tiny-hd128"]
    assert cfg.n_embd // cfg.n_head == 128
    g = build_gpt2_graph(cfg)
    gpu = Executor(g, torch.device("cuda", 0), seed=0, use_cuda_graph=False)
    graph = Executor(g, torch.device("cuda", 0), seed=0, use_cuda_graph=True)
    cpu = Executor(g, torch.device("cpu"), seed=0)
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (cfg.batch, cfg.n_ctx), dtype=torch.int32)
    lab = torch.roll(tok, -1, 1)
    lg, lgr, lc = [], [], []
    for _ in range(4):
        lg.append(float(gpu.step({"tokens": tok.cuda(), "labels": lab.cuda()})[0]))
        lgr.append(float(graph.step({"tokens": tok.cuda(), "labels": lab.cuda()})[0]))
        lc.append(float(cpu.step({"tokens": tok, "labels": lab})[0]))
    assert lg[-1] < lg[0] and lgr[-1] < lgr[0]
    for a, b, c in zip(lg, lgr, lc):
        assert abs(a - c) / abs(c) < 2e-2, (lg, lc)
        assert abs(b - a) < 2e-2 * abs(a), (lgr, lg)


def test_traced_sdpa_block_with_128_wide_heads(monkeypatch):
    """A torch block written with F.scaled_dot_product_attention and 128-wide heads traces onto the attention op, runs on
    our kernels and trains like eager PyTorch."""
    import torch.nn as nn
    import torch.nn.functional as F
    from tepdist_b200.frontend.trace import trace
    from tepdist_b200.runtime.executor import Executor
    B, S, C, H, V = 2, 256, 256, 2, 128

    class Block(nn.Module):
        def __init__(self):
            super().__init__()
            self.emb = nn.Embedding(V, C)
            self.ln1, self.ln2 = nn.LayerNorm(C), nn.LayerNorm(C)
            self.qkv, self.proj = nn.Linear(C, 3 * C), nn.Linear(C, C)
            self.fc, self.out = nn.Linear(C, 4 * C), nn.Linear(4 * C, C)
            self.head = nn.Linear(C, V, bias=False)

        def forward(self, tokens):
            x = self.emb(tokens)
            q, k, v = self.qkv(self.ln1(x)).chunk(3, dim=-1)
            q, k, v = (t.view(B, S, H, C // H).transpose(1, 2) for t in (q, k, v))
            a = F.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(B, S, C)
            x = x + self.proj(a)
            x = x + self.out(F.gelu(self.fc(self.ln2(x)), approximate="tanh"))
            return self.head(x)

    torch.manual_seed(0)
    net = Block()
    tok = torch.randint(0, V, (B, S))
    lab = torch.randint(0, V, (B, S))
    tr = trace(net, {"tokens": tok}, loss="cross_entropy", label_example=lab.int(), optimizer="sgd", lr=0.1,
               compute_dtype="bf16")
    assert any(n.op == "attention" for n in tr.graph.nodes)
    net = net.cuda()
    ops = ar.kernels_only(monkeypatch)
    ex = Executor(tr.graph, torch.device("cuda", 0), use_cuda_graph=False)
    tr.load_state_dict_into(ex, net.state_dict())
    opt = torch.optim.SGD(net.parameters(), lr=0.1)
    tok, lab = tok.cuda(), lab.cuda()
    n0 = ops.launch_count()
    for _ in range(3):
        ref = F.cross_entropy(net(tok).view(-1, V), lab.view(-1))
        opt.zero_grad(); ref.backward(); opt.step()
        (l,) = ex.step({"tokens": tok.int(), "labels": lab.int()})
        assert abs(float(l) - float(ref)) < 2e-2 * abs(float(ref)), (float(l), float(ref))
    assert ops.launch_count() > n0
