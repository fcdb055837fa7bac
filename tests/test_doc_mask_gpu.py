"""GPU numerics of document-masked causal attention and per-document positions (packed rows): the doc_starts kernel, the
DOC instantiations of the flash forward / backward at D = 64 / 128 (and padded 32 / 80, ragged S) against the fp64 reference
of attention_reference.py, the per-document embedding, and whole GPT-2 steps against the CPU executor.  Every case checks
that our kernels ran: the launch counter grows and the torch-math attention paths are turned into errors."""
import pytest
import torch

import attention_reference as ar
import kernel_checks as kc

pytestmark = pytest.mark.gpu

EOT = 999


def _tokens(layout: str, B: int, S: int) -> torch.Tensor:
    """int32 [B, S] tokens whose EOT positions give the named document layout in row 0; the other rows differ (none / one EOT)."""
    g = torch.Generator().manual_seed(sum(map(ord, layout)) + S)
    tok = torch.randint(0, EOT, (B, S), generator=g, dtype=torch.int32)
    marks = {
        "len1": [5, 6, S // 2, S // 2 + 1],                       # documents of length 1 (position 6, S/2 + 1)
        "on_boundary": [63, 127, 191, 255, 639],                   # documents starting exactly at 64 / 128 / ... boundaries
        "before_boundary": [62, 126, 254, 510],                    # ... and 1 before them
        "nan_tile": [199],                                         # rows 200.. see all of KV tile 0 masked (the safe max)
        "many_short": torch.randint(1, 40, (S,), generator=g).cumsum(0).tolist(),
    }[layout]
    marks = [p for p in marks if p < S]
    tok[0, marks] = EOT
    if B > 1:
        tok[1, S // 3] = EOT
    return tok.cuda()


@pytest.mark.parametrize("S", [128, 1000, 1024, 4096])
@pytest.mark.parametrize("D", [64, 128, 32, 80])
@pytest.mark.parametrize("layout", ["len1", "on_boundary", "before_boundary", "nan_tile", "many_short"])
def test_doc_masked_attention_matches_fp64_reference(layout, D, S, monkeypatch):
    ops = ar.kernels_only(monkeypatch)
    B, H = 2, 2
    ds = ops.doc_starts(_tokens(layout, B, S), EOT)
    qkv, q, k, v = kc._qkv(B, S, H, D, seed=S + D)
    do = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
    n0 = ops.launch_count()
    o, lse = ops.attention_fwd(q, k, v, causal=True, doc_start=ds)
    dq, dk, dv = ops.attention_bwd(do, q, k, v, o, lse, causal=True, doc_start=ds)
    torch.cuda.synchronize()
    assert ops.launch_count() >= n0 + 4
    ar.reference(q, k, v, do, True, ds).check(o=o, lse=lse, dq=dq, dk=dk, dv=dv)


@pytest.mark.parametrize("S", [1, 255, 256, 257, 1000, 4096])
def test_doc_starts_kernel_matches_reference(S, monkeypatch):
    ops = ar.kernels_only(monkeypatch)
    g = torch.Generator().manual_seed(S)
    tok = torch.randint(0, 20, (3, S), generator=g, dtype=torch.int32)
    tok[1] = EOT   # consecutive EOTs everywhere
    tok[2, 0] = EOT
    n0 = ops.launch_count()
    got = ops.doc_starts(tok.cuda(), 7)
    got_all = ops.doc_starts(tok.cuda(), EOT)
    assert ops.launch_count() == n0 + 2
    assert torch.equal(got.cpu(), ops.doc_starts(tok, 7))
    assert torch.equal(got_all.cpu(), ops.doc_starts(tok, EOT))


@pytest.mark.parametrize("D,S", [(64, 1024), (128, 1024), (64, 4096), (128, 4096)])
def test_all_zero_doc_start_equals_plain_causal_kernel(D, S, monkeypatch):
    """With every document start at 0 the DOC kernels do the plain kernels' arithmetic in the same order.  O, lse, dK and dV
    are bit-identical; dQ is summed over KV blocks with fp32 atomics, whose order differs between any two runs (of the plain
    kernel too), so it is compared to rounding."""
    ops = ar.kernels_only(monkeypatch)
    B, H = 2, 4
    qkv, q, k, v = kc._qkv(B, S, H, D, seed=11)
    do = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
    zero = torch.zeros(B, S, dtype=torch.int32, device="cuda")
    o0, lse0 = ops.attention_fwd(q, k, v, causal=True)
    o1, lse1 = ops.attention_fwd(q, k, v, causal=True, doc_start=zero)
    g0 = ops.attention_bwd(do, q, k, v, o0, lse0, causal=True)
    g1 = ops.attention_bwd(do, q, k, v, o0, lse0, causal=True, doc_start=zero)
    torch.cuda.synchronize()
    assert torch.equal(o0, o1) and torch.equal(lse0, lse1)
    assert torch.equal(g0[1], g1[1]) and torch.equal(g0[2], g1[2])
    assert kc._rel_err(g1[0], g0[0]) < 1e-2


def test_per_document_embedding_is_exact(monkeypatch):
    ops = ar.kernels_only(monkeypatch)
    B, S, C, V = 3, 1024, 256, 1000
    tok = _tokens("many_short", B, S)
    ds = ops.doc_starts(tok, EOT)
    g = torch.Generator().manual_seed(2)
    wte = torch.randn(V, C, generator=g).to(torch.bfloat16).cuda()
    wpe = torch.randn(S, C, generator=g).to(torch.bfloat16).cuda()
    dout = torch.randint(-3, 4, (B, S, C), generator=g).to(torch.bfloat16).cuda()   # integer values: every fp32 sum is exact
    n0 = ops.launch_count()
    out = ops.embedding_fwd(tok, wte, wpe, doc_start=ds)
    dwte = torch.full((V, C), 0.5, device="cuda")
    dwpe = torch.full((S, C), 0.5, device="cuda")
    ops.embedding_bwd(tok, dout, dwte, dwpe, doc_start=ds)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0 + 2
    rwte, rwpe = torch.full((V, C), 0.5), torch.full((S, C), 0.5)
    ops.embedding_bwd(tok.cpu(), dout.cpu(), rwte, rwpe, doc_start=ds.cpu())
    assert torch.equal(out.cpu(), ops.embedding_fwd(tok.cpu(), wte.cpu(), wpe.cpu(), doc_start=ds.cpu()))
    assert torch.equal(dwte.cpu(), rwte) and torch.equal(dwpe.cpu(), rwpe)
    pos = torch.arange(S, device="cuda") - ds
    assert int(pos.min()) == 0 and int(pos.max()) < S and int((pos == 0).sum()) > B


@pytest.mark.parametrize("name", ["tiny", "tiny-hd128"])
def test_gpt2_with_documents_trains_and_matches_cpu_reference(name, monkeypatch):
    ops = ar.kernels_only(monkeypatch)
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    from tepdist_b200.runtime.executor import Executor
    cfg = CONFIGS[name]
    g = build_gpt2_graph(cfg, eot_token=EOT, reset_position_ids=True)
    gpu = Executor(g, torch.device("cuda", 0), seed=0, use_cuda_graph=False)
    graph = Executor(g, torch.device("cuda", 0), seed=0, use_cuda_graph=True)
    cpu = Executor(g, torch.device("cpu"), seed=0)
    tok = _tokens("many_short", cfg.batch, cfg.n_ctx).cpu()
    lab = torch.roll(tok, -1, 1)
    lg, lgr, lc = [], [], []
    n0 = ops.launch_count()
    for _ in range(4):
        lg.append(float(gpu.step({"tokens": tok.cuda(), "labels": lab.cuda()})[0]))
        lgr.append(float(graph.step({"tokens": tok.cuda(), "labels": lab.cuda()})[0]))
        lc.append(float(cpu.step({"tokens": tok, "labels": lab})[0]))
    assert ops.launch_count() > n0
    assert lg[-1] < lg[0] and lgr[-1] < lgr[0]
    for a, b, c in zip(lg, lgr, lc):
        assert abs(a - c) / abs(c) < 2e-2, (lg, lc)
        assert abs(b - a) < 2e-2 * abs(a), (lgr, lg)
