"""Dropout on the H100 (DESIGN.md "Dropout"): the kernels' masks equal the host mask bit for bit (the elementwise kernel on
ones; the attention kernels read back through O with uniform probabilities and a one-hot V), attention forward / backward
with dropout against an fp64 reference that uses the host mask, whole GPT-2 steps with all three dropouts against the fp32
CPU executor, and CUDA-graph replay (the step is read from device memory, not frozen into the graph)."""
import math
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture
def ops(monkeypatch):
    """The kernel layer; torch-math attention and torch-fallback warnings are failures."""
    from tepdist_b200 import ops as _ops
    from tepdist_b200.ops import attention
    _ops.lib()
    ref_fwd = attention._ref_fwd

    def fail(*a, **k):
        raise AssertionError("fell back to torch math instead of our kernel")

    monkeypatch.setattr(attention, "_ref_fwd", lambda q, *a, **k: fail() if q.is_cuda else ref_fwd(q, *a, **k))
    monkeypatch.setattr(attention, "_warn_torch_math", fail)
    monkeypatch.setattr(_ops, "_warn_once", fail)
    return _ops


def _state(step, micro=0):
    return torch.tensor([step, micro], dtype=torch.int64, device="cuda")


# ------------------------------------------------------------------ masks, bit for bit
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_elementwise_kernel_mask_equals_host_mask(ops, p):
    from tepdist_b200 import _C
    thr = ops.dropout_threshold(p)
    scale = torch.tensor(256.0 / (256 - thr)).to(torch.bfloat16).item()
    # a [2, 96, 256] shard at (batch 1 + micro-batch 1 x 2, sequence 64, column 128) of a [6, 256, 512] tensor
    rng = ops.DropoutRng(123456789012345, _state(7, 1), 3, offsets=(1, 64, 128), micro=(2, 0, 0), global_shape=(6, 256, 512))
    x = torch.ones(2, 96, 256, device="cuda", dtype=torch.bfloat16)
    n0 = ops.launch_count()
    y = ops.dropout(x, p, rng)
    res = torch.randn(2, 96, 256, device="cuda").to(torch.bfloat16)
    y2 = ops.dropout_add(x, res, p, rng)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0 + 2
    keep = torch.from_numpy(_C.dropout_keep(123456789012345, 7, 3, thr, [6, 256, 512], [3, 64, 128], [2, 96, 256], False)).bool()
    assert torch.equal((y.cpu() != 0), keep)
    assert torch.equal(y.cpu()[keep], torch.full((int(keep.sum()),), scale, dtype=torch.bfloat16))
    want = (keep.float() * (256.0 / (256 - thr)) + res.cpu().float()).to(torch.bfloat16)
    assert torch.equal(y2.cpu(), want)


def _one_hot_v(B, S, H, D, k0):
    v = torch.zeros(B, S, H, D, device="cuda", dtype=torch.bfloat16)
    n = min(D, S - k0)
    v[:, k0 + torch.arange(n, device="cuda"), :, torch.arange(n, device="cuda")] = 1.0
    return v, n


ATTN_MASK_CASES = [   # (B, S, H, D, causal, doc, b_off, h_off, Bg, Hg)
    (2, 256, 2, 64, False, False, 0, 0, 2, 2),
    (2, 256, 2, 128, False, False, 3, 5, 6, 8),        # a shard: batch offset 3 of 6, heads 5.. of 8
    (2, 256, 2, 64, True, True, 1, 2, 4, 4),
    (1, 384, 2, 128, True, True, 0, 1, 1, 3),
    (2, 200, 2, 64, True, False, 0, 0, 2, 2),          # ragged causal S: zero-padded onto S = 256
]


@pytest.mark.parametrize("B,S,H,D,causal,doc,b_off,h_off,Bg,Hg", ATTN_MASK_CASES)
def test_attention_kernel_mask_equals_host_mask(ops, B, S, H, D, causal, doc, b_off, h_off, Bg, Hg):
    """q = k = 0: P is uniform over the visible keys, so with V one-hot over keys [k0, k0 + D) O[q, d] is nonzero exactly where
    key k0 + d is visible from q and kept."""
    from tepdist_b200.ops.attention import keep_mask
    p = 0.25
    rng = ops.DropoutRng(99, _state(11), 7, offsets=(b_off, 0, h_off * D), global_shape=(Bg, S, Hg * D))
    q = torch.zeros(B, S, H, D, device="cuda", dtype=torch.bfloat16)
    ds = None
    vis = torch.ones(S, S, dtype=torch.bool)
    if causal:
        vis = vis.tril()
    vis = vis.expand(B, H, S, S)
    if doc:
        starts = torch.zeros(B, S, dtype=torch.int32)
        for b in range(B):
            for cut in (37 + 50 * b, S // 2 + 3):
                starts[b, cut:] = cut
        ds = starts.cuda()
        keys = torch.arange(S)
        vis = vis & (keys.view(1, 1, 1, S) >= starts.long().view(B, 1, S, 1))
    want = keep_mask(rng, p, B, H, S, D) & vis
    got = torch.zeros(B, H, S, S, dtype=torch.bool)
    for k0 in range(0, S, D):
        v, n = _one_hot_v(B, S, H, D, k0)
        n0 = ops.launch_count()
        o, _ = ops.attention_fwd(q, q, v, causal=causal, doc_start=ds, pdrop=p, rng=rng)
        torch.cuda.synchronize()
        assert ops.launch_count() > n0
        got[..., k0:k0 + n] = (o.float().cpu().permute(0, 2, 1, 3)[..., :n] != 0)
    assert torch.equal(got, want), (got != want).sum().item()


# ------------------------------------------------------------------ numerics against fp64
def _ref(q, k, v, do, causal, z, doc=None):
    """fp64 autograd attention with the scaled keep mask z [B, H, S, S] on the probabilities -> (o, lse, dq, dk, dv)."""
    S, D = q.shape[1], q.shape[3]
    qf, kf, vf = (t.double().detach().clone().requires_grad_(True) for t in (q, k, v))
    s = torch.einsum("bqhd,bkhd->bhqk", qf, kf) * D ** -0.5
    if causal:
        vis = torch.ones(S, S, dtype=torch.bool, device=q.device).tril()
        if doc is not None:
            vis = vis & (torch.arange(S, device=q.device).view(1, 1, S) >= doc.long().unsqueeze(-1)).unsqueeze(1)
        s = s.masked_fill(~vis, float("-inf"))
    o = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1) * z, vf)
    o.backward(do.double())
    return o.detach(), torch.logsumexp(s, -1).detach(), qf.grad, kf.grad, vf.grad


def _close(got, want, rel, what):
    """As test_attention_hd64_gpu.py: norm-relative error under `rel`, every element within 4 rel of the largest magnitude."""
    got = got.double()
    assert torch.isfinite(got).all(), f"{what}: non-finite values"
    err_norm = ((got - want).norm() / (want.norm() + 1e-12)).item()
    assert err_norm < rel, (what, err_norm)
    err = (got - want).abs().max().item()
    assert err <= 4 * rel * want.abs().max().item() + 1e-3, (what, err, want.abs().max().item())


NUM_CASES = [   # (B, S, H, D, causal, doc): the 345M and 1.3B step shapes
    (4, 1024, 16, 64, True, False),
    (4, 1024, 16, 64, False, False),
    (1, 2048, 16, 128, True, False),
    (1, 2048, 16, 128, False, False),
    (2, 1024, 16, 64, True, True),
    (1, 2048, 8, 128, True, True),
]


@pytest.mark.parametrize("B,S,H,D,causal,doc", NUM_CASES)
def test_attention_with_dropout_matches_fp64(ops, B, S, H, D, causal, doc):
    from tepdist_b200.ops.attention import keep_mask
    p = 0.1
    g = torch.Generator(device="cuda").manual_seed(S + H + D)
    qkv = torch.randn(B, S, H, 3, D, device="cuda", generator=g).to(torch.bfloat16)
    do = torch.randn(B, S, H, D, device="cuda", generator=g).to(torch.bfloat16)
    q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    ds = None
    if doc:
        tok = torch.randint(0, 50, (B, S), generator=torch.Generator().manual_seed(1), dtype=torch.int32)
        tok[:, S // 3] = 0
        tok[:, S // 2 + 5] = 0
        ds = ops.doc_starts(tok.cuda(), 0)
    rng = ops.DropoutRng(5, _state(3), 2, global_shape=(B, S, H * D))
    n0 = ops.launch_count()
    o, lse = ops.attention_fwd(q, k, v, causal=causal, doc_start=ds, pdrop=p, rng=rng)
    dq, dk, dv = ops.attention_bwd(do, q, k, v, o, lse, causal=causal, doc_start=ds, pdrop=p, rng=rng)
    torch.cuda.synchronize()
    assert ops.launch_count() >= n0 + 4
    z = keep_mask(rng, p, B, H, S, D).cuda().double() * (256.0 / (256 - ops.dropout_threshold(p)))
    o_ref, lse_ref, *g_ref = _ref(q, k, v, do, causal, z, ds)
    del z
    _close(o, o_ref, 2e-2, "o")
    _close(lse, lse_ref, 1e-3, "lse")
    for name, got, want in zip(("dq", "dk", "dv"), (dq, dk, dv), g_ref):
        _close(got, want, 3e-2, name)


# ------------------------------------------------------------------ whole steps
def test_gpt2_345m_widths_with_dropout_gradient_by_gradient(ops):
    """One layer at the 345M widths with embedding, attention and residual dropout: every parameter's gradient against the
    fp32 CPU executor, which draws its masks from the host function.  Step 1 eager, step 2 CUDA-graph capture + replay, step 3
    replay: a step frozen into the graph would give step 3 step 2's masks and fail the comparison."""
    sys.path.insert(0, HERE)
    from test_step_numerics_gpu import step_checks
    from tepdist_b200.models.gpt2 import GPT2Config, build_gpt2_graph
    from tepdist_b200.runtime.executor import Executor
    cfg = GPT2Config(1, 1024, 16, 1024, 50257, 4, embd_pdrop=0.1, attn_pdrop=0.1, resid_pdrop=0.1)
    g = build_gpt2_graph(cfg)
    gpu = Executor(g, torch.device("cuda", 0), seed=4, use_cuda_graph=True)
    cpu = Executor(g, torch.device("cpu"), seed=4)
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (cfg.batch, cfg.n_ctx), dtype=torch.int32)
    lab = torch.roll(tok, -1, 1)
    fg, fc = {"tokens": tok.cuda(), "labels": lab.cuda()}, {"tokens": tok, "labels": lab}
    for s, label in enumerate(("345M + dropout step 1 (eager)", "step 2 (capture + replay)", "step 3 (replay)")):
        n0 = ops.launch_count()
        step_checks(gpu, cpu, fg, fc, label)
        assert ops.launch_count() > n0
        assert (gpu._graph is None) == (s == 0)


def test_cuda_graph_replays_read_the_current_step(ops):
    """A captured dropout reads (step, micro-batch) from device memory: replays after updating the state give each step's
    host mask, and consecutive replays differ; four GPT-2 steps under capture equal four eager steps (up to the last-bit
    spread the fp32 atomics of the backward give between any two runs: a step with another step's masks differs by
    orders of magnitude more)."""
    from tepdist_b200 import _C
    thr = ops.dropout_threshold(0.1)
    state = _state(1)
    x = torch.ones(4, 64, 256, device="cuda", dtype=torch.bfloat16)
    rng = ops.DropoutRng(8, state, 1)
    ops.dropout(x, 0.1, rng)                 # warm-up outside capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = ops.dropout(x, 0.1, rng)
    prev = None
    for step in (2, 3, 4):
        state[0].fill_(step)
        graph.replay()
        torch.cuda.synchronize()
        keep = torch.from_numpy(_C.dropout_keep(8, step, 1, thr, [4, 64, 256], [0, 0, 0], [4, 64, 256], False)).bool()
        got = y.cpu() != 0
        assert torch.equal(got, keep), step
        assert prev is None or not torch.equal(got, prev)
        prev = got

    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    from tepdist_b200.runtime.executor import Executor
    import dataclasses
    cfg = dataclasses.replace(CONFIGS["tiny"], embd_pdrop=0.1, attn_pdrop=0.1, resid_pdrop=0.1)
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (cfg.batch, cfg.n_ctx), dtype=torch.int32, device="cuda")
    feeds = {"tokens": tok, "labels": torch.roll(tok, -1, 1)}
    losses = {}
    for graphed in (False, True):
        ex = Executor(build_gpt2_graph(cfg), torch.device("cuda", 0), seed=2, use_cuda_graph=graphed)
        losses[graphed] = [float(ex.step(feeds)[0]) for _ in range(4)]
        assert (ex._graph is not None) == graphed
    assert losses[True] == pytest.approx(losses[False], rel=1e-5, abs=0), losses


def test_pipeline_slot_replays_use_their_micro_batch(tmp_path):
    """A pipeline stage captures its bodies once per slot and replays them for other micro-batches.  One stage, two
    micro-batches, one slot: micro-batch 1 replays the CUDA graphs captured for micro-batch 0, so a micro-batch index frozen
    at capture would give it micro-batch 0's masks.  Four steps with real capture and replay equal four eager pipeline steps
    (to the run-to-run spread of fp32 atomics)."""
    import subprocess
    out = str(tmp_path / "pp1.pt")
    pr = subprocess.run([sys.executable, os.path.join(HERE, "dropout_worker.py"), "--pp1", out], capture_output=True, text=True,
                        timeout=600)
    assert pr.returncode == 0, pr.stderr[-3000:]
    res = torch.load(out)
    eager, graphed = res[False], res[True]
    assert not eager["use_graph"] and graphed["use_graph"] and graphed["slots"] == 1, graphed
    assert graphed["graph_stats"]["captured"] > 0 and graphed["graph_stats"]["replayed"] > 0, graphed
    assert graphed["losses"] == pytest.approx(eager["losses"], rel=1e-5, abs=0), res
