"""Packed-document training on the CPU reference path: document starts, document-masked causal attention, per-document
positions, the planner's candidates for them, and multi-process (gloo) parity."""
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

from tepdist_b200 import _C, ops
from tepdist_b200.api import Trainer
from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
from tepdist_b200.planner import to_native
from tepdist_b200.runtime.executor import Executor

HERE = os.path.dirname(os.path.abspath(__file__))
EOT = 7


def _doc_starts_loop(tok: torch.Tensor, eot: int) -> torch.Tensor:
    B, S = tok.shape
    out = torch.zeros(B, S, dtype=torch.int32)
    for b in range(B):
        start = 0
        for s in range(S):
            out[b, s] = start
            if int(tok[b, s]) == eot:
                start = s + 1
    return out


@pytest.mark.parametrize("marks", [[], [0], [31], [0, 1, 2], [5, 6, 20, 21, 31], [3, 17]], ids=str)
def test_doc_starts_edge_cases(marks):
    tok = torch.zeros(2, 32, dtype=torch.int32)
    tok[0, marks] = EOT
    tok[1, [m for m in range(32) if m not in marks][:1]] = EOT    # the other row: one EOT at the first free position
    got = ops.doc_starts(tok, EOT)
    assert got.dtype == torch.int32 and got.shape == tok.shape
    assert torch.equal(got, _doc_starts_loop(tok, EOT))
    assert bool((got[:, 1:] >= got[:, :-1]).all())
    if not marks:
        assert int(got[0].max()) == 0
    if 31 in marks:      # an EOT in the last position starts no document inside the row
        assert int(got[0, 31]) == (max([m for m in marks if m < 31], default=-1) + 1)


def _qkv(B, S, H, D, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, S, H, D, generator=g, dtype=torch.float64).float() for _ in range(4)]


@pytest.mark.parametrize("lengths", [[1, 40, 23], [64], [17, 17, 17, 13], [1, 1, 1, 61]], ids=str)
def test_reference_attention_with_documents_equals_each_document_alone(lengths):
    B, H, D = 2, 2, 16
    S = sum(lengths)
    q, k, v, do = _qkv(B, S, H, D)
    tok = torch.zeros(B, S, dtype=torch.int32)
    tok[0, torch.tensor(lengths).cumsum(0) - 1] = EOT
    tok[1, torch.tensor(lengths[::-1]).cumsum(0) - 1] = EOT     # the other row: the same documents in reverse order
    ds = ops.doc_starts(tok, EOT)
    o, lse = ops.attention_fwd(q, k, v, causal=True, doc_start=ds)
    dq, dk, dv = ops.attention_bwd(do, q, k, v, o, lse, causal=True, doc_start=ds)
    for b in range(B):
        starts = sorted(set(ds[b].tolist()))
        bounds = starts + [S]
        for s0, s1 in zip(bounds[:-1], bounds[1:]):
            sl = slice(s0, s1)
            part = [t[b:b + 1, sl] for t in (q, k, v)]
            o1, lse1 = ops.attention_fwd(*part, causal=True)
            g1 = ops.attention_bwd(do[b:b + 1, sl], *part, o1, lse1, causal=True)
            torch.testing.assert_close(o[b:b + 1, sl], o1, rtol=1e-6, atol=1e-6)
            torch.testing.assert_close(lse[b:b + 1, :, sl], lse1, rtol=1e-6, atol=1e-6)
            for got, want in zip((dq, dk, dv), g1):
                torch.testing.assert_close(got[b:b + 1, sl], want, rtol=1e-5, atol=1e-6)


def test_document_mask_needs_causal_attention():
    q, k, v, _ = _qkv(1, 8, 1, 8)
    with pytest.raises(ValueError, match="causal"):
        ops.attention_fwd(q, k, v, causal=False, doc_start=torch.zeros(1, 8, dtype=torch.int32))
    from tepdist_b200.frontend.builder import GraphBuilder
    b = GraphBuilder()
    tok = b.input("tokens", (1, 8), "i32")
    qkv = b.input("qkv", (1, 8, 24), "bf16")
    with pytest.raises(ValueError, match="causal"):
        b.attention(qkv, 1, causal=False, doc_starts=b.doc_starts(tok, EOT))
    with pytest.raises(ValueError, match="eot_token"):
        build_gpt2_graph(CONFIGS["tiny"], reset_position_ids=True)


def test_per_document_positions_reference():
    B, S, C, V = 2, 12, 8, 16
    g = torch.Generator().manual_seed(1)
    tok = torch.randint(0, V, (B, S), generator=g, dtype=torch.int32)
    tok[0, [3, 4, 9]] = EOT
    ds = ops.doc_starts(tok, EOT)
    wte, wpe = torch.randn(V, C, generator=g), torch.randn(S, C, generator=g)
    out = ops.embedding_fwd(tok, wte, wpe, doc_start=ds)
    pos = torch.arange(S) - ds.long()
    assert int(pos[0, 4]) == 0 and int(pos[0, 5]) == 0 and int(pos[0, 10]) == 0 and int(pos[0, 9]) == 4
    torch.testing.assert_close(out, wte[tok.long()] + wpe[pos], rtol=0, atol=0)
    dout = torch.randn(B, S, C, generator=g)
    dwte, dwpe = torch.zeros(V, C), torch.zeros(S, C)
    ops.embedding_bwd(tok, dout, dwte, dwpe, doc_start=ds)
    want = torch.zeros(S, C, dtype=torch.float64)
    for b in range(B):
        for s in range(S):
            want[pos[b, s]] += dout[b, s].double()
    torch.testing.assert_close(dwpe.double(), want, rtol=1e-6, atol=1e-6)


def _losses(g, tok, steps=3):
    ex = Executor(g, torch.device("cpu"), seed=0, use_cuda_graph=False)
    feeds = {"tokens": tok, "labels": torch.roll(tok, -1, 1)}
    return [float(ex.step(feeds)[0]) for _ in range(steps)]


@pytest.mark.parametrize("reset", [False, True])
def test_eot_model_equals_plain_model_on_rows_without_eot(reset):
    cfg = CONFIGS["tiny"]
    tok = torch.randint(0, EOT, (cfg.batch, cfg.n_ctx), generator=torch.Generator().manual_seed(0), dtype=torch.int32)
    plain = _losses(build_gpt2_graph(cfg), tok)
    g = build_gpt2_graph(cfg, eot_token=EOT, reset_position_ids=reset)
    assert g.meta["model"]["eot_token"] == EOT and g.meta["model"]["reset_position_ids"] is reset
    assert sum(n.op == "doc_starts" for n in g.nodes) == 1
    assert plain == _losses(g, tok)
    tok[0, [10, 50, 51]] = EOT     # with documents the model computes something else
    assert _losses(build_gpt2_graph(cfg), tok) != _losses(g, tok)


def _plan_tags(g, num, **kw):
    cg = to_native(g)
    o = _C.SpmdOptions()
    o.num = num
    for k, v in kw.items():
        setattr(o, k, v)
    plan = _C.plan_spmd_level(cg, o)
    return {(cg.node_op(i), plan.choice[i].tag) for i in range(cg.num_nodes())
            if cg.node_op(i) in ("attention", "attention_bwd", "embedding", "embedding_bwd", "doc_starts")}


def test_no_sequence_split_for_document_masked_attention_or_embedding():
    cfg = CONFIGS["tiny"]
    # batch-1 long context: the plain model shards attention over heads and everything token-wise over the sequence; with
    # per-document positions the embedding keeps the sequence whole
    for batch, kw in ((1, dict(collective_latency_bytes=0)), (4, {}), (1, dict(context_parallel=True))):
        tags = _plan_tags(build_gpt2_graph(cfg, batch=batch, eot_token=EOT, reset_position_ids=True), 2, **kw)
        assert tags and not any(t == "seq" for _, t in tags), (batch, kw, tags)
        assert {op for op, _ in tags} == {"attention", "attention_bwd", "embedding", "embedding_bwd", "doc_starts"}
    # (the plain model's context-parallel plan does take the sequence split, so the option above is live)
    assert ("attention", "seq") in _plan_tags(build_gpt2_graph(cfg, batch=1), 2, context_parallel=True)


@pytest.mark.parametrize("strategy", ["cp", "dp2cp2"])
def test_context_parallel_strategies_refuse_document_masks(strategy):
    g = build_gpt2_graph(CONFIGS["tiny"], eot_token=EOT)
    with pytest.raises(ValueError, match="document-masked"):
        Trainer(g, strategy=strategy, device=torch.device("cpu"), use_cuda_graph=False)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


_STRATEGIES = ["dp", "tp", "pp2m2"]
_RESULT = {}


@pytest.mark.parametrize("strategy", _STRATEGIES)
def test_world2_matches_single_process_with_documents_across_shard_boundaries(strategy, tmp_path):
    sys.path.insert(0, HERE)
    import doc_mask_worker
    if not _RESULT:
        out = str(tmp_path / "out.json")
        env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="2")
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
               "--master-port", str(_free_port()), os.path.join(HERE, "doc_mask_worker.py"), "+".join(_STRATEGIES), out]
        pr = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
        assert pr.returncode == 0, pr.stderr[-3000:]
        _RESULT.update(json.load(open(out)))
        _RESULT["ref"] = doc_mask_worker.run("auto")
    got, ref = _RESULT[strategy], _RESULT["ref"]
    assert got["losses"][-1] < got["losses"][0]
    assert got["parallelism"].startswith(strategy[:2]), got
    for a, b in zip(got["losses"], ref["losses"]):
        assert abs(a - b) <= 2e-4 * max(1.0, abs(b)), (strategy, got, ref)
