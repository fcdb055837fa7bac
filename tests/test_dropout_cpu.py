"""Dropout (DESIGN.md "Dropout") without a GPU: the host mask, the graph the builder makes, what the planner refuses, plan
invariance (every plan drops exactly the elements one process drops) and checkpoint resume."""
import dataclasses
import math
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from tepdist_b200 import _C, ops
from tepdist_b200.api import Trainer
from tepdist_b200.frontend.builder import GraphBuilder
from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
from tepdist_b200.planner import to_native

HERE = os.path.dirname(os.path.abspath(__file__))


# ------------------------------------------------------------------ host mask
def _keep(seed, step, site, thr, shape, start=None, length=None, attention=False):
    start = start or [0] * len(shape)
    length = length or [s - a for s, a in zip(shape, start)]
    return _C.dropout_keep(seed, step, site, thr, list(shape), list(start), list(length), attention)


@pytest.mark.parametrize("attention", [False, True])
@pytest.mark.parametrize("p", [0.05, 0.1, 0.5, 0.9])
def test_keep_fraction_within_binomial_bounds(p, attention):
    thr = ops.dropout_threshold(p)
    shape = (2, 3, 256, 256) if attention else (512, 768)
    k = _keep(7, 1, 1, thr, shape, attention=attention)
    n = k.size
    q = 1 - thr / 256
    assert abs(k.mean() - q) <= 6 * math.sqrt(q * (1 - q) / n), (k.mean(), q)


def test_threshold_quantises_p_to_a_256th_and_refuses_out_of_range():
    assert ops.dropout_threshold(0.1) == 26 and ops.dropout_threshold(0.0) == 0 and ops.dropout_threshold(0.5) == 128
    for bad in (-0.1, 1.0, 1.5):
        with pytest.raises(ValueError, match="dropout probability"):
            ops.dropout_threshold(bad)


@pytest.mark.parametrize("attention", [False, True])
def test_masks_depend_on_seed_step_and_site_and_nothing_else(attention):
    shape = (2, 2, 64, 64) if attention else (64, 128)
    base = _keep(1, 5, 2, 26, shape, attention=attention)
    assert np.array_equal(base, _keep(1, 5, 2, 26, shape, attention=attention))
    for other in ((2, 5, 2), (1, 6, 2), (1, 5, 3)):
        k = _keep(*other, 26, shape, attention=attention)
        assert 0.1 < (k != base).mean() < 0.3, other          # independent masks at q = 230/256 differ on ~18 %


@pytest.mark.parametrize("attention", [False, True])
def test_every_box_equals_the_slice_of_the_whole_mask(attention):
    shape = (3, 4, 80, 80) if attention else (6, 40, 96)
    whole = _keep(11, 3, 4, 60, shape, attention=attention)
    rng = np.random.default_rng(0)
    for _ in range(12):
        start = [int(rng.integers(0, s)) for s in shape]
        length = [int(rng.integers(1, s - a + 1)) for s, a in zip(shape, start)]
        box = _keep(11, 3, 4, 60, shape, start, length, attention)
        assert np.array_equal(box, whole[tuple(slice(a, a + n) for a, n in zip(start, length))]), (start, length)


def test_elementwise_rows_are_the_flattened_leading_coordinates():
    a = _keep(3, 1, 1, 100, (4, 6, 32))
    b = _keep(3, 1, 1, 100, (24, 32))
    assert np.array_equal(a.reshape(24, 32), b)


def test_cpu_dropout_op_applies_the_scaled_host_mask():
    x = torch.randn(4, 6, 32)
    res = torch.randn(4, 6, 32)
    rng = ops.DropoutRng(9, torch.tensor([2, 0]), 5)
    keep = torch.from_numpy(_keep(9, 2, 5, 26, (4, 6, 32))).bool()
    y = ops.dropout_add(x, res, 0.1, rng)
    torch.testing.assert_close(y, torch.where(keep, x * 256 / 230, torch.zeros(())) + res, rtol=0, atol=1e-6)
    # a shard at (batch 1, sequence 2) of the global tensor gets the slice of the global mask
    sh = ops.DropoutRng(9, torch.tensor([2, 0]), 5, offsets=(1, 2, 0), global_shape=(4, 6, 32))
    y2 = ops.dropout(x[1:3, 2:5], 0.1, sh)
    torch.testing.assert_close(y2, torch.where(keep[1:3, 2:5], x[1:3, 2:5] * 256 / 230, torch.zeros(())), rtol=0, atol=1e-6)


# ------------------------------------------------------------------ graphs and refusals
def _sig(g):
    return [(n.op, n.name, [v.key() for v in n.inputs], [(tuple(t.shape), t.dtype) for t in n.outputs],
             sorted((k, repr(v)) for k, v in n.attrs.items())) for n in g.nodes]


def test_zero_probabilities_build_the_graph_without_dropout():
    cfg = CONFIGS["tiny"]
    zero = dataclasses.replace(cfg, embd_pdrop=0.0, attn_pdrop=0.0, resid_pdrop=0.0)
    g0, g = build_gpt2_graph(cfg), build_gpt2_graph(zero)
    assert _sig(g0) == _sig(g)
    assert not any("drop" in n.op or "pdrop" in n.attrs for n in g.nodes)
    assert sum(n.op == "linear" and n.attrs.get("residual") for n in g.nodes) == 2 * cfg.n_layer
    b = GraphBuilder()
    x = b.input("x", (2, 16), "f32")
    assert b.dropout(x, 0.0) is x and len(b.g.nodes) == 1


def test_dropout_graph_sites_and_gradients():
    cfg = dataclasses.replace(CONFIGS["tiny"], embd_pdrop=0.1, attn_pdrop=0.1, resid_pdrop=0.1)
    g = build_gpt2_graph(cfg)
    fwd = [n for n in g.nodes if n.op in ("dropout", "dropout_add") or (n.op == "attention" and "pdrop" in n.attrs)]
    assert len(fwd) == 1 + 3 * cfg.n_layer
    sites = [n.attrs["site"] for n in fwd]
    assert len(set(sites)) == len(sites)
    bwd_sites = sorted(n.attrs["site"] for n in g.nodes if n.op == "dropout_bwd") + \
        sorted(n.attrs["site"] for n in g.nodes if n.op == "attention_bwd")
    assert sorted(bwd_sites) == sorted(sites)          # every backward applies its forward's mask


@pytest.mark.parametrize("p", [-0.1, 1.0])
def test_builder_refuses_probabilities_outside_zero_one(p):
    b = GraphBuilder()
    x = b.input("x", (2, 8, 48), "bf16")
    for call in (lambda: b.dropout(x, p), lambda: b.dropout_add(x, x, p), lambda: b.attention(x, heads=2, pdrop=p)):
        with pytest.raises(ValueError, match=r"outside \[0, 1\)"):
            call()


@pytest.mark.parametrize("strategy", ["cp", "dp2cp2"])
def test_context_parallel_strategies_refuse_attention_dropout(strategy):
    g = build_gpt2_graph(dataclasses.replace(CONFIGS["tiny"], attn_pdrop=0.1))
    with pytest.raises(ValueError, match="attention dropout"):
        Trainer(g, strategy=strategy, device=torch.device("cpu"), use_cuda_graph=False)


def _attention_tags(g, **kw):
    cg = to_native(g)
    o = _C.SpmdOptions()
    o.num = 2
    for k, v in kw.items():
        setattr(o, k, v)
    plan = _C.plan_spmd_level(cg, o)
    return {(cg.node_op(i), plan.choice[i].tag) for i in range(cg.num_nodes()) if cg.node_op(i) in ("attention", "attention_bwd")}


def test_no_ring_candidate_for_attention_dropout():
    cfg = CONFIGS["tiny"]
    assert ("attention", "seq") in _attention_tags(build_gpt2_graph(cfg, batch=1), context_parallel=True)
    for kw in (dict(context_parallel=True), dict(collective_latency_bytes=0), {}):
        tags = _attention_tags(build_gpt2_graph(dataclasses.replace(cfg, attn_pdrop=0.1), batch=1), **kw)
        assert tags and not any(t == "seq" for _, t in tags), (kw, tags)
    # residual / embedding dropout alone leave the ring available
    assert ("attention", "seq") in _attention_tags(
        build_gpt2_graph(dataclasses.replace(cfg, embd_pdrop=0.1, resid_pdrop=0.1), batch=1), context_parallel=True)


# ------------------------------------------------------------------ plans: every plan drops what one process drops
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


_RESULTS = {}


def _run_world(world, strategies, tmp_path, extra_env=None):
    key = (world, "+".join(strategies), tuple(sorted((extra_env or {}).items())))
    if key not in _RESULTS:
        out = str(tmp_path / "out.pt")
        env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="2", **(extra_env or {}))
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
               "127.0.0.1", "--master-port", str(_free_port()), os.path.join(HERE, "dropout_worker.py"), "+".join(strategies), out]
        pr = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
        assert pr.returncode == 0, pr.stderr[-4000:]
        _RESULTS[key] = torch.load(out)
    return _RESULTS[key]


def _reference(which="all"):
    if ("ref", which) not in _RESULTS:
        sys.path.insert(0, HERE)
        import dropout_worker
        _RESULTS[("ref", which)] = dropout_worker.run("auto/" + which)
    return _RESULTS[("ref", which)]


def _assert_same(got, ref, what):
    for a, b in zip(got["losses"], ref["losses"]):
        assert abs(a - b) <= 2e-5 * max(1.0, abs(b)), (what, got["losses"], ref["losses"])
    assert sorted(got["grads"]) == sorted(ref["grads"])
    for k, r in ref["grads"].items():
        gk = got["grads"][k]
        scale = float(r.abs().max()) + 1e-6
        err = float((gk - r).abs().max())
        assert err <= 2e-3 * scale, (what, k, err, scale)


_WORLD2 = ["dp", "tp", "tpsp", "pp2m2"]


@pytest.mark.parametrize("strategy", _WORLD2)
def test_world2_plans_drop_what_one_process_drops(strategy, tmp_path):
    got = _run_world(2, _WORLD2, tmp_path)[strategy]
    assert got["parallelism"] is not None and got["losses"][-1] < got["losses"][0]
    _assert_same(got, _reference(), strategy)


def test_head_split_attention_dropout_drops_what_one_process_drops(tmp_path):
    """Attention dropout alone under tp: every attention node is split over heads (qkv [B, S, 3C / 2], heads / 2), so the
    kernels run at a nonzero global head offset on rank 1."""
    got = _run_world(2, ["tp/attn"], tmp_path)["tp/attn"]
    cfg = CONFIGS["tiny"]
    B, S, C, H = 4, cfg.n_ctx, cfg.n_embd, cfg.n_head
    assert got["attention"] and all(heads == H // 2 and shape == (B, S, 3 * C // 2) for _, heads, shape in got["attention"]), \
        got["attention"]
    _assert_same(got, _reference("attn"), "tp, attention dropout only")


def test_world4_dp2tp2_drops_what_one_process_drops(tmp_path):
    _assert_same(_run_world(4, ["dp2tp2"], tmp_path)["dp2tp2"], _reference(), "dp2tp2")


def test_pipeline_slots_replayed_for_other_micro_batches_use_their_offsets(tmp_path):
    """Stage bodies are captured once per slot and replayed for other micro-batches.  Emulated on CPU (a replay re-runs the
    nodes), this checks the slot bookkeeping with dropout on; that a real replay reads the micro-batch index staged for it,
    not one frozen at capture, is checked on the GPU (test_dropout_gpu.py::test_pipeline_slot_replays_use_their_micro_batch)."""
    got = _run_world(2, ["pp2m2"], tmp_path, {"TEPDIST_PP_GRAPH_EMULATE": "1"})["pp2m2"]
    assert got["replayed"] and got["replayed"] > 0, got["replayed"]
    _assert_same(got, _reference(), "pp2m2 (graph emulation)")


# ------------------------------------------------------------------ resume
def test_resumed_run_drops_the_same_elements(tmp_path):
    sys.path.insert(0, HERE)
    import dropout_worker
    cfg = dropout_worker.model()
    f = dropout_worker.feeds(cfg)

    def trainer(seed):
        return Trainer(build_gpt2_graph(cfg, batch=4, optimizer="sgd", lr=dropout_worker.LR), device=torch.device("cpu"),
                       use_cuda_graph=False, seed=seed)
    tr = trainer(3)
    for _ in range(2):
        tr.step(f)
    tr.save(str(tmp_path), 2)
    before = {k: v.clone() for k, v in tr.full_state_dict().items()}
    loss3 = tr.step(f)
    after = tr.full_state_dict()
    tr2 = trainer(17)               # another seed: the checkpoint carries the dropout key along
    assert tr2.restore(str(tmp_path)) == 2
    loss3b = tr2.step(f)
    after2 = tr2.full_state_dict()
    assert loss3b == pytest.approx(loss3, rel=1e-6, abs=1e-6)
    for k in after:
        torch.testing.assert_close((before[k] - after2[k]), (before[k] - after[k]), rtol=1e-5, atol=1e-7)
