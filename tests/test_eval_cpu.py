"""Evaluation step (Executor.evaluate / Trainer.evaluate) without a GPU: the CPU executor, every plan over gloo against one
process, the refusals, and that interleaved evaluations leave training bit-identical."""
import dataclasses
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import eval_worker  # noqa: E402


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


_JOBS = {}


def _job(cases, world, tmp_path_factory):
    """All cases of one world size in one torchrun job (start-up and imports dominate a tiny case)."""
    key = ("+".join(cases), world)
    if key not in _JOBS:
        out = str(tmp_path_factory.mktemp("eval") / "out.json")
        env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
        env.pop("WORLD_SIZE", None)
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
               "127.0.0.1", "--master-port", str(_free_port()), os.path.join(HERE, "eval_worker.py"), key[0], out]
        pr = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
        assert pr.returncode == 0, pr.stderr[-3000:]
        _JOBS[key] = json.load(open(out))
    return _JOBS[key]


WORLD2 = ["eval:dp", "eval:tp", "eval:tpsp", "eval:cp", "eval:pp2m2", "interleave:dp", "interleave:pp2m2", "refuse:pp2m2"]
# pp2m2 on 4 ranks: two stages, each split over 2 ranks (the loss triple is summed over the stage's own split only)
WORLD4 = ["eval:dp2tp2", "eval:pp2m2"]


@pytest.fixture(scope="module")
def single():
    return eval_worker.case_eval("auto")


def _tiny():
    from tepdist_b200.models.gpt2 import CONFIGS
    return CONFIGS["tiny"]


def _close(got, ref):
    for (s, n), (rs, rn) in zip(got, ref):
        assert n == rn
        assert abs(s / n - rs / rn) <= 2e-4 * max(1.0, abs(rs / rn)), (got, ref)


def test_single_process_matches_step_loss_and_torch():
    """With dropout 0 the evaluation of a batch is the loss the next training step reports for it (before its update)."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import build_gpt2_graph
    cfg = _tiny()
    tr = Trainer(build_gpt2_graph(cfg, batch=4), device=torch.device("cpu"), use_cuda_graph=False)
    feeds = eval_worker.batch(cfg, ignore=False)
    s, n = tr.evaluate(feeds)
    assert n == 4 * cfg.n_ctx
    loss = tr.step(feeds)
    assert abs(s / n - loss) <= 1e-5 * abs(loss)
    assert tr.exec.step_count == 1


def test_ignored_labels_are_not_counted():
    from tepdist_b200 import ops
    torch.manual_seed(1)
    logits = torch.randn(6, 24)
    labels = torch.tensor([3, -1, 19, 20, 25, -7])   # vocab 20: 20 and 25 are bad, -1 / -7 ignored
    out, rows = ops.xent_fwd(logits, labels, 20)
    ref = torch.logsumexp(logits[:, :20].double(), -1) - logits.double()[torch.arange(6), labels.clamp(0, 19)]
    assert out[1].item() == 2 and out[2].item() == 2
    assert abs(out[0].item() - (ref[0] + ref[2]).item()) < 1e-5
    assert rows[1].item() == rows[3].item() == rows[4].item() == rows[5].item() == 0.0


def test_bad_label_raises_and_changes_nothing():
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import build_gpt2_graph
    cfg = _tiny()
    tr = Trainer(build_gpt2_graph(cfg, batch=4), device=torch.device("cpu"), use_cuda_graph=False)
    feeds = eval_worker.batch(cfg)
    feeds["labels"][2, 7] = cfg.n_vocab
    before = {k: v.clone() for k, v in tr.state_dict().items()}
    with pytest.raises(ValueError, match="vocabulary"):
        tr.evaluate(feeds)
    ex = tr.exec
    assert ex.step_count == 0 and not ex.ln_stats and not ex._moe_routes
    assert all(torch.equal(before[k], v) for k, v in tr.state_dict().items())


def test_batchnorm_graph_is_refused():
    from tepdist_b200.models.smoke import build_conv_graph
    from tepdist_b200.runtime.executor import Executor
    ex = Executor(build_conv_graph(), torch.device("cpu"))
    with pytest.raises(ValueError, match="BatchNorm"):
        ex.evaluate({})


def test_pipeline_refuses_like_one_executor(tmp_path_factory):
    """Under a pipeline plan the same graphs are refused, on every rank, before any stage runs."""
    got = _job(WORLD2, 2, tmp_path_factory)["refuse:pp2m2"]
    assert got["batchnorm"] and "BatchNorm" in got["batchnorm"], got
    assert got["not_xent"] and "softmax_xent" in got["not_xent"], got


def test_loss_other_than_softmax_xent_is_refused():
    from tepdist_b200.models.smoke import build_mlp_graph
    from tepdist_b200.runtime.executor import Executor
    ex = Executor(build_mlp_graph(), torch.device("cpu"))
    with pytest.raises(ValueError, match="softmax_xent"):
        ex.evaluate({})


def test_moe_evaluation_keeps_no_route_tables():
    """GPT-MoE's forward fills route tables for its einsums; an evaluation leaves none behind and changes no step counter."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt_moe import MoEConfig, build_gpt_moe_graph
    cfg = MoEConfig(n_layer=1, hidden=64, ffn=128, n_head=2, experts=4, capacity=16, groups=2, seq=32, batch=2, vocab=500)
    tr = Trainer(build_gpt_moe_graph(cfg), device=torch.device("cpu"), use_cuda_graph=False)
    torch.manual_seed(0)
    inp = [n for n in tr.exec.g.inputs()]
    feeds = {n.name: torch.randint(0, cfg.vocab, tuple(n.outputs[0].shape), dtype=torch.int32) for n in inp}
    s, n = tr.evaluate(feeds)
    assert n > 0 and s > 0
    assert not tr.exec._moe_routes and not tr.exec.ln_stats and tr.exec.step_count == 0


def test_dropout_is_off_in_evaluation():
    """GPT-2 with p = 0.1 everywhere evaluates exactly like the same weights with p = 0."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import build_gpt2_graph
    cfg = _tiny()
    feeds = eval_worker.batch(cfg)
    res = []
    for p in (0.0, 0.1):
        c = dataclasses.replace(cfg, embd_pdrop=p, attn_pdrop=p, resid_pdrop=p)
        tr = Trainer(build_gpt2_graph(c, batch=4), device=torch.device("cpu"), use_cuda_graph=False)
        res.append(tr.evaluate(feeds))
    assert res[0][1] == res[1][1]
    assert abs(res[0][0] - res[1][0]) <= 1e-5 * abs(res[0][0])


@pytest.mark.parametrize("case,world", [(c, 2) for c in WORLD2 if c.startswith("eval:")] + [(c, 4) for c in WORLD4])
def test_plan_matches_single_process(case, world, single, tmp_path_factory):
    got = _job(WORLD2 if world == 2 else WORLD4, world, tmp_path_factory)[case]
    assert got["same_on_every_rank"], got
    _close(got["eval"], single["eval"])
    assert got["eval"][0][1] == 4 * _tiny().n_ctx - 5      # the five ignored labels


@pytest.mark.parametrize("case", ["interleave:dp", "interleave:pp2m2"])
def test_interleaved_evaluation_leaves_training_unchanged(case, tmp_path_factory):
    got = _job(WORLD2, 2, tmp_path_factory)[case]
    assert got["plain"] == got["interleaved"], got
