"""Worker for multi-process CPU (gloo) tests: python tests/dist_worker.py <case> <out.json> under torchrun env."""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _dev():
    """CPU (gloo) by default; TEPDIST_TEST_DEVICE=cuda runs the same cases on GPUs over NCCL (tests/test_plans_multi_gpu.py)."""
    if os.environ.get("TEPDIST_TEST_DEVICE") == "cuda":
        return torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    return torch.device("cpu")


def case_gpt2(strategy, feed_shards=False, batch=4):
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    cfg = CONFIGS["tiny"]
    if strategy.startswith(("pp", "cp", "dp2cp")) and int(os.environ.get("WORLD_SIZE", "1")) == 1:
        strategy = "auto"   # single-process oracle
    if os.environ.get("TEPDIST_TEST_NCTX"):     # (GPU runs of the ring: blocks of 128 tokens go through the wgmma kernels)
        import dataclasses
        cfg = dataclasses.replace(cfg, n_ctx=int(os.environ["TEPDIST_TEST_NCTX"]))
    g = build_gpt2_graph(cfg, batch=batch)
    tr = Trainer(g, strategy=strategy, device=_dev(), use_cuda_graph=False)
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (batch, cfg.n_ctx), dtype=torch.int32)
    lab = torch.roll(tok, -1, 1)
    if feed_shards and tr.world > 1:   # data-loader contract: every rank feeds only its own sequences
        per = 4 // tr.world
        tok, lab = tok[tr.rank * per:(tr.rank + 1) * per], lab[tr.rank * per:(tr.rank + 1) * per]
    losses = [tr.step({"tokens": tok, "labels": lab}) for _ in range(4)]   # global batch fed: ranks take their shards
    res = {"losses": losses, "parallelism": tr.plan_info.get("parallelism"), "collectives": tr.plan_info.get("collectives")}
    worker = getattr(tr.exec, "worker", None)
    if worker is not None:   # pipeline: receive-buffer ring statistics of every stage worker
        stats = [None] * tr.world
        dist.all_gather_object(stats, dict(worker.ring_stats, stage=worker.stage, sync_recvs=worker.sync_recvs))
        res["ring"] = stats
        gst = [None] * tr.world
        dist.all_gather_object(gst, dict(worker.graph_stats, slots=worker.num_slots, stage=worker.stage))
        res["graphs"] = gst
    return res


def case_ckpt(strategy):
    """Train 2 steps under `strategy`, save a sharded checkpoint into $TEPDIST_TEST_CKPT, train 2 more steps."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    cfg = CONFIGS["tiny"]
    g = build_gpt2_graph(cfg, batch=4, optimizer=os.environ.get("TEPDIST_TEST_OPT", "adamw"))
    tr = Trainer(g, strategy=strategy, device=_dev(), use_cuda_graph=False)
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (4, cfg.n_ctx), dtype=torch.int32)
    feeds = {"tokens": tok, "labels": torch.roll(tok, -1, 1)}
    before = [tr.step(feeds) for _ in range(2)]
    tr.save(os.environ["TEPDIST_TEST_CKPT"], global_step=2)
    after = [tr.step(feeds) for _ in range(2)]
    return {"losses": before + after, "parallelism": tr.plan_info.get("parallelism"), "collectives": tr.plan_info.get("collectives")}


def case_resume(strategy):
    """Start a fresh job under `strategy` (different seed), restore the latest checkpoint in $TEPDIST_TEST_CKPT, train 2 steps."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    cfg = CONFIGS["tiny"]
    tr = Trainer(build_gpt2_graph(cfg, batch=4, optimizer=os.environ.get("TEPDIST_TEST_OPT", "adamw")), strategy=strategy,
                 device=_dev(), use_cuda_graph=False, seed=123)
    step = tr.restore(os.environ["TEPDIST_TEST_CKPT"])
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (4, cfg.n_ctx), dtype=torch.int32)
    feeds = {"tokens": tok, "labels": torch.roll(tok, -1, 1)}
    return {"losses": [tr.step(feeds) for _ in range(2)], "parallelism": tr.plan_info.get("parallelism"), "collectives": None, "step": step}


def case_state(strategy):
    """After a few sharded-optimizer steps every rank's state_dict must hold the SAME, fully updated master weights."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    cfg = CONFIGS["tiny"]
    tr = Trainer(build_gpt2_graph(cfg, batch=4), strategy=strategy, device=_dev(), use_cuda_graph=False)
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (4, cfg.n_ctx), dtype=torch.int32)
    feeds = {"tokens": tok, "labels": torch.roll(tok, -1, 1)}
    losses = [tr.step(feeds) for _ in range(3)]
    sd = tr.state_dict()
    keys = sorted(k for k in sd if not k.endswith(("/m", "/v")))
    sig = torch.tensor([float(sd[k].double().sum()) for k in keys] + [float(sd[k].double().abs().sum()) for k in keys], dtype=torch.float64)
    spread = 0.0
    if dist.is_initialized():
        lo, hi = sig.clone(), sig.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN)
        dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        spread = float((hi - lo).abs().max())
    return {"losses": losses, "signature": sig.tolist(), "rank_spread": spread, "parallelism": tr.plan_info.get("parallelism"),
            "collectives": tr.plan_info.get("collectives")}


def case_clip(strategy):
    """GPT-2 tiny with global-norm and per-tensor gradient clipping at a threshold that bites on every step."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    cfg = CONFIGS["tiny"]
    if strategy.startswith(("pp", "dp2")) and int(os.environ.get("WORLD_SIZE", "1")) == 1:
        strategy = "auto"
    out = {}
    for mode in ("none", "global", "local"):     # (SGD: AdamW would be invariant to a uniform rescaling of the gradients)
        g = build_gpt2_graph(cfg, batch=4, optimizer="sgd")
        g.meta["optimizer"].update(lr=0.5)
        if mode != "none":
            g.meta["optimizer"].update(clip_norm=mode, clip_norm_value=0.05)
        tr = Trainer(g, strategy=strategy, device=_dev(), use_cuda_graph=False)
        torch.manual_seed(0)
        tok = torch.randint(0, cfg.n_vocab, (4, cfg.n_ctx), dtype=torch.int32)
        out[mode] = [tr.step({"tokens": tok, "labels": torch.roll(tok, -1, 1)}) for _ in range(4)]
    return {"losses": [], "parallelism": strategy, "collectives": None, "clip": out}


def case_sched(strategy):
    """Warm-up + cosine schedule that travels with the graph; AdamW (flat / sharded-optimizer kernels read the rate from the device
    tensor) and SGD (host-scalar rate)."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    cfg = CONFIGS["tiny"]
    if strategy.startswith("pp") and int(os.environ.get("WORLD_SIZE", "1")) == 1:
        strategy = "auto"
    out = {}
    for opt, lr in (("adamw", 0.02), ("sgd", 0.5)):
        g = build_gpt2_graph(cfg, batch=4, optimizer=opt, schedule={"kind": "warmup_cosine", "warmup_steps": 2, "total_steps": 5, "end_ratio": 0.1})
        g.meta["optimizer"]["lr"] = lr
        tr = Trainer(g, strategy=strategy, device=_dev(), use_cuda_graph=False)
        torch.manual_seed(0)
        tok = torch.randint(0, cfg.n_vocab, (4, cfg.n_ctx), dtype=torch.int32)
        out[opt] = [tr.step({"tokens": tok, "labels": torch.roll(tok, -1, 1)}) for _ in range(5)]
    return {"losses": [], "parallelism": strategy, "collectives": None, "sched": out}


def case_fullstate(strategy):
    """Whole variables (+ moments) assembled on rank 0 by Trainer.full_state_dict after 3 steps: names, shapes and a value signature."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    cfg = CONFIGS["tiny"]
    if strategy.startswith(("pp", "dp2")) and int(os.environ.get("WORLD_SIZE", "1")) == 1:
        strategy = "auto"
    tr = Trainer(build_gpt2_graph(cfg, batch=4), strategy=strategy, device=_dev(), use_cuda_graph=False)
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (4, cfg.n_ctx), dtype=torch.int32)
    feeds = {"tokens": tok, "labels": torch.roll(tok, -1, 1)}
    losses = [tr.step(feeds) for _ in range(3)]
    sd = tr.full_state_dict(moments=True)
    keys = sorted(sd)
    return {"losses": losses, "parallelism": tr.plan_info.get("parallelism"), "collectives": None, "keys": keys,
            "shapes": [list(sd[k].shape) for k in keys],
            "signature": [float(sd[k].double().sum()) for k in keys] + [float(sd[k].double().abs().sum()) for k in keys]}


class _EmulatedGemmAllReduce:
    """CPU stand-in for parallel.symm.GemmAllReduceMC with the same call contract: row-parallel partial GEMM, sum over the
    group, + bias + residual.  Lets the EXECUTOR side of the fused tensor-parallel path (chain detection, aliasing of the
    all_reduce / add nodes, bias / residual plumbing, liveness) run under gloo; the multimem kernels are not involved."""
    calls = 0

    def __init__(self, M, N, group, ctx):
        self.M, self.N, self.group = M, N, group

    def new_output(self):
        return torch.empty(self.M, self.N)

    def __call__(self, x, w, out, bias=None, residual=None, b_mn=False, block_n=0):
        type(self).calls += 1
        y = x.float() @ (w.float() if b_mn else w.float().t())
        dist.all_reduce(y, group=self.group)
        if bias is not None:
            y = y + bias.float()
        if residual is not None:
            y = y + residual.float().reshape(self.M, self.N)
        out.copy_(y.to(out.dtype))
        return out


def case_tpfused(strategy):
    from tepdist_b200.runtime import executor as ex_mod
    ex_mod.TP_FUSED, ex_mod.TP_FUSED_IMPL = True, _EmulatedGemmAllReduce
    res = case_gpt2("tp")
    res["fused_calls"] = _EmulatedGemmAllReduce.calls
    return res


def case_manualdp(strategy):
    """No planner: every rank runs the UNSHARDED graph on its half of the batch through a bare Executor, gradients are
    averaged by the `grad_sync` hook (parallel/dp.py, bucketed all-reduce over the flat gradient buffer)."""
    from tepdist_b200.api import init_distributed
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    from tepdist_b200.parallel.dp import make_nccl_grad_sync
    from tepdist_b200.runtime.executor import Executor
    ctx = init_distributed()
    world, rank = ctx["world"], ctx["rank"]
    cfg = CONFIGS["tiny"]
    per = 4 // world
    ex = Executor(build_gpt2_graph(cfg, batch=per), _dev(), seed=0, use_cuda_graph=False,
                  grad_sync=make_nccl_grad_sync(bucket_elems=10000) if world > 1 else None)
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (4, cfg.n_ctx), dtype=torch.int32)
    lab = torch.roll(tok, -1, 1)
    losses = []
    for _ in range(4):
        l = ex.step({"tokens": tok[rank * per:(rank + 1) * per], "labels": lab[rank * per:(rank + 1) * per]})[0].float().reshape(1)
        if world > 1:
            dist.all_reduce(l)
        losses.append(float(l) / world)
    return {"losses": losses, "parallelism": "manual-dp", "collectives": None}


def case_opts(strategy):
    """Every reduction-carrying optimizer under `strategy`: losses + how many updates acted on a shard of their variable."""
    from tepdist_b200.api import Trainer
    from test_optimizers_cpu import CASES, build_mlp
    out = {}
    # (a toy MLP: price bytes only so the planner still splits it Megatron-style -- with the per-collective latency term it is,
    # correctly, data parallel, and no update would act on a stored shard)
    os.environ["TEPDIST_COLL_LATENCY_BYTES"] = "0"
    for case in ("momentum", "lamb", "adafactor", "adafactor_relative_step", "sm3", "sm3_momentum"):
        hp = CASES[case][0]
        tr = Trainer(build_mlp(case.split("_")[0], **hp), strategy=strategy, device=_dev(), use_cuda_graph=False, seed=5)
        torch.manual_seed(1)
        losses = [tr.step({"x": torch.randn(8, 16), "t": torch.randn(8, 4)}) for _ in range(6)]
        g = getattr(tr.exec, "g", None)
        sharded = 0
        if g is not None:
            for n in g.nodes:
                if n.op.startswith("apply_"):
                    src = g.nodes[n.inputs[0].node]
                    sharded += int(src.op == "dynamic_slice" or "shard_dims" in src.attrs)
        out[case] = {"losses": losses, "sharded_updates": sharded}
    del os.environ["TEPDIST_COLL_LATENCY_BYTES"]
    return {"losses": [], "parallelism": strategy, "collectives": None, "opts": out}


def case_optsgpt(strategy):
    """GPT-2 tiny with the reduction-carrying optimizers: the cost-based plan is data parallel with ZeRO-sharded updates
    (reduce_scatter -> apply on dynamic_slice(variable) -> all_gather), i.e. the update sees a dim-0 chunk of every variable."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    cfg = CONFIGS["tiny"]
    out = {}
    for kind in ("lamb", "adafactor", "sm3"):
        tr = Trainer(build_gpt2_graph(cfg, batch=4, optimizer=kind), strategy=strategy, device=_dev(), use_cuda_graph=False)
        torch.manual_seed(0)
        tok = torch.randint(0, cfg.n_vocab, (4, cfg.n_ctx), dtype=torch.int32)
        losses = [tr.step({"tokens": tok, "labels": torch.roll(tok, -1, 1)}) for _ in range(4)]
        g = getattr(tr.exec, "g", None)
        chunked = sum(1 for n in g.nodes if n.op.startswith("apply_") and g.nodes[n.inputs[0].node].op == "dynamic_slice") if g else 0
        out[kind] = {"losses": losses, "sharded_updates": chunked}
    return {"losses": [], "parallelism": strategy, "collectives": None, "opts": out}


def case_conv(strategy):
    """Small conv net with BatchNorm (models/smoke.py): under a batch split the BN statistics must be completed across ranks."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.smoke import build_conv_graph
    g = build_conv_graph(batch=8)
    tr = Trainer(g, strategy=strategy, device=_dev(), use_cuda_graph=False)
    torch.manual_seed(0)
    feeds = {"x": torch.randn(8, 3, 16, 16), "t": torch.randn(8, 10)}
    losses = [tr.step(feeds) for _ in range(4)]
    gg = getattr(tr.exec, "g", None)
    synced = sum(1 for n in gg.nodes if n.op.startswith("batchnorm") and n.attrs.get("sync_levels")) if gg is not None else 0
    return {"losses": losses, "parallelism": tr.plan_info.get("parallelism"), "collectives": tr.plan_info.get("collectives"), "synced_bn": synced}


def case_mlp(strategy):
    """examples/smoke_testing-style 2-layer MLP; planner emits a DP shard on CPU/gloo world_size=2 (BASELINE config 1)."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.smoke import build_mlp_graph
    g = build_mlp_graph(batch=8)
    tr = Trainer(g, strategy=strategy, device=_dev(), use_cuda_graph=False)
    torch.manual_seed(0)
    x, t = torch.randn(8, 16), torch.rand(8, 4)
    losses = [tr.step({"x": x, "t": t}) for _ in range(5)]
    return {"losses": losses, "parallelism": tr.plan_info.get("parallelism"), "collectives": tr.plan_info.get("collectives")}


def case_moe(strategy):
    """GPT-MoE tiny: with weights forced sharded the planner picks expert parallelism (all-to-all dispatch/combine)."""
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt_moe import build_moe_ffn_graph
    g = build_moe_ffn_graph(groups=4, tokens_per_group=32, model=32, hidden=64, experts=4, capacity=16)
    if strategy == "ep":
        strategy = "tp"     # var_mem_limit=1 => weights must be stored sharded; expert dim is the cheapest split
    tr = Trainer(g, strategy=strategy, device=_dev(), use_cuda_graph=False)
    torch.manual_seed(0)
    x, t = torch.randn(4, 32, 32), torch.randn(4, 32, 32)
    losses = [tr.step({"x": x, "t": t}) for _ in range(4)]
    return {"losses": losses, "parallelism": tr.plan_info.get("parallelism"), "collectives": tr.plan_info.get("collectives")}


def case_collectives(strategy):
    """Collective lowering on its own (reference xla/tests/dapple_all_gather_test.cc Dim0 / Dim1 / Dim1_2x3, dapple_all_to_all_test.cc,
    dapple_all_reduce tests): every collective op of the IR on every dim of a rank-3 tensor, on each level of the mesh named by
    `strategy` ("1d": one level over the world; "2d": 2 x (world/2)), against the result computed locally from the known contents of
    every rank's shard.  Returns the number of checks and the list of failures."""
    from types import SimpleNamespace
    from tepdist_b200.parallel.collectives import CollectiveRunner
    from tepdist_b200.parallel.mesh import DeviceMesh
    from tepdist_b200.api import init_distributed
    dev = _dev()
    init_distributed("nccl" if dev.type == "cuda" else "gloo")
    world, rank = dist.get_world_size(), dist.get_rank()
    nums = [world] if strategy in ("auto", "1d") else [2, world // 2]
    mesh = DeviceMesh(nums, [False] * len(nums), rank=rank, world=world)
    mesh.build_process_groups()
    run = CollectiveRunner(mesh)
    shape = (8, 8, 16)      # every dim divisible by 2, 4 and 8

    def content(r, sh=shape):        # what global rank r holds
        g = torch.Generator().manual_seed(100 + r)
        return torch.randint(-8, 9, sh, generator=g).float()       # small integers: every reduction is exact in fp32 (and bf16 sums)
    fails, checks = [], 0
    for lvl, num in enumerate(nums):
        ranks = mesh.group_ranks(lvl)
        me = mesh.index_in_group(lvl)
        mine = content(rank).to(dev)
        node = lambda op, **a: SimpleNamespace(op=op, attrs=dict(a, level=lvl, num=num))

        def check(tag, got, want):
            nonlocal checks
            checks += 1
            if tuple(got.shape) != tuple(want.shape) or not torch.equal(got.cpu(), want):
                fails.append(f"level{lvl} {tag}")
        total = sum(content(r) for r in ranks)
        check("all_reduce", run.run(node("all_reduce", reduce=0), [mine])[0], total)
        for d in range(3):
            check(f"all_gather dim{d}", run.run(node("all_gather", dim=d), [mine])[0], torch.cat([content(r) for r in ranks], d))
            sz = shape[d] // num
            check(f"reduce_scatter dim{d}", run.run(node("reduce_scatter", dim=d, reduce=0), [mine])[0], total.narrow(d, me * sz, sz))
            check(f"dynamic_slice dim{d}", run.run(node("dynamic_slice", dim=d), [mine])[0], content(rank).narrow(d, me * sz, sz))
            for cd in range(3):
                if cd == d:
                    continue
                # split `d` -> split `cd` reshard: piece `me` (along d) of every peer, concatenated along cd in group order
                want = torch.cat([content(r).narrow(d, me * sz, sz) for r in ranks], cd)
                check(f"all_to_all split{d} concat{cd}", run.run(node("all_to_all", split_dim=d, concat_dim=cd), [mine])[0], want)
    return {"losses": [], "parallelism": strategy, "collectives": None, "checks": checks, "fails": fails}


def case_ring(strategy):
    """parallel/ring_attention.py on its own: contiguous and zig-zag K / V rings (forward + backward) against full-sequence
    attention, every rank checking its own block; reports the largest error and each layout's per-rank work (block products)."""
    from tepdist_b200.api import init_distributed
    from tepdist_b200.ops.attention import attention_bwd, attention_fwd
    from tepdist_b200.parallel.ring_attention import RingAttention
    init_distributed("gloo")
    r, n = dist.get_rank(), dist.get_world_size()
    torch.manual_seed(0)
    B, S, H, D = 2, 16 * n, 2, 16
    qkv, do = torch.randn(B, S, H, 3, D), torch.randn(B, S, H, D)
    q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    res = {"losses": [], "parallelism": None, "collectives": None}
    L = S // n
    sl = slice(r * L, (r + 1) * L)
    sums = [None] * n      # every rank must have drawn the same tensors (the reference and the ring are compared rank by rank)
    dist.all_gather_object(sums, (float(qkv.double().sum()), float(qkv.double().abs().sum()), float(do.double().sum())))
    res["inputs_identical"] = all(s_ == sums[0] for s_ in sums)
    for causal in (True, False):
        o, lse = attention_fwd(q, k, v, causal=causal)
        grads = attention_bwd(do, q, k, v, o, lse, causal=causal)
        for zz in (False, True):
            ring = RingAttention(dist.group.WORLD, list(range(n)), r, zigzag=zz)
            o2, lse2 = ring.forward(q[:, sl], k[:, sl], v[:, sl], causal=causal)
            g2 = ring.backward(do[:, sl], q[:, sl], k[:, sl], v[:, sl], o2, lse2, causal=causal)
            work = ring.block_products
            o3, _ = ring.forward(q[:, sl], k[:, sl], v[:, sl], causal=causal)      # (diagnostic: is a deviation reproducible in-process?)
            again = (o3 - o2).abs().max().item()
            errs = [(o2 - o[:, sl]).abs().max().item()] + [(a - b[:, sl]).abs().max().item() for a, b in zip(g2, grads)] + [again]
            stats = [None] * n
            dist.all_gather_object(stats, (errs, work))
            res[f"{'causal' if causal else 'full'}_{'zigzag' if zz else 'contiguous'}"] = {
                "err": max(max(e) for e, _ in stats), "work": [w for _, w in stats], "per_rank_o_dq_dk_dv_again": [e for e, _ in stats]}
    return res


if __name__ == "__main__":
    case, out = sys.argv[1], sys.argv[2]
    CASES_ = {"gpt2": case_gpt2, "gpt2s": lambda st: case_gpt2(st, True), "gpt2b1": lambda st: case_gpt2(st, False, 1), "mlp": case_mlp, "moe": case_moe, "ckpt": case_ckpt, "state": case_state, "tpfused": case_tpfused, "manualdp": case_manualdp, "opts": case_opts, "optsgpt": case_optsgpt, "conv": case_conv, "resume": case_resume, "fullstate": case_fullstate, "clip": case_clip, "sched": case_sched, "collectives": case_collectives, "ring": case_ring}

    def run_case(c):
        name, _, strat = c.partition(":")
        return CASES_[name](strat or "auto")
    # "a:x+b:y": several cases in ONE job (the process start-up and the imports dominate a tiny case); results keyed by case
    res = {c: run_case(c) for c in case.split("+")} if "+" in case else run_case(case)
    if int(os.environ.get("RANK", "0")) == 0:
        json.dump(res, open(out, "w"))
    if dist.is_initialized():
        dist.barrier()
        # leave without tearing the process group down: destroying gloo groups while their worker threads are still draining
        # aborted once under load ("terminate called without an active exception", exit -6) after the results were written
        sys.stdout.flush()
        sys.stderr.flush()
        os._exit(0)
