"""The multi-tensor momentum, LAMB, Adafactor and SM3 kernels (ops/csrc/optim_sm90.cu) element by element against their
specification, runtime/optimizers.py, evaluated in fp64 on the CPU with the kernels' fp32 constants and the same `hyper`;
determinism and CUDA-graph replay; and whole GPT-2 and GPT-MoE steps on the executor's whole-variable path.

Tolerances.  Every slot and master element is compared as |got - ref| <= 2 u |ref| + tol * scale, where u = 2^-24 covers the
final fp32 rounding and `scale` is the largest |ref| of that tensor for slots, and the largest |step| (|p_ref - p_pre|) of the
variable for the master.  `tol` (OPT_TOL) is measured, not derived: the kernels reduce over up to 51 M terms per variable
(row and column sums, RMS, norms) in a different order from torch, with --use_fast_math's approximate sqrt / rsqrt /
division, and the error of such a sum depends on its data.  Every run prints the worst value of each kind; the bounds are
about twice the worst measured on an H100 80GB HBM3 at 700 W.  The bf16 compute copy is compared bit for bit with
master.to(bf16).
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
FTZ = 2.0 ** -125
# bound on |got - ref| / scale per optimizer kind (see the module docstring).  Worst measured over every case below on an
# H100 80GB HBM3 at 700 W: momentum 3.8e-8, LAMB 4.1e-7, Adafactor 2.1e-6 (the 345M + rank-3 set), SM3 1.8e-7.
OPT_TOL = {"apply_momentum": 8e-8, "apply_lamb": 8e-7, "apply_adafactor": 4.5e-6, "apply_sm3": 3.5e-7}
WORST = {}

SHAPES_345M = [(50304, 1024), (1024, 1024), (3072, 1024), (4096, 1024), (1024, 4096), (1024,), (3072,), (4096,)]
SHAPES_RAGGED = [(1000, 130), (7, 3), (1, 5), (5, 1), (1001,)]
SHAPE_RANK3 = [(8, 768, 6144)]
SMALL = [(1000, 130), (7, 3), (1, 5), (5, 1), (1001,), (256, 1024), (3, 40, 136), (4096,)]


@pytest.fixture
def ops(monkeypatch):
    """The kernel layer, with every torch-fallback warning turned into a failure and the torch update rules refusing
    CUDA tensors (the kernels must do all the work)."""
    from tepdist_b200 import ops as _ops
    from tepdist_b200.runtime import optimizers
    _ops.lib()

    def fallback(msg):
        raise AssertionError(f"torch fallback instead of our kernel: {msg}")
    monkeypatch.setattr(_ops, "_warn_once", fallback)
    for k, fn in list(optimizers.STEP.items()):
        def refuse(p, *a, _fn=fn, **kw):
            assert not p.is_cuda, "runtime/optimizers.py ran on CUDA tensors"
            return _fn(p, *a, **kw)
        monkeypatch.setitem(optimizers.STEP, k, refuse)
    return _ops


def f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def opt_f32(opt):
    """The optimizer settings as the fp32 constants the kernels compute with."""
    return {k: (f32(v) if isinstance(v, float) else v) for k, v in opt.items()}


class Vars:
    """Variables laid out like VariableStore: 128-element aligned in flat fp32 master / grad and bf16 buffers."""

    def __init__(self, op, opt, shapes, decays=None, seed=0, zero=()):
        from tepdist_b200 import ops
        self.op, self.opt, self.shapes = op, opt, [tuple(s) for s in shapes]
        self.decays = decays or [len(s) >= 2 for s in self.shapes]
        self.offs, off = [], 0
        for s in self.shapes:
            self.offs.append(off)
            off += -(-math.prod(s) // 128) * 128
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.gen = g
        self.master = torch.randn(off, device="cuda", generator=g) * 0.05
        for i in zero:
            self.view(self.master, i).zero_()
        self.grad = torch.zeros(off, device="cuda")
        self.compute = self.master.to(torch.bfloat16)
        self.slots = [[torch.zeros(ss, device="cuda") for ss in ops.optim_slot_shapes(op, s, opt)] for s in self.shapes]
        self.plan = ops.OptimPlan(op, opt, [(o, s, sl, d) for o, s, sl, d in zip(self.offs, self.shapes, self.slots, self.decays)],
                                  torch.device("cuda"))

    def view(self, buf, i):
        return buf[self.offs[i]:self.offs[i] + math.prod(self.shapes[i])].view(self.shapes[i])

    def new_grads(self, scale=1.0):
        self.grad.normal_(generator=self.gen).mul_(scale)

    def state(self):
        return self.master.clone(), [[s.clone() for s in sl] for sl in self.slots]


def hyper_for(opt, step, lr):
    from tepdist_b200.runtime.optimizers import host_hyper
    return torch.tensor(host_hyper(opt, step, lr), dtype=torch.float32, device="cuda")


def check_close(what, got, ref, scale, kind):
    got = got.double().cpu()
    err = (got - ref).abs() - 2 * U32 * ref.abs() - FTZ
    worst = float(err.max()) / max(scale, 1e-30) if err.numel() else 0.0
    WORST[kind] = max(WORST.get(kind, 0.0), worst)
    assert worst <= OPT_TOL[kind], f"{what}: off by {worst:.3e} of its scale (bound {OPT_TOL[kind]:.1e})"


def check_update(vs, pre_master, pre_slots, grad, hyper, label):
    """fp64 runtime/optimizers.py rule on the pre-step state and the given gradient vs the kernels' result."""
    from tepdist_b200.runtime.optimizers import STEP, Shards
    o = opt_f32(vs.opt)
    h = hyper.double().cpu()
    for i, shape in enumerate(vs.shapes):
        p = vs.view(pre_master, i).double().cpu()
        p0 = p.clone()
        gr = vs.view(grad, i).double().cpu()
        sl = [s.double().cpu() for s in pre_slots[i]]
        STEP[vs.op](p, gr, sl, o, h, Shards(), decay=vs.decays[i])
        step = float((p - p0).abs().max())
        check_close(f"{label} {shape} master", vs.view(vs.master, i), p, step, vs.op)
        for k, (got, ref) in enumerate(zip(vs.slots[i], sl)):
            check_close(f"{label} {shape} slot {k}", got, ref, float(ref.abs().max()), vs.op)
    assert torch.equal(vs.compute.view(torch.int16), vs.master.to(torch.bfloat16).view(torch.int16)), f"{label}: bf16 copy"


def run_case(ops, op, opt, shapes, steps=3, lr=1e-2, **kw):
    WORST.pop(op, None)
    vs = Vars(op, opt, shapes, **kw)
    for s in range(1, steps + 1):
        vs.new_grads(scale=1.0 / s)
        hyper = hyper_for(opt, s, lr * (1.0 + 0.5 * s))       # a different learning rate every step
        pm, ps = vs.state()
        n0 = ops.launch_count()
        ops.optim_step(vs.plan, vs.master, vs.grad, vs.compute, hyper)
        assert ops.launch_count() - n0 == ops.OPTIM_LAUNCHES[op]
        torch.cuda.synchronize()
        check_update(vs, pm, ps, vs.grad, hyper, f"{op} {opt} step {s}")
    print(f"\n{op} {opt}: worst {WORST[op]:.2e} of scale (bound {OPT_TOL[op]:.1e})")
    return vs


ALL = SHAPES_345M + SHAPES_RAGGED + SHAPE_RANK3


def test_momentum_against_fp64(ops):
    run_case(ops, "apply_momentum", dict(lr=1e-2, momentum=0.9), ALL)
    run_case(ops, "apply_momentum", dict(lr=1e-2, momentum=0.8, nesterov=True), SMALL)


def test_lamb_against_fp64(ops):
    run_case(ops, "apply_lamb", dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-6, weight_decay=0.01), ALL)
    # an all-zero variable (|p| = 0: ratio 1) and a zero-initialised bias; adapt_all adapts the no-decay variables too
    run_case(ops, "apply_lamb", dict(lr=1e-2, beta1=0.8, beta2=0.99, eps=1e-6, weight_decay=0.1, adapt_all=True), SMALL,
             zero=(0, 4))
    run_case(ops, "apply_lamb", dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-6, weight_decay=0.0), SMALL, zero=(1, 4))


def test_adafactor_against_fp64(ops):
    run_case(ops, "apply_adafactor", dict(lr=1e-2), ALL)
    run_case(ops, "apply_adafactor", dict(lr=None, weight_decay=0.01), SMALL)                 # relative step, wd decay vs no-decay
    run_case(ops, "apply_adafactor", dict(lr=1e-2, factored=False), SMALL)
    run_case(ops, "apply_adafactor", dict(lr=1e-2, clipping_threshold=None, decay_rate=0.9), SMALL)
    run_case(ops, "apply_adafactor", dict(lr=1e-2, multiply_by_parameter_scale=False, clipping_threshold=0.5), SMALL)


def test_sm3_against_fp64(ops):
    run_case(ops, "apply_sm3", dict(lr=1e-2), ALL)
    run_case(ops, "apply_sm3", dict(lr=1e-2, momentum=0.9), SMALL)


@pytest.mark.parametrize("op,opt", [("apply_momentum", dict(lr=1e-2, momentum=0.9, nesterov=True)),
                                    ("apply_lamb", dict(lr=1e-2, weight_decay=0.01)),
                                    ("apply_adafactor", dict(lr=None, weight_decay=0.01)),
                                    ("apply_sm3", dict(lr=1e-2, momentum=0.9))])
def test_deterministic_and_graph_replay_equals_eager(ops, op, opt):
    """Two eager runs give the same bits; one capture replayed three times with new gradients and `hyper` equals them."""
    shapes = [(3072, 1024), (1000, 130), (8, 96, 384), (4096,), (1001,)]
    grads = []
    gen = torch.Generator(device="cuda").manual_seed(7)
    for s in range(3):
        grads.append(torch.randn(Vars(op, opt, shapes).grad.numel(), device="cuda", generator=gen) / (s + 1))
    hypers = [hyper_for(opt, s + 1, 1e-2 * (s + 1)) for s in range(3)]

    def eager():
        vs = Vars(op, opt, shapes, seed=3)
        out = []
        for s in range(3):
            ops.optim_step(vs.plan, vs.master, grads[s], vs.compute, hypers[s])
            out.append((vs.master.clone(), vs.compute.clone(), [t.clone() for sl in vs.slots for t in sl]))
        return out
    a, b = eager(), eager()
    for s in range(3):
        assert torch.equal(a[s][0].view(torch.int32), b[s][0].view(torch.int32)), f"eager run differs at step {s + 1}"
        assert all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a[s][2], b[s][2]))

    vs = Vars(op, opt, shapes, seed=3)
    g_in, h_in = grads[0].clone(), hypers[0].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    pm, ps = vs.state()
    with torch.cuda.stream(side), torch.cuda.graph(graph):
        ops.optim_step(vs.plan, vs.master, g_in, vs.compute, h_in)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    vs.master.copy_(pm)                            # (capture records, it does not run)
    for sl, s0 in zip(vs.slots, ps):
        for t, t0 in zip(sl, s0):
            t.copy_(t0)
    for s in range(3):
        g_in.copy_(grads[s]); h_in.copy_(hypers[s])
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(vs.master.view(torch.int32), a[s][0].view(torch.int32)), f"replay {s + 1}: master differs from eager"
        assert torch.equal(vs.compute.view(torch.int16), a[s][1].view(torch.int16)), f"replay {s + 1}: bf16 copy differs"
        got = [t for sl in vs.slots for t in sl]
        assert all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(got, a[s][2])), f"replay {s + 1}: slots"


# ------------------------------------------------------------------ whole steps on the executor's whole-variable path
def whole_steps(ops, monkeypatch, g, tol, sched, feeds, label):
    """Step 1 eager, step 2 capture + replay, step 3 replay.  Each step: every parameter's gradient against the fp32 CPU
    executor (same pre-step master and slots), then the update against the fp64 rule on the GPU's own gradient."""
    from tepdist_b200.runtime.executor import Executor
    gpu = Executor(g, torch.device("cuda", 0), seed=0, use_cuda_graph=True)
    cpu = Executor(g, torch.device("cpu"), seed=0)
    assert gpu.optim_plan is not None and gpu.fused_apply_ok and cpu.optim_plan is not None
    gpu.set_lr_schedule(sched)
    cpu.set_lr_schedule(sched)
    op = gpu.optim_plan.op
    calls = []
    real = ops.optim_step

    def counted(plan, master, *a):
        n0 = ops.launch_count()
        real(plan, master, *a)
        if master.is_cuda:               # (the CPU oracle takes the same path through the CPU branch)
            calls.append(ops.launch_count() - n0)
    monkeypatch.setattr(ops, "optim_step", counted)
    gs, cs = gpu.store, cpu.store
    slot_nodes = [n for n in gpu.g.nodes if n.op == "state"]
    fg, fc = feeds
    for s in range(3):
        cs.master.copy_(gs.master.cpu())
        for buf in ("m", "v"):
            if getattr(gs, buf) is not None:
                getattr(cs, buf).copy_(getattr(gs, buf).cpu())
        for n in slot_nodes:
            if not gs._flat_slot(n):
                cs.state[n.id].copy_(gs.state[n.id].cpu())
        pre_master = gs.master.clone()
        pre_slots = [[s_.clone() for s_ in sl] for _, _, sl, _ in gpu.optim_plan.variables]
        cpu.step_count = gpu.step_count
        gpu.step(fg)
        torch.cuda.synchronize()
        cpu.step(fc)
        worst = 0.0
        for pid in gs.order:
            name = gs.names[pid]
            gg, r = gs.grad_view(pid).double().cpu(), cs.grad_view(pid).double()
            rel = float((gg - r).norm() / r.norm().clamp_min(1e-30))
            worst = max(worst, rel / tol(name))
            assert rel <= tol(name), f"{label} step {s + 1}: gradient of {name} off by {rel:.3e} (bound {tol(name)})"
        print(f"\n{label} step {s + 1}: worst gradient error {worst:.2f} of its bound")
        vs = _PlanVars(gpu)
        WORST.pop(op, None)
        check_update(vs, pre_master, pre_slots, gs.grad, gpu.hyper, f"{label} step {s + 1}")
        print(f"{label} step {s + 1}: update worst {WORST[op]:.2e} of scale (bound {OPT_TOL[op]:.1e})")
        assert (gpu._graph is None) == (s == 0)
    assert calls == [ops.OPTIM_LAUNCHES[op]] * 2, calls      # eager step and capture; a replay runs no Python
    print(f"{label}: optimizer launches per step {calls[0]} for {len(gpu.optim_plan.variables)} variables")


class _PlanVars(Vars):
    """The executor's variables seen through the Vars interface of check_update."""

    def __init__(self, ex):
        p = ex.optim_plan
        self.op, self.opt = p.op, p.opt
        self.offs = [o for o, _, _, _ in p.variables]
        self.shapes = [tuple(s) for _, s, _, _ in p.variables]
        self.slots = [sl for _, _, sl, _ in p.variables]
        self.decays = [d for _, _, _, d in p.variables]
        self.master, self.compute = ex.store.master, ex.store.compute


@pytest.mark.parametrize("optimizer", ["adafactor", "lamb", "sm3", "momentum"])
def test_gpt2_345m_widths_steps(ops, monkeypatch, optimizer):
    """One layer at the 345M widths, 4096 tokens (gradient bounds: test_step_numerics_gpu.GRAD_TOL)."""
    from test_step_numerics_gpu import grad_tol
    from tepdist_b200.models.gpt2 import GPT2Config, build_gpt2_graph
    cfg = GPT2Config(1, 1024, 16, 1024, 50257, 4)
    hp = {"momentum": dict(momentum=0.9)}.get(optimizer, {})
    g = build_gpt2_graph(cfg, optimizer=optimizer, **hp)
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (cfg.batch, cfg.n_ctx), dtype=torch.int32)
    lab = torch.roll(tok, -1, 1)
    feeds = ({"tokens": tok.cuda(), "labels": lab.cuda()}, {"tokens": tok, "labels": lab})
    whole_steps(ops, monkeypatch, g, grad_tol, lambda step: cfg.lr * min(1.0, step / 4), feeds, f"GPT-2 345M {optimizer}")


@pytest.mark.parametrize("optimizer", ["adafactor", "sm3"])
def test_gpt_moe_steps(ops, monkeypatch, optimizer):
    """Two layers at the reference widths (the rank-3 expert weights [8, 768, 6144]); the oracle routes as the GPU did
    (gradient bounds: test_moe_numerics_gpu.MOE_GRAD_TOL)."""
    from test_moe_numerics_gpu import moe_grad_tol
    from tepdist_b200.models.gpt_moe import MoEConfig, build_gpt_moe_graph
    from tepdist_b200.runtime.executor import Executor
    cfg = MoEConfig(n_layer=2, hidden=768, ffn=6144, n_head=16, experts=8, capacity=256, groups=2, seq=1024, batch=2)
    g = build_gpt_moe_graph(cfg, optimizer=optimizer)
    assert any(len(n.outputs[0].shape) == 3 for n in g.params())
    choices = {}
    real_choices = Executor._moe_choices

    def moe_choices(self, n, gates):
        if gates.is_cuda:
            choices[n.id] = real_choices(self, n, gates)
        return choices[n.id] if gates.is_cuda else choices[n.id].cpu()
    monkeypatch.setattr(Executor, "_moe_choices", moe_choices)
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.vocab, (cfg.batch, cfg.seq), dtype=torch.int32)
    lab = torch.roll(tok, -1, 1)
    feeds = ({"tokens": tok.cuda(), "labels": lab.cuda()}, {"tokens": tok, "labels": lab})
    whole_steps(ops, monkeypatch, g, moe_grad_tol, lambda step: 1e-4 * min(1.0, step / 4), feeds, f"GPT-MoE {optimizer}")
