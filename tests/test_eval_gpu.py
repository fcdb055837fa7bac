"""Evaluation step on the GPU: the forward-only loss kernel against fp64, the single-output GELU GEMM epilogue against the
other GELU paths, whole-model evaluation against the fp32 CPU executor, and that evaluations leave the training state untouched."""
import dataclasses
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

EPS32 = 2.0 ** -24           # fp32 unit roundoff
EPI_DIRECT, EPI_GELU_DUAL, EPI_BIAS_GELU = 0, 4, 8     # ops/csrc/gemm_sm90.cu enum Epi


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from tepdist_b200 import ops as o
    o.lib()
    return o


# ============================================================================================== loss kernel
def xent_ref(logits, labels, V):
    """fp64 logsumexp - logit[label] of the same bf16 logits, and a bound on each row's fp32 error.

    The kernel computes s = sum_j exp(x_j - m) and loss = log(s) + m - x_label in fp32:
      * each exp: its argument x_j - m (exact: both bf16-representable differences of values this size) is multiplied by
        log2(e) with one rounding, |x_j - m| eps absolute, then ex2.approx (2 ulp): relative error (|x - m|_max + 2) eps;
      * the sum: one thread adds at most K = ceil(V / 8 / 512) * 8 terms in sequence, then 9 + 5 shuffle / shared-memory merges,
        each merge rescaling with one more exp: relative error (K + 14 (|x - m|_max + 3)) eps;
      * log(s) by lg2.approx times ln 2: 4 eps relative, so 4 |log s| eps absolute; the relative error of s adds as is;
      * the two additions: 2 (|log s| + |m| + |x_label|) eps.
    The bound is twice the sum of these terms."""
    x = logits.double()[:, :V]
    lab = labels.long()
    valid = (lab >= 0) & (lab < V)
    m = x.max(-1).values
    s = torch.exp(x - m[:, None]).sum(-1)
    xl = x.gather(1, lab.clamp(0, V - 1)[:, None]).squeeze(1)
    loss = torch.where(valid, torch.log(s) + m - xl, torch.zeros_like(m))
    R = (torch.where(torch.isfinite(x), x, m[:, None]) - m[:, None]).abs().max(-1).values    # over the finite logits
    K = math.ceil(V / 8 / 512) * 8
    rel_s = (R + 2) * EPS32 + (K + 14 * (R + 3)) * EPS32
    bound = 2 * (rel_s + 4 * torch.log(s).abs() * EPS32 + 2 * (torch.log(s).abs() + m.abs() + xl.abs()) * EPS32)
    return loss, torch.where(valid, bound, torch.zeros_like(bound)), valid


@pytest.mark.parametrize("T,V,Vp", [(4096, 50257, 50304), (1000, 1001, 1008), (64, 13, 16), (333, 4095, 8192)])
def test_xent_fwd_against_fp64(ops, T, V, Vp):
    torch.manual_seed(T + V)
    logits = (torch.randn(T, Vp, device="cuda") * 3).to(torch.bfloat16)
    logits[:, V:] = 1e4        # padded columns must not take part
    # every 5th row starts with 8 in-vocabulary -inf logits: the first vector thread 0 reads holds no finite value
    logits[::5, :8] = float("-inf")
    labels = torch.randint(0, V, (T,), device="cuda", dtype=torch.int32)
    labels[::5] = V - 1
    labels[::7] = -1           # ignored
    labels[3::11] = V + (torch.arange(len(labels[3::11]), device="cuda", dtype=torch.int32) % (Vp - V + 3))   # bad
    before = logits.clone()
    out, rows = ops.xent_fwd(logits, labels, V)
    torch.cuda.synchronize()
    assert torch.equal(logits, before), "xent_fwd wrote the logits"
    ref, bound, valid = xent_ref(logits, labels, V)
    err = (rows.double() - ref).abs()
    worst = float((err / bound.clamp_min(1e-30))[valid].max())
    print(f"\nxent_fwd [{T}, {Vp}] V={V}: worst err / bound {worst:.3f}")
    assert worst <= 1.0
    assert torch.equal(rows[~valid], torch.zeros_like(rows[~valid]))
    assert int(out[1]) == int(valid.sum()) and int(out[2]) == int((labels >= V).sum())
    assert abs(float(out[0]) - float(ref.sum())) <= float(bound.sum()) + 1e-9 * abs(float(ref.sum()))
    # the fused training kernel's rows agree within the two kernels' bounds
    lab_ok = torch.where(valid, labels, torch.zeros_like(labels))
    _, rows_fb = ops.xent_fwd_bwd(logits.clone(), lab_ok, V, 1.0)
    assert bool(((rows_fb.double() - rows.double()).abs() <= 2 * bound + 1e-30)[valid].all())
    # deterministic: ten calls, the same bits
    sums = [ops.xent_fwd(logits, labels, V)[0].clone() for _ in range(10)]
    assert all(torch.equal(s, sums[0]) for s in sums)


# ============================================================================================== EPI_BIAS_GELU
def _last_epi(ops):
    return ops.lib().tepd_gemm_last_epi()


@pytest.mark.parametrize("M,N,K,block_n", [(256, 512, 128, 128), (256, 512, 128, 256), (300, 1000, 192, 0),
                                           (4096, 4096, 1024, 0)])
def test_bias_gelu_epilogue_bit_identical(ops, M, N, K, block_n):
    """Integer operands: alpha * acc + bias is exact in fp32, so every GELU path sees the same input and must give the same
    bits.  The staged single-output kind is taken for an aligned output, the fragment stores for a padded row pitch."""
    torch.manual_seed(M + N)
    a = torch.randint(-2, 3, (M, K), device="cuda").to(torch.bfloat16)
    b = torch.randint(-2, 3, (N, K), device="cuda").to(torch.bfloat16)
    bias = torch.randint(-4, 5, (N,), device="cuda").float()
    staged = ops.gemm(a, b, bias=bias, act="gelu", block_n=block_n)
    assert _last_epi(ops) == EPI_BIAS_GELU
    buf = torch.full((M, N + 4), float("nan"), device="cuda", dtype=torch.bfloat16)
    direct = ops.gemm(a, b, bias=bias, act="gelu", out=buf[:, :N], block_n=block_n)
    assert _last_epi(ops) == EPI_DIRECT
    pre, act = torch.empty_like(staged), torch.empty_like(staged)
    ops.gemm(a, b, bias=bias, act="gelu", out=pre, out2=act, block_n=block_n)
    assert _last_epi(ops) == EPI_GELU_DUAL
    torch.cuda.synchronize()
    assert torch.equal(staged, direct)
    assert torch.equal(staged, act)
    x = (a.double() @ b.double().t() + bias.double())
    ref = 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))
    assert float((staged.double() - ref).abs().max()) <= float((ref.abs() * 2.0 ** -8 + 1e-2).max())


# ============================================================================================== whole models
def _pair(g, seed=0):
    from tepdist_b200.runtime.executor import Executor
    gpu = Executor(g, torch.device("cuda", 0), seed=seed)
    # weights away from their initialisation (every variable + N(0, 0.05^2)): the logits spread over a range of order one, so
    # the loss depends on every layer, and evaluating with dropout on would move it well beyond MODEL_TOL
    gen = torch.Generator(device="cuda").manual_seed(seed + 7)
    gpu.store.master.add_(torch.randn(gpu.store.master.shape, generator=gen, device="cuda") * 0.05)
    gpu.store.sync_compute()
    cpu = Executor(g, torch.device("cpu"), seed=seed)
    cpu.store.master.copy_(gpu.store.master.cpu())
    return gpu, cpu


def _gpt2_feeds(cfg, batch, eot=None):
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (batch, cfg.n_ctx), dtype=torch.int32)
    if eot is not None:
        tok[:, ::37] = eot
    lab = torch.roll(tok, -1, 1)
    lab[0, -7:] = -1
    return {"tokens": tok, "labels": lab}


# Bound on |mean loss (GPU) - mean loss (fp32 CPU executor)| / mean loss.  The GPU forward computes in bf16 (weights and every
# activation rounded to 8 significant bits), so this is measured, not derived: on an H100 80GB HBM3 at 700 W the largest value
# over these models (with the perturbed weights of _pair) was 4.6e-5 (tiny-eot), and the bound is about four times that.  It
# is tight enough to tell dropout on from dropout off: evaluating GPT-2 tiny with its p = 0.1 dropout on moves the loss by
# 1.0e-3 relative (see test_gpt2_evaluation_against_fp32_executor[tiny-dropout]).
MODEL_TOL = 2e-4


def _check_model(gpu, cpu, feeds, label):
    fg = {k: v.cuda() for k, v in feeds.items()}
    ev_gpu = gpu.evaluate(fg).cpu()
    ev_cpu = cpu.evaluate(feeds)
    n_ref = int(((feeds["labels"] >= 0)).sum())
    assert int(ev_gpu[1]) == int(ev_cpu[1]) == n_ref and int(ev_gpu[2]) == 0
    mg, mc = float(ev_gpu[0] / ev_gpu[1]), float(ev_cpu[0] / ev_cpu[1])
    rel = abs(mg - mc) / abs(mc)
    print(f"\n{label}: eval loss GPU {mg:.6f} CPU {mc:.6f} rel {rel:.2e} (bound {MODEL_TOL:.2e})")
    assert rel <= MODEL_TOL
    return mg


@pytest.mark.parametrize("name", ["tiny", "tiny-hd128", "345m-2l", "tiny-eot", "tiny-dropout"])
def test_gpt2_evaluation_against_fp32_executor(ops, name):
    from tepdist_b200.models.gpt2 import CONFIGS, GPT2Config, build_gpt2_graph
    eot = None
    if name == "345m-2l":
        cfg, batch = GPT2Config(2, 1024, 16, 1024, 50257, 2), 2
    else:
        cfg, batch = CONFIGS[name.replace("-eot", "").replace("-dropout", "")], 4
    kw = {}
    if name == "tiny-eot":
        eot, kw = 0, {"eot_token": 0, "reset_position_ids": True}
    g = build_gpt2_graph(cfg, batch=batch, **kw)
    gpu, cpu = _pair(g)
    feeds = _gpt2_feeds(cfg, batch, eot)
    m0 = _check_model(gpu, cpu, feeds, name)
    if name == "tiny-dropout":
        # the p = 0.1 model evaluates like the p = 0 model with the same weights, and its training step -- the same forward
        # with dropout on -- reports a loss MODEL_TOL cannot mistake for it
        c1 = dataclasses.replace(cfg, embd_pdrop=0.1, attn_pdrop=0.1, resid_pdrop=0.1)
        gpu1, cpu1 = _pair(build_gpt2_graph(c1, batch=batch))
        m1 = _check_model(gpu1, cpu1, feeds, name + " p=0.1")
        assert abs(m1 - m0) <= MODEL_TOL * abs(m0)
        full = {"tokens": feeds["tokens"].cuda(), "labels": torch.roll(feeds["tokens"], -1, 1).cuda()}
        for ex, dropout in ((gpu, False), (gpu1, True)):
            ev = ex.evaluate(full)
            mean = float(ev[0] / ev[1])
            train = float(ex.step(full)[0])      # (the loss before this step's update)
            print(f"dropout {dropout}: eval {mean:.6f} training forward {train:.6f}")
            if dropout:
                assert abs(train - mean) > 2 * MODEL_TOL * abs(mean)
            else:
                assert abs(train - mean) <= 1e-5 * abs(mean)


def test_gpt_moe_evaluation_against_fp32_executor(ops):
    from tepdist_b200.models.gpt_moe import MoEConfig, build_gpt_moe_graph
    cfg = MoEConfig(n_layer=2, hidden=256, ffn=1024, n_head=4, experts=4, capacity=128, groups=2, seq=256, batch=2)
    g = build_gpt_moe_graph(cfg)
    gpu, cpu = _pair(g)
    torch.manual_seed(0)
    feeds = {n.name: torch.randint(0, cfg.vocab, tuple(n.outputs[0].shape), dtype=torch.int32) for n in g.inputs()}
    lab = [k for k in feeds if "label" in k][0]
    feeds[lab].view(-1)[:9] = -1
    ev_gpu = gpu.evaluate({k: v.cuda() for k, v in feeds.items()}).cpu()
    ev_cpu = cpu.evaluate(feeds)
    assert int(ev_gpu[1]) == int(ev_cpu[1]) == feeds[lab].numel() - 9
    rel = abs(float(ev_gpu[0] - ev_cpu[0])) / abs(float(ev_cpu[0]))
    print(f"\nGPT-MoE eval: rel {rel:.2e}")
    assert rel <= MODEL_TOL
    assert not gpu._moe_routes and gpu.step_count == 0


# ============================================================================================== training untouched
def _training_state(ex):
    """Every device value a captured training step reads besides its own graph pool, and the host counters it uses."""
    st = ex.store
    return ([t.clone() for t in (st.master, st.compute, st.grad, st.m, st.v, ex.rng_state, ex.hyper)] +
            [t.clone() for t in ex._static_in.values()] + [t.clone() for t in ex._static_out],
            (ex.step_count, ex.lr_now, len(ex.ln_stats), len(ex._moe_routes)))


def test_evaluation_leaves_graph_training_state_untouched(ops):
    """GPT-2 with dropout 0.1 and a warm-up schedule, CUDA graph on: evaluations after steps 2 and 4 (the first eager, the
    second captured) change no bit of anything the training graph reads.  (Two training runs are not compared with each
    other: the step's own fp32 atomics -- the loss sum, the attention dQ accumulation -- already differ between runs.)"""
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    from tepdist_b200.runtime.executor import Executor
    cfg = dataclasses.replace(CONFIGS["tiny"], embd_pdrop=0.1, attn_pdrop=0.1, resid_pdrop=0.1)
    f = {k: v.cuda() for k, v in _gpt2_feeds(cfg, 4).items()}
    feeds = {"tokens": f["tokens"], "labels": torch.roll(f["tokens"], -1, 1)}
    ex = Executor(build_gpt2_graph(cfg, batch=4), torch.device("cuda", 0), seed=0, use_cuda_graph=True)
    ex.set_lr_schedule(lambda step: 1e-3 * min(1.0, step / 4))
    losses = []
    for i in range(1, 7):
        losses.append(float(ex.step(feeds)[0]))
        if i in (2, 4):
            torch.cuda.synchronize()
            before, counters = _training_state(ex)
            ex.evaluate(f)
            torch.cuda.synchronize()
            after, counters2 = _training_state(ex)
            assert counters == counters2
            assert all(torch.equal(a, b) for a, b in zip(before, after))
    assert ex._eval_graph is not None and all(math.isfinite(x) for x in losses)
    assert losses[-1] < losses[0]
    # graph replays against an eager evaluation of the same weights: the same bits
    replays = [ex.evaluate(f).clone() for _ in range(3)]
    eager = Executor(build_gpt2_graph(cfg, batch=4), torch.device("cuda", 0), seed=1)
    eager.store.master.copy_(ex.store.master)
    eager.store.compute.copy_(ex.store.compute)
    e = eager.evaluate(f)
    torch.cuda.synchronize()
    assert all(torch.equal(x, e) for x in replays), (replays, e)


def test_evaluation_peak_memory_below_training_step(ops):
    from tepdist_b200.models.gpt2 import GPT2Config, build_gpt2_graph
    from tepdist_b200.runtime.executor import Executor
    cfg = GPT2Config(2, 1024, 16, 1024, 50257, 4)
    ex = Executor(build_gpt2_graph(cfg), torch.device("cuda", 0), seed=0)
    f = {k: v.cuda() for k, v in _gpt2_feeds(cfg, 4).items()}
    feeds = {"tokens": f["tokens"], "labels": torch.roll(f["tokens"], -1, 1)}
    ex.step(feeds)
    ex.evaluate(f)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ex.step(feeds)
    torch.cuda.synchronize()
    train = torch.cuda.max_memory_allocated() - base
    torch.cuda.reset_peak_memory_stats()
    ex.evaluate(f)
    torch.cuda.synchronize()
    ev = torch.cuda.max_memory_allocated() - base
    print(f"\npeak above the resident state: training step {train / 2**20:.0f} MiB, evaluation {ev / 2**20:.0f} MiB")
    assert ev < train
