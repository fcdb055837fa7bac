"""The data-parallel sharded AdamW step (`fused_rs_adamw_ag_kernel`, ops/csrc/comm_sm90.cu) element by element, on one GPU.

The kernel sums the peers' gradient chunks, applies AdamW to the chunk this rank owns and stores the bf16 result into every
peer's parameter buffer.  Nothing inside it synchronises across ranks: its peers are just pointers.  So one GPU plays n
ranks here: every virtual rank has its own gradient, parameter, master, m and v buffers on the same device, and the ranks'
calls run one after another on one stream, through `FusedShardedOptimizer.step` -- the executor's own call -- over
stand-ins for the symmetric buffers.  The property checked is the one a data-parallel user relies on: after the step every
replica holds exactly what the one-GPU `adamw_kernel` computes from the summed gradient.

Gradients are dyadic (small integers times 2^-12), so every sum over ranks is exact in fp32 and "the summed gradient" is one
well-defined tensor.  The cross-rank barriers are never launched: with n > 1 on one device they would wait for peers that
do not exist.
"""
import ctypes
import dataclasses

import pytest
import torch
from test_step_numerics_gpu import adamw_ref, close, gen, ops  # noqa: F401  (ops: the kernel-layer fixture)

pytestmark = pytest.mark.gpu

B1, B2, EPS, WD = 0.9, 0.95, 1e-8, 0.1
NAN32 = 0x7FC0DEAD          # NaN sentinels with a payload, compared by bit pattern
NAN16 = 0x7FC1
WRONG = dict(lr=123.0, step=1000, grad_scale=7.0)   # host scalars of ops.adamw_step: the kernel must take `hyper` instead


class _Peers:
    """Stand-in for parallel.symm.SymmetricBuffer: every virtual rank's buffer is a plain tensor on this device."""

    def __init__(self, lib, bufs, rank):
        self.lib = lib
        self.ptr_array = (ctypes.c_void_p * len(bufs))(*[b.data_ptr() for b in bufs])
        self.local_ptr = bufs[rank].data_ptr()
        self.world, self.rank = len(bufs), rank


def virtual_ranks(ops, grads, params):
    """One FusedShardedOptimizer per virtual rank over the given per-rank buffers (unicast path, no barrier)."""
    from tepdist_b200.parallel import symm
    lib = ops.lib()
    symm._sigs(lib)
    out = []
    for r in range(len(grads)):
        fo = object.__new__(symm.FusedShardedOptimizer)
        fo.g, fo.p = _Peers(lib, grads, r), _Peers(lib, params, r)
        fo.world, fo.rank = len(grads), r
        fo.g16, fo.mc, fo.dry, fo.mc_ctas = None, None, False, 0
        fo._barrier = None        # a barrier call would fail here instead of spinning on peers that do not exist
        out.append(fo)
    return out


def sentinel(n, dtype=torch.float32):
    if dtype == torch.float32:
        return torch.full((n,), NAN32, dtype=torch.int32, device="cuda").view(torch.float32)
    return torch.full((n,), NAN16, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def same_bits(what, got, want):
    g, w = bits(got), bits(want)
    bad = g != w
    if bool(bad.any()):
        i = int(bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {g.numel()} elements differ in their bits; first at {i}: "
                             f"{got[i].item()!r} vs {want[i].item()!r}")


def dyadic(n):
    return torch.randint(-1024, 1025, (n,), device="cuda", generator=gen()).float() * 2.0 ** -12


def hyper_for(s):
    """{lr, bc1, bc2, grad scale} of step s + 1, as the executor's device `hyper` tensor carries them."""
    return torch.tensor([1e-2 * (s + 1) / 3, 1 - B1 ** (s + 1), 1 - B2 ** (s + 1), 0.25], device="cuda")


def _seed(s):
    gen().manual_seed(s)
    torch.manual_seed(s)


REPORT = {}


def _record(key, ratio):
    REPORT[key] = max(REPORT.get(key, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, v in sorted(REPORT.items()):
        print(f"largest |kernel - fp64| / tolerance, {k}: {v:.3g}")


# ============================================================================================== the kernel over one range
class RangeCase:
    """n virtual ranks sharing one flat range [s0, e0) of `chunk` elements per rank, inside buffers padded with NaN
    sentinels.  Rank r owns [s0 + r chunk, s0 + (r + 1) chunk); its master / m / v hold values only there."""

    def __init__(self, ops, n, chunk, n_decay, local_grad=False, lead=64, trail=68):
        self.ops, self.n, self.chunk, self.local = ops, n, chunk, local_grad
        self.N, self.s0, self.e0 = lead + n * chunk + trail, lead, lead + n * chunk
        self.nd = n_decay
        self.own = [(self.s0 + r * chunk, self.s0 + (r + 1) * chunk) for r in range(n)]
        L = self.e0 - self.s0
        self.P0 = torch.randn(L, device="cuda", generator=gen())
        self.M0 = torch.randn(L, device="cuda", generator=gen()) * 1e-2
        self.V0 = torch.rand(L, device="cuda", generator=gen()) * 1e-3 + 1e-6
        # per step: every rank's gradient of the range (local_grad: the one complete gradient every rank holds)
        self.steps = [([dyadic(L) for _ in range(1 if local_grad else n)], hyper_for(s)) for s in range(3)]
        self.grads = [sentinel(self.N) for _ in range(n)]
        self.params = [sentinel(self.N, torch.bfloat16) for _ in range(n)]
        self.state = [[sentinel(self.N) for _ in range(3)] for _ in range(n)]     # master, m, v per rank
        self.hyper = torch.zeros(4, device="cuda")
        self.fos = virtual_ranks(ops, self.grads, self.params)

    def reset(self):
        for r, (a, b) in enumerate(self.own):
            for buf, init in zip(self.state[r], (self.P0, self.M0, self.V0)):
                buf.copy_(sentinel(self.N))
                buf[a:b].copy_(init[a - self.s0:b - self.s0])
            self.params[r].copy_(sentinel(self.N, torch.bfloat16))

    def load(self, s):
        gs, h = self.steps[s]
        if not self.local:
            for r in range(self.n):
                self.grads[r][self.s0:self.e0].copy_(gs[r])
        self.hyper.copy_(h)

    def launch_all(self, s, ctas):
        """Every rank's call, rank by rank.  local_grad: before rank r's call only r's gradient buffer holds the
        gradient; every peer's is NaN, so reading any of them would poison the result."""
        for r, fo in enumerate(self.fos):
            a, b = self.own[r]
            if self.local:
                for q in range(self.n):
                    self.grads[q].copy_(sentinel(self.N))
                self.grads[r][self.s0:self.e0].copy_(self.steps[s][0][0])
            fo.step(*self.state[r], a, b, self.nd, self.hyper, B1, B2, EPS, WD, ctas=ctas, local_grad=self.local)

    def summed(self, s):
        gs = self.steps[s][0]
        return gs[0] if self.local else torch.stack([g.double() for g in gs]).sum(0).float()

    def gathered(self, k):
        """The owners' chunks of master (k = 0), m (1) or v (2), put back together over [s0, e0)."""
        return torch.cat([self.state[r][k][a:b] for r, (a, b) in enumerate(self.own)])

    def snapshot(self):
        return [self.gathered(k).clone() for k in range(3)] + [p.clone() for p in self.params]

    def check_sentinels(self, what):
        for r, (a, b) in enumerate(self.own):
            for k, name in enumerate(("master", "m", "v")):
                buf = bits(self.state[r][k])
                assert bool((buf[:a] == NAN32).all() and (buf[b:] == NAN32).all()), f"{what}: rank {r} {name} written outside its chunk"
            pb = bits(self.params[r])
            assert bool((pb[:self.s0] == NAN16).all() and (pb[self.e0:] == NAN16).all()), f"{what}: rank {r} parameters written outside the range"
            gb = bits(self.grads[r])
            assert bool((gb[:self.s0] == NAN32).all() and (gb[self.e0:] == NAN32).all()), f"{what}: rank {r} gradient buffer written"


def run_eager(case, ctas, tag):
    """Three steps; each checked against fp64 and bit for bit against ops.adamw_step on the summed gradient."""
    ops, s0, e0 = case.ops, case.s0, case.e0
    case.reset()
    nd_local = min(max(case.nd - s0, 0), e0 - s0)
    P, M, V = case.P0.clone(), case.M0.clone(), case.V0.clone()
    snaps = []
    for s in range(3):
        case.load(s)
        n0 = ops.launch_count()
        case.launch_all(s, ctas)
        assert ops.launch_count() == n0 + case.n
        torch.cuda.synchronize()
        G = case.summed(s)
        p_ref, m_ref, v_ref, (tp, tm, tv) = adamw_ref(P, G, M, V, case.hyper, nd_local, B1, B2, EPS, WD)
        got = case.snapshot()
        for k, (name, ref, tol) in enumerate((("master", p_ref, tp), ("m", m_ref, tm), ("v", v_ref, tv))):
            _record(f"{'local_grad' if case.local else 'summed'} {name}", close(f"{tag} step {s + 1} {name}", got[k], ref, tol))
        pb = torch.empty(e0 - s0, dtype=torch.bfloat16, device="cuda")
        ops.adamw_step(P, G, M, V, pb, nd_local, WRONG["lr"], B1, B2, EPS, WD, WRONG["step"],
                       grad_scale=WRONG["grad_scale"], hyper=case.hyper)
        for name, a, b in (("master", got[0], P), ("m", got[1], M), ("v", got[2], V)):
            same_bits(f"{tag} step {s + 1} {name} vs ops.adamw_step", a, b)
        same_bits(f"{tag} step {s + 1} bf16 copy vs ops.adamw_step", pb, P.to(torch.bfloat16))
        for r in range(case.n):
            same_bits(f"{tag} step {s + 1} rank {r} parameters vs bf16(master)", case.params[r][s0:e0], got[0].to(torch.bfloat16))
        case.check_sentinels(f"{tag} step {s + 1}")
        snaps.append(got)
    return snaps


N_VIRTUAL = (1, 2, 3, 4, 8)
CHUNK = 4 * 10_001           # whole float4s, not whole 8-element groups


def _decay_at(where, n, s0):
    mid = n // 2
    return s0 + mid * CHUNK + (4 * 37 + 2 if where == "float4" else 0)


@pytest.mark.parametrize("where", ["float4", "chunk"])
@pytest.mark.parametrize("n", N_VIRTUAL)
def test_sharded_adamw_equals_one_gpu_adamw_on_the_summed_gradient(ops, n, where):
    """Decay boundary inside a float4 (where="float4") or exactly on a chunk boundary (where="chunk"); three steps with
    non-zero moments; CTA counts 1, the overlap budget and the default give the same bits; then every rank's calls, captured
    once in a CUDA graph and replayed with new gradients and `hyper`, reproduce the eager bits."""
    _seed(40 + n)
    case = RangeCase(ops, n, CHUNK, _decay_at(where, n, 64))
    runs = {ctas: run_eager(case, ctas, f"n={n} decay@{where} ctas={ctas}") for ctas in (1, ops._sms() // 2, 0)}
    ref = runs[0]
    for ctas, snaps in runs.items():
        for s, (a, b) in enumerate(zip(snaps, ref)):
            for k, (x, y) in enumerate(zip(a, b)):
                same_bits(f"n={n} ctas={ctas} vs default, step {s + 1}, output {k}", x, y)

    case.reset()
    case.load(0)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side), torch.cuda.graph(graph):
        case.launch_all(0, 0)
    torch.cuda.current_stream().wait_stream(side)
    case.reset()                                    # (capture records, it does not run)
    for s in range(3):
        case.load(s)
        graph.replay()
        torch.cuda.synchronize()
        for k, (x, y) in enumerate(zip(case.snapshot(), ref[s])):
            same_bits(f"n={n} graph replay {s + 1}, output {k}", x, y)
        case.check_sentinels(f"n={n} graph replay {s + 1}")


@pytest.mark.parametrize("n", N_VIRTUAL)
def test_local_gradient_mode_reads_only_the_local_gradient(ops, n):
    """local_grad=True (replicated-gradient variables): the update uses the rank's own complete gradient and still stores
    the bf16 result to every rank.  Every peer's gradient buffer is NaN during each rank's call."""
    _seed(60 + n)
    case = RangeCase(ops, n, CHUNK, _decay_at("float4", n, 64), local_grad=True)
    run_eager(case, 0, f"n={n} local_grad")


def test_misaligned_ranges_and_too_many_ranks_are_refused_before_any_launch(ops):
    _seed(70)
    n, N = 2, 4096
    grads = [dyadic(N) for _ in range(n)]
    params = [sentinel(N, torch.bfloat16) for _ in range(n)]
    state = [sentinel(N) for _ in range(3)]
    before = [t.clone() for t in grads + params + state]
    hyper = hyper_for(0)
    fo = virtual_ranks(ops, grads, params)[0]
    for begin, end in ((2, 1024), (0, 1022), (4, 1030)):
        n0 = ops.launch_count()
        with pytest.raises(RuntimeError, match="fused_rs_adamw_ag"):
            fo.step(*state, begin, end, 512, hyper, B1, B2, EPS, WD)
        assert ops.launch_count() == n0
    nine = virtual_ranks(ops, [grads[0]] * 9, [params[0]] * 9)[0]
    for local in (False, True):
        n0 = ops.launch_count()
        with pytest.raises(RuntimeError, match="fused_rs_adamw_ag"):
            nine.step(*state, 0, 1024, 512, hyper, B1, B2, EPS, WD, local_grad=local)
        assert ops.launch_count() == n0
    torch.cuda.synchronize()
    for i, (t, t0) in enumerate(zip(grads + params + state, before)):
        same_bits(f"buffer {i} after refused calls", t, t0)


# ============================================================================================== the executor's layout
@pytest.fixture
def gpt2_layout(monkeypatch):
    """flat_zero_layout of the two-layer GPT-2 at the 345M widths, planned "dp" over n ranks (store laid out on the meta
    device, as the executor lays it out)."""
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    from tepdist_b200.parallel import plan_spmd
    from tepdist_b200.runtime import executor as ex

    monkeypatch.setattr(ex, "init_tensor", lambda init, full, seed, name, shard=None: ex.shard_of(torch.empty(full, device="meta"), *shard))
    g = build_gpt2_graph(dataclasses.replace(CONFIGS["345M"], n_layer=2), batch=8)

    def make(n):
        gs, _ = plan_spmd(g, n, "dp")
        fz = ex.Executor._analyze_flat_zero(gs)
        st = ex.VariableStore(gs, torch.device("meta"), tail=fz["irregular_params"], tail_align=n * ex._ALIGN)
        lay = ex.flat_zero_layout(st, fz, n, dict(gs.meta.get("optimizer") or {}))
        assert lay is not None and not fz["irregular_params"] and not lay.replicated
        return st, lay
    return make


@pytest.mark.parametrize("branch", ["fused", "nccl"])
@pytest.mark.parametrize("n", [2, 4, 8])
def test_layout_composes_to_one_whole_buffer_adamw(ops, gpt2_layout, n, branch):
    """Every virtual rank runs the calls the layout gives it, in the executor's order and with its CTA budgets (fused
    branch: FusedShardedOptimizer.step; NCCL branch: ops.adamw_step on the owned slice of the summed gradient, then the
    owners' bf16 chunks copied to every rank as the all-gather would).  Every rank's bf16 parameters, and the owners'
    master / m / v chunks put back together, must equal ONE whole-buffer ops.adamw_step bit for bit."""
    st, lay = gpt2_layout(n)
    _seed(80 + n)
    T = lay.total
    P0 = torch.randn(T, device="cuda", generator=gen()) * 0.02
    M0 = torch.randn(T, device="cuda", generator=gen()) * 1e-3
    V0 = torch.rand(T, device="cuda", generator=gen()) * 1e-5 + 1e-9
    grads = [dyadic(T) for _ in range(n)]
    G = grads[0].clone()
    for g_ in grads[1:]:
        G += g_                   # exact: dyadic values
    hyper = hyper_for(1)
    P, M, V = P0.clone(), M0.clone(), V0.clone()
    pb = torch.empty(T, dtype=torch.bfloat16, device="cuda")
    ops.adamw_step(P, G, M, V, pb, st.n_decay, WRONG["lr"], B1, B2, EPS, WD, WRONG["step"], grad_scale=WRONG["grad_scale"], hyper=hyper)

    params = [sentinel(T, torch.bfloat16) for _ in range(n)]
    state = [[P0.clone(), M0.clone(), V0.clone()] for _ in range(n)]
    overlap = ops._sms() // 2
    if branch == "fused":
        fos = virtual_ranks(ops, grads, params)
        for r in range(n):
            calls = lay.calls(r)
            for j, (a, b, nd, local) in enumerate(calls):
                fos[r].step(*state[r], a, b, nd, hyper, B1, B2, EPS, WD, ctas=0 if j == len(calls) - 1 else overlap,
                            local_grad=local)
    else:
        # as the collectives place them: reduce_scatter_tensor gives rank r the sum of every rank's r-th chunk of the bucket,
        # all_gather_into_tensor puts rank q's slice at the q-th chunk of every rank's bucket
        for r in range(n):
            for i in lay.order():
                s0, e0, _, _ = lay.ranges[i]
                a, b, nd, local = lay.call(i, r)
                c = (e0 - s0) // n
                red = grads[r][a:b] if local else G[s0 + r * c:s0 + (r + 1) * c]
                ops.adamw_step(state[r][0][a:b], red, state[r][1][a:b], state[r][2][a:b], params[r][a:b],
                               lay.local_decay(a, b, nd), WRONG["lr"], B1, B2, EPS, WD, WRONG["step"],
                               grad_scale=WRONG["grad_scale"], hyper=hyper)
        for i, (s0, e0, _, _) in enumerate(lay.ranges):
            c = (e0 - s0) // n
            sent = [params[q][slice(*lay.call(i, q)[:2])].clone() for q in range(n)]
            for r in range(n):
                for q in range(n):
                    params[r][s0 + q * c:s0 + (q + 1) * c].copy_(sent[q])
    torch.cuda.synchronize()

    covered = sorted((s0, e0) for s0, e0, _, _ in lay.ranges)
    assert covered[0][0] == 0 and covered[-1][1] == T and all(x[1] == y[0] for x, y in zip(covered, covered[1:]))
    for r in range(n):
        same_bits(f"{branch} n={n}: rank {r} parameters vs whole-buffer adamw", params[r], pb)
    for k, (name, want) in enumerate((("master", P), ("m", M), ("v", V))):
        owned = torch.empty_like(want)
        for r in range(n):
            for a, b, _, _ in lay.calls(r):
                owned[a:b] = state[r][k][a:b]
        same_bits(f"{branch} n={n}: owners' {name} chunks vs whole-buffer adamw", owned, want)
