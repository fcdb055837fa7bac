"""Element-by-element numerics of the kernels a GPT-MoE training step launches (the route-table row gathers of
moe_sm90.cu, ops.einsum on the batched wgmma GEMM, the top-2 routing of moe_dispatch_mask), and every parameter's
gradient of whole GPT-MoE steps against the fp32 CPU executor routed like the GPU.

Conventions as in test_step_numerics_gpu.py: every case checks that our kernel ran, and compares each element with a
reference computed in fp64 from the same bf16 / fp32 inputs; bit for bit where the arithmetic is exact, otherwise within a
per-element bound derived from the kernel's arithmetic and stated beside the case.  Route tables are always in bounds:
rc in [0, C) (dropped routes included), re in [-1, E), slot_src in [-1, S).
"""
import ctypes
import re
import time

import pytest
import torch

from test_step_numerics_gpu import (FTZ, U32, bf16_tol, close, exact, gen, ints, launched, ops, randn,  # noqa: F401
                                    step_checks, _seed)

pytestmark = pytest.mark.gpu

NAN = float("nan")


class _RecordingLib:
    """Wraps the kernel library and counts calls per entry point.  Before forwarding a call to a MoE route-table kernel (whose
    operands are all distinct tensors) it fails if two of its pointer arguments are equal: an operand whose temporary copy
    was freed before the launch, its address handed to the next operand's copy.  With `forbid` set, every call fails before
    it is forwarded (a case in which no kernel may run)."""

    def __init__(self, real, sig):
        self.real, self.sig, self.calls, self.forbid = real, sig, {}, False

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        kinds = getattr(self.sig, name)

        def call(*args):
            assert not self.forbid, f"{name} was called where no kernel may run"
            if name.startswith("tepd_moe_"):
                ptrs = [a for a, k in zip(args[:-1], kinds[:-1]) if k is ctypes.c_void_p and a]   # (the last is the stream)
                assert len(set(ptrs)) == len(ptrs), f"{name}: two pointer arguments share an address: {ptrs}"
            self.calls[name] = self.calls.get(name, 0) + 1
            return fn(*args)
        return call

    def total(self):
        return sum(self.calls.values())


@pytest.fixture
def recorded(ops, monkeypatch):
    lib = _RecordingLib(ops.lib(), ops._Sig)
    monkeypatch.setattr(ops, "lib", lambda: lib)
    return lib


# ============================================================================================== A. route-table kernels
# (G, S, E, C, M): the step shape; M = 8 / 264 / 776, whose M / 8 vectors leave the 32 lanes a partial last pass; odd
# (G, E, C) = (3, 5, 7), so the grid's last block is partial; G > 1 with S != C.
ROUTE_SHAPES = [(2, 1024, 8, 256, 768), (2, 64, 4, 16, 8), (2, 64, 4, 16, 264), (2, 64, 4, 16, 776), (3, 10, 5, 7, 24),
                (4, 96, 6, 40, 128)]
ROUTE_IDS = ["G{}S{}E{}C{}M{}".format(*s) for s in ROUTE_SHAPES]


def slot_tables(G, S, E, C):
    """slot_src int32 [G, E, C] in [-1, S) and w fp32 [G, E, C].  About a quarter of the slots are empty; valid slots never
    name token 0 (the row an empty slot's address is computed from) and several slots share token 1; some valid slots
    have w = 0."""
    slot_src = torch.randint(1, S, (G, E, C), device="cuda", generator=gen(), dtype=torch.int32)
    slot_src[torch.rand(G, E, C, device="cuda", generator=gen()) < 0.25] = -1
    slot_src[:, 0, 0] = -1
    slot_src[:, :, C - 1] = 1                                   # token 1 in E slots of every group
    w = (torch.rand(G, E, C, device="cuda", generator=gen()) * 1.9 + 0.1) * (torch.randint(0, 2, (G, E, C), device="cuda",
                                                                                           generator=gen()) * 2 - 1)
    w[torch.rand(G, E, C, device="cuda", generator=gen()) < 0.1] = 0.0
    return slot_src, w


def gather_src(G, S, M, slot_src):
    """src [G, S, M] bf16: random rows, NaN in every row no valid slot names (token 0 among them)."""
    src = randn(G, S, M)
    named = torch.zeros(G, S + 1, dtype=torch.bool, device="cuda")
    named.scatter_(1, (slot_src.long() % (S + 1)).reshape(G, -1), True)         # -1 lands in the dummy column S
    src[~named[:, :S]] = NAN
    return src


def gather_ref(src, slot_src, w):
    """bf16(fp32(w * src)) where slot_src >= 0 (the fp64 product of an fp32 and a bf16 is exact, then the kernel's two
    round-to-nearest steps), +0 elsewhere; [E, G, C, M]."""
    G = src.shape[0]
    valid = (slot_src >= 0).unsqueeze(-1)
    rows = src.double()[torch.arange(G, device="cuda").view(G, 1, 1), slot_src.clamp(min=0).long()]      # [G, E, C, M]
    prod = (w.double().unsqueeze(-1) * rows).float().to(torch.bfloat16)
    return torch.where(valid, prod, torch.zeros_like(prod)).permute(1, 0, 2, 3).contiguous()


@pytest.mark.parametrize("G,S,E,C,M", ROUTE_SHAPES, ids=ROUTE_IDS)
def test_moe_gather_scale_exact(ops, G, S, E, C, M):
    """Bit for bit: empty slots are +0 (their NaN row 0 must not leak), w = 0 on a negative value gives -0 exactly as the
    fp32 product does, one token fills several slots."""
    _seed(G * S + M)
    slot_src, w = slot_tables(G, S, E, C)
    src = gather_src(G, S, M, slot_src)
    out = launched(ops, ops.moe_gather_scale, src, slot_src, w, E, C)
    ref = gather_ref(src, slot_src, w)
    neg_zero = (ref.view(torch.int16) == torch.tensor(-0x8000, dtype=torch.int16, device="cuda"))
    assert bool(neg_zero.any()) and bool((slot_src < 0).any()), "case lost its -0 products or its empty slots"
    exact(f"moe_gather_scale {G}x{S}x{E}x{C}x{M}", out, ref)


def route_tables(G, S, E, C, K):
    """re int32 [G, S, K] in [-1, E), rc in [0, C - 1) for kept routes and C - 1 for dropped ones, gw fp32 with gw != 0 on
    dropped routes too.  Tokens 0 and S - 1 of every group have all K routes dropped."""
    re_ = torch.randint(0, E, (G, S, K), device="cuda", generator=gen(), dtype=torch.int32)
    drop = torch.rand(G, S, K, device="cuda", generator=gen()) < 0.2
    drop[:, 0] = drop[:, -1] = True
    re_[drop] = -1
    rc = torch.randint(0, C - 1, (G, S, K), device="cuda", generator=gen(), dtype=torch.int32)
    rc[drop] = C - 1
    gw = torch.rand(G, S, K, device="cuda", generator=gen()) * 1.9 + 0.1
    return re_, rc, gw, drop


def expert_rows(y, re_, rc):
    """y[re, g, rc, :] in fp64 for every route ([G, S, K, M]); dropped routes read row (0, g, C - 1)."""
    G = re_.shape[0]
    return y.double()[re_.clamp(min=0).long(), torch.arange(G, device="cuda").view(G, 1, 1), rc.long()]


@pytest.mark.parametrize("K", [1, 2, 4])
@pytest.mark.parametrize("G,S,E,C,M", ROUTE_SHAPES, ids=ROUTE_IDS)
def test_moe_combine_sum(ops, G, S, E, C, M, K):
    """Dyadic data (integer y, gw in multiples of 1/8, |sum| <= 24): every fp32 partial sum is exact, so bit for bit.  Random
    data: K products and K additions in fp32 (FMA-contracted or not), within K u sum|gw y| before the bf16 store.  Slot
    C - 1 of every expert holds NaN and only dropped routes (gw != 0) name it; tokens whose routes are all dropped give +0."""
    _seed(G * S * K + M)
    re_, rc, gw, drop = route_tables(G, S, E, C, K)
    for data in ("dyadic", "random"):
        if data == "dyadic":
            y = ints(E, G, C, M)
            w = torch.randint(-16, 17, (G, S, K), device="cuda", generator=gen()).float() / 8
        else:
            y, w = randn(E, G, C, M), gw * torch.where(torch.rand(G, S, K, device="cuda", generator=gen()) < 0.5, -1.0, 1.0)
        y[:, :, C - 1] = NAN
        out = launched(ops, ops.moe_combine_sum, y, re_, rc, w, S)
        terms = torch.where(drop.unsqueeze(-1), torch.zeros((), dtype=torch.float64, device="cuda"),
                            w.double().unsqueeze(-1) * expert_rows(y, re_, rc))
        ref = terms.sum(2) + 0.0                              # (+0.0: an all-dropped row is +0, as the kernel's accumulator)
        what = f"moe_combine_sum {data} {G}x{S}x{E}x{C}x{M} K={K}"
        if data == "dyadic":
            exact(what, out, ref.float().to(torch.bfloat16))
        else:
            close(what, out, ref, bf16_tol(ref, K * U32 * terms.abs().sum(2)))
        exact(f"{what}: all-dropped tokens", out[:, [0, S - 1]], torch.zeros(G, 2, M, dtype=torch.bfloat16, device="cuda"))


@pytest.mark.parametrize("K", [1, 2, 4])
@pytest.mark.parametrize("G,S,E,C,M", ROUTE_SHAPES, ids=ROUTE_IDS)
def test_moe_route_dots(ops, G, S, E, C, M, K):
    """Integer operands with products <= 9 (sums below 9 M < 2^24): exact in any order, so bit for bit.  Random data: each
    lane sums M / 256 runs of 8 products, then 5 shuffle levels: within M u sum|a b|.  Dropped routes are exactly 0 (their
    row C - 1 holds NaN)."""
    _seed(G * S * K + M + 1)
    re_, rc, _, drop = route_tables(G, S, E, C, K)
    for data in ("integer", "random"):
        a, b = (ints(G, S, M), ints(E, G, C, M)) if data == "integer" else (randn(G, S, M), randn(E, G, C, M))
        b[:, :, C - 1] = NAN
        dots = launched(ops, ops.moe_route_dots, a, b, re_, rc)
        prods = torch.where(drop.unsqueeze(-1), torch.zeros((), dtype=torch.float64, device="cuda"),
                            a.double().unsqueeze(2) * expert_rows(b, re_, rc))
        ref = prods.sum(-1)
        what = f"moe_route_dots {data} {G}x{S}x{E}x{C}x{M} K={K}"
        if data == "integer":
            exact(what, dots, ref)
        else:
            close(what, dots, ref, M * U32 * prods.abs().sum(-1) + FTZ)
        assert bool((dots[drop] == 0).all()), f"{what}: a dropped route is not 0"


def strided(t):
    """The same values as a non-contiguous view (every other element of the last dim of a buffer twice as wide)."""
    buf = torch.full(t.shape[:-1] + (2 * t.shape[-1],), 7, dtype=t.dtype, device=t.device)
    v = buf[..., ::2]
    v.copy_(t)
    assert not v.is_contiguous()
    return v


def test_moe_wrappers_non_contiguous_operands(ops, recorded):
    """Every operand of each wrapper as a non-contiguous view, with same-sized pairs (slot_src / w, re / rc / gw): the result
    equals the contiguous call bit for bit, and no call hands the kernel two operands at one address."""
    _seed(50)
    G, S, E, C, M, K = 2, 64, 4, 16, 264, 2
    slot_src, w = slot_tables(G, S, E, C)
    src = gather_src(G, S, M, slot_src)
    want = launched(ops, ops.moe_gather_scale, src, slot_src, w, E, C)
    exact("moe_gather_scale, strided operands", launched(ops, ops.moe_gather_scale, strided(src), strided(slot_src),
                                                        strided(w), E, C), want)
    re_, rc, gw, _ = route_tables(G, S, E, C, K)
    y = randn(E, G, C, M)
    want = launched(ops, ops.moe_combine_sum, y, re_, rc, gw, S)
    exact("moe_combine_sum, strided operands", launched(ops, ops.moe_combine_sum, strided(y), strided(re_), strided(rc),
                                                       strided(gw), S), want)
    a = randn(G, S, M)
    want = launched(ops, ops.moe_route_dots, a, y, re_, rc)
    exact("moe_route_dots, strided operands", launched(ops, ops.moe_route_dots, strided(a), strided(y), strided(re_),
                                                      strided(rc)), want)
    assert recorded.calls == {"tepd_moe_gather_scale": 2, "tepd_moe_combine_sum": 2, "tepd_moe_route_dots": 2}, recorded.calls


def test_moe_wrappers_refuse_bad_tables(ops, recorded):
    """The kernels trust the tables: a non-int32 index table, a non-fp32 weight or a table whose shape does not match the
    data operand is refused before any launch (several of these would make the kernel read outside its tensors)."""
    _seed(51)
    G, S, E, C, M, K = 2, 64, 4, 16, 64, 2
    slot_src, w = slot_tables(G, S, E, C)
    src = gather_src(G, S, M, slot_src)
    re_, rc, gw, _ = route_tables(G, S, E, C, K)
    y, a = randn(E, G, C, M), randn(G, S, M)
    bad = [
        (ops.moe_gather_scale, (src, slot_src.long(), w, E, C), "slot_src"),
        (ops.moe_gather_scale, (src, slot_src, w.double(), E, C), "w"),
        (ops.moe_gather_scale, (src, slot_src, w.bfloat16(), E, C), "w"),
        (ops.moe_gather_scale, (src, slot_src[:, :, :C - 1], w[:, :, :C - 1], E, C), "slot_src"),
        (ops.moe_gather_scale, (src[:1], slot_src, w, E, C), "slot_src"),
        (ops.moe_combine_sum, (y, re_.long(), rc, gw, S), "re"),
        (ops.moe_combine_sum, (y, re_, rc.short(), gw, S), "rc"),
        (ops.moe_combine_sum, (y, re_, rc, gw.bfloat16(), S), "gw"),
        (ops.moe_combine_sum, (y, re_, rc, gw, S - 1), "re"),
        (ops.moe_combine_sum, (y, re_, rc[:, :, :1], gw, S), "rc"),
        (ops.moe_combine_sum, (y[:, :1], re_, rc, gw, S), "re"),
        (ops.moe_route_dots, (a, y, re_.long(), rc), "re"),
        (ops.moe_route_dots, (a, y, re_, rc.float()), "rc"),
        (ops.moe_route_dots, (a, y, re_[:1], rc[:1]), "re"),
        (ops.moe_route_dots, (a[:1], y, re_[:1], rc[:1]), "b must be"),
        (ops.moe_route_dots, (a, y[..., :M - 8], re_, rc), "b must be"),
    ]
    n0 = ops.launch_count()
    recorded.forbid = True
    for fn, args, match in bad:
        with pytest.raises(ValueError, match=match):
            fn(*args)
    assert ops.launch_count() == n0 and recorded.total() == 0, recorded.calls


# ============================================================================================== B. ops.einsum, exact
# Integer operands in [-3, 3]: every product is at most 9 and the longest contraction (H = 6144) sums to at most 55,296 <
# 2^24, so the fp32 accumulator of any schedule is exact and the bf16 output equals the round-to-nearest-even cast of the
# fp64 einsum.  Each call must be exactly one launch of the GEMM (ops.einsum falls back to torch.einsum silently).
EINSUM_EQS = ["GSEC,GSM->EGCM", "EGCM,EMH->EGCH", "EGCH,EHM->EGCM", "GSEC,EGCM->GSM",           # forward
              "EGCM,GSM->GSEC", "GSEC,EGCM->GSM", "EGCH,EMH->EGCM", "EGCM,EGCH->EMH",           # vjps w.r.t. each operand
              "EGCM,EHM->EGCH", "EGCH,EGCM->EHM", "GSM,EGCM->GSEC", "GSEC,GSM->EGCM"]


def einsum_case(ops, recorded, eq, a, b):
    ia, ib = eq.split("->")[0].split(",")
    n0 = recorded.calls.get("tepd_gemm_bf16", 0)
    t0 = recorded.total()
    got = launched(ops, ops.einsum, eq, a, b)
    assert recorded.calls.get("tepd_gemm_bf16", 0) == n0 + 1 and recorded.total() == t0 + 1, f"{eq}: {recorded.calls}"
    ref = torch.einsum(eq, a.double(), b.double())
    assert tuple(got.shape) == tuple(ref.shape), (eq, tuple(got.shape), tuple(ref.shape))
    exact(f"einsum {eq} {tuple(a.shape)} x {tuple(b.shape)}", got, ref.float().to(torch.bfloat16))


@pytest.mark.parametrize("E", [8, 1], ids=["E8", "E1-local-expert"])
def test_einsum_moe_equations_exact(ops, recorded, E):
    """All 12 GPT-MoE equations at the step shape (E, G, S, C, M, H) = (8, 2, 1024, 256, 768, 6144), and at E = 1 (the local
    expert under EP-8, where the expert FCs and their gradients are one 2-D GEMM)."""
    _seed(60 + E)
    G, S, C, M, H = 2, 1024, 256, 768, 6144
    dims = dict(E=E, G=G, S=S, C=C, M=M, H=H)
    t = {k: ints(*(dims[c] for c in k)) for k in ("GSEC", "GSM", "EGCM", "EMH", "EGCH", "EHM")}
    for eq in EINSUM_EQS:
        ia, ib = eq.split("->")[0].split(",")
        einsum_case(ops, recorded, eq, t[ia], t[ib])


def test_einsum_copy_path_and_output_permute_exact(ops, recorded):
    """A non-contiguous operand on either side (the lowering copies it into [batch, rows, cols]), and output orders that differ
    from the GEMM's [batch, M, N] (the final permute)."""
    _seed(62)
    E, G, C, M, H = 4, 2, 128, 264, 520
    x, wi, wo = ints(E, G, C, M), ints(E, M, H), ints(E, H, M)
    einsum_case(ops, recorded, "EGCM,EMH->EGCH", x, strided(wi))
    einsum_case(ops, recorded, "EGCM,EMH->EGCH", strided(x), wi)
    einsum_case(ops, recorded, "EGCH,EGCM->EHM", strided(ints(E, G, C, H)), x)
    for eq in ("EGCM,EMH->GCEH", "EGCM,EMH->HEGC", "EGCH,EHM->MGEC"):
        ia, ib = eq.split("->")[0].split(",")
        a, b = {"EGCM": x, "EGCH": ints(E, G, C, H)}[ia], {"EMH": wi, "EHM": wo}[ib]
        einsum_case(ops, recorded, eq, a, b)


# ============================================================================================== C. routing
def gshard_top2(gates, C, k=2):
    """Plain statement of GShard top-k routing on fp64 gates [G, S, E]: round r takes each token's r-th largest gate (lowest
    expert index on ties); slots are handed out in token order; round r + 1 positions come after every claim of rounds <= r;
    a claim at position >= C is dropped.  -> choices, dense mask (fp32 gate of each kept claim at [g, s, e, pos]), re, rc,
    gw, slot_src, slot_w as Python lists."""
    G, S, E = len(gates), len(gates[0]), len(gates[0][0])
    choices = [[sorted(range(E), key=lambda e: (-gates[g][s][e], e))[:k] for s in range(S)] for g in range(G)]
    mask = [[[[0.0] * C for _ in range(E)] for _ in range(S)] for _ in range(G)]
    re_ = [[[-1] * k for _ in range(S)] for _ in range(G)]
    rc = [[[None] * k for _ in range(S)] for _ in range(G)]
    gw = [[[0.0] * k for _ in range(S)] for _ in range(G)]
    slot_src = [[[-1] * C for _ in range(E)] for _ in range(G)]
    slot_w = [[[0.0] * C for _ in range(E)] for _ in range(G)]
    for g in range(G):
        claims = [0] * E
        for r in range(k):
            for s in range(S):
                e = choices[g][s][r]
                pos = claims[e]
                claims[e] += 1
                if pos >= C:
                    continue
                assert slot_src[g][e][pos] == -1, "two tokens in one slot"
                mask[g][s][e][pos] = gates[g][s][e]
                re_[g][s][r], rc[g][s][r], gw[g][s][r] = e, pos, gates[g][s][e]
                slot_src[g][e][pos], slot_w[g][e][pos] = s, gates[g][s][e]
    return choices, mask, re_, rc, gw, slot_src, slot_w


def routing_logits(kind, G, S, E):
    """bf16 gate logits [G, S, E].  'ties': multiples of 1/2 in [-2, 2], so many tokens have equal gates among their top
    three; 'overflow': experts 0 and 1 favoured by +3 for most tokens; 'unpicked': expert E - 1 at -30 for every token."""
    if kind == "ties":
        lg = torch.randint(-4, 5, (G, S, E), device="cuda", generator=gen()).float() / 2
    else:
        lg = torch.randn(G, S, E, device="cuda", generator=gen())
        if kind == "overflow":
            lg[:, : 3 * S // 4, :2] += 3
        else:
            lg[..., E - 1] = -30
    return lg.to(torch.bfloat16)


@pytest.mark.parametrize("kind", ["ties", "overflow", "unpicked"])
def test_moe_dispatch_mask_matches_gshard_top2(ops, kind):
    """moe_dispatch_mask on the GPU executor of the MoE FFN graph (2 groups x 256 tokens, 8 experts, capacity 48, so the 512
    claims of a group exceed some experts' capacity), its gates set through the gate weight: W_gate = [I | 0] makes the
    gate logits the first E features of x exactly.  The dense mask bf16(gate) * sel, re, rc, gw, slot_src and slot_w must
    equal the fp64 statement of GShard routing on the captured fp32 gates exactly."""
    from tepdist_b200.models.gpt_moe import build_moe_ffn_graph
    from tepdist_b200.runtime.executor import Executor
    G, S, Mm, E, C = 2, 256, 64, 8, 48
    _seed(70)
    g = build_moe_ffn_graph(groups=G, tokens_per_group=S, model=Mm, hidden=128, experts=E, capacity=C)
    ex = Executor(g, torch.device("cuda", 0), seed=0, use_cuda_graph=False)
    ex.store.load_state_dict({"moe/gate/w": torch.eye(E, Mm)})
    x = randn(G, S, Mm)
    x[..., :E] = routing_logits(kind, G, S, E)
    seen = {}
    real_exec = ex._exec

    def exec_(n, ins, feeds):
        outs = real_exec(n, ins, feeds)
        if n.op == "moe_dispatch_mask":
            seen["gates"], seen["mask"], seen["id"] = ins[0].clone(), outs[0].clone(), n.id
        return outs
    ex._exec = exec_
    n0 = ops.launch_count()
    ex.step({"x": x, "t": randn(G, S, Mm)})
    torch.cuda.synchronize()
    assert ops.launch_count() > n0
    gates = seen["gates"]
    assert gates.dtype == torch.float32
    choices, mask, re_r, rc_r, gw_r, src_r, w_r = gshard_top2(gates.double().tolist(), C)
    rt = ex._moe_routes[(0, seen["id"])]

    # the gates have what this case is for
    top = gates.sort(-1, descending=True).values
    demand = torch.zeros(G, E, dtype=torch.long)
    for gi in range(G):
        for s in range(S):
            for e in choices[gi][s]:
                demand[gi, e] += 1
    if kind == "ties":
        assert int((top[..., 1] == top[..., 2]).sum() + (top[..., 0] == top[..., 1]).sum()) > S // 4, "too few exact ties"
    if kind == "overflow":
        assert int(demand.max()) > C
    if kind == "unpicked":
        assert bool((demand[:, E - 1] == 0).all())
    assert int(demand.max()) > C, "case lost its dropped claims"

    dev = lambda v, dt: torch.tensor(v, dtype=dt, device="cuda")
    exact(f"{kind}: dense mask", seen["mask"], dev(mask, torch.float64).float().to(torch.bfloat16))
    exact(f"{kind}: re", rt["re"], dev(re_r, torch.float64))
    kept = dev(re_r, torch.int64) >= 0
    rc_got = rt["rc"].long()
    assert bool(((rc_got >= 0) & (rc_got < C)).all()), "rc out of [0, C)"
    rc_ref = torch.tensor([[[-1 if c is None else c for c in t] for t in grp] for grp in rc_r], device="cuda")
    assert torch.equal(torch.where(kept, rc_got, -1), rc_ref), f"{kind}: rc differs on kept routes"
    exact(f"{kind}: gw", rt["gw"], dev(gw_r, torch.float64))
    assert rt["slot_src"].dtype == torch.int32 and rt["slot_w"].dtype == torch.float32
    exact(f"{kind}: slot_src", rt["slot_src"], dev(src_r, torch.float64))
    exact(f"{kind}: slot_w", rt["slot_w"], dev(w_r, torch.float64))
    exact(f"{kind}: executor's choices", ex._moe_choices(g.nodes[seen["id"]], gates), dev(choices, torch.float64))


# ============================================================================================== D. whole GPT-MoE steps
# Bound on each parameter's relative gradient error ||g_gpu - g_cpu|| / ||g_cpu|| against the fp32 CPU executor, keyed by
# the name without "model/" and "h<l>/" (the dense layer 0 and the attention / LayerNorms of MoE layer 1 share a key).  The
# oracle routes tokens as the GPU did (the GPU's expert choices, see Executor._moe_choices), so the comparison is of the
# same discrete routing (it would have chosen 32 to 51 of the 4096 routes differently on its own).  These bounds are
# measured, not derived: on an H100 80GB HBM3 at 700 W the largest values over the three steps were 3.2e-3 (ln_f/b) to
# 1.27e-2 (moe/gate/w), the expert FC weights 1.0e-2 although the einsum stores their gradients as bf16 before they are
# added to the fp32 buffer; each bound is about twice that kind's largest value.
MOE_GRAD_TOL = {"wte": 1.5e-2, "wpe": 1.5e-2, "attn/c_attn/w": 1.8e-2, "attn/c_attn/b": 1.6e-2, "attn/c_proj/w": 1.7e-2,
                "attn/c_proj/b": 1.5e-2, "ln_1/g": 1.8e-2, "ln_1/b": 1.6e-2, "ln_2/g": 2.5e-2, "ln_2/b": 2.2e-2,
                "mlp/c_fc/w": 1.4e-2, "mlp/c_fc/b": 1.3e-2, "mlp/c_proj/w": 1.4e-2, "mlp/c_proj/b": 1.1e-2,
                "moe/gate/w": 2.6e-2, "moe/expert_fc/wi": 2.1e-2, "moe/expert_fc/wo": 2.1e-2, "ln_f/g": 1.3e-2, "ln_f/b": 7e-3,
                "output": 1.3e-2}


def moe_kind(name):
    return re.sub(r"^model/(h\d+/)?", "", name)


def moe_grad_tol(name):
    return MOE_GRAD_TOL[moe_kind(name)]


def test_gpt_moe_steps_gradient_by_gradient(ops, recorded):
    """Two layers at the reference widths (layer 0 dense, layer 1 MoE: 8 experts, capacity 256, 2 groups of 1024 tokens as
    in the reference's 8 groups x batch 8).  Step 1 eager, step 2 CUDA-graph capture + replay, step 3 replay.  Every MoE
    einsum runs one route-table kernel, every other einsum one GEMM; each step drops at least one route and leaves at least
    one slot empty."""
    from tepdist_b200.models.gpt_moe import MoEConfig, build_gpt_moe_graph
    from tepdist_b200.runtime.executor import Executor
    cfg = MoEConfig(n_layer=2, hidden=768, ffn=6144, n_head=16, experts=8, capacity=256, groups=2, seq=1024, batch=2)
    g = build_gpt_moe_graph(cfg)
    gpu = Executor(g, torch.device("cuda", 0), seed=0, use_cuda_graph=True)
    cpu = Executor(g, torch.device("cpu"), seed=0)
    sched = lambda step: 1e-4 * min(1.0, step / 4)
    gpu.set_lr_schedule(sched)
    cpu.set_lr_schedule(sched)
    assert len(gpu._moe_einsum) == 6, gpu._moe_einsum
    masks = [n for n in g.nodes if n.op == "moe_dispatch_mask"]
    assert len(masks) == 1

    # the GPU's expert choices of every mask node (forward and backward), held so that CUDA-graph replays refresh them
    choices = {}
    real_choices = gpu._moe_choices

    def gpu_choices(n, gates):
        choices[n.id] = real_choices(n, gates)
        return choices[n.id]
    gpu._moe_choices = gpu_choices
    flips = []

    def cpu_choices(n, gates):
        got = choices[n.id].cpu()
        if n.op == "moe_dispatch_mask":
            flips.append(int((Executor._moe_choices(cpu, n, gates) != got).sum()))
        return got
    cpu._moe_choices = cpu_choices

    # one kernel per einsum node: route-table kernels for the six MoE einsums, the GEMM for the rest
    real_exec = gpu._exec

    def exec_(n, ins, feeds):
        before = dict(recorded.calls)
        outs = real_exec(n, ins, feeds)
        if n.op == "einsum":
            new = {k: v - before.get(k, 0) for k, v in recorded.calls.items() if v != before.get(k, 0)}
            if n.id in gpu._moe_einsum:
                kind = gpu._moe_einsum[n.id][0]
                want = {{"gather": "tepd_moe_gather_scale", "combine": "tepd_moe_combine_sum"}.get(kind, "tepd_moe_route_dots"): 1}
            else:
                want = {"tepd_gemm_bf16": 1}
            assert new == want, f"einsum {n.name} ({n.attrs.get('eq')}): launched {new}, expected {want}"
        return outs
    gpu._exec = exec_

    torch.manual_seed(0)
    tok = torch.randint(0, cfg.vocab, (cfg.batch, cfg.seq), dtype=torch.int32)
    lab = torch.roll(tok, -1, 1)
    fg, fc = {"tokens": tok.cuda(), "labels": lab.cuda()}, {"tokens": tok, "labels": lab}
    t0 = time.perf_counter()
    by_kind = {}
    for s, label in enumerate(("GPT-MoE step 1 (eager)", "GPT-MoE step 2 (capture + replay)", "GPT-MoE step 3 (replay)")):
        n0, c0 = ops.launch_count(), dict(recorded.calls)
        flips.clear()
        worst = step_checks(gpu, cpu, fg, fc, label, tol=moe_grad_tol)
        assert ops.launch_count() > n0
        assert (gpu._graph is None) == (s == 0)
        moe_calls = sum(v - c0.get(k, 0) for k, v in recorded.calls.items() if k.startswith("tepd_moe_"))
        assert moe_calls == (6 if s < 2 else 0), moe_calls      # (a replay runs no Python: its launches are the capture's)
        rt = gpu._moe_routes[(0, masks[0].id)]
        dropped, empty = int((rt["re"] < 0).sum()), int((rt["slot_src"] < 0).sum())
        print(f"  routes the fp32 oracle would have chosen differently: {flips[0]} of {rt['re'].numel()}; "
              f"dropped routes {dropped}, empty slots {empty}")
        assert dropped > 0 and empty > 0, (dropped, empty)
        for name, rel in worst.items():
            by_kind[moe_kind(name)] = max(by_kind.get(moe_kind(name), 0.0), rel)
    print("  largest relative error by kind over the steps: " + ", ".join(f"{k} {v:.2e}" for k, v in sorted(by_kind.items())))
    print(f"GPT-MoE steps with oracle: {time.perf_counter() - t0:.1f} s")
