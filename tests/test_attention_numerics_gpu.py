"""The flash-attention kernels (ops/csrc/attention_sm90.cu) element by element against the fp64 reference of
attention_reference.py, under its per-element bounds: head widths 64 and 128 and the widths padded onto them, sequence lengths
from one tile to 4096 and ragged causal ones, odd head counts, q / k / v as views of a fused qkv buffer and of head-major
storage, the dqkv_out path, and repeat determinism.  Then the context-parallel ring: its three small kernels (log-sum-exp
merge, fp32 accumulation, pack) and `RingAttention` itself, its ranks run as threads of this process on one GPU."""
import collections
import threading
import types

import pytest
import torch
import torch.distributed as dist

import attention_reference as ar

pytestmark = pytest.mark.gpu


def _inputs(B, S, H, D, layout, seed):
    """q, k, v [B, S, H, D] views sharing strides (as the kernels require) and a contiguous dO."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if layout == "fused":        # slices of the qkv projection output [B, S, H, 3, D], as the executor passes them
        qkv = torch.randn(B, S, H, 3, D, device="cuda", generator=g).to(torch.bfloat16)
        q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    else:                        # head-major [3, B, H, S, D] storage seen as bshd: stride_h > stride_s
        qkv = torch.randn(3, B, H, S, D, device="cuda", generator=g).to(torch.bfloat16)
        q, k, v = (t.permute(0, 2, 1, 3) for t in qkv)
        assert q.stride(2) > q.stride(1)
    do = torch.randn(B, S, H, D, device="cuda", generator=g).to(torch.bfloat16)
    return q, k, v, do


CASES = [   # (B, S, H, D, causal, layout)
    (2, 128, 2, 64, True, "fused"),
    (2, 256, 3, 64, False, "fused"),
    (2, 1024, 3, 64, True, "head_major"),
    (1, 4096, 2, 64, True, "fused"),
    (1, 4096, 1, 64, False, "head_major"),
    (2, 128, 1, 128, True, "head_major"),
    (2, 256, 3, 128, False, "fused"),
    (1, 1024, 3, 128, True, "fused"),
    (1, 4096, 2, 128, True, "head_major"),
    (2, 256, 2, 32, True, "fused"),          # widths zero-padded onto the 64 / 128 kernels
    (2, 1024, 3, 48, True, "head_major"),
    (2, 256, 2, 80, False, "fused"),
    (1, 1024, 3, 96, True, "fused"),
    (2, 256, 2, 112, True, "head_major"),
    (2, 200, 3, 64, True, "fused"),          # ragged causal sequences, padded to a multiple of 128
    (1, 1000, 2, 128, True, "head_major"),
    (2, 1000, 3, 48, True, "fused"),
]


@pytest.mark.parametrize("B,S,H,D,causal,layout", CASES,
                         ids=[f"B{b}-S{s}-H{h}-D{d}-{'causal' if c else 'full'}-{l}" for b, s, h, d, c, l in CASES])
def test_attention_matches_fp64_within_bounds_and_repeats(B, S, H, D, causal, layout, monkeypatch):
    """The second call writes its gradients into a NaN-filled dqkv_out buffer: it must fill every element, reproduce O, lse, dK
    and dV bit for bit, and keep dQ (summed over key blocks with fp32 reduce-adds in no fixed order) within its bound."""
    ops = ar.kernels_only(monkeypatch)
    q, k, v, do = _inputs(B, S, H, D, layout, seed=S + H + D)
    n0 = ops.launch_count()
    o, lse = ops.attention_fwd(q, k, v, causal=causal)
    dq, dk, dv = ops.attention_bwd(do, q, k, v, o, lse, causal=causal)
    buf = torch.full((B, S, H, 3, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    o2, lse2 = ops.attention_fwd(q, k, v, causal=causal)
    ops.attention_bwd(do, q, k, v, o2, lse2, causal=causal, dqkv_out=buf)
    torch.cuda.synchronize()
    assert ops.launch_count() >= n0 + 8, "attention kernels did not run"
    ref = ar.reference(q, k, v, do, causal)
    ref.check(o=o, lse=lse, dq=dq, dk=dk, dv=dv)
    assert torch.equal(o, o2) and torch.equal(lse, lse2)
    assert torch.equal(buf[:, :, :, 1], dk) and torch.equal(buf[:, :, :, 2], dv)
    ref.check(dq=buf[:, :, :, 0])


# ------------------------------------------------------------------ the ring's three kernels
def _spread(*shape, seed):
    """fp32 values over six decades, both signs."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g) * 10.0 ** torch.empty(*shape, device="cuda").uniform_(-3, 3, generator=g)


def test_ring_pack_is_the_round_to_nearest_even_cast(monkeypatch):
    ops = ar.kernels_only(monkeypatch)
    from tepdist_b200.ops.attention import attn_ring_pack
    B, L, H, D = 2, 256, 3, 64
    dq_acc, kv_acc = _spread(B, L, H, D, seed=1), _spread(B, L, H, 2, D, seed=2)
    out = torch.full((B, L, H, 3, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    n0 = ops.launch_count()
    attn_ring_pack(dq_acc, kv_acc, out)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0 + 1
    assert torch.equal(out[:, :, :, 0], dq_acc.to(torch.bfloat16))
    assert torch.equal(out[:, :, :, 1:], kv_acc.to(torch.bfloat16))


def test_ring_accum_is_an_exact_fp32_add_in_order(monkeypatch):
    """Three partials into the accumulators, compared with the same fp32 additions in the same order, bit for bit."""
    ops = ar.kernels_only(monkeypatch)
    from tepdist_b200.ops.attention import attn_ring_accum_
    B, L, H, D = 2, 256, 3, 128
    dq_acc, kv_acc = _spread(B, L, H, D, seed=3), _spread(B, L, H, 2, D, seed=4)
    want_q, want_kv = dq_acc.clone(), kv_acc.clone()
    n0 = ops.launch_count()
    for i in range(3):
        part = _spread(B, L, H, 3, D, seed=5 + i).to(torch.bfloat16)
        attn_ring_accum_(dq_acc, kv_acc, part)
        want_q += part[:, :, :, 0].float()
        want_kv += part[:, :, :, 1:].float()
    torch.cuda.synchronize()
    assert ops.launch_count() == n0 + 3
    assert torch.equal(dq_acc, want_q) and torch.equal(kv_acc, want_kv)


@pytest.mark.parametrize("D", [64, 128])
def test_ring_merge_matches_fp64_log_sum_exp(D, monkeypatch):
    """o_acc <- (w_a o_acc + w_j o_j), lse <- log(e^lse_acc + e^lse_j), w = e^(lse - lse_new), against fp64.  The kernel's
    __expf / __logf are ex2 / lg2 approximations (relative resp. absolute error about 2^-22) of fp32 arguments, whose rounding
    adds 2^-24 of the argument: the new log-sum-exp is off by e_lse <= 2^-20 + 2^-22 (|lse_acc - new| + |lse_j - new| + |new|),
    each weight relatively by e_lse + 2^-21 + 2^-23 |lse - new|, and the fp32 products and sum by 2^-23 of each term.  The
    bound is twice that."""
    ops = ar.kernels_only(monkeypatch)
    from tepdist_b200.ops.attention import attn_merge_
    B, L, H = 2, 256, 3
    g = torch.Generator(device="cuda").manual_seed(D)
    o_acc = torch.randn(B, L, H, D, device="cuda", generator=g)
    o_j = torch.randn(B, L, H, D, device="cuda", generator=g).to(torch.bfloat16)
    lse_acc = torch.empty(B, H, L, device="cuda").uniform_(-5, 15, generator=g)
    lse_j = lse_acc + torch.empty(B, H, L, device="cuda").uniform_(-12, 12, generator=g)
    lse_out = torch.full_like(lse_acc, float("nan"))
    first = torch.full_like(o_acc, float("nan"))
    first_lse = torch.full_like(lse_acc, float("nan"))
    n0 = ops.launch_count()
    attn_merge_(first, lse_acc, first_lse, o_j, lse_j, True)
    o_in = o_acc.clone()
    attn_merge_(o_acc, lse_acc, lse_out, o_j, lse_j, False)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0 + 2
    assert torch.equal(first, o_j.float()) and torch.equal(first_lse, lse_j)
    la, lj = lse_acc.double(), lse_j.double()
    new = torch.logaddexp(la, lj)
    e_lse = 2.0 ** -20 + 2.0 ** -22 * ((la - new).abs() + (lj - new).abs() + new.abs())
    ar.check(lse_out, new, 2 * e_lse, "lse")
    bshd = lambda t: t.permute(0, 2, 1).unsqueeze(-1)
    wa, wj = bshd(torch.exp(la - new)), bshd(torch.exp(lj - new))
    ea = bshd(e_lse + 2.0 ** -21 + 2.0 ** -23 * (la - new).abs()) + 2.0 ** -23
    ej = bshd(e_lse + 2.0 ** -21 + 2.0 ** -23 * (lj - new).abs()) + 2.0 ** -23
    ta, tj = wa * o_in.double(), wj * o_j.double()
    ar.check(o_acc, ta + tj, 2 * (ea * ta.abs() + ej * tj.abs()), "o")


# ------------------------------------------------------------------ RingAttention over virtual ranks
class _VirtualP2P:
    """torch.distributed's point-to-point calls between ranks that are threads of this process, on one GPU and its shared
    stream.  A send snapshots its tensor (a clone enqueued on the stream behind the writes that produced it); a receive's wait
    copies the message that matches it by (source, destination, posting order), or fails after `timeout` seconds.

    The attention kernels are not re-entrant: tepd_attn_bwd keeps process-wide workspaces (delta_buf and the fp32 dQ
    accumulator) shared by each call's delta, backward and dQ-cast launches, and ctypes releases the GIL during a call, so two
    ranks enqueueing at once could interleave those launches and corrupt each other's dQ.  One rank at a time therefore holds
    `baton` and enqueues GPU work; it lets go of the baton only while it blocks in a wait."""

    def __init__(self, timeout: float = 120.0):
        self.baton = threading.Condition()
        self.timeout = timeout
        self.msgs = {}
        self.sent, self.posted = collections.Counter(), collections.Counter()
        self.me = threading.local()
        self.failed = None

    def isend(self, tensor, dst, group=None):
        key = (self.me.rank, dst, self.sent[self.me.rank, dst])
        self.sent[self.me.rank, dst] += 1
        self.msgs[key] = tensor.clone()
        self.baton.notify_all()
        return types.SimpleNamespace(wait=lambda: None)

    def irecv(self, tensor, src, group=None):
        key = (src, self.me.rank, self.posted[src, self.me.rank])
        self.posted[src, self.me.rank] += 1

        def wait():
            if not self.baton.wait_for(lambda: key in self.msgs or self.failed is not None, self.timeout):
                raise TimeoutError(f"virtual rank {key[1]}: message {key[2]} from rank {key[0]} not sent within {self.timeout} s")
            if self.failed is not None:
                raise RuntimeError("another virtual rank failed") from self.failed
            tensor.copy_(self.msgs.pop(key))
        return types.SimpleNamespace(wait=wait)

    def patch(self, monkeypatch):
        monkeypatch.setattr(dist, "P2POp", lambda op, tensor, peer, group=None: (op, tensor, peer, group))
        monkeypatch.setattr(dist, "batch_isend_irecv", lambda ops_: [op(t, peer, g) for op, t, peer, g in ops_])
        monkeypatch.setattr(dist, "isend", self.isend)
        monkeypatch.setattr(dist, "irecv", self.irecv)

    def run(self, n: int, fn) -> list:
        """fn(rank) on n threads, each holding the baton outside its waits; their results in rank order."""
        out, errors = [None] * n, []

        def body(r):
            self.me.rank = r
            with self.baton:
                try:
                    out[r] = fn(r)
                except BaseException as e:   # noqa: BLE001 -- re-raised in the calling thread
                    errors.append(e)
                    self.failed = e
                    self.baton.notify_all()

        threads = [threading.Thread(target=body, args=(r,)) for r in range(n)]
        for t in threads:
            t.start()
        for t in threads:
            t.join(2 * self.timeout)
        assert not any(t.is_alive() for t in threads), "a virtual rank did not finish"
        if errors:
            raise errors[0]
        assert not self.msgs, f"messages never received: {sorted(self.msgs)}"
        return out


RING_CASES = [(n, zigzag, causal, D) for n in (2, 4) for zigzag, causal in ((False, True), (False, False), (True, True))
              for D in (64, 128)]


@pytest.mark.parametrize("n,zigzag,causal,D", RING_CASES,
                         ids=[f"n{n}-{'zigzag' if z else 'contiguous'}-{'causal' if c else 'full'}-D{d}" for n, z, c, d in RING_CASES])
def test_ring_attention_over_virtual_ranks_matches_fp64(n, zigzag, causal, D, monkeypatch):
    """Every rank's block of O, lse, dQ, dK and dV against full-sequence fp64 attention, and each rank's work in block products: 2 r + 1 for a contiguous causal ring, n on every rank for the zig-zag one."""
    from tepdist_b200.parallel.ring_attention import RingAttention
    ops = ar.kernels_only(monkeypatch)
    B, S, H = 1, 1024, 2
    L = S // n
    q, k, v, do = _inputs(B, S, H, D, "fused", seed=n + D)
    p2p = _VirtualP2P()
    p2p.patch(monkeypatch)
    rings = [RingAttention(None, list(range(n)), r, zigzag=zigzag) for r in range(n)]
    blk = lambda t, r: t[:, r * L:(r + 1) * L]
    n0 = ops.launch_count()
    fwd = p2p.run(n, lambda r: rings[r].forward(blk(q, r), blk(k, r), blk(v, r), causal))
    bwd = p2p.run(n, lambda r: [t.clone() for t in rings[r].backward(blk(do, r), blk(q, r), blk(k, r), blk(v, r), *fwd[r], causal)])
    torch.cuda.synchronize()
    assert ops.launch_count() > n0 + 4 * n
    if zigzag:   # the log-sum-exp stays in the zig-zag layout: rank r holds chunks r and 2n - 1 - r of 2n
        c = L // 2
        lse = torch.empty(B, H, S, device="cuda")
        for r in range(n):
            lse[:, :, r * c:(r + 1) * c] = fwd[r][1][:, :, :c]
            lse[:, :, (2 * n - 1 - r) * c:(2 * n - r) * c] = fwd[r][1][:, :, c:]
    else:
        lse = torch.cat([f[1] for f in fwd], 2)
    cat = lambda ts: torch.cat(ts, 1)
    ref = ar.reference(q, k, v, do, causal, blocks=2 * n if zigzag else n)   # zig-zag: up to 2n - 1 merges into a late row
    ref.check(o=cat([f[0] for f in fwd]), lse=lse, dq=cat([g[0] for g in bwd]), dk=cat([g[1] for g in bwd]),
              dv=cat([g[2] for g in bwd]))
    work = [ring.block_products for ring in rings]
    if not causal:
        assert work == [2.0 * n] * n
    elif zigzag:
        assert work == [float(n)] * n
    else:
        assert work == [2.0 * r + 1 for r in range(n)]
