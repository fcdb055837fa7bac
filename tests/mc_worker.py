"""2+ GPU worker: NVLS substrate (VMM allocation + multicast binding) and the multimem kernels of ops/csrc/vmm_sm90.cu
against plain references, plus timing against NCCL.  Writes a JSON report; prints one line per stage so a failure is
attributable from the log alone."""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def ev_ms(fn, iters=20, warm=5, graph=True):
    """Device time per call, max over ranks.  The calls are replayed from a CUDA graph (20 per replay) so the number
    is the kernels' time, not the Python launch path's."""
    for _ in range(warm):
        fn()
    dist.barrier(); torch.cuda.synchronize()
    g = None
    if graph:
        try:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=s):
                    for _ in range(iters):
                        fn()
            torch.cuda.current_stream().wait_stream(s)
            g.replay()
        except Exception as e:  # noqa: BLE001
            print("graph capture failed, timing eager:", type(e).__name__, e, flush=True)
            g = None
    dist.barrier(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 3 if g is not None else 1
    e0.record()
    for _ in range(reps):
        if g is not None:
            g.replay()
        else:
            for _ in range(iters):
                fn()
    e1.record()
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / (iters * reps)], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


def say(*a):
    print(f"[r{dist.get_rank()}]", *a, flush=True)


def main():
    out = sys.argv[1]
    from tepdist_b200 import ops
    from tepdist_b200.api import init_distributed
    from tepdist_b200.parallel import symm
    ctx = init_distributed()
    rank, n = ctx["rank"], ctx["world"]
    dev = torch.device("cuda", ctx["local_rank"])
    res = {"world": n}
    res["backend"] = symm.symm_backend()
    say("backend", res["backend"])
    if res["backend"] != "vmm":
        if rank == 0:
            json.dump(res, open(out, "w"))
        return
    mc = symm.McContext()
    say("context up: granularity-rounded flag buffer", mc.flags.nbytes)
    for _ in range(3):
        mc.barrier()
    torch.cuda.synchronize()
    mc.check()
    res["barrier_ok"] = True

    # ---- unicast peer mapping through the VMM handles: write own rank id, read every rank's through its mapping.  The
    # views are put on THIS device explicitly: a pointer query would name the GPU the peer's pages live on.
    probe = symm.SymmetricBuffer(4096)
    probe.tensor(torch.float32)[:1024] = float(rank + 1)
    torch.cuda.synchronize(); dist.barrier()
    acc = torch.zeros(1024, device=dev)
    for r in range(n):
        pages = torch._C._construct_storage_from_data_pointer(probe.ptrs[r], dev, probe.nbytes)
        acc += torch.empty(0, dtype=torch.float32, device=dev).set_(pages, 0, (1024,))
    torch.cuda.synchronize()
    res["peer_read_ok"] = bool((acc == n * (n + 1) / 2).all().item())
    say("peer read", res["peer_read_ok"])

    # ---- all-reduce numerics (+ bias + residual epilogue)
    torch.manual_seed(1234 + rank)
    M, N = 4096, 1024
    buf = symm.SymmetricBuffer(M * N * 2)
    x = (torch.randn(M, N, device=dev) * 0.5).to(torch.bfloat16)
    torch.manual_seed(99)
    bias = torch.randn(N, device=dev)                             # replicated
    resid = torch.randn(M, N, device=dev).to(torch.bfloat16)      # replicated
    ref = x.float().clone()
    dist.all_reduce(ref)
    view = buf.tensor(torch.bfloat16, M * N).view(M, N)
    view.copy_(x)
    mc.all_reduce_bf16_(buf, M * N, N)
    torch.cuda.synchronize(); mc.check()
    res["ar_relerr"] = float((view.float() - ref).norm() / ref.norm())
    view.copy_(x)
    mc.all_reduce_bf16_(buf, M * N, N, bias=bias, residual=resid)
    torch.cuda.synchronize(); mc.check()
    ref2 = ref + bias + resid.float()
    res["ar_epi_relerr"] = float((view.float() - ref2).norm() / ref2.norm())
    say("all-reduce relerr", res["ar_relerr"], res["ar_epi_relerr"])

    # ---- timing vs NCCL: 8 MB (TP activations of the 345M model at batch 4) and 64 MB
    for mb in (8, 64):
        numel = mb * 1024 * 1024 // 2
        b2 = symm.SymmetricBuffer(numel * 2)
        t = torch.randn(numel, device=dev).to(torch.bfloat16)
        for ctas in (16, 32, 64, 128):
            res[f"ar_{mb}MB_mc_ctas{ctas}_us"] = 1e3 * ev_ms(lambda: mc.all_reduce_bf16_(b2, numel, 1024, ctas=ctas))
        res[f"ar_{mb}MB_nccl_us"] = 1e3 * ev_ms(lambda: dist.all_reduce(t))
        torch.cuda.synchronize(); mc.check()
        say(mb, "MB:", {k: round(v, 1) for k, v in res.items() if k.startswith(f"ar_{mb}MB")})

    # ---- optimizer step over NVLS: reduce-scatter (fp32 and bf16 wire) + AdamW + bf16 all-gather
    lib = ops.lib()
    P = 8 * 1024 * 1024
    hyper = torch.tensor([1e-3, 1 - 0.9, 1 - 0.999, 1.0 / n, 0, 0, 0, 0], device=dev, dtype=torch.float32)
    torch.manual_seed(7)
    master0 = torch.randn(P, device=dev)
    for wire in ("f32", "bf16"):
        torch.manual_seed(100 + rank)
        g = torch.randn(P, device=dev)
        gbuf = symm.SymmetricBuffer(P * (4 if wire == "f32" else 2))
        pbuf = symm.SymmetricBuffer(P * 2)
        if wire == "f32":
            gbuf.tensor(torch.float32, P).copy_(g)
            gsum = g.clone()
        else:
            gb = g.to(torch.bfloat16)
            gbuf.tensor(torch.bfloat16, P).copy_(gb)
            gsum = gb.float()
        dist.all_reduce(gsum)
        master = master0.clone(); m = torch.zeros(P, device=dev); v = torch.zeros(P, device=dev)
        per = P // n
        b, e = rank * per, (rank + 1) * per
        mc.barrier()
        rc = lib.tepd_mc_rs_adamw_ag(gbuf.mc_ptr, pbuf.mc_ptr, master.data_ptr(), m.data_ptr(), v.data_ptr(), b, e, P, 0.9, 0.999,
                                     1e-8, 0.01, hyper.data_ptr(), int(wire == "bf16"), 0, torch.cuda.current_stream().cuda_stream)
        assert rc == 0, rc
        mc.barrier()
        torch.cuda.synchronize(); mc.check()
        # reference: plain AdamW on the whole vector with the all-reduced gradient
        gg = gsum / n
        mr = 0.1 * gg; vr = 0.001 * gg * gg
        pr = master0 - 1e-3 * ((mr / 0.1) / ((vr / 0.001).sqrt() + 1e-8) + 0.01 * master0)
        got = pbuf.tensor(torch.bfloat16, P).float()
        res[f"opt_{wire}_relerr"] = float((got - pr).norm() / pr.norm())
        res[f"opt_{wire}_master_relerr"] = float((master[b:e] - pr[b:e]).norm() / pr[b:e].norm())
        say("optimizer", wire, res[f"opt_{wire}_relerr"], res[f"opt_{wire}_master_relerr"])

        def step():
            mc.barrier()
            lib.tepd_mc_rs_adamw_ag(gbuf.mc_ptr, pbuf.mc_ptr, master.data_ptr(), m.data_ptr(), v.data_ptr(), b, e, P, 0.9, 0.999, 1e-8,
                                    0.01, hyper.data_ptr(), int(wire == "bf16"), 0, torch.cuda.current_stream().cuda_stream)
            mc.barrier()
        res[f"opt_{wire}_us_8M"] = 1e3 * ev_ms(step)
    # the round-1 unicast kernel on the same problem
    gi = symm.SymmetricBuffer(P * 4, backend="ipc"); pi = symm.SymmetricBuffer(P * 2, backend="ipc")
    fo = symm.FusedShardedOptimizer(gi, pi)
    master = master0.clone(); m = torch.zeros(P, device=dev); v = torch.zeros(P, device=dev)
    per = P // n

    def step_ipc():
        fo.barrier()
        fo.step(master, m, v, rank * per, (rank + 1) * per, P, hyper, 0.9, 0.999, 1e-8, 0.01)
        fo.barrier()
    res["opt_unicast_us_8M"] = 1e3 * ev_ms(step_ipc)
    say("optimizer timing", {k: round(v, 1) for k, v in res.items() if k.endswith("us_8M")})
    if rank == 0:
        json.dump(res, open(out, "w"), indent=1)
        print(json.dumps(res))
    dist.barrier()
    torch.cuda.synchronize()
    os._exit(0)


if __name__ == "__main__":
    main()
