"""2+ GPU worker: fused expert-parallel MoE forward (fp8 dispatch + wgmma fp8 FC) vs a dense fp32 reference."""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    out = sys.argv[1]
    from tepdist_b200.api import init_distributed
    from tepdist_b200.parallel.moe import FusedMoE, route_top_k
    ctx = init_distributed()
    rank, n = ctx["rank"], ctx["world"]
    dev = torch.device("cuda", ctx["local_rank"])
    M, H, E, C, T = 768, 3072, 8, 256, 1024        # gpt_moe: hidden 768, 8 experts, capacity 256 (ffn reduced for the test)
    torch.manual_seed(0)
    W1 = (torch.randn(E, H, M, device=dev) * 0.03).bfloat16()
    B1 = torch.randn(E, H, device=dev) * 0.01
    W2 = (torch.randn(E, M, H, device=dev) * 0.02).bfloat16()
    Wg = torch.randn(M, E, device=dev) * 0.1
    torch.manual_seed(100 + rank)
    x = torch.randn(T, M, device=dev).bfloat16()
    gates = torch.softmax(x.float() @ Wg, -1)
    route, gate = route_top_k(gates, C, 2)
    El = E // n
    moe = FusedMoE(M, H, E, C, W1[rank * El:(rank + 1) * El], B1[rank * El:(rank + 1) * El], W2[rank * El:(rank + 1) * El])
    y = moe.forward(x, route, gate)
    torch.cuda.synchronize()
    # dense reference for this rank's tokens (all experts are known to every rank in the test)
    ref = torch.zeros(T, M, device=dev)
    for k in range(2):
        e = (route[:, k] >> 16).long()
        ok = route[:, k] >= 0
        for ee in range(E):
            m = ok & (e == ee)
            if m.any():
                hcur = torch.nn.functional.gelu(x[m].float() @ W1[ee].float().t() + B1[ee], approximate="tanh")
                ref[m] += gate[m, k, None] * (hcur.bfloat16().float() @ W2[ee].float().t())
    err = float((y.float() - ref).norm() / ref.norm())
    res = {"relerr": err, "dropped": int((route < 0).sum()), "world": n}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        moe.forward(x, route, gate)
    dist.barrier(); torch.cuda.synchronize()
    e0.record()
    for _ in range(10):
        moe.forward(x, route, gate)
    e1.record(); torch.cuda.synchronize()
    res["fused_forward_ms"] = e0.elapsed_time(e1) / 10
    if rank == 0:
        json.dump(res, open(out, "w"))
        print("MOEFUSED", json.dumps(res))
    dist.barrier(); torch.cuda.synchronize()
    os._exit(0)


if __name__ == "__main__":
    main()
