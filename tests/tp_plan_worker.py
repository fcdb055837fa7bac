"""2+ GPU worker: tensor-parallel plan of GPT-2 executed (a) with NCCL collectives and (b) with the fused GEMM -> all-reduce
path (TEPDIST_TP_FUSED=1, parallel/symm.py GemmAllReduceMC) -- loss trajectories must agree with each other and with one GPU."""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    out = sys.argv[1]
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    from tepdist_b200.runtime import executor as ex_mod
    cfg = CONFIGS["tiny"]
    g = build_gpt2_graph(cfg, batch=4)       # 4 x 128 tokens: M = 512 = 2 ranks x 2 m-blocks
    torch.manual_seed(0)
    tok = torch.randint(0, cfg.n_vocab, (4, cfg.n_ctx), dtype=torch.int32)
    lab = torch.roll(tok, -1, 1)
    res = {}
    for tag, fused in (("nccl", False), ("fused", True)):
        ex_mod.TP_FUSED = fused
        tr = Trainer(g, strategy="tp", use_cuda_graph=False, comm_mode="fused")
        res[tag] = [tr.step({"tokens": tok, "labels": lab}) for _ in range(5)]
        res[tag + "_chains"] = len(getattr(tr.exec, "tp_fuse", {}) or {})
        res["parallelism"] = tr.plan_info.get("parallelism")
    if dist.get_rank() == 0:
        ref = ex_mod.Executor(g, torch.device("cuda", 0), seed=0)
        res["single"] = [float(ref.step({"tokens": tok.cuda(), "labels": lab.cuda()})[0]) for _ in range(5)]
        json.dump(res, open(out, "w"))
        print("TPPLAN", json.dumps(res))
    dist.barrier()
    torch.cuda.synchronize()
    os._exit(0)


if __name__ == "__main__":
    main()
