#!/usr/bin/env python
"""Optimizer phase of a training step: the multi-tensor kernels (ops.optim_step, optim_sm90.cu) against the torch path
(runtime/optimizers.py STEP per variable plus the bf16 copy-back, what Executor._apply_one runs), on the same tensors.

Variable sets: GPT-2 345M (24 layers, 406 M elements) and GPT-MoE at the reference widths (8 layers, 8 experts of
768 x 6144).  Each path is captured once in a CUDA graph; the graphs are replayed alternately and timed with CUDA events.
The bytes each kernel update must move per element are counted from the kernels' passes (`kernel_bytes`, not measured);
bytes / 3.35 TB/s (H100 SXM HBM3) is the floor the achieved time is compared with.

`--e2e`: steady-state step time of the training loop of examples/gpt2/train.py (345M, batch 4, one GPU) per optimizer.
Writes JSON to --out (default: a temporary directory) and prints it."""
import argparse
import json
import math
import os
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tepdist_b200 import ops  # noqa: E402
from tepdist_b200.runtime.optimizers import STEP, Shards, host_hyper  # noqa: E402

HBM = 3.35e12
KINDS = {"apply_momentum": dict(lr=1e-3, momentum=0.9), "apply_lamb": dict(lr=1e-3, weight_decay=0.01),
         "apply_adafactor": dict(lr=1e-3), "apply_sm3": dict(lr=1e-3)}


def variable_sets():
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    from tepdist_b200.models.gpt_moe import MoEConfig, build_gpt_moe_graph
    out = {}
    for name, g in (("gpt2-345M", build_gpt2_graph(CONFIGS["345M"])), ("gpt-moe", build_gpt_moe_graph(MoEConfig()))):
        out[name] = [(tuple(n.outputs[0].shape), bool(n.attrs.get("decay", True))) for n in g.params()]
    return out


def kernel_bytes(op, opt, shape):
    """HBM bytes per step of one variable on the kernel path (fp32 = 4 B, bf16 copy = 2 B; reduced slots and partials
    are a few floats per row / column and are left out)."""
    n = math.prod(shape)
    if op == "apply_momentum":          # read g, p, mom; write p, mom, bf16
        return 22 * n
    if op == "apply_lamb":              # pass 1: read g, m, v, p, write m, v; pass 2: read m, v, p, write p, bf16
        return 42 * n
    if op == "apply_adafactor":
        if len(shape) >= 2 and opt.get("factored", True):   # g, p | g | g, p, write p, bf16
            return 26 * n
        return 34 * n                   # g, vf, write vf, p | g, vf, p, write p, bf16
    mom = 8 if opt.get("momentum", 0.0) > 0 else 0
    if len(shape) >= 2:                 # SM3: read g, p, write p, bf16 (+ momentum read / write)
        return (14 + mom) * n
    return (22 + mom) * n               # + the accumulator read / write


class Phase:
    def __init__(self, op, opt, shapes):
        self.op, self.opt = op, opt
        self.shapes = [s for s, _ in shapes]
        self.decays = [d for _, d in shapes]
        self.offs, off = [], 0
        for s in self.shapes:
            self.offs.append(off)
            off += -(-math.prod(s) // 128) * 128
        self.n = sum(math.prod(s) for s in self.shapes)
        self.master = torch.randn(off, device="cuda") * 0.02
        self.grad = torch.randn(off, device="cuda") * 1e-3
        self.compute = self.master.to(torch.bfloat16)
        self.slots = [[torch.zeros(ss, device="cuda") for ss in ops.optim_slot_shapes(op, s, opt)] for s in self.shapes]
        self.plan = ops.OptimPlan(op, opt, list(zip(self.offs, self.shapes, self.slots, self.decays)), torch.device("cuda"))
        self.hyper = torch.tensor(host_hyper(opt, 10, opt.get("lr") or 0.0), dtype=torch.float32, device="cuda")

    def view(self, buf, i):
        return buf[self.offs[i]:self.offs[i] + math.prod(self.shapes[i])].view(self.shapes[i])

    def kernel(self):
        ops.optim_step(self.plan, self.master, self.grad, self.compute, self.hyper)

    def torch_path(self):
        for i, s in enumerate(self.shapes):
            p = self.view(self.master, i)
            STEP[self.op](p, self.view(self.grad, i).float().contiguous(), self.slots[i], self.opt, self.hyper, Shards(),
                          decay=self.decays[i])
            self.view(self.compute, i).copy_(p.to(torch.bfloat16))

    def bytes(self):
        return sum(kernel_bytes(self.op, self.opt, s) for s in self.shapes)


def capture(fn):
    fn()                                # warm-up: allocations, module loads
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side), torch.cuda.graph(g):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    return g


def time_alternating(graphs, rounds, reps):
    ms = {k: [] for k in graphs}
    for _ in range(rounds):
        for k, g in graphs.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                g.replay()
            b.record()
            torch.cuda.synchronize()
            ms[k].append(a.elapsed_time(b) / reps)
    return {k: sorted(v)[len(v) // 2] for k, v in ms.items()}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (x.strip() for x in q.split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:       # (the numbers are still the device's; the card description is then missing)
        return {"gpu": torch.cuda.get_device_name(), "card_query_error": str(e)}


def e2e(optimizers, steps, warmup):
    from tepdist_b200.api import Trainer
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    cfg = CONFIGS["345M"]
    out = {}
    for opt in optimizers:
        g = build_gpt2_graph(cfg, batch=4, optimizer=opt)
        tr = Trainer(g, strategy="auto", comm_mode="fused")
        gen = torch.Generator().manual_seed(0)
        tok = torch.randint(0, cfg.n_vocab, (4, cfg.n_ctx), generator=gen, dtype=torch.int32)
        feeds = {"tokens": tok, "labels": torch.roll(tok, -1, 1)}
        for _ in range(warmup):
            tr.step(feeds)
        t0 = time.perf_counter()
        for _ in range(steps):
            loss = tr.step(feeds)        # returns the loss as a Python float: the step has finished
        dt = (time.perf_counter() - t0) / steps
        out[opt] = {"ms_per_step": 1e3 * dt, "loss": loss, "path": "kernels" if getattr(tr.exec, "optim_plan", None) else "flat"}
        print(f"e2e {opt}: {1e3 * dt:.1f} ms/step", flush=True)
        del tr
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sets", default="gpt2-345M,gpt-moe")
    ap.add_argument("--kinds", default=",".join(KINDS))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--e2e", action="store_true")
    ap.add_argument("--e2e-steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this benchmark measures the device")
    ops.lib()
    res = {"card": card(), "hbm_bytes_per_s": HBM, "sets": {}}
    sets = variable_sets()
    for sname in a.sets.split(","):
        for op in a.kinds.split(","):
            ph = Phase(op, KINDS[op], sets[sname])
            graphs = {"kernel": capture(ph.kernel), "torch": capture(ph.torch_path)}
            t = time_alternating(graphs, a.rounds, a.reps)
            floor_ms = 1e3 * ph.bytes() / HBM
            r = {"elements": ph.n, "variables": len(ph.shapes), "kernel_launches": ops.OPTIM_LAUNCHES[op],
                 "kernel_ms": t["kernel"], "torch_ms": t["torch"], "bytes_per_element": ph.bytes() / ph.n,
                 "hbm_floor_ms": floor_ms, "share_of_floor": floor_ms / t["kernel"]}
            res["sets"].setdefault(sname, {})[op] = r
            print(f"{sname} {op}: kernel {t['kernel']:.2f} ms, torch {t['torch']:.2f} ms, {r['bytes_per_element']:.1f} B/elem, "
                  f"floor {floor_ms:.2f} ms ({100 * r['share_of_floor']:.0f}% of it reached)", flush=True)
            del graphs, ph
            torch.cuda.empty_cache()
    if a.e2e:
        res["e2e_gpt2_345M"] = e2e(["adamw", "adafactor", "lamb", "sm3"], a.e2e_steps, 3)
    res["card_after"] = card()
    out = a.out or os.path.join(tempfile.mkdtemp(), "optimizer_step.json")
    with open(out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
