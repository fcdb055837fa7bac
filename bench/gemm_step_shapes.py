"""Time the GEMM calls of one GPT-2 345M training step (4 x 1024 = 4096 tokens) with the epilogues the executor gives them,
next to torch.matmul (cuBLAS) on the same operands.

Each row is one distinct call of the step: its shape, its epilogue and its schedule (the weight gradients are run the way
`Executor` runs them: plain fp32 stores when `ops.wgrad_prefers_store` says so, otherwise red.add into a zeroed slot with the
split-K / stream-K choice of `ops.gemm`).  `calls` is how often the step makes that call, so the sum of calls x ms is the
step's GEMM time as these kernels run it in isolation.  As in the step, the calls are replayed from a CUDA graph (ten
calls per graph), so the host-side launch cost is not in the time; the zero-fill of a red.add slot is not timed either
(the step zero-fills all such slots at once).  Times are CUDA-event means over enough replays to span `--window` ms
after warm-up.  The card name, power limit and max SM clock are read in the same run.

    python bench/gemm_step_shapes.py [--window 200] [--json out.json] [--compare DIR] [--wgrad-breakdown]

--compare DIR: the first run writes every GEMM output to DIR; a later run (another build) compares its outputs with those
element by element and prints how many elements differ and by how much.

--wgrad-breakdown: instead of the step table, time each weight-gradient shape four ways, plain stores without split-K,
to tell the cost of the fp32 output from the cost of the MN-major A operand: A MN-major as the step runs it (dy [T, n_out])
or K-major (dy^T made contiguous before timing), each with an fp32 output and with a bf16 output.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


def _card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name()


def _time_ms(fn, window_ms: float, warmup: int = 5, per_graph: int = 10) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(per_graph):
            fn()
    fn = graph.replay
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(3):
        fn()
    b.record()
    torch.cuda.synchronize()
    iters = max(10, int(window_ms / max(1e-3, a.elapsed_time(b) / 3)))
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters / per_graph


def cases(T: int = 4096, C: int = 1024, Vp: int = 50304, L: int = 24):
    """(name, calls per step, M, N, K, builder); builder(gen) -> (ours, torch_ref, out) closures over seeded operands."""
    from tepdist_b200 import ops
    dev = "cuda"

    def rnd(gen, *shape, scale=1.0):
        return (torch.randn(*shape, generator=gen, device=dev) * scale).to(torch.bfloat16)

    def fwd(N, K, bias=True, residual=False, gelu=False):
        def build(gen):
            x, w = rnd(gen, T, K), rnd(gen, N, K, scale=0.03)
            b = rnd(gen, N) if bias else None
            res = rnd(gen, T, N) if residual else None
            out = torch.empty(T, N, dtype=torch.bfloat16, device=dev)
            out2 = torch.empty_like(out) if gelu else None

            def ours():
                ops.gemm(x, w, bias=b, residual=res, act="gelu" if gelu else None, out=out, out2=out2)
            return ours, lambda: torch.matmul(x, w.t()), (out, out2) if gelu else (out,)
        return build

    def dgrad(N, K, gelu_bwd=False):   # dx [T, N] = dy [T, K] @ W [K, N]
        def build(gen):
            dy, w = rnd(gen, T, K), rnd(gen, K, N, scale=0.03)
            aux = rnd(gen, T, N) if gelu_bwd else None
            out = torch.empty(T, N, dtype=torch.bfloat16, device=dev)

            def ours():
                ops.gemm(dy, w, b_mn=True, out=out, act="gelu_bwd" if gelu_bwd else None, aux=aux)
            return ours, lambda: torch.matmul(dy, w), (out,)
        return build

    def wgrad(n_out, k_in):   # dW [n_out, k_in] = dy^T [n_out, T] @ x [T, k_in], as Executor._exec("linear_wgrad")
        store = ops.wgrad_prefers_store(n_out, k_in)

        def build(gen):
            dy, x = rnd(gen, T, n_out), rnd(gen, T, k_in)
            out = torch.zeros(n_out, k_in, dtype=torch.float32, device=dev)

            def ours():
                ops.gemm(dy, x, a_mn=True, b_mn=True, out=out, accumulate=not store, split_k=1 if store else 0)
            return ours, lambda: torch.matmul(dy.t(), x), (out,)
        return build, "store" if store else "red.add"

    rows = [
        ("qkv fwd", L, T, 3 * C, C, "bias", fwd(3 * C, C)),
        ("attn/c_proj fwd", L, T, C, C, "bias+residual", fwd(C, C, residual=True)),
        ("mlp/c_fc fwd", L, T, 4 * C, C, "bias+gelu dual", fwd(4 * C, C, gelu=True)),
        ("mlp/c_proj fwd", L, T, C, 4 * C, "bias+residual", fwd(C, 4 * C, residual=True)),
        ("lm_head fwd", 1, T, Vp, C, "none", fwd(Vp, C, bias=False)),
        ("qkv dgrad", L, T, C, 3 * C, "none", dgrad(C, 3 * C)),
        ("attn/c_proj dgrad", L, T, C, C, "none", dgrad(C, C)),
        ("mlp/c_fc dgrad", L, T, C, 4 * C, "none", dgrad(C, 4 * C)),
        ("mlp/c_proj dgrad", L, T, 4 * C, C, "gelu'", dgrad(4 * C, C, gelu_bwd=True)),
        ("lm_head dgrad", 1, T, C, Vp, "none", dgrad(C, Vp)),
    ]
    for name, n_out, k_in in (("qkv", 3 * C, C), ("attn/c_proj", C, C), ("mlp/c_fc", 4 * C, C), ("mlp/c_proj", C, 4 * C),
                              ("lm_head", Vp, C)):
        b, kind = wgrad(n_out, k_in)
        rows.append((f"{name} wgrad", 1 if name == "lm_head" else L, n_out, k_in, T, f"fp32 {kind}", b))
    return rows


def wgrad_breakdown(window_ms: float, T: int = 4096, C: int = 1024, Vp: int = 50304) -> list:
    """Weight-gradient shapes dW [n_out, k_in] = dy^T @ x, plain stores, four variants: (a) A MN-major, fp32 out (the
    step's call when it stores); (b) A MN-major, bf16 out; (c) A K-major, fp32 out; (d) A K-major, bf16 out (the
    data-gradient layout)."""
    from tepdist_b200 import ops
    print(f"{'wgrad':12s} {'M':>5} {'N':>5} {'K':>5} | {'(a) MN f32':>10} {'(b) MN bf16':>11} {'(c) K f32':>10} "
          f"{'(d) K bf16':>10}  (ms per call)")
    rows = []
    for i, (name, n_out, k_in) in enumerate((("qkv", 3 * C, C), ("attn/c_proj", C, C), ("mlp/c_fc", 4 * C, C),
                                             ("mlp/c_proj", C, 4 * C), ("lm_head", Vp, C))):
        gen = torch.Generator(device="cuda")
        gen.manual_seed(4321 + i)
        dy = torch.randn(T, n_out, generator=gen, device="cuda").to(torch.bfloat16)
        x = torch.randn(T, k_in, generator=gen, device="cuda").to(torch.bfloat16)
        dyt = dy.t().contiguous()
        r = {"wgrad": name, "M": n_out, "N": k_in, "K": T}
        for key, a, a_mn, dt in (("a_mn_f32", dy, True, torch.float32), ("a_mn_bf16", dy, True, torch.bfloat16),
                                 ("a_k_f32", dyt, False, torch.float32), ("a_k_bf16", dyt, False, torch.bfloat16)):
            out = torch.empty(n_out, k_in, dtype=dt, device="cuda")

            def ours(a=a, a_mn=a_mn, out=out):
                ops.gemm(a, x, a_mn=a_mn, b_mn=True, out=out, split_k=1)
            n0 = ops.launch_count()
            ours()
            assert ops.launch_count() > n0, f"{name}: our GEMM kernel did not run"
            r[key] = _time_ms(ours, window_ms)
            del out
        print(f"{name:12s} {n_out:5d} {k_in:5d} {T:5d} | {r['a_mn_f32']:10.3f} {r['a_mn_bf16']:11.3f} {r['a_k_f32']:10.3f} "
              f"{r['a_k_bf16']:10.3f}", flush=True)
        rows.append(r)
        del dy, x, dyt
        torch.cuda.empty_cache()
    return rows


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--window", type=float, default=200.0, help="ms of back-to-back calls per measurement")
    ap.add_argument("--json", default=None)
    ap.add_argument("--compare", metavar="DIR", default=None)
    ap.add_argument("--wgrad-breakdown", action="store_true", help="time the weight-gradient shapes four ways (see above)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gemm_step_shapes.py: no CUDA GPU; the timings are only meaningful on the H100")
    from tepdist_b200 import ops
    ops.lib()
    card = _card()
    print(f"# card: {card}  (name, power limit, max SM clock)")
    if a.wgrad_breakdown:
        rows = wgrad_breakdown(a.window)
        if a.json:
            with open(a.json, "w") as fh:
                json.dump({"card": card, "wgrad_breakdown": rows}, fh, indent=1)
        return
    print(f"{'gemm':18s} {'M':>5} {'N':>6} {'K':>6} {'epilogue':15s} {'calls':>5} | {'ours ms':>8} {'TFLOP/s':>7} | "
          f"{'cuBLAS ms':>9} {'TFLOP/s':>7} | {'calls x ours':>12} {'calls x cuBLAS':>14}")
    rows, tot, tot_ref = [], 0.0, 0.0
    if a.compare:
        os.makedirs(a.compare, exist_ok=True)
    for i, (name, calls, M, N, K, epi, build) in enumerate(cases()):
        gen = torch.Generator(device="cuda")
        gen.manual_seed(1234 + i)
        ours, ref, outs = build(gen)
        n0 = ops.launch_count()
        ours()
        assert ops.launch_count() > n0, f"{name}: our GEMM kernel did not run"
        ms = _time_ms(ours, a.window)
        ms_ref = _time_ms(ref, a.window)
        fl = 2.0 * M * N * K
        r = {"gemm": name, "M": M, "N": N, "K": K, "epilogue": epi, "calls": calls, "ms": ms, "tflops": fl / ms / 1e9,
             "cublas_ms": ms_ref, "cublas_tflops": fl / ms_ref / 1e9}
        tot += calls * ms
        tot_ref += calls * ms_ref
        print(f"{name:18s} {M:5d} {N:6d} {K:6d} {epi:15s} {calls:5d} | {ms:8.3f} {r['tflops']:7.1f} | {ms_ref:9.3f} "
              f"{r['cublas_tflops']:7.1f} | {calls * ms:12.2f} {calls * ms_ref:14.2f}", flush=True)
        if a.compare:
            outs[0].zero_()   # one call into a zeroed output (the red.add rows accumulated over the timing)
            ours()
            torch.cuda.synchronize()
            for j, o in enumerate(outs):
                path = os.path.join(a.compare, f"{i:02d}_{j}.pt")
                if os.path.exists(path):
                    prev = torch.load(path, map_location="cuda")
                    diff = (o.float() - prev.float()).abs()
                    r[f"diff_elems_{j}"] = int((o.view(torch.int16 if o.dtype == torch.bfloat16 else torch.int32)
                                                != prev.view(torch.int16 if prev.dtype == torch.bfloat16 else torch.int32))
                                               .sum())
                    r[f"max_abs_diff_{j}"] = float(diff.max())
                    print(f"    output {j}: {r[f'diff_elems_{j}']} of {o.numel()} elements differ from {path}, "
                          f"max |diff| {r[f'max_abs_diff_{j}']:.3g}", flush=True)
                else:
                    torch.save(o.cpu(), path)
        rows.append(r)
        del ours, ref, outs
        torch.cuda.empty_cache()
    print(f"{'step GEMM total':18s} {'':36s} | {'':8s} {'':7s} | {'':9s} {'':7s} | {tot:12.2f} {tot_ref:14.2f}")
    if a.json:
        with open(a.json, "w") as fh:
            json.dump({"card": card, "rows": rows, "step_gemm_ms": tot, "step_cublas_ms": tot_ref}, fh, indent=1)


if __name__ == "__main__":
    main()
