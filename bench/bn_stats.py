"""BatchNorm forward and backward at the shapes one Wide-ResNet training step runs them (model type 0, image 224, batch 4 by
default: the distinct [N, C, H, W] of the step's BatchNorm layers, with how many layers have each).

Per shape: the time of one `ops.batchnorm_fwd` and one `ops.batchnorm_bwd` call, from CUDA graphs of `--iters` calls each
(as the executor replays them, so host overhead is not in the number), CUDA-event mean over `--reps` replays after one
warm-up replay.  GB/s counts the bytes the algorithm has to move: forward reads x and writes y (4 bytes per element),
backward reads dy and x and writes dx (6 bytes per element).  The step total weighs each shape by its layer count.
`--lib` times another build of the kernel library (for example the parent commit's) in the same way, so two builds can be
compared from alternating runs.  The card name, power limit and max SM clock are read (read-only nvidia-smi query) in
the same run.

    python bench/bn_stats.py [--model-type 0] [--image 224] [--batch 4] [--iters 20] [--reps 10] [--lib PATH] [--json out.json]
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from attention_heads import _card  # noqa: E402


def step_shapes(model_type: int, image: int, batch: int):
    from tepdist_b200.models.wide_resnet import WideResNetConfig, build_wide_resnet_graph
    g = build_wide_resnet_graph(WideResNetConfig(model_type=model_type, batch=batch, image=image))
    return collections.Counter(tuple(g.type_of(n.inputs[0]).shape) for n in g.nodes if n.op == "batchnorm")


def graph_ms(fn, iters: int, reps: int) -> float:
    """Mean time of one fn() call, replayed from a CUDA graph of `iters` calls."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()                                                    # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(iters):
            fn()
    graph.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        graph.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / (reps * iters)


def run(shape, iters: int, reps: int) -> dict:
    from tepdist_b200 import ops
    N, C, H, W = shape
    torch.manual_seed(0)
    x = (torch.randn(N, H, W, C, device="cuda") * 2 + 0.5).to(torch.bfloat16).permute(0, 3, 1, 2)
    dy = torch.randn(N, H, W, C, device="cuda").to(torch.bfloat16).permute(0, 3, 1, 2)
    gamma, beta = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda")
    n0 = ops.launch_count()
    _, mean, rstd = ops.batchnorm_fwd(x, gamma, beta, 1e-5)
    assert ops.launch_count() > n0, "BatchNorm kernels did not run"
    fwd = lambda: ops.batchnorm_fwd(x, gamma, beta, 1e-5)  # noqa: E731
    bwd = lambda: ops.batchnorm_bwd(dy, x, gamma, mean, rstd)  # noqa: E731
    r = {"shape": [N, C, H, W], "fwd_ms": graph_ms(fwd, iters, reps), "bwd_ms": graph_ms(bwd, iters, reps)}
    el = N * C * H * W
    r["fwd_GBps"] = 4 * el / r["fwd_ms"] / 1e6
    r["bwd_GBps"] = 6 * el / r["bwd_ms"] / 1e6
    return r


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model-type", type=int, default=0)
    ap.add_argument("--image", type=int, default=224)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--lib", default=None, help="kernel library to time instead of the in-tree build")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from tepdist_b200 import ops
    if args.lib:
        ops._LIB_PATH = os.path.abspath(args.lib)
    ops.lib()
    shapes = step_shapes(args.model_type, args.image, args.batch)
    print(f"# {_card()}; library {ops._LIB_PATH}")
    print(f"{'N, C, H, W':>22} {'layers':>6} {'fwd ms':>8} {'GB/s':>6} {'bwd ms':>8} {'GB/s':>6}")
    rows, tot_f, tot_b = [], 0.0, 0.0
    for shape, count in sorted(shapes.items(), key=lambda kv: (kv[0][2], kv[0][1])):
        r = run(shape, args.iters, args.reps)
        r["layers"] = count
        rows.append(r)
        tot_f += count * r["fwd_ms"]
        tot_b += count * r["bwd_ms"]
        print(f"{str(tuple(shape)):>22} {count:>6} {r['fwd_ms']:>8.4f} {r['fwd_GBps']:>6.0f} {r['bwd_ms']:>8.4f} {r['bwd_GBps']:>6.0f}")
    print(f"step total (layers x ms): forward {tot_f:.3f} ms, backward {tot_b:.3f} ms")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": _card(), "lib": ops._LIB_PATH, "shapes": rows, "fwd_total_ms": tot_f, "bwd_total_ms": tot_b}, f,
                      indent=1)


if __name__ == "__main__":
    main()
