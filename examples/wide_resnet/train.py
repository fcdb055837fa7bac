#!/usr/bin/env python
"""Wide-ResNet with fake ImageNet input (reference examples/wide_resnet/resnet_train.py: prints examples/sec, sec/batch)."""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tepdist_b200.api import Trainer  # noqa: E402
from tepdist_b200.models.wide_resnet import WideResNetConfig, build_wide_resnet_graph  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model-type", type=int, default=1)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--image", type=int, default=224)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--strategy", default="auto")
    ap.add_argument("--optimizer", default="adamw", choices=["adamw", "adam", "momentum", "sgd"],
                    help="reference: AdamOptimizer(0.1) in train_imagenet.py, MomentumOptimizer(0.01, 0.9) in resnet_train.py")
    ap.add_argument("--lr", type=float, default=None)
    ap.add_argument("--no-graph", action="store_true", help="run the step eagerly (default: whole step replayed from a CUDA graph)")
    ap.add_argument("--graph", action="store_true", help="(default; kept for compatibility)")
    a = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    cfg = WideResNetConfig(model_type=a.model_type, batch=a.batch * world, image=a.image)
    if a.lr is not None:
        cfg.lr = a.lr
    elif a.optimizer in ("momentum", "sgd"):
        cfg.lr = 0.01
    tr = Trainer(build_wide_resnet_graph(cfg, optimizer=a.optimizer), strategy=a.strategy, use_cuda_graph=not a.no_graph)
    dt = torch.bfloat16 if tr.device.type == "cuda" else torch.float32
    feeds = {"images": torch.full((cfg.batch, 3, a.image, a.image), 0.5, dtype=dt), "labels": torch.ones(cfg.batch, dtype=torch.int32)}
    last = time.time()
    for i in range(a.steps):
        loss = tr.step(feeds)
        if tr.rank == 0 and (i + 1) % 5 == 0:
            d = (time.time() - last) / 5
            last = time.time()
            print(f"step {i + 1}, loss = {loss:.3f} ({cfg.batch / d:.1f} examples/sec; {d:.3f} sec/batch)")
    os._exit(0)


if __name__ == "__main__":
    main()
