"""PyTorch client frontend: torch.fx -> planner IR.

The reference's client is patched TensorFlow that clusters the whole training step into one XLA computation
(SURVEY §2.F F1-F4).  Here an `nn.Module` is symbolically traced with torch.fx, shapes are propagated, every call is
mapped onto a planner-IR op, the loss is attached, and `build_training_step` appends backward + optimizer so the server
receives ONE graph per training step.  Module parameters become `parameter` nodes whose initial values are shipped as
init specs (random-init models) or loaded afterwards through `load_state_dict`.
"""
from __future__ import annotations

import math
import operator
from typing import Any, Dict, Optional

import torch
import torch.fx as fx
import torch.nn as nn
import torch.nn.functional as F
from torch.fx.passes.shape_prop import ShapeProp

from ..ir import Graph, Value
from .builder import GraphBuilder, build_training_step

_DT = {torch.float32: "f32", torch.bfloat16: "bf16", torch.float16: "f16", torch.int32: "i32", torch.int64: "i64", torch.bool: "bool"}


class TraceResult:
    def __init__(self, graph: Graph, param_names: Dict[str, str]):
        self.graph = graph
        self.param_names = param_names   # IR parameter name -> module state_dict key

    def load_state_dict_into(self, executor, state_dict: Dict[str, torch.Tensor]) -> None:
        """Copy a module's weights into a built executor's variable store (same values as the eager module)."""
        sd = {}
        for ir_name, key in self.param_names.items():
            sd[ir_name] = state_dict[key].detach().float()
        executor.store.load_state_dict(sd)


def optimizer_from_torch(opt: "torch.optim.Optimizer"):
    """(kind, hyper-parameters) of frontend.builder.apply_optimizer for a torch.optim instance, so that a user's unmodified
    optimizer object can be handed to `trace` (the reference's client likewise takes the user's TF optimizer as it is).
    Supported: SGD (with / without momentum, Nesterov), Adam (without the coupled L2 term), AdamW; one parameter group."""
    groups = opt.param_groups
    keys = [k for k in groups[0] if k != "params"]
    if any(any(g[k] != groups[0][k] for k in keys) for g in groups[1:]):
        raise NotImplementedError("parameter groups with different hyper-parameters; mark variables with decay=False in the graph instead")
    g = groups[0]
    for flag in ("amsgrad", "maximize", "capturable_unsupported"):
        if g.get(flag):
            raise NotImplementedError(f"{type(opt).__name__}({flag}=True)")
    if isinstance(opt, torch.optim.AdamW) or (isinstance(opt, torch.optim.Adam) and g.get("decoupled_weight_decay")):
        return "adamw", dict(lr=g["lr"], beta1=g["betas"][0], beta2=g["betas"][1], eps=g["eps"], weight_decay=g["weight_decay"])
    if isinstance(opt, torch.optim.Adam):
        if g["weight_decay"]:
            raise NotImplementedError("Adam(weight_decay != 0) adds an L2 term to the gradient; use AdamW (decoupled) instead")
        return "adam", dict(lr=g["lr"], beta1=g["betas"][0], beta2=g["betas"][1], eps=g["eps"])
    if isinstance(opt, torch.optim.SGD):
        if g["weight_decay"] or g["dampening"]:
            raise NotImplementedError("SGD(weight_decay / dampening != 0)")
        if g["momentum"]:
            return "momentum", dict(lr=g["lr"], momentum=g["momentum"], nesterov=bool(g["nesterov"]))
        return "sgd", dict(lr=g["lr"])
    raise NotImplementedError(f"{type(opt).__name__}: pass optimizer=<one of frontend.builder.OPTIMIZERS> and its hyper-parameters instead")


def trace(module: nn.Module, example_inputs: Dict[str, torch.Tensor], loss: str = "cross_entropy", label_name: str = "labels",
          label_example: Optional[torch.Tensor] = None, optimizer: Any = "adamw", compute_dtype: str = "f32", **hp) -> TraceResult:
    """`module(**example_inputs)` must return logits / predictions; `loss` in {"cross_entropy", "mse"}.  `optimizer`: a kind
    from frontend.builder.OPTIMIZERS with its hyper-parameters as keyword arguments, or a torch.optim instance."""
    decay_all = False
    if isinstance(optimizer, torch.optim.Optimizer):
        optimizer, from_opt = optimizer_from_torch(optimizer)
        hp = {**from_opt, **hp}
        decay_all = True      # torch applies a group's weight_decay to every parameter of the group, biases and norms included
    gm = fx.symbolic_trace(module)
    names = list(example_inputs)
    ShapeProp(gm).propagate(*[example_inputs[k] for k in names])
    b = GraphBuilder(type(module).__name__, compute_dtype=compute_dtype)
    env: Dict[str, Any] = {}
    pnames: Dict[str, str] = {}
    mods = dict(gm.named_modules())
    params = dict(gm.named_parameters())

    def dt(t: torch.dtype) -> str:
        d = _DT[t]
        return compute_dtype if d in ("f32", "bf16", "f16") else ("i32" if d == "i64" else d)

    def param(key: str, shape, kind="normal", std=0.02, value=0.0, transpose=False) -> Value:
        if key in env:
            return env[key]
        init = {"kind": "constant", "value": value} if kind == "constant" else {"kind": kind, "std": std}
        v = b.parameter(key.replace(".", "/"), tuple(shape), init)
        pnames[key.replace(".", "/")] = key
        env[key] = v
        return v

    def val(a):
        if isinstance(a, fx.Node):
            return env[a.name]
        return a

    for node in gm.graph.nodes:
        tm = node.meta.get("tensor_meta")
        if node.op == "placeholder":
            t = example_inputs[node.name]
            env[node.name] = b.input(node.name, tuple(t.shape), dt(t.dtype))
        elif node.op == "get_attr":
            p = params[node.target]
            env[node.name] = param(node.target, p.shape, std=float(p.std()) if p.numel() > 1 else 0.02)
        elif node.op == "call_module":
            m = mods[node.target]
            x = val(node.args[0])
            key = node.target
            if isinstance(m, nn.Linear):
                w = param(key + ".weight", m.weight.shape, std=1.0 / math.sqrt(m.in_features))
                bias = param(key + ".bias", m.bias.shape, "constant") if m.bias is not None else None
                env[node.name] = b.linear(x, w, bias, name=key.replace(".", "/"))
            elif isinstance(m, nn.LayerNorm):
                g = param(key + ".weight", m.weight.shape, "constant", value=1.0)
                be = param(key + ".bias", m.bias.shape, "constant")
                env[node.name] = b.layernorm(x, g, be, m.eps, name=key.replace(".", "/"))
            elif isinstance(m, nn.GELU):
                env[node.name] = b.gelu(x)
            elif isinstance(m, nn.ReLU):
                env[node.name] = b.relu(x)
            elif isinstance(m, nn.Tanh):
                env[node.name] = b.tanh(x)
            elif isinstance(m, nn.Embedding):
                w = param(key + ".weight", m.weight.shape, std=0.02)
                env[node.name] = b.gather_rows(w, x, name=key.replace(".", "/"))
            elif isinstance(m, nn.Conv2d):
                w = param(key + ".weight", m.weight.shape, std=math.sqrt(2.0 / (m.in_channels * m.kernel_size[0] * m.kernel_size[1])))
                y = b.conv2d(x, w, m.stride[0], m.padding[0], name=key.replace(".", "/"))
                if m.bias is not None:
                    bias = param(key + ".bias", m.bias.shape, "constant")
                    y = b.add(y, b.broadcast(bias, b.t(y).shape, [1]))
                env[node.name] = y
            elif isinstance(m, nn.BatchNorm2d):
                g = param(key + ".weight", m.weight.shape, "constant", value=1.0)
                be = param(key + ".bias", m.bias.shape, "constant")
                env[node.name] = b.batchnorm(x, g, be, m.eps, name=key.replace(".", "/"))
            elif isinstance(m, nn.MaxPool2d):
                k = m.kernel_size if isinstance(m.kernel_size, int) else m.kernel_size[0]
                s = m.stride if isinstance(m.stride, int) else m.stride[0]
                p = m.padding if isinstance(m.padding, int) else m.padding[0]
                env[node.name] = b.maxpool2d(x, k, s, p)
            elif isinstance(m, nn.AdaptiveAvgPool2d):
                env[node.name] = b.reshape(b.global_avgpool(x), tuple(tm.shape))
            elif isinstance(m, (nn.Dropout, nn.Identity)):
                env[node.name] = x       # (the reference's dropout is a no-op as well)
            elif isinstance(m, nn.Flatten):
                env[node.name] = b.reshape(x, tuple(tm.shape))
            else:
                raise NotImplementedError(f"module {type(m).__name__}")
        elif node.op in ("call_function", "call_method"):
            t = node.target
            a = [val(x) for x in node.args]
            if t in (operator.add, torch.add, "add"):
                env[node.name] = b.add(a[0], a[1]) if isinstance(a[1], Value) else b.add(a[0], b.constant(float(a[1])))
            elif t in (operator.sub, torch.sub):
                env[node.name] = b.sub(a[0], a[1])
            elif t in (operator.mul, torch.mul, "mul"):
                env[node.name] = b.mul(a[0], a[1]) if isinstance(a[1], Value) else b.scale(a[0], float(a[1]))
            elif t in (operator.truediv, torch.div):
                env[node.name] = b.div(a[0], a[1]) if isinstance(a[1], Value) else b.scale(a[0], 1.0 / float(a[1]))
            elif t in (torch.matmul, operator.matmul, "matmul"):
                env[node.name] = b.matmul(a[0], a[1])
            elif t in (F.relu, torch.relu, "relu"):
                env[node.name] = b.relu(a[0])
            elif t in (F.gelu,):
                env[node.name] = b.gelu(a[0])
            elif t in (torch.tanh, "tanh"):
                env[node.name] = b.tanh(a[0])
            elif t in (F.softmax, torch.softmax, "softmax"):
                dim = node.kwargs.get("dim", a[1] if len(a) > 1 else -1)
                env[node.name] = b.softmax(a[0], dim)
            elif t in ("view", "reshape", torch.reshape, torch.flatten, "flatten"):
                env[node.name] = b.reshape(a[0], tuple(tm.shape))
            elif t in ("transpose", torch.transpose):
                r = len(b.t(a[0]).shape)
                perm = list(range(r))
                d0, d1 = a[1] % r, a[2] % r
                perm[d0], perm[d1] = perm[d1], perm[d0]
                env[node.name] = b.transpose(a[0], perm)
            elif t in ("permute", torch.permute):
                perm = a[1] if isinstance(a[1], (list, tuple)) else a[1:]
                env[node.name] = b.transpose(a[0], list(perm))
            elif t in ("contiguous", "float", "to"):
                env[node.name] = a[0]
            elif t is F.scaled_dot_product_attention:
                # q, k, v: [B, H, S, D] -> the fused attention op (one wgmma flash-attention kernel on the GPU) on the
                # heads-major packed layout [B, S, H, 3, D]
                if node.kwargs.get("attn_mask") is not None or node.kwargs.get("dropout_p", 0.0):
                    raise NotImplementedError("scaled_dot_product_attention: attn_mask / dropout are not supported")
                q, k, v = a[0], a[1], a[2]
                B_, H_, S_, D_ = b.t(q).shape
                pk = [b.reshape(b.transpose(x_, [0, 2, 1, 3]), (B_, S_, H_, 1, D_)) for x_ in (q, k, v)]
                qkv = b.reshape(b.concat(pk, 3), (B_, S_, 3 * H_ * D_))
                o = b.attention(qkv, heads=H_, causal=bool(node.kwargs.get("is_causal", False)), name=node.name)
                env[node.name] = b.transpose(b.reshape(o, (B_, S_, H_, D_)), [0, 2, 1, 3])
            elif t in ("chunk", torch.chunk, "split", torch.split):
                src = a[0]
                shp = b.t(src).shape
                dim = node.kwargs.get("dim", a[2] if len(a) > 2 else (0 if t in ("split", torch.split) else 0))
                dim = dim % len(shp)
                if t in ("chunk", torch.chunk):
                    n_ = int(a[1])
                    sizes = [shp[dim] // n_] * n_
                else:
                    sz = a[1]
                    sizes = list(sz) if isinstance(sz, (list, tuple)) else [int(sz)] * (shp[dim] // int(sz))
                parts, off = [], 0
                for sz_ in sizes:
                    st_ = [0] * len(shp)
                    li_ = list(shp)
                    st_[dim], li_[dim] = off, off + sz_
                    parts.append(b.slice(src, st_, li_))
                    off += sz_
                env[node.name] = tuple(parts)
            elif t is operator.getitem:
                if isinstance(a[0], tuple):
                    env[node.name] = a[0][a[1]]
                else:
                    raise NotImplementedError("getitem on a tensor")
            elif t in ("size",):
                shp = b.t(a[0]).shape
                env[node.name] = shp if len(a) == 1 else shp[a[1]]
            else:
                raise NotImplementedError(f"function {t}")
        elif node.op == "output":
            out = val(node.args[0])
            if loss == "cross_entropy":
                lab = b.input(label_name, tuple(label_example.shape), "i32")
                loss_v = b.softmax_xent(out, lab, name="loss")
            elif loss == "mse":
                tgt = b.input(label_name, tuple(label_example.shape), compute_dtype)
                d = b.sub(out, tgt)
                loss_v = b.reduce_mean(b.mul(d, d), list(range(len(b.t(out).shape))), name="loss")
            else:
                raise ValueError(loss)
    if decay_all:
        for n in b.g.nodes:
            if n.op == "parameter":
                n.attrs["decay"] = True
    g = build_training_step(b, loss_v, optimizer, **hp)
    return TraceResult(g, pnames)
