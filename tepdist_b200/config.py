"""Flag system wiring: ServiceEnv (C++, csrc/service_env.{h,cc}) -> planner / runtime options.

Reference parity (SURVEY 2.E E1, 5.6): `ServiceEnv` loads defaults -> JSON file (`CONFIG_FILE`, default config.json) ->
environment variables, and every planner/runtime component reads its knobs from it (service_env.h:46-74).  Only keys the
user actually set (in the environment or the JSON file) override what the Python API was called with, so library callers
and tests keep their explicit arguments.
"""
from __future__ import annotations

import json
import os
from typing import Any, Dict, Optional, Set

_ENV = None
_EXPLICIT: Set[str] = set()


def env(reload: bool = False):
    """The process-wide ServiceEnv, loaded once (reload=True re-reads file + environment, used by tests)."""
    global _ENV, _EXPLICIT
    from . import _C
    if _ENV is None or reload:
        e = _C.ServiceEnv.instance()
        cfg = os.environ.get("CONFIG_FILE", "config.json")
        e.load(cfg)
        keys = set(e.keys())
        explicit = {k for k in keys if k in os.environ}
        try:
            with open(cfg) as f:
                explicit |= {k for k in json.load(f) if k in keys}
        except (OSError, ValueError):
            pass
        _ENV, _EXPLICIT = e, explicit
    return _ENV


def is_set(key: str) -> bool:
    env()
    return key in _EXPLICIT


def _take(out: Dict[str, Any], field: str, key: str, kind: str, scale: float = 1.0) -> None:
    if not is_set(key):
        return
    e = env()
    if kind == "bool":
        out[field] = e.get_bool(key)
    elif kind == "int":
        out[field] = int(e.get_int(key))
    else:
        out[field] = e.get_double(key) * scale


def spmd_overrides() -> Dict[str, Any]:
    """SpmdOptions fields set by the user (VAR_MEM_LIMIT, COST_FACTOR, OPT_LEVEL, IGNORE_ANNOTATION, AUX_AFFINITY,
    FORWARD_SUB_GRAPH_NUM, ILP_TIME_LIMIT [minutes])."""
    o: Dict[str, Any] = {}
    _take(o, "var_mem_limit", "VAR_MEM_LIMIT", "float")
    _take(o, "cost_factor", "COST_FACTOR", "float")
    _take(o, "opt_level", "OPT_LEVEL", "int")
    _take(o, "ignore_annotation", "IGNORE_ANNOTATION", "bool")
    _take(o, "aux_affinity", "AUX_AFFINITY", "bool")
    _take(o, "forward_sub_graph_num", "FORWARD_SUB_GRAPH_NUM", "int")
    _take(o, "ilp_time_limit_s", "ILP_TIME_LIMIT", "float", 60.0)
    _take(o, "num_threads", "ILP_NUM_THREADS", "int")      # sub-graph problems solved concurrently
    import os
    if os.environ.get("TEPDIST_COLL_LATENCY_BYTES") is not None:   # per-collective latency term of the SPMD cost (bytes of wire
        o["collective_latency_bytes"] = float(os.environ["TEPDIST_COLL_LATENCY_BYTES"])   # time; 0 = byte counts only)
    return o


def auto_parallel_overrides() -> Dict[str, Any]:
    o: Dict[str, Any] = {}
    _take(o, "unbalanced_ratio", "UNBALANCED_RATIO", "float")
    if is_set("RULE_MODE") and env().get_bool("RULE_MODE"):
        o["spmd_rule_mode"] = True
    return o


def schedule_overrides() -> Dict[str, Any]:
    o: Dict[str, Any] = {}
    _take(o, "micro_num_limit", "MICRO_NUM_LIMIT", "int")
    _take(o, "buffer_save", "BUFFER_SAVE", "bool")
    _take(o, "reorder_send", "MULTI_REORDER", "bool")      # the scheduler's send hoisting (closest counterpart)
    _take(o, "early_ga", "EARLY_GA", "bool")               # default here: true (GA is where a micro-batch is released)
    _take(o, "group_sched_count", "GROUP_SCHED_COUNT", "int")   # micro-batch groups with their own 1F1B window (task_scheduler.cc:125)
    if os.environ.get("TEPDIST_RECV_RING"):                     # native knob: receive-buffer ring size per class (tests, experiments)
        o["recv_ring"] = int(os.environ["TEPDIST_RECV_RING"])
    return o


def hw_profile():
    """HW_PROFILE: cost-model constants of the planner / evaluator -- "h100" (default) or "reference_v100" (the reference's
    15 TFLOP/s / 300 GB/s constants, evaluator.h:47-56)."""
    from . import _C
    name = env().get("HW_PROFILE") if is_set("HW_PROFILE") else "h100"
    if name not in ("h100", "reference_v100"):
        raise ValueError(f"HW_PROFILE={name!r}: expected 'h100' or 'reference_v100'")
    return _C.HwProfile.reference_v100() if name == "reference_v100" else _C.HwProfile.h100()


def pp_bandwidth() -> Optional[float]:
    """PP_BANDWIDTH (GB/s) for pipeline send/recv cost in the task scheduler; None = the hardware profile's link bandwidth."""
    return env().get_double("PP_BANDWIDTH") * 1e9 if is_set("PP_BANDWIDTH") else None


def check_num_gradients(n_apply: int) -> None:
    """NUM_GRADIENTS: the reference's sanity check that the client's training graph has the expected number of gradients."""
    if is_set("NUM_GRADIENTS"):
        want = int(env().get_int("NUM_GRADIENTS"))
        if want > 0 and want != n_apply:
            raise ValueError(f"NUM_GRADIENTS={want} but the training step updates {n_apply} variables")


# Accepted for compatibility with the reference's config files but without effect here (and why):
#   ASYNC_SEND            pipeline sends are always isend: a blocking send can deadlock two stages that send to each other at the
#                         same point of the 1F1B steady state (their receives are posted later in their own task lists)
#   DISABLE_BUFFER_ALIAS  variables are always updated in place in the flat store
#   CLUSTER_SPEC, FRONTEND informational (set by the launcher)
INERT_KEYS = ("ASYNC_SEND", "DISABLE_BUFFER_ALIAS", "CLUSTER_SPEC", "FRONTEND")


def resolve_strategy(strategy: str) -> str:
    """"auto" defers to the flags: NUM_STAGES>1 -> config-mode pipeline, RULE_MODE -> rule planner."""
    if strategy != "auto":
        return strategy
    e = env()
    if is_set("NUM_STAGES") and e.get_int("NUM_STAGES") > 1:
        m = e.get_int("NUM_MICRO_BATCHES") if is_set("NUM_MICRO_BATCHES") else 0
        return f"pp{e.get_int('NUM_STAGES')}" + (f"m{m}" if m > 0 else "")
    if is_set("RULE_MODE") and e.get_bool("RULE_MODE"):
        return "rule"
    return strategy


def comm_mode(requested: Optional[str]) -> str:
    if requested is not None:
        return requested
    return env().get("COMM_MODE") or "fused"


def comm_dtype():
    """FP16_COMM: fp32 sum-reductions travel in 16 bit (bf16 here; custom_collective_expander.cc FP16 wrap)."""
    import torch
    return torch.bfloat16 if is_set("FP16_COMM") and env().get_bool("FP16_COMM") else None


def async_recv() -> bool:
    """ASYNC_RECV (default true): a pipeline receive is posted at its Recv task and awaited at the Input task of its micro-batch.
    false: awaited right at the Recv task (a debugging aid: serialises communication with compute; deadlock-free because the
    scheduler places every Recv after the start of its Send)."""
    return env().get_bool("ASYNC_RECV") if is_set("ASYNC_RECV") else True


def fake_input() -> bool:
    return is_set("FAKE_INPUT") and env().get_bool("FAKE_INPUT")


def debug() -> bool:
    return (is_set("DEBUG") and env().get_bool("DEBUG")) or (is_set("DUMP_ARTIFACTS") and env().get_bool("DUMP_ARTIFACTS"))
