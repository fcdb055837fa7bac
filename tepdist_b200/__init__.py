"""tepdist_b200 — a H100-native automatic distributed-training system with TePDist's capabilities.

Layers (see DESIGN.md): PyTorch client frontend -> planner IR -> C++ planner (SPMD cones/ILP, pipeline
stage ILP, sync-free micro-batching) -> transforms -> task-graph runtime -> sm_90a kernels + NCCL /
peer-memory collectives.
"""
__version__ = "0.1.0"
