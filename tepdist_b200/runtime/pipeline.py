"""Pipeline-parallel worker: executes this rank's ordered task list (1F1B schedule from the C++ scheduler).

Reference parity (SURVEY §3.3, D8, K4, Appendix E): DAPPLEExecutable::ExecuteTaskList — per task: Input (wait recv),
Compute (enqueue the stage executable), Output, Send / Recv (NCCL p2p on side streams, event-synchronised), GAInit / GA,
and the optimizer (AG) on the last micro-batch.  Ranks execute their static lists in lock-step order, which is what
makes the send/recv pairing deadlock-free (no dynamic dependency tracking at run time).
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from ..ir import Graph, Node, Value
from .executor import Executor, shard_of


def elide_shared_level_collectives(g: Graph, shared_levels: List[int]) -> Tuple[Graph, List[Tuple[int, int]]]:
    """Collectives on a time-multiplexed (micro-batch) level are not communication: the reduction over micro-batches
    is gradient accumulation (GA).  Rewire their users to the operand; return the fetches that must be SUMMED over
    micro-batches (e.g. the loss)."""
    alias: Dict[Tuple[int, int], Value] = {}

    def res(v: Value) -> Value:
        while v.key() in alias:
            v = alias[v.key()]
        return v

    out = Graph(g.name)
    out.meta = dict(g.meta)
    idmap: Dict[int, int] = {}
    summed: List[Tuple[int, int]] = []
    for n in g.nodes:
        if n.op in ("all_reduce", "reduce_scatter", "all_gather", "dynamic_slice") and int(n.attrs.get("level", -1)) in shared_levels \
                and n.op == "all_reduce":
            alias[(n.id, 0)] = n.inputs[0]
            continue
        ins = []
        for v in n.inputs:
            r = res(v)
            ins.append(Value(idmap[r.node], r.idx))
        nn = out.add(n.op, ins, n.outputs, dict(n.attrs), n.name, n.group, n.backward)
        nn.stage = n.stage
        idmap[n.id] = nn.id
    for v in g.outputs:
        r = res(v)
        if r.key() != v.key():
            summed.append((idmap[r.node], r.idx))
        out.outputs.append(Value(idmap[r.node], r.idx))
    for var, v in g.updates.items():
        r = res(v)
        out.updates[idmap[var]] = Value(idmap[r.node], r.idx)
    for n in out.nodes:
        if "slot_of" in n.attrs and n.attrs["slot_of"] in idmap:
            n.attrs["slot_of"] = idmap[n.attrs["slot_of"]]
    out._next_group = g._next_group
    return out, summed


class StageWorker:
    """One pipeline stage on one rank."""

    def __init__(self, graph: Graph, stage: int, num_stages: int, num_micro: int, micro_level: int, device: torch.device,
                 peer_prev: Optional[int], peer_next: Optional[int], seed: int = 0, collective: Any = None,
                 coords: Optional[Dict[int, int]] = None, comm_mode: str = "nccl", use_cuda_graph: bool = False):
        self.stage, self.S, self.M, self.micro_level = stage, num_stages, num_micro, micro_level
        # CUDA graphs of the stage bodies (reference: each stage is ONE compiled executable per direction, virtual_client.cc:
        # 1662-1807; here the interpreter would otherwise pay ~30 us of Python per kernel, 7000+ kernels per step): the forward
        # and the backward body of a micro-batch are captured once per in-flight SLOT (activations of slot k live in graph k's
        # private pool; receive buffers, input staging and outputs have fixed addresses per slot) and replayed afterwards
        import os
        # TEPDIST_PP_GRAPH_EMULATE=1 (CPU tests): same slot / staging / fixed-address bookkeeping, but a "replay" re-executes the
        # body eagerly and copies its results into the tensors recorded at "capture" -- a slot reused while its previous owner is
        # still live, a stale staging buffer or a mis-wired receive slot then shows up as a wrong loss without any GPU
        self.graph_emulate = os.environ.get("TEPDIST_PP_GRAPH_EMULATE") == "1"
        self.use_graph = (bool(use_cuda_graph) and device.type == "cuda") or self.graph_emulate
        self.graphs: Dict[Tuple[bool, int], Any] = {}
        self.graph_env: Dict[Tuple[bool, int], Dict[Tuple[int, int], torch.Tensor]] = {}
        self._static_feeds: Dict[int, Dict[str, torch.Tensor]] = {}
        self.slot_of: Dict[int, int] = {}
        self.num_slots = 0
        self.steps_run = 0
        self.graph_stats = {"captured": 0, "replayed": 0}
        self.peer_prev, self.peer_next = peer_prev, peer_next
        g, self.summed = elide_shared_level_collectives(graph, [micro_level] if num_micro > 1 else [])
        # this stage's slice of the program: sources it owns + its compute nodes.  WHICH nodes run per micro-batch forward /
        # per micro-batch backward / once per step, and WHICH values cross which stage boundary, is not derived here: it is the
        # DefContext tree of the C++ core (SyncFreeDecompose + StageDecompose, csrc/auto_parallel.cc) for exactly this graph
        self.full = g
        from .. import _C
        from ..planner import to_native
        cg = to_native(g)
        self.decomposition = _C.sync_free_decompose(cg, micro_level if num_micro > 1 else -1)
        self.transfers = _C.stage_decompose(cg, num_stages, self.decomposition)
        ctx = {(c.kind, c.stage): c for c in self.decomposition.ctx}
        mine = [n for n in g.nodes if n.stage == stage]
        self.sub, self.idmap = self._extract(g, mine)
        self.exec = Executor(self.sub, device, seed=seed, collective=collective, coords=dict(coords or {}), comm_mode=comm_mode)
        self.exec.grad_accumulate = True    # gradients accumulate over micro-batches: atomically-added, zero-filled slots
        self.exec.micro_level = micro_level if num_micro > 1 else None
        self._slot_rng: Dict[int, torch.Tensor] = {}   # dropout (step, micro-batch) words read by slot k's captured bodies
        spmd = 1
        if collective is not None:
            spmd = max(1, collective.mesh.world // max(1, num_stages))
        self.exec.pipeline_norm_divisor = spmd   # global-norm clipping: stage sums are added up over the whole job
        self.exec._plan_store_init()
        ex = self.exec
        if num_stages > 1:
            fwd_ids = {self.idmap[i] for i in ctx[("stage_fwd", stage)].nodes if i in self.idmap}
            bwd_ids = {self.idmap[i] for i in ctx[("stage_bwd", stage)].nodes if i in self.idmap}
        else:   # one stage: the CG context is the whole per-micro-batch program
            cgc = next(c for c in self.decomposition.ctx if c.kind == "cg")
            fwd_ids = {self.idmap[i] for i in cgc.nodes if i in self.idmap and not g.nodes[i].backward}
            bwd_ids = {self.idmap[i] for i in cgc.nodes if i in self.idmap and g.nodes[i].backward}
        # the forward list additionally materialises the sources this stage owns (variables / constants live in ENTRY)
        self.fwd_nodes = [n for n in self.sub.nodes if (n.id in fwd_ids or (n.op in ("parameter", "constant") and not n.backward))
                          and n.id not in ex.post_apply]
        self.bwd_nodes = [n for n in self.sub.nodes if n.id in bwd_ids and n.id not in ex.post_apply]
        self.env: Dict[int, Dict[Tuple[int, int], torch.Tensor]] = {}
        # persistent receive buffers: (backward, value key, slot) -> (buffer, micro-batch that owns it this step)
        self._ring: Dict[Tuple[bool, Tuple[int, int], int], Tuple[torch.Tensor, Optional[int]]] = {}
        self.ring_stats = {"alloc": 0, "reuse": 0, "miss": 0}
        self.pending_send: List[Any] = []
        from .. import config
        self.async_recv = config.async_recv()
        self.sync_recvs = 0
        self.loss_acc: Optional[torch.Tensor] = None
        # values the optimizer phase reads from the environment (gradients of variables that are not flat-bound, and
        # anything else the apply / post-apply nodes consume from the per-micro-batch part)
        pre = {n.id for n in self.fwd_nodes} | {n.id for n in self.bwd_nodes}
        self.acc_keys = set()
        for n in self.sub.nodes:
            if n.id in ex.post_apply or n.op.startswith("apply_"):
                for v in n.inputs:
                    if v.node in pre and v.key() not in ex.grad_binding and self.sub.nodes[v.node].op not in ("parameter", "state"):
                        self.acc_keys.add(v.key())
        self.acc_env: Dict[Tuple[int, int], torch.Tensor] = {}

    # ------------------------------------------------------------------ sub-graph extraction
    def _extract(self, g: Graph, mine: List[Node]):
        """Copy this stage's nodes; values produced on other stages become `boundary` placeholder nodes that are filled
        by Recv tasks (threaded through intermediate stages by the transfer plan)."""
        sub = Graph(f"{g.name}.stage{self.stage}")
        sub.meta = dict(g.meta)
        idmap: Dict[int, int] = {}
        self.boundary_in: Dict[Tuple[int, int], int] = {}   # full-graph value -> placeholder node id in sub
        mine_ids = {n.id for n in mine}
        for n in mine:
            ins = []
            for v in n.inputs:
                if v.node in mine_ids:
                    ins.append(Value(idmap[v.node], v.idx))
                else:
                    key = v.key()
                    if key not in self.boundary_in:
                        bn = sub.add("boundary", [], [g.type_of(v)], {"src": list(key)}, f"recv_{v.node}_{v.idx}", -1,
                                     g.nodes[v.node].backward)
                        self.boundary_in[key] = bn.id
                    ins.append(Value(self.boundary_in[key], 0))
            nn = sub.add(n.op, ins, n.outputs, dict(n.attrs), n.name, n.group, n.backward)
            nn.stage = n.stage
            idmap[n.id] = nn.id
        for v in g.outputs:
            if v.node in mine_ids:
                sub.outputs.append(Value(idmap[v.node], v.idx))
        for var, v in g.updates.items():
            if var in mine_ids and v.node in mine_ids:
                sub.updates[idmap[var]] = Value(idmap[v.node], v.idx)
        for n in sub.nodes:
            if "slot_of" in n.attrs and n.attrs["slot_of"] in idmap:
                n.attrs["slot_of"] = idmap[n.attrs["slot_of"]]
        return sub, idmap

    # ------------------------------------------------------------------ transfer plan (neighbour-only, B4)
    def plan_transfers(self) -> None:
        """For every boundary (s, s+1) and direction, the ordered list of full-graph values that cross it -- the StageTransfer
        list of the C++ StageDecompose pass (values consumed k stages away hop through each intermediate stage).  Every rank
        decomposes the same graph, hence derives the same lists in the same order."""
        fwd: Dict[int, List[Tuple[int, int]]] = {b: [] for b in range(self.S - 1)}   # boundary b: stage b -> b+1
        bwd: Dict[int, List[Tuple[int, int]]] = {b: [] for b in range(self.S - 1)}   # boundary b: stage b+1 -> b
        for t in self.transfers:
            if t.backward:
                bwd[t.to_stage].append(tuple(t.value))
            else:
                fwd[t.from_stage].append(tuple(t.value))
        self.xfer_fwd, self.xfer_bwd = fwd, bwd

    # ------------------------------------------------------------------ phases
    def _micro_env(self, m: int) -> Dict[Tuple[int, int], torch.Tensor]:
        return self.env.setdefault(m, {})

    def _run_nodes(self, nodes: List[Node], m: int, feeds: Dict[str, torch.Tensor], accumulate: bool = True) -> None:
        ex = self.exec
        ex.coords[self.micro_level] = m
        ex._tag = m
        env = self._micro_env(m)
        for n in nodes:
            if n.op == "boundary":
                continue
            try:
                ins = [env[v.key()] for v in n.inputs]
            except KeyError as e:
                miss = self.sub.nodes[e.args[0][0]]
                raise RuntimeError(f"stage {self.stage} micro {m}: node {n.id} {n.op} '{n.name}' needs value of node {miss.id} "
                                   f"{miss.op} '{miss.name}' (backward={miss.backward}, post_apply={miss.id in ex.post_apply}) "
                                   f"which has not been produced") from e
            if n.id in ex.alias_of:
                outs = [env[ex.alias_of[n.id]]]
            else:
                ex._env = env
                outs = ex._exec(n, ins, feeds)
            for i, t in enumerate(outs):
                env[(n.id, i)] = t
                pid = ex.grad_binding.get((n.id, i))
                if pid is not None and ex.fused_apply_ok:
                    gv = ex.store.grad_view(pid)
                    if t.data_ptr() != gv.data_ptr():
                        gv.add_(t.reshape(gv.shape).to(gv.dtype))
                if accumulate and (n.id, i) in self.acc_keys:
                    self._accumulate_extra((n.id, i), t)

    def _accumulate_extra(self, key: Tuple[int, int], t: torch.Tensor) -> None:
        """Gradients outside the flat buffer: accumulate over micro-batches (GA)."""
        if key in self.acc_env:
            self.acc_env[key] = self.acc_env[key] + t
        else:
            self.acc_env[key] = t.clone()

    # ------------------------------------------------------------------ CUDA graphs of the stage bodies
    def plan_slots(self, task_list: List[Dict[str, Any]]) -> None:
        """Static slot of every micro-batch: taken at the first task that touches it (a hoisted forward Recv or the forward
        Compute), returned where the scheduler's GC plan releases the micro-batch.  The number of slots is what the schedule
        keeps in flight on this stage (1F1B: at most stages - stage; GROUP_SCHED_COUNT groups: more)."""
        free: List[int] = []
        slot_of: Dict[int, int] = {}
        n = 0
        for t in task_list:
            m = t["micro"]
            if m is not None and m >= 0 and m not in slot_of and t["type"] in ("Recv", "Compute", "Input") and not t["backward"]:
                if free:
                    free.sort()
                    slot_of[m] = free.pop(0)
                else:
                    slot_of[m] = n
                    n += 1
            for dead in t.get("release", ()):
                if dead in slot_of:
                    free.append(slot_of[dead])
        self.slot_of, self.num_slots = slot_of, n

    def _drop_state(self, slot: Optional[int], m: int) -> None:
        """Point the dropout kernels at the (step, micro-batch) words for micro-batch m: the executor's own for an eager body,
        slot k's fixed-address copy for a captured one (a replay for another micro-batch then reads that micro-batch's index,
        staged here like the inputs, not the one frozen at capture)."""
        ex = self.exec
        if not ex.has_dropout:
            return
        if slot is None:
            st = ex.rng_state
        else:
            st = self._slot_rng.get(slot)
            if st is None:
                st = self._slot_rng[slot] = torch.zeros(2, dtype=torch.int64, device=ex.device)
            st[0].fill_(ex.step_count)
        st[1].fill_(m)
        ex.drop_state = st

    def _stage_feeds(self, slot: int, m: int, feeds: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        """Per-slot staging of the fed inputs this stage consumes: micro-batch m's shard is copied into a fixed buffer (the
        captured body reads that address)."""
        ex = self.exec
        ex.coords[self.micro_level] = m
        self._drop_state(slot, m)
        out = self._static_feeds.setdefault(slot, {})
        dev = ex.device
        for n in self.sub.nodes:
            if n.op != "input" or n.name not in feeds:
                continue
            t = feeds[n.name]
            if t.device != dev:
                t = t.to(dev, non_blocking=True)
            want = tuple(n.outputs[0].shape)
            if tuple(t.shape) != want:
                t = shard_of(t, n.attrs, ex.coords)
            if tuple(t.shape) != want:
                raise ValueError(f"pipeline stage {self.stage}: input '{n.name}' fed with shape {tuple(feeds[n.name].shape)}; with CUDA "
                                 f"graphs the GLOBAL batch {tuple(n.attrs.get('full_shape', want))} must be fed on every rank")
            if n.name not in out:
                out[n.name] = t.contiguous().clone()
            else:
                out[n.name].copy_(t, non_blocking=True)
        return out

    def _run_phase(self, bwd: bool, m: int, feeds: Dict[str, torch.Tensor]) -> None:
        nodes = self.bwd_nodes if bwd else self.fwd_nodes
        if not self.use_graph or self.steps_run < 1 or m not in self.slot_of:
            self._drop_state(None, m)
            self._run_nodes(nodes, m, feeds)          # eager (first step = warm-up: lazy allocations, kernel attributes)
            return
        slot = self.slot_of[m]
        key = (bwd, slot)
        sfeeds = self._stage_feeds(slot, m, feeds)
        env = self._micro_env(m)
        if key not in self.graphs:
            before = set(env)
            if self.graph_emulate:
                self._run_nodes(nodes, m, sfeeds, accumulate=False)
                self.graphs[key] = "emulated"
            else:
                cur = torch.cuda.current_stream()
                side = getattr(self, "_cap_stream", None)
                if side is None:
                    side = self._cap_stream = torch.cuda.Stream()
                side.wait_stream(cur)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.stream(side):
                    # thread-local capture mode: NCCL's watchdog thread and in-flight p2p of other streams stay legal; no device-
                    # wide synchronisation here (a peer may be waiting for data this rank has already queued)
                    g.capture_begin(capture_error_mode="thread_local")
                    try:
                        self._run_nodes(nodes, m, sfeeds, accumulate=False)
                    finally:
                        g.capture_end()
                cur.wait_stream(side)
                self.graphs[key] = g
                g.replay()                            # capture records, it does not execute
            self.graph_env[key] = {k: v for k, v in env.items() if k not in before}
            self.graph_stats["captured"] += 1
        elif self.graph_emulate:
            scratch = dict(env)
            self.env[m] = scratch
            self._run_nodes(nodes, m, sfeeds, accumulate=False)
            self.env[m] = env
            for k, v in self.graph_env[key].items():
                if scratch[k].data_ptr() != v.data_ptr():
                    v.copy_(scratch[k])
            env.update(self.graph_env[key])
            self.graph_stats["replayed"] += 1
        else:
            env.update(self.graph_env[key])
            self.graphs[key].replay()
            self.graph_stats["replayed"] += 1
        for k in self.acc_keys:
            if k in self.graph_env[key]:
                self._accumulate_extra(k, self.graph_env[key][k])

    def begin_step(self) -> None:
        self.exec.step_count += 1
        self.exec._set_hyper()
        self.exec.store.grad.zero_()       # GAInit
        self.env.clear()
        for rk, (buf, _) in list(self._ring.items()):   # every slot is free at a step boundary
            self._ring[rk] = (buf, None)
        self.acc_env = {}
        self.loss_acc = None

    def forward(self, m: int, feeds: Dict[str, torch.Tensor]) -> None:
        self._run_phase(False, m, feeds)

    def backward(self, m: int, feeds: Dict[str, torch.Tensor]) -> None:
        self._run_phase(True, m, feeds)
        env = self._micro_env(m)
        for v in self.sub.outputs:   # fetches (loss) are summed over micro-batches
            if v.key() in env:
                t = env[v.key()].detach().float()
                self.loss_acc = t.clone() if self.loss_acc is None else self.loss_acc + t

    def release(self, m: int) -> None:
        """GC: every activation of micro-batch m is dead (its backward ran and its gradients were sent).  Called where
        the task list says so (`release` entries, derived from the C++ GC plan -- reference D5 MakeTaskGraphGCPlan)."""
        self.env.pop(m, None)
        self._threaded.pop(m, None)

    def apply(self, feeds: Dict[str, torch.Tensor]) -> None:
        """AG: gradient sync over the SPMD level (if any) + optimizer + post-update re-layouts, once per step."""
        self.exec.run_optimizer(self.acc_env, feeds)

    # ------------------------------------------------------------------ p2p
    def _values_for(self, boundary: int, backward: bool) -> List[Tuple[int, int]]:
        return (self.xfer_bwd if backward else self.xfer_fwd)[boundary]

    def _lookup(self, m: int, key: Tuple[int, int]) -> torch.Tensor:
        env = self._micro_env(m)
        if key[0] in self.idmap:                       # produced here
            return env[(self.idmap[key[0]], key[1])]
        return env[(self.boundary_in[key], 0)] if key in self.boundary_in else self._threaded[m][key]

    def send(self, m: int, backward: bool) -> List[Any]:
        boundary = self.stage - 1 if backward else self.stage
        peer = self.peer_prev if backward else self.peer_next
        works = []
        for key in self._values_for(boundary, backward):
            t = self._lookup(m, key).contiguous()
            works.append((dist.isend(t, peer), t))   # keep the payload alive until the send completes
        return works

    def _recv_buffer(self, m: int, backward: bool, key: Tuple[int, int], slot: int) -> torch.Tensor:
        """Receive buffer for value `key` of micro-batch m.  slot >= 0 (BUFFER_SAVE): slot `slot` of the persistent ring of
        this (direction, value) class, whose size the scheduler chose (groups x in-flight limit, or TEPDIST_RECV_RING) --
        reference execution_state.cc:219 recv_dapple_buffer_ptr_[key][buffer_id].  A slot whose previous micro-batch has
        not been released yet cannot be waited for here (its release is later in THIS worker's task list; the reference
        waits on the consumer's event from another thread), so such a receive gets a fresh buffer and is counted as a miss."""
        from .executor import torch_dtype
        dev = self.exec.device
        tt = self.full.type_of(Value(*key))

        def fresh():
            return torch.empty(tt.shape, dtype=torch_dtype(tt.dtype, dev), device=dev)
        if slot < 0:
            return fresh()
        rk = (backward, key, slot)
        ent = self._ring.get(rk)
        if ent is not None:
            buf, owner = ent
            if owner != m and (owner in self.env or owner in self._threaded):
                if self.use_graph:
                    raise RuntimeError(f"stage {self.stage}: receive slot {slot} of micro-batch {m} is still owned by {owner}")
                self.ring_stats["miss"] += 1
                return fresh()
            for w, t in self.pending_send:          # a pass-through send may still be reading the slot
                if t.data_ptr() == buf.data_ptr():
                    w.wait()
            self.ring_stats["reuse"] += 1
        else:
            buf = fresh()
            self.ring_stats["alloc"] += 1
        self._ring[rk] = (buf, m)
        return buf

    def recv(self, m: int, backward: bool, slot: int = -1) -> List[Any]:
        boundary = self.stage if backward else self.stage - 1
        peer = self.peer_next if backward else self.peer_prev
        env = self._micro_env(m)
        works = []
        if self.use_graph and m in self.slot_of:
            slot = self.slot_of[m]       # the receive ring is indexed by the graph slot: captured bodies read fixed addresses
        for key in self._values_for(boundary, backward):
            buf = self._recv_buffer(m, backward, key, slot)
            works.append(dist.irecv(buf, peer))
            if key in self.boundary_in:
                env[(self.boundary_in[key], 0)] = buf
            self._threaded.setdefault(m, {})[key] = buf   # may only pass through to the next stage
        return works

    _threaded: Dict[int, Dict[Tuple[int, int], torch.Tensor]] = {}

    def evaluate_forward(self, m: int, feeds: Dict[str, torch.Tensor]) -> None:
        """Micro-batch m's forward body, eagerly and in evaluation mode (Executor.run_eval_nodes); on the stage that holds
        the loss its triple is added into eval_acc."""
        ex = self.exec
        if self._eval_free is None:
            # nodes downstream of the loss (the reduction of the loss output a plan may add) have no use in an evaluation
            after = {n.id for n in self.fwd_nodes if n.op == "softmax_xent"}
            for n in self.fwd_nodes:
                if any(v.node in after for v in n.inputs):
                    after.add(n.id)
            self._eval_nodes = [n for n in self.fwd_nodes if n.op == "softmax_xent" or n.id not in after]
            self._eval_free = ex._plan_eval(self.sub, self._eval_nodes)[1]
            out = self._values_for(self.stage, False) if self.stage < self.S - 1 else []
            sent = {(self.idmap[k[0]], k[1]) if k[0] in self.idmap else (self.boundary_in.get(k), 0) for k in out}
            for ks in self._eval_free.values():     # values sent to the next stage live until the Send task
                ks[:] = [k for k in ks if k not in sent]
        ex.coords[self.micro_level] = m
        t = ex.run_eval_nodes(self._eval_nodes, self._eval_free, self._micro_env(m), feeds, ("eval", m))
        if t is not None:
            self.eval_acc = t.clone() if self.eval_acc is None else self.eval_acc + t

    eval_acc: Optional[torch.Tensor] = None
    _eval_free: Optional[Dict[int, List[Tuple[int, int]]]] = None
    _eval_nodes: List[Node] = []


def run_pipeline_eval(worker: StageWorker, task_list: List[Dict[str, Any]], feeds: Dict[str, torch.Tensor]) -> Optional[torch.Tensor]:
    """One evaluation pass: this device's task list without the backward tasks and the optimizer (AG); every stage body runs
    eagerly with dropout off.  Returns the loss triple summed over the micro-batches on the stage that holds the loss, None
    elsewhere.  Nothing of the training step's state is touched: receive buffers are fresh (not the slot ring the captured
    bodies read), and every micro-batch environment is released by the end of the call."""
    worker.eval_acc = None
    worker.env.clear()
    worker._threaded = {}
    use_graph, worker.use_graph = worker.use_graph, False     # (recv: fresh buffers instead of the graph slots' ring)
    pending_recv: Dict[int, List[Any]] = {}
    pending_send: List[Any] = []
    try:
        for t in task_list:
            kind, m, bwd = t["type"], t["micro"], t["backward"]
            if not bwd:
                if kind == "Recv":
                    pending_recv[m] = worker.recv(m, False, -1)
                elif kind == "Input":
                    for w in pending_recv.pop(m, []):
                        w.wait()
                elif kind == "Compute":
                    worker.evaluate_forward(m, feeds)
                elif kind == "Send":
                    pending_send += worker.send(m, False)
            for dead in t.get("release", ()):
                worker.release(dead)
        for w, _ in pending_send:
            w.wait()
    finally:
        worker.use_graph = use_graph
        worker.env.clear()
        worker._threaded = {}
    return worker.eval_acc


def run_pipeline_step(worker: StageWorker, task_list: List[Dict[str, Any]], feeds: Dict[str, torch.Tensor]) -> Optional[float]:
    """Execute one training step by walking this device's ordered task list."""
    if worker.use_graph and getattr(worker, "_slots_for", None) is not task_list:
        worker.plan_slots(task_list)
        worker._slots_for = task_list
    worker.begin_step()
    timing = getattr(worker, "timing", False) and worker.exec.device.type == "cuda"
    spans: List[Tuple[Any, Any]] = []
    if timing:
        t_begin = torch.cuda.Event(enable_timing=True)
        t_begin.record()
    worker._threaded = {}
    pending_recv: Dict[Tuple[int, bool], List[Any]] = {}
    pending_send = worker.pending_send = []
    for t in task_list:
        kind, m, bwd = t["type"], t["micro"], t["backward"]
        if kind == "Recv":
            pending_recv[(m, bwd)] = worker.recv(m, bwd, t.get("buffer_id", -1))
            if not worker.async_recv:            # ASYNC_RECV=false: block here instead of at the Input task
                for w in pending_recv.pop((m, bwd)):
                    w.wait()
                worker.sync_recvs += 1
        elif kind == "Input":
            for w in pending_recv.pop((m, bwd), []):
                w.wait()
        elif kind == "Compute":
            if timing:
                a, b_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
            (worker.backward if bwd else worker.forward)(m, feeds)
            if timing:
                b_.record()
                spans.append((a, b_))
        elif kind == "Send":
            pending_send += worker.send(m, bwd)   # (work, payload) pairs: payloads stay referenced until waited
        elif kind == "AG":
            for w, _ in pending_send:
                w.wait()
            del pending_send[:]
            worker.apply(feeds)
        for dead in t.get("release", ()):         # the scheduler's GC plan (task_graph.cc ComputeReleasePlan) decides
            worker.release(dead)
    for w, _ in pending_send:
        w.wait()
    worker.steps_run += 1
    if timing:
        # measured bubble of THIS stage: share of the step (first task .. last send completed) in which no stage body ran
        t_end = torch.cuda.Event(enable_timing=True)
        t_end.record()
        torch.cuda.synchronize()
        busy = sum(a.elapsed_time(b_) for a, b_ in spans)
        total = t_begin.elapsed_time(t_end)
        worker.last_timing = {"busy_ms": busy, "step_ms": total, "bubble": 1.0 - busy / total if total > 0 else 0.0}
    return None if worker.loss_acc is None else float(worker.loss_acc)
