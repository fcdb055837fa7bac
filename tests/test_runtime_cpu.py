"""CPU tests for the C++ runtime core: slice utils + sharded Philox init (mirrors the reference's only unit tests,
pjrt/slice_utils_test.cc and pjrt/initializers_test.cc — SURVEY §4), device mesh, task DAG, scheduler, ServiceEnv."""
import json
import os

import numpy as np
import pytest

from tepdist_b200 import _C

S, G = _C.DimStrategy.split, _C.DimStrategy.glue


# ------------------------------------------------------------------------------------------------ slice utils
def _full(shape):
    return np.arange(int(np.prod(shape)), dtype=np.float32).reshape(shape)


def test_slice_major_minor_and_two_dims():
    x = _full((4, 6))
    np.testing.assert_array_equal(_C.slice_copy(x, [4, 6], [S(0, 2)], [1]), x[2:4])           # major dim
    np.testing.assert_array_equal(_C.slice_copy(x, [4, 6], [S(1, 3)], [2]), x[:, 4:6])        # minor dim
    np.testing.assert_array_equal(_C.slice_copy(x, [4, 6], [S(0, 2), S(1, 2)], [1, 0]), x[2:4, 0:3])   # two levels / two dims
    np.testing.assert_array_equal(_C.slice_copy(x, [4, 6], [G()], [0]), x)                    # no dist spec


def test_slice_same_dim_twice_and_strided():
    x = _full((8, 3))
    # same dim cut by two levels (micro-batch x SPMD): second level acts inside the first level's shard
    got = _C.slice_copy(x, [8, 3], [S(0, 2), S(0, 2)], [1, 0])
    np.testing.assert_array_equal(got, x[4:6])
    # layout-aware split: within every block of 4 rows shard k owns the k-th half
    got = _C.slice_copy(x, [8, 3], [S(0, 2, 4)], [1])
    np.testing.assert_array_equal(got, np.concatenate([x[2:4], x[6:8]]))
    runs = _C.slice_runs([8, 3], [S(0, 2, 4)], [1])
    assert runs == [(6, 6), (18, 6)]


# ------------------------------------------------------------------------------------------------ sharded init
@pytest.mark.parametrize("kind", ["uniform", "normal", "truncated_normal"])
@pytest.mark.parametrize("shape,levels,ids", [
    ([16, 8], [S(0, 4)], [2]),                 # shard on top dim
    ([6, 10], [S(1, 2)], [1]),                 # shard on inner dim
    ([7, 13], [G()], [0]),                     # replication, prime sizes
    ([3, 5, 8], [S(2, 4)], [3]),               # multi-dimension
    ([12, 6], [S(0, 2), S(1, 3)], [1, 2]),     # two levels
    ([2, 3], [S(1, 3)], [0]),                  # size < group in the other dim
])
def test_sharded_philox_equals_slice_of_full(kind, shape, levels, ids):
    n = int(np.prod(shape))
    full = np.asarray(_C.philox_fill(kind, 1234, 0, n, 0.5, 2.0, -1.0, 3.0)).reshape(shape)
    shard = np.asarray(_C.philox_fill_shard(kind, 1234, shape, levels, ids, 0.5, 2.0, -1.0, 3.0))
    ref = np.asarray(_C.slice_copy(full, shape, levels, ids))
    np.testing.assert_array_equal(shard, ref)   # bit exact


def test_philox_statistics_and_offsets():
    a = np.asarray(_C.philox_fill("normal", 7, 0, 200000, 0.0, 1.0, 0, 1))
    assert abs(a.mean()) < 0.01 and abs(a.std() - 1.0) < 0.01
    b = np.asarray(_C.philox_fill("normal", 7, 1000, 50, 0.0, 1.0, 0, 1))
    np.testing.assert_array_equal(b, a[1000:1050])          # any window of the stream is reproducible (multi-thread fill)
    t = np.asarray(_C.philox_fill("truncated_normal", 9, 0, 100000, 0.0, 1.0, 0, 1))
    assert np.abs(t).max() <= 2.0
    u = np.asarray(_C.philox_fill("uniform", 9, 0, 100000, 0, 1, 2.0, 5.0))
    assert u.min() >= 2.0 and u.max() <= 5.0 and abs(u.mean() - 3.5) < 0.02


# ------------------------------------------------------------------------------------------------ device mesh
def test_comm_dev_manager_groups():
    m = _C.CommDevManager()
    # level 0 = micro-batch (shared), level 1 = SPMD(2), level 2 = stage(4); stage rotated outermost
    m.build([8, 2, 4], [True, False, False], [2, 1, 0], 2, 4)
    assert m.total_devices() == 8
    assert m.global_device([5, 1, 3]) == 3 * 2 + 1          # micro id contributes nothing
    assert m.coords(7) == [0, 1, 3]
    assert m.group_of(5, 1).devices == [4, 5] and m.rank_in_group(5, 1) == 1
    assert m.group_of(5, 2).devices == [1, 3, 5, 7] and m.rank_in_group(5, 2) == 2
    assert len(m.all_groups(1)) == 4 and len(m.all_groups(2)) == 2
    assert m.worker_of(5) == 1 and m.local_device(5) == 1
    assert m.group_spans_workers(m.group_of(5, 2)) and not m.group_spans_workers(m.group_of(5, 1))


# ------------------------------------------------------------------------------------------------ task DAG + scheduler
def _spec(S_, M, spmd=1):
    sp = _C.PipelineSpec()
    sp.num_stages, sp.num_micro, sp.spmd = S_, M, spmd
    sp.fwd_seconds = [1e-3] * S_
    sp.bwd_seconds = [2e-3] * S_
    sp.ag_seconds = [5e-4] * S_
    sp.act_bytes = [1e9] * S_
    sp.boundary_bytes = [8e6] * (S_ - 1)
    return sp


def test_task_dag_structure_and_dominance():
    sp = _spec(4, 8, 2)
    dag = _C.build_pipeline_task_dag(sp)
    kinds = [n.type for n in dag.nodes]
    assert kinds.count(_C.TaskType.Compute) == 2 * 4 * 8
    assert kinds.count(_C.TaskType.Send) == kinds.count(_C.TaskType.Recv) == 2 * 3 * 8
    assert kinds.count(_C.TaskType.GA) == 4 * 8 and kinds.count(_C.TaskType.AG) == 4 and kinds.count(_C.TaskType.GAInit) == 4
    assert len(dag.topo_order()) == len(dag.nodes)
    idom = dag.dominance_tree()
    assert idom[dag.source] == dag.source and all(i >= 0 for i in idom)
    for n in dag.nodes:
        if n.type == _C.TaskType.Send:
            assert abs(n.device - n.peer_device) == sp.spmd       # neighbour stages only
    assert "digraph" in dag.to_dot()


def test_scheduler_is_1f1b_and_bounds_memory():
    S_, M = 4, 8
    sp = _spec(S_, M)
    dag = _C.build_pipeline_task_dag(sp)
    sch = _C.schedule_tasks(dag, sp, _C.ScheduleOptions())
    # per-device order respects dependencies
    pos = {}
    for dev, tasks in sch.device_tasks.items():
        for i, t in enumerate(tasks):
            pos[t] = (dev, i)
    for n in dag.nodes:
        for c in n.children:
            if pos[n.id][0] == pos[c][0]:
                assert pos[n.id][1] < pos[c][1]
            assert sch.finish[n.id] <= sch.start[c] + 1e-12
    # 1F1B: stage s never holds more than S - s forward activations
    for dev in range(S_):
        assert sch.peak_bytes[dev] <= (S_ - dev) * 1e9 + 1
    # pipeline efficiency close to the 1F1B ideal: (M * (f+b)) / ((M + S - 1) * (f+b))
    ideal = (M + S_ - 1) * 3e-3 + 5e-4
    assert sch.makespan < ideal * 1.15
    assert 0 < sch.bubble_ratio < 0.45 and not sch.oom
    # last stage alternates F and B from the start (steady 1F1B)
    last = [dag.nodes[t].name for t in sch.device_tasks[S_ - 1] if dag.nodes[t].type == _C.TaskType.Compute]
    assert last[:4] == ["F.s3.m0", "B.s3.m0", "F.s3.m1", "B.s3.m1"]
    # GPipe-style (no cap) uses more memory on stage 0
    o = _C.ScheduleOptions(); o.micro_num_limit = M
    dag2 = _C.build_pipeline_task_dag(sp)
    sch2 = _C.schedule_tasks(dag2, sp, o)
    assert sch2.peak_bytes[0] >= sch.peak_bytes[0]
    # GC plan: every task's output is released exactly once on its device list
    rel = [r for n in dag.nodes for r in n.mem_to_release]
    assert len(rel) == len(set(rel))
    assert any(n.buffer_id >= 0 for n in dag.nodes if n.type == _C.TaskType.Recv)


def test_scheduler_early_ga_and_receive_ring_options():
    """EARLY_GA (reference task_scheduler.cc:1367 ReorderGA; default on here): gradient accumulation of micro-batch m directly
    follows its backward bundle, so the micro-batch is released at once; off: GA yields to any ready compute and ends up later
    in the device order, at no cost in makespan.  GROUP_SCHED_COUNT: independent 1F1B windows per micro-batch group; the ring of
    receive-buffer slots per class covers what can be in flight."""
    S_, M = 4, 8
    sp = _spec(S_, M)

    def run(**kw):
        o = _C.ScheduleOptions()
        for k, v in kw.items():
            setattr(o, k, v)
        dag = _C.build_pipeline_task_dag(sp)
        return dag, _C.schedule_tasks(dag, sp, o)

    def ga_lag(dag, sch):
        lag = 0
        for tasks in sch.device_tasks.values():
            names = [dag.nodes[t].name for t in tasks]
            for i, nme in enumerate(names):
                if nme.startswith("ga."):
                    s, m = nme.split(".")[1:]
                    lag += i - names.index(f"out.B.{s}.{m}")
        return lag
    assert _C.ScheduleOptions().early_ga and _C.ScheduleOptions().group_sched_count == 0
    d1, early = run()
    d2, lazy = run(early_ga=False)
    n_ga = S_ * M
    assert ga_lag(d1, early) <= 2 * n_ga            # right behind out.B (a hoisted Send may sit in between)
    assert ga_lag(d2, lazy) > ga_lag(d1, early)
    assert abs(lazy.makespan - early.makespan) < 1e-4
    for dag, sch in ((d1, early), (d2, lazy)):      # both are valid orders of the DAG
        pos = {t: (dev, i) for dev, tasks in sch.device_tasks.items() for i, t in enumerate(tasks)}
        assert all(pos[n.id][1] < pos[c][1] for n in dag.nodes for c in n.children if pos[n.id][0] == pos[c][0])
    # GROUP_SCHED_COUNT: micro-batch m is scheduled in group m % G, every group with its own 1F1B window -> up to G x (S - s)
    # forward activations in flight on stage s, at no loss in makespan; a valid order of the DAG
    def peak_in_flight(dag, sch, dev):
        live = peak = 0
        for t in sch.device_tasks[dev]:
            n = dag.nodes[t]
            if n.type == _C.TaskType.Compute:
                live += -1 if n.backward else 1
                peak = max(peak, live)
        return peak
    d1g, one = run(group_sched_count=1)
    d2g, two = run(group_sched_count=2)
    assert [dag_n.name for dag_n in (d1g.nodes[t] for t in one.device_tasks[0])] == [d1.nodes[t].name for t in early.device_tasks[0]]
    for dev in range(S_):
        assert peak_in_flight(d1g, one, dev) <= S_ - dev
        assert peak_in_flight(d2g, two, dev) <= 2 * (S_ - dev)
    assert peak_in_flight(d2g, two, 0) > peak_in_flight(d1g, one, 0)
    assert two.makespan <= one.makespan * 1.02
    pos = {t: (dev, i) for dev, tasks in two.device_tasks.items() for i, t in enumerate(tasks)}
    assert all(pos[n.id][1] < pos[c][1] for n in d2g.nodes for c in n.children if pos[n.id][0] == pos[c][0])
    # receive ring: default = groups x in-flight limit (never undersized); `recv_ring` overrides it; `buffer_reused` marks the
    # receives that take over a slot from an earlier receive of their class
    for kw, ring in (({}, S_), ({"group_sched_count": 2}, 2 * S_), ({"recv_ring": 2}, 2), ({"recv_ring": 3, "group_sched_count": 2}, 3)):
        dag, _ = run(**kw)
        for st in range(S_):
            for bwd in (False, True):
                rc = sorted((n.micro, n.buffer_id, n.buffer_reused) for n in dag.nodes
                            if n.type == _C.TaskType.Recv and n.stage == st and n.backward == bwd)
                if rc:
                    assert {b for _, b, _ in rc} == set(range(min(ring, M)))
                    assert sum(1 for _, _, r in rc if not r) == min(ring, M) and len(rc) == M
    dag, _ = run(buffer_save=False)
    assert all(n.buffer_id < 0 for n in dag.nodes)


def test_flat_moment_buffers_exist_for_adamw_even_when_every_slot_node_is_chunk_shaped():
    """The sharded-optimizer path addresses m / v by flat offset.  In a plan where every variable is ZeRO-sharded all `state` nodes
    have chunk shapes, so none of them maps onto the flat buffers -- the buffers must be allocated regardless (a refactoring of
    ensure_slots briefly tied the allocation to the existence of a whole-shaped slot; the 8-GPU GPT-2 plan has next to none)."""
    import torch
    from tepdist_b200.frontend.builder import GraphBuilder, build_training_step
    from tepdist_b200.ir import TensorType
    from tepdist_b200.runtime.executor import Executor, VariableStore
    b = GraphBuilder("chunked", compute_dtype="f32")
    x = b.input("x", (4, 8), "f32")
    w = b.parameter("w", (8, 8), {"kind": "normal", "std": 0.1})
    g = build_training_step(b, b.reduce_mean(b.matmul(x, w), [0, 1], name="loss"), "adamw", lr=0.1)
    for n in g.nodes:                       # what the SPMD transform does to the slots of a ZeRO-sharded variable
        if n.op == "state":
            n.outputs[0] = TensorType((4, 8), "f32")
    st = VariableStore(g, torch.device("cpu"))
    assert not any(st._flat_slot(n) for n in st._state_nodes)
    st.ensure_slots()
    assert st.m is None                     # no whole-shaped slot and nobody asked for flat moments
    st.ensure_slots(flat_moments=True)
    assert st.m is not None and st.v is not None and st.m.numel() == st.master.numel()
    # the executor asks for them whenever the graph updates with AdamW
    g2 = build_training_step(*(lambda bb: (bb, bb.reduce_mean(bb.matmul(bb.input("x", (4, 8), "f32"), bb.parameter("w", (8, 8), {"kind": "normal", "std": 0.1})), [0, 1], name="loss")))(GraphBuilder("whole", compute_dtype="f32")), "adamw", lr=0.1)
    ex = Executor(g2, torch.device("cpu"), use_cuda_graph=False)
    assert ex.store.m is not None


def test_scheduler_reports_oom():
    sp = _spec(2, 4)
    sp.mem_limit = 1.5e9
    dag = _C.build_pipeline_task_dag(sp)
    assert _C.schedule_tasks(dag, sp, _C.ScheduleOptions()).oom


# ------------------------------------------------------------------------------------------------ config
def test_service_env_load_order(tmp_path, monkeypatch):
    env = _C.ServiceEnv.instance()
    env.load(str(tmp_path / "none.json"))
    assert env.get_int("OPT_LEVEL") == 2 and env.get_bool("BUFFER_SAVE") and "VAR_MEM_LIMIT" in env.keys()
    cfg = tmp_path / "config.json"
    cfg.write_text(json.dumps({"NUM_STAGES": 4, "COST_FACTOR": 2.5, "RULE_MODE": True, "BOGUS": 1}))
    monkeypatch.setenv("NUM_STAGES", "2")      # env overrides the file, with a warning
    warnings = env.load(str(cfg))
    assert env.get_int("NUM_STAGES") == 2 and env.get_double("COST_FACTOR") == 2.5 and env.get_bool("RULE_MODE")
    assert any("BOGUS" in w for w in warnings) and any("NUM_STAGES" in w for w in warnings)
    assert "NUM_STAGES=2" in env.dump()
    with pytest.raises(IndexError):
        env.get("NOPE")
    # a reload starts from the defaults again: nothing of the previous load (or of set()) may linger
    env.set("OPT_LEVEL", "0")
    monkeypatch.delenv("NUM_STAGES")
    env.load(str(tmp_path / "missing.json"))
    assert env.get_int("NUM_STAGES") == 0 and env.get_double("COST_FACTOR") == 1.0 and not env.get_bool("RULE_MODE")
    assert env.get_int("OPT_LEVEL") == 2


def test_profile_and_plan_artifact_dumps(tmp_path):
    """Executor.profile gives a per-node / per-op time table + chrome trace; DEBUG artefacts are written (SURVEY 5.1)."""
    import torch
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    from tepdist_b200.parallel import plan_spmd
    from tepdist_b200.runtime.executor import Executor
    from tepdist_b200.utils import trace
    cfg = CONFIGS["tiny"]
    g = build_gpt2_graph(cfg, batch=2)
    ex = Executor(g, torch.device("cpu"), use_cuda_graph=False)
    tok = torch.randint(0, cfg.n_vocab, (2, cfg.n_ctx), dtype=torch.int32)
    prof = ex.profile({"tokens": tok, "labels": torch.roll(tok, -1, 1)}, chrome_trace=str(tmp_path / "trace.json"))
    assert prof["total_ms"] > 0 and "linear" in prof["by_op"] and "optimizer" in prof["by_op"]
    assert sum(prof["by_op"].values()) <= prof["total_ms"] * 1.05
    ev = json.load(open(tmp_path / "trace.json"))["traceEvents"]
    assert len(ev) == len(prof["nodes"]) > 20
    sharded, info = plan_spmd(g, 2, "auto")
    d = trace.dump_plan_artifacts(sharded, info, str(tmp_path / "dump"))
    for f in ("strategies.txt", "plan.json", "step_graph.dot"):
        assert os.path.getsize(os.path.join(d, f)) > 0
    assert "all_reduce" in open(os.path.join(d, "step_graph.dot")).read() or "reduce_scatter" in open(os.path.join(d, "step_graph.dot")).read()


def test_tp_all_reduce_chains_are_found_for_fusion():
    """Megatron plan of GPT-2: every row-parallel projection is linear -> all_reduce -> +bias -> +residual, every
    column-parallel input gradient is linear_dgrad -> all_reduce; these are the chains the fused GEMM -> all-reduce path
    (parallel/symm.py GemmAllReduceMC, TEPDIST_TP_FUSED=1) takes over."""
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    from tepdist_b200.parallel import plan_spmd
    from tepdist_b200.runtime.executor import Executor
    cfg = CONFIGS["tiny"]
    sharded, info = plan_spmd(build_gpt2_graph(cfg, batch=4), 2, "tp")
    chains = Executor.find_tp_chains(sharded)
    fwd = [c for lid, c in chains.items() if sharded.nodes[lid].op == "linear"]
    bwd = [c for lid, c in chains.items() if sharded.nodes[lid].op == "linear_dgrad"]
    assert len(fwd) == 2 * cfg.n_layer, (len(fwd), info["collectives"])
    assert all(c["bias"] is not None and c["res"] is not None and len(c["chain"]) == 3 for c in fwd)
    assert len(bwd) >= 2 * cfg.n_layer and all(c["M"] == 4 * cfg.n_ctx and c["num"] == 2 for c in bwd)
    # a data-parallel plan has nothing to fuse
    dp, _ = plan_spmd(build_gpt2_graph(cfg, batch=4), 2, "auto")
    assert Executor.find_tp_chains(dp) == {}


def test_python_device_mesh_agrees_with_cxx_comm_dev_manager():
    """The runtime addresses devices through parallel/mesh.py::DeviceMesh, a Python mirror of the C++ CommDevManager (which is
    otherwise only unit-tested).  Two implementations of the same mixed-radix addressing must not drift: compare coordinates,
    the communicator of every device at every level, rank-in-group and the inverse mapping for many meshes, with
    time-multiplexed (share_dev) levels and non-trivial placement layouts -- including the shapes the runtime builds
    (pure SPMD, dp x tp, micro x spmd x stage with the stage level outermost)."""
    import itertools
    from tepdist_b200.parallel.mesh import DeviceMesh
    cases = []
    for nums in ([2], [8], [2, 2], [4, 2], [2, 4], [2, 2, 2], [3, 2], [2, 3, 2]):
        L = len(nums)
        for shared in itertools.product([False, True], repeat=L):
            if all(shared):
                continue
            for layout in itertools.permutations(range(L)):
                cases.append((list(nums), list(shared), list(layout)))
    cases.append(([4, 2, 2], [True, False, False], [2, 0, 1]))      # micro(shared) x spmd x stage, stage outermost (build_pipeline)
    assert len(cases) >= 100
    for nums, shared, layout in cases:
        mgr = _C.CommDevManager()
        mgr.build(nums, shared, layout)
        world = mgr.total_devices()
        for dev in range(world):
            mesh = DeviceMesh(nums, shared, layout, rank=dev, world=world)
            assert mesh.total_devices == world, (nums, shared, layout)
            cc = mgr.coords(dev)
            pc = mesh.coords()
            for lvl in range(len(nums)):
                if shared[lvl]:
                    assert cc[lvl] == 0 and lvl not in pc, (nums, shared, layout, dev, lvl)
                    continue
                assert pc[lvl] == cc[lvl], (nums, shared, layout, dev, lvl, pc, cc)
                assert mesh.group_ranks(lvl) == list(mgr.group_of(dev, lvl).devices), (nums, shared, layout, dev, lvl)
                assert mesh.index_in_group(lvl) == mgr.rank_in_group(dev, lvl)
            ids = [cc[l] for l in range(len(nums))]
            assert mgr.global_device(ids) == dev == mesh.device_of({l: cc[l] for l in range(len(nums)) if not shared[l]})
        for lvl in range(len(nums)):
            if not shared[lvl]:
                assert sorted(map(tuple, DeviceMesh(nums, shared, layout, rank=0, world=world).all_groups(lvl))) == \
                    sorted(tuple(g.devices) for g in mgr.all_groups(lvl)), (nums, shared, layout, lvl)


def test_variable_store_fills_only_its_shard_bit_identically(monkeypatch):
    """Sharded variables are generated shard-only (C++ SliceRuns + counter-based Philox) and must equal, bit for bit, the
    slice of a full-tensor fill; and the full-size generator must not be touched for them (that is the point: the reference's
    multi-billion-parameter configs do not fit a per-rank full copy)."""
    import torch
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    from tepdist_b200.parallel import plan_spmd, plan_spmd_mesh
    from tepdist_b200.runtime.executor import VariableStore, shard_of
    from tepdist_b200.utils import init as init_mod
    g = build_gpt2_graph(CONFIGS["tiny"], batch=4)
    plans = [(plan_spmd(g, 2, "tp")[0], [{0: 0}, {0: 1}]),
             (plan_spmd_mesh(g, [2, 2], ["tp", "dp"])[0], [{0: 0, 1: 0}, {0: 1, 1: 0}, {0: 0, 1: 1}, {0: 1, 1: 1}])]
    for sharded, all_coords in plans:
        n_sharded = sum(1 for n in sharded.params() if n.attrs.get("shard_dims"))
        assert n_sharded > 4
        for coords in all_coords:
            full_calls = []
            real_fill = init_mod.init_tensor

            def spy(spec, shape, seed, name, shard=None):
                if shard is None and spec.get("kind", "constant") != "constant":
                    full_calls.append(name)
                return real_fill(spec, shape, seed, name, shard)
            monkeypatch.setattr("tepdist_b200.runtime.executor.init_tensor", spy)
            # the shard branch has a fallback that regenerates the full tensor: make sure it is NOT what ran
            full_sizes = []
            real_philox = _C.philox_fill
            monkeypatch.setattr(_C, "philox_fill", lambda kind, seed, off, n, *a: (full_sizes.append(n), real_philox(kind, seed, off, n, *a))[1])
            st = VariableStore(sharded, torch.device("cpu"), seed=5, coords=coords)
            monkeypatch.undo()
            assert not full_calls, full_calls[:3]
            whole = [int(np.prod(st.shape[n.id])) for n in sharded.params() if not n.attrs.get("shard_dims") and
                     n.attrs.get("init", {}).get("kind", "constant") != "constant"]
            assert sorted(full_sizes) == sorted(whole), "full-size Philox fills happened for sharded variables"
            for n in sharded.params():
                full = tuple(n.attrs.get("full_shape", st.shape[n.id]))
                oracle = shard_of(init_mod.init_tensor(n.attrs.get("init", {"kind": "constant", "value": 0.0}), full, 5, n.name),
                                  n.attrs, coords)
                assert torch.equal(st.master_view(n.id), oracle.reshape(st.shape[n.id])), (n.name, coords)


def test_einsum_lowering_to_batched_gemm_matches_torch_einsum():
    """ops.einsum brings any batch / M / N / K index pattern to ONE [batch, M, K] x [batch, K, N] GEMM call (either operand
    major, copies only when the memory order forces one): every GPT-MoE einsum (dispatch, expert FCs, combine) and the
    gradient einsums the autodiff derives from them must equal torch.einsum.  (CPU: the GEMM is its fp32 reference path.)"""
    import torch
    from tepdist_b200 import ops
    torch.manual_seed(0)
    G, S, E, C, M, H = 2, 16, 4, 8, 24, 32
    t = {"GSEC": torch.randn(G, S, E, C), "GSM": torch.randn(G, S, M), "EGCM": torch.randn(E, G, C, M), "EMH": torch.randn(E, M, H),
         "EGCH": torch.randn(E, G, C, H), "EHM": torch.randn(E, H, M)}
    eqs = ["GSEC,GSM->EGCM", "EGCM,EMH->EGCH", "EGCH,EHM->EGCM", "GSEC,EGCM->GSM",           # forward
           "EGCM,GSM->GSEC", "GSEC,EGCM->GSM", "EGCH,EMH->EGCM", "EGCM,EGCH->EMH",           # vjps w.r.t. each operand
           "EGCM,EHM->EGCH", "EGCH,EGCM->EHM", "GSM,EGCM->GSEC", "GSEC,GSM->EGCM"]
    for eq in eqs:
        ia, ib = eq.split("->")[0].split(",")
        got = ops.einsum(eq, t[ia], t[ib], _force=True)
        ref = torch.einsum(eq, t[ia], t[ib])
        # (the GEMM entry point rounds its result to bf16 like the kernel does: compare in relative Frobenius norm)
        assert got.shape == ref.shape and float((got.float() - ref).norm() / ref.norm()) < 1e-2, eq
    # patterns the lowering does not cover fall back to torch.einsum
    x = torch.randn(4, 8)
    assert torch.allclose(ops.einsum("ab,ab->a", x, x, _force=True), (x * x).sum(1), atol=1e-5)


def test_moe_route_table_path_equals_the_dense_einsums():
    """GPT-MoE's dispatch / combine einsums (and the four gradient einsums around them) run as route-table row gathers when their
    mask comes from moe_dispatch_mask.  Same losses and same updated weights as the dense-einsum execution, step by step, on
    the MoE FFN graph and on a tiny GPT-MoE -- forward, backward and token dropping (capacity smaller than the demand) included."""
    import torch
    from tepdist_b200.models.gpt_moe import MoEConfig, build_gpt_moe_graph, build_moe_ffn_graph
    from tepdist_b200.runtime import executor as ex_mod
    from tepdist_b200.runtime.executor import Executor

    def run(g, feeds, sparse):
        ex_mod.MOE_SPARSE = sparse
        try:
            ex = Executor(g, torch.device("cpu"), seed=0, use_cuda_graph=False)
            n_sparse = len(ex._moe_einsum)
            losses = [float(ex.step(feeds)[0]) for _ in range(3)]
            return losses, ex.store.state_dict(), n_sparse
        finally:
            ex_mod.MOE_SPARSE = True

    torch.manual_seed(0)
    g = build_moe_ffn_graph(groups=4, tokens_per_group=32, model=32, hidden=64, experts=4, capacity=8)     # capacity 8 < 32 * 2 / 4: drops
    feeds = {"x": torch.randn(4, 32, 32), "t": torch.randn(4, 32, 32)}
    ld, sd, nd = run(g, feeds, False)
    ls, ss, ns = run(g, feeds, True)
    assert nd == 0 and ns == 5, (nd, ns)          # dispatch, combine + their gradient einsums (x is an input here: no d x)
    for a, b in zip(ls, ld):
        assert abs(a - b) <= 1e-5 * max(1.0, abs(b)), (ls, ld)
    for k in sd:
        assert torch.allclose(ss[k].float(), sd[k].float(), atol=1e-5, rtol=1e-4), k
    cfg = MoEConfig(n_layer=2, hidden=64, ffn=128, n_head=2, experts=4, capacity=16, groups=2, seq=64, batch=2, vocab=500)
    g2 = build_gpt_moe_graph(cfg)
    tok = torch.randint(0, cfg.vocab, (cfg.batch, cfg.seq), dtype=torch.int32)
    f2 = {"tokens": tok, "labels": torch.roll(tok, -1, 1)}
    ld, _, _ = run(g2, f2, False)
    ls, _, ns = run(g2, f2, True)
    assert ns == 6 and all(abs(a - b) <= 1e-5 * max(1.0, abs(b)) for a, b in zip(ls, ld)), (ls, ld)


def test_flat_bucket_policy_is_graded_aligned_and_covers_the_buffer():
    """B7 (storage-order variant, executed by the runtime): bucket boundaries over the flat gradient buffer start small and double
    up to the cap, only ever fall on variable starts that are multiples of the chunk granularity, and tile [0, end) exactly."""
    offs, o = [], 0
    sizes = [1 << 20] * 12 + [3 << 20] * 30 + [50 << 20, 1 << 18, 1 << 18]
    for sz in sizes:
        offs.append(o)
        o += sz
    end = o
    gran = 8 * 128
    b = list(_C.plan_flat_buckets(offs, end, gran, 4 << 20, 48 << 20))
    assert b[0] == 0 and b[-1] == end and b == sorted(set(b))
    assert all(x in offs and x % gran == 0 for x in b[1:-1])
    widths = [b[i + 1] - b[i] for i in range(len(b) - 1)]
    assert widths[0] >= 4 << 20 and widths[0] < widths[2]             # graded: the first buckets are the small ones
    assert all(w >= min(48 << 20, (4 << 20) << min(i, 16)) or i == len(widths) - 1 for i, w in enumerate(widths))
    # the same policy the executor used to compute in Python
    ref = [0]
    for off in offs[1:]:
        want = min(48 << 20, (4 << 20) << min(len(ref) - 1, 16))
        if off - ref[-1] >= want and off % gran == 0:
            ref.append(off)
    ref.append(end)
    assert b == ref


def test_pipeline_slot_assignment_follows_the_release_plan():
    """CUDA-graph stage bodies: slots are taken at a micro-batch's first task (a hoisted forward Recv counts) and returned where the
    scheduler releases the micro-batch -- never more slots than micro-batches in flight, never a slot shared by two live ones."""
    import types
    from tepdist_b200.models.gpt2 import CONFIGS, build_gpt2_graph
    from tepdist_b200.parallel import plan_pipeline
    from tepdist_b200.runtime.pipeline import StageWorker
    g = build_gpt2_graph(CONFIGS["tiny"], batch=8)
    _, info, tasks = plan_pipeline(g, 4, 4, 8)
    for dev, lst in tasks.items():
        w = types.SimpleNamespace()
        StageWorker.plan_slots(w, lst)
        assert set(w.slot_of) == set(range(8)) and 1 <= w.num_slots <= 4 + 1, (dev, w.slot_of)
        live = {}
        for t in lst:
            m = t["micro"]
            if m is not None and m >= 0 and not t["backward"] and t["type"] in ("Recv", "Compute", "Input") and m not in live.values():
                assert w.slot_of[m] not in live, (dev, m, live)
                live[w.slot_of[m]] = m
            for dead in t.get("release", ()):
                live.pop(w.slot_of[dead], None)


def test_ring_attention_block_schedule_equals_full_attention():
    """Every virtual rank's ring schedule (causal diagonal block, unmasked earlier blocks, log-sum-exp merge, backward blocks fed
    the global log-sum-exp, fp32 dK / dV accumulation) reproduces full-sequence attention and its gradients (fp32, CPU branch of
    the same functions the GPU test drives through the kernels)."""
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import kernel_checks as kc
    errs = kc.check_ring_blocks("cpu")
    assert errs and max(errs.values()) < 1e-5, errs
