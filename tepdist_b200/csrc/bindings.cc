// pybind11 surface of the C++ core (module tepdist_b200._C).
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include "cost.h"
#include "ir.h"
#include "pbqp.h"
#include "rules.h"
#include "spmd_planner.h"

namespace py = pybind11;
using namespace tepdist;

void BindPlanner(py::module_& m);   // planner_bindings.cc (auto_parallel, stage, syncfree, evaluator, transforms)
void BindRuntime(py::module_& m);   // runtime_bindings.cc (dev mesh, task graph, scheduler, slicing, philox)

static Attr ToAttr(const py::handle& h) {
  if (py::isinstance<py::bool_>(h)) return h.cast<bool>();
  if (py::isinstance<py::int_>(h)) return (int64_t)h.cast<long long>();
  if (py::isinstance<py::float_>(h)) return h.cast<double>();
  if (py::isinstance<py::str>(h)) return h.cast<std::string>();
  if (py::isinstance<py::list>(h) || py::isinstance<py::tuple>(h)) {
    std::vector<int64_t> v;
    for (auto x : h) {
      if (!py::isinstance<py::int_>(x)) return std::string(py::str(h));
      v.push_back((int64_t)x.cast<long long>());
    }
    return v;
  }
  return std::string(py::str(h));
}
static py::object FromAttr(const Attr& a) {
  if (auto p = std::get_if<int64_t>(&a)) return py::int_(*p);
  if (auto p = std::get_if<double>(&a)) return py::float_(*p);
  if (auto p = std::get_if<std::string>(&a)) return py::str(*p);
  if (auto p = std::get_if<bool>(&a)) return py::bool_(*p);
  if (auto p = std::get_if<std::vector<int64_t>>(&a)) return py::cast(*p);
  return py::none();
}

PYBIND11_MODULE(_C, m) {
  m.doc() = "tepdist_b200 native core: planner IR, sharding rules, SPMD/pipeline planners, transforms, runtime";

  py::class_<DimStrategy>(m, "DimStrategy")
      .def(py::init<>())
      .def_static("glue", &DimStrategy::Glue)
      .def_static("split", &DimStrategy::Split, py::arg("dim"), py::arg("num"), py::arg("stride") = 0)
      .def_static("partial_", &DimStrategy::Partial, py::arg("num"), py::arg("kind") = 0)
      .def_readwrite("dim", &DimStrategy::dim)
      .def_readwrite("num", &DimStrategy::num)
      .def_readwrite("stride", &DimStrategy::stride)
      .def_readwrite("partial", &DimStrategy::partial)
      .def_readwrite("reduce_kind", &DimStrategy::reduce_kind)
      .def("is_glue", &DimStrategy::is_glue)
      .def("is_split", &DimStrategy::is_split)
      .def("__eq__", [](const DimStrategy& a, const DimStrategy& b) { return a == b; })
      .def("__repr__", &DimStrategy::str)
      .def("apply_to_shape", [](const DimStrategy& s, std::vector<int64_t> from, std::vector<int64_t> to) {
        return s.ApplyToShape(TensorType{from, "f32"}, TensorType{to, "f32"});
      })
      .def("stride_on_elements", [](const DimStrategy& s, std::vector<int64_t> shape) {
        return s.StrideOnElements(TensorType{shape, "f32"});
      });

  py::class_<DistSpec>(m, "DistSpec")
      .def(py::init<>())
      .def_readwrite("levels", &DistSpec::levels)
      .def_readwrite("stage", &DistSpec::stage)
      .def("__repr__", &DistSpec::str);

  py::class_<Candidate>(m, "Candidate")
      .def_readonly("ins", &Candidate::ins)
      .def_readonly("outs", &Candidate::outs)
      .def_readonly("node_cost", &Candidate::node_cost)
      .def_readonly("tag", &Candidate::tag)
      .def("__repr__", [](const Candidate& c) {
        std::string s = "[" + c.tag + "] (";
        for (size_t i = 0; i < c.ins.size(); ++i) s += (i ? "," : "") + c.ins[i].str();
        s += ")->(";
        for (size_t i = 0; i < c.outs.size(); ++i) s += (i ? "," : "") + c.outs[i].str();
        return s + ")";
      });

  py::class_<Graph>(m, "Graph")
      .def(py::init<>())
      .def_readwrite("name", &Graph::name)
      .def_readwrite("split_nums", &Graph::split_nums)
      .def_readwrite("share_dev", &Graph::share_dev)
      .def_readwrite("placement_layout", &Graph::placement_layout)
      .def_readwrite("stage_split_ordinal", &Graph::stage_split_ordinal)
      .def_readwrite("meta", &Graph::meta)
      .def("add_node",
           [](Graph& g, const std::string& op, const std::vector<std::pair<int, int>>& inputs,
              const std::vector<std::pair<std::vector<int64_t>, std::string>>& outs, const py::dict& attrs,
              const std::string& name, int group, bool backward) {
             std::vector<ValueRef> in;
             for (auto& p : inputs) in.push_back({p.first, p.second});
             std::vector<TensorType> ot;
             for (auto& o : outs) ot.push_back({o.first, o.second});
             std::map<std::string, Attr> at;
             for (auto kv : attrs) {
               if (py::isinstance<py::dict>(kv.second)) continue;  // nested dicts (init specs) stay client-side
               at[kv.first.cast<std::string>()] = ToAttr(kv.second);
             }
             return g.AddNode(op, in, ot, at, name, group, backward);
           })
      .def("set_outputs", [](Graph& g, const std::vector<std::pair<int, int>>& o) {
        g.outputs.clear();
        for (auto& p : o) g.outputs.push_back({p.first, p.second});
      })
      .def("set_update", [](Graph& g, int var, int node, int idx) { g.updates[var] = {node, idx}; })
      .def("num_nodes", [](const Graph& g) { return g.nodes.size(); })
      .def("node_op", [](const Graph& g, int i) { return g.nodes[i].op; })
      .def("node_name", [](const Graph& g, int i) { return g.nodes[i].name; })
      .def("node_stage", [](const Graph& g, int i) { return g.nodes[i].stage; })
      .def("set_node_stage", [](Graph& g, int i, int s) { g.nodes[i].stage = s; })
      .def("node_group", [](const Graph& g, int i) { return g.nodes[i].group; })
      .def("node_backward", [](const Graph& g, int i) { return g.nodes[i].backward; })
      .def("node_inputs", [](const Graph& g, int i) {
        std::vector<std::pair<int, int>> r;
        for (auto& v : g.nodes[i].inputs) r.push_back({v.node, v.idx});
        return r;
      })
      .def("node_outputs", [](const Graph& g, int i) {
        std::vector<std::pair<std::vector<int64_t>, std::string>> r;
        for (auto& t : g.nodes[i].outputs) r.push_back({t.dims, t.dtype});
        return r;
      })
      .def("node_attrs", [](const Graph& g, int i) {
        py::dict d;
        for (auto& kv : g.nodes[i].attrs) d[py::str(kv.first)] = FromAttr(kv.second);
        return d;
      })
      .def("set_node_attr", [](Graph& g, int i, const std::string& k, py::object v) { g.nodes[i].attrs[k] = ToAttr(v); })
      .def("erase_node_attr", [](Graph& g, int i, const std::string& k) { g.nodes[i].attrs.erase(k); })
      .def("node_dist", [](const Graph& g, int i) { return g.nodes[i].dist; })
      .def("outputs", [](const Graph& g) {
        std::vector<std::pair<int, int>> r;
        for (auto& v : g.outputs) r.push_back({v.node, v.idx});
        return r;
      })
      .def("updates", [](const Graph& g) {
        std::vector<std::tuple<int, int, int>> r;
        for (auto& kv : g.updates) r.push_back({kv.first, kv.second.node, kv.second.idx});
        return r;
      })
      .def("node_flops", [](const Graph& g, int i) { return NodeFlops(g, g.nodes[i]); })
      .def("dump", &Graph::Dump, py::arg("with_dist") = true)
      .def("clone", [](const Graph& g) { return Graph(g); });

  m.def("enumerate_candidates", [](const Graph& g, int node, int num, bool allow_glue) {
    RuleOptions o;
    o.allow_glue_compute_intensive = allow_glue;
    return EnumerateCandidates(g, g.nodes[node], num, o);
  }, py::arg("graph"), py::arg("node"), py::arg("num"), py::arg("allow_glue") = false);
  m.def("forward_infer", [](const Graph& g, int node, int num, int operand, const DimStrategy& s) {
    return ForwardInfer(g, g.nodes[node], num, operand, s);
  });
  m.def("back_infer", [](const Graph& g, int node, int num, int out, const DimStrategy& s) {
    return BackInfer(g, g.nodes[node], num, out, s);
  });
  m.def("reshard_kind", [](const DimStrategy& a, const DimStrategy& b) { return std::string(ReshardName(ClassifyReshard(a, b))); });
  m.def("reshard_cost", &ReshardCost, py::arg("from_"), py::arg("to"), py::arg("bytes"), py::arg("n"), py::arg("cost_factor") = 1.0);
  m.def("find_critical_nodes", &FindCriticalNodes, py::arg("graph"), py::arg("min_segment_flops_frac") = 0.0);
  m.def("find_critical_nodes_by_main_path", &FindCriticalNodesByMainPath);

  py::class_<HwProfile>(m, "HwProfile")
      .def(py::init<>())
      .def_static("h100", &HwProfile::H100)
      .def_static("reference_v100", &HwProfile::ReferenceV100)
      .def_readwrite("name", &HwProfile::name)
      .def_readwrite("flops", &HwProfile::flops)
      .def_readwrite("hbm_bw", &HwProfile::hbm_bw)
      .def_readwrite("link_bw", &HwProfile::link_bw)
      .def_readwrite("inter_node_bw", &HwProfile::inter_node_bw)
      .def_readwrite("coll_latency", &HwProfile::coll_latency)
      .def_readwrite("small_batch_half_rows", &HwProfile::small_batch_half_rows)
      .def("exposed_comm_fraction", &HwProfile::ExposedCommFraction)
      .def("compute_slowdown", &HwProfile::ComputeSlowdown)
      .def_readwrite("mem_bytes", &HwProfile::mem_bytes)
      .def_readwrite("var_mem_limit", &HwProfile::var_mem_limit);

  py::class_<SpmdOptions>(m, "SpmdOptions")
      .def(py::init<>())
      .def_readwrite("num", &SpmdOptions::num)
      .def_readwrite("var_mem_limit", &SpmdOptions::var_mem_limit)
      .def_readwrite("mem_split_min_rank", &SpmdOptions::mem_split_min_rank)
      .def_readwrite("context_parallel", &SpmdOptions::context_parallel)
      .def_readwrite("sequence_parallel", &SpmdOptions::sequence_parallel)
      .def_readwrite("share_relayout_cost", &SpmdOptions::share_relayout_cost)
      .def_readwrite("num_threads", &SpmdOptions::num_threads)
      .def_readwrite("collective_latency_bytes", &SpmdOptions::collective_latency_bytes)
      .def_readwrite("min_segment_flops_frac", &SpmdOptions::min_segment_flops_frac)
      .def_readwrite("cost_factor", &SpmdOptions::cost_factor)
      .def_readwrite("opt_level", &SpmdOptions::opt_level)
      .def_readwrite("ignore_annotation", &SpmdOptions::ignore_annotation)
      .def_readwrite("aux_affinity", &SpmdOptions::aux_affinity)
      .def_readwrite("forward_sub_graph_num", &SpmdOptions::forward_sub_graph_num)
      .def_readwrite("ilp_time_limit_s", &SpmdOptions::ilp_time_limit_s)
      .def_readwrite("replicate_penalty", &SpmdOptions::replicate_penalty)
      .def_readwrite("memory_weight", &SpmdOptions::memory_weight)
      .def_readwrite("hw", &SpmdOptions::hw);
  py::class_<SpmdStats>(m, "SpmdStats")
      .def_readonly("comm_bytes", &SpmdStats::comm_bytes)
      .def_readonly("solve_seconds", &SpmdStats::solve_seconds)
      .def_readonly("num_subgraphs", &SpmdStats::num_subgraphs)
      .def_readonly("distinct_subgraphs", &SpmdStats::distinct_subgraphs)
      .def_readonly("core_nodes_max", &SpmdStats::core_nodes_max)
      .def_readonly("optimal", &SpmdStats::optimal)
      .def_readonly("var_bytes_per_device", &SpmdStats::var_bytes_per_device)
      .def_readonly("forced_weight_splits", &SpmdStats::forced_weight_splits)
      .def_readonly("infeasible_subgraphs", &SpmdStats::infeasible_subgraphs)
      .def_readonly("threads_used", &SpmdStats::threads_used)
      .def_readonly("ignored_annotations", &SpmdStats::ignored_annotations)
      .def_readonly("collectives", &SpmdStats::collectives);
  py::class_<SpmdPlan>(m, "SpmdPlan")
      .def_readonly("choice", &SpmdPlan::choice)
      .def_readonly("stats", &SpmdPlan::stats);
  m.def("plan_spmd_level", [](Graph& g, const SpmdOptions& o) { return PlanSpmdLevel(&g, o); });
  m.def("plan_spmd_by_rules", [](Graph& g, const SpmdOptions& o) { return PlanSpmdByRules(&g, o); });
  m.def("dump_strategies", &DumpStrategies);
  m.def("verify_infer", [](const Graph& g, int num) { return VerifyInfer(g, num); });
  m.def("unknown_ops", [](bool clear) { return UnknownOps(clear); }, py::arg("clear") = true);

  py::class_<PBQP>(m, "PBQP")
      .def(py::init<>())
      .def("add_node", &PBQP::AddNode)
      .def("add_edge", &PBQP::AddEdge)
      .def("evaluate", &PBQP::Evaluate)
      .def("solve", [](PBQP& q, double tl) {
        auto r = q.Solve(tl);
        py::dict d;
        d["choice"] = r.choice; d["cost"] = r.cost; d["optimal"] = r.optimal;
        d["core_nodes"] = r.core_nodes; d["reduced_nodes"] = r.reduced_nodes; d["bb_nodes"] = r.bb_nodes;
        return d;
      }, py::arg("time_limit_s") = 30.0);

  BindPlanner(m);
  BindRuntime(m);
}
