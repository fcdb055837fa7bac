#include "auto_parallel.h"

#include <algorithm>
#include <cmath>
#include <set>
#include <sstream>

#include "rules.h"

namespace tepdist {

// =============================================================================== sync-free analysis
SyncFreeResult SyncFreeAnalysis(const Graph& g, int num_micro) {
  SyncFreeResult best;
  best.num_micro = num_micro;
  if (num_micro <= 1) { best.ok = true; best.reason = "single micro-batch"; return best; }
  std::vector<int> inputs;
  int max_rank = 0;
  for (auto& n : g.nodes)
    if (n.op == "input" && n.outputs[0].rank() > 0) { inputs.push_back(n.id); max_rank = std::max(max_rank, n.outputs[0].rank()); }
  if (inputs.empty()) { best.reason = "no sample inputs"; return best; }
  SpmdOptions so;
  so.num = num_micro;
  so.ignore_annotation = false;
  for (int d = 0; d < max_rank; ++d) {
    // proposal: every sample input that has dim d (divisible) is split on it
    Graph c = g;
    std::map<int, int> dims;
    for (int id : inputs) {
      const TensorType& t = c.nodes[id].outputs[0];
      if (d < t.rank() && t.dims[d] % num_micro == 0 && t.dims[d] >= num_micro) {
        c.nodes[id].attrs["shard_dim"] = (int64_t)d;
        dims[id] = d;
      } else {
        c.nodes[id].attrs.erase("shard_dim");
      }
    }
    for (auto& n : c.nodes)
      if (n.op != "input") n.attrs.erase("shard_dim");
    if (dims.empty()) continue;
    SpmdPlan plan = PlanSpmdByRules(&c, so);
    int split = 0;
    std::vector<ValueRef> sync;
    for (auto& n : c.nodes)
      for (int o = 0; o < (int)n.outputs.size(); ++o) {
        const DimStrategy& s = plan.choice[n.id].outs[o];
        if (s.is_split()) ++split;
        if (s.partial) sync.push_back({n.id, o});
      }
    // validation (reference Validate, :182-226): the partial points must form a clean cut — nothing computed from
    // a reduced value may flow back into per-micro-batch (split) computation
    std::set<int> after;  // nodes that consume reduced values (transitively)
    bool clean = true;
    for (auto& n : c.nodes) {
      bool aft = false;
      for (int k = 0; k < (int)n.inputs.size(); ++k) {
        const ValueRef& v = n.inputs[k];
        const DimStrategy& ps = plan.choice[v.node].outs[v.idx];
        if (after.count(v.node) || (ps.partial && !plan.choice[n.id].ins[k].partial)) aft = true;
      }
      if (aft) {
        after.insert(n.id);
        for (auto& s : plan.choice[n.id].outs)
          if (s.is_split() || s.partial) clean = false;
      }
    }
    // a sequence split that runs through attention is NOT sync-free: the "seq" candidate communicates inside the node (K / V ring)
    for (auto& n : c.nodes)
      if ((n.op == "attention" || n.op == "attention_bwd") && plan.choice[n.id].tag == "seq") clean = false;
    if (!clean) continue;
    if (split > best.num_split_values) {
      best.ok = true;
      best.num_split_values = split;
      best.input_split_dim = dims;
      best.sync_points = sync;
      best.plan = plan;
      best.reason = "split dim " + std::to_string(d);
    }
  }
  if (!best.ok) best.reason = "no valid micro-batch split";
  return best;
}

// =============================================================================== decomposition
std::string Decomposition::Dump() const {
  std::ostringstream o;
  for (size_t i = 0; i < ctx.size(); ++i) {
    const DefContext& c = ctx[i];
    o << "[" << i << "] " << c.name << " kind=" << c.kind << " stage=" << c.stage << " nodes=" << c.nodes.size()
      << " in=" << c.inputs.size() << " out=" << c.outputs.size() << " gflops=" << c.gflops
      << (c.per_micro_batch ? " per-micro" : "") << " children=[";
    for (size_t k = 0; k < c.children.size(); ++k) o << (k ? "," : "") << c.children[k];
    o << "]\n";
  }
  return o.str();
}

namespace {
void FillIo(const Graph& g, DefContext* c) {
  std::set<int> mine(c->nodes.begin(), c->nodes.end());
  std::set<ValueRef> ins, outs;
  std::set<ValueRef> fetch(g.outputs.begin(), g.outputs.end());
  for (int id : c->nodes) {
    const Node& n = g.nodes[id];
    c->gflops += NodeFlops(g, n) / 1e9;
    for (auto& v : n.inputs)
      if (!mine.count(v.node)) ins.insert(v);
    for (int o = 0; o < (int)n.outputs.size(); ++o) {
      ValueRef v{id, o};
      bool ext = fetch.count(v) > 0;
      for (auto& u : g.users(v))
        if (!mine.count(u.node)) ext = true;
      for (auto& kv : g.updates)
        if (kv.second == v) ext = true;
      if (ext) outs.insert(v);
    }
  }
  c->inputs.assign(ins.begin(), ins.end());
  c->outputs.assign(outs.begin(), outs.end());
  for (auto& v : c->inputs) c->in_bytes += (double)g.type(v).bytes();
  for (auto& v : c->outputs) c->out_bytes += (double)g.type(v).bytes();
}
}  // namespace

Decomposition SyncFreeDecompose(const Graph& g, int micro_level) {
  Decomposition d;
  // sync points: collectives on the micro-batch level; when no such level exists (single micro-batch) the cut is
  // at the gradient operands of the apply nodes (so CG/AG still exist and GA degenerates to a move)
  std::set<int> sync_nodes;
  for (auto& n : g.nodes)
    if ((n.op == "all_reduce" || n.op == "reduce_scatter") && n.attr_i("level", -1) == micro_level) sync_nodes.insert(n.id);
  std::set<int> ag;  // everything downstream of a sync point or an apply node
  for (auto& n : g.nodes) {
    bool down = n.op.rfind("apply_", 0) == 0;
    for (auto& v : n.inputs)
      if (ag.count(v.node) || sync_nodes.count(v.node)) down = true;
    if (down && !sync_nodes.count(n.id)) ag.insert(n.id);
  }
  if (sync_nodes.empty())
    for (auto& n : g.nodes)
      if (n.op.rfind("apply_", 0) == 0) d.accumulators.push_back(n.inputs[1]);
  for (int id : sync_nodes) d.accumulators.push_back(g.nodes[id].inputs[0]);

  DefContext entry, cg, gainit, ga, agc;
  entry.name = "ENTRY"; entry.kind = "entry";
  cg.name = "CG"; cg.kind = "cg"; cg.per_micro_batch = true;
  gainit.name = "GAINIT"; gainit.kind = "gainit";
  ga.name = "GA"; ga.kind = "ga"; ga.per_micro_batch = true;
  agc.name = "AG"; agc.kind = "ag";
  for (auto& n : g.nodes) {
    entry.nodes.push_back(n.id);
    if (IsVariable(n.op)) continue;  // variables are entry arguments shared by CG and AG
    if (sync_nodes.count(n.id)) ga.nodes.push_back(n.id);
    else if (ag.count(n.id)) agc.nodes.push_back(n.id);
    else cg.nodes.push_back(n.id);
  }
  FillIo(g, &cg);
  FillIo(g, &ga);
  FillIo(g, &agc);
  gainit.outputs = d.accumulators;
  for (auto& v : d.accumulators) gainit.out_bytes += (double)g.type(v).bytes();
  entry.children = {1, 2, 3, 4};
  d.ctx = {entry, cg, gainit, ga, agc};
  // provenance of every input of GA / AG
  auto owner = [&](int node) {
    if (std::binary_search(d.ctx[1].nodes.begin(), d.ctx[1].nodes.end(), node)) return 1;
    if (std::binary_search(d.ctx[3].nodes.begin(), d.ctx[3].nodes.end(), node)) return 3;
    if (std::binary_search(d.ctx[4].nodes.begin(), d.ctx[4].nodes.end(), node)) return 4;
    return -1;
  };
  for (int ci : {1, 3, 4})
    for (int i = 0; i < (int)d.ctx[ci].inputs.size(); ++i) d.ctx[ci].input_def[i] = owner(d.ctx[ci].inputs[i].node);
  return d;
}

std::vector<StageTransfer> StageDecompose(const Graph& g, int num_stages, Decomposition* d) {
  std::vector<StageTransfer> xfers;
  if (num_stages <= 1) return xfers;
  const int cg_idx = 1, ag_idx = 4;
  std::vector<int> child_f(num_stages), child_b(num_stages), child_a(num_stages);
  auto make = [&](const std::string& nm, const std::string& kind, int s, bool per_micro, int parent) {
    DefContext c;
    c.name = nm; c.kind = kind; c.stage = s; c.per_micro_batch = per_micro;
    d->ctx.push_back(c);
    int idx = (int)d->ctx.size() - 1;
    d->ctx[parent].children.push_back(idx);
    return idx;
  };
  for (int s = 0; s < num_stages; ++s) {
    child_f[s] = make("CG_SLICE_" + std::to_string(s) + "_F", "stage_fwd", s, true, cg_idx);
    child_b[s] = make("CG_SLICE_" + std::to_string(s) + "_B", "stage_bwd", s, true, cg_idx);
    child_a[s] = make("AG_SLICE_" + std::to_string(s), "stage_ag", s, false, ag_idx);
  }
  for (int id : d->ctx[cg_idx].nodes) {
    const Node& n = g.nodes[id];
    int s = std::min(std::max(n.stage, 0), num_stages - 1);
    d->ctx[n.backward ? child_b[s] : child_f[s]].nodes.push_back(id);
  }
  for (int id : d->ctx[ag_idx].nodes) {
    const Node& n = g.nodes[id];
    int s = std::min(std::max(n.stage, 0), num_stages - 1);
    d->ctx[child_a[s]].nodes.push_back(id);
  }
  for (int s = 0; s < num_stages; ++s) {
    FillIo(g, &d->ctx[child_f[s]]);
    FillIo(g, &d->ctx[child_b[s]]);
    FillIo(g, &d->ctx[child_a[s]]);
  }
  // cross-stage transfer optimisation: a value consumed k stages away hops through every intermediate stage
  std::set<std::tuple<int, int, int, int>> seen;  // (value node, idx, from, to)
  for (auto& n : g.nodes) {
    if (IsVariable(n.op)) continue;
    for (auto& v : n.inputs) {
      const Node& p = g.nodes[v.node];
      if (IsVariable(p.op) || p.op == "constant") continue;
      int a = p.stage, b = n.stage;
      if (a < 0 || b < 0 || a == b) continue;
      const int step = b > a ? 1 : -1;
      for (int s = a; s != b; s += step)
        if (seen.insert({v.node, v.idx, s, s + step}).second)
          xfers.push_back({v, s, s + step, step < 0, (double)g.type(v).bytes()});
    }
  }
  return xfers;
}

// =============================================================================== evaluator
std::string EvalResult::str() const {
  std::ostringstream o;
  o << "duration=" << total_duration * 1e3 << "ms compute=" << compute_time * 1e3 << "ms comm=" << comm_time * 1e3
    << "ms p2p=" << p2p_time * 1e3 << "ms gpu_eff=" << gpu_efficiency << " coll_ratio=" << coll_ratio
    << " bubble=" << bubble_ratio << " mem/dev=" << mem_bytes_per_device / 1e9 << "GB" << (feasible ? "" : " INFEASIBLE");
  return o.str();
}

EvalResult Evaluate(const EvalInput& in, const HwProfile& hw) {
  EvalResult r;
  const int S = std::max(1, in.num_stages), M = std::max(1, in.num_micro), n = std::max(1, in.spmd);
  // per-stage, per-micro-batch forward / backward compute (backward = 2x forward)
  std::vector<double> f(S), b(S);
  double total_flops = 0;
  for (int s = 0; s < S; ++s) {
    double fl = s < (int)in.stage_flops.size() ? in.stage_flops[s] : 0.0;
    total_flops += fl;
    const double t = fl / n / M / hw.flops * hw.ComputeSlowdown(in.rows_per_micro);
    f[s] = t / 3.0;
    b[s] = t * 2.0 / 3.0;
  }
  const double comm_mb = in.spmd_comm_bytes > 0 ? CollectiveSeconds(hw, in.spmd_comm_bytes / M) * in.exposed_comm_fraction : 0.0;
  const double xfer = (S > 1) ? CollectiveSeconds(hw, in.cut_bytes / std::max(1, S - 1) / 2.0 / n) : 0.0;  // one boundary, one direction
  // forward wave then backward wave (reference evaluator.cc:131-267): fill + steady state + drain
  double fill = 0, drain = 0, steady = 0;
  for (int s = 0; s < S; ++s) {
    fill += f[s] + (s + 1 < S ? xfer : 0.0);
    drain += b[s] + (s > 0 ? xfer : 0.0);
    steady = std::max(steady, f[s] + b[s] + comm_mb / S);
  }
  r.total_duration = fill + drain + (M - 1) * steady + comm_mb / S;
  r.compute_time = total_flops / (S * n) / hw.flops * hw.ComputeSlowdown(in.rows_per_micro);
  r.comm_time = comm_mb * M / S;
  r.p2p_time = S > 1 ? 2.0 * (S - 1) * xfer : 0.0;
  r.gpu_efficiency = r.compute_time / r.total_duration;
  r.coll_ratio = r.comm_time / r.total_duration;
  r.bubble_ratio = std::max(0.0, 1.0 - (r.compute_time + r.comm_time) / r.total_duration);
  // memory: variables sharded by the SPMD plan only if it chose to; conservatively whole / stages, plus
  // activations of the in-flight micro-batches (1F1B keeps <= S in flight)
  r.mem_bytes_per_device = in.var_bytes / S + in.act_bytes / S / n * std::min(M, S) / std::max(1, M);
  r.feasible = r.mem_bytes_per_device < hw.mem_bytes;
  return r;
}

// =============================================================================== orchestrator
std::string DeviceSplitProposal::str() const {
  std::ostringstream o;
  o << "stages=" << stages << " spmd=" << spmd << " micro=" << micro;
  return o.str();
}

std::vector<DeviceSplitProposal> GenerateSplitProposals(int num_devices, int64_t batch, bool allow_pipeline) {
  std::vector<DeviceSplitProposal> out;
  for (int s = 1; s <= num_devices; s *= 2) {
    if (num_devices % s) continue;
    if (s > 1 && !allow_pipeline) break;
    DeviceSplitProposal p;
    p.stages = s;
    p.spmd = num_devices / s;
    if (s == 1) {
      p.micro = 1;
      out.push_back(p);
      continue;
    }
    // pipeline needs micro-batching: counts from max(2S-1, 2) upward that divide the batch (reference
    // sync_free_splitting_analysis.cc:63-149); also try twice that for a smaller bubble
    int found = 0;
    for (int64_t m = std::max(2 * s - 1, 2); m <= batch && found < 2; ++m)
      if (batch % m == 0 && (batch / m) % std::max(1, p.spmd) == 0) { p.micro = (int)m; out.push_back(p); ++found; m = 2 * m - 1; }
    if (!found)
      for (int64_t m = s; m <= batch && !found; ++m)
        if (batch % m == 0) { p.micro = (int)m; out.push_back(p); ++found; }
  }
  return out;
}

namespace {
int64_t BatchOf(const Graph& g) {
  for (auto& n : g.nodes)
    if (n.op == "input" && n.outputs[0].rank() > 0) return n.outputs[0].dims[0];
  return 1;
}
double VarBytes(const Graph& g) {
  double b = 0;
  bool adam = false;
  for (auto& n : g.nodes) adam |= n.op == "apply_adamw" || n.op == "apply_lamb";
  for (auto& n : g.nodes)
    if (n.op == "parameter") b += (double)n.outputs[0].numel() * (adam ? 18.0 : 10.0);
  return b;
}
double ActBytes(const Graph& g) {
  double b = 0;
  for (auto& n : g.nodes)
    if (!n.backward && !IsSource(n.op) && n.op.rfind("apply_", 0) != 0)
      for (auto& t : n.outputs) b += (double)t.bytes();
  return b;
}
}  // namespace

ParallelPlan AutoParallelRun(const Graph& g, const AutoParallelOptions& opt) {
  ParallelPlan best;
  std::ostringstream log;
  std::vector<DeviceSplitProposal> props;
  const int64_t batch = BatchOf(g);
  if (opt.mode == "config") {
    DeviceSplitProposal p;
    p.stages = std::max(1, opt.num_stages);
    p.spmd = std::max(1, opt.num_devices / p.stages);
    p.micro = std::max(1, opt.num_micro_batches);
    props.push_back(p);
  } else if (opt.mode == "rule") {
    DeviceSplitProposal p;
    p.spmd = opt.num_devices;
    props.push_back(p);
  } else {
    props = GenerateSplitProposals(opt.num_devices, batch, opt.allow_pipeline);
  }
  bool have = false;
  for (auto& p : props) {
    ParallelPlan cand;
    cand.proposal = p;
    Graph cur = g;
    cur.split_nums.clear();
    cur.share_dev.clear();
    int level = 0;
    bool ok = true;
    // 1. micro-batch (sync-free) level: time-multiplexed on the same devices
    if (p.micro > 1) {
      cand.sync_free = SyncFreeAnalysis(cur, p.micro);
      if (!cand.sync_free.ok) { log << "[skip] " << p.str() << ": " << cand.sync_free.reason << "\n"; continue; }
      cur.record_split(p.micro, true);
      Graph t = SpmdTransform(cur, cand.sync_free.plan, level, p.micro);
      cur = std::move(t);
      ++level;
    }
    // 2. SPMD level
    double spmd_comm = 0;
    if (p.spmd > 1) {
      SpmdOptions so = opt.spmd;
      so.num = p.spmd;
      const bool rule = opt.mode == "rule" || opt.spmd_rule_mode;
      if (rule) {
        so.ignore_annotation = false;
        for (auto& n : cur.nodes)   // sample inputs are split on their batch dim unless the user annotated otherwise
          if (n.op == "input" && !n.has("shard_dim") && n.outputs[0].rank() > 0) n.attrs["shard_dim"] = (int64_t)0;
      }
      SpmdPlan plan = rule ? PlanSpmdByRules(&cur, so) : PlanSpmdLevel(&cur, so);
      cand.spmd_stats = plan.stats;
      spmd_comm = plan.stats.comm_bytes;
      cur.record_split(p.spmd, false);
      TransformStats ts;
      Graph t = SpmdTransform(cur, plan, level, p.spmd, &ts);
      if (rule) spmd_comm = ts.comm_bytes;
      cur = std::move(t);
      ++level;
    }
    // 3. pipeline stages
    EvalInput ei;
    ei.num_stages = p.stages; ei.num_micro = p.micro; ei.spmd = p.spmd;
    if (p.stages > 1) {
      StagePlanOptions so;
      so.num_stages = p.stages;
      so.unbalanced_ratio = opt.unbalanced_ratio;
      cand.stage_plan = PlanStages(&cur, so);
      ei.stage_flops = cand.stage_plan.stage_flops;
      for (auto& f : ei.stage_flops) f *= (double)p.micro * p.spmd;  // sketch flops are per micro-batch per shard
      ei.cut_bytes = cand.stage_plan.cut_bytes * p.spmd;
    } else {
      double fl = 0;
      for (auto& n : g.nodes) fl += NodeFlops(g, n);
      ei.stage_flops = {fl};
      for (auto& n : cur.nodes) n.stage = 0;
    }
    // gradient collectives overlap with backward (side stream); activation collectives are exposed
    ei.spmd_comm_bytes = spmd_comm * p.micro;
    ei.exposed_comm_fraction = opt.exposed_comm_fraction >= 0 ? opt.exposed_comm_fraction : opt.hw.ExposedCommFraction(p.spmd);
    ei.var_bytes = VarBytes(g);
    ei.act_bytes = ActBytes(g);
    {   // rows one device works on per micro-batch: the sample inputs' leading extent (tokens = every element of an integer
        // input; feature tensors: everything but the innermost dim), split over the SPMD group and the micro-batches
      double rows = 0;
      for (auto& n : g.nodes)
        if (n.op == "input" && !n.outputs.empty()) {
          const TensorType& t = n.outputs[0];
          double r = (double)t.numel();
          if (t.dtype != "i32" && t.dtype != "i64" && t.rank() > 1) r /= (double)t.dims.back();
          rows = std::max(rows, r);
        }
      ei.rows_per_micro = rows / std::max(1, p.spmd) / std::max(1, p.micro);
    }
    cand.eval = Evaluate(ei, opt.hw);
    cand.graph = std::move(cur);
    log << "[candidate] " << p.str() << " -> " << cand.eval.str() << "\n";
    best.candidates.push_back({p.str(), cand.eval.total_duration});
    if (!ok) continue;
    if (!have || (cand.eval.feasible && !best.eval.feasible) ||
        (cand.eval.feasible == best.eval.feasible && cand.eval.total_duration < best.eval.total_duration)) {
      auto keep = best.candidates;
      best = std::move(cand);
      best.candidates = keep;
      have = true;
    }
  }
  if (have) log << "[Strategy] " << best.proposal.str() << " " << best.eval.str() << "\n";
  best.log = log.str();
  return best;
}

}  // namespace tepdist
