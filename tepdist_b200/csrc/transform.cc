#include "transform.h"

#include <algorithm>
#include <set>
#include <sstream>
#include <stdexcept>

#include "cost.h"
#include "rules.h"

namespace tepdist {

std::string TransformStats::CommInfo() const {
  std::ostringstream o;
  o << "num_ar=" << num_all_reduce << " num_ag=" << num_all_gather << " num_aa=" << num_all_to_all
    << " num_rs=" << num_reduce_scatter << " num_ds=" << num_dynamic_slice << " total_cost=" << comm_bytes;
  return o.str();
}

namespace {

struct Rewriter {
  const Graph& g;
  const SpmdPlan& plan;
  int level, num;
  TransformStats* stats;
  Graph out;
  std::map<ValueRef, ValueRef> vmap;                                  // old value -> new value (in produced layout)
  std::map<ValueRef, DimStrategy> produced;                           // old value -> layout of vmap[v]
  std::map<std::pair<ValueRef, std::string>, ValueRef> reshard_cache;  // (old value, target) -> new value

  TensorType Sharded(const TensorType& t, const DimStrategy& s) const { return ShardType(t, s); }

  ValueRef Emit(const std::string& op, std::vector<ValueRef> ins, std::vector<TensorType> outs,
                std::map<std::string, Attr> attrs, const std::string& name, int group, bool backward) {
    int id = out.AddNode(op, ins, outs, attrs, name, group, backward);
    return ValueRef{id, 0};
  }

  // new value holding old value `v` in layout `to`
  ValueRef DoReshard(ValueRef v, const DimStrategy& to, const Node& user) {
    const DimStrategy& from = produced.at(v);
    tepdist::Reshard kind = ClassifyReshard(from, to);
    if (kind == Reshard::kNone) return vmap.at(v);
    auto key = std::make_pair(v, to.str());
    auto it = reshard_cache.find(key);
    if (it != reshard_cache.end()) return it->second;  // reference: dedup identical reshards per source
    const TensorType& full = g.type(v);
    const Node& prod = g.nodes[v.node];
    std::map<std::string, Attr> a;
    a["level"] = (int64_t)level;
    a["num"] = (int64_t)num;
    ValueRef nv;
    const double B = (double)full.bytes();
    const std::string nm = prod.name + "/";
    switch (kind) {
      case Reshard::kDynamicSlice:
        a["dim"] = (int64_t)to.dim;
        nv = Emit("dynamic_slice", {vmap.at(v)}, {Sharded(full, to)}, a, nm + "ds", prod.group, user.backward);
        if (stats) stats->num_dynamic_slice++;
        break;
      case Reshard::kAllGather:
        a["dim"] = (int64_t)from.dim;
        nv = Emit("all_gather", {vmap.at(v)}, {full}, a, nm + "ag", prod.group, user.backward);
        if (stats) { stats->num_all_gather++; stats->comm_bytes += ReshardBytes(kind, B, num); }
        break;
      case Reshard::kAllToAll: {
        a["split_dim"] = (int64_t)to.dim;
        a["concat_dim"] = (int64_t)from.dim;
        nv = Emit("all_to_all", {vmap.at(v)}, {Sharded(full, to)}, a, nm + "a2a", prod.group, user.backward);
        if (stats) { stats->num_all_to_all++; stats->comm_bytes += ReshardBytes(kind, B, num); }
        break;
      }
      case Reshard::kAllReduce:
        a["reduce"] = (int64_t)from.reduce_kind;
        nv = Emit("all_reduce", {vmap.at(v)}, {full}, a, nm + "ar", prod.group, user.backward);
        if (stats) { stats->num_all_reduce++; stats->comm_bytes += ReshardBytes(kind, B, num); }
        break;
      case Reshard::kReduceScatter:
        a["reduce"] = (int64_t)from.reduce_kind;
        a["dim"] = (int64_t)to.dim;
        nv = Emit("reduce_scatter", {vmap.at(v)}, {Sharded(full, to)}, a, nm + "rs", prod.group, user.backward);
        if (stats) { stats->num_reduce_scatter++; stats->comm_bytes += ReshardBytes(kind, B, num); }
        break;
      default:
        nv = vmap.at(v);
    }
    reshard_cache[key] = nv;
    return nv;
  }

  void FixAttrs(const Node& n, const Candidate& c, std::map<std::string, Attr>& a, const std::vector<TensorType>& outs) {
    const std::string& op = n.op;
    auto set_shape = [&](const char* key, const TensorType& t) { a[key] = t.dims; };
    if (op == "reshape" || op == "broadcast" || op == "pad_zero") set_shape("shape", outs[0]);
    if (op == "slice") {
      auto lim = n.attr_v("limits");
      if (c.outs[0].is_split()) lim[c.outs[0].dim] /= num;
      a["limits"] = lim;
    }
    if (op == "attention" || op == "attention_bwd") {
      if (c.tag == "heads") a["heads"] = (int64_t)(n.attr_i("heads") / num);
      if (c.tag == "seq") {   // context parallel: the runtime runs the K / V ring over the ranks of this level
        std::vector<int64_t> lv = n.attr_v("cp_levels"), nm = n.attr_v("cp_nums");
        lv.push_back((int64_t)level);
        nm.push_back((int64_t)num);
        a["cp_levels"] = lv;
        a["cp_nums"] = nm;
      }
    }
    const bool dropout = op == "dropout" || op == "dropout_bwd" || op == "dropout_add" ||
                         ((op == "attention" || op == "attention_bwd") && n.has("pdrop") && n.attr_f("pdrop") > 0.0);
    if (dropout) {
      // a dropout mask is defined on GLOBAL coordinates: remember the unsharded output shape and how every level cut it, so
      // the runtime can turn its mesh coordinates into the shard's offsets (runtime/executor.py Executor._drop_rng)
      if (!n.has("drop_full")) a["drop_full"] = n.outputs[0].dims;
      if (c.outs[0].is_split()) {
        std::vector<int64_t> dims = n.attr_v("drop_dims"), nums = n.attr_v("drop_nums"), lvls = n.attr_v("drop_levels");
        dims.push_back(c.outs[0].dim);
        nums.push_back(num);
        lvls.push_back(level);
        a["drop_dims"] = dims; a["drop_nums"] = nums; a["drop_levels"] = lvls;
      }
    }
    if (op == "softmax_xent") {
      const TensorType& l = g.type(n.inputs[0]);
      int64_t tokens = n.has("global_tokens") ? n.attr_i("global_tokens") : l.numel() / l.dims.back();
      a["global_tokens"] = tokens;
      if (c.ins[0].is_split()) {
        // the tokens are split over this level (the loss has no vocab candidate): an evaluation step sums its (loss, token
        // count) over exactly the levels recorded here
        std::vector<int64_t> lv = n.attr_v("token_levels"), nm = n.attr_v("token_nums");
        lv.push_back((int64_t)level);
        nm.push_back((int64_t)num);
        a["token_levels"] = lv;
        a["token_nums"] = nm;
      }
    }
    if (op == "reduce_mean" && c.outs[0].partial) {
      const TensorType& x = g.type(n.inputs[0]);
      int64_t cnt = 1;
      for (auto ax : n.attr_v("axes")) cnt *= x.dims[ax];
      a["mean_divisor"] = n.has("mean_divisor") ? n.attr_i("mean_divisor") : cnt;
    }
    if ((op == "batchnorm" || op == "batchnorm_bwd") && c.tag == "batch") {
      // the batch statistics span every level that splits the batch: the runtime completes them across those levels
      std::vector<int64_t> lv = n.attr_v("sync_levels"), nm = n.attr_v("sync_nums");
      lv.push_back((int64_t)level);
      nm.push_back((int64_t)num);
      a["sync_levels"] = lv;
      a["sync_nums"] = nm;
    }
    if (IsSource(op) && op != "constant" && c.outs[0].is_split()) {
      // sharded variable / input: remember how this level cut the FULL tensor so init / feeding can slice
      std::vector<int64_t> dims = n.attr_v("shard_dims"), nums = n.attr_v("shard_nums"), lvls = n.attr_v("shard_levels");
      dims.push_back(c.outs[0].dim);
      nums.push_back(num);
      lvls.push_back(level);
      a["shard_dims"] = dims; a["shard_nums"] = nums; a["shard_levels"] = lvls;
      if (!n.has("full_shape")) a["full_shape"] = n.outputs[0].dims;
    }
    if (IsSource(op) && !n.has("full_shape") && !a.count("full_shape")) a["full_shape"] = n.outputs[0].dims;
    if (n.has("slot_of")) {  // node ids change under the rewrite: keep the slot -> variable link valid
      auto it = vmap.find(ValueRef{(int)n.attr_i("slot_of"), 0});
      if (it != vmap.end()) a["slot_of"] = (int64_t)it->second.node;
    }
  }

  void Run() {
    out.name = g.name;
    out.split_nums = g.split_nums;
    out.share_dev = g.share_dev;
    out.placement_layout = g.placement_layout;
    out.meta = g.meta;
    for (const Node& n : g.nodes) {
      const Candidate& c = plan.choice[n.id];
      std::vector<ValueRef> ins;
      for (int k = 0; k < (int)n.inputs.size(); ++k) ins.push_back(DoReshard(n.inputs[k], c.ins[k], n));
      std::vector<TensorType> outs;
      for (int o = 0; o < (int)n.outputs.size(); ++o) outs.push_back(Sharded(n.outputs[o], c.outs[o]));
      std::map<std::string, Attr> a = n.attrs;
      FixAttrs(n, c, a, outs);

      // "contract_rs<d>": row-parallel linear whose reduction is a reduce-scatter over dim d inside the node (rules.cc LinearRule)
      const bool rs_inside = n.op == "linear" && c.tag.rfind("contract_rs", 0) == 0;
      const bool unfuse = rs_inside || (n.op == "linear" && c.outs[0].partial && (n.attr_b("bias") || n.attr_b("residual")));
      if (!unfuse) {
        int id = out.AddNode(n.op, ins, outs, a, n.name, n.group, n.backward);
        out.nodes[id].stage = n.stage;
        for (int o = 0; o < (int)n.outputs.size(); ++o) {
          out.nodes[id].dist[o] = n.dist[o];
          vmap[ValueRef{n.id, o}] = ValueRef{id, o};
          produced[ValueRef{n.id, o}] = c.outs[o];
        }
        continue;
      }
      // row-parallel linear with fused epilogue: the bias / residual must be added once, after the reduction.
      // y_partial = x_s w_s ; y = reduce(y_partial) ; y += b (+ res).  reduce = reduce-scatter when every consumer
      // wants the same split layout (new vs the reference, which never emits reduce-scatter), else all-reduce.
      std::map<std::string, Attr> la = a;
      la["bias"] = false;
      la["residual"] = false;
      const DimStrategy partial = DimStrategy::Partial(num, 0);
      std::vector<TensorType> louts = outs;
      if (rs_inside) louts[0] = Sharded(n.outputs[0], partial);     // the GEMM itself produces the full-shape partial sum
      int lid = out.AddNode("linear", {ins[0], ins[1]}, louts, la, n.name, n.group, n.backward);
      out.nodes[lid].stage = n.stage;
      ValueRef self{n.id, 0};
      DimStrategy want = DimStrategy::Glue();
      if (rs_inside) {
        want = c.outs[0];
      } else {
        bool first = true, same = true;
        for (auto& u : g.users(self)) {
          const DimStrategy& need = plan.choice[u.node].ins[u.operand];
          if (need.partial) { same = false; break; }
          if (first) { want = need; first = false; }
          else if (need != want) same = false;
        }
        if (!same || first) want = DimStrategy::Glue();
      }
      vmap[self] = ValueRef{lid, 0};
      produced[self] = rs_inside ? partial : c.outs[0];
      ValueRef red = DoReshard(self, want, n);
      for (auto it = reshard_cache.begin(); it != reshard_cache.end();)  // cached entries refer to the pre-epilogue value
        it = (it->first.first == self) ? reshard_cache.erase(it) : std::next(it);
      ValueRef cur = red;
      TensorType yt = Sharded(n.outputs[0], want);
      int k = 2;
      if (n.attr_b("bias")) {
        ValueRef bv = n.inputs[k++];
        DimStrategy bs = want.is_split() && want.dim == n.outputs[0].rank() - 1 ? DimStrategy::Split(0, num) : DimStrategy::Glue();
        ValueRef b = DoReshard(bv, bs, n);
        cur = Emit("add", {cur, b}, {yt}, {}, n.name + "/bias", n.group, n.backward);
      }
      if (n.attr_b("residual")) {
        ValueRef rv = n.inputs[k++];
        ValueRef r = DoReshard(rv, want, n);
        cur = Emit("add", {cur, r}, {yt}, {}, n.name + "/res", n.group, n.backward);
      }
      vmap[self] = cur;
      produced[self] = want;
    }
    // fetches are always returned replicated
    for (auto& v : g.outputs) out.outputs.push_back(DoReshard(v, DimStrategy::Glue(), g.nodes[v.node]));
    // updated value must land in its variable's storage layout (In/Out affinity)
    for (auto& kv : g.updates) {
      const DimStrategy& store = plan.choice[kv.first].outs[0];
      out.updates[vmap.at(ValueRef{kv.first, 0}).node] = DoReshard(kv.second, store, g.nodes[kv.second.node]);
    }
    // collectives were appended after their producers but possibly after their users' position: re-sort
    TopoSort();
  }

  void TopoSort() {
    // Nodes were emitted in a valid order already (a reshard is emitted right before its first user and cached
    // for later users), so nothing to do; keep the hook for safety checks.
    for (auto& n : out.nodes)
      for (auto& v : n.inputs)
        if (v.node >= n.id) throw std::runtime_error("SpmdTransform produced a non-topological graph at " + n.name);
  }
};

}  // namespace

Graph SpmdTransform(const Graph& g, const SpmdPlan& plan, int level, int num, TransformStats* stats) {
  Rewriter r{g, plan, level, num, stats, Graph(), {}, {}, {}};
  r.Run();
  return std::move(r.out);
}

int CombineGradientCollectives(Graph* g, int64_t bucket_bytes, int max_per_bucket) {
  // gradient collectives = all_reduce / reduce_scatter whose result feeds an apply_* node
  int bucket = 0, in_bucket = 0;
  int64_t fill = 0;
  std::string cur_kind;
  int64_t cur_level = -1;
  bool any = false;
  for (auto& n : g->nodes) {
    if (n.op != "all_reduce" && n.op != "reduce_scatter") continue;
    bool grad = false;
    for (auto& u : g->users(ValueRef{n.id, 0}))
      if (g->nodes[u.node].op.rfind("apply_", 0) == 0 && u.operand == 1) grad = true;
    if (!grad) continue;
    const int64_t bytes = g->type(n.inputs[0]).bytes();
    const int64_t lvl = n.attr_i("level");
    if (any && (n.op != cur_kind || lvl != cur_level || fill + bytes > bucket_bytes || in_bucket >= max_per_bucket)) {
      ++bucket;
      fill = 0;
      in_bucket = 0;
    }
    any = true;
    cur_kind = n.op;
    cur_level = lvl;
    n.attrs["bucket"] = (int64_t)bucket;
    n.attrs["bucket_offset"] = fill;
    fill += bytes;
    ++in_bucket;
  }
  return any ? bucket + 1 : 0;
}

std::vector<int64_t> PlanFlatBuckets(const std::vector<int64_t>& offsets, int64_t end, int64_t gran, int64_t first, int64_t cap) {
  std::vector<int64_t> bounds = {0};
  for (size_t i = 1; i < offsets.size(); ++i) {
    const int64_t off = offsets[i];
    const int shift = (int)std::min<size_t>(bounds.size() - 1, 16);
    const int64_t want = std::min(cap, first << shift);
    if (off - bounds.back() >= want && gran > 0 && off % gran == 0) bounds.push_back(off);
  }
  bounds.push_back(end);
  return bounds;
}

int LivenessOptimize(Graph* g, int64_t min_bytes) {
  // B6 (reference hlo_liveness_optimizer.cc:26-54): a converted copy of a variable that has several users -- typically one
  // in the forward and one in the backward pass -- stays alive from its first to its last user, i.e. for most of the step.
  // Give every user after the first its own copy of the convert, placed immediately in front of that user (same group /
  // direction / stage as the user), so each copy lives only for the duration of one consumer and the run-time GC can
  // free it right away.  Rebuilds the node list (ids change); returns the number of copies made.
  const int n0 = (int)g->nodes.size();
  std::vector<char> target(n0, 0);
  bool any = false;
  for (int i = 0; i < n0; ++i) {
    const Node& n = g->nodes[i];
    if (n.op != "cast" || n.inputs.size() != 1 || g->nodes[n.inputs[0].node].op != "parameter") continue;
    if (n.outputs[0].bytes() < min_bytes) continue;
    std::set<int> user_nodes;
    for (auto& u : g->users(ValueRef{i, 0})) user_nodes.insert(u.node);
    if (user_nodes.size() > 1) target[i] = 1, any = true;
  }
  if (!any) return 0;
  std::vector<Node> out;
  out.reserve(n0 + 16);
  std::vector<int> remap(n0, -1);
  std::vector<char> used(n0, 0);
  int dup = 0;
  for (int i = 0; i < n0; ++i) {
    Node n = g->nodes[i];
    std::map<int, int> local;   // target cast -> copy used by THIS node (several operands may read the same cast)
    for (auto& v : n.inputs) {
      const int src = v.node;
      if (!target[src]) {
        v.node = remap[src];
        continue;
      }
      auto it = local.find(src);
      if (it != local.end()) {
        v.node = it->second;
        continue;
      }
      int use = remap[src];
      if (used[src]) {
        Node c = g->nodes[src];
        c.inputs[0].node = remap[c.inputs[0].node];
        c.id = (int)out.size();
        c.name += ".dup" + std::to_string(++dup);
        c.group = n.group;
        c.backward = n.backward;
        c.stage = n.stage;
        out.push_back(c);
        use = c.id;
      }
      used[src] = 1;
      local[src] = use;
      v.node = use;
    }
    n.id = (int)out.size();
    remap[i] = n.id;
    out.push_back(std::move(n));
  }
  g->nodes = std::move(out);
  for (auto& v : g->outputs) v.node = remap[v.node];
  std::map<int, ValueRef> upd;
  for (auto& kv : g->updates) upd[remap[kv.first]] = ValueRef{remap[kv.second.node], kv.second.idx};
  g->updates = std::move(upd);
  g->InvalidateUsers();
  return dup;
}

}  // namespace tepdist
