// Cost-based SPMD strategy planner for ONE mesh level.
//
// Reference parity (SURVEY §2.A A5, A6, A8): CostSpmdStrategy::StrategyPlanning
// (xla/service/parallel/cost_spmd_strategy.cc:4782-4916): seed from user annotations -> memory plan
// (SplitPlanByMemCost) -> critical-node decomposition of the forward graph into sub-graphs with the backward
// ops attached by op_group (FindSubGraphs/ExpandSubGraphs) -> per sub-graph strategy selection (DP inside
// cones + ILP across cones == PBQP reductions + branch&bound here) for every (head, tail) strategy pair ->
// DP across sub-graphs keyed on the separator strategy -> post-process -> record DistSpec on every value.
// InstAffinityMap's In/Out affinity (variable <-> updated output) and Var/Aux affinity (variable <-> slots)
// are expressed as edges of the same optimisation problem.
#pragma once
#include <map>
#include <string>
#include <vector>

#include "cost.h"
#include "ir.h"
#include "rules.h"

namespace tepdist {

struct SpmdOptions {
  int num = 2;                       // devices at this mesh level
  double var_mem_limit = HwProfile().var_mem_limit;   // VAR_MEM_LIMIT (bytes per device for variables + slots + grads)
  int num_threads = 1;               // ILP_NUM_THREADS: sub-graph problems solved concurrently (same plan, less wall time)
  bool share_relayout_cost = false;  // experimental: split a value's re-layout price over its consumers (see EdgeCost)
  bool sequence_parallel = false;    // tensor-parallel plans may use the reduce-scatter / all-gather (Megatron sequence-parallel) form
  bool context_parallel = false;     // attention never reshards to heads: the sequence split stays, K / V ride a ring ("cp" strategy)
  int mem_split_min_rank = 1;        // memory plan: only variables of at least this rank may be FORCED to be stored sharded
                                     // (2 = matrices only: Megatron-style tensor parallelism keeps biases / LayerNorm vectors whole)
  double cost_factor = 1.0;          // COST_FACTOR (all-to-all weight)
  int opt_level = 2;                 // OPT_LEVEL: >=3 one whole-graph problem, <3 sub-graph DP
  bool ignore_annotation = true;     // IGNORE_ANNOTATION
  bool aux_affinity = false;         // AUX_AFFINITY (variable <-> optimizer slots share a layout)
  int forward_sub_graph_num = 0;     // FORWARD_SUB_GRAPH_NUM: 0 = cut at every separator
  double min_segment_flops_frac = 0; // tiny-node clustering: separators cutting off less than this share of the forward FLOPs are dropped
  double ilp_time_limit_s = 20.0;    // ILP_TIME_LIMIT
  double replicate_penalty = 1e-3;   // per byte of activation computed redundantly (keeps free splits split)
  double memory_weight = 0.0;        // per byte of variable state stored per device (0: memory only via VAR_MEM_LIMIT)
  double shard_storage_penalty = 1e-6;  // tie-break: keep variables stored whole unless sharding saves traffic
  double collective_latency_bytes = -1; // per-collective launch + sync latency, in bytes of wire time, added to every edge whose
                                        // re-layout launches a collective in the activation path (< 0: hw.coll_latency *
                                        // hw.link_bw; 0 disables).  Gradient / parameter collectives are bucketed by the
                                        // runtime (a handful of launches per step whatever the number of variables) and pay none.
  HwProfile hw;
};

struct SpmdStats {
  double comm_bytes = 0;       // objective: per-device bytes moved by the inserted collectives
  double solve_seconds = 0;
  int num_subgraphs = 0;
  int distinct_subgraphs = 0;  // after structural memoisation
  int core_nodes_max = 0;      // largest irreducible ("ILP") core
  bool optimal = true;
  double var_bytes_per_device = 0;
  int forced_weight_splits = 0;
  int ignored_annotations = 0;   // user split / replicate annotations no candidate of the node can honour
  int threads_used = 1;          // worker threads that solved the sub-graph problems (SpmdOptions::num_threads)
  int infeasible_subgraphs = 0;  // sub-graphs without a consistent assignment (their nodes keep candidate 0): a planner defect if > 0
  std::map<std::string, int> collectives;  // kind -> count implied by the chosen plan
};

struct SpmdPlan {
  // chosen candidate per node (ins = layout each operand must arrive in, outs = produced layouts)
  std::vector<Candidate> choice;
  SpmdStats stats;
};

// Forward separators: forward values through which ALL forward dataflow passes (the reference's critical nodes,
// GraphSketch::FindCriticalInsts — FreedomDegree()==0 on the heavy path).
// Critical nodes = separators of the forward dataflow (reference GraphSketch, hlo_graph_sketch.cc:1288-1336: the nodes of the
// max-FLOPs main path whose FreedomDegree is 0).  Computed by a liveness scan: after a critical node executes, its output is
// the ONLY live forward value, i.e. no value bypasses it -- which is the FreedomDegree == 0 condition and puts the node on every
// source-to-loss path, the heaviest one included.  `min_segment_flops_frac` > 0 additionally drops separators that would cut off
// a sub-graph with less than that share of the forward FLOPs (the reference's tiny-node clustering): their nodes are merged
// into the following sub-graph.
std::vector<int> FindCriticalNodes(const Graph& g, double min_segment_flops_frac = 0.0);
// The same set from the DEFINITION (independent implementation used to verify the scan): the forward nodes that lie on the
// max-FLOPs source-to-loss path and have no bypassing forward edge (every forward edge (u, v) with topological position
// pos(u) < pos(c) < pos(v) is absent).
std::vector<int> FindCriticalNodesByMainPath(const Graph& g);

// Plans one level and appends the chosen DimStrategy to every value's DistSpec (levels.push_back).
SpmdPlan PlanSpmdLevel(Graph* g, const SpmdOptions& opt);

// Rule / annotation driven planner (reference FastSpmdStrategy, RULE_MODE=true): propagate the user's
// split / replicate annotations with InferGraph, everything undecided stays replicated.
SpmdPlan PlanSpmdByRules(Graph* g, const SpmdOptions& opt);

std::string DumpStrategies(const Graph& g, const SpmdPlan& plan);  // "strategies.txt" artefact

}  // namespace tepdist
