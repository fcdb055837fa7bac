// ServiceEnv: the server-side flag system (reference xla/service/service_env.{h,cc}: an X-macro table of typed
// options; load order defaults -> JSON file (CONFIG_FILE, default config.json) -> environment variables, which
// override with a warning; the effective config is printed).  SURVEY E1 / §5.6.
#pragma once
#include <map>
#include <string>
#include <vector>

namespace tepdist {

#define TEPDIST_SERVICE_OPTIONS(X)                                                                  \
  X(DEBUG, "false", "verbose per-task timing and planner artefact dumps")                          \
  X(CLUSTER_SPEC, "", "path of the cluster JSON (master / workers: ip, port, gpu_ids)")            \
  X(RULE_MODE, "false", "annotation/rule driven planner instead of the cost-based one")            \
  X(IGNORE_ANNOTATION, "true", "ignore user sharding annotations in cost mode")                    \
  X(AUX_AFFINITY, "false", "force optimizer slots to share their variable's layout")               \
  X(COST_FACTOR, "1.0", "weight of all-to-all bytes in the planner objective")                     \
  X(FP16_COMM, "false", "communicate fp32 reductions in 16-bit (bf16)")                    \
  X(NUM_GRADIENTS, "0", "expected number of gradient tensors (sanity check)")                      \
  X(FORWARD_SUB_GRAPH_NUM, "0", "number of forward sub-graphs for the sub-graph DP (0 = every separator)") \
  X(VAR_MEM_LIMIT, "60000000000", "bytes per device for variables+slots+grads before weights are force-sharded") \
  X(OPT_LEVEL, "2", ">=3 whole-graph problem; <3 sub-graph DP; <1 fast inference only")            \
  X(UNBALANCED_RATIO, "0.08", "per-stage FLOPs slack of the pipeline planner")                     \
  X(NUM_MICRO_BATCHES, "0", "config mode: micro-batches")                                          \
  X(NUM_STAGES, "0", "config mode: pipeline stages")                                               \
  X(MICRO_NUM_LIMIT, "0", "forward micro-batches in flight per stage (0 = #stages => 1F1B)")       \
  X(GROUP_SCHED_COUNT, "1", "micro-batch groups (m % count) with their own 1F1B window (reference default: 2)")                            \
  X(PP_BANDWIDTH, "770", "GB/s assumed for pipeline p2p")                                          \
  X(ILP_TIME_LIMIT, "1", "minutes per exact solve before the greedy fallback")                     \
  X(ILP_NUM_THREADS, "1", "solver threads")                                                        \
  X(BUFFER_SAVE, "true", "reuse pipeline receive buffers")                                         \
  X(EARLY_GA, "true", "schedule gradient accumulation right after each backward (reference default: false)")                      \
  X(ASYNC_RECV, "true", "receive on a side stream")                                                \
  X(ASYNC_SEND, "true", "send on a side stream")                                                   \
  X(MULTI_REORDER, "true", "iterate send/GA reordering to a fixpoint")                             \
  X(FAKE_INPUT, "false", "cache the first step's inputs and reuse them")                           \
  X(DISABLE_BUFFER_ALIAS, "false", "debug: do not alias variable inputs/outputs")                  \
  X(FRONTEND, "torch", "client frontend name")                                                     \
  X(DUMP_ARTIFACTS, "false", "write strategies/cone/comm/stage/task-graph dumps (reference DUMP_LLVM_PTX analogue)") \
  X(COMM_MODE, "fused", "fused = peer-memory sm_90a kernels, nccl = reference-semantics baseline") \
  X(HW_PROFILE, "h100", "cost-model constants: h100 | reference_v100")

class ServiceEnv {
 public:
  static ServiceEnv* Instance();
  // defaults -> JSON file (CONFIG_FILE env or argument; missing file is fine) -> environment overrides
  std::vector<std::string> Load(const std::string& config_file = "");
  std::string Get(const std::string& key) const;
  long long GetInt(const std::string& key) const;
  double GetDouble(const std::string& key) const;
  bool GetBool(const std::string& key) const;
  void Set(const std::string& key, const std::string& value);
  std::vector<std::string> Keys() const;
  std::string Dump() const;

 private:
  ServiceEnv();
  std::map<std::string, std::string> values_, help_;
  std::vector<std::string> order_;
};

}  // namespace tepdist
