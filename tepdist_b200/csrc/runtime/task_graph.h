// Task-graph runtime IR, DAG construction, cost-based list scheduler, execution plan, GC / buffer-reuse plans.
//
// Reference parity (SURVEY §2.D D2-D6): xla/pjrt/task_graph.{h,cc}, task_scheduler.{h,cc}, execution_plan.{h,cc},
// lifetime_tracker.{h,cc}.  One TaskNode per (stage, micro-batch, phase) compute, explicit Send/Recv pairs on every
// cross-device edge, gradient accumulation tasks, optimizer (AG) tasks; a discrete-event list scheduler with the
// reference's priorities (GA first, smaller micro-batch first, forward admission capped at MICRO_NUM_LIMIT in
// flight => 1F1B, AG last, sends only when the peer can take them) but REAL cost estimates (FLOPs / bytes) instead
// of unit costs; per-device ordered task lists are what each rank executes in lock-step (static schedule =>
// deadlock-free send/recv pairing).
#pragma once
#include <map>
#include <string>
#include <vector>

#include "cost.h"

namespace tepdist {

enum class TaskType { kSplit, kInput, kCompute, kOutput, kSend, kRecv, kGAInit, kGA, kAG, kMerge };
const char* TaskTypeName(TaskType t);

struct TaskNode {
  int id = 0;
  TaskType type = TaskType::kCompute;
  std::string name;
  int stage = 0;          // pipeline stage (device group)
  int micro = -1;         // micro-batch id (-1: per step)
  bool backward = false;
  int device = 0;         // representative global device (first device of the stage's SPMD group)
  int peer_device = -1;   // send/recv partner
  double cost = 0;        // seconds
  double out_bytes = 0;   // bytes this task keeps alive until its consumers finish
  std::vector<int> parents, children;
  std::vector<int> mem_to_release;  // GC plan: task outputs that die after this task (D5 MakeTaskGraphGCPlan)
  int buffer_id = -1;     // recv-buffer reuse class slot (BUFFER_SAVE)
  bool buffer_reused = false;  // slot had an earlier user this step: the receiver must wait for that user's release
  int def_ctx = -1;       // index of the DefContext this task executes
};

class TaskDAG {
 public:
  std::vector<TaskNode> nodes;
  int AddNode(TaskType t, const std::string& name, int stage, int micro, bool backward, double cost, double out_bytes);
  void AddEdge(int from, int to);
  std::vector<int> TopoOrder() const;
  // immediate dominators (Cooper-Harvey-Kennedy) with the Split source as root
  std::vector<int> BuildDominanceTree() const;
  std::string ToDot() const;
  int source = -1, sink = -1;
};

struct PipelineSpec {
  int num_stages = 1, num_micro = 1, spmd = 1;
  std::vector<double> fwd_seconds, bwd_seconds;  // per stage, per micro-batch
  std::vector<double> ag_seconds;                // optimizer per stage
  std::vector<double> act_bytes;                 // activation bytes stashed per (stage, micro) between fwd and bwd
  std::vector<double> boundary_bytes;            // bytes crossing boundary s -> s+1 per micro-batch (one direction)
  double p2p_bw = 7.7e11, p2p_latency = 5e-6;
  double mem_limit = HwProfile().mem_bytes;
};
// D3 CompileTaskDAG + CrossDeviceCalibration: per (stage, micro) Input/Compute/Output bundles for fwd and bwd, GA per
// micro, GAInit/AG per stage, Send/Recv on every stage boundary.
TaskDAG BuildPipelineTaskDAG(const PipelineSpec& spec);

struct ScheduleOptions {
  int micro_num_limit = 0;       // MICRO_NUM_LIMIT: forward micro-batches in flight per stage (0 => num_stages => 1F1B)
  bool early_ga = true;          // EARLY_GA: accumulate (and release the micro-batch) right after its backward; false: when idle
  bool reorder_send = true;      // ReorderSend: hoist sends right after their producer
  bool buffer_save = true;       // BUFFER_SAVE: recv buffer reuse classes
  int group_sched_count = 0;     // GROUP_SCHED_COUNT: micro-batch m is scheduled in group m % count, each group with its own
                                 // 1F1B admission window (0 / 1: one group)
  int recv_ring = 0;             // receive-buffer ring size per class (0 => groups x in-flight limit: never undersized)
};
struct Schedule {
  std::map<int, std::vector<int>> device_tasks;  // device -> ordered task ids
  std::vector<double> start, finish;             // per task
  double makespan = 0;
  std::map<int, double> peak_bytes;              // device -> peak live activation bytes
  bool oom = false;
  double bubble_ratio = 0;
  std::string Dump(const TaskDAG& dag) const;
};
Schedule ScheduleTasks(TaskDAG* dag, const PipelineSpec& spec, const ScheduleOptions& opt);

// D3 proper: the same DAG compiled from the DefContext tree of a decomposed plan (compile_task_dag.cc); fills `spec_out` with
// the costs it derived so the scheduler prices the same numbers.  (Declared here, defined next to the planner types.)
struct Decomposition;
struct StageTransfer;
class Graph;
TaskDAG CompileTaskDAG(const Graph& g, const Decomposition& d, const std::vector<StageTransfer>& xfers, int num_micro, int spmd,
                       const HwProfile& hw, PipelineSpec* spec_out);

// D6 OutputBuffersLifeTimeTracker: ref-count every task output along a linear execution order; returns for each
// position the outputs that become dead right after it.
std::vector<std::vector<int>> ComputeReleasePlan(const TaskDAG& dag, const std::vector<int>& order);

}  // namespace tepdist
