// Communication / compute cost model.
//
// Reference parity (SURVEY §2.A A7, A11): Cost() / DataTransferSize() (cost_spmd_strategy.cc:74-174),
// PerfUtils (performance_utils.cc), Evaluator constants (evaluator.h:45-57).  Re-parameterised for one
// 8xH100 SXM NVSwitch box (single bandwidth tier + launch latency); the reference's V100 numbers stay selectable
// as the "reference" profile.
#pragma once
#include <string>

#include "ir.h"

namespace tepdist {

struct HwProfile {
  std::string name = "h100";
  double flops = 7e14;           // dense bf16 FLOP/s per GPU a GEMM sustains (about 70 % of the 989 TFLOP/s data-sheet peak)
  double hbm_bw = 3.35e12;       // B/s (HBM3, data sheet)
  double link_bw = 4.5e11;       // B/s per direction per GPU through NVSwitch (NVLink 4, data sheet)
  double inter_node_bw = 5.0e10; // B/s (unused on one box)
  double coll_latency = 8e-6;    // s per collective launch/sync
  double mem_bytes = 80e9 * 0.9;       // usable device memory (pipeline schedules, plan feasibility)
  double var_mem_limit = 60e9;         // default VAR_MEM_LIMIT: variables + optimizer slots + gradients per device before the
                                       // planner forces weights to be stored sharded (leaves ~20 GB for activations / workspaces)
  // Share of the SPMD collectives' wire time that is NOT hidden under compute, by group size (the fused bucketed
  // reduce-scatter + AdamW + all-gather runs on a side stream; larger groups leave less of it hidden).  Not measured on
  // H100: these values were calibrated on a different GPU generation and are kept until they are re-measured.
  double ExposedCommFraction(int n) const {
    if (name == "reference_v100") return 1.0;          // the reference issues every collective in-stream
    if (n <= 2) return 0.33;
    if (n <= 4) return 0.70;
    return 0.90;
  }
  // Tensor-core work on few rows runs far below the sustained rate (tile-count quantisation on 132 SMs, per-kernel prologue /
  // epilogue against a few us of MMAs): time = flops / rate * (1 + half_rows / rows).  half_rows is not measured on H100
  // either (same carry-over as ExposedCommFraction).
  double small_batch_half_rows = 4096;
  double ComputeSlowdown(double rows) const { return (rows > 0 && name != "reference_v100") ? 1.0 + small_batch_half_rows / rows : 1.0; }
  static HwProfile H100() { return HwProfile(); }
  static HwProfile ReferenceV100() {
    HwProfile h;
    h.name = "reference_v100";
    h.flops = 15e12; h.hbm_bw = 9e11; h.link_bw = 300e9; h.inter_node_bw = 3.125e9; h.coll_latency = 0;
    h.mem_bytes = 32e9 * 0.9;
    h.var_mem_limit = 24e9;
    return h;
  }
};

enum class Reshard { kNone, kDynamicSlice, kAllGather, kAllToAll, kAllReduce, kReduceScatter, kInvalid };
const char* ReshardName(Reshard r);

// What it takes to turn a value laid out as `from` into layout `to`.
Reshard ClassifyReshard(const DimStrategy& from, const DimStrategy& to);
// Bytes each device moves for that reshard (B = full tensor bytes, n = group size).
//   AR = 2B(n-1)/n   AG = B - B/n   RS = B(n-1)/n   A2A = (B/n - B/n^2) * cost_factor   slice ~ 0
double ReshardBytes(Reshard kind, double full_bytes, int n, double cost_factor = 1.0);
double ReshardCost(const DimStrategy& from, const DimStrategy& to, double full_bytes, int n, double cost_factor = 1.0);
// Seconds for a collective of `bytes` per device.
double CollectiveSeconds(const HwProfile& hw, double bytes, bool spans_nodes = false);

constexpr double kInfCost = 1e30;

}  // namespace tepdist
