// Host-side shard slicing and sharded deterministic initialisation.
//
// Reference parity (SURVEY D11, D13): SliceUtils (xla/pjrt/slice_utils.h: N-d strided shard copy for multi-level and
// stride-on-dim splits; GetSliceStartOffsetOnSrc returns (offset, len) runs) and the Philox initialisers
// (xla/pjrt/initializers.{h,cc}, fill_philox_random.h): every worker fills ONLY its shard, bit-identical to the
// corresponding slice of an unsharded initialisation.
#pragma once
#include <cstdint>
#include <string>
#include <utility>
#include <vector>

#include "ir.h"

namespace tepdist {

// Contiguous (element offset, length) runs, in shard order, that make up the shard of `shape` selected by
// applying every split level in `levels` with the per-level index `ids` (levels[i] is glue/partial => no cut).
std::vector<std::pair<int64_t, int64_t>> SliceRuns(const std::vector<int64_t>& shape, const std::vector<DimStrategy>& levels,
                                                   const std::vector<int>& ids);
std::vector<int64_t> ShardShape(const std::vector<int64_t>& shape, const std::vector<DimStrategy>& levels);
// Copy the shard out of a full row-major buffer (elem_size bytes per element).
void SliceCopy(const uint8_t* src, uint8_t* dst, int64_t elem_size, const std::vector<int64_t>& shape,
               const std::vector<DimStrategy>& levels, const std::vector<int>& ids);

// Philox4x32-10 stream keyed by `seed`; element i of the logical tensor depends only on (seed, i).
void PhiloxFill(const std::string& kind, uint64_t seed, int64_t offset, int64_t n, float mean, float stddev, float lo, float hi,
                float* out);
// Fill exactly the shard described by (shape, levels, ids): equals SliceCopy of a full PhiloxFill.
std::vector<float> PhiloxFillShard(const std::string& kind, uint64_t seed, const std::vector<int64_t>& shape,
                                   const std::vector<DimStrategy>& levels, const std::vector<int>& ids, float mean, float stddev,
                                   float lo, float hi);

// Dropout keep mask (DESIGN.md "Dropout"): out[e] = 1 iff element e of the box [start, start + len) of a tensor of GLOBAL
// shape `shape` is kept.  Philox4x32-10 keyed by `seed`, counter (column group, row, step, site); an element is kept iff its
// byte of the call's 16 is >= thr.  Elementwise: row = the flattened leading coordinates, 16 consecutive columns per call.
// attention (shape [B, H, S, S], (b, h, query, key)): one call per (b, h, 16-query block, 32-key block, query % 8,
// (key % 8) / 2), the 16 elements a thread of the forward kernel holds in its score fragment.  The CUDA kernels
// (ops/csrc/dropout_philox.cuh) produce the same bits.
void DropoutKeep(uint64_t seed, uint32_t step, uint32_t site, int thr, bool attention, const std::vector<int64_t>& shape,
                 const std::vector<int64_t>& start, const std::vector<int64_t>& len, uint8_t* out);

}  // namespace tepdist
