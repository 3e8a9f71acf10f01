// agg_jit.h — run-time specialisation of the fused filter -> hash-aggregate kernel and of the two
// passes of the partitioned aggregation.
//
// The reference interprets its plan per block (FilterExecutor + AggregateHashTable dispatch over
// dynamic `dyn AggregateFunction`s, aggregate_function.rs); the precompiled kernels here interpret
// a by-value plan per ROW (op if-chains, slot selects, runtime-constant modulo).  An operator instead
// asks for a kernel compiled for its plan: the plan is printed as one `constexpr StaticPlan`, NVRTC
// compiles agg_kernels.cuh against it for sm_90a (once per plan shape and process; ~0.5 s), and the
// cubin is loaded through the runtime's library API.  No NVRTC on the machine, or a failed
// compilation, leaves the operator on the precompiled kernels — same results, more instructions.
#pragma once
#include <string>

#include "plan.h"

namespace dbx {

struct AggJitKernels {
  cudaKernel_t fast = nullptr;  // whole tiles of plain 8-byte columns (FAST)
  cudaKernel_t gen = nullptr;   // any column layout, direct row order
  cudaKernel_t part = nullptr;  // pass 1 of the partitioned aggregation (filter_partition_body)
  cudaKernel_t part_ring = nullptr;  // the same on the bulk-copy ring (filter_partition_ring_body)
  cudaKernel_t slice = nullptr; // pass 2 in shared memory (slice_agg_body)
  bool ok() const { return fast && gen; }
  bool two_pass_ok() const { return part && part_ring && slice; }
};

// Text of the StaticPlan initialiser for a plan; empty when the plan cannot be specialised.
std::string agg_jit_plan_text(const StaticPlan& sp);
// Returns the kernels for (plan text, slot count), compiling on first use.  `compile_only`
// stops after NVRTC (no GPU needed: used by the CPU test-suite); out may then be nullptr.
bool agg_jit_get(const std::string& plan_text, int n_slots, AggJitKernels* out, std::string* why, bool compile_only = false);

// One kernel of a generated translation unit (see eval.cu): compiled once per distinct source text.
bool jit_get_kernel(const std::string& source, const char* name, cudaKernel_t* out, std::string* why, bool compile_only = false);

}  // namespace dbx
