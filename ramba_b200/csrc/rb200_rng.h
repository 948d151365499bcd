// rb200_rng.h — parameters and host-side plan of the random fill kernel (rb200_rng.cu).
#pragma once
#include <cuda_runtime.h>

#include <string>

#include "../../include/ramba_b200.h"

namespace rb200 {

constexpr int kRngMaxTail = 4;  // affine instructions after the draw (`low + (high - low) * u`, `loc + scale * z`)

struct RngParams {
  char* out;                          // the one contiguous destination view, in the form's own dtype
  int form;                           // rb200_philox_form
  int ndim;
  long long shape[RB200_MAX_DIMS];    // itershape
  long long gstart[RB200_MAX_DIMS];   // global_start
  long long mult[RB200_MAX_DIMS];     // linear index: g0, then lin = lin * mult[d] + g_d for d = 1.. (Horner form)
  long long rows, inner;              // the box as [rows][inner]: every row is one run of consecutive linear indices
  long long per_row;                  // blocks a row touches (upper bound over the alignments of its first index)
  long long items;                    // rows * per_row
  unsigned long long key, bound;
  int n_tail;
  int tail_op[kRngMaxTail];           // RB200_OP_ADD / SUB / MUL with the accumulator as a and a scalar as b
  unsigned long long tail_scal[kRngMaxTail];
};

struct RngPlan {
  RngParams P;
  long long blocks;
};

// A plain draw: the linear index from the IOTAs, one PHILOX, an optional affine tail in the draw's class, and one
// unmasked store to a view in that class's own dtype that is contiguous over the range.  false: anything else.
bool plan_rng(const rb200_fused_op* op, int sms, RngPlan& T);
// one line for rb200_describe_plan
std::string describe_rng(const RngPlan& T);
cudaError_t launch_rng(const RngPlan& T, cudaStream_t stream);

}  // namespace rb200
