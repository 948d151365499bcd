#pragma once
// Grouped reduction along one axis (rb200_group.cu): rb200_group_reduce of include/ramba_b200.h.
#include <cuda_runtime.h>

#include "../../include/ramba_b200.h"

namespace rb200 {

enum GroupForm { GFORM_ROW = 0, GFORM_COLUMN = 1, GFORM_GENERAL = 2 };

// A validated view split around the grouped axis, with the plan the launch and the description share.  Kept dims are the
// dims before the axis then the dims after it, unit dims dropped and contiguous neighbours merged on each side.
struct GroupPlan {
  const char* base;
  int elem_bytes;
  int nk;                  // kept dims (0..4)
  long long kshape[RB200_MAX_DIMS - 1];
  long long kstride[RB200_MAX_DIMS - 1];
  long long L, sa;         // extent and element stride of the grouped axis
  long long O, I, nkept;   // outer / inner element counts, nkept = O * I
  int G;
  int form;
  long long C;             // positions per chunk: chunk s covers [s*C, min((s+1)*C, L))
  int S;                   // chunks; their partials are folded in chunk order
  int K;                   // row form: CTAs per row (K > 1: ncl == 1 and partials go through scratch)
  int ncl;                 // row form: chunks per CTA, folded in shared memory
  long long ctas;
  long long scratch_bytes;
};

void make_group_plan(const rb200_index_view& v, int axis, int n_groups, GroupPlan* P);
const char* group_form_name(int form);
cudaError_t launch_group(const GroupPlan& P, int src_dtype, int op, const long long* offsets, const long long* members, const double* center,
                         void* out, void* scratch, cudaStream_t stream);

}  // namespace rb200
