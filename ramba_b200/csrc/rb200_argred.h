#pragma once
// First-occurrence index reductions (rb200_argred.cu): rb200_arg_reduce of include/ramba_b200.h.
#include <cuda_runtime.h>

#include "../../include/ramba_b200.h"

namespace rb200 {

enum ArgForm { AFORM_GLOBAL = 0, AFORM_ROW = 1, AFORM_COLUMN = 2, AFORM_GENERAL = 3 };

// A validated view and the plan the launch and the description share.  Global form: `dims` are the view's dims (unit
// dims dropped; bind_arg_coords merges the ones that are contiguous in memory AND in the global flat index).  Axis
// forms: `dims` are the kept dims (the dims before the axis then the dims after it, unit dims dropped, neighbours that
// are contiguous in memory merged), walked in C order to give the contiguous output.
struct ArgPlan {
  const char* base;
  int form;
  int nd;
  long long shape[RB200_MAX_DIMS];
  long long stride[RB200_MAX_DIMS];   // elements in memory
  long long gstride[RB200_MAX_DIMS];  // global form: flat-index stride of each dim (bind_arg_coords)
  long long g0;                       // global form: flat index of the view's first element; axis forms: origin[axis]
  long long L, sa;                    // axis forms: extent and element stride of the reduced axis; global: element count
  long long n_out;                    // outputs (1 for the global form)
  long long C;                        // positions per chunk of the walk
  int S;                              // chunks per output; S > 1: (key, index) partials go to scratch and a fold ends
  long long ctas;
  long long scratch_bytes;
};

void make_arg_plan(const rb200_index_view& v, int axis, ArgPlan* P);
void bind_arg_coords(const rb200_index_view& v, int axis, const long long* origin, const long long* gstride, ArgPlan* P);
const char* arg_form_name(int form);
cudaError_t launch_arg(const ArgPlan& P, int src_dtype, int op, long long* out_idx, long long* out_key, void* scratch, cudaStream_t stream);

}  // namespace rb200
