#pragma once
// Integer-array indexing kernels (rb200_index.cu): gather, scatter and route of include/ramba_b200.h.
#include <cuda_runtime.h>

#include "../../include/ramba_b200.h"

namespace rb200 {

// A validated rb200_index_view after dropping unit dims and merging dims that are contiguous with each other, so that a
// C-contiguous N-d view takes the flat 1-D path.
struct IdxView {
  char* base;
  int ndim;
  int elem_bytes;
  long long size;
  long long shape[RB200_MAX_DIMS];
  long long stride[RB200_MAX_DIMS];
};

// A validated rb200_route_table, copied into the kernel's parameters (under 4 KB).
struct RouteParams {
  int ndim, n_ranks;
  long long size;
  long long shape[RB200_MAX_DIMS];
  int n_cells[RB200_MAX_DIMS];
  int cut_start[RB200_MAX_DIMS];
  long long cuts[RB200_MAX_ROUTE_CUTS];
  int owner[RB200_MAX_ROUTE_CELLS];
  long long offset[RB200_MAX_ROUTE_CELLS];
  long long stride[RB200_MAX_ROUTE_CELLS * RB200_MAX_DIMS];
};

IdxView collapse_index_view(const rb200_index_view& v);
cudaError_t launch_gather(const IdxView& v, const long long* lin, long long n, void* out, unsigned long long* bad, int sms, cudaStream_t stream);
cudaError_t launch_scatter(const IdxView& v, const long long* lin, long long n, const void* values, unsigned long long* bad, int sms,
                           cudaStream_t stream);
long long route_scratch_bytes(long long n, int n_ranks);
cudaError_t launch_route(const RouteParams& R, const long long* lin, long long n, long long* offsets, long long* slots, long long* counts,
                         unsigned long long* bad, void* scratch, int sms, cudaStream_t stream);

}  // namespace rb200
