#pragma once
// Stream compaction (rb200_compact.cu): rb200_compact_count and rb200_compact of include/ramba_b200.h.
#include <cuda_runtime.h>

#include "../../include/ramba_b200.h"

namespace rb200 {

// A validated condition view cut into runs and chunks, shared by the two kernels and the description.  The view's
// C-order positions 0..n-1 form n_runs runs of run_len positions; run r is cut into cpr chunks of at most
// RB200_COMPACT_CHUNK positions.  Chunk (r, c) has index q = c * n_runs + r.  A CTA covers one chunk when
// run_len >= RB200_COMPACT_CHUNK, otherwise runs_per_cta whole runs (one chunk each).
struct CompactView {
  const char* base;
  int nd;  // dims after dropping unit dims and merging the ones that are contiguous in memory
  int eb;
  long long shape[RB200_MAX_DIMS];
  long long stride[RB200_MAX_DIMS];  // elements
};

#ifdef __CUDACC__
// element offset of C-order position p of a view
__device__ __forceinline__ long long c_offset(const CompactView& v, long long p) {
  if (v.nd == 1) return p * v.stride[0];
  long long off = 0;
#pragma unroll
  for (int d = RB200_MAX_DIMS - 1; d >= 0; --d) {
    if (d < v.nd) {
      if (d == 0) {
        off += p * v.stride[0];
      } else {
        const long long q = p / v.shape[d];
        off += (p - q * v.shape[d]) * v.stride[d];
        p = q;
      }
    }
  }
  return off;
}
#endif

struct CompactPlan {
  CompactView cond;
  long long n, run_len, n_runs, cpr, runs_per_cta, ctas;
};

// the payload of rb200_compact
struct CompactOut {
  int form;
  CompactView values;                       // VALUES
  int k;                                    // COORDS: streams (the view's dims)
  long long cshape[RB200_MAX_DIMS];         // COORDS / FLAT: the view's shape (unit dims kept)
  long long origin[RB200_MAX_DIMS];         // COORDS: global coordinate of element (0, ..., 0)
  long long gstride[RB200_MAX_DIMS];        // FLAT: C-order strides of the global shape
  long long g0;                             // FLAT: flat index of element (0, ..., 0)
  void* out[RB200_MAX_DIMS];
};

CompactView make_compact_view(const rb200_index_view& v);
void make_compact_plan(const rb200_index_view& cond, long long run_len, CompactPlan* P);
cudaError_t launch_compact_count(const CompactPlan& P, bool is_float, long long* counts, cudaStream_t stream);
cudaError_t launch_compact(const CompactPlan& P, bool is_float, const long long* counts, const long long* incl, const long long* run_base,
                           const CompactOut& O, cudaStream_t stream);

}  // namespace rb200
