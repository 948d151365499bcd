#pragma once
// Order statistics (rb200_select.cu): rb200_select_count, rb200_select_choose and rb200_select_rows of
// include/ramba_b200.h.
#include <cuda_runtime.h>

#include "../../include/ramba_b200.h"
#include "rb200_compact.h"

namespace rb200 {

enum SelectForm { SELECT_ROW = 0, SELECT_PASS = 1 };

// A validated selection: the source view cut into S segments of L positions, K targets each, and the plan every launch
// and the description share.  Pass form: CTA c covers segment c / cps, positions [(c % cps) * chunk, ...) of it.
struct SelectPlan {
  CompactView src;
  int src_dtype, bits;            // bits: key width (64 or 32)
  long long n, L, S, K;           // S: the view's segments
  long long GS;                   // segments of the whole array (the digit width and compaction rule follow it)
  int form;
  bool vec;                       // 16-byte loads: one aligned unit-stride run, segments whole vectors
  int digit, passes;              // pass form: digit width and passes; row form: 8 and bits / 8
  long long chunk, cps, ctas;     // pass form: positions per CTA, CTAs per segment, CTAs
  long long rows, groups;         // pass form: count rows per launch, launches per pass
  long long shared_bytes;         // dynamic shared memory per CTA
  long long counts_bytes;         // pass form: S * K * 2^digit int64
  long long cand_cap;             // pass form, one segment: compaction buffer keys
};

// segments: 0, or the segments of the whole array when the view holds a rank's part of them (then the pass form)
void make_select_plan(const rb200_index_view& src, int src_dtype, long long seg_len, long long targets, long long segments, bool no_row,
                      SelectPlan* P);
const char* select_form_name(int form);
cudaError_t launch_select_count(const SelectPlan& P, const rb200_select_state& S, int pass, int mode, cudaStream_t stream);
cudaError_t launch_select_choose(const SelectPlan& P, const rb200_select_state& S, int pass, cudaStream_t stream);
cudaError_t launch_select_rows(const SelectPlan& P, const long long* rank_table, bool skip_nan, unsigned long long* keys, long long* nans,
                               cudaStream_t stream);

}  // namespace rb200
