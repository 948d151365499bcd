// rb200_stream.h — parameters and host-side plan of the streaming kernels (rb200_stream.cu) and of the map + reduce
// kernels they hand over to (rb200_mapred.cu).
#pragma once
#include <cuda_runtime.h>

#include <string>

#include "rb200_lean.cuh"
#include "rb200_mapred.h"
#include "rb200_terms.h"

namespace rb200 {

constexpr int kStreamMaxStaged = 4;
constexpr int kStreamTile = LV * kThreads;  // 2048

struct StreamStaged {
  const char* base;
  int es;        // element size (4 / 8)
  int dview;     // the same view in the direct table (ragged last tile)
  unsigned off;  // byte offset inside a stage
  int pad;
};

struct StreamHoist {
  int direct, reg, is_f32_class;
};

struct StreamParams {
  int mode;
  long long total, n_tiles;                  // mode 0
  long long R, C, rows_per_split;            // mode 1: box [R][C]
  int n_chunks, n_split;
  int n_staged, depth;
  unsigned stage_bytes;
  StreamStaged staged[kStreamMaxStaged];
  int n_direct;
  LDirect direct[RB200_MAX_VIEWS];           // s1: row stride (mode 1), s2: element / column stride
  int n_hoist;
  StreamHoist hoist[kStreamMaxStaged];
  int n_insns, n_regs;
  LInsn insns[RB200_MAX_INSNS];
  u64 scal[RB200_MAX_SCALARS];
  int n_reds;
  KRed reds[RB200_MAX_REDS];
  u64* red_partials;
  unsigned int* red_counter;
  // term form (n_terms > 0, stream_terms_kernel): tile = tv * 256 elements (tv is always LV); steps [0, n32) in float32,
  // the rest in float64
  int tv, n_terms, n32;
  int n_thoist;                      // column mode: row-broadcast operands copied once per CTA into shared memory
  int thoist_direct[kStreamMaxStaged];
  TermStep terms[kMaxTerms];
};
constexpr int X_HOIST = 3;  // TermStep.xkind of the streaming kernel: element of a hoisted (row-broadcast) operand

struct StreamPlan {
  StreamParams P;
  size_t smem;
  long long blocks;
  int eff;  // column mode: splits actually written
  bool use_mr;  // the map + reduce kernels of rb200_mapred.cu run this op list
  MrParams mr;
};

// mode 0 (a contiguous 1-D space, optional global reductions) or mode 1 (one axis reduction over the rows of a [R][C]
// box into n_split row slices; T.eff of them are written).  false: the op list is not of this form.  use_terms /
// use_mapred: the term kernel and the map + reduce kernels may be chosen
bool plan_stream(const rb200_fused_op* op, int sms, int n_split, bool use_terms, bool use_mapred, StreamPlan& T);
// one line for rb200_describe_plan
std::string describe_stream(const StreamPlan& T);
cudaError_t launch_stream(const StreamPlan& T, cudaStream_t stream);

}  // namespace rb200
