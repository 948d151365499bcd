#pragma once
#include <string>

#include "rb200_vm.cuh"

namespace rb200 {
constexpr int kV = 4;   // elements per thread per tile (N-d and axis kernels)
constexpr int kV1 = 8;  // elements per thread per tile of the 1-D kernel (halves the per-instruction decode cost)
// launchers (one translation unit per kernel instantiation so that they compile in parallel)
cudaError_t launch_vm_elementwise_nd1(const KParams& P, unsigned blocks, size_t smem, cudaStream_t stream);
cudaError_t launch_vm_elementwise_nd2(const KParams& P, unsigned blocks, size_t smem, cudaStream_t stream);
cudaError_t launch_vm_elementwise_nd3(const KParams& P, unsigned blocks, size_t smem, cudaStream_t stream);
cudaError_t launch_vm_elementwise_nd5(const KParams& P, unsigned blocks, size_t smem, cudaStream_t stream);
cudaError_t launch_vm_elementwise_lean(const KParams& P, unsigned blocks, size_t smem, cudaStream_t stream);
cudaError_t launch_vm_elementwise_ax1d(const KParams& P, unsigned blocks, size_t smem, cudaStream_t stream);
cudaError_t launch_vm_axis_reduce(const KParams& P, unsigned blocks, size_t smem, cudaStream_t stream);

// the general interpreter's plan (rb200_interp_plan.cu): an elementwise op list (with global reductions) or an axis
// reduction; for the axis forms the kernel writes splits [0, n_written) of the requested ones
enum InterpForm { INTERP_ELEMENTWISE, INTERP_AXIS_AS_1D, INTERP_AXIS_REDUCE };
struct InterpPlan {
  InterpForm form;
  KParams k;
  bool lean;  // INTERP_ELEMENTWISE, 1-D: the lean instantiation (handler ids are lean ids)
  bool per_tile;  // the lean kernel runs one CTA per tile instead of a persistent grid walking the tiles
  long long blocks;
  size_t smem;
  int n_written;
};
// any valid, non-empty op list.  row_mode / lean / per_tile: the N-d row tiling, the lean 1-D kernel and its grid of
// one CTA per tile may be chosen
void plan_interp(const rb200_fused_op* op, int sms, bool row_mode, bool lean, bool per_tile, InterpPlan& I);
// one line for rb200_describe_plan
std::string describe_interp(const rb200_fused_op* op, const InterpPlan& I);

long long scan_scratch_bytes(long long n_outer, long long len, long long n_inner);
cudaError_t launch_scan(const void* src, void* dst, int dtype, long long n_outer, long long len, long long n_inner, int op, const void* carry, void* totals,
                        void* scratch, int sms, cudaStream_t stream, bool* supported);
}  // namespace rb200
