#pragma once
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
long long scan_scratch_bytes(long long n_outer, long long len, long long n_inner);
cudaError_t launch_scan(const void* src, void* dst, int dtype, long long n_outer, long long len, long long n_inner, int op, const void* carry, void* totals,
                        void* scratch, int sms, cudaStream_t stream, bool* supported);
}  // namespace rb200
