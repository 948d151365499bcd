// rb200_elementwise_lean.cu — the lean instantiation of the 1-D elementwise kernel (lean handler set only; see
// vm_elementwise_kernel in rb200_elementwise.cuh and lean_interp_eligible in rb200_interp_plan.cu).
#include "rb200_elementwise.cuh"
namespace rb200 {
cudaError_t launch_vm_elementwise_lean(const KParams& P, unsigned blocks, size_t smem, cudaStream_t stream) {
  return launch_vm_elementwise_nd<kV1, 1, false, true>(P, blocks, smem, stream);
}
}  // namespace rb200
