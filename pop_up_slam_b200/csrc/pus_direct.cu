// pus_direct.cu -- the third instantiation of the device code (pus::kdirect): the persistent kernel of handles in direct
// linear-solver mode (pus_set_linear_solver(h, 1)), whose LM / GN / update driver factors the reduced pose system by a dense
// Cholesky instead of running PCG (DESIGN.md section 5).  A kernel of its own, so that the default PCG kernel (pus::kplain)
// is compiled exactly as without it.  Single-GPU only: the spanning hooks are compiled out.
#include <cuda_runtime.h>

#include "pus_graph.hpp"

namespace pus {
namespace kdirect {
#define PUS_NO_SPAN 1
#define PUS_DIRECT 1
#include "pus_kernels.cuh"
#include "pus_driver.cuh"
#undef PUS_DIRECT
#undef PUS_NO_SPAN
}  // namespace kdirect

void* direct_kernel_ptr() { return (void*)kdirect::lm_kernel; }
size_t direct_devgraph_bytes() { return sizeof(kdirect::DevGraph); }
cudaError_t direct_kernel_prepare() {
  return cudaFuncSetAttribute(kdirect::lm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kdirect::kSmemBytes);
}
}  // namespace pus
