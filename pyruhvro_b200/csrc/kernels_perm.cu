// The permissive instance of the interpreter's fused decode pass (rv_schema_permissive): records with a record error
// become null rows and are listed instead of failing the call (dev_kernels.cuh fused_body<W, true>).  It has a
// translation unit of its own: the interpreter's fused body is the longest compile of the library, and _build.py
// compiles the sources side by side.
#include "kernels.cuh"

#include "dev_kernels.cuh"
#include "interp.cuh"

namespace rv {
namespace {

__global__ void __launch_bounds__(kBlock) fused_kernel_perm(const DecodeParams p) { fused_body<InterpWalker, true>(p, int(blockIdx.x)); }

}  // namespace

cudaError_t prepare_kernels_permissive() {
    cudaError_t e = cudaFuncSetAttribute(fused_kernel_perm, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(fused_kernel_perm, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    return e;
}

void launch_fused_permissive(const DecodeParams& p, size_t smem, cudaStream_t s) {
    fused_kernel_perm<<<unsigned(p.n_tiles), kBlock, smem, s>>>(p);
}

}  // namespace rv
