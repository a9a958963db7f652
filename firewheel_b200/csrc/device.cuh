// device.cuh — the ordering primitives every kernel source shares, and the one host launcher for kernels that need launch attributes.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <utility>

namespace fw {

// Programmatic dependent launch (sm_90+): a kernel launched with the PDL attribute may start while its predecessor in the stream
// is still running; it must not touch the predecessor's results before pdl_wait(). pdl_launch_dependents() lets the next kernel
// of the stream start early in the same way.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// gpu-scope acquire load / release store of a flag word that other CTAs or another stream's kernels poll
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) { asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

// cudaLaunchKernelEx with `smem` bytes of dynamic shared memory; pdl: launch with programmatic stream serialization (the kernel
// then orders itself after its predecessor with pdl_wait()).
template <class... KArgs, class... Args>
static cudaError_t launch_ex(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = pdl ? attr : nullptr; cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

}  // namespace fw
