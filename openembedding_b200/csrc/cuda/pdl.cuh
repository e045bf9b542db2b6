// Programmatic dependent launch (PDL) for the kernels of a training step.
//
// A step is ~25 short kernels (3-40 us each); at that size the launch latency, the CTA ramp-up
// and the setup code of a kernel (barrier init, tensor-map prefetch, descriptor staging) are a
// visible fraction of its run time. Every hot kernel therefore
//   * is launched with cudaLaunchAttributeProgrammaticStreamSerialization, so the stream (or
//     the captured graph edge) lets it start while its predecessor is still draining,
//   * calls pdl_trigger() first thing (its own successor may be scheduled as soon as all of
//     its CTAs are resident) and
//   * calls pdl_wait() after its setup code and BEFORE its first global-memory access that
//     depends on -- or could race with -- the predecessor: griddepcontrol.wait returns when the
//     preceding grid has completed and its memory operations are visible.
// Nothing before pdl_wait() may read data produced on the device or write global memory.
// EXB_PDL=0 in the environment turns the launch attribute off (the device instructions are
// then no-ops).
#pragma once
#include <cuda_runtime.h>
#include <cstdlib>
#include <utility>

namespace exb {

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

inline bool pdl_enabled() {
    static int on = -1;
    if (on < 0) {
        const char* e = getenv("EXB_PDL");
        on = (e && e[0] == '0') ? 0 : 1;
    }
    return on == 1;
}

template <class... KArgs, class... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(std::forward<Args>(args))...);
}

}  // namespace exb
