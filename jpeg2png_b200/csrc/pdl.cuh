// pdl.cuh — programmatic dependent launch (griddepcontrol, sm_90+) for the kernels of an iteration.
//
// The solver is a chain of short kernels (4K: 114 us + 131 us per iteration; 1080p and the strips of a
// multi-GPU frame: a few tens of us each).  Launched the plain way, kernel n+1 cannot place a CTA
// before kernel n has drained and flushed: launch latency, the ramp of the first wave and the first
// DRAM round trip are paid in the open, every kernel, every iteration.  With the
// programmatic-stream-serialization launch attribute the CTAs of kernel n+1 become resident as soon
// as every CTA of kernel n has executed `launch_dependents` and an SM has room; they run whatever
// does not depend on kernel n (index set-up, tables, prefetch of buffers kernel n does not write)
// and block in `griddepcontrol.wait` until kernel n has completed and its writes are visible.
//
// Rule that keeps the chain safe: a kernel executes launch_dependents only AFTER its own wait has
// returned, so at most two grids are in flight and a kernel's pre-wait section can only overlap its
// immediate predecessor.  What each kernel does before its wait is stated at its pdl_wait().
// A kernel launched without the attribute sees both instructions as no-ops.
#pragma once
#include <cuda_runtime.h>
#include <stdlib.h>

#include <utility>

namespace j2p {

#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#endif

// J2P_PDL=0: launch the kernels of an iteration without the programmatic-dependent-launch attribute (A/B aid)
inline bool pdl_enabled() {
    static const bool on = [] {
        const char *e = getenv("J2P_PDL");
        return !(e && *e == '0');
    }();
    return on;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_chain(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args &&...args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

}  // namespace j2p
