// mixed.cu — libj2pmixed.so: the grouped iteration kernels behind j2p_session_iterate_group.
//
// A group is several sessions whose frames differ in size.  Each kernel of an iteration is launched
// once for the whole group: the grid is flat, and CTA i reads entry i of a CTA table built by
// session.cu (geometry.cuh, GroupCta).  The entry names the session (its descriptor, GroupFrame, with
// the buffers of the current parity) and the block index the CTA would have in that session's own
// batch launch, so every frame is cut into the CTAs, bands and tiles its own session launches, its sums
// of g^2 go to its own partials and ticket and fold in the same order.  The bodies are the solver's
// (gradient_packed_body.inc, project_tile_body.inc, project_tile22_body.cuh), run with batch addressing.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../csrc/geometry.cuh"
#include "../csrc/gradient_packed_body.cuh"
#include "../csrc/project_tile22_body.cuh"
#include "../csrc/project_tile_body.cuh"

namespace j2p {

template <int NC_, bool TGV_, int GPM_>
__global__ void J2P_GRAD_BOUNDS k_gradient_packed_grouped(const GroupFrame *__restrict__ frames, const GroupCta *__restrict__ ctas, const float factor) {
    constexpr int NC = NC_, GPM = GPM_;
    constexpr bool TGV = TGV_, BATCH = true;
    const GroupCta e = ctas[blockIdx.x];
    const GroupGeo geo(e);
    const FrameDev &F = frames[e.d].F;
    const int band_rows = frames[e.d].band_rows;
    constexpr bool REC = false;
    const RecDev R{};
#include "../csrc/gradient_packed_body.inc"
}

// One CTA per SM fewer than k_project_tile: at its 64 registers the body spilled (4 bytes) with the table
// entry and the descriptor's addressing on top of a batch launch's.
template <bool RES_>
__global__ void __launch_bounds__(PT_NT, J2P_TILE_MIN_CTAS - 1) k_project_tile_grouped(const GroupFrame *__restrict__ frames, const GroupCta *__restrict__ ctas,
                                                                                  const float factor) {
    constexpr bool RES = RES_, BATCH = true;
    // the CTA's entry and its session's descriptor in shared memory: read through a global pointer, the
    // descriptor's fields would cost the body registers that a kernel parameter block does not
    __shared__ FrameDev F;
    __shared__ GroupCta e;
    const unsigned d = ctas[blockIdx.x].d;
    for (unsigned i = threadIdx.x; i < sizeof(FrameDev) / 8; i += blockDim.x)
        reinterpret_cast<uint2 *>(&F)[i] = reinterpret_cast<const uint2 *>(&frames[d].F)[i];
    if (threadIdx.x == 0) e = ctas[blockIdx.x];
    __syncthreads();
    const GroupGeo geo(e);
    const int c0 = (int)e.c;                 // the plane; bx is the CTA column within it
    constexpr bool REC = false;
    const RecDev R{};
#include "../csrc/project_tile_body.inc"
}

__global__ void __launch_bounds__(P22_NT, 3) k_project_tile22_grouped(const GroupFrame *__restrict__ frames, const GroupCta *__restrict__ ctas,
                                                                     const float factor) {
    const GroupCta e = ctas[blockIdx.x];
    project_tile22_body<true>(frames[e.d].F, (int)e.c, factor, GroupGeo(e));   // e.c: the plane; bx: the CTA column within it
}

__global__ void k_step_uncovered_grouped(const GroupFrame *__restrict__ frames, const GroupCta *__restrict__ ctas, const float factor) {
    const GroupCta e = ctas[blockIdx.x];
    step_uncovered_body<true>(frames[e.d].F, (int)e.c, factor, GroupGeo(e));
}

__global__ void k_step_uncovered22_grouped(const GroupFrame *__restrict__ frames, const GroupCta *__restrict__ ctas, const float factor) {
    const GroupCta e = ctas[blockIdx.x];
    step_uncovered22_body<true>(frames[e.d].F, (int)e.c, factor, GroupGeo(e));
}

template <bool TGV, int GPM>
static void *grad_kernel(int nc) {
    switch (nc) {
        case 1: return (void *)k_gradient_packed_grouped<1, TGV, GPM>;
        case 2: return (void *)k_gradient_packed_grouped<2, TGV, GPM>;
        default: return (void *)k_gradient_packed_grouped<3, TGV, GPM>;
    }
}

// the kernel of slot k (GroupKernel) for nc planes per frame
static void *kernel_of(int k, int nc, bool tgv) {
    switch (k) {
        case GK_GRAD + 0: return tgv ? grad_kernel<true, 0>(nc) : grad_kernel<false, 0>(nc);
        case GK_GRAD + 1: return tgv ? grad_kernel<true, 1>(nc) : grad_kernel<false, 1>(nc);
        case GK_GRAD + 2: return tgv ? (void *)k_gradient_packed_grouped<3, true, 2> : (void *)k_gradient_packed_grouped<3, false, 2>;
        case GK_TILE + 0: return (void *)k_project_tile_grouped<false>;
        case GK_TILE + 1: return (void *)k_project_tile_grouped<true>;
        case GK_TILE22: return (void *)k_project_tile22_grouped;
        case GK_UNCOVERED: return (void *)k_step_uncovered_grouped;
        default: return (void *)k_step_uncovered22_grouped;
    }
}

}  // namespace j2p

using namespace j2p;

// Once per device (the current one): the dynamic shared memory of the 2x2 tile kernel.
extern "C" int j2p_mixed_configure(void) {
    const cudaError_t e = cudaFuncSetAttribute(k_project_tile22_grouped, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P22_SMEM);
    if (e != cudaSuccess) cudaGetLastError();
    return (int)e;
}

// One iteration of a group on `stream`: the launches of L in GroupKernel order, each over its slice of
// the CTA table.  frames: the descriptors of this iteration's parity.  *nlaunch: kernels launched.
// Returns a cudaError_t.
extern "C" int j2p_mixed_iterate(const GroupFrame *frames, const GroupCta *ctas, const GroupLaunch *L, int nc, int tgv, float factor,
                                 void *stream, int *nlaunch) {
    const cudaStream_t s = (cudaStream_t)stream;
    *nlaunch = 0;
    for (int k = 0; k < GK_COUNT; k++) {
        if (L->count[k] == 0) continue;
        const GroupCta *slice = ctas + L->first[k];
        void *args[] = {(void *)&frames, (void *)&slice, (void *)&factor};
        const bool uncovered = k == GK_UNCOVERED || k == GK_UNCOVERED22;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(L->count[k]);
        cfg.blockDim = dim3(k < GK_TILE ? GM_NT : (k == GK_TILE22 ? P22_NT : (uncovered ? 256 : PT_NT)));
        cfg.dynamicSmemBytes = k == GK_TILE22 ? P22_SMEM : 0;
        cfg.stream = s;
        // the chain of the single-frame path (pdl.cuh): the gradient and the tile projections are programmatic
        // dependents of the kernel before them; the uncovered-pixel kernels are plain launches
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = !uncovered && pdl_enabled() ? 1 : 0;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        const cudaError_t e = cudaLaunchKernelExC(&cfg, kernel_of(k, nc, tgv != 0), args);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return (int)e;
        }
        *nlaunch += 1;
    }
    return (int)cudaSuccess;
}
