// project_generic_body.cuh — the constants and plane descriptor of the generic projection k_project<SW, SH>
// (kernels_project.cu), shared with its recording variant k_project_rec (objective/objective.cu).  The
// body itself is project_generic_body.inc.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.cuh"
#include "numerics.cuh"
#include "project_common.cuh"
#include "record.cuh"
#include "strip_sync.cuh"

namespace j2p {

// ------------------------------------------------------------------------------------------
// k_project — 8 threads per coefficient block (thread j owns row j), 32 blocks per CTA.
// Template <SW, SH>: compile-time sampling factors of the plane (float4 I/O, stepped values of
// the whole footprint kept in registers); SW == 0 selects the run-time generic path.
// ------------------------------------------------------------------------------------------
#ifndef J2P_PBW_LOG2
#define J2P_PBW_LOG2 5     // CTA tile = 2^k blocks wide: 32 x 1 blocks = 1 KB contiguous per plane row (DRAM locality)
#endif
constexpr int P_NT = 256, P_BW = 1 << J2P_PBW_LOG2, P_BH = (P_NT / 8) / P_BW;   // CTA tile in coefficient blocks

struct ProjPlane {
    int c;          // plane index
    int gx;         // CTAs per row
};

#ifndef J2P_PROJ_MIN_CTAS
#define J2P_PROJ_MIN_CTAS 4     // resident CTAs per SM for full-resolution planes (register bound 64)
#endif

}  // namespace j2p
