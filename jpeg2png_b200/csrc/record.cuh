// record.cuh — what the recording kernels of libj2pobjective.so (objective/objective.cu) take besides
// the frame descriptor: where the objective of every iteration goes (j2p_session_record_objective).
//
// The sub-gradient kernel sums a1·|∇x| (TV) and a2·|∇²x| (TGV) per source pixel in fp64 (compute.c:91,
// :155) into slots 3 and 4 of its per-CTA partials; the projection sums (residual/q)^2 per coefficient
// block in fp64 (compute_simd_step.c:22-26) and writes one partial per CTA (per block for the generic
// k_project) and plane.  The frame's last sub-gradient CTA of iteration i folds both, in a fixed order,
// into row i of the history: tv, tv2 of iteration i and the DCT distance the projection of iteration
// i-1 left (0 for iteration 0, session.cu).  Passed as a separate kernel parameter: FrameDev, and with
// it every existing kernel's parameter block, stays as it is.
#pragma once

namespace j2p {

constexpr int REC_FIELDS = 5;         // per frame and iteration: tv, tv2, prob of planes 0, 1, 2 (raw sums)

struct RecDev {
    double *hist;                     // [iterations][nframes][REC_FIELDS]
    double *pp;                       // projection partials [nframes][3][pp_stride]
    unsigned iter;                    // the iteration of this launch
    unsigned nframes;                 // frames per history row
    unsigned pp_stride;               // partials per plane slot
    unsigned pp_count[3];             // partials the projection of one frame writes per plane
    unsigned row0;                    // projection launches: the first CTA row of this launch in its plane
};

}  // namespace j2p
