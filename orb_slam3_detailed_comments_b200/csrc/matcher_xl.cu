// matcher_xl.cu -- the ORBmatcher searches in their global-memory form (matcher_core.cuh GlobalFrame), for frames and keyframes
// whose shared-memory form does not fit a CTA (launch_proj, matcher.cu, decides per call).  Its own library,
// liborbslam3_b200_match_xl.so, linked by liborbslam3_b200.so.
#include "matcher_core.cuh"

namespace orb {

// One CTA per frame writes the FrameFeat block (and for the grid searches the GridFeat block, after k_frame_grid) that the
// shared-memory form stages in every CTA.
__global__ void __launch_bounds__(1024) k_stage_frames_xl(const __grid_constant__ ProjParams P, const GlobalFrame S) {
    const int frame = blockIdx.x;
    FrameFeat F;
    int N, row0;
    stage_frame(P, P.frame_image[frame], S.featBlocks + (size_t)frame * S.featStride, F, N, row0);
    if (S.gridBlocks) {
        GridFeat GF;
        stage_grid(P, frame, S.gridBlocks + (size_t)frame * S.gridStride, GF, N, row0);
    }
}

template <int G>
__global__ void __launch_bounds__(PM_WARPS * 32) k_proj_candidates_grp_xl(const __grid_constant__ ProjParams P, const GlobalFrame S) {
    proj_candidates_grp_body<G>(P, S);
}

__global__ void __launch_bounds__(PM_WARPS * 32) k_proj_candidates_xl(const __grid_constant__ ProjParams P, const GlobalFrame S) {
    proj_candidates_body(P, S);
}

__global__ void __launch_bounds__(256) k_proj_resolve_xl(const __grid_constant__ ProjParams P, const GlobalFrame S) {
#include "matcher_resolve.inc"
}

__global__ void __launch_bounds__(PR_THREADS) k_proj_resolve_par_xl(const __grid_constant__ ProjParams P, const GlobalFrame S) {
#include "matcher_resolve_par.inc"
}

cudaError_t proj_xl_set_smem(size_t resolve_par_bytes, size_t resolve_bytes) {
    const cudaError_t e = cudaFuncSetAttribute(k_proj_resolve_par_xl, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)resolve_par_bytes);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(k_proj_resolve_xl, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)resolve_bytes);
}

cudaError_t launch_proj_xl(ProjXlKernel kernel, dim3 grid, size_t smem, cudaStream_t st, const ProjParams& P, const GlobalFrame& S) {
    switch (kernel) {
        case PXL_STAGE: return launch_p(k_stage_frames_xl, grid, dim3(1024), smem, st, P, S);
        case PXL_CAND_G4: return launch_p(k_proj_candidates_grp_xl<4>, grid, dim3(PM_WARPS * 32), smem, st, P, S);
        case PXL_CAND_G8: return launch_p(k_proj_candidates_grp_xl<8>, grid, dim3(PM_WARPS * 32), smem, st, P, S);
        case PXL_CAND_G16: return launch_p(k_proj_candidates_grp_xl<16>, grid, dim3(PM_WARPS * 32), smem, st, P, S);
        case PXL_CAND: return launch_p(k_proj_candidates_xl, grid, dim3(PM_WARPS * 32), smem, st, P, S);
        case PXL_RESOLVE_PAR: return launch_p(k_proj_resolve_par_xl, grid, dim3(PR_THREADS), smem, st, P, S);
        case PXL_RESOLVE: return launch_p(k_proj_resolve_xl, grid, dim3(256), smem, st, P, S);
    }
    return cudaErrorInvalidValue;
}

}  // namespace orb
