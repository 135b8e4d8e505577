// replay.cu -- batched sequence replay: the tracking-thread step of a batch of stereo or monocular frames through ONE pair of calls,
// host buffers in / host buffers out (include/orbslam3_b200.h: orbr_submit / orbr_collect).
//
// What the reference's Tracking thread does per frame -- Frame::Frame (both eyes through ORBextractor::operator(),
// Frame.cc:136-141; ComputeStereoMatches, Frame.cc:1102), TrackWithMotionModel (SearchByProjection(cur, last), PoseOptimization,
// Tracking.cc:3389-3443), TrackLocalMap (SearchByProjection(F, local map points), PoseOptimization, Tracking.cc:4052, 3522) --
// queued for n_frames frames at once on the handle's stream: one H2D of the images, one H2D per query array, the kernels, and
// the small count tables back.  A monocular step (orbr_step::monocular) extracts one image per frame with vLappingArea = {0, 1000}
// (Frame.cc:380) and skips ComputeStereoMatches; everything after the extraction is shared.  orbr_submit returns as soon as
// everything is queued; orbr_collect waits for the counts, reads back exactly the rows the batch produced and waits once more.
// Colour or differently sized camera images (orbr_step::image_format, src_*) go up as they are and become grey level-0 images on the
// device (k_ingest) before the extraction.  An RGB-D step (orbr_step::depth_maps) extracts one image per frame with vLappingArea = {0, 0}
// and takes mvuRight / mvDepth from the raw depth maps (k_stereo_rgbd, orbm_stereo_rgbd_batch) in place of ComputeStereoMatches.
// A host thread that keeps several handles in flight (submit k+1 .. k+H-1 before collect k) overlaps uploads, kernels and
// downloads of different handles without more threads.
#include <string.h>

#include <algorithm>
#include <vector>

#include "extractor.h"
#include "devmath.cuh"

using namespace orb;
using namespace orbdev;

struct orbr_state {
    // device copies of the host query arrays + device-side results of one step, carved from one allocation
    uint8_t* d_buf = nullptr;
    size_t bytes = 0;
    bool pending = false;
    int n_frames = 0, nimg = 0, nq_last = 0, nq_local = 0, with_po = 0;
    bool mono = false;
    cudaEvent_t ev_counts = nullptr;
    // result pointers inside d_buf
    int *d_fm = nullptr, *d_nm_last = nullptr, *d_match = nullptr, *d_nm_local = nullptr;
    int *d_eoff[2] = {}, *d_efeat[2] = {}, *d_inl[2] = {};
    float *d_exw = nullptr, *d_eobs = nullptr, *d_ew = nullptr;
    double* d_pose[2] = {};
    uint8_t* d_outl[2] = {};
    int* h_eoff = nullptr;   // pinned: edge_offset tables of both PoseOptimization calls ([2][n_frames + 1])
    size_t h_eoff_bytes = 0;
    // chained flow: Frame::isInFrustum outputs per local map point + the frame's Sophus::SE3f after the first PoseOptimization
    int chain_np = -1;
    uint8_t* d_cview = nullptr;
    float *d_cpx = nullptr, *d_cpy = nullptr, *d_cpxr = nullptr, *d_cvc = nullptr, *d_cdepth = nullptr, *d_posef = nullptr;
    int* d_clevel = nullptr;
};


// ---- the chained flow's glue kernels -------------------------------------------------------------------------------------
namespace orb {

// After the motion-model search and its PoseOptimization, one CTA per frame:
//   seen[q] = 1 for every LastFrame map point the search put into the frame (pMP->mnLastFrameSeen = mCurrentFrame.mnId,
//             Tracking.cc:3997-4000 -- set for outliers too, :3460);
//   features whose map point came out an outlier are released (mvpMapPoints[i] = NULL, Tracking.cc:3447-3470);
//   claimed[row] = the feature still holds a map point with Observations() > 0 (what ORBmatcher.cc:116-118 tests);
//   the optimised pose -> Sophus::SE3f (Optimizer.cc:406-410: rotation().cast<float>(), translation().cast<float>(); SO3's
//   constructor normalises the quaternion, so3.hpp:297-303, with Eigen's 4-float reduction (x^2 + z^2) + (y^2 + w^2)) ->
//   mRcw / mtcw / mOw (Frame::UpdatePoseMatrices, Frame.cc:592-599: Eigen's toRotationMatrix, Sophus' inverse()).
__global__ void __launch_bounds__(256) k_chain_after_motion(const int* __restrict__ fimg, const int* __restrict__ offsets, const int* __restrict__ nkp,
                                                            int maxFeat, const int* __restrict__ qoff, const uint8_t* __restrict__ obs,
                                                            const int* __restrict__ eoff, const int* __restrict__ efeat,
                                                            const uint8_t* __restrict__ outl, const double* __restrict__ pose1,
                                                            int* __restrict__ fm, uint8_t* __restrict__ seen, uint8_t* __restrict__ claimed,
                                                            float* __restrict__ posef, float* __restrict__ Rcw, float* __restrict__ tcw,
                                                            float* __restrict__ Ow) {
    const int f = blockIdx.x, img = fimg[f], row0 = offsets[img], N = min(nkp[img], maxFeat);
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const int q = fm[row0 + i];
        if (q >= 0) seen[q] = 1;            // q indexes the whole batch's query arrays: frames do not collide
    }
    __syncthreads();
    for (int e = eoff[f] + threadIdx.x; e < eoff[f + 1]; e += blockDim.x)
        if (outl[e]) fm[row0 + efeat[e]] = -1;
    __syncthreads();
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const int q = fm[row0 + i];
        claimed[row0 + i] = (q >= 0 && (!obs || obs[q])) ? 1 : 0;
    }
    if (threadIdx.x == 0) {
        const double* p = pose1 + 7 * f;
        float qx = (float)p[0], qy = (float)p[1], qz = (float)p[2], qw = (float)p[3];
        const float tx = (float)p[4], ty = (float)p[5], tz = (float)p[6];
        const float len = fsqrt(fadd(fadd(fmul(qx, qx), fmul(qz, qz)), fadd(fmul(qy, qy), fmul(qw, qw))));
        qx = fdiv(qx, len); qy = fdiv(qy, len); qz = fdiv(qz, len); qw = fdiv(qw, len);
        float* o = posef + 7 * f;
        o[0] = qx; o[1] = qy; o[2] = qz; o[3] = qw; o[4] = tx; o[5] = ty; o[6] = tz;
        // Eigen::QuaternionBase::toRotationMatrix
        const float t2x = fmul(2.f, qx), t2y = fmul(2.f, qy), t2z = fmul(2.f, qz);
        const float twx = fmul(t2x, qw), twy = fmul(t2y, qw), twz = fmul(t2z, qw);
        const float txx = fmul(t2x, qx), txy = fmul(t2y, qx), txz = fmul(t2z, qx), tyy = fmul(t2y, qy), tyz = fmul(t2z, qy), tzz = fmul(t2z, qz);
        float* R = Rcw + 9 * f;
        R[0] = fsub(1.f, fadd(tyy, tzz)); R[1] = fsub(txy, twz); R[2] = fadd(txz, twy);
        R[3] = fadd(txy, twz); R[4] = fsub(1.f, fadd(txx, tzz)); R[5] = fsub(tyz, twx);
        R[6] = fsub(txz, twy); R[7] = fadd(tyz, twx); R[8] = fsub(1.f, fadd(txx, tyy));
        tcw[3 * f] = tx; tcw[3 * f + 1] = ty; tcw[3 * f + 2] = tz;
        // mOw = mTcw.inverse().translation() = conj(q) * (t * -1)   (se3.hpp inverse(), so3.hpp:358-367 point action)
        const float ix = -qx, iy = -qy, iz = -qz, px = fmul(tx, -1.f), py = fmul(ty, -1.f), pz = fmul(tz, -1.f);
        const float uvx = fsub(fmul(iy, pz), fmul(iz, py)), uvy = fsub(fmul(iz, px), fmul(ix, pz)), uvz = fsub(fmul(ix, py), fmul(iy, px));
        const float ux = fadd(uvx, uvx), uy = fadd(uvy, uvy), uz = fadd(uvz, uvz);
        const float cx = fsub(fmul(iy, uz), fmul(iz, uy)), cy = fsub(fmul(iz, ux), fmul(ix, uz)), cz = fsub(fmul(ix, uy), fmul(iy, ux));
        Ow[3 * f] = fadd(fadd(px, fmul(qw, ux)), cx); Ow[3 * f + 1] = fadd(fadd(py, fmul(qw, uy)), cy); Ow[3 * f + 2] = fadd(fadd(pz, fmul(qw, uz)), cz);
    }
}

// local map points the motion-model search already put into the frame are not projected again (Tracking.cc:3997-4000, 4013-4014)
__global__ void __launch_bounds__(256) k_chain_skip_seen(const int* __restrict__ poff, const int* __restrict__ qoffL, const int* __restrict__ lastq,
                                                         const uint8_t* __restrict__ seen, uint8_t* __restrict__ in_view, float* __restrict__ px,
                                                         float* __restrict__ py, float* __restrict__ pxr, int* __restrict__ level,
                                                         float* __restrict__ vc, float* __restrict__ depth) {
    const int f = blockIdx.y, i = poff[f] + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= poff[f + 1]) return;
    const int lq = lastq[i];
    if (lq >= 0 && seen[qoffL[f] + lq]) { in_view[i] = 0; px[i] = -1.f; py[i] = -1.f; pxr[i] = -1.f; level[i] = -1; vc[i] = 0.f; depth[i] = 0.f; }
}

}  // namespace orb

void orbr_release(orbx_handle* h) {   // called by orbx_destroy
    if (!h || !h->replay) return;
    orbr_state* r = h->replay;
    if (r->d_buf) cudaFree(r->d_buf);
    if (r->ev_counts) cudaEventDestroy(r->ev_counts);
    if (r->h_eoff) cudaFreeHost(r->h_eoff);
    delete r;
    h->replay = nullptr;
}

extern "C" orb_status orbr_submit(orbx_handle* h, const orbm_camera* cam, const orbr_step* S) {
    if (!h || !cam || !S || S->n_frames < 1 || !S->images) return set_error(ORB_ERR_INVALID, "bad arguments");
    const bool mono = S->monocular != 0, rgbd = S->depth_maps != nullptr;
    if (mono && rgbd) return set_error(ORB_ERR_INVALID, "a step is monocular or RGB-D, not both");
    const int nf = S->n_frames, nimg = (mono || rgbd) ? nf : 2 * nf;   // monocular, RGB-D: image f is frame f; stereo: eyes 2f, 2f + 1
    if (nimg > h->cfg.max_batch)
        return set_error(ORB_ERR_INVALID, nimg == nf ? "n_frames exceeds the handle's max_batch" : "2 * n_frames exceeds the handle's max_batch");
    if (h->capturing) return set_error(ORB_ERR_INVALID, "orbr_submit cannot run inside a graph capture");
    const orbm_last_queries* QL = S->last;
    const orbm_local_queries* QC = S->local;
    if (QL && (QL->n_frames != nf || !QL->frame_image || !QL->query_offset || !QL->Tcw || !QL->direction)) return set_error(ORB_ERR_INVALID, "bad last-frame query set");
    if (QC && (QC->n_frames != nf || !QC->frame_image || !QC->query_offset)) return set_error(ORB_ERR_INVALID, "bad local-map query set");
    const orbr_chain* CH = S->chain;
    if (CH && (!QL || QC || !S->pose || !QL->world_pos || !CH->point_offset || !CH->world_pos || !CH->normal || !CH->max_dist || !CH->min_dist ||
               !CH->desc || !CH->last_query))
        return set_error(ORB_ERR_INVALID, "the chained flow needs `last` (with world positions), `pose`, no `local`, and every array of orbr_chain");
    if (S->pose_optimization && (!S->pose || (QL && !QL->world_pos) || (QC && !S->local_world_pos)))
        return set_error(ORB_ERR_INVALID, "pose_optimization needs pose and the world positions of the queries");
    // camera images as they arrive: converted to grey and resized on the device (orbx_extract_batch_device_format)
    ImageSource src{S->image_format, S->src_width, S->src_height, S->src_stride, S->src_image_stride_bytes};
    const bool ingest = src.format || src.w || src.h || src.stride || src.image_stride;
    if (ingest) {
        const orb_status s = check_source(src, S->width, S->height);
        if (s != ORB_OK) return s;
    }
    DepthSource dsrc{S->depth_format, S->depth_stride, S->depth_image_stride_bytes};
    if (rgbd) {
        if (ingest && (src.w != S->width || src.h != S->height))
            return set_error(ORB_ERR_UNSUPPORTED, "RGB-D camera images of another size than width x height: System::TrackRGBD's resize of the depth "
                                                  "map is not built");
        const orb_status s = check_depth(dsrc, nf, S->width, S->height);
        if (s != ORB_OK) return s;
    }
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    if (!h->replay) {
        h->replay = new orbr_state();
        ORB_CUDA(cudaEventCreateWithFlags(&h->replay->ev_counts, cudaEventDisableTiming));
    }
    orbr_state* r = h->replay;
    if (r->pending) return set_error(ORB_ERR_INVALID, "the previous step of this handle has not been collected");
    const int nqL = QL ? QL->query_offset[nf] : 0, nqC = QC ? QC->query_offset[nf] : (CH ? CH->point_offset[nf] : 0);
    int maxqL = 0, maxqC = 0;
    if (CH)
        for (int f = 0; f < nf; ++f) {
            if (CH->point_offset[f + 1] < CH->point_offset[f]) return set_error(ORB_ERR_INVALID, "bad point table");
            maxqC = std::max(maxqC, CH->point_offset[f + 1] - CH->point_offset[f]);
        }
    for (int f = 0; f < nf; ++f) {
        if (QL) {
            if (QL->query_offset[f + 1] < QL->query_offset[f] || QL->frame_image[f] < 0 || QL->frame_image[f] >= nimg) return set_error(ORB_ERR_INVALID, "bad frame table");
            // bMono: the monocular search never looks forward or backward (ORBmatcher.cc:1967-1971)
            if (mono && QL->direction[f] != 0) return set_error(ORB_ERR_INVALID, "a monocular step needs direction 0 for every frame");
            maxqL = std::max(maxqL, QL->query_offset[f + 1] - QL->query_offset[f]);
        }
        if (QC) {
            if (QC->query_offset[f + 1] < QC->query_offset[f] || QC->frame_image[f] < 0 || QC->frame_image[f] >= nimg) return set_error(ORB_ERR_INVALID, "bad frame table");
            maxqC = std::max(maxqC, QC->query_offset[f + 1] - QC->query_offset[f]);
        }
    }
    const size_t rows_cap = h->out_rows;   // compact rows a batch of max_batch images can produce
    const bool po = S->pose_optimization != 0 || CH != nullptr;
    cudaStream_t st = h->stream;
    // ---- both eyes of every frame through the extractor, then ComputeStereoMatches; or the one image of every monocular frame
    //      with vLappingArea = {0, 1000} (Frame.cc:380) and no stereo: mvuRight stays -1 for the searches and PoseOptimization; or the
    //      one image of every RGB-D frame with {0, 0}, then ComputeStereoFromRGBD from its depth map ----
    orb_status s = ingest ? extract_batch_source(h, S->images, nimg, S->width, S->height, src, 0, mono ? 1000 : 0)
                          : orbx_extract_batch(h, S->images, nimg, S->width, S->height, S->stride, S->image_stride_bytes, 0, mono ? 1000 : 0, nullptr, nullptr);
    if (s != ORB_OK) return s;
    if (rgbd) s = orbm_stereo_rgbd_batch(h, nf, S->depth_maps, dsrc.format, (int32_t)dsrc.stride, dsrc.image_stride, S->depth_factor, 0, S->bf);
    else if (!mono) s = orbm_stereo_batch(h, nf, S->bf, S->b);
    if (s != ORB_OK) return s;
    // ---- the step's device block, carved after the extraction is queued so that only the query copies precede the first search.
    //      The chained flow and the local-map flow share the frame table, offsets, descriptors and world positions of their queries ----
    struct Ptrs {
        int *fimgL, *qoffL, *dirL, *octL; float *tcwL, *xwL, *angL; uint8_t *descL, *obsL;
        int *fimgC, *qoffC, *lvlC; float *pxC, *pyC, *pxrC, *vcC, *tdC, *xwC; uint8_t *descC, *claimC, *viewC;
        float* pose;
        float *nrmK, *mxK, *mnK, *RcwK, *tcwK, *OwK; int* lastqK; uint8_t* seenK;
    } D{};
    const int* fimgC = CH ? QL->frame_image : QC ? QC->frame_image : nullptr;
    const int* qoffC = CH ? CH->point_offset : QC ? QC->query_offset : nullptr;
    const uint8_t* descC = CH ? CH->desc : QC ? QC->desc : nullptr;
    const float* xwC = CH ? CH->world_pos : po ? S->local_world_pos : nullptr;
    auto layout = [&](Carve& c) {
        if (QL) {
            D.fimgL = stage_in(c, QL->frame_image, nf, false); D.qoffL = stage_in(c, QL->query_offset, nf + 1, false);
            D.dirL = stage_in(c, QL->direction, nf, false); D.tcwL = stage_in(c, QL->Tcw, (size_t)nf * 7, false);
            D.xwL = stage_in(c, QL->world_pos, (size_t)nqL * 3, false); D.octL = stage_in(c, QL->last_octave, nqL, false);
            D.angL = stage_in(c, QL->last_angle, nqL, false); D.descL = stage_in(c, QL->desc, (size_t)nqL * 32, false);
            D.obsL = stage_in(c, QL->obs_positive, nqL, false);
        }
        D.fimgC = stage_in(c, fimgC, nf, false); D.qoffC = stage_in(c, qoffC, nf + 1, false);
        D.descC = stage_in(c, descC, (size_t)nqC * 32, false); D.xwC = stage_in(c, xwC, (size_t)nqC * 3, false);
        if (QC) {
            D.pxC = stage_in(c, QC->proj_x, nqC, false); D.pyC = stage_in(c, QC->proj_y, nqC, false); D.pxrC = stage_in(c, QC->proj_xr, nqC, false);
            D.lvlC = stage_in(c, QC->level, nqC, false); D.vcC = stage_in(c, QC->view_cos, nqC, false); D.tdC = stage_in(c, QC->track_depth, nqC, false);
            D.viewC = stage_in(c, QC->in_view, nqC, false);
        }
        if (CH) {
            D.nrmK = stage_in(c, CH->normal, (size_t)nqC * 3, false); D.mxK = stage_in(c, CH->max_dist, nqC, false);
            D.mnK = stage_in(c, CH->min_dist, nqC, false); D.lastqK = stage_in(c, CH->last_query, nqC, false);
        }
        D.pose = stage_in(c, po ? S->pose : nullptr, (size_t)nf * 7, false);
        D.claimC = c.take<uint8_t>(rows_cap);
        r->d_fm = c.take<int>(rows_cap); r->d_nm_last = c.take<int>(nf); r->d_match = c.take<int>(nqC); r->d_nm_local = c.take<int>(nf);
        for (int k = 0; k < 2; ++k) {
            r->d_eoff[k] = c.take<int>(nf + 1); r->d_efeat[k] = c.take<int>(po ? rows_cap : 1); r->d_inl[k] = c.take<int>(nf);
            r->d_pose[k] = c.take<double>((size_t)nf * 7); r->d_outl[k] = c.take<uint8_t>(po ? rows_cap : 1);
        }
        r->d_exw = c.take<float>(po ? rows_cap * 3 : 1); r->d_eobs = c.take<float>(po ? rows_cap * 3 : 1); r->d_ew = c.take<float>(po ? rows_cap : 1);
        const size_t npK = CH ? (size_t)nqC : 0;
        D.RcwK = c.take<float>((size_t)nf * 9); D.tcwK = c.take<float>((size_t)nf * 3); D.OwK = c.take<float>((size_t)nf * 3);
        D.seenK = c.take<uint8_t>(CH ? (size_t)nqL : 0);
        r->d_cview = c.take<uint8_t>(npK); r->d_cpx = c.take<float>(npK); r->d_cpy = c.take<float>(npK); r->d_cpxr = c.take<float>(npK);
        r->d_clevel = c.take<int>(npK); r->d_cvc = c.take<float>(npK); r->d_cdepth = c.take<float>(npK); r->d_posef = c.take<float>((size_t)nf * 7);
    };
    if ((s = carve_scratch(r->bytes, r->d_buf, h->capturing, st, layout).status) != ORB_OK ||
        (s = grow_pinned(r->h_eoff_bytes, r->h_eoff, sizeof(int) * 2 * (nf + 1))) != ORB_OK)
        return s;
    const int qb0 = h->q_total_bound, qb1 = h->q_frame_bound, qb2 = h->rows_bound;
    auto restore = [&]() { h->q_total_bound = qb0; h->q_frame_bound = qb1; h->rows_bound = qb2; };
    // ---- TrackWithMotionModel: SearchByProjection(cur, last) [+ PoseOptimization] ----
    if (QL) {
        orbm_last_queries q{};
        q.n_frames = nf; q.on_device = 1; q.frame_image = D.fimgL; q.query_offset = D.qoffL; q.Tcw = D.tcwL; q.direction = D.dirL;
        q.world_pos = D.xwL; q.last_octave = D.octL; q.last_angle = D.angL; q.desc = D.descL; q.obs_positive = D.obsL;
        h->q_total_bound = std::max(nqL, 1); h->q_frame_bound = std::max(maxqL, 1); h->rows_bound = (int)rows_cap;   // exact: the host tables are at hand
        s = orbm_search_last_frame(h, cam, &q, S->th_last, S->check_orientation_last, r->d_fm, r->d_nm_last);
        restore();
        if (s != ORB_OK) return s;
        if (po) {
            orbo_edge_source es{nf, D.fimgL, r->d_fm, nullptr, nullptr, D.xwL};
            if ((s = orbo_pose_edges(h, &es, r->d_eoff[0], r->d_efeat[0], r->d_exw, r->d_eobs, r->d_ew)) != ORB_OK) return s;
            orbo_pose_problems pp{nf, 1, r->d_eoff[0], D.pose, r->d_exw, r->d_eobs, r->d_ew, cam->fx, cam->fy, cam->cx, cam->cy, cam->bf, (int32_t)rows_cap};
            if ((s = orbo_pose_optimization(h, &pp, r->d_pose[0], r->d_outl[0], r->d_inl[0], nullptr)) != ORB_OK) return s;
            ORB_CUDA(cudaMemcpyAsync(r->h_eoff, r->d_eoff[0], sizeof(int) * (nf + 1), cudaMemcpyDeviceToHost, st));
        }
    }
    // ---- the chained flow: outlier release, pose -> Sophus::SE3f, isInFrustum, local-map search, second PoseOptimization ----
    if (CH) {
        ORB_CUDA(cudaMemsetAsync(D.seenK, 0, std::max(nqL, 1), st));
        k_chain_after_motion<<<nf, 256, 0, st>>>(D.fimgL, h->d_offsets, h->d_nkp, h->geom.kpTotal, D.qoffL, D.obsL, r->d_eoff[0],
                                                 r->d_efeat[0], r->d_outl[0], r->d_pose[0], r->d_fm, D.seenK, D.claimC, r->d_posef, D.RcwK, D.tcwK, D.OwK);
        ORB_LAUNCHED();
        orbf_frustum_points fp{};
        fp.n_frames = nf; fp.on_device = 1; fp.point_offset = D.qoffC; fp.Rcw = D.RcwK; fp.tcw = D.tcwK; fp.Ow = D.OwK; fp.world_pos = D.xwC;
        fp.normal = D.nrmK; fp.max_dist = D.mxK; fp.min_dist = D.mnK; fp.n_points_max = std::max(maxqC, 1);
        if ((s = orbf_is_in_frustum(h, cam, &fp, CH->viewing_cos_limit, r->d_cview, r->d_cpx, r->d_cpy, r->d_cpxr, r->d_clevel, r->d_cvc, r->d_cdepth)) != ORB_OK)
            return s;
        if (maxqC > 0) {
            k_chain_skip_seen<<<dim3((maxqC + 255) / 256, nf), 256, 0, st>>>(D.qoffC, D.qoffL, D.lastqK, D.seenK, r->d_cview, r->d_cpx, r->d_cpy, r->d_cpxr,
                                                                           r->d_clevel, r->d_cvc, r->d_cdepth);
            ORB_LAUNCHED();
        }
        orbm_local_queries q{};
        q.n_frames = nf; q.on_device = 1; q.frame_image = D.fimgC; q.query_offset = D.qoffC; q.proj_x = r->d_cpx; q.proj_y = r->d_cpy; q.proj_xr = r->d_cpxr;
        q.level = r->d_clevel; q.view_cos = r->d_cvc; q.track_depth = r->d_cdepth; q.desc = D.descC; q.feature_claimed = D.claimC; q.in_view = r->d_cview;
        h->q_total_bound = std::max(nqC, 1); h->q_frame_bound = std::max(maxqC, 1); h->rows_bound = (int)rows_cap;
        s = orbm_search_local_points(h, cam, &q, S->th_local, S->nnratio_local, S->far_points, S->th_far, r->d_match, r->d_nm_local);
        restore();
        if (s != ORB_OK) return s;
        // PoseOptimization over every map point the frame holds now: the motion-model survivors and the local-map matches
        orbo_edge_source es{nf, D.fimgC, r->d_fm, D.qoffC, r->d_match, D.xwL, D.xwC};
        if ((s = orbo_pose_edges(h, &es, r->d_eoff[1], r->d_efeat[1], r->d_exw, r->d_eobs, r->d_ew)) != ORB_OK) return s;
        orbo_pose_problems pp{nf, 1, r->d_eoff[1], r->d_posef, r->d_exw, r->d_eobs, r->d_ew, cam->fx, cam->fy, cam->cx, cam->cy, cam->bf, (int32_t)rows_cap};
        if ((s = orbo_pose_optimization(h, &pp, r->d_pose[1], r->d_outl[1], r->d_inl[1], nullptr)) != ORB_OK) return s;
        ORB_CUDA(cudaMemcpyAsync(r->h_eoff + (nf + 1), r->d_eoff[1], sizeof(int) * (nf + 1), cudaMemcpyDeviceToHost, st));
        ORB_CUDA(cudaGetLastError());
    }
    // ---- TrackLocalMap: SearchByProjection(F, local map points) [+ PoseOptimization] ----
    if (QC) {
        if (QC->feature_claimed) return set_error(ORB_ERR_UNSUPPORTED, "orbr_submit: feature_claimed refers to rows that do not exist yet; pass NULL");
        orbm_local_queries q{};
        q.n_frames = nf; q.on_device = 1; q.frame_image = D.fimgC; q.query_offset = D.qoffC; q.proj_x = D.pxC; q.proj_y = D.pyC; q.proj_xr = D.pxrC;
        q.level = D.lvlC; q.view_cos = D.vcC; q.track_depth = D.tdC; q.desc = D.descC; q.feature_claimed = nullptr;
        q.in_view = D.viewC;
        h->q_total_bound = std::max(nqC, 1); h->q_frame_bound = std::max(maxqC, 1); h->rows_bound = (int)rows_cap;
        s = orbm_search_local_points(h, cam, &q, S->th_local, S->nnratio_local, S->far_points, S->th_far, r->d_match, r->d_nm_local);
        restore();
        if (s != ORB_OK) return s;
        if (po) {
            orbo_edge_source es{nf, D.fimgC, nullptr, D.qoffC, r->d_match, D.xwC};
            if ((s = orbo_pose_edges(h, &es, r->d_eoff[1], r->d_efeat[1], r->d_exw, r->d_eobs, r->d_ew)) != ORB_OK) return s;
            orbo_pose_problems pp{nf, 1, r->d_eoff[1], D.pose, r->d_exw, r->d_eobs, r->d_ew, cam->fx, cam->fy, cam->cx, cam->cy, cam->bf, (int32_t)rows_cap};
            if ((s = orbo_pose_optimization(h, &pp, r->d_pose[1], r->d_outl[1], r->d_inl[1], nullptr)) != ORB_OK) return s;
            ORB_CUDA(cudaMemcpyAsync(r->h_eoff + (nf + 1), r->d_eoff[1], sizeof(int) * (nf + 1), cudaMemcpyDeviceToHost, st));
        }
    }
    // ---- the small tables back: per-image counts / offsets and the capacity flags ----
    if ((s = queue_counts(h)) != ORB_OK) return s;
    ORB_CUDA(cudaEventRecord(r->ev_counts, st));
    r->pending = true;
    r->n_frames = nf; r->nimg = nimg; r->mono = mono;
    r->nq_last = QL ? nqL : -1; r->nq_local = (QC || CH) ? nqC : -1; r->with_po = po ? 1 : 0; r->chain_np = CH ? nqC : -1;
    return ORB_OK;
}

extern "C" orb_status orbr_collect(orbx_handle* h, const orbr_results* O, int32_t* total_rows_out) {
    if (!h || !O || !h->replay || !h->replay->pending) return set_error(ORB_ERR_INVALID, "no submitted step to collect");
    orbr_state* r = h->replay;
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    ORB_CUDA(cudaEventSynchronize(r->ev_counts));
    r->pending = false;
    const int nimg = r->nimg, nf = r->n_frames;
    orb_status s = latch_counts(h);
    if (s != ORB_OK) return s;
    const int rows = image_row0(h, nimg);
    if (total_rows_out) *total_rows_out = rows;
    if (O->n) for (int b = 0; b < nimg; ++b) O->n[b] = image_features(h, b);
    if (O->offsets) for (int b = 0; b <= nimg; ++b) O->offsets[b] = image_row0(h, b);
    if (rows > O->cap_rows) return set_error(ORB_ERR_CAPACITY, "result buffers smaller than the batch result");
    cudaStream_t st = h->stream;
    auto down = [&](void* dst, const void* src, size_t bytes) -> orb_status {
        if (dst && bytes) ORB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st));
        return ORB_OK;
    };
    if ((s = down(O->keypoints, h->d_kps, sizeof(orbx_keypoint) * (size_t)rows)) != ORB_OK || (s = down(O->descriptors, h->d_desc, 32 * (size_t)rows)) != ORB_OK)
        return s;
    if (r->mono) {   // the monocular Frame stores mvuRight = mvDepth = -1; d_uright may still hold an earlier stereo batch
        if (O->uright) std::fill(O->uright, O->uright + rows, -1.0f);
        if (O->depth) std::fill(O->depth, O->depth + rows, -1.0f);
    } else if ((s = down(O->uright, h->d_uright, 4 * (size_t)rows)) != ORB_OK || (s = down(O->depth, h->d_depth, 4 * (size_t)rows)) != ORB_OK)
        return s;
    if (r->nq_last >= 0) {
        if ((s = down(O->last_feature_match, r->d_fm, 4 * (size_t)rows)) != ORB_OK || (s = down(O->last_nmatches, r->d_nm_last, 4 * (size_t)nf)) != ORB_OK) return s;
    }
    if (r->nq_local >= 0) {
        if ((s = down(O->local_match, r->d_match, 4 * (size_t)r->nq_local)) != ORB_OK || (s = down(O->local_nmatches, r->d_nm_local, 4 * (size_t)nf)) != ORB_OK) return s;
    }
    if (r->with_po) {
        for (int k = 0; k < 2; ++k) {
            if ((k == 0 ? r->nq_last : r->nq_local) < 0) continue;
            const int* eoff = r->h_eoff + k * (nf + 1);
            const int ne = eoff[nf];
            if (ne > O->cap_rows) return set_error(ORB_ERR_CAPACITY, "edge buffers smaller than the result");
            if (O->edge_offset[k]) memcpy(O->edge_offset[k], eoff, sizeof(int) * (nf + 1));
            if ((s = down(O->pose[k], r->d_pose[k], 56 * (size_t)nf)) != ORB_OK || (s = down(O->inliers[k], r->d_inl[k], 4 * (size_t)nf)) != ORB_OK ||
                (s = down(O->edge_feature[k], r->d_efeat[k], 4 * (size_t)ne)) != ORB_OK || (s = down(O->edge_outlier[k], r->d_outl[k], (size_t)ne)) != ORB_OK)
                return s;
        }
    }
    if (r->chain_np >= 0) {
        const size_t np = (size_t)r->chain_np;
        if ((s = down(O->chain_in_view, r->d_cview, np)) != ORB_OK || (s = down(O->chain_proj_x, r->d_cpx, 4 * np)) != ORB_OK ||
            (s = down(O->chain_proj_y, r->d_cpy, 4 * np)) != ORB_OK || (s = down(O->chain_proj_xr, r->d_cpxr, 4 * np)) != ORB_OK ||
            (s = down(O->chain_level, r->d_clevel, 4 * np)) != ORB_OK || (s = down(O->chain_view_cos, r->d_cvc, 4 * np)) != ORB_OK ||
            (s = down(O->chain_pose_f, r->d_posef, 28 * (size_t)nf)) != ORB_OK)
            return s;
    }
    ORB_CUDA(cudaStreamSynchronize(st));
    return ORB_OK;
}

// ---- keyframe state of one frame as a fixed-capacity block in device memory (what replicas sharing a map exchange) ----------
// KeyFrame::KeyFrame(Frame&) (KeyFrame.cc:45-90) keeps mvKeysUn, mvuRight, mDescriptors and the pose of the frame; this is that
// state in the layout of replay.pack_keyframe: [int32 n][pose 7 x f32][n x (x, y) f32][n x octave i32][n x uright f32][n x 32 B].
namespace orb {
__global__ void __launch_bounds__(256) k_pack_keyframe(const orbx_keypoint* __restrict__ kps, const uint8_t* __restrict__ desc,
                                                       const float* __restrict__ uright, const int* __restrict__ nkp,
                                                       const int* __restrict__ offsets, int image, const float* __restrict__ pose7,
                                                       uint8_t* __restrict__ block, int cap) {
    const int n = min(nkp[image], cap), row0 = offsets[image];
    if (blockIdx.x == 0 && threadIdx.x < 8) {
        if (threadIdx.x == 0) reinterpret_cast<int*>(block)[0] = n;
        else reinterpret_cast<float*>(block)[threadIdx.x] = pose7[threadIdx.x - 1];
    }
    float2* xy = reinterpret_cast<float2*>(block + 32);
    int* oct = reinterpret_cast<int*>(block + 32 + 8 * (size_t)n);
    float* ur = reinterpret_cast<float*>(block + 32 + 12 * (size_t)n);
    uint4* dd = reinterpret_cast<uint4*>(block + 32 + 16 * (size_t)n);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const orbx_keypoint k = kps[row0 + i];
        xy[i] = make_float2(k.x, k.y);
        oct[i] = k.octave;
        ur[i] = uright ? uright[row0 + i] : -1.f;
        const uint4* s = reinterpret_cast<const uint4*>(desc + 32 * (size_t)(row0 + i));
        dd[2 * i] = s[0];
        dd[2 * i + 1] = s[1];
    }
}
}  // namespace orb

extern "C" size_t orbx_keyframe_block_bytes(const orbx_handle* h) {
    return h ? 32 + (size_t)orbx_max_features(h) * 48 : 0;
}

extern "C" orb_status orbx_pack_keyframe_device(orbx_handle* h, int32_t image, const float* d_pose7, uint8_t* d_block, size_t block_bytes) {
    if (!h || !d_pose7 || !d_block || image < 0 || image >= h->last_batch) return set_error(ORB_ERR_INVALID, "bad arguments");
    if (block_bytes < orbx_keyframe_block_bytes(h) || ((uintptr_t)d_block & 15)) return set_error(ORB_ERR_INVALID, "block too small or not 16-byte aligned");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    k_pack_keyframe<<<8, 256, 0, h->stream>>>(h->d_kps, h->d_desc, h->stereo_valid ? h->d_uright : nullptr, h->d_nkp, h->d_offsets, image, d_pose7,
                                              d_block, orbx_max_features(h));
    ORB_LAUNCHED();
    ORB_CUDA(cudaGetLastError());
    return ORB_OK;
}
