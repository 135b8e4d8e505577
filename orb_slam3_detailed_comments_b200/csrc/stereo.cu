// stereo.cu -- Frame::ComputeStereoMatches (/root/reference/src/Frame.cc:1102-1358) and Frame::ComputeStereoFromRGBD on the device.
// One warp per LEFT keypoint: lanes stride over the right image's keypoints (row-band, octave and
// disparity-range gates, then 256-bit Hamming with __popc), shuffle arg-min with index tie-break
// (= "first strictly smaller" in ascending right index), 11x11 SAD over 11 shifts on the raw pyramid
// level, parabola refinement.  A second kernel applies the 2.1 * median SAD filter per frame.
#include <algorithm>

#include <stdlib.h>

#include "extractor.h"
#include "devmath.cuh"
#include "stereo_core.cuh"
#include "rgbd_core.cuh"

using namespace orb;
using namespace orbdev;

namespace orb {

struct StereoSide {
    const orbx_keypoint* kps;
    const uint8_t* desc;
    const int* offsets;  // first compact row of every image
    const int* nkp;
};

struct StereoParams {
    StereoSide L, R;
    int strideL, baseL, strideR, baseR;  // image index of pair p: p*stride + base
    float bf, b;
    float* uright;   // indexed by LEFT compact row
    float* depth;
    int* sad;
    int maxRight;    // capacity of the shared-memory staging of right keypoints
};

#define ST_WARPS 8

__global__ void __launch_bounds__(ST_WARPS * 32) k_stereo_match(const __grid_constant__ StereoParams P,
                                                               const __grid_constant__ ExtractGeom gL,
                                                               const __grid_constant__ ExtractGeom gR) {
    extern __shared__ __align__(16) unsigned char st_smem[];
    const int pair = blockIdx.y;
    const int imgL = pair * P.strideL + P.baseL, imgR = pair * P.strideR + P.baseR;
    const int N = P.L.nkp[imgL], Nr = min(P.R.nkp[imgR], P.maxRight);
    const int rowL0 = P.L.offsets[imgL], rowR0 = P.R.offsets[imgR];
    if (blockIdx.x * ST_WARPS >= N) return;
    // stage the right keypoints: x, (minr | maxr << 16), octave   (Frame.cc:1134-1156)
    float* s_x = reinterpret_cast<float*>(st_smem);
    int* s_band = reinterpret_cast<int*>(st_smem + 4 * (size_t)P.maxRight);
    int8_t* s_oct = reinterpret_cast<int8_t*>(st_smem + 8 * (size_t)P.maxRight);
    for (int j = threadIdx.x; j < Nr; j += blockDim.x) {
        const orbx_keypoint k = P.R.kps[rowR0 + j];
        const float r = fmul(2.0f, gR.lv[k.octave].scale);   // mvScaleFactors of the frame (= left extractor's)
        const int maxr = (int)ceilf(fadd(k.y, r)), minr = (int)floorf(fsub(k.y, r));
        s_x[j] = k.x;
        s_band[j] = (minr & 0xffff) | (maxr << 16);
        s_oct[j] = (int8_t)k.octave;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int iL = blockIdx.x * ST_WARPS + (threadIdx.x >> 5);
    if (iL >= N) return;
    const int rowL = rowL0 + iL;
    const orbx_keypoint kpL = P.L.kps[rowL];
    float out_u = -1.0f, out_d = -1.0f;
    int out_sad = -1;
    const float minZ = P.b, maxD = fdiv(P.bf, minZ);
    const float uL = kpL.x, vL = kpL.y;
    const int vLi = (int)vL;
    const float minU = fsub(uL, maxD), maxU = uL;
    uint32_t best = (100u << 16) | 0xffffu;   // TH_HIGH, ORBmatcher.cc:36
    if (!(maxU < 0)) {
        const uint4* dl = reinterpret_cast<const uint4*>(P.L.desc + (size_t)rowL * 32);
        const uint4 a0 = __ldg(dl), a1 = __ldg(dl + 1);
        for (int j = lane; j < Nr; j += 32) {
            const int band = s_band[j];
            const int minr = (int)(int16_t)(band & 0xffff), maxr = band >> 16;
            const int oc = s_oct[j];
            const float uR = s_x[j];
            if (vLi < minr || vLi > maxr) continue;
            if (oc < kpL.octave - 1 || oc > kpL.octave + 1) continue;
            if (!(uR >= minU && uR <= maxU)) continue;
            const uint4* dr = reinterpret_cast<const uint4*>(P.R.desc + (size_t)(rowR0 + j) * 32);
            const uint4 b0 = __ldg(dr), b1 = __ldg(dr + 1);
            const uint32_t d = __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
                               __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
            const uint32_t key = (d << 16) | (uint32_t)j;
            best = min(best, key);   // equal distance keeps the smaller right index: strict '<' in ascending order
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
    const int bestDist = (int)(best >> 16), bestIdxR = (int)(best & 0xffffu);
    if (bestDist < 75 && bestDist < 100) {   // thOrbDist = (TH_HIGH + TH_LOW) / 2
        const float uR0 = s_x[bestIdxR];
        const int oct = kpL.octave;
        const float sf = gL.lv[oct].inv_scale;
        const float scaleduL = roundf(fmul(kpL.x, sf)), scaledvL = roundf(fmul(kpL.y, sf)), scaleduR0 = roundf(fmul(uR0, sf));
        const LevelGeom& GL = gL.lv[oct];
        const LevelGeom& GR = gR.lv[oct];
        const float iniu = scaleduR0, endu = fadd(scaleduR0, 11.0f);   // scaleduR0 + L - w, scaleduR0 + L + w + 1
        if (!(iniu < 0 || endu >= (float)GR.w)) {
            const int cy = (int)scaledvL, cxL = (int)scaleduL, cxR = (int)scaleduR0;
            int part[11];
#pragma unroll
            for (int s = 0; s < 11; ++s) part[s] = 0;
            if (lane < 11) {
                const int y = cy + lane - 5;
                const uint8_t* pl = GL.base + (int64_t)imgL * GL.img_stride + (int64_t)y * GL.pitch + (cxL - 5);
                const uint8_t* pr = GR.base + (int64_t)imgR * GR.img_stride + (int64_t)y * GR.pitch + (cxR - 10);
                int l[11], r[21];
#pragma unroll
                for (int k = 0; k < 11; ++k) l[k] = __ldg(pl + k);
#pragma unroll
                for (int k = 0; k < 21; ++k) r[k] = __ldg(pr + k);
#pragma unroll
                for (int s = 0; s < 11; ++s) {
                    int acc = 0;
#pragma unroll
                    for (int k = 0; k < 11; ++k) acc += abs(l[k] - r[s + k]);
                    part[s] = acc;
                }
            }
            int bestSad = 0x7fffffff, bestinc = 0;
            float dists[11];
#pragma unroll
            for (int s = 0; s < 11; ++s) {
                int v = part[s];
#pragma unroll
                for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);   // lanes 0..15 hold the rows
                v = __shfl_sync(0xffffffffu, v, 0);
                dists[s] = (float)v;
                if (v < bestSad) {   // (float)dist < (int)bestDist with exact small integers
                    bestSad = v;
                    bestinc = s - 5;
                }
            }
            if (bestinc != -5 && bestinc != 5) {
                const float d1 = dists[5 + bestinc - 1], d2 = dists[5 + bestinc], d3 = dists[5 + bestinc + 1];
                const float deltaR = fdiv(fsub(d1, d3), fmul(2.0f, fsub(fadd(d1, d3), fmul(2.0f, d2))));
                if (!(deltaR < -1 || deltaR > 1)) {
                    float bestuR = fmul(GL.scale, fadd(fadd(scaleduR0, (float)bestinc), deltaR));
                    float disparity = fsub(uL, bestuR);
                    if (disparity >= 0 && disparity < maxD) {
                        if (disparity <= 0) {
                            disparity = 0.01f;
                            bestuR = (float)((double)uL - 0.01);
                        }
                        out_d = fdiv(P.bf, disparity);
                        out_u = bestuR;
                        out_sad = bestSad;
                    }
                }
            }
        }
    }
    if (lane == 0) {
        P.uright[rowL] = out_u;
        P.depth[rowL] = out_d;
        P.sad[rowL] = out_sad;
    }
}

// Variant 1 (the default; ORB_STEREO_VARIANT=0 selects k_stereo_match; host-emulated in tests/host_emul, device parity in tests/test_zz_stereo_v1_gpu.py): one THREAD per left keypoint,
// the right keypoints bucketed by image row once per CTA -- see stereo_core.cuh.  k_stereo_match above keeps its round-1 machine code.
#define ST1_THREADS 128

__global__ void __launch_bounds__(ST1_THREADS) k_stereo_match_v1(const __grid_constant__ StereoParams P,
                                                               const __grid_constant__ ExtractGeom gL,
                                                               const __grid_constant__ ExtractGeom gR) {
    extern __shared__ __align__(16) unsigned char st_smem[];
    __shared__ StLevel s_lv[ORB_MAX_LEVELS];
    const int pair = blockIdx.y;
    const int imgL = pair * P.strideL + P.baseL, imgR = pair * P.strideR + P.baseR;
    const int N = P.L.nkp[imgL], Nr = min(P.R.nkp[imgR], P.maxRight);
    const int rowL0 = P.L.offsets[imgL], rowR0 = P.R.offsets[imgR];
    if ((int)(blockIdx.x * ST1_THREADS) >= N) return;     // uniform per CTA
    const int H = gR.lv[0].h;
    float* s_x = reinterpret_cast<float*>(st_smem);
    int* s_band = reinterpret_cast<int*>(st_smem + 4 * (size_t)P.maxRight);
    int* s_ent = reinterpret_cast<int*>(st_smem + 8 * (size_t)P.maxRight);
    int* s_off = reinterpret_cast<int*>(st_smem + 12 * (size_t)P.maxRight);          // H + 1 offsets
    int* s_cur = s_off + (H + 1);                                                     // H fill cursors
    signed char* s_oct = reinterpret_cast<signed char*>(s_cur + H);
    for (int i = threadIdx.x; i <= H; i += blockDim.x) s_off[i] = 0;
    if (threadIdx.x < gL.nlevels) {
        const int l = threadIdx.x;
        StLevel v;
        v.L = gL.lv[l].base + (int64_t)imgL * gL.lv[l].img_stride;
        v.R = gR.lv[l].base + (int64_t)imgR * gR.lv[l].img_stride;
        v.pitchL = gL.lv[l].pitch; v.pitchR = gR.lv[l].pitch; v.wR = gR.lv[l].w;
        v.scale = gL.lv[l].scale; v.inv_scale = gL.lv[l].inv_scale;
        s_lv[l] = v;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < Nr; j += blockDim.x) {   // stage + count: x, (minr | maxr << 16), octave   (Frame.cc:1134-1156)
        const orbx_keypoint k = P.R.kps[rowR0 + j];
        const float r = fmul(2.0f, gR.lv[k.octave].scale);
        const int maxr = (int)ceilf(fadd(k.y, r)), minr = (int)floorf(fsub(k.y, r));
        s_x[j] = k.x;
        s_band[j] = (minr & 0xffff) | (maxr << 16);
        s_oct[j] = (signed char)k.octave;
        atomicAdd(&s_off[st_row_bucket(k.y, H) + 1], 1);
    }
    __syncthreads();
    if (threadIdx.x < 32) {                                 // inclusive scan of the H bucket counts by one warp
        int carry = 0;
        for (int base = 1; base <= H; base += 32) {
            const int i = base + (int)threadIdx.x;
            int v = i <= H ? s_off[i] : 0;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, v, o);
                if ((int)threadIdx.x >= o) v += u;
            }
            if (i <= H) s_off[i] = v + carry;
            carry += __shfl_sync(0xffffffffu, v, 31);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < H; i += blockDim.x) s_cur[i] = s_off[i];
    __syncthreads();
    for (int j = threadIdx.x; j < Nr; j += blockDim.x) {
        const int bkt = st_row_bucket(P.R.kps[rowR0 + j].y, H);
        s_ent[atomicAdd(&s_cur[bkt], 1)] = j;
    }
    __syncthreads();
    const int iL = blockIdx.x * ST1_THREADS + threadIdx.x;
    if (iL >= N) return;
    StRight R;
    R.x = s_x; R.band = s_band; R.oct = s_oct; R.row_off = s_off; R.row_ent = s_ent;
    R.H = H; R.W = st_scan_window(gR.lv[gR.nlevels - 1].scale);
    const int rowL = rowL0 + iL;
    const orbx_keypoint kpL = P.L.kps[rowL];
    float u, d;
    int sad;
    stereo_match_one(kpL.x, kpL.y, kpL.octave, reinterpret_cast<const uint32_t*>(P.L.desc + (size_t)rowL * 32), R,
                     P.R.desc + (size_t)rowR0 * 32, s_lv, P.bf, P.b, &u, &d, &sad);
    P.uright[rowL] = u;
    P.depth[rowL] = d;
    P.sad[rowL] = sad;
}

// Frame.cc:1338-1357: drop matches whose SAD >= 1.5 * 1.4 * median SAD.  One CTA per frame.
__global__ void __launch_bounds__(256) k_stereo_median(const __grid_constant__ StereoParams P) {
    extern __shared__ int md_sad[];
    __shared__ int s_cnt, s_median;
    const int imgL = blockIdx.x * P.strideL + P.baseL;
    const int N = P.L.nkp[imgL], row0 = P.L.offsets[imgL];
    if (threadIdx.x == 0) { s_cnt = 0; s_median = -1; }
    for (int i = threadIdx.x; i < N; i += blockDim.x) md_sad[i] = P.sad[row0 + i];
    __syncthreads();
    int local = 0;
    for (int i = threadIdx.x; i < N; i += blockDim.x) local += md_sad[i] >= 0;
    if (local) atomicAdd(&s_cnt, local);
    __syncthreads();
    const int cnt = s_cnt;
    if (cnt == 0) return;
    const int target = cnt / 2;   // vDistIdx[vDistIdx.size() / 2] of the (SAD, iL)-sorted pairs: only its SAD matters
    // two-pass radix select on the 16-bit SAD (<= 121 * 255): high byte, then low byte
    __shared__ int s_hist[256];
    __shared__ int s_hi, s_rem;
    for (int pass = 0; pass < 2; ++pass) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) s_hist[i] = 0;
        __syncthreads();
        for (int i = threadIdx.x; i < N; i += blockDim.x) {
            const int v = md_sad[i];
            if (v < 0) continue;
            if (pass == 0) atomicAdd(&s_hist[(v >> 8) & 0xff], 1);
            else if ((v >> 8) == s_hi) atomicAdd(&s_hist[v & 0xff], 1);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int rem = pass == 0 ? target : s_rem, b = 0;
            while (b < 255 && rem >= s_hist[b]) { rem -= s_hist[b]; ++b; }
            if (pass == 0) { s_hi = b; s_rem = rem; }
            else s_median = (s_hi << 8) | b;
        }
        __syncthreads();
    }
    const float thDist = fmul(1.5f * 1.4f, (float)s_median);
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const int v = md_sad[i];
        if (v >= 0 && !((float)v < thDist)) {
            P.uright[row0 + i] = -1.0f;
            P.depth[row0 + i] = -1.0f;
        }
    }
}

}  // namespace orb

static orb_status run_stereo(orbx_handle* hl, orbx_handle* hr, int n_pairs, int strideL, int baseL, int strideR, int baseR,
                             float bf, float b) {
    if (!hl || !hr || n_pairs < 1) return set_error(ORB_ERR_INVALID, "bad stereo arguments");
    if (hl->last_batch < (n_pairs - 1) * strideL + baseL + 1 || hr->last_batch < (n_pairs - 1) * strideR + baseR + 1)
        return set_error(ORB_ERR_INVALID, "stereo pairs exceed the last extracted batch");
    if (hl->cfg.device != hr->cfg.device || hl->cur_w != hr->cur_w || hl->cur_h != hr->cur_h ||
        hl->cfg.n_levels != hr->cfg.n_levels)
        return set_error(ORB_ERR_INVALID, "left/right extractors must share device, image size and pyramid");
    if (!(b > 0.f)) return set_error(ORB_ERR_INVALID, "baseline must be positive");
    ORB_CUDA(cudaSetDevice(hl->cfg.device));
    const char* venv = getenv("ORB_STEREO_VARIANT");      // read at every call: a test can switch variants inside one process
    const int variant = venv && atoi(venv) == 0 ? 0 : 1;   // default 1 (k_stereo_match_v1) since its round-2 device run
    const size_t maxRight = hr->geom.kpTotal, H = hr->geom.lv[0].h;
    const size_t smem1 = 13 * maxRight + 4 * (2 * H + 2) + 64, smem = 9 * maxRight + 16, smem2 = 4 * (size_t)hl->geom.kpTotal + 16;
    static const size_t v1Static = static_smem(k_stereo_match_v1), v0Static = static_smem(k_stereo_match), medStatic = static_smem(k_stereo_median);
    orb_status s;
    if ((s = variant == 1 ? check_smem(hl, smem1, v1Static, "k_stereo_match_v1") : check_smem(hl, smem, v0Static, "k_stereo_match")) != ORB_OK ||
        (s = check_smem(hl, smem2, medStatic, "k_stereo_median")) != ORB_OK)
        return s;
    cudaStream_t st = hl->stream;
    if (hr != hl) {   // order after the right extractor's work
        ORB_CUDA(cudaEventRecord(hr->ev_fork, hr->stream));
        ORB_CUDA(cudaStreamWaitEvent(st, hr->ev_fork, 0));
    }
    StereoParams P;
    P.L = {hl->d_kps, hl->d_desc, hl->d_offsets, hl->d_nkp};
    P.R = {hr->d_kps, hr->d_desc, hr->d_offsets, hr->d_nkp};
    P.strideL = strideL; P.baseL = baseL; P.strideR = strideR; P.baseR = baseR;
    P.bf = bf; P.b = b;
    P.uright = hl->d_uright; P.depth = hl->d_depth; P.sad = hl->d_sad;
    P.maxRight = hr->geom.kpTotal;
    if (variant == 1) {
        ORB_CUDA(cudaFuncSetAttribute(k_stereo_match_v1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(smem1, (size_t)1024)));
        dim3 grid1((hl->geom.kpTotal + ST1_THREADS - 1) / ST1_THREADS, n_pairs);
        launch_p(k_stereo_match_v1, grid1, dim3(ST1_THREADS), smem1, st, P, hl->geom, hr->geom);
    } else {
        ORB_CUDA(cudaFuncSetAttribute(k_stereo_match, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(smem, (size_t)1024)));
        dim3 grid((hl->geom.kpTotal + ST_WARPS - 1) / ST_WARPS, n_pairs);
        k_stereo_match<<<grid, ST_WARPS * 32, smem, st>>>(P, hl->geom, hr->geom);
    }
    ORB_LAUNCHED();
    ORB_CUDA(cudaFuncSetAttribute(k_stereo_median, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(smem2, (size_t)1024)));
    launch_p(k_stereo_median, dim3(n_pairs), dim3(256), smem2, st, P);
    ORB_LAUNCHED();
    ORB_CUDA(cudaGetLastError());
    hl->stereo_valid = true;
    return ORB_OK;
}

extern "C" orb_status orbm_stereo_batch(orbx_handle* h, int32_t n_pairs, float bf, float b) {
    return run_stereo(h, h, n_pairs, 2, 0, 2, 1, bf, b);
}

// the uright / depth rows [0, n) of the last stereo batch, as many as the caller's `cap` rows hold
static orb_status download_stereo_rows(orbx_handle* h, int n, float* uright, float* depth, int32_t cap, const char* too_small) {
    const int rows = std::min(n, (int)cap);
    if (rows > 0) {
        if (uright) ORB_CUDA(cudaMemcpyAsync(uright, h->d_uright, sizeof(float) * (size_t)rows, cudaMemcpyDeviceToHost, h->stream));
        if (depth) ORB_CUDA(cudaMemcpyAsync(depth, h->d_depth, sizeof(float) * (size_t)rows, cudaMemcpyDeviceToHost, h->stream));
        ORB_CUDA(cudaStreamSynchronize(h->stream));
    }
    return n > cap ? set_error(ORB_ERR_CAPACITY, too_small) : ORB_OK;
}

extern "C" orb_status orbm_stereo_download(orbx_handle* h, float* uright, float* depth, int32_t cap_rows) {
    int total = 0;
    orb_status s = batch_rows(h, &total);
    if (s != ORB_OK) return s;
    return download_stereo_rows(h, total, uright, depth, cap_rows, "output buffer smaller than the batch result");
}

extern "C" orb_status orbm_stereo_pair(orbx_handle* left, orbx_handle* right, float bf, float b, float* uright, float* depth,
                                       int32_t cap) {
    orb_status s = run_stereo(left, right, 1, 1, 0, 1, 0, bf, b);
    if (s != ORB_OK) return s;
    s = orbx_counts(left, nullptr, nullptr, nullptr);
    if (s != ORB_OK) return s;
    return download_stereo_rows(left, image_features(left, 0), uright, depth, cap, "output buffer smaller than N");
}

// ---- Frame::ComputeStereoFromRGBD ----------------------------------------------------------------------------------------------------
namespace orb {

// One thread per keypoint row of each image (rgbd_core.cuh rgbd_row); blockIdx.y is the image.  Only the sampled depth pixels are
// read and converted.
__global__ void __launch_bounds__(128) k_stereo_rgbd(const __grid_constant__ orbdev::RgbdPlan P) {
    const int img = blockIdx.y, i = blockIdx.x * 128 + threadIdx.x;
    if (i >= P.nkp[img]) return;
    const int row = P.offsets[img] + i;
    const float x = P.kps[row].x, y = P.kps[row].y;
    float u, d;
    orbdev::rgbd_row(P.depth + (int64_t)img * P.image_stride, P.stride, P.format, P.scaled != 0, P.factor, x, y, P.bf, &u, &d);
    P.uright[row] = u;
    P.depth_out[row] = d;
}

}  // namespace orb

orb_status check_depth(DepthSource& d, int n_images, int w, int hh) {
    if (d.format != ORB_DEPTH_U16 && d.format != ORB_DEPTH_F32) return set_error(ORB_ERR_INVALID, "unknown depth format");
    const int64_t elem = d.format == ORB_DEPTH_U16 ? 2 : 4, row = (int64_t)w * elem;
    if (d.stride == 0) d.stride = row;
    if (d.image_stride == 0) d.image_stride = (size_t)d.stride * hh;
    if (d.stride < row || d.stride > INT32_MAX || d.stride % elem || d.image_stride % elem ||
        (n_images > 1 && d.image_stride < (size_t)d.stride * hh))
        return set_error(ORB_ERR_INVALID, "depth stride shorter than a row (or a map) or not a multiple of the element size");
    return ORB_OK;
}

extern "C" orb_status orbm_stereo_rgbd_batch(orbx_handle* h, int32_t n_images, const void* depth, int32_t depth_format, int32_t stride_bytes,
                                             size_t image_stride_bytes, float depth_factor, int32_t on_device, float bf) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) return set_error(ORB_ERR_NO_DEVICE, "no CUDA device: this library has no CPU fallback");
    if (!h || !depth) return set_error(ORB_ERR_INVALID, "null handle or depth map");
    if (n_images < 1 || n_images > h->last_batch) return set_error(ORB_ERR_INVALID, "n_images exceeds the last extracted batch");
    DepthSource D{depth_format, stride_bytes, image_stride_bytes};
    orb_status s = check_depth(D, n_images, h->cur_w, h->cur_h);
    if (s != ORB_OK) return s;
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    const uint8_t* src = static_cast<const uint8_t*>(depth);
    if (!on_device) {   // the maps go up tight into the handle's buffer
        const size_t row = (size_t)h->cur_w * (D.format == ORB_DEPTH_U16 ? 2 : 4), img = row * h->cur_h;
        if ((s = grow_device(h->dmap_bytes, h->d_dmap, img * n_images, h->capturing)) != ORB_OK) return s;
        if ((s = copy_images(h, h->d_dmap, row, src, D.stride, D.image_stride, row, h->cur_h, n_images, cudaMemcpyHostToDevice)) != ORB_OK) return s;
        src = h->d_dmap;
        D.stride = (int64_t)row;
        D.image_stride = img;
    }
    const orbdev::RgbdPlan P{src, (int64_t)D.image_stride, D.stride, D.format, orbdev::rgbd_scaled(D.format, depth_factor) ? 1 : 0, depth_factor, bf,
                             h->d_kps, h->d_offsets, h->d_nkp, h->d_uright, h->d_depth};
    k_stereo_rgbd<<<dim3((h->geom.kpTotal + 127) / 128, n_images), 128, 0, h->stream>>>(P);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(ORB_ERR_CUDA, std::string("k_stereo_rgbd: ") + cudaGetErrorString(e));
    ORB_LAUNCHED();
    h->stereo_valid = true;
    return ORB_OK;
}
