// knn.cu -- K9: brute-force 256-bit Hamming 2-nearest-neighbour search, cv::BFMatcher(cv::NORM_HAMMING).knnMatch(query, train,
// matches, 2) as Frame::ComputeStereoFishEyeMatches calls it (/root/reference/src/Frame.cc:1553; include/Frame.h: BFmatcher), batched
// over independent (query set, train set) pairs.  A thread keeps one query descriptor in registers and the best two
// (distance, train index) keys; the train descriptors stream through shared memory in tiles that every thread reads at the same
// address (broadcast).  Keys order like OpenCV's result: ascending distance, ties by ascending train index (probed against
// cv2 4.13; tests/test_knn_cpu.py).
// STATUS: written after the last GPU run of round 1 -- the GPU test is opt-in (ORB_FIRST_CONTACT=1) until its first device run.
#include <stdlib.h>

#include <algorithm>

#include "extractor.h"

using namespace orb;

namespace {

constexpr int KNN_THREADS = 256;
constexpr int KNN_TILE = 128;       // train descriptors per shared-memory tile (4 KB)

struct KnnParams {
    int n_pairs;
    const int* q_off;       // [n_pairs + 1]
    const int* t_off;       // [n_pairs + 1]
    const uint8_t* q_desc;  // 32 bytes per row
    const uint8_t* t_desc;
    int* idx;               // [rows][2], -1 = no such neighbour
    int* dist;              // [rows][2]
};

// ---- TMA (1-D bulk copy) staging of the train tiles, double-buffered: ORB_KNN_TMA=1 -----------------------------------------------
// A tile is 128 consecutive 32-byte rows: one contiguous, 16-byte aligned 4 KB span -- exactly what cp.async.bulk moves without a
// tensor map.  One thread arms an mbarrier with the byte count and issues the copy of tile n + 1 while all threads work on tile n.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "KNN_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra KNN_DONE;\n"
        "bra KNN_WAIT;\n"
        "KNN_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

__global__ void __launch_bounds__(KNN_THREADS) k_hamming_knn2_tma(const __grid_constant__ KnnParams P) {
    __shared__ __align__(128) uint4 s_t[2][KNN_TILE * 2];
    __shared__ __align__(8) uint64_t s_bar[2];
    const int pair = blockIdx.y;
    const int q0 = P.q_off[pair], nq = P.q_off[pair + 1] - q0;
    const int t0 = P.t_off[pair], nt = P.t_off[pair + 1] - t0;
    if ((int)(blockIdx.x * KNN_THREADS) >= nq) return;     // uniform per CTA
    const int q = blockIdx.x * KNN_THREADS + threadIdx.x;
    const bool active = q < nq;
    uint4 a0 = make_uint4(0, 0, 0, 0), a1 = a0;
    if (active) {
        const uint4* qp = reinterpret_cast<const uint4*>(P.q_desc + (size_t)(q0 + q) * 32);
        a0 = __ldg(qp);
        a1 = __ldg(qp + 1);
    }
    if (threadIdx.x == 0) {
        mbar_init(&s_bar[0], 1);
        mbar_init(&s_bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int ntiles = (nt + KNN_TILE - 1) / KNN_TILE;
    const uint8_t* tbase = P.t_desc + (size_t)t0 * 32;
    auto issue = [&](int n) {
        const int m = min(KNN_TILE, nt - n * KNN_TILE);
        mbar_expect_tx(&s_bar[n & 1], (uint32_t)m * 32u);
        bulk_g2s(&s_t[n & 1][0], tbase + (size_t)n * KNN_TILE * 32, (uint32_t)m * 32u, &s_bar[n & 1]);
    };
    if (threadIdx.x == 0 && ntiles > 0) issue(0);
    uint32_t best0 = 0xffffffffu, best1 = 0xffffffffu;
    for (int n = 0; n < ntiles; ++n) {
        if (threadIdx.x == 0 && n + 1 < ntiles) issue(n + 1);       // its buffer was last read in iteration n - 1 (barrier below)
        mbar_wait(&s_bar[n & 1], (uint32_t)((n >> 1) & 1));
        const int m = min(KNN_TILE, nt - n * KNN_TILE), base = n * KNN_TILE;
        const uint4* tile = s_t[n & 1];
        if (active) {
#pragma unroll 4
            for (int j = 0; j < m; ++j) {
                const uint4 b0 = tile[2 * j], b1 = tile[2 * j + 1];
                const uint32_t d = __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
                                   __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
                const uint32_t key = (d << 20) | (uint32_t)(base + j);
                const uint32_t lo = min(best0, key);
                best1 = min(best1, max(best0, key));
                best0 = lo;
            }
        }
        __syncthreads();                                             // everyone is done with this buffer
    }
    if (active) {
        const size_t r = 2 * (size_t)(q0 + q);
        P.idx[r] = best0 == 0xffffffffu ? -1 : (int)(best0 & 0xfffffu);
        P.dist[r] = best0 == 0xffffffffu ? -1 : (int)(best0 >> 20);
        P.idx[r + 1] = best1 == 0xffffffffu ? -1 : (int)(best1 & 0xfffffu);
        P.dist[r + 1] = best1 == 0xffffffffu ? -1 : (int)(best1 >> 20);
    }
}

// blockIdx.y = pair, blockIdx.x = tile of KNN_THREADS queries
__global__ void __launch_bounds__(KNN_THREADS) k_hamming_knn2(const __grid_constant__ KnnParams P) {
    __shared__ uint4 s_t[KNN_TILE * 2];
    const int pair = blockIdx.y;
    const int q0 = P.q_off[pair], nq = P.q_off[pair + 1] - q0;
    const int t0 = P.t_off[pair], nt = P.t_off[pair + 1] - t0;
    if ((int)(blockIdx.x * KNN_THREADS) >= nq) return;     // uniform per CTA
    const int q = blockIdx.x * KNN_THREADS + threadIdx.x;
    const bool active = q < nq;
    uint4 a0 = make_uint4(0, 0, 0, 0), a1 = a0;
    if (active) {
        const uint4* qp = reinterpret_cast<const uint4*>(P.q_desc + (size_t)(q0 + q) * 32);
        a0 = __ldg(qp);
        a1 = __ldg(qp + 1);
    }
    uint32_t best0 = 0xffffffffu, best1 = 0xffffffffu;     // distance << 20 | train index  (train sets of < 2^20 rows)
    for (int base = 0; base < nt; base += KNN_TILE) {
        const int m = min(KNN_TILE, nt - base);
        __syncthreads();                                   // the previous tile is no longer read
        const uint4* tp = reinterpret_cast<const uint4*>(P.t_desc + (size_t)(t0 + base) * 32);
        for (int i = threadIdx.x; i < 2 * m; i += KNN_THREADS) s_t[i] = __ldg(tp + i);
        __syncthreads();
        if (active) {
#pragma unroll 4
            for (int j = 0; j < m; ++j) {
                const uint4 b0 = s_t[2 * j], b1 = s_t[2 * j + 1];
                const uint32_t d = __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
                                   __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
                const uint32_t key = (d << 20) | (uint32_t)(base + j);
                const uint32_t lo = min(best0, key);        // sorted insert into (best0, best1)
                best1 = min(best1, max(best0, key));
                best0 = lo;
            }
        }
    }
    if (active) {
        const size_t r = 2 * (size_t)(q0 + q);
        P.idx[r] = best0 == 0xffffffffu ? -1 : (int)(best0 & 0xfffffu);
        P.dist[r] = best0 == 0xffffffffu ? -1 : (int)(best0 >> 20);
        P.idx[r + 1] = best1 == 0xffffffffu ? -1 : (int)(best1 & 0xfffffu);
        P.dist[r + 1] = best1 == 0xffffffffu ? -1 : (int)(best1 >> 20);
    }
}

}  // namespace

extern "C" orb_status orbm_hamming_knn2(orbx_handle* h, int32_t n_pairs, const int32_t* query_offset, const uint8_t* query_desc,
                                        const int32_t* train_offset, const uint8_t* train_desc, int32_t* idx_out, int32_t* dist_out) {
    if (!h || n_pairs < 0 || !query_offset || !train_offset || !idx_out || !dist_out) return set_error(ORB_ERR_INVALID, "bad arguments");
    if (n_pairs == 0) return ORB_OK;
    const int nq = query_offset[n_pairs], nt = train_offset[n_pairs];
    if (query_offset[0] != 0 || train_offset[0] != 0 || nq < 0 || nt < 0 || (nq > 0 && !query_desc) || (nt > 0 && !train_desc))
        return set_error(ORB_ERR_INVALID, "bad descriptor tables");
    int maxq = 0;
    for (int i = 0; i < n_pairs; ++i) {
        if (query_offset[i + 1] < query_offset[i] || train_offset[i + 1] < train_offset[i]) return set_error(ORB_ERR_INVALID, "offsets must ascend");
        if (train_offset[i + 1] - train_offset[i] >= (1 << 20)) return set_error(ORB_ERR_UNSUPPORTED, "train set of 2^20 rows or more");
        maxq = std::max(maxq, query_offset[i + 1] - query_offset[i]);
    }
    if (nq == 0) return ORB_OK;
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    const size_t np = (size_t)n_pairs;
    KnnParams P;
    P.n_pairs = n_pairs;
    cudaStream_t st = h->stream;
    auto layout = [&](Carve& c) {
        P.q_off = stage_in(c, query_offset, np + 1, false); P.t_off = stage_in(c, train_offset, np + 1, false);
        P.q_desc = stage_in(c, query_desc, (size_t)nq * 32, false);
        P.t_desc = train_desc ? stage_in(c, train_desc, (size_t)nt * 32, false) : c.take<uint8_t>(32);   // a real address even with no train rows
        P.idx = stage_out(c, idx_out, (size_t)nq * 2, false);
        P.dist = stage_out(c, dist_out, (size_t)nq * 2, false);
    };
    const Carve c = carve_scratch(h->po_bytes, h->d_po, h->capturing, st, layout);
    if (c.status != ORB_OK) return c.status;
    const char* tma = getenv("ORB_KNN_TMA");       // 1: train tiles by cp.async.bulk + mbarrier, double-buffered
    if (tma && atoi(tma) == 1) k_hamming_knn2_tma<<<dim3((maxq + KNN_THREADS - 1) / KNN_THREADS, n_pairs), KNN_THREADS, 0, st>>>(P);
    else k_hamming_knn2<<<dim3((maxq + KNN_THREADS - 1) / KNN_THREADS, n_pairs), KNN_THREADS, 0, st>>>(P);
    ORB_LAUNCHED();
    ORB_CUDA(cudaGetLastError());
    return copy_out(c);
}
