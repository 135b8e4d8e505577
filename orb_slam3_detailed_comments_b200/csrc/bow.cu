// bow.cu -- Frame::ComputeBoW / KeyFrame::ComputeBoW on the device: DBoW2's vocabulary-tree transform of every descriptor
// of a batch (TemplatedVocabulary<FORB::TDescriptor, FORB>::transform, Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1127-1260)
// and the BowVector assembly (BowVector::addWeight / normalize, BowVector.cpp:34-84) for TF_IDF weighting + L1 scoring,
// the configuration ORBvoc.txt is loaded with (TemplatedVocabulary.h:56, ORBVocabulary.h).
//   /root/reference/src/Frame.cc:984-997  mpORBvocabulary->transform(vCurrentDesc, mBowVec, mFeatVec, 4)
// The vocabulary (flattened by the caller from the DBoW2 object it loaded) lives in HBM: children as CSR, 32-byte node
// descriptors, word id and idf weight per leaf.  A 16-lane group walks one descriptor down the tree: lane c takes child c,
// the group's minimum with the first-child tie-break picks the branch.
#include <algorithm>
#include <vector>

#include "extractor.h"

using namespace orb;

struct orbv_vocabulary {
    int device = 0;
    int n_nodes = 0, L = 0, max_children = 0;
    uint8_t* d_buf = nullptr;   // the five arrays below, carved from one block
    int* d_child_off = nullptr;
    int* d_child = nullptr;
    uint8_t* d_desc = nullptr;
    int* d_word = nullptr;
    double* d_weight = nullptr;
};

namespace orb {

struct BowParams {
    const int* child_off;
    const int* child;
    const uint8_t* ndesc;
    const int* nword;
    const double* nweight;
    int nid_level;            // L - levelsup
    const uint8_t* desc;      // descriptors of the batch (compact rows)
    int rows;
    int* word;                // per row
    int* node;
    double* weight;
    // BowVector assembly
    const int* offsets;       // compact row offset per image
    const int* nkp;
    int maxFeat;
    int* bow_count;           // [n_images]
    int* bow_word;            // [n_images][maxFeat]
    double* bow_weight;
};

__global__ void __launch_bounds__(256) k_bow_transform(const __grid_constant__ BowParams P) {
    const int sub = threadIdx.x & 15;
    const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    if (row >= P.rows) return;   // uniform per 16-lane group
    const unsigned gmask = 0xffffu << (threadIdx.x & 16);
    const uint4* q4 = reinterpret_cast<const uint4*>(P.desc + (size_t)row * 32);
    const uint4 a0 = __ldg(q4), a1 = __ldg(q4 + 1);
    int final_id = 0, level = 0, nid = 0;
    for (;;) {
        const int c0 = P.child_off[final_id], c1 = P.child_off[final_id + 1];
        if (c0 == c1) break;                           // isLeaf()
        ++level;
        uint32_t best = 0xffffffffu;                   // distance << 16 | child position: '<' keeps the first minimum
        for (int base = c0; base < c1; base += 16) {
            const int c = base + sub;
            if (c < c1) {
                const uint4* d4 = reinterpret_cast<const uint4*>(P.ndesc + (size_t)P.child[c] * 32);
                const uint4 b0 = __ldg(d4), b1 = __ldg(d4 + 1);
                const uint32_t d = __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
                                   __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
                best = min(best, (d << 16) | (uint32_t)(c - c0));
            }
        }
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(gmask, best, o, 16));
        final_id = P.child[c0 + (int)(best & 0xffffu)];
        if (level == P.nid_level) nid = final_id;
    }
    if (sub == 0) {
        P.word[row] = P.nword[final_id];
        P.node[row] = nid;                              // nid_level <= 0: the root (0)
        P.weight[row] = P.nweight[final_id];
    }
}

// BowVector of one image: (word, feature) keys of the features with weight > 0, bitonic sort, then the map semantics
// replayed by one thread -- per-word sums in feature order, the L1 norm in ascending word order (BowVector.cpp:34-84) --
// so every double is bit-identical to the reference's.
__global__ void __launch_bounds__(256) k_bow_vector(const __grid_constant__ BowParams P) {
    extern __shared__ unsigned long long bw_keys[];
    const int img = blockIdx.x;
    const int N = min(P.nkp[img], P.maxFeat), row0 = P.offsets[img];
    int npow = 2;
    while (npow < N) npow <<= 1;
    for (int i = threadIdx.x; i < npow; i += blockDim.x) {
        unsigned long long k = ~0ull;
        if (i < N && P.weight[row0 + i] > 0) k = ((unsigned long long)(unsigned)P.word[row0 + i] << 32) | (unsigned)i;
        bw_keys[i] = k;
    }
    __syncthreads();
    for (int k = 2; k <= npow; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < (npow >> 1); i += blockDim.x) {
                const int l = ((i & ~(j - 1)) << 1) | (i & (j - 1)), r = l | j;
                const unsigned long long a = bw_keys[l], b = bw_keys[r];
                if ((a > b) == ((l & k) == 0)) { bw_keys[l] = b; bw_keys[r] = a; }
            }
            __syncthreads();
        }
    if (threadIdx.x == 0) {
        int* ow = P.bow_word + (size_t)img * P.maxFeat;
        double* ov = P.bow_weight + (size_t)img * P.maxFeat;
        int n = 0;
        for (int i = 0; i < N; ++i) {
            const unsigned long long k = bw_keys[i];
            if (k == ~0ull) break;
            const int w = (int)(k >> 32), f = (int)(k & 0xffffffffu);
            const double v = P.weight[row0 + f];
            if (n > 0 && ow[n - 1] == w) ov[n - 1] += v;        // addWeight: vit->second += v
            else { ow[n] = w; ov[n] = v; ++n; }
        }
        double norm = 0.0;
        for (int i = 0; i < n; ++i) norm += fabs(ov[i]);         // normalize(L1)
        if (norm > 0.0)
            for (int i = 0; i < n; ++i) ov[i] /= norm;
        P.bow_count[img] = n;
    }
}

}  // namespace orb

extern "C" orb_status orbv_create(int32_t device, int32_t n_nodes, int32_t depth_levels, const int32_t* child_offset, const int32_t* child_ids,
                                  const uint8_t* node_desc, const int32_t* node_word, const double* node_weight, orbv_vocabulary** out) {
    if (!out || n_nodes < 1 || !child_offset || !child_ids || !node_desc || !node_word || !node_weight || child_offset[0] != 0)
        return set_error(ORB_ERR_INVALID, "bad arguments");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) return set_error(ORB_ERR_NO_DEVICE, "no CUDA device: this library has no CPU fallback");
    ORB_CUDA(cudaSetDevice(device));
    const int nchild = child_offset[n_nodes];
    if (nchild != n_nodes - 1) return set_error(ORB_ERR_INVALID, "the children lists must cover every node but the root exactly once");
    orbv_vocabulary* v = new orbv_vocabulary();
    v->device = device; v->n_nodes = n_nodes; v->L = depth_levels;
    for (int i = 0; i < n_nodes; ++i) v->max_children = std::max(v->max_children, child_offset[i + 1] - child_offset[i]);
    auto layout = [&](Carve& c) {
        v->d_child_off = stage_in(c, child_offset, (size_t)n_nodes + 1, false);
        v->d_child = stage_in(c, child_ids, (size_t)nchild, false);
        v->d_desc = stage_in(c, node_desc, (size_t)n_nodes * 32, false);
        v->d_word = stage_in(c, node_word, (size_t)n_nodes, false);
        v->d_weight = stage_in(c, node_weight, (size_t)n_nodes, false);
    };
    orb_status s = carve_exact(v->d_buf, nullptr, layout).status;
    if (s == ORB_OK && cudaStreamSynchronize(nullptr) != cudaSuccess) s = set_error(ORB_ERR_CUDA, "vocabulary upload failed");
    if (s != ORB_OK) {
        orbv_destroy(v);
        return s;
    }
    *out = v;
    return ORB_OK;
}

extern "C" void orbv_destroy(orbv_vocabulary* v) {
    if (!v) return;
    cudaSetDevice(v->device);
    if (v->d_buf) cudaFree(v->d_buf);
    delete v;
}

extern "C" orb_status orbv_transform(orbx_handle* h, const orbv_vocabulary* voc, int32_t levelsup, int32_t on_device, int32_t* word_out,
                                     int32_t* node_out, double* weight_out, int32_t* bow_count_out, int32_t* bow_word_out, double* bow_weight_out) {
    if (!h || !voc || !word_out || !node_out || !weight_out) return set_error(ORB_ERR_INVALID, "bad arguments");
    if (voc->device != h->cfg.device) return set_error(ORB_ERR_INVALID, "vocabulary and extractor live on different devices");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    int rows = 0;
    orb_status s = batch_rows(h, &rows);
    if (s != ORB_OK) return s;
    const int nimg = h->last_batch;
    const bool dev = on_device != 0, want_bow = bow_count_out && bow_word_out && bow_weight_out;
    const int maxFeat = h->geom.kpTotal;
    int npow = 2;
    while (npow < maxFeat) npow <<= 1;
    static const size_t bowStatic = static_smem(k_bow_vector);
    if (want_bow && ((s = check_frame_rows(maxFeat, "frame")) != ORB_OK || (s = check_smem(h, (size_t)npow * 8, bowStatic, "k_bow_vector")) != ORB_OK))
        return s;
    BowParams P{};
    P.child_off = voc->d_child_off; P.child = voc->d_child; P.ndesc = voc->d_desc; P.nword = voc->d_word; P.nweight = voc->d_weight;
    P.nid_level = voc->L - levelsup;
    P.desc = h->d_desc; P.rows = rows;
    P.offsets = h->d_offsets; P.nkp = h->d_nkp; P.maxFeat = maxFeat;
    // results staging shares the pose-optimisation buffer (not the matcher stage: its feature_node input may live there)
    auto layout = [&](Carve& c) {
        P.word = stage_out(c, word_out, rows, dev);
        P.node = stage_out(c, node_out, rows, dev);
        P.weight = stage_out(c, weight_out, rows, dev);
        if (want_bow) {
            P.bow_count = stage_out(c, bow_count_out, nimg, dev);
            P.bow_word = stage_out(c, bow_word_out, (size_t)nimg * maxFeat, dev);
            P.bow_weight = stage_out(c, bow_weight_out, (size_t)nimg * maxFeat, dev);
        }
    };
    const Carve c = carve_scratch(h->po_bytes, h->d_po, h->capturing, h->stream, layout);
    if (c.status != ORB_OK) return c.status;
    cudaStream_t st = h->stream;
    if (rows > 0) {
        k_bow_transform<<<(rows * 16 + 255) / 256, 256, 0, st>>>(P);
        ORB_LAUNCHED();
    }
    if (want_bow) {
        ORB_CUDA(cudaFuncSetAttribute(k_bow_vector, cudaFuncAttributeMaxDynamicSharedMemorySize, npow * 8));
        k_bow_vector<<<nimg, 256, (size_t)npow * 8, st>>>(P);
        ORB_LAUNCHED();
    }
    ORB_CUDA(cudaGetLastError());
    return dev ? ORB_OK : copy_out(c);
}
