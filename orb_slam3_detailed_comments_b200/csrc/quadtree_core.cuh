// quadtree_core.cuh -- DistributeOctTree (/root/reference/src/ORBextractor.cc:711-1057) re-designed
// for one CTA per (image, level).
//
// The reference walks a std::list of nodes that each own a copy of their keypoints.  Here:
//   * every candidate computes its own root-to-leaf path (it depends only on its coordinates) and is
//     packed into ONE sort element [root:2 | path:2 bits/depth | score:8] (QtForm below: 32 bits and 11
//     depths for regions up to 2048 px, 64 bits and 12 depths up to 4096 px);
//   * the words are sorted (bitonic, in shared memory), after which every tree node is a contiguous
//     range and "DivideNode" is three binary searches -- no keypoint is ever moved again;
//   * the node list is an array rebuilt per round with prefix sums (the list order, push_front
//     order, the 3*nToExpand rule, the std::sort tie order and the early break of the ordered
//     phase are reproduced exactly -- SURVEY App. B items 2-6);
//   * each surviving leaf picks its best candidate (max score, ties -> reference candidate order).
//
// Capacity: the list never exceeds max(N + 3, 4 * nIni).  A sweep only starts when the previous one
// ended with S + 3 * nToExpand <= N (otherwise the ordered phase takes over) and a sweep replaces
// each of the nToExpand multi-point nodes by at most 4 children, so it ends with at most
// S + 3 * nToExpand <= N nodes; the ordered phase breaks as soon as N is reached (<= N + 3).
//
// The code is written as barrier-separated SPMD phases (QT_PAR_FOR / QT_SYNC) so the identical source
// also compiles as sequential host code for tests/host_emul (no GPU in the build container).
#pragma once
#include "devmath.cuh"

namespace orbdev {

// The two forms of the sort element; the algorithm below is written once and instantiated for both.  A region of side
// 2^depths px is one pixel wide after `depths` halvings, so the path identifies the candidate's pixel.
//   uint32_t: [root:2 | path:22 | score:8]                  regions up to 2048 px (k_quadtree, k_quadtree_v1)
//   uint64_t: [0:30 | root:2 | path:24 | score:8]           regions up to 4096 px (k_quadtree_v1_k64)
// QtNode::pd holds depth << pd_shift | prefix; the prefix of a depth-d node has 2 + 2d bits.
template <typename E> struct QtForm;
template <> struct QtForm<uint32_t> { static constexpr int depths = 11, max_dim = 2048, pd_shift = 24; };
template <> struct QtForm<uint64_t> { static constexpr int depths = 12, max_dim = 4096, pd_shift = 28; };
template <typename E> ORB_HD constexpr int qt_elem_bits() { return 10 + 2 * QtForm<E>::depths; }

#if defined(__CUDA_ARCH__)
#define QT_PAR_FOR(i, n) for (int i = threadIdx.x; i < (n); i += blockDim.x)
#define QT_SYNC() __syncthreads()
#define QT_SERIAL if (threadIdx.x == 0)
#define QT_NTHREADS ((int)blockDim.x)
#elif defined(QT_EMUL_THREADS)
// tests/host_emul/qt_mt.cpp: host threads play the CTA with a real barrier (ThreadSanitizer then sees a missing QT_SYNC as a race)
extern thread_local int qt_tid;
extern int qt_nthreads;
void qt_barrier();
#define QT_PAR_FOR(i, n) for (int i = orbdev::qt_tid; i < (n); i += orbdev::qt_nthreads)
#define QT_SYNC() orbdev::qt_barrier()
#define QT_SERIAL if (orbdev::qt_tid == 0)
#define QT_NTHREADS (orbdev::qt_nthreads)
#elif defined(QT_HOST_COUNT_SYNCS)
// host, one thread, counting the barriers a CTA would execute (tests/host_emul: the barrier budget of the two variants)
extern long qt_sync_count;
#define QT_PAR_FOR(i, n) for (int i = 0; i < (n); ++i)
#define QT_SYNC() ((void)++orbdev::qt_sync_count)
#define QT_SERIAL
#define QT_NTHREADS 1
#else
#define QT_PAR_FOR(i, n) for (int i = 0; i < (n); ++i)
#define QT_SYNC() ((void)0)
#define QT_SERIAL
#define QT_NTHREADS 1
#endif

// Phase clocks of the device build (-DQT_PROFILE only: tools/qt_phases.py): thread 0 of every CTA adds the cycles between ticks to
// g_qt_prof[slot]; slot = 16 * (level-0 CTA ? 0 : 1) + phase.  Compiled out of the product library.
#if defined(__CUDACC__) && defined(QT_PROFILE)
__device__ long long g_qt_prof[32];
#endif
#if defined(__CUDA_ARCH__) && defined(QT_PROFILE)
#define QT_PROF_BEGIN() long long qt_tl_ = clock64()
#define QT_TICK(g, k) { const long long t_ = clock64(); if (threadIdx.x == 0) atomicAdd((unsigned long long*)&g_qt_prof[(g).prof_base + (k)], (unsigned long long)(t_ - qt_tl_)); qt_tl_ = t_; }
#else
#define QT_PROF_BEGIN() ((void)0)
#define QT_TICK(g, k) {}
#endif

struct QtNode {      // 20 bytes
    int lo, hi;      // candidate range [lo,hi) in the sorted array
    uint32_t pd;     // depth << QtForm::pd_shift | prefix (root + 2*depth path bits)
    int16_t ulx, uly, urx, bry;
};

struct QtItem {      // one entry of vSizeAndPointerToNode: (count, node)
    uint32_t cnt;
    uint32_t ulx_pos;  // UL.x << 16 | position of the node in the current list
};

struct QtGeom {
    int regionW, regionH;  // maxX-minX, maxY-minY
    int nIni;
    float hX;
    int N;                 // features wanted at this level
    int wCell, hCell, nCols;  // FAST cell grid (defines the reference's candidate order)
#if defined(QT_PROFILE)
    int prof_base;
#endif
};

// workspace layout for `cap` nodes; all pointers may be shared or global memory
struct QtWork {
    QtNode* cur;
    QtNode* nxt;
    int* bnd;        // 3*cap child boundaries
    int* m;          // cap: non-empty children / scan scratch
    int* x;          // cap: expandable children / scan scratch
    int* f;          // cap: flags / scan scratch
    QtItem* items;   // cap
    QtItem* items2;  // cap
    int* scan_tmp;   // 40 ints, then 34 64-bit slots for qt_exscan3
    int cap;
};

ORB_HD int qt_node_cap(int N) { return N + 20; }

ORB_HD size_t qt_work_bytes(int cap) {
    return (size_t)cap * (2 * sizeof(QtNode) + 3 * 4 + 3 * 4 + 2 * sizeof(QtItem)) + (40 + 72) * 4 + 64;   // scan_tmp: 40 ints + 34 x 64 bit (qt_exscan3)
}

ORB_HD void qt_work_carve(QtWork& w, void* base, int cap) {
    char* p = (char*)base;
    w.cap = cap;
    w.cur = (QtNode*)p; p += sizeof(QtNode) * cap;
    w.nxt = (QtNode*)p; p += sizeof(QtNode) * cap;
    w.bnd = (int*)p; p += 12 * (size_t)cap;
    w.m = (int*)p; p += 4 * (size_t)cap;
    w.x = (int*)p; p += 4 * (size_t)cap;
    w.f = (int*)p; p += 4 * (size_t)cap;
    w.items = (QtItem*)p; p += sizeof(QtItem) * cap;
    w.items2 = (QtItem*)p; p += sizeof(QtItem) * cap;
    w.scan_tmp = (int*)p;
}

// packed candidate as produced by the FAST kernel: x_rel | y_rel << 12 | score << 24 (coords relative
// to (minBorderX, minBorderY) = (16,16))
ORB_HD uint32_t qt_pack_cand(int x, int y, int score) { return (uint32_t)x | ((uint32_t)y << 12) | ((uint32_t)score << 24); }

// sortable element of a candidate
template <typename E = uint32_t>
ORB_HD E qt_element(uint32_t cand, const QtGeom& g) {
    const int x = cand & 0xfff, y = (cand >> 12) & 0xfff;
    const int root = (int)fdiv((float)x, g.hX);
    QtBox b = qt_root_box(root, g.hX, g.regionH);
    E key = (E)root;
    for (int d = 0; d < QtForm<E>::depths; ++d) {
        const int mx = b.ulx + ((b.urx - b.ulx + 1) >> 1);
        const int my = b.uly + ((b.bry - b.uly + 1) >> 1);
        const int q = (x < mx ? 0 : 1) | (y < my ? 0 : 2);
        key = (key << 2) | (E)q;
        b = qt_child_box(b, q);
    }
    return (key << 8) | (E)(cand >> 24);
}

// recover (x_rel, y_rel) of an element by replaying its path: after QtForm<E>::depths halvings the box is
// at most one pixel wide, so its upper-left corner is the point.
template <typename E>
ORB_HD void qt_element_xy(E e, const QtGeom& g, int* x, int* y) {
    const int root = (int)(e >> (qt_elem_bits<E>() - 2));
    QtBox b = qt_root_box(root, g.hX, g.regionH);
    for (int d = 0; d < QtForm<E>::depths; ++d) b = qt_child_box(b, (int)((e >> (qt_elem_bits<E>() - 4 - 2 * d)) & 3u));
    *x = b.ulx;
    *y = b.uly;
}

template <typename E = uint32_t>
ORB_HD int qt_node_shift(int depth) { return qt_elem_bits<E>() - 2 - 2 * depth; }

template <typename E>
ORB_HD int qt_lower_bound(const E* a, int lo, int hi, E v) {
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// in-place exclusive scan of a[0..n); returns the total.  Must be called by the whole CTA.
#if defined(__CUDA_ARCH__)
__device__ inline int qt_exscan(int* a, int n, int* tmp) {
    const int nt = blockDim.x, tid = threadIdx.x;
    const int chunk = (n + nt - 1) / nt;
    const int b = min(tid * chunk, n), e = min(b + chunk, n);
    int s = 0;
    for (int i = b; i < e; ++i) s += a[i];
    int inc = s;
    const int lane = tid & 31, wid = tid >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) tmp[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        const int nw = (nt + 31) >> 5;
        int v = lane < nw ? tmp[lane] : 0, iv = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, iv, o);
            if (lane >= o) iv += u;
        }
        if (lane < nw) tmp[lane] = iv - v;
        if (lane == 31) tmp[32] = iv;
    }
    __syncthreads();
    int run = tmp[wid] + inc - s;
    const int total = tmp[32];
    for (int i = b; i < e; ++i) {
        const int v = a[i];
        a[i] = run;
        run += v;
    }
    __syncthreads();
    return total;
}
#elif defined(QT_EMUL_THREADS)
inline int qt_exscan(int* a, int n, int* tmp) {
    qt_barrier();
    if (qt_tid == 0) {
        int run = 0;
        for (int i = 0; i < n; ++i) {
            const int v = a[i];
            a[i] = run;
            run += v;
        }
        tmp[32] = run;
    }
    qt_barrier();
    const int total = tmp[32];
    qt_barrier();
    return total;
}
#else
inline int qt_exscan(int* a, int n, int*) {
    int run = 0;
    for (int i = 0; i < n; ++i) {
        const int v = a[i];
        a[i] = run;
        run += v;
    }
    return run;
}
#endif

// three in-place exclusive scans at once (the sweep's non-empty children, expandable children and kept-node flags: one pass and
// three barriers instead of three passes and nine).  Fields of 21 bits: every sum is below 4 * cap.  Whole CTA.
#if defined(__CUDA_ARCH__)
__device__ inline void qt_exscan3(int* a, int* b, int* c, int n, int* tmp, int* ta, int* tb, int* tc) {
    unsigned long long* t64 = reinterpret_cast<unsigned long long*>(tmp + 40);
    const int nt = blockDim.x, tid = threadIdx.x;
    const int chunk = (n + nt - 1) / nt;
    const int lo = min(tid * chunk, n), hi = min(lo + chunk, n);
    unsigned long long s = 0;
    for (int i = lo; i < hi; ++i) s += (unsigned long long)a[i] | ((unsigned long long)b[i] << 21) | ((unsigned long long)c[i] << 42);
    unsigned long long inc = s;
    const int lane = tid & 31, wid = tid >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) t64[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        const int nw = (nt + 31) >> 5;
        unsigned long long v = lane < nw ? t64[lane] : 0ull, iv = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long u = __shfl_up_sync(0xffffffffu, iv, o);
            if (lane >= o) iv += u;
        }
        if (lane < nw) t64[lane] = iv - v;
        if (lane == 31) t64[32] = iv;
    }
    __syncthreads();
    unsigned long long run = t64[wid] + inc - s;
    const unsigned long long total = t64[32];
    for (int i = lo; i < hi; ++i) {
        const unsigned long long v = (unsigned long long)a[i] | ((unsigned long long)b[i] << 21) | ((unsigned long long)c[i] << 42);
        a[i] = (int)(run & 0x1fffffull); b[i] = (int)((run >> 21) & 0x1fffffull); c[i] = (int)(run >> 42);
        run += v;
    }
    __syncthreads();
    *ta = (int)(total & 0x1fffffull); *tb = (int)((total >> 21) & 0x1fffffull); *tc = (int)(total >> 42);
}
#else
inline void qt_exscan3(int* a, int* b, int* c, int n, int* tmp, int* ta, int* tb, int* tc) {
    *ta = qt_exscan(a, n, tmp);
    *tb = qt_exscan(b, n, tmp);
    *tc = qt_exscan(c, n, tmp);
}
#endif

// bitonic sort of arr[0..npow) (npow a power of two), ascending
template <typename E>
ORB_HD void qt_bitonic_sort(E* arr, int npow) {
    for (int k = 2; k <= npow; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            QT_PAR_FOR(i, npow >> 1) {
                const int l = ((i & ~(j - 1)) << 1) | (i & (j - 1));
                const int r = l | j;
                const E a = arr[l], b = arr[r];
                const bool up = (l & k) == 0;
                if ((a > b) == up) {
                    arr[l] = b;
                    arr[r] = a;
                }
            }
            QT_SYNC();
        }
    }
}

// children of node `nd`: boundaries b[0..2] (b0=lo, b4=hi implicit) -> counts; returns m | x << 8
template <typename E>
ORB_HD int qt_split(const E* arr, const QtNode& nd, int* b3) {
    const int depth = (int)(nd.pd >> QtForm<E>::pd_shift);
    const uint32_t pref = nd.pd & ((1u << QtForm<E>::pd_shift) - 1u);
    const int sh = qt_node_shift<E>(depth + 1);
    int prev = nd.lo, m = 0, x = 0;
    for (int q = 1; q <= 4; ++q) {
        const int b = (q < 4) ? qt_lower_bound(arr, prev, nd.hi, (E)((pref << 2) | (uint32_t)q) << sh) : nd.hi;
        if (q < 4) b3[q - 1] = b;
        const int c = b - prev;
        m += c > 0;
        x += c > 1;
        prev = b;
    }
    return m | (x << 8);
}

template <typename E>
ORB_HD QtNode qt_child(const QtNode& nd, const int* b3, int q) {
    const int depth = (int)(nd.pd >> QtForm<E>::pd_shift);
    const uint32_t pref = nd.pd & ((1u << QtForm<E>::pd_shift) - 1u);
    QtBox pb;
    pb.ulx = nd.ulx; pb.uly = nd.uly; pb.urx = nd.urx; pb.bry = nd.bry;
    const QtBox cb = qt_child_box(pb, q);
    QtNode c;
    c.lo = q == 0 ? nd.lo : b3[q - 1];
    c.hi = q == 3 ? nd.hi : b3[q];
    c.pd = ((uint32_t)(depth + 1) << QtForm<E>::pd_shift) | ((pref << 2) | (uint32_t)q);
    c.ulx = (int16_t)cb.ulx; c.uly = (int16_t)cb.uly; c.urx = (int16_t)cb.urx; c.bry = (int16_t)cb.bry;
    return c;
}

template <typename E>
ORB_HD bool qt_expandable(const QtNode& nd) { return (nd.hi - nd.lo) > 1 && (int)(nd.pd >> QtForm<E>::pd_shift) < QtForm<E>::depths; }

// compareNodes (ORBextractor.cc:676-697) orders by (point count, UL.x): one 48-bit key, compared without branches
ORB_HD uint64_t qt_item_key(const QtItem& a) { return ((uint64_t)a.cnt << 16) | (uint64_t)(a.ulx_pos >> 16); }
ORB_HD bool qt_item_less(const QtItem& a, const QtItem& b) { return qt_item_key(a) < qt_item_key(b); }

// std::sort on QtItem with the libstdc++ sequence of moves (devmath.cuh std_sort, specialised)
ORB_HD void qt_std_sort_items(QtItem* a, int n) {
    // QtItem and SortItem differ only in the comparator; map to (key,val) where key orders like
    // compareNodes: cnt (32 bits) then ulx (16 bits) -> 48-bit key does not fit SortItem, so the
    // algorithm is instantiated again here on QtItem.
    if (n <= 1) return;
    int lg = 0;
    for (int t = n; t > 1; t >>= 1) ++lg;
    int sf[64], sl[64], sd[64];
    int sp = 1;
    sf[0] = 0; sl[0] = n; sd[0] = 2 * lg;
    while (sp > 0) {
        --sp;
        int first = sf[sp], last = sl[sp], depth = sd[sp];
        while (last - first > 16) {
            if (depth == 0) {
                // heap sort fallback (__partial_sort(first,last,last))
                QtItem* h = a + first;
                const int len = last - first;
                // __make_heap
                for (int parent = (len - 2) / 2;; --parent) {
                    QtItem v = h[parent];
                    int hole = parent, child = parent;
                    while (child < (len - 1) / 2) {
                        child = 2 * (child + 1);
                        if (qt_item_less(h[child], h[child - 1])) --child;
                        h[hole] = h[child];
                        hole = child;
                    }
                    if ((len & 1) == 0 && child == (len - 2) / 2) {
                        child = 2 * (child + 1);
                        h[hole] = h[child - 1];
                        hole = child - 1;
                    }
                    int par = (hole - 1) / 2;
                    while (hole > parent && qt_item_less(h[par], v)) {
                        h[hole] = h[par];
                        hole = par;
                        par = (hole - 1) / 2;
                    }
                    h[hole] = v;
                    if (parent == 0) break;
                }
                for (int end = len - 1; end > 0; --end) {  // __sort_heap
                    QtItem v = h[end];
                    h[end] = h[0];
                    int hole = 0, child = 0;
                    const int l2 = end;
                    while (child < (l2 - 1) / 2) {
                        child = 2 * (child + 1);
                        if (qt_item_less(h[child], h[child - 1])) --child;
                        h[hole] = h[child];
                        hole = child;
                    }
                    if ((l2 & 1) == 0 && child == (l2 - 2) / 2) {
                        child = 2 * (child + 1);
                        h[hole] = h[child - 1];
                        hole = child - 1;
                    }
                    int par = (hole - 1) / 2;
                    while (hole > 0 && qt_item_less(h[par], v)) {
                        h[hole] = h[par];
                        hole = par;
                        par = (hole - 1) / 2;
                    }
                    h[hole] = v;
                }
                break;
            }
            --depth;
            const int mid = first + (last - first) / 2;
            {
                const int A = first + 1, B = mid, C = last - 1;
                int pick;
                if (qt_item_less(a[A], a[B])) {
                    if (qt_item_less(a[B], a[C])) pick = B;
                    else if (qt_item_less(a[A], a[C])) pick = C;
                    else pick = A;
                } else if (qt_item_less(a[A], a[C])) pick = A;
                else if (qt_item_less(a[B], a[C])) pick = C;
                else pick = B;
                QtItem t = a[first]; a[first] = a[pick]; a[pick] = t;
            }
            int lo = first + 1, hi = last;
            while (true) {
                while (qt_item_less(a[lo], a[first])) ++lo;
                --hi;
                while (qt_item_less(a[first], a[hi])) --hi;
                if (!(lo < hi)) break;
                QtItem t = a[lo]; a[lo] = a[hi]; a[hi] = t;
                ++lo;
            }
            sf[sp] = lo; sl[sp] = last; sd[sp] = depth;
            ++sp;
            last = lo;
        }
    }
    const int head = n > 16 ? 16 : n;
    for (int i = 1; i < head; ++i) {  // __insertion_sort(first, first+16)
        if (qt_item_less(a[i], a[0])) {
            QtItem v = a[i];
            for (int j = i; j > 0; --j) a[j] = a[j - 1];
            a[0] = v;
        } else {
            QtItem v = a[i];
            int j = i;
            while (qt_item_less(v, a[j - 1])) { a[j] = a[j - 1]; --j; }
            a[j] = v;
        }
    }
    for (int i = 16; i < n; ++i) {  // __unguarded_insertion_sort
        QtItem v = a[i];
        int j = i;
        while (qt_item_less(v, a[j - 1])) { a[j] = a[j - 1]; --j; }
        a[j] = v;
    }
}

}  // namespace orbdev
#include "quadtree_sort_par.cuh"
namespace orbdev {

// reference candidate order (cell row, cell col, y, x) as one comparable key
ORB_HD uint64_t qt_order_key(int x, int y, const QtGeom& g) {
    const int ci = (y - 3) / g.hCell, cj = (x - 3) / g.wCell;
    return ((uint64_t)(ci * g.nCols + cj) << 24) | ((uint64_t)y << 12) | (uint64_t)x;
}

// ---------------------------------------------------------------------------------------------
// the distribution itself.  arr: n sorted elements.  out[t] = packed candidate (x|y<<12|score<<24)
// of the t-th node of the final list.  Returns the list length (uniform across the CTA), or -1
// when the workspace capacity would be exceeded.
// ---------------------------------------------------------------------------------------------
// VARIANT 0: the ordered phase's std::sort by one thread (GPU-validated in round 1).  VARIANT 1: the same moves spread over the
// CTA (quadtree_sort_par.cuh; host-emulated in tests/test_quadtree_emul.py; the default since its round-2 device run).
template <int VARIANT, typename Key>
ORB_HD int qt_distribute_v(const Key* arr, int n, const QtGeom& g, QtWork& w, uint32_t* out) {
    // roots (ORBextractor.cc:718-786): non-empty ones, in order
    QT_PROF_BEGIN();
    int S = 0;
    QT_SERIAL {
        int lo = 0, cnt = 0;
        for (int r = 0; r < g.nIni; ++r) {
            const int hi = (r == 3) ? n : qt_lower_bound(arr, lo, n, (Key)(r + 1) << (qt_elem_bits<Key>() - 2));
            if (hi > lo) {
                QtNode nd;
                const QtBox b = qt_root_box(r, g.hX, g.regionH);
                nd.lo = lo; nd.hi = hi; nd.pd = (uint32_t)r;
                nd.ulx = (int16_t)b.ulx; nd.uly = 0; nd.urx = (int16_t)b.urx; nd.bry = (int16_t)b.bry;
                w.cur[cnt++] = nd;
            }
            lo = hi;
        }
        w.scan_tmp[36] = cnt;
    }
    QT_SYNC();
    S = w.scan_tmp[36];
    QT_SYNC();

    bool finish = (S == 0);
    QT_TICK(g, 2)
    while (!finish) {
        const int prevS = S;
        // ---- one sweep over the list (ORBextractor.cc:814-906) --------------------------------
        QT_PAR_FOR(t, S) {
            const QtNode nd = w.cur[t];
            if (qt_expandable<Key>(nd)) {
                const int mx = qt_split(arr, nd, &w.bnd[3 * t]);
                w.m[t] = mx & 0xff;
                w.x[t] = mx >> 8;
                w.f[t] = 0;
            } else {
                w.m[t] = 0;
                w.x[t] = 0;
                w.f[t] = 1;
            }
        }
        QT_SYNC();
        // keep a copy of m (needed after the scan) in the upper half of bnd? -> recompute instead:
        int E, X, NM;   // m[t] = sum_{t'<t} m, x[t] = sum_{t'<t} x, f[t] = rank among kept nodes
        qt_exscan3(w.m, w.x, w.f, S, w.scan_tmp, &E, &X, &NM);
        if (E + NM > w.cap) return -1;
        QT_PAR_FOR(t, S) {
            const QtNode nd = w.cur[t];
            if (!qt_expandable<Key>(nd)) {
                w.nxt[E + w.f[t]] = nd;
            } else {
                const int* b3 = &w.bnd[3 * t];
                int cnts[4];
                cnts[0] = b3[0] - nd.lo; cnts[1] = b3[1] - b3[0]; cnts[2] = b3[2] - b3[1]; cnts[3] = nd.hi - b3[2];
                const int mt = (cnts[0] > 0) + (cnts[1] > 0) + (cnts[2] > 0) + (cnts[3] > 0);
                // block of node t starts after the blocks of all LATER expandable nodes
                const int base = E - w.m[t] - mt;
                int r = 0;
                int pos[4];
                for (int q = 3; q >= 0; --q)
                    if (cnts[q] > 0) {
                        pos[q] = base + r;
                        w.nxt[base + r] = qt_child<Key>(nd, b3, q);
                        ++r;
                    }
                int rr = 0;
                for (int q = 0; q < 4; ++q)
                    if (cnts[q] > 1) {
                        QtItem it;
                        it.cnt = (uint32_t)cnts[q];
                        const QtNode c = w.nxt[pos[q]];
                        it.ulx_pos = ((uint32_t)(uint16_t)c.ulx << 16) | (uint32_t)pos[q];
                        w.items[w.x[t] + rr] = it;
                        ++rr;
                    }
            }
        }
        QT_SYNC();
        S = E + NM;
        { QtNode* t = w.cur; w.cur = w.nxt; w.nxt = t; }
        int nItems = X;
        QT_TICK(g, 3)
        if (S >= g.N || S == prevS) {
            finish = true;
        } else if (S + 3 * nItems > g.N) {
            // ---- ordered phase (ORBextractor.cc:932-1016) -------------------------------------
            while (!finish) {
                const int prev2 = S;
                if (nItems == 0) {  // nothing left to divide: the list stops growing
                    finish = true;
                    break;
                }
                if (VARIANT == 0) {
                    QT_SERIAL { qt_std_sort_items(w.items, nItems); }
                    QT_SYNC();
                } else {
                    qt_std_sort_items_par(w.items, nItems, w.items2, w.m, w.bnd, w.f, w.scan_tmp, 6 * w.cap);   // bnd | m | x | f are contiguous: 6 * cap ints from w.bnd
                }
                QT_TICK(g, 4)
                // processing order p = 0.. corresponds to sorted index j = nItems-1-p
                QT_PAR_FOR(p, nItems) {
                    const QtItem it = w.items[nItems - 1 - p];
                    const QtNode nd = w.cur[it.ulx_pos & 0xffffu];
                    const int mx = qt_split(arr, nd, &w.bnd[3 * p]);
                    w.m[p] = (mx & 0xff) - 1;  // growth of the list when this node is divided
                    w.x[p] = mx >> 8;
                }
                QT_SYNC();
                qt_exscan(w.m, nItems, w.scan_tmp);  // m[p] = growth before p
                // K = number of nodes divided before the `break`
                QT_SERIAL { w.scan_tmp[37] = 0; }
                QT_SYNC();
                {
                    int local = 0;
                    QT_PAR_FOR(p, nItems) {
                        // size after dividing p: prev2 + m[p] + growth(p); still below N => continue
                        const QtItem it = w.items[nItems - 1 - p];
                        const QtNode nd = w.cur[it.ulx_pos & 0xffffu];
                        const int* b3 = &w.bnd[3 * p];
                        const int mt = ((b3[0] - nd.lo) > 0) + ((b3[1] - b3[0]) > 0) + ((b3[2] - b3[1]) > 0) + ((nd.hi - b3[2]) > 0);
                        if (prev2 + w.m[p] + mt - 1 < g.N) ++local;
                    }
#if defined(__CUDA_ARCH__)
                    if (local) atomicAdd(&w.scan_tmp[37], local);
#elif defined(QT_EMUL_THREADS)
                    if (local) __atomic_fetch_add(&w.scan_tmp[37], local, __ATOMIC_RELAXED);
#else
                    w.scan_tmp[37] += local;
#endif
                }
                QT_SYNC();
                int K = w.scan_tmp[37] + 1;
                if (K > nItems) K = nItems;
                QT_SYNC();
                // flags over the current list: 1 = kept; positions of divided nodes get 0
                QT_PAR_FOR(t, S) w.f[t] = 1;
                QT_SYNC();
                QT_PAR_FOR(p, K) w.f[w.items[nItems - 1 - p].ulx_pos & 0xffffu] = 0;
                QT_SYNC();
                const int kept = qt_exscan(w.f, S, w.scan_tmp);
                // children blocks: total Ek, block of p starts after the blocks of later p' < K
                // growth prefix m[p] = sum_{p'<p} (mt-1)  =>  sum_{p'<p} mt = m[p] + p
                int Ek;
                {
                    const QtItem it = w.items[nItems - 1 - (K - 1)];
                    const QtNode nd = w.cur[it.ulx_pos & 0xffffu];
                    const int* b3 = &w.bnd[3 * (K - 1)];
                    const int mt = ((b3[0] - nd.lo) > 0) + ((b3[1] - b3[0]) > 0) + ((b3[2] - b3[1]) > 0) + ((nd.hi - b3[2]) > 0);
                    Ek = w.m[K - 1] + (K - 1) + mt;
                }
                if (Ek + kept > w.cap) return -1;
                const int Xk = qt_exscan(w.x, K, w.scan_tmp);  // x[p] = items created before p
                QT_TICK(g, 5)
                QT_PAR_FOR(t, S) {
                    // kept nodes keep their relative order behind all new children
                    const QtNode nd = w.cur[t];
                    bool is_kept;
                    if (t + 1 < S) is_kept = w.f[t + 1] != w.f[t]; else is_kept = (kept != w.f[t]);
                    if (is_kept) w.nxt[Ek + w.f[t]] = nd;
                }
                QT_PAR_FOR(p, K) {
                    const QtItem it = w.items[nItems - 1 - p];
                    const QtNode nd = w.cur[it.ulx_pos & 0xffffu];
                    const int* b3 = &w.bnd[3 * p];
                    int cnts[4];
                    cnts[0] = b3[0] - nd.lo; cnts[1] = b3[1] - b3[0]; cnts[2] = b3[2] - b3[1]; cnts[3] = nd.hi - b3[2];
                    const int mt = (cnts[0] > 0) + (cnts[1] > 0) + (cnts[2] > 0) + (cnts[3] > 0);
                    const int before = w.m[p] + p;          // children created before p
                    const int base = Ek - before - mt;      // later-divided nodes sit in front
                    int r = 0;
                    int pos[4];
                    for (int q = 3; q >= 0; --q)
                        if (cnts[q] > 0) {
                            pos[q] = base + r;
                            w.nxt[base + r] = qt_child<Key>(nd, b3, q);
                            ++r;
                        }
                    int rr = 0;
                    for (int q = 0; q < 4; ++q)
                        if (cnts[q] > 1) {
                            QtItem ni;
                            ni.cnt = (uint32_t)cnts[q];
                            const QtBox cb = qt_child_box(QtBox{nd.ulx, nd.uly, nd.urx, nd.bry}, q);
                            ni.ulx_pos = ((uint32_t)(uint16_t)cb.ulx << 16) | (uint32_t)pos[q];
                            w.items2[w.x[p] + rr] = ni;
                            ++rr;
                        }
                }
                QT_SYNC();
                S = Ek + kept;
                nItems = Xk;
                { QtNode* t = w.cur; w.cur = w.nxt; w.nxt = t; }
                { QtItem* t = w.items; w.items = w.items2; w.items2 = t; }
                QT_TICK(g, 6)
                if (S >= g.N || S == prev2) finish = true;
            }
        }
    }
    // ---- best candidate of every leaf (ORBextractor.cc:1028-1053) ------------------------------
    QT_PAR_FOR(t, S) {
        const QtNode nd = w.cur[t];
        Key best = arr[nd.lo];
        int bx, by;
        qt_element_xy(best, g, &bx, &by);
        uint64_t bkey = qt_order_key(bx, by, g);
        for (int i = nd.lo + 1; i < nd.hi; ++i) {
            const Key e = arr[i];
            const uint32_t se = (uint32_t)e & 0xffu, sb = (uint32_t)best & 0xffu;
            if (se < sb) continue;
            int ex, ey;
            qt_element_xy(e, g, &ex, &ey);
            const uint64_t ekey = qt_order_key(ex, ey, g);
            if (se > sb || ekey < bkey) {
                best = e; bx = ex; by = ey; bkey = ekey;
            }
        }
        out[t] = qt_pack_cand(bx, by, (int)((uint32_t)best & 0xffu));
    }
    QT_SYNC();
    QT_TICK(g, 7)
    return S;
}

template <typename E>
ORB_HD int qt_distribute(const E* arr, int n, const QtGeom& g, QtWork& w, uint32_t* out) {
    return qt_distribute_v<0>(arr, n, g, w, out);
}

}  // namespace orbdev
