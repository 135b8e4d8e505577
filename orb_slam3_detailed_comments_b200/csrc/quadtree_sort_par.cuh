// quadtree_sort_par.cuh -- std::sort(vSizeAndPointerToNode.begin(), end(), compareNodes) of DistributeOctTree's ordered phase
// (/root/reference/src/ORBextractor.cc:932-940) with libstdc++'s exact sequence of moves, but spread over the CTA.
//
// compareNodes orders by (point count, UL.x) only, nodes tie often, and the reference then divides the tied nodes in whatever order
// libstdc++'s introsort left them -- so the permutation itself is part of the result.  quadtree_core.cuh's qt_std_sort_items is a
// one-thread transcription (ncu, round 1: ~30 % of k_quadtree's stall samples are the other 255 threads waiting for it at the
// barrier).  The same moves, restructured:
//   * __introsort_loop recurses on the right part and iterates on the left: the segments alive at one recursion depth are
//     disjoint, so a GENERATION of segments is processed concurrently, one thread per segment, with the transcription's own
//     median-of-three + unguarded partition (or heap sort when the depth limit is hit); the critical path becomes
//     n + n/2 + n/4 + ... instead of n log2(n / 16);
//   * __final_insertion_sort only ever moves an element in front of strictly greater ones, i.e. it is a STABLE sort of whatever
//     the partitioning left: every thread computes the stable rank of one element instead (n <= a few hundred).
// Included by quadtree_core.cuh (uses QtItem, qt_item_less, qt_exscan and the QT_ SPMD macros).
#pragma once

namespace orbdev {

// one __introsort_loop step on [first, last): pivot to a[first] (__move_median_to_first), __unguarded_partition; returns the cut
ORB_HD int qt_sortpar_partition(QtItem* a, int first, int last) {
    const int mid = first + (last - first) / 2;
    const int A = first + 1, B = mid, C = last - 1;
    int pick;
    if (qt_item_less(a[A], a[B])) {
        if (qt_item_less(a[B], a[C])) pick = B;
        else if (qt_item_less(a[A], a[C])) pick = C;
        else pick = A;
    } else if (qt_item_less(a[A], a[C])) pick = A;
    else if (qt_item_less(a[B], a[C])) pick = C;
    else pick = B;
    { const QtItem t = a[first]; a[first] = a[pick]; a[pick] = t; }
    const uint64_t pv = qt_item_key(a[first]);
    int lo = first + 1, hi = last;
    // The two scans of __unguarded_partition read four items per round trip (the loads are independent, the tests sequential): the
    // chain of one shared-memory latency per element was the critical path of the whole ordered phase (phase clocks, round 2).
    // Reads run at most three items past a scan's stopping point: inside the workspace on the device, inside the padding the host
    // harnesses allocate (tests/host_emul).
#if defined(QT_EMUL_THREADS)
    // threaded host emulation (ThreadSanitizer): one item per read -- a speculative read may land in a segment another thread is
    // partitioning, which is harmless (the value is never used) but is a data race by the letter
    while (true) {
        while (qt_item_key(a[lo]) < pv) ++lo;
        --hi;
        while (pv < qt_item_key(a[hi])) --hi;
        if (!(lo < hi)) break;
        const QtItem t = a[lo]; a[lo] = a[hi]; a[hi] = t;
        ++lo;
    }
#else
    while (true) {
        while (true) {
            const uint64_t k0 = qt_item_key(a[lo]), k1 = qt_item_key(a[lo + 1]), k2 = qt_item_key(a[lo + 2]), k3 = qt_item_key(a[lo + 3]);
            if (!(k0 < pv)) break;
            ++lo;
            if (!(k1 < pv)) break;
            ++lo;
            if (!(k2 < pv)) break;
            ++lo;
            if (!(k3 < pv)) break;
            ++lo;
        }
        --hi;
        while (true) {
            const uint64_t k0 = qt_item_key(a[hi]), k1 = qt_item_key(a[hi - 1]), k2 = qt_item_key(a[hi - 2]), k3 = qt_item_key(a[hi - 3]);
            if (!(pv < k0)) break;
            --hi;
            if (!(pv < k1)) break;
            --hi;
            if (!(pv < k2)) break;
            --hi;
            if (!(pv < k3)) break;
            --hi;
        }
        if (!(lo < hi)) break;
        const QtItem t = a[lo]; a[lo] = a[hi]; a[hi] = t;
        ++lo;
    }
#endif
    return lo;
}

// __partial_sort(first, last, last) == __make_heap + __sort_heap on h[0..len)
ORB_HD void qt_sortpar_heapsort(QtItem* h, int len) {
    for (int parent = (len - 2) / 2;; --parent) {
        const QtItem v = h[parent];
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
    for (int end = len - 1; end > 0; --end) {
        const QtItem v = h[end];
        h[end] = h[0];
        int hole = 0, child = 0;
        while (child < (end - 1) / 2) {
            child = 2 * (child + 1);
            if (qt_item_less(h[child], h[child - 1])) --child;
            h[hole] = h[child];
            hole = child;
        }
        if ((end & 1) == 0 && child == (end - 2) / 2) {
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
}


#if defined(__CUDACC__)
// One __introsort_loop step on [first, last) by a whole WARP, with exactly the result of qt_sortpar_partition.
// __unguarded_partition alternates two scans: `lo` runs up to the next item that is NOT LESS than the pivot, `hi` down to the next
// item that is NOT GREATER, the two are swapped, and so on until the scans meet.  Between two swaps both scans only cross items no
// earlier swap has touched, so the k-th stop of `lo` is the k-th position L_k (ascending, from first + 1) whose ORIGINAL key is not
// less than the pivot, the k-th stop of `hi` the k-th position R_k (descending, from last - 1; `first` itself, which holds the pivot,
// is the final sentinel) whose original key is not greater: swap k happens while L_k < R_k, and the scans meet at
// min(L_j, R_{j-1}) for the first j that fails (the item swapped into R_{j-1} stops `lo` if no untouched one does first).
// So: two ballot-ranked position lists, the swaps of all k < j at once, one formula for the cut.  (Phase clocks, round 2: one
// thread's chain of dependent swaps over ~250 items with many equal keys was the largest phase of the level-0 CTA.)
// scratch: 2 * (last - first) ints.  All 32 lanes call with the same arguments; returns the cut in every lane.
__device__ inline int qt_sortpar_partition_warp(QtItem* a, int first, int last, int* scratch, int lane) {
    const unsigned lt = (1u << lane) - 1u;
    if (lane == 0) {
        const int mid = first + (last - first) / 2;
        const int A = first + 1, B = mid, C = last - 1;
        int pick;
        if (qt_item_less(a[A], a[B])) {
            if (qt_item_less(a[B], a[C])) pick = B;
            else if (qt_item_less(a[A], a[C])) pick = C;
            else pick = A;
        } else if (qt_item_less(a[A], a[C])) pick = A;
        else if (qt_item_less(a[B], a[C])) pick = C;
        else pick = B;
        const QtItem t = a[first]; a[first] = a[pick]; a[pick] = t;
    }
    __syncwarp();
    const uint64_t pv = qt_item_key(a[first]);
    const int len = last - first;
    int* Lpos = scratch;          // ascending positions with key >= pivot
    int* Rpos = scratch + len;    // ascending positions with key <= pivot; Rpos[0] = first (the pivot itself)
    if (lane == 0) Rpos[0] = first;
    int nL = 0, nR = 1;
    for (int base = first + 1; base < last; base += 32) {
        const int p = base + lane;
        bool fl = false, fr = false;
        if (p < last) {
            const uint64_t k = qt_item_key(a[p]);
            fl = !(k < pv);
            fr = !(pv < k);
        }
        const unsigned ml = __ballot_sync(0xffffffffu, fl), mr = __ballot_sync(0xffffffffu, fr);
        if (fl) Lpos[nL + __popc(ml & lt)] = p;
        if (fr) Rpos[nR + __popc(mr & lt)] = p;
        nL += __popc(ml);
        nR += __popc(mr);
    }
    __syncwarp();
    const int kmax = nL < nR ? nL : nR;
    int j = 0;
    for (int base = 0; base < kmax; base += 32) {
        const int k = base + lane;
        int lp = 0, rp = 0;
        bool c = false;
        if (k < kmax) {
            lp = Lpos[k];
            rp = Rpos[nR - 1 - k];
            c = lp < rp;
        }
        const unsigned m = __ballot_sync(0xffffffffu, c);
        if (c) { const QtItem t = a[lp]; a[lp] = a[rp]; a[rp] = t; }     // the pairs of all k < j are disjoint positions
        j += __popc(m);
        if (m != 0xffffffffu) break;      // warp-uniform: L_k < R_k holds for a prefix of k only
    }
    __syncwarp();
    int cut;
    if (j == 0) cut = Lpos[0];            // exists: the median-of-three leaves an item >= pivot inside (first, last)
    else {
        const int rprev = Rpos[nR - j];   // R_{j-1}
        cut = (j < nL && Lpos[j] < rprev) ? Lpos[j] : rprev;
    }
    __syncwarp();
    return cut;
}
#define QT_COOP_MIN 40    // segments longer than this are partitioned by the whole warp, shorter ones one per lane
#endif

// a[0..n) sorted exactly as std::sort(a, a + n, compareNodes) leaves it.  tmp: n items.  seg / nxt: 3 ints per segment slot each
// (first, last, depth), room for n / 8 + 2 slots; flag: 2 * (n / 8 + 2) ints; scan_tmp: qt_exscan's scratch.  Whole CTA; returns after a
// barrier.  Every segment on a list is longer than 16, so a generation holds at most n / 17 of them.
ORB_HD void qt_std_sort_items_par(QtItem* a, int n, QtItem* tmp, int* seg, int* nxt, int* flag, int* scan_tmp, int nxt_ints) {
    if (n <= 1) return;   // uniform
    if (n > 16) {
        int lg = 0;
        for (int t = n; t > 1; t >>= 1) ++lg;
#if defined(__CUDA_ARCH__)
        // device: the generations are run by warp 0 alone -- a generation has at most n / 17 segments (one lane each), and its five
        // CTA barriers (partition | scan x 3 | scatter) become __syncwarp; the other warps wait at the one barrier below
        if (threadIdx.x < 32) {
            const int lane = threadIdx.x;
            const unsigned lt = (1u << lane) - 1u;
            int* cur = seg;      // 3 ints per segment: first, last, depth
            int* oth = nxt;
            if (lane == 0) { cur[0] = 0; cur[1] = n; cur[2] = 2 * lg; }
            __syncwarp();
            int nseg = 1;
            while (nseg > 0) {
                int off = 0;
                for (int base = 0; base < nseg; base += 32) {
                    const int sI = base + lane;
                    int first = 0, cut = 0, last = 0, depth = 0;
                    bool l_alive = false, r_alive = false;
                    const bool mine = sI < nseg;
                    if (mine) { first = cur[3 * sI]; last = cur[3 * sI + 1]; depth = cur[3 * sI + 2]; cut = first; }
                    // long segments first, one after the other, by the whole warp (tmp is free until the rank phase: its scratch)
                    const bool big = mine && depth != 0 && last - first > QT_COOP_MIN;
                    unsigned mb = __ballot_sync(0xffffffffu, big);
                    while (mb) {
                        const int src = __ffs(mb) - 1;
                        mb &= mb - 1;
                        const int f = __shfl_sync(0xffffffffu, first, src), l_ = __shfl_sync(0xffffffffu, last, src);
                        const int c = qt_sortpar_partition_warp(a, f, l_, reinterpret_cast<int*>(tmp), lane);
                        if (lane == src) cut = c;
                    }
                    if (mine && !big) {
                        if (depth == 0) qt_sortpar_heapsort(a + first, last - first);
                        else cut = qt_sortpar_partition(a, first, last);
                    }
                    if (mine) {
                        l_alive = depth != 0 && cut - first > 16;
                        r_alive = depth != 0 && last - cut > 16;
                    }
                    const unsigned ml = __ballot_sync(0xffffffffu, l_alive), mr = __ballot_sync(0xffffffffu, r_alive);
                    const int pos = off + __popc(ml & lt) + __popc(mr & lt);
                    if (l_alive) { oth[3 * pos] = first; oth[3 * pos + 1] = cut; oth[3 * pos + 2] = depth - 1; }
                    if (r_alive) { const int pr = pos + (l_alive ? 1 : 0); oth[3 * pr] = cut; oth[3 * pr + 1] = last; oth[3 * pr + 2] = depth - 1; }
                    off += __popc(ml) + __popc(mr);
                }
                __syncwarp();
                nseg = off;
                { int* t_ = cur; cur = oth; oth = t_; }
            }
        }
        QT_SYNC();
#else
        QT_SERIAL { seg[0] = 0; seg[1] = n; seg[2] = 2 * lg; }
        QT_SYNC();
        int nseg = 1;
        const int nslots_max = n / 8 + 2;     // 2 * (n / 17) slots at most
        while (nseg > 0) {
            QT_PAR_FOR(s, nseg) {
                const int first = seg[3 * s], last = seg[3 * s + 1], depth = seg[3 * s + 2];
                int cut = first;
                if (depth == 0) qt_sortpar_heapsort(a + first, last - first);      // this segment is finished
                else cut = qt_sortpar_partition(a, first, last);
                // children: the left part [first, cut) and the right part [cut, last), alive while longer than 16
                const bool l_alive = depth != 0 && cut - first > 16, r_alive = depth != 0 && last - cut > 16;
                nxt[3 * (2 * s)] = first; nxt[3 * (2 * s) + 1] = cut; nxt[3 * (2 * s) + 2] = depth - 1;
                nxt[3 * (2 * s + 1)] = cut; nxt[3 * (2 * s + 1) + 1] = last; nxt[3 * (2 * s + 1) + 2] = depth - 1;
                flag[2 * s] = flag[nslots_max + 2 * s] = l_alive ? 1 : 0;
                flag[2 * s + 1] = flag[nslots_max + 2 * s + 1] = r_alive ? 1 : 0;
            }
            QT_SYNC();
            // compact the alive children into the next generation's list: the flags live twice (the scan turns one copy into ranks);
            // `seg` is dead once the partitions are done, so the survivors are scattered straight into it
            const int nslots = 2 * nseg;
            const int alive = qt_exscan(flag, nslots, scan_tmp);
            QT_PAR_FOR(s, nslots) {
                if (flag[nslots_max + s]) {
                    const int d = flag[s];
                    seg[3 * d] = nxt[3 * s];
                    seg[3 * d + 1] = nxt[3 * s + 1];
                    seg[3 * d + 2] = nxt[3 * s + 2];
                }
            }
            QT_SYNC();
            nseg = alive;
        }
#endif
    }
    // __final_insertion_sort == stable sort of the current arrangement: rank(i) = #{j : key_j < key_i} + #{j < i : key_j == key_i}.
    // G threads share an item (each counts over a slice of j; nxt is free by now and holds the partial counts).
    int G = 1;
    while (G < 4 && 2 * G * n <= QT_NTHREADS && 2 * G * n <= nxt_ints) G <<= 1;
    const int slice = (n + G - 1) / G;
    QT_PAR_FOR(t, n * G) {
        const int i = t / G, part = t - i * G;
        const uint64_t kv = qt_item_key(a[i]);
        const int j0 = part * slice, j1 = (j0 + slice < n) ? j0 + slice : n;
        int rank = 0;
        for (int j = j0; j < j1; ++j) {
            const uint64_t ku = qt_item_key(a[j]);
            rank += (ku < kv ? 1 : 0) + ((ku == kv) & (j < i) ? 1 : 0);
        }
        nxt[t] = rank;
    }
    QT_SYNC();
    QT_PAR_FOR(i, n) {
        int rank = 0;
        for (int k = 0; k < G; ++k) rank += nxt[i * G + k];
        tmp[rank] = a[i];
    }
    QT_SYNC();
    QT_PAR_FOR(i, n) a[i] = tmp[i];
    QT_SYNC();
}

// Bitonic sort with two butterfly stages per pass (kept as the stepping stone to qt_bitonic_sort_r8 below, which k_quadtree_v1 uses).  For one merge size k the stages j = k/2 ... 1
// are taken in pairs (j, j/2): a thread loads the four elements that differ in bits j and j/2, does both compare-exchange
// levels in registers and stores them -- half the barriers and half the shared-memory round trips of qt_bitonic_sort; an odd
// stage count leaves one ordinary pass (j = 1).  Keys are unique per candidate pixel (root | path | score), so any correct sort
// yields the same array.
ORB_HD void qt_bitonic_sort_r4(uint32_t* arr, int npow) {
    for (int k = 2; k <= npow; k <<= 1) {
        int j = k >> 1;
        for (; j >= 2; j >>= 2) {
            const int h = j >> 1;
            QT_PAR_FOR(i, npow >> 2) {
                const int l0 = (i & (h - 1)) | ((i & ~(h - 1)) << 2);   // i spread over the index bits other than h and j = 2h
                uint32_t a0 = arr[l0], a1 = arr[l0 | h], a2 = arr[l0 | j], a3 = arr[l0 | j | h];
                const bool up = (l0 & k) == 0;
                uint32_t x;
                if ((a0 > a2) == up) { x = a0; a0 = a2; a2 = x; }
                if ((a1 > a3) == up) { x = a1; a1 = a3; a3 = x; }
                if ((a0 > a1) == up) { x = a0; a0 = a1; a1 = x; }
                if ((a2 > a3) == up) { x = a2; a2 = a3; a3 = x; }
                arr[l0] = a0; arr[l0 | h] = a1; arr[l0 | j] = a2; arr[l0 | j | h] = a3;
            }
            QT_SYNC();
        }
        if (j == 1) {
            QT_PAR_FOR(i, npow >> 1) {
                const int l = i << 1, r = l | 1;
                const uint32_t a = arr[l], b = arr[r];
                if ((a > b) == ((l & k) == 0)) { arr[l] = b; arr[r] = a; }
            }
            QT_SYNC();
        }
    }
}

// The same with up to THREE butterfly stages per pass (strides j, j/2, j/4: eight elements per thread, twelve compare-exchanges in
// registers); a remainder of two stages takes the four-element step, of one the ordinary pass.  8192 elements: 35 barriers instead
// of 49 (91 for one stage per pass).
ORB_HD void qt_bitonic_sort_r8(uint32_t* arr, int npow) {
#define QT_CX(x, y) { if (((x) > (y)) == up) { const uint32_t t_ = (x); (x) = (y); (y) = t_; } }
    for (int k = 2; k <= npow; k <<= 1) {
        int j = k >> 1;
        for (; j >= 4; j >>= 3) {
            const int h = j >> 1, q = j >> 2;
            QT_PAR_FOR(i, npow >> 3) {
                const int l0 = (i & (q - 1)) | ((i & ~(q - 1)) << 3);   // i spread over the index bits other than q, h = 2q, j = 4q
                uint32_t a0 = arr[l0], a1 = arr[l0 | q], a2 = arr[l0 | h], a3 = arr[l0 | h | q];
                uint32_t a4 = arr[l0 | j], a5 = arr[l0 | j | q], a6 = arr[l0 | j | h], a7 = arr[l0 | j | h | q];
                const bool up = (l0 & k) == 0;
                QT_CX(a0, a4) QT_CX(a1, a5) QT_CX(a2, a6) QT_CX(a3, a7)        // stride j
                QT_CX(a0, a2) QT_CX(a1, a3) QT_CX(a4, a6) QT_CX(a5, a7)        // stride h
                QT_CX(a0, a1) QT_CX(a2, a3) QT_CX(a4, a5) QT_CX(a6, a7)        // stride q
                arr[l0] = a0; arr[l0 | q] = a1; arr[l0 | h] = a2; arr[l0 | h | q] = a3;
                arr[l0 | j] = a4; arr[l0 | j | q] = a5; arr[l0 | j | h] = a6; arr[l0 | j | h | q] = a7;
            }
            QT_SYNC();
        }
        if (j == 2) {          // two stages left: strides 2 and 1
            QT_PAR_FOR(i, npow >> 2) {
                const int l0 = i << 2;
                uint32_t a0 = arr[l0], a1 = arr[l0 | 1], a2 = arr[l0 | 2], a3 = arr[l0 | 3];
                const bool up = (l0 & k) == 0;
                QT_CX(a0, a2) QT_CX(a1, a3) QT_CX(a0, a1) QT_CX(a2, a3)
                arr[l0] = a0; arr[l0 | 1] = a1; arr[l0 | 2] = a2; arr[l0 | 3] = a3;
            }
            QT_SYNC();
        } else if (j == 1) {   // one stage left
            QT_PAR_FOR(i, npow >> 1) {
                const int l = i << 1;
                uint32_t a0 = arr[l], a1 = arr[l | 1];
                const bool up = (l & k) == 0;
                QT_CX(a0, a1)
                arr[l] = a0; arr[l | 1] = a1;
            }
            QT_SYNC();
        }
    }
#undef QT_CX
}

#if defined(__CUDACC__)
// ---- device only: bitonic sort whose strides <= 128 never touch shared memory -----------------------------------------------
// Under ncu qt_bitonic_sort_r8 was a large share of k_quadtree_v1 (the larger at levels 1-7) and took four
// times the ideal shared-memory wavefronts -- in the passes with strides < 32 a thread's eight elements are 8 / 4 / 2 words apart
// from its neighbour's, an 8- / 4- / 2-way bank conflict on all sixteen accesses.  Here a warp owns 256 consecutive elements: lane
// i holds arr[base + 4 i .. + 3] and arr[base + 128 + 4 i .. + 3] (two conflict-free 128-bit accesses), so strides 128, 2 and 1 are
// compare-exchanges between a lane's own registers and strides 64 .. 4 are one shuffle each with lane ^ 16 .. lane ^ 1.  All merges
// up to 256 run in one such pass; a larger merge takes shared-memory passes (three / two / one stage each, strides >= 256 only:
// conflict-free) followed by one warp pass.  8192 elements: 13 barriers (35 before, 91 with one stage per pass).  Keys are unique,
// so any correct sort gives the same array.
__device__ __forceinline__ void qt_warp_stages(uint32_t (&v)[8], int idx0, int k, int jstart, int lane) {
#define QT_IDX(e) (idx0 + ((e) & 3) + (((e) >> 2) << 7))
#define QT_CXU(x, y, up) { const uint32_t lo_ = min((x), (y)), hi_ = max((x), (y)); (x) = (up) ? lo_ : hi_; (y) = (up) ? hi_ : lo_; }
#pragma unroll
    for (int s = 7; s >= 0; --s) {
        const int j = 1 << s;
        if (j > jstart) continue;
        if (s == 7) {
#pragma unroll
            for (int e = 0; e < 4; ++e) QT_CXU(v[e], v[e + 4], (QT_IDX(e) & k) == 0)
        } else if (s >= 2) {
            const int m = j >> 2;
            const bool lower = (lane & m) == 0;
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const bool up = (QT_IDX(e) & k) == 0;
                const uint32_t other = __shfl_xor_sync(0xffffffffu, v[e], m);
                v[e] = (lower == up) ? min(v[e], other) : max(v[e], other);
            }
        } else if (s == 1) {
            QT_CXU(v[0], v[2], (QT_IDX(0) & k) == 0) QT_CXU(v[1], v[3], (QT_IDX(1) & k) == 0)
            QT_CXU(v[4], v[6], (QT_IDX(4) & k) == 0) QT_CXU(v[5], v[7], (QT_IDX(5) & k) == 0)
        } else {
            QT_CXU(v[0], v[1], (QT_IDX(0) & k) == 0) QT_CXU(v[2], v[3], (QT_IDX(2) & k) == 0)
            QT_CXU(v[4], v[5], (QT_IDX(4) & k) == 0) QT_CXU(v[6], v[7], (QT_IDX(6) & k) == 0)
        }
    }
#undef QT_IDX
#undef QT_CXU
}

// npow: a power of two >= 256; arr 16-byte aligned; whole CTA (blockDim a multiple of 32); returns after a barrier
__device__ inline void qt_bitonic_sort_w(uint32_t* arr, int npow) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5, nblk = npow >> 8;
#define QT_CX(x, y) { if (((x) > (y)) == up) { const uint32_t t_ = (x); (x) = (y); (y) = t_; } }
    for (int kk = 256; kk <= npow; kk <<= 1) {
        // shared-memory passes for the strides >= 256 of merge size kk (none for kk == 256)
        int j = kk >> 1;
        for (; j >= 1024; j >>= 3) {
            const int h = j >> 1, q = j >> 2;
            for (int i = threadIdx.x; i < (npow >> 3); i += blockDim.x) {
                const int l0 = (i & (q - 1)) | ((i & ~(q - 1)) << 3);
                uint32_t a0 = arr[l0], a1 = arr[l0 | q], a2 = arr[l0 | h], a3 = arr[l0 | h | q];
                uint32_t a4 = arr[l0 | j], a5 = arr[l0 | j | q], a6 = arr[l0 | j | h], a7 = arr[l0 | j | h | q];
                const bool up = (l0 & kk) == 0;
                QT_CX(a0, a4) QT_CX(a1, a5) QT_CX(a2, a6) QT_CX(a3, a7)
                QT_CX(a0, a2) QT_CX(a1, a3) QT_CX(a4, a6) QT_CX(a5, a7)
                QT_CX(a0, a1) QT_CX(a2, a3) QT_CX(a4, a5) QT_CX(a6, a7)
                arr[l0] = a0; arr[l0 | q] = a1; arr[l0 | h] = a2; arr[l0 | h | q] = a3;
                arr[l0 | j] = a4; arr[l0 | j | q] = a5; arr[l0 | j | h] = a6; arr[l0 | j | h | q] = a7;
            }
            __syncthreads();
        }
        if (j == 512) {          // strides 512 and 256
            for (int i = threadIdx.x; i < (npow >> 2); i += blockDim.x) {
                const int l0 = (i & 255) | ((i & ~255) << 2);
                uint32_t a0 = arr[l0], a1 = arr[l0 | 256], a2 = arr[l0 | 512], a3 = arr[l0 | 768];
                const bool up = (l0 & kk) == 0;
                QT_CX(a0, a2) QT_CX(a1, a3) QT_CX(a0, a1) QT_CX(a2, a3)
                arr[l0] = a0; arr[l0 | 256] = a1; arr[l0 | 512] = a2; arr[l0 | 768] = a3;
            }
            __syncthreads();
        } else if (j == 256) {   // stride 256 alone
            for (int i = threadIdx.x; i < (npow >> 1); i += blockDim.x) {
                const int l0 = (i & 255) | ((i & ~255) << 1);
                uint32_t a0 = arr[l0], a1 = arr[l0 | 256];
                const bool up = (l0 & kk) == 0;
                QT_CX(a0, a1)
                arr[l0] = a0; arr[l0 | 256] = a1;
            }
            __syncthreads();
        }
        // warp pass: strides 128 .. 1 of merge size kk; for kk == 256 every merge from 2 up to 256
        for (int b = warp; b < nblk; b += nwarps) {
            const int base = b << 8, idx0 = base + 4 * lane;
            uint4* p0 = reinterpret_cast<uint4*>(arr + idx0);
            uint4* p1 = reinterpret_cast<uint4*>(arr + idx0 + 128);
            const uint4 x0 = *p0, x1 = *p1;
            uint32_t v[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
            if (kk == 256) {
                for (int k = 2; k <= 256; k <<= 1) qt_warp_stages(v, idx0, k, k >> 1, lane);
            } else {
                qt_warp_stages(v, idx0, kk, 128, lane);
            }
            *p0 = make_uint4(v[0], v[1], v[2], v[3]);
            *p1 = make_uint4(v[4], v[5], v[6], v[7]);
        }
        __syncthreads();
    }
#undef QT_CX
}
#endif  // __CUDACC__

}  // namespace orbdev
