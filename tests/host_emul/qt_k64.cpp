// tests/host_emul/qt_k64.cpp -- csrc/quadtree_core.cuh on either sort element (QtForm<uint32_t> / QtForm<uint64_t>), compiled three
// ways from this one file:
//   default                  one host thread
//   -DQT_EMUL_THREADS        T host threads that play one CTA with a real barrier (built with -fsanitize=thread: a missing QT_SYNC
//                            is reported as a data race, exit code 66)
//   -DQT_HOST_COUNT_SYNCS    one thread counting the barriers a CTA would execute (printed on stdout)
// Usage: qt_k64 <in.bin> <out.bin> <threads> <element bits: 32 | 64>
//   in:  int32 n regionW regionH N wCell hCell nCols variant, then n x (x, y, score)      out: int32 S, then S x (x, y, score)
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>
#if defined(QT_EMUL_THREADS)
#include <barrier>
#include <thread>
#endif

#include "../../orb_slam3_detailed_comments_b200/csrc/devmath.cuh"
#if defined(QT_HOST_COUNT_SYNCS)
namespace orbdev { long qt_sync_count = 0; }
#endif
#include "../../orb_slam3_detailed_comments_b200/csrc/quadtree_core.cuh"

#if defined(QT_EMUL_THREADS)
namespace orbdev {
thread_local int qt_tid = 0;
int qt_nthreads = 1;
static std::barrier<>* g_bar = nullptr;
void qt_barrier() { g_bar->arrive_and_wait(); }
}
#endif
using namespace orbdev;

template <typename E>
static int run(const std::vector<int32_t>& c, int n, const QtGeom& g, int variant, int T, std::vector<uint32_t>& out) {
    int npow = 2;
    while (npow < n) npow <<= 1;
    std::vector<E> arr(npow, ~(E)0);
    for (int i = 0; i < n; ++i) arr[i] = qt_element<E>(qt_pack_cand(c[3 * i], c[3 * i + 1], c[3 * i + 2]), g);
    const int cap = g.N + 20;
    std::vector<char> ws(qt_work_bytes(cap));
    out.assign(cap + 4, 0);
    auto body = [&]() {
        if (variant == 0) qt_bitonic_sort(arr.data(), npow); else qt_bitonic_sort_r8(arr.data(), npow);
        QtWork w;                             // per-thread copy of the workspace descriptor, like the kernel's registers
        qt_work_carve(w, ws.data(), cap);
        return variant == 0 ? qt_distribute_v<0>(arr.data(), n, g, w, out.data()) : qt_distribute_v<1>(arr.data(), n, g, w, out.data());
    };
#if defined(QT_EMUL_THREADS)
    qt_nthreads = T;
    std::barrier<> bar(T);
    g_bar = &bar;
    std::vector<int> S(T, -9);
    std::vector<std::thread> th;
    for (int t = 0; t < T; ++t)
        th.emplace_back([&, t] {
            qt_tid = t;
            S[t] = body();
        });
    for (auto& t : th) t.join();
    for (int t = 1; t < T; ++t)
        if (S[t] != S[0]) return -1000;   // the return value must be uniform across the CTA
    return S[0];
#else
    (void)T;
#if defined(QT_HOST_COUNT_SYNCS)
    qt_sync_count = 0;
#endif
    const int S = body();
#if defined(QT_HOST_COUNT_SYNCS)
    printf("%ld %d\n", qt_sync_count, npow);
#endif
    return S;
#endif
}

int main(int argc, char** argv) {
    if (argc < 5) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    int32_t hdr[8];
    if (fread(hdr, 4, 8, f) != 8) return 2;
    const int n = hdr[0], variant = hdr[7];
    std::vector<int32_t> c(3 * (size_t)n + 3);
    if (n && fread(c.data(), 4, 3 * (size_t)n, f) != 3 * (size_t)n) return 2;
    fclose(f);
    QtGeom g;
    g.regionW = hdr[1]; g.regionH = hdr[2];
    g.nIni = (int)std::round((float)g.regionW / (float)g.regionH);
    g.hX = (float)g.regionW / (float)g.nIni;
    g.N = hdr[3]; g.wCell = hdr[4]; g.hCell = hdr[5]; g.nCols = hdr[6];
    std::vector<uint32_t> out;
    const int T = atoi(argv[3]);
    const int S = atoi(argv[4]) == 64 ? run<uint64_t>(c, n, g, variant, T, out) : run<uint32_t>(c, n, g, variant, T, out);
    if (S == -1000) return 4;
    FILE* o = fopen(argv[2], "wb");
    if (!o) return 2;
    const int32_t s32 = S;
    fwrite(&s32, 4, 1, o);
    for (int i = 0; i < S; ++i) {
        const int32_t r[3] = {(int32_t)(out[i] & 0xfff), (int32_t)((out[i] >> 12) & 0xfff), (int32_t)(out[i] >> 24)};
        fwrite(r, 4, 3, o);
    }
    fclose(o);
    return 0;
}
