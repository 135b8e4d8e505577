// liba.cu -- Optimizer::LocalInertialBA's numeric core on the device (include/orbslam3_b200.h, liba_*).
// The algorithm lives in liba_core.cuh as barrier-separated SPMD phases shared with the CPU emulation harness; this file is
// the launch wrapper: one thread-block cluster (or one CTA) per window, everything for a window in one blob (liba_pack.h),
// fp64 throughout.
#include <cuda_runtime.h>
#include <stdlib.h>

#include <vector>

#include "common.cuh"
#include "liba_pack.h"
#include "scratch.h"

using namespace orb;

static_assert(sizeof(liba_problem) == 232 && sizeof(liba_result) == 80, "C ABI layout (include/orbslam3_b200.h)");

namespace {

constexpr int LIBA_THREADS = 256;
constexpr int LIBA_CS_MAX = 8;       // CTAs (SMs) per window: a portable-size thread-block cluster

// One team (a cluster of `cs` CTAs, or one CTA) per window; blocks of a cluster are consecutive in x.
__global__ void __launch_bounds__(LIBA_THREADS) k_liba(const LibaDev* __restrict__ problems, int cs) {
    __shared__ double s_red[LIBA_THREADS / 32];
    LibaDev P = problems[blockIdx.x / cs];
    P.red = s_red;
    P.cs = cs;
    P.rank = blockIdx.x % cs;
    P.l_id = threadIdx.x;
    P.l_stride = blockDim.x;
    P.t_id = P.rank * blockDim.x + threadIdx.x;
    P.t_stride = cs * blockDim.x;
    liba_optimize(P);
}

}  // namespace

struct liba_handle {
    int device = 0;
    cudaStream_t stream = nullptr;
    uint8_t* d_buf = nullptr;
    size_t d_bytes = 0;
    uint8_t* h_buf = nullptr;
    size_t h_bytes = 0;
    int n_sms = 1;
};

extern "C" orb_status liba_create(int32_t device, liba_handle** out) {
    if (!out) return set_error(ORB_ERR_INVALID, "null argument");
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev)
        return set_error(ORB_ERR_NO_DEVICE, "no usable CUDA device (this library has no CPU fallback)");
    ORB_CUDA(cudaSetDevice(device));
    liba_handle* h = new liba_handle();
    h->device = device;
    h->n_sms = device_sm_count(device);
    if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete h;
        return set_error(ORB_ERR_CUDA, "cudaStreamCreate failed");
    }
    ORB_CUDA(cudaFuncSetAttribute(k_liba, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));   // 16-CTA clusters for one or two windows
    *out = h;
    return ORB_OK;
}

extern "C" void liba_destroy(liba_handle* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (h->d_buf) cudaFree(h->d_buf);
    if (h->h_buf) cudaFreeHost(h->h_buf);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

extern "C" orb_status liba_solve(liba_handle* h, int32_t n_problems, const liba_problem* in, liba_result* out) {
    if (!h || !in || !out || n_problems < 0) return set_error(ORB_ERR_INVALID, "null argument");
    if (n_problems == 0) return ORB_OK;
    ORB_CUDA(cudaSetDevice(h->device));
    for (int i = 0; i < n_problems; ++i) {
        const liba_problem& p = in[i];
        if (p.n_kf <= 0 || p.n_mp < 0 || p.n_edges < 0 || p.n_links < 0 || !p.state || !p.fixed || !out[i].state || !out[i].point ||
            (p.n_mp && !p.point) || (p.n_edges && (!p.edge_kf || !p.edge_mp || !p.obs || !p.inv_sigma2)) || (p.n_links && !p.links))
            return set_error(ORB_ERR_INVALID, "liba_problem: missing array");
        for (int e = 0; e < p.n_edges; ++e)
            if (p.edge_kf[e] < 0 || p.edge_kf[e] >= p.n_kf || p.edge_mp[e] < 0 || p.edge_mp[e] >= p.n_mp)
                return set_error(ORB_ERR_INVALID, "liba_problem: edge index out of range");
        for (int l = 0; l < p.n_links; ++l)
            if (p.links[l].k1 < 0 || p.links[l].k1 >= p.n_kf || p.links[l].k2 < 0 || p.links[l].k2 >= p.n_kf)
                return set_error(ORB_ERR_INVALID, "liba_problem: link index out of range");
    }
    // blob: [LibaDev x n] then per problem io | in | work
    std::vector<LibaLayout> lay(n_problems);
    std::vector<size_t> base(n_problems);
    size_t total = ((sizeof(LibaDev) * (size_t)n_problems) + 255) & ~(size_t)255;
    for (int i = 0; i < n_problems; ++i) {
        lay[i] = liba_pack(in[i], nullptr, nullptr, nullptr);
        if (lay[i].total == 0) return set_error(ORB_ERR_INVALID, "liba_problem: two links join the same keyframe pair (or > 65535 keyframes)");
        base[i] = total;
        total += (lay[i].total + 255) & ~(size_t)255;
    }
    orb_status s = grow_device(h->d_bytes, h->d_buf, total, false);
    if (s != ORB_OK || (s = grow_pinned(h->h_bytes, h->h_buf, total)) != ORB_OK) return s;
    LibaDev* hdev = reinterpret_cast<LibaDev*>(h->h_buf);
    ORB_CUDA(cudaMemsetAsync(h->d_buf, 0, total, h->stream));
    for (int i = 0; i < n_problems; ++i) liba_pack(in[i], h->h_buf + base[i], h->d_buf + base[i], &hdev[i]);
    ORB_CUDA(cudaMemcpyAsync(h->d_buf, h->h_buf, sizeof(LibaDev) * (size_t)n_problems, cudaMemcpyHostToDevice, h->stream));
    for (int i = 0; i < n_problems; ++i)
        ORB_CUDA(cudaMemcpyAsync(h->d_buf + base[i], h->h_buf + base[i], lay[i].io_bytes + lay[i].in_bytes, cudaMemcpyHostToDevice, h->stream));
    // one or two windows get a cluster of 16 SMs each (the non-portable size), small batches 8, large ones fewer
    // (ORB_LIBA_CLUSTER = 1 | 2 | 4 | 8 | 16 overrides: a tuning knob)
    const int sms = h->n_sms;
    int cs = n_problems <= 2 ? 16 : ((n_problems * LIBA_CS_MAX <= sms) ? LIBA_CS_MAX : (n_problems * 4 <= sms ? 4 : (n_problems * 2 <= sms ? 2 : 1)));
    if (const char* e = getenv("ORB_LIBA_CLUSTER")) {
        const int v = atoi(e);
        if (v == 1 || v == 2 || v == 4 || v == 8 || v == 16) cs = v;
    }
    ORB_CUDA(fit_cluster_size(k_liba, &cs, LIBA_THREADS, 0));
    {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(n_problems * cs);
        cfg.blockDim = dim3(LIBA_THREADS);
        cfg.dynamicSmemBytes = 0;
        cfg.stream = h->stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = cs;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        ORB_CUDA(cudaLaunchKernelEx(&cfg, k_liba, reinterpret_cast<const LibaDev*>(h->d_buf), cs));
    }
    ORB_LAUNCHED();
    ORB_CUDA(cudaGetLastError());
    for (int i = 0; i < n_problems; ++i)
        ORB_CUDA(cudaMemcpyAsync(h->h_buf + base[i], h->d_buf + base[i], lay[i].io_bytes, cudaMemcpyDeviceToHost, h->stream));
    ORB_CUDA(cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n_problems; ++i) liba_unpack(in[i], h->h_buf + base[i], hdev[i], h->d_buf + base[i], &out[i]);
    return ORB_OK;
}

// ---- host helper: the information matrices of one link from IMU::Preintegrated::C ---------------------------------------------
namespace {

bool invert_n(const double* A, int n, double* out) {      // Gauss-Jordan with partial pivoting (Eigen's inverse() is PartialPivLU)
    std::vector<double> a(A, A + n * n);
    for (int i = 0; i < n * n; ++i) out[i] = (i / n == i % n) ? 1.0 : 0.0;
    for (int c = 0; c < n; ++c) {
        int piv = c;
        for (int r = c + 1; r < n; ++r) if (fabs(a[r * n + c]) > fabs(a[piv * n + c])) piv = r;
        if (!(fabs(a[piv * n + c]) > 0)) return false;
        if (piv != c) for (int k = 0; k < n; ++k) { std::swap(a[c * n + k], a[piv * n + k]); std::swap(out[c * n + k], out[piv * n + k]); }
        const double d = 1.0 / a[c * n + c];
        for (int k = 0; k < n; ++k) { a[c * n + k] *= d; out[c * n + k] *= d; }
        for (int r = 0; r < n; ++r) {
            if (r == c) continue;
            const double f = a[r * n + c];
            if (f == 0.0) continue;
            for (int k = 0; k < n; ++k) { a[r * n + k] -= f * a[c * n + k]; out[r * n + k] -= f * out[c * n + k]; }
        }
    }
    return true;
}

void jacobi_eigen(double* A, int n, double* V) {          // cyclic Jacobi: A (symmetric) -> diagonal, V = eigenvectors (columns)
    for (int i = 0; i < n * n; ++i) V[i] = (i / n == i % n) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 64; ++sweep) {
        double off = 0, diag = 0;
        for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) (i == j ? diag : off) += A[i * n + j] * A[i * n + j];
        if (off <= 1e-32 * diag) break;
        for (int p = 0; p < n; ++p)
            for (int q = p + 1; q < n; ++q) {
                if (A[p * n + q] == 0.0) continue;
                const double theta = (A[q * n + q] - A[p * n + p]) / (2.0 * A[p * n + q]);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < n; ++k) { const double akp = A[k * n + p], akq = A[k * n + q]; A[k * n + p] = c * akp - s * akq; A[k * n + q] = s * akp + c * akq; }
                for (int k = 0; k < n; ++k) { const double apk = A[p * n + k], aqk = A[q * n + k]; A[p * n + k] = c * apk - s * aqk; A[q * n + k] = s * apk + c * aqk; }
                for (int k = 0; k < n; ++k) { const double vkp = V[k * n + p], vkq = V[k * n + q]; V[k * n + p] = c * vkp - s * vkq; V[k * n + q] = s * vkp + c * vkq; }
            }
    }
}

}  // namespace

extern "C" orb_status liba_link_information(const float* C15, int32_t oldest, double* info81, double* infoG9, double* infoA9) {
    if (!C15 || !info81 || !infoG9 || !infoA9) return set_error(ORB_ERR_INVALID, "null argument");
    double M[81], Mi[81], V[81];
    for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) M[9 * i + j] = (double)C15[15 * i + j];
    if (!invert_n(M, 9, Mi)) return set_error(ORB_ERR_INVALID, "liba_link_information: singular covariance block");
    for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) M[9 * i + j] = (Mi[9 * i + j] + Mi[9 * j + i]) / 2;      // G2oTypes.cc:577
    jacobi_eigen(M, 9, V);
    double eig[9];
    for (int i = 0; i < 9; ++i) eig[i] = M[9 * i + i] < 1e-12 ? 0.0 : M[9 * i + i];                                    // G2oTypes.cc:580-583
    const double scale = oldest ? 1e-2 : 1.0;                                                                         // Optimizer.cc:2477-2478
    for (int i = 0; i < 9; ++i)
        for (int j = 0; j < 9; ++j) {
            double s = 0;
            for (int k = 0; k < 9; ++k) s += V[9 * i + k] * eig[k] * V[9 * j + k];
            info81[9 * i + j] = s * scale;
        }
    for (int b = 0; b < 2; ++b) {
        double B[9];
        const int o = 9 + 3 * b;
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) B[3 * i + j] = (double)C15[15 * (o + i) + o + j];
        if (!invert_n(B, 3, b == 0 ? infoG9 : infoA9)) return set_error(ORB_ERR_INVALID, "liba_link_information: singular random-walk covariance");
    }
    return ORB_OK;
}
