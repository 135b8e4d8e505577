// tests/host/lba_stub.cc -- TEST INFRASTRUCTURE (CPU tier): lba_solve_bool over the oracle (orc_lba) instead of the GPU, so that
// host/Optimizer_lba_b200.cc -- window selection, flattening, outlier pass, write-back -- can run without a GPU next to the
// reference's own function (tests/test_host_lba_vs_ref.py).  Never linked into the product.
#include <cstdint>
#include <vector>

#include "orbslam3_b200.h"

extern "C" int orc_lba(int nKF, int nMP, int nE, double* pose, const uint8_t* fixed, double* point, const int* ekf, const int* emp, const double* obs,
                       const double* invs2, const double* cam5, double lambdaInit, int maxIters, const volatile int* stop_flag, double* edge_chi2,
                       uint8_t* edge_depth_pos, double* stats);

extern "C" {
const char* orb_last_error(void) { return "lba_stub"; }
lba_handle* orb_b200_lba_handle(void) { static int dummy; return reinterpret_cast<lba_handle*>(&dummy); }

orb_status lba_solve_bool(lba_handle*, const lba_problem* in, lba_result* out, const volatile uint8_t* stop_flag) {
    std::vector<double> pose(in->pose, in->pose + 7 * (size_t)in->n_kf), point(in->point, in->point + 3 * (size_t)in->n_mp);
    const double cam5[5] = {in->fx, in->fy, in->cx, in->cy, in->bf};
    volatile int stop = (stop_flag && *stop_flag) ? 1 : 0;
    double stats[8] = {0};
    std::vector<double> chi2(in->n_edges + 1);
    std::vector<uint8_t> dpos(in->n_edges + 1);
    const int it = orc_lba(in->n_kf, in->n_mp, in->n_edges, pose.data(), in->fixed, point.data(), in->edge_kf, in->edge_mp, in->obs, in->inv_sigma2, cam5,
                           in->lambda_init, in->max_iters, &stop, chi2.data(), dpos.data(), stats);
    for (size_t i = 0; i < pose.size(); ++i) out->pose[i] = pose[i];
    for (size_t i = 0; i < point.size(); ++i) out->point[i] = point[i];
    for (int e = 0; e < in->n_edges; ++e) {
        if (out->edge_chi2) out->edge_chi2[e] = chi2[e];
        if (out->edge_depth_positive) out->edge_depth_positive[e] = dpos[e];
    }
    out->iterations = it; out->trials = (int)stats[3]; out->lambda = stats[1]; out->chi2 = stats[2]; out->chi2_initial = stats[4];
    return ORB_OK;
}
}
