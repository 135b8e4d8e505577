// tests/host/liba_stub.cc -- TEST INFRASTRUCTURE (CPU tier): liba_solve over the oracle (orc_liba) instead of the GPU, so that
// host/Optimizer_liba_b200.cc -- temporal window, fixed keyframes, flattening, outlier pass, failure rule, write-back -- can run without
// a GPU next to the reference's own function (tests/test_host_liba_vs_ref.py).  liba_link_information (a host-only helper, no device
// work) comes from liborbslam3_b200.so in both binaries.  Never linked into the product.
#include <cstdint>
#include <vector>

#include "orbslam3_b200.h"

extern "C" int orc_liba(int nKF, int nMP, int nE, int nL, double* state, const uint8_t* fixed, double* point, const int* ekf, const int* emp,
                        const double* obs, const double* invs2, const double* Tcb12, const double* cam5, const void* links_raw, double lambdaInit,
                        int maxIters, double* edge_chi2, double* link_chi2, double* stats, uint8_t* edge_depth_positive);
extern "C" int orc_inertial_link_size();

extern "C" {
void* liba_mock_camera() { static double storage[4]; return storage; }   // a GeometricCamera object for the mock keyframes (the stand-in class is empty)
orb_status liba_create(int32_t, liba_handle** out) { static int dummy; *out = reinterpret_cast<liba_handle*>(&dummy); return ORB_OK; }
void liba_destroy(liba_handle*) {}

orb_status liba_solve(liba_handle*, int32_t n_problems, const liba_problem* in, liba_result* out) {
    if (orc_inertial_link_size() != (int)sizeof(liba_link)) return ORB_ERR_INVALID;
    for (int q = 0; q < n_problems; ++q) {
        const liba_problem& P = in[q];
        liba_result& R = out[q];
        std::vector<double> state(P.state, P.state + 21 * (size_t)P.n_kf), point(P.point, P.point + 3 * (size_t)P.n_mp);
        point.resize(point.size() + 3);
        const double cam5[5] = {P.fx, P.fy, P.cx, P.cy, P.bf};
        std::vector<double> chi2(P.n_edges + 1), lchi(3 * (size_t)P.n_links + 3);
        std::vector<uint8_t> dpos(P.n_edges + 1);
        double stats[8] = {0};
        const int it = orc_liba(P.n_kf, P.n_mp, P.n_edges, P.n_links, state.data(), P.fixed, point.data(), P.edge_kf, P.edge_mp, P.obs, P.inv_sigma2, P.Tcb,
                                cam5, P.links, P.lambda_init, P.max_iters, chi2.data(), lchi.data(), stats, dpos.data());
        for (size_t i = 0; i < 21 * (size_t)P.n_kf; ++i) R.state[i] = state[i];
        for (size_t i = 0; i < 3 * (size_t)P.n_mp; ++i) R.point[i] = point[i];
        for (int e = 0; e < P.n_edges; ++e) {
            if (R.edge_chi2) R.edge_chi2[e] = chi2[e];
            if (R.edge_depth_positive) R.edge_depth_positive[e] = dpos[e];
        }
        if (R.link_chi2) for (int i = 0; i < 3 * P.n_links; ++i) R.link_chi2[i] = lchi[i];
        R.iterations = it; R.trials = (int)stats[3]; R.lambda = stats[1]; R.chi2 = stats[2]; R.chi2_initial = stats[4]; R.chi2_last_trial = stats[5];
    }
    return ORB_OK;
}
}
