// Optimizer_liba_b200.cc -- Optimizer::LocalInertialBA (/root/reference/src/Optimizer.cc:2203-2812) on the GPU.
//
// Compiled against the reference's UNMODIFIED include/Optimizer.h (signature :86).  What stays on the host is what touches the map's
// objects: the temporal window (the keyframe and its mPrevKF chain, :2217-2245), its map points (:2248-2270), the fixed keyframes
// (the one before the window and one other observer per point, :2272-2340), flattening them into the arrays liba_solve takes
// (vertices :2363-2424, inertial links :2427-2510, reprojection edges :2548-2660), the outlier pass (:2690-2726), the failure rule
// (:2731-2735) and the write-back under the map mutex (:2738-2808).  Everything g2o did in between -- VertexPose / Velocity / GyroBias /
// AccBias, EdgeInertial / EdgeGyroRW / EdgeAccRW / EdgeMono / EdgeStereo with their Huber kernels, BlockSolverX, the Levenberg loop -- is
// one kernel launch (k_liba, csrc/liba.cu) behind liba_solve.
// Link before the reference's Optimizer.o with -Wl,--allow-multiple-definition, or exclude that one body from Optimizer.cc.
//
// Differences a caller can see, all below float resolution of the written poses or refused loudly:
//  * VertexPose starts from the keyframe's float Tcw AND its float body pose (ImuCamPose's constructor, G2oTypes.cc:30-70) and only
//    recomputes Rcw = Rcb Rbw at its first update; liba_solve takes the body pose and derives the camera pose from it at every evaluation
//    (the two differ by float rounding of the keyframe's own members, ~1e-7).  tbc is derived from Tcb, not read from mImuCalib.mTbc.
//  * not built: optimisable keyframes without IMU (bImu false: pose-only vertices inside an inertial window) and right-camera
//    observations of two-camera rigs (EdgeMono(1), :2622-2657) -- such a window is refused with an exception.
//  * GeometricCamera::uncertainty2 (:2583, :2609) is 1.0f in both camera models of the tree (Pinhole.h, KannalaBrandt8.h); x / 1.0f == x.
//  * `assert(mit->second >= 3)` (:2664) is compiled out of the reference's Release build; it is not evaluated here.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <list>
#include <map>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "Optimizer.h"        // the reference's header
#include "orb_b200_host.h"

namespace {

struct LibaRegistry {
    std::mutex mu;
    liba_handle* h = nullptr;
    ~LibaRegistry() { if (h) liba_destroy(h); }
};

liba_handle* liba_handle_of_process() {   // one LocalInertialBA workspace per process (created on first use, released at exit)
    static LibaRegistry r;
    std::lock_guard<std::mutex> lk(r.mu);
    if (!r.h) orb_b200::check(liba_create(orb_b200::device_ordinal(), &r.h), "liba_create");
    return r.h;
}

template <class M3>
void put3x3(float* dst, const M3& m) { for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) dst[3 * r + c] = m(r, c); }

}  // namespace

namespace ORB_SLAM3 {

void Optimizer::LocalInertialBA(KeyFrame* pKF, bool* pbStopFlag, Map* pMap, int& num_fixedKF, int& num_OptKF, int& num_MPs, int& num_edges,
                                bool bLarge, bool bRecInit) {
    (void)pbStopFlag;   // the reference installs the flag AFTER optimize() (:2683-2685): it never stops this optimisation
    (void)num_fixedKF; (void)num_OptKF; (void)num_MPs; (void)num_edges;   // never assigned by the reference either
    Map* pCurrentMap = pKF->GetMap();
    const int maxOpt = bLarge ? 25 : 10, opt_it = bLarge ? 4 : 10;
    const int Nd = std::min((int)pCurrentMap->KeyFramesInMap() - 2, maxOpt);
    const unsigned long ba_id = pKF->mnId;

    // ---- temporal window: the keyframe and its predecessors ----
    std::vector<KeyFrame*> vOpt;
    vOpt.reserve(Nd > 0 ? Nd : 1);
    vOpt.push_back(pKF);
    pKF->mnBALocalForKF = ba_id;
    for (int i = 1; i < Nd; ++i) {
        KeyFrame* prev = vOpt.back()->mPrevKF;
        if (!prev) break;
        vOpt.push_back(prev);
        prev->mnBALocalForKF = ba_id;
    }
    // ---- their map points, in keyframe then feature order ----
    std::vector<MapPoint*> vPoints;
    for (KeyFrame* k : vOpt) {
        const std::vector<MapPoint*> vpMPs = k->GetMapPointMatches();
        for (MapPoint* pMP : vpMPs)
            if (pMP && !pMP->isBad() && pMP->mnBALocalForKF != ba_id) {
                vPoints.push_back(pMP);
                pMP->mnBALocalForKF = ba_id;
            }
    }
    // ---- fixed keyframes: the one before the window (or, without one, the window's oldest), then one other observer per point ----
    std::vector<KeyFrame*> vFixed;
    if (vOpt.back()->mPrevKF) {
        vFixed.push_back(vOpt.back()->mPrevKF);
        vOpt.back()->mPrevKF->mnBAFixedForKF = ba_id;
    } else {
        vOpt.back()->mnBALocalForKF = 0;
        vOpt.back()->mnBAFixedForKF = ba_id;
        vFixed.push_back(vOpt.back());
        vOpt.pop_back();
    }
    // (covisible optimisable keyframes: maxCovKF = 0, the loop at :2289 leaves at its first test)
    const size_t maxFixKF = 200;
    std::vector<std::map<KeyFrame*, std::tuple<int, int>>> vObs(vPoints.size());   // one GetObservations() snapshot per point, reused below
    for (size_t p = 0; p < vPoints.size(); ++p) {
        vObs[p] = vPoints[p]->GetObservations();
        if (vFixed.size() >= maxFixKF) continue;   // :2337 leaves the marking loop; the snapshots are still needed for the edges
        for (const auto& ob : vObs[p]) {
            KeyFrame* pKFi = ob.first;
            if (pKFi->mnBALocalForKF != ba_id && pKFi->mnBAFixedForKF != ba_id) {
                pKFi->mnBAFixedForKF = ba_id;
                if (!pKFi->isBad()) {
                    vFixed.push_back(pKFi);
                    break;   // one new fixed keyframe per point
                }
            }
        }
    }

    // ---- vertices: per keyframe Rwb twb v bg ba (ImuCamPose + VertexVelocity / GyroBias / AccBias), optimisable ones first ----
    const int N = (int)vOpt.size(), nKF = N + (int)vFixed.size(), nMP = (int)vPoints.size();
    std::vector<double> state((size_t)nKF * 21, 0.0);
    std::vector<uint8_t> fixed(nKF, 0);
    std::unordered_map<KeyFrame*, int> kfIndex;
    kfIndex.reserve((size_t)nKF * 2);
    const Sophus::SE3f Tcb = pKF->mImuCalib.mTcb;
    auto add_kf = [&](KeyFrame* k, bool isFixed) {
        const int i = (int)kfIndex.size();
        kfIndex[k] = i;
        double* S = &state[(size_t)i * 21];
        const Eigen::Matrix3d Rwb = k->GetImuRotation().cast<double>();
        const Eigen::Vector3d twb = k->GetImuPosition().cast<double>();
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) S[3 * r + c] = Rwb(r, c);
        for (int c = 0; c < 3; ++c) S[9 + c] = twb(c);
        if (k->bImu) {
            const Eigen::Vector3d v = k->GetVelocity().cast<double>(), bg = k->GetGyroBias().cast<double>(), ba = k->GetAccBias().cast<double>();
            for (int c = 0; c < 3; ++c) { S[12 + c] = v(c); S[15 + c] = bg(c); S[18 + c] = ba(c); }
        } else if (!isFixed) {
            throw orb_b200::Error("LocalInertialBA: an optimisable keyframe without IMU (bImu false) is not built on the GPU path");
        }
        const Sophus::SE3f Tk = k->mImuCalib.mTcb;
        for (int r = 0; r < 3; ++r) {
            if (Tk.translation()(r) != Tcb.translation()(r)) throw orb_b200::Error("LocalInertialBA: keyframes of one window with different IMU calibrations");
            for (int c = 0; c < 3; ++c)
                if (Tk.rotationMatrix()(r, c) != Tcb.rotationMatrix()(r, c)) throw orb_b200::Error("LocalInertialBA: keyframes of one window with different IMU calibrations");
        }
        fixed[i] = isFixed ? 1 : 0;
    };
    for (KeyFrame* k : vOpt) add_kf(k, false);
    for (KeyFrame* k : vFixed) add_kf(k, true);

    // ---- inertial links: EdgeInertial + EdgeGyroRW + EdgeAccRW between each optimisable keyframe and its predecessor ----
    std::vector<liba_link> links;
    links.reserve(N);
    for (int i = 0; i < N; ++i) {
        KeyFrame* k = vOpt[i];
        if (!k->mPrevKF) continue;                                                   // "NOT INERTIAL LINK TO PREVIOUS FRAME"
        if (!(k->bImu && k->mPrevKF->bImu && k->mpImuPreintegrated)) continue;       // "ERROR building inertial edge"
        IMU::Preintegrated* pre = k->mpImuPreintegrated;
        pre->SetNewBias(k->mPrevKF->GetImuBias());
        const auto it = kfIndex.find(k->mPrevKF);
        if (it == kfIndex.end()) continue;                                            // a vertex is missing: the reference prints and skips
        liba_link L;
        L.k1 = it->second; L.k2 = i; L.robust = (i == N - 1 || bRecInit) ? 1 : 0; L.pad = 0;
        L.dt = pre->dT;
        put3x3(L.dR, pre->dR); put3x3(L.JRg, pre->JRg); put3x3(L.JVg, pre->JVg); put3x3(L.JVa, pre->JVa); put3x3(L.JPg, pre->JPg); put3x3(L.JPa, pre->JPa);
        for (int c = 0; c < 3; ++c) { L.dV[c] = pre->dV(c); L.dP[c] = pre->dP(c); }
        L.bias[0] = pre->b.bax; L.bias[1] = pre->b.bay; L.bias[2] = pre->b.baz; L.bias[3] = pre->b.bwx; L.bias[4] = pre->b.bwy; L.bias[5] = pre->b.bwz;
        float C[225];
        for (int r = 0; r < 15; ++r) for (int c = 0; c < 15; ++c) C[15 * r + c] = pre->C(r, c);
        orb_b200::check(liba_link_information(C, i == N - 1 ? 1 : 0, L.info, L.infoG, L.infoA), "liba_link_information");
        links.push_back(L);
    }

    // ---- reprojection edges, by point then by observer (the observation map's order) ----
    std::vector<int32_t> edge_kf, edge_mp;
    std::vector<double> obs, inv_sigma2, point((size_t)nMP * 3);
    std::vector<KeyFrame*> edgeKF;
    const float fx = pKF->fx, fy = pKF->fy, cx = pKF->cx, cy = pKF->cy, bf = pKF->mbf;
    for (int p = 0; p < nMP; ++p) {
        const Eigen::Vector3d X = vPoints[p]->GetWorldPos().cast<double>();
        point[3 * (size_t)p] = X(0); point[3 * (size_t)p + 1] = X(1); point[3 * (size_t)p + 2] = X(2);
        for (const auto& ob : vObs[p]) {
            KeyFrame* pKFi = ob.first;
            if (pKFi->mnBALocalForKF != ba_id && pKFi->mnBAFixedForKF != ba_id) continue;
            if (pKFi->isBad() || pKFi->GetMap() != pCurrentMap) continue;
            if (pKFi->mpCamera2) throw orb_b200::Error("LocalInertialBA: a keyframe with a second camera (EdgeMono(1)) is not built on the GPU path");
            const int leftIndex = std::get<0>(ob.second);
            if (leftIndex == -1) continue;
            const auto it = kfIndex.find(pKFi);
            if (it == kfIndex.end()) continue;   // marked fixed but bad at marking time and alive now: no vertex, g2o would reject the edge
            if (pKFi->fx != fx || pKFi->fy != fy || pKFi->cx != cx || pKFi->cy != cy || pKFi->mbf != bf)
                throw orb_b200::Error("LocalInertialBA: keyframes of one window with different intrinsics");
            const cv::KeyPoint& kpUn = pKFi->mvKeysUn[leftIndex];
            const float ur = pKFi->mvuRight[leftIndex];
            edge_kf.push_back(it->second);
            edge_mp.push_back(p);
            obs.push_back(kpUn.pt.x); obs.push_back(kpUn.pt.y); obs.push_back(ur < 0 ? -1.0 : (double)ur);   // < 0: EdgeMono, else EdgeStereo
            inv_sigma2.push_back(pKFi->mvInvLevelSigma2[kpUn.octave]);
            edgeKF.push_back(pKFi);
        }
    }
    const int nE = (int)edge_kf.size();

    // ---- optimizer.optimize(opt_it) on the device ----
    std::vector<double> state_out((size_t)nKF * 21), point_out((size_t)(nMP > 0 ? nMP : 1) * 3), chi2(nE > 0 ? nE : 1);
    std::vector<uint8_t> depth_ok(nE > 0 ? nE : 1);
    liba_problem in;
    in.n_kf = nKF; in.n_mp = nMP; in.n_edges = nE; in.n_links = (int)links.size();
    in.state = state.data(); in.fixed = fixed.data(); in.point = point.data(); in.edge_kf = edge_kf.data(); in.edge_mp = edge_mp.data();
    in.obs = obs.data(); in.inv_sigma2 = inv_sigma2.data(); in.links = links.data();
    const Eigen::Matrix3d Rcb = Tcb.rotationMatrix().cast<double>();
    const Eigen::Vector3d tcb = Tcb.translation().cast<double>();
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) in.Tcb[3 * r + c] = Rcb(r, c); in.Tcb[9 + r] = tcb(r); }
    in.fx = fx; in.fy = fy; in.cx = cx; in.cy = cy; in.bf = bf;
    in.lambda_init = bLarge ? 1e-2 : 1e0;   // :2349, :2355
    in.max_iters = opt_it;
    liba_result out;
    out.state = state_out.data(); out.point = point_out.data(); out.edge_chi2 = chi2.data(); out.link_chi2 = nullptr;
    out.edge_depth_positive = depth_ok.data();
    orb_b200::check(liba_solve(liba_handle_of_process(), 1, &in, &out), "liba_solve");
    const float err = (float)out.chi2_initial, err_end = (float)out.chi2_last_trial;   // :2672, :2685 (activeRobustChi2 into float)

    // ---- outliers: monocular edges first, then stereo edges, each in creation order (:2690-2726) ----
    const float chi2Mono2 = 5.991f, chi2Stereo2 = 7.815f;
    std::vector<std::pair<KeyFrame*, MapPoint*>> vToErase;
    vToErase.reserve(nE);
    for (int pass = 0; pass < 2; ++pass)
        for (int e = 0; e < nE; ++e) {
            const bool mono = obs[3 * (size_t)e + 2] < 0;
            if (mono != (pass == 0)) continue;
            MapPoint* pMP = vPoints[edge_mp[e]];
            if (mono) {
                const bool bClose = pMP->mTrackDepth < 10.f;
                if (pMP->isBad()) continue;
                if ((chi2[e] > chi2Mono2 && !bClose) || (chi2[e] > 1.5f * chi2Mono2 && bClose) || !depth_ok[e]) vToErase.push_back(std::make_pair(edgeKF[e], pMP));
            } else {
                if (pMP->isBad()) continue;
                if (chi2[e] > chi2Stereo2) vToErase.push_back(std::make_pair(edgeKF[e], pMP));
            }
        }

    // ---- under the map mutex: failure rule, erasures, write-back (:2729-2811) ----
    std::unique_lock<std::mutex> lock(pMap->mMutexMapUpdate);
    if ((2 * err < err_end || std::isnan(err) || std::isnan(err_end)) && !bLarge) return;   // "FAIL LOCAL-INERTIAL BA!!!!" (the marks stay, as in the reference)
    for (auto& er : vToErase) {
        er.first->EraseMapPointMatch(er.second);
        er.second->EraseObservation(er.first);
    }
    for (KeyFrame* k : vFixed) k->mnBAFixedForKF = 0;
    for (int i = 0; i < N; ++i) {
        KeyFrame* k = vOpt[i];
        const double* S = &state_out[(size_t)i * 21];
        if (std::memcmp(S, &state[(size_t)i * 21], 12 * sizeof(double)) != 0) {
            Eigen::Matrix3d Rbw;    // ImuCamPose::Update (G2oTypes.cc:236-243): Rcw = Rcb Rbw, tcw = Rcb tbw + tcb
            Eigen::Vector3d twb(S[9], S[10], S[11]);
            for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) Rbw(r, c) = S[3 * c + r];
            const Eigen::Vector3d tbw = -(Rbw * twb);
            const Eigen::Matrix3d Rcw = Rcb * Rbw;
            const Eigen::Vector3d tcw = Rcb * tbw + tcb;
            k->SetPose(Sophus::SE3f(Rcw.cast<float>(), tcw.cast<float>()));
        } else {   // no accepted step moved this vertex: it still holds the keyframe's own Tcw (the constructor's copy)
            k->SetPose(Sophus::SE3f(k->GetRotation(), k->GetTranslation()));
        }
        k->mnBALocalForKF = 0;
        if (k->bImu) {
            k->SetVelocity(Eigen::Vector3d(S[12], S[13], S[14]).cast<float>());
            k->SetNewBias(IMU::Bias(S[18], S[19], S[20], S[15], S[16], S[17]));   // (acc, gyro), doubles narrowed by the const float& parameters
        }
    }
    for (int p = 0; p < nMP; ++p) {
        const Eigen::Vector3d X(point_out[3 * (size_t)p], point_out[3 * (size_t)p + 1], point_out[3 * (size_t)p + 2]);
        vPoints[p]->SetWorldPos(X.cast<float>());
        vPoints[p]->UpdateNormalAndDepth();
    }
    pMap->IncreaseChangeIndex();
}

}  // namespace ORB_SLAM3
