// Optimizer_lba_b200.cc -- Optimizer::LocalBundleAdjustment (/root/reference/src/Optimizer.cc:1740-2188) on the GPU.
//
// Compiled against the reference's UNMODIFIED include/Optimizer.h (signature :59).  What stays on the host is what touches the
// map's objects: choosing the local window (:1744-1855), flattening it into the SoA problem the solver takes (:1873-2091),
// sorting out the outliers (:2107-2150) and writing the result back under the map mutex (:2153-2187).  Everything g2o did
// in between -- linearisation of the mono / stereo reprojection edges with Huber kernels, the Schur-reduced normal equations, the
// dense LDL^T, the Levenberg loop with its accept / reject rule -- is ONE kernel launch (k_lba, csrc/lba.cu) behind lba_solve_bool.
// Link before the reference's Optimizer.o with -Wl,--allow-multiple-definition, or exclude that one body from Optimizer.cc.
// Not built: right-camera observations of fisheye rigs (EdgeSE3ProjectXYZToBody, :2049-2086) -- such a window is refused.
#include <cmath>
#include <list>
#include <map>
#include <unordered_map>
#include <vector>

#include "Optimizer.h"        // the reference's header
#include "orb_b200_host.h"

namespace ORB_SLAM3 {

void Optimizer::LocalBundleAdjustment(KeyFrame* pKF, bool* pbStopFlag, Map* pMap, int& num_fixedKF, int& num_OptKF, int& num_MPs,
                                      int& num_edges) {
    (void)num_MPs;   // the reference never assigns it in this overload either
    // ---- local window: the keyframe, its covisible neighbours, every point they see, every other observer as a fixed camera ----
    std::vector<KeyFrame*> vLocal;
    vLocal.push_back(pKF);
    pKF->mnBALocalForKF = pKF->mnId;
    Map* pCurrentMap = pKF->GetMap();
    const std::vector<KeyFrame*> vNeigh = pKF->GetVectorCovisibleKeyFrames();
    for (KeyFrame* pKFi : vNeigh) {
        pKFi->mnBALocalForKF = pKF->mnId;
        if (!pKFi->isBad() && pKFi->GetMap() == pCurrentMap) vLocal.push_back(pKFi);
    }
    num_fixedKF = 0;
    std::vector<MapPoint*> vPoints;
    for (KeyFrame* pKFi : vLocal) {
        if (pKFi->mnId == pMap->GetInitKFid()) num_fixedKF = 1;
        const std::vector<MapPoint*> vpMPs = pKFi->GetMapPointMatches();
        for (MapPoint* pMP : vpMPs)
            if (pMP && !pMP->isBad() && pMP->GetMap() == pCurrentMap && pMP->mnBALocalForKF != pKF->mnId) {
                vPoints.push_back(pMP);
                pMP->mnBALocalForKF = pKF->mnId;
            }
    }
    std::vector<KeyFrame*> vFixed;
    std::vector<std::map<KeyFrame*, std::tuple<int, int>>> vObs(vPoints.size());   // one GetObservations() snapshot per point, reused below
    for (size_t p = 0; p < vPoints.size(); ++p) {
        vObs[p] = vPoints[p]->GetObservations();
        for (const auto& ob : vObs[p]) {
            KeyFrame* pKFi = ob.first;
            if (pKFi->mnBALocalForKF != pKF->mnId && pKFi->mnBAFixedForKF != pKF->mnId) {
                pKFi->mnBAFixedForKF = pKF->mnId;
                if (!pKFi->isBad() && pKFi->GetMap() == pCurrentMap) vFixed.push_back(pKFi);
            }
        }
    }
    num_fixedKF = (int)vFixed.size() + num_fixedKF;
    if (num_fixedKF == 0) return;   // :1851 "LBA aborted"

    // ---- flatten: poses (quaternion + translation, float -> double as g2o::SE3Quat takes them), points, edges by point ----
    pCurrentMap->msOptKFs.clear();
    pCurrentMap->msFixedKFs.clear();
    const int nKF = (int)(vLocal.size() + vFixed.size()), nMP = (int)vPoints.size();
    std::vector<double> pose((size_t)nKF * 7), point((size_t)nMP * 3);
    std::vector<uint8_t> fixed(nKF);
    std::unordered_map<KeyFrame*, int> kfIndex;
    kfIndex.reserve(nKF * 2);
    auto add_kf = [&](KeyFrame* k, bool isFixed) {
        const int i = (int)kfIndex.size();
        kfIndex[k] = i;
        const Sophus::SE3f Tcw = k->GetPose();
        const Eigen::Quaterniond q = Tcw.unit_quaternion().cast<double>();
        const Eigen::Vector3d t = Tcw.translation().cast<double>();
        double* P = &pose[(size_t)i * 7];
        P[0] = q.x(); P[1] = q.y(); P[2] = q.z(); P[3] = q.w(); P[4] = t(0); P[5] = t(1); P[6] = t(2);
        fixed[i] = isFixed ? 1 : 0;
    };
    for (KeyFrame* k : vLocal) {
        add_kf(k, k->mnId == pMap->GetInitKFid());
        pCurrentMap->msOptKFs.insert(k->mnId);
    }
    num_OptKF = (int)vLocal.size();
    for (KeyFrame* k : vFixed) {
        add_kf(k, true);
        pCurrentMap->msFixedKFs.insert(k->mnId);
    }
    std::vector<int32_t> edge_kf, edge_mp;
    std::vector<double> obs, inv_sigma2;
    std::vector<KeyFrame*> edgeKF;      // vpEdgeKFMono / vpEdgeKFStereo, in creation order
    const float fx = pKF->fx, fy = pKF->fy, cx = pKF->cx, cy = pKF->cy, bf = pKF->mbf;
    for (int p = 0; p < nMP; ++p) {
        const Eigen::Vector3d X = vPoints[p]->GetWorldPos().cast<double>();
        point[3 * (size_t)p] = X(0); point[3 * (size_t)p + 1] = X(1); point[3 * (size_t)p + 2] = X(2);
        for (const auto& ob : vObs[p]) {
            KeyFrame* pKFi = ob.first;
            if (pKFi->isBad() || pKFi->GetMap() != pCurrentMap) continue;
            if (pKFi->mpCamera2) throw orb_b200::Error("LocalBundleAdjustment: a keyframe with a second camera (EdgeSE3ProjectXYZToBody) is not built on the GPU path");
            const int leftIndex = std::get<0>(ob.second);
            if (leftIndex == -1) continue;
            const auto it = kfIndex.find(pKFi);
            if (it == kfIndex.end()) continue;   // cannot happen: every live observer is local or fixed
            if (pKFi->fx != fx || pKFi->fy != fy || pKFi->cx != cx || pKFi->cy != cy || pKFi->mbf != bf)
                throw orb_b200::Error("LocalBundleAdjustment: keyframes of one window with different intrinsics");
            const cv::KeyPoint& kpUn = pKFi->mvKeysUn[leftIndex];
            const float ur = pKFi->mvuRight[leftIndex];
            edge_kf.push_back(it->second);
            edge_mp.push_back(p);
            obs.push_back(kpUn.pt.x); obs.push_back(kpUn.pt.y); obs.push_back(ur < 0 ? -1.0 : (double)ur);   // < 0: EdgeSE3ProjectXYZ, else EdgeStereoSE3ProjectXYZ
            inv_sigma2.push_back(pKFi->mvInvLevelSigma2[kpUn.octave]);
            edgeKF.push_back(pKFi);
        }
    }
    const int nE = (int)edge_kf.size();
    num_edges = nE;
    if (pbStopFlag && *pbStopFlag) return;   // :2093-2095

    // ---- optimizer.optimize(10) on the device ----
    std::vector<double> pose_out((size_t)nKF * 7), point_out((size_t)nMP * 3), chi2(nE > 0 ? nE : 1);
    std::vector<uint8_t> depth_ok(nE > 0 ? nE : 1);
    lba_problem in;
    in.n_kf = nKF; in.n_mp = nMP; in.n_edges = nE;
    in.pose = pose.data(); in.fixed = fixed.data(); in.point = point.data(); in.edge_kf = edge_kf.data(); in.edge_mp = edge_mp.data();
    in.obs = obs.data(); in.inv_sigma2 = inv_sigma2.data();
    in.fx = fx; in.fy = fy; in.cx = cx; in.cy = cy; in.bf = bf;
    in.lambda_init = pMap->IsInertial() ? 100.0 : 0.0;   // :1867-1868
    in.max_iters = 10;
    lba_result out;
    out.pose = pose_out.data(); out.point = point_out.data(); out.edge_chi2 = chi2.data(); out.edge_depth_positive = depth_ok.data();
    static_assert(sizeof(bool) == 1, "bool* pbStopFlag is relayed as one byte");
    orb_b200::check(lba_solve_bool(orb_b200_lba_handle(), &in, &out, reinterpret_cast<const volatile uint8_t*>(pbStopFlag)), "lba_solve_bool");

    // ---- outliers: monocular edges first, then stereo edges, each in creation order (:2107-2150) ----
    std::vector<std::pair<KeyFrame*, MapPoint*>> vToErase;
    vToErase.reserve(nE);
    for (int pass = 0; pass < 2; ++pass)
        for (int e = 0; e < nE; ++e) {
            const bool mono = obs[3 * (size_t)e + 2] < 0;
            if (mono != (pass == 0)) continue;
            MapPoint* pMP = vPoints[edge_mp[e]];
            if (pMP->isBad()) continue;
            if (chi2[e] > (mono ? 5.991 : 7.815) || !depth_ok[e]) vToErase.push_back(std::make_pair(edgeKF[e], pMP));
        }

    // ---- write-back under the map mutex (:2153-2187) ----
    std::unique_lock<std::mutex> lock(pMap->mMutexMapUpdate);
    for (auto& er : vToErase) {
        er.first->EraseMapPointMatch(er.second);
        er.second->EraseObservation(er.first);
    }
    for (size_t i = 0; i < vLocal.size(); ++i) {
        const double* P = &pose_out[i * 7];
        const Eigen::Quaterniond q(P[3], P[0], P[1], P[2]);
        const Eigen::Vector3d t(P[4], P[5], P[6]);
        vLocal[i]->SetPose(Sophus::SE3f(q.cast<float>(), t.cast<float>()));
    }
    for (int p = 0; p < nMP; ++p) {
        const Eigen::Vector3d X(point_out[3 * (size_t)p], point_out[3 * (size_t)p + 1], point_out[3 * (size_t)p + 2]);
        vPoints[p]->SetWorldPos(X.cast<float>());
        vPoints[p]->UpdateNormalAndDepth();
    }
    pMap->IncreaseChangeIndex();
}

}  // namespace ORB_SLAM3
