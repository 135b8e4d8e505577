// Optimizer.h -- stand-in for the reference's include/Optimizer.h: the members of ORB_SLAM3::Optimizer that the host units
// host/Optimizer_lba_b200.cc, Optimizer_pose_b200.cc and Optimizer_liba_b200.cc define, as the reference declares them.  Used by
// tests/host/build.sh and build_units.sh only when no reference checkout is given (see ORBextractor.h here).
#ifndef OPTIMIZER_H
#define OPTIMIZER_H
namespace ORB_SLAM3 {
class Optimizer {
   public:
    void static LocalBundleAdjustment(KeyFrame* pKF, bool* pbStopFlag, Map* pMap, int& num_fixedKF, int& num_OptKF, int& num_MPs,
                                      int& num_edges);
    int static PoseOptimization(Frame* pFrame);
    void static LocalInertialBA(KeyFrame* pKF, bool* pbStopFlag, Map* pMap, int& num_fixedKF, int& num_OptKF, int& num_MPs, int& num_edges,
                                bool bLarge = false, bool bRecInit = false);
};
}  // namespace ORB_SLAM3
#endif
