// Optimizer.h -- stand-in for the reference's include/Optimizer.h: Optimizer::LocalBundleAdjustment as the reference declares it,
// the member host/Optimizer_lba_b200.cc defines.  Used by tests/host/build.sh only when no reference checkout is given (see
// ORBextractor.h here).
#ifndef OPTIMIZER_H
#define OPTIMIZER_H
namespace ORB_SLAM3 {
class Optimizer {
   public:
    void static LocalBundleAdjustment(KeyFrame* pKF, bool* pbStopFlag, Map* pMap, int& num_fixedKF, int& num_OptKF, int& num_MPs,
                                      int& num_edges);
};
}  // namespace ORB_SLAM3
#endif
