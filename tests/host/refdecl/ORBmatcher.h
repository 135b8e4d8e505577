// ORBmatcher.h -- stand-in for the reference's include/ORBmatcher.h: the members of ORB_SLAM3::ORBmatcher that the host units
// (host/ORBmatcher_b200.cc, ORBmatcher_bow_b200.cc, ORBmatcher_init_b200.cc, ORBmatcher_triangulation_b200.cc, ORBmatcher_fuse_b200.cc,
// ORBmatcher_reloc_b200.cc, ORBmatcher_sim3_b200.cc) define, with the reference's signatures and default arguments.  Used by
// tests/host/build.sh and build_units.sh only when no reference checkout is given (see ORBextractor.h here).
#ifndef ORBMATCHER_H
#define ORBMATCHER_H
#include <set>
#include <utility>
#include <vector>
namespace ORB_SLAM3 {
class ORBmatcher {
   public:
    ORBmatcher(float nnratio = 0.6, bool checkOri = true);
    static int DescriptorDistance(const cv::Mat& a, const cv::Mat& b);
    int SearchByProjection(Frame& F, const std::vector<MapPoint*>& vpMapPoints, const float th = 3, const bool bFarPoints = false,
                           const float thFarPoints = 50.0f);
    int SearchByProjection(Frame& CurrentFrame, const Frame& LastFrame, const float th, const bool bMono);
    int SearchByProjection(Frame& CurrentFrame, KeyFrame* pKF, const std::set<MapPoint*>& sAlreadyFound, const float th, const int ORBdist);
    int SearchByProjection(KeyFrame* pKF, Sophus::Sim3<float>& Scw, const std::vector<MapPoint*>& vpPoints, std::vector<MapPoint*>& vpMatched, int th,
                           float ratioHamming = 1.0);
    int SearchByProjection(KeyFrame* pKF, Sophus::Sim3<float>& Scw, const std::vector<MapPoint*>& vpPoints, const std::vector<KeyFrame*>& vpPointsKFs,
                           std::vector<MapPoint*>& vpMatched, std::vector<KeyFrame*>& vpMatchedKF, int th, float ratioHamming = 1.0);
    int SearchByBoW(KeyFrame* pKF, Frame& F, std::vector<MapPoint*>& vpMapPointMatches);
    int SearchByBoW(KeyFrame* pKF1, KeyFrame* pKF2, std::vector<MapPoint*>& vpMatches12);
    int SearchForInitialization(Frame& F1, Frame& F2, std::vector<cv::Point2f>& vbPrevMatched, std::vector<int>& vnMatches12, int windowSize = 10);
    int SearchForTriangulation(KeyFrame* pKF1, KeyFrame* pKF2, std::vector<std::pair<size_t, size_t> >& vMatchedPairs, const bool bOnlyStereo,
                               const bool bCoarse = false);
    int Fuse(KeyFrame* pKF, const std::vector<MapPoint*>& vpMapPoints, const float th = 3.0, const bool bRight = false);
    int Fuse(KeyFrame* pKF, Sophus::Sim3f& Scw, const std::vector<MapPoint*>& vpPoints, float th, std::vector<MapPoint*>& vpReplacePoint);
   public:
    static const int TH_LOW;
    static const int TH_HIGH;
    static const int HISTO_LENGTH;
   protected:
    float RadiusByViewingCos(const float& viewCos);
    void ComputeThreeMaxima(std::vector<int>* histo, const int L, int& ind1, int& ind2, int& ind3);
    float mfNNratio;
    bool mbCheckOrientation;
};
}  // namespace ORB_SLAM3
#endif
