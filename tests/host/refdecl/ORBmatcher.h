// ORBmatcher.h -- stand-in for the reference's include/ORBmatcher.h: the members of ORB_SLAM3::ORBmatcher that the per-frame unit
// host/ORBmatcher_b200.cc defines, with the reference's signatures and default arguments.  Used by tests/host/build.sh only when no
// reference checkout is given (see ORBextractor.h here).
#ifndef ORBMATCHER_H
#define ORBMATCHER_H
#include <vector>
namespace ORB_SLAM3 {
class ORBmatcher {
   public:
    ORBmatcher(float nnratio = 0.6, bool checkOri = true);
    static int DescriptorDistance(const cv::Mat& a, const cv::Mat& b);
    int SearchByProjection(Frame& F, const std::vector<MapPoint*>& vpMapPoints, const float th = 3, const bool bFarPoints = false,
                           const float thFarPoints = 50.0f);
    int SearchByProjection(Frame& CurrentFrame, const Frame& LastFrame, const float th, const bool bMono);
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
