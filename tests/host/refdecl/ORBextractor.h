// ORBextractor.h -- stand-in for the reference's include/ORBextractor.h: the ORB_SLAM3::ORBextractor declaration (constructor,
// operator(), getters, the protected members host/ORBextractor_b200.cc fills) as the reference declares it.  Used by
// tests/host/build.sh only when no reference checkout is given, so that tests/host/host_boundary builds from the repository alone;
// with ORB_REFERENCE_ROOT set, the real header is used and tests/test_host_shim.py compares the skeletons with it.
#ifndef ORBEXTRACTOR_H
#define ORBEXTRACTOR_H
#include <list>
#include <vector>
#include <opencv2/opencv.hpp>
namespace ORB_SLAM3 {
class ORBextractor {
   public:
    ORBextractor(int nfeatures, float scaleFactor, int nlevels, int iniThFAST, int minThFAST);
    ~ORBextractor() {}
    int operator()(cv::InputArray _image, cv::InputArray _mask, std::vector<cv::KeyPoint>& _keypoints, cv::OutputArray _descriptors,
                   std::vector<int>& vLappingArea);
    int inline GetLevels() { return nlevels; }
    float inline GetScaleFactor() { return scaleFactor; }
    std::vector<float> inline GetScaleFactors() { return mvScaleFactor; }
    std::vector<float> inline GetInverseScaleFactors() { return mvInvScaleFactor; }
    std::vector<float> inline GetScaleSigmaSquares() { return mvLevelSigma2; }
    std::vector<float> inline GetInverseScaleSigmaSquares() { return mvInvLevelSigma2; }
    std::vector<cv::Mat> mvImagePyramid;
   protected:
    std::vector<cv::Point> pattern;
    int nfeatures;
    double scaleFactor;
    int nlevels;
    int iniThFAST;
    int minThFAST;
    std::vector<int> mnFeaturesPerLevel;
    std::vector<int> umax;
    std::vector<float> mvScaleFactor;
    std::vector<float> mvInvScaleFactor;
    std::vector<float> mvLevelSigma2;
    std::vector<float> mvInvLevelSigma2;
};
}  // namespace ORB_SLAM3
#endif
