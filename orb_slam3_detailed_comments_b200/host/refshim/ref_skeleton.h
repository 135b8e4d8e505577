// refshim/ref_skeleton.h -- SKELETONS of the reference's Frame / KeyFrame / MapPoint / Map classes for the compile check and the
// marshaling tests of the host translation units (host/ORBmatcher_b200.cc, Frame_stereo_b200.cc, Optimizer_lba_b200.cc).
//
// The reference's own include/Frame.h, KeyFrame.h, MapPoint.h, Map.h pull in the whole system (Sophus, g2o, DBoW2, boost
// serialization, Pangolin through Tracking.h); none of that exists in this image.  This header is pre-included (g++ -include) and
// defines those headers' include guards, so that the reference's UNMODIFIED include/ORBmatcher.h and include/Optimizer.h -- the
// class declarations our translation units implement -- are parsed against these skeletons instead.
//
// Every member between "//@ref <header>" and "//@end" is declared EXACTLY as in that reference header; tests/test_host_shim.py
// checks each such line against the header's text.  Only members our translation units touch are listed.  Bodies (a mock map for
// tests/host/) are in ref_skeleton_impl.h.  A real integration does not use this file: it compiles the same translation units
// against the real headers.
#pragma once
#define FRAME_H
#define KEYFRAME_H
#define MAPPOINT_H
#define MAP_H
#define LOOPCLOSING_H

#include <list>
#include <map>
#include <mutex>
#include <set>
#include <tuple>
#include <vector>

#include "Eigen/Core"
#include "opencv2/opencv.hpp"
#include "sophus/se3.hpp"
#include "sophus/sim3.hpp"
#include "ORBextractor.h"   // the reference's own header (it needs nothing but <opencv2/opencv.hpp>)

namespace g2o { class Sim3; }
#ifdef ORB_REFSHIM_FUSE  // host/ORBmatcher_fuse_b200.cc
#define ORB_REFSHIM_TRI
#endif
#ifdef ORB_REFSHIM_VOC   // host/Frame_bow_b200.cc: what Thirdparty/DBoW2/DBoW2/{BowVector.h, FeatureVector.h, TemplatedVocabulary.h} declare, as far as
#define ORB_REFSHIM_BOW   // Frame::ComputeBoW and the flattening of the vocabulary touch it (the nodes are PROTECTED members there too)
namespace DBoW2 {
typedef unsigned int WordId;
typedef double WordValue;
class BowVector : public std::map<WordId, WordValue> {};
}
#endif
#ifdef ORB_REFSHIM_BOW   // host/ORBmatcher_bow_b200.cc: Thirdparty/DBoW2/DBoW2/FeatureVector.h:23-27 is `class FeatureVector: public std::map<NodeId, std::vector<unsigned int> >`
namespace DBoW2 {
typedef unsigned int NodeId;
class FeatureVector : public std::map<NodeId, std::vector<unsigned int> > {
   public:
    void addFeature(NodeId id, unsigned int i_feature) { (*this)[id].push_back(i_feature); }   // FeatureVector.cpp:27-41
};
}
#endif
#ifdef ORB_REFSHIM_VOC
namespace DBoW2 {
template <class TDescriptor, class F>
class TemplatedVocabulary {   // TemplatedVocabulary.h:297-329 (Node), :408-427 (the protected members)
   public:
    struct Node {
        NodeId id;
        WordValue weight;
        std::vector<NodeId> children;
        NodeId parent;
        TDescriptor descriptor;
        WordId word_id;
        Node() : id(0), weight(0), parent(0), word_id(0) {}
        inline bool isLeaf() const { return children.empty(); }
    };
    void mock_set(int L, const std::vector<Node>& nodes) { m_L = L; m_nodes = nodes; }
   protected:
    int m_k = 0;
    int m_L = 0;
    std::vector<Node> m_nodes;
};
struct FORB { typedef cv::Mat TDescriptor; };
}
namespace ORB_SLAM3 { typedef DBoW2::TemplatedVocabulary<DBoW2::FORB::TDescriptor, DBoW2::FORB> ORBVocabulary; }   // include/ORBVocabulary.h:30-31
#endif

using namespace std;   // the reference headers rely on it (ORBmatcher.h:64 `vector<pair<size_t, size_t> >`, Optimizer.h:64 `map<...>`)

namespace ORB_SLAM3 {

class KeyFrame;
class MapPoint;
class Map;
class Frame;
class GeometricCamera;

#ifdef ORB_REFSHIM_LIBA   // host/Optimizer_liba_b200.cc (LocalInertialBA) and the reference's own function next to it (tests/host/build_liba_cpu.sh)
namespace IMU {
class Bias {
   public:
//@ref ImuTypes.h
    Bias():bax(0),bay(0),baz(0),bwx(0),bwy(0),bwz(0){}
    Bias(const float &b_acc_x, const float &b_acc_y, const float &b_acc_z,
            const float &b_ang_vel_x, const float &b_ang_vel_y, const float &b_ang_vel_z):
            bax(b_acc_x), bay(b_acc_y), baz(b_acc_z), bwx(b_ang_vel_x), bwy(b_ang_vel_y), bwz(b_ang_vel_z){}
    float bax, bay, baz;
    float bwx, bwy, bwz;
//@end
};
class Calib {
   public:
//@ref ImuTypes.h
    Sophus::SE3<float> mTcb;
    Sophus::SE3<float> mTbc;
//@end
};
class Preintegrated {
   public:
//@ref ImuTypes.h
    void SetNewBias(const Bias &bu_);
    float dT;
    Eigen::Matrix<float,15,15> C;
    Bias b;
    Eigen::Matrix3f dR;
    Eigen::Vector3f dV, dP;
    Eigen::Matrix3f JRg, JVg, JVa, JPg, JPa;
//@end
    // mock state (tests/host only)
    Bias mock_bu;
    int mock_bias_sets = 0;
};
}  // namespace IMU
#endif

class LoopClosing {
   public:
    typedef std::map<KeyFrame*, g2o::Sim3*> KeyFrameAndPose;   // placeholder: Optimizer.h names the type in signatures we do not implement
};

class Map {
   public:
//@ref Map.h
    long unsigned int GetInitKFid();
    void IncreaseChangeIndex();
    bool IsInertial();
    std::mutex mMutexMapUpdate;
    std::set<long unsigned int> msOptKFs;
    std::set<long unsigned int> msFixedKFs;
//@end
#ifdef ORB_REFSHIM_LIBA
//@ref Map.h
    long unsigned  KeyFramesInMap();
//@end
    long unsigned mock_n_keyframes = 0;
#endif
    // mock state (tests/host only)
    long unsigned int mock_init_kf_id = 0;
    bool mock_inertial = false;
    int mock_change_index = 0;
};

class MapPoint {
   public:
//@ref MapPoint.h
    void SetWorldPos(const Eigen::Vector3f &Pos);
    Eigen::Vector3f GetWorldPos();
    Eigen::Vector3f GetNormal();
    std::map<KeyFrame*,std::tuple<int,int>> GetObservations();
    int Observations();
    void EraseObservation(KeyFrame* pKF, bool erase = true);
    bool isBad();
    cv::Mat GetDescriptor();
    void UpdateNormalAndDepth();
    Map* GetMap();
    long unsigned int mnId;
    float mTrackProjX;
    float mTrackProjY;
    float mTrackDepth;
    float mTrackProjXR;
    bool mbTrackInView, mbTrackInViewR;
    int mnTrackScaleLevel, mnTrackScaleLevelR;
    float mTrackViewCos, mTrackViewCosR;
    long unsigned int mnBALocalForKF;
//@end
#ifdef ORB_REFSHIM_POSE   // host/Optimizer_pose_b200.cc (PoseOptimization)
//@ref MapPoint.h
    static std::mutex mGlobalMutex;
//@end
#endif
#ifdef ORB_REFSHIM_FUSE
//@ref MapPoint.h
    void AddObservation(KeyFrame* pKF,int idx);
    bool IsInKeyFrame(KeyFrame* pKF);
    void Replace(MapPoint* pMP);
//@end
    void mock_set_distances(float mn, float mx) { mfMinDistance = mn; mfMaxDistance = mx; }
    int mock_id = -1;
   protected:
//@ref MapPoint.h
     float mfMinDistance;
     float mfMaxDistance;
//@end
   public:
#endif
    // mock state (tests/host only)
    Eigen::Vector3f mock_pos, mock_normal;
    std::map<KeyFrame*, std::tuple<int, int>> mock_obs;
    cv::Mat mock_desc;
    Map* mock_map = nullptr;
    bool mock_bad = false;
    int mock_normal_updates = 0;
    MapPoint() : mnId(0), mTrackProjX(0), mTrackProjY(0), mTrackDepth(0), mTrackProjXR(0), mbTrackInView(false), mbTrackInViewR(false),
                 mnTrackScaleLevel(0), mnTrackScaleLevelR(0), mTrackViewCos(0), mTrackViewCosR(0), mnBALocalForKF(0) {}
};

class KeyFrame {
   public:
//@ref KeyFrame.h
    void SetPose(const Sophus::SE3f &Tcw);
    Sophus::SE3f GetPose();
    std::vector<KeyFrame* > GetVectorCovisibleKeyFrames();
    void EraseMapPointMatch(MapPoint* pMP);
    std::vector<MapPoint*> GetMapPointMatches();
    bool isBad();
    Map* GetMap();
    long unsigned int mnId;
    long unsigned int mnBALocalForKF;
    long unsigned int mnBAFixedForKF;
    const float fx, fy, cx, cy, invfx, invfy, mbf, mb, mThDepth;
    const std::vector<cv::KeyPoint> mvKeys;
    const std::vector<cv::KeyPoint> mvKeysUn;
    const std::vector<float> mvuRight; // negative value for monocular points
    const cv::Mat mDescriptors;
    const std::vector<float> mvInvLevelSigma2;
    GeometricCamera* mpCamera, *mpCamera2;
    const int NLeft, NRight;
//@end
#ifdef ORB_REFSHIM_REF_LBA   // only when the REFERENCE's own LocalBundleAdjustment is compiled over this skeleton (tests/host/build_lba_cpu.sh)
//@ref KeyFrame.h
    Sophus::SE3f GetRelativePoseTrl();
    const std::vector<cv::KeyPoint> mvKeysRight;
//@end
#endif
#ifdef ORB_REFSHIM_BOW
//@ref KeyFrame.h
    DBoW2::FeatureVector mFeatVec;
//@end
#endif
#ifdef ORB_REFSHIM_TRI   // host/ORBmatcher_triangulation_b200.cc
//@ref KeyFrame.h
    Sophus::SE3f GetPoseInverse();
    Eigen::Vector3f GetCameraCenter();
//@end
#endif
#ifdef ORB_REFSHIM_FUSE
//@ref KeyFrame.h
    void AddMapPoint(MapPoint* pMP, const size_t &idx);
    MapPoint* GetMapPoint(const size_t &idx);
    std::set<MapPoint*> GetMapPoints();
    const int mnMinX;
    const int mnMinY;
    const int mnMaxX;
    const int mnMaxY;
//@end
#endif
#ifdef ORB_REFSHIM_LIBA
//@ref KeyFrame.h
    void SetVelocity(const Eigen::Vector3f &Vw_);
    Eigen::Vector3f GetImuPosition();
    Eigen::Matrix3f GetImuRotation();
    Eigen::Matrix3f GetRotation();
    Eigen::Vector3f GetTranslation();
    Eigen::Vector3f GetVelocity();
    void SetNewBias(const IMU::Bias &b);
    Eigen::Vector3f GetGyroBias();
    Eigen::Vector3f GetAccBias();
    IMU::Bias GetImuBias();
    bool bImu;
    KeyFrame* mPrevKF;
    IMU::Preintegrated* mpImuPreintegrated;
    IMU::Calib mImuCalib;
//@end
    // mock state (tests/host only): the body pose is kept next to the camera pose, as the reference keyframe does (SetPose updates both)
    Eigen::Vector3f mock_vel;
    IMU::Bias mock_bias;
    int mock_vel_sets = 0, mock_bias_sets = 0;
#endif
    // mock state (tests/host only)
    Sophus::SE3f mock_Tcw;
    std::vector<KeyFrame*> mock_covisible;
    std::vector<MapPoint*> mock_matches;
    Map* mock_map = nullptr;
    bool mock_bad = false;
    int mock_pose_sets = 0;
    KeyFrame(long unsigned int id, float fx_, float fy_, float cx_, float cy_, float bf_, float b_, const std::vector<cv::KeyPoint>& keysUn,
             const std::vector<float>& uRight, const std::vector<float>& invSigma2)
        : mnId(id), mnBALocalForKF(0), mnBAFixedForKF(0), fx(fx_), fy(fy_), cx(cx_), cy(cy_), invfx(1.f / fx_), invfy(1.f / fy_), mbf(bf_),
          mb(b_), mThDepth(0), mvKeys(keysUn), mvKeysUn(keysUn), mvuRight(uRight), mDescriptors(), mvInvLevelSigma2(invSigma2),
          mpCamera(nullptr), mpCamera2(nullptr), NLeft(-1), NRight(-1)
#ifdef ORB_REFSHIM_REF_LBA
          , mvKeysRight()
#endif
#ifdef ORB_REFSHIM_FUSE
          , mnMinX(0), mnMinY(0), mnMaxX(0), mnMaxY(0)
#endif
#ifdef ORB_REFSHIM_LIBA
          , bImu(false), mPrevKF(nullptr), mpImuPreintegrated(nullptr)
#endif
    {}
};

class Frame {
   public:
//@ref Frame.h
    void ComputeStereoMatches();
    void ComputeStereoFromRGBD(const cv::Mat &imDepth);
    inline Sophus::SE3<float> GetPose() const {
        return mTcw;
    }
    ORBextractor* mpORBextractorLeft, *mpORBextractorRight;
    static float fx;
    static float fy;
    static float cx;
    static float cy;
    float mbf;
    float mb;
    int N;
    std::vector<cv::KeyPoint> mvKeys, mvKeysRight;
    std::vector<cv::KeyPoint> mvKeysUn;
    std::vector<MapPoint*> mvpMapPoints;
    std::vector<float> mvuRight;
    std::vector<float> mvDepth;
    cv::Mat mDescriptors, mDescriptorsRight;
    std::vector<bool> mvbOutlier;
    static float mnMinX;
    static float mnMaxX;
    static float mnMinY;
    static float mnMaxY;
    GeometricCamera* mpCamera, *mpCamera2;
    int Nleft, Nright;
    Sophus::SE3<float> mTcw;
//@end
#ifdef ORB_REFSHIM_BOW
//@ref Frame.h
    DBoW2::FeatureVector mFeatVec;
//@end
#endif
#ifdef ORB_REFSHIM_VOC
//@ref Frame.h
    void ComputeBoW();
    ORBVocabulary* mpORBvocabulary;
    DBoW2::BowVector mBowVec;
//@end
#endif
#ifdef ORB_REFSHIM_POSE
//@ref Frame.h
    void SetPose(const Sophus::SE3<float> &Tcw);
    vector<float> mvInvLevelSigma2;
//@end
    int mock_pose_sets = 0;
#endif
    Frame() : mpORBextractorLeft(nullptr), mpORBextractorRight(nullptr), mbf(0), mb(0), N(0), mpCamera(nullptr), mpCamera2(nullptr), Nleft(-1), Nright(-1) {}
};

}  // namespace ORB_SLAM3
