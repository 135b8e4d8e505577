// orb_b200_host.h -- shared by the host translation units that stand in for the reference's src/ORBextractor.cc and for the
// hot members of src/ORBmatcher.cc, src/Frame.cc, src/Optimizer.cc.  They only marshal: all arithmetic runs on the GPU behind
// the C ABI (include/orbslam3_b200.h).  There is no CPU fallback: a failed call throws orb_b200::Error (the reference has no error
// channel at these call sites; an uncaught exception terminates like its asserts do, a caught one lets the application decide).
#pragma once
#include <cstdlib>
#include <stdexcept>
#include <string>

#include "orbslam3_b200.h"

namespace orb_b200 {

struct Error : std::runtime_error {
    explicit Error(const std::string& what) : std::runtime_error(what) {}
};

inline void check(orb_status s, const char* what) {
    if (s != ORB_OK) throw Error(std::string("ORB-SLAM3 GPU path: ") + what + ": " + orb_last_error());
}

// the CUDA device every workspace of the host units is created on: $ORB_B200_DEVICE, else 0
inline int device_ordinal() {
    const char* d = std::getenv("ORB_B200_DEVICE");
    return d ? std::atoi(d) : 0;
}

}  // namespace orb_b200

// The device handle behind a reference ORBextractor object (host/ORBextractor_b200.cc keeps the table: the reference class has
// no spare member).  NULL when the object was not created by our constructor.
extern "C" orbx_handle* orb_b200_handle_of(const void* orb_extractor);
// Releases one extractor's device workspace early (all are released at process exit).
extern "C" void orb_b200_release(const void* orb_extractor);
// One LocalBundleAdjustment solver workspace per process (created on first use, released at exit).
extern "C" lba_handle* orb_b200_lba_handle(void);
// The workspace the keyframe-to-keyframe searches run on (host/ORBmatcher_bow_b200.cc keeps it): they see no Frame, hence no extractor to
// take one from.  Any live extractor handle of the process serves; SearchByBoW(KeyFrame*, Frame&) sets its frame's when none is set.
extern "C" void orb_b200_use_handle_for_keyframe_searches(orbx_handle* h);
extern "C" orbx_handle* orb_b200_keyframe_search_handle(void);
