#!/bin/bash
# Builds tests/host/rgbd_member: Frame::ComputeStereoFromRGBD (host/Frame_stereo_b200.cc) with the extractor and matcher units it works
# with, linked with the library, against the reference's own headers when a reference checkout is given, else against the stand-in
# declarations of tests/host/refdecl, with the skeletons and miniature third-party headers of orb_slam3_detailed_comments_b200/host/refshim.
# Run by __graft_entry__.build(); the binary is git-ignored.
set -e
ROOT="$(cd "$(dirname "$0")/../.." && pwd)"
REF="${ORB_REFERENCE_ROOT:-/root/reference}"
H="$ROOT/orb_slam3_detailed_comments_b200/host"
if [ -f "$REF/include/ORBmatcher.h" ]; then DECL=(-I "$REF/include" -I "$REF"); else DECL=(-I "$ROOT/tests/host/refdecl"); fi
g++ -std=c++14 -O1 -Wall -Wno-unused-function -Wno-comment -include "$H/refshim/ref_skeleton.h" -I "$H/refshim" "${DECL[@]}" \
    -I "$ROOT/include" -I "$H" "$ROOT/tests/host/rgbd_member.cc" "$H/ORBextractor_b200.cc" "$H/Frame_stereo_b200.cc" "$H/ORBmatcher_b200.cc" \
    -L "$ROOT/orb_slam3_detailed_comments_b200/lib" -lorbslam3_b200 -Wl,-rpath,'$ORIGIN/../../orb_slam3_detailed_comments_b200/lib' -lpthread \
    -o "$ROOT/tests/host/rgbd_member"
