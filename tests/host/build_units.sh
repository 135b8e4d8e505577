#!/bin/bash
# Builds tests/host/host_units: all thirteen host translation units + the test driver, against the reference's own headers when a reference
# checkout is given, else against the stand-in declarations of tests/host/refdecl, with the skeleton map and the miniature third-party headers
# of orb_slam3_detailed_comments_b200/host/refshim.  The C ABI calls the units make are wrapped (-Wl,--wrap=): the driver records each call's
# inputs and outputs before and after forwarding it to liborbslam3_b200.  A binary of its own, so that host_boundary does not depend on it.
# Run by __graft_entry__.build() after build.sh; the binary is git-ignored.
set -e
ROOT="$(cd "$(dirname "$0")/../.." && pwd)"
REF="${ORB_REFERENCE_ROOT:-/root/reference}"
H="$ROOT/orb_slam3_detailed_comments_b200/host"
if [ -f "$REF/include/ORBmatcher.h" ]; then DECL=(-I "$REF/include" -I "$REF"); else DECL=(-I "$ROOT/tests/host/refdecl"); fi
WRAP=""
for f in orbm_search_bow orbm_search_bow_keyframes orbm_search_initialization orbm_search_triangulation orbm_search_keyframe orbv_create orbv_transform \
         orbo_pose_optimization liba_solve; do WRAP="$WRAP,--wrap=$f"; done
# every skeleton section at once; _TRI and _BOW are given empty, as ref_skeleton.h defines them again (refshim/sophus/se3.hpp reads _TRI first)
g++ -std=c++14 -O1 -DORB_REFSHIM_BOW= -DORB_REFSHIM_TRI= -DORB_REFSHIM_FUSE -DORB_REFSHIM_VOC -DORB_REFSHIM_POSE -DORB_REFSHIM_LIBA -Wall -Wno-unused-function -Wno-comment -Wno-reorder \
    -include "$H/refshim/ref_skeleton.h" -I "$H/refshim" "${DECL[@]}" -I "$ROOT/include" -I "$H" "$ROOT/tests/host/host_units.cc" \
    "$H/ORBextractor_b200.cc" "$H/Frame_stereo_b200.cc" "$H/ORBmatcher_b200.cc" "$H/Optimizer_lba_b200.cc" \
    "$H/ORBmatcher_bow_b200.cc" "$H/ORBmatcher_triangulation_b200.cc" "$H/ORBmatcher_init_b200.cc" "$H/ORBmatcher_fuse_b200.cc" \
    "$H/ORBmatcher_reloc_b200.cc" "$H/ORBmatcher_sim3_b200.cc" "$H/Frame_bow_b200.cc" "$H/Optimizer_pose_b200.cc" "$H/Optimizer_liba_b200.cc" \
    -L "$ROOT/orb_slam3_detailed_comments_b200/lib" -lorbslam3_b200 -Wl"$WRAP" \
    -Wl,-rpath,'$ORIGIN/../../orb_slam3_detailed_comments_b200/lib' -lpthread -o "$ROOT/tests/host/host_units"
