// k_ingest's per-thread body (csrc/resize_core.cuh ig_pixels4) compiled for the host: tests/test_oracle_ingest_cpu.py runs it over
// whole images against the oracle and cv2.
#include <cstdint>

#include "../../orb_slam3_detailed_comments_b200/csrc/resize_core.cuh"

extern "C" void emul_ingest(const uint8_t* src, int format, int sw, int sh, int spitch, uint8_t* dst, int dw, int dh, int dpitch) {
    const orbdev::IngestPlan P = orbdev::ig_plan(src, 0, format, sw, sh, spitch, dst, 0, dw, dh, dpitch);
    for (int y = 0; y < dh; ++y)
        for (int x4 = 0; x4 < dw; x4 += 4) *reinterpret_cast<uint32_t*>(dst + (int64_t)y * dpitch + x4) = orbdev::ig_pixels4(P, src, x4, y);
}
