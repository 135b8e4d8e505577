// Host build of csrc/blur_mma.cuh's fragment builder for tests/test_blur_mma_emul.py: the table the handle uploads for k_blur_mma.
#include "../../orb_slam3_detailed_comments_b200/csrc/blur_mma.cuh"

extern "C" void emul_blur_fragments(uint32_t* frag) { orbdev::bm_fragments(frag); }
extern "C" int emul_blur_tile(int* tw_th_srow) {
    tw_th_srow[0] = BM_TW;
    tw_th_srow[1] = BM_TH;
    tw_th_srow[2] = BM_SROW;
    return 0;
}
