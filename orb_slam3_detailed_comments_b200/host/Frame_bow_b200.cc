// Frame_bow_b200.cc -- Frame::ComputeBoW (/root/reference/src/Frame.cc:984-997) on the GPU.
//
// Compiled against the reference's headers.  mpORBvocabulary->transform(descriptors, mBowVec, mFeatVec, 4) -- DBoW2's tree walk of every
// descriptor, TF-IDF weights, the L1-normalised BowVector and the level-4 FeatureVector -- is orbv_transform over the descriptors the
// frame's extractor left on the device.  On the host: the vocabulary is flattened ONCE per ORBVocabulary object into orbv_create's arrays
// (node 0 = root, children in m_nodes[i].children order, descriptors, word ids, weights, m_L), and the two containers are filled the way
// DBoW2 fills them: BowVector entries in ascending word order, feature i under its node iff its word's weight is > 0
// (TemplatedVocabulary.h:1153-1157).  The vocabulary's nodes are protected members of DBoW2::TemplatedVocabulary; they are read through
// a derived class (no change to the reference's headers).  KeyFrame::ComputeBoW (KeyFrame.cc:101-112) has the same body.
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "Frame.h"             // the reference's header (here: the skeleton that stands in for it)
#include "marshal.h"

namespace {

struct VocabularyAccess : ORB_SLAM3::ORBVocabulary {
    typedef ORB_SLAM3::ORBVocabulary Base;
    static const std::vector<Node>& nodes(const Base& v) { return v.*(&VocabularyAccess::m_nodes); }
    static int depth_levels(const Base& v) { return v.*(&VocabularyAccess::m_L); }
};

struct VocabularyCache {
    std::mutex mu;
    std::map<const ORB_SLAM3::ORBVocabulary*, orbv_vocabulary*> byObject;
    ~VocabularyCache() { for (auto& kv : byObject) orbv_destroy(kv.second); }
};

const orbv_vocabulary* device_vocabulary(const ORB_SLAM3::ORBVocabulary* voc) {
    static VocabularyCache cache;
    std::lock_guard<std::mutex> lk(cache.mu);
    auto it = cache.byObject.find(voc);
    if (it != cache.byObject.end()) return it->second;
    const auto& nodes = VocabularyAccess::nodes(*voc);
    const int n = (int)nodes.size();
    if (n == 0) throw orb_b200::Error("Frame::ComputeBoW: empty vocabulary");
    std::vector<int32_t> child_offset(n + 1, 0), child_ids, word(n, -1);
    std::vector<uint8_t> desc((size_t)n * 32, 0);
    std::vector<double> weight(n, 0.0);
    for (int i = 0; i < n; ++i) {
        const auto& nd = nodes[i];
        for (size_t c = 0; c < nd.children.size(); ++c) child_ids.push_back((int32_t)nd.children[c]);
        child_offset[i + 1] = (int32_t)child_ids.size();
        if (i > 0 && !nd.descriptor.empty()) std::memcpy(&desc[(size_t)i * 32], nd.descriptor.template ptr<unsigned char>(), 32);   // the root has no descriptor
        if (nd.isLeaf() && i > 0) { word[i] = (int32_t)nd.word_id; weight[i] = nd.weight; }
    }
    orbv_vocabulary* out = nullptr;
    orb_b200::check(orbv_create(orb_b200::device_ordinal(), n, VocabularyAccess::depth_levels(*voc), child_offset.data(), child_ids.data(), desc.data(), word.data(), weight.data(), &out),
                    "orbv_create");
    cache.byObject[voc] = out;
    return out;
}

}  // namespace

namespace ORB_SLAM3 {

void Frame::ComputeBoW() {
    if (!mBowVec.empty()) return;
    orbx_handle* h = orb_b200::resident_frame(*this, "Frame::ComputeBoW");
    mFeatVec.clear();
    if (N == 0) return;
    const orbv_vocabulary* voc = device_vocabulary(mpORBvocabulary);
    const int cap = orbx_max_features(h);
    std::vector<int32_t> word(N), node(N), bow_word(cap > N ? cap : N);
    std::vector<double> weight(N), bow_weight(cap > N ? cap : N);
    int32_t bow_count = 0;
    orb_b200::check(orbv_transform(h, voc, 4, 0, word.data(), node.data(), weight.data(), &bow_count, bow_word.data(), bow_weight.data()), "orbv_transform");
    for (int k = 0; k < bow_count; ++k) mBowVec.insert(mBowVec.end(), std::make_pair((DBoW2::WordId)bow_word[k], (DBoW2::WordValue)bow_weight[k]));
    for (int i = 0; i < N; ++i)
        if (weight[i] > 0) mFeatVec.addFeature((DBoW2::NodeId)node[i], (unsigned int)i);
}

}  // namespace ORB_SLAM3
