// TEST INFRASTRUCTURE ONLY (oracle/).  C entry points around the reference's DBoW2 (Thirdparty/DBoW2: TemplatedVocabulary.h, FORB.cpp,
// ScoringObject.cpp, BowVector.cpp, FeatureVector.cpp, DUtils) and src/KeyFrameDatabase.cc, all compiled VERBATIM where they lie
// (oracle/Makefile target `ref`, _ref/libdbowref.so; oracle/dbowshim/pre.hpp).  Pins the vocabulary text loader, transform(),
// the L1 score and the loop / relocalisation candidate detection of the restatements (and of the CUDA library) to that source.
#include <cstdint>
#include <cstring>
#include <memory>
#include <vector>

#include "KeyFrameDatabase.h"

using namespace ORB_SLAM2;

namespace {
DBoW2::BowVector make_bow(const uint32_t* w, const double* v, int n) {
    DBoW2::BowVector b;
    for (int i = 0; i < n; i++) b.insert(b.end(), std::make_pair((DBoW2::WordId)w[i], (DBoW2::WordValue)v[i]));
    return b;
}
// The tree as TemplatedVocabulary keeps it (the protected m_nodes), read through a pointer to member formed in a derived class.
struct VocNodes : ORBVocabulary {
    static const std::vector<Node>& of(const ORBVocabulary& v) { return v.*(&VocNodes::m_nodes); }
};
}  // namespace

extern "C" {

void* dbowref_voc_load_text(const char* path) {
    ORBVocabulary* voc = new ORBVocabulary();
    if (!voc->loadFromTextFile(path)) { delete voc; return nullptr; }
    return voc;
}
void dbowref_voc_destroy(void* h) { delete static_cast<ORBVocabulary*>(h); }
int dbowref_voc_words(void* h) { return (int)static_cast<ORBVocabulary*>(h)->size(); }
int dbowref_voc_nodes(void* h) { return (int)VocNodes::of(*static_cast<ORBVocabulary*>(h)).size(); }
// Node by node: parent, leaf flag, 32-byte descriptor (zeros for the root), weight; k and L of the tree.
void dbowref_voc_export(void* h, int32_t* parent, uint8_t* is_leaf, uint8_t* desc, double* weight, int* k, int* L) {
    const ORBVocabulary* voc = static_cast<ORBVocabulary*>(h);
    const auto& nodes = VocNodes::of(*voc);
    for (size_t i = 0; i < nodes.size(); i++) {
        parent[i] = (int32_t)nodes[i].parent;
        is_leaf[i] = nodes[i].isLeaf() ? 1 : 0;
        weight[i] = nodes[i].weight;
        std::memset(desc + i * 32, 0, 32);
        if (!nodes[i].descriptor.empty()) std::memcpy(desc + i * 32, nodes[i].descriptor.data, 32);
    }
    *k = voc->getBranchingFactor();
    *L = voc->getDepthLevels();
}

// TemplatedVocabulary::transform(features, BowVector, FeatureVector, levelsup) — Frame::ComputeBoW (src/Frame.cc:395-402)
int dbowref_transform(void* h, const uint8_t* desc, int n, int levelsup, uint32_t* bow_word, double* bow_val, int* n_bow,
                      uint32_t* fv_node, int32_t* fv_start, uint32_t* fv_idx, int* n_nodes) {
    ORBVocabulary* voc = static_cast<ORBVocabulary*>(h);
    std::vector<cv::Mat> feats(n);
    for (int i = 0; i < n; i++) { feats[i] = cv::Mat(1, 32, CV_8U); std::memcpy(feats[i].data, desc + (size_t)i * 32, 32); }
    DBoW2::BowVector bow;
    DBoW2::FeatureVector fv;
    voc->transform(feats, bow, fv, levelsup);
    int k = 0;
    for (const auto& e : bow) { bow_word[k] = e.first; bow_val[k] = e.second; k++; }
    *n_bow = k;
    int a = 0, p = 0;
    for (const auto& e : fv) {
        fv_node[a] = e.first; fv_start[a] = p;
        for (unsigned int f : e.second) fv_idx[p++] = f;
        a++;
    }
    fv_start[a] = p;
    *n_nodes = a;
    return k;
}

// TemplatedVocabulary::score -> L1Scoring::score (ScoringObject.cpp:23-71)
double dbowref_score(void* h, const uint32_t* w1, const double* v1, int n1, const uint32_t* w2, const double* v2, int n2) {
    return static_cast<ORBVocabulary*>(h)->score(make_bow(w1, v1, n1), make_bow(w2, v2, n2));
}

// KeyFrameDatabase::add for keyframes 0..n_kf-1 (in order), then DetectRelocalizationCandidates (loop = 0) or
// DetectLoopCandidates(query keyframe with `connected`, minScore) (loop = 1).  neigh: n_kf x 10, -1 padded, best first.
int dbowref_detect_candidates(void* h, int loop, int n_kf, const int32_t* kf_start, const uint32_t* kf_word, const double* kf_value,
                              const uint32_t* q_word, const double* q_value, int nq, const uint8_t* connected, const int32_t* neigh,
                              float minScore, int32_t* out) {
    ORBVocabulary* voc = static_cast<ORBVocabulary*>(h);
    KeyFrameDatabase db(*voc);
    std::vector<KeyFrame> kfs(n_kf);
    for (int k = 0; k < n_kf; k++) {
        kfs[k].mnId = k;
        kfs[k].mBowVec = make_bow(kf_word + kf_start[k], kf_value + kf_start[k], kf_start[k + 1] - kf_start[k]);
        for (int j = 0; j < 10 && neigh[(size_t)k * 10 + j] >= 0; j++) kfs[k].covisible.push_back(&kfs[neigh[(size_t)k * 10 + j]]);
    }
    for (int k = 0; k < n_kf; k++) db.add(&kfs[k]);
    std::vector<KeyFrame*> res;
    if (loop) {
        KeyFrame q;
        q.mnId = n_kf + 7;
        q.mBowVec = make_bow(q_word, q_value, nq);
        for (int k = 0; k < n_kf; k++) if (connected && connected[k]) q.connected.insert(&kfs[k]);
        res = db.DetectLoopCandidates(&q, minScore);
    } else {
        Frame F;
        F.mnId = n_kf + 7;
        F.mBowVec = make_bow(q_word, q_value, nq);
        res = db.DetectRelocalizationCandidates(&F);
    }
    for (size_t i = 0; i < res.size(); i++) out[i] = (int32_t)(res[i] - &kfs[0]);
    return (int)res.size();
}

// A SEQUENCE of DetectRelocalizationCandidates calls on the same database and KeyFrame objects: KeyFrame::mRelocScore persists
// between the queries, and the covisibility accumulation (:262-275) reads it for neighbours the current query did not score.
// q_start: n_q + 1 offsets into q_word / q_value; out: n_q rows of `out_stride` slots, out_n[i] = candidates of query i.
int dbowref_reloc_sequence(void* h, int n_kf, const int32_t* kf_start, const uint32_t* kf_word, const double* kf_value, int n_q,
                           const int32_t* q_start, const uint32_t* q_word, const double* q_value, const int32_t* neigh, int32_t* out,
                           int out_stride, int32_t* out_n) {
    ORBVocabulary* voc = static_cast<ORBVocabulary*>(h);
    KeyFrameDatabase db(*voc);
    std::vector<KeyFrame> kfs(n_kf);
    for (int k = 0; k < n_kf; k++) {
        kfs[k].mnId = k;
        kfs[k].mBowVec = make_bow(kf_word + kf_start[k], kf_value + kf_start[k], kf_start[k + 1] - kf_start[k]);
        for (int j = 0; j < 10 && neigh[(size_t)k * 10 + j] >= 0; j++) kfs[k].covisible.push_back(&kfs[neigh[(size_t)k * 10 + j]]);
    }
    for (int k = 0; k < n_kf; k++) db.add(&kfs[k]);
    for (int i = 0; i < n_q; i++) {
        Frame F;
        F.mnId = n_kf + 7 + i;
        F.mBowVec = make_bow(q_word + q_start[i], q_value + q_start[i], q_start[i + 1] - q_start[i]);
        const std::vector<KeyFrame*> res = db.DetectRelocalizationCandidates(&F);
        out_n[i] = (int32_t)res.size();
        for (size_t j = 0; j < res.size() && (int)j < out_stride; j++) out[(size_t)i * out_stride + j] = (int32_t)(res[j] - &kfs[0]);
    }
    return 0;
}

}  // extern "C"
