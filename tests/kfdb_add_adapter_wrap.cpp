// Drives borb::adapt::kfdb_add_resident (include/borb_kfdb_adapters.hpp) on a stand-in KeyFrame with the reference's member names,
// next to borb::adapt::kfdb_add on the keyframe's host view, so that tests/test_gpu_kfdb_add_frames.py can check that both leave the
// same database.  Compiled by the test (g++, oracle/cvmini for cv::Mat / cv::KeyPoint, linked against libborb.so).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <exception>
#include <map>
#include <vector>

#include <opencv2/core/core.hpp>

namespace stub {
struct KeyFrame {
    int N = 0;
    std::vector<cv::KeyPoint> mvKeysUn;
    cv::Mat mDescriptors;
    std::vector<float> mvuRight, mvScaleFactors, mvLevelSigma2;
    std::map<unsigned, double> mBowVec;
    std::map<unsigned, std::vector<unsigned> > mFeatVec;
};
}  // namespace stub

#define BORB_ADAPTER_NO_EXTRACTOR
#include "borb_kfdb_adapters.hpp"

namespace {
// every live slot of a database: counts, whole device block and host row copies
std::vector<std::vector<uint8_t> > snapshot(borb_kfdb* db) {
    int32_t n = 0;
    borb::check(borb_kfdb_size(db, &n, nullptr), "borb_kfdb_size");
    std::vector<std::vector<uint8_t> > out(n);
    for (int32_t s = 0; s < n; s++) {
        int32_t c[4];
        uint64_t bytes = 0;
        borb::check(borb_debug_kfdb_read(db, s, c, &bytes, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr),
                    "borb_debug_kfdb_read");
        std::vector<uint8_t>& o = out[s];
        o.assign(16 + bytes + (size_t)c[1] * 8, 0);
        std::memcpy(o.data(), c, 16);
        borb::check(borb_debug_kfdb_read(db, s, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                                         reinterpret_cast<uint32_t*>(o.data() + 16 + bytes), o.data() + 16),
                    "borb_debug_kfdb_read");
    }
    return out;
}
}  // namespace

// n_kf keyframes: host views (keys, desc, FeatureVector, BowVector) and their resident frames (BoW computed at the same levelsup);
// has_mp[k] may be NULL.  Keyframe k goes to database A through kfdb_add and to database B through kfdb_add_resident.  Returns 0
// when both databases hold the same slots byte for byte and map every keyframe to the same slot, 2 (with err) when they differ.
extern "C" int kfdb_add_adapter_run(int n_kf, const int32_t* n_feat, const void* const* keys, const uint8_t* const* desc, const int32_t* n_nodes,
                                    const uint32_t* const* fv_node, const int32_t* const* fv_start, const uint32_t* const* fv_idx,
                                    const int32_t* n_bow, const uint32_t* const* bow_word, const double* const* bow_value,
                                    const uint8_t* const* has_mp, void* const* frames, char* err, int errlen) {
    try {
        std::vector<stub::KeyFrame> kf(n_kf);
        borb::adapt::KfdbState<stub::KeyFrame> A, B;
        for (int k = 0; k < n_kf; k++) {
            stub::KeyFrame& K = kf[k];
            const int n = n_feat[k];
            K.N = n;
            K.mvKeysUn.resize(n);
            if (n) std::memcpy(K.mvKeysUn.data(), keys[k], (size_t)n * sizeof(cv::KeyPoint));
            K.mDescriptors = cv::Mat(n, 32, CV_8U);
            if (n) std::memcpy(K.mDescriptors.data, desc[k], (size_t)n * 32);
            for (int a = 0; a < n_nodes[k]; a++)
                K.mFeatVec[fv_node[k][a]] = std::vector<unsigned>(fv_idx[k] + fv_start[k][a], fv_idx[k] + fv_start[k][a + 1]);
            for (int i = 0; i < n_bow[k]; i++) K.mBowVec[bow_word[k][i]] = bow_value[k][i];
            const borb::adapt::FlatFeatVec<std::map<unsigned, std::vector<unsigned> > > fv(K.mFeatVec);
            const borb_keyframe_view v = borb::adapt::keyframe_view(&K, has_mp[k], fv.view());
            borb::adapt::kfdb_add(A, &K, &v);
            borb::adapt::kfdb_add_resident(B, &K, static_cast<const borb_frame*>(frames[k]), has_mp[k]);
        }
        for (int k = 0; k < n_kf; k++)
            if (A.slot_of.at(&kf[k]) != B.slot_of.at(&kf[k]) || B.kf_of_slot[B.slot_of.at(&kf[k])] != &kf[k]) {
                std::snprintf(err, errlen, "keyframe %d: slot %d through kfdb_add, %d through kfdb_add_resident", k, A.slot_of.at(&kf[k]),
                              B.slot_of.at(&kf[k]));
                return 2;
            }
        const std::vector<std::vector<uint8_t> > a = snapshot(A.db), b = snapshot(B.db);
        if (a.size() != b.size()) { std::snprintf(err, errlen, "%zu slots vs %zu", a.size(), b.size()); return 2; }
        for (size_t s = 0; s < a.size(); s++)
            if (a[s] != b[s]) { std::snprintf(err, errlen, "slot %zu differs", s); return 2; }
        uint64_t ba = 0, bb = 0;
        borb::check(borb_kfdb_size(A.db, nullptr, &ba), "borb_kfdb_size");
        borb::check(borb_kfdb_size(B.db, nullptr, &bb), "borb_kfdb_size");
        if (ba != bb) { std::snprintf(err, errlen, "%llu device bytes vs %llu", (unsigned long long)ba, (unsigned long long)bb); return 2; }
        return 0;
    } catch (const std::exception& e) {
        std::snprintf(err, errlen, "%s", e.what());
        return 1;
    }
}
