// Drives borb::adapt::kfdb_search_loop_candidates (include/borb_kfdb_adapters.hpp) — the code INTEGRATION.md puts into
// LoopClosing::ComputeSim3 — on stand-in KeyFrame / MapPoint types that carry the reference's member names, so that
// tests/test_gpu_kfdb_loop.py can compare its vpMatches12 with the verbatim ORBmatcher::SearchByBoW(KeyFrame*, KeyFrame*).
// Compiled by the test (g++, oracle/cvmini for cv::Mat / cv::KeyPoint, linked against libborb.so).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <exception>
#include <map>
#include <vector>

#include <opencv2/core/core.hpp>

namespace stub {
struct MapPoint {
    int kf = -1, idx = -1;                         // which keyframe feature this point stands for
    bool bad = false;
    bool isBad() { return bad; }
};
struct KeyFrame {
    int N = 0;
    std::vector<cv::KeyPoint> mvKeysUn;
    cv::Mat mDescriptors;
    std::vector<float> mvuRight, mvScaleFactors, mvLevelSigma2;
    std::map<unsigned, double> mBowVec;
    std::map<unsigned, std::vector<unsigned> > mFeatVec;
    std::vector<MapPoint*> mps;
    std::vector<MapPoint*> GetMapPointMatches() { return mps; }
};
}  // namespace stub

#define BORB_ADAPTER_NO_EXTRACTOR
#include "borb_kfdb_adapters.hpp"

// state[k][i]: 0 no MapPoint, 1 a good one, 2 a bad one.  add_state is what the database is given at add(), now_state what
// GetMapPointMatches() returns when the search runs.  erase >= 0 erases that keyframe from the database before the search.
// match: n_cand x n_feat[query], the candidate feature whose MapPoint vvpMatches[c][i] holds, or -1.
extern "C" int loop_adapter_run(int n_kf, const int32_t* n_feat, const void* const* keys, const uint8_t* const* desc, const int32_t* n_nodes,
                                const uint32_t* const* fv_node, const int32_t* const* fv_start, const uint32_t* const* fv_idx,
                                const uint8_t* const* add_state, const uint8_t* const* now_state, int query, int n_cand, const int32_t* cand,
                                int erase, float nnratio, int check_ori, int32_t* counts, int32_t* match, char* err, int errlen) {
    try {
        std::vector<stub::KeyFrame> kf(n_kf);
        std::vector<std::vector<stub::MapPoint> > pts(n_kf);
        borb::adapt::KfdbState<stub::KeyFrame> S;
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
            pts[k].resize(n);
            K.mps.assign(n, nullptr);
            for (int i = 0; i < n; i++) {
                pts[k][i].kf = k; pts[k][i].idx = i;
                if (add_state[k][i]) { pts[k][i].bad = add_state[k][i] == 2; K.mps[i] = &pts[k][i]; }
            }
            // KeyFrameDatabase::add of integration/KeyFrameDatabase_borb.cc
            const std::vector<stub::MapPoint*> mps = K.GetMapPointMatches();
            std::vector<uint8_t> has_mp(mps.size());
            for (size_t i = 0; i < mps.size(); i++) has_mp[i] = mps[i] && !mps[i]->isBad();
            const borb::adapt::FlatFeatVec<std::map<unsigned, std::vector<unsigned> > > fv(K.mFeatVec);
            const borb_keyframe_view v = borb::adapt::keyframe_view(&K, has_mp.data(), fv.view());
            borb::adapt::kfdb_add(S, &K, &v);
        }
        for (int k = 0; k < n_kf; k++)                       // MapPoints culled, added or set bad since add()
            for (int i = 0; i < n_feat[k]; i++) {
                kf[k].mps[i] = nullptr;
                if (now_state[k][i]) { pts[k][i].bad = now_state[k][i] == 2; kf[k].mps[i] = &pts[k][i]; }
            }
        if (erase >= 0) borb::adapt::kfdb_erase(S, &kf[erase]);
        std::vector<stub::KeyFrame*> cands(n_cand);
        for (int c = 0; c < n_cand; c++) cands[c] = &kf[cand[c]];
        std::vector<std::vector<stub::MapPoint*> > vvp;
        const std::vector<int> nm = borb::adapt::kfdb_search_loop_candidates<stub::KeyFrame, stub::MapPoint>(S, &kf[query], cands, nnratio,
                                                                                                             check_ori != 0, vvp);
        const int n1 = n_feat[query];
        for (int c = 0; c < n_cand; c++) {
            counts[c] = nm[c];
            if ((int)vvp[c].size() != n1) { std::snprintf(err, errlen, "vpMatches12 of candidate %d has %zu entries", c, vvp[c].size()); return 2; }
            for (int i = 0; i < n1; i++) {
                const stub::MapPoint* p = vvp[c][i];
                if (p && p->kf != cand[c]) { std::snprintf(err, errlen, "candidate %d row %d holds a point of keyframe %d", c, i, p->kf); return 2; }
                match[(size_t)c * n1 + i] = p ? p->idx : -1;
            }
        }
        return 0;
    } catch (const std::exception& e) {
        std::snprintf(err, errlen, "%s", e.what());
        return 1;
    }
}
