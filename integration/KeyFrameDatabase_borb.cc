// Drop-in replacement of the reference's src/KeyFrameDatabase.cc: same class, same methods (include/KeyFrameDatabase.h:41-75 is
// used UNCHANGED), the keyframes' BowVectors — and their descriptors, for ORBmatcher::SearchByBoW against the database — live in
// HBM (borb_kfdb), and the inverted-file walk + mpVoc->score() loop of DetectLoopCandidates / DetectRelocalizationCandidates is
// one borb_kfdb_query launch (include/borb_kfdb_adapters.hpp).  The header has no room for new members, so the per-database
// state (device handle, KeyFrame* <-> slot maps) sits in a side table keyed by `this`; mvInvertedFile stays empty.
//
// CMake:  replace src/KeyFrameDatabase.cc by this file, add ${BORB_DIR}/include to the include path, link libborb.so.
// Define BORB_KFDB_SCORING_ONLY to keep only the BowVectors resident (no descriptors: SearchByBoW then uses host views).
#include "KeyFrameDatabase.h"

#include "KeyFrame.h"
#include "Frame.h"

#include <memory>
#include <mutex>
#include <unordered_map>

#include "borb_kfdb_adapters.hpp"

namespace ORB_SLAM2 {

namespace {
typedef borb::adapt::KfdbState<KeyFrame> State;
std::mutex g_states_mu;
std::unordered_map<const KeyFrameDatabase*, std::unique_ptr<State> > g_states;
State& state_of(const KeyFrameDatabase* db) {
    std::lock_guard<std::mutex> lk(g_states_mu);
    std::unique_ptr<State>& p = g_states[db];
    if (!p) p.reset(new State());
    return *p;
}
}  // namespace

KeyFrameDatabase::KeyFrameDatabase(const ORBVocabulary& voc) : mpVoc(&voc) {
    std::lock_guard<std::mutex> lk(g_states_mu);
    g_states.erase(this);                     // an earlier database at the same address is gone
}

void KeyFrameDatabase::add(KeyFrame* pKF) {
#ifdef BORB_KFDB_SCORING_ONLY
    borb::adapt::kfdb_add(state_of(this), pKF, (const borb_keyframe_view*)nullptr);
#else
    // features for the resident SearchByBoW: mvKeysUn, mDescriptors, mFeatVec, has_mp[i] = MapPoint present and not bad
    const std::vector<MapPoint*> mps = pKF->GetMapPointMatches();
    std::vector<uint8_t> has_mp(mps.size());
    for (size_t i = 0; i < mps.size(); i++) has_mp[i] = mps[i] && !mps[i]->isBad();
    const borb::adapt::FlatFeatVec<DBoW2::FeatureVector> fv(pKF->mFeatVec);
    const borb_keyframe_view v = borb::adapt::keyframe_view(pKF, has_mp.data(), fv.view());
    borb::adapt::kfdb_add(state_of(this), pKF, &v);
#endif
}

void KeyFrameDatabase::erase(KeyFrame* pKF) { borb::adapt::kfdb_erase(state_of(this), pKF); }

void KeyFrameDatabase::clear() { borb::adapt::kfdb_clear(state_of(this)); }

std::vector<KeyFrame*> KeyFrameDatabase::DetectLoopCandidates(KeyFrame* pKF, float minScore) {
    return borb::adapt::kfdb_detect_loop(state_of(this), pKF, minScore);
}

std::vector<KeyFrame*> KeyFrameDatabase::DetectRelocalizationCandidates(Frame* F) {
    return borb::adapt::kfdb_detect_relocalization(state_of(this), F);
}

#ifndef BORB_KFDB_SCORING_ONLY
// LoopClosing::ComputeSim3's SearchByBoW(mpCurrentKF, pKF, vvpMapPointMatches[i]) (src/LoopClosing.cc:251-280) for every candidate
// in one call on the resident keyframes (INTEGRATION.md shows the change to ComputeSim3).  Returns nmatches per candidate.
std::vector<int> SearchLoopCandidatesByBoW(KeyFrameDatabase* pDB, KeyFrame* pKF, const std::vector<KeyFrame*>& candidates, float nnratio,
                                           bool checkOri, std::vector<std::vector<MapPoint*> >& vvpMatches) {
    return borb::adapt::kfdb_search_loop_candidates<KeyFrame, MapPoint>(state_of(pDB), pKF, candidates, nnratio, checkOri, vvpMatches);
}
#endif

}  // namespace ORB_SLAM2
