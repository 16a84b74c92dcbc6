// borb_kfdb_adapters.hpp — header-only adapter for ORB_SLAM2::KeyFrameDatabase (reference include/KeyFrameDatabase.h:41-75,
// src/KeyFrameDatabase.cc): add / erase / clear keep the keyframes' BowVectors (and, when the caller supplies a keyframe view,
// their descriptors for SearchByBoW) resident in HBM; DetectLoopCandidates / DetectRelocalizationCandidates replace the
// inverted-file walk and the mpVoc->score() loop by ONE borb_kfdb_query launch (shared-word count, float L1 score and first
// shared word of EVERY keyframe) and then run the reference's remaining, pointer-graph part — thresholds, covisibility
// accumulation over KeyFrame::GetBestCovisibilityKeyFrames(10), the KeyFrame::mn{Loop,Reloc}{Query,Words} / m{Loop,Reloc}Score
// bookkeeping fields — on the calling thread, written here from the procedure's definition (SURVEY §8 f1).
// Templated on the reference's KeyFrame / Frame types; integration/KeyFrameDatabase_borb.cc instantiates it as the drop-in
// replacement of src/KeyFrameDatabase.cc.  tests/test_gpu_adapters.py EXECUTES it on the GPU through the same C wrapper
// (oracle/dbowref_wrap.cpp) that drives the verbatim KeyFrameDatabase.cc, single queries and query sequences.
//
// Include AFTER <opencv2/core/core.hpp> and borb_matcher_adapters.hpp (thread_matcher, check).
#pragma once
#include <algorithm>
#include <cstdint>
#include <list>
#include <mutex>
#include <set>
#include <stdexcept>
#include <unordered_map>
#include <utility>
#include <vector>

#include "borb_matcher_adapters.hpp"

namespace borb {
namespace adapt {

template <class KeyFrameT>
struct KfdbState {
    borb_kfdb* db = nullptr;
    int device = 0;
    std::mutex mu;                                        // KeyFrameDatabase::mMutex: add / erase / Detect* run on different threads
    std::unordered_map<KeyFrameT*, int32_t> slot_of;
    std::vector<KeyFrameT*> kf_of_slot;                   // slots are never reused: slot order == insertion order into the word lists
    ~KfdbState() { if (db) borb_kfdb_destroy(db); }
    void ensure() { if (!db) check(borb_kfdb_create(device, &db), "borb_kfdb_create"); }
};

// DBoW2::BowVector (std::map<WordId, WordValue>) -> ascending arrays
template <class BowVec>
inline void flat_bow(const BowVec& b, std::vector<uint32_t>& w, std::vector<double>& v) {
    w.clear(); v.clear();
    w.reserve(b.size()); v.reserve(b.size());
    for (const auto& kv : b) { w.push_back((uint32_t)kv.first); v.push_back((double)kv.second); }
}

// KeyFrameDatabase::add (:41-47).  `view` = the keyframe's features for the resident SearchByBoW (keyframe_view of
// borb_matcher_adapters.hpp), or nullptr to keep only the BowVector (scoring only).
template <class KeyFrameT>
inline void kfdb_add(KfdbState<KeyFrameT>& S, KeyFrameT* pKF, const borb_keyframe_view* view) {
    std::lock_guard<std::mutex> lk(S.mu);
    S.ensure();
    std::vector<uint32_t> w; std::vector<double> v;
    flat_bow(pKF->mBowVec, w, v);
    borb_keyframe_view none = {};
    int32_t slot = -1;
    check(borb_kfdb_add(S.db, view ? view : &none, w.data(), v.data(), (int)w.size(), &slot), "borb_kfdb_add");
    if ((size_t)slot >= S.kf_of_slot.size()) S.kf_of_slot.resize((size_t)slot + 1, nullptr);
    S.kf_of_slot[slot] = pKF;
    S.slot_of[pKF] = slot;
}

// KeyFrameDatabase::add (:41-47) of a keyframe whose Frame is still resident (`f`, BoW computed by borb_frames_compute_bow at the
// database's levelsup): the keyframe's features and BowVector are taken from the device, only has_mp (f's n entries, MapPoint present
// && !isBad(); nullptr: none) crosses PCIe.  The database ends as kfdb_add with the keyframe's view leaves it.  Many streams at once:
// borb_kfdb_add_frames with one job per stream, then the slot bookkeeping below per job.
template <class KeyFrameT>
inline void kfdb_add_resident(KfdbState<KeyFrameT>& S, KeyFrameT* pKF, const borb_frame* f, const uint8_t* has_mp) {
    std::lock_guard<std::mutex> lk(S.mu);
    S.ensure();
    int32_t slot = -1;
    const borb_kfdb_add_job job = {S.db, f, has_mp, &slot};
    check(borb_kfdb_add_frames(thread_matcher(S.device), &job, 1), "borb_kfdb_add_frames");
    if ((size_t)slot >= S.kf_of_slot.size()) S.kf_of_slot.resize((size_t)slot + 1, nullptr);
    S.kf_of_slot[slot] = pKF;
    S.slot_of[pKF] = slot;
}

template <class KeyFrameT>
inline void kfdb_erase(KfdbState<KeyFrameT>& S, KeyFrameT* pKF) {          // :49-66
    std::lock_guard<std::mutex> lk(S.mu);
    auto it = S.slot_of.find(pKF);
    if (it == S.slot_of.end()) return;
    check(borb_kfdb_erase(S.db, it->second), "borb_kfdb_erase");
    S.kf_of_slot[it->second] = nullptr;
    S.slot_of.erase(it);
}

template <class KeyFrameT>
inline void kfdb_clear(KfdbState<KeyFrameT>& S) {                          // :68-73
    std::lock_guard<std::mutex> lk(S.mu);
    if (S.db) check(borb_kfdb_clear(S.db), "borb_kfdb_clear");
    S.slot_of.clear(); S.kf_of_slot.clear();
}

// The data-parallel part of both Detect* procedures: per slot the shared-word count, the float score and the first shared word.
struct KfdbScores { std::vector<int32_t> common; std::vector<float> score; std::vector<uint32_t> first; int n = 0; };
template <class KeyFrameT, class BowVec>
inline KfdbScores kfdb_scores(KfdbState<KeyFrameT>& S, const BowVec& query) {
    KfdbScores R;
    if (!S.db) return R;
    std::vector<uint32_t> w; std::vector<double> v;
    flat_bow(query, w, v);
    const size_t cap = S.kf_of_slot.size();
    R.common.assign(cap ? cap : 1, 0); R.score.assign(cap ? cap : 1, 0.f); R.first.assign(cap ? cap : 1, 0xFFFFFFFFu);
    int32_t n = 0;
    check(borb_kfdb_query(thread_matcher(S.device), S.db, w.data(), v.data(), (int)w.size(), R.common.data(), R.score.data(), R.first.data(),
                          (int)cap, &n), "borb_kfdb_query");
    R.n = n;
    return R;
}

// lKFsSharingWords: the keyframes that share a word with the query, in the order the inverted-file walk meets them — ascending
// first shared word, then insertion order into that word's list (== slot order) — minus `skip`.
template <class KeyFrameT>
inline std::vector<int32_t> sharing_order(const KfdbState<KeyFrameT>& S, const KfdbScores& R, const std::set<KeyFrameT*>* skip) {
    std::vector<int32_t> s;
    for (int32_t i = 0; i < R.n; i++)
        if (R.common[i] > 0 && S.kf_of_slot[i] && !(skip && skip->count(S.kf_of_slot[i]))) s.push_back(i);
    std::stable_sort(s.begin(), s.end(), [&](int32_t a, int32_t b) { return R.first[a] < R.first[b]; });
    return s;
}

// KeyFrameDatabase::DetectRelocalizationCandidates (:199-310)
template <class KeyFrameT, class FrameT>
inline std::vector<KeyFrameT*> kfdb_detect_relocalization(KfdbState<KeyFrameT>& S, FrameT* F) {
    std::lock_guard<std::mutex> lk(S.mu);
    const KfdbScores R = kfdb_scores(S, F->mBowVec);
    const std::vector<int32_t> sharing = sharing_order(S, R, (const std::set<KeyFrameT*>*)nullptr);
    if (sharing.empty()) return std::vector<KeyFrameT*>();
    int maxCommonWords = 0;
    for (int32_t s : sharing) {
        KeyFrameT* k = S.kf_of_slot[s];
        k->mnRelocQuery = F->mnId; k->mnRelocWords = R.common[s];                 // the walk's bookkeeping (:211-224)
        if (R.common[s] > maxCommonWords) maxCommonWords = R.common[s];
    }
    const int minCommonWords = maxCommonWords * 0.8f;
    std::list<std::pair<float, KeyFrameT*> > scored;
    for (int32_t s : sharing)
        if (R.common[s] > minCommonWords) {
            KeyFrameT* k = S.kf_of_slot[s];
            k->mRelocScore = R.score[s];
            scored.push_back(std::make_pair(R.score[s], k));
        }
    if (scored.empty()) return std::vector<KeyFrameT*>();
    std::list<std::pair<float, KeyFrameT*> > acc;
    float bestAccScore = 0;
    for (const auto& it : scored) {
        KeyFrameT* pKFi = it.second;
        const std::vector<KeyFrameT*> neigh = pKFi->GetBestCovisibilityKeyFrames(10);
        float bestScore = it.first, accScore = bestScore;
        KeyFrameT* pBestKF = pKFi;
        for (KeyFrameT* pKF2 : neigh) {
            if (pKF2->mnRelocQuery != F->mnId) continue;
            accScore += pKF2->mRelocScore;                 // this query's score, or the one an earlier query left (below minCommonWords)
            if (pKF2->mRelocScore > bestScore) { pBestKF = pKF2; bestScore = pKF2->mRelocScore; }
        }
        acc.push_back(std::make_pair(accScore, pBestKF));
        if (accScore > bestAccScore) bestAccScore = accScore;
    }
    const float minScoreToRetain = 0.75f * bestAccScore;
    std::set<KeyFrameT*> added;
    std::vector<KeyFrameT*> out;
    out.reserve(acc.size());
    for (const auto& it : acc)
        if (it.first > minScoreToRetain && !added.count(it.second)) { out.push_back(it.second); added.insert(it.second); }
    return out;
}

// KeyFrameDatabase::DetectLoopCandidates (:76-197)
template <class KeyFrameT>
inline std::vector<KeyFrameT*> kfdb_detect_loop(KfdbState<KeyFrameT>& S, KeyFrameT* pKF, float minScore) {
    const std::set<KeyFrameT*> connected = pKF->GetConnectedKeyFrames();
    std::lock_guard<std::mutex> lk(S.mu);
    const KfdbScores R = kfdb_scores(S, pKF->mBowVec);
    const std::vector<int32_t> sharing = sharing_order(S, R, &connected);
    if (sharing.empty()) return std::vector<KeyFrameT*>();
    int maxCommonWords = 0;
    for (int32_t s : sharing) {
        KeyFrameT* k = S.kf_of_slot[s];
        k->mnLoopQuery = pKF->mnId; k->mnLoopWords = R.common[s];
        if (R.common[s] > maxCommonWords) maxCommonWords = R.common[s];
    }
    const int minCommonWords = maxCommonWords * 0.8f;
    std::list<std::pair<float, KeyFrameT*> > scored;
    for (int32_t s : sharing)
        if (R.common[s] > minCommonWords) {
            KeyFrameT* k = S.kf_of_slot[s];
            k->mLoopScore = R.score[s];
            if (R.score[s] >= minScore) scored.push_back(std::make_pair(R.score[s], k));
        }
    if (scored.empty()) return std::vector<KeyFrameT*>();
    std::list<std::pair<float, KeyFrameT*> > acc;
    float bestAccScore = minScore;
    for (const auto& it : scored) {
        KeyFrameT* pKFi = it.second;
        const std::vector<KeyFrameT*> neigh = pKFi->GetBestCovisibilityKeyFrames(10);
        float bestScore = it.first, accScore = it.first;
        KeyFrameT* pBestKF = pKFi;
        for (KeyFrameT* pKF2 : neigh) {
            if (pKF2->mnLoopQuery == pKF->mnId && pKF2->mnLoopWords > minCommonWords) {
                accScore += pKF2->mLoopScore;
                if (pKF2->mLoopScore > bestScore) { pBestKF = pKF2; bestScore = pKF2->mLoopScore; }
            }
        }
        acc.push_back(std::make_pair(accScore, pBestKF));
        if (accScore > bestAccScore) bestAccScore = accScore;
    }
    const float minScoreToRetain = 0.75f * bestAccScore;
    std::set<KeyFrameT*> added;
    std::vector<KeyFrameT*> out;
    out.reserve(acc.size());
    for (const auto& it : acc)
        if (it.first > minScoreToRetain && !added.count(it.second)) { out.push_back(it.second); added.insert(it.second); }
    return out;
}

// ORBmatcher::SearchByBoW(KeyFrame* pKF, KeyFrame* pKFi, vpMatches12) (src/ORBmatcher.cc:522-655) of the loop-closing keyframe
// against every keyframe of `candidates` in ONE borb_search_by_bow_kf_db_pairs call (LoopClosing::ComputeSim3, :251-280).  Every
// keyframe must have been added with its features.  The MapPoint masks of the query and the candidates are refreshed from
// GetMapPointMatches() first (what the reference reads at call time) in one borb_kfdb_set_has_mp_batch, then vvpMatches[i] is
// rebuilt as SearchByBoWKF rebuilds vpMatches12.  A candidate that has left the database meanwhile (erased after it passed
// DetectLoopCandidates) gets 0 matches, which ComputeSim3 discards.  Returns the counts.
template <class KeyFrameT, class MapPointT>
inline std::vector<int> kfdb_search_loop_candidates(KfdbState<KeyFrameT>& S, KeyFrameT* pKF, const std::vector<KeyFrameT*>& candidates,
                                                    float nnratio, bool checkOri, std::vector<std::vector<MapPointT*> >& vvpMatches) {
    const size_t nc = candidates.size();
    vvpMatches.assign(nc, std::vector<MapPointT*>());
    std::vector<int> counts(nc, 0);
    const std::vector<MapPointT*> vpMapPoints1 = pKF->GetMapPointMatches();
    for (size_t i = 0; i < nc; i++) vvpMatches[i].assign(vpMapPoints1.size(), static_cast<MapPointT*>(nullptr));
    if (nc == 0) return counts;
    std::lock_guard<std::mutex> lk(S.mu);
    const auto qit = S.slot_of.find(pKF);
    if (qit == S.slot_of.end()) throw std::runtime_error("kfdb_search_loop_candidates: the loop-closing keyframe is not in the database");
    std::vector<size_t> live;                                        // candidates still in the database
    std::vector<int32_t> slots, mask_slots(1, qit->second);
    std::vector<std::vector<MapPointT*> > mps2(nc);
    std::vector<std::vector<uint8_t> > masks(1);
    auto good = [](const std::vector<MapPointT*>& mps) {
        std::vector<uint8_t> hm(mps.size());
        for (size_t i = 0; i < mps.size(); i++) hm[i] = mps[i] && !mps[i]->isBad();                // :558-562, :574-580
        return hm;
    };
    masks[0] = good(vpMapPoints1);
    for (size_t i = 0; i < nc; i++) {
        const auto it = S.slot_of.find(candidates[i]);
        if (it == S.slot_of.end()) continue;
        live.push_back(i);
        slots.push_back(it->second);
        mps2[i] = candidates[i]->GetMapPointMatches();
        if (candidates[i] != pKF) { mask_slots.push_back(it->second); masks.push_back(good(mps2[i])); }
    }
    if (live.empty()) return counts;
    std::vector<const uint8_t*> mask_ptr(masks.size());
    for (size_t i = 0; i < masks.size(); i++) mask_ptr[i] = masks[i].data();
    check(borb_kfdb_set_has_mp_batch(S.db, (int)mask_slots.size(), mask_slots.data(), mask_ptr.data()), "borb_kfdb_set_has_mp_batch");
    const int nl = (int)live.size();
    std::vector<int32_t> nm(nl), off(nl);
    std::vector<uint32_t> pairs(vpMapPoints1.size() * nl + 1);
    int32_t total = 0;
    check(borb_search_by_bow_kf_db_pairs(thread_matcher(S.device), S.db, qit->second, slots.data(), nl, nnratio, checkOri, nm.data(), off.data(),
                                         pairs.data(), (int)pairs.size(), &total), "borb_search_by_bow_kf_db_pairs");
    for (int k = 0; k < nl; k++) {
        const size_t i = live[k];
        counts[i] = nm[k];
        for (int32_t p = off[k]; p < off[k] + nm[k]; p++)
            vvpMatches[i][pairs[p] & 0xFFFFu] = mps2[i][pairs[p] >> 16];                            // :602
    }
    return counts;
}

}  // namespace adapt
}  // namespace borb
