// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle/orb_prims.h / orb_port.h headers).
// Line-by-line restatements, on POD arrays, of the matcher side of the hot path:
//   Frame::AssignFeaturesToGrid / PosInGrid / GetFeaturesInArea   src/Frame.cc:230-245, 382-392, 327-380
//   ORBmatcher::SearchByProjection(Frame&, vector<MapPoint*>&, th) src/ORBmatcher.cc:45-137
//   ORBmatcher::SearchByBoW(KeyFrame*, Frame&, ...)               src/ORBmatcher.cc:159-288
//   ORBmatcher::SearchByBoW(KeyFrame*, KeyFrame*, ...)            src/ORBmatcher.cc:522-655
//   ORBmatcher::SearchForTriangulation                            src/ORBmatcher.cc:657-823, CheckDistEpipolarLine :140-157
//   ORBmatcher::ComputeThreeMaxima / DescriptorDistance           src/ORBmatcher.cc:1601-1663
//   TemplatedVocabulary::transform / loadFromTextFile             Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1127-1259, 1338-1424
// (further down: the other SearchByProjection overloads, SearchForInitialization, SearchBySim3, Fuse x2, Frame::isInFrustum,
//  MapPoint::PredictScale / ComputeDistinctiveDescriptors, L1Scoring::score, KeyFrameDatabase candidate detection.)
// The reference holds no tests for these functions ("parity unpinned" by the reference itself — SURVEY.md §8c).  The
// restatements are pinned to the reference SOURCE instead: src/ORBmatcher.cc and src/Frame.cc are compiled verbatim
// against plain-data stand-ins of the types they point to (oracle/_ref/libmatchref.so, libframeref.so; oracle/Makefile)
// and tests/test_oracle_match_ref.py / test_oracle_frame_ref.py assert equality on every fixture.  The vocabulary,
// scoring and keyframe-database functions have no such pin (re-derived a second time in numpy, tests/test_oracle_match.py).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <random>
#include <string>
#include <vector>

#include "orb_port.h"

namespace {
constexpr int TH_HIGH = 100, TH_LOW = 50, HISTO_LENGTH = 30;
constexpr int GRID_COLS = 64, GRID_ROWS = 48;   // include/Frame.h:37-38

struct Grid {
    float minX, minY, maxX, maxY, invW, invH;
    std::vector<std::vector<int>> cell;   // [x*ROWS + y], insertion order
};

Grid build_grid(const orbport_kp* k, int n, float minX, float minY, float maxX, float maxY) {
    Grid g;
    g.minX = minX; g.minY = minY; g.maxX = maxX; g.maxY = maxY;
    g.invW = (float)GRID_COLS / (float)(maxX - minX);     // Frame.cc:101-102
    g.invH = (float)GRID_ROWS / (float)(maxY - minY);
    g.cell.assign(GRID_COLS * GRID_ROWS, {});
    for (int i = 0; i < n; i++) {
        const int px = (int)std::round((k[i].x - minX) * g.invW);   // PosInGrid :384-385
        const int py = (int)std::round((k[i].y - minY) * g.invH);
        if (px < 0 || px >= GRID_COLS || py < 0 || py >= GRID_ROWS) continue;
        g.cell[px * GRID_ROWS + py].push_back(i);
    }
    return g;
}

std::vector<int> features_in_area(const Grid& g, const orbport_kp* k, float x, float y, float r, int minLevel, int maxLevel) {
    std::vector<int> out;
    // a NaN centre (a point at the camera centre, orbport_is_in_frustum): the reference's (int)floor(NaN) is INT_MIN on x86,
    // which empties the window; said here without the undefined conversion
    if (!(x == x) || !(y == y)) return out;
    const int nMinCellX = std::max(0, (int)std::floor((x - g.minX - r) * g.invW));
    if (nMinCellX >= GRID_COLS) return out;
    const int nMaxCellX = std::min(GRID_COLS - 1, (int)std::ceil((x - g.minX + r) * g.invW));
    if (nMaxCellX < 0) return out;
    const int nMinCellY = std::max(0, (int)std::floor((y - g.minY - r) * g.invH));
    if (nMinCellY >= GRID_ROWS) return out;
    const int nMaxCellY = std::min(GRID_ROWS - 1, (int)std::ceil((y - g.minY + r) * g.invH));
    if (nMaxCellY < 0) return out;
    const bool bCheckLevels = (minLevel > 0) || (maxLevel >= 0);
    for (int ix = nMinCellX; ix <= nMaxCellX; ix++)
        for (int iy = nMinCellY; iy <= nMaxCellY; iy++)
            for (int idx : g.cell[ix * GRID_ROWS + iy]) {
                const orbport_kp& kp = k[idx];
                if (bCheckLevels) {
                    if (kp.octave < minLevel) continue;
                    if (maxLevel >= 0 && kp.octave > maxLevel) continue;
                }
                const float distx = kp.x - x, disty = kp.y - y;
                if (std::fabs(distx) < r && std::fabs(disty) < r) out.push_back(idx);
            }
    return out;
}

void three_maxima(const std::vector<int>* histo, int L, int& ind1, int& ind2, int& ind3) {
    int max1 = 0, max2 = 0, max3 = 0;
    for (int i = 0; i < L; i++) {
        const int s = (int)histo[i].size();
        if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }
        else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }
        else if (s > max3) { max3 = s; ind3 = i; }
    }
    if (max2 < 0.1f * (float)max1) { ind2 = -1; ind3 = -1; }
    else if (max3 < 0.1f * (float)max1) { ind3 = -1; }
}

int rot_bin(float a1, float a2) {
    const float factor = 1.0f / HISTO_LENGTH;
    float rot = a1 - a2;
    if (rot < 0.0) rot += 360.0f;
    int bin = (int)std::round(rot * factor);
    if (bin == HISTO_LENGTH) bin = 0;
    return bin;
}

struct FeatVec { int nn; const uint32_t* node; const int32_t* start; const uint32_t* idx; };

}  // namespace

extern "C" {

int orbport_features_in_area(const orbport_kp* k, int n, float minX, float minY, float maxX, float maxY, float x, float y, float r,
                             int minLevel, int maxLevel, int32_t* out, int cap) {
    Grid g = build_grid(k, n, minX, minY, maxX, maxY);
    std::vector<int> v = features_in_area(g, k, x, y, r, minLevel, maxLevel);
    for (int i = 0; i < (int)v.size() && i < cap; i++) out[i] = v[i];
    return (int)v.size();
}

// build_grid flattened the way the device keeps it: cell c = x*GRID_ROWS + y holds cell_idx[cell_start[c] .. cell_start[c+1])
// in insertion order (cell_start: GRID_COLS*GRID_ROWS + 1 entries, cell_idx: n).  Returns the number of features in the grid.
int orbport_assign_grid(const orbport_kp* k, int n, float minX, float minY, float maxX, float maxY, int32_t* cell_start, int32_t* cell_idx) {
    const Grid g = build_grid(k, n, minX, minY, maxX, maxY);
    int r = 0;
    for (int c = 0; c < GRID_COLS * GRID_ROWS; c++) {
        cell_start[c] = r;
        for (int i : g.cell[c]) cell_idx[r++] = i;
    }
    cell_start[GRID_COLS * GRID_ROWS] = r;
    return r;
}

// match_feat[iMP] = frame feature index claimed by map point iMP, or -1.  occupied may be NULL.
int orbport_search_by_projection(const orbport_kp* keys_un, const uint8_t* desc, const float* u_right, const uint8_t* occupied, int N,
                                 float minX, float minY, float maxX, float maxY, const float* scale_factors, int n_mp,
                                 const float* proj_x, const float* proj_y, const float* proj_xr, const int32_t* level,
                                 const float* view_cos, const uint8_t* mp_desc, const uint8_t* mp_valid, const uint8_t* mp_has_obs,
                                 float th, float nnratio, int32_t* match_feat) {
    Grid g = build_grid(keys_un, N, minX, minY, maxX, maxY);
    std::vector<char> held(N, 0);          // F.mvpMapPoints[idx] && Observations()>0
    for (int i = 0; i < N; i++) held[i] = occupied ? (occupied[i] != 0) : 0;
    int nmatches = 0;
    const bool bFactor = th != 1.0;
    for (int iMP = 0; iMP < n_mp; iMP++) {
        match_feat[iMP] = -1;
        if (mp_valid && !mp_valid[iMP]) continue;
        const int nPredictedLevel = level[iMP];
        float r = view_cos[iMP] > 0.998 ? 2.5 : 4.0;
        if (bFactor) r *= th;
        const std::vector<int> vIndices = features_in_area(g, keys_un, proj_x[iMP], proj_y[iMP], r * scale_factors[nPredictedLevel],
                                                           nPredictedLevel - 1, nPredictedLevel);
        if (vIndices.empty()) continue;
        const uint8_t* MPdescriptor = mp_desc + (size_t)iMP * 32;
        int bestDist = 256, bestLevel = -1, bestDist2 = 256, bestLevel2 = -1, bestIdx = -1;
        for (int idx : vIndices) {
            if (held[idx]) continue;
            if (u_right && u_right[idx] > 0) {
                const float er = std::fabs(proj_xr[iMP] - u_right[idx]);
                if (er > r * scale_factors[nPredictedLevel]) continue;
            }
            const int dist = orbport_hamming(MPdescriptor, desc + (size_t)idx * 32);
            if (dist < bestDist) { bestDist2 = bestDist; bestDist = dist; bestLevel2 = bestLevel; bestLevel = keys_un[idx].octave; bestIdx = idx; }
            else if (dist < bestDist2) { bestLevel2 = keys_un[idx].octave; bestDist2 = dist; }
        }
        if (bestDist <= TH_HIGH) {
            if (bestLevel == bestLevel2 && bestDist > nnratio * bestDist2) continue;
            match_feat[iMP] = bestIdx;
            // F.mvpMapPoints[bestIdx]=pMP: later map points skip it only if pMP->Observations()>0 (:87-89)
            held[bestIdx] = mp_has_obs ? (mp_has_obs[iMP] != 0) : 1;
            nmatches++;
        }
    }
    return nmatches;
}

// SearchByBoW(KeyFrame*, Frame&): match_f[F.N] = KF feature whose MapPoint the frame feature received, or -1.
int orbport_search_by_bow_kf_f(const orbport_kp* kf_keys, const uint8_t* kf_desc, const uint8_t* kf_has_mp, int kf_n, int kf_nn,
                               const uint32_t* kf_node, const int32_t* kf_start, const uint32_t* kf_idx, const orbport_kp* f_keys,
                               const uint8_t* f_desc, int f_n, int f_nn, const uint32_t* f_node, const int32_t* f_start,
                               const uint32_t* f_idx, float nnratio, int check_ori, int32_t* match_f) {
    (void)kf_n;
    for (int i = 0; i < f_n; i++) match_f[i] = -1;
    int nmatches = 0;
    std::vector<int> rotHist[HISTO_LENGTH];
    int a = 0, b = 0;
    while (a < kf_nn && b < f_nn) {
        if (kf_node[a] == f_node[b]) {
            for (int iKF = kf_start[a]; iKF < kf_start[a + 1]; iKF++) {
                const unsigned realIdxKF = kf_idx[iKF];
                if (!kf_has_mp[realIdxKF]) continue;
                const uint8_t* dKF = kf_desc + (size_t)realIdxKF * 32;
                int bestDist1 = 256, bestIdxF = -1, bestDist2 = 256;
                for (int iF = f_start[b]; iF < f_start[b + 1]; iF++) {
                    const unsigned realIdxF = f_idx[iF];
                    if (match_f[realIdxF] >= 0) continue;
                    const int dist = orbport_hamming(dKF, f_desc + (size_t)realIdxF * 32);
                    if (dist < bestDist1) { bestDist2 = bestDist1; bestDist1 = dist; bestIdxF = realIdxF; }
                    else if (dist < bestDist2) bestDist2 = dist;
                }
                if (bestDist1 <= TH_LOW) {
                    if ((float)bestDist1 < nnratio * (float)bestDist2) {
                        match_f[bestIdxF] = (int)realIdxKF;
                        if (check_ori) rotHist[rot_bin(kf_keys[realIdxKF].angle, f_keys[bestIdxF].angle)].push_back(bestIdxF);
                        nmatches++;
                    }
                }
            }
            a++; b++;
        } else if (kf_node[a] < f_node[b]) {
            a = (int)(std::lower_bound(kf_node, kf_node + kf_nn, f_node[b]) - kf_node);
        } else {
            b = (int)(std::lower_bound(f_node, f_node + f_nn, kf_node[a]) - f_node);
        }
    }
    if (check_ori) {
        int ind1 = -1, ind2 = -1, ind3 = -1;
        three_maxima(rotHist, HISTO_LENGTH, ind1, ind2, ind3);
        for (int i = 0; i < HISTO_LENGTH; i++) {
            if (i == ind1 || i == ind2 || i == ind3) continue;
            for (int j : rotHist[i]) { match_f[j] = -1; nmatches--; }
        }
    }
    return nmatches;
}

// SearchByBoW(KeyFrame*, KeyFrame*): match12[kf1.N] = index in KF2 or -1.
int orbport_search_by_bow_kf_kf(const orbport_kp* k1, const uint8_t* d1, const uint8_t* has_mp1, int n1, int nn1, const uint32_t* node1,
                                const int32_t* start1, const uint32_t* idx1, const orbport_kp* k2, const uint8_t* d2,
                                const uint8_t* has_mp2, int n2, int nn2, const uint32_t* node2, const int32_t* start2,
                                const uint32_t* idx2, float nnratio, int check_ori, int32_t* match12) {
    for (int i = 0; i < n1; i++) match12[i] = -1;
    std::vector<char> vbMatched2(n2, 0);
    std::vector<int> rotHist[HISTO_LENGTH];
    int nmatches = 0, a = 0, b = 0;
    while (a < nn1 && b < nn2) {
        if (node1[a] == node2[b]) {
            for (int i1 = start1[a]; i1 < start1[a + 1]; i1++) {
                const unsigned i = idx1[i1];
                if (!has_mp1[i]) continue;
                int bestDist1 = 256, bestIdx2 = -1, bestDist2 = 256;
                for (int i2 = start2[b]; i2 < start2[b + 1]; i2++) {
                    const unsigned j = idx2[i2];
                    if (vbMatched2[j] || !has_mp2[j]) continue;
                    const int dist = orbport_hamming(d1 + (size_t)i * 32, d2 + (size_t)j * 32);
                    if (dist < bestDist1) { bestDist2 = bestDist1; bestDist1 = dist; bestIdx2 = j; }
                    else if (dist < bestDist2) bestDist2 = dist;
                }
                if (bestDist1 < TH_LOW) {
                    if ((float)bestDist1 < nnratio * (float)bestDist2) {
                        match12[i] = bestIdx2;
                        vbMatched2[bestIdx2] = 1;
                        if (check_ori) rotHist[rot_bin(k1[i].angle, k2[bestIdx2].angle)].push_back(i);
                        nmatches++;
                    }
                }
            }
            a++; b++;
        } else if (node1[a] < node2[b]) {
            a = (int)(std::lower_bound(node1, node1 + nn1, node2[b]) - node1);
        } else {
            b = (int)(std::lower_bound(node2, node2 + nn2, node1[a]) - node2);
        }
    }
    if (check_ori) {
        int ind1 = -1, ind2 = -1, ind3 = -1;
        three_maxima(rotHist, HISTO_LENGTH, ind1, ind2, ind3);
        for (int i = 0; i < HISTO_LENGTH; i++) {
            if (i == ind1 || i == ind2 || i == ind3) continue;
            for (int j : rotHist[i]) { match12[j] = -1; nmatches--; }
        }
    }
    return nmatches;
}

// SearchForTriangulation: pairs[2*m] (idx1, idx2) ascending idx1; returns m.  ex,ey: epipole of KF1's centre in KF2
// (ORBmatcher.cc:663-670, computed by the caller); F12 row-major 3x3; sf2/sigma2_2: KF2's mvScaleFactors / mvLevelSigma2.
int orbport_search_for_triangulation(const orbport_kp* k1, const uint8_t* d1, const uint8_t* has_mp1, const float* ur1, int n1, int nn1,
                                     const uint32_t* node1, const int32_t* start1, const uint32_t* idx1, const orbport_kp* k2,
                                     const uint8_t* d2, const uint8_t* has_mp2, const float* ur2, int n2, int nn2, const uint32_t* node2,
                                     const int32_t* start2, const uint32_t* idx2, const float* F12, float ex, float ey,
                                     const float* sf2, const float* sigma2_2, int only_stereo, int check_ori, int32_t* pairs) {
    (void)n2;
    int nmatches = 0;
    std::vector<int> vMatches12(n1, -1);
    std::vector<int> rotHist[HISTO_LENGTH];
    int a = 0, b = 0;
    while (a < nn1 && b < nn2) {
        if (node1[a] == node2[b]) {
            for (int i1 = start1[a]; i1 < start1[a + 1]; i1++) {
                const unsigned i = idx1[i1];
                if (has_mp1[i]) continue;
                const bool bStereo1 = ur1 && ur1[i] >= 0;
                if (only_stereo && !bStereo1) continue;
                const orbport_kp& kp1 = k1[i];
                int bestDist = TH_LOW, bestIdx2 = -1;
                for (int i2 = start2[b]; i2 < start2[b + 1]; i2++) {
                    const unsigned j = idx2[i2];
                    if (has_mp2[j]) continue;             // vbMatched2 is never set in the reference (:677,:725)
                    const bool bStereo2 = ur2 && ur2[j] >= 0;
                    if (only_stereo && !bStereo2) continue;
                    const int dist = orbport_hamming(d1 + (size_t)i * 32, d2 + (size_t)j * 32);
                    if (dist > TH_LOW || dist > bestDist) continue;
                    const orbport_kp& kp2 = k2[j];
                    if (!bStereo1 && !bStereo2) {
                        const float distex = ex - kp2.x, distey = ey - kp2.y;
                        if (distex * distex + distey * distey < 100 * sf2[kp2.octave]) continue;
                    }
                    // CheckDistEpipolarLine (:140-157)
                    const float la = kp1.x * F12[0] + kp1.y * F12[3] + F12[6];
                    const float lb = kp1.x * F12[1] + kp1.y * F12[4] + F12[7];
                    const float lc = kp1.x * F12[2] + kp1.y * F12[5] + F12[8];
                    const float num = la * kp2.x + lb * kp2.y + lc;
                    const float den = la * la + lb * lb;
                    if (den == 0) continue;
                    const float dsqr = num * num / den;
                    if (dsqr < 3.84 * sigma2_2[kp2.octave]) { bestIdx2 = j; bestDist = dist; }
                }
                if (bestIdx2 >= 0) {
                    vMatches12[i] = bestIdx2;
                    nmatches++;
                    if (check_ori) rotHist[rot_bin(kp1.angle, k2[bestIdx2].angle)].push_back(i);
                }
            }
            a++; b++;
        } else if (node1[a] < node2[b]) {
            a = (int)(std::lower_bound(node1, node1 + nn1, node2[b]) - node1);
        } else {
            b = (int)(std::lower_bound(node2, node2 + nn2, node1[a]) - node2);
        }
    }
    if (check_ori) {
        int ind1 = -1, ind2 = -1, ind3 = -1;
        three_maxima(rotHist, HISTO_LENGTH, ind1, ind2, ind3);
        for (int i = 0; i < HISTO_LENGTH; i++) {
            if (i == ind1 || i == ind2 || i == ind3) continue;
            for (int j : rotHist[i]) { vMatches12[j] = -1; nmatches--; }
        }
    }
    int m = 0;
    for (int i = 0; i < n1; i++) {
        if (vMatches12[i] < 0) continue;
        pairs[2 * m] = i; pairs[2 * m + 1] = vMatches12[i];
        m++;
    }
    return m;
}

// ------------------------------------------------------------------------------------------ vocabulary
struct OVoc {
    int k, L;
    std::vector<int> parent;                 // node 0 = root
    std::vector<std::vector<int>> children;
    std::vector<uint8_t> desc;               // nodes x 32
    std::vector<double> weight;
    std::vector<int> word_id;                // -1 for inner nodes
    std::vector<char> leaf;
};

static void voc_add(OVoc* v, int pid, bool leaf, const uint8_t* d, double w, int& nwords) {
    const int nid = (int)v->parent.size();
    v->parent.push_back(pid);
    v->children.emplace_back();
    v->children[pid].push_back(nid);
    v->desc.insert(v->desc.end(), d, d + 32);
    v->weight.push_back(w);
    v->leaf.push_back(leaf);
    v->word_id.push_back(leaf ? nwords++ : -1);
}

static OVoc* voc_new(int k, int L) {
    OVoc* v = new OVoc();
    v->k = k; v->L = L;
    v->parent.push_back(0); v->children.emplace_back(); v->desc.assign(32, 0); v->weight.push_back(0); v->leaf.push_back(0); v->word_id.push_back(-1);
    return v;
}

// Text format of Vocabulary/ORBvoc.txt (TemplatedVocabulary.h:1338-1424): "k L scoring weighting", then one line per
// node "parent isLeaf d0..d31 weight".  (The reference's `while(!f.eof())` also turns a trailing empty line into a
// garbage child of the root; that artefact is not reproduced.)
void* orbport_voc_load_text(const char* path) {
    // plain C stdio (this library may be linked with a static libstdc++, whose iostreams must not be used from a dlopen'ed .so)
    FILE* f = std::fopen(path, "r");
    if (!f) return nullptr;
    std::vector<char> line(1 << 16);
    if (!std::fgets(line.data(), (int)line.size(), f)) { std::fclose(f); return nullptr; }
    int k = -1, L = -1, n1 = -1, n2 = -1;
    if (std::sscanf(line.data(), "%d %d %d %d", &k, &L, &n1, &n2) != 4 || k < 0 || k > 20 || L < 1 || L > 10 || n1 < 0 || n1 > 5 || n2 < 0 || n2 > 3) {
        std::fclose(f);
        return nullptr;
    }
    OVoc* v = voc_new(k, L);
    int nwords = 0;
    while (std::fgets(line.data(), (int)line.size(), f)) {
        char* p = line.data();
        char* end = nullptr;
        const long pid = std::strtol(p, &end, 10);
        if (end == p) continue;                       // blank line
        p = end;
        const long isLeaf = std::strtol(p, &end, 10); p = end;
        uint8_t d[32];
        for (int i = 0; i < 32; i++) { d[i] = (uint8_t)std::strtol(p, &end, 10); p = end; }
        const double w = std::strtod(p, &end);
        voc_add(v, (int)pid, isLeaf > 0, d, w, nwords);
    }
    std::fclose(f);
    return v;
}

// Seeded random tree of ORBvoc's shape (k children per inner node, L levels, leaves at depth L).
void* orbport_voc_random(int k, int L, unsigned seed) {
    OVoc* v = voc_new(k, L);
    std::mt19937 rng(seed);
    int nwords = 0;
    std::vector<int> frontier = {0};
    for (int depth = 1; depth <= L; depth++) {
        std::vector<int> next;
        for (int p : frontier)
            for (int c = 0; c < k; c++) {
                uint8_t d[32];
                for (int i = 0; i < 32; i += 4) { uint32_t r = rng(); std::memcpy(d + i, &r, 4); }
                const double w = depth == L ? 0.5 + (rng() % 100000) / 10000.0 : 0.0;
                next.push_back((int)v->parent.size());
                voc_add(v, p, depth == L, d, w, nwords);
            }
        frontier.swap(next);
    }
    return v;
}

void orbport_voc_free(void* h) { delete (OVoc*)h; }
int orbport_voc_nodes(void* h) { return (int)((OVoc*)h)->parent.size(); }
// flat export (nodes in id order): parent, is_leaf, word_id, descriptor, weight
void orbport_voc_export(void* h, int32_t* parent, uint8_t* is_leaf, int32_t* word_id, uint8_t* desc, double* weight, int* k, int* L) {
    OVoc* v = (OVoc*)h;
    const int n = (int)v->parent.size();
    for (int i = 0; i < n; i++) { parent[i] = v->parent[i]; is_leaf[i] = v->leaf[i]; word_id[i] = v->word_id[i]; weight[i] = v->weight[i]; }
    std::memcpy(desc, v->desc.data(), (size_t)n * 32);
    *k = v->k; *L = v->L;
}

// transform(feature, word_id, weight, nid, levelsup) for n features (TemplatedVocabulary.h:1218-1259)
void orbport_voc_transform(void* h, const uint8_t* desc, int n, int levelsup, int32_t* word, double* weight, int32_t* node) {
    OVoc* v = (OVoc*)h;
    const int nid_level = v->L - levelsup;
    for (int f = 0; f < n; f++) {
        const uint8_t* feat = desc + (size_t)f * 32;
        int nid = 0;
        if (nid_level <= 0) nid = 0;
        int final_id = 0, current_level = 0;
        do {
            ++current_level;
            const std::vector<int>& nodes = v->children[final_id];
            final_id = nodes[0];
            double best_d = orbport_hamming(feat, &v->desc[(size_t)final_id * 32]);
            for (size_t c = 1; c < nodes.size(); c++) {
                const double d = orbport_hamming(feat, &v->desc[(size_t)nodes[c] * 32]);
                if (d < best_d) { best_d = d; final_id = nodes[c]; }
            }
            if (current_level == nid_level) nid = final_id;
        } while (!v->leaf[final_id]);
        word[f] = v->word_id[final_id];
        weight[f] = v->weight[final_id];
        node[f] = nid;
    }
}

double orbport_bow_score_l1(const uint32_t* w1, const double* v1, int n1, const uint32_t* w2, const double* v2, int n2, int32_t* common, uint32_t* first);

// TemplatedVocabulary::transform(features, BowVector&, FeatureVector&, levelsup) (TemplatedVocabulary.h:1127-1194) for TF-IDF / L1:
// std::map bookkeeping as the reference does it, flattened to arrays (words ascending; nodes ascending, features in order).
void orbport_compute_bow(void* h, const uint8_t* desc, int n, int levelsup, uint32_t* bow_word, double* bow_value, int32_t* n_bow,
                         uint32_t* fv_node, int32_t* fv_start, uint32_t* fv_idx, int32_t* n_nodes) {
    std::vector<int32_t> word(n > 0 ? n : 1), node(n > 0 ? n : 1);
    std::vector<double> weight(n > 0 ? n : 1);
    orbport_voc_transform(h, desc, n, levelsup, word.data(), weight.data(), node.data());
    std::map<uint32_t, double> bow;
    std::map<uint32_t, std::vector<uint32_t>> fv;
    for (int i = 0; i < n; i++)
        if (weight[i] > 0) {
            auto it = bow.lower_bound((uint32_t)word[i]);                         // BowVector::addWeight
            if (it != bow.end() && !(bow.key_comp()((uint32_t)word[i], it->first))) it->second += weight[i];
            else bow.insert(it, std::make_pair((uint32_t)word[i], weight[i]));
            fv[(uint32_t)node[i]].push_back((uint32_t)i);                         // FeatureVector::addFeature
        }
    double norm = 0.0;                                                            // BowVector::normalize(L1)
    for (auto& kv : bow) norm += std::fabs(kv.second);
    if (norm > 0.0) for (auto& kv : bow) kv.second /= norm;
    int nb = 0;
    for (auto& kv : bow) { bow_word[nb] = kv.first; bow_value[nb] = kv.second; nb++; }
    int nn = 0, pos = 0;
    fv_start[0] = 0;
    for (auto& kv : fv) {
        fv_node[nn] = kv.first;
        for (uint32_t f : kv.second) fv_idx[pos++] = f;
        fv_start[++nn] = pos;
    }
    *n_bow = nb; *n_nodes = nn;
}

// the scoring loop of KeyFrameDatabase::Detect*Candidates (src/KeyFrameDatabase.cc:127,:240) over n_kf keyframes whose BowVectors
// are concatenated (offsets kf_off[n_kf + 1]): float si = mpVoc->score(query, kf)
void orbport_bow_score_sweep(const uint32_t* q_word, const double* q_value, int nq, const uint32_t* kf_word, const double* kf_value,
                             const int32_t* kf_off, int n_kf, float* score, int32_t* common) {
    for (int k = 0; k < n_kf; k++) {
        int32_t c = 0; uint32_t first = 0;
        score[k] = (float)orbport_bow_score_l1(q_word, q_value, nq, kf_word + kf_off[k], kf_value + kf_off[k], kf_off[k + 1] - kf_off[k], &c, &first);
        if (common) common[k] = c;
    }
}

}  // extern "C"

// ORBmatcher::SearchByProjection(Frame &CurrentFrame, const Frame &LastFrame, th, bMono) — src/ORBmatcher.cc:1328-1470.
// world_pos: x3Dw of LastFrame.mvpMapPoints[i] (n_last x 3); valid[i] = pMP && !mvbOutlier[i]; has_obs[i] = pMP->Observations()>0;
// Tcw: CurrentFrame.mTcw rows 0..2 (3x4 row-major).  forward/backward: the bForward / bBackward flags of :1348-1349
// (computed by the caller from the two poses).  cv::Mat products are float32 (r0*p0 + r1*p1) + r2*p2, then + t (SURVEY §8 a13).
// state_cur[i2]: >=0 index of the LastFrame feature whose MapPoint ended up in CurrentFrame.mvpMapPoints[i2]; -1 untouched;
// -2 set to NULL by the rotation-consistency cull (:1456-1466).
extern "C" int orbport_search_by_projection_last(const orbport_kp* cur_keys_un, const uint8_t* cur_desc, const float* cur_u_right,
                                                 const uint8_t* cur_occupied, int n_cur, float minX, float minY, float maxX, float maxY,
                                                 const float* scale_factors, const orbport_kp* last_keys, const float* world_pos,
                                                 const uint8_t* last_desc, const uint8_t* valid, const uint8_t* has_obs, int n_last,
                                                 const float* Tcw, float fx, float fy, float cx, float cy, float bf, float th, int forward,
                                                 int backward, int check_ori, int32_t* state_cur) {
    Grid g = build_grid(cur_keys_un, n_cur, minX, minY, maxX, maxY);
    std::vector<char> held(n_cur, 0);
    for (int i = 0; i < n_cur; i++) { held[i] = cur_occupied ? (cur_occupied[i] != 0) : 0; state_cur[i] = -1; }
    int nmatches = 0;
    std::vector<int> rotHist[HISTO_LENGTH];
    for (int i = 0; i < n_last; i++) {
        if (valid && !valid[i]) continue;
        const float* P = world_pos + 3 * (size_t)i;
        const float xc = ((Tcw[0] * P[0] + Tcw[1] * P[1]) + Tcw[2] * P[2]) + Tcw[3];
        const float yc = ((Tcw[4] * P[0] + Tcw[5] * P[1]) + Tcw[6] * P[2]) + Tcw[7];
        const float zc = ((Tcw[8] * P[0] + Tcw[9] * P[1]) + Tcw[10] * P[2]) + Tcw[11];
        const float invzc = 1.0 / zc;
        if (invzc < 0) continue;
        const float u = fx * xc * invzc + cx;
        const float v = fy * yc * invzc + cy;
        if (u < minX || u > maxX) continue;
        if (v < minY || v > maxY) continue;
        const int nLastOctave = last_keys[i].octave;
        const float radius = th * scale_factors[nLastOctave];
        std::vector<int> vIndices2;
        if (forward) vIndices2 = features_in_area(g, cur_keys_un, u, v, radius, nLastOctave, -1);
        else if (backward) vIndices2 = features_in_area(g, cur_keys_un, u, v, radius, 0, nLastOctave);
        else vIndices2 = features_in_area(g, cur_keys_un, u, v, radius, nLastOctave - 1, nLastOctave + 1);
        if (vIndices2.empty()) continue;
        const uint8_t* dMP = last_desc + (size_t)i * 32;
        int bestDist = 256, bestIdx2 = -1;
        for (int i2 : vIndices2) {
            if (held[i2]) continue;
            if (cur_u_right && cur_u_right[i2] > 0) {
                const float ur = u - bf * invzc;
                const float er = std::fabs(ur - cur_u_right[i2]);
                if (er > radius) continue;
            }
            const int dist = orbport_hamming(dMP, cur_desc + (size_t)i2 * 32);
            if (dist < bestDist) { bestDist = dist; bestIdx2 = i2; }
        }
        if (bestDist <= TH_HIGH) {
            state_cur[bestIdx2] = i;
            held[bestIdx2] = has_obs ? (has_obs[i] != 0) : 1;
            nmatches++;
            if (check_ori) rotHist[rot_bin(last_keys[i].angle, cur_keys_un[bestIdx2].angle)].push_back(bestIdx2);
        }
    }
    if (check_ori) {
        int ind1 = -1, ind2 = -1, ind3 = -1;
        three_maxima(rotHist, HISTO_LENGTH, ind1, ind2, ind3);
        for (int i = 0; i < HISTO_LENGTH; i++)
            if (i != ind1 && i != ind2 && i != ind3)
                for (int j : rotHist[i]) { state_cur[j] = -2; nmatches--; }
    }
    return nmatches;
}

// ---------------------------------------------------------------------------------------------------------------
// MapPoint::PredictScale (reference src/MapPoint.cc:385-417): log/ceil resolve to the float overloads
// (TemplatedVocabulary.h:36 puts `using namespace std` in scope), i.e. glibc logf.
static int predict_scale(float mfMaxDistance, float currentDist, float logScaleFactor, int nScaleLevels) {
    const float ratio = mfMaxDistance / currentDist;
    int nScale = (int)std::ceil(std::log(ratio) / logScaleFactor);
    if (nScale < 0) nScale = 0;
    else if (nScale >= nScaleLevels) nScale = nScaleLevels - 1;
    return nScale;
}
// cv::norm(3x1 CV_32F) (NORM_L2): squares accumulated in double in index order, sqrt in double, result narrowed by the caller
static float norm3(const float* v) {
    double s = 0;
    for (int i = 0; i < 3; i++) { const double d = v[i]; s += d * d; }
    return (float)std::sqrt(s);
}
// cv::Mat::dot of two 3x1 CV_32F: products and sum in double, index order
static double dot3(const float* a, const float* b) {
    double s = 0;
    for (int i = 0; i < 3; i++) s += (double)a[i] * b[i];
    return s;
}

// ORBmatcher::SearchByProjection(Frame &CurrentFrame, KeyFrame *pKF, const set<MapPoint*> &sAlreadyFound, th, ORBdist)
// reference src/ORBmatcher.cc:1472-1599 (Tracking::Relocalization, src/Tracking.cc:1396,1410).
// Query i = pKF->GetMapPointMatches()[i]; valid[i] = pMP && !pMP->isBad() && !sAlreadyFound.count(pMP);
// cur_occupied[i2] = CurrentFrame.mvpMapPoints[i2] != NULL; Ow = -Rcw.t()*tcw computed by the caller (:1478).
extern "C" int orbport_search_by_projection_kf(const orbport_kp* cur_keys_un, const uint8_t* cur_desc, const uint8_t* cur_occupied, int n_cur,
                                               float minX, float minY, float maxX, float maxY, const float* scale_factors, int n_levels,
                                               float log_scale_factor, const float* kf_angle, const float* world_pos, const uint8_t* mp_desc,
                                               const float* max_distance, const float* min_distance, const uint8_t* valid, int n_q,
                                               const float* Tcw, const float* Ow, float fx, float fy, float cx, float cy, float th,
                                               int ORBdist, int check_ori, int32_t* state_cur) {
    Grid g = build_grid(cur_keys_un, n_cur, minX, minY, maxX, maxY);
    std::vector<char> held(n_cur, 0);
    for (int i = 0; i < n_cur; i++) { held[i] = cur_occupied ? (cur_occupied[i] != 0) : 0; state_cur[i] = -1; }
    int nmatches = 0;
    std::vector<int> rotHist[HISTO_LENGTH];
    for (int i = 0; i < n_q; i++) {
        if (valid && !valid[i]) continue;
        const float* P = world_pos + 3 * (size_t)i;
        const float xc = ((Tcw[0] * P[0] + Tcw[1] * P[1]) + Tcw[2] * P[2]) + Tcw[3];
        const float yc = ((Tcw[4] * P[0] + Tcw[5] * P[1]) + Tcw[6] * P[2]) + Tcw[7];
        const float zc = ((Tcw[8] * P[0] + Tcw[9] * P[1]) + Tcw[10] * P[2]) + Tcw[11];
        const float invzc = 1.0 / zc;
        const float u = fx * xc * invzc + cx;
        const float v = fy * yc * invzc + cy;
        if (u < minX || u > maxX) continue;
        if (v < minY || v > maxY) continue;
        if (!(u == u) || !(v == v)) continue;                 // NaN would index the grid with an undefined int in the reference
        const float PO[3] = {P[0] - Ow[0], P[1] - Ow[1], P[2] - Ow[2]};
        const float dist3D = norm3(PO);
        const float maxDistance = 1.2f * max_distance[i];     // MapPoint::GetMaxDistanceInvariance (MapPoint.cc:379-383)
        const float minDistance = 0.8f * min_distance[i];     // GetMinDistanceInvariance (:373-377)
        if (dist3D < minDistance || dist3D > maxDistance) continue;
        const int nPredictedLevel = predict_scale(max_distance[i], dist3D, log_scale_factor, n_levels);
        const float radius = th * scale_factors[nPredictedLevel];
        const std::vector<int> vIndices2 = features_in_area(g, cur_keys_un, u, v, radius, nPredictedLevel - 1, nPredictedLevel + 1);
        if (vIndices2.empty()) continue;
        const uint8_t* dMP = mp_desc + (size_t)i * 32;
        int bestDist = 256, bestIdx2 = -1;
        for (int i2 : vIndices2) {
            if (held[i2]) continue;
            const int dist = orbport_hamming(dMP, cur_desc + (size_t)i2 * 32);
            if (dist < bestDist) { bestDist = dist; bestIdx2 = i2; }
        }
        if (bestDist <= ORBdist) {
            state_cur[bestIdx2] = i;
            held[bestIdx2] = 1;
            nmatches++;
            if (check_ori) rotHist[rot_bin(kf_angle[i], cur_keys_un[bestIdx2].angle)].push_back(bestIdx2);
        }
    }
    if (check_ori) {
        int ind1 = -1, ind2 = -1, ind3 = -1;
        three_maxima(rotHist, HISTO_LENGTH, ind1, ind2, ind3);
        for (int i = 0; i < HISTO_LENGTH; i++)
            if (i != ind1 && i != ind2 && i != ind3)
                for (int j : rotHist[i]) { state_cur[j] = -2; nmatches--; }
    }
    return nmatches;
}

// ORBmatcher::SearchByProjection(KeyFrame* pKF, cv::Mat Scw, const vector<MapPoint*> &vpPoints, vector<MapPoint*> &vpMatched, int th)
// reference src/ORBmatcher.cc:290-403 (LoopClosing::ComputeSim3, src/LoopClosing.cc:391).
// Tcw = [Rcw | tcw] AFTER the scale has been divided out (:299-302), Ow = -Rcw.t()*tcw (:303): the caller's cv::Mat
// lines. valid[i] = !vpPoints[i]->isBad() && !spAlreadyFound.count(vpPoints[i]); kf_matched[idx] = vpMatched[idx] != NULL.
// state_kf[idx] = index into vpPoints of the point now in vpMatched[idx], -1 = untouched.
extern "C" int orbport_search_by_projection_sim3(const orbport_kp* kf_keys_un, const uint8_t* kf_desc, const uint8_t* kf_matched, int n_kf,
                                                 float minX, float minY, float maxX, float maxY, const float* scale_factors, int n_levels,
                                                 float log_scale_factor, const float* world_pos, const uint8_t* mp_desc,
                                                 const float* max_distance, const float* min_distance, const float* normal,
                                                 const uint8_t* valid, int n_q, const float* Tcw, const float* Ow, float fx, float fy,
                                                 float cx, float cy, int th, int32_t* state_kf) {
    Grid g = build_grid(kf_keys_un, n_kf, minX, minY, maxX, maxY);
    std::vector<char> held(n_kf, 0);
    for (int i = 0; i < n_kf; i++) { held[i] = kf_matched ? (kf_matched[i] != 0) : 0; state_kf[i] = -1; }
    int nmatches = 0;
    for (int iMP = 0; iMP < n_q; iMP++) {
        if (valid && !valid[iMP]) continue;
        const float* P = world_pos + 3 * (size_t)iMP;
        const float p3Dc[3] = {((Tcw[0] * P[0] + Tcw[1] * P[1]) + Tcw[2] * P[2]) + Tcw[3],
                               ((Tcw[4] * P[0] + Tcw[5] * P[1]) + Tcw[6] * P[2]) + Tcw[7],
                               ((Tcw[8] * P[0] + Tcw[9] * P[1]) + Tcw[10] * P[2]) + Tcw[11]};
        if (p3Dc[2] < 0.0) continue;
        const float invz = 1 / p3Dc[2];
        const float x = p3Dc[0] * invz;
        const float y = p3Dc[1] * invz;
        const float u = fx * x + cx;
        const float v = fy * y + cy;
        if (!(u >= minX && u < maxX && v >= minY && v < maxY)) continue;       // KeyFrame::IsInImage (KeyFrame.cc:610-613)
        const float maxDistance = 1.2f * max_distance[iMP];
        const float minDistance = 0.8f * min_distance[iMP];
        const float PO[3] = {P[0] - Ow[0], P[1] - Ow[1], P[2] - Ow[2]};
        const float dist = norm3(PO);
        if (dist < minDistance || dist > maxDistance) continue;
        if (dot3(PO, normal + 3 * (size_t)iMP) < 0.5 * dist) continue;          // viewing angle < 60 deg (:354-357)
        const int nPredictedLevel = predict_scale(max_distance[iMP], dist, log_scale_factor, n_levels);
        const float radius = th * scale_factors[nPredictedLevel];
        const std::vector<int> vIndices = features_in_area(g, kf_keys_un, u, v, radius, -1, -1);   // KeyFrame::GetFeaturesInArea: no levels
        if (vIndices.empty()) continue;
        const uint8_t* dMP = mp_desc + (size_t)iMP * 32;
        int bestDist = 256, bestIdx = -1;
        for (int idx : vIndices) {
            if (held[idx]) continue;
            const int kpLevel = kf_keys_un[idx].octave;
            if (kpLevel < nPredictedLevel - 1 || kpLevel > nPredictedLevel) continue;
            const int dist2 = orbport_hamming(dMP, kf_desc + (size_t)idx * 32);
            if (dist2 < bestDist) { bestDist = dist2; bestIdx = idx; }
        }
        if (bestDist <= TH_LOW) {
            state_kf[bestIdx] = iMP;
            held[bestIdx] = 1;
            nmatches++;
        }
    }
    return nmatches;
}

// ---------------------------------------------------------------------------------------------------------------
// ORBmatcher::Fuse(KeyFrame *pKF, const vector<MapPoint *> &vpMapPoints, const float th) — reference
// src/ORBmatcher.cc:825-970 (LocalMapping::SearchInNeighbors, src/LocalMapping.cc:483-511), and
// ORBmatcher::Fuse(KeyFrame *pKF, cv::Mat Scw, vpPoints, th, vpReplacePoint) — :972-1100 (LoopClosing::SearchAndFuse).
// The search part only: best_idx[i] = keyframe feature selected for point i (bestDist <= TH_LOW), else -1.  The map
// mutation that follows (:947-966 / :1077-1090: Replace / AddObservation / AddMapPoint) does not feed back into the
// search of later points except through `isBad()` / `IsInKeyFrame()` of a point that occurs twice in the list; the
// adapter applies best_idx in order and re-evaluates those two tests when it does.
// scw_variant = 0: invz = 1/z in float, stereo/mono reprojection gates (7.8 / 5.99); 1: invz = 1.0/z, no gates.
extern "C" int orbport_fuse(const orbport_kp* kf_keys_un, const uint8_t* kf_desc, const float* kf_u_right, const float* inv_level_sigma2,
                            int n_kf, float minX, float minY, float maxX, float maxY, const float* scale_factors, int n_levels,
                            float log_scale_factor, const float* world_pos, const uint8_t* mp_desc, const float* max_distance,
                            const float* min_distance, const float* normal, const uint8_t* valid, int n_q, const float* Tcw,
                            const float* Ow, float fx, float fy, float cx, float cy, float bf, float th, int scw_variant,
                            int32_t* best_idx) {
    Grid g = build_grid(kf_keys_un, n_kf, minX, minY, maxX, maxY);
    int nFound = 0;
    for (int i = 0; i < n_q; i++) {
        best_idx[i] = -1;
        if (valid && !valid[i]) continue;
        const float* P = world_pos + 3 * (size_t)i;
        const float p3Dc[3] = {((Tcw[0] * P[0] + Tcw[1] * P[1]) + Tcw[2] * P[2]) + Tcw[3],
                               ((Tcw[4] * P[0] + Tcw[5] * P[1]) + Tcw[6] * P[2]) + Tcw[7],
                               ((Tcw[8] * P[0] + Tcw[9] * P[1]) + Tcw[10] * P[2]) + Tcw[11]};
        if (p3Dc[2] < 0.0f) continue;
        float invz;
        if (scw_variant) invz = 1.0 / p3Dc[2]; else invz = 1 / p3Dc[2];
        const float x = p3Dc[0] * invz;
        const float y = p3Dc[1] * invz;
        const float u = fx * x + cx;
        const float v = fy * y + cy;
        if (!(u >= minX && u < maxX && v >= minY && v < maxY)) continue;
        const float ur = u - bf * invz;
        const float maxDistance = 1.2f * max_distance[i];
        const float minDistance = 0.8f * min_distance[i];
        const float PO[3] = {P[0] - Ow[0], P[1] - Ow[1], P[2] - Ow[2]};
        const float dist3D = norm3(PO);
        if (dist3D < minDistance || dist3D > maxDistance) continue;
        if (dot3(PO, normal + 3 * (size_t)i) < 0.5 * dist3D) continue;
        const int nPredictedLevel = predict_scale(max_distance[i], dist3D, log_scale_factor, n_levels);
        const float radius = th * scale_factors[nPredictedLevel];
        const std::vector<int> vIndices = features_in_area(g, kf_keys_un, u, v, radius, -1, -1);
        if (vIndices.empty()) continue;
        const uint8_t* dMP = mp_desc + (size_t)i * 32;
        int bestDist = 256, bestIdx = -1;
        for (int idx : vIndices) {
            const orbport_kp& kp = kf_keys_un[idx];
            const int kpLevel = kp.octave;
            if (kpLevel < nPredictedLevel - 1 || kpLevel > nPredictedLevel) continue;
            if (!scw_variant) {
                if (kf_u_right && kf_u_right[idx] >= 0) {
                    const float ex = u - kp.x, ey = v - kp.y, er = ur - kf_u_right[idx];
                    const float e2 = ex * ex + ey * ey + er * er;
                    if (e2 * inv_level_sigma2[kpLevel] > 7.8) continue;
                } else {
                    const float ex = u - kp.x, ey = v - kp.y;
                    const float e2 = ex * ex + ey * ey;
                    if (e2 * inv_level_sigma2[kpLevel] > 5.99) continue;
                }
            }
            const int dist = orbport_hamming(dMP, kf_desc + (size_t)idx * 32);
            if (dist < bestDist) { bestDist = dist; bestIdx = idx; }
        }
        if (bestDist <= TH_LOW) { best_idx[i] = bestIdx; nFound++; }
    }
    return nFound;
}

// One direction of ORBmatcher::SearchBySim3 (:1146-1222 / :1224-1300): MapPoints of keyframe A (world_pos, through
// A's pose Taw then the similarity [sRba | tba]) searched among keyframe B's features.  match[i] = B feature or -1.
static void sim3_direction(const orbport_kp* kB, const uint8_t* dB, int nB, const float* boundsB, const float* sfB, int n_levels,
                           float log_scale, const float* world_pos, const uint8_t* mp_desc, const float* max_distance,
                           const float* min_distance, const uint8_t* valid, int nA, const float* Taw, const float* Sba, float fx,
                           float fy, float cx, float cy, float th, int32_t* match) {
    Grid g = build_grid(kB, nB, boundsB[0], boundsB[1], boundsB[2], boundsB[3]);
    for (int i = 0; i < nA; i++) {
        match[i] = -1;
        if (valid && !valid[i]) continue;
        const float* P = world_pos + 3 * (size_t)i;
        const float a[3] = {((Taw[0] * P[0] + Taw[1] * P[1]) + Taw[2] * P[2]) + Taw[3],
                            ((Taw[4] * P[0] + Taw[5] * P[1]) + Taw[6] * P[2]) + Taw[7],
                            ((Taw[8] * P[0] + Taw[9] * P[1]) + Taw[10] * P[2]) + Taw[11]};
        const float b[3] = {((Sba[0] * a[0] + Sba[1] * a[1]) + Sba[2] * a[2]) + Sba[3],
                            ((Sba[4] * a[0] + Sba[5] * a[1]) + Sba[6] * a[2]) + Sba[7],
                            ((Sba[8] * a[0] + Sba[9] * a[1]) + Sba[10] * a[2]) + Sba[11]};
        if (b[2] < 0.0) continue;
        const float invz = 1.0 / b[2];
        const float x = b[0] * invz;
        const float y = b[1] * invz;
        const float u = fx * x + cx;
        const float v = fy * y + cy;
        if (!(u >= boundsB[0] && u < boundsB[2] && v >= boundsB[1] && v < boundsB[3])) continue;
        const float maxDistance = 1.2f * max_distance[i];
        const float minDistance = 0.8f * min_distance[i];
        const float dist3D = norm3(b);
        if (dist3D < minDistance || dist3D > maxDistance) continue;
        const int nPredictedLevel = predict_scale(max_distance[i], dist3D, log_scale, n_levels);
        const float radius = th * sfB[nPredictedLevel];
        const std::vector<int> vIndices = features_in_area(g, kB, u, v, radius, -1, -1);
        if (vIndices.empty()) continue;
        const uint8_t* dMP = mp_desc + (size_t)i * 32;
        int bestDist = INT32_MAX, bestIdx = -1;
        for (int idx : vIndices) {
            if (kB[idx].octave < nPredictedLevel - 1 || kB[idx].octave > nPredictedLevel) continue;
            const int dist = orbport_hamming(dMP, dB + (size_t)idx * 32);
            if (dist < bestDist) { bestDist = dist; bestIdx = idx; }
        }
        if (bestDist <= TH_HIGH) match[i] = bestIdx;
    }
}

// ORBmatcher::SearchBySim3(pKF1, pKF2, vpMatches12, s12, R12, t12, th) — reference src/ORBmatcher.cc:1102-1326
// (LoopClosing::ComputeSim3, src/LoopClosing.cc:375-378).  T1w/T2w = keyframe poses (3x4); S12 = [s12*R12 | t12] and
// S21 = [(1/s12)*R12^T | -sR21*t12] as the caller's cv::Mat lines produce them (:1119-1122).
// valid1[i1] = vpMapPoints1[i1] && !vbAlreadyMatched1[i1] && !isBad() (same for 2).  Both projections use pKF1's
// intrinsics (:1105-1108) — replicated.  match12[i1] = index in KF2 of the agreed match, else -1.
extern "C" int orbport_search_by_sim3(const orbport_kp* k1, const uint8_t* d1, int n1, const float* bounds1, const float* sf1,
                                      float log_scale1, const orbport_kp* k2, const uint8_t* d2, int n2, const float* bounds2,
                                      const float* sf2, float log_scale2, int n_levels, const float* wp1, const uint8_t* md1,
                                      const float* max1, const float* min1, const uint8_t* valid1, const float* wp2,
                                      const uint8_t* md2, const float* max2, const float* min2, const uint8_t* valid2,
                                      const float* T1w, const float* T2w, const float* S12, const float* S21, float fx, float fy,
                                      float cx, float cy, float th, int32_t* match12) {
    std::vector<int32_t> vnMatch1(n1 > 0 ? n1 : 1, -1), vnMatch2(n2 > 0 ? n2 : 1, -1);
    sim3_direction(k2, d2, n2, bounds2, sf2, n_levels, log_scale2, wp1, md1, max1, min1, valid1, n1, T1w, S21, fx, fy, cx, cy, th, vnMatch1.data());
    sim3_direction(k1, d1, n1, bounds1, sf1, n_levels, log_scale1, wp2, md2, max2, min2, valid2, n2, T2w, S12, fx, fy, cx, cy, th, vnMatch2.data());
    int nFound = 0;
    for (int i1 = 0; i1 < n1; i1++) {
        match12[i1] = -1;
        const int idx2 = vnMatch1[i1];
        if (idx2 >= 0) {
            const int idx1 = vnMatch2[idx2];
            if (idx1 == i1) { match12[i1] = idx2; nFound++; }
        }
    }
    return nFound;
}

// ORBmatcher::SearchForInitialization(Frame &F1, Frame &F2, vector<cv::Point2f> &vbPrevMatched, vector<int> &vnMatches12,
// int windowSize) — reference src/ORBmatcher.cc:405-520 (Tracking::MonocularInitialization, src/Tracking.cc:599).
// prev_matched: n1 x 2 floats, updated in place (:513-517).
extern "C" int orbport_search_for_initialization(const orbport_kp* k1, const uint8_t* d1, int n1, const orbport_kp* k2, const uint8_t* d2,
                                                 int n2, float minX, float minY, float maxX, float maxY, float* prev_matched,
                                                 int windowSize, float nnratio, int check_ori, int32_t* vnMatches12) {
    Grid g = build_grid(k2, n2, minX, minY, maxX, maxY);
    int nmatches = 0;
    for (int i = 0; i < n1; i++) vnMatches12[i] = -1;
    std::vector<int> rotHist[HISTO_LENGTH];
    std::vector<int> vMatchedDistance(n2, INT32_MAX);
    std::vector<int> vnMatches21(n2, -1);
    for (int i1 = 0; i1 < n1; i1++) {
        const int level1 = k1[i1].octave;
        if (level1 > 0) continue;
        const std::vector<int> vIndices2 = features_in_area(g, k2, prev_matched[2 * i1], prev_matched[2 * i1 + 1], (float)windowSize, level1, level1);
        if (vIndices2.empty()) continue;
        const uint8_t* dd1 = d1 + (size_t)i1 * 32;
        int bestDist = INT32_MAX, bestDist2 = INT32_MAX, bestIdx2 = -1;
        for (int i2 : vIndices2) {
            const int dist = orbport_hamming(dd1, d2 + (size_t)i2 * 32);
            if (vMatchedDistance[i2] <= dist) continue;
            if (dist < bestDist) { bestDist2 = bestDist; bestDist = dist; bestIdx2 = i2; }
            else if (dist < bestDist2) bestDist2 = dist;
        }
        if (bestDist <= TH_LOW) {
            if (bestDist < (float)bestDist2 * nnratio) {
                if (vnMatches21[bestIdx2] >= 0) { vnMatches12[vnMatches21[bestIdx2]] = -1; nmatches--; }
                vnMatches12[i1] = bestIdx2;
                vnMatches21[bestIdx2] = i1;
                vMatchedDistance[bestIdx2] = bestDist;
                nmatches++;
                if (check_ori) rotHist[rot_bin(k1[i1].angle, k2[bestIdx2].angle)].push_back(i1);
            }
        }
    }
    if (check_ori) {
        int ind1 = -1, ind2 = -1, ind3 = -1;
        three_maxima(rotHist, HISTO_LENGTH, ind1, ind2, ind3);
        for (int i = 0; i < HISTO_LENGTH; i++) {
            if (i == ind1 || i == ind2 || i == ind3) continue;
            for (int idx1 : rotHist[i])
                if (vnMatches12[idx1] >= 0) { vnMatches12[idx1] = -1; nmatches--; }
        }
    }
    for (int i1 = 0; i1 < n1; i1++)
        if (vnMatches12[i1] >= 0) { prev_matched[2 * i1] = k2[vnMatches12[i1]].x; prev_matched[2 * i1 + 1] = k2[vnMatches12[i1]].y; }
    return nmatches;
}

// MapPoint::ComputeDistinctiveDescriptors — reference src/MapPoint.cc:242-307: among the N descriptors observing a
// MapPoint, the one with the least median Hamming distance to the rest (median = sorted row[(int)(0.5*(N-1))], the
// row including the zero self-distance; first minimum wins).  Returns the index, -1 for N == 0.
extern "C" int orbport_distinctive_descriptor(const uint8_t* desc, int N) {
    if (N <= 0) return -1;
    std::vector<std::vector<float>> Distances(N, std::vector<float>(N, 0.f));
    for (int i = 0; i < N; i++) {
        Distances[i][i] = 0;
        for (int j = i + 1; j < N; j++) {
            const int distij = orbport_hamming(desc + (size_t)i * 32, desc + (size_t)j * 32);
            Distances[i][j] = (float)distij;
            Distances[j][i] = (float)distij;
        }
    }
    int BestMedian = INT32_MAX, BestIdx = 0;
    for (int i = 0; i < N; i++) {
        std::vector<int> vDists(Distances[i].begin(), Distances[i].end());
        std::sort(vDists.begin(), vDists.end());
        const int median = vDists[(size_t)(0.5 * (N - 1))];
        if (median < BestMedian) { BestMedian = median; BestIdx = i; }
    }
    return BestIdx;
}

// DBoW2::L1Scoring::score — reference Thirdparty/DBoW2/DBoW2/ScoringObject.cpp:23-71 — on two BowVectors given as
// ascending (word, value) arrays, and the common-word count KeyFrameDatabase::DetectRelocalizationCandidates /
// DetectLoopCandidates accumulate through the inverted file (src/KeyFrameDatabase.cc:211-224, :91-108).
extern "C" double orbport_bow_score_l1(const uint32_t* w1, const double* v1, int n1, const uint32_t* w2, const double* v2, int n2,
                                       int32_t* common_words, uint32_t* first_common_word) {
    double score = 0;
    int i = 0, j = 0, common = 0;
    uint32_t first = 0xFFFFFFFFu;
    while (i < n1 && j < n2) {
        if (w1[i] == w2[j]) {
            const double vi = v1[i], wi = v2[j];
            score += std::fabs(vi - wi) - std::fabs(vi) - std::fabs(wi);
            if (!common) first = w1[i];
            common++; ++i; ++j;
        } else if (w1[i] < w2[j]) {
            i = (int)(std::lower_bound(w1 + i, w1 + n1, w2[j]) - w1);
        } else {
            j = (int)(std::lower_bound(w2 + j, w2 + n2, w1[i]) - w2);
        }
    }
    if (common_words) *common_words = common;
    if (first_common_word) *first_common_word = first;
    return -score / 2.0;
}

// KeyFrameDatabase::add (src/KeyFrameDatabase.cc:41-47) + DetectRelocalizationCandidates (:199-310), restated with a real
// inverted file.  Keyframes 0..n_kf-1 are added in index order; kf_start/kf_word/kf_value = their BowVectors (CSR,
// ascending words); neigh = GetBestCovisibilityKeyFrames(10) per keyframe as n_kf x 10 indices (-1 padded).
// Returns the number of candidates written to out (keyframe indices, in the reference's output order).
extern "C" int orbport_detect_reloc_candidates(int n_kf, const int32_t* kf_start, const uint32_t* kf_word, const double* kf_value,
                                               int n_words, const uint32_t* q_word, const double* q_value, int nq,
                                               const int32_t* neigh, int32_t* out) {
    std::vector<std::vector<int>> mvInvertedFile(n_words);
    for (int k = 0; k < n_kf; k++)
        for (int e = kf_start[k]; e < kf_start[k + 1]; e++) mvInvertedFile[kf_word[e]].push_back(k);
    std::vector<int> mnRelocWords(n_kf, 0);
    std::vector<char> queried(n_kf, 0);          // pKFi->mnRelocQuery == F->mnId
    std::vector<float> mRelocScore(n_kf, 0.f);
    std::vector<int> lKFsSharingWords;
    for (int i = 0; i < nq; i++) {
        if (q_word[i] >= (uint32_t)n_words) continue;
        for (int pKFi : mvInvertedFile[q_word[i]]) {
            if (!queried[pKFi]) { mnRelocWords[pKFi] = 0; queried[pKFi] = 1; lKFsSharingWords.push_back(pKFi); }
            mnRelocWords[pKFi]++;
        }
    }
    if (lKFsSharingWords.empty()) return 0;
    int maxCommonWords = 0;
    for (int k : lKFsSharingWords) if (mnRelocWords[k] > maxCommonWords) maxCommonWords = mnRelocWords[k];
    const int minCommonWords = maxCommonWords * 0.8f;
    std::vector<std::pair<float, int>> lScoreAndMatch;
    for (int k : lKFsSharingWords) {
        if (mnRelocWords[k] > minCommonWords) {
            const int s0 = kf_start[k], n2 = kf_start[k + 1] - s0;
            const float si = (float)orbport_bow_score_l1(q_word, q_value, nq, kf_word + s0, kf_value + s0, n2, nullptr, nullptr);
            mRelocScore[k] = si;
            lScoreAndMatch.push_back({si, k});
        }
    }
    if (lScoreAndMatch.empty()) return 0;
    std::vector<std::pair<float, int>> lAccScoreAndMatch;
    float bestAccScore = 0;
    for (auto& it : lScoreAndMatch) {
        const int pKFi = it.second;
        float bestScore = it.first;
        float accScore = bestScore;
        int pBestKF = pKFi;
        for (int j = 0; j < 10; j++) {
            const int pKF2 = neigh[(size_t)pKFi * 10 + j];
            if (pKF2 < 0) break;
            if (!queried[pKF2]) continue;
            accScore += mRelocScore[pKF2];
            if (mRelocScore[pKF2] > bestScore) { pBestKF = pKF2; bestScore = mRelocScore[pKF2]; }
        }
        lAccScoreAndMatch.push_back({accScore, pBestKF});
        if (accScore > bestAccScore) bestAccScore = accScore;
    }
    const float minScoreToRetain = 0.75f * bestAccScore;
    std::vector<char> added(n_kf, 0);
    int n_out = 0;
    for (auto& it : lAccScoreAndMatch) {
        if (it.first > minScoreToRetain && !added[it.second]) { out[n_out++] = it.second; added[it.second] = 1; }
    }
    return n_out;
}

// Frame::isInFrustum — reference src/Frame.cc:269-325, for n MapPoints (Tracking::SearchLocalPoints, src/Tracking.cc:1167-1180).
// Tcw = [mRcw | mtcw], Ow = mOw.  Outputs are the fields the reference stores on the MapPoint: mbTrackInView,
// mTrackProjX, mTrackProjY, mTrackProjXR, mnTrackScaleLevel, mTrackViewCos (untouched where in_view = 0).  A point at the
// camera centre (PcZ == 0) projects to NaN, and NaN passes every test that follows: with mfMinDistance == 0 the point is in
// view with NaN track fields and level 0, as in the reference; features_in_area then finds nothing for it.
extern "C" int orbport_is_in_frustum(const float* world_pos, const float* normal, const float* max_distance, const float* min_distance,
                                     const uint8_t* valid, int n, const float* Tcw, const float* Ow, float fx, float fy, float cx,
                                     float cy, float mbf, float minX, float minY, float maxX, float maxY, float viewingCosLimit,
                                     float log_scale_factor, int n_levels, uint8_t* in_view, float* proj_x, float* proj_y,
                                     float* proj_xr, int32_t* level, float* view_cos) {
    int count = 0;
    for (int i = 0; i < n; i++) {
        in_view[i] = 0;
        if (valid && !valid[i]) continue;
        const float* P = world_pos + 3 * (size_t)i;
        const float PcX = ((Tcw[0] * P[0] + Tcw[1] * P[1]) + Tcw[2] * P[2]) + Tcw[3];
        const float PcY = ((Tcw[4] * P[0] + Tcw[5] * P[1]) + Tcw[6] * P[2]) + Tcw[7];
        const float PcZ = ((Tcw[8] * P[0] + Tcw[9] * P[1]) + Tcw[10] * P[2]) + Tcw[11];
        if (PcZ < 0.0f) continue;
        const float invz = 1.0f / PcZ;
        const float u = fx * PcX * invz + cx;
        const float v = fy * PcY * invz + cy;
        if (u < minX || u > maxX) continue;
        if (v < minY || v > maxY) continue;
        const float maxDistance = 1.2f * max_distance[i];
        const float minDistance = 0.8f * min_distance[i];
        const float PO[3] = {P[0] - Ow[0], P[1] - Ow[1], P[2] - Ow[2]};
        const float dist = norm3(PO);
        if (dist < minDistance || dist > maxDistance) continue;
        const float viewCos = dot3(PO, normal + 3 * (size_t)i) / dist;
        if (viewCos < viewingCosLimit) continue;
        const int nPredictedLevel = predict_scale(max_distance[i], dist, log_scale_factor, n_levels);
        in_view[i] = 1;
        proj_x[i] = u;
        proj_xr[i] = u - mbf * invz;
        proj_y[i] = v;
        level[i] = nPredictedLevel;
        view_cos[i] = viewCos;
        count++;
    }
    return count;
}

// KeyFrameDatabase::DetectLoopCandidates(KeyFrame* pKF, float minScore) — reference src/KeyFrameDatabase.cc:76-197, restated
// with a real inverted file like orbport_detect_reloc_candidates.  connected[k] = 1 if keyframe k is in
// pKF->GetConnectedKeyFrames() (the query keyframe itself is normally not in the database yet, :LoopClosing.cc:147).
extern "C" int orbport_detect_loop_candidates(int n_kf, const int32_t* kf_start, const uint32_t* kf_word, const double* kf_value,
                                              int n_words, const uint32_t* q_word, const double* q_value, int nq,
                                              const uint8_t* connected, const int32_t* neigh, float minScore, int32_t* out) {
    std::vector<std::vector<int>> mvInvertedFile(n_words);
    for (int k = 0; k < n_kf; k++)
        for (int e = kf_start[k]; e < kf_start[k + 1]; e++) mvInvertedFile[kf_word[e]].push_back(k);
    std::vector<int> mnLoopWords(n_kf, 0);
    std::vector<char> queried(n_kf, 0);           // pKFi->mnLoopQuery == pKF->mnId
    std::vector<float> mLoopScore(n_kf, 0.f);
    std::vector<int> lKFsSharingWords;
    for (int i = 0; i < nq; i++) {
        if (q_word[i] >= (uint32_t)n_words) continue;
        for (int pKFi : mvInvertedFile[q_word[i]]) {
            if (!queried[pKFi]) {
                mnLoopWords[pKFi] = 0;
                if (!connected[pKFi]) { queried[pKFi] = 1; lKFsSharingWords.push_back(pKFi); }
            }
            mnLoopWords[pKFi]++;
        }
    }
    if (lKFsSharingWords.empty()) return 0;
    std::vector<std::pair<float, int>> lScoreAndMatch;
    int maxCommonWords = 0;
    for (int k : lKFsSharingWords) if (mnLoopWords[k] > maxCommonWords) maxCommonWords = mnLoopWords[k];
    const int minCommonWords = maxCommonWords * 0.8f;
    for (int k : lKFsSharingWords) {
        if (mnLoopWords[k] > minCommonWords) {
            const int s0 = kf_start[k], n2 = kf_start[k + 1] - s0;
            const float si = (float)orbport_bow_score_l1(q_word, q_value, nq, kf_word + s0, kf_value + s0, n2, nullptr, nullptr);
            mLoopScore[k] = si;
            if (si >= minScore) lScoreAndMatch.push_back({si, k});
        }
    }
    if (lScoreAndMatch.empty()) return 0;
    std::vector<std::pair<float, int>> lAccScoreAndMatch;
    float bestAccScore = minScore;
    for (auto& it : lScoreAndMatch) {
        const int pKFi = it.second;
        float bestScore = it.first;
        float accScore = it.first;
        int pBestKF = pKFi;
        for (int j = 0; j < 10; j++) {
            const int pKF2 = neigh[(size_t)pKFi * 10 + j];
            if (pKF2 < 0) break;
            if (queried[pKF2] && mnLoopWords[pKF2] > minCommonWords) {
                accScore += mLoopScore[pKF2];
                if (mLoopScore[pKF2] > bestScore) { pBestKF = pKF2; bestScore = mLoopScore[pKF2]; }
            }
        }
        lAccScoreAndMatch.push_back({accScore, pBestKF});
        if (accScore > bestAccScore) bestAccScore = accScore;
    }
    const float minScoreToRetain = 0.75f * bestAccScore;
    std::vector<char> added(n_kf, 0);
    int n_out = 0;
    for (auto& it : lAccScoreAndMatch)
        if (it.first > minScoreToRetain && !added[it.second]) { out[n_out++] = it.second; added[it.second] = 1; }
    return n_out;
}

// element-wise MapPoint::PredictScale, exported for tests/test_oracle_map_ref.py
extern "C" void orbport_predict_scale(const float* max_distance, const float* dist, int n, float log_scale, int n_levels, int32_t* out) {
    for (int i = 0; i < n; i++) out[i] = predict_scale(max_distance[i], dist[i], log_scale, n_levels);
}
