// Windowed projection search shared by every ORBmatcher::SearchByProjection overload, Fuse and SearchBySim3
// (reference src/ORBmatcher.cc:45-129, 290-403, 825-1100, 1102-1326, 1328-1599) — candidate enumeration and the
// order-dependent claim resolution; fuse_batch_kernel (below) is the list-free search of both Fuse overloads.
//
//   proj_candidates_kernel   Frame::GetFeaturesInArea (src/Frame.cc:327-380) + the per-candidate gates + DescriptorDistance,
//       a warp per query.  Lanes take different GRID CELLS of the query window (a cell holds ~0.3 features, so a lane per
//       feature of one cell would idle 31 lanes), a warp scan turns the per-cell pass counts into list offsets — the list keeps
//       the reference's (ix, iy, insertion) order — then lanes take list ENTRIES for the 256-bit distances.  The list is finally
//       sorted by (distance, position): every consumer needs the lexicographic minimum / second minimum under some exclusion
//       set, which on a sorted list is "the first entries that are not excluded".
//   proj_resolve_kernel<LAST>   the reference's sequential side effect: a query skips features that an EARLIER query of the same
//       call has claimed (:87-89,:123 / :1401-1403,:1428).  The CTA takes a WAVE of up to 1024 consecutive queries, a thread per
//       query: every thread picks the first non-excluded entries of its sorted list, where "excluded" = held before the wave or
//       currently claimed by an EARLIER query of the wave (shared-memory tag per feature, atomicMin of the thread id); claims are
//       republished and the picks repeated until no thread changes.  Query 0 is right after one round, a query whose chain of
//       earlier competitors has depth d after d + 1 rounds: the fixpoint is the sequential result, reached in 2-4 rounds unless
//       neighbouring queries really fight over features.  (A single warp walking the queries costs ~5 cycles per dependent
//       instruction with nothing to hide them: 2 us per 32 queries; the waves make the depth of the conflict chain, not the
//       number of queries, the cost.)
//       LAST = false: best / second-best + ratio test (:98-121), out[query] = feature.
//       LAST = true : best only, threshold th_dist, out[feature] = query, match events for the rotation histogram (:1426-1466).
// All float tests use _rn intrinsics (no FMA contraction) so comparisons match the reference bit for bit.
#include "borb_match.h"

namespace borb {

namespace {

constexpr int HISTO_LENGTH = 30;
constexpr int SORT_CAP = 128;               // lists up to this length are sorted; longer ones keep position order (flagged)
constexpr int RES_K = 4;                    // list entries per query staged in shared memory by the resolve kernel

__device__ __forceinline__ int ham_words(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b) {
    int d = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) d += __popc(a[i] ^ b[i]);
    return d;
}

__device__ __forceinline__ int rot_bin(float a1, float a2) {
    float rot = __fsub_rn(a1, a2);
    if (rot < 0.0f) rot = __fadd_rn(rot, 360.0f);
    int bin = (int)roundf(__fmul_rn(rot, 1.0f / HISTO_LENGTH));
    if (bin == HISTO_LENGTH) bin = 0;
    return bin;
}

__device__ void three_maxima(const int* cnt, int& ind1, int& ind2, int& ind3) {        // ORBmatcher::ComputeThreeMaxima (:1601-1642)
    int max1 = 0, max2 = 0, max3 = 0;
    ind1 = ind2 = ind3 = -1;
    for (int i = 0; i < HISTO_LENGTH; i++) {
        const int s = cnt[i];
        if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }
        else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }
        else if (s > max3) { max3 = s; ind3 = i; }
    }
    if ((float)max2 < 0.1f * (float)max1) { ind2 = -1; ind3 = -1; }
    else if ((float)max3 < 0.1f * (float)max1) { ind3 = -1; }
}

__device__ __forceinline__ unsigned warp_min(unsigned v) { return __reduce_min_sync(0xFFFFFFFFu, v); }

// The cell window of GetFeaturesInArea(x, y, rs) (Frame.cc:327-380) on A's grid: columns c0x..c1x, rows c0y..c1y; false when
// it is empty.  A NaN centre (a point at the camera centre, Frame::isInFrustum) has an empty window: the reference's
// (int)floor(NaN) is INT_MIN on x86, while the device conversion gives 0, which would make the window cell (0, 0).
__device__ __forceinline__ bool area_window(const ProjArgs& A, float x, float y, float rs, int& c0x, int& c1x, int& c0y, int& c1y) {
    if (!(x == x) || !(y == y)) return false;
    c0x = max(0, (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(x, A.minX), rs), A.invW)));
    c1x = min(GRID_COLS - 1, (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(x, A.minX), rs), A.invW)));
    c0y = max(0, (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(y, A.minY), rs), A.invH)));
    c1y = min(GRID_ROWS - 1, (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(y, A.minY), rs), A.invH)));
    return !(c0x >= GRID_COLS || c1x < 0 || c0y >= GRID_ROWS || c1y < 0);
}

// The per-candidate gates of the windowed searches: GetFeaturesInArea's level range and square, then the stereo consistency
// of SearchByProjection (:91-96) where u_right is given (Fuse passes none: its stereo test is the reprojection gate)
__device__ __forceinline__ bool area_passes(const borb_keypoint& kp, const float* __restrict__ u_right, int idx, float x, float y, float xr,
                                            float rs, int minLevel, int maxLevel) {
    if ((minLevel > 0) || (maxLevel >= 0)) {                 // bCheckLevels
        if (kp.octave < minLevel) return false;
        if (maxLevel >= 0 && kp.octave > maxLevel) return false;
    }
    const float dx = __fsub_rn(kp.x, x), dy = __fsub_rn(kp.y, y);
    if (!(fabsf(dx) < rs && fabsf(dy) < rs)) return false;
    if (u_right != nullptr) {
        const float ur = u_right[idx];
        if (ur > 0) {
            const float er = fabsf(__fsub_rn(xr, ur));
            if (er > rs) return false;
        }
    }
    return true;
}

}  // namespace

// cand entry: idx | dist << 16 | octave << 25;   cand_cnt = count | CAND_UNSORTED
__device__ __forceinline__ void candidates_body(const ProjArgs& A) {
    const int lane = threadIdx.x & 31;
    const int iMP = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (iMP >= A.n_mp) return;
    uint32_t* out = A.cand + (size_t)iMP * A.n;
    int count = 0;
    bool unsorted = false;
    // Every per-query input is fetched up front, independent loads back to back: in the small-call path they live in pinned
    // HOST memory (borb_match_host.cu: Call::dev) and a dependent chain of PCIe round trips would dominate the kernel.
    const uint8_t valid_q = A.mp_valid != nullptr ? A.mp_valid[iMP] : (uint8_t)1;
    const int lvl_q = (A.mode == 0) ? A.level[iMP] : 0;
    const float vc_q = (A.mode == 0) ? A.view_cos[iMP] : 0.f;
    const float x = A.proj_x[iMP], y = A.proj_y[iMP];
    const float xr = A.proj_xr[iMP];
    const uint4 dm0 = reinterpret_cast<const uint4*>(A.mp_desc)[(size_t)iMP * 2], dm1 = reinterpret_cast<const uint4*>(A.mp_desc)[(size_t)iMP * 2 + 1];
    const uint32_t dm[8] = {dm0.x, dm0.y, dm0.z, dm0.w, dm1.x, dm1.y, dm1.z, dm1.w};
    if (valid_q) {
        float rs;
        int minLevel, maxLevel;
        if (A.mode == 0) {
            const int lvl = lvl_q;
            float r = vc_q > 0.998 ? 2.5f : 4.0f;     // RadiusByViewingCos (:131-137)
            if (A.th != 1.0f) r = __fmul_rn(r, A.th);
            rs = __fmul_rn(r, A.scale_factors[lvl]);
            minLevel = lvl - 1; maxLevel = lvl;
        } else {
            rs = A.q_radius[iMP]; minLevel = A.q_minl[iMP]; maxLevel = A.q_maxl[iMP];
        }
        // GetFeaturesInArea(x, y, rs, minLevel, maxLevel)  (Frame.cc:327-380)
        int c0x, c1x, c0y, c1y;
        if (area_window(A, x, y, rs, c0x, c1x, c0y, c1y)) {
            auto passes = [&](int idx) -> bool { return area_passes(A.keys[idx], A.u_right, idx, x, y, xr, rs, minLevel, maxLevel); };
            // ---- 1. a lane per grid cell, cells in (ix outer, iy inner) order
            const int ncy = c1y - c0y + 1, C = (c1x - c0x + 1) * ncy;
            for (int cb = 0; cb < C; cb += 32) {
                const int c = cb + lane;
                int s0 = 0, s1 = 0;
                if (c < C) {
                    const int qx = c / ncy;
                    const int cell = (c0x + qx) * GRID_ROWS + c0y + (c - qx * ncy);
                    s0 = A.cell_start[cell]; s1 = A.cell_start[cell + 1];
                }
                int np = 0;
                for (int e = s0; e < s1; e++) np += passes(A.cell_idx[e]) ? 1 : 0;
                int incl = np;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= o) incl += t; }
                int w = count + incl - np;
                if (np > 0)
                    for (int e = s0; e < s1; e++) { const int idx = A.cell_idx[e]; if (passes(idx)) out[w++] = (uint32_t)idx; }
                count += __shfl_sync(0xFFFFFFFFu, incl, 31);
            }
            __syncwarp();
            // ---- 2. a lane per list entry: 256-bit distance
            for (int e = lane; e < count; e += 32) {
                const int idx = (int)out[e];
                const int dist = ham_words(dm, reinterpret_cast<const uint32_t*>(A.desc + (size_t)idx * 32));
                out[e] = (uint32_t)idx | ((uint32_t)dist << 16) | ((uint32_t)A.keys[idx].octave << 25);
            }
            __syncwarp();
            // ---- 3. sort by (distance, position)
            if (count > 1 && count <= 32) {
                const uint32_t ent = lane < count ? out[lane] : 0u;
                const uint32_t key = lane < count ? ((((ent >> 16) & 0x1FFu) << 16) | (uint32_t)lane) : 0xFFFFFFFFu;
                int rank = 0;
#pragma unroll
                for (int j = 0; j < 32; j++) rank += __shfl_sync(0xFFFFFFFFu, key, j) < key ? 1 : 0;
                __syncwarp();
                if (lane < count) out[rank] = ent;
            } else if (count > 32 && count <= SORT_CAP) {
                uint32_t ent[SORT_CAP / 32];
                int rank[SORT_CAP / 32];
#pragma unroll
                for (int t = 0; t < SORT_CAP / 32; t++) { const int e = lane + 32 * t; ent[t] = e < count ? out[e] : 0u; rank[t] = 0; }
                for (int j = 0; j < count; j++) {
                    const uint32_t kj = (((out[j] >> 16) & 0x1FFu) << 16) | (uint32_t)j;
#pragma unroll
                    for (int t = 0; t < SORT_CAP / 32; t++) {
                        const uint32_t key = (((ent[t] >> 16) & 0x1FFu) << 16) | (uint32_t)(lane + 32 * t);
                        rank[t] += kj < key ? 1 : 0;
                    }
                }
                __syncwarp();
#pragma unroll
                for (int t = 0; t < SORT_CAP / 32; t++)
                    if (lane + 32 * t < count) out[rank[t]] = ent[t];
            } else if (count > SORT_CAP) unsorted = true;
        }
    }
    if (lane == 0) A.cand_cnt[iMP] = count | (unsorted ? CAND_UNSORTED : 0);
}

__global__ void __launch_bounds__(256) proj_candidates_kernel(ProjArgs A) { candidates_body(A); }
// one launch for many independent (frame, MapPoint list) jobs: grid.y = job, the job's arguments come from device memory
__global__ void __launch_bounds__(256) proj_candidates_batch_kernel(const ProjArgs* __restrict__ jobs) { candidates_body(jobs[blockIdx.y]); }

// The search part of both Fuse overloads (:825-970, :972-1100) for a table of jobs, a warp per (job, query point) on grid
// (points / 8, jobs), after project_points (variant 2) wrote the windows.  The candidate enumeration and the first-minimum
// search are one pass, with no candidate list: the grid is sorted by cell = ix * GRID_ROWS + iy, so for each column ix of the
// window the window's cells are ONE contiguous range of cell_idx.  Lanes stride over that range (coalesced), apply the area
// gates and the reprojection gates (:907-931), and keep min((dist << 16) | e) with e the position in cell_idx: ascending e is
// the (ix, iy, insertion) order of GetFeaturesInArea, so the warp minimum is the reference's `dist < bestDist` first minimum.
__global__ void __launch_bounds__(256) fuse_batch_kernel(const FuseJob* __restrict__ jobs) {
    const FuseJob& J = jobs[blockIdx.y];
    const ProjArgs& A = J.A;
    const int lane = threadIdx.x & 31;
    const int iq = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (iq >= A.n_mp) return;
    unsigned best = 0xFFFFFFFFu;
    if (A.mp_valid[iq]) {
        const float x = A.proj_x[iq], y = A.proj_y[iq], xr = A.proj_xr[iq], rs = A.q_radius[iq];
        const int minLevel = A.q_minl[iq], maxLevel = A.q_maxl[iq];
        int c0x, c1x, c0y, c1y;
        if (area_window(A, x, y, rs, c0x, c1x, c0y, c1y)) {
            const uint4 dm0 = reinterpret_cast<const uint4*>(A.mp_desc)[(size_t)iq * 2], dm1 = reinterpret_cast<const uint4*>(A.mp_desc)[(size_t)iq * 2 + 1];
            const uint32_t dm[8] = {dm0.x, dm0.y, dm0.z, dm0.w, dm1.x, dm1.y, dm1.z, dm1.w};
            for (int ix = c0x; ix <= c1x; ix++) {
                const int e1 = A.cell_start[ix * GRID_ROWS + c1y + 1];
                for (int e = A.cell_start[ix * GRID_ROWS + c0y] + lane; e < e1; e += 32) {
                    const int idx = A.cell_idx[e];
                    const borb_keypoint kp = A.keys[idx];
                    if (!area_passes(kp, nullptr, idx, x, y, xr, rs, minLevel, maxLevel)) continue;
                    if (J.inv_sigma2 != nullptr) {                      // Fuse(pKF, vpMapPoints, th) reprojection gates (:907-931)
                        const float ex = __fsub_rn(x, kp.x), ey = __fsub_rn(y, kp.y);
                        const float kr = A.u_right != nullptr ? A.u_right[idx] : -1.0f;
                        const float inv = J.inv_sigma2[kp.octave];
                        if (kr >= 0) {
                            const float er = __fsub_rn(xr, kr);
                            const float e2 = __fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(er, er));
                            if ((double)__fmul_rn(e2, inv) > 7.8) continue;
                        } else {
                            const float e2 = __fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey));
                            if ((double)__fmul_rn(e2, inv) > 5.99) continue;
                        }
                    }
                    const int dist = ham_words(dm, reinterpret_cast<const uint32_t*>(A.desc + (size_t)idx * 32));
                    best = min(best, ((unsigned)dist << 16) | (unsigned)e);
                }
            }
        }
    }
    best = warp_min(best);
    if (lane == 0) {
        int out = -1;
        if (best != 0xFFFFFFFFu && (int)(best >> 16) <= A.th_dist) { out = A.cell_idx[best & 0xFFFFu]; atomicAdd(J.n_found, 1); }
        A.out_match[iq] = out;
    }
}

void launch_fuse_search(const FuseJob* d_jobs, int n_jobs, int max_nq, cudaStream_t s) {
    fuse_batch_kernel<<<dim3((max_nq + 7) / 8, n_jobs), 256, 0, s>>>(d_jobs);
}

size_t resolve_smem_bytes(int n, int n_mp) {
    return ((size_t)(n + 31) / 32 + (size_t)n + (size_t)n_mp * RES_K + (size_t)n_mp) * 4 + (size_t)n_mp + 64;
}

// out_match: the per-feature state (LAST) or the per-query match, then the match count
template <bool LAST>
__device__ __forceinline__ void resolve_body(const ProjArgs& A) {
    const borb_keypoint* __restrict__ cur_keys = A.keys;
    int32_t* __restrict__ out = A.out_match;
    int32_t* __restrict__ ev_idx = A.ev_idx;
    uint8_t* __restrict__ ev_bin = A.ev_bin;
    int* __restrict__ n_matches = reinterpret_cast<int*>(A.out_match + (LAST ? A.n : A.n_mp));
    extern __shared__ uint32_t rsm[];
    __shared__ int hist[32];
    __shared__ int cnt_nm, cnt_ev, cnt_rm;
    const int tid = threadIdx.x, lane = tid & 31, T = blockDim.x;
    const int words = (A.n + 31) / 32;
    uint32_t* held = rsm;                                   // bit per frame feature: occupied before the call or claimed during it
    uint32_t* tag = held + words;                           // per feature: lowest lane of the current batch claiming it
    uint32_t* ent = tag + A.n;                              // first RES_K entries of every list
    int* cnts = reinterpret_cast<int*>(ent + (size_t)A.n_mp * RES_K);
    uint8_t* obs = reinterpret_cast<uint8_t*>(cnts + A.n_mp);
    for (int i0 = 0; i0 < words * 32; i0 += T) {            // T is a multiple of 32: a warp builds one word per pass with a ballot
        const int i = i0 + tid;
        const bool occ = A.occupied != nullptr && i < A.n && A.occupied[i] != 0;
        const unsigned bits = __ballot_sync(0xFFFFFFFFu, occ);
        if (lane == 0 && (i >> 5) < words) held[i >> 5] = bits;
    }
    for (int i = tid; i < A.n; i += T) tag[i] = 0xFFFFFFFFu;
    for (int iq = tid; iq < A.n_mp; iq += T) {
        // the first RES_K entries are read unconditionally (the row has A.n >= 1 slots) so that the loads do not wait for the count
        uint32_t e[RES_K];
#pragma unroll
        for (int k = 0; k < RES_K; k++) e[k] = k < A.n ? A.cand[(size_t)iq * A.n + k] : 0u;
        const int c = A.cand_cnt[iq];
        cnts[iq] = c;
        obs[iq] = (A.mp_has_obs == nullptr || A.mp_has_obs[iq]) ? 1 : 0;
#pragma unroll
        for (int k = 0; k < RES_K; k++) ent[iq * RES_K + k] = k < (c & CAND_COUNT_MASK) ? e[k] : 0u;
    }
    if (LAST) for (int i = tid; i < A.n; i += T) out[i] = -1;
    if (tid < 32) hist[tid] = 0;
    if (tid == 0) { cnt_nm = 0; cnt_ev = 0; cnt_rm = 0; }
    __syncthreads();

    // ---- waves of T consecutive queries, a thread per query; tag = lowest thread of the wave currently claiming the feature
    for (int base = 0; base < A.n_mp; base += T) {
        const int iq = base + tid;
        const int craw = iq < A.n_mp ? cnts[iq] : 0;
        const int cnt = craw & CAND_COUNT_MASK;
        const bool sorted = !(craw & CAND_UNSORTED);
        const bool active = cnt > 0;
        const bool has_obs = iq < A.n_mp && obs[iq];
        const uint32_t* glist = A.cand + (size_t)(iq < A.n_mp ? iq : 0) * A.n;
        int prev = -1, claim = -1, m = -1;
        while (true) {
            m = -1;
            if (active) {
                // first (and for the ratio test second) entry that is neither held nor claimed by an earlier query of the wave
                uint32_t e1 = 0xFFFFFFFFu, e2 = 0xFFFFFFFFu;
                if (sorted) {
                    for (int p = 0; p < cnt; p++) {
                        const uint32_t e = p < RES_K ? ent[iq * RES_K + p] : glist[p];
                        const int idx = e & 0xFFFF;
                        if (((held[idx >> 5] >> (idx & 31)) & 1u) || tag[idx] < (uint32_t)tid) continue;
                        if (e1 == 0xFFFFFFFFu) { e1 = e; if (LAST) break; }
                        else { e2 = e; break; }
                    }
                } else {                                     // list longer than SORT_CAP: full scan in position order
                    unsigned k1 = 0xFFFFFFFFu, k2 = 0xFFFFFFFFu;
                    for (int p = 0; p < cnt; p++) {
                        const uint32_t e = glist[p];
                        const int idx = e & 0xFFFF;
                        if (((held[idx >> 5] >> (idx & 31)) & 1u) || tag[idx] < (uint32_t)tid) continue;
                        const unsigned key = (((e >> 16) & 0x1FFu) << 16) | (unsigned)p;
                        if (key < k1) { k2 = k1; k1 = key; } else if (key < k2) k2 = key;
                    }
                    if (k1 != 0xFFFFFFFFu) e1 = glist[k1 & 0xFFFFu];
                    if (k2 != 0xFFFFFFFFu) e2 = glist[k2 & 0xFFFFu];
                }
                if (e1 != 0xFFFFFFFFu) {
                    const int bestDist = (int)((e1 >> 16) & 0x1FFu);
                    if (LAST) {
                        if (bestDist <= A.th_dist) m = (int)(e1 & 0xFFFF);
                    } else if (bestDist <= TH_HIGH) {
                        const int bestLevel = (int)(e1 >> 25);
                        int bestDist2 = 256, bestLevel2 = -1;
                        if (e2 != 0xFFFFFFFFu) { bestDist2 = (int)((e2 >> 16) & 0x1FFu); bestLevel2 = (int)(e2 >> 25); }
                        if (!(bestLevel == bestLevel2 && (float)bestDist > __fmul_rn(A.nnratio, (float)bestDist2))) m = (int)(e1 & 0xFFFF);
                    }
                }
            }
            claim = (m >= 0 && has_obs) ? m : -1;             // only MapPoints with observations block later queries (:87-89)
            if (!__syncthreads_or(claim != prev)) break;      // (also: every pick has read the tags before they change)
            if (prev >= 0) tag[prev] = 0xFFFFFFFFu;
            __syncthreads();
            if (claim >= 0) atomicMin(&tag[claim], (uint32_t)tid);
            __syncthreads();
            prev = claim;
        }
        // commit the wave
        if (claim >= 0) { atomicOr(&held[claim >> 5], 1u << (claim & 31)); tag[claim] = 0xFFFFFFFFu; }
        const unsigned accm = __ballot_sync(0xFFFFFFFFu, m >= 0);
        if (LAST) {
            int ebase = 0;
            if (lane == 0 && accm) ebase = atomicAdd(&cnt_ev, __popc(accm));
            ebase = __shfl_sync(0xFFFFFFFFu, ebase, 0);
            if (m >= 0) {
                atomicMax(&out[m], iq);                       // CurrentFrame.mvpMapPoints[bestIdx2] = pMP: a later query overwrites (:1428)
                ev_idx[ebase + __popc(accm & ((1u << lane) - 1))] = m | (iq << 16);     // match event: feature | query << 16
            }
        } else if (iq < A.n_mp) out[iq] = m;
        if (lane == 0 && accm) atomicAdd(&cnt_nm, __popc(accm));
        __syncthreads();
    }
    if (LAST && A.check_ori) {
        __threadfence_block();
        __syncthreads();
        const int nev = cnt_ev;
        // rotation histogram over the MATCH EVENTS (a feature re-claimed later appears twice, exactly as rotHist does)
        for (int e = tid; e < nev; e += T) {
            const int ev = ev_idx[e];
            const int b = rot_bin(A.q_angle[ev >> 16], cur_keys[ev & 0xFFFF].angle);
            ev_bin[e] = (uint8_t)b;
            atomicAdd(&hist[b], 1);
        }
        __syncthreads();
        int i1, i2, i3;
        three_maxima(hist, i1, i2, i3);
        // culling is order independent for the final state: every event of a culled bin nulls its feature
        int removed = 0;
        for (int e = tid; e < nev; e += T) {
            const int b = ev_bin[e];
            if (b != i1 && b != i2 && b != i3) { out[ev_idx[e] & 0xFFFF] = -2; removed++; }
        }
        if (removed) atomicAdd(&cnt_rm, removed);
    }
    __syncthreads();
    if (tid == 0) *n_matches = cnt_nm - cnt_rm;
}

template <bool LAST>
__global__ void __launch_bounds__(1024) proj_resolve_kernel(ProjArgs A) { resolve_body<LAST>(A); }
// a CTA per job (SearchByProjection(F, vpMapPoints) or (CurrentFrame, LastFrame) of many independent frames in one launch);
// the block size follows the largest job, and the wave fixpoint is the sequential result for any block size
template <bool LAST>
__global__ void __launch_bounds__(1024) proj_resolve_batch_kernel(const ProjArgs* __restrict__ jobs) {
    const ProjArgs& A = jobs[blockIdx.x];
    if (A.n_mp <= 0) return;                        // a job without work (no MapPoints / empty frame) carries null pointers
    resolve_body<LAST>(A);
}

void launch_candidates(const ProjArgs& A, cudaStream_t s) {
    if (A.n_mp > 0) proj_candidates_kernel<<<(A.n_mp + 7) / 8, 256, 0, s>>>(A);
}

int launch_projection_batch(const ProjArgs* d_jobs, const ProjArgs& one, int n_jobs, int max_n, int max_n_mp, cudaStream_t s, bool last) {
    if (n_jobs <= 0 || max_n_mp <= 0) return 0;
    if (n_jobs == 1) {
        launch_candidates(one, s);
        launch_resolve(one, last, s);
        return 2;
    }
    proj_candidates_batch_kernel<<<dim3((max_n_mp + 7) / 8, n_jobs), 256, 0, s>>>(d_jobs);
    const size_t smem = resolve_smem_bytes(max_n, max_n_mp);
    const int threads = max_n_mp > 512 ? 1024 : (max_n_mp > 256 ? 512 : 256);
    if (last) {
        allow_max_smem((const void*)proj_resolve_batch_kernel<true>);
        proj_resolve_batch_kernel<true><<<n_jobs, threads, smem, s>>>(d_jobs);
    } else {
        allow_max_smem((const void*)proj_resolve_batch_kernel<false>);
        proj_resolve_batch_kernel<false><<<n_jobs, threads, smem, s>>>(d_jobs);
    }
    return 2;
}

void launch_resolve(const ProjArgs& A, bool last, cudaStream_t s) {
    const size_t smem = resolve_smem_bytes(A.n, A.n_mp);
    const int threads = A.n_mp > 512 ? 1024 : (A.n_mp > 256 ? 512 : 256);     // one wave covers the whole call when it can
    if (last) {
        allow_max_smem((const void*)proj_resolve_kernel<true>);
        proj_resolve_kernel<true><<<1, threads, smem, s>>>(A);
    } else {
        allow_max_smem((const void*)proj_resolve_kernel<false>);
        proj_resolve_kernel<false><<<1, threads, smem, s>>>(A);
    }
}

}  // namespace borb
