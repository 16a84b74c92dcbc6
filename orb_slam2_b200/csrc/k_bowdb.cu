// SearchByBoW(KeyFrame*, Frame&, vpMapPointMatches) (reference src/ORBmatcher.cc:159-288) of ONE frame against MANY keyframes
// of the device-resident database in one launch — relocalisation / loop-closure candidates (src/Tracking.cc:1357-1377),
// BASELINE configs[4]: 2000 keyframes x ~1200 features = 76.8 MB of descriptors + 9.6 MB of feature-vector data per query.
//
// Layout.  A keyframe is stored in the database as a STREAM RECORD: its features permuted into FeatureVector order (node id
// ascending, feature index ascending inside a node — the order of the reference's two nested loops, :180-205), so that the
// descriptors of a node are consecutive 32-byte rows and every keyframe byte is read exactly once.  The query frame is packed
// the same way on the device (bowdb_pack_kernel, plus a work list), fetched into shared memory ONCE per (persistent, one per SM)
// CTA with a 1-D TMA bulk copy (cp.async.bulk + mbarrier) and reused for every keyframe.
//
// Jobs.  One launch sequence (pack, match, finalize) serves many frames, each against its own database and keyframe list
// (borb_search_by_bow_db_batch; a single call is the one-job case): every job has its own block, work counter, match table,
// histograms and pair cursor.
//
// Work decomposition.  A frame feature lives in exactly one node, so the greedy "frame feature already claimed" skip (:209)
// never crosses nodes: a (keyframe, node) bucket is an independent claim scope.  An ITEM is (one node of the query frame, a
// range of <= 32 keyframes); warps take items from an atomic counter, widest buckets first, keyframes per item ~ 1 / nt^2.
// Inside an item every row (keyframe feature with a good MapPoint, :196-202) meets the SAME nt columns (frame features of
// the node): lane = row with its descriptor in registers, the column loop has a warp-uniform trip count and broadcast
// shared-memory loads; best / second best == lexicographic min / second min of (distance, column).  Only rows that have a
// distance <= TH_LOW at all can match or claim (:226); those are replayed in (keyframe, row) order against the bucket's
// claim bits with the ratio test of :228 (a row whose best or second best was claimed meanwhile is rescanned by the warp).
// A match goes to a (keyframe x frame-position) table and bumps the keyframe's rotation histogram; a second kernel (CTA per
// keyframe) applies ComputeThreeMaxima (:267-285) and compacts the survivors into (frame feature, keyframe feature) pairs in
// (node, frame feature) order — deterministic output.
//
// Bound: not HBM (96 MB of keyframe records per 2000-keyframe sweep) but the integer pipes and the per-item / per-batch
// bookkeeping around the column loop (ham256<MODE>: 8 POPC, 4 POPC + carry-save tree, or 5 POPC + three 3:2 compressors).
#include "borb_match.h"
#include "match_rules.cuh"

namespace borb {

namespace {

constexpr int BDB_WARPS = 32;                 // one 1024-thread CTA per SM (64 registers): 32 warps share one copy of the query frame
constexpr int BDB_CTAS = 1;
constexpr int BDB_QCAP = 64;                  // pending-row ring per warp
constexpr int BDB_CLAIM_WORDS = MATCH_MAX_FEATURES / 32;
constexpr int BDB_WARP_BYTES = BDB_CLAIM_WORDS * 4 + 32 * 24 + BDB_QCAP * 48;   // claim bits | keyframe runs of the batch | pending rows (descriptor halves, meta)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// 256-bit Hamming distance.  MODE 0: 8 POPC (descriptor_distance).  MODE 1: full carry-save adder tree, 4 POPC + 17 LOP3.  MODE 2
// (default): three 3:2 compressors, 5 POPC + 6 LOP3.  POPC issues at a quarter of LOP3's rate (16 vs 64 results per clock per SM on
// sm_90, CUDA C++ Programming Guide throughput table): per distance MODE 0 is all POPC, MODE 1 shifts most of the work to LOP3,
// MODE 2 balances the two.
template <int MODE>
__device__ __forceinline__ int ham256(const uint4 a0, const uint4 a1, const uint4 b0, const uint4 b1) {
    if (MODE == 0) return descriptor_distance(a0, a1, b0, b1);
    const uint32_t x0 = a0.x ^ b0.x, x1 = a0.y ^ b0.y, x2 = a0.z ^ b0.z, x3 = a0.w ^ b0.w;
    const uint32_t x4 = a1.x ^ b1.x, x5 = a1.y ^ b1.y, x6 = a1.z ^ b1.z, x7 = a1.w ^ b1.w;
    const uint32_t s1 = x0 ^ x1 ^ x2, c1 = (x0 & x1) | (x2 & (x0 ^ x1));
    const uint32_t s2 = x3 ^ x4 ^ x5, c2 = (x3 & x4) | (x5 & (x3 ^ x4));
    const uint32_t s3 = s1 ^ s2 ^ x6, c3 = (s1 & s2) | (x6 & (s1 ^ s2));
    if (MODE == 2) return (__popc(s3) + __popc(x7)) + 2 * (__popc(c1) + __popc(c2) + __popc(c3));
    // full tree: 8 words -> bit planes of weight 1, 2, 4, 8
    const uint32_t ones = s3 ^ x7, c4 = s3 & x7;
    const uint32_t s5 = c1 ^ c2 ^ c3, c5 = (c1 & c2) | (c3 & (c1 ^ c2));
    const uint32_t twos = s5 ^ c4, c6 = s5 & c4;
    const uint32_t fours = c5 ^ c6, eights = c5 & c6;
    return __popc(ones) + 2 * __popc(twos) + 4 * __popc(fours) + 8 * __popc(eights);
}

}  // namespace

struct KfRun { const uint2* meta; const uint4* desc; int rs, off; };     // rows rs.. of one keyframe's bucket; off = first row's rank in the batch

// The items of one job, taken by this CTA's warps until the job's work counter is exhausted.  fb: the job's frame block, in
// shared memory (FSM) or in global memory; ws: the warp's scratch.
template <int CSA, bool FSM>
__device__ __forceinline__ void bowdb_job_items(const BowDbArgs& A, const BowDbJob& J, const uint8_t* fb, uint8_t* ws) {
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const unsigned lt_mask = (1u << lane) - 1u;
    const FrameBlockHdr* H = reinterpret_cast<const FrameBlockHdr*>(fb);
    const int mf = H->m, np = H->np;
    const uint32_t* fnode = reinterpret_cast<const uint32_t*>(fb + H->off_node);
    const int32_t* fstart = reinterpret_cast<const int32_t*>(fb + H->off_start);
    const float* fangle = reinterpret_cast<const float*>(fb + H->off_angle);
    const uint4* fdesc = reinterpret_cast<const uint4*>(fb + H->off_desc);
    const int32_t* pnode = reinterpret_cast<const int32_t*>(fb + H->off_pnode);
    const int32_t* pcs = reinterpret_cast<const int32_t*>(fb + H->off_pcs);
    const int32_t* pstart = reinterpret_cast<const int32_t*>(fb + H->off_pstart);

    uint32_t* claim = reinterpret_cast<uint32_t*>(ws);                                   // claimed columns when the bucket is wider than 32
    KfRun* run = reinterpret_cast<KfRun*>(ws + BDB_CLAIM_WORDS * 4);                      // the <= 32 keyframes of the current batch
    // ring of pending rows with a good MapPoint: descriptor halves and {row, run, meta.x, meta.y}
    uint4* qd0 = reinterpret_cast<uint4*>(ws + BDB_CLAIM_WORDS * 4 + 32 * sizeof(KfRun));
    uint4* qd1 = qd0 + BDB_QCAP;
    int4* qm = reinterpret_cast<int4*>(qd1 + BDB_QCAP);

    const int items = pstart[np];
    const int warps_total = gridDim.x * (blockDim.x >> 5);
    int it_static = blockIdx.x + gridDim.x * wrp;                 // static schedule: consecutive (similar-cost) items go to different SMs
    while (true) {
        int it = 0;
        if (A.static_sched) { it = it_static; it_static += warps_total; }
        else {
            if (lane == 0) it = atomicAdd(J.ctr, 1);
            it = __shfl_sync(0xFFFFFFFFu, it, 0);
        }
        if (it >= items) break;
        int lo = 0, hi = np;                                      // largest p with pstart[p] <= it
        while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (pstart[mid] <= it) lo = mid; else hi = mid; }
        const int bf = pnode[lo], cs = pcs[lo];
        const int k0 = (it - pstart[lo]) * cs, k1 = min(J.n_kf, k0 + cs);
        const uint32_t node = fnode[bf];
        const int ts = fstart[bf], nt = fstart[bf + 1] - ts;       // nt > 0 by construction of the work list
        const bool wide = nt > 32;
        const uint4* fd = fdesc + (size_t)ts * 2;

        {
            const int kb = k0;                                    // an item holds at most 32 keyframes (the host's work list)
            // ---- lane j: keyframe kb + j; find the bucket of `node` in its FeatureVector (ascending node ids)
            const int k = kb + lane;
            int rs = 0, cnt = 0;
            const uint2* kmeta = nullptr; const uint4* kdesc = nullptr;
            if (k < k1) {
                const KfStream* Kp = J.table + (J.slots ? J.slots[k] : k);
                const int nn = Kp->nn;
                if (nn > 0) {
                    const uint32_t* kn = Kp->node;
                    int idx = min(bf, nn - 1);                    // both lists are ascending subsets of the same level: try the same rank first
                    if (kn[idx] != node) {
                        int l2 = 0, h2 = nn;
                        while (l2 < h2) { const int mid = (l2 + h2) >> 1; if (kn[mid] < node) l2 = mid + 1; else h2 = mid; }
                        idx = (l2 < nn && kn[l2] == node) ? l2 : -1;
                    }
                    if (idx >= 0) {
                        const int32_t* st = Kp->start;
                        rs = st[idx]; cnt = st[idx + 1] - rs;
                        kmeta = Kp->meta; kdesc = reinterpret_cast<const uint4*>(Kp->desc);
                    }
                }
            }
            int incl = cnt;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= o) incl += t; }
            const int total = __shfl_sync(0xFFFFFFFFu, incl, 31);
            __syncwarp();
            run[lane] = KfRun{kmeta, kdesc, rs, incl - cnt};
            __syncwarp();
            int cur_run = -1;                  // keyframe (lane index of the batch) the claim state below belongs to
            uint32_t claimed = 0;
            int qn = 0, qh = 0;                // ring: qn pending rows starting at slot qh

            // One batch: lane j owns the j-th pending row (rows stay in (keyframe, FeatureVector) order), its 256-bit descriptor
            // in registers, and scans the nt columns: best / second best == lexicographic min / second min of (distance, column)
            // (:207-224).  Then the rows that have a distance <= TH_LOW at all are replayed in row order against the claim state
            // of their keyframe (:209, :226-251); every other row can neither match nor claim.
            auto process = [&](int n_act) {
                const bool act = lane < n_act;
                int4 e = make_int4(0, 0, 0, 0);
                uint4 q0 = make_uint4(0, 0, 0, 0), q1 = q0;
                if (act) { const int sl = (qh + lane) & (BDB_QCAP - 1); e = qm[sl]; q0 = qd0[sl]; q1 = qd1[sl]; }
                unsigned k1v = 0xFFFFFFFFu, k2v = 0xFFFFFFFFu;
#pragma unroll 2
                for (int c = 0; c < nt; c++) {
                    const int d = ham256<CSA>(q0, q1, fd[2 * c], fd[2 * c + 1]);
                    const unsigned key = ((unsigned)d << 16) | (unsigned)c;
                    k2v = min(k2v, max(k1v, key));                 // second smallest so far (k1v <= k2v always)
                    k1v = min(k1v, key);
                }
                unsigned low = __ballot_sync(0xFFFFFFFFu, act && (k1v >> 16) <= (unsigned)TH_LOW);
                while (low) {
                    const int L = __ffs(low) - 1;
                    low &= low - 1;
                    const int rL = __shfl_sync(0xFFFFFFFFu, e.y, L);
                    unsigned kk1 = __shfl_sync(0xFFFFFFFFu, k1v, L), kk2 = __shfl_sync(0xFFFFFFFFu, k2v, L);
                    if (rL != cur_run) {
                        cur_run = rL; claimed = 0;
                        if (wide) { for (int w = lane; w < ((nt + 31) >> 5); w += 32) claim[w] = 0; __syncwarp(); }
                    }
                    auto is_claimed = [&](unsigned col) -> bool { return wide ? ((claim[col >> 5] >> (col & 31)) & 1u) != 0 : ((claimed >> col) & 1u) != 0; };
                    const bool stale = is_claimed(kk1 & 0xFFFFu) || (kk2 != 0xFFFFFFFFu && is_claimed(kk2 & 0xFFFFu));
                    if (stale) {
                        // a claimed column is this row's best or second best: rescan the bucket without the claimed columns, all lanes
                        uint4 r0v, r1v;
                        r0v.x = __shfl_sync(0xFFFFFFFFu, q0.x, L); r0v.y = __shfl_sync(0xFFFFFFFFu, q0.y, L);
                        r0v.z = __shfl_sync(0xFFFFFFFFu, q0.z, L); r0v.w = __shfl_sync(0xFFFFFFFFu, q0.w, L);
                        r1v.x = __shfl_sync(0xFFFFFFFFu, q1.x, L); r1v.y = __shfl_sync(0xFFFFFFFFu, q1.y, L);
                        r1v.z = __shfl_sync(0xFFFFFFFFu, q1.z, L); r1v.w = __shfl_sync(0xFFFFFFFFu, q1.w, L);
                        unsigned m1 = 0xFFFFFFFFu, m2 = 0xFFFFFFFFu;
                        for (int col = lane; col < nt; col += 32) {
                            if (is_claimed((unsigned)col)) continue;
                            const int d = ham256<CSA>(r0v, r1v, fd[2 * col], fd[2 * col + 1]);
                            const unsigned key = ((unsigned)d << 16) | (unsigned)col;
                            if (key < m1) { m2 = m1; m1 = key; } else if (key < m2) m2 = key;
                        }
                        kk1 = __reduce_min_sync(0xFFFFFFFFu, m1);
                        kk2 = __reduce_min_sync(0xFFFFFFFFu, m1 == kk1 ? m2 : m1);
                    }
                    if (kk1 == 0xFFFFFFFFu) continue;
                    const int bestDist1 = (int)(kk1 >> 16);
                    if (bestDist1 > TH_LOW) continue;                                          // :226
                    const int bestDist2 = kk2 == 0xFFFFFFFFu ? 256 : (int)(kk2 >> 16);
                    if (!((float)bestDist1 < __fmul_rn(A.nnratio, (float)bestDist2))) continue;   // :228
                    const unsigned pb = kk1 & 0xFFFFu;
                    if (wide) { if (lane == 0) claim[pb >> 5] |= 1u << (pb & 31); __syncwarp(); }
                    else claimed |= 1u << pb;
                    const uint32_t mx = (uint32_t)__shfl_sync(0xFFFFFFFFu, e.z, L), my = (uint32_t)__shfl_sync(0xFFFFFFFFu, e.w, L);
                    if (lane == 0) {
                        const int bin = A.check_ori ? rot_bin(__uint_as_float(my), fangle[ts + pb]) : 0;
                        J.table_out[(size_t)(kb + rL) * mf + ts + pb] = (mx & 0xFFFFu) | ((uint32_t)bin << 16);   // vpMapPointMatches[bestIdxF] = pMP (:232)
                        atomicAdd(&J.hist_out[(size_t)(kb + rL) * 32 + bin], 1);                                     // rotHist[bin].push_back (:241)
                    }
                }
            };

            // rows of the batch in (keyframe, row) order, 32 at a time; the loads of the next 32 are issued before the pending
            // ones are processed, so their latency overlaps the column loop
            auto fetch = [&](int base, int& src, int& row, uint2& meta, uint4& d0, uint4& d1) {
                const int pos = base + lane;
                src = 0; row = 0; meta = make_uint2(0u, 0u); d0 = make_uint4(0, 0, 0, 0); d1 = d0;
                if (pos < total) {
                    int l3 = 0, h3 = 32;                          // largest j with run[j].off <= pos (empty runs share their successor's off: pick the last)
                    while (h3 - l3 > 1) { const int mid = (l3 + h3) >> 1; if (run[mid].off <= pos) l3 = mid; else h3 = mid; }
                    src = l3;
                    const KfRun r = run[src];
                    row = r.rs + (pos - r.off);
                    meta = r.meta[row];                           // feature | good-MapPoint flag << 16 | ..., angle
                    d0 = r.desc[(size_t)row * 2]; d1 = r.desc[(size_t)row * 2 + 1];
                }
            };
            int src, row; uint2 meta; uint4 d0, d1;
            fetch(0, src, row, meta, d0, d1);
            for (int base = 0; base < total; base += 32) {
                const bool ok = ((meta.x >> 16) & 1u) != 0;       // good MapPoint (:196-202)
                const unsigned okm = __ballot_sync(0xFFFFFFFFu, ok);
                if (ok) {
                    const int sl = (qh + qn + __popc(okm & lt_mask)) & (BDB_QCAP - 1);
                    qm[sl] = make_int4(row, src, (int)meta.x, (int)meta.y); qd0[sl] = d0; qd1[sl] = d1;
                }
                qn += __popc(okm);
                if (base + 32 < total) fetch(base + 32, src, row, meta, d0, d1);
                __syncwarp();
                if (qn >= 32) {
                    process(32);
                    qh = (qh + 32) & (BDB_QCAP - 1); qn -= 32;
                    __syncwarp();
                }
            }
            if (qn > 0) { process(qn); __syncwarp(); }
        }
    }
}

// SearchByBoW(KeyFrame* pKF1, KeyFrame* pKF2) (src/ORBmatcher.cc:522-655) of the loop-closing keyframe (the query, a slot of the
// database packed into the block like a frame) against many candidates: the roles of the two sides swap.  Rows are the QUERY's
// features with a good MapPoint (:558-562), shared by every candidate; columns are the candidate's bucket features with a good
// MapPoint (:574-580), and the claims sit on them (vbMatched2, :576, :603).  A candidate feature lies in one node, so a (candidate,
// node) bucket is still an independent claim scope.  An item is (query node, <= 32 candidates); lane j finds candidate j's bucket,
// then the warp takes the candidates one after the other: lane = query row (32 at a time, descriptor from the block), the column
// loop over the candidate's bucket is warp-uniform (broadcast loads).  Best / second best are the lexicographic min / second min of
// (distance, column) — the first minimum in the candidate's FeatureVector order wins (:586-595).  Rows with a distance below TH_LOW
// at all are replayed in row order against the bucket's claims, a row whose best or second best was claimed meanwhile rescanned by
// the warp, with the strict gate of :598 and the ratio test of :600.  The match goes to the (candidate x query position) table as
// candidate feature | bin << 16, the bin of query angle - candidate angle (:607), so the relocalisation finalize culls and compacts it.
template <bool FSM>
__device__ __forceinline__ void bowkf_job_items(const BowDbArgs& A, const BowDbJob& J, const uint8_t* fb, uint8_t* ws) {
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const FrameBlockHdr* H = reinterpret_cast<const FrameBlockHdr*>(fb);
    const int mf = H->m, np = H->np;
    const uint32_t* fnode = reinterpret_cast<const uint32_t*>(fb + H->off_node);
    const int32_t* fstart = reinterpret_cast<const int32_t*>(fb + H->off_start);
    const float* fangle = reinterpret_cast<const float*>(fb + H->off_angle);
    const uint4* fdesc = reinterpret_cast<const uint4*>(fb + H->off_desc);
    const int32_t* pnode = reinterpret_cast<const int32_t*>(fb + H->off_pnode);
    const int32_t* pcs = reinterpret_cast<const int32_t*>(fb + H->off_pcs);
    const int32_t* pstart = reinterpret_cast<const int32_t*>(fb + H->off_pstart);
    const uint2* qmeta = J.q_meta;                                // the query's rows, in block order: the good-MapPoint flag
    uint32_t* claim = reinterpret_cast<uint32_t*>(ws);            // claimed columns when the bucket is wider than 32

    const int items = pstart[np];
    const int warps_total = gridDim.x * (blockDim.x >> 5);
    int it_static = blockIdx.x + gridDim.x * wrp;
    while (true) {
        int it = 0;
        if (A.static_sched) { it = it_static; it_static += warps_total; }
        else {
            if (lane == 0) it = atomicAdd(J.ctr, 1);
            it = __shfl_sync(0xFFFFFFFFu, it, 0);
        }
        if (it >= items) break;
        int lo = 0, hi = np;                                      // largest p with pstart[p] <= it
        while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (pstart[mid] <= it) lo = mid; else hi = mid; }
        const int bf = pnode[lo], cs = pcs[lo];
        const int k0 = (it - pstart[lo]) * cs, k1 = min(J.n_kf, k0 + cs);
        const uint32_t node = fnode[bf];
        const int ts = fstart[bf], nt = fstart[bf + 1] - ts;

        // lane j: candidate k0 + j; the bucket of `node` in its FeatureVector (ascending node ids)
        const int k = k0 + lane;
        int rs = 0, cnt = 0;
        const uint2* kmeta = nullptr; const uint4* kdesc = nullptr;
        if (k < k1) {
            const KfStream* Kp = J.table + (J.slots ? J.slots[k] : k);
            const int nn = Kp->nn;
            if (nn > 0) {
                const uint32_t* kn = Kp->node;
                int idx = min(bf, nn - 1);
                if (kn[idx] != node) {
                    int l2 = 0, h2 = nn;
                    while (l2 < h2) { const int mid = (l2 + h2) >> 1; if (kn[mid] < node) l2 = mid + 1; else h2 = mid; }
                    idx = (l2 < nn && kn[l2] == node) ? l2 : -1;
                }
                if (idx >= 0) {
                    rs = Kp->start[idx]; cnt = Kp->start[idx + 1] - rs;
                    kmeta = Kp->meta + rs; kdesc = reinterpret_cast<const uint4*>(Kp->desc) + (size_t)rs * 2;
                }
            }
        }
        unsigned todo = __ballot_sync(0xFFFFFFFFu, cnt > 0);
        while (todo) {
            const int src = __ffs(todo) - 1;
            todo &= todo - 1;
            const int nc = __shfl_sync(0xFFFFFFFFu, cnt, src);
            const uint2* cm = reinterpret_cast<const uint2*>(__shfl_sync(0xFFFFFFFFu, reinterpret_cast<unsigned long long>(kmeta), src));
            const uint4* cd = reinterpret_cast<const uint4*>(__shfl_sync(0xFFFFFFFFu, reinterpret_cast<unsigned long long>(kdesc), src));
            const bool wide = nc > 32;
            uint32_t claimed = 0;
            if (wide) { for (int w = lane; w < ((nc + 31) >> 5); w += 32) claim[w] = 0; __syncwarp(); }
            auto is_claimed = [&](unsigned col) -> bool { return wide ? ((claim[col >> 5] >> (col & 31)) & 1u) != 0 : ((claimed >> col) & 1u) != 0; };
            auto good = [&](int col) -> bool { return ((cm[col].x >> 16) & 1u) != 0; };
            for (int r0 = 0; r0 < nt; r0 += 32) {
                const int r = ts + r0 + lane;
                const bool act = r0 + lane < nt && ((qmeta[r].x >> 16) & 1u) != 0;
                uint4 q0 = make_uint4(0, 0, 0, 0), q1 = q0;
                if (act) { q0 = fdesc[2 * r]; q1 = fdesc[2 * r + 1]; }
                unsigned k1v = 0xFFFFFFFFu, k2v = 0xFFFFFFFFu;
                for (int c = 0; c < nc; c++) {
                    if (!good(c)) continue;                                        // warp-uniform
                    const int d = ham256<2>(q0, q1, cd[2 * c], cd[2 * c + 1]);
                    const unsigned key = ((unsigned)d << 16) | (unsigned)c;
                    k2v = min(k2v, max(k1v, key));
                    k1v = min(k1v, key);
                }
                unsigned low = __ballot_sync(0xFFFFFFFFu, act && (k1v >> 16) < (unsigned)TH_LOW);
                while (low) {
                    const int L = __ffs(low) - 1;
                    low &= low - 1;
                    unsigned kk1 = __shfl_sync(0xFFFFFFFFu, k1v, L), kk2 = __shfl_sync(0xFFFFFFFFu, k2v, L);
                    const bool stale = is_claimed(kk1 & 0xFFFFu) || (kk2 != 0xFFFFFFFFu && is_claimed(kk2 & 0xFFFFu));
                    if (stale) {
                        uint4 r0v, r1v;
                        r0v.x = __shfl_sync(0xFFFFFFFFu, q0.x, L); r0v.y = __shfl_sync(0xFFFFFFFFu, q0.y, L);
                        r0v.z = __shfl_sync(0xFFFFFFFFu, q0.z, L); r0v.w = __shfl_sync(0xFFFFFFFFu, q0.w, L);
                        r1v.x = __shfl_sync(0xFFFFFFFFu, q1.x, L); r1v.y = __shfl_sync(0xFFFFFFFFu, q1.y, L);
                        r1v.z = __shfl_sync(0xFFFFFFFFu, q1.z, L); r1v.w = __shfl_sync(0xFFFFFFFFu, q1.w, L);
                        unsigned m1 = 0xFFFFFFFFu, m2 = 0xFFFFFFFFu;
                        for (int col = lane; col < nc; col += 32) {
                            if (is_claimed((unsigned)col) || !good(col)) continue;
                            const int d = ham256<2>(r0v, r1v, cd[2 * col], cd[2 * col + 1]);
                            const unsigned key = ((unsigned)d << 16) | (unsigned)col;
                            if (key < m1) { m2 = m1; m1 = key; } else if (key < m2) m2 = key;
                        }
                        kk1 = __reduce_min_sync(0xFFFFFFFFu, m1);
                        kk2 = __reduce_min_sync(0xFFFFFFFFu, m1 == kk1 ? m2 : m1);
                    }
                    if (kk1 == 0xFFFFFFFFu) continue;
                    const int bestDist1 = (int)(kk1 >> 16);
                    if (bestDist1 >= TH_LOW) continue;                                         // :598
                    const int bestDist2 = kk2 == 0xFFFFFFFFu ? 256 : (int)(kk2 >> 16);
                    if (!((float)bestDist1 < __fmul_rn(A.nnratio, (float)bestDist2))) continue;   // :600
                    const unsigned pb = kk1 & 0xFFFFu;
                    if (wide) { if (lane == 0) claim[pb >> 5] |= 1u << (pb & 31); __syncwarp(); }
                    else claimed |= 1u << pb;
                    if (lane == 0) {
                        const uint2 cv = cm[pb];
                        const int pos = ts + r0 + L;
                        const int bin = A.check_ori ? rot_bin(fangle[pos], __uint_as_float(cv.y)) : 0;
                        J.table_out[(size_t)(k0 + src) * mf + pos] = (cv.x & 0xFFFFu) | ((uint32_t)bin << 16);   // vpMatches12[idx1] (:602)
                        atomicAdd(&J.hist_out[(size_t)(k0 + src) * 32 + bin], 1);                                 // rotHist[bin] (:614)
                    }
                }
            }
            __syncwarp();                                         // the claim words are reset for the next candidate
        }
    }
}

// Job scheduling.  A call with one job (every single call) passes it as a kernel parameter (ONE_SMEM / ONE_GLOBAL): its fields stay
// in the constant bank instead of registers, which keeps the item loop at the register budget of 64.  A job table (TABLE):
// a CTA works on one job at a time: its warps take the job's items from the job's counter, and only when that
// counter is exhausted (for every warp: a barrier) does the CTA move on, to the next job (in job order, wrapping) that still has
// items.  So a CTA visits a job at most once, and fetches a shared-memory frame block (one 1-D TMA bulk copy) only for a job it
// is about to work on.  CTAs start at jobs spread over the job table, so many small jobs are taken by different CTAs.  Blocks
// that do not fit next to the warp scratch are read through L1 from global memory (FSM = false), in the same launch.
// KFKF selects the items of SearchByBoW(KeyFrame*, KeyFrame*) (bowkf_job_items) instead of those of (KeyFrame*, Frame&).
enum { ONE_SMEM = 0, ONE_GLOBAL = 1, TABLE = 2 };
template <int CSA, bool FSM, bool KFKF>
__device__ __forceinline__ void job_items(const BowDbArgs& A, const BowDbJob& J, const uint8_t* fb, uint8_t* ws) {
    if constexpr (KFKF) bowkf_job_items<FSM>(A, J, fb, ws);
    else bowdb_job_items<CSA, FSM>(A, J, fb, ws);
}
template <int CSA, int KIND, bool KFKF>
__device__ __forceinline__ void bowdb_match(const BowDbArgs& A, int smem_frame, const BowDbJob& J0) {
    extern __shared__ __align__(128) uint8_t sm[];
    __shared__ __align__(8) unsigned long long bar;
    __shared__ BowDbJob sJ;
    __shared__ int s_job, s_next, s_left, s_loads;     // the job cursor (the next job to look at, jobs not looked at) and the block loads so far
    const int tid = threadIdx.x;
    if (KIND == ONE_GLOBAL) { job_items<CSA, false, KFKF>(A, J0, J0.frame_block, sm + (size_t)(tid >> 5) * BDB_WARP_BYTES); return; }
    if (KIND == ONE_SMEM) {
        if (tid == 0) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bar)));
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar)), "r"((uint32_t)J0.frame_bytes) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(smem_u32(sm)), "l"(reinterpret_cast<uint64_t>(J0.frame_block)), "r"((uint32_t)J0.frame_bytes), "r"(smem_u32(&bar))
                         : "memory");
        }
        __syncthreads();
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "BOWDB_WAIT1:\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n"
            "@p bra BOWDB_DONE1;\n"
            "bra BOWDB_WAIT1;\n"
            "BOWDB_DONE1:\n"
            "}\n" ::"r"(smem_u32(&bar))
            : "memory");
        job_items<CSA, true, KFKF>(A, J0, sm, sm + (((size_t)smem_frame + 127) & ~size_t(127)) + (size_t)(tid >> 5) * BDB_WARP_BYTES);
        return;
    }
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        s_next = A.static_sched ? 0 : (int)((long long)blockIdx.x * A.n_jobs / gridDim.x); s_left = A.n_jobs; s_loads = 0;
    }
    while (true) {
        if (tid == 0) {
            int pick = -1, next = s_next, left = s_left;
            for (; left > 0 && pick < 0; left--) {
                const int* c = A.jobs[next].ctr;
                if (A.static_sched || *(volatile const int*)c < *(volatile const int*)(c + 1)) pick = next;
                next = next + 1 == A.n_jobs ? 0 : next + 1;
            }
            s_next = next; s_left = left; s_job = pick;
            if (pick >= 0) sJ = A.jobs[pick];
        }
        __syncthreads();
        uint8_t* ws = sm + (((size_t)smem_frame + 127) & ~size_t(127)) + (size_t)(tid >> 5) * BDB_WARP_BYTES;
        if (s_job < 0) break;
        if (sJ.frame_in_smem) {
            if (tid == 0) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");          // the previous block was read through the generic proxy
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar)), "r"((uint32_t)sJ.frame_bytes) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(smem_u32(sm)), "l"(reinterpret_cast<uint64_t>(sJ.frame_block)), "r"((uint32_t)sJ.frame_bytes), "r"(smem_u32(&bar))
                             : "memory");
            }
            asm volatile(
                "{\n"
                ".reg .pred p;\n"
                "BOWDB_WAIT:\n"
                "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
                "@p bra BOWDB_DONE;\n"
                "bra BOWDB_WAIT;\n"
                "BOWDB_DONE:\n"
                "}\n" ::"r"(smem_u32(&bar)), "r"((uint32_t)s_loads & 1u)
                : "memory");
            job_items<CSA, true, KFKF>(A, sJ, sm, ws);
        } else {
            job_items<CSA, false, KFKF>(A, sJ, sJ.frame_block, ws);
        }
        __syncthreads();                                          // every warp is done with this job's block
        if (tid == 0 && sJ.frame_in_smem) s_loads++;
    }
}
template <int CSA, int KIND>
__global__ void __launch_bounds__(32 * BDB_WARPS, BDB_CTAS) bowdb_match_kernel(BowDbArgs A, int smem_frame, const __grid_constant__ BowDbJob J0) {
    bowdb_match<CSA, KIND, false>(A, smem_frame, J0);
}
// One distance arithmetic (MODE 2, the default) only: borb_debug_set_bow_csa applies to bowdb_match_kernel.
template <int KIND>
__global__ void __launch_bounds__(32 * BDB_WARPS, BDB_CTAS) bowkf_match_kernel(BowDbArgs A, int smem_frame, const __grid_constant__ BowDbJob J0) {
    bowdb_match<2, KIND, true>(A, smem_frame, J0);
}

// Rotation-consistency cull and compaction, a 128-thread CTA per keyframe.  table_out row: one u32 per frame position
// (FeatureVector order): keyframe feature | bin << 16, or 0xFFFFFFFF.  Survivors are written in frame-position order.
// A warp owns a contiguous quarter of the row (its entries stay in registers between the passes when the row has at most
// FIN_THREADS * FIN_REG positions), so the ordered compaction needs ballots and ONE block-level exchange of the warp totals.
constexpr int FIN_THREADS = 128;
constexpr int FIN_REG = 16;
__global__ void __launch_bounds__(FIN_THREADS) bowdb_finalize_kernel(BowDbArgs A) {
    __shared__ int hist[32];
    __shared__ int warp_cnt[FIN_THREADS / 32];
    __shared__ int s_off, s_i1, s_i2, s_i3, s_job;
    const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
    if (tid == 0) {                                                       // the job of this CTA: largest j with kf_base <= blockIdx.x
        int lo = 0, hi = A.n_jobs;
        while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (A.jobs[mid].kf_base <= (int)blockIdx.x) lo = mid; else hi = mid; }
        s_job = lo;
    }
    __syncthreads();
    const BowDbJob& J = A.jobs[s_job];
    const int k = blockIdx.x - J.kf_base, mf = J.m;
    const uint16_t* forig = reinterpret_cast<const uint16_t*>(J.frame_block + frame_block_layout(J.nn, mf, J.n).off_orig);
    if (tid < 32) hist[tid] = J.hist_out[(size_t)k * 32 + tid];              // rotation histogram accumulated by the match kernel
    const uint32_t* row = J.table_out + (size_t)k * mf;
    const int per_warp = (((mf + FIN_THREADS / 32 - 1) / (FIN_THREADS / 32)) + 31) & ~31;      // positions per warp, whole 32-steps
    const int w0 = wrp * per_warp, w1 = min(mf, w0 + per_warp);
    const bool in_regs = per_warp <= 32 * FIN_REG;
    const bool need_rows = J.pairs != nullptr || J.dense != nullptr;
    uint32_t e[FIN_REG];
#pragma unroll
    for (int t = 0; t < FIN_REG; t++) {
        const int i = w0 + t * 32 + lane;
        e[t] = (need_rows && in_regs && i < w1) ? row[i] : 0xFFFFFFFFu;
    }
    __syncthreads();
    if (tid == 0) {
        int i1 = -1, i2 = -1, i3 = -1, kept = 0;
        if (A.check_ori) {
            three_maxima(hist, i1, i2, i3);
            for (int b = 0; b < HISTO_LENGTH; b++) if (b == i1 || b == i2 || b == i3) kept += hist[b];
        } else {
            for (int b = 0; b < 32; b++) kept += hist[b];
        }
        const int off = J.pairs ? atomicAdd(J.ctr + 2, kept) : 0;
        J.n_matches[k] = kept;                                           // nmatches after the cull (:267-285)
        if (J.pair_off) J.pair_off[k] = off;
        s_off = off; s_i1 = i1; s_i2 = i2; s_i3 = i3;
    }
    __syncthreads();
    if (!J.pairs && !J.dense) return;
    const int i1 = s_i1, i2 = s_i2, i3 = s_i3;
    auto kept_entry = [&](uint32_t v) -> bool {
        if (v == 0xFFFFFFFFu) return false;
        if (!A.check_ori) return true;
        const int b = (int)((v >> 16) & 31);
        return b == i1 || b == i2 || b == i3;
    };
    // survivors per warp
    int mine = 0;
    if (in_regs) {
#pragma unroll
        for (int t = 0; t < FIN_REG; t++) mine += kept_entry(e[t]) ? 1 : 0;
    } else {
        for (int i = w0 + lane; i < w1; i += 32) mine += kept_entry(row[i]) ? 1 : 0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xFFFFFFFFu, mine, o);
    if (lane == 0) warp_cnt[wrp] = mine;
    __syncthreads();
    int run = s_off;
    for (int w = 0; w < wrp; w++) run += warp_cnt[w];
    auto emit = [&](uint32_t v, int i) {
        const bool keep = kept_entry(v);
        const unsigned bal = __ballot_sync(0xFFFFFFFFu, keep);
        if (keep) {
            const int j = (int)forig[i], r = (int)(v & 0xFFFFu);
            if (J.pairs) { const int pos = run + __popc(bal & ((1u << lane) - 1)); if (pos < J.pairs_cap) J.pairs[pos] = (uint32_t)j | ((uint32_t)r << 16); }
            if (J.dense) J.dense[(size_t)k * J.dense_stride + j] = r;
        }
        run += __popc(bal);
    };
    if (in_regs) {
#pragma unroll
        for (int t = 0; t < FIN_REG; t++) emit(e[t], w0 + t * 32 + lane);
    } else {
        for (int i0 = w0; i0 < w1; i0 += 32) { const int i = i0 + lane; emit(i < w1 ? row[i] : 0xFFFFFFFFu, i); }
    }
}

// Warps per CTA: as many as fit beside the query frame in one SM's shared memory (one CTA per SM), at least 8.
static int bowdb_warps(int frame_bytes, bool fsm) {
    const size_t frame = fsm ? (((size_t)frame_bytes + 127) & ~size_t(127)) : 0;
    const size_t budget = 226 * 1024;
    if (frame + 8 * (size_t)BDB_WARP_BYTES > budget) return 0;
    const int w = (int)((budget - frame) / BDB_WARP_BYTES);
    return w > BDB_WARPS ? BDB_WARPS : w;
}

bool bowdb_frame_fits_smem(int frame_bytes) { return bowdb_warps(frame_bytes, true) >= 8; }

// The query frame's block (FrameBlockHdr + sections), one CTA per job: the FeatureVector's node and start arrays; orig, angle and
// desc of every feature inside a node in FeatureVector order; and the work list - the non-empty nodes stable-sorted widest first
// (the long items start first), keyframes per item cs = clamp(item_target / nt^2, 1, 32) so that an item is a few hundred
// column-loop iterations whatever the bucket width (a keyframe's bucket of the node is about as full as the frame's), and the
// item prefix pstart.  Also resets the job's work counter and pair cursor and stores its item count next to them.
// Shared memory: 8 B per sort key (next power of two >= nn, at least 32).
// KFKF: the query is a database slot; its stream rows are already in FeatureVector order, with the feature index and angle in
// q_meta, so row r is copied as it is.
constexpr int PACK_THREADS = 512;
template <bool KFKF>
__device__ __forceinline__ void bowdb_pack(const BowDbJob* __restrict__ jobs) {
    extern __shared__ __align__(16) uint64_t pk_sm[];
    __shared__ int warp_sums[PACK_THREADS / 32];
    __shared__ int s_np;
    const BowDbJob& J = jobs[blockIdx.x];
    const int tid = threadIdx.x, T = blockDim.x, lane = tid & 31, wrp = tid >> 5;
    const int nn = J.nn, m = J.m;
    FrameBlockHdr h = frame_block_layout(nn, m, J.n);
    uint8_t* dst = J.frame_block;
    uint32_t* node = reinterpret_cast<uint32_t*>(dst + h.off_node);
    int32_t* start = reinterpret_cast<int32_t*>(dst + h.off_start);
    uint16_t* orig = reinterpret_cast<uint16_t*>(dst + h.off_orig);
    float* angle = reinterpret_cast<float*>(dst + h.off_angle);
    uint4* desc = reinterpret_cast<uint4*>(dst + h.off_desc);
    const uint4* src = reinterpret_cast<const uint4*>(J.desc);
    for (int i = tid; i < nn; i += T) node[i] = J.fv_node[i];
    for (int i = tid; i <= nn; i += T) start[i] = nn > 0 ? J.fv_start[i] : 0;
    for (int t = tid; t < 2 * m; t += T) {                                // a thread per descriptor half
        const int r = t >> 1;
        if constexpr (KFKF) {
            desc[t] = src[t];
            if ((t & 1) == 0) { const uint2 mt = J.q_meta[r]; orig[r] = (uint16_t)(mt.x & 0xFFFFu); angle[r] = __uint_as_float(mt.y); }
        } else {
            const uint32_t j = J.fv_idx[r];
            desc[t] = src[(size_t)j * 2 + (t & 1)];
            if ((t & 1) == 0) { orig[r] = (uint16_t)j; angle[r] = J.keys[j].angle; }
        }
    }
    // work list: (widest first, then node index) as one ascending 64-bit key; empty nodes sort last
    int K = 32;
    while (K < nn) K <<= 1;
    uint64_t* keys = pk_sm;
    int mine = 0;
    for (int i = tid; i < K; i += T) {
        const int w = i < nn ? J.fv_start[i + 1] - J.fv_start[i] : 0;
        keys[i] = w > 0 ? ((uint64_t)(0xFFFFFFFFu - (uint32_t)w) << 32) | (uint32_t)i : ~0ull;
        mine += w > 0;
    }
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xFFFFFFFFu, mine, o);
    if (lane == 0) warp_sums[wrp] = mine;
    __syncthreads();
    if (tid == 0) { int a = 0; for (int w = 0; w < T / 32; w++) a += warp_sums[w]; s_np = a; }
    bitonic_sort_u64(keys, K);                                            // starts and ends with a barrier: s_np is visible
    const int np = s_np;                                                  // non-empty nodes
    int32_t* pnode = reinterpret_cast<int32_t*>(dst + h.off_pnode);
    int32_t* pcs = reinterpret_cast<int32_t*>(dst + h.off_pcs);
    int32_t* pstart = reinterpret_cast<int32_t*>(dst + h.off_pstart);
    // each thread owns a contiguous chunk of the list: its item count, then an exclusive scan of the chunk totals
    const int chunk = (np + T - 1) / T, c0 = min(np, tid * chunk), c1 = min(np, c0 + chunk);
    int items = 0;
    for (int p = c0; p < c1; p++) {
        const int a = (int)(uint32_t)keys[p];
        const long long nt = J.fv_start[a + 1] - J.fv_start[a];
        long long cs = J.item_target / (nt * nt);
        cs = cs < 1 ? 1 : (cs > 32 ? 32 : cs);                            // one 32-lane batch of keyframes per item at most
        pnode[p] = a; pcs[p] = (int32_t)cs;
        items += (int)((J.n_kf + cs - 1) / cs);
    }
    int incl = items;
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) warp_sums[wrp] = incl;
    __syncthreads();
    int before = incl - items, total = 0;
    for (int w = 0; w < T / 32; w++) { const int v = warp_sums[w]; if (w < wrp) before += v; total += v; }
    for (int p = c0; p < c1; p++) { pstart[p] = before; before += (int)((J.n_kf + pcs[p] - 1) / pcs[p]); }
    if (tid == 0) {
        pstart[np] = total;
        h.np = np;
        *reinterpret_cast<FrameBlockHdr*>(dst) = h;
        J.ctr[0] = 0; J.ctr[1] = total; J.ctr[2] = 0;
    }
}
__global__ void __launch_bounds__(PACK_THREADS) bowdb_pack_kernel(const BowDbJob* __restrict__ jobs) { bowdb_pack<false>(jobs); }
__global__ void __launch_bounds__(PACK_THREADS) bowkf_pack_kernel(const BowDbJob* __restrict__ jobs) { bowdb_pack<true>(jobs); }

int launch_bowdb(const BowDbArgs& A, const BowDbJob& one, int max_smem_frame, long long max_items, int total_kf, int max_nn, int csa, int n_sm,
                 bool kfkf, cudaStream_t s) {
    int K = 32;
    while (K < max_nn) K <<= 1;
    void (*pack)(const BowDbJob*) = kfkf ? bowkf_pack_kernel : bowdb_pack_kernel;
    allow_max_smem((const void*)pack);
    pack<<<A.n_jobs, PACK_THREADS, (size_t)K * 8, s>>>(A.jobs);
    const bool fsm = max_smem_frame > 0;
    const int warps = bowdb_warps(max_smem_frame, fsm);
    const size_t smem = (fsm ? (((size_t)max_smem_frame + 127) & ~size_t(127)) : 0) + (size_t)warps * BDB_WARP_BYTES;
    long long ctas = (max_items + warps - 1) / warps;
    if (ctas > n_sm * BDB_CTAS) ctas = n_sm * BDB_CTAS;
    if (ctas < 1) ctas = 1;
    // one job: passed as a parameter; its block decides the frame's memory
    const int kind = A.n_jobs > 1 ? TABLE : (one.frame_in_smem ? ONE_SMEM : ONE_GLOBAL);
    void (*kern)(BowDbArgs, int, BowDbJob) = nullptr;
    if (kfkf) kern = kind == TABLE ? bowkf_match_kernel<TABLE> : (kind == ONE_SMEM ? bowkf_match_kernel<ONE_SMEM> : bowkf_match_kernel<ONE_GLOBAL>);
    else switch (csa * 3 + kind) {
        case 0: kern = bowdb_match_kernel<0, ONE_SMEM>; break;
        case 1: kern = bowdb_match_kernel<0, ONE_GLOBAL>; break;
        case 2: kern = bowdb_match_kernel<0, TABLE>; break;
        case 3: kern = bowdb_match_kernel<1, ONE_SMEM>; break;
        case 4: kern = bowdb_match_kernel<1, ONE_GLOBAL>; break;
        case 5: kern = bowdb_match_kernel<1, TABLE>; break;
        case 6: kern = bowdb_match_kernel<2, ONE_SMEM>; break;
        case 7: kern = bowdb_match_kernel<2, ONE_GLOBAL>; break;
        default: kern = bowdb_match_kernel<2, TABLE>; break;
    }
    allow_max_smem((const void*)kern);
    kern<<<(int)ctas, 32 * warps, smem, s>>>(A, fsm ? max_smem_frame : 0, one);
    bowdb_finalize_kernel<<<total_kf, FIN_THREADS, 0, s>>>(A);
    return 3;
}

// KeyFrameDatabase::add of a resident frame with its BoW (borb_kfdb_add_frames), a CTA per job: the block that borb_kfdb_add packs
// on the host, byte for byte (kfdb_block_layout; every byte outside the sections is written 0).  Row r of the FeatureVector holds
// feature j = fv_idx[r] of node a, the largest a with fv_start[a] <= r; its record is {j | has_mp[j] != 0 << 16 | a << 17, bits of
// mvKeysUn[j].angle}, and its descriptor is gathered as two uint4, a thread per half, as bowdb_pack does.  The records also go to
// meta_out, the host's copy.
constexpr int INSERT_THREADS = 256;
__global__ void __launch_bounds__(INSERT_THREADS) kfdb_insert_kernel(const KfdbInsertJob* __restrict__ jobs) {
    const KfdbInsertJob& J = jobs[blockIdx.x];
    const int tid = threadIdx.x, T = blockDim.x;
    const int nn = J.nn, m = J.m, nb = J.n_bow;
    const KfdbBlock L = kfdb_block_layout(nn, m, nb);
    uint8_t* blk = J.block;
    auto zero = [&](size_t lo, size_t hi) { for (size_t i = lo + tid; i < hi; i += T) blk[i] = 0; };
    zero(L.node + (size_t)nn * 4, L.start);
    zero(L.start + (size_t)(nn + 1) * 4, L.meta);
    zero(L.meta + (size_t)m * 8, L.desc);
    zero(L.desc + (size_t)m * 32, L.bow_word);
    zero(L.bow_word + (size_t)nb * 4, L.bow_value);
    zero(L.bow_value + (size_t)nb * 8, L.bytes);
    uint32_t* node = reinterpret_cast<uint32_t*>(blk + L.node);
    int32_t* start = reinterpret_cast<int32_t*>(blk + L.start);
    uint2* meta = reinterpret_cast<uint2*>(blk + L.meta);
    uint4* desc = reinterpret_cast<uint4*>(blk + L.desc);
    const uint4* src = reinterpret_cast<const uint4*>(J.desc);
    for (int i = tid; i < nn; i += T) node[i] = J.fv_node[i];
    for (int i = tid; i <= nn; i += T) start[i] = nn > 0 ? J.fv_start[i] : 0;
    for (int t = tid; t < 2 * m; t += T) {
        const int r = t >> 1;
        const uint32_t j = J.fv_idx[r];
        desc[t] = src[(size_t)j * 2 + (t & 1)];
        if ((t & 1) == 0) {
            int lo = 0, hi = nn;                                  // the row's node: largest a with fv_start[a] <= r
            while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (J.fv_start[mid] <= r) lo = mid; else hi = mid; }
            const uint32_t good = (J.has_mp && J.has_mp[j]) ? 0x10000u : 0u;
            const uint2 rec = make_uint2(j | good | ((uint32_t)lo << 17), __float_as_uint(J.keys[j].angle));
            meta[r] = rec;
            J.meta_out[r] = rec;
        }
    }
    uint32_t* bw = reinterpret_cast<uint32_t*>(blk + L.bow_word);
    double* bv = reinterpret_cast<double*>(blk + L.bow_value);
    for (int i = tid; i < nb; i += T) { bw[i] = J.bow_word[i]; bv[i] = J.bow_value[i]; }
}

int launch_kfdb_insert(const KfdbInsertJob* d_jobs, int n_jobs, cudaStream_t s) {
    if (n_jobs <= 0) return 0;
    kfdb_insert_kernel<<<n_jobs, INSERT_THREADS, 0, s>>>(d_jobs);
    return 1;
}

}  // namespace borb
