// Hamming-distance matchers of the ORB front-end (reference src/ORBmatcher.cc) and the BoW feeder.
//
//   grid_sort_kernel      Frame::AssignFeaturesToGrid (src/Frame.cc:230-245): (cell, insertion) order by a bitonic sort in shared
//       memory.  The windowed search itself (GetFeaturesInArea + claim resolution) lives in k_proj.cu.
//   project_points_kernel the pose projections / frustum tests that feed it (src/ORBmatcher.cc:290-403,1328-1599, src/Frame.cc:269-325).
//   bow_match_kernel      SearchByBoW(KeyFrame*,Frame&) (:159-288) and SearchByBoW(KeyFrame*,KeyFrame*) (:522-655) over a
//       table of pairs: a CTA per (keyframe, target) pair deals the FeatureVector nodes to 8 warps (a feature lives in
//       exactly one node, so the greedy "already claimed" skip, :209/:576, never crosses nodes); per node the distance matrix is
//       computed with all lanes busy, then the rows are replayed in order; rotation-histogram cull (:267-285) at the end.
//       (The database-resident search of one frame against thousands of keyframes is k_bowdb.cu.)
//   triangulation_kernel  SearchForTriangulation (:657-823) over a table of jobs, a CTA per job: no sequential dependence
//       (vbMatched2 is never set in the reference), "dist<=bestDist, later wins" == min over (distance, -position); epipolar
//       tests as :140-157.
//   bow_transform_kernel  TemplatedVocabulary::transform (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1218-1259):
//       a warp per descriptor descends the tree, lanes = children, first-wins argmin (bow_transform_batch_kernel: the same
//       descent for many resident frames, grid.y = frame).
//   bow_build_kernel      the BowVector / FeatureVector bookkeeping of transform (:1150-1194) on the device, a CTA per frame.
//   match_math_probe_kernel  tests only (borb_debug_eval_math): glibc_logf and predict_scale on given inputs, swept over every
//       input against glibc and MapPoint::PredictScale by tests/test_gpu_device_math.py.
// All float tests use _rn intrinsics (no FMA contraction) so comparisons match the reference bit for bit.
//
// Bound: latency / POPC issue (15 thread-ops/clk/SM measured); the batch (map points, keyframes) supplies parallelism.
#include "borb_match.h"

namespace borb {

namespace {

constexpr int HISTO_LENGTH = 30;

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

// ORBmatcher::ComputeThreeMaxima (:1601-1642) on bin counts
__device__ void three_maxima(const int* cnt, int& ind1, int& ind2, int& ind3) {
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

__device__ __forceinline__ unsigned warp_min(unsigned v) {
    return __reduce_min_sync(0xFFFFFFFFu, v);        // REDUX: one instruction instead of a 5-step shuffle chain (the replays are latency chains)
}

}  // namespace

// ------------------------------------------------------------------------------------------------ grid
// One CTA: sorts (cell, feature index) keys in shared memory; writes cell_start[GRID_CELLS+1] and cell_idx[] in
// (cell, insertion) order — the layout of Frame::mGrid[x][y] (cell = x*48 + y).
__global__ void __launch_bounds__(1024) grid_sort_kernel(const borb_keypoint* __restrict__ keys, int n, float minX, float minY,
                                                         float invW, float invH, int K, int* __restrict__ cell_start,
                                                         int* __restrict__ cell_idx) {
    extern __shared__ uint32_t skeys[];
    const int tid = threadIdx.x, T = blockDim.x;
    for (int i = tid; i < K; i += T) {
        uint32_t key = 0xFFFFFFFFu;
        if (i < n) {
            const int px = (int)roundf(__fmul_rn(__fsub_rn(keys[i].x, minX), invW));   // PosInGrid (Frame.cc:384-385)
            const int py = (int)roundf(__fmul_rn(__fsub_rn(keys[i].y, minY), invH));
            if (px >= 0 && px < GRID_COLS && py >= 0 && py < GRID_ROWS) key = ((uint32_t)(px * GRID_ROWS + py) << 16) | (uint32_t)i;
        }
        skeys[i] = key;
    }
    __syncthreads();
    for (int kk = 2; kk <= K; kk <<= 1)
        for (int j = kk >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < K; i += T) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const bool asc = (i & kk) == 0;
                    const uint32_t a = skeys[i], b = skeys[ixj];
                    if ((a > b) == asc) { skeys[i] = b; skeys[ixj] = a; }
                }
            }
            __syncthreads();
        }
    for (int r = tid; r < K; r += T) {
        const uint32_t key = skeys[r];
        const int cell = key == 0xFFFFFFFFu ? GRID_CELLS : (int)(key >> 16);
        const int prev = r == 0 ? -1 : (skeys[r - 1] == 0xFFFFFFFFu ? GRID_CELLS : (int)(skeys[r - 1] >> 16));
        if (key != 0xFFFFFFFFu) cell_idx[r] = (int)(key & 0xFFFFu);
        for (int c = prev + 1; c <= cell && c <= GRID_CELLS; c++) cell_start[c] = r;
        if (r == K - 1 && cell < GRID_CELLS)
            for (int c = cell + 1; c <= GRID_CELLS; c++) cell_start[c] = K;
    }
}

// ------------------------------------------------------------------------------------------------ projection
// (candidate enumeration and claim resolution: k_proj.cu)

// glibc (>= 2.28) logf for positive normal finite x — the function MapPoint::PredictScale calls (src/MapPoint.cc:393,410;
// `log` resolves to the float overload).  ARM optimized-routines algorithm in double; the device function itself is compared
// with glibc for every positive normal float, and predict_scale for every float ratio, through match_math_probe_kernel
// (tests/test_gpu_device_math.py, DESIGN.md).
struct LogfTab { double invc[16], logc[16]; double ln2, a0, a1, a2; };
__device__ const LogfTab d_logf = {
    {0x1.661ec79f8f3bep+0, 0x1.571ed4aaf883dp+0, 0x1.49539f0f010bp+0, 0x1.3c995b0b80385p+0, 0x1.30d190c8864a5p+0, 0x1.25e227b0b8eap+0,
     0x1.1bb4a4a1a343fp+0, 0x1.12358f08ae5bap+0, 0x1.0953f419900a7p+0, 0x1p+0, 0x1.e608cfd9a47acp-1, 0x1.ca4b31f026aap-1,
     0x1.b2036576afce6p-1, 0x1.9c2d163a1aa2dp-1, 0x1.886e6037841edp-1, 0x1.767dcf5534862p-1},
    {-0x1.57bf7808caadep-2, -0x1.2bef0a7c06ddbp-2, -0x1.01eae7f513a67p-2, -0x1.b31d8a68224e9p-3, -0x1.6574f0ac07758p-3,
     -0x1.1aa2bc79c81p-3, -0x1.a4e76ce8c0e5ep-4, -0x1.1973c5a611cccp-4, -0x1.252f438e10c1ep-5, 0x0p+0, 0x1.aa5aa5df25984p-5,
     0x1.c5e53aa362eb4p-4, 0x1.526e57720db08p-3, 0x1.bc2860d22477p-3, 0x1.1058bc8a07ee1p-2, 0x1.4043057b6ee09p-2},
    0x1.62e42fefa39efp-1, -0x1.00ea348b88334p-2, 0x1.5575b0be00b6ap-2, -0x1.ffffef20a4123p-2};

__device__ __forceinline__ float glibc_logf(float x) {
    const uint32_t ix = __float_as_uint(x);
    if (ix == 0x3f800000u) return 0.f;
    const uint32_t tmp = ix - 0x3f330000u;
    const int i = (tmp >> 19) & 15;
    const int k = (int)tmp >> 23;
    const uint32_t iz = ix - (tmp & (0x1ffu << 23));
    const double z = (double)__uint_as_float(iz);
    const double r = __dsub_rn(__dmul_rn(z, d_logf.invc[i]), 1.0);
    const double y0 = __dadd_rn(d_logf.logc[i], __dmul_rn((double)k, d_logf.ln2));
    const double r2 = __dmul_rn(r, r);
    double y = __dadd_rn(__dmul_rn(d_logf.a1, r), d_logf.a2);
    y = __dadd_rn(__dmul_rn(d_logf.a0, r2), y);
    y = __dadd_rn(__dmul_rn(y, r2), __dadd_rn(y0, r));
    return (float)y;
}

// MapPoint::PredictScale (src/MapPoint.cc:385-417)
__device__ __forceinline__ int predict_scale(float max_distance, float dist, float log_scale, int n_levels) {
    const float ratio = __fdiv_rn(max_distance, dist);
    const uint32_t ir = __float_as_uint(ratio);
    int nScale = 0;             // ratio <= 0, subnormal, inf or NaN: the reference's (int) conversion lands below 0 -> clamped to 0
    if (ir >= 0x00800000u && ir < 0x7f800000u) {
        const float q = ceilf(__fdiv_rn(glibc_logf(ratio), log_scale));
        nScale = q >= 2147483648.f || !(q == q) ? 0 : (q <= -2147483648.f ? 0 : (int)q);
    }
    if (nScale < 0) nScale = 0;
    else if (nScale >= n_levels) nScale = n_levels - 1;
    return nScale;
}

// Test probe (borb_debug_eval_math fn 3-4): the very glibc_logf / predict_scale that project_points_kernel inlines, compiled in
// this translation unit with its flags.  fn 3 logf(a) (defined for positive normal a); fn 4 PredictScale(max_distance = a,
// dist = b, log_scale, n_levels) as int32.
__global__ void match_math_probe_kernel(int fn, const float* __restrict__ a, const float* __restrict__ b, int n, float log_scale,
                                        int n_levels, void* __restrict__ out) {
    for (long long i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        if (fn == 3) static_cast<float*>(out)[i] = glibc_logf(a[i]);
        else static_cast<int*>(out)[i] = predict_scale(a[i], b[i], log_scale, n_levels);
    }
}

int launch_match_math_probe(int fn, const float* a, const float* b, int n, float log_scale, int n_levels, void* out,
                            cudaStream_t s) {
    match_math_probe_kernel<<<std::min((n + 255) / 256, 8192), 256, 0, s>>>(fn, a, b, n, log_scale, n_levels, out);
    return 1;
}

// Projection of query point i with the 3x4 pose, for the three SearchByProjection overloads that take world points and for
// Frame::isInFrustum.
__device__ __forceinline__ void project_point(const LastArgs& L, int i) {
    bool ok = L.valid_in == nullptr || L.valid_in[i] != 0;
    float u = 0.f, v = 0.f, ur = 0.f, radius = 0.f, ang = 0.f;
    int minl = 0, maxl = -1;
    if (ok) {
        const float* P = L.world_pos + 3 * (size_t)i;
        const float p0 = P[0], p1 = P[1], p2 = P[2];
        // cv::Mat 3x3 * 3x1 + 3x1 in float32: (r0*p0 + r1*p1) + r2*p2, then + t  (SURVEY a13)
        const float xc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(L.T[0], p0), __fmul_rn(L.T[1], p1)), __fmul_rn(L.T[2], p2)), L.T[3]);
        const float yc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(L.T[4], p0), __fmul_rn(L.T[5], p1)), __fmul_rn(L.T[6], p2)), L.T[7]);
        const float zc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(L.T[8], p0), __fmul_rn(L.T[9], p1)), __fmul_rn(L.T[10], p2)), L.T[11]);
        float q0 = xc, q1 = yc, q2 = zc;                                     // the point in the camera the features belong to
        if (L.variant == 2 && L.chain) {                                      // p3Dc2 = sR21*p3Dc1 + t21 (:1158)
            q0 = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(L.T2[0], xc), __fmul_rn(L.T2[1], yc)), __fmul_rn(L.T2[2], zc)), L.T2[3]);
            q1 = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(L.T2[4], xc), __fmul_rn(L.T2[5], yc)), __fmul_rn(L.T2[6], zc)), L.T2[7]);
            q2 = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(L.T2[8], xc), __fmul_rn(L.T2[9], yc)), __fmul_rn(L.T2[10], zc)), L.T2[11]);
        }
        if (L.variant == 3) {                                                 // Frame::isInFrustum (src/Frame.cc:269-325)
            if (zc < 0.0f) ok = false;
            const float invz = __fdiv_rn(1.0f, zc);                           // 1.0f/PcZ (:286)
            u = __fadd_rn(__fmul_rn(__fmul_rn(L.fx, xc), invz), L.cx);
            v = __fadd_rn(__fmul_rn(__fmul_rn(L.fy, yc), invz), L.cy);
            // no NaN test: at PcZ == 0 (a point at the camera centre) u and v are NaN and pass, as in the reference; the
            // track fields then hold NaN and the search window is empty (area_window)
            if (u < L.minX || u > L.maxX || v < L.minY || v > L.maxY) ok = false;
            ur = __fsub_rn(u, __fmul_rn(L.bf, invz));                         // mTrackProjXR (:319)
        } else if (L.variant == 2) {
            if (q2 < 0.0f) ok = false;                                        // depth must be positive (:329-330)
            const float invz = L.invz_double ? (float)(1.0 / (double)q2) : __fdiv_rn(1.0f, q2);   // (:1014,:1164) / (:333,:861)
            const float x = __fmul_rn(q0, invz), y = __fmul_rn(q1, invz);
            u = __fadd_rn(__fmul_rn(L.fx, x), L.cx);
            v = __fadd_rn(__fmul_rn(L.fy, y), L.cy);
            if (!(u >= L.minX && u < L.maxX && v >= L.minY && v < L.maxY)) ok = false;     // KeyFrame::IsInImage
            ur = __fsub_rn(u, __fmul_rn(L.bf, invz));                         // (:873)
        } else {
            const float invzc = (float)(1.0 / (double)zc);                   // 1.0/x3Dc.at<float>(2) (:1365, :1503)
            if (L.variant == 0 && invzc < 0) ok = false;                      // (:1367-1368); the keyframe overload has no such test
            u = __fadd_rn(__fmul_rn(__fmul_rn(L.fx, xc), invzc), L.cx);
            v = __fadd_rn(__fmul_rn(__fmul_rn(L.fy, yc), invzc), L.cy);
            if (u < L.minX || u > L.maxX || v < L.minY || v > L.maxY) ok = false;
            if (!(u == u) || !(v == v)) ok = false;                           // NaN never reaches a defined grid cell in the reference either
            ur = __fsub_rn(u, __fmul_rn(L.bf, invzc));
        }
        if (L.variant == 0) {
            const int oct = L.last_keys[i].octave;
            radius = __fmul_rn(L.th, L.scale_factors[oct]);
            if (L.forward) { minl = oct; maxl = -1; }
            else if (L.backward) { minl = 0; maxl = oct; }
            else { minl = oct - 1; maxl = oct + 1; }
            ang = L.last_keys[i].angle;
        } else if (ok) {
            // PO = p3Dw - Ow (float); cv::norm accumulates the squares in double, in index order
            const bool cam = L.variant == 2 && L.chain;                       // SearchBySim3: dist3D = cv::norm(p3Dc2) (:1177)
            const float o0 = cam ? q0 : __fsub_rn(p0, L.Ow[0]), o1 = cam ? q1 : __fsub_rn(p1, L.Ow[1]), o2 = cam ? q2 : __fsub_rn(p2, L.Ow[2]);
            const double d0 = o0, d1 = o1, d2 = o2;
            const float dist = (float)sqrt(__dadd_rn(__dadd_rn(__dmul_rn(d0, d0), __dmul_rn(d1, d1)), __dmul_rn(d2, d2)));
            const float mx = L.max_distance[i];
            const float maxD = __fmul_rn(1.2f, mx), minD = __fmul_rn(0.8f, L.min_distance[i]);
            if (dist < minD || dist > maxD) ok = false;
            if (ok && L.variant == 2 && L.use_normal) {                       // viewing angle below 60 degrees (:354-357)
                const float* N = L.normal + 3 * (size_t)i;
                const double dot = __dadd_rn(__dadd_rn(__dmul_rn(d0, (double)N[0]), __dmul_rn(d1, (double)N[1])), __dmul_rn(d2, (double)N[2]));
                if (dot < __dmul_rn(0.5, (double)dist)) ok = false;
            }
            float vcos = 0.f;
            if (ok && L.variant == 3) {                                       // viewCos = PO.dot(Pn)/dist (:305-308)
                const float* N = L.normal + 3 * (size_t)i;
                const double dot = __dadd_rn(__dadd_rn(__dmul_rn(d0, (double)N[0]), __dmul_rn(d1, (double)N[1])), __dmul_rn(d2, (double)N[2]));
                vcos = (float)__ddiv_rn(dot, (double)dist);
                if (vcos < L.view_cos_limit) ok = false;
            }
            if (ok) {
                const int lvl = predict_scale(mx, dist, L.log_scale, L.n_levels);
                radius = __fmul_rn(L.th, L.scale_factors[lvl]);
                minl = lvl - 1;
                maxl = L.variant == 1 ? lvl + 1 : lvl;
                if (L.variant == 3) { L.level_out[i] = lvl; L.viewcos_out[i] = vcos; }
            }
            ang = L.q_angle_in != nullptr ? L.q_angle_in[i] : 0.f;
        }
    }
    if (L.variant == 3 && !ok) { u = 0.f; v = 0.f; ur = 0.f; }              // the MapPoint's track fields stay untouched (reported as 0)
    L.proj_x[i] = u; L.proj_y[i] = v; L.proj_xr[i] = ur; L.radius[i] = radius; L.minl[i] = minl; L.maxl[i] = maxl;
    L.angle[i] = ang;
    L.valid_out[i] = ok ? 1 : 0;
}

__global__ void __launch_bounds__(256) project_points_kernel(LastArgs L) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < L.n_last) project_point(L, i);
}
// one launch for many independent jobs (borb_search_local_points_batch / borb_search_by_projection_last_batch): grid.y = job,
// the job's arguments come from device memory; a job without points has n_last = 0
__global__ void __launch_bounds__(256) project_points_batch_kernel(const LastArgs* __restrict__ jobs) {
    const LastArgs& L = jobs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < L.n_last) project_point(L, i);
}

// SearchForInitialization (:405-520): one warp replays F1's level-0 features in order.  A candidate i2 is skipped
// when an earlier feature already holds it with a distance <= ours (vMatchedDistance, :441-442); a better match
// displaces the earlier owner (:462-466).  vMatchedDistance / vnMatches21 live in shared memory.
__global__ void __launch_bounds__(32) init_resolve_kernel(ProjArgs A, const borb_keypoint* __restrict__ keys1, int n1,
                                                          int32_t* __restrict__ match12, int32_t* __restrict__ ev_idx,
                                                          uint8_t* __restrict__ ev_bin, float* __restrict__ prev, int* __restrict__ n_matches) {
    extern __shared__ uint32_t smem_init[];
    uint16_t* matchedDist = reinterpret_cast<uint16_t*>(smem_init);           // 0xFFFF = INT_MAX
    uint16_t* owner = matchedDist + ((A.n + 1) & ~1);                          // 0xFFFF = -1
    __shared__ int hist[32];
    const int lane = threadIdx.x;
    for (int i = lane; i < A.n; i += 32) { matchedDist[i] = 0xFFFFu; owner[i] = 0xFFFFu; }
    for (int i = lane; i < n1; i += 32) match12[i] = -1;
    hist[lane] = 0;
    __syncwarp();
    int nm = 0, nev = 0;
    for (int i1 = 0; i1 < n1; i1++) {
        const int cnt = A.cand_cnt[i1] & CAND_COUNT_MASK;
        if (cnt == 0) continue;
        const uint32_t* c = A.cand + (size_t)i1 * A.n;
        unsigned k1 = 0xFFFFFFFFu, k2 = 0xFFFFFFFFu;
        for (int p = lane; p < cnt; p += 32) {
            const uint32_t e = c[p];
            const unsigned dist = (e >> 16) & 0x1FFu;
            if ((unsigned)matchedDist[e & 0xFFFF] <= dist) continue;
            const unsigned key = (dist << 16) | (unsigned)p;
            if (key < k1) { k2 = k1; k1 = key; } else if (key < k2) k2 = key;
        }
        const unsigned best = warp_min(k1);
        const unsigned second = warp_min(k1 == best ? k2 : k1);
        if (best != 0xFFFFFFFFu) {
            const int bestDist = (int)(best >> 16);
            const float bd2 = second != 0xFFFFFFFFu ? (float)(int)(second >> 16) : 2147483648.f;      // (float)INT_MAX
            if (bestDist <= TH_LOW && (float)bestDist < __fmul_rn(bd2, A.nnratio)) {
                const int i2 = (int)(c[best & 0xFFFFu] & 0xFFFF);
                const int prevOwner = owner[i2];
                __syncwarp();                                    // every lane has read the owner before lane 0 replaces it
                if (prevOwner != 0xFFFF) nm--;
                nm++;
                if (lane == 0) {
                    if (prevOwner != 0xFFFF) match12[prevOwner] = -1;
                    match12[i1] = i2;
                    owner[i2] = (uint16_t)i1;
                    matchedDist[i2] = (uint16_t)bestDist;
                    if (A.check_ori) {
                        const int b = rot_bin(keys1[i1].angle, A.keys[i2].angle);
                        ev_idx[nev] = i1; ev_bin[nev] = (uint8_t)b;
                        hist[b]++;
                    }
                }
                nev++;
            }
        }
        __syncwarp();
    }
    if (A.check_ori) {
        int i1m, i2m, i3m;
        three_maxima(hist, i1m, i2m, i3m);
        int removed = 0;
        for (int e = lane; e < nev; e += 32) {                   // every F1 feature appears at most once in the histogram
            const int b = ev_bin[e];
            if (b != i1m && b != i2m && b != i3m && match12[ev_idx[e]] >= 0) { match12[ev_idx[e]] = -1; removed++; }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) removed += __shfl_xor_sync(0xFFFFFFFFu, removed, off);
        nm -= removed;
    }
    __syncwarp();
    for (int i = lane; i < n1; i += 32) {                        // update vbPrevMatched (:513-517)
        const int m = match12[i];
        if (m >= 0) { prev[2 * i] = A.keys[m].x; prev[2 * i + 1] = A.keys[m].y; }
    }
    if (lane == 0) *n_matches = nm;
}

// MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:242-307), batched: a warp per MapPoint, a lane per row of the
// distance matrix.  The row median (sorted row[(int)(0.5*(N-1))], self-distance included) comes from a 257-bin counting
// histogram kept in local memory; first minimal median wins (lowest row index).
__global__ void __launch_bounds__(128) distinctive_kernel(const uint8_t* __restrict__ desc, const int32_t* __restrict__ offsets,
                                                          int n_points, int32_t* __restrict__ best_idx) {
    const int lane = threadIdx.x & 31;
    const int pt = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (pt >= n_points) return;
    const int o0 = offsets[pt], N = offsets[pt + 1] - o0;
    if (N <= 0) { if (lane == 0) best_idx[pt] = -1; return; }
    const uint32_t* D = reinterpret_cast<const uint32_t*>(desc) + (size_t)o0 * 8;
    const int k = (int)(0.5 * (double)(N - 1));
    unsigned bestKey = 0xFFFFFFFFu;                              // median << 20 | row
    for (int i = lane; i < N; i += 32) {
        uint16_t hist[257];
#pragma unroll 1
        for (int b = 0; b < 257; b++) hist[b] = 0;
        uint32_t a[8];
#pragma unroll
        for (int w = 0; w < 8; w++) a[w] = D[(size_t)i * 8 + w];
#pragma unroll 1
        for (int j = 0; j < N; j++) {
            int d = 0;
#pragma unroll
            for (int w = 0; w < 8; w++) d += __popc(a[w] ^ D[(size_t)j * 8 + w]);
            hist[d]++;
        }
        int cum = 0, median = 256;
#pragma unroll 1
        for (int b = 0; b < 257; b++) {
            cum += hist[b];
            if (cum > k) { median = b; break; }
        }
        bestKey = min(bestKey, ((unsigned)median << 20) | (unsigned)i);
    }
    bestKey = warp_min(bestKey);
    if (lane == 0) best_idx[pt] = (int)(bestKey & 0xFFFFFu);
}

// KeyFrameDatabase query (src/KeyFrameDatabase.cc:76-197, 199-310): for every keyframe of the device-resident database,
// the number of words it shares with the query BowVector (what the inverted-file walk counts, :211-224) and
// DBoW2::L1Scoring::score (ScoringObject.cpp:23-71).  A warp per keyframe: lanes take 32 consecutive keyframe words,
// binary-search them in the query, and the matching terms are added in ascending word order (double, the order of the
// reference's merge loop) so that the score is bit-identical.
__global__ void __launch_bounds__(256) kfdb_score_kernel(const KfdbQueryJob* __restrict__ jobs, int in_smem) {
    extern __shared__ __align__(16) uint8_t kq_sm[];
    const KfdbQueryJob& J = jobs[blockIdx.y];                         // grid.y = job
    const int n_slots = J.n_slots, nq = J.nq;
    if ((int)blockIdx.x * (int)(blockDim.x >> 5) >= n_slots) return;  // the grid is sized for the largest database
    const int lane = threadIdx.x & 31;
    // the query BowVector is probed ~10 x per keyframe word: keep it in shared memory (values first: 8-byte aligned)
    const uint32_t* qword = J.qword;
    const double* qvalue = J.qvalue;
    if (in_smem) {
        double* sv = reinterpret_cast<double*>(kq_sm);
        uint32_t* sw = reinterpret_cast<uint32_t*>(sv + nq);
        for (int i = threadIdx.x; i < nq; i += blockDim.x) { sv[i] = J.qvalue[i]; sw[i] = J.qword[i]; }
        __syncthreads();
        qword = sw; qvalue = sv;
    }
    const BowDev* __restrict__ table = J.table;
    int32_t* __restrict__ common = J.common;
    float* __restrict__ score = J.score;
    uint32_t* __restrict__ first_word = J.first_word;
    const int warps_total = gridDim.x * (blockDim.x >> 5);
    const int steps = nq > 0 ? 32 - __clz(nq) : 0;                    // iterations that finish any lower_bound over nq entries
    constexpr int U = 8;                                              // keyframe words per lane in flight: the loads and the U searches overlap
    for (int slot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); slot < n_slots; slot += warps_total) {
        const BowDev kf = table[slot];
        double acc = 0.0;
        int ncommon = 0;
        uint32_t first = 0xFFFFFFFFu;
        for (int base = 0; base < kf.n; base += 32 * U) {
            uint32_t w[U];
            int lo[U], hi[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const int i = base + u * 32 + lane;
                w[u] = i < kf.n ? kf.word[i] : 0xFFFFFFFFu;
                lo[u] = 0; hi[u] = i < kf.n ? nq : 0;
            }
            for (int st = 0; st < steps; st++) {                      // lower_bound of w[u] in the query words, U searches interleaved
#pragma unroll
                for (int u = 0; u < U; u++) {
                    if (lo[u] < hi[u]) {
                        const int mid = (lo[u] + hi[u]) >> 1;
                        if (qword[mid] < w[u]) lo[u] = mid + 1; else hi[u] = mid;
                    }
                }
            }
            double term[U];
            bool found[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const int i = base + u * 32 + lane;
                found[u] = i < kf.n && lo[u] < nq && qword[lo[u]] == w[u];
                term[u] = 0.0;
                if (found[u]) {
                    const double vi = qvalue[lo[u]], wi = kf.value[i];   // v1 = query (F->mBowVec), v2 = keyframe
                    term[u] = __dsub_rn(__dsub_rn(fabs(__dsub_rn(vi, wi)), fabs(vi)), fabs(wi));
                }
            }
#pragma unroll
            for (int u = 0; u < U; u++) {
                unsigned bal = __ballot_sync(0xFFFFFFFFu, found[u]);
                if (bal && first == 0xFFFFFFFFu) first = __shfl_sync(0xFFFFFFFFu, w[u], __ffs(bal) - 1);
                ncommon += __popc(bal);
                while (bal) {                                         // ordered accumulation: ascending word id
                    const int src = __ffs(bal) - 1;
                    bal &= bal - 1;
                    acc = __dadd_rn(acc, __shfl_sync(0xFFFFFFFFu, term[u], src));
                }
            }
        }
        if (lane == 0) {
            common[slot] = ncommon;
            score[slot] = (float)(-acc / 2.0);                        // float si = mpVoc->score(...) (:240)
            first_word[slot] = first;
        }
    }
}

// ------------------------------------------------------------------------------------------------ BoW guided search
// mode 0: SearchByBoW(KeyFrame*, Frame&)   — q = keyframe (needs has_mp), t = frame;   out match[t.n]  = q index
// mode 1: SearchByBoW(KeyFrame*, KeyFrame*) — q = kf1, t = kf2 (both need has_mp);      out match[q.n]  = t index
// Per shared node the nq x nt distance matrix is computed first, all lanes busy and all loads in flight at once
// (the greedy claim makes the ROWS sequential, not the distances); the replay then walks the rows over the
// matrix in shared memory.  BOW_DCAP matrix entries per warp; wider nodes are processed in row chunks.
constexpr int BOW_WARPS = 8;        // warps per (keyframe, frame) pair: FeatureVector nodes are independent (a feature lives in
                                    // exactly one node, so claims never cross nodes) and are dealt round-robin to the warps
constexpr int BOW_DCAP = 1024;      // distance-matrix entries per warp
constexpr int BOW_JCAP = 1024;      // widest target bucket the matrix path handles; beyond it rows fall back to direct evaluation
constexpr int BOW_RCAP = 256;       // rows per chunk
constexpr int BOW_WARP_WORDS = BOW_DCAP / 2 + BOW_JCAP / 2 + BOW_RCAP / 2;

// A CTA per pair: pair p searches qs[p] against ts[p] and writes its match (and rotation bins) at out_off[p].
__global__ void __launch_bounds__(32 * BOW_WARPS) bow_match_kernel(const KfDev* __restrict__ qs, const KfDev* __restrict__ ts, int mode,
                                                                   float nnratio, int check_ori, int32_t* __restrict__ match,
                                                                   const size_t* __restrict__ out_off, uint8_t* __restrict__ bins,
                                                                   int32_t* __restrict__ n_matches, int max_t) {
    extern __shared__ uint32_t sm[];
    __shared__ int hist[32];
    __shared__ int nm_total;
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5, tid = threadIdx.x;
    const int pair = blockIdx.x;
    const int words = (max_t + 31) / 32;
    uint32_t* claimed = sm;                                                      // bit per target feature, shared by the CTA
    uint16_t* D = reinterpret_cast<uint16_t*>(sm + words + (size_t)wrp * BOW_WARP_WORDS);   // distances of the current row chunk
    uint16_t* J = D + BOW_DCAP;                                                  // target feature per column (0xFFFF = unusable)
    uint16_t* R = J + BOW_JCAP;                                                  // query feature per row of the chunk
    const KfDev q = qs[pair];
    const KfDev t = ts[pair];
    const size_t o0 = out_off[pair];
    int32_t* out = match + o0;
    uint8_t* bin = bins + o0;
    const int nout = mode == 0 ? t.n : q.n;
    for (int i = tid; i < nout; i += 32 * BOW_WARPS) out[i] = -1;
    for (int w = tid; w < words; w += 32 * BOW_WARPS) claimed[w] = 0;
    if (tid < 32) hist[tid] = 0;
    if (tid == 0) nm_total = 0;
    __syncthreads();
    int nm = 0;
    int lo = 0;                                                                  // merge-join cursor in the target's node list (:180-264)
    for (int a = wrp; a < q.nn; a += BOW_WARPS) {
        const uint32_t node = q.node[a];
        // advance the cursor to the first target node >= node: 32 nodes per probe
        while (lo < t.nn) {
            const int c = lo + lane;
            const unsigned ge = __ballot_sync(0xFFFFFFFFu, c >= t.nn || t.node[c] >= node);
            if (ge) { lo += __ffs(ge) - 1; break; }
            lo += 32;
        }
        if (lo >= t.nn) break;
        if (t.node[lo] != node) continue;
        const int ts0 = t.start[lo], nt = t.start[lo + 1] - ts0;
        const int qs0 = q.start[a], nq = q.start[a + 1] - qs0;
        if (nt <= 0 || nq <= 0) continue;
        const bool matrix = nt <= BOW_JCAP;
        __syncwarp();
        if (matrix) {
            for (int p = lane; p < nt; p += 32) {
                const int j = (int)t.idx[ts0 + p];
                J[p] = (mode == 1 && (t.has_mp == nullptr || !t.has_mp[j])) ? 0xFFFFu : (uint16_t)j;
            }
        }
        const int rows_per_chunk = matrix ? min(BOW_RCAP, max(1, BOW_DCAP / nt)) : BOW_RCAP;
        for (int r0 = 0; r0 < nq; r0 += rows_per_chunk) {
            const int nr = min(rows_per_chunk, nq - r0);
            __syncwarp();
            for (int i = lane; i < nr; i += 32) R[i] = (uint16_t)q.idx[qs0 + r0 + i];
            __syncwarp();
            if (matrix && nr * nt <= BOW_DCAP) {
                for (int e = lane; e < nr * nt; e += 32) {
                    const int i = e / nt, p = e - i * nt;
                    const int j = J[p];
                    D[e] = j == 0xFFFF ? (uint16_t)0x1FF
                                       : (uint16_t)ham_words(reinterpret_cast<const uint32_t*>(q.desc + (size_t)R[i] * 32),
                                                             reinterpret_cast<const uint32_t*>(t.desc + (size_t)j * 32));
                }
            }
            const bool have_d = matrix && nr * nt <= BOW_DCAP;                   // (a single row wider than the matrix is evaluated directly)
            __syncwarp();
            for (int g0 = 0; g0 < nr; g0 += 32) {
                // row metadata for 32 rows at once: one round of global latency instead of one per row
                const int il = g0 + lane;
                const int r_l = il < nr ? (int)R[il] : 0;
                const bool ok_l = il < nr && q.has_mp != nullptr && q.has_mp[r_l] != 0;
                const float ang_l = (ok_l && check_ori) ? q.keys[r_l].angle : 0.f;
                const unsigned okmask = __ballot_sync(0xFFFFFFFFu, ok_l);
                const int ng = min(32, nr - g0);
                for (int ii = 0; ii < ng; ii++) {
                    if (!((okmask >> ii) & 1u)) continue;
                    const int i = g0 + ii;
                    const int r = __shfl_sync(0xFFFFFFFFu, r_l, ii);
                    const float qa = __shfl_sync(0xFFFFFFFFu, ang_l, ii);
                    unsigned k1 = 0xFFFFFFFFu, k2 = 0xFFFFFFFFu;
                    if (have_d) {
                        for (int p = lane; p < nt; p += 32) {
                            const int j = J[p];
                            if (j == 0xFFFF || ((claimed[j >> 5] >> (j & 31)) & 1u)) continue;
                            const unsigned key = ((unsigned)D[i * nt + p] << 16) | (unsigned)p;
                            if (key < k1) { k2 = k1; k1 = key; } else if (key < k2) k2 = key;
                        }
                    } else {                                                      // bucket wider than the matrix: direct evaluation
                        const uint32_t* dq = reinterpret_cast<const uint32_t*>(q.desc + (size_t)r * 32);
                        for (int p = lane; p < nt; p += 32) {
                            const int j = (int)t.idx[ts0 + p];
                            if ((claimed[j >> 5] >> (j & 31)) & 1u) continue;
                            if (mode == 1 && (t.has_mp == nullptr || !t.has_mp[j])) continue;
                            const int dist = ham_words(dq, reinterpret_cast<const uint32_t*>(t.desc + (size_t)j * 32));
                            const unsigned key = ((unsigned)dist << 16) | (unsigned)p;
                            if (key < k1) { k2 = k1; k1 = key; } else if (key < k2) k2 = key;
                        }
                    }
                    const unsigned best = warp_min(k1);
                    const unsigned second = warp_min(k1 == best ? k2 : k1);
                    if (best == 0xFFFFFFFFu) continue;
                    const int bestDist1 = (int)(best >> 16);
                    const int bestDist2 = second == 0xFFFFFFFFu ? 256 : (int)(second >> 16);
                    const bool pass = mode == 0 ? (bestDist1 <= TH_LOW) : (bestDist1 < TH_LOW);
                    if (pass && (float)bestDist1 < __fmul_rn(nnratio, (float)bestDist2)) {
                        const int pb = (int)(best & 0xFFFFu);
                        const int j = (int)t.idx[ts0 + pb];
                        if (lane == 0) {
                            atomicOr(&claimed[j >> 5], 1u << (j & 31));          // other warps own other nodes' bits of the same word
                            const int o = mode == 0 ? j : r;
                            out[o] = mode == 0 ? r : j;
                            if (check_ori) {
                                const int b2 = rot_bin(qa, t.keys[j].angle);
                                bin[o] = (uint8_t)b2;
                                atomicAdd(&hist[b2], 1);
                            }
                        }
                        nm++;
                        __syncwarp();
                    }
                }
            }
        }
    }
    if (lane == 0 && nm) atomicAdd(&nm_total, nm);
    __threadfence_block();
    __syncthreads();
    if (wrp != 0) return;
    nm = nm_total;
    if (check_ori) {
        int i1, i2, i3;
        three_maxima(hist, i1, i2, i3);
        int removed = 0;
        for (int i = lane; i < nout; i += 32)
            if (out[i] >= 0) {
                const int b2 = bin[i];
                if (b2 != i1 && b2 != i2 && b2 != i3) { out[i] = -1; removed++; }
            }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) removed += __shfl_xor_sync(0xFFFFFFFFu, removed, off);
        nm -= removed;
    }
    if (lane == 0) n_matches[pair] = nm;
}

// ------------------------------------------------------------------------------------------------ triangulation
// A CTA per job (borb_search_for_triangulation is the one-job case); the rows of a job are independent, so warps take kf1's
// FeatureVector nodes round robin, and the job's pairs are compacted in idx1 order into its own region.
__global__ void __launch_bounds__(256) triangulation_kernel(const TriJob* __restrict__ jobs, int check_ori) {
    __shared__ int hist[32];
    __shared__ int top[3];
    __shared__ int wsum[9];
    const TriJob& T = jobs[blockIdx.x];
    const KfDev& q = T.q;
    const KfDev& t = T.t;
    int32_t* __restrict__ vmatch = T.vmatch;
    uint8_t* __restrict__ bins = T.bins;
    int32_t* __restrict__ pairs = T.pairs;
    const int cap = T.cap;
    const int tid = threadIdx.x, lane = tid & 31, wrp = tid >> 5;
    for (int i = tid; i < q.n; i += 256) vmatch[i] = -1;
    if (tid < 32) hist[tid] = 0;
    __syncthreads();
    for (int a = wrp; a < q.nn; a += 8) {
        const uint32_t node = q.node[a];
        int lo = 0, hi = t.nn;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (t.node[mid] < node) lo = mid + 1; else hi = mid; }
        if (lo >= t.nn || t.node[lo] != node) continue;
        const int ts0 = t.start[lo], ts1 = t.start[lo + 1];
        for (int iq = q.start[a]; iq < q.start[a + 1]; iq++) {
            const int i = (int)q.idx[iq];
            if (q.has_mp != nullptr && q.has_mp[i]) continue;              // already has a MapPoint (:699-703)
            const bool bStereo1 = q.u_right != nullptr && q.u_right[i] >= 0;
            if (T.only_stereo && !bStereo1) continue;
            const borb_keypoint kp1 = q.keys[i];
            const uint32_t* d1 = reinterpret_cast<const uint32_t*>(q.desc + (size_t)i * 32);
            // epipolar line of kp1 in image 2 (CheckDistEpipolarLine, :142-145)
            const float la = __fadd_rn(__fadd_rn(__fmul_rn(kp1.x, T.F[0]), __fmul_rn(kp1.y, T.F[3])), T.F[6]);
            const float lb = __fadd_rn(__fadd_rn(__fmul_rn(kp1.x, T.F[1]), __fmul_rn(kp1.y, T.F[4])), T.F[7]);
            const float lc = __fadd_rn(__fadd_rn(__fmul_rn(kp1.x, T.F[2]), __fmul_rn(kp1.y, T.F[5])), T.F[8]);
            const float den = __fadd_rn(__fmul_rn(la, la), __fmul_rn(lb, lb));
            unsigned bestKey = 0xFFFFFFFFu;
            for (int p = ts0 + lane; p < ts1; p += 32) {
                const int j = (int)t.idx[p];
                if (t.has_mp != nullptr && t.has_mp[j]) continue;
                const bool bStereo2 = t.u_right != nullptr && t.u_right[j] >= 0;
                if (T.only_stereo && !bStereo2) continue;
                const int dist = ham_words(d1, reinterpret_cast<const uint32_t*>(t.desc + (size_t)j * 32));
                if (dist > TH_LOW) continue;
                const borb_keypoint kp2 = t.keys[j];
                if (!bStereo1 && !bStereo2) {
                    const float distex = __fsub_rn(T.ex, kp2.x), distey = __fsub_rn(T.ey, kp2.y);
                    if (__fadd_rn(__fmul_rn(distex, distex), __fmul_rn(distey, distey)) < __fmul_rn(100.0f, t.scale_factors[kp2.octave])) continue;
                }
                const float num = __fadd_rn(__fadd_rn(__fmul_rn(la, kp2.x), __fmul_rn(lb, kp2.y)), lc);
                if (den == 0) continue;
                const float dsqr = __fdiv_rn(__fmul_rn(num, num), den);
                if (!((double)dsqr < 3.84 * (double)t.level_sigma2[kp2.octave])) continue;
                // "dist <= bestDist, later wins" (:738-755)  ==  min over (dist, -position)
                bestKey = min(bestKey, ((unsigned)dist << 16) | (unsigned)(0xFFFF - (p - ts0)));
            }
            bestKey = warp_min(bestKey);
            if (bestKey != 0xFFFFFFFFu && lane == 0) {
                const int j = (int)t.idx[ts0 + (0xFFFF - (int)(bestKey & 0xFFFFu))];
                vmatch[i] = j;
                if (check_ori) {
                    const int b = rot_bin(kp1.angle, t.keys[j].angle);
                    bins[i] = (uint8_t)b;
                    atomicAdd(&hist[b], 1);
                }
            }
        }
    }
    __syncthreads();
    if (check_ori) {
        if (tid == 0) { int a, b, c; three_maxima(hist, a, b, c); top[0] = a; top[1] = b; top[2] = c; }
        __syncthreads();
        for (int i = tid; i < q.n; i += 256)
            if (vmatch[i] >= 0) { const int b = bins[i]; if (b != top[0] && b != top[1] && b != top[2]) vmatch[i] = -1; }
        __syncthreads();
    }
    // ordered compaction into (idx1, idx2) pairs, ascending idx1 (:812-820)
    int running = 0;
    for (int base = 0; base < q.n; base += 256) {
        const int i = base + tid;
        const int v = i < q.n ? vmatch[i] : -1;
        const unsigned bal = __ballot_sync(0xFFFFFFFFu, v >= 0);
        if (lane == 0) wsum[wrp] = __popc(bal);
        __syncthreads();
        int off = running;
        for (int w = 0; w < wrp; w++) off += wsum[w];
        int tot = 0;
        for (int w = 0; w < 8; w++) tot += wsum[w];
        if (v >= 0) {
            const int pos = off + __popc(bal & ((1u << lane) - 1));
            if (pos < cap) { pairs[2 * pos] = i; pairs[2 * pos + 1] = v; }
        }
        running += tot;
        __syncthreads();
    }
    if (tid == 0) *T.n_pairs = running;
}

// ------------------------------------------------------------------------------------------------ vocabulary
// descent of feature f (a warp)
__device__ __forceinline__ void bow_descend(const VocDev& V, const uint8_t* __restrict__ desc, int f, int levelsup, int32_t* __restrict__ word,
                                            double* __restrict__ weight, int32_t* __restrict__ node) {
    const int lane = threadIdx.x & 31;
    // the descriptor is read ONCE into registers: `desc` may be pinned host memory (borb_bow_transform reads it in place)
    const uint4 f0 = reinterpret_cast<const uint4*>(desc)[(size_t)f * 2], f1 = reinterpret_cast<const uint4*>(desc)[(size_t)f * 2 + 1];
    const uint32_t feat[8] = {f0.x, f0.y, f0.z, f0.w, f1.x, f1.y, f1.z, f1.w};
    const int nid_level = V.L - levelsup;
    int nid = 0, final_id = 0, level = 0;
    while (true) {
        const int c0 = V.child_start[final_id], c1 = V.child_start[final_id + 1];
        if (c1 == c0) break;                                  // leaf (isLeaf() == children.empty())
        ++level;
        unsigned best = 0xFFFFFFFFu;
        for (int c = c0 + lane; c < c1; c += 32) {
            const int id = V.child_ids[c];
            const int d = ham_words(feat, reinterpret_cast<const uint32_t*>(V.desc + (size_t)id * 32));
            // distance <= 256 in the top 9 bits, the child's rank in the low 23 (borb_voc_create refuses wider nodes)
            best = min(best, ((unsigned)d << 23) | (unsigned)(c - c0));     // strict '<': first child wins ties (:1244)
        }
        best = warp_min(best);
        final_id = V.child_ids[c0 + (int)(best & 0x7FFFFFu)];
        if (level == nid_level) nid = final_id;
    }
    if (lane == 0) {
        word[f] = V.word_id[final_id];
        weight[f] = V.weight[final_id];
        node[f] = nid;
    }
}

__global__ void __launch_bounds__(256) bow_transform_kernel(VocDev V, const uint8_t* __restrict__ desc, int n, int levelsup,
                                                            int32_t* __restrict__ word, double* __restrict__ weight,
                                                            int32_t* __restrict__ node) {
    const int f = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (f < n) bow_descend(V, desc, f, levelsup, word, weight, node);
}
// many resident frames in one launch (borb_frames_compute_bow): grid.y = frame, results in the frame's device scratch
__global__ void __launch_bounds__(256) bow_transform_batch_kernel(VocDev V, const BowFrameJob* __restrict__ jobs, int levelsup) {
    const BowFrameJob& J = jobs[blockIdx.y];
    const int f = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (f < J.n) bow_descend(V, J.desc, f, levelsup, J.word, J.weight, J.node);
}

namespace {
// Exclusive prefix count of the run heads among sorted keys [0, m): a head is the first key of a run of equal high words.
// Each thread owns the contiguous chunk [c0, c1); returns the number of heads before c0, and the total in *total.
__device__ int count_heads_before(const uint64_t* k, int m, int c0, int c1, int* warp_sums, int* total) {
    int c = 0;
    for (int r = c0; r < c1; r++) c += (r == 0 || (k[r] >> 32) != (k[r - 1] >> 32)) ? 1 : 0;
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int incl = c;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const int v = __shfl_up_sync(0xFFFFFFFFu, incl, off);
        if (lane >= off) incl += v;
    }
    if (lane == 31) warp_sums[wrp] = incl;
    __syncthreads();
    int before = incl - c, all = 0;
    for (int w = 0; w < nw; w++) {
        const int s = warp_sums[w];
        if (w < wrp) before += s;
        all += s;
    }
    *total = all;
    __syncthreads();                                                     // warp_sums is reused by the next call
    return before;
}
}  // namespace

// The bookkeeping half of TemplatedVocabulary::transform (TemplatedVocabulary.h:1150-1194) for one frame per CTA, from the
// per-feature (word, weight, node) of the descent — what borb_compute_bow does on the host, bit for bit:
//   kept features (weight > 0: stop words drop out of both vectors, :1157) sorted by (word, feature) and by (node, feature);
//   per word run the weights summed in feature order (BowVector::addWeight, `vit->second += v`); the L1 norm summed in word order
//   (BowVector::normalize, BowVector.cpp:62-83) as one sequential chain of double adds (a tree reduction would round differently);
//   every value divided by it when it is > 0; the FeatureVector as CSR from the node order.
// Shared memory: 16 B per key slot (K = next power of two >= n, at least 32): the sort keys, then the run values.
__global__ void __launch_bounds__(1024) bow_build_kernel(const BowFrameJob* __restrict__ jobs) {
    extern __shared__ __align__(16) uint64_t bb_sm[];
    __shared__ int warp_sums[32];
    __shared__ int s_m;
    __shared__ double s_norm;
    const BowFrameJob& J = jobs[blockIdx.x];
    const int n = J.n, tid = threadIdx.x, T = blockDim.x;
    int K = 32;
    while (K < n) K <<= 1;
    uint64_t* keys = bb_sm;
    double* vals = reinterpret_cast<double*>(bb_sm + K);
    constexpr uint64_t NONE = ~0ull;                                     // dropped feature / padding: sorts last
    const int chunk = (K + T - 1) / T;                                   // the contiguous slice of sorted keys a thread scans
    const int c0 = min(K, tid * chunk), c1 = min(K, c0 + chunk);
    if (tid == 0) s_m = 0;
    // ---- BowVector: (word, feature) order
    for (int i = tid; i < K; i += T) keys[i] = (i < n && J.weight[i] > 0.0) ? ((uint64_t)(uint32_t)J.word[i] << 32) | (uint32_t)i : NONE;
    __syncthreads();
    bitonic_sort_u64(keys, K);
    for (int r = c0; r < c1; r++)                                        // m = number of kept features = first NONE
        if (keys[r] != NONE && (r + 1 == K || keys[r + 1] == NONE)) s_m = r + 1;
    __syncthreads();
    const int m = s_m;
    int nb = 0;
    int q = count_heads_before(keys, m, c0, min(c1, m), warp_sums, &nb);
    for (int r = c0; r < min(c1, m); r++) {
        const uint32_t w = (uint32_t)(keys[r] >> 32);
        if (r > 0 && (uint32_t)(keys[r - 1] >> 32) == w) continue;
        double v = J.weight[(uint32_t)keys[r]];
        for (int e = r + 1; e < m && (uint32_t)(keys[e] >> 32) == w; e++) v = __dadd_rn(v, J.weight[(uint32_t)keys[e]]);   // in feature order
        vals[q] = v;
        J.dst.word[q] = w;
        if (J.copy.word) J.copy.word[q] = w;
        q++;
    }
    __syncthreads();
    if (tid == 0) {                                                      // the serial chain of BowVector::normalize
        double norm = 0.0;
#pragma unroll 8
        for (int k = 0; k < nb; k++) norm = __dadd_rn(norm, fabs(vals[k]));
        s_norm = norm;
    }
    __syncthreads();
    const double norm = s_norm;
    for (int k = tid; k < nb; k += T) {
        const double v = norm > 0.0 ? __ddiv_rn(vals[k], norm) : vals[k];
        J.dst.value[k] = v;
        if (J.copy.word) J.copy.value[k] = v;
    }
    // ---- FeatureVector: (node, feature) order; the kept set is the same
    for (int i = tid; i < K; i += T) keys[i] = (i < n && J.weight[i] > 0.0) ? ((uint64_t)(uint32_t)J.node[i] << 32) | (uint32_t)i : NONE;
    __syncthreads();
    bitonic_sort_u64(keys, K);
    int nn = 0;
    q = count_heads_before(keys, m, c0, min(c1, m), warp_sums, &nn);
    for (int r = c0; r < min(c1, m); r++) {
        const uint32_t nd = (uint32_t)(keys[r] >> 32), f = (uint32_t)keys[r];
        if (r == 0 || (uint32_t)(keys[r - 1] >> 32) != nd) {
            J.dst.node[q] = nd; J.dst.start[q] = r;
            if (J.copy.word) { J.copy.node[q] = nd; J.copy.start[q] = r; }
            q++;
        }
        J.dst.idx[r] = f;
        if (J.copy.word) J.copy.idx[r] = f;
    }
    if (tid == 0) {
        J.dst.start[nn] = m;
        if (J.copy.word) J.copy.start[nn] = m;
        J.counts[0] = nb;
        J.counts[1] = nn;
        J.counts[2] = m;
    }
}

// ------------------------------------------------------------------------------------------------ launchers
int launch_grid_sort(const borb_keypoint* keys, int n, float minX, float minY, float invW, float invH, int* cell_start, int* cell_idx,
                     cudaStream_t s) {
    int K = 32;
    while (K < n) K <<= 1;
    allow_max_smem((const void*)grid_sort_kernel);
    grid_sort_kernel<<<1, 1024, K * 4, s>>>(keys, n, minX, minY, invW, invH, K, cell_start, cell_idx);
    return 1;
}
int launch_initialization(const ProjArgs& A, const borb_keypoint* keys1, int n1, int32_t* match12, int32_t* ev_idx, uint8_t* ev_bin,
                          float* prev, int* n_matches, cudaStream_t s) {
    launch_candidates(A, s);
    const size_t smem = (size_t)((A.n + 1) & ~1) * 2 + (size_t)A.n * 2 + 16;
    init_resolve_kernel<<<1, 32, smem, s>>>(A, keys1, n1, match12, ev_idx, ev_bin, prev, n_matches);
    return 2;
}
int launch_kfdb_score(const KfdbQueryJob* d_jobs, int n_jobs, int max_slots, int max_nq, int n_sm, cudaStream_t s) {
    if (n_jobs > 0 && max_slots > 0) {
        const size_t smem = (size_t)max_nq * 12 + 16;
        const int in_smem = smem <= 160 * 1024;
        if (in_smem) allow_max_smem((const void*)kfdb_score_kernel);
        int ctas = (max_slots + 3) / 4;                               // 4 keyframes (warps) per CTA: 2000 keyframes spread over all SMs
        const int cap = std::max(1, n_sm * 8 / n_jobs);               // persistent: the query is staged once per CTA
        if (ctas > cap) ctas = cap;
        kfdb_score_kernel<<<dim3(ctas, n_jobs), 128, in_smem ? smem : 0, s>>>(d_jobs, in_smem);
    }
    return 1;
}
int launch_distinctive(const uint8_t* desc, const int32_t* offsets, int n_points, int32_t* best_idx, cudaStream_t s) {
    if (n_points > 0) distinctive_kernel<<<(n_points + 3) / 4, 128, 0, s>>>(desc, offsets, n_points, best_idx);
    return 1;
}
int launch_point_projection_batch(const LastArgs* d_last, const ProjArgs* d_jobs, const LastArgs& one_last, const ProjArgs& one, int n_jobs,
                                  int max_nq, int max_n, int max_n_mp, bool last, cudaStream_t s) {
    if (n_jobs <= 0 || max_nq <= 0) return 0;
    if (n_jobs == 1) project_points_kernel<<<(one_last.n_last + 255) / 256, 256, 0, s>>>(one_last);
    else project_points_batch_kernel<<<dim3((max_nq + 255) / 256, n_jobs), 256, 0, s>>>(d_last);
    return 1 + launch_projection_batch(d_jobs, one, n_jobs, max_n, max_n_mp, s, last);
}
int launch_bow_match(const KfDev* qs, const KfDev* ts, int n_pairs, int mode, float nnratio, int check_ori, int32_t* match,
                     const size_t* out_off, uint8_t* bins, int32_t* n_matches, int max_t, cudaStream_t s) {
    const int words = (max_t + 31) / 32;
    const size_t smem = (size_t)(words + BOW_WARPS * BOW_WARP_WORDS) * 4;
    allow_max_smem((const void*)bow_match_kernel);
    bow_match_kernel<<<n_pairs, 32 * BOW_WARPS, smem, s>>>(qs, ts, mode, nnratio, check_ori, match, out_off, bins, n_matches, max_t);
    return 1;
}
int launch_triangulation(const TriJob* d_jobs, int n_jobs, int check_ori, cudaStream_t s) {
    if (n_jobs <= 0) return 0;
    triangulation_kernel<<<n_jobs, 256, 0, s>>>(d_jobs, check_ori);
    return 1;
}
int launch_fuse_batch(const LastArgs* d_last, const FuseJob* d_jobs, int n_jobs, int max_nq, cudaStream_t s) {
    if (n_jobs <= 0 || max_nq <= 0) return 0;
    project_points_batch_kernel<<<dim3((max_nq + 255) / 256, n_jobs), 256, 0, s>>>(d_last);
    launch_fuse_search(d_jobs, n_jobs, max_nq, s);
    return 2;
}
int launch_bow_transform(const VocDev& V, const uint8_t* desc, int n, int levelsup, int32_t* word, double* weight, int32_t* node,
                         cudaStream_t s) {
    if (n > 0) bow_transform_kernel<<<(n + 7) / 8, 256, 0, s>>>(V, desc, n, levelsup, word, weight, node);
    return 1;
}
int launch_bow_frames(const VocDev& V, const BowFrameJob* d_jobs, int n_frames, int max_n, int levelsup, cudaStream_t s) {
    if (n_frames <= 0) return 0;
    bow_transform_batch_kernel<<<dim3((max(max_n, 1) + 7) / 8, n_frames), 256, 0, s>>>(V, d_jobs, levelsup);
    int K = 32;
    while (K < max_n) K <<= 1;
    allow_max_smem((const void*)bow_build_kernel);
    bow_build_kernel<<<n_frames, 1024, (size_t)K * 16, s>>>(d_jobs);
    return 2;
}

}  // namespace borb
