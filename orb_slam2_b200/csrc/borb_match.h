// Internal declarations for the matcher / vocabulary part of libborb.  Not part of the C ABI.
#pragma once
#include "borb_internal.h"

// Device-resident Frame (include/borb.h: borb_frame_create / borb_frame_from_extractor): what the windowed searches read of a
// Frame — mvKeysUn, mDescriptors, mvuRight, mvScaleFactors and the 64x48 feature grid (Frame::AssignFeaturesToGrid) — kept in
// HBM across the matcher calls of one Track().
struct borb_frame {
    int device = 0;
    int n = 0, n_levels = 0;
    float min_x = 0, min_y = 0, max_x = 0, max_y = 0;
    uint8_t* block = nullptr;       // one allocation: keys | desc | u_right | depth | scale factors | cell_start | cell_idx |
                                    //                 bow_value | bow_word | fv_node | fv_start | fv_idx
    size_t block_bytes = 0;
    int cap = 0;                    // features the block can hold
    borb_keypoint* keys = nullptr;
    uint8_t* desc = nullptr;
    float* u_right = nullptr;       // null: monocular
    float* depth = nullptr;
    float* ur_store = nullptr;      // storage behind u_right / depth (always allocated)
    float* depth_store = nullptr;
    float* sf = nullptr;
    int* cell_start = nullptr;
    int* cell_idx = nullptr;
    // Frame::mBowVec / mFeatVec (borb_frames_compute_bow): BowVector in word order, FeatureVector as CSR (cap entries each,
    // fv_start cap + 1); valid only while has_bow, which frame_alloc clears
    double* bow_value = nullptr;
    uint32_t* bow_word = nullptr;
    uint32_t* fv_node = nullptr;
    int32_t* fv_start = nullptr;
    uint32_t* fv_idx = nullptr;
    bool has_bow = false;
    int n_bow = 0, n_nodes = 0, n_fv = 0;   // n_fv = fv_start[n_nodes]: features inside the FeatureVector's nodes
    cudaEvent_t ready = nullptr;    // recorded after the last kernel that writes the block
};

extern "C" void borb_voc_adopt_ownership(borb_voc* v);     // internal (borb_nccl.cu): the vocabulary now owns its blob

namespace borb {

constexpr int GRID_COLS = 64, GRID_ROWS = 48;     // FRAME_GRID_COLS / FRAME_GRID_ROWS (include/Frame.h:37-38)
constexpr int GRID_CELLS = GRID_COLS * GRID_ROWS;
constexpr int CAND_UNSORTED = 0x40000000;           // flag in cand_cnt: list longer than the sort capacity, kept in position order
constexpr int CAND_COUNT_MASK = 0x3FFFFFFF;
constexpr int MATCH_MAX_FEATURES = 8192;          // per frame / keyframe (grid sort and claim bitsets live in smem)
static_assert(MATCH_MAX_FEATURES == BORB_MATCH_MAX_FEATURES, "include/borb.h documents this limit");

struct ProjArgs {                 // device pointers
    int n;                        // frame features
    const borb_keypoint* keys;
    const uint8_t* desc;
    const float* u_right;         // may be null
    const uint8_t* occupied;      // may be null
    float minX, minY, invW, invH;
    const float* scale_factors;
    const int* cell_start;
    const int* cell_idx;
    int n_mp;
    const float *proj_x, *proj_y, *proj_xr, *view_cos;
    const int32_t* level;
    const uint8_t* mp_desc;
    const uint8_t* mp_valid;      // may be null
    const uint8_t* mp_has_obs;    // may be null
    float th, nnratio;
    uint32_t* cand;               // n_mp x n
    int* cand_cnt;                // n_mp
    // mode 1 (SearchByProjection(CurrentFrame, LastFrame)): the window is precomputed per query by project_points_kernel
    const float* q_radius;        // null in mode 0
    const int32_t* q_minl;
    const int32_t* q_maxl;
    int mode;                     // 0: local map points (ratio test), 1: last frame (best only, rotation histogram)
    int check_ori;
    const float* q_angle;         // mode 1: mvKeysUn[i].angle of the query
    int th_dist;                  // mode 1: accept bestDist <= th_dist (TH_HIGH / ORBdist / TH_LOW)
    // where the resolve / fuse kernels write the results
    int32_t* out_match;           // n_mp entries (mode 1 resolve: the per-feature state, n entries), then the match count
    int32_t* ev_idx;              // mode 1: match events of the rotation histogram, n_mp entries
    uint8_t* ev_bin;
};

struct FuseJob {                  // one job of fuse_batch_kernel (k_proj.cu)
    ProjArgs A;                   // the keyframe (u_right null for the Scw overload) and the windows project_points wrote (mode 1
                                  // fields); th_dist = TH_LOW; out_match = best_idx, n_mp entries
    const float* inv_sigma2;      // mvInvLevelSigma2: the reprojection gates of Fuse(pKF, vpMapPoints, th); null for the Scw overload
    int* n_found;
};

struct Sim3AgreeJob {             // one SearchBySim3 of sim3_agree_batch_kernel (k_proj.cu)
    const int32_t* match1;        // KF1's points searched in KF2: n1 entries, a KF2 feature or -1 (fuse_batch_kernel's best_idx)
    const int32_t* match2;        // KF2's points searched in KF1: n2 entries
    int n1, n2;                   // n1 = 0: nothing to do (the host wrote the result of a job without features)
    int32_t* match12;             // n1 entries
    int* n_found;                 // preset to 0
};

constexpr int INIT_K = 8;         // window entries per F1 feature kept by init_prefix_kernel

struct InitJob {                  // one SearchForInitialization of init_prefix / init_replay (k_proj.cu)
    ProjArgs A;                   // F2 = the current frame: keys, descriptors, grid and bounds (bind_frame_fields)
    const borb_keypoint* keys1;   // F1 = the initial frame
    const uint8_t* desc1;
    int n1;                       // 0: nothing to do (the host wrote the result of a job without features)
    float window;                 // (float)windowSize
    const float* prev_in;         // vbPrevMatched, n1 x 2
    uint32_t* prefix;             // scratch, n1 x INIT_K: the smallest window keys as F2 feature | dist << 16, in (dist, e) order
    int* win_count;               // scratch, n1: the window's entries (0: skipped feature or empty window)
    int32_t* out;                 // n1 entries of vnMatches12, then the match count
    float* prev_out;              // n1 x 2: vbPrevMatched after the call (:513-517)
};

struct LastArgs {                 // inputs of project_points_kernel
    int variant;                  // 0: (CurrentFrame, LastFrame) :1328   1: (CurrentFrame, KeyFrame) :1472   2: (KeyFrame, Scw) :290
                                  // 3: Frame::isInFrustum (src/Frame.cc:269-325), feeding SearchByProjection(F, vpMapPoints)
    float view_cos_limit;         // variant 3
    int32_t* level_out;           // variant 3: mnTrackScaleLevel
    float* viewcos_out;           // variant 3: mTrackViewCos
    int n_last;
    const borb_keypoint* last_keys;   // variant 0 only (octave, angle of the last-frame feature)
    const float* q_angle_in;      // variant 1: angle of the observing keyframe feature (may be null)
    const float* max_distance;    // variants 1, 2
    const float* min_distance;
    const float* normal;          // variant 2, n x 3
    float Ow[3];
    float log_scale;
    int n_levels;
    // variant 2 options (Fuse x2, SearchBySim3 directions share its code path)
    int invz_double;              // invz = 1.0/z evaluated in double (:1014, :1164) instead of 1/z in float (:333, :861)
    int use_normal;               // viewing-angle gate PO.dot(Pn) < 0.5*dist
    int chain;                    // second transform T2 applied to the camera-frame point; distance = |point in camera 2| (:1157-1177)
    float T2[12];
    const float* world_pos;       // n_last x 3
    const uint8_t* valid_in;      // may be null
    float T[12];                  // Tcw rows 0..2
    float fx, fy, cx, cy, bf, th;
    float minX, minY, maxX, maxY;
    const float* scale_factors;
    int forward, backward;
    float *proj_x, *proj_y, *proj_xr, *radius, *angle;
    int32_t *minl, *maxl;
    uint8_t* valid_out;
};

struct KfDev {                    // device-side borb_keyframe_view
    int n, nn;
    const borb_keypoint* keys;
    const uint8_t* desc;
    const uint8_t* has_mp;        // may be null
    const float* u_right;         // may be null
    const uint32_t* node;
    const int32_t* start;
    const uint32_t* idx;
    const float* scale_factors;
    const float* level_sigma2;
};

struct BowDev {                   // one keyframe's BowVector in the device-resident database (null / 0 when erased)
    const uint32_t* word;         // ascending
    const double* value;
    int n;
};

struct KfStream {                  // one keyframe of the device-resident database, features permuted into FeatureVector order
    const uint32_t* node;         // nn node ids, ascending
    const int32_t* start;         // nn + 1 row offsets
    const uint2* meta;            // m rows: x = feature index (mFeatVec order: node, then feature index) | good-MapPoint flag << 16
                                  //             | index of the row's node in node[] << 17 (nn <= MATCH_MAX_FEATURES < 2^15),
                                  //         y = bits of mvKeysUn[feature].angle
    const uint8_t* desc;          // m x 32, 16-byte aligned
    int nn, m, n, pad;
    const void* pad2[2];
};

// One keyframe's device block in the database (borb_kfdb_add, borb_kfdb_add_frames): the KfStream and BowDev sections
//   node[nn] | start[nn + 1] | meta[m] uint2 | desc[m][32] | bow words[n_bow] | bow values[n_bow]
// each 256-byte aligned, then 256 bytes of tail; every byte outside the sections is 0.
struct KfdbBlock { size_t node, start, meta, desc, bow_word, bow_value, bytes; };
__host__ __device__ inline KfdbBlock kfdb_block_layout(int nn, int m, int n_bow) {
    size_t off = 0;
    auto put = [&](size_t bytes) { off = (off + 255) & ~size_t(255); const size_t o = off; off += bytes; return o; };
    KfdbBlock L;
    L.node = put((size_t)nn * 4); L.start = put((size_t)(nn + 1) * 4); L.meta = put((size_t)m * 8); L.desc = put((size_t)m * 32);
    L.bow_word = put((size_t)n_bow * 4); L.bow_value = put((size_t)n_bow * 8);
    L.bytes = off + 256;
    return L;
}

struct KfdbInsertJob {            // one keyframe of kfdb_insert_kernel (k_bowdb.cu): a resident frame with BoW -> its database block
    const uint32_t* fv_node;      // the frame's FeatureVector (nn nodes, m = fv_start[nn] rows) and BowVector
    const int32_t* fv_start;
    const uint32_t* fv_idx;
    const borb_keypoint* keys;
    const uint8_t* desc;
    const uint32_t* bow_word;
    const double* bow_value;
    const uint8_t* has_mp;        // n entries, may be null
    int nn, m, n_bow, pad;
    uint8_t* block;               // kfdb_block_layout(nn, m, n_bow), written whole
    uint2* meta_out;              // m rows: a copy of the row records for the host (pinned, device-addressable)
};

// Packed query frame of the database search (k_bowdb.cu), built on the device by bowdb_pack_kernel: header, then 16-byte
// aligned sections
//   node[nn] u32 ascending | start[nn+1] i32 | orig[m] u16 | angle[m] f32 | desc[m][32]     (m = features inside nodes)
//   work list (np = non-empty frame nodes, widest bucket first): pnode[np] i32 node index | pcs[np] i32 keyframes per item |
//   pstart[np+1] i32 cumulative item count
struct FrameBlockHdr { int32_t nn, m, n, off_node, off_start, off_orig, off_angle, off_desc, bytes, np, off_pnode, off_pcs, off_pstart, pad[3]; };

// The section offsets and the size of the block of a frame with nn FeatureVector nodes holding m of its n features.
__host__ __device__ inline FrameBlockHdr frame_block_layout(int nn, int m, int n) {
    FrameBlockHdr h{};
    int off = (int)sizeof(FrameBlockHdr);
    auto put = [&](int bytes) { off = (off + 15) & ~15; const int o = off; off += bytes; return o; };
    h.nn = nn; h.m = m; h.n = n;
    h.off_node = put(nn * 4); h.off_start = put((nn + 1) * 4); h.off_orig = put(m * 2);
    h.off_angle = put(m * 4); h.off_desc = put(m * 32);
    h.off_pnode = put(nn * 4); h.off_pcs = put(nn * 4); h.off_pstart = put((nn + 1) * 4);
    h.bytes = (off + 15) & ~15;
    return h;
}

// One frame of the database search (borb_search_by_bow_db*, borb_search_by_bow_db_batch): read by bowdb_pack_kernel,
// bowdb_match_kernel and bowdb_finalize_kernel (k_bowdb.cu).
struct BowDbJob {
    // the frame: FeatureVector (CSR), keypoints (angle) and descriptors, resident or staged from a host view
    const uint32_t* fv_node;
    const int32_t* fv_start;      // nn + 1
    const uint32_t* fv_idx;       // m
    union {
        const borb_keypoint* keys;
        const uint2* q_meta;      // SearchByBoW(KeyFrame*, KeyFrame*): the query slot's KfStream rows (fv_node / fv_start / desc are
    };                            // its stream's, desc in row order, fv_idx unused)
    const uint8_t* desc;          // n x 32, 16-byte aligned
    int nn, m, n, item_target;    // item_target: keyframes per work item = item_target / nt^2, clamped to 1..32
    uint8_t* frame_block;         // FrameBlockHdr + sections, 128-byte aligned, frame_bytes = frame_block_layout(nn, m, n).bytes
    int frame_bytes, frame_in_smem;
    // the keyframes
    const KfStream* table;        // the job's database, one entry per slot (nn = 0: erased)
    const int32_t* slots;         // n_kf slots to search, or null = slots 0..n_kf-1
    int n_kf, kf_base;            // kf_base: the job's first finalize CTA (sum of n_kf of the jobs before it)
    int* ctr;                     // [0] work counter, [1] work items (written by the packer), [2] pair cursor
    uint32_t* table_out;          // n_kf x m, preset to 0xFFFFFFFF
    int* hist_out;                // n_kf x 32 rotation-histogram counters, preset to 0
    // results
    int32_t* n_matches;           // n_kf
    int32_t* pair_off;            // n_kf (may be null)
    uint32_t* pairs;              // frame feature | keyframe feature << 16 (may be null), pairs_cap entries
    int pairs_cap;
    int dense_stride;
    int32_t* dense;               // n_kf x dense_stride preset to -1 (may be null): match[k][frame feature] = keyframe feature
};

struct BowDbArgs {                // the launch sequence of the database search over a job table in device memory
    const BowDbJob* jobs;
    int n_jobs;
    int static_sched;             // 1: item i of every job -> warp i mod (warps), 0: atomic work counter per job
    float nnratio;
    int check_ori;
};

struct KfdbQueryJob {             // one query of kfdb_score_kernel (k_match.cu)
    const BowDev* table;          // the job's database, one entry per slot
    int n_slots, nq;
    const uint32_t* qword;        // the query BowVector, ascending words
    const double* qvalue;
    int32_t* common;              // n_slots entries each
    float* score;
    uint32_t* first_word;
};

// ascending bitonic sort of K (a power of two) 64-bit keys in shared memory by the whole CTA; ends with a barrier
__device__ inline void bitonic_sort_u64(uint64_t* k, int K) {
    const int half = K >> 1;
    for (int kk = 2; kk <= K; kk <<= 1)
        for (int j = kk >> 1; j > 0; j >>= 1) {
            for (int p = threadIdx.x; p < half; p += blockDim.x) {
                const int i = ((p & ~(j - 1)) << 1) | (p & (j - 1));          // lower element of the p-th compare pair
                const uint64_t a = k[i], b = k[i + j];
                if ((a > b) == ((i & kk) == 0)) { k[i] = b; k[i + j] = a; }
            }
            __syncthreads();
        }
}

struct FrameJob {                 // one frame of borb_frames_from_extractor (k_frame.cu); a grid-only row sets keys, the grid, n and the bounds
    const borb_keypoint* src_keys;   // the extractor's mvKeys of that image
    const uint8_t* src_desc;
    const float* src_ur;             // stereo: the extractor's mvuRight / mvDepth of the pair
    const float* src_depth;
    const void* depth_img;           // RGB-D: depth map in HBM (w x h, tight rows)
    borb_keypoint* keys;             // destination borb_frame fields
    uint8_t* desc;
    float* u_right;
    float* depth;
    int* cell_start;
    int* cell_idx;
    int n;
    float min_x, min_y, inv_w, inv_h;
};

struct TriJob {                   // one SearchForTriangulation of triangulation_kernel (k_match.cu), a CTA per job
    KfDev q, t;                   // kf1, kf2
    float F[9];
    float ex, ey;
    int only_stereo;
    int32_t* vmatch;              // scratch, q.n entries
    uint8_t* bins;                // scratch, q.n entries
    int32_t* pairs;               // 2 * cap ints
    int cap;
    int32_t* n_pairs;
};

struct DistinctArgs {             // MapPoint::ComputeDistinctiveDescriptors of n_points points (distinctive_kernel, k_match.cu)
    const uint8_t* const* src;    // row sources: descriptor arrays of 32-byte rows, 16-byte aligned
    const int32_t* obs_src;       // observation o = row obs_row[o] of src[obs_src[o]]; null: row o of src[0]
    const int32_t* obs_row;
    const int32_t* offsets;       // n_points + 1: point p owns observations offsets[p] .. offsets[p+1]-1
    int n_points;
    int32_t* best_idx;            // n_points: the chosen observation, relative to offsets[p] (-1: none)
    uint8_t* desc_out;            // n_points x 32: the chosen row, untouched where best_idx is -1; may be null
};

struct BowTables {                // a BowVector (word order) and a FeatureVector (CSR); word == null: not written
    uint32_t* word;
    double* value;
    uint32_t* node;
    int32_t* start;               // n_nodes + 1
    uint32_t* idx;
};

struct BowFrameJob {              // one frame of a BoW call (bow_transform_batch_kernel, bow_build_kernel)
    const uint8_t* desc;          // a resident frame's descriptors, or staged host ones
    int n;
    int32_t* word;                // word id, word weight, node id per feature (the descent's output): scratch, or the results of
    double* weight;               // a descent-only call
    int32_t* node;
    BowTables dst;                // a resident frame's storage, or result slots
    BowTables copy;               // the same tables again, for the host (may be unset)
    int32_t* counts;              // n_bow, n_nodes, fv_start[n_nodes]
};

struct VocDev {                   // views into the packed blob
    int n_nodes, k, L;
    const uint8_t* desc;          // n_nodes x 32
    const double* weight;
    const int32_t* word_id;       // -1 for inner nodes
    const int32_t* child_start;   // n_nodes + 1
    const int32_t* child_ids;     // n_nodes - 1
};

void launch_candidates(const ProjArgs& A, cudaStream_t s);
// candidates and resolve (last: resolve<true>) of n_jobs jobs: one job runs the by-value kernels on `one` (the host copy of job 0),
// more run the *_batch_kernels over the ProjArgs table d_jobs (unused for one job)
int launch_projection_batch(const ProjArgs* d_jobs, const ProjArgs& one, int n_jobs, int max_n, int max_n_mp, cudaStream_t s, bool last = false);
// project_points, then launch_projection_batch; one job by value (one_last, one), more over the LastArgs / ProjArgs tables
int launch_point_projection_batch(const LastArgs* d_last, const ProjArgs* d_jobs, const LastArgs& one_last, const ProjArgs& one, int n_jobs,
                                  int max_nq, int max_n, int max_n_mp, bool last, cudaStream_t s);
void launch_resolve(const ProjArgs& A, bool last, cudaStream_t s);
// SearchForInitialization of n_jobs jobs in 2 launches: one job by value (`one`), more over the InitJob table d_jobs;
// max_n1 / max_n2 = the most features of an initial / current frame of a live job
int launch_init_batch(const InitJob* d_jobs, const InitJob& one, int n_jobs, int max_n1, int max_n2, float nnratio, int check_ori,
                      cudaStream_t s);
// n_jobs queries (a job table in device memory) in one launch; max_slots / max_nq: the largest n_slots / nq of the jobs
int launch_kfdb_score(const KfdbQueryJob* d_jobs, int n_jobs, int max_slots, int max_nq, int n_sm, cudaStream_t s);
int launch_distinctive(const DistinctArgs& A, cudaStream_t s);
// n_pairs searches in one launch (tables in device memory): pair p matches qs[p] against ts[p] and writes its output (mode 0: ts[p].n
// entries, mode 1: qs[p].n) at match + out_off[p], its rotation bins at bins + out_off[p]; max_t = the largest ts[p].n
int launch_bow_match(const KfDev* qs, const KfDev* ts, int n_pairs, int mode, float nnratio, int check_ori, int32_t* match,
                     const size_t* out_off, uint8_t* bins, int32_t* n_matches, int max_t, cudaStream_t s);
void host_image_bounds(int w, int h, const borb_camera& c, float* b4);
int launch_frame_build(const FrameJob* d_jobs, int n_jobs, int max_n, const borb_camera& cam, int mode, int depth_type, float depth_factor, int w,
                       int h, int out_cap, borb_keypoint* keys_out, float* ur_out, float* depth_out, cudaStream_t s);
// Frame::AssignFeaturesToGrid of n_jobs frames (a FrameJob table the kernel can read) in one launch; max_n = the most keys of a job
int launch_grid_sort(const FrameJob* d_jobs, int n_jobs, int max_n, cudaStream_t s);
// Copies whose lengths are device-side counts (an extraction's keypoint count, a grid's size), written by host_copy_kernel straight
// into mapped pinned memory: only the bytes of the counted elements cross PCIe and the host needs no count beforehand.
struct HostCopy {
    const void* src;
    void* dst;
    const int* count;     // elements: *count, or `fixed` when null
    int fixed;
    int elem_words;       // 32-bit words per element
};
struct HostCopies { HostCopy seg[8]; int n; };
int launch_host_copy(const HostCopies& c, cudaStream_t s);
// pack + match + finalize over A.jobs (3 launches): one = a host copy of job 0 (what the match kernel reads of a single job),
// max_smem_frame = largest frame_bytes of the jobs with frame_in_smem, max_items = an upper bound of the work items of all jobs,
// total_kf = sum of their n_kf; kfkf: the jobs are SearchByBoW(KeyFrame*, KeyFrame*) of a database slot against candidates
int launch_bowdb(const BowDbArgs& A, const BowDbJob& one, int max_smem_frame, long long max_items, int total_kf, int max_nn, int csa, int n_sm,
                 bool kfkf, cudaStream_t s);
bool bowdb_frame_fits_smem(int frame_bytes);
// n_jobs database blocks (a job table in device memory) in one launch, a CTA per job
int launch_kfdb_insert(const KfdbInsertJob* d_jobs, int n_jobs, cudaStream_t s);
// n_jobs searches (a job table in device memory) in one launch
int launch_triangulation(const TriJob* d_jobs, int n_jobs, int check_ori, cudaStream_t s);
// project_points over a LastArgs table (variant 2), then fuse_batch_kernel over a FuseJob table: 2 launches; max_nq = most points of a job
int launch_fuse_batch(const LastArgs* d_last, const FuseJob* d_jobs, int n_jobs, int max_nq, cudaStream_t s);
void launch_fuse_search(const FuseJob* d_jobs, int n_jobs, int max_nq, cudaStream_t s);
// SearchBySim3 of n_jobs jobs in 3 launches: launch_fuse_batch over the 2 n_jobs direction entries of d_last / d_dirs (job j: 2j and
// 2j + 1), then sim3_agree_batch_kernel over d_jobs; max_nq = most points of a direction, max_n1 = most KF1 features of a job
int launch_sim3_batch(const LastArgs* d_last, const FuseJob* d_dirs, const Sim3AgreeJob* d_jobs, int n_jobs, int max_nq, int max_n1,
                      cudaStream_t s);
// descent + bookkeeping for n_frames frames (a job table the kernels can read): 2 launches, descent_only: 1
int launch_bow_frames(const VocDev& V, const BowFrameJob* d_jobs, int n_frames, int max_n, int levelsup, bool descent_only, cudaStream_t s);

}  // namespace borb
