// Host side of the matcher / vocabulary entry points of the C ABI (include/borb.h): snapshots arrive as plain host
// arrays, are staged into one device arena per call, and every result is produced by the CUDA kernels in k_match.cu.
#include <algorithm>
#include <atomic>
#include <cassert>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <optional>
#include <string>

#include "borb_match.h"

using namespace borb;

// What a Call runs on: a device, a stream and the grow-only buffers it stages through.  A matcher and a vocabulary each carry one.
struct CallBuffers {
    int device = 0;
    cudaStream_t stream = nullptr;
    uint8_t* arena = nullptr;       // device scratch, grow-only
    size_t arena_bytes = 0;
    uint8_t* h_stage = nullptr;     // pinned staging mirror of the arena's input part
    size_t h_bytes = 0;
    uint8_t* h_out = nullptr;       // pinned landing buffer for results (one D2H per call)
    size_t h_out_bytes = 0;
};

struct borb_matcher : CallBuffers {
    uint64_t launches = 0;
    int n_sm = 1;                   // the device's multiprocessor count (sizes the persistent grids)
    std::vector<int32_t> sel;       // indices of the valid queries of the current call
    cudaEvent_t ev_a = nullptr, ev_b = nullptr;   // cross-stream ordering with an extractor handle (borb_frames_from_extractor)
    cudaEvent_t ev_r = nullptr;     // borb_frame_from_extractors: the right handle's extraction before the left stream's association
    bool timing = false;            // borb_matcher_set_timing: CUDA events around the kernels of the database search
    cudaEvent_t t0 = nullptr, t1 = nullptr;
    float last_ms = 0.f;
};

struct borb_voc : CallBuffers {     // the buffers of borb_bow_transform / borb_compute_bow
    bool owns = true;
    uint8_t* blob = nullptr;        // device
    size_t bytes = 0;
    VocDev dev;
    std::mutex mu;                  // a single call holds it until its results are copied out: every caller shares the buffers
};

namespace {

constexpr size_t ZERO_COPY_MAX = 96 * 1024;       // inputs up to this size may be read in place by the kernels (each byte is read once)

// One call on a matcher's or a vocabulary's buffers and stream.  Its layout comes first, as offsets: staged inputs, then device-only
// scratch, then result slots.
// begin() grows the buffers, after which addresses exist; commit() moves the inputs with one H2D copy and finish() brings the result
// region back with one D2H copy and synchronises.  Kernels read the inputs from the arena or, for a small in-place call, from the
// pinned staging buffer itself (device-addressable, UVA: no H2D copy and no DMA latency).  They write results to the arena, or
// straight into the pinned landing buffer.
class Call {
public:
    explicit Call(CallBuffers* b) : b_(b) {}
    // a staged input; src == nullptr: filled through host<T>() after begin()
    size_t in(const void* src, size_t bytes) {
        assert(!begun_ && in_end_ == off_);              // every input comes before any scratch
        const size_t o = put(bytes);
        items_.push_back({src, o, bytes});
        in_end_ = off_;
        return o;
    }
    size_t scratch(size_t bytes) { assert(!begun_); return put(bytes); }
    // a slot of the result region, 16-byte aligned
    size_t result(size_t bytes) {
        assert(!begun_);
        const size_t o = (res_bytes_ + 15) & ~size_t(15);
        res_bytes_ = o + bytes;
        return o;
    }
    // in_place: the kernels read the inputs from the staging buffer if they fit ZERO_COPY_MAX
    borb_status begin(bool in_place = false) {
        assert(!begun_);
        in_place_ = in_place && in_end_ <= ZERO_COPY_MAX;
        res_off_ = put(res_bytes_);
        BORB_CUDA(cudaSetDevice(b_->device));
        borb_status s;
        if ((s = grow_device(b_->arena, b_->arena_bytes, off_)) != BORB_OK) return s;
        if ((s = grow_pinned(b_->h_stage, b_->h_bytes, in_end_)) != BORB_OK) return s;
        if (res_bytes_ && (s = grow_pinned(b_->h_out, b_->h_out_bytes, res_bytes_ + 4096)) != BORB_OK) return s;
        BORB_CUDA(cudaStreamSynchronize(b_->stream));   // the staging buffer may still feed an earlier copy
        if (const int p = poison_byte(); p >= 0) {      // borb_debug_set_poison: everything this call has not written yet
            std::memset(b_->h_stage, p, in_end_);        // the alignment gaps between the inputs included
            std::memset(b_->h_out, p, res_bytes_);
            BORB_CUDA(cudaMemsetAsync(b_->arena + in_end_, p, off_ - in_end_, b_->stream));
        }
        for (const Item& it : items_)
            if (it.src) std::memcpy(b_->h_stage + it.off, it.src, it.bytes);
        begun_ = true;
        return BORB_OK;
    }
    bool in_place() const { return in_place_; }
    // the staging copy of an input
    template <class T> T* host(size_t off) const { assert(begun_ && off < in_end_); return reinterpret_cast<T*>(b_->h_stage + off); }
    // where kernels read an input or use scratch
    uint8_t* dev(size_t off) const { assert(begun_); return (in_place_ && off < in_end_ ? b_->h_stage : b_->arena) + off; }
    // where kernels write a result: the arena (brought back by finish()), or direct: the landing buffer
    uint8_t* res(size_t off, bool direct) {
        assert(begun_);
        download_ |= !direct;
        return (direct ? b_->h_out : b_->arena + res_off_) + off;
    }
    borb_status commit() {
        assert(begun_);
        if (in_end_ && !in_place_) BORB_CUDA(cudaMemcpyAsync(b_->arena, b_->h_stage, in_end_, cudaMemcpyHostToDevice, b_->stream));
        return BORB_OK;
    }
    borb_status wait(const borb_frame* f) const {
        BORB_CUDA(cudaStreamWaitEvent(b_->stream, f->ready, 0));
        return BORB_OK;
    }
    borb_status finish() {
        BORB_CUDA(cudaGetLastError());
        if (download_ && res_bytes_) BORB_CUDA(cudaMemcpyAsync(b_->h_out, b_->arena + res_off_, res_bytes_, cudaMemcpyDeviceToHost, b_->stream));
        BORB_CUDA(cudaStreamSynchronize(b_->stream));
        return BORB_OK;
    }
    // the landing buffer, after finish()
    const uint8_t* out(size_t off) const { return b_->h_out + off; }

private:
    struct Item { const void* src; size_t off, bytes; };
    size_t put(size_t bytes) { off_ = (off_ + 255) & ~size_t(255); const size_t o = off_; off_ += bytes; return o; }
    // grow-only buffers; the stream is synchronised first because queued work may still use the old one
    borb_status grow_device(uint8_t*& p, size_t& have, size_t bytes) {
        if (have >= bytes) return BORB_OK;
        BORB_CUDA(cudaStreamSynchronize(b_->stream));
        cudaFree(p);
        p = nullptr; have = 0;
        const size_t want = bytes + bytes / 2 + (1 << 20);
        BORB_CUDA(cudaMalloc(&p, want));
        have = want;
        return BORB_OK;
    }
    borb_status grow_pinned(uint8_t*& p, size_t& have, size_t bytes) {
        if (have >= bytes) return BORB_OK;
        BORB_CUDA(cudaStreamSynchronize(b_->stream));
        if (p) cudaFreeHost(p);
        p = nullptr; have = 0;
        const size_t want = bytes + bytes / 2 + (1 << 16);
        BORB_CUDA(cudaMallocHost(&p, want));
        have = want;
        return BORB_OK;
    }
    CallBuffers* b_;
    std::vector<Item> items_;
    size_t off_ = 0, in_end_ = 0, res_bytes_ = 0, res_off_ = 0;
    bool begun_ = false, in_place_ = false, download_ = false;
};

// after the stream's queued work: frees the buffers and the stream
void free_call_buffers(CallBuffers& b) {
    cudaSetDevice(b.device);
    if (b.stream) cudaStreamSynchronize(b.stream);
    cudaFree(b.arena);
    if (b.h_stage) cudaFreeHost(b.h_stage);
    if (b.h_out) cudaFreeHost(b.h_out);
    if (b.stream) cudaStreamDestroy(b.stream);
}

// ---- frame side of the windowed searches: staged from the host view per call, or taken from a device-resident borb_frame
struct FrameInfo { int n, n_levels; float min_x, min_y, max_x, max_y, inv_w, inv_h; bool has_ur; const borb_frame* rf; };
struct FrameStage { size_t keys = 0, desc = 0, ur = 0, occ = 0, sf = 0, cs = 0, ci = 0; bool ur_p = false, occ_p = false; };

FrameInfo frame_info(const borb_frame_view* F) {
    FrameInfo I{};
    I.rf = F->resident;
    if (I.rf) {
        I.n = I.rf->n; I.n_levels = I.rf->n_levels; I.min_x = I.rf->min_x; I.min_y = I.rf->min_y; I.max_x = I.rf->max_x; I.max_y = I.rf->max_y;
        I.has_ur = I.rf->u_right != nullptr;
    } else {
        I.n = F->n; I.n_levels = F->n_levels; I.min_x = F->min_x; I.min_y = F->min_y; I.max_x = F->max_x; I.max_y = F->max_y;
        I.has_ur = F->u_right != nullptr;
    }
    I.inv_w = (float)GRID_COLS / (float)(I.max_x - I.min_x);      // mfGridElementWidthInv (Frame.cc:101)
    I.inv_h = (float)GRID_ROWS / (float)(I.max_y - I.min_y);
    return I;
}
// Frame::AssignFeaturesToGrid of the host views of one call, all in one launch_grid_sort over a FrameJob table of which a view
// fills only the grid fields.  stage_frame counts the views before Call::begin(); stage() then adds the table as an input after the
// views' own, add() fills a view's row once addresses exist, and launch() builds every grid after commit().  A view without
// features is never searched and gets no grid.
class HostGrids {
public:
    void count(const FrameInfo& I) { if (!I.rf && I.n > 0) cap_++; }
    void stage(Call& c) { if (cap_ > 0) off_ = c.in(nullptr, (size_t)cap_ * sizeof(FrameJob)); }
    void add(const Call& c, const FrameInfo& I, borb_keypoint* keys, int* cell_start, int* cell_idx) {
        if (I.rf || I.n == 0) return;
        assert(n_ < cap_);
        FrameJob J{};
        J.keys = keys; J.cell_start = cell_start; J.cell_idx = cell_idx;
        J.n = I.n; J.min_x = I.min_x; J.min_y = I.min_y; J.inv_w = I.inv_w; J.inv_h = I.inv_h;
        c.host<FrameJob>(off_)[n_++] = J;
        max_n_ = std::max(max_n_, I.n);
    }
    int launch(const Call& c, cudaStream_t s) const { return n_ > 0 ? launch_grid_sort((const FrameJob*)c.dev(off_), n_, max_n_, s) : 0; }

private:
    int cap_ = 0, n_ = 0, max_n_ = 0;
    size_t off_ = 0;
};
// the per-call inputs of the frame (everything for a host view; only `occupied` for a resident frame); g counts a host view's grid
FrameStage stage_frame(Call& c, const borb_frame_view* F, const FrameInfo& I, bool want_ur, HostGrids& g) {
    FrameStage fs;
    g.count(I);
    if (!I.rf) {
        fs.keys = c.in(F->keys_un, (size_t)I.n * sizeof(borb_keypoint));
        fs.desc = c.in(F->desc, (size_t)I.n * 32);
        fs.ur_p = want_ur && F->u_right != nullptr;
        if (fs.ur_p) fs.ur = c.in(F->u_right, (size_t)I.n * 4);
        fs.sf = c.in(F->scale_factors, (size_t)(F->scale_factors ? I.n_levels : 0) * 4);
    } else fs.ur_p = want_ur && I.has_ur;
    fs.occ_p = F->occupied != nullptr;
    if (fs.occ_p) fs.occ = c.in(F->occupied, (size_t)I.n);
    return fs;
}
void reserve_grid(Call& c, const FrameInfo& I, FrameStage& fs) {
    if (I.rf) return;
    fs.cs = c.scratch((size_t)(GRID_CELLS + 1) * 4);
    fs.ci = c.scratch((size_t)MATCH_MAX_FEATURES * 4 + 16);
}
// the frame fields of A: the resident frame's, or those of a host view staged at fs, whose grid row g gets
void bind_frame_fields(const FrameInfo& I, const FrameStage& fs, const Call& c, HostGrids& g, ProjArgs& A) {
    A.n = I.n;
    A.minX = I.min_x; A.minY = I.min_y; A.invW = I.inv_w; A.invH = I.inv_h;
    if (const borb_frame* rf = I.rf) {
        A.keys = rf->keys; A.desc = rf->desc; A.u_right = fs.ur_p ? rf->u_right : nullptr; A.scale_factors = rf->sf;
        A.cell_start = rf->cell_start; A.cell_idx = rf->cell_idx;
        return;
    }
    A.keys = (const borb_keypoint*)c.dev(fs.keys); A.desc = c.dev(fs.desc);
    A.u_right = fs.ur_p ? (const float*)c.dev(fs.ur) : nullptr;
    A.scale_factors = (const float*)c.dev(fs.sf);
    A.cell_start = (const int*)c.dev(fs.cs); A.cell_idx = (const int*)c.dev(fs.ci);
    g.add(c, I, (borb_keypoint*)c.dev(fs.keys), (int*)c.dev(fs.cs), (int*)c.dev(fs.ci));
}
// The per-job kernel arguments of a Tracking-thread search.  One job is launched by value (the single calls: no table crosses PCIe);
// more go to a staged table that the *_batch_kernels read.
template <class T> struct JobTable {
    int n;
    size_t off = 0;
    T one{};
    JobTable(Call& c, int n_jobs) : n(n_jobs) { if (n > 1) off = c.in(nullptr, (size_t)n * sizeof(T)); }
    T* host(const Call& c) { return n > 1 ? c.host<T>(off) : &one; }               // after begin()
    const T* dev(const Call& c) const { return n > 1 ? (const T*)c.dev(off) : nullptr; }
};
// A host view's octaves index the level tables in the kernels (mvInvLevelSigma2 in Fuse, mvScaleFactors / mvLevelSigma2 in
// SearchForTriangulation) and are packed into 7 bits of a projection search's candidate entries, where the ratio test compares
// them; so every octave must lie in [0, n_levels), as the extractor makes them.
borb_status check_octaves(const borb_keypoint* k, int n, int n_levels, const char* what) {
    for (int i = 0; i < n; i++)
        if (k[i].octave < 0 || k[i].octave >= n_levels) {
            set_error("%s keypoint %d: octave %d outside [0, %d)", what, i, k[i].octave, n_levels);
            return BORB_ERR_INVALID_ARG;
        }
    return BORB_OK;
}
borb_status check_frame(const borb_frame_view* F, const FrameInfo& I, const borb_matcher* m, const char* what = "frame") {
    if (I.n < 0 || I.n > MATCH_MAX_FEATURES) { set_error("frame has %d features (limit %d)", I.n, MATCH_MAX_FEATURES); return BORB_ERR_INVALID_ARG; }
    if (I.rf) {
        if (I.rf->device != m->device) { set_error("resident frame and matcher live on different devices"); return BORB_ERR_INVALID_ARG; }
        return BORB_OK;
    }
    if (I.n > 0 && (!F->keys_un || !F->desc)) { set_error("incomplete frame view"); return BORB_ERR_INVALID_ARG; }
    if (I.n_levels < 1 || !F->scale_factors || !(I.max_x > I.min_x) || !(I.max_y > I.min_y)) { set_error("incomplete frame view"); return BORB_ERR_INVALID_ARG; }
    return check_octaves(F->keys_un, I.n, I.n_levels, what);
}
// error text of a check shared by the single calls and the batches: the batches prefix it with the job index
borb_status job_fail(bool batch, int j, borb_status s) {
    if (!batch) return s;
    const std::string e = borb_last_error();
    set_error("job %d: %s", j, e.c_str());
    return s;
}
// the candidate search reads its queries from what project_points_kernel wrote
void wire_projection(const LastArgs& L, ProjArgs& A) {
    A.n_mp = L.n_last;
    A.proj_x = L.proj_x; A.proj_y = L.proj_y; A.proj_xr = L.proj_xr; A.mp_valid = L.valid_out;
    A.level = L.level_out; A.view_cos = L.viewcos_out;                                   // variant 3 (mode 0)
    A.q_radius = L.radius; A.q_minl = L.minl; A.q_maxl = L.maxl; A.q_angle = L.angle;   // mode 1
}
// a result block of n entries followed by the match count
void read_counted(const uint8_t* r, int n, int32_t* out, int32_t* count) {
    std::memcpy(out, r, (size_t)n * 4);
    std::memcpy(count, r + (size_t)n * 4, 4);
}

// The checks of a host view, FeatureVector included: the kernels index shared and global memory with its node ranges and feature
// indices, and the staging sizes its uploads from start[n_nodes].
borb_status check_kf(const borb_keyframe_view* v, const char* what) {
    if (!v || v->n < 0 || v->n > MATCH_MAX_FEATURES || (v->n > 0 && (!v->keys_un || !v->desc)) ||
        (v->n_levels < 1 && (v->scale_factors || v->level_sigma2))) {
        set_error("%s: bad keyframe view (n=%d, limit %d)", what, v ? v->n : -1, MATCH_MAX_FEATURES);
        return BORB_ERR_INVALID_ARG;
    }
    if (v->n_levels > 0) {                  // every view with level tables (the searches without them read no octave)
        const borb_status s = check_octaves(v->keys_un, v->n, v->n_levels, what);
        if (s != BORB_OK) return s;
    }
    const borb_featvec_view& fv = v->fv;
    if (fv.n_nodes < 0 || (fv.n_nodes > 0 && (!fv.node_id || !fv.start || !fv.feat_idx))) {
        set_error("%s: bad feature vector", what);
        return BORB_ERR_INVALID_ARG;
    }
    if (fv.n_nodes == 0) return BORB_OK;
    for (int a = 0; a < fv.n_nodes; a++)
        if (fv.start[a + 1] < fv.start[a] || (a == 0 ? fv.start[0] < 0 : fv.node_id[a] <= fv.node_id[a - 1])) {
            set_error("%s: FeatureVector nodes must ascend", what);
            return BORB_ERR_INVALID_ARG;
        }
    for (int r = 0; r < fv.start[fv.n_nodes]; r++)
        if (fv.feat_idx[r] >= (uint32_t)v->n) {
            set_error("%s: FeatureVector index %u outside the keyframe's %d features", what, fv.feat_idx[r], v->n);
            return BORB_ERR_INVALID_ARG;
        }
    return BORB_OK;
}

const borb_keyframe_view NO_VIEW{};          // the view of a resident side that takes nothing from the caller

// One side of a BoW-guided search (SearchByBoW, SearchForTriangulation, the frame of the database search): a host view v, staged per
// call, or a resident frame rf with its BoW, of which only v's has_mp and level_sigma2, when given, cross PCIe.  stage() comes before
// Call::begin(), bind() after it.
struct KfSide {
    const borb_keyframe_view* v = &NO_VIEW;
    const borb_frame* rf = nullptr;
    size_t keys = 0, desc = 0, has_mp = 0, u_right = 0, node = 0, start = 0, idx = 0, sf = 0, sig = 0;

    int n() const { return rf ? rf->n : v->n; }
    int nn() const { return rf ? rf->n_nodes : v->fv.n_nodes; }
    int m() const { return rf ? rf->n_fv : (v->fv.n_nodes > 0 ? v->fv.start[v->fv.n_nodes] : 0); }   // features inside the nodes
    void stage(Call& c) {
        if (v->has_mp) has_mp = c.in(v->has_mp, (size_t)n());
        if (v->level_sigma2) sig = c.in(v->level_sigma2, (size_t)(rf ? rf->n_levels : v->n_levels) * 4);
        if (rf) return;
        keys = c.in(v->keys_un, (size_t)v->n * sizeof(borb_keypoint));
        desc = c.in(v->desc, (size_t)v->n * 32);
        if (v->u_right) u_right = c.in(v->u_right, (size_t)v->n * 4);
        node = c.in(v->fv.node_id, (size_t)nn() * 4);
        start = c.in(v->fv.start, (size_t)(nn() > 0 ? nn() + 1 : 0) * 4);
        idx = c.in(v->fv.feat_idx, (size_t)m() * 4);
        if (v->scale_factors) sf = c.in(v->scale_factors, (size_t)v->n_levels * 4);
    }
    KfDev bind(const Call& c) const {
        KfDev d{};
        d.n = n(); d.nn = nn();
        d.has_mp = v->has_mp ? c.dev(has_mp) : nullptr;
        d.level_sigma2 = v->level_sigma2 ? reinterpret_cast<const float*>(c.dev(sig)) : nullptr;
        if (rf) {
            d.keys = rf->keys; d.desc = rf->desc; d.u_right = rf->u_right; d.scale_factors = rf->sf;
            d.node = rf->fv_node; d.start = rf->fv_start; d.idx = rf->fv_idx;
            return d;
        }
        d.keys = reinterpret_cast<const borb_keypoint*>(c.dev(keys));
        d.desc = c.dev(desc);
        d.u_right = v->u_right ? reinterpret_cast<const float*>(c.dev(u_right)) : nullptr;
        d.scale_factors = v->scale_factors ? reinterpret_cast<const float*>(c.dev(sf)) : nullptr;
        d.node = reinterpret_cast<const uint32_t*>(c.dev(node));
        d.start = reinterpret_cast<const int32_t*>(c.dev(start));
        d.idx = reinterpret_cast<const uint32_t*>(c.dev(idx));
        return d;
    }
};

// packed vocabulary blob: header {magic, n_nodes, k, L, offsets...} followed by 256-byte aligned sections
struct VocHeader { uint32_t magic; int32_t n_nodes, k, L; uint64_t off_desc, off_weight, off_word, off_cstart, off_cids, bytes; };
constexpr uint32_t VOC_MAGIC = 0x42564f43u;   // "BVOC"

void voc_views(borb_voc* v, const VocHeader& h) {
    v->dev.n_nodes = h.n_nodes; v->dev.k = h.k; v->dev.L = h.L;
    v->dev.desc = v->blob + h.off_desc;
    v->dev.weight = reinterpret_cast<const double*>(v->blob + h.off_weight);
    v->dev.word_id = reinterpret_cast<const int32_t*>(v->blob + h.off_word);
    v->dev.child_start = reinterpret_cast<const int32_t*>(v->blob + h.off_cstart);
    v->dev.child_ids = reinterpret_cast<const int32_t*>(v->blob + h.off_cids);
}

// One frame of a BoW call: a resident frame f, whose tables get the vectors, or the caller's n host descriptors desc, staged,
// whose vectors go to result slots.  The host copies it wants: the vectors and their counts, or with descent only the
// per-feature word / weight / node; a null pointer is not copied.
struct BowSide {
    borb_frame* f = nullptr;
    const uint8_t* desc = nullptr;
    int n = 0;
    BowTables out{};
    int32_t* n_bow = nullptr;
    int32_t* n_nodes = nullptr;
    int32_t* word = nullptr;
    double* weight = nullptr;
    int32_t* node = nullptr;
};

// TemplatedVocabulary::transform of n_jobs frames on one Call: the descent (bow_transform_batch_kernel) and, unless descent_only,
// the BowVector / FeatureVector bookkeeping (bow_build_kernel); one synchronisation.  A resident frame waits for its ready event,
// and gets it recorded again and its counts set.
borb_status bow_jobs(CallBuffers* cb, const VocDev& V, const BowSide* S, int n_jobs, int levelsup, bool descent_only, uint64_t* launches) {
    Call c(cb);
    const size_t o_jobs = c.in(nullptr, (size_t)n_jobs * sizeof(BowFrameJob));     // filled in place
    std::vector<size_t> o_desc(n_jobs, 0), o_scr(n_jobs), o_res(n_jobs, 0);
    std::vector<char> has_res(n_jobs, 0);
    int max_n = 0;
    for (int i = 0; i < n_jobs; i++) {
        if (!S[i].f) o_desc[i] = c.in(S[i].desc, (size_t)S[i].n * 32);
        max_n = std::max(max_n, S[i].n);
    }
    const size_t o_jobs_dev = c.scratch((size_t)n_jobs * sizeof(BowFrameJob));   // the job table the kernels read
    const size_t r_cnt = c.result((size_t)n_jobs * 12);     // (n_bow, n_nodes, fv_start[n_nodes]) of every frame, then the tables
    for (int i = 0; i < n_jobs; i++) {
        const BowSide& b = S[i];
        const size_t n = (size_t)b.n;
        o_scr[i] = descent_only ? c.result(n * 16) : c.scratch(n * 16);        // weight f64 | word i32 | node i32
        has_res[i] = !descent_only && (!b.f || b.out.word || b.out.value || b.out.node || b.out.start || b.out.idx);
        if (has_res[i]) o_res[i] = c.result(n * 24 + 4);                        // value | word | node | start | idx
    }
    // Small inputs are read in place, as the descent reads each descriptor once.  The job table is not: every warp of both kernels
    // reads its job, which from pinned memory costs a PCIe round trip per warp (DESIGN §5, "The single calls later became one-frame
    // jobs"), so it gets a device copy of its own.  Results: a small call on host descriptors only (a single call) has the kernels
    // write them straight into the pinned landing buffer, so no D2H copy; otherwise they come back in one download.
    borb_status s;
    if ((s = c.begin(true)) != BORB_OK) return s;
    const bool direct = c.in_place() && std::none_of(S, S + n_jobs, [](const BowSide& b) { return b.f != nullptr; });
    BowFrameJob* hj = c.host<BowFrameJob>(o_jobs);
    for (int i = 0; i < n_jobs; i++) {
        const BowSide& b = S[i];
        const size_t n = (size_t)b.n;
        BowFrameJob J{};
        J.desc = b.f ? b.f->desc : c.dev(o_desc[i]); J.n = b.n;
        uint8_t* w = descent_only ? c.res(o_scr[i], direct) : c.dev(o_scr[i]);
        J.weight = (double*)w; J.word = (int32_t*)(w + n * 8); J.node = (int32_t*)(w + n * 12);
        if (has_res[i]) {
            uint8_t* r = c.res(o_res[i], direct);
            (b.f ? J.copy : J.dst) = BowTables{(uint32_t*)(r + n * 8), (double*)r, (uint32_t*)(r + n * 12), (int32_t*)(r + n * 16), (uint32_t*)(r + n * 20 + 4)};
        }
        if (b.f && !descent_only) {
            J.dst = BowTables{b.f->bow_word, b.f->bow_value, b.f->fv_node, b.f->fv_start, b.f->fv_idx};
            b.f->has_bow = false;                       // the storage is rewritten from here on
        }
        J.counts = (int32_t*)c.res(r_cnt, direct) + 3 * i;
        hj[i] = J;
    }
    if ((s = c.commit()) != BORB_OK) return s;
    const size_t o_table = c.in_place() ? o_jobs_dev : o_jobs;
    if (c.in_place()) BORB_CUDA(cudaMemcpyAsync(c.dev(o_table), hj, (size_t)n_jobs * sizeof(BowFrameJob), cudaMemcpyHostToDevice, cb->stream));
    for (int i = 0; i < n_jobs; i++)
        if (S[i].f && (s = c.wait(S[i].f)) != BORB_OK) return s;
    const int nl = launch_bow_frames(V, (const BowFrameJob*)c.dev(o_table), n_jobs, max_n, levelsup, descent_only, cb->stream);
    if (launches) *launches += nl;
    for (int i = 0; i < n_jobs; i++)
        if (S[i].f) BORB_CUDA(cudaEventRecord(S[i].f->ready, cb->stream));
    if ((s = c.finish()) != BORB_OK) return s;
    for (int i = 0; i < n_jobs; i++) {
        const BowSide& b = S[i];
        const size_t n = (size_t)b.n;
        if (descent_only) {
            const uint8_t* w = c.out(o_scr[i]);
            std::memcpy(b.weight, w, n * 8); std::memcpy(b.word, w + n * 8, n * 4); std::memcpy(b.node, w + n * 12, n * 4);
            continue;
        }
        int32_t cnt[3];
        std::memcpy(cnt, c.out(r_cnt) + (size_t)i * 12, 12);
        if (b.f) { b.f->n_bow = cnt[0]; b.f->n_nodes = cnt[1]; b.f->n_fv = cnt[2]; b.f->has_bow = true; }
        if (b.n_bow) *b.n_bow = cnt[0];
        if (b.n_nodes) *b.n_nodes = cnt[1];
        if (!has_res[i]) continue;
        const uint8_t* r = c.out(o_res[i]);
        if (b.out.value) std::memcpy(b.out.value, r, (size_t)cnt[0] * 8);
        if (b.out.word) std::memcpy(b.out.word, r + n * 8, (size_t)cnt[0] * 4);
        if (b.out.node) std::memcpy(b.out.node, r + n * 12, (size_t)cnt[1] * 4);
        if (b.out.start) std::memcpy(b.out.start, r + n * 16, (size_t)(cnt[1] + 1) * 4);
        if (b.out.idx) std::memcpy(b.out.idx, r + n * 20 + 4, (size_t)cnt[2] * 4);
    }
    return BORB_OK;
}

}  // namespace

extern "C" {

borb_status borb_matcher_create(int device, borb_matcher** out) {
    if (!out) return BORB_ERR_INVALID_ARG;
    *out = nullptr;
    int ndev = 0;
    borb_status st = borb_device_count(&ndev);
    if (st != BORB_OK) return st;
    if (ndev < 1) { set_error("no CUDA device visible; libborb has no CPU fallback"); return BORB_ERR_NO_DEVICE; }
    if (device < 0 || device >= ndev) { set_error("device %d out of range", device); return BORB_ERR_INVALID_ARG; }
    borb_matcher* m = new borb_matcher();
    m->device = device;
    cudaError_t e = cudaSetDevice(device);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&m->n_sm, cudaDevAttrMultiProcessorCount, device);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) { set_error("CUDA init failed: %s", cudaGetErrorString(e)); delete m; return BORB_ERR_CUDA; }
    if (m->n_sm < 1) m->n_sm = 1;
    *out = m;
    return BORB_OK;
}

borb_status borb_matcher_destroy(borb_matcher* m) {
    if (!m) return BORB_OK;
    free_call_buffers(*m);
    if (m->ev_a) { cudaEventDestroy(m->ev_a); cudaEventDestroy(m->ev_b); }
    if (m->ev_r) cudaEventDestroy(m->ev_r);
    if (m->t0) { cudaEventDestroy(m->t0); cudaEventDestroy(m->t1); }
    delete m;
    return BORB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Device-resident Frame.  Blocks of destroyed frames are recycled (a tracker creates one per camera frame).
namespace {
std::mutex g_frame_pool_mu;
std::vector<borb_frame*> g_frame_pool;

borb_status frame_alloc(int device, int n, int n_levels, bool stereo, borb_frame** out) {
    borb_frame* f = nullptr;
    {
        std::lock_guard<std::mutex> lk(g_frame_pool_mu);
        for (size_t i = 0; i < g_frame_pool.size(); i++)
            if (g_frame_pool[i]->device == device && g_frame_pool[i]->cap >= n) { f = g_frame_pool[i]; g_frame_pool.erase(g_frame_pool.begin() + i); break; }
    }
    if (!f) {
        f = new borb_frame();
        f->device = device;
        f->cap = n < 2048 ? 2048 : ((n + 1023) & ~1023);
        size_t off = 0;
        auto put = [&](size_t bytes) { off = (off + 255) & ~size_t(255); const size_t o = off; off += bytes; return o; };
        const size_t o_k = put((size_t)f->cap * sizeof(borb_keypoint)), o_d = put((size_t)f->cap * 32), o_u = put((size_t)f->cap * 4), o_z = put((size_t)f->cap * 4);
        const size_t o_s = put(BORB_MAX_LEVELS * 4), o_cs = put((size_t)(GRID_CELLS + 1) * 4), o_ci = put((size_t)MATCH_MAX_FEATURES * 4 + 16);
        const size_t o_bv = put((size_t)f->cap * 8), o_bw = put((size_t)f->cap * 4), o_fn = put((size_t)f->cap * 4);
        const size_t o_fs = put((size_t)(f->cap + 1) * 4), o_fi = put((size_t)f->cap * 4);
        cudaError_t e = cudaMalloc(&f->block, off + 256);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&f->ready, cudaEventDisableTiming);
        if (e != cudaSuccess) { set_error("frame allocation failed: %s", cudaGetErrorString(e)); cudaFree(f->block); delete f; return BORB_ERR_CUDA; }
        f->block_bytes = off + 256;
        f->keys = (borb_keypoint*)(f->block + o_k); f->desc = f->block + o_d; f->ur_store = (float*)(f->block + o_u); f->depth_store = (float*)(f->block + o_z);
        f->sf = (float*)(f->block + o_s); f->cell_start = (int*)(f->block + o_cs); f->cell_idx = (int*)(f->block + o_ci);
        f->bow_value = (double*)(f->block + o_bv); f->bow_word = (uint32_t*)(f->block + o_bw); f->fv_node = (uint32_t*)(f->block + o_fn);
        f->fv_start = (int32_t*)(f->block + o_fs); f->fv_idx = (uint32_t*)(f->block + o_fi);
    }
    f->has_bow = false;                // a new frame, or a recycled block that still holds another frame's vectors
    f->n_bow = f->n_nodes = f->n_fv = 0;
    // u_right / depth storage always exists; the pointers are nulled for a monocular frame
    f->u_right = stereo ? f->ur_store : nullptr;
    f->depth = stereo ? f->depth_store : nullptr;
    f->n = n; f->n_levels = n_levels;
    *out = f;
    return BORB_OK;
}
// borb_debug_set_poison: the whole block of a frame handed out by frame_alloc, new or recycled, on the stream that then writes it
borb_status poison_frame(const borb_frame* f, cudaStream_t s) {
    const int p = poison_byte();
    if (p >= 0) BORB_CUDA(cudaMemsetAsync(f->block, p, f->block_bytes, s));
    return BORB_OK;
}
}  // namespace

borb_status borb_frame_create(borb_matcher* m, const borb_frame_view* v, borb_frame** out) {
    if (!m || !v || !out) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    *out = nullptr;
    if (v->resident) { set_error("the view already refers to a resident frame"); return BORB_ERR_INVALID_ARG; }
    const FrameInfo I = frame_info(v);
    borb_status s = check_frame(v, I, m);
    if (s != BORB_OK) return s;
    if (I.n_levels > BORB_MAX_LEVELS) { set_error("too many levels"); return BORB_ERR_INVALID_ARG; }
    BORB_CUDA(cudaSetDevice(m->device));
    borb_frame* f = nullptr;
    if ((s = frame_alloc(m->device, I.n, I.n_levels, v->u_right != nullptr, &f)) != BORB_OK) return s;
    f->depth = nullptr;                 // a view carries mvuRight but no mvDepth: nothing is written to depth_store
    f->min_x = I.min_x; f->min_y = I.min_y; f->max_x = I.max_x; f->max_y = I.max_y;
    Call c(m);
    HostGrids g;                                         // the frame's grid, built in its block
    borb_frame_view V = *v;
    V.occupied = nullptr;                                // a per-call input of the searches, not part of the frame
    const FrameStage fs = stage_frame(c, &V, I, true, g);
    g.stage(c);
    if ((s = c.begin()) != BORB_OK) { borb_frame_destroy(f); return s; }
    g.add(c, I, f->keys, f->cell_start, f->cell_idx);
    if ((s = c.commit()) != BORB_OK) { borb_frame_destroy(f); return s; }
    cudaStream_t q = m->stream;
    if ((s = poison_frame(f, q)) != BORB_OK) return s;
    if (I.n > 0) {
        BORB_CUDA(cudaMemcpyAsync(f->keys, c.dev(fs.keys), (size_t)I.n * sizeof(borb_keypoint), cudaMemcpyDeviceToDevice, q));
        BORB_CUDA(cudaMemcpyAsync(f->desc, c.dev(fs.desc), (size_t)I.n * 32, cudaMemcpyDeviceToDevice, q));
        if (fs.ur_p) BORB_CUDA(cudaMemcpyAsync(f->u_right, c.dev(fs.ur), (size_t)I.n * 4, cudaMemcpyDeviceToDevice, q));
    }
    BORB_CUDA(cudaMemcpyAsync(f->sf, c.dev(fs.sf), (size_t)I.n_levels * 4, cudaMemcpyDeviceToDevice, q));
    m->launches += g.launch(c, q);
    if (I.n == 0) BORB_CUDA(cudaMemsetAsync(f->cell_start, 0, (size_t)(GRID_CELLS + 1) * 4, q));
    BORB_CUDA(cudaEventRecord(f->ready, q));
    if ((s = c.finish()) != BORB_OK) return s;       // the staging arena is reused by the next call on this matcher
    *out = f;
    return BORB_OK;
}

borb_status borb_frame_destroy(borb_frame* f) {
    if (!f) return BORB_OK;
    std::lock_guard<std::mutex> lk(g_frame_pool_mu);
    if (g_frame_pool.size() < 1024) { g_frame_pool.push_back(f); return BORB_OK; }     // ~235 KB each (2048 features); a multi-stream server keeps hundreds alive
    cudaSetDevice(f->device);
    cudaEventSynchronize(f->ready);
    cudaFree(f->block);
    cudaEventDestroy(f->ready);
    delete f;
    return BORB_OK;
}

namespace {
// What borb_frame_from_extractors adds to the one-frame build of image 0: the extractors' own keypoints and descriptors and the
// feature grid, copied into the same result region as mvKeysUn / mvuRight / mvDepth.
struct FrameHostCopies {
    borb_frame_host* host;
    const borb_extractor* right;    // stereo: mvKeysRight / mDescriptorsRight come from image 0 of this handle
    int n_right;
};

borb_status check_frames_args(borb_matcher* m, borb_extractor* e, const borb_camera* cam, int mode, const void* depth, int depth_type) {
    depth_type &= 3;
    if (mode < 0 || mode > 2 || (mode == 2 && !depth) || (depth_type != 0 && depth_type != 1)) { set_error("bad mode / depth arguments"); return BORB_ERR_INVALID_ARG; }
    if (!e->have_geom || e->last_n_images < 1) { set_error("no extracted batch on this extractor handle"); return BORB_ERR_STATE; }
    if (e->device != m->device) { set_error("extractor and matcher live on different devices"); return BORB_ERR_INVALID_ARG; }
    (void)cam;
    return BORB_OK;
}

borb_status build_frames(borb_matcher* m, borb_extractor* e, const int32_t* images, int n_frames, const int32_t* n_keys,
                         const borb_camera* cam, int mode, const void* const* depth, int depth_type, float depth_factor,
                         int depth_stride_bytes, borb_keypoint* keys_un, float* u_right, float* depth_out, int cap,
                         float* bounds4, borb_frame** frames, const FrameHostCopies* hc);
}  // namespace

borb_status borb_frames_from_extractor(borb_matcher* m, borb_extractor* e, const int32_t* images, int n_frames, const int32_t* n_keys,
                                       const borb_camera* cam, int mode, const void* const* depth, int depth_type, float depth_factor,
                                       int depth_stride_bytes, borb_keypoint* keys_un, float* u_right, float* depth_out, int cap,
                                       float* bounds4, borb_frame** frames) {
    if (!m || !e || !cam || !frames || n_frames < 0 || (n_frames > 0 && (!images || !n_keys))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_status s = check_frames_args(m, e, cam, mode, depth, depth_type);
    if (s != BORB_OK) return s;
    if ((keys_un || u_right || depth_out) && cap < 0) { set_error("negative capacity"); return BORB_ERR_INVALID_ARG; }
    return build_frames(m, e, images, n_frames, n_keys, cam, mode, depth, depth_type, depth_factor, depth_stride_bytes, keys_un, u_right,
                        depth_out, cap, bounds4, frames, nullptr);
}

borb_status borb_frame_from_extractors(borb_matcher* m, borb_extractor* left, borb_extractor* right, const borb_camera* cam, int mode,
                                       float b, const void* depth, int depth_type, float depth_factor, int depth_stride_bytes,
                                       borb_frame_host* host, borb_frame** out) {
    if (!m) { set_error("null argument: m"); return BORB_ERR_INVALID_ARG; }
    if (!left) { set_error("null argument: left"); return BORB_ERR_INVALID_ARG; }
    if (!cam) { set_error("null argument: cam"); return BORB_ERR_INVALID_ARG; }
    if (!host) { set_error("null argument: host"); return BORB_ERR_INVALID_ARG; }
    if (!out) { set_error("null argument: out"); return BORB_ERR_INVALID_ARG; }
    *out = nullptr;
    host->n = host->n_right = 0;
    if (host->cap < 0) { set_error("host->cap is negative (%d)", host->cap); return BORB_ERR_INVALID_ARG; }
    if ((mode == 1) != (right != nullptr)) { set_error("right: a stereo frame (mode 1) takes a right handle, other modes none"); return BORB_ERR_INVALID_ARG; }
    if (right == left) { set_error("right: the same handle as left"); return BORB_ERR_INVALID_ARG; }
    if (mode == 1 && !(b > 0.f)) { set_error("b: mb = mbf/fx must be positive (%g)", (double)b); return BORB_ERR_INVALID_ARG; }
    borb_status s = check_frames_args(m, left, cam, mode, depth, depth_type);
    if (s != BORB_OK) return s;
    if (right && (s = check_stereo_pair(left, right)) != BORB_OK) return s;
    // the frame is built before its keypoint counts reach the host: everything is sized by the handles' capacities (one image each)
    const int bound = left->geom.sel_image_stride, bound_r = right ? right->geom.sel_image_stride : 0;
    if (bound > MATCH_MAX_FEATURES || bound_r > MATCH_MAX_FEATURES) {
        set_error("left/right: up to %d / %d keypoints per image (limit %d per frame)", bound, bound_r, MATCH_MAX_FEATURES);
        return BORB_ERR_INVALID_ARG;
    }
    if (host->cap < bound || host->cap < bound_r) {
        set_error("host->cap %d: the handles return up to %d / %d keypoints (borb_extractor_capacity)", host->cap, bound, bound_r);
        return BORB_ERR_CAPACITY;
    }
    BORB_CUDA(cudaSetDevice(m->device));
    if (right) {    // the association on the left stream reads the right handle's extraction: ordered by an event, not by the host
        if (!m->ev_r) BORB_CUDA(cudaEventCreateWithFlags(&m->ev_r, cudaEventDisableTiming));
        BORB_CUDA(cudaEventRecord(m->ev_r, right->stream));
        BORB_CUDA(cudaStreamWaitEvent(left->stream, m->ev_r, 0));
        if ((s = enqueue_stereo_pair(left, right, cam->bf, b)) != BORB_OK) return s;
    }
    const int32_t image = 0;
    const FrameHostCopies hc{host, right, bound_r};
    return build_frames(m, left, &image, 1, &bound, cam, mode, mode == 2 ? &depth : nullptr, depth_type, depth_factor, depth_stride_bytes,
                        host->keys_un, host->u_right, host->depth, bound, host->bounds, out, &hc);
}

namespace {
borb_status build_frames(borb_matcher* m, borb_extractor* e, const int32_t* images, int n_frames, const int32_t* n_keys,
                         const borb_camera* cam, int mode, const void* const* depth, int depth_type, float depth_factor,
                         int depth_stride_bytes, borb_keypoint* keys_un, float* u_right, float* depth_out, int cap,
                         float* bounds4, borb_frame** frames, const FrameHostCopies* hc) {
    const bool depth_on_device = (depth_type & 4) != 0;
    depth_type &= 3;
    const Geometry& g = e->geom;
    const int w = g.w, h = g.h, nl = g.nlevels;
    float b4[4];
    host_image_bounds(w, h, *cam, b4);
    if (bounds4) std::memcpy(bounds4, b4, sizeof(b4));
    for (int i = 0; i < n_frames; i++) frames[i] = nullptr;
    if (n_frames == 0) return BORB_OK;
    int max_n = 0;
    for (int i = 0; i < n_frames; i++) {
        if (images[i] < 0 || images[i] >= e->last_n_images) { set_error("image %d is not part of the extractor's last batch", images[i]); return BORB_ERR_INVALID_ARG; }
        if (n_keys[i] < 0 || n_keys[i] > g.sel_image_stride || n_keys[i] > MATCH_MAX_FEATURES) { set_error("frame %d: %d keypoints outside [0, %d]", i, n_keys[i], MATCH_MAX_FEATURES); return BORB_ERR_INVALID_ARG; }
        if (mode == 1 && (images[i] & 1)) { set_error("stereo mode takes LEFT images (even indices) of borb_stereo_frames"); return BORB_ERR_INVALID_ARG; }
        if (mode == 2 && !depth[i]) { set_error("frame %d: null depth map", i); return BORB_ERR_INVALID_ARG; }
        max_n = n_keys[i] > max_n ? n_keys[i] : max_n;
    }
    BORB_CUDA(cudaSetDevice(m->device));
    borb_status s = BORB_OK;
    for (int i = 0; i < n_frames && s == BORB_OK; i++) {
        s = frame_alloc(m->device, n_keys[i], nl, mode != 0, &frames[i]);
        if (s == BORB_OK) { frames[i]->min_x = b4[0]; frames[i]->min_y = b4[1]; frames[i]->max_x = b4[2]; frames[i]->max_y = b4[3]; }
    }
    auto fail = [&](borb_status st) { for (int i = 0; i < n_frames; i++) { borb_frame_destroy(frames[i]); frames[i] = nullptr; } return st; };
    if (s != BORB_OK) return fail(s);
    const size_t px = depth_type == 1 ? 2 : 4;
    const size_t depth_img_bytes = (mode == 2 && !depth_on_device) ? (size_t)w * h * px : 0;
    if (mode == 2 && !depth_on_device && depth_stride_bytes < (int)(w * px)) { set_error("depth stride %d smaller than a row", depth_stride_bytes); return fail(BORB_ERR_INVALID_ARG); }
    const int ocap = (keys_un || u_right || depth_out) ? cap : 0;
    Call c(m);
    const size_t o_jobs = c.in(nullptr, (size_t)n_frames * sizeof(FrameJob));     // filled in place
    const size_t o_sf = c.in(e->scale.data(), (size_t)nl * 4);
    const size_t o_depth = c.scratch(depth_img_bytes * n_frames + 16);
    // the requested outputs; the kernel writes depth_out wherever it writes u_right
    const size_t kb = keys_un ? (size_t)n_frames * ocap * sizeof(borb_keypoint) : 0, fb = (u_right || depth_out) ? (size_t)n_frames * ocap * 4 : 0;
    const size_t r_k = c.result(kb), r_u = c.result(fb), r_d = c.result(fb);
    // borb_frame_from_extractors: one frame, image 0, sized by the handles' capacities; its counts, mvKeys / mDescriptors (and the
    // right image's) and the grid join the results, and every result is written straight into the landing buffer by the kernels,
    // only as many elements as the device-side counts say
    borb_frame_host* H = hc ? hc->host : nullptr;
    const bool direct = H != nullptr;
    const size_t n0 = (size_t)n_keys[0], nr = hc ? (size_t)hc->n_right : 0;
    const bool want_grid = H && (H->cell_start || H->cell_idx);
    const size_t xk = H && H->keys ? n0 * sizeof(borb_keypoint) : 0, xd = H && H->desc ? n0 * 32 : 0;
    const size_t xkr = H && H->keys_right ? nr * sizeof(borb_keypoint) : 0, xdr = H && H->desc_right ? nr * 32 : 0;
    const size_t xcs = want_grid ? (size_t)(GRID_CELLS + 1) * 4 : 0, xci = H && H->cell_idx ? n0 * 4 : 0;
    const size_t r_xk = c.result(xk), r_xd = c.result(xd), r_xkr = c.result(xkr), r_xdr = c.result(xdr), r_xcs = c.result(xcs), r_xci = c.result(xci);
    const size_t r_cnt = c.result(H ? 2 * sizeof(int32_t) : 0);
    if ((s = c.begin()) != BORB_OK) return fail(s);
    FrameJob* hj = c.host<FrameJob>(o_jobs);
    const float invW = (float)GRID_COLS / (float)(b4[2] - b4[0]), invH = (float)GRID_ROWS / (float)(b4[3] - b4[1]);
    for (int i = 0; i < n_frames; i++) {
        FrameJob& J = hj[i];
        borb_frame* f = frames[i];
        const int img = images[i];
        J.src_keys = e->ws.kps + (size_t)img * g.sel_image_stride;
        J.src_desc = e->ws.desc + (size_t)img * g.sel_image_stride * 32;
        J.src_ur = mode == 1 ? e->ws.u_right + (size_t)(img / 2) * g.sel_image_stride : nullptr;
        J.src_depth = mode == 1 ? e->ws.depth + (size_t)(img / 2) * g.sel_image_stride : nullptr;
        J.depth_img = mode == 2 ? (depth_on_device ? depth[i] : (const void*)(c.dev(o_depth) + (size_t)i * depth_img_bytes)) : nullptr;
        J.keys = f->keys; J.desc = f->desc; J.u_right = f->ur_store; J.depth = f->depth_store;
        J.cell_start = f->cell_start; J.cell_idx = f->cell_idx;
        J.n = n_keys[i]; J.min_x = b4[0]; J.min_y = b4[1]; J.inv_w = invW; J.inv_h = invH;
    }
    if ((s = c.commit()) != BORB_OK) return fail(s);
    cudaStream_t q = m->stream;
    // the extractor's results must be complete, and its next batch must not overwrite them while they are being read
    if (!m->ev_a) { BORB_CUDA(cudaEventCreateWithFlags(&m->ev_a, cudaEventDisableTiming)); BORB_CUDA(cudaEventCreateWithFlags(&m->ev_b, cudaEventDisableTiming)); }
    BORB_CUDA(cudaEventRecord(m->ev_a, e->stream));
    BORB_CUDA(cudaStreamWaitEvent(q, m->ev_a, 0));
    for (int i = 0; i < n_frames; i++)
        if ((s = poison_frame(frames[i], q)) != BORB_OK) return fail(s);
    if (mode == 2 && !depth_on_device)
        for (int i = 0; i < n_frames; i++)
            BORB_CUDA(cudaMemcpy2DAsync(c.dev(o_depth) + (size_t)i * depth_img_bytes, (size_t)w * px, depth[i], (size_t)depth_stride_bytes, (size_t)w * px, h,
                                        cudaMemcpyHostToDevice, q));
    for (int i = 0; i < n_frames; i++) BORB_CUDA(cudaMemcpyAsync(frames[i]->sf, c.dev(o_sf), (size_t)nl * 4, cudaMemcpyDeviceToDevice, q));
    // the frame's keypoint count is the extraction's, read on the device
    if (H) BORB_CUDA(cudaMemcpyAsync(c.dev(o_jobs) + offsetof(FrameJob, n), e->ws.nkp, sizeof(int), cudaMemcpyDeviceToDevice, q));
    m->launches += launch_frame_build((const FrameJob*)c.dev(o_jobs), n_frames, max_n, *cam, mode, depth_type, depth_factor, w, h, ocap,
                                      keys_un ? (borb_keypoint*)c.res(r_k, direct) : nullptr, fb ? (float*)c.res(r_u, direct) : nullptr,
                                      (float*)c.res(r_d, direct), q);
    if (H) {
        const int* cnt_r = hc->right ? hc->right->ws.nkp : nullptr;
        HostCopies hcp{};
        auto seg = [&](size_t r, size_t bytes, const void* src, const int* count, int fixed, int elem_words) {
            if (bytes) hcp.seg[hcp.n++] = HostCopy{src, c.res(r, true), count, fixed, elem_words};
        };
        seg(r_cnt, 4, e->ws.nkp, nullptr, 1, 1);
        seg(r_cnt + 4, hc->right ? 4 : 0, cnt_r, nullptr, 1, 1);
        seg(r_xk, xk, e->ws.kps, e->ws.nkp, 0, sizeof(borb_keypoint) / 4);
        seg(r_xd, xd, e->ws.desc, e->ws.nkp, 0, 8);
        seg(r_xkr, xkr, hc->right ? (const void*)hc->right->ws.kps : nullptr, cnt_r, 0, sizeof(borb_keypoint) / 4);
        seg(r_xdr, xdr, hc->right ? (const void*)hc->right->ws.desc : nullptr, cnt_r, 0, 8);
        seg(r_xcs, xcs, frames[0]->cell_start, nullptr, GRID_CELLS + 1, 1);
        seg(r_xci, xci, frames[0]->cell_idx, frames[0]->cell_start + GRID_CELLS, 0, 1);
        m->launches += launch_host_copy(hcp, q);
    }
    for (int i = 0; i < n_frames; i++) BORB_CUDA(cudaEventRecord(frames[i]->ready, q));
    BORB_CUDA(cudaEventRecord(m->ev_b, q));
    BORB_CUDA(cudaStreamWaitEvent(e->stream, m->ev_b, 0));
    if (hc && hc->right) BORB_CUDA(cudaStreamWaitEvent(hc->right->stream, m->ev_b, 0));
    if ((s = c.finish()) != BORB_OK) return s;
    if (H) {    // the one wait is over: the counts are known
        const int32_t* cnt = (const int32_t*)c.out(r_cnt);
        const int n = cnt[0], n_r = hc->right ? cnt[1] : 0;
        if (n < 0 || (size_t)n > n0 || n_r < 0 || (size_t)n_r > nr) { set_error("keypoint counts %d / %d beyond the handles' capacities", n, n_r); return fail(BORB_ERR_STATE); }
        frames[0]->n = n;
        H->n = n; H->n_right = n_r;
        if (keys_un) std::memcpy(keys_un, c.out(r_k), (size_t)n * sizeof(borb_keypoint));
        if (u_right) std::memcpy(u_right, c.out(r_u), (size_t)n * 4);
        if (depth_out) std::memcpy(depth_out, c.out(r_d), (size_t)n * 4);
        if (xk) std::memcpy(H->keys, c.out(r_xk), (size_t)n * sizeof(borb_keypoint));
        if (xd) std::memcpy(H->desc, c.out(r_xd), (size_t)n * 32);
        if (xkr) std::memcpy(H->keys_right, c.out(r_xkr), (size_t)n_r * sizeof(borb_keypoint));
        if (xdr) std::memcpy(H->desc_right, c.out(r_xdr), (size_t)n_r * 32);
        if (want_grid) {
            const int32_t* cs = (const int32_t*)c.out(r_xcs);
            const int in_grid = cs[GRID_CELLS];
            if (in_grid < 0 || in_grid > n) { set_error("grid of %d entries for %d features", in_grid, n); return fail(BORB_ERR_STATE); }
            if (H->cell_start) std::memcpy(H->cell_start, cs, xcs);
            if (H->cell_idx && in_grid > 0) std::memcpy(H->cell_idx, c.out(r_xci), (size_t)in_grid * 4);
        }
        return BORB_OK;
    }
    if (ocap > 0) {
        if (keys_un) std::memcpy(keys_un, c.out(r_k), kb);
        if (u_right) std::memcpy(u_right, c.out(r_u), fb);
        if (depth_out) std::memcpy(depth_out, c.out(r_d), fb);
    }
    return BORB_OK;
}
}  // namespace

borb_status borb_frame_info(const borb_frame* f, int32_t* n, int32_t* n_levels, int32_t* has_u_right) {
    if (!f) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (n) *n = f->n;
    if (n_levels) *n_levels = f->n_levels;
    if (has_u_right) *has_u_right = f->u_right != nullptr;
    return BORB_OK;
}

borb_status borb_debug_frame_read(const borb_frame* f, borb_keypoint* keys, uint8_t* desc, float* u_right, float* depth, int32_t* cell_start,
                                  int32_t* cell_idx) {
    if (!f) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if ((u_right || depth) && !f->u_right) { set_error("a monocular frame has no mvuRight / mvDepth"); return BORB_ERR_INVALID_ARG; }
    if (depth && !f->depth) { set_error("a frame made by borb_frame_create has no mvDepth"); return BORB_ERR_INVALID_ARG; }
    BORB_CUDA(cudaSetDevice(f->device));
    BORB_CUDA(cudaEventSynchronize(f->ready));
    const size_t n = (size_t)f->n;
    if (n > 0) {
        if (keys) BORB_CUDA(cudaMemcpy(keys, f->keys, n * sizeof(borb_keypoint), cudaMemcpyDeviceToHost));
        if (desc) BORB_CUDA(cudaMemcpy(desc, f->desc, n * 32, cudaMemcpyDeviceToHost));
        if (u_right) BORB_CUDA(cudaMemcpy(u_right, f->u_right, n * 4, cudaMemcpyDeviceToHost));
        if (depth) BORB_CUDA(cudaMemcpy(depth, f->depth, n * 4, cudaMemcpyDeviceToHost));
    }
    std::vector<int32_t> cs(GRID_CELLS + 1);
    BORB_CUDA(cudaMemcpy(cs.data(), f->cell_start, cs.size() * 4, cudaMemcpyDeviceToHost));
    if (cell_start) std::memcpy(cell_start, cs.data(), cs.size() * 4);
    const int in_grid = cs[GRID_CELLS];
    if (in_grid < 0 || (size_t)in_grid > n) { set_error("grid of %d entries for %d features", in_grid, f->n); return BORB_ERR_STATE; }
    if (cell_idx && in_grid > 0) BORB_CUDA(cudaMemcpy(cell_idx, f->cell_idx, (size_t)in_grid * 4, cudaMemcpyDeviceToHost));
    return BORB_OK;
}

// ---- SearchByProjection(F, vpMapPoints, th): one (frame, map point list) pair of borb_search_by_projection or of
// borb_search_by_projection_batch
namespace {
// a pair without map points or without frame features needs no more than the first checks
borb_status check_mappoints(const borb_frame_view* F, const FrameInfo& I, const borb_mappoint_view* P, const borb_matcher* m) {
    borb_status s = check_frame(F, I, m);
    if (s != BORB_OK) return s;
    if (P->n < 0 || P->n > MATCH_MAX_FEATURES) { set_error("%d map points (limit %d per call)", P->n, MATCH_MAX_FEATURES); return BORB_ERR_INVALID_ARG; }
    if (P->n == 0 || I.n == 0) return BORB_OK;
    if (!P->proj_x || !P->proj_y || !P->proj_xr || !P->level || !P->view_cos || !P->desc) { set_error("incomplete map point view"); return BORB_ERR_INVALID_ARG; }
    for (int i = 0; i < P->n; i++)
        if ((!P->valid || P->valid[i]) && (P->level[i] < 0 || P->level[i] >= I.n_levels)) { set_error("map point %d: predicted level out of range", i); return BORB_ERR_INVALID_ARG; }
    return BORB_OK;
}

struct MapPointsOff { FrameStage fs; size_t px, py, pxr, lvl, vc, md, val, obs, cand, cc; };

MapPointsOff stage_mappoints(Call& c, const borb_frame_view* F, const FrameInfo& I, const borb_mappoint_view* P, HostGrids& g) {
    MapPointsOff o{};
    const size_t n = (size_t)P->n;
    o.fs = stage_frame(c, F, I, true, g);
    o.px = c.in(P->proj_x, n * 4); o.py = c.in(P->proj_y, n * 4); o.pxr = c.in(P->proj_xr, n * 4);
    o.lvl = c.in(P->level, n * 4); o.vc = c.in(P->view_cos, n * 4); o.md = c.in(P->desc, n * 32);
    o.val = P->valid ? c.in(P->valid, n) : 0;
    o.obs = P->has_obs ? c.in(P->has_obs, n) : 0;
    return o;
}
// device-only scratch, laid out after every input
void reserve_mappoints(Call& c, const FrameInfo& I, const borb_mappoint_view* P, MapPointsOff& o) {
    reserve_grid(c, I, o.fs);
    o.cand = c.scratch((size_t)P->n * I.n * 4); o.cc = c.scratch((size_t)P->n * 4);
}
// the map point side of A (the frame side comes from bind_frame_fields); out: P->n matches followed by the count
void bind_mappoints(const MapPointsOff& o, const borb_mappoint_view* P, const Call& c, float th, float nnratio, int32_t* out, ProjArgs& A) {
    A.occupied = o.fs.occ_p ? c.dev(o.fs.occ) : nullptr;
    A.n_mp = P->n; A.proj_x = (const float*)c.dev(o.px); A.proj_y = (const float*)c.dev(o.py); A.proj_xr = (const float*)c.dev(o.pxr);
    A.view_cos = (const float*)c.dev(o.vc); A.level = (const int32_t*)c.dev(o.lvl); A.mp_desc = c.dev(o.md);
    A.mp_valid = P->valid ? c.dev(o.val) : nullptr; A.mp_has_obs = P->has_obs ? c.dev(o.obs) : nullptr;
    A.th = th; A.nnratio = nnratio; A.th_dist = TH_HIGH;
    A.cand = (uint32_t*)c.dev(o.cand); A.cand_cnt = (int*)c.dev(o.cc);
    A.mode = 0;
    A.out_match = out;
}

// Shared body of borb_search_by_projection (one job, a host view or a resident frame) and borb_search_by_projection_batch (resident
// frames).  The per-frame call is a few microseconds of kernel work behind ~20 us of launch + synchronisation, so independent camera
// streams are batched the same way the extractor batches their images: one launch pair and one synchronisation for every job.
borb_status projection_jobs(borb_matcher* m, const borb_frame_view* frames, const borb_mappoint_view* points, int n_jobs, float th,
                            float nnratio, int32_t* const* match_feat, int32_t* n_matches, bool batch) {
    struct Job { FrameInfo I; bool live; MapPointsOff o; size_t res; };
    std::vector<Job> J(n_jobs);
    int max_n = 1, max_n_mp = 0;
    for (int j = 0; j < n_jobs; j++) {
        const borb_mappoint_view* P = &points[j];
        if (batch && !frames[j].resident) { set_error("job %d: borb_search_by_projection_batch needs device-resident frames (borb_frame_view::resident)", j); return BORB_ERR_INVALID_ARG; }
        if (batch && !match_feat[j]) { set_error("job %d: null output", j); return BORB_ERR_INVALID_ARG; }
        const FrameInfo I = J[j].I = frame_info(&frames[j]);
        borb_status s = check_mappoints(&frames[j], I, P, m);
        if (s != BORB_OK) return job_fail(batch, j, s);
        J[j].live = P->n > 0 && I.n > 0;
    }
    for (int j = 0; j < n_jobs; j++) {                  // every job has passed its checks: a refused call writes nothing
        n_matches[j] = 0;
        if (!J[j].live) { std::fill_n(match_feat[j], points[j].n, -1); continue; }
        max_n = std::max(max_n, J[j].I.n); max_n_mp = std::max(max_n_mp, points[j].n);
    }
    if (max_n_mp == 0) return BORB_OK;
    Call c(m);
    HostGrids g;
    for (int j = 0; j < n_jobs; j++)
        if (J[j].live) J[j].o = stage_mappoints(c, &frames[j], J[j].I, &points[j], g);
    JobTable<ProjArgs> jt(c, n_jobs);
    g.stage(c);
    for (int j = 0; j < n_jobs; j++) {
        if (!J[j].live) continue;
        reserve_mappoints(c, J[j].I, &points[j], J[j].o);
        J[j].res = c.result((size_t)points[j].n * 4 + 4);
    }
    borb_status s;
    if ((s = c.begin(n_jobs == 1 && J[0].I.rf)) != BORB_OK) return s;
    const bool direct = c.in_place() || n_jobs > 1;      // results land in the pinned landing buffer (UVA): no D2H copy
    ProjArgs* hj = jt.host(c);
    for (int j = 0; j < n_jobs; j++) {
        ProjArgs A{};
        if (J[j].live) {
            bind_frame_fields(J[j].I, J[j].o.fs, c, g, A);
            bind_mappoints(J[j].o, &points[j], c, th, nnratio, (int32_t*)c.res(J[j].res, direct), A);
        }                                                // a dead job keeps n_mp = 0: both kernels skip it
        hj[j] = A;
    }
    if ((s = c.commit()) != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++)
        if (J[j].live && J[j].I.rf && (s = c.wait(J[j].I.rf)) != BORB_OK) return s;
    m->launches += g.launch(c, m->stream);
    m->launches += launch_projection_batch(jt.dev(c), hj[0], n_jobs, max_n, max_n_mp, m->stream);
    if ((s = c.finish()) != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++)
        if (J[j].live) read_counted(c.out(J[j].res), points[j].n, match_feat[j], &n_matches[j]);
    return BORB_OK;
}
}  // namespace

borb_status borb_search_by_projection(borb_matcher* m, const borb_frame_view* F, const borb_mappoint_view* P, float th, float nnratio,
                                      int32_t* match_feat, int32_t* n_matches) {
    if (!m || !F || !P || !match_feat || !n_matches) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    return projection_jobs(m, F, P, 1, th, nnratio, &match_feat, n_matches, false);
}

// Frames must be device-resident (borb_frames_from_extractor / borb_frame_create).
borb_status borb_search_by_projection_batch(borb_matcher* m, const borb_frame_view* frames, const borb_mappoint_view* points, int n_jobs,
                                            float th, float nnratio, int32_t* const* match_feat, int32_t* n_matches) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && (!frames || !points || !match_feat || !n_matches))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    return projection_jobs(m, frames, points, n_jobs, th, nnratio, match_feat, n_matches, true);
}

// Shared body of the three SearchByProjection overloads that project world points with a pose:
// variant 0 (CurrentFrame, LastFrame) :1328, 1 (CurrentFrame, KeyFrame) :1472, 2 (KeyFrame, Scw) :290.
struct PointQuery {
    int variant, n;
    const borb_keypoint* keys;      // variant 0
    const float* world_pos;
    const uint8_t* desc;
    const uint8_t* valid;
    const uint8_t* has_obs;         // variant 0
    const float* max_distance;      // variants 1, 2
    const float* min_distance;
    const float* normal;            // variant 2
    const float* angle;             // variant 1
    const float* Tcw;
    const float* Ow;
    float fx, fy, cx, cy, bf, th, log_scale;
    int forward, backward, check_ori, th_dist;
    // variant 2 family (order-independent overloads share the projection code)
    int invz_double, use_normal, chain;
    const float* T2;                // chain: [sR | t] applied after Tcw
    int chi2;                       // Fuse(pKF, ...) reprojection gates
    const float* inv_sigma2;        // chi2: mvInvLevelSigma2 (n_levels)
};

namespace {
// a query without points or a frame without features needs no more than the first checks
borb_status check_query(const borb_frame_view* F, const FrameInfo& I, const PointQuery& Q, const borb_matcher* m) {
    borb_status s = check_frame(F, I, m);
    if (s != BORB_OK) return s;
    if (Q.n < 0 || Q.n > MATCH_MAX_FEATURES) { set_error("%d query points (limit %d per call)", Q.n, MATCH_MAX_FEATURES); return BORB_ERR_INVALID_ARG; }
    if (I.n == 0 || Q.n == 0) return BORB_OK;
    if (!Q.world_pos || !Q.desc) { set_error("incomplete query view"); return BORB_ERR_INVALID_ARG; }
    if (Q.variant == 0) {
        if (!Q.keys) { set_error("incomplete last-frame view"); return BORB_ERR_INVALID_ARG; }
        for (int i = 0; i < Q.n; i++)
            if (Q.keys[i].octave < 0 || Q.keys[i].octave >= I.n_levels) { set_error("last-frame keypoint %d: octave out of range", i); return BORB_ERR_INVALID_ARG; }
    } else {
        if (!Q.max_distance || !Q.min_distance || (!Q.Ow && !Q.chain) || (Q.variant == 2 && Q.use_normal && !Q.normal) ||
            (Q.variant == 1 && Q.check_ori && !Q.angle) || (Q.chain && !Q.T2) || (Q.chi2 && !Q.inv_sigma2)) {
            set_error("incomplete world-points view"); return BORB_ERR_INVALID_ARG;
        }
        if (!(Q.log_scale > 0.f)) { set_error("log_scale_factor must be positive (Frame::mfLogScaleFactor)"); return BORB_ERR_INVALID_ARG; }
    }
    return BORB_OK;
}

struct QueryOff { FrameStage fs; size_t lk, wp, md, vin, obs, mx, mn, nr, qa, is2, px, py, pxr, rad, ang, minl, maxl, val, cand, cc, evi, evb; };

QueryOff stage_query(Call& c, const borb_frame_view* F, const FrameInfo& I, const PointQuery& Q, HostGrids& g) {
    QueryOff o{};
    const size_t nq = (size_t)Q.n;
    o.fs = stage_frame(c, F, I, Q.variant == 0 || Q.chi2, g);
    o.lk = Q.keys ? c.in(Q.keys, nq * sizeof(borb_keypoint)) : 0;
    o.wp = c.in(Q.world_pos, nq * 12);
    o.md = c.in(Q.desc, nq * 32);
    o.vin = Q.valid ? c.in(Q.valid, nq) : 0;
    o.obs = Q.has_obs ? c.in(Q.has_obs, nq) : 0;
    o.mx = Q.max_distance ? c.in(Q.max_distance, nq * 4) : 0;
    o.mn = Q.min_distance ? c.in(Q.min_distance, nq * 4) : 0;
    o.nr = Q.normal ? c.in(Q.normal, nq * 12) : 0;
    o.qa = Q.angle ? c.in(Q.angle, nq * 4) : 0;
    o.is2 = Q.chi2 ? c.in(Q.inv_sigma2, (size_t)I.n_levels * 4) : 0;
    return o;
}
// device-only scratch of project_points (and the grid of a host view), laid out after every input
void reserve_projection(Call& c, const FrameInfo& I, const PointQuery& Q, QueryOff& o) {
    const size_t nq = (size_t)Q.n;
    reserve_grid(c, I, o.fs);
    o.px = c.scratch(nq * 4); o.py = c.scratch(nq * 4); o.pxr = c.scratch(nq * 4); o.rad = c.scratch(nq * 4);
    o.ang = c.scratch(nq * 4); o.minl = c.scratch(nq * 4); o.maxl = c.scratch(nq * 4); o.val = c.scratch(nq);
}
// the same plus the candidate lists and the match events of the resolve kernel
void reserve_query(Call& c, const FrameInfo& I, const PointQuery& Q, QueryOff& o) {
    const size_t nq = (size_t)Q.n;
    reserve_projection(c, I, Q, o);
    o.cand = c.scratch(nq * I.n * 4); o.cc = c.scratch(nq * 4);
    o.evi = c.scratch(nq * 4); o.evb = c.scratch(nq);
}
// L and the query side of A (the frame side comes from bind_frame_fields); out: where the search kernel writes (the resolve kernel:
// I.n entries of state followed by the match count; fuse_batch_kernel: one entry per query)
void bind_query(const QueryOff& o, const PointQuery& Q, const FrameInfo& I, const Call& c, int32_t* out, LastArgs& L, ProjArgs& A) {
    L.variant = Q.variant;
    L.n_last = Q.n; L.last_keys = Q.keys ? (const borb_keypoint*)c.dev(o.lk) : nullptr; L.world_pos = (const float*)c.dev(o.wp);
    L.q_angle_in = Q.angle ? (const float*)c.dev(o.qa) : nullptr;
    L.max_distance = Q.max_distance ? (const float*)c.dev(o.mx) : nullptr;
    L.min_distance = Q.min_distance ? (const float*)c.dev(o.mn) : nullptr;
    L.normal = Q.normal ? (const float*)c.dev(o.nr) : nullptr;
    for (int i = 0; i < 3; i++) L.Ow[i] = Q.Ow ? Q.Ow[i] : 0.f;
    L.log_scale = Q.log_scale; L.n_levels = I.n_levels;
    L.invz_double = Q.invz_double; L.use_normal = Q.use_normal; L.chain = Q.chain;
    for (int i = 0; i < 12; i++) L.T2[i] = Q.chain ? Q.T2[i] : 0.f;
    L.valid_in = Q.valid ? c.dev(o.vin) : nullptr;
    for (int i = 0; i < 12; i++) L.T[i] = Q.Tcw[i];
    L.fx = Q.fx; L.fy = Q.fy; L.cx = Q.cx; L.cy = Q.cy; L.bf = Q.bf; L.th = Q.th;
    L.minX = I.min_x; L.minY = I.min_y; L.maxX = I.max_x; L.maxY = I.max_y;
    L.scale_factors = A.scale_factors;
    L.forward = Q.forward; L.backward = Q.backward;
    L.proj_x = (float*)c.dev(o.px); L.proj_y = (float*)c.dev(o.py); L.proj_xr = (float*)c.dev(o.pxr); L.radius = (float*)c.dev(o.rad);
    L.angle = (float*)c.dev(o.ang); L.minl = (int32_t*)c.dev(o.minl); L.maxl = (int32_t*)c.dev(o.maxl); L.valid_out = c.dev(o.val);
    A.occupied = o.fs.occ_p ? c.dev(o.fs.occ) : nullptr;
    wire_projection(L, A);
    A.mp_desc = c.dev(o.md); A.mp_has_obs = Q.has_obs ? c.dev(o.obs) : nullptr;
    A.th = Q.th; A.nnratio = 0.f;
    A.cand = (uint32_t*)c.dev(o.cand); A.cand_cnt = (int*)c.dev(o.cc);
    A.mode = 1; A.check_ori = Q.check_ori; A.th_dist = Q.th_dist;
    A.out_match = out; A.ev_idx = (int32_t*)c.dev(o.evi); A.ev_bin = c.dev(o.evb);
}
// SearchByProjection(CurrentFrame, LastFrame) of one camera stream
PointQuery last_frame_query(const borb_last_frame_job& B, int check_orientation) {
    PointQuery Q{};
    Q.variant = 0; Q.n = B.last.n; Q.keys = B.last.keys_un; Q.world_pos = B.last.world_pos; Q.desc = B.last.desc; Q.valid = B.last.valid;
    Q.has_obs = B.last.has_obs;
    Q.Tcw = B.Tcw; Q.fx = B.fx; Q.fy = B.fy; Q.cx = B.cx; Q.cy = B.cy; Q.bf = B.bf; Q.th = B.th; Q.forward = B.forward; Q.backward = B.backward;
    Q.check_ori = check_orientation; Q.th_dist = TH_HIGH;                  // (:1426)
    return Q;
}
// SearchByProjection(CurrentFrame, pKF, sAlreadyFound, th, ORBdist) of one relocalising camera stream
PointQuery kf_query(const borb_kf_projection_job& B, int check_orientation) {
    PointQuery Q{};
    Q.variant = 1; Q.n = B.pts.n; Q.world_pos = B.pts.world_pos; Q.desc = B.pts.desc; Q.valid = B.pts.valid;
    Q.max_distance = B.pts.max_distance; Q.min_distance = B.pts.min_distance; Q.angle = B.pts.angle;
    Q.Tcw = B.Tcw; Q.Ow = B.Ow; Q.fx = B.fx; Q.fy = B.fy; Q.cx = B.cx; Q.cy = B.cy; Q.th = B.th; Q.log_scale = B.log_scale_factor;
    Q.check_ori = check_orientation; Q.th_dist = B.orb_dist;
    return Q;
}
// SearchByProjection(pKF, Scw, vpPoints, vpMatched, th) of one loop-closing camera stream
PointQuery sim3_projection_query(const borb_sim3_projection_job& B) {
    PointQuery Q{};
    Q.variant = 2; Q.n = B.pts.n; Q.world_pos = B.pts.world_pos; Q.desc = B.pts.desc; Q.valid = B.pts.valid;
    Q.max_distance = B.pts.max_distance; Q.min_distance = B.pts.min_distance; Q.normal = B.pts.normal;
    Q.Tcw = B.Tcw; Q.Ow = B.Ow; Q.fx = B.fx; Q.fy = B.fy; Q.cx = B.cx; Q.cy = B.cy; Q.th = (float)B.th; Q.log_scale = B.log_scale_factor;
    Q.check_ori = 0; Q.th_dist = TH_LOW;                                   // (:394)
    Q.use_normal = 1;
    return Q;
}

// one (frame, query) pair of point_query_jobs; state: the job's output, the frame's n entries
struct PointJob { const borb_frame_view* F; PointQuery Q; int32_t* state; };

// Shared body of borb_search_by_projection_last / _kf / _sim3 and of their _batch forms (resident frames): project_points,
// candidates and resolve<true>, one synchronisation.  batch: the name of the batched entry point (its errors name the job), null for
// a single call.  The state stays in the arena, not in mapped host memory: resolve<true> writes it with atomicMax.
borb_status point_query_jobs(borb_matcher* m, const PointJob* jobs, int n_jobs, int32_t* n_matches, const char* batch) {
    struct Job { FrameInfo I; bool live; QueryOff o; size_t res; };
    std::vector<Job> J(n_jobs);
    int max_n = 1, max_nq = 0;
    for (int j = 0; j < n_jobs; j++) {
        const PointQuery& Q = jobs[j].Q;
        if (batch && !jobs[j].F->resident) { set_error("job %d: %s needs device-resident frames (borb_frame_view::resident)", j, batch); return BORB_ERR_INVALID_ARG; }
        if (batch && !jobs[j].state) { set_error("job %d: null output", j); return BORB_ERR_INVALID_ARG; }
        const FrameInfo I = J[j].I = frame_info(jobs[j].F);
        borb_status s = check_query(jobs[j].F, I, Q, m);
        if (s != BORB_OK) return job_fail(batch != nullptr, j, s);
        J[j].live = I.n > 0 && Q.n > 0;
        if (J[j].live) { max_n = std::max(max_n, I.n); max_nq = std::max(max_nq, Q.n); }
    }
    for (int j = 0; j < n_jobs; j++) { n_matches[j] = 0; std::fill_n(jobs[j].state, J[j].I.n, -1); }   // every job passed its checks
    if (max_nq == 0) return BORB_OK;
    Call c(m);
    HostGrids g;
    for (int j = 0; j < n_jobs; j++)
        if (J[j].live) J[j].o = stage_query(c, jobs[j].F, J[j].I, jobs[j].Q, g);
    JobTable<LastArgs> lt(c, n_jobs);
    JobTable<ProjArgs> jt(c, n_jobs);
    g.stage(c);
    for (int j = 0; j < n_jobs; j++) {
        if (!J[j].live) continue;
        reserve_query(c, J[j].I, jobs[j].Q, J[j].o);
        J[j].res = c.result((size_t)J[j].I.n * 4 + 4);
    }
    borb_status s;
    if ((s = c.begin(n_jobs == 1 && J[0].I.rf)) != BORB_OK) return s;
    LastArgs* hl = lt.host(c);
    ProjArgs* hj = jt.host(c);
    for (int j = 0; j < n_jobs; j++) {
        LastArgs L{};
        ProjArgs A{};
        if (J[j].live) {
            bind_frame_fields(J[j].I, J[j].o.fs, c, g, A);
            bind_query(J[j].o, jobs[j].Q, J[j].I, c, (int32_t*)c.res(J[j].res, false), L, A);
        }                                            // a job without work keeps n_last = n_mp = 0: every kernel skips it
        hl[j] = L;
        hj[j] = A;
    }
    if ((s = c.commit()) != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++)
        if (J[j].live && J[j].I.rf && (s = c.wait(J[j].I.rf)) != BORB_OK) return s;
    m->launches += g.launch(c, m->stream);
    m->launches += launch_point_projection_batch(lt.dev(c), jt.dev(c), hl[0], hj[0], n_jobs, max_nq, max_n, max_nq, true, m->stream);
    if ((s = c.finish()) != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++)
        if (J[j].live) read_counted(c.out(J[j].res), J[j].I.n, jobs[j].state, &n_matches[j]);
    return BORB_OK;
}
}  // namespace

borb_status borb_search_by_projection_last(borb_matcher* m, const borb_frame_view* F, const borb_lastframe_view* Lf, const float* Tcw,
                                           float fx, float fy, float cx, float cy, float bf, float th, int forward, int backward,
                                           int check_orientation, int32_t* state_cur, int32_t* n_matches) {
    if (!m || !F || !Lf || !Tcw || !state_cur || !n_matches) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_last_frame_job B{};
    B.last = *Lf;
    std::memcpy(B.Tcw, Tcw, sizeof(B.Tcw));
    B.fx = fx; B.fy = fy; B.cx = cx; B.cy = cy; B.bf = bf; B.th = th; B.forward = forward; B.backward = backward;
    const PointJob P{F, last_frame_query(B, check_orientation), state_cur};
    return point_query_jobs(m, &P, 1, n_matches, nullptr);
}

borb_status borb_search_by_projection_kf(borb_matcher* m, const borb_frame_view* cur, const borb_worldpoints_view* pts, const float* Tcw,
                                         const float* Ow, float fx, float fy, float cx, float cy, float log_scale_factor, float th,
                                         int orb_dist, int check_orientation, int32_t* state_cur, int32_t* n_matches) {
    if (!m || !cur || !pts || !Tcw || !Ow || !state_cur || !n_matches) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_kf_projection_job B{};
    B.pts = *pts;
    std::memcpy(B.Tcw, Tcw, sizeof(B.Tcw)); std::memcpy(B.Ow, Ow, sizeof(B.Ow));
    B.fx = fx; B.fy = fy; B.cx = cx; B.cy = cy; B.log_scale_factor = log_scale_factor; B.th = th; B.orb_dist = orb_dist;
    const PointJob P{cur, kf_query(B, check_orientation), state_cur};
    return point_query_jobs(m, &P, 1, n_matches, nullptr);
}

borb_status borb_search_by_projection_sim3(borb_matcher* m, const borb_frame_view* kf, const borb_worldpoints_view* pts, const float* Tcw,
                                           const float* Ow, float fx, float fy, float cx, float cy, float log_scale_factor, int th,
                                           int32_t* state_kf, int32_t* n_matches) {
    if (!m || !kf || !pts || !Tcw || !Ow || !state_kf || !n_matches) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_sim3_projection_job B{};
    B.pts = *pts;
    std::memcpy(B.Tcw, Tcw, sizeof(B.Tcw)); std::memcpy(B.Ow, Ow, sizeof(B.Ow));
    B.fx = fx; B.fy = fy; B.cx = cx; B.cy = cy; B.log_scale_factor = log_scale_factor; B.th = th;
    const PointJob P{kf, sim3_projection_query(B), state_kf};
    return point_query_jobs(m, &P, 1, n_matches, nullptr);
}

borb_status borb_search_by_projection_last_batch(borb_matcher* m, const borb_last_frame_job* jobs, int n_jobs, int check_orientation,
                                                 int32_t* n_matches) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && (!jobs || !n_matches))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    std::vector<PointJob> P(n_jobs);
    for (int j = 0; j < n_jobs; j++) P[j] = PointJob{&jobs[j].cur, last_frame_query(jobs[j], check_orientation), jobs[j].state_cur};
    return point_query_jobs(m, P.data(), n_jobs, n_matches, "borb_search_by_projection_last_batch");
}

borb_status borb_search_by_projection_kf_batch(borb_matcher* m, const borb_kf_projection_job* jobs, int n_jobs, int check_orientation,
                                               int32_t* n_matches) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && (!jobs || !n_matches))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    std::vector<PointJob> P(n_jobs);
    for (int j = 0; j < n_jobs; j++) P[j] = PointJob{&jobs[j].cur, kf_query(jobs[j], check_orientation), jobs[j].state_cur};
    return point_query_jobs(m, P.data(), n_jobs, n_matches, "borb_search_by_projection_kf_batch");
}

borb_status borb_search_by_projection_sim3_batch(borb_matcher* m, const borb_sim3_projection_job* jobs, int n_jobs, int32_t* n_matches) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && (!jobs || !n_matches))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    std::vector<PointJob> P(n_jobs);
    for (int j = 0; j < n_jobs; j++) P[j] = PointJob{&jobs[j].kf, sim3_projection_query(jobs[j]), jobs[j].state_kf};
    return point_query_jobs(m, P.data(), n_jobs, n_matches, "borb_search_by_projection_sim3_batch");
}

// ---- the search part of Fuse: borb_fuse is the one-job case of borb_fuse_batch (project_points + fuse_batch_kernel, one
// synchronisation).  The scratch of a job is its projections: fuse_batch_kernel takes the first minimum without candidate lists.
namespace {
borb_status fuse_jobs(borb_matcher* m, const borb_fuse_job* jobs, int n_jobs, bool batch, int32_t* n_found) {
    struct Job { borb_frame_view kf; PointQuery Q; FrameInfo I; bool live; QueryOff o; size_t res; };
    std::vector<Job> J(n_jobs);
    int max_nq = 0;
    for (int j = 0; j < n_jobs; j++) {
        const borb_fuse_job& B = jobs[j];
        if (!B.scw_variant && !B.inv_level_sigma2) { set_error("Fuse(pKF, vpMapPoints, th) needs mvInvLevelSigma2"); return job_fail(batch, j, BORB_ERR_INVALID_ARG); }
        PointQuery& Q = J[j].Q;
        Q.variant = 2; Q.n = B.pts.n; Q.world_pos = B.pts.world_pos; Q.desc = B.pts.desc; Q.valid = B.pts.valid;
        Q.max_distance = B.pts.max_distance; Q.min_distance = B.pts.min_distance; Q.normal = B.pts.normal;
        Q.Tcw = B.Tcw; Q.Ow = B.Ow; Q.fx = B.fx; Q.fy = B.fy; Q.cx = B.cx; Q.cy = B.cy; Q.bf = B.bf; Q.th = B.th; Q.log_scale = B.log_scale_factor;
        Q.th_dist = TH_LOW;                                                // (:944, :1075)
        Q.use_normal = 1;
        Q.invz_double = B.scw_variant ? 1 : 0;                             // 1.0/z (:1014) vs 1/z (:861)
        Q.chi2 = B.scw_variant ? 0 : 1; Q.inv_sigma2 = B.inv_level_sigma2;
        // occupancy plays no role in either Fuse (the MapPoint already in the slot is handled by the caller, :947-960)
        J[j].kf = B.kf;
        J[j].kf.occupied = nullptr;
        const FrameInfo I = J[j].I = frame_info(&J[j].kf);
        const borb_status s = check_query(&J[j].kf, I, Q, m);
        if (s != BORB_OK) return job_fail(batch, j, s);
        J[j].live = I.n > 0 && Q.n > 0;
        if (J[j].live) max_nq = std::max(max_nq, Q.n);
    }
    for (int j = 0; j < n_jobs; j++) { n_found[j] = 0; std::fill_n(jobs[j].best_idx, J[j].Q.n, -1); }   // every job passed its checks
    if (max_nq == 0) return BORB_OK;
    Call c(m);
    HostGrids g;
    for (int j = 0; j < n_jobs; j++)
        if (J[j].live) J[j].o = stage_query(c, &J[j].kf, J[j].I, J[j].Q, g);
    const size_t o_last = c.in(nullptr, (size_t)n_jobs * sizeof(LastArgs)), o_jobs = c.in(nullptr, (size_t)n_jobs * sizeof(FuseJob));
    g.stage(c);
    const size_t r_cnt = c.result((size_t)n_jobs * 4);     // n_found of every job, then every job's best_idx
    for (int j = 0; j < n_jobs; j++) {
        if (!J[j].live) continue;
        reserve_projection(c, J[j].I, J[j].Q, J[j].o);
        J[j].res = c.result((size_t)J[j].Q.n * 4);
    }
    borb_status s;
    if ((s = c.begin()) != BORB_OK) return s;
    LastArgs* hl = c.host<LastArgs>(o_last);
    FuseJob* hj = c.host<FuseJob>(o_jobs);
    for (int j = 0; j < n_jobs; j++) {
        LastArgs L{};
        FuseJob F{};
        if (J[j].live) {
            bind_frame_fields(J[j].I, J[j].o.fs, c, g, F.A);
            bind_query(J[j].o, J[j].Q, J[j].I, c, (int32_t*)c.res(J[j].res, false), L, F.A);
            F.inv_sigma2 = J[j].Q.chi2 ? (const float*)c.dev(J[j].o.is2) : nullptr;
            F.n_found = (int*)c.res(r_cnt, false) + j;
        }                                            // a job without work keeps n_last = n_mp = 0: both kernels skip it
        hl[j] = L;
        hj[j] = F;
    }
    if ((s = c.commit()) != BORB_OK) return s;
    BORB_CUDA(cudaMemsetAsync(c.res(r_cnt, false), 0, (size_t)n_jobs * 4, m->stream));
    for (int j = 0; j < n_jobs; j++)
        if (J[j].live && J[j].I.rf && (s = c.wait(J[j].I.rf)) != BORB_OK) return s;
    m->launches += g.launch(c, m->stream);
    m->launches += launch_fuse_batch((const LastArgs*)c.dev(o_last), (const FuseJob*)c.dev(o_jobs), n_jobs, max_nq, m->stream);
    if ((s = c.finish()) != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++) {
        std::memcpy(&n_found[j], c.out(r_cnt) + (size_t)j * 4, 4);
        if (J[j].live) std::memcpy(jobs[j].best_idx, c.out(J[j].res), (size_t)J[j].Q.n * 4);
    }
    return BORB_OK;
}
}  // namespace

borb_status borb_fuse(borb_matcher* m, const borb_frame_view* kf, const float* inv_level_sigma2, const borb_worldpoints_view* pts,
                      const float* Tcw, const float* Ow, float fx, float fy, float cx, float cy, float bf, float log_scale_factor,
                      float th, int scw_variant, int32_t* best_idx, int32_t* n_found) {
    if (!m || !kf || !pts || !Tcw || !Ow || !best_idx || !n_found) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_fuse_job B{};
    B.kf = *kf; B.inv_level_sigma2 = inv_level_sigma2; B.pts = *pts;
    std::memcpy(B.Tcw, Tcw, sizeof(B.Tcw)); std::memcpy(B.Ow, Ow, sizeof(B.Ow));
    B.fx = fx; B.fy = fy; B.cx = cx; B.cy = cy; B.bf = bf; B.log_scale_factor = log_scale_factor; B.th = th;
    B.scw_variant = scw_variant; B.best_idx = best_idx;
    return fuse_jobs(m, &B, 1, false, n_found);
}

borb_status borb_fuse_batch(borb_matcher* m, const borb_fuse_job* jobs, int n_jobs, int32_t* n_found) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && (!jobs || !n_found))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    for (int j = 0; j < n_jobs; j++) {
        if (!jobs[j].kf.resident) { set_error("job %d: borb_fuse_batch needs device-resident keyframes (borb_frame_view::resident)", j); return BORB_ERR_INVALID_ARG; }
        if (!jobs[j].best_idx) { set_error("job %d: null output", j); return BORB_ERR_INVALID_ARG; }
    }
    return fuse_jobs(m, jobs, n_jobs, true, n_found);
}

// ---- SearchBySim3: borb_search_by_sim3 is the one-job case of borb_search_by_sim3_batch.  A job is two direction jobs of
// fuse_batch_kernel, both in one launch pair, whose matches stay in the arena; sim3_agree_batch_kernel then keeps the pairs the two
// directions agree on.  3 launches and one synchronisation whatever n_jobs is; the scratch of a direction is its projections and its
// matches, with no candidate list.
namespace {
// the points P of one keyframe, seen from camera 1 or 2 (Tw: that camera's pose) and chained into the other camera by S
PointQuery sim3_direction(const borb_sim3_job& B, const borb_worldpoints_view& P, const float* Tw, const float* S, float log_scale) {
    PointQuery Q{};
    Q.variant = 2; Q.n = P.n; Q.world_pos = P.world_pos; Q.desc = P.desc; Q.valid = P.valid;
    Q.max_distance = P.max_distance; Q.min_distance = P.min_distance;
    Q.Tcw = Tw; Q.chain = 1; Q.T2 = S; Q.fx = B.fx; Q.fy = B.fy; Q.cx = B.cx; Q.cy = B.cy; Q.th = B.th; Q.log_scale = log_scale;
    Q.th_dist = TH_HIGH; Q.invz_double = 1;                                // (:1221, :1301); invz = 1.0/z (:1166, :1246)
    return Q;
}

borb_status sim3_jobs(borb_matcher* m, const borb_sim3_job* jobs, int n_jobs, bool batch, int32_t* n_found) {
    // direction 2j: KF1's points into KF2 (:1146-1222); 2j + 1: KF2's points into KF1 (:1224-1300)
    struct Dir { borb_frame_view kf; PointQuery Q; FrameInfo I; QueryOff o; size_t out = 0; };
    std::vector<Dir> D(2 * (size_t)n_jobs);
    std::vector<size_t> res(n_jobs);
    std::vector<char> live(n_jobs);
    int max_nq = 0, max_n1 = 0;
    for (int j = 0; j < n_jobs; j++) {
        const borb_sim3_job& B = jobs[j];
        Dir& d12 = D[2 * (size_t)j];
        Dir& d21 = D[2 * (size_t)j + 1];
        d12.kf = B.kf2; d12.Q = sim3_direction(B, B.pts1, B.T1w, B.S21, B.log_scale_factor2);
        d21.kf = B.kf1; d21.Q = sim3_direction(B, B.pts2, B.T2w, B.S12, B.log_scale_factor1);
        d12.kf.occupied = d21.kf.occupied = nullptr;               // vpMatches12 enters through pts*.valid (:1130-1155)
        d12.I = frame_info(&d12.kf);
        d21.I = frame_info(&d21.kf);
        const int n1 = d21.I.n, n2 = d12.I.n;
        if (B.pts1.n != n1 || B.pts2.n != n2) {
            set_error("SearchBySim3: one MapPoint slot per keyframe feature (GetMapPointMatches)");
            return job_fail(batch, j, BORB_ERR_INVALID_ARG);
        }
        borb_status s = check_query(&d12.kf, d12.I, d12.Q, m);
        if (s == BORB_OK) s = check_query(&d21.kf, d21.I, d21.Q, m);
        if (s != BORB_OK) return job_fail(batch, j, s);
        live[j] = n1 > 0 && n2 > 0;
        if (live[j]) { max_nq = std::max(max_nq, std::max(n1, n2)); max_n1 = std::max(max_n1, n1); }
    }
    for (int j = 0; j < n_jobs; j++) { n_found[j] = 0; std::fill_n(jobs[j].match12, D[2 * (size_t)j + 1].I.n, -1); }   // every job passed its checks
    if (max_nq == 0) return BORB_OK;
    const size_t nd = D.size();
    Call c(m);
    HostGrids g;
    for (size_t k = 0; k < nd; k++)
        if (live[k / 2]) D[k].o = stage_query(c, &D[k].kf, D[k].I, D[k].Q, g);
    const size_t o_last = c.in(nullptr, nd * sizeof(LastArgs)), o_dirs = c.in(nullptr, nd * sizeof(FuseJob));
    const size_t o_jobs = c.in(nullptr, (size_t)n_jobs * sizeof(Sim3AgreeJob));
    g.stage(c);
    const size_t o_sink = c.scratch(nd * 4);                   // fuse_batch_kernel's per-direction counts: the agreement test counts instead
    const size_t r_cnt = c.result((size_t)n_jobs * 4);         // n_found of every job, then every job's match12
    for (size_t k = 0; k < nd; k++) {
        if (!live[k / 2]) continue;
        reserve_projection(c, D[k].I, D[k].Q, D[k].o);
        D[k].out = c.scratch((size_t)D[k].Q.n * 4);
    }
    for (int j = 0; j < n_jobs; j++)
        if (live[j]) res[j] = c.result((size_t)jobs[j].pts1.n * 4);
    borb_status s;
    if ((s = c.begin()) != BORB_OK) return s;
    LastArgs* hl = c.host<LastArgs>(o_last);
    FuseJob* hd = c.host<FuseJob>(o_dirs);
    Sim3AgreeJob* hj = c.host<Sim3AgreeJob>(o_jobs);
    for (size_t k = 0; k < nd; k++) {
        LastArgs L{};
        FuseJob F{};
        if (live[k / 2]) {
            bind_frame_fields(D[k].I, D[k].o.fs, c, g, F.A);       // no u_right: stage_frame is asked for none without chi2
            bind_query(D[k].o, D[k].Q, D[k].I, c, (int32_t*)c.dev(D[k].out), L, F.A);
            F.n_found = (int*)c.dev(o_sink) + k;
        }                                            // a job without work keeps n_last = n_mp = n1 = 0: every kernel skips it
        hl[k] = L;
        hd[k] = F;
    }
    for (int j = 0; j < n_jobs; j++) {
        Sim3AgreeJob A{};
        if (live[j]) {
            A.match1 = (const int32_t*)c.dev(D[2 * (size_t)j].out); A.match2 = (const int32_t*)c.dev(D[2 * (size_t)j + 1].out);
            A.n1 = jobs[j].pts1.n; A.n2 = jobs[j].pts2.n;
            A.match12 = (int32_t*)c.res(res[j], false);
            A.n_found = (int*)c.res(r_cnt, false) + j;
        }
        hj[j] = A;
    }
    if ((s = c.commit()) != BORB_OK) return s;
    BORB_CUDA(cudaMemsetAsync(c.res(r_cnt, false), 0, (size_t)n_jobs * 4, m->stream));
    for (size_t k = 0; k < nd; k++)
        if (live[k / 2] && D[k].I.rf && (s = c.wait(D[k].I.rf)) != BORB_OK) return s;
    m->launches += g.launch(c, m->stream);                   // both keyframes of host views: one launch
    m->launches += launch_sim3_batch((const LastArgs*)c.dev(o_last), (const FuseJob*)c.dev(o_dirs), (const Sim3AgreeJob*)c.dev(o_jobs), n_jobs,
                                     max_nq, max_n1, m->stream);
    if ((s = c.finish()) != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++) {
        std::memcpy(&n_found[j], c.out(r_cnt) + (size_t)j * 4, 4);
        if (live[j]) std::memcpy(jobs[j].match12, c.out(res[j]), (size_t)jobs[j].pts1.n * 4);
    }
    return BORB_OK;
}
}  // namespace

borb_status borb_search_by_sim3(borb_matcher* m, const borb_frame_view* kf1, const borb_frame_view* kf2, const borb_worldpoints_view* pts1,
                                const borb_worldpoints_view* pts2, const float* T1w, const float* T2w, const float* S12, const float* S21,
                                float fx, float fy, float cx, float cy, float log_scale_factor1, float log_scale_factor2, float th,
                                int32_t* match12, int32_t* n_found) {
    if (!m || !kf1 || !kf2 || !pts1 || !pts2 || !T1w || !T2w || !S12 || !S21 || !match12 || !n_found) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_sim3_job B{};
    B.kf1 = *kf1; B.kf2 = *kf2; B.pts1 = *pts1; B.pts2 = *pts2;
    std::memcpy(B.T1w, T1w, sizeof(B.T1w)); std::memcpy(B.T2w, T2w, sizeof(B.T2w));
    std::memcpy(B.S12, S12, sizeof(B.S12)); std::memcpy(B.S21, S21, sizeof(B.S21));
    B.fx = fx; B.fy = fy; B.cx = cx; B.cy = cy; B.log_scale_factor1 = log_scale_factor1; B.log_scale_factor2 = log_scale_factor2; B.th = th;
    B.match12 = match12;
    return sim3_jobs(m, &B, 1, false, n_found);
}

borb_status borb_search_by_sim3_batch(borb_matcher* m, const borb_sim3_job* jobs, int n_jobs, int32_t* n_found) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && (!jobs || !n_found))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    for (int j = 0; j < n_jobs; j++) {
        if (!jobs[j].kf1.resident || !jobs[j].kf2.resident) {
            set_error("job %d: borb_search_by_sim3_batch needs device-resident keyframes (borb_frame_view::resident)", j);
            return BORB_ERR_INVALID_ARG;
        }
        if (!jobs[j].match12) { set_error("job %d: null output", j); return BORB_ERR_INVALID_ARG; }
    }
    return sim3_jobs(m, jobs, n_jobs, true, n_found);
}

// ---- Tracking::SearchLocalPoints: one camera stream of borb_search_local_points or of borb_search_local_points_batch
namespace {
// a job without points needs no more than the first checks
borb_status check_local(const borb_local_points_job& B, const FrameInfo& I, const borb_matcher* m) {
    borb_status s = check_frame(&B.frame, I, m);
    if (s != BORB_OK) return s;
    const borb_worldpoints_view& P = B.pts;
    if (P.n < 0) { set_error("negative point count"); return BORB_ERR_INVALID_ARG; }
    if (P.n == 0) return BORB_OK;
    if (!P.world_pos || !P.desc || !P.max_distance || !P.min_distance || !P.normal) { set_error("incomplete world-points view"); return BORB_ERR_INVALID_ARG; }
    if (!(B.log_scale_factor > 0.f)) { set_error("log_scale_factor must be positive (Frame::mfLogScaleFactor)"); return BORB_ERR_INVALID_ARG; }
    return BORB_OK;
}

// sel0 / nq: the job's valid points are sel[sel0 .. sel0 + nq); gather: not every point is valid
struct LocalOff { FrameStage fs; size_t sel0; int nq; bool gather; size_t wp, md, obs, mx, mn, nr, rad, ang, minl, maxl, cand, cc; };

// Resets the job's outputs (not in view, no match) and appends its valid points to sel.  Only the points that reach isInFrustum
// travel (src/Tracking.cc:1171-1175 skips the already-matched and the bad ones): a KITTI-scale local map lists ten thousand points
// of which a fraction is valid, and the reference has no limit on the list.
// the outputs of a point the search does not reach; written once every job of the call has passed its checks
void clear_local(const borb_local_points_job& B) {
    for (int i = 0; i < B.pts.n; i++) {
        B.in_view[i] = 0; B.match_feat[i] = -1;
        if (B.proj_x) B.proj_x[i] = 0.f;
        if (B.proj_y) B.proj_y[i] = 0.f;
        if (B.proj_xr) B.proj_xr[i] = 0.f;
        if (B.level) B.level[i] = 0;
        if (B.view_cos) B.view_cos[i] = 0.f;
    }
}
borb_status select_local(const borb_local_points_job& B, std::vector<int32_t>& sel, LocalOff& o) {
    const borb_worldpoints_view& P = B.pts;
    o.sel0 = sel.size();
    for (int i = 0; i < P.n; i++)
        if (!P.valid || P.valid[i]) sel.push_back(i);
    o.nq = (int)(sel.size() - o.sel0);
    o.gather = o.nq != P.n;
    if (o.nq > MATCH_MAX_FEATURES) { set_error("%d valid local map points (limit %d per call)", o.nq, MATCH_MAX_FEATURES); return BORB_ERR_INVALID_ARG; }
    return BORB_OK;
}
// gathered inputs are written straight into the pinned staging buffer once the layout is known (src = nullptr): gather_local
void stage_local(Call& c, const borb_local_points_job& B, const FrameInfo& I, LocalOff& o, HostGrids& grids) {
    const borb_worldpoints_view& P = B.pts;
    const size_t nq = (size_t)o.nq;
    const bool g = o.gather;
    o.fs = stage_frame(c, &B.frame, I, true, grids);
    o.wp = c.in(g ? nullptr : P.world_pos, nq * 12); o.md = c.in(g ? nullptr : P.desc, nq * 32);
    o.obs = B.has_obs ? c.in(g ? nullptr : B.has_obs, nq) : 0;
    o.mx = c.in(g ? nullptr : P.max_distance, nq * 4); o.mn = c.in(g ? nullptr : P.min_distance, nq * 4);
    o.nr = c.in(g ? nullptr : P.normal, nq * 12);
}
// device-only scratch, laid out after every input
void reserve_local(Call& c, const FrameInfo& I, LocalOff& o) {
    const size_t nq = (size_t)o.nq;
    reserve_grid(c, I, o.fs);
    o.rad = c.scratch(nq * 4); o.ang = c.scratch(nq * 4); o.minl = c.scratch(nq * 4); o.maxl = c.scratch(nq * 4);
    o.cand = c.scratch(nq * std::max(I.n, 1) * 4); o.cc = c.scratch(nq * 4);
}
// h: the staging buffer
void gather_local(uint8_t* h, const LocalOff& o, const borb_local_points_job& B, const std::vector<int32_t>& sel) {
    const borb_worldpoints_view& P = B.pts;
    for (int k = 0; k < o.nq; k++) {
        const int i = sel[o.sel0 + k];
        std::memcpy(h + o.wp + (size_t)k * 12, P.world_pos + (size_t)i * 3, 12);
        std::memcpy(h + o.md + (size_t)k * 32, P.desc + (size_t)i * 32, 32);
        if (B.has_obs) h[o.obs + k] = B.has_obs[i];
        std::memcpy(h + o.mx + (size_t)k * 4, P.max_distance + i, 4);
        std::memcpy(h + o.mn + (size_t)k * 4, P.min_distance + i, 4);
        std::memcpy(h + o.nr + (size_t)k * 12, P.normal + (size_t)i * 3, 12);
    }
}
// the results of a job, contiguous so that ONE device-to-host copy brings them back: px | py | pxr | level | viewcos | match | nm | valid
size_t local_res_bytes(int nq) { return (size_t)nq * 25 + 16; }
// L and the point side of A (the frame side comes from bind_frame_fields).  r: the job's result block (zeroed: level | viewcos of
// points outside the frustum read as 0)
void bind_local(const LocalOff& o, const borb_local_points_job& B, const FrameInfo& I, float viewing_cos_limit, float nnratio, const Call& c,
                uint8_t* r, LastArgs& L, ProjArgs& A) {
    const int nq = o.nq;
    L.variant = 3; L.n_last = nq; L.world_pos = (const float*)c.dev(o.wp);
    L.max_distance = (const float*)c.dev(o.mx); L.min_distance = (const float*)c.dev(o.mn); L.normal = (const float*)c.dev(o.nr);
    for (int i = 0; i < 3; i++) L.Ow[i] = B.Ow[i];
    L.log_scale = B.log_scale_factor; L.n_levels = I.n_levels; L.view_cos_limit = viewing_cos_limit;
    L.valid_in = nullptr;
    for (int i = 0; i < 12; i++) L.T[i] = B.Tcw[i];
    L.fx = B.fx; L.fy = B.fy; L.cx = B.cx; L.cy = B.cy; L.bf = B.mbf; L.th = B.th;
    L.minX = I.min_x; L.minY = I.min_y; L.maxX = I.max_x; L.maxY = I.max_y;
    L.scale_factors = A.scale_factors;
    L.proj_x = (float*)r; L.proj_y = L.proj_x + nq; L.proj_xr = L.proj_y + nq;
    L.level_out = (int32_t*)(L.proj_xr + nq); L.viewcos_out = (float*)(L.level_out + nq);
    L.valid_out = r + (size_t)nq * 24 + 16;
    L.radius = (float*)c.dev(o.rad); L.angle = (float*)c.dev(o.ang); L.minl = (int32_t*)c.dev(o.minl); L.maxl = (int32_t*)c.dev(o.maxl);
    A.occupied = o.fs.occ_p ? c.dev(o.fs.occ) : nullptr;
    wire_projection(L, A);
    A.mp_desc = c.dev(o.md); A.mp_has_obs = B.has_obs ? c.dev(o.obs) : nullptr;
    A.th = B.th; A.nnratio = nnratio; A.th_dist = TH_HIGH;
    A.cand = (uint32_t*)c.dev(o.cand); A.cand_cnt = (int*)c.dev(o.cc);
    A.mode = 0;
    A.out_match = (int32_t*)(L.viewcos_out + nq);
}
// search = 0: the frame has no features and every match stays -1
void scatter_local(const uint8_t* r, const LocalOff& o, const borb_local_points_job& B, const std::vector<int32_t>& sel, bool search,
                   int32_t* n_matches) {
    const int nq = o.nq;
    const float* rpx = (const float*)r; const float* rpy = rpx + nq; const float* rpxr = rpy + nq;
    const int32_t* rlvl = (const int32_t*)(rpxr + nq); const float* rvc = (const float*)(rlvl + nq);
    const int32_t* rmatch = (const int32_t*)(rvc + nq);
    const uint8_t* rval = r + (size_t)nq * 24 + 16;
    if (search) *n_matches = *(const int32_t*)(rmatch + nq);
    for (int k = 0; k < nq; k++) {
        const int i = sel[o.sel0 + k];
        B.in_view[i] = rval[k];
        if (search) B.match_feat[i] = rmatch[k];
        if (B.proj_x) B.proj_x[i] = rpx[k];
        if (B.proj_y) B.proj_y[i] = rpy[k];
        if (B.proj_xr) B.proj_xr[i] = rpxr[k];
        if (B.level) B.level[i] = rlvl[k];
        if (B.view_cos) B.view_cos[i] = rvc[k];
    }
}

// Shared body of borb_search_local_points (one job, a host view or a resident frame) and borb_search_local_points_batch (resident
// frames): project_points, candidates and resolve, one synchronisation.  Every job's results go to one region of the arena, zeroed
// first, that comes back with ONE device-to-host copy.
borb_status local_points_jobs(borb_matcher* m, const borb_local_points_job* jobs, int n_jobs, float viewing_cos_limit, float nnratio,
                              int32_t* n_matches, bool batch) {
    // search: valid points on a frame with features (otherwise only isInFrustum runs)
    struct Job { FrameInfo I; bool search; LocalOff o; size_t res; };
    std::vector<Job> J(n_jobs);
    std::vector<int32_t>& sel = m->sel;
    sel.clear();
    int max_nq = 0, max_n = 1, max_n_mp = 0;
    for (int j = 0; j < n_jobs; j++) {
        const borb_local_points_job& B = jobs[j];
        if (batch && !B.frame.resident) { set_error("job %d: borb_search_local_points_batch needs device-resident frames (borb_frame_view::resident)", j); return BORB_ERR_INVALID_ARG; }
        if (batch && (!B.in_view || !B.match_feat)) { set_error("job %d: null output", j); return BORB_ERR_INVALID_ARG; }
        const FrameInfo I = J[j].I = frame_info(&B.frame);
        borb_status s = check_local(B, I, m);
        if (s == BORB_OK) s = select_local(B, sel, J[j].o);
        if (s != BORB_OK) return job_fail(batch, j, s);
        const int nq = J[j].o.nq;
        J[j].search = nq > 0 && I.n > 0;
        max_nq = std::max(max_nq, nq);
        if (J[j].search) { max_n = std::max(max_n, I.n); max_n_mp = std::max(max_n_mp, nq); }
    }
    for (int j = 0; j < n_jobs; j++) { n_matches[j] = 0; clear_local(jobs[j]); }   // every job passed its checks
    if (max_nq == 0) return BORB_OK;
    Call c(m);
    HostGrids g;
    for (int j = 0; j < n_jobs; j++)
        if (J[j].o.nq > 0) stage_local(c, jobs[j], J[j].I, J[j].o, g);
    JobTable<LastArgs> lt(c, n_jobs);
    JobTable<ProjArgs> jt(c, n_jobs);
    g.stage(c);
    size_t res_end = 0;
    for (int j = 0; j < n_jobs; j++) {
        if (J[j].o.nq == 0) continue;
        reserve_local(c, J[j].I, J[j].o);
        J[j].res = c.result(local_res_bytes(J[j].o.nq));
        res_end = J[j].res + local_res_bytes(J[j].o.nq);
    }
    borb_status s;
    if ((s = c.begin(n_jobs == 1 && J[0].I.rf)) != BORB_OK) return s;
    LastArgs* hl = lt.host(c);
    ProjArgs* hj = jt.host(c);
    for (int j = 0; j < n_jobs; j++) {
        const LocalOff& o = J[j].o;
        LastArgs L{};
        ProjArgs A{};
        if (o.nq > 0) {
            if (o.gather) gather_local(c.host<uint8_t>(0), o, jobs[j], sel);
            bind_frame_fields(J[j].I, o.fs, c, g, A);
            bind_local(o, jobs[j], J[j].I, viewing_cos_limit, nnratio, c, c.res(J[j].res, false), L, A);
            if (!J[j].search) A.n_mp = 0;              // a frame without features: candidates and resolve skip the job
        }                                            // a job without valid points keeps n_last = 0 as well
        hl[j] = L;
        hj[j] = A;
    }
    if ((s = c.commit()) != BORB_OK) return s;
    BORB_CUDA(cudaMemsetAsync(c.res(0, false), 0, res_end, m->stream));
    for (int j = 0; j < n_jobs; j++)
        if (J[j].o.nq > 0 && J[j].I.rf && (s = c.wait(J[j].I.rf)) != BORB_OK) return s;
    m->launches += g.launch(c, m->stream);
    m->launches += launch_point_projection_batch(lt.dev(c), jt.dev(c), hl[0], hj[0], n_jobs, max_nq, max_n, max_n_mp, false, m->stream);
    if ((s = c.finish()) != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++)
        if (J[j].o.nq > 0) scatter_local(c.out(J[j].res), J[j].o, jobs[j], sel, J[j].search, &n_matches[j]);
    return BORB_OK;
}
}  // namespace

borb_status borb_search_local_points(borb_matcher* m, const borb_frame_view* F, const borb_worldpoints_view* pts, const uint8_t* has_obs,
                                     const float* Tcw, const float* Ow, float fx, float fy, float cx, float cy, float mbf,
                                     float viewing_cos_limit, float log_scale_factor, float th, float nnratio, uint8_t* in_view,
                                     float* proj_x, float* proj_y, float* proj_xr, int32_t* level, float* view_cos,
                                     int32_t* match_feat, int32_t* n_matches) {
    if (!m || !F || !pts || !Tcw || !Ow || !in_view || !match_feat || !n_matches) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_local_points_job B{};
    B.frame = *F; B.pts = *pts; B.has_obs = has_obs;
    std::memcpy(B.Tcw, Tcw, sizeof(B.Tcw)); std::memcpy(B.Ow, Ow, sizeof(B.Ow));
    B.fx = fx; B.fy = fy; B.cx = cx; B.cy = cy; B.mbf = mbf; B.log_scale_factor = log_scale_factor; B.th = th;
    B.in_view = in_view; B.proj_x = proj_x; B.proj_y = proj_y; B.proj_xr = proj_xr; B.level = level; B.view_cos = view_cos; B.match_feat = match_feat;
    return local_points_jobs(m, &B, 1, viewing_cos_limit, nnratio, n_matches, false);
}

borb_status borb_search_local_points_batch(borb_matcher* m, const borb_local_points_job* jobs, int n_jobs, float viewing_cos_limit,
                                           float nnratio, int32_t* n_matches) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && (!jobs || !n_matches))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    return local_points_jobs(m, jobs, n_jobs, viewing_cos_limit, nnratio, n_matches, true);
}

// ---- SearchForInitialization: borb_search_for_initialization is the one-job case of borb_search_for_initialization_batch
// (init_prefix + init_replay, k_proj.cu, one synchronisation).  The scratch of a job is O(n1), with no n1 x n2 candidate list.
namespace {
// Tracking::MonocularInitialization of one or many camera streams.  Each job has two frame sides, F1 (initial) and F2 (current).
// host == nullptr: the batch, whose jobs read their resident frames in place (keys, descriptors and F2's grid as built), so that only
// vbPrevMatched crosses PCIe.  Otherwise host = {F1, F2}, the single call's host views, of which only keys_un and desc are staged
// and F2's grid is built in call scratch.
borb_status init_jobs(borb_matcher* m, const borb_init_job* jobs, int n_jobs, const borb_frame_view* host, float nnratio,
                      int check_orientation, int32_t* n_matches) {
    const bool batch = host == nullptr;
    struct Job { borb_frame_view F[2]; FrameInfo I[2]; FrameStage fs[2]; bool live = false; size_t prev = 0, pre = 0, cnt = 0, res = 0, rprev = 0; };
    std::vector<Job> J(n_jobs);
    for (int j = 0; j < n_jobs; j++) {
        const borb_init_job& B = jobs[j];
        Job& o = J[j];
        if (batch) {
            if (!B.initial || !B.current) { set_error("job %d: null frame (the batch takes device-resident frames)", j); return BORB_ERR_INVALID_ARG; }
            o.F[0].resident = B.initial; o.F[1].resident = B.current;
        } else {
            o.F[0] = host[0]; o.F[1] = host[1];
        }
        for (int k = 0; k < 2; k++) {
            o.I[k] = frame_info(&o.F[k]);
            const borb_status s = batch ? check_frame(&o.F[k], o.I[k], m) : BORB_OK;     // the single call checks its views itself
            if (s != BORB_OK) return job_fail(batch, j, s);
        }
        if (o.I[0].n > 0 && (!B.prev_matched || !B.matches12)) { set_error("job %d: null prev_matched or matches12", j); return BORB_ERR_INVALID_ARG; }
    }
    int max_n1 = 0, max_n2 = 0;
    for (int j = 0; j < n_jobs; j++) {                  // a job without features: matches12 -1, prev_matched untouched
        const int n1 = J[j].I[0].n, n2 = J[j].I[1].n;
        n_matches[j] = 0;
        J[j].live = n1 > 0 && n2 > 0;
        if (!J[j].live) { std::fill_n(jobs[j].matches12, n1, -1); continue; }
        max_n1 = std::max(max_n1, n1); max_n2 = std::max(max_n2, n2);
    }
    if (max_n1 == 0) return BORB_OK;
    Call c(m);
    HostGrids g;
    for (int j = 0; j < n_jobs; j++) {
        Job& o = J[j];
        if (!o.live) continue;
        for (int k = 0; k < 2; k++)
            if (!o.I[k].rf) {                            // of a host view, only what the init kernels read
                o.fs[k].keys = c.in(o.F[k].keys_un, (size_t)o.I[k].n * sizeof(borb_keypoint));
                o.fs[k].desc = c.in(o.F[k].desc, (size_t)o.I[k].n * 32);
            }
        g.count(o.I[1]);                                 // F2's grid
        o.prev = c.in(jobs[j].prev_matched, (size_t)o.I[0].n * 8);
    }
    JobTable<InitJob> jt(c, n_jobs);
    g.stage(c);
    for (int j = 0; j < n_jobs; j++) {
        Job& o = J[j];
        if (!o.live) continue;
        const size_t n1 = (size_t)o.I[0].n;
        o.pre = c.scratch(n1 * INIT_K * 4);
        o.cnt = c.scratch(n1 * 4);
        reserve_grid(c, o.I[1], o.fs[1]);
        o.res = c.result(n1 * 4 + 4);
        o.rprev = c.result(n1 * 8);
    }
    borb_status s;
    // in place only for the batch: the kernels read a staged F2 more than once (ZERO_COPY_MAX)
    if ((s = c.begin(batch && n_jobs == 1)) != BORB_OK) return s;
    InitJob* hj = jt.host(c);
    for (int j = 0; j < n_jobs; j++) {
        const Job& o = J[j];
        InitJob I{};
        if (o.live) {                                    // a dead job keeps n1 = 0: both kernels skip it
            bind_frame_fields(o.I[1], o.fs[1], c, g, I.A);
            const borb_frame* f1 = o.I[0].rf;
            I.keys1 = f1 ? f1->keys : (const borb_keypoint*)c.dev(o.fs[0].keys);
            I.desc1 = f1 ? f1->desc : c.dev(o.fs[0].desc);
            I.n1 = o.I[0].n;
            I.window = (float)jobs[j].window_size;
            I.prev_in = (const float*)c.dev(o.prev);
            I.prefix = (uint32_t*)c.dev(o.pre); I.win_count = (int*)c.dev(o.cnt);
            I.out = (int32_t*)c.res(o.res, true); I.prev_out = (float*)c.res(o.rprev, true);     // straight into the landing buffer
        }
        hj[j] = I;
    }
    if ((s = c.commit()) != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++)
        for (int k = 0; k < 2; k++)
            if (J[j].live && J[j].I[k].rf && (s = c.wait(J[j].I[k].rf)) != BORB_OK) return s;
    m->launches += g.launch(c, m->stream);
    m->launches += launch_init_batch(jt.dev(c), hj[0], n_jobs, max_n1, max_n2, nnratio, check_orientation, m->stream);
    if ((s = c.finish()) != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++) {
        if (!J[j].live) continue;
        read_counted(c.out(J[j].res), J[j].I[0].n, jobs[j].matches12, &n_matches[j]);
        std::memcpy(jobs[j].prev_matched, c.out(J[j].rprev), (size_t)J[j].I[0].n * 8);
    }
    return BORB_OK;
}
}  // namespace

borb_status borb_search_for_initialization(borb_matcher* m, const borb_frame_view* f1, const borb_frame_view* f2, float* prev_matched,
                                           int window_size, float nnratio, int check_orientation, int32_t* matches12, int32_t* n_matches) {
    if (!m || !f1 || !f2 || !prev_matched || !matches12 || !n_matches) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (f1->n < 0 || f1->n > MATCH_MAX_FEATURES || f2->n < 0 || f2->n > MATCH_MAX_FEATURES) { set_error("feature count outside [0,%d]", MATCH_MAX_FEATURES); return BORB_ERR_INVALID_ARG; }
    if (f1->n > 0 && f2->n > 0) {
        if (!f1->keys_un || !f1->desc || !f2->keys_un || !f2->desc || !(f2->max_x > f2->min_x) || !(f2->max_y > f2->min_y)) {
            set_error("incomplete frame view"); return BORB_ERR_INVALID_ARG;
        }
        // a negative F1 octave would skip the reference's level test (GetFeaturesInArea with bCheckLevels false).  The search reads
        // no level table, so a view without one (n_levels < 1) has only the sign of its octaves checked
        const auto levels = [](int n) { return n > 0 ? n : INT_MAX; };
        borb_status s = check_octaves(f1->keys_un, f1->n, levels(f1->n_levels), "initial frame");
        if (s == BORB_OK) s = check_octaves(f2->keys_un, f2->n, levels(f2->n_levels), "current frame");
        if (s != BORB_OK) return s;
    }
    *n_matches = 0;
    for (int i = 0; i < f1->n; i++) matches12[i] = -1;
    if (f1->n == 0 || f2->n == 0) return BORB_OK;
    borb_frame_view V[2] = {*f1, *f2};
    V[0].resident = V[1].resident = nullptr;            // the host fields are read, never the resident frame
    borb_init_job B{};
    B.prev_matched = prev_matched; B.window_size = window_size; B.matches12 = matches12;
    return init_jobs(m, &B, 1, V, nnratio, check_orientation, n_matches);
}

borb_status borb_search_for_initialization_batch(borb_matcher* m, const borb_init_job* jobs, int n_jobs, float nnratio, int check_orientation,
                                                 int32_t* n_matches) {
    if (!m || n_jobs < 0) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (n_jobs > 0 && (!jobs || !n_matches)) { set_error("job 0: null job table or n_matches"); return BORB_ERR_INVALID_ARG; }
    return init_jobs(m, jobs, n_jobs, nullptr, nnratio, check_orientation, n_matches);
}

borb_status borb_distinctive_descriptors(borb_matcher* m, const uint8_t* desc, const int32_t* offsets, int n_points, int32_t* best_idx) {
    if (!m || !offsets || !best_idx || n_points < 0) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (n_points == 0) return BORB_OK;
    const int total_desc = offsets[n_points];
    for (int i = 0; i < n_points; i++)
        if (offsets[i + 1] < offsets[i] || offsets[i] < 0 || offsets[i + 1] - offsets[i] >= (1 << 16)) { set_error("offsets must ascend; at most 65535 observations per MapPoint"); return BORB_ERR_INVALID_ARG; }
    if (total_desc > 0 && !desc) { set_error("null descriptors"); return BORB_ERR_INVALID_ARG; }
    Call c(m);
    const size_t o_src = c.in(nullptr, sizeof(const uint8_t*));     // the one row source: the staged rows, filled in place
    const size_t o_d = c.in(desc, (size_t)total_desc * 32);
    const size_t o_o = c.in(offsets, (size_t)(n_points + 1) * 4);
    const size_t r_b = c.result((size_t)n_points * 4);
    borb_status s;
    if ((s = c.begin()) != BORB_OK) return s;
    *c.host<const uint8_t*>(o_src) = c.dev(o_d);
    if ((s = c.commit()) != BORB_OK) return s;
    const DistinctArgs A{(const uint8_t* const*)c.dev(o_src), nullptr, nullptr, (const int32_t*)c.dev(o_o), n_points,
                         (int32_t*)c.res(r_b, false), nullptr};
    m->launches += launch_distinctive(A, m->stream);
    if ((s = c.finish()) != BORB_OK) return s;
    std::memcpy(best_idx, c.out(r_b), (size_t)n_points * 4);
    return BORB_OK;
}

// The rows are read in place from the resident frames: only the observation tables, the offsets and the frame table go up, and only
// best_idx and the chosen rows come down.
borb_status borb_distinctive_descriptors_frames(borb_matcher* m, const borb_frame* const* frames, int n_frames, const int32_t* obs_frame,
                                                const int32_t* obs_idx, const int32_t* offsets, int n_points, int32_t* best_idx,
                                                uint8_t* desc_out) {
    if (!m || n_frames < 0 || n_points < 0 || (n_frames > 0 && !frames) || (n_points > 0 && !offsets)) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (n_points > 0 && (!best_idx || !desc_out)) { set_error("null best_idx or desc_out"); return BORB_ERR_INVALID_ARG; }
    for (int f = 0; f < n_frames; f++) {
        if (!frames[f]) { set_error("frame %d: not a device-resident frame", f); return BORB_ERR_INVALID_ARG; }
        if (frames[f]->device != m->device) { set_error("frame %d and matcher live on different devices", f); return BORB_ERR_INVALID_ARG; }
    }
    if (n_points == 0) return BORB_OK;
    if (offsets[0] != 0) { set_error("point 0: offsets must start at 0 (got %d)", offsets[0]); return BORB_ERR_INVALID_ARG; }
    for (int p = 0; p < n_points; p++)
        if (offsets[p + 1] < offsets[p] || offsets[p + 1] - offsets[p] >= (1 << 16)) {
            set_error("point %d: offsets must ascend; at most 65535 observations per MapPoint (got %d .. %d)", p, offsets[p], offsets[p + 1]);
            return BORB_ERR_INVALID_ARG;
        }
    const int total = offsets[n_points];
    if (total > 0 && (!obs_frame || !obs_idx)) { set_error("null obs_frame or obs_idx"); return BORB_ERR_INVALID_ARG; }
    for (int p = 0; p < n_points; p++)
        for (int o = offsets[p]; o < offsets[p + 1]; o++) {
            const int f = obs_frame[o];
            if (f < 0 || f >= n_frames) { set_error("point %d: observation %d names frame %d outside the table's %d", p, o, f, n_frames); return BORB_ERR_INVALID_ARG; }
            if (obs_idx[o] < 0 || obs_idx[o] >= frames[f]->n) {
                set_error("point %d: observation %d reads feature %d of frame %d, which has %d", p, o, obs_idx[o], f, frames[f]->n);
                return BORB_ERR_INVALID_ARG;
            }
        }
    if (total == 0) {                                   // no observation: nothing to launch
        for (int p = 0; p < n_points; p++) best_idx[p] = -1;
        return BORB_OK;
    }
    Call c(m);
    const size_t o_src = c.in(nullptr, (size_t)n_frames * sizeof(const uint8_t*));   // the frames' descriptor arrays, filled in place
    const size_t o_of = c.in(obs_frame, (size_t)total * 4), o_oi = c.in(obs_idx, (size_t)total * 4);
    const size_t o_o = c.in(offsets, (size_t)(n_points + 1) * 4);
    const size_t r_b = c.result((size_t)n_points * 4), r_d = c.result((size_t)n_points * 32);
    borb_status s;
    if ((s = c.begin()) != BORB_OK) return s;
    const uint8_t** src = c.host<const uint8_t*>(o_src);
    for (int f = 0; f < n_frames; f++) src[f] = frames[f]->desc;
    if ((s = c.commit()) != BORB_OK) return s;
    std::vector<const borb_frame*> wait(frames, frames + n_frames);
    std::sort(wait.begin(), wait.end());
    wait.erase(std::unique(wait.begin(), wait.end()), wait.end());
    for (const borb_frame* f : wait)
        if ((s = c.wait(f)) != BORB_OK) return s;
    const DistinctArgs A{(const uint8_t* const*)c.dev(o_src), (const int32_t*)c.dev(o_of), (const int32_t*)c.dev(o_oi), (const int32_t*)c.dev(o_o),
                         n_points, (int32_t*)c.res(r_b, false), c.res(r_d, false)};
    m->launches += launch_distinctive(A, m->stream);
    if ((s = c.finish()) != BORB_OK) return s;
    std::memcpy(best_idx, c.out(r_b), (size_t)n_points * 4);
    for (int p = 0; p < n_points; p++)
        if (best_idx[p] >= 0) std::memcpy(desc_out + (size_t)p * 32, c.out(r_d) + (size_t)p * 32, 32);
    return BORB_OK;
}

// ---- SearchByBoW: borb_search_by_bow (keyframes against one frame), borb_search_by_bow_kf (one keyframe pair) and
// borb_search_by_bow_batch (TrackReferenceKeyFrame of many camera streams: a keyframe against its own resident frame with BoW) are
// jobs of one launch of bow_match_kernel and one synchronisation.
namespace {
// Where an argument error lies, as its text names it: "job j", or for a BowVector reference of borb_bow_score_batch "job j query"
// (ref == QUERY_REF) or "job j target t" (ref = t).
constexpr int NO_REF = -2, QUERY_REF = -1;
std::string job_at(int j, int ref = NO_REF) {
    std::string s = "job " + std::to_string(j);
    if (ref == QUERY_REF) s += " query";
    else if (ref >= 0) s += " target " + std::to_string(ref);
    return s;
}

borb_status check_resident_bow(const borb_frame* f, const borb_matcher* m, int j, const char* what, int ref = NO_REF) {
    if (!f) { set_error("%s: %s is not a device-resident frame", job_at(j, ref).c_str(), what); return BORB_ERR_INVALID_ARG; }
    if (f->device != m->device) { set_error("%s: %s and matcher live on different devices", job_at(j, ref).c_str(), what); return BORB_ERR_INVALID_ARG; }
    if (!f->has_bow) { set_error("%s: %s has no BoW (borb_frames_compute_bow)", job_at(j, ref).c_str(), what); return BORB_ERR_INVALID_ARG; }
    if (f->n > MATCH_MAX_FEATURES) {
        set_error("%s: %s has %d features (limit %d)", job_at(j, ref).c_str(), what, f->n, MATCH_MAX_FEATURES);
        return BORB_ERR_INVALID_ARG;
    }
    return BORB_OK;
}

// q: the keyframe; t: the frame (mode 0) or kf2 (mode 1); match: t.n() entries (mode 0) or q.n() (mode 1)
struct BowJob { KfSide q, t; int32_t* match; };

// The arguments are checked by the callers.  Consecutive jobs with the same target share its staging.
borb_status bow_jobs(borb_matcher* m, std::vector<BowJob>& J, int mode, float nnratio, int check_ori, int32_t* n_matches) {
    const int n_jobs = (int)J.size();
    std::vector<size_t> off(n_jobs + 1, 0);           // each job's matches in the result block
    int max_t = 0;
    for (int j = 0; j < n_jobs; j++) {
        off[j + 1] = off[j] + (size_t)(mode == 0 ? J[j].t.n() : J[j].q.n());
        max_t = std::max(max_t, J[j].t.n());
    }
    Call c(m);
    for (int j = 0; j < n_jobs; j++) {
        J[j].q.stage(c);
        if (j > 0 && J[j].t.v == J[j - 1].t.v && J[j].t.rf == J[j - 1].t.rf) J[j].t = J[j - 1].t;
        else J[j].t.stage(c);
    }
    const size_t o_q = c.in(nullptr, (size_t)n_jobs * sizeof(KfDev)), o_t = c.in(nullptr, (size_t)n_jobs * sizeof(KfDev));   // filled in place
    const size_t o_off = c.in(nullptr, (size_t)n_jobs * sizeof(size_t));
    const size_t o_bins = c.scratch(off[n_jobs] + 16);
    const size_t r_cnt = c.result((size_t)n_jobs * 4), r_match = c.result(off[n_jobs] * 4);     // n_matches of every job, then every job's matches
    borb_status s;
    if ((s = c.begin()) != BORB_OK) return s;
    KfDev* hq = c.host<KfDev>(o_q);
    KfDev* ht = c.host<KfDev>(o_t);
    size_t* hoff = c.host<size_t>(o_off);
    for (int j = 0; j < n_jobs; j++) {
        hq[j] = J[j].q.bind(c);
        ht[j] = J[j].t.bind(c);
        hoff[j] = off[j];
    }
    if ((s = c.commit()) != BORB_OK) return s;
    for (const BowJob& B : J) {
        if (B.q.rf && (s = c.wait(B.q.rf)) != BORB_OK) return s;
        if (B.t.rf && (s = c.wait(B.t.rf)) != BORB_OK) return s;
    }
    m->launches += launch_bow_match((const KfDev*)c.dev(o_q), (const KfDev*)c.dev(o_t), n_jobs, mode, nnratio, check_ori,
                                    (int32_t*)c.res(r_match, false), (const size_t*)c.dev(o_off), c.dev(o_bins), (int32_t*)c.res(r_cnt, false),
                                    max_t, m->stream);
    if ((s = c.finish()) != BORB_OK) return s;
    std::memcpy(n_matches, c.out(r_cnt), (size_t)n_jobs * 4);
    for (int j = 0; j < n_jobs; j++) std::memcpy(J[j].match, c.out(r_match) + off[j] * 4, (off[j + 1] - off[j]) * 4);
    return BORB_OK;
}
}  // namespace

borb_status borb_search_by_bow(borb_matcher* m, const borb_keyframe_view* kfs, int n_kf, const borb_keyframe_view* frame, float nnratio,
                               int check_orientation, int32_t* match, int32_t* n_matches) {
    if (!m || !frame || !match || !n_matches || n_kf < 0 || (n_kf > 0 && !kfs)) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_status s = check_kf(frame, "borb_search_by_bow(frame)");
    for (int i = 0; i < n_kf && s == BORB_OK; i++) s = check_kf(&kfs[i], "borb_search_by_bow(keyframe)");
    if (s != BORB_OK) return s;
    if (n_kf == 0) return BORB_OK;
    std::vector<BowJob> J(n_kf);
    for (int i = 0; i < n_kf; i++) J[i] = BowJob{KfSide{&kfs[i]}, KfSide{frame}, match + (size_t)i * frame->n};
    return bow_jobs(m, J, 0, nnratio, check_orientation, n_matches);
}

borb_status borb_search_by_bow_kf(borb_matcher* m, const borb_keyframe_view* kf1, const borb_keyframe_view* kf2, float nnratio,
                                  int check_orientation, int32_t* match12, int32_t* n_matches) {
    if (!m || !kf1 || !kf2 || !match12 || !n_matches) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_status s = check_kf(kf1, "borb_search_by_bow_kf(kf1)");
    if (s == BORB_OK) s = check_kf(kf2, "borb_search_by_bow_kf(kf2)");
    if (s != BORB_OK) return s;
    std::vector<BowJob> J{BowJob{KfSide{kf1}, KfSide{kf2}, match12}};
    return bow_jobs(m, J, 1, nnratio, check_orientation, n_matches);
}

borb_status borb_search_by_bow_batch(borb_matcher* m, const borb_bow_job* jobs, int n_jobs, float nnratio, int check_orientation,
                                     int32_t* n_matches) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && (!jobs || !n_matches))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (n_jobs == 0) return BORB_OK;
    std::vector<BowJob> J(n_jobs);
    for (int j = 0; j < n_jobs; j++) {
        const borb_bow_job& B = jobs[j];
        borb_status s = check_resident_bow(B.frame, m, j, "frame");
        if (s != BORB_OK) return s;
        if (!B.match) { set_error("job %d: null output", j); return BORB_ERR_INVALID_ARG; }
        if (B.kf_frame) {
            if ((s = check_resident_bow(B.kf_frame, m, j, "kf_frame")) != BORB_OK) return s;
        } else if ((s = check_kf(&B.kf, "keyframe")) != BORB_OK) return job_fail(true, j, s);
        J[j] = BowJob{KfSide{&B.kf, B.kf_frame}, KfSide{&NO_VIEW, B.frame}, B.match};
    }
    std::fill_n(n_matches, n_jobs, 0);                  // every job passed its checks
    return bow_jobs(m, J, 0, nnratio, check_orientation, n_matches);
}

// ---------------------------------------------------------------------------------------------------------------
// Device-resident keyframe database: KeyFrameDatabase (src/KeyFrameDatabase.cc) + the keyframe-side inputs of SearchByBoW.
// A keyframe is kept as a STREAM RECORD (k_bowdb.cu): features permuted into FeatureVector order so that a node's
// descriptors are consecutive rows.  The reference guards add / erase / Detect*Candidates with mMutex (they run on the
// LoopClosing, Tracking and LocalMapping threads); the handle carries the same mutex.
struct borb_kfdb {
    int device = 0;
    std::mutex mu;
    struct Entry {
        uint8_t* block = nullptr;
        KfStream stream{};
        BowDev bow{nullptr, nullptr, 0};
        uint8_t* d_meta = nullptr;           // m x 8 bytes inside block (row order)
        std::vector<uint16_t> orig;          // host copy of the row -> feature permutation
        std::vector<uint32_t> meta;          // host copy of the row records (borb_kfdb_set_has_mp rewrites the flag)
        int n = 0;
        bool alive = false;
    };
    std::vector<Entry> entries;
    BowDev* d_table = nullptr;      // mirrors entries[*].bow
    KfStream* d_stream = nullptr;   // mirrors entries[*].stream
    size_t table_cap = 0;
    bool dirty = true;
    size_t bytes = 0;
    int n_sm = 0;
};

borb_status borb_kfdb_create(int device, borb_kfdb** out) {
    if (!out) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) { set_error("no CUDA device: the keyframe database is GPU-resident"); return BORB_ERR_NO_DEVICE; }
    if (device < 0 || device >= n) { set_error("device %d out of range", device); return BORB_ERR_INVALID_ARG; }
    borb_kfdb* db = new borb_kfdb();
    db->device = device;
    cudaDeviceGetAttribute(&db->n_sm, cudaDevAttrMultiProcessorCount, device);
    if (db->n_sm < 1) db->n_sm = 1;
    *out = db;
    return BORB_OK;
}

static void kfdb_clear_locked(borb_kfdb* db) {
    cudaSetDevice(db->device);
    cudaDeviceSynchronize();
    for (auto& e : db->entries) cudaFree(e.block);
    db->entries.clear();
    db->dirty = true;
    db->bytes = 0;
}

borb_status borb_kfdb_clear(borb_kfdb* db) {
    if (!db) return BORB_OK;
    std::lock_guard<std::mutex> lk(db->mu);
    kfdb_clear_locked(db);
    return BORB_OK;
}

borb_status borb_kfdb_destroy(borb_kfdb* db) {
    if (!db) return BORB_OK;
    { std::lock_guard<std::mutex> lk(db->mu); kfdb_clear_locked(db); cudaFree(db->d_table); cudaFree(db->d_stream); }
    delete db;
    return BORB_OK;
}

// Appends a keyframe whose device block (kfdb_block_layout(nn, m, n_bow), complete) holds the row records `meta` (m x 2 u32, row
// order) and returns its slot; the caller holds db->mu.  The one place that points a slot's KfStream and BowDev into its block and
// keeps the host copies of the rows (borb_kfdb_set_has_mp rewrites their flag), for borb_kfdb_add and borb_kfdb_add_frames alike.
static int32_t kfdb_append_locked(borb_kfdb* db, uint8_t* block, int nn, int m, int n, int n_bow, const uint32_t* meta) {
    const KfdbBlock L = kfdb_block_layout(nn, m, n_bow);
    borb_kfdb::Entry e;
    e.block = block;
    e.orig.resize(m);
    e.meta.assign(meta, meta + (size_t)m * 2);
    for (int r = 0; r < m; r++) e.orig[r] = (uint16_t)(meta[2 * r] & 0xFFFFu);
    e.stream.node = (const uint32_t*)(block + L.node); e.stream.start = (const int32_t*)(block + L.start);
    e.stream.meta = (const uint2*)(block + L.meta); e.stream.desc = block + L.desc;
    e.stream.nn = nn; e.stream.m = m; e.stream.n = n; e.stream.pad = 0;
    e.d_meta = block + L.meta;
    e.n = n;
    e.bow.word = (const uint32_t*)(block + L.bow_word); e.bow.value = (const double*)(block + L.bow_value); e.bow.n = n_bow;
    e.alive = true;
    db->entries.push_back(std::move(e));
    db->dirty = true;
    db->bytes += L.bytes;
    return (int32_t)db->entries.size() - 1;
}

borb_status borb_kfdb_add(borb_kfdb* db, const borb_keyframe_view* kf, const uint32_t* bow_word, const double* bow_value, int n_bow,
                          int32_t* slot_out) {
    if (!db || !kf || !slot_out || n_bow < 0 || (n_bow > 0 && (!bow_word || !bow_value))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_status s = check_kf(kf, "borb_kfdb_add");
    if (s != BORB_OK) return s;
    for (int i = 1; i < n_bow; i++)
        if (bow_word[i] <= bow_word[i - 1]) { set_error("BowVector words must ascend (std::map order)"); return BORB_ERR_INVALID_ARG; }
    const int nn = kf->fv.n_nodes;
    const int m = nn > 0 ? kf->fv.start[nn] : 0;
    std::lock_guard<std::mutex> lk(db->mu);
    BORB_CUDA(cudaSetDevice(db->device));
    // one device block per keyframe, packed here and uploaded whole (kfdb_insert_kernel writes the same bytes from a resident frame)
    const KfdbBlock L = kfdb_block_layout(nn, m, n_bow);
    std::vector<uint8_t> h(L.bytes, 0);
    uint32_t* meta = reinterpret_cast<uint32_t*>(&h[L.meta]);
    if (nn) {
        std::memcpy(&h[L.node], kf->fv.node_id, (size_t)nn * 4);
        std::memcpy(&h[L.start], kf->fv.start, (size_t)(nn + 1) * 4);
        int a = 0;                                                     // node index of row r (rows are grouped by node)
        for (int r = 0; r < m; r++) {
            while (a + 1 < nn && r >= kf->fv.start[a + 1]) a++;
            const uint32_t f = kf->fv.feat_idx[r];
            meta[2 * r] = f | ((kf->has_mp && kf->has_mp[f]) ? 0x10000u : 0u) | ((uint32_t)a << 17);
            std::memcpy(&meta[2 * r + 1], &kf->keys_un[f].angle, 4);
            std::memcpy(&h[L.desc + (size_t)r * 32], kf->desc + (size_t)f * 32, 32);
        }
    }
    if (n_bow) { std::memcpy(&h[L.bow_word], bow_word, (size_t)n_bow * 4); std::memcpy(&h[L.bow_value], bow_value, (size_t)n_bow * 8); }
    uint8_t* block = nullptr;
    BORB_CUDA(cudaMalloc(&block, L.bytes));
    cudaError_t ce = poison_byte() >= 0 ? cudaMemset(block, poison_byte(), L.bytes) : cudaSuccess;   // borb_debug_set_poison
    if (ce == cudaSuccess) ce = cudaMemcpy(block, h.data(), L.bytes, cudaMemcpyHostToDevice);
    if (ce != cudaSuccess) { cudaFree(block); BORB_CUDA(ce); }
    *slot_out = kfdb_append_locked(db, block, nn, m, kf->n, n_bow, meta);
    return BORB_OK;
}

borb_status borb_kfdb_erase(borb_kfdb* db, int32_t slot) {
    if (!db) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    std::lock_guard<std::mutex> lk(db->mu);
    if (slot < 0 || slot >= (int)db->entries.size() || !db->entries[slot].alive) { set_error("bad keyframe slot"); return BORB_ERR_INVALID_ARG; }
    BORB_CUDA(cudaSetDevice(db->device));
    BORB_CUDA(cudaDeviceSynchronize());           // queries enqueued under the mutex may still be reading the block
    borb_kfdb::Entry& e = db->entries[slot];
    cudaFree(e.block);
    e = borb_kfdb::Entry();
    db->dirty = true;
    return BORB_OK;
}

borb_status borb_kfdb_set_has_mp_batch(borb_kfdb* db, int n, const int32_t* slots, const uint8_t* const* has_mp) {
    if (!db || n < 0 || (n > 0 && (!slots || !has_mp))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    std::lock_guard<std::mutex> lk(db->mu);
    for (int i = 0; i < n; i++) {
        if (!has_mp[i]) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
        if (slots[i] < 0 || slots[i] >= (int)db->entries.size() || !db->entries[slots[i]].alive) { set_error("bad keyframe slot"); return BORB_ERR_INVALID_ARG; }
    }
    if (n == 0) return BORB_OK;
    BORB_CUDA(cudaSetDevice(db->device));
    BORB_CUDA(cudaDeviceSynchronize());           // a search enqueued under the mutex may still be reading the records
    for (int i = 0; i < n; i++) {
        borb_kfdb::Entry& e = db->entries[slots[i]];
        for (size_t r = 0; r < e.orig.size(); r++) e.meta[2 * r] = (e.meta[2 * r] & ~0x10000u) | (has_mp[i][e.orig[r]] ? 0x10000u : 0u);
        if (!e.meta.empty()) BORB_CUDA(cudaMemcpy(e.d_meta, e.meta.data(), e.meta.size() * 4, cudaMemcpyHostToDevice));
    }
    return BORB_OK;
}

borb_status borb_kfdb_set_has_mp(borb_kfdb* db, int32_t slot, const uint8_t* has_mp) {
    return borb_kfdb_set_has_mp_batch(db, 1, &slot, &has_mp);
}

borb_status borb_kfdb_size(const borb_kfdb* db, int32_t* n_slots, uint64_t* device_bytes) {
    if (!db) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    std::lock_guard<std::mutex> lk(const_cast<borb_kfdb*>(db)->mu);
    if (n_slots) *n_slots = (int32_t)db->entries.size();
    if (device_bytes) *device_bytes = db->bytes;
    return BORB_OK;
}

// caller holds db->mu
static borb_status kfdb_sync_table(borb_kfdb* db) {
    if (!db->dirty) return BORB_OK;
    const size_t n = db->entries.size();
    if (n > db->table_cap) {
        BORB_CUDA(cudaDeviceSynchronize());
        cudaFree(db->d_table); db->d_table = nullptr;
        cudaFree(db->d_stream); db->d_stream = nullptr;
        db->table_cap = n + n / 2 + 64;
        BORB_CUDA(cudaMalloc(&db->d_table, db->table_cap * sizeof(BowDev)));
        BORB_CUDA(cudaMalloc(&db->d_stream, db->table_cap * sizeof(KfStream)));
        if (const int p = poison_byte(); p >= 0) {      // borb_debug_set_poison: the entries past the live slots are never written
            BORB_CUDA(cudaMemset(db->d_table, p, db->table_cap * sizeof(BowDev)));
            BORB_CUDA(cudaMemset(db->d_stream, p, db->table_cap * sizeof(KfStream)));
        }
    }
    std::vector<BowDev> t(n);
    std::vector<KfStream> st(n);
    for (size_t i = 0; i < n; i++) {
        t[i] = db->entries[i].alive ? db->entries[i].bow : BowDev{nullptr, nullptr, 0};
        st[i] = db->entries[i].alive ? db->entries[i].stream : KfStream{};
    }
    if (n) {
        BORB_CUDA(cudaMemcpy(db->d_table, t.data(), n * sizeof(BowDev), cudaMemcpyHostToDevice));
        BORB_CUDA(cudaMemcpy(db->d_stream, st.data(), n * sizeof(KfStream), cudaMemcpyHostToDevice));
    }
    db->dirty = false;
    return BORB_OK;
}

static std::atomic<int> g_bow_csa{2};
static std::atomic<int> g_bow_item_target{8192};   // keyframes per work item = target / nt^2 (tuning knob of the measurement scripts)
static std::atomic<int> g_bow_static{0};
borb_status borb_debug_set_bow_item_target(int t) { g_bow_static.store(t < 0 ? 1 : 0); if (t < 0) t = -t; g_bow_item_target.store(t < 1 ? 1 : t); return BORB_OK; }
borb_status borb_debug_set_bow_csa(int mode) { g_bow_csa.store(mode < 0 ? 0 : (mode > 2 ? 2 : mode)); return BORB_OK; }

namespace {

// Every distinct database of a call, locked in address order (two concurrent batches over the same databases cannot deadlock),
// held across the table sync and the kernel enqueue (erase() and set_has_mp() synchronise the device before they touch a block).
struct DbLocks {
    std::vector<borb_kfdb*> dbs;
    std::vector<std::unique_lock<std::mutex>> held;
    explicit DbLocks(std::vector<borb_kfdb*> all) : dbs(std::move(all)) {
        std::sort(dbs.begin(), dbs.end(), std::less<borb_kfdb*>());
        dbs.erase(std::unique(dbs.begin(), dbs.end()), dbs.end());
        for (borb_kfdb* db : dbs) held.emplace_back(db->mu);
    }
    borb_status sync() {
        for (borb_kfdb* db : dbs) { borb_status st = kfdb_sync_table(db); if (st != BORB_OK) return st; }
        return BORB_OK;
    }
    void unlock() { held.clear(); }
};

// A job of borb_bow_score_batch, resolved under the database locks: the query and the targets as device BowVectors, and the
// resident frames among them, whose ready events the launch waits on.
struct BowTable {
    BowDev query;
    std::vector<BowDev> targets;
    std::vector<const borb_frame*> frames;
};

// One query of the database score: the BowVector comes from the host (word / value) or from a resident frame, and is scored
// against every slot of db; or, with a table, the table's query is scored against its targets (db, frame and word unused).
struct QueryJob {
    borb_kfdb* db;
    const borb_frame* frame;
    const uint32_t* word; const double* value; int n_bow;
    int32_t* common; float* score; uint32_t* first_word;      // common, first_word and n_slots may be null with a table
    int cap; int32_t* n_slots;
    const BowTable* table = nullptr;
};

// Shared body of borb_kfdb_query, borb_kfdb_query_batch and borb_bow_score_batch: one launch of kfdb_score_kernel for every job
// (none when no job has a slot or a target) and one synchronisation.  The arguments are checked by the callers.  held: the
// databases' locks, taken by a caller that resolved its tables under them (released once the kernel is enqueued); without it, the
// jobs' databases are locked here.
borb_status kfdb_query_jobs(borb_matcher* m, const QueryJob* q, int n_jobs, bool batch, DbLocks* held = nullptr) {
    std::vector<int> ns(n_jobs);
    std::vector<size_t> o_w(n_jobs, 0), o_v(n_jobs, 0), o_t(n_jobs, 0), ho(n_jobs, 0);
    int max_slots = 0, max_nq = 0;
    Call c(m);
    {
        std::optional<DbLocks> own;
        if (!held) {
            std::vector<borb_kfdb*> dbs(n_jobs);
            for (int j = 0; j < n_jobs; j++) dbs[j] = q[j].db;
            own.emplace(std::move(dbs));
        }
        DbLocks& lk = held ? *held : *own;
        for (int j = 0; j < n_jobs; j++) {
            ns[j] = q[j].table ? (int)q[j].table->targets.size() : (int)q[j].db->entries.size();
            if (q[j].n_slots) *q[j].n_slots = ns[j];
        }
        for (int j = 0; j < n_jobs; j++)
            if (q[j].cap < ns[j]) { set_error("output capacity %d < %d database slots", q[j].cap, ns[j]); return job_fail(batch, j, BORB_ERR_CAPACITY); }
        for (int j = 0; j < n_jobs; j++) {
            max_slots = std::max(max_slots, ns[j]);
            max_nq = std::max(max_nq, q[j].table ? q[j].table->query.n : q[j].frame ? q[j].frame->n_bow : q[j].n_bow);
        }
        if (max_slots == 0) return BORB_OK;
        BORB_CUDA(cudaSetDevice(m->device));
        borb_status s;
        if (std::any_of(q, q + n_jobs, [](const QueryJob& x) { return !x.table; }) && (s = lk.sync()) != BORB_OK) return s;
        for (int j = 0; j < n_jobs; j++) {
            if (q[j].table) o_t[j] = c.in(q[j].table->targets.data(), (size_t)ns[j] * sizeof(BowDev));
            else if (!q[j].frame) { o_w[j] = c.in(q[j].word, (size_t)q[j].n_bow * 4); o_v[j] = c.in(q[j].value, (size_t)q[j].n_bow * 8); }
        }
        const size_t o_jobs = c.in(nullptr, (size_t)n_jobs * sizeof(KfdbQueryJob));     // filled in place
        for (int j = 0; j < n_jobs; j++) ho[j] = c.result((size_t)ns[j] * 12);
        if ((s = c.begin()) != BORB_OK) return s;
        KfdbQueryJob* hj = c.host<KfdbQueryJob>(o_jobs);
        for (int j = 0; j < n_jobs; j++) {
            // the three result arrays are written by the kernel straight into the pinned landing buffer (device-addressable, UVA)
            uint8_t* o = c.res(ho[j], true);
            KfdbQueryJob J{};
            J.n_slots = ns[j];
            if (const BowTable* T = q[j].table) {
                J.table = (const BowDev*)c.dev(o_t[j]);
                J.qword = T->query.word; J.qvalue = T->query.value; J.nq = T->query.n;
            } else {
                J.table = q[j].db->d_table;
                if (q[j].frame) { J.qword = q[j].frame->bow_word; J.qvalue = q[j].frame->bow_value; J.nq = q[j].frame->n_bow; }
                else { J.qword = (const uint32_t*)c.dev(o_w[j]); J.qvalue = (const double*)c.dev(o_v[j]); J.nq = q[j].n_bow; }
            }
            J.common = (int32_t*)o; J.score = (float*)(o + (size_t)ns[j] * 4); J.first_word = (uint32_t*)(o + (size_t)ns[j] * 8);
            hj[j] = J;
        }
        if ((s = c.commit()) != BORB_OK) return s;
        for (int j = 0; j < n_jobs; j++) {
            if (q[j].frame && (s = c.wait(q[j].frame)) != BORB_OK) return s;
            if (q[j].table)
                for (const borb_frame* f : q[j].table->frames)
                    if ((s = c.wait(f)) != BORB_OK) return s;
        }
        m->launches += launch_kfdb_score((const KfdbQueryJob*)c.dev(o_jobs), n_jobs, max_slots, max_nq, m->n_sm, m->stream);
        lk.unlock();
    }
    const borb_status s = c.finish();
    if (s != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++) {
        const uint8_t* o = c.out(ho[j]);
        if (q[j].common) std::memcpy(q[j].common, o, (size_t)ns[j] * 4);
        if (ns[j]) std::memcpy(q[j].score, o + (size_t)ns[j] * 4, (size_t)ns[j] * 4);
        if (q[j].first_word) std::memcpy(q[j].first_word, o + (size_t)ns[j] * 8, (size_t)ns[j] * 4);
    }
    return BORB_OK;
}

// One frame of the database search: a resident frame with its BoW, or a host view.
struct SearchJob {
    borb_kfdb* db;
    const borb_frame* frame;
    const borb_keyframe_view* view;
    const int32_t* slots; int n_kf;
    int32_t* dense;                    // borb_search_by_bow_db: match[k * n + j]
    int32_t* n_matches; int32_t* pair_offset; uint32_t* pairs; int pairs_cap; int32_t* n_pairs_total;
    int32_t query_slot;                // SearchByBoW(KeyFrame*, KeyFrame*): the query keyframe, a slot of db (frame and view unused)
};

// Shared body of borb_search_by_bow_db, _db_pairs and _db_batch, and (kfkf) of borb_search_by_bow_kf_db_pairs and _batch: pack,
// match and finalize over the job table (3 launches; none when no job has a keyframe and a feature inside a node) and one
// synchronisation.  The arguments are checked by the callers, except the slot lists and the query slots, which are checked here under
// the database locks (a batch checks every job with keyframes, a single call only one that has work, as before).
borb_status bowdb_jobs(borb_matcher* m, const SearchJob* J, int n_jobs, float nnratio, int check_ori, bool batch, bool kfkf = false) {
    struct Plan { KfSide f; int nn, m, n; bool work; FrameBlockHdr h; size_t o_fb, o_sl, o_ctr, o_hist, o_tab, o_dense, ho; };
    std::vector<Plan> P(n_jobs);
    for (int j = 0; j < n_jobs; j++) {
        const SearchJob& S = J[j];
        Plan& p = P[j];
        if (!kfkf) {
            p.f = S.frame ? KfSide{&NO_VIEW, S.frame} : KfSide{S.view};
            p.nn = p.f.nn(); p.m = p.f.m(); p.n = p.f.n();
        }                                                              // else: read from the database under its lock
        p.work = S.n_kf > 0 && (kfkf || p.m > 0);
        if (S.n_pairs_total) *S.n_pairs_total = 0;
        if (S.dense) for (size_t i = 0; i < (size_t)S.n_kf * p.n; i++) S.dense[i] = -1;
        for (int i = 0; i < S.n_kf; i++) { S.n_matches[i] = 0; if (S.pair_offset) S.pair_offset[i] = 0; }
    }
    std::vector<int> work;
    Call c(m);
    {
        std::vector<borb_kfdb*> dbs(n_jobs);
        for (int j = 0; j < n_jobs; j++) dbs[j] = J[j].db;
        DbLocks lk(std::move(dbs));
        for (int j = 0; j < n_jobs; j++) {
            const SearchJob& S = J[j];
            if (kfkf) {
                const int q = S.query_slot;
                if (q < 0 || q >= (int)S.db->entries.size() || !S.db->entries[q].alive || S.db->entries[q].n == 0) {
                    set_error("query slot %d is not a live keyframe added with features", q);
                    return job_fail(batch, j, BORB_ERR_INVALID_ARG);
                }
                const KfStream& st = S.db->entries[q].stream;
                P[j].nn = st.nn; P[j].m = st.m; P[j].n = st.n;
                P[j].work = S.n_kf > 0 && st.m > 0;
            }
            if (S.n_kf == 0 || (!batch && !P[j].work)) continue;      // the single calls return zeros before looking at the slots
            const int n_slots = (int)S.db->entries.size();
            if (!S.slots && S.n_kf != n_slots) { set_error("slots == NULL searches every slot: n_kf must be %d", n_slots); return job_fail(batch, j, BORB_ERR_INVALID_ARG); }
            if (S.slots)
                for (int i = 0; i < S.n_kf; i++)
                    if (S.slots[i] < 0 || S.slots[i] >= n_slots || !S.db->entries[S.slots[i]].alive) { set_error("slot %d is not a live keyframe", S.slots[i]); return job_fail(batch, j, BORB_ERR_INVALID_ARG); }
        }
        for (int j = 0; j < n_jobs; j++) if (P[j].work) work.push_back(j);
        const int nw = (int)work.size();
        if (nw == 0) return BORB_OK;
        BORB_CUDA(cudaSetDevice(m->device));
        borb_status s = lk.sync();
        if (s != BORB_OK) return s;
        for (int j : work) {
            const SearchJob& S = J[j];
            Plan& p = P[j];
            if (!kfkf) p.f.stage(c);                                   // a host view is packed on the device like a resident frame
            p.o_sl = S.slots ? c.in(S.slots, (size_t)S.n_kf * 4) : 0;
        }
        const size_t o_jobs = c.in(nullptr, (size_t)nw * sizeof(BowDbJob));       // filled in place
        size_t hist_bytes = 0, tab_bytes = 0;
        for (int j : work) { hist_bytes += (size_t)J[j].n_kf * 32 * 4; tab_bytes += (size_t)J[j].n_kf * P[j].m * 4; }
        const size_t o_hist = c.scratch(hist_bytes), o_tab = c.scratch(tab_bytes);
        size_t hist_off = o_hist, tab_off = o_tab;
        int max_smem_frame = 0, max_nn = 0, total_kf = 0;
        long long max_items = 0;
        for (int j : work) {
            const SearchJob& S = J[j];
            Plan& p = P[j];
            p.h = frame_block_layout(p.nn, p.m, p.n);
            p.o_fb = c.scratch((size_t)p.h.bytes);
            p.o_ctr = c.scratch(16);
            p.o_hist = hist_off; hist_off += (size_t)S.n_kf * 32 * 4;
            p.o_tab = tab_off; tab_off += (size_t)S.n_kf * p.m * 4;
            p.o_dense = S.dense ? c.scratch((size_t)S.n_kf * p.n * 4) : 0;
            p.ho = c.result((size_t)S.n_kf * 8 + (S.pairs ? (size_t)S.pairs_cap * 4 : 0));
            if (bowdb_frame_fits_smem(p.h.bytes)) max_smem_frame = std::max(max_smem_frame, p.h.bytes);
            max_nn = std::max(max_nn, p.nn);
            max_items += (long long)std::min(p.nn, p.m) * S.n_kf;
            total_kf += S.n_kf;
        }
        if ((s = c.begin()) != BORB_OK) return s;
        BowDbJob* hj = c.host<BowDbJob>(o_jobs);
        int kf_base = 0;
        for (int w = 0; w < nw; w++) {
            const SearchJob& S = J[work[w]];
            const Plan& p = P[work[w]];
            BowDbJob D{};
            if (kfkf) {
                const KfStream& st = S.db->entries[S.query_slot].stream;
                D.fv_node = st.node; D.fv_start = st.start; D.q_meta = st.meta; D.desc = st.desc;
            } else {
                const KfDev f = p.f.bind(c);
                D.fv_node = f.node; D.fv_start = f.start; D.fv_idx = f.idx; D.keys = f.keys; D.desc = f.desc;
            }
            D.nn = p.nn; D.m = p.m; D.n = p.n; D.item_target = g_bow_item_target.load();
            D.frame_block = c.dev(p.o_fb); D.frame_bytes = p.h.bytes; D.frame_in_smem = bowdb_frame_fits_smem(p.h.bytes) ? 1 : 0;
            D.table = S.db->d_stream; D.slots = S.slots ? (const int32_t*)c.dev(p.o_sl) : nullptr;
            D.n_kf = S.n_kf; D.kf_base = kf_base; kf_base += S.n_kf;
            D.ctr = (int*)c.dev(p.o_ctr);
            D.table_out = (uint32_t*)c.dev(p.o_tab); D.hist_out = (int*)c.dev(p.o_hist);
            // counts, offsets and the compact pair list are written by the finalize kernel straight into the pinned landing buffer
            // (device-addressable, UVA) - no device-to-host copies; the dense table (MBs) still goes through one copy
            uint8_t* o = c.res(p.ho, true);
            D.n_matches = (int32_t*)o; D.pair_off = (int32_t*)(o + (size_t)S.n_kf * 4);
            D.pairs = S.pairs ? (uint32_t*)(o + (size_t)S.n_kf * 8) : nullptr; D.pairs_cap = S.pairs_cap;
            D.dense = S.dense ? (int32_t*)c.dev(p.o_dense) : nullptr; D.dense_stride = p.n;
            hj[w] = D;
        }
        if ((s = c.commit()) != BORB_OK) return s;
        BORB_CUDA(cudaMemsetAsync(c.dev(o_hist), 0, hist_bytes, m->stream));
        BORB_CUDA(cudaMemsetAsync(c.dev(o_tab), 0xFF, tab_bytes, m->stream));
        for (int j : work) {
            if (J[j].dense) BORB_CUDA(cudaMemsetAsync(c.dev(P[j].o_dense), 0xFF, (size_t)J[j].n_kf * P[j].n * 4, m->stream));
            if (J[j].frame && (s = c.wait(J[j].frame)) != BORB_OK) return s;
        }
        BowDbArgs A{};
        A.jobs = (const BowDbJob*)c.dev(o_jobs); A.n_jobs = nw; A.static_sched = g_bow_static.load();
        A.nnratio = nnratio; A.check_ori = check_ori;
        if (m->timing) BORB_CUDA(cudaEventRecord(m->t0, m->stream));
        m->launches += launch_bowdb(A, hj[0], max_smem_frame, max_items, total_kf, max_nn, g_bow_csa.load(), J[work[0]].db->n_sm, kfkf,
                                   m->stream);
        if (m->timing) BORB_CUDA(cudaEventRecord(m->t1, m->stream));
        for (int j : work)
            if (J[j].dense) BORB_CUDA(cudaMemcpyAsync(J[j].dense, c.dev(P[j].o_dense), (size_t)J[j].n_kf * P[j].n * 4, cudaMemcpyDeviceToHost, m->stream));
    }
    if (const borb_status s = c.finish(); s != BORB_OK) return s;
    if (m->timing) { float ms = 0.f; if (cudaEventElapsedTime(&ms, m->t0, m->t1) == cudaSuccess) m->last_ms = ms; else cudaGetLastError(); }
    int overflow = -1;
    long long over_total = 0;
    for (int j : work) {
        const SearchJob& S = J[j];
        const uint8_t* o = c.out(P[j].ho);
        std::memcpy(S.n_matches, o, (size_t)S.n_kf * 4);
        if (S.pair_offset) std::memcpy(S.pair_offset, o + (size_t)S.n_kf * 4, (size_t)S.n_kf * 4);
        if (!S.pairs) continue;
        long long total_pairs = 0;
        for (int i = 0; i < S.n_kf; i++) total_pairs += S.n_matches[i];
        if (S.n_pairs_total) *S.n_pairs_total = (int32_t)total_pairs;
        const long long ncopy = total_pairs < S.pairs_cap ? total_pairs : S.pairs_cap;
        if (ncopy > 0) std::memcpy(S.pairs, o + (size_t)S.n_kf * 8, (size_t)ncopy * 4);
        if (total_pairs > S.pairs_cap && overflow < 0) { overflow = j; over_total = total_pairs; }
    }
    if (overflow >= 0) {
        set_error("%lld matched pairs, capacity %d", over_total, J[overflow].pairs_cap);
        return job_fail(batch, overflow, BORB_ERR_CAPACITY);
    }
    return BORB_OK;
}

// the checks of the single database searches on their host view
borb_status check_db_view(borb_matcher* m, borb_kfdb* db, const borb_keyframe_view* frame) {
    if (m->device != db->device) { set_error("matcher and keyframe database live on different devices"); return BORB_ERR_INVALID_ARG; }
    return check_kf(frame, "SearchByBoW(database, frame)");
}

// the checks of a batch job's database, and of its resident frame unless it searches a database slot (f == NULL, kfkf)
borb_status check_db_job(borb_matcher* m, borb_kfdb* db, const borb_frame* f, int j, bool kfkf = false) {
    if (!db) { set_error("job %d: null database", j); return BORB_ERR_INVALID_ARG; }
    if (db->device != m->device) { set_error("job %d: database and matcher live on different devices", j); return BORB_ERR_INVALID_ARG; }
    return kfkf ? BORB_OK : check_resident_bow(f, m, j, "frame");
}

}  // namespace

borb_status borb_kfdb_query(borb_matcher* m, borb_kfdb* db, const uint32_t* bow_word, const double* bow_value, int n_bow,
                            int32_t* common_words, float* score, uint32_t* first_word, int cap, int32_t* n_slots) {
    if (!m || !db || !common_words || !score || !first_word || !n_slots || n_bow < 0 || (n_bow > 0 && (!bow_word || !bow_value))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (m->device != db->device) { set_error("matcher and keyframe database live on different devices"); return BORB_ERR_INVALID_ARG; }
    for (int i = 1; i < n_bow; i++)
        if (bow_word[i] <= bow_word[i - 1]) { set_error("BowVector words must ascend (std::map order)"); return BORB_ERR_INVALID_ARG; }
    const QueryJob q{db, nullptr, bow_word, bow_value, n_bow, common_words, score, first_word, cap, n_slots};
    return kfdb_query_jobs(m, &q, 1, false);
}

borb_status borb_kfdb_query_batch(borb_matcher* m, const borb_kfdb_query_job* jobs, int n_jobs) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && !jobs)) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (n_jobs == 0) return BORB_OK;
    std::vector<QueryJob> q(n_jobs);
    for (int j = 0; j < n_jobs; j++) {
        const borb_kfdb_query_job& B = jobs[j];
        borb_status s = check_db_job(m, B.db, B.frame, j);
        if (s != BORB_OK) return s;
        if (!B.common_words || !B.score || !B.first_word || !B.n_slots) { set_error("job %d: null output", j); return BORB_ERR_INVALID_ARG; }
        q[j] = QueryJob{B.db, B.frame, nullptr, nullptr, 0, B.common_words, B.score, B.first_word, B.cap, B.n_slots};
    }
    return kfdb_query_jobs(m, q.data(), n_jobs, true);
}

// The frames are checked first; the slots are resolved to their BowVectors under the databases' locks, which are held until the
// kernel is enqueued (a concurrent erase synchronises the device before it frees a block).
borb_status borb_bow_score_batch(borb_matcher* m, const borb_bow_score_job* jobs, int n_jobs) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && !jobs)) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (n_jobs == 0) return BORB_OK;
    std::vector<borb_kfdb*> dbs;
    auto check_ref = [&](const borb_bow_ref& r, int j, int ref) {
        if (r.frame) return check_resident_bow(r.frame, m, j, "frame", ref);
        if (!r.db) { set_error("%s: neither a frame nor a database", job_at(j, ref).c_str()); return BORB_ERR_INVALID_ARG; }
        if (r.db->device != m->device) { set_error("%s: database and matcher live on different devices", job_at(j, ref).c_str()); return BORB_ERR_INVALID_ARG; }
        dbs.push_back(r.db);
        return BORB_OK;
    };
    for (int j = 0; j < n_jobs; j++) {
        const borb_bow_score_job& B = jobs[j];
        if (B.n_targets < 0) { set_error("job %d: n_targets %d < 0", j, B.n_targets); return BORB_ERR_INVALID_ARG; }
        if (B.n_targets > 0 && (!B.targets || !B.score)) { set_error("job %d: null targets or score", j); return BORB_ERR_INVALID_ARG; }
        borb_status s = check_ref(B.query, j, QUERY_REF);
        for (int t = 0; t < B.n_targets && s == BORB_OK; t++) s = check_ref(B.targets[t], j, t);
        if (s != BORB_OK) return s;
    }
    DbLocks lk(std::move(dbs));
    std::vector<BowTable> T(n_jobs);
    auto resolve = [&](const borb_bow_ref& r, int j, int ref, BowTable& tab, BowDev& out) {
        if (r.frame) {
            out = BowDev{r.frame->bow_word, r.frame->bow_value, r.frame->n_bow};
            tab.frames.push_back(r.frame);
            return BORB_OK;
        }
        if (r.slot < 0 || r.slot >= (int)r.db->entries.size() || !r.db->entries[r.slot].alive) {
            set_error("%s: slot %d is not a live keyframe", job_at(j, ref).c_str(), r.slot);
            return BORB_ERR_INVALID_ARG;
        }
        out = r.db->entries[r.slot].bow;
        return BORB_OK;
    };
    std::vector<QueryJob> q(n_jobs);
    for (int j = 0; j < n_jobs; j++) {
        const borb_bow_score_job& B = jobs[j];
        BowTable& tab = T[j];
        tab.targets.resize(B.n_targets);
        borb_status s = resolve(B.query, j, QUERY_REF, tab, tab.query);
        for (int t = 0; t < B.n_targets && s == BORB_OK; t++) s = resolve(B.targets[t], j, t, tab, tab.targets[t]);
        if (s != BORB_OK) return s;
        std::sort(tab.frames.begin(), tab.frames.end());
        tab.frames.erase(std::unique(tab.frames.begin(), tab.frames.end()), tab.frames.end());
        q[j] = QueryJob{nullptr, nullptr, nullptr, nullptr, 0, nullptr, B.score, nullptr, B.n_targets, nullptr, &tab};
    }
    return kfdb_query_jobs(m, q.data(), n_jobs, true, &lk);
}

// Every job's block is allocated and written by one launch of kfdb_insert_kernel before any database is locked; the slots are
// appended in job order under the locks once the blocks are complete, so no search ever sees a partial block.
borb_status borb_kfdb_add_frames(borb_matcher* m, const borb_kfdb_add_job* jobs, int n_jobs) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && !jobs)) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (n_jobs == 0) return BORB_OK;
    for (int j = 0; j < n_jobs; j++) {
        const borb_kfdb_add_job& B = jobs[j];
        const borb_status s = check_db_job(m, B.db, B.frame, j);
        if (s != BORB_OK) return s;
        if (!B.slot_out) { set_error("job %d: null slot_out", j); return BORB_ERR_INVALID_ARG; }
    }
    BORB_CUDA(cudaSetDevice(m->device));
    std::vector<uint8_t*> blocks(n_jobs, nullptr);
    auto fail = [&](borb_status s) { for (uint8_t* b : blocks) cudaFree(b); return s; };
    Call c(m);
    std::vector<size_t> o_hm(n_jobs, 0), r_meta(n_jobs, 0);
    for (int j = 0; j < n_jobs; j++)
        if (jobs[j].has_mp && jobs[j].frame->n > 0) o_hm[j] = c.in(jobs[j].has_mp, (size_t)jobs[j].frame->n);
    const size_t o_jobs = c.in(nullptr, (size_t)n_jobs * sizeof(KfdbInsertJob));     // filled in place
    for (int j = 0; j < n_jobs; j++) r_meta[j] = c.result((size_t)jobs[j].frame->n_fv * 8);
    for (int j = 0; j < n_jobs; j++) {
        const borb_frame* f = jobs[j].frame;
        const cudaError_t e = cudaMalloc(&blocks[j], kfdb_block_layout(f->n_nodes, f->n_fv, f->n_bow).bytes);
        if (e != cudaSuccess) { blocks[j] = nullptr; set_error("job %d: keyframe block allocation failed: %s", j, cudaGetErrorString(e)); return fail(BORB_ERR_CUDA); }
        if (poison_byte() >= 0)                          // borb_debug_set_poison, ahead of kfdb_insert_kernel on the same stream
            BORB_CUDA(cudaMemsetAsync(blocks[j], poison_byte(), kfdb_block_layout(f->n_nodes, f->n_fv, f->n_bow).bytes, m->stream));
    }
    borb_status s;
    if ((s = c.begin()) != BORB_OK) return fail(s);
    KfdbInsertJob* hj = c.host<KfdbInsertJob>(o_jobs);
    for (int j = 0; j < n_jobs; j++) {
        const borb_frame* f = jobs[j].frame;
        KfdbInsertJob J{};
        J.fv_node = f->fv_node; J.fv_start = f->fv_start; J.fv_idx = f->fv_idx; J.keys = f->keys; J.desc = f->desc;
        J.bow_word = f->bow_word; J.bow_value = f->bow_value;
        J.has_mp = (jobs[j].has_mp && f->n > 0) ? c.dev(o_hm[j]) : nullptr;
        J.nn = f->n_nodes; J.m = f->n_fv; J.n_bow = f->n_bow;
        J.block = blocks[j];
        // the row records for the host copies are written by the kernel straight into the pinned landing buffer (UVA)
        J.meta_out = f->n_fv > 0 ? reinterpret_cast<uint2*>(c.res(r_meta[j], true)) : nullptr;
        hj[j] = J;
    }
    if ((s = c.commit()) != BORB_OK) return fail(s);
    for (int j = 0; j < n_jobs; j++)
        if ((s = c.wait(jobs[j].frame)) != BORB_OK) return fail(s);
    m->launches += launch_kfdb_insert((const KfdbInsertJob*)c.dev(o_jobs), n_jobs, m->stream);
    if ((s = c.finish()) != BORB_OK) return fail(s);
    std::vector<borb_kfdb*> dbs(n_jobs);
    for (int j = 0; j < n_jobs; j++) dbs[j] = jobs[j].db;
    DbLocks lk(std::move(dbs));
    for (int j = 0; j < n_jobs; j++) {
        const borb_frame* f = jobs[j].frame;
        *jobs[j].slot_out = kfdb_append_locked(jobs[j].db, blocks[j], f->n_nodes, f->n_fv, f->n, f->n_bow,
                                               reinterpret_cast<const uint32_t*>(c.out(r_meta[j])));
    }
    return BORB_OK;
}

borb_status borb_debug_kfdb_read(borb_kfdb* db, int32_t slot, int32_t* counts4, uint64_t* block_bytes, uint32_t* node, int32_t* start,
                                 uint32_t* meta, uint8_t* desc, uint32_t* bow_word, double* bow_value, uint32_t* host_meta, uint8_t* block) {
    if (!db) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    std::lock_guard<std::mutex> lk(db->mu);
    if (slot < 0 || slot >= (int)db->entries.size() || !db->entries[slot].alive) { set_error("bad keyframe slot"); return BORB_ERR_INVALID_ARG; }
    const borb_kfdb::Entry& e = db->entries[slot];
    const int nn = e.stream.nn, m = e.stream.m, nb = e.bow.n;
    const KfdbBlock L = kfdb_block_layout(nn, m, nb);
    if (counts4) { counts4[0] = nn; counts4[1] = m; counts4[2] = e.n; counts4[3] = nb; }
    if (block_bytes) *block_bytes = L.bytes;
    BORB_CUDA(cudaSetDevice(db->device));
    auto get = [&](void* dst, size_t off, size_t bytes) -> borb_status {
        if (dst && bytes) BORB_CUDA(cudaMemcpy(dst, e.block + off, bytes, cudaMemcpyDeviceToHost));
        return BORB_OK;
    };
    borb_status s;
    if ((s = get(node, L.node, (size_t)nn * 4)) != BORB_OK || (s = get(start, L.start, (size_t)(nn + 1) * 4)) != BORB_OK ||
        (s = get(meta, L.meta, (size_t)m * 8)) != BORB_OK || (s = get(desc, L.desc, (size_t)m * 32)) != BORB_OK ||
        (s = get(bow_word, L.bow_word, (size_t)nb * 4)) != BORB_OK || (s = get(bow_value, L.bow_value, (size_t)nb * 8)) != BORB_OK ||
        (s = get(block, 0, L.bytes)) != BORB_OK)
        return s;
    if (host_meta && m > 0) std::memcpy(host_meta, e.meta.data(), (size_t)m * 8);
    return BORB_OK;
}

borb_status borb_search_by_bow_db(borb_matcher* m, borb_kfdb* db, const int32_t* slots, int n_kf, const borb_keyframe_view* frame,
                                  float nnratio, int check_orientation, int32_t* match, int32_t* n_matches) {
    if (!m || !db || !frame || !match || !n_matches || n_kf < 0) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_status s = check_db_view(m, db, frame);
    if (s != BORB_OK) return s;
    const SearchJob J{db, nullptr, frame, slots, n_kf, match, n_matches, nullptr, nullptr, 0, nullptr};
    return bowdb_jobs(m, &J, 1, nnratio, check_orientation, false);
}

borb_status borb_search_by_bow_db_pairs(borb_matcher* m, borb_kfdb* db, const int32_t* slots, int n_kf, const borb_keyframe_view* frame,
                                        float nnratio, int check_orientation, int32_t* n_matches, int32_t* pair_offset, uint32_t* pairs,
                                        int pairs_cap, int32_t* n_pairs_total) {
    if (!m || !db || !frame || !n_matches || n_kf < 0 || pairs_cap < 0 || (pairs && !pair_offset)) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_status s = check_db_view(m, db, frame);
    if (s != BORB_OK) return s;
    const SearchJob J{db, nullptr, frame, slots, n_kf, nullptr, n_matches, pair_offset, pairs, pairs_cap, n_pairs_total};
    return bowdb_jobs(m, &J, 1, nnratio, check_orientation, false);
}

borb_status borb_search_by_bow_db_batch(borb_matcher* m, const borb_bow_db_job* jobs, int n_jobs, float nnratio, int check_orientation) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && !jobs)) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (n_jobs == 0) return BORB_OK;
    std::vector<SearchJob> S(n_jobs);
    for (int j = 0; j < n_jobs; j++) {
        const borb_bow_db_job& B = jobs[j];
        borb_status s = check_db_job(m, B.db, B.frame, j);
        if (s != BORB_OK) return s;
        if (B.n_kf < 0 || B.pairs_cap < 0 || (B.n_kf > 0 && !B.n_matches)) { set_error("job %d: null output or negative count", j); return BORB_ERR_INVALID_ARG; }
        if (B.pairs && !B.pair_offset) { set_error("job %d: pairs without pair_offset", j); return BORB_ERR_INVALID_ARG; }
        S[j] = SearchJob{B.db, B.frame, nullptr, B.slots, B.n_kf, nullptr, B.n_matches, B.pair_offset, B.pairs, B.pairs_cap, B.n_pairs_total};
    }
    return bowdb_jobs(m, S.data(), n_jobs, nnratio, check_orientation, true);
}

borb_status borb_search_by_bow_kf_db_batch(borb_matcher* m, const borb_bow_kf_db_job* jobs, int n_jobs, float nnratio, int check_orientation) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && !jobs)) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (n_jobs == 0) return BORB_OK;
    std::vector<SearchJob> S(n_jobs);
    for (int j = 0; j < n_jobs; j++) {
        const borb_bow_kf_db_job& B = jobs[j];
        borb_status s = check_db_job(m, B.db, nullptr, j, true);
        if (s != BORB_OK) return s;
        if (B.n_kf < 0 || B.pairs_cap < 0 || (B.n_kf > 0 && !B.n_matches)) { set_error("job %d: null output or negative count", j); return BORB_ERR_INVALID_ARG; }
        if (B.pairs && !B.pair_offset) { set_error("job %d: pairs without pair_offset", j); return BORB_ERR_INVALID_ARG; }
        S[j] = SearchJob{B.db, nullptr, nullptr, B.slots, B.n_kf, nullptr, B.n_matches, B.pair_offset, B.pairs, B.pairs_cap, B.n_pairs_total,
                         B.query_slot};
    }
    return bowdb_jobs(m, S.data(), n_jobs, nnratio, check_orientation, true, true);
}

borb_status borb_search_by_bow_kf_db_pairs(borb_matcher* m, borb_kfdb* db, int32_t query_slot, const int32_t* slots, int n_kf, float nnratio,
                                           int check_orientation, int32_t* n_matches, int32_t* pair_offset, uint32_t* pairs, int pairs_cap,
                                           int32_t* n_pairs_total) {
    const borb_bow_kf_db_job J{db, query_slot, slots, n_kf, n_matches, pair_offset, pairs, pairs_cap, n_pairs_total};
    return borb_search_by_bow_kf_db_batch(m, &J, 1, nnratio, check_orientation);
}

// ---- SearchForTriangulation: borb_search_for_triangulation is the one-job case of borb_search_for_triangulation_batch (one launch
// of triangulation_kernel, a CTA per job, and one synchronisation).  Each side is a host view or a resident frame with its BoW.
namespace {
borb_status triangulation_jobs(borb_matcher* m, const borb_triangulation_job* jobs, int n_jobs, int check_ori, bool batch) {
    struct Job { KfSide s1, s2; bool live; int cap; size_t vm, bins, res; };
    std::vector<Job> J(n_jobs);
    for (int j = 0; j < n_jobs; j++) {
        const borb_triangulation_job& B = jobs[j];
        if (!B.pairs || !B.n_pairs || B.cap < 0) { set_error("job %d: null output or negative capacity", j); return BORB_ERR_INVALID_ARG; }
        borb_status s = BORB_OK;
        if (B.kf1_frame) s = check_resident_bow(B.kf1_frame, m, j, "kf1_frame");
        else if ((s = check_kf(&B.kf1, batch ? "kf1" : "borb_search_for_triangulation(kf1)")) != BORB_OK) return job_fail(batch, j, s);
        if (s != BORB_OK) return s;
        if (B.kf2_frame) s = check_resident_bow(B.kf2_frame, m, j, "kf2_frame");
        else if ((s = check_kf(&B.kf2, batch ? "kf2" : "borb_search_for_triangulation(kf2)")) != BORB_OK) return job_fail(batch, j, s);
        if (s != BORB_OK) return s;
        if (!B.kf2.level_sigma2 || (!B.kf2_frame && !B.kf2.scale_factors)) {
            set_error("kf2 needs scale_factors and level_sigma2");
            return job_fail(batch, j, BORB_ERR_INVALID_ARG);
        }
        Job& Q = J[j];
        Q.s1 = KfSide{&B.kf1, B.kf1_frame};
        Q.s2 = KfSide{&B.kf2, B.kf2_frame};
        Q.live = Q.s1.n() > 0 && Q.s1.nn() > 0 && Q.s2.n() > 0 && Q.s2.nn() > 0;
        Q.cap = std::min(B.cap, Q.s1.n());           // a job has at most one pair per kf1 feature
    }
    for (int j = 0; j < n_jobs; j++) *jobs[j].n_pairs = 0;      // every job passed its checks
    std::vector<int> live;
    for (int j = 0; j < n_jobs; j++) if (J[j].live) live.push_back(j);
    const int nl = (int)live.size();
    if (nl == 0) return BORB_OK;
    Call c(m);
    for (int j : live) {
        J[j].s1.stage(c);
        J[j].s2.stage(c);
    }
    const size_t o_jobs = c.in(nullptr, (size_t)nl * sizeof(TriJob));          // filled in place
    const size_t r_cnt = c.result((size_t)nl * 4);       // n_pairs of every live job, then every job's pairs
    for (int j : live) {
        Job& Q = J[j];
        Q.vm = c.scratch((size_t)Q.s1.n() * 4); Q.bins = c.scratch((size_t)Q.s1.n());
        Q.res = c.result((size_t)Q.cap * 8);
    }
    borb_status s;
    if ((s = c.begin()) != BORB_OK) return s;
    TriJob* hj = c.host<TriJob>(o_jobs);
    for (int k = 0; k < nl; k++) {
        const borb_triangulation_job& B = jobs[live[k]];
        const Job& Q = J[live[k]];
        TriJob T{};
        T.q = Q.s1.bind(c);
        T.t = Q.s2.bind(c);
        for (int i = 0; i < 9; i++) T.F[i] = B.F12[i];
        T.ex = B.ex; T.ey = B.ey; T.only_stereo = B.only_stereo;
        T.vmatch = (int32_t*)c.dev(Q.vm); T.bins = c.dev(Q.bins);
        T.pairs = (int32_t*)c.res(Q.res, false); T.cap = Q.cap; T.n_pairs = (int32_t*)c.res(r_cnt, false) + k;
        hj[k] = T;
    }
    if ((s = c.commit()) != BORB_OK) return s;
    for (int j : live) {
        if (jobs[j].kf1_frame && (s = c.wait(jobs[j].kf1_frame)) != BORB_OK) return s;
        if (jobs[j].kf2_frame && (s = c.wait(jobs[j].kf2_frame)) != BORB_OK) return s;
    }
    m->launches += launch_triangulation((const TriJob*)c.dev(o_jobs), nl, check_ori, m->stream);
    if ((s = c.finish()) != BORB_OK) return s;
    int overflow = -1;
    for (int k = 0; k < nl; k++) {
        const borb_triangulation_job& B = jobs[live[k]];
        std::memcpy(B.n_pairs, c.out(r_cnt) + (size_t)k * 4, 4);
        const int np = std::min(*B.n_pairs, B.cap);
        if (np > 0) std::memcpy(B.pairs, c.out(J[live[k]].res), (size_t)np * 8);
        if (*B.n_pairs > B.cap && overflow < 0) overflow = live[k];
    }
    if (overflow >= 0) {
        set_error("%d pairs, capacity %d", *jobs[overflow].n_pairs, jobs[overflow].cap);
        return job_fail(batch, overflow, BORB_ERR_CAPACITY);
    }
    return BORB_OK;
}
}  // namespace

borb_status borb_search_for_triangulation(borb_matcher* m, const borb_keyframe_view* kf1, const borb_keyframe_view* kf2, const float* F12,
                                          float ex, float ey, int only_stereo, int check_orientation, int32_t* pairs, int cap,
                                          int32_t* n_pairs) {
    if (!m || !kf1 || !kf2 || !F12 || !pairs || !n_pairs || cap < 0) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_triangulation_job B{};
    B.kf1 = *kf1; B.kf2 = *kf2;
    std::memcpy(B.F12, F12, sizeof(B.F12));
    B.ex = ex; B.ey = ey; B.only_stereo = only_stereo; B.pairs = pairs; B.cap = cap; B.n_pairs = n_pairs;
    return triangulation_jobs(m, &B, 1, check_orientation, false);
}

borb_status borb_search_for_triangulation_batch(borb_matcher* m, const borb_triangulation_job* jobs, int n_jobs, int check_orientation) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && !jobs)) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    return triangulation_jobs(m, jobs, n_jobs, check_orientation, true);
}

// ------------------------------------------------------------------------------------------------ vocabulary
borb_status borb_voc_create(const int32_t* parent, const uint8_t* is_leaf, const uint8_t* desc, const double* weight, int n_nodes, int k,
                            int L, int device, borb_voc** out) {
    if (!parent || !is_leaf || !desc || !weight || !out || n_nodes < 2) { set_error("bad vocabulary arrays"); return BORB_ERR_INVALID_ARG; }
    *out = nullptr;
    for (int i = 1; i < n_nodes; i++)
        if (parent[i] < 0 || parent[i] >= i) { set_error("node %d: parent %d must precede it", i, parent[i]); return BORB_ERR_INVALID_ARG; }
    int ndev = 0;
    borb_status s = borb_device_count(&ndev);
    if (s != BORB_OK) return s;
    if (device < 0 || device >= ndev) { set_error("device %d out of range", device); return ndev < 1 ? BORB_ERR_NO_DEVICE : BORB_ERR_INVALID_ARG; }
    // children in order of appearance; word ids in order of leaf appearance (loadFromTextFile :1378-1420)
    std::vector<int32_t> cstart(n_nodes + 1, 0), cids(n_nodes > 1 ? n_nodes - 1 : 0), word(n_nodes, -1);
    for (int i = 1; i < n_nodes; i++) cstart[parent[i] + 1]++;
    for (int i = 0; i < n_nodes; i++)                  // the descent packs a child's rank into 23 bits (bow_descend, k_match.cu)
        if (cstart[i + 1] >= (1 << 23)) { set_error("node %d: %d children, limit %d", i, cstart[i + 1], (1 << 23) - 1); return BORB_ERR_INVALID_ARG; }
    for (int i = 0; i < n_nodes; i++) cstart[i + 1] += cstart[i];
    std::vector<int32_t> fill(cstart.begin(), cstart.end() - 1);
    for (int i = 1; i < n_nodes; i++) cids[fill[parent[i]]++] = i;
    int nw = 0;
    for (int i = 1; i < n_nodes; i++) if (is_leaf[i]) word[i] = nw++;
    VocHeader h{};
    h.magic = VOC_MAGIC; h.n_nodes = n_nodes; h.k = k; h.L = L;
    size_t off = 256;
    auto sec = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) & ~size_t(255); return o; };
    h.off_desc = sec((size_t)n_nodes * 32); h.off_weight = sec((size_t)n_nodes * 8); h.off_word = sec((size_t)n_nodes * 4);
    h.off_cstart = sec((size_t)(n_nodes + 1) * 4); h.off_cids = sec((size_t)(n_nodes > 1 ? n_nodes - 1 : 1) * 4);
    h.bytes = off;
    std::vector<uint8_t> host(off, 0);
    std::memcpy(host.data(), &h, sizeof(h));
    std::memcpy(host.data() + h.off_desc, desc, (size_t)n_nodes * 32);
    std::memcpy(host.data() + h.off_weight, weight, (size_t)n_nodes * 8);
    std::memcpy(host.data() + h.off_word, word.data(), (size_t)n_nodes * 4);
    std::memcpy(host.data() + h.off_cstart, cstart.data(), (size_t)(n_nodes + 1) * 4);
    if (n_nodes > 1) std::memcpy(host.data() + h.off_cids, cids.data(), (size_t)(n_nodes - 1) * 4);
    borb_voc* v = new borb_voc();
    v->device = device; v->bytes = off;
    cudaError_t e = cudaSetDevice(device);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&v->stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMalloc(&v->blob, off);
    if (e == cudaSuccess) e = cudaMemcpy(v->blob, host.data(), off, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { set_error("vocabulary upload failed: %s", cudaGetErrorString(e)); cudaFree(v->blob); delete v; return BORB_ERR_CUDA; }
    voc_views(v, h);
    *out = v;
    return BORB_OK;
}

borb_status borb_voc_load_text(const char* path, int device, borb_voc** out) {
    if (!path || !out) return BORB_ERR_INVALID_ARG;
    FILE* f = std::fopen(path, "r");
    if (!f) { set_error("cannot open %s", path); return BORB_ERR_INVALID_ARG; }
    std::vector<char> line(1 << 16);
    int k = -1, L = -1, n1 = -1, n2 = -1;
    if (!std::fgets(line.data(), (int)line.size(), f) || std::sscanf(line.data(), "%d %d %d %d", &k, &L, &n1, &n2) != 4 || k < 0 || k > 20 ||
        L < 1 || L > 10 || n1 < 0 || n1 > 5 || n2 < 0 || n2 > 3) {
        std::fclose(f);
        set_error("%s is not a vocabulary text file", path);
        return BORB_ERR_INVALID_ARG;
    }
    std::vector<int32_t> parent(1, 0);
    std::vector<uint8_t> leaf(1, 0), desc(32, 0);
    std::vector<double> weight(1, 0.0);
    while (std::fgets(line.data(), (int)line.size(), f)) {
        char* p = line.data();
        char* end = nullptr;
        const long pid = std::strtol(p, &end, 10);
        if (end == p) continue;     // blank line (the reference's eof loop turns a trailing blank line into a garbage node)
        p = end;
        const long isLeaf = std::strtol(p, &end, 10); p = end;
        uint8_t d[32];
        for (int i = 0; i < 32; i++) { d[i] = (uint8_t)std::strtol(p, &end, 10); p = end; }
        const double w = std::strtod(p, &end);
        parent.push_back((int32_t)pid); leaf.push_back(isLeaf > 0); weight.push_back(w);
        desc.insert(desc.end(), d, d + 32);
    }
    std::fclose(f);
    return borb_voc_create(parent.data(), leaf.data(), desc.data(), weight.data(), (int)parent.size(), k, L, device, out);
}

borb_status borb_voc_destroy(borb_voc* v) {
    if (!v) return BORB_OK;
    free_call_buffers(*v);
    if (v->owns) cudaFree(v->blob);
    delete v;
    return BORB_OK;
}

borb_status borb_voc_blob(const borb_voc* v, void** d_blob, size_t* bytes) {
    if (!v || !d_blob || !bytes) return BORB_ERR_INVALID_ARG;
    *d_blob = v->blob; *bytes = v->bytes;
    return BORB_OK;
}

borb_status borb_voc_from_blob(void* d_blob, size_t bytes, int device, borb_voc** out) {
    if (!d_blob || !out || bytes < sizeof(VocHeader)) return BORB_ERR_INVALID_ARG;
    *out = nullptr;
    BORB_CUDA(cudaSetDevice(device));
    VocHeader h;
    BORB_CUDA(cudaMemcpy(&h, d_blob, sizeof(h), cudaMemcpyDeviceToHost));
    if (h.magic != VOC_MAGIC || h.bytes != bytes) { set_error("not a packed vocabulary blob"); return BORB_ERR_INVALID_ARG; }
    borb_voc* v = new borb_voc();
    v->device = device; v->owns = false; v->blob = (uint8_t*)d_blob; v->bytes = bytes;
    cudaError_t e = cudaStreamCreateWithFlags(&v->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) { set_error("stream: %s", cudaGetErrorString(e)); delete v; return BORB_ERR_CUDA; }
    voc_views(v, h);
    *out = v;
    return BORB_OK;
}

// internal: the vocabulary takes ownership of a blob it adopted (receiver side of borb_voc_broadcast)
extern "C" void borb_voc_adopt_ownership(borb_voc* v) { if (v) v->owns = true; }

borb_status borb_bow_transform(borb_voc* v, const uint8_t* desc, int n, int levelsup, int32_t* word, double* weight, int32_t* node) {
    if (!v || n < 0 || (n > 0 && (!desc || !word || !weight || !node))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (n == 0) return BORB_OK;
    BowSide b;
    b.desc = desc; b.n = n; b.word = word; b.weight = weight; b.node = node;
    // Tracking (Frame::ComputeBoW) and LocalMapping (KeyFrame::ComputeBoW) transform on one vocabulary, as DBoW2's const transform
    // allows: one call at a time owns its buffers, from the staging to the copy out
    std::lock_guard<std::mutex> lk(v->mu);
    return bow_jobs(v, v->dev, &b, 1, levelsup, true, nullptr);
}

// Frame::ComputeBoW / KeyFrame::ComputeBoW (src/Frame.cc:395-402, src/KeyFrame.cc:59-68): the one-frame case of
// borb_frames_compute_bow on the caller's host descriptors, under the vocabulary's lock.
borb_status borb_compute_bow(borb_voc* v, const uint8_t* desc, int n, int levelsup, uint32_t* bow_word, double* bow_value, int32_t* n_bow,
                             uint32_t* fv_node, int32_t* fv_start, uint32_t* fv_idx, int32_t* n_nodes) {
    if (!v || n < 0 || !n_bow || !n_nodes || (n > 0 && (!desc || !bow_word || !bow_value || !fv_node || !fv_start || !fv_idx))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    *n_bow = 0; *n_nodes = 0;
    if (fv_start) fv_start[0] = 0;
    // bow_build_kernel keeps 16 B of shared memory per key slot, the next power of two >= n: 8192 features is the most a block can hold
    if (n > MATCH_MAX_FEATURES) { set_error("%d features (limit %d)", n, MATCH_MAX_FEATURES); return BORB_ERR_INVALID_ARG; }
    if (n == 0) return BORB_OK;
    BowSide b;
    b.desc = desc; b.n = n; b.out = BowTables{bow_word, bow_value, fv_node, fv_start, fv_idx}; b.n_bow = n_bow; b.n_nodes = n_nodes;
    std::lock_guard<std::mutex> lk(v->mu);
    return bow_jobs(v, v->dev, &b, 1, levelsup, false, nullptr);
}

// Frame::ComputeBoW for many resident frames: the tree descent and the ordered-map bookkeeping of TemplatedVocabulary::transform
// (TemplatedVocabulary.h:1150-1194) both on the device (bow_transform_batch_kernel, bow_build_kernel), two launches and one
// synchronisation; the vectors stay with the frames for borb_search_by_bow_batch.  Of the vocabulary it reads only the immutable
// blob (v->dev), on the matcher's buffers and stream, so it takes no vocabulary lock.
borb_status borb_frames_compute_bow(borb_matcher* m, borb_voc* v, borb_frame* const* frames, int n_frames, int levelsup,
                                    uint32_t* const* bow_word, double* const* bow_value, int32_t* n_bow, uint32_t* const* fv_node,
                                    int32_t* const* fv_start, uint32_t* const* fv_idx, int32_t* n_nodes) {
    if (!m || !v || n_frames < 0 || (n_frames > 0 && !frames)) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (n_frames == 0) return BORB_OK;
    if (v->device != m->device) { set_error("vocabulary and matcher live on different devices"); return BORB_ERR_INVALID_ARG; }
    std::vector<BowSide> S(n_frames);
    for (int i = 0; i < n_frames; i++) {
        borb_frame* f = frames[i];
        if (!f) { set_error("frame %d: not a device-resident frame", i); return BORB_ERR_INVALID_ARG; }
        if (f->device != m->device) { set_error("frame %d: frame and matcher live on different devices", i); return BORB_ERR_INVALID_ARG; }
        if (f->n < 0 || f->n > MATCH_MAX_FEATURES) { set_error("frame %d: %d features (limit %d)", i, f->n, MATCH_MAX_FEATURES); return BORB_ERR_INVALID_ARG; }
        S[i].f = f; S[i].n = f->n;
        S[i].out = BowTables{bow_word ? bow_word[i] : nullptr, bow_value ? bow_value[i] : nullptr, fv_node ? fv_node[i] : nullptr,
                             fv_start ? fv_start[i] : nullptr, fv_idx ? fv_idx[i] : nullptr};
        S[i].n_bow = n_bow ? n_bow + i : nullptr;
        S[i].n_nodes = n_nodes ? n_nodes + i : nullptr;
    }
    return bow_jobs(m, v->dev, S.data(), n_frames, levelsup, false, &m->launches);
}

// Device time (CUDA events on the matcher's stream) of the kernels of the last database search on this handle, for bench.py's roofline.
borb_status borb_matcher_set_timing(borb_matcher* m, int enable) {
    if (!m) return BORB_ERR_INVALID_ARG;
    BORB_CUDA(cudaSetDevice(m->device));
    if (enable && !m->t0) { BORB_CUDA(cudaEventCreate(&m->t0)); BORB_CUDA(cudaEventCreate(&m->t1)); }
    m->timing = enable != 0;
    m->last_ms = 0.f;
    return BORB_OK;
}
borb_status borb_matcher_last_kernel_ms(borb_matcher* m, float* ms) {
    if (!m || !ms) return BORB_ERR_INVALID_ARG;
    *ms = m->last_ms;
    return BORB_OK;
}
borb_status borb_matcher_launch_count(const borb_matcher* m, uint64_t* n) {
    if (!m || !n) return BORB_ERR_INVALID_ARG;
    *n = m->launches;
    return BORB_OK;
}

}  // extern "C"
