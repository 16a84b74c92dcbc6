// Host side of the matcher / vocabulary entry points of the C ABI (include/borb.h): snapshots arrive as plain host
// arrays, are staged into one device arena per call, and every result is produced by the CUDA kernels in k_match.cu.
#include <algorithm>
#include <atomic>
#include <cassert>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>

#include "borb_match.h"

using namespace borb;

struct borb_matcher {
    int device = 0;
    cudaStream_t stream = nullptr;
    uint8_t* arena = nullptr;       // device scratch, grow-only
    size_t arena_bytes = 0, arena_off = 0;
    uint8_t* h_stage = nullptr;     // pinned staging mirror of the arena's input part
    size_t h_bytes = 0;
    uint64_t launches = 0;
    int32_t* aux = nullptr;         // small device buffer that survives an arena re-layout (SearchBySim3: first direction's matches)
    size_t aux_count = 0;
    uint8_t* h_out = nullptr;       // pinned landing buffer for results (one D2H per call)
    size_t h_out_bytes = 0;
    std::vector<int32_t> sel;       // indices of the valid queries of the current call
    cudaEvent_t ev_a = nullptr, ev_b = nullptr;   // cross-stream ordering with an extractor handle (borb_frames_from_extractor)
    bool timing = false;            // borb_matcher_set_timing: CUDA events around the kernels of the database search
    cudaEvent_t t0 = nullptr, t1 = nullptr;
    float last_ms = 0.f;
};

struct borb_voc {
    int device = 0;
    bool owns = true;
    uint8_t* blob = nullptr;        // device
    size_t bytes = 0;
    VocDev dev;
    cudaStream_t stream = nullptr;
    uint8_t* scratch = nullptr;     // pinned HOST buffer of borb_bow_transform: descriptors in, (weight, word, node) out - the kernel reads
    size_t scratch_bytes = 0;       // and writes it in place (UVA), so a call is one launch and one synchronize.  One caller at a time per handle.
};

namespace {

constexpr size_t ZERO_COPY_MAX = 96 * 1024;       // inputs up to this size may be read in place by the kernels (each byte is read once)

// One matcher call on m->stream.  Its layout comes first, as offsets: staged inputs, then device-only scratch, then result slots.
// begin() grows the buffers, after which addresses exist; commit() moves the inputs with one H2D copy and finish() brings the result
// region back with one D2H copy and synchronises.  Kernels read the inputs from the arena or, for a small in-place call, from the
// pinned staging buffer itself (device-addressable, UVA: no H2D copy and no DMA latency).  They write results to the arena, or
// straight into the pinned landing buffer.
class Call {
public:
    explicit Call(borb_matcher* m) : m_(m) {}
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
        BORB_CUDA(cudaSetDevice(m_->device));
        borb_status s;
        if ((s = grow_device(m_->arena, m_->arena_bytes, off_)) != BORB_OK) return s;
        if ((s = grow_pinned(m_->h_stage, m_->h_bytes, in_end_)) != BORB_OK) return s;
        if (res_bytes_ && (s = grow_pinned(m_->h_out, m_->h_out_bytes, res_bytes_ + 4096)) != BORB_OK) return s;
        BORB_CUDA(cudaStreamSynchronize(m_->stream));   // the staging buffer may still feed an earlier copy
        for (const Item& it : items_)
            if (it.src) std::memcpy(m_->h_stage + it.off, it.src, it.bytes);
        begun_ = true;
        return BORB_OK;
    }
    bool in_place() const { return in_place_; }
    // the staging copy of an input
    template <class T> T* host(size_t off) const { assert(begun_ && off < in_end_); return reinterpret_cast<T*>(m_->h_stage + off); }
    // where kernels read an input or use scratch
    uint8_t* dev(size_t off) const { assert(begun_); return (in_place_ && off < in_end_ ? m_->h_stage : m_->arena) + off; }
    // where kernels write a result: the arena (brought back by finish()), or direct: the landing buffer
    uint8_t* res(size_t off, bool direct) {
        assert(begun_);
        download_ |= !direct;
        return (direct ? m_->h_out : m_->arena + res_off_) + off;
    }
    borb_status commit() {
        assert(begun_);
        if (in_end_ && !in_place_) BORB_CUDA(cudaMemcpyAsync(m_->arena, m_->h_stage, in_end_, cudaMemcpyHostToDevice, m_->stream));
        return BORB_OK;
    }
    borb_status wait(const borb_frame* f) const {
        BORB_CUDA(cudaStreamWaitEvent(m_->stream, f->ready, 0));
        return BORB_OK;
    }
    borb_status finish() {
        BORB_CUDA(cudaGetLastError());
        if (download_ && res_bytes_) BORB_CUDA(cudaMemcpyAsync(m_->h_out, m_->arena + res_off_, res_bytes_, cudaMemcpyDeviceToHost, m_->stream));
        BORB_CUDA(cudaStreamSynchronize(m_->stream));
        return BORB_OK;
    }
    // the landing buffer, after finish()
    const uint8_t* out(size_t off) const { return m_->h_out + off; }

private:
    struct Item { const void* src; size_t off, bytes; };
    size_t put(size_t bytes) { off_ = (off_ + 255) & ~size_t(255); const size_t o = off_; off_ += bytes; return o; }
    // grow-only buffers; the stream is synchronised first because queued work may still use the old one
    borb_status grow_device(uint8_t*& p, size_t& have, size_t bytes) {
        if (have >= bytes) return BORB_OK;
        BORB_CUDA(cudaStreamSynchronize(m_->stream));
        cudaFree(p);
        p = nullptr; have = 0;
        const size_t want = bytes + bytes / 2 + (1 << 20);
        BORB_CUDA(cudaMalloc(&p, want));
        have = want;
        return BORB_OK;
    }
    borb_status grow_pinned(uint8_t*& p, size_t& have, size_t bytes) {
        if (have >= bytes) return BORB_OK;
        BORB_CUDA(cudaStreamSynchronize(m_->stream));
        if (p) cudaFreeHost(p);
        p = nullptr; have = 0;
        const size_t want = bytes + bytes / 2 + (1 << 16);
        BORB_CUDA(cudaMallocHost(&p, want));
        have = want;
        return BORB_OK;
    }
    borb_matcher* m_;
    std::vector<Item> items_;
    size_t off_ = 0, in_end_ = 0, res_bytes_ = 0, res_off_ = 0;
    bool begun_ = false, in_place_ = false, download_ = false;
};

// ---- frame side of the windowed searches: staged from the host view per call, or taken from a device-resident borb_frame
struct FrameInfo { int n, n_levels; float min_x, min_y, max_x, max_y; bool has_ur; const borb_frame* rf; };
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
    return I;
}
// the per-call inputs of the frame (everything for a host view; only `occupied` for a resident frame)
FrameStage stage_frame(Call& c, const borb_frame_view* F, const FrameInfo& I, bool want_ur) {
    FrameStage fs;
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
// the frame fields of A that a device-resident frame provides
void bind_resident(const borb_frame* rf, ProjArgs& A) {
    A.n = rf->n;
    A.minX = rf->min_x; A.minY = rf->min_y;
    A.invW = (float)GRID_COLS / (float)(rf->max_x - rf->min_x);      // mfGridElementWidthInv (Frame.cc:101)
    A.invH = (float)GRID_ROWS / (float)(rf->max_y - rf->min_y);
    A.keys = rf->keys; A.desc = rf->desc; A.u_right = rf->u_right; A.scale_factors = rf->sf;
    A.cell_start = rf->cell_start; A.cell_idx = rf->cell_idx;
}
// the frame fields of A: the resident frame's, or those of a host view staged at fs
void bind_frame_fields(const FrameInfo& I, const FrameStage& fs, const Call& c, ProjArgs& A) {
    if (I.rf) {
        bind_resident(I.rf, A);
        if (!fs.ur_p) A.u_right = nullptr;
        return;
    }
    A.n = I.n;
    A.minX = I.min_x; A.minY = I.min_y;
    A.invW = (float)GRID_COLS / (float)(I.max_x - I.min_x);
    A.invH = (float)GRID_ROWS / (float)(I.max_y - I.min_y);
    A.keys = (const borb_keypoint*)c.dev(fs.keys); A.desc = c.dev(fs.desc);
    A.u_right = fs.ur_p ? (const float*)c.dev(fs.ur) : nullptr;
    A.scale_factors = (const float*)c.dev(fs.sf);
    A.cell_start = (const int*)c.dev(fs.cs); A.cell_idx = (const int*)c.dev(fs.ci);
}
// after commit(): builds the grid of a host view bound by bind_frame_fields, waits for the resident frame otherwise
borb_status prepare_frame(borb_matcher* m, const Call& c, const FrameInfo& I, const ProjArgs& A) {
    if (I.rf) return c.wait(I.rf);
    if (I.n > 0) m->launches += launch_grid_sort(A.keys, A.n, A.minX, A.minY, A.invW, A.invH, (int*)A.cell_start, (int*)A.cell_idx, m->stream);
    else BORB_CUDA(cudaMemsetAsync((void*)A.cell_start, 0, (size_t)(GRID_CELLS + 1) * 4, m->stream));
    return BORB_OK;
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
borb_status check_frame(const borb_frame_view* F, const FrameInfo& I, const borb_matcher* m) {
    if (I.n < 0 || I.n > MATCH_MAX_FEATURES) { set_error("frame has %d features (limit %d)", I.n, MATCH_MAX_FEATURES); return BORB_ERR_INVALID_ARG; }
    if (I.rf) {
        if (I.rf->device != m->device) { set_error("resident frame and matcher live on different devices"); return BORB_ERR_INVALID_ARG; }
        return BORB_OK;
    }
    if (I.n > 0 && (!F->keys_un || !F->desc)) { set_error("incomplete frame view"); return BORB_ERR_INVALID_ARG; }
    if (I.n_levels < 1 || !F->scale_factors || !(I.max_x > I.min_x) || !(I.max_y > I.min_y)) { set_error("incomplete frame view"); return BORB_ERR_INVALID_ARG; }
    return BORB_OK;
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

struct KfOffsets { size_t keys, desc, has_mp, u_right, node, start, idx, sf, sig; bool has_mp_p, ur_p; };

borb_status check_kf(const borb_keyframe_view* v, const char* what) {
    if (!v || v->n < 0 || v->n > MATCH_MAX_FEATURES || (v->n > 0 && (!v->keys_un || !v->desc))) {
        set_error("%s: bad keyframe view (n=%d, limit %d)", what, v ? v->n : -1, MATCH_MAX_FEATURES);
        return BORB_ERR_INVALID_ARG;
    }
    if (v->fv.n_nodes < 0 || (v->fv.n_nodes > 0 && (!v->fv.node_id || !v->fv.start || !v->fv.feat_idx))) {
        set_error("%s: bad feature vector", what);
        return BORB_ERR_INVALID_ARG;
    }
    return BORB_OK;
}

KfOffsets stage_kf(Call& c, const borb_keyframe_view* v) {
    KfOffsets o{};
    o.keys = c.in(v->keys_un, (size_t)v->n * sizeof(borb_keypoint));
    o.desc = c.in(v->desc, (size_t)v->n * 32);
    o.has_mp_p = v->has_mp != nullptr;
    o.has_mp = o.has_mp_p ? c.in(v->has_mp, (size_t)v->n) : 0;
    o.ur_p = v->u_right != nullptr;
    o.u_right = o.ur_p ? c.in(v->u_right, (size_t)v->n * 4) : 0;
    o.node = c.in(v->fv.node_id, (size_t)v->fv.n_nodes * 4);
    o.start = c.in(v->fv.start, (size_t)(v->fv.n_nodes + 1) * 4);
    const int total = v->fv.n_nodes > 0 ? v->fv.start[v->fv.n_nodes] : 0;
    o.idx = c.in(v->fv.feat_idx, (size_t)total * 4);
    o.sf = c.in(v->scale_factors, (size_t)(v->scale_factors ? v->n_levels : 0) * 4);
    o.sig = c.in(v->level_sigma2, (size_t)(v->level_sigma2 ? v->n_levels : 0) * 4);
    return o;
}

KfDev kf_dev(const Call& c, const borb_keyframe_view* v, const KfOffsets& o) {
    KfDev d;
    d.n = v->n; d.nn = v->fv.n_nodes;
    d.keys = reinterpret_cast<const borb_keypoint*>(c.dev(o.keys));
    d.desc = c.dev(o.desc);
    d.has_mp = o.has_mp_p ? c.dev(o.has_mp) : nullptr;
    d.u_right = o.ur_p ? reinterpret_cast<const float*>(c.dev(o.u_right)) : nullptr;
    d.node = reinterpret_cast<const uint32_t*>(c.dev(o.node));
    d.start = reinterpret_cast<const int32_t*>(c.dev(o.start));
    d.idx = reinterpret_cast<const uint32_t*>(c.dev(o.idx));
    d.scale_factors = reinterpret_cast<const float*>(c.dev(o.sf));
    d.level_sigma2 = reinterpret_cast<const float*>(c.dev(o.sig));
    return d;
}

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
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) { set_error("CUDA init failed: %s", cudaGetErrorString(e)); delete m; return BORB_ERR_CUDA; }
    *out = m;
    return BORB_OK;
}

borb_status borb_matcher_destroy(borb_matcher* m) {
    if (!m) return BORB_OK;
    cudaSetDevice(m->device);
    if (m->stream) cudaStreamSynchronize(m->stream);
    cudaFree(m->arena);
    cudaFree(m->aux);
    if (m->h_stage) cudaFreeHost(m->h_stage);
    if (m->h_out) cudaFreeHost(m->h_out);
    if (m->ev_a) { cudaEventDestroy(m->ev_a); cudaEventDestroy(m->ev_b); }
    if (m->t0) { cudaEventDestroy(m->t0); cudaEventDestroy(m->t1); }
    if (m->stream) cudaStreamDestroy(m->stream);
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
    f->has_bow = false;                 // a new frame, or a recycled block that still holds another frame's vectors
    f->n_bow = f->n_nodes = f->n_fv = 0;
    // u_right / depth storage always exists; the pointers are nulled for a monocular frame
    f->u_right = stereo ? f->ur_store : nullptr;
    f->depth = stereo ? f->depth_store : nullptr;
    f->n = n; f->n_levels = n_levels;
    *out = f;
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
    f->min_x = I.min_x; f->min_y = I.min_y; f->max_x = I.max_x; f->max_y = I.max_y;
    Call c(m);
    const size_t o_k = c.in(v->keys_un, (size_t)I.n * sizeof(borb_keypoint)), o_d = c.in(v->desc, (size_t)I.n * 32);
    const size_t o_u = v->u_right ? c.in(v->u_right, (size_t)I.n * 4) : 0;
    const size_t o_s = c.in(v->scale_factors, (size_t)I.n_levels * 4);
    if ((s = c.begin()) != BORB_OK || (s = c.commit()) != BORB_OK) { borb_frame_destroy(f); return s; }
    cudaStream_t q = m->stream;
    if (I.n > 0) {
        BORB_CUDA(cudaMemcpyAsync(f->keys, c.dev(o_k), (size_t)I.n * sizeof(borb_keypoint), cudaMemcpyDeviceToDevice, q));
        BORB_CUDA(cudaMemcpyAsync(f->desc, c.dev(o_d), (size_t)I.n * 32, cudaMemcpyDeviceToDevice, q));
        if (v->u_right) BORB_CUDA(cudaMemcpyAsync(f->u_right, c.dev(o_u), (size_t)I.n * 4, cudaMemcpyDeviceToDevice, q));
    }
    BORB_CUDA(cudaMemcpyAsync(f->sf, c.dev(o_s), (size_t)I.n_levels * 4, cudaMemcpyDeviceToDevice, q));
    const float invW = (float)GRID_COLS / (float)(I.max_x - I.min_x), invH = (float)GRID_ROWS / (float)(I.max_y - I.min_y);
    if (I.n > 0) m->launches += launch_grid_sort(f->keys, I.n, I.min_x, I.min_y, invW, invH, f->cell_start, f->cell_idx, q);
    else BORB_CUDA(cudaMemsetAsync(f->cell_start, 0, (size_t)(GRID_CELLS + 1) * 4, q));
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

borb_status borb_frames_from_extractor(borb_matcher* m, borb_extractor* e, const int32_t* images, int n_frames, const int32_t* n_keys,
                                       const borb_camera* cam, int mode, const void* const* depth, int depth_type, float depth_factor,
                                       int depth_stride_bytes, borb_keypoint* keys_un, float* u_right, float* depth_out, int cap,
                                       float* bounds4, borb_frame** frames) {
    if (!m || !e || !cam || !frames || n_frames < 0 || (n_frames > 0 && (!images || !n_keys))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    const bool depth_on_device = (depth_type & 4) != 0;
    depth_type &= 3;
    if (mode < 0 || mode > 2 || (mode == 2 && !depth) || (depth_type != 0 && depth_type != 1)) { set_error("bad mode / depth arguments"); return BORB_ERR_INVALID_ARG; }
    if (!e->have_geom || e->last_n_images < 1) { set_error("no extracted batch on this extractor handle"); return BORB_ERR_STATE; }
    if (e->device != m->device) { set_error("extractor and matcher live on different devices"); return BORB_ERR_INVALID_ARG; }
    if ((keys_un || u_right || depth_out) && cap < 0) { set_error("negative capacity"); return BORB_ERR_INVALID_ARG; }
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
    if (mode == 2 && !depth_on_device)
        for (int i = 0; i < n_frames; i++)
            BORB_CUDA(cudaMemcpy2DAsync(c.dev(o_depth) + (size_t)i * depth_img_bytes, (size_t)w * px, depth[i], (size_t)depth_stride_bytes, (size_t)w * px, h,
                                        cudaMemcpyHostToDevice, q));
    for (int i = 0; i < n_frames; i++) BORB_CUDA(cudaMemcpyAsync(frames[i]->sf, c.dev(o_sf), (size_t)nl * 4, cudaMemcpyDeviceToDevice, q));
    m->launches += launch_frame_build((const FrameJob*)c.dev(o_jobs), n_frames, max_n, *cam, mode, depth_type, depth_factor, w, h, ocap,
                                      keys_un ? (borb_keypoint*)c.res(r_k, false) : nullptr, fb ? (float*)c.res(r_u, false) : nullptr,
                                      (float*)c.res(r_d, false), q);
    for (int i = 0; i < n_frames; i++) BORB_CUDA(cudaEventRecord(frames[i]->ready, q));
    BORB_CUDA(cudaEventRecord(m->ev_b, q));
    BORB_CUDA(cudaStreamWaitEvent(e->stream, m->ev_b, 0));
    if ((s = c.finish()) != BORB_OK) return s;
    if (ocap > 0) {
        if (keys_un) std::memcpy(keys_un, c.out(r_k), kb);
        if (u_right) std::memcpy(u_right, c.out(r_u), fb);
        if (depth_out) std::memcpy(depth_out, c.out(r_d), fb);
    }
    return BORB_OK;
}

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

MapPointsOff stage_mappoints(Call& c, const borb_frame_view* F, const FrameInfo& I, const borb_mappoint_view* P) {
    MapPointsOff o{};
    const size_t n = (size_t)P->n;
    o.fs = stage_frame(c, F, I, true);
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
        n_matches[j] = 0;
        if (batch && !frames[j].resident) { set_error("job %d: borb_search_by_projection_batch needs device-resident frames (borb_frame_view::resident)", j); return BORB_ERR_INVALID_ARG; }
        if (batch && !match_feat[j]) { set_error("job %d: null output", j); return BORB_ERR_INVALID_ARG; }
        const FrameInfo I = J[j].I = frame_info(&frames[j]);
        borb_status s = check_mappoints(&frames[j], I, P, m);
        if (s != BORB_OK) return job_fail(batch, j, s);
        J[j].live = P->n > 0 && I.n > 0;
        if (!J[j].live) { std::fill_n(match_feat[j], P->n, -1); continue; }
        max_n = std::max(max_n, I.n); max_n_mp = std::max(max_n_mp, P->n);
    }
    if (max_n_mp == 0) return BORB_OK;
    Call c(m);
    for (int j = 0; j < n_jobs; j++)
        if (J[j].live) J[j].o = stage_mappoints(c, &frames[j], J[j].I, &points[j]);
    JobTable<ProjArgs> jt(c, n_jobs);
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
            bind_frame_fields(J[j].I, J[j].o.fs, c, A);
            bind_mappoints(J[j].o, &points[j], c, th, nnratio, (int32_t*)c.res(J[j].res, direct), A);
        }                                                // a dead job keeps n_mp = 0: both kernels skip it
        hj[j] = A;
    }
    if ((s = c.commit()) != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++)
        if (J[j].live && (s = prepare_frame(m, c, J[j].I, hj[j])) != BORB_OK) return s;
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
    int argmin;                     // 1: per-query first-minimum (no claim replay); `state` then has Q.n entries
    int chi2;                       // Fuse(pKF, ...) reprojection gates
    const float* inv_sigma2;        // chi2: mvInvLevelSigma2 (n_levels)
    int to_aux;                     // 1: leave the result in m->aux + aux_off (device) instead of downloading it
    size_t aux_off;
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

QueryOff stage_query(Call& c, const borb_frame_view* F, const FrameInfo& I, const PointQuery& Q) {
    QueryOff o{};
    const size_t nq = (size_t)Q.n;
    o.fs = stage_frame(c, F, I, Q.variant == 0 || Q.chi2);
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
// the same plus the candidate lists and the match events of the resolve / argmin kernels
void reserve_query(Call& c, const FrameInfo& I, const PointQuery& Q, QueryOff& o) {
    const size_t nq = (size_t)Q.n;
    reserve_projection(c, I, Q, o);
    o.cand = c.scratch(nq * I.n * 4); o.cc = c.scratch(nq * 4);
    o.evi = c.scratch(nq * 4); o.evb = c.scratch(nq);
}
// L and the query side of A (the frame side comes from bind_frame_fields); out: the state (argmin: Q.n entries, otherwise I.n)
// followed by the match count
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

// one (frame, query) pair of point_query_jobs; state: the job's output (argmin: Q.n entries, otherwise the frame's n), or null (to_aux)
struct PointJob { const borb_frame_view* F; PointQuery Q; int32_t* state; };

// Shared body of borb_search_by_projection_last / _kf / _sim3, of the two directions of borb_search_by_sim3 (argmin, to_aux: one job
// only) and of borb_search_by_projection_last_batch (resident frames): project_points, candidates and resolve<true> (or argmin),
// one synchronisation.  The state stays in the arena, not in mapped host memory: resolve<true> writes it with atomicMax.
borb_status point_query_jobs(borb_matcher* m, const PointJob* jobs, int n_jobs, int32_t* n_matches, bool batch) {
    struct Job { FrameInfo I; bool live; QueryOff o; size_t res; };
    std::vector<Job> J(n_jobs);
    int max_n = 1, max_nq = 0;
    for (int j = 0; j < n_jobs; j++) {
        const PointQuery& Q = jobs[j].Q;
        assert(n_jobs == 1 || (!Q.argmin && !Q.to_aux));
        n_matches[j] = 0;
        if (batch && !jobs[j].F->resident) { set_error("job %d: borb_search_by_projection_last_batch needs device-resident frames (borb_frame_view::resident)", j); return BORB_ERR_INVALID_ARG; }
        if (batch && !jobs[j].state) { set_error("job %d: null output", j); return BORB_ERR_INVALID_ARG; }
        const FrameInfo I = J[j].I = frame_info(jobs[j].F);
        borb_status s = check_query(jobs[j].F, I, Q, m);
        if (s != BORB_OK) return job_fail(batch, j, s);
        if (jobs[j].state) std::fill_n(jobs[j].state, Q.argmin ? Q.n : I.n, -1);
        if (Q.to_aux && Q.n > 0) {      // caller sized m->aux; "no match" everywhere until the kernels say otherwise
            BORB_CUDA(cudaSetDevice(m->device));
            BORB_CUDA(cudaMemsetAsync(m->aux + Q.aux_off, 0xFF, (size_t)Q.n * 4, m->stream));
        }
        J[j].live = I.n > 0 && Q.n > 0;
        if (J[j].live) { max_n = std::max(max_n, I.n); max_nq = std::max(max_nq, Q.n); }
    }
    if (max_nq == 0) return BORB_OK;
    Call c(m);
    for (int j = 0; j < n_jobs; j++)
        if (J[j].live) J[j].o = stage_query(c, jobs[j].F, J[j].I, jobs[j].Q);
    JobTable<LastArgs> lt(c, n_jobs);
    JobTable<ProjArgs> jt(c, n_jobs);
    for (int j = 0; j < n_jobs; j++) {
        if (!J[j].live) continue;
        const PointQuery& Q = jobs[j].Q;
        reserve_query(c, J[j].I, Q, J[j].o);
        const size_t bytes = (size_t)(Q.argmin ? Q.n : J[j].I.n) * 4 + 4;
        J[j].res = Q.to_aux ? c.scratch(bytes) : c.result(bytes);
    }
    borb_status s;
    if ((s = c.begin(n_jobs == 1 && J[0].I.rf)) != BORB_OK) return s;
    LastArgs* hl = lt.host(c);
    ProjArgs* hj = jt.host(c);
    for (int j = 0; j < n_jobs; j++) {
        LastArgs L{};
        ProjArgs A{};
        if (J[j].live) {
            const PointQuery& Q = jobs[j].Q;
            bind_frame_fields(J[j].I, J[j].o.fs, c, A);
            bind_query(J[j].o, Q, J[j].I, c, (int32_t*)(Q.to_aux ? c.dev(J[j].res) : c.res(J[j].res, false)), L, A);
        }                                            // a job without work keeps n_last = n_mp = 0: every kernel skips it
        hl[j] = L;
        hj[j] = A;
    }
    if ((s = c.commit()) != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++)
        if (J[j].live && (s = prepare_frame(m, c, J[j].I, hj[j])) != BORB_OK) return s;
    const PointQuery& Q0 = jobs[0].Q;
    if (Q0.argmin) m->launches += launch_projection_argmin(hl[0], hj[0], m->stream);
    else m->launches += launch_point_projection_batch(lt.dev(c), jt.dev(c), hl[0], hj[0], n_jobs, max_nq, max_n, max_nq, true, m->stream);
    if (Q0.to_aux) BORB_CUDA(cudaMemcpyAsync(m->aux + Q0.aux_off, c.dev(J[0].res), (size_t)Q0.n * 4, cudaMemcpyDeviceToDevice, m->stream));
    if ((s = c.finish()) != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++)
        if (J[j].live && !jobs[j].Q.to_aux)
            read_counted(c.out(J[j].res), jobs[j].Q.argmin ? jobs[j].Q.n : J[j].I.n, jobs[j].state, &n_matches[j]);
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
    return point_query_jobs(m, &P, 1, n_matches, false);
}

borb_status borb_search_by_projection_kf(borb_matcher* m, const borb_frame_view* cur, const borb_worldpoints_view* pts, const float* Tcw,
                                         const float* Ow, float fx, float fy, float cx, float cy, float log_scale_factor, float th,
                                         int orb_dist, int check_orientation, int32_t* state_cur, int32_t* n_matches) {
    if (!m || !cur || !pts || !Tcw || !Ow || !state_cur || !n_matches) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    PointQuery Q{};
    Q.variant = 1; Q.n = pts->n; Q.world_pos = pts->world_pos; Q.desc = pts->desc; Q.valid = pts->valid;
    Q.max_distance = pts->max_distance; Q.min_distance = pts->min_distance; Q.angle = pts->angle;
    Q.Tcw = Tcw; Q.Ow = Ow; Q.fx = fx; Q.fy = fy; Q.cx = cx; Q.cy = cy; Q.th = th; Q.log_scale = log_scale_factor;
    Q.check_ori = check_orientation; Q.th_dist = orb_dist;
    const PointJob P{cur, Q, state_cur};
    return point_query_jobs(m, &P, 1, n_matches, false);
}

borb_status borb_search_by_projection_sim3(borb_matcher* m, const borb_frame_view* kf, const borb_worldpoints_view* pts, const float* Tcw,
                                           const float* Ow, float fx, float fy, float cx, float cy, float log_scale_factor, int th,
                                           int32_t* state_kf, int32_t* n_matches) {
    if (!m || !kf || !pts || !Tcw || !Ow || !state_kf || !n_matches) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    PointQuery Q{};
    Q.variant = 2; Q.n = pts->n; Q.world_pos = pts->world_pos; Q.desc = pts->desc; Q.valid = pts->valid;
    Q.max_distance = pts->max_distance; Q.min_distance = pts->min_distance; Q.normal = pts->normal;
    Q.Tcw = Tcw; Q.Ow = Ow; Q.fx = fx; Q.fy = fy; Q.cx = cx; Q.cy = cy; Q.th = (float)th; Q.log_scale = log_scale_factor;
    Q.check_ori = 0; Q.th_dist = 50;                                       // TH_LOW (:394)
    Q.use_normal = 1;
    const PointJob P{kf, Q, state_kf};
    return point_query_jobs(m, &P, 1, n_matches, false);
}

borb_status borb_search_by_projection_last_batch(borb_matcher* m, const borb_last_frame_job* jobs, int n_jobs, int check_orientation,
                                                 int32_t* n_matches) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && (!jobs || !n_matches))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    std::vector<PointJob> P(n_jobs);
    for (int j = 0; j < n_jobs; j++) P[j] = PointJob{&jobs[j].cur, last_frame_query(jobs[j], check_orientation), jobs[j].state_cur};
    return point_query_jobs(m, P.data(), n_jobs, n_matches, true);
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
        n_found[j] = 0;
        if (!B.scw_variant && !B.inv_level_sigma2) { set_error("Fuse(pKF, vpMapPoints, th) needs mvInvLevelSigma2"); return job_fail(batch, j, BORB_ERR_INVALID_ARG); }
        PointQuery& Q = J[j].Q;
        Q.variant = 2; Q.n = B.pts.n; Q.world_pos = B.pts.world_pos; Q.desc = B.pts.desc; Q.valid = B.pts.valid;
        Q.max_distance = B.pts.max_distance; Q.min_distance = B.pts.min_distance; Q.normal = B.pts.normal;
        Q.Tcw = B.Tcw; Q.Ow = B.Ow; Q.fx = B.fx; Q.fy = B.fy; Q.cx = B.cx; Q.cy = B.cy; Q.bf = B.bf; Q.th = B.th; Q.log_scale = B.log_scale_factor;
        Q.th_dist = TH_LOW;                                                // (:944, :1075)
        Q.use_normal = 1; Q.argmin = 1;
        Q.invz_double = B.scw_variant ? 1 : 0;                             // 1.0/z (:1014) vs 1/z (:861)
        Q.chi2 = B.scw_variant ? 0 : 1; Q.inv_sigma2 = B.inv_level_sigma2;
        // occupancy plays no role in either Fuse (the MapPoint already in the slot is handled by the caller, :947-960)
        J[j].kf = B.kf;
        J[j].kf.occupied = nullptr;
        const FrameInfo I = J[j].I = frame_info(&J[j].kf);
        const borb_status s = check_query(&J[j].kf, I, Q, m);
        if (s != BORB_OK) return job_fail(batch, j, s);
        std::fill_n(B.best_idx, Q.n, -1);
        J[j].live = I.n > 0 && Q.n > 0;
        if (J[j].live) max_nq = std::max(max_nq, Q.n);
    }
    if (max_nq == 0) return BORB_OK;
    Call c(m);
    for (int j = 0; j < n_jobs; j++)
        if (J[j].live) J[j].o = stage_query(c, &J[j].kf, J[j].I, J[j].Q);
    const size_t o_last = c.in(nullptr, (size_t)n_jobs * sizeof(LastArgs)), o_jobs = c.in(nullptr, (size_t)n_jobs * sizeof(FuseJob));
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
            bind_frame_fields(J[j].I, J[j].o.fs, c, F.A);
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
        if (J[j].live && (s = prepare_frame(m, c, J[j].I, hj[j].A)) != BORB_OK) return s;
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

borb_status borb_search_by_sim3(borb_matcher* m, const borb_frame_view* kf1, const borb_frame_view* kf2, const borb_worldpoints_view* pts1,
                                const borb_worldpoints_view* pts2, const float* T1w, const float* T2w, const float* S12, const float* S21,
                                float fx, float fy, float cx, float cy, float log_scale_factor1, float log_scale_factor2, float th,
                                int32_t* match12, int32_t* n_found) {
    if (!m || !kf1 || !kf2 || !pts1 || !pts2 || !T1w || !T2w || !S12 || !S21 || !match12 || !n_found) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    *n_found = 0;
    const int n1 = frame_info(kf1).n, n2 = frame_info(kf2).n;
    if (pts1->n != n1 || pts2->n != n2) { set_error("SearchBySim3: one MapPoint slot per keyframe feature (GetMapPointMatches)"); return BORB_ERR_INVALID_ARG; }
    for (int i = 0; i < n1; i++) match12[i] = -1;
    if (n1 == 0 || n2 == 0) return BORB_OK;
    borb_frame_view F1 = *kf1, F2 = *kf2;
    F1.occupied = nullptr; F2.occupied = nullptr;
    BORB_CUDA(cudaSetDevice(m->device));
    const size_t need = (size_t)n1 + (size_t)n2;
    if (m->aux_count < need) {
        cudaFree(m->aux); m->aux = nullptr; m->aux_count = 0;
        BORB_CUDA(cudaMalloc(&m->aux, need * 4));
        m->aux_count = need;
    }
    int32_t nm = 0;
    // KF1's points into KF2 (:1146-1222) and KF2's points into KF1 (:1224-1300); both results stay on the device
    PointQuery Q{};
    Q.variant = 2; Q.n = pts1->n; Q.world_pos = pts1->world_pos; Q.desc = pts1->desc; Q.valid = pts1->valid;
    Q.max_distance = pts1->max_distance; Q.min_distance = pts1->min_distance;
    Q.Tcw = T1w; Q.chain = 1; Q.T2 = S21; Q.fx = fx; Q.fy = fy; Q.cx = cx; Q.cy = cy; Q.th = th; Q.log_scale = log_scale_factor2;
    Q.th_dist = 100; Q.argmin = 1; Q.invz_double = 1; Q.to_aux = 1; Q.aux_off = 0;        // TH_HIGH (:1218)
    const PointJob P{&F2, Q, nullptr};
    borb_status s = point_query_jobs(m, &P, 1, &nm, false);
    if (s != BORB_OK) return s;
    PointQuery R{};
    R.variant = 2; R.n = pts2->n; R.world_pos = pts2->world_pos; R.desc = pts2->desc; R.valid = pts2->valid;
    R.max_distance = pts2->max_distance; R.min_distance = pts2->min_distance;
    R.Tcw = T2w; R.chain = 1; R.T2 = S12; R.fx = fx; R.fy = fy; R.cx = cx; R.cy = cy; R.th = th; R.log_scale = log_scale_factor1;
    R.th_dist = 100; R.argmin = 1; R.invz_double = 1; R.to_aux = 1; R.aux_off = (size_t)n1;
    const PointJob PR{&F1, R, nullptr};
    s = point_query_jobs(m, &PR, 1, &nm, false);
    if (s != BORB_OK) return s;
    // agreement test (:1302-1323) on the device
    Call c(m);
    const size_t r_out = c.result((size_t)n1 * 4), r_nf = c.result(4);
    if ((s = c.begin()) != BORB_OK) return s;
    m->launches += launch_sim3_agree(m->aux, m->aux + n1, n1, n2, (int32_t*)c.res(r_out, false), (int*)c.res(r_nf, false), m->stream);
    if ((s = c.finish()) != BORB_OK) return s;
    std::memcpy(match12, c.out(r_out), (size_t)n1 * 4);
    std::memcpy(n_found, c.out(r_nf), 4);
    return BORB_OK;
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
borb_status select_local(const borb_local_points_job& B, std::vector<int32_t>& sel, LocalOff& o) {
    const borb_worldpoints_view& P = B.pts;
    for (int i = 0; i < P.n; i++) {
        B.in_view[i] = 0; B.match_feat[i] = -1;
        if (B.proj_x) B.proj_x[i] = 0.f;
        if (B.proj_y) B.proj_y[i] = 0.f;
        if (B.proj_xr) B.proj_xr[i] = 0.f;
        if (B.level) B.level[i] = 0;
        if (B.view_cos) B.view_cos[i] = 0.f;
    }
    o.sel0 = sel.size();
    for (int i = 0; i < P.n; i++)
        if (!P.valid || P.valid[i]) sel.push_back(i);
    o.nq = (int)(sel.size() - o.sel0);
    o.gather = o.nq != P.n;
    if (o.nq > MATCH_MAX_FEATURES) { set_error("%d valid local map points (limit %d per call)", o.nq, MATCH_MAX_FEATURES); return BORB_ERR_INVALID_ARG; }
    return BORB_OK;
}
// gathered inputs are written straight into the pinned staging buffer once the layout is known (src = nullptr): gather_local
void stage_local(Call& c, const borb_local_points_job& B, const FrameInfo& I, LocalOff& o) {
    const borb_worldpoints_view& P = B.pts;
    const size_t nq = (size_t)o.nq;
    const bool g = o.gather;
    o.fs = stage_frame(c, &B.frame, I, true);
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
        n_matches[j] = 0;
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
    if (max_nq == 0) return BORB_OK;
    Call c(m);
    for (int j = 0; j < n_jobs; j++)
        if (J[j].o.nq > 0) stage_local(c, jobs[j], J[j].I, J[j].o);
    JobTable<LastArgs> lt(c, n_jobs);
    JobTable<ProjArgs> jt(c, n_jobs);
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
            bind_frame_fields(J[j].I, o.fs, c, A);
            bind_local(o, jobs[j], J[j].I, viewing_cos_limit, nnratio, c, c.res(J[j].res, false), L, A);
            if (!J[j].search) A.n_mp = 0;              // a frame without features: candidates and resolve skip the job
        }                                            // a job without valid points keeps n_last = 0 as well
        hl[j] = L;
        hj[j] = A;
    }
    if ((s = c.commit()) != BORB_OK) return s;
    BORB_CUDA(cudaMemsetAsync(c.res(0, false), 0, res_end, m->stream));
    for (int j = 0; j < n_jobs; j++)
        if (J[j].o.nq > 0 && (s = prepare_frame(m, c, J[j].I, hj[j])) != BORB_OK) return s;
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

borb_status borb_search_for_initialization(borb_matcher* m, const borb_frame_view* f1, const borb_frame_view* f2, float* prev_matched,
                                           int window_size, float nnratio, int check_orientation, int32_t* matches12, int32_t* n_matches) {
    if (!m || !f1 || !f2 || !prev_matched || !matches12 || !n_matches) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    *n_matches = 0;
    if (f1->n < 0 || f1->n > MATCH_MAX_FEATURES || f2->n < 0 || f2->n > MATCH_MAX_FEATURES) { set_error("feature count outside [0,%d]", MATCH_MAX_FEATURES); return BORB_ERR_INVALID_ARG; }
    for (int i = 0; i < f1->n; i++) matches12[i] = -1;
    if (f1->n == 0 || f2->n == 0) return BORB_OK;
    if (!f1->keys_un || !f1->desc || !f2->keys_un || !f2->desc || !(f2->max_x > f2->min_x) || !(f2->max_y > f2->min_y)) {
        set_error("incomplete frame view"); return BORB_ERR_INVALID_ARG;
    }
    const int n1 = f1->n;
    // the query windows are data the caller already has: vbPrevMatched as centre, windowSize as radius, level 0 only (:421-427)
    std::vector<float> px(n1), py(n1), rad(n1, (float)window_size);
    std::vector<int32_t> zero(n1, 0);
    std::vector<uint8_t> valid(n1);
    for (int i = 0; i < n1; i++) { px[i] = prev_matched[2 * i]; py[i] = prev_matched[2 * i + 1]; valid[i] = f1->keys_un[i].octave > 0 ? 0 : 1; }
    Call c(m);
    const size_t o_k2 = c.in(f2->keys_un, (size_t)f2->n * sizeof(borb_keypoint));
    const size_t o_d2 = c.in(f2->desc, (size_t)f2->n * 32);
    const size_t o_k1 = c.in(f1->keys_un, (size_t)n1 * sizeof(borb_keypoint));
    const size_t o_d1 = c.in(f1->desc, (size_t)n1 * 32);
    const size_t o_px = c.in(px.data(), (size_t)n1 * 4), o_py = c.in(py.data(), (size_t)n1 * 4), o_rad = c.in(rad.data(), (size_t)n1 * 4);
    const size_t o_lv = c.in(zero.data(), (size_t)n1 * 4), o_val = c.in(valid.data(), (size_t)n1);
    const size_t o_prev = c.in(prev_matched, (size_t)n1 * 8);
    const size_t o_cs = c.scratch((size_t)(GRID_CELLS + 1) * 4), o_ci = c.scratch((size_t)MATCH_MAX_FEATURES * 4 + 16);
    const size_t o_cand = c.scratch((size_t)n1 * f2->n * 4), o_cc = c.scratch((size_t)n1 * 4);
    const size_t o_m12 = c.scratch((size_t)n1 * 4), o_evi = c.scratch((size_t)n1 * 4), o_evb = c.scratch((size_t)n1), o_nm = c.scratch(16);
    borb_status s;
    if ((s = c.begin()) != BORB_OK || (s = c.commit()) != BORB_OK) return s;
    ProjArgs A{};
    A.n = f2->n; A.keys = (const borb_keypoint*)c.dev(o_k2); A.desc = c.dev(o_d2);
    A.u_right = nullptr; A.occupied = nullptr;
    A.minX = f2->min_x; A.minY = f2->min_y;
    A.invW = (float)GRID_COLS / (float)(f2->max_x - f2->min_x);
    A.invH = (float)GRID_ROWS / (float)(f2->max_y - f2->min_y);
    A.scale_factors = nullptr;
    A.cell_start = (const int*)c.dev(o_cs); A.cell_idx = (const int*)c.dev(o_ci);
    A.n_mp = n1; A.proj_x = (const float*)c.dev(o_px); A.proj_y = (const float*)c.dev(o_py); A.proj_xr = (const float*)c.dev(o_px);
    A.mp_desc = c.dev(o_d1); A.mp_valid = c.dev(o_val); A.mp_has_obs = nullptr;
    A.th = 1.f; A.nnratio = nnratio;
    A.cand = (uint32_t*)c.dev(o_cand); A.cand_cnt = (int*)c.dev(o_cc);
    A.q_radius = (const float*)c.dev(o_rad); A.q_minl = (const int32_t*)c.dev(o_lv); A.q_maxl = (const int32_t*)c.dev(o_lv);
    A.mode = 1; A.check_ori = check_orientation; A.th_dist = 50;
    m->launches += launch_grid_sort(A.keys, A.n, A.minX, A.minY, A.invW, A.invH, (int*)c.dev(o_cs), (int*)c.dev(o_ci), m->stream);
    m->launches += launch_initialization(A, (const borb_keypoint*)c.dev(o_k1), n1, (int32_t*)c.dev(o_m12), (int32_t*)c.dev(o_evi), c.dev(o_evb),
                                         (float*)c.dev(o_prev), (int*)c.dev(o_nm), m->stream);
    // vbPrevMatched is updated on its staged copy: the three results go straight to the caller's arrays
    BORB_CUDA(cudaMemcpyAsync(matches12, c.dev(o_m12), (size_t)n1 * 4, cudaMemcpyDeviceToHost, m->stream));
    BORB_CUDA(cudaMemcpyAsync(prev_matched, c.dev(o_prev), (size_t)n1 * 8, cudaMemcpyDeviceToHost, m->stream));
    BORB_CUDA(cudaMemcpyAsync(n_matches, c.dev(o_nm), 4, cudaMemcpyDeviceToHost, m->stream));
    return c.finish();
}

borb_status borb_distinctive_descriptors(borb_matcher* m, const uint8_t* desc, const int32_t* offsets, int n_points, int32_t* best_idx) {
    if (!m || !offsets || !best_idx || n_points < 0) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (n_points == 0) return BORB_OK;
    const int total_desc = offsets[n_points];
    for (int i = 0; i < n_points; i++)
        if (offsets[i + 1] < offsets[i] || offsets[i] < 0 || offsets[i + 1] - offsets[i] >= (1 << 16)) { set_error("offsets must ascend; at most 65535 observations per MapPoint"); return BORB_ERR_INVALID_ARG; }
    if (total_desc > 0 && !desc) { set_error("null descriptors"); return BORB_ERR_INVALID_ARG; }
    Call c(m);
    const size_t o_d = c.in(desc, (size_t)total_desc * 32);
    const size_t o_o = c.in(offsets, (size_t)(n_points + 1) * 4);
    const size_t r_b = c.result((size_t)n_points * 4);
    borb_status s;
    if ((s = c.begin()) != BORB_OK || (s = c.commit()) != BORB_OK) return s;
    m->launches += launch_distinctive(c.dev(o_d), (const int32_t*)c.dev(o_o), n_points, (int32_t*)c.res(r_b, false), m->stream);
    if ((s = c.finish()) != BORB_OK) return s;
    std::memcpy(best_idx, c.out(r_b), (size_t)n_points * 4);
    return BORB_OK;
}

static borb_status bow_common(borb_matcher* m, const borb_keyframe_view* qs, int n_q, const borb_keyframe_view* t, int mode, float nnratio,
                              int check_ori, int32_t* match, int32_t* n_matches) {
    // mode 0: qs[0..n_q) keyframes vs ONE frame t, out stride t->n.   mode 1: n_q == 1, q = kf1, t = kf2, out stride q->n.
    Call c(m);
    std::vector<KfOffsets> qo(n_q);
    for (int i = 0; i < n_q; i++) qo[i] = stage_kf(c, &qs[i]);
    const KfOffsets to = stage_kf(c, t);
    const size_t o_qd = c.in(nullptr, (size_t)n_q * sizeof(KfDev)), o_td = c.in(nullptr, sizeof(KfDev));     // filled in place
    const int out_stride = mode == 0 ? t->n : qs[0].n;
    const size_t o_bins = c.scratch((size_t)n_q * (out_stride > 0 ? out_stride : 1));
    const size_t r_match = c.result((size_t)n_q * (out_stride > 0 ? out_stride : 1) * 4), r_nm = c.result((size_t)n_q * 4);
    borb_status s;
    if ((s = c.begin()) != BORB_OK) return s;
    KfDev* hq = c.host<KfDev>(o_qd);
    for (int i = 0; i < n_q; i++) hq[i] = kf_dev(c, &qs[i], qo[i]);
    *c.host<KfDev>(o_td) = kf_dev(c, t, to);
    if ((s = c.commit()) != BORB_OK) return s;
    m->launches += launch_bow_match((const KfDev*)c.dev(o_qd), (const KfDev*)c.dev(o_td), n_q, mode, nnratio, check_ori, (int32_t*)c.res(r_match, false),
                                    out_stride, nullptr, c.dev(o_bins), (int32_t*)c.res(r_nm, false), t->n, m->stream);
    if ((s = c.finish()) != BORB_OK) return s;
    if (out_stride > 0) std::memcpy(match, c.out(r_match), (size_t)n_q * out_stride * 4);
    std::memcpy(n_matches, c.out(r_nm), (size_t)n_q * 4);
    return BORB_OK;
}

borb_status borb_search_by_bow(borb_matcher* m, const borb_keyframe_view* kfs, int n_kf, const borb_keyframe_view* frame, float nnratio,
                               int check_orientation, int32_t* match, int32_t* n_matches) {
    if (!m || !frame || !match || !n_matches || n_kf < 0 || (n_kf > 0 && !kfs)) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_status s = check_kf(frame, "borb_search_by_bow(frame)");
    for (int i = 0; i < n_kf && s == BORB_OK; i++) s = check_kf(&kfs[i], "borb_search_by_bow(keyframe)");
    if (s != BORB_OK) return s;
    if (n_kf == 0) return BORB_OK;
    return bow_common(m, kfs, n_kf, frame, 0, nnratio, check_orientation, match, n_matches);
}

borb_status borb_search_by_bow_kf(borb_matcher* m, const borb_keyframe_view* kf1, const borb_keyframe_view* kf2, float nnratio,
                                  int check_orientation, int32_t* match12, int32_t* n_matches) {
    if (!m || !kf1 || !kf2 || !match12 || !n_matches) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_status s = check_kf(kf1, "borb_search_by_bow_kf(kf1)");
    if (s == BORB_OK) s = check_kf(kf2, "borb_search_by_bow_kf(kf2)");
    if (s != BORB_OK) return s;
    return bow_common(m, kf1, 1, kf2, 1, nnratio, check_orientation, match12, n_matches);
}

// ---- TrackReferenceKeyFrame's SearchByBoW(KeyFrame*, Frame&) for many camera streams in one launch: each job's frame is resident
// with its BoW (borb_frames_compute_bow); its keyframe is a host view, or a resident frame of which only has_mp crosses PCIe.
namespace {
borb_status check_resident_bow(const borb_frame* f, const borb_matcher* m, int j, const char* what) {
    if (!f) { set_error("job %d: %s is not a device-resident frame", j, what); return BORB_ERR_INVALID_ARG; }
    if (f->device != m->device) { set_error("job %d: %s and matcher live on different devices", j, what); return BORB_ERR_INVALID_ARG; }
    if (!f->has_bow) { set_error("job %d: %s has no BoW (borb_frames_compute_bow)", j, what); return BORB_ERR_INVALID_ARG; }
    if (f->n > MATCH_MAX_FEATURES) { set_error("job %d: %s has %d features (limit %d)", j, what, f->n, MATCH_MAX_FEATURES); return BORB_ERR_INVALID_ARG; }
    return BORB_OK;
}
// a resident frame as the SearchByBoW side of a KfDev (has_mp from the caller)
KfDev resident_kf_dev(const borb_frame* f, const uint8_t* has_mp) {
    KfDev d{};
    d.n = f->n; d.nn = f->n_nodes;
    d.keys = f->keys; d.desc = f->desc; d.has_mp = has_mp; d.u_right = f->u_right;
    d.node = f->fv_node; d.start = f->fv_start; d.idx = f->fv_idx;
    d.scale_factors = f->sf;
    return d;
}
}  // namespace

borb_status borb_search_by_bow_batch(borb_matcher* m, const borb_bow_job* jobs, int n_jobs, float nnratio, int check_orientation,
                                     int32_t* n_matches) {
    if (!m || n_jobs < 0 || (n_jobs > 0 && (!jobs || !n_matches))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (n_jobs == 0) return BORB_OK;
    int max_t = 0;
    std::vector<size_t> off(n_jobs);                  // each job's matches in the result block (frames differ in n)
    size_t total_n = 0;
    for (int j = 0; j < n_jobs; j++) {
        const borb_bow_job& B = jobs[j];
        n_matches[j] = 0;
        borb_status s = check_resident_bow(B.frame, m, j, "frame");
        if (s != BORB_OK) return s;
        if (!B.match) { set_error("job %d: null output", j); return BORB_ERR_INVALID_ARG; }
        if (B.kf_frame) {
            if ((s = check_resident_bow(B.kf_frame, m, j, "kf_frame")) != BORB_OK) return s;
        } else if ((s = check_kf(&B.kf, "keyframe")) != BORB_OK) return job_fail(true, j, s);
        max_t = std::max(max_t, B.frame->n);
        off[j] = total_n; total_n += (size_t)B.frame->n;
    }
    Call c(m);
    std::vector<KfOffsets> ko(n_jobs);
    std::vector<size_t> o_hm(n_jobs, 0);
    for (int j = 0; j < n_jobs; j++) {
        const borb_bow_job& B = jobs[j];
        if (!B.kf_frame) ko[j] = stage_kf(c, &B.kf);
        else if (B.kf.has_mp) o_hm[j] = c.in(B.kf.has_mp, (size_t)B.kf_frame->n);
    }
    const size_t o_q = c.in(nullptr, (size_t)n_jobs * sizeof(KfDev)), o_t = c.in(nullptr, (size_t)n_jobs * sizeof(KfDev));   // filled in place
    const size_t o_off = c.in(nullptr, (size_t)n_jobs * sizeof(size_t));
    const size_t o_bins = c.scratch(total_n + 16);
    const size_t r_cnt = c.result((size_t)n_jobs * 4), r_match = c.result(total_n * 4);     // n_matches of every job, then every job's matches
    borb_status s;
    if ((s = c.begin()) != BORB_OK) return s;
    KfDev* hq = c.host<KfDev>(o_q);
    KfDev* ht = c.host<KfDev>(o_t);
    size_t* hoff = c.host<size_t>(o_off);
    for (int j = 0; j < n_jobs; j++) {
        const borb_bow_job& B = jobs[j];
        hq[j] = B.kf_frame ? resident_kf_dev(B.kf_frame, B.kf.has_mp ? c.dev(o_hm[j]) : nullptr) : kf_dev(c, &B.kf, ko[j]);
        ht[j] = resident_kf_dev(B.frame, nullptr);
        hoff[j] = off[j];
    }
    if ((s = c.commit()) != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++) {
        if ((s = c.wait(jobs[j].frame)) != BORB_OK) return s;
        if (jobs[j].kf_frame && (s = c.wait(jobs[j].kf_frame)) != BORB_OK) return s;
    }
    m->launches += launch_bow_match((const KfDev*)c.dev(o_q), (const KfDev*)c.dev(o_t), n_jobs, 0, nnratio, check_orientation,
                                    (int32_t*)c.res(r_match, false), 0, (const size_t*)c.dev(o_off), c.dev(o_bins), (int32_t*)c.res(r_cnt, false),
                                    max_t, m->stream);
    if ((s = c.finish()) != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++) {
        std::memcpy(&n_matches[j], c.out(r_cnt) + (size_t)j * 4, 4);
        std::memcpy(jobs[j].match, c.out(r_match) + off[j] * 4, (size_t)jobs[j].frame->n * 4);
    }
    return BORB_OK;
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

borb_status borb_kfdb_add(borb_kfdb* db, const borb_keyframe_view* kf, const uint32_t* bow_word, const double* bow_value, int n_bow,
                          int32_t* slot_out) {
    if (!db || !kf || !slot_out || n_bow < 0 || (n_bow > 0 && (!bow_word || !bow_value))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_status s = check_kf(kf, "borb_kfdb_add");
    if (s != BORB_OK) return s;
    for (int i = 1; i < n_bow; i++)
        if (bow_word[i] <= bow_word[i - 1]) { set_error("BowVector words must ascend (std::map order)"); return BORB_ERR_INVALID_ARG; }
    const int nn = kf->fv.n_nodes;
    const int m = nn > 0 ? kf->fv.start[nn] : 0;
    for (int a = 0; a < nn; a++)
        if (kf->fv.start[a + 1] < kf->fv.start[a] || (a > 0 && kf->fv.node_id[a] <= kf->fv.node_id[a - 1])) { set_error("FeatureVector nodes must ascend"); return BORB_ERR_INVALID_ARG; }
    for (int r = 0; r < m; r++)
        if (kf->fv.feat_idx[r] >= (uint32_t)kf->n) { set_error("FeatureVector index %u outside the keyframe's %d features", kf->fv.feat_idx[r], kf->n); return BORB_ERR_INVALID_ARG; }
    std::lock_guard<std::mutex> lk(db->mu);
    BORB_CUDA(cudaSetDevice(db->device));
    // one device block per keyframe: [node | start | orig | angle | hasmp | desc (rows in FeatureVector order) | bow words | bow values]
    size_t off = 0;
    auto put = [&](size_t bytes) { off = (off + 255) & ~size_t(255); const size_t o = off; off += bytes; return o; };
    const size_t o_node = put((size_t)nn * 4), o_start = put((size_t)(nn + 1) * 4), o_meta = put((size_t)m * 8), o_desc = put((size_t)m * 32);
    const size_t o_bw = put((size_t)n_bow * 4), o_bv = put((size_t)n_bow * 8);
    const size_t total = off + 256;
    std::vector<uint8_t> h(total, 0);
    borb_kfdb::Entry e;
    e.orig.resize(m);
    if (nn) {
        std::memcpy(&h[o_node], kf->fv.node_id, (size_t)nn * 4);
        std::memcpy(&h[o_start], kf->fv.start, (size_t)(nn + 1) * 4);
        uint32_t* meta = reinterpret_cast<uint32_t*>(&h[o_meta]);
        e.meta.resize((size_t)m * 2);
        int a = 0;                                                     // node index of row r (rows are grouped by node)
        for (int r = 0; r < m; r++) {
            while (a + 1 < nn && r >= kf->fv.start[a + 1]) a++;
            const uint32_t f = kf->fv.feat_idx[r];
            e.orig[r] = (uint16_t)f;
            meta[2 * r] = f | ((kf->has_mp && kf->has_mp[f]) ? 0x10000u : 0u) | ((uint32_t)a << 17);
            std::memcpy(&meta[2 * r + 1], &kf->keys_un[f].angle, 4);
            e.meta[2 * r] = meta[2 * r]; e.meta[2 * r + 1] = meta[2 * r + 1];
            std::memcpy(&h[o_desc + (size_t)r * 32], kf->desc + (size_t)f * 32, 32);
        }
    }
    if (n_bow) { std::memcpy(&h[o_bw], bow_word, (size_t)n_bow * 4); std::memcpy(&h[o_bv], bow_value, (size_t)n_bow * 8); }
    BORB_CUDA(cudaMalloc(&e.block, total));
    BORB_CUDA(cudaMemcpy(e.block, h.data(), total, cudaMemcpyHostToDevice));
    uint8_t* b = e.block;
    e.stream.node = (const uint32_t*)(b + o_node); e.stream.start = (const int32_t*)(b + o_start); e.stream.meta = (const uint2*)(b + o_meta);
    e.stream.desc = b + o_desc;
    e.stream.nn = nn; e.stream.m = m; e.stream.n = kf->n; e.stream.pad = 0;
    e.d_meta = b + o_meta;
    e.n = kf->n;
    e.bow.word = (const uint32_t*)(b + o_bw); e.bow.value = (const double*)(b + o_bv); e.bow.n = n_bow;
    e.alive = true;
    db->entries.push_back(std::move(e));
    db->dirty = true;
    db->bytes += total;
    *slot_out = (int32_t)db->entries.size() - 1;
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

borb_status borb_kfdb_set_has_mp(borb_kfdb* db, int32_t slot, const uint8_t* has_mp) {
    if (!db || !has_mp) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    std::lock_guard<std::mutex> lk(db->mu);
    if (slot < 0 || slot >= (int)db->entries.size() || !db->entries[slot].alive) { set_error("bad keyframe slot"); return BORB_ERR_INVALID_ARG; }
    BORB_CUDA(cudaSetDevice(db->device));
    borb_kfdb::Entry& e = db->entries[slot];
    for (size_t r = 0; r < e.orig.size(); r++) e.meta[2 * r] = (e.meta[2 * r] & ~0x10000u) | (has_mp[e.orig[r]] ? 0x10000u : 0u);
    BORB_CUDA(cudaDeviceSynchronize());           // a search enqueued under the mutex may still be reading the records
    if (!e.meta.empty()) BORB_CUDA(cudaMemcpy(e.d_meta, e.meta.data(), e.meta.size() * 4, cudaMemcpyHostToDevice));
    return BORB_OK;
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
};

// One query of the database score: the BowVector comes from the host (word / value) or from a resident frame.
struct QueryJob {
    borb_kfdb* db;
    const borb_frame* frame;
    const uint32_t* word; const double* value; int n_bow;
    int32_t* common; float* score; uint32_t* first_word;
    int cap; int32_t* n_slots;
};

// Shared body of borb_kfdb_query and borb_kfdb_query_batch: one launch of kfdb_score_kernel for every job (none when no database
// has a slot) and one synchronisation.  The arguments are checked by the callers.
borb_status kfdb_query_jobs(borb_matcher* m, const QueryJob* q, int n_jobs, bool batch) {
    std::vector<int> ns(n_jobs);
    std::vector<size_t> o_w(n_jobs, 0), o_v(n_jobs, 0), ho(n_jobs, 0);
    int max_slots = 0, max_nq = 0;
    Call c(m);
    {
        std::vector<borb_kfdb*> dbs(n_jobs);
        for (int j = 0; j < n_jobs; j++) dbs[j] = q[j].db;
        DbLocks lk(std::move(dbs));
        for (int j = 0; j < n_jobs; j++) {
            ns[j] = (int)q[j].db->entries.size();
            *q[j].n_slots = ns[j];
        }
        for (int j = 0; j < n_jobs; j++)
            if (q[j].cap < ns[j]) { set_error("output capacity %d < %d database slots", q[j].cap, ns[j]); return job_fail(batch, j, BORB_ERR_CAPACITY); }
        for (int j = 0; j < n_jobs; j++) {
            max_slots = std::max(max_slots, ns[j]);
            max_nq = std::max(max_nq, q[j].frame ? q[j].frame->n_bow : q[j].n_bow);
        }
        if (max_slots == 0) return BORB_OK;
        BORB_CUDA(cudaSetDevice(m->device));
        borb_status s = lk.sync();
        if (s != BORB_OK) return s;
        for (int j = 0; j < n_jobs; j++)
            if (!q[j].frame) { o_w[j] = c.in(q[j].word, (size_t)q[j].n_bow * 4); o_v[j] = c.in(q[j].value, (size_t)q[j].n_bow * 8); }
        const size_t o_jobs = c.in(nullptr, (size_t)n_jobs * sizeof(KfdbQueryJob));     // filled in place
        for (int j = 0; j < n_jobs; j++) ho[j] = c.result((size_t)ns[j] * 12);
        if ((s = c.begin()) != BORB_OK) return s;
        KfdbQueryJob* hj = c.host<KfdbQueryJob>(o_jobs);
        for (int j = 0; j < n_jobs; j++) {
            // the three result arrays are written by the kernel straight into the pinned landing buffer (device-addressable, UVA)
            uint8_t* o = c.res(ho[j], true);
            KfdbQueryJob J{};
            J.table = q[j].db->d_table; J.n_slots = ns[j];
            if (q[j].frame) { J.qword = q[j].frame->bow_word; J.qvalue = q[j].frame->bow_value; J.nq = q[j].frame->n_bow; }
            else { J.qword = (const uint32_t*)c.dev(o_w[j]); J.qvalue = (const double*)c.dev(o_v[j]); J.nq = q[j].n_bow; }
            J.common = (int32_t*)o; J.score = (float*)(o + (size_t)ns[j] * 4); J.first_word = (uint32_t*)(o + (size_t)ns[j] * 8);
            hj[j] = J;
        }
        if ((s = c.commit()) != BORB_OK) return s;
        for (int j = 0; j < n_jobs; j++)
            if (q[j].frame && (s = c.wait(q[j].frame)) != BORB_OK) return s;
        m->launches += launch_kfdb_score((const KfdbQueryJob*)c.dev(o_jobs), n_jobs, max_slots, max_nq, q[0].db->n_sm, m->stream);
    }
    const borb_status s = c.finish();
    if (s != BORB_OK) return s;
    for (int j = 0; j < n_jobs; j++) {
        const uint8_t* o = c.out(ho[j]);
        std::memcpy(q[j].common, o, (size_t)ns[j] * 4);
        std::memcpy(q[j].score, o + (size_t)ns[j] * 4, (size_t)ns[j] * 4);
        std::memcpy(q[j].first_word, o + (size_t)ns[j] * 8, (size_t)ns[j] * 4);
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
};

// Shared body of borb_search_by_bow_db, _db_pairs and _db_batch: pack, match and finalize over the job table (3 launches; none when
// no job has a keyframe and a feature inside a node) and one synchronisation.  The arguments are checked by the callers, except the
// slot lists, which are checked here under the database locks (a batch checks every job with keyframes, a single call only one
// that has work, as before).
borb_status bowdb_jobs(borb_matcher* m, const SearchJob* J, int n_jobs, float nnratio, int check_ori, bool batch) {
    struct Plan { int nn, m, n; bool work; FrameBlockHdr h; size_t o_node, o_start, o_idx, o_keys, o_desc, o_fb, o_sl, o_ctr, o_hist, o_tab, o_dense, ho; };
    std::vector<Plan> P(n_jobs);
    for (int j = 0; j < n_jobs; j++) {
        const SearchJob& S = J[j];
        Plan& p = P[j];
        if (S.frame) { p.nn = S.frame->n_nodes; p.m = S.frame->n_fv; p.n = S.frame->n; }
        else { p.nn = S.view->fv.n_nodes; p.m = p.nn > 0 ? S.view->fv.start[p.nn] : 0; p.n = S.view->n; }
        p.work = S.n_kf > 0 && p.m > 0;
        if (S.n_pairs_total) *S.n_pairs_total = 0;
        if (S.dense) for (size_t i = 0; i < (size_t)S.n_kf * p.n; i++) S.dense[i] = -1;
        for (int i = 0; i < S.n_kf; i++) { S.n_matches[i] = 0; if (S.pair_offset) S.pair_offset[i] = 0; }
    }
    std::vector<int> work;
    for (int j = 0; j < n_jobs; j++) if (P[j].work) work.push_back(j);
    const int nw = (int)work.size();
    Call c(m);
    {
        std::vector<borb_kfdb*> dbs(n_jobs);
        for (int j = 0; j < n_jobs; j++) dbs[j] = J[j].db;
        DbLocks lk(std::move(dbs));
        for (int j = 0; j < n_jobs; j++) {
            const SearchJob& S = J[j];
            if (S.n_kf == 0 || (!batch && !P[j].work)) continue;      // the single calls return zeros before looking at the slots
            const int n_slots = (int)S.db->entries.size();
            if (!S.slots && S.n_kf != n_slots) { set_error("slots == NULL searches every slot: n_kf must be %d", n_slots); return job_fail(batch, j, BORB_ERR_INVALID_ARG); }
            if (S.slots)
                for (int i = 0; i < S.n_kf; i++)
                    if (S.slots[i] < 0 || S.slots[i] >= n_slots || !S.db->entries[S.slots[i]].alive) { set_error("slot %d is not a live keyframe", S.slots[i]); return job_fail(batch, j, BORB_ERR_INVALID_ARG); }
        }
        if (nw == 0) return BORB_OK;
        BORB_CUDA(cudaSetDevice(m->device));
        borb_status s = lk.sync();
        if (s != BORB_OK) return s;
        for (int j : work) {
            const SearchJob& S = J[j];
            Plan& p = P[j];
            if (!S.frame) {                                            // a host view: its raw arrays, packed on the device like a resident frame
                const borb_keyframe_view* v = S.view;
                p.o_node = c.in(v->fv.node_id, (size_t)p.nn * 4); p.o_start = c.in(v->fv.start, (size_t)(p.nn + 1) * 4);
                p.o_idx = c.in(v->fv.feat_idx, (size_t)p.m * 4);
                p.o_keys = c.in(v->keys_un, (size_t)p.n * sizeof(borb_keypoint)); p.o_desc = c.in(v->desc, (size_t)p.n * 32);
            }
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
            if (S.frame) {
                D.fv_node = S.frame->fv_node; D.fv_start = S.frame->fv_start; D.fv_idx = S.frame->fv_idx;
                D.keys = S.frame->keys; D.desc = S.frame->desc;
            } else {
                D.fv_node = (const uint32_t*)c.dev(p.o_node); D.fv_start = (const int32_t*)c.dev(p.o_start); D.fv_idx = (const uint32_t*)c.dev(p.o_idx);
                D.keys = (const borb_keypoint*)c.dev(p.o_keys); D.desc = c.dev(p.o_desc);
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
        m->launches += launch_bowdb(A, hj[0], max_smem_frame, max_items, total_kf, max_nn, g_bow_csa.load(), J[work[0]].db->n_sm, m->stream);
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
borb_status check_db_view(borb_matcher* m, borb_kfdb* db, const borb_keyframe_view* frame, int n_kf) {
    if (m->device != db->device) { set_error("matcher and keyframe database live on different devices"); return BORB_ERR_INVALID_ARG; }
    borb_status s = check_kf(frame, "SearchByBoW(database, frame)");
    if (s != BORB_OK || n_kf == 0) return s;
    const int nn = frame->fv.n_nodes, mf = nn > 0 ? frame->fv.start[nn] : 0;
    for (int a = 0; a < nn; a++)
        if (frame->fv.start[a + 1] < frame->fv.start[a] || (a > 0 && frame->fv.node_id[a] <= frame->fv.node_id[a - 1])) { set_error("FeatureVector nodes must ascend"); return BORB_ERR_INVALID_ARG; }
    for (int r = 0; r < mf; r++)
        if (frame->fv.feat_idx[r] >= (uint32_t)frame->n) { set_error("FeatureVector index outside the frame's features"); return BORB_ERR_INVALID_ARG; }
    return BORB_OK;
}

// the checks of a batch job's database and resident frame
borb_status check_db_job(borb_matcher* m, borb_kfdb* db, const borb_frame* f, int j) {
    if (!db) { set_error("job %d: null database", j); return BORB_ERR_INVALID_ARG; }
    if (db->device != m->device) { set_error("job %d: database and matcher live on different devices", j); return BORB_ERR_INVALID_ARG; }
    return check_resident_bow(f, m, j, "frame");
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

borb_status borb_search_by_bow_db(borb_matcher* m, borb_kfdb* db, const int32_t* slots, int n_kf, const borb_keyframe_view* frame,
                                  float nnratio, int check_orientation, int32_t* match, int32_t* n_matches) {
    if (!m || !db || !frame || !match || !n_matches || n_kf < 0) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_status s = check_db_view(m, db, frame, n_kf);
    if (s != BORB_OK) return s;
    const SearchJob J{db, nullptr, frame, slots, n_kf, match, n_matches, nullptr, nullptr, 0, nullptr};
    return bowdb_jobs(m, &J, 1, nnratio, check_orientation, false);
}

borb_status borb_search_by_bow_db_pairs(borb_matcher* m, borb_kfdb* db, const int32_t* slots, int n_kf, const borb_keyframe_view* frame,
                                        float nnratio, int check_orientation, int32_t* n_matches, int32_t* pair_offset, uint32_t* pairs,
                                        int pairs_cap, int32_t* n_pairs_total) {
    if (!m || !db || !frame || !n_matches || n_kf < 0 || pairs_cap < 0 || (pairs && !pair_offset)) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    borb_status s = check_db_view(m, db, frame, n_kf);
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

// ---- SearchForTriangulation: borb_search_for_triangulation is the one-job case of borb_search_for_triangulation_batch (one launch
// of triangulation_kernel, a CTA per job, and one synchronisation).  Each side is a host view or a resident frame with its BoW.
namespace {
borb_status triangulation_jobs(borb_matcher* m, const borb_triangulation_job* jobs, int n_jobs, int check_ori, bool batch) {
    struct Side { int n, nn; KfOffsets o; size_t o_hm, o_sig; };
    struct Job { Side s1, s2; bool live; int cap; size_t vm, bins, res; };
    std::vector<Job> J(n_jobs);
    for (int j = 0; j < n_jobs; j++) {
        const borb_triangulation_job& B = jobs[j];
        if (!B.pairs || !B.n_pairs || B.cap < 0) { set_error("job %d: null output or negative capacity", j); return BORB_ERR_INVALID_ARG; }
        *B.n_pairs = 0;
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
        Q.s1.n = B.kf1_frame ? B.kf1_frame->n : B.kf1.n; Q.s1.nn = B.kf1_frame ? B.kf1_frame->n_nodes : B.kf1.fv.n_nodes;
        Q.s2.n = B.kf2_frame ? B.kf2_frame->n : B.kf2.n; Q.s2.nn = B.kf2_frame ? B.kf2_frame->n_nodes : B.kf2.fv.n_nodes;
        Q.live = Q.s1.n > 0 && Q.s1.nn > 0 && Q.s2.n > 0 && Q.s2.nn > 0;
        Q.cap = std::min(B.cap, Q.s1.n);             // a job has at most one pair per kf1 feature
    }
    std::vector<int> live;
    for (int j = 0; j < n_jobs; j++) if (J[j].live) live.push_back(j);
    const int nl = (int)live.size();
    if (nl == 0) return BORB_OK;
    Call c(m);
    for (int j : live) {
        const borb_triangulation_job& B = jobs[j];
        Job& Q = J[j];
        if (!B.kf1_frame) Q.s1.o = stage_kf(c, &B.kf1);
        else if (B.kf1.has_mp) Q.s1.o_hm = c.in(B.kf1.has_mp, (size_t)Q.s1.n);
        if (!B.kf2_frame) Q.s2.o = stage_kf(c, &B.kf2);
        else {
            if (B.kf2.has_mp) Q.s2.o_hm = c.in(B.kf2.has_mp, (size_t)Q.s2.n);
            Q.s2.o_sig = c.in(B.kf2.level_sigma2, (size_t)B.kf2_frame->n_levels * 4);
        }
    }
    const size_t o_jobs = c.in(nullptr, (size_t)nl * sizeof(TriJob));          // filled in place
    const size_t r_cnt = c.result((size_t)nl * 4);       // n_pairs of every live job, then every job's pairs
    for (int j : live) {
        Job& Q = J[j];
        Q.vm = c.scratch((size_t)Q.s1.n * 4); Q.bins = c.scratch((size_t)Q.s1.n);
        Q.res = c.result((size_t)Q.cap * 8);
    }
    borb_status s;
    if ((s = c.begin()) != BORB_OK) return s;
    TriJob* hj = c.host<TriJob>(o_jobs);
    for (int k = 0; k < nl; k++) {
        const borb_triangulation_job& B = jobs[live[k]];
        const Job& Q = J[live[k]];
        TriJob T{};
        T.q = B.kf1_frame ? resident_kf_dev(B.kf1_frame, B.kf1.has_mp ? c.dev(Q.s1.o_hm) : nullptr) : kf_dev(c, &B.kf1, Q.s1.o);
        if (B.kf2_frame) {
            T.t = resident_kf_dev(B.kf2_frame, B.kf2.has_mp ? c.dev(Q.s2.o_hm) : nullptr);
            T.t.level_sigma2 = (const float*)c.dev(Q.s2.o_sig);
        } else T.t = kf_dev(c, &B.kf2, Q.s2.o);
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
    cudaSetDevice(v->device);
    if (v->stream) cudaStreamSynchronize(v->stream);
    if (v->owns) cudaFree(v->blob);
    if (v->scratch) cudaFreeHost(v->scratch);
    if (v->stream) cudaStreamDestroy(v->stream);
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
    BORB_CUDA(cudaSetDevice(v->device));
    const size_t need = (size_t)n * (32 + 4 + 8 + 4) + 1024;
    if (v->scratch_bytes < need) {
        BORB_CUDA(cudaStreamSynchronize(v->stream));
        if (v->scratch) cudaFreeHost(v->scratch);
        v->scratch = nullptr; v->scratch_bytes = 0;
        BORB_CUDA(cudaMallocHost(&v->scratch, need * 2));
        v->scratch_bytes = need * 2;
    }
    uint8_t* h_desc = v->scratch;
    double* h_w = (double*)(v->scratch + (((size_t)n * 32 + 255) & ~size_t(255)));
    int32_t* h_word = (int32_t*)(h_w + n);
    int32_t* h_node = h_word + n;
    std::memcpy(h_desc, desc, (size_t)n * 32);
    launch_bow_transform(v->dev, h_desc, n, levelsup, h_word, h_w, h_node, v->stream);
    BORB_CUDA(cudaGetLastError());
    BORB_CUDA(cudaStreamSynchronize(v->stream));
    std::memcpy(word, h_word, (size_t)n * 4);
    std::memcpy(weight, h_w, (size_t)n * 8);
    std::memcpy(node, h_node, (size_t)n * 4);
    return BORB_OK;
}

// Frame::ComputeBoW / KeyFrame::ComputeBoW (src/Frame.cc:395-402, src/KeyFrame.cc:59-68): the tree descent on the GPU
// (borb_bow_transform), then the ordered-map bookkeeping of TemplatedVocabulary::transform (TemplatedVocabulary.h:1150-1194) in
// C++: BowVector::addWeight in feature order for every feature whose word weight is > 0, L1 normalisation with the norm summed
// in word order (BowVector.cpp:60-79), FeatureVector::addFeature in feature order.
borb_status borb_compute_bow(borb_voc* v, const uint8_t* desc, int n, int levelsup, uint32_t* bow_word, double* bow_value, int32_t* n_bow,
                             uint32_t* fv_node, int32_t* fv_start, uint32_t* fv_idx, int32_t* n_nodes) {
    if (!v || n < 0 || !n_bow || !n_nodes || (n > 0 && (!desc || !bow_word || !bow_value || !fv_node || !fv_start || !fv_idx))) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    *n_bow = 0; *n_nodes = 0;
    if (fv_start) fv_start[0] = 0;
    if (n == 0) return BORB_OK;
    std::vector<int32_t> word(n), node(n);
    std::vector<double> weight(n);
    borb_status s = borb_bow_transform(v, desc, n, levelsup, word.data(), weight.data(), node.data());
    if (s != BORB_OK) return s;
    // kept features ordered by word / by node, equal keys in feature order (what std::map insertion in feature order gives):
    // one 64-bit key (id << 32 | feature) per feature, plain sort
    std::vector<uint64_t> kw, kn;
    kw.reserve(n); kn.reserve(n);
    for (int i = 0; i < n; i++)
        if (weight[i] > 0) { kw.push_back(((uint64_t)(uint32_t)word[i] << 32) | (uint32_t)i); kn.push_back(((uint64_t)(uint32_t)node[i] << 32) | (uint32_t)i); }
    std::sort(kw.begin(), kw.end());
    std::sort(kn.begin(), kn.end());
    std::vector<int32_t> byw(kw.size()), byn(kn.size());
    for (size_t k = 0; k < kw.size(); k++) { byw[k] = (int32_t)(kw[k] & 0xFFFFFFFFu); byn[k] = (int32_t)(kn[k] & 0xFFFFFFFFu); }
    int nb = 0;
    for (size_t k = 0; k < byw.size(); k++) {
        const int i = byw[k];
        if (nb > 0 && bow_word[nb - 1] == (uint32_t)word[i]) bow_value[nb - 1] += weight[i];     // vit->second += v
        else { bow_word[nb] = (uint32_t)word[i]; bow_value[nb] = weight[i]; nb++; }
    }
    double norm = 0.0;
    for (int k = 0; k < nb; k++) norm += std::fabs(bow_value[k]);
    if (norm > 0.0) for (int k = 0; k < nb; k++) bow_value[k] /= norm;
    int nn = 0;
    for (size_t k = 0; k < byn.size(); k++) {
        const int i = byn[k];
        if (nn == 0 || fv_node[nn - 1] != (uint32_t)node[i]) { fv_node[nn] = (uint32_t)node[i]; fv_start[nn] = (int32_t)k; nn++; }
        fv_idx[k] = (uint32_t)i;
    }
    fv_start[nn] = (int32_t)byn.size();
    *n_bow = nb; *n_nodes = nn;
    return BORB_OK;
}

// Frame::ComputeBoW for many resident frames: borb_compute_bow's descent and bookkeeping both on the device (bow_transform_batch_kernel,
// bow_build_kernel), two launches and one synchronisation; the vectors stay with the frames for borb_search_by_bow_batch.
borb_status borb_frames_compute_bow(borb_matcher* m, borb_voc* v, borb_frame* const* frames, int n_frames, int levelsup,
                                    uint32_t* const* bow_word, double* const* bow_value, int32_t* n_bow, uint32_t* const* fv_node,
                                    int32_t* const* fv_start, uint32_t* const* fv_idx, int32_t* n_nodes) {
    if (!m || !v || n_frames < 0 || (n_frames > 0 && !frames)) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    if (n_frames == 0) return BORB_OK;
    if (v->device != m->device) { set_error("vocabulary and matcher live on different devices"); return BORB_ERR_INVALID_ARG; }
    int max_n = 0;
    for (int i = 0; i < n_frames; i++) {
        const borb_frame* f = frames[i];
        if (!f) { set_error("frame %d: not a device-resident frame", i); return BORB_ERR_INVALID_ARG; }
        if (f->device != m->device) { set_error("frame %d: frame and matcher live on different devices", i); return BORB_ERR_INVALID_ARG; }
        if (f->n < 0 || f->n > MATCH_MAX_FEATURES) { set_error("frame %d: %d features (limit %d)", i, f->n, MATCH_MAX_FEATURES); return BORB_ERR_INVALID_ARG; }
        max_n = std::max(max_n, f->n);
    }
    auto wants = [&](int i) {
        return (bow_word && bow_word[i]) || (bow_value && bow_value[i]) || (fv_node && fv_node[i]) || (fv_start && fv_start[i]) || (fv_idx && fv_idx[i]);
    };
    Call c(m);
    const size_t o_jobs = c.in(nullptr, (size_t)n_frames * sizeof(BowFrameJob));     // filled in place
    std::vector<size_t> o_scr(n_frames), o_copy(n_frames, 0);
    const size_t r_cnt = c.result((size_t)n_frames * 12);     // (n_bow, n_nodes, fv_start[n_nodes]) of every frame, then the host copies
    for (int i = 0; i < n_frames; i++) {
        const size_t n = (size_t)frames[i]->n;
        o_scr[i] = c.scratch(n * 16);                   // weight f64 | word i32 | node i32
        if (wants(i)) o_copy[i] = c.result(n * 24 + 4);   // value | word | node | start | idx
    }
    borb_status s;
    if ((s = c.begin()) != BORB_OK) return s;
    BowFrameJob* hj = c.host<BowFrameJob>(o_jobs);
    for (int i = 0; i < n_frames; i++) {
        borb_frame* f = frames[i];
        const size_t n = (size_t)f->n;
        BowFrameJob J{};
        J.desc = f->desc; J.n = f->n;
        uint8_t* w = c.dev(o_scr[i]);
        J.weight = (double*)w; J.word = (int32_t*)(w + n * 8); J.node = (int32_t*)(w + n * 12);
        J.dst = BowTables{f->bow_word, f->bow_value, f->fv_node, f->fv_start, f->fv_idx};
        if (wants(i)) {
            uint8_t* cp = c.res(o_copy[i], false);
            J.copy = BowTables{(uint32_t*)(cp + n * 8), (double*)cp, (uint32_t*)(cp + n * 12), (int32_t*)(cp + n * 16), (uint32_t*)(cp + n * 20 + 4)};
        }
        J.counts = (int32_t*)c.res(r_cnt, false) + 3 * i;
        hj[i] = J;
        f->has_bow = false;                             // the storage is rewritten from here on
    }
    if ((s = c.commit()) != BORB_OK) return s;
    for (int i = 0; i < n_frames; i++)
        if ((s = c.wait(frames[i])) != BORB_OK) return s;
    m->launches += launch_bow_frames(v->dev, (const BowFrameJob*)c.dev(o_jobs), n_frames, max_n, levelsup, m->stream);
    for (int i = 0; i < n_frames; i++) BORB_CUDA(cudaEventRecord(frames[i]->ready, m->stream));
    if ((s = c.finish()) != BORB_OK) return s;
    for (int i = 0; i < n_frames; i++) {
        borb_frame* f = frames[i];
        int32_t cnt[3];
        std::memcpy(cnt, c.out(r_cnt) + (size_t)i * 12, 12);
        f->n_bow = cnt[0]; f->n_nodes = cnt[1]; f->n_fv = cnt[2]; f->has_bow = true;
        if (n_bow) n_bow[i] = cnt[0];
        if (n_nodes) n_nodes[i] = cnt[1];
        if (!wants(i)) continue;
        const size_t n = (size_t)f->n;
        const uint8_t* cp = c.out(o_copy[i]);
        if (bow_value && bow_value[i]) std::memcpy(bow_value[i], cp, (size_t)cnt[0] * 8);
        if (bow_word && bow_word[i]) std::memcpy(bow_word[i], cp + n * 8, (size_t)cnt[0] * 4);
        if (fv_node && fv_node[i]) std::memcpy(fv_node[i], cp + n * 12, (size_t)cnt[1] * 4);
        if (fv_start && fv_start[i]) std::memcpy(fv_start[i], cp + n * 16, (size_t)(cnt[1] + 1) * 4);
        if (fv_idx && fv_idx[i]) std::memcpy(fv_idx[i], cp + n * 20 + 4, (size_t)cnt[2] * 4);
    }
    return BORB_OK;
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
