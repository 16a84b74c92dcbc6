// Host side of libborb: C ABI (include/borb.h), geometry/tables, workspace, launch orchestration.
// No CPU compute path exists here: every entry point that produces results launches CUDA kernels.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "borb_internal.h"

namespace borb {

static thread_local std::string tl_error;
void set_error(const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    tl_error = buf;
}

bool allow_max_smem(const void* func) {
    static std::mutex mu;
    static std::vector<std::pair<const void*, int>> done;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return false;
    std::lock_guard<std::mutex> lk(mu);
    for (auto& d : done)
        if (d.first == func && d.second == dev) return true;
    cudaFuncAttributes fa;
    int optin = 0;
    cudaError_t e = cudaFuncGetAttributes(&fa, func);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes);
    if (e != cudaSuccess) { set_error("raising the shared-memory limit failed: %s", cudaGetErrorString(e)); cudaGetLastError(); return false; }
    done.push_back({func, dev});
    return true;
}

namespace {

inline int cv_round_f(float v) { return (int)lrintf(v); }     // cvRound: round-half-even
inline int align_up(int v, int a) { return (v + a - 1) / a * a; }

// Scale tables and per-level quotas exactly as the reference constructor derives them
// (src/ORBextractor.cc:410-470): float chain with a double scaleFactor member, cvRound quotas, umax.
void init_tables(borb_extractor* e) {
    const int L = e->cfg.n_levels;
    const double sf = (double)e->cfg.scale_factor;
    e->scale.assign(L, 1.f); e->sigma2.assign(L, 1.f); e->inv_scale.assign(L, 1.f); e->inv_sigma2.assign(L, 1.f);
    for (int i = 1; i < L; i++) {
        e->scale[i] = (float)((double)e->scale[i - 1] * sf);
        e->sigma2[i] = e->scale[i] * e->scale[i];
    }
    for (int i = 0; i < L; i++) { e->inv_scale[i] = 1.0f / e->scale[i]; e->inv_sigma2[i] = 1.0f / e->sigma2[i]; }
    e->per_level.assign(L, 0);
    const float factor = (float)(1.0 / sf);
    float want = (float)e->cfg.n_features * (1.f - factor) / (1.f - (float)std::pow((double)factor, (double)L));
    int sum = 0;
    for (int l = 0; l < L - 1; l++) {
        e->per_level[l] = cv_round_f(want);
        sum += e->per_level[l];
        want *= factor;
    }
    e->per_level[L - 1] = e->cfg.n_features - sum > 0 ? e->cfg.n_features - sum : 0;
    // circular patch row extents
    const int vmax = (int)std::floor(HALF_PATCH * std::sqrt(2.f) / 2 + 1);
    const int vmin = (int)std::ceil(HALF_PATCH * std::sqrt(2.f) / 2);
    for (int v = 0; v < 16; v++) e->umax[v] = 0;
    for (int v = 0; v <= vmax; ++v) e->umax[v] = (int)lrint(std::sqrt((double)HALF_PATCH * HALF_PATCH - (double)v * v));
    for (int v = HALF_PATCH, v0 = 0; v >= vmin; --v) {
        while (e->umax[v0] == e->umax[v0 + 1]) ++v0;
        e->umax[v] = v0;
        ++v0;
    }
}

// cv::resize INTER_LINEAR 8U coefficient tables (OpenCV imgproc/resize.cpp): {offset, c0, c1, 0} int16 quadruples.
// `extra` > 0 appends entries for the reflect-101 padding columns dst .. dst+extra-1 (copies of the reflected column).
// The entry count is padded to an even number so that every table starts 16-byte aligned.
void resize_table(int src, int dst, bool clamp_edges, int extra, std::vector<int16_t>& out) {
    const double inv = (double)dst / src, scale = 1. / inv;
    const size_t first = out.size();
    for (int d = 0; d < dst; d++) {
        float f = (float)((d + 0.5) * scale - 0.5);
        int s = (int)std::floor(f);
        f -= s;
        if (clamp_edges) {
            if (s < 0) { f = 0; s = 0; }
            if (s >= src - 1) { f = 0; s = src - 1; }
        }
        out.push_back((int16_t)s);
        out.push_back((int16_t)cv_round_f((1.f - f) * 2048.f));
        out.push_back((int16_t)cv_round_f(f * 2048.f));
        out.push_back(0);
    }
    for (int k = 0; k < extra; k++) {
        int r = 2 * dst - 2 - (dst + k);            // reflect-101 of column dst+k
        if (r < 0) r = 0;
        for (int j = 0; j < 4; j++) out.push_back(out[first + (size_t)r * 4 + j]);
    }
    if (((out.size() - first) / 4) & 1) for (int j = 0; j < 4; j++) out.push_back(0);
}

// The x table again, per group of 4 destination columns (one thread of pyr_resize_kernel): {c0, c1, base, selectors}.
// base = first byte of the aligned 12-byte source window the group reads (same in all 4 entries); the selectors
// are the two PRMT controls that pull source bytes (ofs, ofs+1) out of the window words (w0,w1) and then w2:
//   t = prmt(w0, w1, s1), pair = prmt(t, w2, s2), s1 = selectors & 0xFF, s2 = selectors >> 8.
// Returns false if some group spans more than 12 bytes (scale factors above ~2): the caller then uses the generic kernel.
bool resize_window_table(const std::vector<int16_t>& tabs, size_t xtab_first, int n_entries, std::vector<int16_t>& out) {
    bool ok = true;
    for (int gq = 0; gq < n_entries; gq += 4) {
        int lo = 1 << 30, hi = 0;
        for (int i = 0; i < 4; i++) {
            const int ofs = tabs[xtab_first + (size_t)(gq + i) * 4];
            lo = std::min(lo, ofs); hi = std::max(hi, ofs);
        }
        const int base = lo & ~3;
        if (hi + 1 - base > 11) ok = false;
        for (int i = 0; i < 4; i++) {
            const int16_t* e = &tabs[xtab_first + (size_t)(gq + i) * 4];
            const int pos = e[0] - base;
            int s1 = 0, s2 = 0x10;
            if (pos <= 6) s1 = pos | ((pos + 1) << 4);
            else if (pos == 7) { s1 = 7; s2 = 0x40; }
            else { const int q = (pos - 8) + 4; s2 = q | ((q + 1) << 4); }
            out.push_back(e[1]);
            out.push_back(e[2]);
            out.push_back((int16_t)base);
            out.push_back((int16_t)((s1 | (s2 << 8)) & 0x7FFF));
        }
    }
    return ok;
}

const int8_t kPattern[1024] = {          // bit_pattern_31_: (x0, y0, x1, y1) per test
#include "orb_pattern.inc"
};

borb_status build_geometry(borb_extractor* e, int w, int h, std::vector<int16_t>& tabs) {
    Geometry& g = e->geom;
    std::memset(&g, 0, sizeof(g));
    const int L = e->cfg.n_levels;
    g.nlevels = L; g.w = w; g.h = h;
    g.fast_mode = e->fast_mode;
    g.ini_th = e->cfg.ini_th_fast < 0 ? 0 : (e->cfg.ini_th_fast > 255 ? 255 : e->cfg.ini_th_fast);
    g.min_th = e->cfg.min_th_fast < 0 ? 0 : (e->cfg.min_th_fast > 255 ? 255 : e->cfg.min_th_fast);
    for (int i = 0; i < 16; i++) g.umax[i] = e->umax[i];
    unsigned pyr_off = 0, cand_off = 0;
    int blk = 0, sel_off = 0, btile = 0;
    tabs.clear();
    for (int l = 0; l < L; l++) {
        LevelGeom& v = g.lv[l];
        v.w = cv_round_f((float)w * e->inv_scale[l]);
        v.h = cv_round_f((float)h * e->inv_scale[l]);
        const float width = (float)(v.w - 2 * MIN_BORDER), height = (float)(v.h - 2 * MIN_BORDER);
        v.nCols = (int)(width / 30.f);
        v.nRows = (int)(height / 30.f);
        if (v.nCols < 1 || v.nRows < 1) {
            set_error("level %d is %dx%d: too small for the 30-px FAST cell grid (reference divides by zero)", l, v.w, v.h);
            return BORB_ERR_UNSUPPORTED;
        }
        v.wCell = (int)std::ceil(width / v.nCols);
        v.hCell = (int)std::ceil(height / v.nRows);
        v.pitch = align_up(v.w + 8, 128);          // >= 8 bytes of reflect-101 padding after every row
        v.pyr_off = pyr_off;
        pyr_off += (unsigned)v.pitch * v.h;
        v.cellsPerBlk = FAST_TILE_W / v.wCell > 0 ? FAST_TILE_W / v.wCell : 1;
        v.rowsPerBlk = fast_rows_per_blk(v.nRows, v.hCell);
        v.blkCols = (v.nCols + v.cellsPerBlk - 1) / v.cellsPerBlk;
        v.blkBase = blk;
        blk += v.blkCols * ((v.nRows + v.rowsPerBlk - 1) / v.rowsPerBlk);
        v.cand_off = cand_off;
        v.cand_cap = v.nCols * v.nRows * ((v.wCell + 1) / 2) * ((v.hCell + 1) / 2);   // strict 3x3 NMS: <=1 per 2x2
        cand_off += (unsigned)align_up(v.cand_cap, 32);
        v.quota = e->per_level[l];
        v.nIni = (int)std::round(width / height);
        if (v.nIni < 1) { set_error("level %d aspect ratio gives zero quadtree roots (reference divides by zero)", l); return BORB_ERR_UNSUPPORTED; }
        v.hX = width / v.nIni;
        v.node_cap = (v.quota > 4 * v.nIni ? v.quota : 4 * v.nIni) + 3;
        v.node_cap = align_up(v.node_cap + 1, 4);
        v.sel_off = sel_off;
        sel_off += v.node_cap;
        v.scale = e->scale[l];
        v.inv_scale = e->inv_scale[l];
        v.patch_size = (float)(int)(PATCH * e->scale[l]);
        g.blur_base[l] = btile;
        btile += ((v.w + BLUR_TILE_W - 1) / BLUR_TILE_W) * ((v.h + BLUR_TILE_H - 1) / BLUR_TILE_H);   // blur_kernel strips
        if (l > 0) {
            const int wpad = (v.w + 8 + 3) & ~3;     // pixels + reflect padding, whole words
            v.xtab_off = (unsigned)(tabs.size() / 4);
            resize_table(g.lv[l - 1].w, v.w, true, wpad - v.w, tabs);
            v.ytab_off = (unsigned)(tabs.size() / 4);
            resize_table(g.lv[l - 1].h, v.h, false, 0, tabs);
            v.xwin_off = (unsigned)(tabs.size() / 4);
            std::vector<int16_t> win;
            v.x_windowed = resize_window_table(tabs, (size_t)v.xtab_off * 4, wpad, win) ? 1 : 0;
            tabs.insert(tabs.end(), win.begin(), win.end());
        }
        if (quadtree_smem_bytes(v.node_cap) > 200 * 1024) {   // also keeps node_cap < 2^14, which the kernel's 16-bit node ids need
            set_error("per-level quota %d exceeds the quadtree kernel's shared-memory envelope", v.quota);
            return BORB_ERR_UNSUPPORTED;
        }
    }
    g.blur_base[L] = btile;
    g.blur_tiles = btile;
    g.fast_blocks = blk;
    g.pyr_image_stride = (unsigned)align_up((int)pyr_off, g.lv[0].pitch);   // whole level-0 rows: lets batches move as one 3-D copy
    g.cand_image_stride = cand_off;
    g.sel_image_stride = sel_off;
    if (sel_off >= 65536) { set_error("keypoint capacity %d exceeds 65535", sel_off); return BORB_ERR_UNSUPPORTED; }
    return BORB_OK;
}

void free_workspace(Workspace& ws) {
    cudaFree(ws.pyr); cudaFree(ws.blur); cudaFree(ws.cand); cudaFree(ws.cand_cnt); cudaFree(ws.pnode); cudaFree(ws.sel);
    cudaFree(ws.sel_cnt); cudaFree(ws.kps); cudaFree(ws.desc); cudaFree(ws.nkp); cudaFree(ws.u_right); cudaFree(ws.depth);
    cudaFree(ws.sad); cudaFree(ws.tabs); cudaFree(ws.brief_slots); cudaFree(ws.pair_idx); cudaFree(ws.st_bins); cudaFree(ws.st_recs); cudaFree(ws.stage);
    free(ws.fast_tmaps); cudaFree(ws.fast_tiles);
    ws = Workspace();
}

borb_status ensure(borb_extractor* e, int w, int h, int n_images) {
    if (w < 1 || h < 1 || w > BORB_MAX_DIM || h > BORB_MAX_DIM) { set_error("image size %dx%d outside [1,%d]", w, h, BORB_MAX_DIM); return BORB_ERR_UNSUPPORTED; }
    BORB_CUDA(cudaSetDevice(e->device));
    const bool same_shape = e->have_geom && e->geom.w == w && e->geom.h == h;
    if (same_shape && e->ws.max_images >= n_images) return BORB_OK;
    BORB_CUDA(cudaStreamSynchronize(e->stream));
    std::vector<int16_t> tabs;
    e->have_geom = false;
    e->last_n_images = 0;
    e->last_stereo_pairs = 0;
    borb_status st = build_geometry(e, w, h, tabs);
    if (st != BORB_OK) return st;
    size_t n = (size_t)(n_images > 2 ? n_images : 2);
    if (same_shape && (size_t)e->ws.max_images > n) n = (size_t)e->ws.max_images;
    free_workspace(e->ws);
    if (e->h_counts) { cudaFreeHost(e->h_counts); e->h_counts = nullptr; }
    e->pair_cache.clear();
    const Geometry& g = e->geom;
    Workspace& ws = e->ws;
    BORB_CUDA(cudaMalloc(&ws.pyr, n * g.pyr_image_stride + 256));      // +slack: aligned word reads may run a few bytes past the last row
    BORB_CUDA(cudaMalloc(&ws.blur, n * g.pyr_image_stride + 256));
    BORB_CUDA(cudaMalloc(&ws.cand, n * g.cand_image_stride * sizeof(uint32_t)));
    BORB_CUDA(cudaMalloc(&ws.pnode, n * g.cand_image_stride * sizeof(int)));
    BORB_CUDA(cudaMalloc(&ws.cand_cnt, n * g.nlevels * sizeof(int)));
    BORB_CUDA(cudaMalloc(&ws.sel, n * g.sel_image_stride * sizeof(uint32_t)));
    BORB_CUDA(cudaMalloc(&ws.sel_cnt, n * g.nlevels * sizeof(int)));
    BORB_CUDA(cudaMalloc(&ws.kps, n * g.sel_image_stride * sizeof(borb_keypoint)));
    BORB_CUDA(cudaMalloc(&ws.desc, n * g.sel_image_stride * 32));
    BORB_CUDA(cudaMalloc(&ws.nkp, n * sizeof(int)));
    BORB_CUDA(cudaMalloc(&ws.u_right, n * g.sel_image_stride * sizeof(float)));
    BORB_CUDA(cudaMalloc(&ws.depth, n * g.sel_image_stride * sizeof(float)));
    BORB_CUDA(cudaMalloc(&ws.sad, n * g.sel_image_stride * sizeof(int)));
    BORB_CUDA(cudaMalloc(&ws.pair_idx, n * 2 * sizeof(int)));
    BORB_CUDA(cudaMalloc(&ws.st_bins, n * stereo_bins_bytes_per_pair()));
    ws.st_recs_bytes = n * (size_t)stereo_rec_stride(g) * stereo_rec_bytes();
    BORB_CUDA(cudaMalloc(&ws.st_recs, ws.st_recs_bytes));
    BORB_CUDA(cudaMalloc(&ws.tabs, (tabs.size() + 4) * sizeof(int16_t)));
    BORB_CUDA(cudaMemcpy(ws.tabs, tabs.data(), tabs.size() * sizeof(int16_t), cudaMemcpyHostToDevice));
    const std::vector<uint32_t>& slots = brief_slot_table();
    BORB_CUDA(cudaMalloc(&ws.brief_slots, slots.size() * sizeof(uint32_t)));
    BORB_CUDA(cudaMemcpy(ws.brief_slots, slots.data(), slots.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    BORB_CUDA(cudaMemset(ws.nkp, 0, n * sizeof(int)));
    BORB_CUDA(cudaMallocHost(&e->h_counts, n * 2 * sizeof(int)));
    ws.max_images = (int)n;
    ws.fast_tmaps = malloc(fast_tmaps_bytes());
    if ((st = build_fast_tmaps(g, ws, ws.fast_tmaps)) != BORB_OK) return st;
    if ((st = build_fast_tiles(g, ws)) != BORB_OK) return st;
    e->have_geom = true;
    return BORB_OK;
}

void drain_timing(borb_extractor* e);
void begin_step(borb_extractor* e) {
    if (!e->timing) return;
    if (e->ev.empty()) {
        e->ev.resize((size_t)borb_extractor::EV_RING * 9);
        for (auto& x : e->ev) cudaEventCreate(&x);
    }
    if (e->ev_pending >= borb_extractor::EV_RING) {   // ring full: drain (costs a sync, only in timing mode)
        cudaStreamSynchronize(e->stream);
        drain_timing(e);
    }
    e->ev_slot = (e->ev_slot + 1) % borb_extractor::EV_RING;
    e->ev_mask[e->ev_slot] = 0;
    e->ev_pending++;
}
void mark(borb_extractor* e, int i) {
    if (!e->timing || e->ev.empty()) return;
    cudaEventRecord(e->ev[(size_t)e->ev_slot * 9 + i], e->stream);
    e->ev_mask[e->ev_slot] |= 1u << i;
}
// After a stream sync: fold the pending slots into stage_ms / stage_sum_ms.
void drain_timing(borb_extractor* e) {
    const int R = borb_extractor::EV_RING;
    for (int k = e->ev_pending - 1; k >= 0; k--) {
        const int slot = ((e->ev_slot - k) % R + R) % R;
        const unsigned m = e->ev_mask[slot];
        for (int i = 0; i < 8; i++) {
            float ms = 0.f;
            // stage i = [mark i, next recorded mark)
            if (m & (1u << i)) {
                int j = i + 1;
                while (j < 9 && !(m & (1u << j))) j++;
                if (j < 9 && cudaEventElapsedTime(&ms, e->ev[(size_t)slot * 9 + i], e->ev[(size_t)slot * 9 + j]) != cudaSuccess) { ms = 0.f; cudaGetLastError(); }
            }
            e->stage_ms[i] = ms;
            e->stage_sum_ms[i] += ms;
        }
        e->stage_steps++;
    }
    e->ev_pending = 0;
}

// Queues pyramid .. descriptors for n images whose level 0 is already in ws.pyr.
borb_status enqueue_extract(borb_extractor* e, int n) {
    const Geometry& g = e->geom;
    Workspace& ws = e->ws;
    cudaStream_t s = e->stream;
    BORB_CUDA(cudaMemsetAsync(ws.cand_cnt, 0, (size_t)n * g.nlevels * sizeof(int), s));
    mark(e, 1);
    e->launches += launch_pyramid(g, ws, n, s);
    mark(e, 2);
    e->launches += launch_fast(g, ws, n, s);
    mark(e, 3);
    e->launches += launch_quadtree(g, ws, n, s);
    mark(e, 4);
    e->launches += launch_blur(g, ws, n, s);
    mark(e, 5);
    e->launches += launch_describe(g, ws, n, s);
    mark(e, 6);
    BORB_CUDA(cudaGetLastError());
    e->last_n_images = n;
    e->last_stereo_pairs = 0;
    return BORB_OK;
}

// With rectification maps installed the caller hands in RAW frames; the pipeline works on the rectified size.
borb_status rectified_size(borb_extractor* e, int w, int h, int* gw, int* gh) {
    if (!e->d_map[0][0]) return BORB_OK;
    if (w != e->map_src_w || h != e->map_src_h) {
        set_error("rectification maps were built for %dx%d raw frames, got %dx%d", e->map_src_w, e->map_src_h, w, h);
        return BORB_ERR_INVALID_ARG;
    }
    *gw = e->map_dst_w; *gh = e->map_dst_h;
    return BORB_OK;
}

// Host images -> level 0.  slots[k] is the host pointer of batch image k (k = 0..n-1).  When the n images form
// one contiguous block in slot order (camera frames in one pinned buffer) they travel as ONE 1-D copy into a
// packed landing buffer and a kernel re-pitches them; otherwise one 2-D copy per image.
borb_status upload_slots(borb_extractor* e, const uint8_t* const* slots, int n, int w, int h, int stride, bool stereo_pairs = false) {
    const Geometry& g = e->geom;
    const int ch = e->in_channels;
    if (stride < w * ch) { set_error("stride %d smaller than a row of %d %d-channel pixels", stride, w, ch); return BORB_ERR_INVALID_ARG; }
    const size_t img_bytes = (size_t)stride * h;
    bool contiguous = n > 1 || ch > 1 || e->d_map[0][0] != nullptr;
    for (int k = 0; k < n; k++) {
        if (!slots[k]) { set_error("image %d is NULL", k); return BORB_ERR_INVALID_ARG; }
        if (slots[k] != slots[0] + (size_t)k * img_bytes) contiguous = false;
    }
    auto need_stage = [&](size_t need) -> borb_status {
        if (e->ws.stage_bytes < need) {
            BORB_CUDA(cudaStreamSynchronize(e->stream));
            cudaFree(e->ws.stage);
            e->ws.stage = nullptr; e->ws.stage_bytes = 0;
            BORB_CUDA(cudaMalloc(&e->ws.stage, need));
            e->ws.stage_bytes = need;
        }
        return BORB_OK;
    };
    if (e->d_map[0][0]) {               // raw frames: rectify while re-pitching (w, h are the RAW size here)
        if (ch != 1) { set_error("rectification maps apply to CV_8UC1 frames"); return BORB_ERR_UNSUPPORTED; }
        const size_t src_img = contiguous ? img_bytes : (size_t)w * h;
        const int src_stride = contiguous ? stride : w;
        borb_status st = need_stage(src_img * n);
        if (st != BORB_OK) return st;
        if (contiguous) BORB_CUDA(cudaMemcpyAsync(e->ws.stage, slots[0], src_img * n, cudaMemcpyHostToDevice, e->stream));
        else
            for (int k = 0; k < n; k++)
                BORB_CUDA(cudaMemcpy2DAsync(e->ws.stage + (size_t)k * src_img, w, slots[k], stride, w, h, cudaMemcpyHostToDevice, e->stream));
        e->launches += launch_repack_remap(g, e->ws, e->ws.stage, src_stride, src_img, w, h, e->d_map[0][0], e->d_map[0][1],
                                           stereo_pairs ? e->d_map[1][0] : nullptr, stereo_pairs ? e->d_map[1][1] : nullptr, n, e->stream);
        return BORB_OK;
    }
    if (contiguous) {
        const size_t need = img_bytes * n;
        borb_status st = need_stage(need);
        if (st != BORB_OK) return st;
        BORB_CUDA(cudaMemcpyAsync(e->ws.stage, slots[0], need, cudaMemcpyHostToDevice, e->stream));
        if (ch == 1) e->launches += launch_repack(g, e->ws, e->ws.stage, stride, img_bytes, n, e->stream);
        else e->launches += launch_repack_color(g, e->ws, e->ws.stage, stride, img_bytes, ch, e->in_rgb, n, e->stream);
        return BORB_OK;
    }
    if (ch > 1) {                       // scattered colour images: packed landing rows, then the converting re-pitch
        const size_t row = (size_t)w * ch;
        borb_status st = need_stage(row * h * n);
        if (st != BORB_OK) return st;
        for (int k = 0; k < n; k++)
            BORB_CUDA(cudaMemcpy2DAsync(e->ws.stage + (size_t)k * row * h, row, slots[k], stride, row, h, cudaMemcpyHostToDevice, e->stream));
        e->launches += launch_repack_color(g, e->ws, e->ws.stage, (int)row, row * h, ch, e->in_rgb, n, e->stream);
        return BORB_OK;
    }
    for (int k = 0; k < n; k++) {
        uint8_t* dst = e->ws.pyr + (size_t)k * g.pyr_image_stride + g.lv[0].pyr_off;
        BORB_CUDA(cudaMemcpy2DAsync(dst, g.lv[0].pitch, slots[k], stride, w, h, cudaMemcpyHostToDevice, e->stream));
    }
    return BORB_OK;
}

// Device images -> level 0.  With rectification maps installed the images are RAW frames (w, h the raw size) and the remap
// reads them in place; stereo_pairs applies set 1 (when installed) to the odd images, as upload_slots does.  The input
// format of host images does not apply: device images are always CV_8UC1.
borb_status upload_device(borb_extractor* e, const uint8_t* d_gray, int n, int w, int h, size_t pitch, size_t image_stride,
                          bool stereo_pairs = false) {
    const Geometry& g = e->geom;
    if (e->d_map[0][0]) {
        if (pitch > (size_t)INT_MAX) { set_error("pitch %zu too large", pitch); return BORB_ERR_INVALID_ARG; }
        e->launches += launch_repack_remap(g, e->ws, d_gray, (int)pitch, image_stride, w, h, e->d_map[0][0], e->d_map[0][1],
                                           stereo_pairs ? e->d_map[1][0] : nullptr, stereo_pairs ? e->d_map[1][1] : nullptr, n, e->stream);
        return BORB_OK;
    }
    cudaMemcpy3DParms p = {};
    p.srcPtr = make_cudaPitchedPtr((void*)d_gray, pitch, w, image_stride / pitch);
    p.dstPtr = make_cudaPitchedPtr(e->ws.pyr + g.lv[0].pyr_off, g.lv[0].pitch, w, g.pyr_image_stride / g.lv[0].pitch);
    if (image_stride % pitch == 0 && g.pyr_image_stride % g.lv[0].pitch == 0) {
        p.extent = make_cudaExtent(w, h, n);
        p.kind = cudaMemcpyDeviceToDevice;
        BORB_CUDA(cudaMemcpy3DAsync(&p, e->stream));
    } else {
        for (int i = 0; i < n; i++)
            BORB_CUDA(cudaMemcpy2DAsync(e->ws.pyr + (size_t)i * g.pyr_image_stride + g.lv[0].pyr_off, g.lv[0].pitch,
                                        d_gray + (size_t)i * image_stride, pitch, w, h, cudaMemcpyDeviceToDevice, e->stream));
    }
    return BORB_OK;
}

// Queues the D2H copies of keypoints / descriptors / counts of images [first, first+count) step `step`.
borb_status download_kps(borb_extractor* e, int first, int count, int step, borb_keypoint* kps, uint8_t* desc, int cap, int* n_out) {
    const Geometry& g = e->geom;
    const int m = cap < g.sel_image_stride ? cap : g.sel_image_stride;
    cudaStream_t s = e->stream;
    if (kps && m > 0)
        BORB_CUDA(cudaMemcpy2DAsync(kps, (size_t)cap * sizeof(borb_keypoint), e->ws.kps + (size_t)first * g.sel_image_stride,
                                    (size_t)step * g.sel_image_stride * sizeof(borb_keypoint), (size_t)m * sizeof(borb_keypoint),
                                    count, cudaMemcpyDeviceToHost, s));
    if (desc && m > 0)
        BORB_CUDA(cudaMemcpy2DAsync(desc, (size_t)cap * 32, e->ws.desc + (size_t)first * g.sel_image_stride * 32,
                                    (size_t)step * g.sel_image_stride * 32, (size_t)m * 32, count, cudaMemcpyDeviceToHost, s));
    if (n_out)
        BORB_CUDA(cudaMemcpy2DAsync(n_out, sizeof(int), e->ws.nkp + first, (size_t)step * sizeof(int), sizeof(int), count,
                                    cudaMemcpyDeviceToHost, s));
    return BORB_OK;
}

borb_status check_args(borb_extractor* e, int n, int w, int h) {
    if (!e) { set_error("null handle"); return BORB_ERR_INVALID_ARG; }
    if (n < 0) { set_error("negative image count"); return BORB_ERR_INVALID_ARG; }
    (void)w; (void)h;
    return BORB_OK;
}

borb_status enqueue_stereo(borb_extractor* eL, borb_extractor* eR, int n_pairs, const int* left_idx, const int* right_idx,
                           float bf, float b) {
    borb_extractor* e = eL;
    const Geometry& g = e->geom;
    std::vector<int> idx(2 * (size_t)n_pairs);
    for (int p = 0; p < n_pairs; p++) {
        idx[2 * p] = left_idx ? left_idx[p] : (eL == eR ? 2 * p : 0);
        idx[2 * p + 1] = right_idx ? right_idx[p] : (eL == eR ? 2 * p + 1 : 0);
        if (idx[2 * p] < 0 || idx[2 * p] >= eL->last_n_images || idx[2 * p + 1] < 0 || idx[2 * p + 1] >= eR->last_n_images) {
            set_error("stereo pair %d refers to an image outside the last batch", p);
            return BORB_ERR_STATE;
        }
    }
    if (n_pairs > e->ws.max_images) { set_error("too many pairs"); return BORB_ERR_INVALID_ARG; }
    if (idx != e->pair_cache) {
        // the (rarely changing) pair table rides through a pinned staging buffer; wait for earlier work so
        // the staging buffer is not overwritten under a pending copy
        BORB_CUDA(cudaStreamSynchronize(e->stream));
        std::memcpy(e->h_counts, idx.data(), idx.size() * sizeof(int));
        BORB_CUDA(cudaMemcpyAsync(e->ws.pair_idx, e->h_counts, idx.size() * sizeof(int), cudaMemcpyHostToDevice, e->stream));
        e->pair_cache = idx;
    }
    // the records are the RIGHT images' keypoints: with two handles the right one may hold more than the left (nfeatures)
    const int rec_stride = stereo_rec_stride(eR->geom);
    const size_t rec_bytes = (size_t)n_pairs * rec_stride * stereo_rec_bytes();
    if (rec_bytes > e->ws.st_recs_bytes) {
        BORB_CUDA(cudaStreamSynchronize(e->stream));      // earlier stereo launches may still read the old buffer
        cudaFree(e->ws.st_recs);
        e->ws.st_recs = nullptr;
        e->ws.st_recs_bytes = 0;
        BORB_CUDA(cudaMalloc(&e->ws.st_recs, rec_bytes));
        e->ws.st_recs_bytes = rec_bytes;
    }
    StereoView L{eL->ws.pyr, eL->ws.kps, eL->ws.desc, eL->ws.nkp, eL->geom.pyr_image_stride, eL->geom.sel_image_stride};
    StereoView R{eR->ws.pyr, eR->ws.kps, eR->ws.desc, eR->ws.nkp, eR->geom.pyr_image_stride, eR->geom.sel_image_stride};
    mark(e, 6);
    e->launches += launch_stereo(g, L, R, e->ws.pair_idx, n_pairs, bf, b, e->ws.u_right, e->ws.depth, e->ws.sad, g.sel_image_stride,
                                 e->ws.st_bins, e->ws.st_recs, rec_stride, e->stream);
    mark(e, 7);
    BORB_CUDA(cudaGetLastError());
    // borb_stereo_frames_results reads pairs in the default layout (left 2p, right 2p+1 of this handle's batch) only
    e->last_stereo_pairs = (eL == eR && !left_idx && !right_idx) ? n_pairs : 0;
    return BORB_OK;
}

borb_status download_stereo(borb_extractor* e, int n_pairs, float* u_right, float* depth, int cap) {
    const Geometry& g = e->geom;
    const int m = cap < g.sel_image_stride ? cap : g.sel_image_stride;
    if (u_right && m > 0)
        BORB_CUDA(cudaMemcpy2DAsync(u_right, (size_t)cap * 4, e->ws.u_right, (size_t)g.sel_image_stride * 4, (size_t)m * 4, n_pairs, cudaMemcpyDeviceToHost, e->stream));
    if (depth && m > 0)
        BORB_CUDA(cudaMemcpy2DAsync(depth, (size_t)cap * 4, e->ws.depth, (size_t)g.sel_image_stride * 4, (size_t)m * 4, n_pairs, cudaMemcpyDeviceToHost, e->stream));
    return BORB_OK;
}

borb_status finish_timing(borb_extractor* e) {
    if (e->timing && e->ev_pending > 0) drain_timing(e);
    return BORB_OK;
}

}  // namespace

// Plain double math is enough here: the order only groups the taps, every order gives the same descriptor.
const std::vector<uint32_t>& brief_slot_table() {
    static const std::vector<uint32_t> table = [] {
        std::vector<uint32_t> t((size_t)BRIEF_BINS * 512);
        int row[512], col[512], order[512];
        for (int b = 0; b < BRIEF_BINS; b++) {
            const double th = (b + 0.5) * (2.0 * 3.14159265358979323846 / BRIEF_BINS);
            const double a = std::cos(th), s = std::sin(th);
            for (int p = 0; p < 512; p++) {
                const int x = kPattern[2 * p], y = kPattern[2 * p + 1];
                row[p] = (int)std::lround(x * s + y * a);
                col[p] = (int)std::lround(x * a - y * s);
                order[p] = p;
            }
            std::sort(order, order + 512, [&](int i, int j) {
                return row[i] != row[j] ? row[i] < row[j] : (col[i] != col[j] ? col[i] < col[j] : i < j);
            });
            for (int k = 0; k < 512; k++) {
                const int p = order[k];
                t[(size_t)b * 512 + k] = (uint32_t)(kPattern[2 * p] + 128) | (uint32_t)(kPattern[2 * p + 1] + 128) << 8 | (uint32_t)p << 16;
            }
        }
        return t;
    }();
    return table;
}

}  // namespace borb

using namespace borb;

extern "C" {

const char* borb_last_error(void) { return tl_error.c_str(); }
const char* borb_status_str(borb_status s) {
    switch (s) {
        case BORB_OK: return "ok";
        case BORB_ERR_INVALID_ARG: return "invalid argument";
        case BORB_ERR_NO_DEVICE: return "no CUDA device (libborb has no CPU path)";
        case BORB_ERR_CUDA: return "CUDA error";
        case BORB_ERR_UNSUPPORTED: return "unsupported shape or quota";
        case BORB_ERR_CAPACITY: return "output capacity too small";
        case BORB_ERR_STATE: return "invalid call order";
    }
    return "unknown";
}
int borb_version(void) { return BORB_VERSION; }

borb_status borb_device_count(int* n) {
    if (!n) return BORB_ERR_INVALID_ARG;
    *n = 0;
    cudaError_t err = cudaGetDeviceCount(n);
    if (err != cudaSuccess) { *n = 0; cudaGetLastError(); set_error("cudaGetDeviceCount: %s", cudaGetErrorString(err)); return BORB_ERR_NO_DEVICE; }
    return BORB_OK;
}

borb_status borb_host_alloc(void** p, size_t bytes) {
    if (!p) return BORB_ERR_INVALID_ARG;
    BORB_CUDA(cudaMallocHost(p, bytes));
    return BORB_OK;
}
borb_status borb_host_free(void* p) {
    if (p) BORB_CUDA(cudaFreeHost(p));
    return BORB_OK;
}

borb_status borb_extractor_create(const borb_extractor_cfg* cfg, int device, borb_extractor** out) {
    if (!cfg || !out) { set_error("null argument"); return BORB_ERR_INVALID_ARG; }
    *out = nullptr;
    if (cfg->n_levels < 1 || cfg->n_levels > BORB_MAX_LEVELS || cfg->n_features < 1 || !(cfg->scale_factor > 1.0f)) {
        set_error("bad extractor cfg (n_features=%d scale=%f levels=%d)", cfg->n_features, cfg->scale_factor, cfg->n_levels);
        return BORB_ERR_INVALID_ARG;
    }
    int ndev = 0;
    borb_status st = borb_device_count(&ndev);
    if (st != BORB_OK) return st;
    if (ndev < 1) { set_error("no CUDA device visible; libborb has no CPU fallback"); return BORB_ERR_NO_DEVICE; }
    if (device < 0 || device >= ndev) { set_error("device %d out of range (%d visible)", device, ndev); return BORB_ERR_INVALID_ARG; }
    borb_extractor* e = new borb_extractor();
    e->cfg = *cfg;
    e->device = device;
    init_tables(e);
    cudaError_t err = cudaSetDevice(device);
    if (err == cudaSuccess) err = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking);
    if (err != cudaSuccess) {
        set_error("CUDA init failed: %s", cudaGetErrorString(err));
        delete e;
        return BORB_ERR_CUDA;
    }
    *out = e;
    return BORB_OK;
}

borb_status borb_extractor_destroy(borb_extractor* e) {
    if (!e) return BORB_OK;
    cudaSetDevice(e->device);
    if (e->stream) cudaStreamSynchronize(e->stream);
    free_workspace(e->ws);
    for (int a = 0; a < 2; a++)
        for (int c = 0; c < 2; c++) cudaFree(e->d_map[a][c]);
    if (e->h_counts) cudaFreeHost(e->h_counts);
    for (auto& x : e->ev) cudaEventDestroy(x);
    if (e->stream) cudaStreamDestroy(e->stream);
    delete e;
    return BORB_OK;
}

borb_status borb_extractor_tables(const borb_extractor* e, float* scale, float* inv_scale, float* sigma2, float* inv_sigma2,
                                  int32_t* features_per_level) {
    if (!e) return BORB_ERR_INVALID_ARG;
    for (int l = 0; l < e->cfg.n_levels; l++) {
        if (scale) scale[l] = e->scale[l];
        if (inv_scale) inv_scale[l] = e->inv_scale[l];
        if (sigma2) sigma2[l] = e->sigma2[l];
        if (inv_sigma2) inv_sigma2[l] = e->inv_sigma2[l];
        if (features_per_level) features_per_level[l] = e->per_level[l];
    }
    return BORB_OK;
}

borb_status borb_extractor_capacity(const borb_extractor* e, int width, int height, int* cap) {
    if (!e || !cap) return BORB_ERR_INVALID_ARG;
    borb_extractor tmp;
    tmp.cfg = e->cfg; tmp.scale = e->scale; tmp.inv_scale = e->inv_scale; tmp.per_level = e->per_level;
    std::memcpy(tmp.umax, e->umax, sizeof(tmp.umax));
    std::vector<int16_t> tabs;
    if (width < 1 || height < 1 || width > BORB_MAX_DIM || height > BORB_MAX_DIM) { set_error("image size out of range"); return BORB_ERR_UNSUPPORTED; }
    borb_status st = build_geometry(&tmp, width, height, tabs);
    if (st != BORB_OK) return st;
    *cap = tmp.geom.sel_image_stride;
    return BORB_OK;
}

borb_status borb_extractor_reserve(borb_extractor* e, int width, int height, int max_images) {
    if (!e || max_images < 1) return BORB_ERR_INVALID_ARG;
    return ensure(e, width, height, max_images);
}

borb_status borb_sync(borb_extractor* e) {
    if (!e) return BORB_ERR_INVALID_ARG;
    BORB_CUDA(cudaSetDevice(e->device));
    BORB_CUDA(cudaStreamSynchronize(e->stream));
    return finish_timing(e);
}

borb_status borb_extract_batch_enqueue(borb_extractor* e, const uint8_t* const* gray, int n, int w, int h, int stride,
                                       borb_keypoint* kps, uint8_t* desc, int cap, int* n_out) {
    borb_status st = check_args(e, n, w, h);
    if (st != BORB_OK) return st;
    if (n == 0) return BORB_OK;
    if (!gray || cap < 0 || stride < w) { set_error("bad arguments"); return BORB_ERR_INVALID_ARG; }
    int gw = w, gh = h;
    if ((st = rectified_size(e, w, h, &gw, &gh)) != BORB_OK) return st;
    if ((st = ensure(e, gw, gh, n)) != BORB_OK) return st;
    begin_step(e);
    mark(e, 0);
    if ((st = upload_slots(e, gray, n, w, h, stride)) != BORB_OK) return st;
    if ((st = enqueue_extract(e, n)) != BORB_OK) return st;
    mark(e, 7);
    st = download_kps(e, 0, n, 1, kps, desc, cap, n_out);
    mark(e, 8);
    return st;
}

borb_status borb_extract_batch(borb_extractor* e, const uint8_t* const* gray, int n, int w, int h, int stride,
                               borb_keypoint* kps, uint8_t* desc, int cap, int* n_out) {
    if (!n_out) { set_error("n_out is required"); return BORB_ERR_INVALID_ARG; }
    borb_status st = borb_extract_batch_enqueue(e, gray, n, w, h, stride, kps, desc, cap, n_out);
    if (st != BORB_OK) return st;
    if (n == 0) return BORB_OK;
    if ((st = borb_sync(e)) != BORB_OK) return st;
    for (int i = 0; i < n; i++)
        if (n_out[i] > cap) { set_error("image %d produced %d keypoints, capacity %d", i, n_out[i], cap); return BORB_ERR_CAPACITY; }
    return BORB_OK;
}

borb_status borb_extract(borb_extractor* e, const uint8_t* gray, int w, int h, int stride, borb_keypoint* kps, uint8_t* desc,
                         int cap, int* n_out) {
    if (!n_out) { set_error("n_out is required"); return BORB_ERR_INVALID_ARG; }
    *n_out = 0;
    if (!gray || w == 0 || h == 0) return BORB_OK;     // empty image: silent return (ORBextractor.cc:1046-1047)
    const uint8_t* one[1] = {gray};
    return borb_extract_batch(e, one, 1, w, h, stride, kps, desc, cap, n_out);
}

borb_status borb_extract_batch_device(borb_extractor* e, const uint8_t* d_gray, int n, int w, int h, size_t pitch,
                                      size_t image_stride, borb_keypoint* kps, uint8_t* desc, int cap, int* n_out) {
    borb_status st = check_args(e, n, w, h);
    if (st != BORB_OK) return st;
    if (n == 0) return BORB_OK;
    if (!d_gray || pitch < (size_t)w) { set_error("bad arguments"); return BORB_ERR_INVALID_ARG; }
    int gw = w, gh = h;
    if ((st = rectified_size(e, w, h, &gw, &gh)) != BORB_OK) return st;
    if ((st = ensure(e, gw, gh, n)) != BORB_OK) return st;
    begin_step(e);
    mark(e, 0);
    if ((st = upload_device(e, d_gray, n, w, h, pitch, image_stride)) != BORB_OK) return st;
    if ((st = enqueue_extract(e, n)) != BORB_OK) return st;
    mark(e, 7);
    if ((st = download_kps(e, 0, n, 1, kps, desc, cap, n_out)) != BORB_OK) return st;
    mark(e, 8);
    return borb_sync(e);
}

borb_status borb_extractor_set_rectify_maps(borb_extractor* e, int which, const float* map_x, const float* map_y, int src_w, int src_h,
                                            int dst_w, int dst_h) {
    if (!e || which < 0 || which > 1) { set_error("bad arguments"); return BORB_ERR_INVALID_ARG; }
    BORB_CUDA(cudaSetDevice(e->device));
    BORB_CUDA(cudaStreamSynchronize(e->stream));
    if (!map_x || !map_y) {                                  // remove (set 0 removes both)
        for (int s2 = which; s2 < 2; s2++)
            for (int c = 0; c < 2; c++) { cudaFree(e->d_map[s2][c]); e->d_map[s2][c] = nullptr; }
        return BORB_OK;
    }
    if (src_w <= 0 || src_h <= 0 || dst_w <= 0 || dst_h <= 0) { set_error("bad map geometry"); return BORB_ERR_INVALID_ARG; }
    if (which == 1 && (!e->d_map[0][0] || src_w != e->map_src_w || src_h != e->map_src_h || dst_w != e->map_dst_w || dst_h != e->map_dst_h)) {
        set_error("install the left maps (set 0) first; both sets share one geometry"); return BORB_ERR_STATE;
    }
    const size_t bytes = (size_t)dst_w * dst_h * sizeof(float);
    const float* src[2] = {map_x, map_y};
    for (int c = 0; c < 2; c++) {
        cudaFree(e->d_map[which][c]); e->d_map[which][c] = nullptr;
        BORB_CUDA(cudaMalloc(&e->d_map[which][c], bytes));
        BORB_CUDA(cudaMemcpy(e->d_map[which][c], src[c], bytes, cudaMemcpyHostToDevice));
    }
    if (which == 0) {
        e->map_src_w = src_w; e->map_src_h = src_h; e->map_dst_w = dst_w; e->map_dst_h = dst_h;
        for (int c = 0; c < 2; c++) { cudaFree(e->d_map[1][c]); e->d_map[1][c] = nullptr; }      // a new left set invalidates the right one
    }
    return BORB_OK;
}

borb_status borb_extractor_set_input_format(borb_extractor* e, int channels, int rgb_order) {
    if (!e) { set_error("null handle"); return BORB_ERR_INVALID_ARG; }
    if (channels != 1 && channels != 3 && channels != 4) { set_error("channels must be 1, 3 or 4 (CV_8UC1 / C3 / C4)"); return BORB_ERR_INVALID_ARG; }
    e->in_channels = channels;
    e->in_rgb = rgb_order ? 1 : 0;
    return BORB_OK;
}

borb_status borb_extractor_pyramid(borb_extractor* e, int image, int level, uint8_t* dst, int* w, int* h) {
    if (!e || !e->have_geom || image < 0 || image >= e->last_n_images || level < 0 || level >= e->geom.nlevels) {
        set_error("no such image/level in the last batch");
        return BORB_ERR_STATE;
    }
    const LevelGeom& L = e->geom.lv[level];
    if (w) *w = L.w;
    if (h) *h = L.h;
    if (!dst) return BORB_OK;
    BORB_CUDA(cudaSetDevice(e->device));
    BORB_CUDA(cudaMemcpy2DAsync(dst, L.w, e->ws.pyr + (size_t)image * e->geom.pyr_image_stride + L.pyr_off, L.pitch, L.w, L.h,
                                cudaMemcpyDeviceToHost, e->stream));
    BORB_CUDA(cudaStreamSynchronize(e->stream));
    return BORB_OK;
}

borb_status borb_debug_blurred(borb_extractor* e, int image, int level, uint8_t* dst, int* w, int* h) {
    if (!e || !e->have_geom || image < 0 || image >= e->last_n_images || level < 0 || level >= e->geom.nlevels) {
        set_error("no such image/level in the last batch");
        return BORB_ERR_STATE;
    }
    const LevelGeom& L = e->geom.lv[level];
    if (w) *w = L.w;
    if (h) *h = L.h;
    if (!dst) return BORB_OK;
    BORB_CUDA(cudaSetDevice(e->device));
    BORB_CUDA(cudaMemcpy2DAsync(dst, L.w, e->ws.blur + (size_t)image * e->geom.pyr_image_stride + L.pyr_off, L.pitch, L.w, L.h,
                                cudaMemcpyDeviceToHost, e->stream));
    BORB_CUDA(cudaStreamSynchronize(e->stream));
    return BORB_OK;
}

static borb_status debug_list(borb_extractor* e, int image, int level, bool selected, int32_t* xys, int cap, int* n_out) {
    if (!e || !n_out || !e->have_geom || image < 0 || image >= e->last_n_images || level < 0 || level >= e->geom.nlevels) {
        set_error("no such image/level in the last batch");
        return BORB_ERR_STATE;
    }
    const Geometry& g = e->geom;
    const LevelGeom& L = g.lv[level];
    BORB_CUDA(cudaSetDevice(e->device));
    BORB_CUDA(cudaStreamSynchronize(e->stream));
    int n = 0;
    BORB_CUDA(cudaMemcpy(&n, (selected ? e->ws.sel_cnt : e->ws.cand_cnt) + image * g.nlevels + level, sizeof(int), cudaMemcpyDeviceToHost));
    *n_out = n;
    const int m = n < cap ? n : cap;
    if (m <= 0 || !xys) return BORB_OK;
    std::vector<uint32_t> raw(m);
    const uint32_t* src = selected ? e->ws.sel + (size_t)image * g.sel_image_stride + L.sel_off
                                   : e->ws.cand + (size_t)image * g.cand_image_stride + L.cand_off;
    BORB_CUDA(cudaMemcpy(raw.data(), src, (size_t)m * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    for (int i = 0; i < m; i++) { xys[3 * i] = xys_x(raw[i]); xys[3 * i + 1] = xys_y(raw[i]); xys[3 * i + 2] = xys_s(raw[i]); }
    return BORB_OK;
}
borb_status borb_debug_candidates(borb_extractor* e, int image, int level, int32_t* xys, int cap, int* n_out) {
    return debug_list(e, image, level, false, xys, cap, n_out);
}
borb_status borb_debug_selected(borb_extractor* e, int image, int level, int32_t* xys, int cap, int* n_out) {
    return debug_list(e, image, level, true, xys, cap, n_out);
}

borb_status borb_debug_set_fast_mode(borb_extractor* e, int mode) {
    if (!e || mode < 0 || mode > 3) { set_error("fast mode must be 0..3"); return BORB_ERR_INVALID_ARG; }
    e->fast_mode = mode;
    if (e->have_geom) e->geom.fast_mode = mode;
    return BORB_OK;
}

borb_status borb_debug_brief_slots(uint32_t* dst, int cap, int* n_bins) {
    if (!n_bins) { set_error("n_bins is NULL"); return BORB_ERR_INVALID_ARG; }
    const std::vector<uint32_t>& t = brief_slot_table();
    *n_bins = BRIEF_BINS;
    if (dst) std::memcpy(dst, t.data(), std::min((size_t)(cap > 0 ? cap : 0), t.size()) * sizeof(uint32_t));
    return BORB_OK;
}

borb_status borb_debug_eval_math(int fn, const float* a, const float* b, int n, float log_scale, int n_levels, void* out) {
    if (fn < 0 || fn > 4) { set_error("eval_math: no function %d (0..4)", fn); return BORB_ERR_INVALID_ARG; }
    if (n < 0) { set_error("eval_math: n = %d", n); return BORB_ERR_INVALID_ARG; }
    const bool binary = fn == 2 || fn == 4;
    if (!a || !out || (binary && !b)) { set_error("eval_math: NULL input or output"); return BORB_ERR_INVALID_ARG; }
    if (n == 0) return BORB_OK;
    struct Buffers {         // released on every return, after the frees have waited for the stream's work
        cudaStream_t s = nullptr;
        float *a = nullptr, *b = nullptr;
        void* out = nullptr;
        ~Buffers() { cudaFree(a); cudaFree(b); cudaFree(out); if (s) cudaStreamDestroy(s); }
    } d;
    const size_t bytes = (size_t)n * sizeof(float);
    BORB_CUDA(cudaStreamCreateWithFlags(&d.s, cudaStreamNonBlocking));
    BORB_CUDA(cudaMalloc(&d.a, bytes));
    BORB_CUDA(cudaMalloc(&d.out, bytes));
    BORB_CUDA(cudaMemcpyAsync(d.a, a, bytes, cudaMemcpyHostToDevice, d.s));
    if (binary) {
        BORB_CUDA(cudaMalloc(&d.b, bytes));
        BORB_CUDA(cudaMemcpyAsync(d.b, b, bytes, cudaMemcpyHostToDevice, d.s));
    }
    if (fn <= 2) launch_describe_math_probe(fn, d.a, d.b, n, static_cast<float*>(d.out), d.s);
    else launch_match_math_probe(fn, d.a, d.b, n, log_scale, n_levels, d.out, d.s);
    BORB_CUDA(cudaGetLastError());
    BORB_CUDA(cudaMemcpyAsync(out, d.out, bytes, cudaMemcpyDeviceToHost, d.s));
    BORB_CUDA(cudaStreamSynchronize(d.s));
    return BORB_OK;
}

borb_status borb_launch_count(const borb_extractor* e, uint64_t* n) {
    if (!e || !n) return BORB_ERR_INVALID_ARG;
    *n = e->launches;
    return BORB_OK;
}
borb_status borb_set_timing(borb_extractor* e, int enable) {
    if (!e) return BORB_ERR_INVALID_ARG;
    e->timing = enable != 0;
    for (int i = 0; i < 8; i++) { e->stage_sum_ms[i] = 0; e->stage_ms[i] = 0; }
    e->stage_steps = 0;
    e->ev_pending = 0;
    return BORB_OK;
}
borb_status borb_stage_times_total(borb_extractor* e, double* ms8, uint64_t* steps) {
    if (!e || !ms8 || !steps) return BORB_ERR_INVALID_ARG;
    for (int i = 0; i < 8; i++) ms8[i] = e->stage_sum_ms[i];
    *steps = e->stage_steps;
    return BORB_OK;
}
borb_status borb_extractor_stream(borb_extractor* e, void** stream) {
    if (!e || !stream) return BORB_ERR_INVALID_ARG;
    *stream = (void*)e->stream;
    return BORB_OK;
}
borb_status borb_stage_times(borb_extractor* e, float* ms8) {
    if (!e || !ms8) return BORB_ERR_INVALID_ARG;
    for (int i = 0; i < 8; i++) ms8[i] = e->stage_ms[i];
    return BORB_OK;
}

// ------------------------------------------------------------------------------------------- stereo
borb_status borb_stereo_match(borb_extractor* e, int n_pairs, const int* left_idx, const int* right_idx, float bf, float b,
                              float* u_right, float* depth, int cap) {
    if (!e || n_pairs < 0 || !(b > 0.f)) { set_error("bad arguments"); return BORB_ERR_INVALID_ARG; }
    if (!e->have_geom || e->last_n_images == 0) { set_error("stereo match before any extract"); return BORB_ERR_STATE; }
    if (n_pairs == 0) return BORB_OK;
    BORB_CUDA(cudaSetDevice(e->device));
    begin_step(e);
    borb_status st = enqueue_stereo(e, e, n_pairs, left_idx, right_idx, bf, b);
    if (st != BORB_OK) return st;
    if ((st = download_stereo(e, n_pairs, u_right, depth, cap)) != BORB_OK) return st;
    mark(e, 8);
    return borb_sync(e);
}

borb_status borb_stereo_match2(borb_extractor* left, borb_extractor* right, float bf, float b, float* u_right, float* depth, int cap) {
    if (!left || !right || !(b > 0.f)) { set_error("bad arguments"); return BORB_ERR_INVALID_ARG; }
    if (!left->have_geom || !right->have_geom || left->last_n_images < 1 || right->last_n_images < 1) { set_error("stereo match before extract"); return BORB_ERR_STATE; }
    if (left->device != right->device || left->geom.w != right->geom.w || left->geom.h != right->geom.h ||
        left->geom.nlevels != right->geom.nlevels) {
        set_error("left/right extractors differ in device or geometry");
        return BORB_ERR_INVALID_ARG;
    }
    // the match kernel reads both pyramids and both keypoint sets with one scale table (level offsets, pitches, row bands)
    for (int l = 0; l < left->geom.nlevels; l++)
        if (left->geom.lv[l].scale != right->geom.lv[l].scale) {
            set_error("left/right extractors differ in scale factor at level %d (%g vs %g)", l, (double)left->geom.lv[l].scale,
                      (double)right->geom.lv[l].scale);
            return BORB_ERR_INVALID_ARG;
        }
    BORB_CUDA(cudaSetDevice(left->device));
    BORB_CUDA(cudaStreamSynchronize(right->stream));   // right results must be complete before left's stream reads them
    begin_step(left);
    borb_status st = enqueue_stereo(left, right, 1, nullptr, nullptr, bf, b);
    if (st != BORB_OK) return st;
    if ((st = download_stereo(left, 1, u_right, depth, cap)) != BORB_OK) return st;
    mark(left, 8);
    return borb_sync(left);
}

borb_status borb_stereo_frames_enqueue(borb_extractor* e, const uint8_t* const* left, const uint8_t* const* right, int n_pairs,
                                       int w, int h, int stride, float bf, float b, borb_keypoint* kps_left, uint8_t* desc_left,
                                       int* n_left, borb_keypoint* kps_right, uint8_t* desc_right, int* n_right, float* u_right,
                                       float* depth, int cap) {
    borb_status st = check_args(e, n_pairs, w, h);
    if (st != BORB_OK) return st;
    if (n_pairs == 0) return BORB_OK;
    if (!left || !right || stride < w || !(b > 0.f)) { set_error("bad arguments"); return BORB_ERR_INVALID_ARG; }
    int gw = w, gh = h;
    if ((st = rectified_size(e, w, h, &gw, &gh)) != BORB_OK) return st;
    if ((st = ensure(e, gw, gh, 2 * n_pairs)) != BORB_OK) return st;
    begin_step(e);
    mark(e, 0);
    {
        std::vector<const uint8_t*> slots(2 * (size_t)n_pairs);
        for (int p = 0; p < n_pairs; p++) { slots[2 * p] = left[p]; slots[2 * p + 1] = right[p]; }
        if ((st = upload_slots(e, slots.data(), 2 * n_pairs, w, h, stride, true)) != BORB_OK) return st;
    }
    if ((st = enqueue_extract(e, 2 * n_pairs)) != BORB_OK) return st;
    if ((st = enqueue_stereo(e, e, n_pairs, nullptr, nullptr, bf, b)) != BORB_OK) return st;
    if ((st = download_kps(e, 0, n_pairs, 2, kps_left, desc_left, cap, n_left)) != BORB_OK) return st;
    if ((st = download_kps(e, 1, n_pairs, 2, kps_right, desc_right, cap, n_right)) != BORB_OK) return st;
    if ((st = download_stereo(e, n_pairs, u_right, depth, cap)) != BORB_OK) return st;
    mark(e, 8);
    return BORB_OK;
}

borb_status borb_stereo_frames(borb_extractor* e, const uint8_t* const* left, const uint8_t* const* right, int n_pairs, int w,
                               int h, int stride, float bf, float b, borb_keypoint* kps_left, uint8_t* desc_left, int* n_left,
                               borb_keypoint* kps_right, uint8_t* desc_right, int* n_right, float* u_right, float* depth, int cap) {
    borb_status st = borb_stereo_frames_enqueue(e, left, right, n_pairs, w, h, stride, bf, b, kps_left, desc_left, n_left,
                                                kps_right, desc_right, n_right, u_right, depth, cap);
    if (st != BORB_OK || n_pairs == 0) return st;
    if ((st = borb_sync(e)) != BORB_OK) return st;
    for (int p = 0; p < n_pairs; p++)
        if ((n_left && n_left[p] > cap) || (n_right && n_right[p] > cap)) { set_error("pair %d exceeds capacity %d", p, cap); return BORB_ERR_CAPACITY; }
    return BORB_OK;
}

borb_status borb_stereo_frames_device_enqueue(borb_extractor* e, const uint8_t* d_gray, int n_pairs, int w, int h, size_t pitch,
                                              size_t image_stride, float bf, float b, int* n_left, int* n_right, float* u_right,
                                              float* depth, int cap) {
    borb_status st = check_args(e, n_pairs, w, h);
    if (st != BORB_OK) return st;
    if (n_pairs == 0) return BORB_OK;
    if (!d_gray || pitch < (size_t)w || !(b > 0.f)) { set_error("bad arguments"); return BORB_ERR_INVALID_ARG; }
    int gw = w, gh = h;
    if ((st = rectified_size(e, w, h, &gw, &gh)) != BORB_OK) return st;
    if ((st = ensure(e, gw, gh, 2 * n_pairs)) != BORB_OK) return st;
    begin_step(e);
    mark(e, 0);
    if ((st = upload_device(e, d_gray, 2 * n_pairs, w, h, pitch, image_stride, true)) != BORB_OK) return st;
    if ((st = enqueue_extract(e, 2 * n_pairs)) != BORB_OK) return st;
    if ((st = enqueue_stereo(e, e, n_pairs, nullptr, nullptr, bf, b)) != BORB_OK) return st;
    if ((st = download_kps(e, 0, n_pairs, 2, nullptr, nullptr, cap, n_left)) != BORB_OK) return st;
    if ((st = download_kps(e, 1, n_pairs, 2, nullptr, nullptr, cap, n_right)) != BORB_OK) return st;
    if ((st = download_stereo(e, n_pairs, u_right, depth, cap)) != BORB_OK) return st;
    mark(e, 8);
    return BORB_OK;
}

borb_status borb_stereo_frames_device(borb_extractor* e, const uint8_t* d_gray, int n_pairs, int w, int h, size_t pitch,
                                      size_t image_stride, float bf, float b, int* n_left, int* n_right, float* u_right,
                                      float* depth, int cap) {
    borb_status st = borb_stereo_frames_device_enqueue(e, d_gray, n_pairs, w, h, pitch, image_stride, bf, b, n_left, n_right,
                                                       u_right, depth, cap);
    if (st != BORB_OK || n_pairs == 0) return st;
    return borb_sync(e);
}

borb_status borb_stereo_frames_results(borb_extractor* e, int n_pairs, borb_keypoint* kps_left, uint8_t* desc_left, int* n_left,
                                       borb_keypoint* kps_right, uint8_t* desc_right, int* n_right, float* u_right, float* depth,
                                       int cap) {
    if (!e || n_pairs < 0 || cap < 0) { set_error("bad arguments"); return BORB_ERR_INVALID_ARG; }
    if (n_pairs == 0) return BORB_OK;
    if (!e->have_geom || n_pairs > e->last_stereo_pairs) {
        set_error("the last call on this handle left stereo results for %d pairs, %d requested", e->last_stereo_pairs, n_pairs);
        return BORB_ERR_STATE;
    }
    BORB_CUDA(cudaSetDevice(e->device));
    borb_status st;
    if ((st = download_kps(e, 0, n_pairs, 2, kps_left, desc_left, cap, n_left)) != BORB_OK) return st;
    if ((st = download_kps(e, 1, n_pairs, 2, kps_right, desc_right, cap, n_right)) != BORB_OK) return st;
    if ((st = download_stereo(e, n_pairs, u_right, depth, cap)) != BORB_OK) return st;
    if ((st = borb_sync(e)) != BORB_OK) return st;
    std::vector<int> counts(2 * (size_t)n_pairs);
    BORB_CUDA(cudaMemcpy(counts.data(), e->ws.nkp, counts.size() * sizeof(int), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < counts.size(); i++)
        if (counts[i] > cap) { set_error("pair %d exceeds capacity %d", (int)(i / 2), cap); return BORB_ERR_CAPACITY; }
    return BORB_OK;
}

}  // extern "C"
