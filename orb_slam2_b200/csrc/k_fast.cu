// FAST-9/16 score map + cell-local strict 3x3 NMS + per-cell ini/min threshold selection, for every
// level of every image of the batch in ONE launch.
//
// Replaces the per-cell cv::FAST loop of ORBextractor::ComputeKeyPointsOctTree (reference
// src/ORBextractor.cc:784-829; OpenCV features2d/fast.cpp FAST_t<16> + cornerScore<16>) using the
// whole-level reformulation of SURVEY §8(a3), verified identical to the per-cell loop in
// tests/test_oracle_extract.py:
//   S(p)    = max over the 16 nine-pixel arcs (both polarities) of min |I_p - I_q|, minus 1
//             (p is a corner at threshold t  <=>  S(p) >= t);
//   keep(p) = S(p) strictly greater than S(q) for the 8-neighbours q that lie in the SAME cell's
//             detection domain (neighbours outside count as 0);
//   a cell emits keep(p) with S>=iniTh if any exists, else keep(p) with S>=minTh.
// One CTA owns `cellsPerBlk` whole cells of one cell row, so NMS and the threshold decision are CTA-local.
//
// Pipeline inside a CTA (v3):
//   0. one elected thread issues a 3-D TMA tile load (cp.async.bulk.tensor, box 160 x (hCell+6) bytes at
//      ((x0-4)&~15, y0-3, image): the inner start coordinate must be 16-byte aligned) into shared memory
//      and everybody waits on its mbarrier;
//   1. a thread owns the 4 pixels of one ALIGNED 32-bit word of the tile and slides down its rows with a
//      7-row register window.  Cheap reject: per even ring position one VABSDIFF4 gives |I_q - I_p| for the
//      4 pixels and three logic ops a per-byte ">t" flag; a FAST-9 arc contains a pixel of each antipodal
//      ring pair, so AND_j (f_j | f_{j+8}) == 0 rejects.  Surviving words are scored EXACTLY: ring
//      differences as s16x2 lanes (two pixels per register), S = max(max_k min_{j<9} d_{k+j},
//      -min_k max_{j<9} d_{k+j}) - 1 with VIMNMX3.S16x2 (min3/max3) networks — the corner test IS the score
//      (corner at t <=> S >= t).  Survivors are pushed to a shared-memory word queue and scored in a second
//      pass with all lanes busy.  This pass runs at iniThFAST only; cells that end up without a kept corner
//      are redone at minThFAST afterwards (pass B), exactly the reference's per-cell fallback;
//   2. cell-local strict NMS over the queued corners;  3. per-cell threshold decision and warp-aggregated
//      append to the global candidate list.
// Output: unordered candidate list per (image, level) of packed (x,y,score); consumers break ties with
// the reference's emission order key (cell row, cell col, y, x), never with list position.
//
// Bound (target): HBM read of the level pixels, once — sum_l w_l*h_l bytes per image.  In practice the integer ALU pipe
// (LOP3/PRMT/VABSDIFF4/VIMNMX3) bounds it: a bit-exact FAST-9 needs tens of integer operations per pixel — see DESIGN.md.
#include <cuda.h>

#include <cstring>

#include "borb_internal.h"

#include <algorithm>
#include <vector>

namespace borb {

namespace {

constexpr int TP = 160;                 // TMA box width == smem tile pitch (bytes).  TMA needs a 16-byte aligned start
                                        // column, so the box starts at xs = (x0-4) & ~15 and domain px xx sits at column xx+off
constexpr int TROWS = 66;               // hCell <= 60, + 3 halo rows above and below
constexpr int QCAP = 60 * 128;          // queue capacity >= every pixel of the largest tile

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// 4-byte window starting DX bytes after the start of W1 (W0|W1|W2 are three consecutive aligned words)
template <int DX>
__device__ __forceinline__ uint32_t win(uint32_t W0, uint32_t W1, uint32_t W2) {
    if (DX == 0) return W1;
    if (DX > 0) return __byte_perm(W1, W2, DX | ((DX + 1) << 4) | ((DX + 2) << 8) | ((DX + 3) << 12));
    constexpr int K = 4 + DX;
    return __byte_perm(W0, W1, K | ((K + 1) << 4) | ((K + 2) << 8) | ((K + 3) << 12));
}

// CONSERVATIVE reject flag, 3 instructions (VABSDIFF4, IADD, LOP3): bit 7 of every byte of the result is set if that
// byte of a = |q - v| exceeds t (K = (127-t)*0x01010101, t <= 127).  Per byte a + (127-t) >= 128 <=> a > t; a byte whose
// sum overflows has a >= 129 (bit 7 of a itself, OR-ed in).  The carry out of an overflowing byte can raise the next
// byte's flag when that byte has a == t exactly: a false "keep", which only sends the word to the exact scoring pass
// (pass 1b decides every corner from exact scores), never a false reject.
__device__ __forceinline__ uint32_t gt_flag(uint32_t q, uint32_t v, uint32_t K) {
    const uint32_t a = __vabsdiffu4(q, v);
    return (a + K) | a;
}

// Exact FAST scores of the 4 pixels of one aligned word.  R0/R1/R2[j]: the three aligned words (px -4..-1, 0..3,
// 4..7 relative to the word) of tile rows dy = j-3.  Returns 4 bytes: S(p) clamped to [0,254]; S(p) >= t <=> p
// is a FAST-9 corner at threshold t (cornerScore<16> of OpenCV for every pixel, both polarities at once).
__device__ __forceinline__ uint32_t score_word(const uint32_t (&R0)[7], const uint32_t (&R1)[7], const uint32_t (&R2)[7]) {
#define ROWJ(dy) R0[(dy) + 3], R1[(dy) + 3], R2[(dy) + 3]
    uint32_t wn[16];
    wn[0] = win<0>(ROWJ(3));    wn[1] = win<1>(ROWJ(3));    wn[2] = win<2>(ROWJ(2));     wn[3] = win<3>(ROWJ(1));
    wn[4] = win<3>(ROWJ(0));    wn[5] = win<3>(ROWJ(-1));   wn[6] = win<2>(ROWJ(-2));    wn[7] = win<1>(ROWJ(-3));
    wn[8] = win<0>(ROWJ(-3));   wn[9] = win<-1>(ROWJ(-3));  wn[10] = win<-2>(ROWJ(-2));  wn[11] = win<-3>(ROWJ(-1));
    wn[12] = win<-3>(ROWJ(0));  wn[13] = win<-3>(ROWJ(1));  wn[14] = win<-2>(ROWJ(2));   wn[15] = win<-1>(ROWJ(3));
#undef ROWJ
    const uint32_t v = R1[3];
    uint32_t res[2];
#pragma unroll
    for (int half = 0; half < 2; half++) {
        // half 0: pixels 0 and 2 (even bytes) as two s16 lanes; half 1: pixels 1 and 3 (odd bytes)
        const uint32_t v2 = half ? __byte_perm(v, 0u, 0x4341) : (v & 0x00FF00FFu);
        const uint32_t nv2 = __vneg2(v2);
        uint32_t d[16];
#pragma unroll
        for (int k = 0; k < 16; k++) {
            const uint32_t q2 = half ? __byte_perm(wn[k], 0u, 0x4341) : (wn[k] & 0x00FF00FFu);
            d[k] = __vadd2(q2, nv2);                       // I_q - I_p per lane, in [-255, 255]
        }
        uint32_t lo3[16], hi3[16];
#pragma unroll
        for (int k = 0; k < 16; k++) {
            lo3[k] = __vimin3_s16x2(d[k], d[(k + 1) & 15], d[(k + 2) & 15]);
            hi3[k] = __vimax3_s16x2(d[k], d[(k + 1) & 15], d[(k + 2) & 15]);
        }
        uint32_t lo9[16], hi9[16];
#pragma unroll
        for (int k = 0; k < 16; k++) {
            lo9[k] = __vimin3_s16x2(lo3[k], lo3[(k + 3) & 15], lo3[(k + 6) & 15]);   // min over the arc k..k+8
            hi9[k] = __vimax3_s16x2(hi3[k], hi3[(k + 3) & 15], hi3[(k + 6) & 15]);   // max over the arc k..k+8
        }
        uint32_t bb[5], dd[5];
#pragma unroll
        for (int k = 0; k < 5; k++) {
            bb[k] = __vimax3_s16x2(lo9[3 * k], lo9[3 * k + 1], lo9[3 * k + 2]);
            dd[k] = __vimin3_s16x2(hi9[3 * k], hi9[3 * k + 1], hi9[3 * k + 2]);
        }
        const uint32_t bright = __vimax3_s16x2(__vimax3_s16x2(bb[0], bb[1], bb[2]), __vimax3_s16x2(bb[3], bb[4], lo9[15]), bb[0]);
        const uint32_t darkm = __vimin3_s16x2(__vimin3_s16x2(dd[0], dd[1], dd[2]), __vimin3_s16x2(dd[3], dd[4], hi9[15]), dd[0]);
        // S = max(bright, -darkm) - 1, clamped at 0
        res[half] = __viaddmax_s16x2_relu(__vmaxs2(bright, __vneg2(darkm)), 0xFFFFFFFFu, 0u);
    }
    // lanes hold 0..254: bytes  px0 = res0.lo, px1 = res1.lo, px2 = res0.hi, px3 = res1.hi
    return res[1] * 256u + res[0];
}

}  // namespace

struct TMaps { CUtensorMap m[BORB_MAX_LEVELS]; };

// One FAST CTA = whole cells of one cell row of one level.  The tile geometry is the same for every image of a batch, so it
// is computed once on the host (build_fast_tiles) instead of ~110 instructions per CTA (8.7 % of the kernel's instructions).
struct __align__(16) FastTile { int16_t l, ncell, x0, x1, y0, y1, wCell, hCell; };

__global__ void __launch_bounds__(256, 4) fast_kernel(const __grid_constant__ Geometry g, const __grid_constant__ TMaps tm,
                                                   const FastTile* __restrict__ tiles, uint32_t* __restrict__ cand, int* __restrict__ cand_cnt) {
    __shared__ __align__(128) uint8_t tile[TROWS * TP];
    __shared__ __align__(16) uint8_t score[60 * TP];     // S(p) in TILE coordinates (same columns as `tile`)
    __shared__ uint16_t queue[QCAP];                      // corners: row << 8 | tile column
    __shared__ uint16_t wqueue[8 * 256];                  // words (row << 5 | lane) deferred to the dense scoring pass: one 256-entry
    __shared__ int wcnt[8];                               // segment per warp (a warp owns <= 8 rows), filled without atomics
    __shared__ __align__(8) unsigned long long bar;
    __shared__ uint32_t scoredRow[60];                    // per tile row: lanes whose word has an exact score in `score`
    __shared__ int qn, needB;
    __shared__ int cellHasIni[128 / 30 + 1];
    __shared__ uint8_t cellOf[128];

    const int img = blockIdx.y;
    const FastTile T = tiles[blockIdx.x];                // one 16-byte load (only non-empty tiles are in the table)
    const int l = T.l, ncell = T.ncell, x0 = T.x0, x1 = T.x1, y0 = T.y0, y1 = T.y1;
    const int wCell = T.wCell, hCell = T.hCell;
    const LevelGeom& L = g.lv[l];
    const int tw = x1 - x0, th = y1 - y0;
    const int tid = threadIdx.x;
    const int lane = tid & 31, wrp = tid >> 5;

    // ---- 0. TMA: tile rows y0-3 .. y0+hCell+2, columns xs .. xs+159 of image `img`, level l
    const int xs = (x0 - 4) & ~15;          // 16-byte aligned box start (TMA requirement)
    const int off = x0 - xs;                // tile column of domain pixel xx = 0   (4..19)
    if (tid == 0) {
        // the issuing thread initialises the barrier itself, so the copy starts before the CTA's first barrier; the other
        // threads see the initialised mbarrier after the __syncthreads() below and only then wait on it
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const uint32_t bytes = (uint32_t)TP * (uint32_t)(hCell + 6);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar)), "r"(bytes) : "memory");
        asm volatile(
            "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
            ::"r"(smem_u32(tile)), "l"(reinterpret_cast<uint64_t>(&tm.m[l])), "r"(xs), "r"(y0 - 3), "r"(img), "r"(smem_u32(&bar))
            : "memory");
    }
    // overlap with the copy: bookkeeping
    if (tid < 128 / 30 + 1) cellHasIni[tid] = 0;
    if (tid < 128) cellOf[tid] = (uint8_t)(tid / wCell);
    if (tid == 0) { qn = 0; needB = 0; }
    __syncthreads();
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "FAST_TMA_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n"
        "@p bra FAST_TMA_DONE;\n"
        "bra FAST_TMA_WAIT;\n"
        "FAST_TMA_DONE:\n"
        "}\n" ::"r"(smem_u32(&bar))
        : "memory");
    // no CTA barrier here: every thread has observed the mbarrier phase itself (acquire), the bookkeeping stores above are
    // ordered by the __syncthreads() before the wait
    if (g.fast_mode == 1) {                 // ablation: tile load only (one word per thread consumed so the copy is observed)
        if (reinterpret_cast<const uint32_t*>(tile)[tid] == 0x12345678u && cand_cnt[0] == -1) cand[0] = 1;
        return;
    }

    // Pass A works at iniThFAST only: a cell falls back to minThFAST only if it has NO kept corner at iniThFAST
    // (ORBextractor.cc:809-816), and a pixel with S < ini can neither be kept at ini nor suppress one that is.
    const int tlow = g.ini_th;
    const uint32_t* T32 = reinterpret_cast<const uint32_t*>(tile);
    uint32_t* S32 = reinterpret_cast<uint32_t*>(score);
    const int wbase = off >> 2;             // lane owns aligned tile word wbase+lane (tile columns 4*(wbase+lane) .. +3)
    const uint32_t T1 = (uint32_t)(127 - min(tlow, 127)) * 0x01010101u;      // gt_flag's K
    const uint32_t TC = (uint32_t)min(max(tlow, 1), 128) * 0x01010101u;   // corner flag: S >= max(tlow,1)
    const bool reject_ok = tlow <= 127;

    // Writes one scored word to the score map and appends its corner pixels (S >= tlow, inside the domain) to the
    // corner queue.  Must be called by all 32 lanes (write = false for lanes without work).
    auto commit = [&](uint32_t sw, int yy, int wc, bool write, int tlow, uint32_t TC, uint32_t needMask) {
        const int col = 4 * wc;
        uint32_t vm = 0;
#pragma unroll
        for (int b = 0; b < 4; b++)
            if (col + b - off >= 0 && col + b - off < tw) vm |= 0x80u << (8 * b);
        if (write) S32[yy * (TP / 4) + wc] = sw;
        // bit 7 per byte: S >= TC byte (TC <= 128)
        uint32_t m = (((sw | 0x80808080u) - TC) | sw) & vm & needMask;
        if (tlow > 128) {       // never used by the reference configs: exact per-byte compare
            m = 0;
#pragma unroll
            for (int b = 0; b < 4; b++)
                if ((int)((sw >> (8 * b)) & 0xFF) >= tlow) m |= 0x80u << (8 * b);
            m &= vm & needMask;
        }
        if (!write) m = 0;
        const unsigned any = __ballot_sync(0xFFFFFFFFu, m != 0);
        if (any) {
            const int c = __popc(m);
            int incl = c;
#pragma unroll
            for (int o2 = 1; o2 < 32; o2 <<= 1) {
                const int t = __shfl_up_sync(0xFFFFFFFFu, incl, o2);
                if (lane >= o2) incl += t;
            }
            int base = 0;
            if (lane == 31) base = atomicAdd(&qn, incl);
            base = __shfl_sync(0xFFFFFFFFu, base, 31) + incl - c;
            uint32_t mm = m;
            while (mm) {
                const int b = (__ffs(mm) - 1) >> 3;
                mm &= mm - 1;
                queue[base++] = (uint16_t)((yy << 8) | (col + b));
            }
        }
    };

    // ---- 1a. slide down the rows: cheap reject, then score in place (dense warps) or defer (sparse warps)
    {
        const int RG = (th + 7) >> 3;                 // rows per warp (8 warps)
        const int yBeg = wrp * RG, yEnd = min(th, yBeg + RG);
        const int wc = wbase + lane;
        uint32_t vmask = 0;
#pragma unroll
        for (int b = 0; b < 4; b++)
            if (4 * wc + b - off >= 0 && 4 * wc + b - off < tw) vmask |= 0x80u << (8 * b);
        // rolling window of 7 tile rows x 3 words; slot (j % 7) holds tile row (yy + j), j = 0..6 <=> dy = j-3
        uint32_t a0[7], a1[7], a2[7];
        int wcount = 0;
        if (yBeg < yEnd) {
#pragma unroll
            for (int j = 0; j < 6; j++) {
                const uint32_t* rp = T32 + (yBeg + j) * (TP / 4) + wc - 1;
                a0[j] = rp[0]; a1[j] = rp[1]; a2[j] = rp[2];
            }
        }
#pragma unroll
        for (int it = 0; it < 8; it++) {
            const int yy = yBeg + it;
            if (yy < yEnd) {          // warp-uniform
                {
                    const uint32_t* rp = T32 + (yy + 6) * (TP / 4) + wc - 1;
                    a0[(it + 6) % 7] = rp[0]; a1[(it + 6) % 7] = rp[1]; a2[(it + 6) % 7] = rp[2];
                }
#define ROW(dy) a0[(it + (dy) + 3) % 7], a1[(it + (dy) + 3) % 7], a2[(it + (dy) + 3) % 7]
                bool keep = vmask != 0;
                if (reject_ok && keep) {
                    const uint32_t v = a1[(it + 3) % 7];
                    uint32_t acc = gt_flag(win<0>(ROW(3)), v, T1) | gt_flag(win<0>(ROW(-3)), v, T1);      // pair (0,8)
                    acc &= gt_flag(win<2>(ROW(2)), v, T1) | gt_flag(win<-2>(ROW(-2)), v, T1);               // (2,10)
                    acc &= gt_flag(win<3>(ROW(0)), v, T1) | gt_flag(win<-3>(ROW(0)), v, T1);                // (4,12)
                    acc &= gt_flag(win<2>(ROW(-2)), v, T1) | gt_flag(win<-2>(ROW(2)), v, T1);               // (6,14)
                    keep = (acc & vmask) != 0;
                }
#undef ROW
                const unsigned bal = __ballot_sync(0xFFFFFFFFu, keep);
                if (lane == 0) scoredRow[yy] = bal;
                // rejected words are final (S < iniTh: recorded as 0); survivors are scored in pass 1b with all lanes busy
                if (!keep && vmask != 0) S32[yy * (TP / 4) + wc] = 0;
                if (keep) wqueue[wrp * 256 + wcount + __popc(bal & ((1u << lane) - 1))] = (uint16_t)((yy << 5) | lane);
                wcount += __popc(bal);               // warp-uniform: the warp's segment needs no atomic
            }
        }
        if (lane == 0) wcnt[wrp] = wcount;
    }
    __syncthreads();
    if (g.fast_mode == 2) {                 // ablation: load + packed reject
        if (wcnt[0] == -1) cand[0] = 1;
        return;
    }

    // ---- 1b. dense scoring pass over the deferred words (the 8 segments read as one list)
    {
        int c[8], nw = 0;
#pragma unroll
        for (int w = 0; w < 8; w++) { c[w] = wcnt[w]; nw += c[w]; }
        for (int eb = 0; eb < nw; eb += 256) {
            const int e = eb + tid;
            uint32_t sw = 0;
            int yy = 0, wc = wbase;
            const bool have = e < nw;
            if (have) {
                int seg = 0, r = e;
#pragma unroll
                for (int w = 0; w < 7; w++)
                    if (seg == w && r >= c[w]) { r -= c[w]; seg = w + 1; }
                const int we = wqueue[seg * 256 + r];
                yy = we >> 5;
                wc = wbase + (we & 31);
                uint32_t R0[7], R1[7], R2[7];
#pragma unroll
                for (int j = 0; j < 7; j++) {
                    const uint32_t* rp = T32 + (yy + j) * (TP / 4) + wc - 1;
                    R0[j] = rp[0]; R1[j] = rp[1]; R2[j] = rp[2];
                }
                sw = score_word(R0, R1, R2);
            }
            commit(sw, yy, wc, have, tlow, TC, 0xFFFFFFFFu);
        }
    }
    __syncthreads();
    int nq = qn;
    if (g.fast_mode == 3) {                 // ablation: load + reject + exact scores
        if (nq == -1) cand[0] = 1;
        return;
    }

    uint32_t* out = cand + (size_t)img * g.cand_image_stride + L.cand_off;
    int* cnt = cand_cnt + img * g.nlevels + l;

    // cell-local strict NMS over queue[0..n) (0xFFFF = dropped); optionally records which cells keep something
    auto nms = [&](int n, bool mark) {
        for (int e = tid; e < n; e += 256) {
            const int q = queue[e];
            const int col = q & 255, yy = q >> 8;
            const int xx = col - off;
            const int s = score[yy * TP + col];
            const int c = cellOf[xx];
            const int cx0 = c * wCell, cx1 = min(cx0 + wCell, tw);
            bool ismax = true;
#pragma unroll
            for (int dy = -1; dy <= 1; dy++)
#pragma unroll
                for (int dx = -1; dx <= 1; dx++) {
                    if (dx == 0 && dy == 0) continue;
                    const int qx = xx + dx, qy = yy + dy;
                    if (qx < cx0 || qx >= cx1 || qy < 0 || qy >= th) continue;
                    if (!(s > (int)score[qy * TP + col + dx])) ismax = false;
                }
            if (ismax) {
                if (mark) cellHasIni[c] = 1;
            } else
                queue[e] = 0xFFFF;
        }
    };
    // warp-aggregated append of the surviving queue entries to the global candidate list
    auto emit = [&](int n) {
        for (int eb = 0; eb < n; eb += 256) {
            const int e = eb + tid;
            int s = 0, xx = 0, yy = 0;
            if (e < n) {
                const int q = queue[e];
                if (q != 0xFFFF) {
                    const int col = q & 255;
                    yy = q >> 8; xx = col - off;
                    s = score[yy * TP + col];
                }
            }
            const unsigned m = __ballot_sync(0xFFFFFFFFu, s > 0);
            if (m) {
                int base = 0;
                if (lane == 0) base = atomicAdd(cnt, __popc(m));
                base = __shfl_sync(0xFFFFFFFFu, base, 0);
                if (s > 0) {
                    const int pos = base + __popc(m & ((1u << lane) - 1));
                    if (pos < L.cand_cap) out[pos] = pack_xys(x0 + xx, y0 + yy, s);
                }
            }
        }
    };

    // ---- 2. pass A: NMS among the S >= iniTh corners; every survivor is emitted and marks its cell
    nms(nq, true);
    __syncthreads();
    emit(nq);
    if (tid < ncell && tid * wCell < tw && !cellHasIni[tid] && g.min_th < g.ini_th) needB = 1;
    __syncthreads();
    if (!needB) return;

    // ---- 3. pass B (rare): cells without any kept iniTh corner are redone at minThFAST (ORBextractor.cc:812-816).
    //         Words of those cells that pass A rejected (S < ini, not necessarily < min) are scored now.
    {
        if (tid == 0) qn = 0;
        __syncthreads();
        const int tmin = g.min_th;
        const uint32_t T1b = (uint32_t)(127 - min(tmin, 127)) * 0x01010101u;
        const uint32_t TCb = (uint32_t)min(max(tmin, 1), 128) * 0x01010101u;
        const int nwords = th * 32;
        for (int wb = 0; wb < nwords; wb += 256) {
            const int widx = wb + tid;
            const int yy = widx >> 5;           // warp-uniform: 32 consecutive threads share a row
            const int wc = wbase + (widx & 31);
            uint32_t needMask = 0, sw = 0;
            bool write = false;
            if (widx < nwords) {
#pragma unroll
                for (int b = 0; b < 4; b++) {
                    const int xx = 4 * wc + b - off;
                    if (xx >= 0 && xx < tw && !cellHasIni[cellOf[xx]]) needMask |= 0x80u << (8 * b);
                }
                if (needMask) {
                    write = true;
                    if ((scoredRow[yy] >> (widx & 31)) & 1u) {
                        sw = S32[yy * (TP / 4) + wc];
                    } else {
                        uint32_t R0[7], R1[7], R2[7];
#pragma unroll
                        for (int j = 0; j < 7; j++) {
                            const uint32_t* rp = T32 + (yy + j) * (TP / 4) + wc - 1;
                            R0[j] = rp[0]; R1[j] = rp[1]; R2[j] = rp[2];
                        }
                        bool keep = true;
                        if (tmin <= 127) {
                            const uint32_t v = R1[3];
#define ROWJ(dy) R0[(dy) + 3], R1[(dy) + 3], R2[(dy) + 3]
                            uint32_t acc = gt_flag(win<0>(ROWJ(3)), v, T1b) | gt_flag(win<0>(ROWJ(-3)), v, T1b);
                            acc &= gt_flag(win<2>(ROWJ(2)), v, T1b) | gt_flag(win<-2>(ROWJ(-2)), v, T1b);
                            acc &= gt_flag(win<3>(ROWJ(0)), v, T1b) | gt_flag(win<-3>(ROWJ(0)), v, T1b);
                            acc &= gt_flag(win<2>(ROWJ(-2)), v, T1b) | gt_flag(win<-2>(ROWJ(2)), v, T1b);
#undef ROWJ
                            keep = (acc & 0x80808080u) != 0;
                        }
                        sw = keep ? score_word(R0, R1, R2) : 0u;
                    }
                }
            }
            commit(sw, yy, wc, write, tmin, TCb, needMask);
        }
        __syncthreads();
        nq = qn;
        nms(nq, false);
        __syncthreads();
        emit(nq);
    }
}

// ---- host: tensor maps (one per level: 3-D {x, y, image} view of the pyramid buffer)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

borb_status build_fast_tmaps(const Geometry& g, const Workspace& ws, void* out_tmaps) {
    static EncodeTiledFn encode = nullptr;
    if (!encode) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
        if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
            set_error("cuTensorMapEncodeTiled unavailable (%s)", cudaGetErrorString(e));
            return BORB_ERR_CUDA;
        }
        encode = (EncodeTiledFn)fn;
    }
    TMaps* tm = reinterpret_cast<TMaps*>(out_tmaps);
    std::memset(tm, 0, sizeof(TMaps));
    for (int l = 0; l < g.nlevels; l++) {
        const LevelGeom& L = g.lv[l];
        cuuint64_t dims[3] = {(cuuint64_t)L.w, (cuuint64_t)L.h, (cuuint64_t)ws.max_images};
        cuuint64_t strides[2] = {(cuuint64_t)L.pitch, (cuuint64_t)g.pyr_image_stride};
        cuuint32_t box[3] = {(cuuint32_t)TP, (cuuint32_t)(L.hCell + 6), 1};
        cuuint32_t estr[3] = {1, 1, 1};
        CUresult r = encode(&tm->m[l], CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, ws.pyr + L.pyr_off, dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) {
            set_error("cuTensorMapEncodeTiled failed for level %d (CUresult %d)", l, (int)r);
            return BORB_ERR_CUDA;
        }
    }
    return BORB_OK;
}

size_t fast_tmaps_bytes() { return sizeof(TMaps); }

// The non-empty tiles of one image in (level, cell row, block column) order - the order the grid had when the kernel derived
// the geometry itself (ORBextractor.cc:781-787 cell grid, cellsPerBlk cells per CTA).
borb_status build_fast_tiles(const Geometry& g, Workspace& ws) {
    std::vector<FastTile> t;
    for (int l = 0; l < g.nlevels; l++) {
        const LevelGeom& L = g.lv[l];
        for (int cellRow = 0; cellRow < L.nRows; cellRow++)
            for (int blkCol = 0; blkCol < L.blkCols; blkCol++) {
                const int cell0 = blkCol * L.cellsPerBlk;
                const int ncell = std::min(L.cellsPerBlk, L.nCols - cell0);
                const int x0 = EDGE + cell0 * L.wCell, x1 = std::min(x0 + ncell * L.wCell, L.w - EDGE);
                const int y0 = EDGE + cellRow * L.hCell, y1 = std::min(y0 + L.hCell, L.h - EDGE);
                if (x0 >= x1 || y0 >= y1) continue;
                FastTile f;
                f.l = (int16_t)l; f.ncell = (int16_t)ncell; f.x0 = (int16_t)x0; f.x1 = (int16_t)x1; f.y0 = (int16_t)y0; f.y1 = (int16_t)y1;
                f.wCell = (int16_t)L.wCell; f.hCell = (int16_t)L.hCell;
                t.push_back(f);
            }
    }
    cudaFree(ws.fast_tiles); ws.fast_tiles = nullptr;
    ws.fast_n_tiles = (int)t.size();
    if (t.empty()) return BORB_OK;
    BORB_CUDA(cudaMalloc(&ws.fast_tiles, t.size() * sizeof(FastTile)));
    BORB_CUDA(cudaMemcpy(ws.fast_tiles, t.data(), t.size() * sizeof(FastTile), cudaMemcpyHostToDevice));
    return BORB_OK;
}

int launch_fast(const Geometry& g, const Workspace& ws, int n_images, cudaStream_t s) {
    if (ws.fast_n_tiles == 0) return 0;
    dim3 grid(ws.fast_n_tiles, n_images);
    fast_kernel<<<grid, 256, 0, s>>>(g, *reinterpret_cast<const TMaps*>(ws.fast_tmaps), reinterpret_cast<const FastTile*>(ws.fast_tiles), ws.cand, ws.cand_cnt);
    return 1;
}

}  // namespace borb
