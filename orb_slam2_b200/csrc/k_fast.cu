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
// One CTA owns `cellsPerBlk` whole cells of each of a band of `rowsPerBlk` cell rows (max(1, FAST_H_BAND / hCell)), so NMS and
// the threshold decision are CTA-local; the band pays the halo rows, the tile load and the barrier chain once for all its rows.
//
// Pipeline inside a CTA:
//   0. one elected thread issues a 3-D TMA tile load (cp.async.bulk.tensor, box 160 x (rowsPerBlk*hCell+6) bytes at
//      ((x0-4)&~15, y0-3, image): the inner start coordinate must be 16-byte aligned) into shared memory
//      and everybody waits on its mbarrier;
//   1a. a thread owns the 4 pixels of one ALIGNED 32-bit word of the tile and slides down its rows with a
//      7-row register window.  Cheap reject: per even ring position one VABSDIFF4 gives |I_q - I_p| for the
//      4 pixels and two more ops a per-byte ">t" flag; a FAST-9 arc contains a pixel of each antipodal
//      ring pair, so AND_j (f_j | f_{j+8}) == 0 rejects the pixel.  Words with a surviving pixel go to the
//      warp's segment of a word queue with their byte flags; the warp then expands its segment into a pixel
//      queue holding only the surviving pixels (about half the pixels of the surviving words);
//   1b. the queued pixels are scored EXACTLY, two per thread: each pixel's 16 ring bytes are gathered from the
//      tile and the two pixels packed into the 16-bit lanes of one register, S = max(max_k min_{j<9} I_{k+j} - I_p,
//      I_p - min_k max_{j<9} I_{k+j}) - 1 with VIMNMX3.S16x2 (min3/max3) networks over the ring intensities — the
//      corner test IS the score (corner at t <=> S >= t).  Pixels that were not scored hold S = 0 in the score map.
//      Phases 1a/1b run at iniThFAST; cells that end up without a kept corner are redone at minThFAST
//      afterwards by the same two phases (pass B), exactly the reference's per-cell fallback;
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
#include <type_traits>
#include <vector>

namespace borb {

namespace {

constexpr int TP = 160;                 // TMA box width == smem tile pitch (bytes).  TMA needs a 16-byte aligned start
                                        // column, so the box starts at xs = (x0-4) & ~15 and domain px xx sits at column xx+off
constexpr int HB = FAST_H_BAND;         // domain rows of the tallest tile: a band of R >= 2 cell rows has R * hCell <= HB rows,
                                        // a one-row band hCell <= 59
static_assert(HB >= 60 && HB <= 127, "a one-row band (hCell <= 59) must fit; collect packs the row into 7 bits");
constexpr int TROWS = HB + 6;           // + 3 halo rows above and below
constexpr int QCAP = HB * 128;          // queue capacity >= every domain pixel of the largest tile
constexpr int RG_MAX = (HB + 7) / 8;    // rows per warp in phase 1a (8 warps)
constexpr int WSEG = RG_MAX * 32;       // one warp's segment of the word queue: at most 32 words per row
constexpr int RMAX = HB / 30;           // cell rows per band (hCell >= 30)
constexpr int NCX = 128 / 30 + 1;       // cell columns per band (wCell >= 30, domain columns < 128)
// dynamic shared memory: tile | score | queue | wqueue
constexpr int SM_SCORE = TROWS * TP, SM_QUEUE = SM_SCORE + HB * TP, SM_WQUEUE = SM_QUEUE + QCAP * 2;
constexpr int FAST_SMEM = SM_WQUEUE + 8 * WSEG * 4;
static_assert(SM_SCORE % 16 == 0 && SM_WQUEUE % 4 == 0, "shared-memory carve-up alignment");

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
// byte's flag when that byte has a == t exactly: a false "keep", which only sends the pixel to the exact scoring pass
// (pass 1b decides every corner from exact scores), never a false reject.
__device__ __forceinline__ uint32_t gt_flag(uint32_t q, uint32_t v, uint32_t K) {
    const uint32_t a = __vabsdiffu4(q, v);
    return (a + K) | a;
}

// Exact FAST scores of two pixels at once, one per 16-bit lane.  d[k] = I_q for ring position k (OpenCV's 16-pixel
// circle, clockwise from (0,+3)), v2 = I_p, all in [0, 255].  Returns per lane S(p) in [0,254]; S(p) >= t <=> p is a
// FAST-9 corner at threshold t (cornerScore<16> of OpenCV, both polarities at once).  The min/max network runs on the
// intensities themselves: min_j (I_qj - I_p) = min_j I_qj - I_p, so I_p is subtracted once at the end, not per ring pixel.
__device__ __forceinline__ uint32_t score_pair(const uint32_t (&d)[16], uint32_t v2) {
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
    // S = max(bright - I_p, I_p - darkm) - 1, clamped at 0 (lanes stay in [-255, 255]: no borrow between lanes)
    return __viaddmax_s16x2_relu(__vmaxs2(__vsub2(bright, v2), __vsub2(v2, darkm)), 0xFFFFFFFFu, 0u);
}

// Exact scores of the pixels at smem addresses pa and pb (tile bytes): lane 0 = S(pa), lane 1 = S(pb).  Each ring byte of
// the two pixels is loaded on its own and the pair is packed into the two s16 lanes.
__device__ __forceinline__ uint32_t score_pixels(const uint8_t* pa, const uint8_t* pb) {
    constexpr int RX[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
    constexpr int RY[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};
    uint32_t d[16];
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const int o = RY[k] * TP + RX[k];
        d[k] = (uint32_t)pa[o] | ((uint32_t)pb[o] << 16);
    }
    return score_pair(d, (uint32_t)pa[0] | ((uint32_t)pb[0] << 16));
}

}  // namespace

struct TMaps { CUtensorMap m[BORB_MAX_LEVELS]; };

// One FAST CTA = whole cells of a band of rowsPerBlk cell rows of one level (the last band of a level may hold fewer cell
// rows).  The tile geometry is the same for every image of a batch, so it is computed once on the host (build_fast_tiles)
// instead of ~110 instructions per CTA (8.7 % of the kernel's instructions).
struct __align__(16) FastTile { int8_t l, ncell, rowsPerBlk, pad; int16_t x0, x1, y0, y1, wCell, hCell; };
static_assert(sizeof(FastTile) == 16, "one 16-byte load per CTA");

// 64 registers and FAST_SMEM (45 KB at HB = 64) + 256 B static shared memory: 4 CTAs/SM
__global__ void __launch_bounds__(256, 4) fast_kernel(const __grid_constant__ Geometry g, const __grid_constant__ TMaps tm,
                                                   const FastTile* __restrict__ tiles, uint32_t* __restrict__ cand, int* __restrict__ cand_cnt) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* tile = smem;                                 // TROWS x TP: the TMA box
    uint8_t* score = smem + SM_SCORE;                     // HB x TP: S(p) in TILE coordinates (same columns as `tile`)
    uint16_t* queue = reinterpret_cast<uint16_t*>(smem + SM_QUEUE);   // QCAP: pixels to score, then (in place) corners:
                                                                      // row << 8 | tile column
    uint32_t* wqueue = reinterpret_cast<uint32_t*>(smem + SM_WQUEUE); // surviving words (reject flags | row << 8 | word column):
                                                          // one WSEG-entry segment per warp (a warp owns <= RG_MAX rows of
                                                          // <= 32 words), filled without atomics
    __shared__ __align__(8) unsigned long long bar;
    __shared__ int pn, qn, needB;
    __shared__ int cellHasIni[RMAX * NCX];                // [cell row of the band][cell]
    __shared__ uint8_t cellOf[128];                       // domain column -> cell of the band row
    __shared__ uint8_t rowOf[HB];                         // domain row -> cell row of the band

    const int img = blockIdx.y;
    const FastTile T = tiles[blockIdx.x];                // one 16-byte load (only non-empty tiles are in the table)
    const int l = T.l, ncell = T.ncell, x0 = T.x0, x1 = T.x1, y0 = T.y0, y1 = T.y1;
    const int wCell = T.wCell, hCell = T.hCell;
    const LevelGeom& L = g.lv[l];
    const int tw = x1 - x0, th = y1 - y0;
    const int tid = threadIdx.x;
    const int lane = tid & 31, wrp = tid >> 5;

    // ---- 0. TMA: tile rows y0-3 .. y0+rowsPerBlk*hCell+2, columns xs .. xs+159 of image `img`, level l
    const int xs = (x0 - 4) & ~15;          // 16-byte aligned box start (TMA requirement)
    const int off = x0 - xs;                // tile column of domain pixel xx = 0   (4..19)
    if (tid == 0) {
        // the issuing thread initialises the barrier itself, so the copy starts before the CTA's first barrier; the other
        // threads see the initialised mbarrier after the __syncthreads() below and only then wait on it
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        // the whole box, rows past the image included (TMA counts its out-of-bounds fill), exactly as the tensor map has it
        const uint32_t bytes = (uint32_t)TP * (uint32_t)fast_box_rows(T.rowsPerBlk, hCell);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar)), "r"(bytes) : "memory");
        asm volatile(
            "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
            ::"r"(smem_u32(tile)), "l"(reinterpret_cast<uint64_t>(&tm.m[l])), "r"(xs), "r"(y0 - 3), "r"(img), "r"(smem_u32(&bar))
            : "memory");
    }
    // overlap with the copy: bookkeeping
    if (tid < RMAX * NCX) cellHasIni[tid] = 0;
    if (tid < 128) cellOf[tid] = (uint8_t)(tid / wCell);
    if (tid < HB) rowOf[tid] = (uint8_t)(tid / hCell);
    if (tid == 0) { pn = 0; qn = 0; needB = 0; }
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

    const uint32_t* T32 = reinterpret_cast<const uint32_t*>(tile);
    uint32_t* S32 = reinterpret_cast<uint32_t*>(score);
    const int wbase = off >> 2;             // in phase 1a lane owns aligned tile word wc (tile columns 4*wc .. 4*wc+3)
    const int wc = wbase + lane;
    uint32_t vmask = 0;                     // bit 7 of each byte of word wc that lies inside the detection domain
#pragma unroll
    for (int b = 0; b < 4; b++)
        if (4 * wc + b - off >= 0 && 4 * wc + b - off < tw) vmask |= 0x80u << (8 * b);

    // ---- 1a. Reject at threshold t, pixel by pixel, among the pixels whose byte of `m` (bit 7) is set, and queue the
    //          survivors.  Words are tested 4 pixels at a time sliding down the rows; surviving words go to the warp's
    //          segment of `wqueue` with their per-byte flags and are then expanded by the same warp into single pixels of
    //          `queue` (order does not matter).  `zero` (pass A, m = the domain): record every domain pixel's score as 0
    //          first, so that pixels rejected here read as S = 0 < t.  Pass A tests every row with mr[0]; pass B (banded)
    //          tests the rows of cell row r of the band with mr[r].
    auto collect = [&](int t, const uint32_t (&mr)[RMAX], bool zero, auto banded) {
        constexpr bool BANDED = decltype(banded)::value;
        const uint32_t K = (uint32_t)(127 - min(t, 127)) * 0x01010101u;      // gt_flag's K
        // the masks are loop invariants the compiler would otherwise rebuild from the tile geometry on every row (≈149
        // instead of ≈83 instructions per row)
        uint32_t mm[RMAX];
#pragma unroll
        for (int r = 0; r < (BANDED ? RMAX : 1); r++) {
            mm[r] = mr[r];
            asm volatile("" : "+r"(mm[r]));
        }
        const bool reject = t <= 127;
        const int RG = (th + 7) >> 3;                 // rows per warp (8 warps), <= RG_MAX
        const int yBeg = wrp * RG, yEnd = min(th, yBeg + RG);
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
        // rows in runs of 7, the window's period: slot indices depend on `it` only modulo 7, so they stay compile-time
        // constants without unrolling all RG_MAX rows (12 rows of a 96-row band, fully unrolled, spilled)
        for (int it0 = 0; it0 < RG; it0 += 7)
#pragma unroll
        for (int it = 0; it < 7; it++) {
            const int yy = yBeg + it0 + it;
            if (yy < yEnd) {          // warp-uniform
                {
                    const uint32_t* rp = T32 + (yy + 6) * (TP / 4) + wc - 1;
                    a0[(it + 6) % 7] = rp[0]; a1[(it + 6) % 7] = rp[1]; a2[(it + 6) % 7] = rp[2];
                }
                uint32_t m = mm[0];
                if constexpr (BANDED) {
#pragma unroll
                    for (int r = 1; r < RMAX; r++)
                        if (yy >= r * hCell) m = mm[r];
                }
#define ROW(dy) a0[(it + (dy) + 3) % 7], a1[(it + (dy) + 3) % 7], a2[(it + (dy) + 3) % 7]
                uint32_t f = m;
                if (reject && m) {
                    const uint32_t v = a1[(it + 3) % 7];
                    uint32_t acc = gt_flag(win<0>(ROW(3)), v, K) | gt_flag(win<0>(ROW(-3)), v, K);      // pair (0,8)
                    acc &= gt_flag(win<2>(ROW(2)), v, K) | gt_flag(win<-2>(ROW(-2)), v, K);               // (2,10)
                    acc &= gt_flag(win<3>(ROW(0)), v, K) | gt_flag(win<-3>(ROW(0)), v, K);                // (4,12)
                    acc &= gt_flag(win<2>(ROW(-2)), v, K) | gt_flag(win<-2>(ROW(2)), v, K);               // (6,14)
                    f = acc & m;
                }
#undef ROW
                const unsigned bal = __ballot_sync(0xFFFFFFFFu, f != 0);
                if (zero && m != 0) S32[yy * (TP / 4) + wc] = 0;
                // flags in bits 7/15/23/31, row in bits 8..14, word column in bits 0..6
                if (f) wqueue[wrp * WSEG + wcount + __popc(bal & ((1u << lane) - 1))] = f | (uint32_t)(yy << 8) | (uint32_t)wc;
                wcount += __popc(bal);               // warp-uniform: the warp's segment needs no atomic
            }
        }
        __syncwarp();
        for (int i = 0; i < wcount; i += 32) {       // warp-uniform
            const uint32_t we = i + lane < wcount ? wqueue[wrp * WSEG + i + lane] : 0u;
            const uint32_t fl = we & 0x80808080u;
            const int c = __popc(fl);
            int incl = c;
#pragma unroll
            for (int o2 = 1; o2 < 32; o2 <<= 1) {
                const int s = __shfl_up_sync(0xFFFFFFFFu, incl, o2);
                if (lane >= o2) incl += s;
            }
            int base = 0;
            if (lane == 31) base = atomicAdd(&pn, incl);
            base = __shfl_sync(0xFFFFFFFFu, base, 31) + incl - c;
            const int e = (int)((we >> 8) & 127) << 8 | (int)(4 * (we & 127));
#pragma unroll
            for (int b = 0; b < 4; b++)
                if (fl & (0x80u << (8 * b))) queue[base++] = (uint16_t)(e + b);
        }
    };

    // ---- 1b. Exact scores of the queued pixels, two per thread (one per s16x2 lane), written to the score map; the
    //          corners (S >= t) go to the corner queue, which reuses the front of the pixel queue.
    auto score_queue = [&](int t) {
        const int np = pn;
        const int tc = max(t, 1);
        for (int rb = 0; rb < np; rb += 512) {       // CTA-uniform: the loop holds a barrier
            const int e0 = rb + wrp * 64 + lane, e1 = e0 + 32;
            const bool va = e0 < np, vb = e1 < np;
            const int qa = va ? queue[e0] : off;      // idle lanes score domain pixel (0, 0)
            const int qb = vb ? queue[e1] : qa;
            // corners found in this round land below rb + 512 (at most one per entry read so far), never on an entry of a
            // later round; the barrier keeps them off the entries of this one until everybody has read them
            __syncthreads();
            if (rb + wrp * 64 < np) {                 // warp-uniform
                const int ia = (qa >> 8) * TP + (qa & 255), ib = (qb >> 8) * TP + (qb & 255);
                const uint32_t s2 = score_pixels(tile + ia + 3 * TP, tile + ib + 3 * TP);
                const int sa = (int)(s2 & 0xFFFFu), sb = (int)(s2 >> 16);
                if (va) score[ia] = (uint8_t)sa;
                if (vb) score[ib] = (uint8_t)sb;
                const bool ca = va && sa >= tc, cb = vb && sb >= tc;
                if (__any_sync(0xFFFFFFFFu, ca || cb)) {
                    const int c = (int)ca + (int)cb;
                    int incl = c;
#pragma unroll
                    for (int o2 = 1; o2 < 32; o2 <<= 1) {
                        const int s = __shfl_up_sync(0xFFFFFFFFu, incl, o2);
                        if (lane >= o2) incl += s;
                    }
                    int base = 0;
                    if (lane == 31) base = atomicAdd(&qn, incl);
                    base = __shfl_sync(0xFFFFFFFFu, base, 31) + incl - c;
                    if (ca) queue[base++] = (uint16_t)qa;
                    if (cb) queue[base] = (uint16_t)qb;
                }
            }
        }
    };

    // Pass A works at iniThFAST only: a cell falls back to minThFAST only if it has NO kept corner at iniThFAST
    // (ORBextractor.cc:809-816), and a pixel with S < ini can neither be kept at ini nor suppress one that is.
    {
        const uint32_t mA[RMAX] = {vmask};
        collect(g.ini_th, mA, true, std::false_type());
    }
    __syncthreads();
    if (g.fast_mode == 2) {                 // ablation: load + packed reject + pixel queue
        if (pn == -1) cand[0] = 1;
        return;
    }
    score_queue(g.ini_th);
    __syncthreads();
    int nq = qn;
    if (g.fast_mode == 3) {                 // ablation: load + reject + exact scores
        if (nq == -1) cand[0] = 1;
        return;
    }

    uint32_t* out = cand + (size_t)img * g.cand_image_stride + L.cand_off;
    int* cnt = cand_cnt + img * g.nlevels + l;

    // cell-local strict NMS over queue[0..n) (0xFFFF = dropped); optionally records which cells keep something.  A
    // neighbour in another cell, whether beside the pixel or in the band's cell row above or below, counts as 0.
    auto nms = [&](int n, bool mark) {
        for (int e = tid; e < n; e += 256) {
            const int q = queue[e];
            const int col = q & 255, yy = q >> 8;
            const int xx = col - off;
            const int s = score[yy * TP + col];
            const int c = cellOf[xx], r = rowOf[yy];
            const int cx0 = c * wCell, cx1 = min(cx0 + wCell, tw);
            const int cy0 = r * hCell, cy1 = min(cy0 + hCell, th);
            bool ismax = true;
#pragma unroll
            for (int dy = -1; dy <= 1; dy++)
#pragma unroll
                for (int dx = -1; dx <= 1; dx++) {
                    if (dx == 0 && dy == 0) continue;
                    const int qx = xx + dx, qy = yy + dy;
                    if (qx < cx0 || qx >= cx1 || qy < cy0 || qy >= cy1) continue;
                    if (!(s > (int)score[qy * TP + col + dx])) ismax = false;
                }
            if (ismax) {
                if (mark) cellHasIni[r * NCX + c] = 1;
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
    if (tid < RMAX * NCX) {
        const int r = tid / NCX, c = tid - r * NCX;
        if (r * hCell < th && c < ncell && c * wCell < tw && !cellHasIni[tid] && g.min_th < g.ini_th) needB = 1;
    }
    __syncthreads();
    if (!needB) return;

    // ---- 3. pass B (rare): cells without any kept iniTh corner are redone at minThFAST (ORBextractor.cc:812-816) by
    //         phases 1a and 1b over the pixels of those cells.  Every pixel with S >= minTh passes the reject at minTh and
    //         is (re)scored, so its score is exact; any other pixel of the cell holds 0 or its exact score, both < minTh.
    {
        uint32_t need[RMAX];                // per cell row of the band: the thread's pixels whose cell needs pass B
#pragma unroll
        for (int r = 0; r < RMAX; r++) {
            need[r] = 0;
#pragma unroll
            for (int b = 0; b < 4; b++) {
                const int xx = 4 * wc + b - off;
                if (xx >= 0 && xx < tw && !cellHasIni[r * NCX + cellOf[xx]]) need[r] |= 0x80u << (8 * b);
            }
        }
        if (tid == 0) { pn = 0; qn = 0; }
        __syncthreads();
        collect(g.min_th, need, false, std::true_type());
        __syncthreads();
        score_queue(g.min_th);
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
        cuuint32_t box[3] = {(cuuint32_t)TP, (cuuint32_t)fast_box_rows(L.rowsPerBlk, L.hCell), 1};
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

// The non-empty tiles of one image in (level, band, block column) order (ORBextractor.cc:781-787 cell grid; cellsPerBlk cells
// of rowsPerBlk cell rows per CTA).  A band spans cell rows [cellRow, cellRow + rowsPerBlk), clipped at the grid's last row and
// its domain at h - EDGE like a single cell row's.
borb_status build_fast_tiles(const Geometry& g, Workspace& ws) {
    std::vector<FastTile> t;
    for (int l = 0; l < g.nlevels; l++) {
        const LevelGeom& L = g.lv[l];
        for (int cellRow = 0; cellRow < L.nRows; cellRow += L.rowsPerBlk)
            for (int blkCol = 0; blkCol < L.blkCols; blkCol++) {
                const int cell0 = blkCol * L.cellsPerBlk;
                const int ncell = std::min(L.cellsPerBlk, L.nCols - cell0);
                const int nrow = std::min(L.rowsPerBlk, L.nRows - cellRow);
                const int x0 = EDGE + cell0 * L.wCell, x1 = std::min(x0 + ncell * L.wCell, L.w - EDGE);
                const int y0 = EDGE + cellRow * L.hCell, y1 = std::min(y0 + nrow * L.hCell, L.h - EDGE);
                if (x0 >= x1 || y0 >= y1) continue;
                FastTile f;
                f.l = (int8_t)l; f.ncell = (int8_t)ncell; f.rowsPerBlk = (int8_t)L.rowsPerBlk; f.pad = 0;
                f.x0 = (int16_t)x0; f.x1 = (int16_t)x1; f.y0 = (int16_t)y0; f.y1 = (int16_t)y1;
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
    allow_max_smem((const void*)fast_kernel);          // once per device
    dim3 grid(ws.fast_n_tiles, n_images);
    fast_kernel<<<grid, 256, FAST_SMEM, s>>>(g, *reinterpret_cast<const TMaps*>(ws.fast_tmaps), reinterpret_cast<const FastTile*>(ws.fast_tiles), ws.cand, ws.cand_cnt);
    return 1;
}

}  // namespace borb
