// Stereo association: warp-per-left-keypoint Hamming search + 11x11 SAD sub-pixel refinement, then a
// per-pair median cull.  Replaces Frame::ComputeStereoMatches (reference src/Frame.cc:466-640).
//
// Kernel 0 (one CTA per pair): bins the right keypoints by image row — every right keypoint is registered in
//   each 8-row bin its band [floor(y-r), ceil(y+r)] touches (count, scan, fill with shared-memory atomics), as a
//   compact 16-byte record {iR, minr|maxr, octave, x}.  A left keypoint then only scans the bin of its own row
//   (~100 records instead of all ~2000 right keypoints).  Order inside a bin is irrelevant (see below).
// Kernel 1 (one warp per left keypoint):
//   candidates = right keypoints whose row band [floor(y-r), ceil(y+r)], r = 2*mvScaleFactors[octave]
//   (:483-493) contains (int)vL (:511), with |octaveR-octaveL| <= 1 (:533) and uR in [uL-maxD, uL]
//   (:516-517,:538); best Hamming < TH_HIGH with first-wins on ties (:522,:543) == min over the packed
//   key (dist<<16 | iR), so no row table / ordering is needed.  If best < (TH_HIGH+TH_LOW)/2 (:471,:552):
//   SAD of centre-subtracted 11x11 patches on the UNBLURRED level kpL.octave over incR in [-5,5]
//   (:556-592, exact integers), reject extremes (:594), parabola (:598-605), rescale (:608), disparity
//   gate and clamp (:610-622).
// Kernel 2 (one CTA per pair): median of the accepted SAD distances (element size/2 of the sorted
//   (dist,iL) list, :626-627), thDist = 1.5f*1.4f*median, invalidate dist >= thDist (:628-639).
// The reference reads the uninitialised member mb at :496; the intended mb = mbf/fx is an argument.
//
// Bound: L2-resident gathers; algorithmic bytes ~0.5 MB per pair (SURVEY §8d).
#include "borb_internal.h"
#include "match_rules.cuh"

namespace borb {

constexpr int SBIN_SHIFT = 3;      // 8 image rows per bin
constexpr int SBIN_MAX = 512;      // bins per pair (images up to 4096 rows)
struct __align__(16) RightRec { int iR; int band; int octave; float x; };   // band = minr | maxr << 16

// grid: (pairs); writes bin_start[pair][nbins+1] and recs[pair][...]
__global__ void __launch_bounds__(256) stereo_bin_kernel(const __grid_constant__ Geometry g, StereoView Rv,
                                                         const int* __restrict__ pair_idx, int* __restrict__ bin_start,
                                                         RightRec* __restrict__ recs, int rec_stride) {
    __shared__ int cnt[SBIN_MAX + 1];
    __shared__ int wsum[40];
    const int pair = blockIdx.x, tid = threadIdx.x;
    const int imR = pair_idx[2 * pair + 1];
    const int nR = Rv.nkp[imR];
    const int nb = min((g.h >> SBIN_SHIFT) + 1, SBIN_MAX);
    const borb_keypoint* kR = Rv.kps + (size_t)imR * Rv.kp_image_stride;
    for (int i = tid; i <= nb; i += 256) cnt[i] = 0;
    __syncthreads();
    for (int i = tid; i < nR; i += 256) {
        const borb_keypoint kr = kR[i];
        const float r = __fmul_rn(2.0f, g.lv[kr.octave].scale);
        const int maxr = (int)ceilf(__fadd_rn(kr.y, r)), minr = (int)floorf(__fsub_rn(kr.y, r));
        const int b0 = max(minr, 0) >> SBIN_SHIFT, b1 = min(min(maxr, g.h - 1) >> SBIN_SHIFT, nb - 1);
        for (int b = b0; b <= b1; b++) atomicAdd(&cnt[b], 1);
    }
    __syncthreads();
    // exclusive scan of cnt[0..nb) (nb <= 512: two elements per thread)
    {
        const int lane = tid & 31, w = tid >> 5;
        const int i0 = 2 * tid, i1 = 2 * tid + 1;
        const int c0 = i0 < nb ? cnt[i0] : 0, c1 = i1 < nb ? cnt[i1] : 0;
        int incl = c0 + c1;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const int t = __shfl_up_sync(0xFFFFFFFFu, incl, off);
            if (lane >= off) incl += t;
        }
        if (lane == 31) wsum[w] = incl;
        __syncthreads();
        if (w == 0) {
            int v = lane < 8 ? wsum[lane] : 0, inc2 = v;
#pragma unroll
            for (int off = 1; off < 8; off <<= 1) {
                const int t = __shfl_up_sync(0xFFFFFFFFu, inc2, off);
                if (lane >= off) inc2 += t;
            }
            if (lane < 8) wsum[8 + lane] = inc2 - v;
            if (lane == 7) wsum[16] = inc2;
        }
        __syncthreads();
        const int base = wsum[8 + w] + incl - (c0 + c1);
        if (i0 < nb) cnt[i0] = base;
        if (i1 < nb) cnt[i1] = base + c0;
        if (tid == 0) cnt[nb] = wsum[16];
        __syncthreads();
    }
    int* bs = bin_start + (size_t)pair * (SBIN_MAX + 1);
    for (int i = tid; i <= nb; i += 256) bs[i] = cnt[i];
    __syncthreads();
    RightRec* out = recs + (size_t)pair * rec_stride;
    for (int i = tid; i < nR; i += 256) {
        const borb_keypoint kr = kR[i];
        const float r = __fmul_rn(2.0f, g.lv[kr.octave].scale);
        const int maxr = (int)ceilf(__fadd_rn(kr.y, r)), minr = (int)floorf(__fsub_rn(kr.y, r));
        const int b0 = max(minr, 0) >> SBIN_SHIFT, b1 = min(min(maxr, g.h - 1) >> SBIN_SHIFT, nb - 1);
        RightRec rec;
        rec.iR = i; rec.band = (minr & 0xFFFF) | (maxr << 16); rec.octave = kr.octave; rec.x = kr.x;
        for (int b = b0; b <= b1; b++) {
            const int pos = atomicAdd(&cnt[b], 1);
            if (pos < rec_stride) out[pos] = rec;
        }
    }
}

// 40 registers (6 CTAs/SM): latency-bound gathers, occupancy pays (0.112 -> 0.101 ms per 32 pairs)
__global__ void __launch_bounds__(256, 6) stereo_match_kernel(const __grid_constant__ Geometry g, StereoView Lv, StereoView Rv,
                                                           const int* __restrict__ pair_idx, float bf, float b,
                                                           float* __restrict__ u_right, float* __restrict__ depth,
                                                           int* __restrict__ sad, int out_stride,
                                                           const int* __restrict__ bin_start, const RightRec* __restrict__ recs,
                                                           int rec_stride) {
    const int pair = blockIdx.y;
    const int imL = pair_idx[2 * pair], imR = pair_idx[2 * pair + 1];
    const int lane = threadIdx.x & 31;
    const int iL = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int nL = Lv.nkp[imL], nR = Rv.nkp[imR];
    if (iL >= nL) return;
    const size_t o = (size_t)pair * out_stride + iL;
    const borb_keypoint* kL = Lv.kps + (size_t)imL * Lv.kp_image_stride;
    const borb_keypoint* kR = Rv.kps + (size_t)imR * Rv.kp_image_stride;
    const uint8_t* dL = Lv.desc + (size_t)imL * Lv.kp_image_stride * 32;
    const uint8_t* dR = Rv.desc + (size_t)imR * Rv.kp_image_stride * 32;

    float uR_out = -1.0f, depth_out = -1.0f;
    int sad_out = -1;

    const borb_keypoint kp = kL[iL];
    const int levelL = kp.octave;
    const float vL = kp.y, uL = kp.x;
    const float maxD = __fdiv_rn(bf, b);            // mbf/minZ, minZ = mb (:496-498)
    const float minU = __fsub_rn(uL, maxD), maxU = uL;   // minD = 0 (:516-517)
    const int row = (int)vL;
    const uint4 a0 = reinterpret_cast<const uint4*>(dL + (size_t)iL * 32)[0];
    const uint4 a1 = reinterpret_cast<const uint4*>(dL + (size_t)iL * 32)[1];
    unsigned best = ((unsigned)TH_HIGH << 16);      // strict '<' against TH_HIGH: keys >= TH_HIGH<<16 never win
    if (!(maxU < 0) && row >= 0 && row < g.h) {
        const int nb = min((g.h >> SBIN_SHIFT) + 1, SBIN_MAX);
        const int bin = min(row >> SBIN_SHIFT, nb - 1);
        const int* bs = bin_start + (size_t)pair * (SBIN_MAX + 1);
        const int e0 = bs[bin], e1 = min(bs[bin + 1], rec_stride);
        const RightRec* rr = recs + (size_t)pair * rec_stride;
        for (int e = e0 + lane; e < e1; e += 32) {
            const RightRec rc = rr[e];
            const int minr = (int)(short)(rc.band & 0xFFFF), maxr = rc.band >> 16;
            if (row < minr || row > maxr) continue;
            if (rc.octave < levelL - 1 || rc.octave > levelL + 1) continue;
            if (rc.x >= minU && rc.x <= maxU) {
                const uint4* b = reinterpret_cast<const uint4*>(dR + (size_t)rc.iR * 32);
                const int dist = descriptor_distance(a0, a1, b[0], b[1]);
                const unsigned key = ((unsigned)dist << 16) | (unsigned)rc.iR;
                best = min(best, key);
            }
        }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) best = min(best, __shfl_xor_sync(0xFFFFFFFFu, best, off));
    const int bestDist = (int)(best >> 16);
    const int thOrbDist = (TH_HIGH + TH_LOW) / 2;
    if (bestDist < thOrbDist) {
        const int bestIdxR = (int)(best & 0xFFFFu);
        const float uR0 = kR[bestIdxR].x;
        const LevelGeom& LG = g.lv[levelL];
        const float sf = LG.inv_scale;
        const int scaleduL = (int)roundf(__fmul_rn(kp.x, sf));
        const int scaledvL = (int)roundf(__fmul_rn(kp.y, sf));
        const int scaleduR0 = (int)roundf(__fmul_rn(uR0, sf));
        const int w = 5, Lh = 5;
        const int iniu = scaleduR0 + Lh - w, endu = scaleduR0 + Lh + w + 1;
        // reference guard (:573-576) plus memory-safety guards the reference leaves to cv::Mat asserts
        const bool ok = !(iniu < 0 || endu >= LG.w) && scaleduR0 - Lh - w >= 0 && scaledvL - w >= 0 &&
                        scaledvL + w < LG.h && scaleduL - w >= 0 && scaleduL + w < LG.w;
        if (ok) {
            const uint8_t* IL = Lv.pyr + (size_t)imL * Lv.pyr_image_stride + LG.pyr_off;
            const uint8_t* IR = Rv.pyr + (size_t)imR * Rv.pyr_image_stride + LG.pyr_off;
            const int cL = IL[(size_t)scaledvL * LG.pitch + scaleduL];
            int il[4];
            int offs[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const int e = lane + 32 * k;
                if (e < 121) {
                    const int yy = e / 11, xx = e - yy * 11;
                    offs[k] = (scaledvL - w + yy) * LG.pitch + (xx - w);
                    il[k] = (int)IL[offs[k] + scaleduL] - cL;
                } else { offs[k] = -1; il[k] = 0; }
            }
            int bestD = 0x7FFFFFFF, bestinc = 0;
            int dists[11];
#pragma unroll
            for (int inc = -5; inc <= 5; inc++) {
                const int uc = scaleduR0 + inc;
                const int cR = IR[(size_t)scaledvL * LG.pitch + uc];
                int s = 0;
#pragma unroll
                for (int k = 0; k < 4; k++)
                    if (offs[k] >= 0) s += abs(il[k] - ((int)IR[offs[k] + uc] - cR));
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, off);
                dists[inc + 5] = s;
                if (s < bestD) { bestD = s; bestinc = inc; }
            }
            if (!(bestinc == -Lh || bestinc == Lh)) {
                float d1 = 0.f, d2 = 0.f, d3 = 0.f;
#pragma unroll
                for (int i = 1; i < 10; i++)
                    if (i == bestinc + 5) { d1 = (float)dists[i - 1]; d2 = (float)dists[i]; d3 = (float)dists[i + 1]; }
                const float num = __fsub_rn(d1, d3);
                const float den = __fmul_rn(2.0f, __fsub_rn(__fadd_rn(d1, d3), __fmul_rn(2.0f, d2)));
                const float deltaR = __fdiv_rn(num, den);
                if (!(deltaR < -1.f || deltaR > 1.f)) {
                    float bestuR = __fmul_rn(LG.scale, __fadd_rn(__fadd_rn((float)scaleduR0, (float)bestinc), deltaR));
                    float disparity = __fsub_rn(uL, bestuR);
                    if (disparity >= 0.f && disparity < maxD) {
                        if (disparity <= 0.f) {
                            disparity = 0.01f;                       // (float)0.01 (:616)
                            bestuR = (float)((double)uL - 0.01);     // uL-0.01 evaluated in double (:617)
                        }
                        depth_out = __fdiv_rn(bf, disparity);
                        uR_out = bestuR;
                        sad_out = bestD;
                    }
                }
            }
        }
    }
    if (lane == 0) {
        u_right[o] = uR_out;
        depth[o] = depth_out;
        sad[o] = sad_out;
    }
}

// One CTA per pair: k-th order statistic by two 256-bin histogram passes (SAD <= 121*510 < 2^16).
__global__ void __launch_bounds__(256) stereo_median_kernel(StereoView Lv, const int* __restrict__ pair_idx,
                                                            float* __restrict__ u_right, float* __restrict__ depth,
                                                            const int* __restrict__ sad, int out_stride) {
    __shared__ int hist[256];
    __shared__ int sel[3];
    const int pair = blockIdx.x;
    const int nL = Lv.nkp[pair_idx[2 * pair]];
    const size_t o = (size_t)pair * out_stride;
    const int tid = threadIdx.x;
    hist[tid] = 0;
    __syncthreads();
    int cnt = 0;
    for (int i = tid; i < nL; i += 256) {
        const int d = sad[o + i];
        if (d >= 0) { atomicAdd(&hist[min(d >> 8, 255)], 1); cnt++; }
    }
    // total number of accepted matches
    __shared__ int tot;
    if (tid == 0) tot = 0;
    __syncthreads();
    if (cnt) atomicAdd(&tot, cnt);
    __syncthreads();
    const int n = tot;
    if (n == 0) return;                       // reference: UB on an empty vDistIdx (:627); nothing to cull
    const int kth = n / 2;
    if (tid == 0) {
        int acc = 0, bin = 0;
        for (; bin < 256; bin++) { if (acc + hist[bin] > kth) break; acc += hist[bin]; }
        sel[0] = bin; sel[1] = kth - acc;
    }
    __syncthreads();
    const int hiBin = sel[0], rem = sel[1];
    __syncthreads();
    hist[tid] = 0;
    __syncthreads();
    for (int i = tid; i < nL; i += 256) {
        const int d = sad[o + i];
        if (d >= 0 && min(d >> 8, 255) == hiBin) atomicAdd(&hist[d & 255], 1);
    }
    __syncthreads();
    if (tid == 0) {
        int acc = 0, bin = 0;
        for (; bin < 256; bin++) { if (acc + hist[bin] > rem) break; acc += hist[bin]; }
        sel[2] = (hiBin << 8) | bin;
    }
    __syncthreads();
    const float median = (float)sel[2];
    const float thDist = __fmul_rn(1.5f * 1.4f, median);
    for (int i = tid; i < nL; i += 256) {
        const int d = sad[o + i];
        if (d >= 0 && !((float)d < thDist)) { u_right[o + i] = -1.0f; depth[o + i] = -1.0f; }
    }
}

// Worst-case records per pair of right images of geometry g (their keypoint capacity): a band spans 2*ceil(2*scale_max)+2 rows, i.e. at most (that >> 3) + 2 bins.
int stereo_rec_stride(const Geometry& g) {
    const int band = 2 * (int)ceilf(2.0f * g.lv[g.nlevels - 1].scale) + 3;
    return g.sel_image_stride * ((band >> SBIN_SHIFT) + 2);
}
size_t stereo_bins_bytes_per_pair() { return (size_t)(SBIN_MAX + 1) * sizeof(int); }
size_t stereo_rec_bytes() { return sizeof(RightRec); }

int launch_stereo(const Geometry& g, const StereoView& L, const StereoView& R, const int* d_pair_idx, int n_pairs,
                  float bf, float b, float* d_u_right, float* d_depth, int* d_sad, int out_stride, int* d_bins, void* d_recs,
                  int rec_stride, cudaStream_t s) {
    stereo_bin_kernel<<<n_pairs, 256, 0, s>>>(g, R, d_pair_idx, d_bins, reinterpret_cast<RightRec*>(d_recs), rec_stride);
    dim3 grid((g.sel_image_stride + 7) / 8, n_pairs);
    stereo_match_kernel<<<grid, 256, 0, s>>>(g, L, R, d_pair_idx, bf, b, d_u_right, d_depth, d_sad, out_stride, d_bins,
                                             reinterpret_cast<const RightRec*>(d_recs), rec_stride);
    stereo_median_kernel<<<n_pairs, 256, 0, s>>>(L, d_pair_idx, d_u_right, d_depth, d_sad, out_stride);
    return 3;
}

}  // namespace borb
