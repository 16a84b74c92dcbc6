// Orientation (intensity centroid) + 256-bit steered BRIEF + final keypoint records: one warp per keypoint.
//
// Replaces, of reference src/ORBextractor.cc:
//   IC_Angle (:77-104) / computeOrientation (:472-479)  — integer moments over the 749-px disc of the
//       UNBLURRED level, angle = cv::fastAtan2((float)m01,(float)m10) (float32 polynomial, no FMA);
//   computeOrbDescriptor (:108-147) with bit_pattern_31_ (:150-408) — a = cosf(t), b = sinf(t),
//       t = angle*(float)(CV_PI/180.f); tap = center[cvRound(x*b+y*a)*step + cvRound(x*a-y*b)] on the
//       BLURRED level; bit k of byte i = tap(16i+2k... ) i.e. test t -> byte t/8, bit t%8;
//   operator() tail (:1059-1104) — levels concatenated 0..n-1, pt *= mvScaleFactor[level], size, octave.
// sinf/cosf: device port (double arithmetic) of the glibc >= 2.28 single-precision kernels the
// reference binary calls on x86-64 (ARM optimized-routines sincosf); checked exhaustively on the CPU
// against glibc for every float in [0, 2*pi] (DESIGN.md).  The 512 taps are fetched in the order of the keypoint's
// orientation bin (brief_slot_table, borb_internal.h): one gather instruction then touches a few adjacent rows of the
// patch (~4 128-byte lines) instead of points spread over the whole 37 x 37 window (~20 lines).  Each tap byte goes to
// its canonical place 2*test + which in the warp's 512 B of shared memory; lane t%32 then reads test t's two bytes as one
// u16 and a warp ballot IS the packed little-endian uint32 of 4 descriptor bytes, so a descriptor is 8 ballots.
//
// Bound: not the tap gathers' L1 wavefronts: cutting their lines from ~20 to ~4 per instruction left the kernel's own time
// unchanged (DESIGN.md §5), and prefetching the blurred window into L1 made it 25 % slower.  What remains is filling the
// 37 x 37 blurred and 31 x 31 level windows of every keypoint from L2 (which of their traffic or latency binds: not
// measured).  The shorter tap instructions do raise the throughput of the whole pipeline with several streams in flight.
#include "borb_internal.h"

namespace borb {

namespace {

// glibc sinf/cosf kernels for |x| < 120 (reduce_fast + degree-8/7 polynomials in double)
struct SinCosTab { double sign[4]; double hpi_inv, hpi, c0, c1, c2, c3, c4, s1, s2, s3; };
__device__ const SinCosTab d_sincos[2] = {
    {{1.0, -1.0, -1.0, 1.0}, 0x1.45F306DC9C883p+23, 0x1.921FB54442D18p0, 0x1p0, -0x1.ffffffd0c621cp-2,
     0x1.55553e1068f19p-5, -0x1.6c087e89a359dp-10, 0x1.99343027bf8c3p-16, -0x1.555545995a603p-3,
     0x1.1107605230bc4p-7, -0x1.994eb3774cf24p-13},
    {{1.0, -1.0, -1.0, 1.0}, 0x1.45F306DC9C883p+23, 0x1.921FB54442D18p0, -0x1p0, 0x1.ffffffd0c621cp-2,
     -0x1.55553e1068f19p-5, 0x1.6c087e89a359dp-10, -0x1.99343027bf8c3p-16, -0x1.555545995a603p-3,
     0x1.1107605230bc4p-7, -0x1.994eb3774cf24p-13}};

__device__ __forceinline__ float sc_poly(double x, double x2, const SinCosTab* p, int n) {
    if ((n & 1) == 0) {
        const double x3 = x * x2;
        const double s1 = p->s2 + x2 * p->s3;
        const double x7 = x3 * x2;
        const double s = x + x3 * p->s1;
        return (float)(s + x7 * s1);
    }
    const double x4 = x2 * x2;
    const double c2 = p->c3 + x2 * p->c4;
    const double c1 = p->c0 + x2 * p->c1;
    const double x6 = x4 * x2;
    const double c = c1 + x4 * p->c2;
    return (float)(c + x6 * c2);
}
// is_cos = 0: sinf(y), 1: cosf(y); valid for 0 <= y < 120
__device__ __forceinline__ float glibc_sincosf(float y, int is_cos) {
    double x = (double)y;
    const SinCosTab* p = &d_sincos[0];
    const unsigned top = (__float_as_uint(y) >> 20) & 0x7ff;
    if (top < ((0x3f490fdbu >> 20) & 0x7ff)) {          // |y| < pi/4 (abstop12 compare)
        const double x2 = x * x;
        if (top < ((0x39800000u >> 20) & 0x7ff)) return is_cos ? 1.0f : y;   // |y| < 2^-12
        return sc_poly(x, x2, p, is_cos);
    }
    const double r = x * p->hpi_inv;
    const int n = ((int)r + 0x800000) >> 24;
    x = x - (double)n * p->hpi;
    const double s = p->sign[n & 3];
    if (n & 2) p = &d_sincos[1];
    return sc_poly(x * s, x * x, p, n ^ is_cos);
}

// cv::fastAtan2 (degrees), float32, every product/sum individually rounded
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {
    const float scale = (float)(180.0 / 3.14159265358979323846);
    const float p1 = 0.9997878412794807f * scale, p3 = -0.3258083974640975f * scale;
    const float p5 = 0.1555786518463281f * scale, p7 = -0.04432655554792128f * scale;
    const float ax = fabsf(x), ay = fabsf(y);
    const float eps = (float)2.2204460492503131e-16;
    float a, c, c2;
    if (ax >= ay) {
        c = __fdiv_rn(ay, __fadd_rn(ax, eps));
        c2 = __fmul_rn(c, c);
        a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
    } else {
        c = __fdiv_rn(ax, __fadd_rn(ay, eps));
        c2 = __fmul_rn(c, c);
        a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
    }
    if (x < 0) a = __fsub_rn(180.f, a);
    if (y < 0) a = __fsub_rn(360.f, a);
    return a;
}

}  // namespace

// 32 registers (8 CTAs/SM): the kernel is bound by gather latency and L1 wavefronts, occupancy pays (0.173 -> 0.150 ms)
__global__ void __launch_bounds__(256, 8) describe_kernel(const __grid_constant__ Geometry g, const uint8_t* __restrict__ pyr,
                                                       const uint8_t* __restrict__ blur, const uint32_t* __restrict__ slots,
                                                       const uint32_t* __restrict__ sel, const int* __restrict__ sel_cnt,
                                                       borb_keypoint* __restrict__ kps, uint8_t* __restrict__ desc,
                                                       int* __restrict__ nkp) {
    __shared__ __align__(4) uint8_t taps[8][512];
    const int img = blockIdx.y;
    const int lane = threadIdx.x & 31;
    const int idx = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    // level lookup through the prefix of per-level counts (levels are concatenated 0..n-1, :1076-1104):
    // lane i holds the inclusive prefix of level i's count; l = number of levels whose prefix is <= idx
    int scan = lane < g.nlevels ? sel_cnt[img * g.nlevels + lane] : 0;
#pragma unroll
    for (int off = 1; off < BORB_MAX_LEVELS; off <<= 1) {
        const int t = __shfl_up_sync(0xFFFFFFFFu, scan, off);
        if (lane >= off) scan += t;
    }
    const int total = __shfl_sync(0xFFFFFFFFu, scan, g.nlevels - 1);
    if (blockIdx.x == 0 && threadIdx.x == 0) nkp[img] = total;
    if (idx >= total) return;
    const int l = __popc(__ballot_sync(0xFFFFFFFFu, lane < g.nlevels && scan <= idx));
    const int base = __shfl_sync(0xFFFFFFFFu, scan, max(l - 1, 0)) & (l > 0 ? -1 : 0);
    const LevelGeom& L = g.lv[l];
    const int pitch = L.pitch;
    const float lscale = L.scale, lpatch = L.patch_size;
    const uint32_t e = sel[(size_t)img * g.sel_image_stride + L.sel_off + (idx - base)];
    const int px = xys_x(e), py = xys_y(e);
    const size_t lvl_off = (size_t)img * g.pyr_image_stride + L.pyr_off;
    // ---- IC_Angle
    // lane = column u of the 31x31 window; the disc is symmetric (umax[v] >= |u| <=> |v| <= umax[|u|]), so a lane's
    // rows are |v| <= vmax.  One multiply-add per pixel: acc += I * (v * 2^13 + 1) carries the column sum (< 2^13) in
    // the low bits and sum_v v*I above them; m10 = sum_u u * (column sum), m01 = sum_u sum_v v * I(u,v).
    const int u = lane - HALF_PATCH;
    const int vmax = lane < 31 ? g.umax[u < 0 ? -u : u] : -1;
    const uint8_t* col = pyr + lvl_off + (size_t)(py - HALF_PATCH) * pitch + (px + u);   // top of this lane's column
    int acc = 0;
#pragma unroll
    for (int vv = -HALF_PATCH; vv <= HALF_PATCH; vv++) {
        if ((vv < 0 ? -vv : vv) <= vmax) acc += (int)*col * (vv * 8192 + 1);
        col += pitch;
    }
    const int colsum = acc & 8191;
    int m01 = acc >> 13;                                   // exact: 0 <= colsum < 2^13
    int m10 = u * colsum;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        m01 += __shfl_xor_sync(0xFFFFFFFFu, m01, off);
        m10 += __shfl_xor_sync(0xFFFFFFFFu, m10, off);
    }
    const float angle = fast_atan2_deg((float)m01, (float)m10);
    // ---- steered BRIEF on the blurred level
    const float factorPI = (float)(3.1415926535897932384626433832795 / 180.f);
    const float t = __fmul_rn(angle, factorPI);
    const float a = glibc_sincosf(t, 1), b = glibc_sincosf(t, 0);
    const uint8_t* cb = blur + lvl_off + (size_t)py * pitch + px;
    const int bin = min((int)(angle * (float)(BRIEF_BINS / 360.0)), BRIEF_BINS - 1);    // fast_atan2_deg may return 360
    const uint32_t* slot = slots + bin * 512 + lane;
    uint8_t* tw = taps[threadIdx.x >> 5];
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const uint32_t s = __ldg(slot + k * 32);
        // x + 128 and y + 128 as the low mantissa bits of 2^23: one PRMT and one exact FADD per coordinate
        const float x = __fsub_rn(__uint_as_float(__byte_perm(s, 0x4B000000u, 0x7440)), 8388736.f);
        const float y = __fsub_rn(__uint_as_float(__byte_perm(s, 0x4B000000u, 0x7441)), 8388736.f);
        const int r = __float2int_rn(__fadd_rn(__fmul_rn(x, b), __fmul_rn(y, a)));
        const int q = __float2int_rn(__fsub_rn(__fmul_rn(x, a), __fmul_rn(y, b)));
        tw[s >> 16] = cb[r * pitch + q];
    }
    __syncwarp();
    unsigned mine = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const unsigned t01 = reinterpret_cast<const uint16_t*>(tw)[j * 32 + lane];    // test 32j + lane: tap 0 low, tap 1 high
        const unsigned word = __ballot_sync(0xFFFFFFFFu, (t01 & 0xFFu) < (t01 >> 8));
        if (lane == j) mine = word;
    }
    const size_t o = (size_t)img * g.sel_image_stride + idx;
    if (lane < 8) reinterpret_cast<unsigned*>(desc + o * 32)[lane] = mine;
    if (lane == 0) {
        borb_keypoint k;
        k.x = __fmul_rn((float)px, lscale);
        k.y = __fmul_rn((float)py, lscale);
        k.size = lpatch;
        k.angle = angle;
        k.response = (float)xys_s(e);
        k.octave = l;
        k.class_id = -1;
        kps[o] = k;
    }
}

int launch_describe(const Geometry& g, const Workspace& ws, int n_images, cudaStream_t s) {
    dim3 grid((g.sel_image_stride + 7) / 8, n_images);
    describe_kernel<<<grid, 256, 0, s>>>(g, ws.pyr, ws.blur, ws.brief_slots, ws.sel, ws.sel_cnt, ws.kps, ws.desc, ws.nkp);
    return 1;
}

}  // namespace borb
