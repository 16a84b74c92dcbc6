// Device rules every ORBmatcher search shares (reference src/ORBmatcher.cc), written once for k_match.cu, k_proj.cu, k_bowdb.cu,
// k_stereo.cu and k_frame.cu.  Device code only.  All float steps use _rn intrinsics (no FMA contraction) so results match the reference bit
// for bit.
#pragma once
#include <climits>
#include <cstdint>

namespace borb {

namespace {

constexpr int HISTO_LENGTH = 30;                 // ORBmatcher::HISTO_LENGTH (:39)

// (int)v as the reference computes it on x86 (cvttss2si): NaN, +-inf and every value outside [-2^31, 2^31) give INT_MIN.  The
// device conversion saturates instead (+inf and large values INT_MAX, NaN 0), which would put a NaN key into grid column 0 and
// turn a window edge past 2^31 into the last grid column.
__device__ __forceinline__ int x86_int(float v) { return (v >= -2147483648.f && v < 2147483648.f) ? (int)v : INT_MIN; }

// ORBmatcher::DescriptorDistance (:1646-1662) of two 256-bit descriptors given as 8 words each
__device__ __forceinline__ int descriptor_distance(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b) {
    int d = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) d += __popc(a[i] ^ b[i]);
    return d;
}

// the same on descriptors held as two uint4 halves each
__device__ __forceinline__ int descriptor_distance(const uint4 a0, const uint4 a1, const uint4 b0, const uint4 b1) {
    const uint32_t x0 = a0.x ^ b0.x, x1 = a0.y ^ b0.y, x2 = a0.z ^ b0.z, x3 = a0.w ^ b0.w;
    const uint32_t x4 = a1.x ^ b1.x, x5 = a1.y ^ b1.y, x6 = a1.z ^ b1.z, x7 = a1.w ^ b1.w;
    return __popc(x0) + __popc(x1) + __popc(x2) + __popc(x3) + __popc(x4) + __popc(x5) + __popc(x6) + __popc(x7);
}

// rotation-histogram bin of an angle difference (:238-243): rot + 360 below 0, round(rot * (1.0f / HISTO_LENGTH)), 30 wraps to 0
__device__ __forceinline__ int rot_bin(float a1, float a2) {
    float rot = __fsub_rn(a1, a2);
    if (rot < 0.0f) rot = __fadd_rn(rot, 360.0f);
    int bin = (int)roundf(__fmul_rn(rot, 1.0f / HISTO_LENGTH));
    if (bin == HISTO_LENGTH) bin = 0;
    return bin;
}

// ORBmatcher::ComputeThreeMaxima (:1601-1642) on bin counts: the three fullest bins, a bin below 0.1 of the fullest dropped as -1
__device__ __forceinline__ void three_maxima(const int* cnt, int& ind1, int& ind2, int& ind3) {
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

// the minimum of v over the warp: the (distance, position) keys of the searches' first-minimum rules
__device__ __forceinline__ unsigned warp_min(unsigned v) {
    return __reduce_min_sync(0xFFFFFFFFu, v);        // REDUX: one instruction instead of a 5-step shuffle chain (the replays are latency chains)
}

}  // namespace

}  // namespace borb
