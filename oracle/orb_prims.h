// ORACLE — TEST INFRASTRUCTURE ONLY.  Never linked into, imported by, or called from the
// product path (orb_slam2_b200/, include/).  Only tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs may use anything under oracle/.
//
// CPU restatements of the five OpenCV primitives that ORB_SLAM2's ORBextractor.cc calls.
// OpenCV is NOT vendored under /root/reference (find_package(OpenCV), CMakeLists.txt:32-38), so
// these follow OpenCV's published algorithms and are pinned bit-exact against cv2 4.13.0
// (tests/test_oracle_prims.py).  Parity statement: "reference logic + OpenCV 4.13 primitive
// semantics"; the reference itself holds no tests / golden vectors ("parity unpinned" by the
// reference, pinned here by cv2 cross-checks).
//
// Call sites replaced (reference file:line):
//   cv::resize INTER_LINEAR     src/ORBextractor.cc:1120
//   cv::copyMakeBorder          src/ORBextractor.cc:1122,1127
//   cv::FAST(…,true) TYPE_9_16  src/ORBextractor.cc:809,814
//   cv::GaussianBlur 7x7 s=2    src/ORBextractor.cc:1086
//   cv::fastAtan2               src/ORBextractor.cc:103
//   cvRound/cvFloor/cvCeil      src/ORBextractor.cc:81,115,119-120,442,456-460,1112
#pragma once
#include <cstdint>
#include <cstring>
#include <cmath>
#include <cfloat>
#include <vector>
#include <algorithm>

namespace orbprims {

// cvRound: round-half-to-even (SSE cvtsd2si / cvtss2si under the default rounding mode).  The 32-bit conversion saturates:
// NaN and results outside int range give INT_MIN (the "integer indefinite" value), never a wrapped 64-bit result.
static inline int cv_round(double v) {
    const long r = std::lrint(v);
    return (v != v || r < INT32_MIN || r > INT32_MAX) ? INT32_MIN : (int)r;
}
static inline int cv_round(float v) {
    const long r = std::lrintf(v);
    return (v != v || r < INT32_MIN || r > INT32_MAX) ? INT32_MIN : (int)r;
}
static inline int cv_floor(double v) { int i = (int)v; return i - (i > v); }
static inline int cv_ceil(double v) { int i = (int)v; return i + (i < v); }

// BORDER_REFLECT_101 index map (gfedcb|abcdefgh|gfedcba)
static inline int reflect101(int p, int len) {
    if (len == 1) return 0;
    while (p < 0 || p >= len) {
        if (p < 0) p = -p;
        else p = 2 * len - 2 - p;
    }
    return p;
}

// ---------------------------------------------------------------------------------------------
// cv::resize, INTER_LINEAR, CV_8UC1: 11-bit fixed-point coefficient tables, (S>>4)*b>>16 vertical
// pass (OpenCV imgproc/resize.cpp: resizeGeneric_ + HResizeLinear + VResizeLinear<uchar,...>).
// ---------------------------------------------------------------------------------------------
static inline void resize_linear_u8(const uint8_t* src, int sw, int sh, size_t sstep,
                                    uint8_t* dst, int dw, int dh, size_t dstep) {
    const double inv_scale_x = (double)dw / sw, inv_scale_y = (double)dh / sh;
    const double scale_x = 1. / inv_scale_x, scale_y = 1. / inv_scale_y;
    std::vector<int> xofs(dw), yofs(dh);
    std::vector<short> ialpha(dw * 2), ibeta(dh * 2);
    for (int dx = 0; dx < dw; dx++) {
        float fx = (float)((dx + 0.5) * scale_x - 0.5);
        int sx = cv_floor(fx);
        fx -= sx;
        if (sx < 0) { fx = 0; sx = 0; }
        if (sx >= sw - 1) { fx = 0; sx = sw - 1; }
        xofs[dx] = sx;
        ialpha[dx * 2] = (short)cv_round((1.f - fx) * 2048.f);
        ialpha[dx * 2 + 1] = (short)cv_round(fx * 2048.f);
    }
    for (int dy = 0; dy < dh; dy++) {
        float fy = (float)((dy + 0.5) * scale_y - 0.5);
        int sy = cv_floor(fy);
        fy -= sy;
        yofs[dy] = sy;
        ibeta[dy * 2] = (short)cv_round((1.f - fy) * 2048.f);
        ibeta[dy * 2 + 1] = (short)cv_round(fy * 2048.f);
    }
    std::vector<int> row0(dw), row1(dw);
    auto hrow = [&](int sy, std::vector<int>& out) {
        sy = sy < 0 ? 0 : (sy >= sh ? sh - 1 : sy);
        const uint8_t* S = src + (size_t)sy * sstep;
        for (int dx = 0; dx < dw; dx++) {
            int sx = xofs[dx];
            int sx1 = sx + 1 < sw ? sx + 1 : sx;
            out[dx] = S[sx] * ialpha[dx * 2] + S[sx1] * ialpha[dx * 2 + 1];
        }
    };
    for (int dy = 0; dy < dh; dy++) {
        hrow(yofs[dy], row0);
        hrow(yofs[dy] + 1, row1);
        const int b0 = ibeta[dy * 2], b1 = ibeta[dy * 2 + 1];
        uint8_t* D = dst + (size_t)dy * dstep;
        for (int x = 0; x < dw; x++)
            D[x] = (uint8_t)((((b0 * (row0[x] >> 4)) >> 16) + ((b1 * (row1[x] >> 4)) >> 16) + 2) >> 2);
    }
}

// ---------------------------------------------------------------------------------------------
// cv::FAST(img, kps, threshold, nonmaxSuppression=true), TYPE_9_16 (OpenCV features2d/fast.cpp,
// FAST_t<16> + cornerScore<16>).  Output raster order; each entry (x, y, score).
// ---------------------------------------------------------------------------------------------
struct FastPt { int x, y, score; };

static inline void fast_offsets16(int pixel[25], int step) {
    static const int offs[16][2] = {{0, 3},  {1, 3},   {2, 2},   {3, 1},  {3, 0},  {3, -1},
                                    {2, -2}, {1, -3},  {0, -3},  {-1, -3}, {-2, -2}, {-3, -1},
                                    {-3, 0}, {-3, 1},  {-2, 2},  {-1, 3}};
    for (int k = 0; k < 16; k++) pixel[k] = offs[k][0] + offs[k][1] * step;
    for (int k = 16; k < 25; k++) pixel[k] = pixel[k - 16];
}

static inline int fast_corner_score16(const uint8_t* ptr, const int pixel[25], int threshold) {
    const int K = 8, N = K * 3 + 1;
    int k, v = ptr[0];
    short d[N];
    for (k = 0; k < N; k++) d[k] = (short)(v - ptr[pixel[k]]);
    int a0 = threshold;
    for (k = 0; k < 16; k += 2) {
        int a = std::min((int)d[k + 1], (int)d[k + 2]);
        a = std::min(a, (int)d[k + 3]);
        if (a <= a0) continue;
        a = std::min(a, (int)d[k + 4]);
        a = std::min(a, (int)d[k + 5]);
        a = std::min(a, (int)d[k + 6]);
        a = std::min(a, (int)d[k + 7]);
        a = std::min(a, (int)d[k + 8]);
        a0 = std::max(a0, std::min(a, (int)d[k]));
        a0 = std::max(a0, std::min(a, (int)d[k + 9]));
    }
    int b0 = -a0;
    for (k = 0; k < 16; k += 2) {
        int b = std::max((int)d[k + 1], (int)d[k + 2]);
        b = std::max(b, (int)d[k + 3]);
        b = std::max(b, (int)d[k + 4]);
        b = std::max(b, (int)d[k + 5]);
        if (b >= b0) continue;
        b = std::max(b, (int)d[k + 6]);
        b = std::max(b, (int)d[k + 7]);
        b = std::max(b, (int)d[k + 8]);
        b0 = std::min(b0, std::max(b, (int)d[k]));
        b0 = std::min(b0, std::max(b, (int)d[k + 9]));
    }
    return -b0 - 1;
}

static inline void fast9_16(const uint8_t* img, int cols, int rows, size_t step, int threshold,
                            bool nms, std::vector<FastPt>& out) {
    out.clear();
    if (cols < 7 || rows < 7) return;
    const int K = 8, N = 25;
    int pixel[25];
    fast_offsets16(pixel, (int)step);
    threshold = std::min(std::max(threshold, 0), 255);
    uint8_t tab[512];
    for (int i = -255; i <= 255; i++) tab[i + 255] = (uint8_t)(i < -threshold ? 1 : i > threshold ? 2 : 0);
    std::vector<uint8_t> sbuf((size_t)cols * 3, 0);
    std::vector<int> cbuf((size_t)(cols + 1) * 3, 0);
    uint8_t* buf[3] = {sbuf.data(), sbuf.data() + cols, sbuf.data() + 2 * cols};
    int* cpbuf[3] = {cbuf.data(), cbuf.data() + cols + 1, cbuf.data() + 2 * (cols + 1)};
    for (int i = 3; i < rows - 2; i++) {
        const uint8_t* ptr = img + (size_t)i * step + 3;
        uint8_t* curr = buf[(i - 3) % 3];
        int* cornerpos = cpbuf[(i - 3) % 3] + 1;
        std::memset(curr, 0, cols);
        int ncorners = 0;
        if (i < rows - 3) {
            for (int j = 3; j < cols - 3; j++, ptr++) {
                int v = ptr[0];
                const uint8_t* t = &tab[0] - v + 255;
                int d = t[ptr[pixel[0]]] | t[ptr[pixel[8]]];
                if (d == 0) continue;
                d &= t[ptr[pixel[2]]] | t[ptr[pixel[10]]];
                d &= t[ptr[pixel[4]]] | t[ptr[pixel[12]]];
                d &= t[ptr[pixel[6]]] | t[ptr[pixel[14]]];
                if (d == 0) continue;
                d &= t[ptr[pixel[1]]] | t[ptr[pixel[9]]];
                d &= t[ptr[pixel[3]]] | t[ptr[pixel[11]]];
                d &= t[ptr[pixel[5]]] | t[ptr[pixel[13]]];
                d &= t[ptr[pixel[7]]] | t[ptr[pixel[15]]];
                if (d & 1) {
                    int vt = v - threshold, count = 0;
                    for (int k = 0; k < N; k++) {
                        int x = ptr[pixel[k]];
                        if (x < vt) {
                            if (++count > K) {
                                cornerpos[ncorners++] = j;
                                if (nms) curr[j] = (uint8_t)fast_corner_score16(ptr, pixel, threshold);
                                break;
                            }
                        } else
                            count = 0;
                    }
                }
                if (d & 2) {
                    int vt = v + threshold, count = 0;
                    for (int k = 0; k < N; k++) {
                        int x = ptr[pixel[k]];
                        if (x > vt) {
                            if (++count > K) {
                                cornerpos[ncorners++] = j;
                                if (nms) curr[j] = (uint8_t)fast_corner_score16(ptr, pixel, threshold);
                                break;
                            }
                        } else
                            count = 0;
                    }
                }
            }
        }
        cornerpos[-1] = ncorners;
        if (i == 3) continue;
        const uint8_t* prev = buf[(i - 4 + 3) % 3];
        const uint8_t* pprev = buf[(i - 5 + 3) % 3];
        cornerpos = cpbuf[(i - 4 + 3) % 3] + 1;
        ncorners = cornerpos[-1];
        for (int k = 0; k < ncorners; k++) {
            int j = cornerpos[k];
            int score = prev[j];
            if (!nms || (score > prev[j + 1] && score > prev[j - 1] && score > pprev[j - 1] &&
                         score > pprev[j] && score > pprev[j + 1] && score > curr[j - 1] &&
                         score > curr[j] && score > curr[j + 1]))
                out.push_back(FastPt{j, i - 1, score});
        }
    }
}

// ---------------------------------------------------------------------------------------------
// cv::GaussianBlur(7x7, sigma 2, BORDER_REFLECT_101) on CV_8UC1 — OpenCV >= 3.4 fixed-point path
// (imgproc/smooth.dispatch.cpp: ufixedpoint16 kernel from getGaussianKernelFixedPoint_ED).
// Kernel bits (x/256): 18 34 48 56 48 34 18.  Row pass exact u16, column pass (sum+2^15)>>16.
// In-place safe (src may equal dst).
// ---------------------------------------------------------------------------------------------
static inline void gaussian_blur7_u8(const uint8_t* src, int w, int h, size_t sstep, uint8_t* dst,
                                     size_t dstep) {
    static const int q[7] = {18, 34, 48, 56, 48, 34, 18};
    std::vector<uint16_t> tmp((size_t)w * h);
    std::vector<int> xi(w + 6);
    for (int x = -3; x < w + 3; x++) xi[x + 3] = reflect101(x, w);
    for (int y = 0; y < h; y++) {
        const uint8_t* S = src + (size_t)y * sstep;
        uint16_t* T = tmp.data() + (size_t)y * w;
        for (int x = 0; x < w; x++) {
            int s = 0;
            for (int k = 0; k < 7; k++) s += q[k] * S[xi[x + k]];
            T[x] = (uint16_t)s;
        }
    }
    for (int y = 0; y < h; y++) {
        const uint16_t* R[7];
        for (int k = 0; k < 7; k++) R[k] = tmp.data() + (size_t)reflect101(y + k - 3, h) * w;
        uint8_t* D = dst + (size_t)y * dstep;
        for (int x = 0; x < w; x++) {
            uint32_t s = 0;
            for (int k = 0; k < 7; k++) s += (uint32_t)q[k] * R[k][x];
            uint32_t v = (s + 32768u) >> 16;
            D[x] = (uint8_t)(v > 255 ? 255 : v);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// cv::fastAtan2(y, x) — degrees in [0,360), float32 7th-order odd polynomial
// (OpenCV core/mathfuncs_core.simd.hpp atan_f32 / fastAtan2 scalar).  Every op is float32,
// no FMA contraction (build with -ffp-contract=off).
// ---------------------------------------------------------------------------------------------
static inline float fast_atan2(float y, float x) {
    const float scale = (float)(180.0 / 3.14159265358979323846);
    const float p1 = 0.9997878412794807f * scale;
    const float p3 = -0.3258083974640975f * scale;
    const float p5 = 0.1555786518463281f * scale;
    const float p7 = -0.04432655554792128f * scale;
    float ax = std::fabs(x), ay = std::fabs(y);
    float a, c, c2;
    if (ax >= ay) {
        c = ay / (ax + (float)DBL_EPSILON);
        c2 = c * c;
        a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    } else {
        c = ax / (ay + (float)DBL_EPSILON);
        c2 = c * c;
        a = 90.f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    }
    if (x < 0) a = 180.f - a;
    if (y < 0) a = 360.f - a;
    return a;
}

// cv::cvtColor(src, dst, COLOR_RGB2GRAY / BGR2GRAY / RGBA2GRAY / BGRA2GRAY) on CV_8U — what Tracking::GrabImage* applies to
// colour frames (reference src/Tracking.cc:172-197).  OpenCV 4.13: Y = (R*9798 + G*19235 + B*3735 + 2^14) >> 15.
static inline void cvt_color_to_gray_u8(const uint8_t* src, int w, int h, size_t sstep, int channels, bool rgb_order, uint8_t* dst,
                                        size_t dstep) {
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const uint8_t* p = src + y * sstep + (size_t)x * channels;
            const int R = rgb_order ? p[0] : p[2], G = p[1], B = rgb_order ? p[2] : p[0];
            dst[y * dstep + x] = (uint8_t)((R * 9798 + G * 19235 + B * 3735 + 16384) >> 15);
        }
}

// cv::remap(src, dst, map_x, map_y, INTER_LINEAR) (BORDER_CONSTANT 0) with CV_32FC1 maps on CV_8UC1 — the per-frame
// rectification of reference Examples/Stereo/stereo_euroc.cc:136-137.  OpenCV fixed point: 1/32-px coordinates by
// cvRound, bilinear weights scaled to 2^15 (exact for 1/32 fractions), result (sum + 2^14) >> 15.
static inline void remap_linear_u8(const uint8_t* src, int sw, int sh, size_t sstep, const float* mx, const float* my, uint8_t* dst,
                                   int dw, int dh, size_t dstep) {
    for (int y = 0; y < dh; y++)
        for (int x = 0; x < dw; x++) {
            const int sx = cv_round(mx[(size_t)y * dw + x] * 32.f), sy = cv_round(my[(size_t)y * dw + x] * 32.f);
            int ix = sx >> 5, iy = sy >> 5;
            ix = ix < -32768 ? -32768 : (ix > 32767 ? 32767 : ix);
            iy = iy < -32768 ? -32768 : (iy > 32767 ? 32767 : iy);
            const int fx = sx & 31, fy = sy & 31;
            auto tap = [&](int yy, int xx) -> int { return (xx >= 0 && xx < sw && yy >= 0 && yy < sh) ? src[yy * sstep + xx] : 0; };
            const int w00 = (32 - fx) * (32 - fy) * 32, w01 = fx * (32 - fy) * 32, w10 = (32 - fx) * fy * 32, w11 = fx * fy * 32;
            dst[y * dstep + x] = (uint8_t)((tap(iy, ix) * w00 + tap(iy, ix + 1) * w01 + tap(iy + 1, ix) * w10 + tap(iy + 1, ix + 1) * w11 + 16384) >> 15);
        }
}

}  // namespace orbprims
