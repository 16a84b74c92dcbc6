// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle/orb_prims.h header).
// C exports of the OpenCV-primitive restatements so tests can pin them against cv2 4.13.
#include "orb_prims.h"

#include <math.h>
#include <thread>

extern "C" {

void orbport_resize_linear(const uint8_t* src, int sw, int sh, int sstep, uint8_t* dst, int dw, int dh, int dstep) {
    orbprims::resize_linear_u8(src, sw, sh, (size_t)sstep, dst, dw, dh, (size_t)dstep);
}
void orbport_gaussian_blur7(const uint8_t* src, int w, int h, int sstep, uint8_t* dst, int dstep) {
    orbprims::gaussian_blur7_u8(src, w, h, (size_t)sstep, dst, (size_t)dstep);
}
// cv::FAST(img, kps, threshold, true): returns count; xys = (x,y,score) triples in raster order
int orbport_fast9(const uint8_t* img, int w, int h, int step, int threshold, int nms, int32_t* xys, int cap) {
    std::vector<orbprims::FastPt> pts;
    orbprims::fast9_16(img, w, h, (size_t)step, threshold, nms != 0, pts);
    for (int i = 0; i < (int)pts.size() && i < cap; i++) { xys[3 * i] = pts[i].x; xys[3 * i + 1] = pts[i].y; xys[3 * i + 2] = pts[i].score; }
    return (int)pts.size();
}
void orbport_fast_atan2(const float* y, const float* x, float* out, int n) {
    for (int i = 0; i < n; i++) out[i] = orbprims::fast_atan2(y[i], x[i]);
}
// The host libm itself (fn 0 ::sinf, 1 ::cosf, 2 ::logf), element-wise over a few threads: the reference the device ports of
// glibc sinf/cosf (describe) and logf (PredictScale) are compared with.  Called through a pointer, so no builtin is folded in.
void orbport_libm(int fn, const float* in, float* out, int64_t n) {
    float (*const f)(float) = fn == 0 ? ::sinf : fn == 1 ? ::cosf : ::logf;
    const int64_t nt = std::max<int64_t>(1, std::min<int64_t>({(int64_t)std::thread::hardware_concurrency(), 16, n / 65536}));
    std::vector<std::thread> pool;
    for (int64_t t = 0; t < nt; t++)
        pool.emplace_back([=] {
            for (int64_t i = n * t / nt; i < n * (t + 1) / nt; i++) out[i] = f(in[i]);
        });
    for (std::thread& th : pool) th.join();
}
int orbport_reflect101(int p, int len) { return orbprims::reflect101(p, len); }
void orbport_cvt_color_to_gray(const uint8_t* src, int w, int h, int sstep, int channels, int rgb_order, uint8_t* dst, int dstep) {
    orbprims::cvt_color_to_gray_u8(src, w, h, (size_t)sstep, channels, rgb_order != 0, dst, (size_t)dstep);
}
void orbport_remap_linear(const uint8_t* src, int sw, int sh, int sstep, const float* mx, const float* my, uint8_t* dst, int dw, int dh,
                          int dstep) {
    orbprims::remap_linear_u8(src, sw, sh, (size_t)sstep, mx, my, dst, dw, dh, (size_t)dstep);
}
}
