// Scale pyramid: level l = fixed-point bilinear downscale of level l-1 (chain), all images of the batch
// per launch.  Replaces ORBextractor::ComputePyramid (reference src/ORBextractor.cc:1107-1132), i.e.
// cv::resize(INTER_LINEAR) on CV_8UC1: 11-bit coefficient tables, horizontal pass in int32, vertical
// pass (((b0*(r0>>4))>>16) + ((b1*(r1>>4))>>16) + 2) >> 2.
//
// Layout: every level row carries >= 8 bytes of reflect-101 padding after its last pixel (the only part of the
// reference's 19-px copyMakeBorder that any later stage needs: the 7x7 blur reads up to 7 bytes past the row end
// as aligned words).  The padding columns are produced here as ordinary pixels through table entries that point at
// the reflected column.
//
// A thread makes 4 destination pixels x ROWS rows.  Per pixel one 8-byte table entry {c0|c1<<16, base|selectors<<16}
// built on the host (borb_host.cu resize_window_table): the two source rows come in as three aligned 32-bit words
// each (the group's 12-byte window), the byte pair (ofs, ofs+1) is pulled out with two table-driven PRMTs and the
// horizontal pass is one IDP.2A (dp2a) per pixel and row; no data-dependent selects or branches.
// Levels whose groups do not fit a 12-byte window (scale factors above ~2) take pyr_resize_generic_kernel.
//
// Bound: ALU/FMA issue (integer work per pixel); traffic sum_{l>=1} w_l*h_l bytes written + read per image.
#include "borb_internal.h"

namespace borb {

template <int ROWS>
__global__ void __launch_bounds__(256, 6) pyr_resize_kernel(const uint8_t* __restrict__ pyr, uint8_t* __restrict__ pyr_out,
                                                         const int16_t* __restrict__ tabs, LevelGeom src, LevelGeom dst,
                                                         unsigned image_stride) {
    const int img = blockIdx.z;
    const int dyb = (blockIdx.y * 8 + threadIdx.y) * ROWS;
    const int dx0 = (blockIdx.x * 32 + threadIdx.x) * 4;
    const int wpad = (dst.w + 8 + 3) & ~3;                  // pixels + reflect padding, whole words
    if (dyb >= dst.h || dx0 >= wpad) return;
    const uint8_t* S = pyr + (size_t)img * image_stride + src.pyr_off;
    uint8_t* D = pyr_out + (size_t)img * image_stride + dst.pyr_off;
    const uint4* xt = reinterpret_cast<const uint4*>(tabs + ((size_t)dst.xwin_off + dx0) * 4);   // 16-byte aligned
    const uint2* yt = reinterpret_cast<const uint2*>(tabs + (size_t)dst.ytab_off * 4);
    const uint4 e01 = xt[0], e23 = xt[1];
    const uint32_t wts[4] = {e01.x, e01.z, e23.x, e23.z};
    const uint32_t ctl[4] = {e01.y, e01.w, e23.y, e23.w};
    const int base = (int)(ctl[0] & 0xFFFF);
    uint32_t ra[ROWS][3], rc[ROWS][3];
    uint32_t B0[ROWS], B1[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; r++) {
        const int dy = min(dyb + r, dst.h - 1);
        const uint2 ye = yt[dy];
        const int sy = (int)(short)(ye.x & 0xFFFF);
        B0[r] = ye.x & 0xFFFF0000u;                         // b0 << 16: (b0 * v) >> 16 == umulhi(b0 << 16, v)
        B1[r] = ye.y << 16;
        const int sy0 = min(max(sy, 0), src.h - 1), sy1 = min(max(sy + 1, 0), src.h - 1);
        const uint32_t* R0 = reinterpret_cast<const uint32_t*>(S + (size_t)sy0 * src.pitch + base);
        const uint32_t* R1 = reinterpret_cast<const uint32_t*>(S + (size_t)sy1 * src.pitch + base);
        ra[r][0] = R0[0]; ra[r][1] = R0[1]; ra[r][2] = R0[2];
        rc[r][0] = R1[0]; rc[r][1] = R1[1]; rc[r][2] = R1[2];
    }
#pragma unroll
    for (int r = 0; r < ROWS; r++) {
        if (dyb + r >= dst.h) break;
        uint32_t v[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const uint32_t s1 = ctl[i] >> 16, s2 = ctl[i] >> 24;        // PRMT reads the low 16 bits only
            const uint32_t p0 = __byte_perm(__byte_perm(ra[r][0], ra[r][1], s1), ra[r][2], s2);
            const uint32_t p1 = __byte_perm(__byte_perm(rc[r][0], rc[r][1], s1), rc[r][2], s2);
            const uint32_t h0 = __dp2a_lo(wts[i], p0, 0u), h1 = __dp2a_lo(wts[i], p1, 0u);
            v[i] = (__umulhi(B0[r], h0 >> 4) + __umulhi(B1[r], h1 >> 4) + 2) >> 2;
        }
        const uint32_t out = __byte_perm(__byte_perm(v[0], v[1], 0x0040), __byte_perm(v[2], v[3], 0x0040), 0x5410);
        // rows are pitch-aligned (pitch % 128 == 0, pitch >= w + 8) and dx0 % 4 == 0: one aligned 32-bit store
        *reinterpret_cast<uint32_t*>(D + (size_t)(dyb + r) * dst.pitch + dx0) = out;
    }
}

// Any scale factor: one destination pixel per thread, byte loads through the plain {ofs, c0, c1} table.
__global__ void __launch_bounds__(256) pyr_resize_generic_kernel(const uint8_t* __restrict__ pyr, uint8_t* __restrict__ pyr_out,
                                                                 const int16_t* __restrict__ tabs, LevelGeom src, LevelGeom dst,
                                                                 unsigned image_stride) {
    const int img = blockIdx.z;
    const int dy = blockIdx.y * 8 + threadIdx.y;
    const int dx = blockIdx.x * 32 + threadIdx.x;
    const int wpad = (dst.w + 8 + 3) & ~3;
    if (dy >= dst.h || dx >= wpad) return;
    const uint8_t* S = pyr + (size_t)img * image_stride + src.pyr_off;
    uint8_t* D = pyr_out + (size_t)img * image_stride + dst.pyr_off;
    const short4 xe = reinterpret_cast<const short4*>(tabs)[(size_t)dst.xtab_off + dx];
    const short4 ye = reinterpret_cast<const short4*>(tabs)[(size_t)dst.ytab_off + dy];
    const int sy0 = min(max((int)ye.x, 0), src.h - 1), sy1 = min(max((int)ye.x + 1, 0), src.h - 1);
    const uint8_t* R0 = S + (size_t)sy0 * src.pitch;
    const uint8_t* R1 = S + (size_t)sy1 * src.pitch;
    const int sx = xe.x;                                     // sx + 1 <= src.w: inside the row's reflect padding
    const int r0 = R0[sx] * xe.y + R0[sx + 1] * xe.z;
    const int r1 = R1[sx] * xe.y + R1[sx + 1] * xe.z;
    D[(size_t)dy * dst.pitch + dx] = (uint8_t)((((ye.y * (r0 >> 4)) >> 16) + ((ye.z * (r1 >> 4)) >> 16) + 2) >> 2);
}

// Level 0 from a tightly packed landing buffer (one big H2D copy) into the pitched pyramid layout.
__global__ void __launch_bounds__(256) repack_kernel(const uint8_t* __restrict__ stage, int src_stride, size_t src_image_bytes,
                                                     uint8_t* __restrict__ pyr, LevelGeom l0, unsigned image_stride) {
    const int img = blockIdx.z, y = blockIdx.y;
    const int x0 = (blockIdx.x * 256 + threadIdx.x) * 4;
    if (x0 >= l0.w) return;
    const uint8_t* S = stage + (size_t)img * src_image_bytes + (size_t)y * src_stride + x0;
    uint32_t v = 0;
#pragma unroll
    for (int i = 0; i < 4; i++)
        if (x0 + i < l0.w) v |= (uint32_t)S[i] << (8 * i);
    *reinterpret_cast<uint32_t*>(pyr + (size_t)img * image_stride + l0.pyr_off + (size_t)y * l0.pitch + x0) = v;
}

// Colour input: Tracking::GrabImage* convert with cv::cvtColor(RGB2GRAY / BGR2GRAY / RGBA2GRAY / BGRA2GRAY) before the
// extractor is called (reference src/Tracking.cc:172-197, 211-223, 243-255).  Fused into the re-pitch of the upload;
// OpenCV 4.13 8-bit semantics (checked exhaustively over all 2^24 colours against cv2):
//   Y = (R*9798 + G*19235 + B*3735 + 2^14) >> 15
__global__ void __launch_bounds__(256) repack_color_kernel(const uint8_t* __restrict__ stage, int src_stride, size_t src_image_bytes,
                                                           int channels, int rgb, uint8_t* __restrict__ pyr, LevelGeom l0,
                                                           unsigned image_stride) {
    const int img = blockIdx.z, y = blockIdx.y;
    const int x0 = (blockIdx.x * 256 + threadIdx.x) * 4;
    if (x0 >= l0.w) return;
    const uint8_t* S = stage + (size_t)img * src_image_bytes + (size_t)y * src_stride + (size_t)x0 * channels;
    const int cr = rgb ? 9798 : 3735, cb = rgb ? 3735 : 9798;      // weight of channel 0 / channel 2
    uint32_t v = 0;
#pragma unroll
    for (int i = 0; i < 4; i++)
        if (x0 + i < l0.w) {
            const uint8_t* px = S + i * channels;
            const int yv = (px[0] * cr + px[1] * 19235 + px[2] * cb + 16384) >> 15;
            v |= (uint32_t)yv << (8 * i);
        }
    *reinterpret_cast<uint32_t*>(pyr + (size_t)img * image_stride + l0.pyr_off + (size_t)y * l0.pitch + x0) = v;
}

// Stereo rectification of the raw camera frame, fused into the upload: cv::remap(im, imRect, M1, M2, cv::INTER_LINEAR) of
// reference Examples/Stereo/stereo_euroc.cc:136-137 with the CV_32FC1 maps of cv::initUndistortRectifyMap (:96-98).
// OpenCV semantics (pinned against cv2.remap in tests/test_oracle_prims.py): coordinates to 1/32 px with cvRound,
//   sx = cvRound(mapx*32), ix = sx >> 5, fx = sx & 31 (same for y); weights (32-fx)(32-fy)*32 ... (sum 2^15, exact);
//   out = (sum w*p + 2^14) >> 15; taps outside the source read 0 (BORDER_CONSTANT).
// Image k of the batch uses map set (k & 1) when two sets are given (left / right), else set 0.
__global__ void __launch_bounds__(256) repack_remap_kernel(const uint8_t* __restrict__ stage, int src_stride, size_t src_image_bytes,
                                                           int src_w, int src_h, const float* __restrict__ mx0,
                                                           const float* __restrict__ my0, const float* __restrict__ mx1,
                                                           const float* __restrict__ my1, uint8_t* __restrict__ pyr, LevelGeom l0,
                                                           unsigned image_stride) {
    const int img = blockIdx.z, y = blockIdx.y;
    const int x0 = (blockIdx.x * 256 + threadIdx.x) * 4;
    if (x0 >= l0.w) return;
    const bool second = (img & 1) && mx1 != nullptr;
    const float* MX = second ? mx1 : mx0;
    const float* MY = second ? my1 : my0;
    const uint8_t* S = stage + (size_t)img * src_image_bytes;
    uint32_t v = 0;
#pragma unroll
    for (int i = 0; i < 4; i++)
        if (x0 + i < l0.w) {
            const size_t o = (size_t)y * l0.w + x0 + i;
            // cvRound gives INT_MIN for NaN (the pixel reads the border); __float2int_rn(NaN) would be 0, i.e. pixel (0, 0).
            // Out-of-range values saturate either way and land outside any source image.
            const float mx = __fmul_rn(MX[o], 32.f), my = __fmul_rn(MY[o], 32.f);
            const int sx = mx == mx ? __float2int_rn(mx) : INT_MIN, sy = my == my ? __float2int_rn(my) : INT_MIN;
            const int ix = max(-32768, min(32767, sx >> 5)), iy = max(-32768, min(32767, sy >> 5));     // saturate_cast<short>
            const int fx = sx & 31, fy = sy & 31;
            auto tap = [&](int yy, int xx) -> int {
                return (xx >= 0 && xx < src_w && yy >= 0 && yy < src_h) ? (int)S[(size_t)yy * src_stride + xx] : 0;
            };
            const int w00 = (32 - fx) * (32 - fy) * 32, w01 = fx * (32 - fy) * 32, w10 = (32 - fx) * fy * 32, w11 = fx * fy * 32;
            const int r = (tap(iy, ix) * w00 + tap(iy, ix + 1) * w01 + tap(iy + 1, ix) * w10 + tap(iy + 1, ix + 1) * w11 + 16384) >> 15;
            v |= (uint32_t)r << (8 * i);
        }
    *reinterpret_cast<uint32_t*>(pyr + (size_t)img * image_stride + l0.pyr_off + (size_t)y * l0.pitch + x0) = v;
}

// reflect-101 padding of level 0 (columns w .. w+7 = columns w-2 .. w-9), after any kind of upload
__global__ void __launch_bounds__(256) pad_level0_kernel(uint8_t* __restrict__ pyr, LevelGeom l0, unsigned image_stride) {
    const int y = blockIdx.x * 256 + threadIdx.x, img = blockIdx.y;
    if (y >= l0.h) return;
    uint8_t* row = pyr + (size_t)img * image_stride + l0.pyr_off + (size_t)y * l0.pitch;
#pragma unroll
    for (int k = 0; k < 8; k++) row[l0.w + k] = row[max(l0.w - 2 - k, 0)];
}

int launch_repack(const Geometry& g, const Workspace& ws, const uint8_t* stage, int src_stride, size_t src_image_bytes,
                  int n_images, cudaStream_t s) {
    dim3 grid((g.lv[0].w + 1023) / 1024, g.lv[0].h, n_images);
    repack_kernel<<<grid, 256, 0, s>>>(stage, src_stride, src_image_bytes, ws.pyr, g.lv[0], g.pyr_image_stride);
    return 1;
}

constexpr int PYR_ROWS = 2;

int launch_repack_remap(const Geometry& g, const Workspace& ws, const uint8_t* stage, int src_stride, size_t src_image_bytes, int src_w,
                        int src_h, const float* mx0, const float* my0, const float* mx1, const float* my1, int n_images, cudaStream_t s) {
    dim3 grid((g.lv[0].w + 1023) / 1024, g.lv[0].h, n_images);
    repack_remap_kernel<<<grid, 256, 0, s>>>(stage, src_stride, src_image_bytes, src_w, src_h, mx0, my0, mx1, my1, ws.pyr, g.lv[0],
                                             g.pyr_image_stride);
    return 1;
}

int launch_repack_color(const Geometry& g, const Workspace& ws, const uint8_t* stage, int src_stride, size_t src_image_bytes, int channels,
                        int rgb, int n_images, cudaStream_t s) {
    dim3 grid((g.lv[0].w + 1023) / 1024, g.lv[0].h, n_images);
    repack_color_kernel<<<grid, 256, 0, s>>>(stage, src_stride, src_image_bytes, channels, rgb, ws.pyr, g.lv[0], g.pyr_image_stride);
    return 1;
}

int launch_pyramid(const Geometry& g, const Workspace& ws, int n_images, cudaStream_t s) {
    int launches = 0;
    pad_level0_kernel<<<dim3((g.lv[0].h + 255) / 256, n_images), 256, 0, s>>>(ws.pyr, g.lv[0], g.pyr_image_stride);
    launches++;
    for (int l = 1; l < g.nlevels; l++) {
        const LevelGeom& d = g.lv[l];
        dim3 block(32, 8);
        if (d.x_windowed) {
            dim3 grid((d.w + 8 + 127) / 128, (d.h + 8 * PYR_ROWS - 1) / (8 * PYR_ROWS), n_images);
            pyr_resize_kernel<PYR_ROWS><<<grid, block, 0, s>>>(ws.pyr, ws.pyr, ws.tabs, g.lv[l - 1], d, g.pyr_image_stride);
        } else {
            dim3 grid((d.w + 8 + 3 + 31) / 32, (d.h + 7) / 8, n_images);
            pyr_resize_generic_kernel<<<grid, block, 0, s>>>(ws.pyr, ws.pyr, ws.tabs, g.lv[l - 1], d, g.pyr_image_stride);
        }
        launches++;
    }
    return launches;
}

}  // namespace borb
