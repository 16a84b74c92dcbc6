// Tail of the Frame constructors on the device (reference src/Frame.cc:61-117 stereo, :119-178 RGB-D, :180-233 monocular), for
// the images an extractor handle has just processed — the keypoints and descriptors never leave HBM between extraction and
// the matcher calls of the same Track():
//   Frame::UndistortKeyPoints      (:404-434)  cv::undistortPoints(mat, mat, mK, mDistCoef, cv::Mat(), mK): double arithmetic,
//                                              five fixed-point iterations of the Brown model, result narrowed to float
//                                              (OpenCV calib3d cvUndistortPointsInternal with its default TermCriteria(MAX_ITER, 5));
//   Frame::ComputeStereoFromRGBD   (:643-664)  d = imDepth.at<float>(v,u) on the DISTORTED keypoint (coordinates truncated),
//                                              mvuRight = kpU.pt.x - mbf/d; the CV_16U -> CV_32F conversion of
//                                              Tracking::GrabImageRGBD (src/Tracking.cc:227-228) is fused into the lookup;
//   Frame::AssignFeaturesToGrid    (:230-245)  one CTA per frame, (cell, insertion) order by a bitonic sort in shared memory.
// A thread per keypoint; frames of a batch are independent jobs (grid.y).  Bound: latency — a frame is ~60 KB.
#include "borb_match.h"
#include "match_rules.cuh"

namespace borb {

// one point through cv::undistortPoints(src, dst, K, D, Mat(), K)
__host__ __device__ inline void undistort_point(float u_in, float v_in, const borb_camera& c, float* xo, float* yo) {
    const double k0 = c.k1, k1 = c.k2, k2 = c.p1, k3 = c.p2, k4 = c.k3;
    const double fx = c.fx, fy = c.fy, cx = c.cx, cy = c.cy;
    const double ifx = 1. / fx, ify = 1. / fy;
    const double u = u_in, v = v_in;
    double x = (u - cx) * ifx, y = (v - cy) * ify;
    const double x0 = x, y0 = y;
    for (int j = 0; j < 5; j++) {
        const double r2 = x * x + y * y;
        // k5..k7 (rational model) are zero: the numerator is (1 + ((0*r2 + 0)*r2 + 0)*r2) = 1 exactly
        const double icdist = 1. / (1 + ((k4 * r2 + k1) * r2 + k0) * r2);
        if (icdist < 0) { x = (u - cx) * ifx; y = (v - cy) * ify; break; }
        const double deltaX = 2 * k2 * x * y + k3 * (r2 + 2 * x * x);
        const double deltaY = k2 * (r2 + 2 * y * y) + 2 * k3 * x * y;
        x = (x0 - deltaX) * icdist; y = (y0 - deltaY) * icdist;
    }
    const double xx = fx * x + cx, yy = fy * y + cy;      // P = K; the zero entries add +-0 and ww = 1/1
    *xo = (float)xx; *yo = (float)yy;
}

void host_image_bounds(int w, int h, const borb_camera& c, float* b4) {       // Frame::ComputeImageBounds (:436-464)
    if (c.k1 != 0.0f) {
        float x[4], y[4];
        const float cu[4] = {0.f, (float)w, 0.f, (float)w}, cv[4] = {0.f, 0.f, (float)h, (float)h};
        for (int i = 0; i < 4; i++) undistort_point(cu[i], cv[i], c, &x[i], &y[i]);
        b4[0] = x[0] < x[2] ? x[0] : x[2]; b4[2] = x[1] > x[3] ? x[1] : x[3];
        b4[1] = y[0] < y[1] ? y[0] : y[1]; b4[3] = y[2] > y[3] ? y[2] : y[3];
    } else { b4[0] = 0.f; b4[1] = 0.f; b4[2] = (float)w; b4[3] = (float)h; }
}

__global__ void __launch_bounds__(256) frame_build_kernel(const FrameJob* __restrict__ jobs, borb_camera cam, int mode, int depth_type,
                                                          float depth_factor, int w, int h, int out_cap, borb_keypoint* __restrict__ keys_out,
                                                          float* __restrict__ ur_out, float* __restrict__ depth_out) {
    const FrameJob J = jobs[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= J.n) return;
    const borb_keypoint kp = J.src_keys[i];
    borb_keypoint ku = kp;
    if (cam.k1 != 0.0f) undistort_point(kp.x, kp.y, cam, &ku.x, &ku.y);
    float ur = -1.f, dp = -1.f;
    if (mode == 2) {                                                    // RGB-D (:643-664)
        const int v = (int)kp.y, u = (int)kp.x;
        if (u >= 0 && v >= 0 && u < w && v < h) {
            float d;
            if (depth_type == 1) d = __fmul_rn((float)reinterpret_cast<const uint16_t*>(J.depth_img)[(size_t)v * w + u], depth_factor);
            else d = reinterpret_cast<const float*>(J.depth_img)[(size_t)v * w + u];
            if (d > 0) { dp = d; ur = __fsub_rn(ku.x, __fdiv_rn(cam.bf, d)); }
        }
    } else if (mode == 1) { ur = J.src_ur[i]; dp = J.src_depth[i]; }    // stereo: the association the extractor handle computed
    J.keys[i] = ku;
    const uint4* sd = reinterpret_cast<const uint4*>(J.src_desc) + (size_t)i * 2;
    uint4* dd = reinterpret_cast<uint4*>(J.desc) + (size_t)i * 2;
    dd[0] = sd[0]; dd[1] = sd[1];
    if (mode != 0) { J.u_right[i] = ur; J.depth[i] = dp; }
    const size_t o = (size_t)blockIdx.y * out_cap + i;
    if (keys_out && i < out_cap) keys_out[o] = ku;
    if (ur_out && i < out_cap) { ur_out[o] = ur; depth_out[o] = dp; }
}

// Frame::AssignFeaturesToGrid for a table of frames, one CTA per job: the frames of borb_frames_from_extractor, and the host views
// and borb_frame_create frames of the matcher calls (borb_match_host.cu), whose rows set only keys, n, the bounds and the grid.
// Sorts (cell, feature index) keys in shared memory; writes cell_start[GRID_CELLS+1] and cell_idx[] in (cell, insertion) order —
// the layout of Frame::mGrid[x][y] (cell = x*48 + y).
__global__ void __launch_bounds__(1024) grid_sort_jobs_kernel(const FrameJob* __restrict__ jobs) {
    extern __shared__ uint32_t skeys[];
    const FrameJob J = jobs[blockIdx.x];
    const int tid = threadIdx.x, T = blockDim.x, n = J.n;
    int K = 32;
    while (K < n) K <<= 1;
    int* cell_start = J.cell_start;
    int* cell_idx = J.cell_idx;
    if (n == 0) { for (int c = tid; c <= GRID_CELLS; c += T) cell_start[c] = 0; return; }
    for (int i = tid; i < K; i += T) {
        uint32_t key = 0xFFFFFFFFu;
        if (i < n) {
            // PosInGrid (Frame.cc:384-385): a NaN coordinate is INT_MIN, so the key is in no cell
            const int px = x86_int(roundf(__fmul_rn(__fsub_rn(J.keys[i].x, J.min_x), J.inv_w)));
            const int py = x86_int(roundf(__fmul_rn(__fsub_rn(J.keys[i].y, J.min_y), J.inv_h)));
            if (px >= 0 && px < GRID_COLS && py >= 0 && py < GRID_ROWS) key = ((uint32_t)(px * GRID_ROWS + py) << 16) | (uint32_t)i;
        }
        skeys[i] = key;
    }
    __syncthreads();
    for (int kk = 2; kk <= K; kk <<= 1)
        for (int j = kk >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < K; i += T) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const bool asc = (i & kk) == 0;
                    const uint32_t a = skeys[i], b = skeys[ixj];
                    if ((a > b) == asc) { skeys[i] = b; skeys[ixj] = a; }
                }
            }
            __syncthreads();
        }
    for (int r = tid; r < K; r += T) {
        const uint32_t key = skeys[r];
        const int cell = key == 0xFFFFFFFFu ? GRID_CELLS : (int)(key >> 16);
        const int prev = r == 0 ? -1 : (skeys[r - 1] == 0xFFFFFFFFu ? GRID_CELLS : (int)(skeys[r - 1] >> 16));
        if (key != 0xFFFFFFFFu) cell_idx[r] = (int)(key & 0xFFFFu);
        for (int c = prev + 1; c <= cell && c <= GRID_CELLS; c++) cell_start[c] = r;
        if (r == K - 1 && cell < GRID_CELLS)
            for (int c = cell + 1; c <= GRID_CELLS; c++) cell_start[c] = K;
    }
}

int launch_frame_build(const FrameJob* d_jobs, int n_jobs, int max_n, const borb_camera& cam, int mode, int depth_type, float depth_factor, int w,
                       int h, int out_cap, borb_keypoint* keys_out, float* ur_out, float* depth_out, cudaStream_t s) {
    if (n_jobs <= 0) return 0;
    int launches = 0;
    if (max_n > 0) {
        dim3 grid((max_n + 255) / 256, n_jobs);
        frame_build_kernel<<<grid, 256, 0, s>>>(d_jobs, cam, mode, depth_type, depth_factor, w, h, out_cap, keys_out, ur_out, depth_out);
        launches++;
    }
    return launches + launch_grid_sort(d_jobs, n_jobs, max_n, s);
}

// One segment per blockIdx.y (borb_frame_from_extractors: the counts, mvKeys, mDescriptors and the right image's, the grid).
__global__ void __launch_bounds__(256) host_copy_kernel(HostCopies c) {
    const HostCopy g = c.seg[blockIdx.y];
    const size_t words = (size_t)(g.count ? *g.count : g.fixed) * (size_t)g.elem_words;
    const uint32_t* __restrict__ src = reinterpret_cast<const uint32_t*>(g.src);
    uint32_t* __restrict__ dst = reinterpret_cast<uint32_t*>(g.dst);
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < words; k += (size_t)gridDim.x * blockDim.x) dst[k] = src[k];
}

int launch_host_copy(const HostCopies& c, cudaStream_t s) {
    if (c.n <= 0) return 0;
    host_copy_kernel<<<dim3(16, c.n), 256, 0, s>>>(c);
    return 1;
}

int launch_grid_sort(const FrameJob* d_jobs, int n_jobs, int max_n, cudaStream_t s) {
    int K = 32;
    while (K < max_n) K <<= 1;
    allow_max_smem((const void*)grid_sort_jobs_kernel);
    grid_sort_jobs_kernel<<<n_jobs, 1024, (size_t)K * 4, s>>>(d_jobs);
    return 1;
}

}  // namespace borb
