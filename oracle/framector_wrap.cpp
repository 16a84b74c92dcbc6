// TEST INFRASTRUCTURE ONLY (oracle/).  The reference's three Frame constructors (src/Frame.cc:61-228), run unmodified.  Linked
// into _ref/libframector.so together with the reference's src/Frame.cc and frameref_wrap.cpp, against the reference's real
// include/Frame.h with oracle/frameshim/pre.hpp force-included (oracle/Makefile).  Used by tests/test_oracle_frame_ctor.py and
// tests/test_gpu_frame_ctor_ref.py (through oracle_lib.ref_frame) to pin whole constructors.
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <new>
#include <vector>

#include "Frame.h"
#include "orb_port.h"

using namespace ORB_SLAM2;

namespace {
std::vector<cv::KeyPoint> keys_of(const orbport_kp* k, int n) {
    static_assert(sizeof(cv::KeyPoint) == sizeof(orbport_kp), "keypoint layout");
    std::vector<cv::KeyPoint> v(n);
    if (n) std::memcpy(v.data(), k, (size_t)n * sizeof(orbport_kp));
    return v;
}
cv::Mat desc_of(const uint8_t* d, int n) {
    cv::Mat m(n > 0 ? n : 1, 32, CV_8U);
    if (n) std::memcpy(m.data, d, (size_t)n * 32);
    return m;
}
}  // namespace

extern "C" {

// One of the three Frame constructors, run unmodified: kind 0 monocular (Frame.cc:174-228), 1 stereo (:61-117), 2 RGB-D
// (:119-171).  Each extractor (left; right for kind 1) replays keys / desc / the pyramid that the verbatim ORBextractor.cc found
// on the image (frameshim/pre.hpp); `tables` holds its mvScaleFactor, mvInvScaleFactor, mvLevelSigma2, mvInvLevelSigma2
// (nlevels each).  The images handed to the constructor are blank w x h matrices: it only reads their size
// (ComputeImageBounds, :436-464).  depth: the h x w CV_32F map Tracking::GrabImageRGBD passes (kind 2).
// The Frame is built by placement-new into zeroed storage whose mb already holds mb_prefill: ComputeStereoMatches reads mb
// (:496-498) before the constructor assigns it (:114), so in the reference that read sees whatever the storage held.
// fresh != 0 sets Frame::mbInitialComputations first, as in a new process; 0 continues the statics of the previous call (a
// Tracking sequence).  A stereo frame with N > 0 whose right image gives no accepted match reaches :627 with vDistIdx empty:
// it reads vDistIdx[0] from storage that :502 reserved but nothing wrote.  That is benign: the loop at :630 does not run, so the
// value is never used.  Outputs (max(nL, nR) entries per array):
//   i_out[9]: mnId, N, mvKeysRight.size(), entries in the grid, mnScaleLevels, mvKeysUn.size(), mvuRight.size(),
//             mvDepth.size(), mbInitialComputations after the call
//   f_out[17]: the statics mnMinX mnMinY mnMaxX mnMaxY, mfGridElementWidthInv, mfGridElementHeightInv, fx fy cx cy invfx invfy;
//              the members mb, mbf, mThDepth, mfScaleFactor, mfLogScaleFactor
//   scales_out: mvScaleFactors, mvInvScaleFactors, mvLevelSigma2, mvInvLevelSigma2 (nlevels each)
//   cell_start / cell_idx: mGrid flattened as frameref_assign_grid does.
// Returns N.
int framector_run(int kind, int fresh, int w, int h, const orbport_kp* kL, const uint8_t* dL, int nL, const orbport_kp* kR,
                  const uint8_t* dR, int nR, const uint8_t* const* pyrL, const uint8_t* const* pyrR, const int* lw, const int* lh,
                  int nlevels, const float* tablesL, const float* tablesR, float scale_factor, const float* K4, const float* dist,
                  int n_dist, float bf, float th_depth, float mb_prefill, const float* depth, int64_t* i_out, float* f_out,
                  float* scales_out, orbport_kp* keys, uint8_t* desc, orbport_kp* keys_right, uint8_t* desc_right,
                  orbport_kp* keys_un, float* u_right, float* depth_out, int32_t* cell_start, int32_t* cell_idx) {
    ORBextractor X[2];
    const orbport_kp* kk[2] = {kL, kR};
    const uint8_t* dd[2] = {dL, dR};
    const int nn[2] = {nL, nR};
    const uint8_t* const* pp[2] = {pyrL, pyrR};
    const float* tt[2] = {tablesL, tablesR};
    for (int s = 0; s < (kind == 1 ? 2 : 1); s++) {
        for (int l = 0; l < nlevels; l++) {
            cv::Mat a(lh[l], lw[l], CV_8U);
            std::memcpy(a.data, pp[s][l], (size_t)lw[l] * lh[l]);
            X[s].mvImagePyramid.push_back(a);
        }
        X[s].mvScaleFactor.assign(tt[s], tt[s] + nlevels);
        X[s].mvInvScaleFactor.assign(tt[s] + nlevels, tt[s] + 2 * nlevels);
        X[s].mvLevelSigma2.assign(tt[s] + 2 * nlevels, tt[s] + 3 * nlevels);
        X[s].mvInvLevelSigma2.assign(tt[s] + 3 * nlevels, tt[s] + 4 * nlevels);
        X[s].scaleFactor = scale_factor;
        X[s].replayKeys = keys_of(kk[s], nn[s]);
        X[s].replayDesc = desc_of(dd[s], nn[s]);
    }
    cv::Mat K(3, 3, CV_32F);
    K.at<float>(0, 0) = K4[0]; K.at<float>(1, 1) = K4[1]; K.at<float>(0, 2) = K4[2]; K.at<float>(1, 2) = K4[3]; K.at<float>(2, 2) = 1.f;
    cv::Mat D(n_dist, 1, CV_32F);
    for (int i = 0; i < n_dist; i++) D.at<float>(i) = dist[i];
    cv::Mat im(h, w, CV_8U), im2(h, w, CV_8U), imDepth(h, w, CV_32F);
    if (kind == 2) std::memcpy(imDepth.data, depth, (size_t)w * h * 4);
    const double timeStamp = 0.0;
    if (fresh) Frame::mbInitialComputations = true;

    void* mem = ::operator new(sizeof(Frame));
    std::memset(mem, 0, sizeof(Frame));
    *reinterpret_cast<float*>(static_cast<char*>(mem) + offsetof(Frame, mb)) = mb_prefill;
    Frame* F;
    if (kind == 1) F = new (mem) Frame(im, im2, timeStamp, &X[0], &X[1], nullptr, K, D, bf, th_depth);
    else if (kind == 2) F = new (mem) Frame(im, imDepth, timeStamp, &X[0], nullptr, K, D, bf, th_depth);
    else F = new (mem) Frame(im, timeStamp, &X[0], nullptr, K, D, bf, th_depth);

    const int N = F->N, Nr = (int)F->mvKeysRight.size();
    if (N > 0) {
        std::memcpy(keys, F->mvKeys.data(), (size_t)N * sizeof(orbport_kp));
        for (int i = 0; i < N; i++) std::memcpy(desc + (size_t)i * 32, F->mDescriptors.ptr<uint8_t>(i), 32);
    }
    if (Nr > 0) {
        std::memcpy(keys_right, F->mvKeysRight.data(), (size_t)Nr * sizeof(orbport_kp));
        for (int i = 0; i < Nr; i++) std::memcpy(desc_right + (size_t)i * 32, F->mDescriptorsRight.ptr<uint8_t>(i), 32);
    }
    if (!F->mvKeysUn.empty()) std::memcpy(keys_un, F->mvKeysUn.data(), F->mvKeysUn.size() * sizeof(orbport_kp));
    for (size_t i = 0; i < F->mvuRight.size(); i++) u_right[i] = F->mvuRight[i];
    for (size_t i = 0; i < F->mvDepth.size(); i++) depth_out[i] = F->mvDepth[i];
    int r = 0;
    for (int x = 0; x < FRAME_GRID_COLS; x++)
        for (int y = 0; y < FRAME_GRID_ROWS; y++) {
            cell_start[x * FRAME_GRID_ROWS + y] = r;
            for (size_t i : F->mGrid[x][y]) cell_idx[r++] = (int32_t)i;
        }
    cell_start[FRAME_GRID_COLS * FRAME_GRID_ROWS] = r;
    const int L = (int)F->mvScaleFactors.size();
    for (int l = 0; l < L && l < nlevels; l++) {
        scales_out[l] = F->mvScaleFactors[l]; scales_out[nlevels + l] = F->mvInvScaleFactors[l];
        scales_out[2 * nlevels + l] = F->mvLevelSigma2[l]; scales_out[3 * nlevels + l] = F->mvInvLevelSigma2[l];
    }
    const int64_t iv[9] = {(int64_t)F->mnId, N, Nr, r, F->mnScaleLevels, (int64_t)F->mvKeysUn.size(), (int64_t)F->mvuRight.size(),
                           (int64_t)F->mvDepth.size(), Frame::mbInitialComputations ? 1 : 0};
    std::memcpy(i_out, iv, sizeof(iv));
    const float fv[17] = {Frame::mnMinX, Frame::mnMinY, Frame::mnMaxX, Frame::mnMaxY, Frame::mfGridElementWidthInv,
                          Frame::mfGridElementHeightInv, Frame::fx, Frame::fy, Frame::cx, Frame::cy, Frame::invfx, Frame::invfy,
                          F->mb, F->mbf, F->mThDepth, F->mfScaleFactor, F->mfLogScaleFactor};
    std::memcpy(f_out, fv, sizeof(fv));
    F->~Frame();
    ::operator delete(mem);
    return N;
}

}  // extern "C"
