// TEST INFRASTRUCTURE ONLY (oracle/).  C entry points around the reference's src/Frame.cc, which oracle/Makefile (target `ref`)
// compiles VERBATIM where it lies, against the reference's real include/Frame.h with oracle/frameshim/pre.hpp force-included
// (plain-data stand-ins for the classes Frame.h merely points to).  Covers Frame::ComputeStereoMatches (:466-640), the feature
// grid AssignFeaturesToGrid / PosInGrid / GetFeaturesInArea (:230-245, :327-392) and Frame::isInFrustum (:269-325).
// Used by tests/test_oracle_frame_ref.py to pin the restatements (orb_port_stereo.cpp, orb_port_match.cpp) to the reference.
#include <cstdint>
#include <cstring>
#include <vector>

#include "Frame.h"
#include "orb_port.h"

namespace ORB_SLAM2 {
// MapPoint::PredictScale(const float&, Frame*) — src/MapPoint.cc:402-417 (restated: MapPoint.cc needs the whole map graph)
int MapPoint::PredictScale(const float& currentDist, Frame* pF) {
    const float ratio = mfMaxDistance / currentDist;
    int nScale = ceil(log(ratio) / pF->mfLogScaleFactor);
    if (nScale < 0) nScale = 0;
    else if (nScale >= pF->mnScaleLevels) nScale = pF->mnScaleLevels - 1;
    return nScale;
}
}  // namespace ORB_SLAM2

using namespace ORB_SLAM2;

namespace {
std::vector<cv::KeyPoint> make_keys(const orbport_kp* k, int n) {
    static_assert(sizeof(cv::KeyPoint) == sizeof(orbport_kp), "keypoint layout");
    std::vector<cv::KeyPoint> v(n);
    if (n) std::memcpy(v.data(), k, (size_t)n * sizeof(orbport_kp));
    return v;
}
cv::Mat make_desc(const uint8_t* d, int n) {
    cv::Mat m(n > 0 ? n : 1, 32, CV_8U);
    if (n) std::memcpy(m.data, d, (size_t)n * 32);
    return m;
}
void set_bounds(float minX, float minY, float maxX, float maxY) {
    Frame::mnMinX = minX; Frame::mnMinY = minY; Frame::mnMaxX = maxX; Frame::mnMaxY = maxY;
    Frame::mfGridElementWidthInv = static_cast<float>(FRAME_GRID_COLS) / static_cast<float>(Frame::mnMaxX - Frame::mnMinX);   // Frame.cc:101-102
    Frame::mfGridElementHeightInv = static_cast<float>(FRAME_GRID_ROWS) / static_cast<float>(Frame::mnMaxY - Frame::mnMinY);
}
}  // namespace

extern "C" {

// Frame::ComputeStereoMatches on given keypoints / descriptors / pyramids (same arguments as orbport_stereo)
int frameref_stereo(const orbport_kp* kL, const uint8_t* dL, int nL, const orbport_kp* kR, const uint8_t* dR, int nR,
                    const uint8_t* const* pyrL, const uint8_t* const* pyrR, const int* lw, const int* lh, int nlevels,
                    const float* scale, const float* inv_scale, float bf, float b, float* uRight, float* depth) {
    ORBextractor L, R;
    for (int l = 0; l < nlevels; l++) {
        cv::Mat a(lh[l], lw[l], CV_8U), c(lh[l], lw[l], CV_8U);
        std::memcpy(a.data, pyrL[l], (size_t)lw[l] * lh[l]);
        std::memcpy(c.data, pyrR[l], (size_t)lw[l] * lh[l]);
        L.mvImagePyramid.push_back(a); R.mvImagePyramid.push_back(c);
    }
    Frame F;
    F.mpORBextractorLeft = &L; F.mpORBextractorRight = &R;
    F.N = nL;
    F.mvKeys = make_keys(kL, nL); F.mvKeysRight = make_keys(kR, nR);
    F.mDescriptors = make_desc(dL, nL); F.mDescriptorsRight = make_desc(dR, nR);
    F.mvScaleFactors.assign(scale, scale + nlevels);
    F.mvInvScaleFactors.assign(inv_scale, inv_scale + nlevels);
    F.mbf = bf;
    F.mb = b;            // the reference reads mb before its constructor assigns it (Frame.cc:496 vs :114); the intended mbf/fx is given
    if (nL == 0 || nR == 0) { for (int i = 0; i < nL; i++) { uRight[i] = -1.f; depth[i] = -1.f; } return 0; }   // :627 is UB on an empty list
    F.ComputeStereoMatches();
    int n = 0;
    for (int i = 0; i < nL; i++) { uRight[i] = F.mvuRight[i]; depth[i] = F.mvDepth[i]; n += F.mvuRight[i] >= 0; }
    return n;
}

// AssignFeaturesToGrid + GetFeaturesInArea (same arguments as orbport_features_in_area)
int frameref_features_in_area(const orbport_kp* k, int n, float minX, float minY, float maxX, float maxY, float x, float y, float r,
                              int minLevel, int maxLevel, int32_t* out, int cap) {
    set_bounds(minX, minY, maxX, maxY);
    Frame F;
    F.N = n;
    F.mvKeysUn = make_keys(k, n);
    F.AssignFeaturesToGrid();
    const std::vector<size_t> v = F.GetFeaturesInArea(x, y, r, minLevel, maxLevel);
    for (int i = 0; i < (int)v.size() && i < cap; i++) out[i] = (int32_t)v[i];
    return (int)v.size();
}

// AssignFeaturesToGrid, with Frame::mGrid flattened the way the device keeps it: cell c = x*FRAME_GRID_ROWS + y holds
// cell_idx[cell_start[c] .. cell_start[c+1]) in insertion order (cell_start: FRAME_GRID_COLS*FRAME_GRID_ROWS + 1 entries,
// cell_idx: n).  Returns the number of features in the grid.
int frameref_assign_grid(const orbport_kp* k, int n, float minX, float minY, float maxX, float maxY, int32_t* cell_start, int32_t* cell_idx) {
    set_bounds(minX, minY, maxX, maxY);
    Frame F;
    F.N = n;
    F.mvKeysUn = make_keys(k, n);
    F.AssignFeaturesToGrid();
    int r = 0;
    for (int x = 0; x < FRAME_GRID_COLS; x++)
        for (int y = 0; y < FRAME_GRID_ROWS; y++) {
            cell_start[x * FRAME_GRID_ROWS + y] = r;
            for (size_t i : F.mGrid[x][y]) cell_idx[r++] = (int32_t)i;
        }
    cell_start[FRAME_GRID_COLS * FRAME_GRID_ROWS] = r;
    return r;
}

// Frame::isInFrustum for n MapPoints (same outputs as orbport_is_in_frustum); the pose goes through SetPose / UpdatePoseMatrices
int frameref_is_in_frustum(const float* world_pos, const float* normal, const float* max_distance, const float* min_distance,
                           const uint8_t* valid, int n, const float* Tcw, float fx, float fy, float cx, float cy, float mbf, float minX,
                           float minY, float maxX, float maxY, float viewingCosLimit, float log_scale_factor, int n_levels,
                           uint8_t* in_view, float* proj_x, float* proj_y, float* proj_xr, int32_t* level, float* view_cos, float* Ow_out) {
    set_bounds(minX, minY, maxX, maxY);
    Frame::fx = fx; Frame::fy = fy; Frame::cx = cx; Frame::cy = cy;
    Frame F;
    F.mbf = mbf; F.mfLogScaleFactor = log_scale_factor; F.mnScaleLevels = n_levels;
    cv::Mat T(4, 4, CV_32F);
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 4; c++) T.at<float>(r, c) = Tcw[4 * r + c];
    T.at<float>(3, 3) = 1.f;
    F.SetPose(T);
    const cv::Mat O = F.GetCameraCenter();
    for (int i = 0; i < 3; i++) Ow_out[i] = O.at<float>(i);
    int count = 0;
    for (int i = 0; i < n; i++) {
        in_view[i] = 0;
        if (valid && !valid[i]) continue;
        MapPoint p;
        p.mWorldPos = cv::Mat(3, 1, CV_32F); p.mNormalVector = cv::Mat(3, 1, CV_32F);
        for (int k = 0; k < 3; k++) { p.mWorldPos.at<float>(k) = world_pos[3 * (size_t)i + k]; p.mNormalVector.at<float>(k) = normal[3 * (size_t)i + k]; }
        p.mfMaxDistance = max_distance[i]; p.mfMinDistance = min_distance[i];
        if (F.isInFrustum(&p, viewingCosLimit)) {
            in_view[i] = 1; proj_x[i] = p.mTrackProjX; proj_y[i] = p.mTrackProjY; proj_xr[i] = p.mTrackProjXR;
            level[i] = p.mnTrackScaleLevel; view_cos[i] = p.mTrackViewCos;
            count++;
        }
    }
    return count;
}

// The RGB-D constructor's data-parallel steps (src/Frame.cc:143-145, :160-176): UndistortKeyPoints (:404-434),
// ComputeStereoFromRGBD (:643-664) and ComputeImageBounds (:436-464), run unmodified.  K4 = fx fy cx cy; dist: n_dist
// coefficients k1 k2 p1 p2 [k3] exactly as Tracking builds mDistCoef (src/Tracking.cc:69-79); depth: h x w floats.
int frameref_rgbd(const orbport_kp* keys, int n, const float* K4, const float* dist, int n_dist, float bf, const float* depth, int w, int h,
                  orbport_kp* keys_un, float* u_right, float* depth_out, float* bounds4) {
    Frame F;
    F.mK = cv::Mat(3, 3, CV_32F);
    F.mK.at<float>(0, 0) = K4[0]; F.mK.at<float>(1, 1) = K4[1]; F.mK.at<float>(0, 2) = K4[2]; F.mK.at<float>(1, 2) = K4[3]; F.mK.at<float>(2, 2) = 1.f;
    F.mDistCoef = cv::Mat(n_dist, 1, CV_32F);
    for (int i = 0; i < n_dist; i++) F.mDistCoef.at<float>(i) = dist[i];
    F.mbf = bf;
    F.N = n;
    F.mvKeys = make_keys(keys, n);
    cv::Mat im(h, w, CV_8U), imDepth(h, w, CV_32F);
    std::memcpy(imDepth.data, depth, (size_t)w * h * 4);
    F.ComputeImageBounds(im);
    bounds4[0] = Frame::mnMinX; bounds4[1] = Frame::mnMinY; bounds4[2] = Frame::mnMaxX; bounds4[3] = Frame::mnMaxY;
    if (n == 0) return 0;
    F.UndistortKeyPoints();
    F.ComputeStereoFromRGBD(imDepth);
    int cnt = 0;
    std::memcpy(keys_un, F.mvKeysUn.data(), (size_t)n * sizeof(orbport_kp));
    for (int i = 0; i < n; i++) { u_right[i] = F.mvuRight[i]; depth_out[i] = F.mvDepth[i]; cnt += F.mvDepth[i] > 0; }
    return cnt;
}

}  // extern "C"
