/* borb.h — C ABI of the CUDA ORB front-end for the H100 (libborb.so).
 *
 * Drop-in boundary for the ONE hot path of raulmur/ORB_SLAM2 (SURVEY.md §8):
 *   ORBextractor::operator()              include/ORBextractor.h:59-61, src/ORBextractor.cc:1043
 *   Frame::ComputeStereoMatches           include/Frame.h:89,            src/Frame.cc:466
 *   ORBmatcher::SearchByProjection (F,MPs) include/ORBmatcher.h:46,       src/ORBmatcher.cc:45
 *   ORBmatcher::SearchByBoW               include/ORBmatcher.h:61-62,    src/ORBmatcher.cc:159,522
 *   ORBmatcher::SearchForTriangulation    include/ORBmatcher.h:69-70,    src/ORBmatcher.cc:657
 *   ORBmatcher::DescriptorDistance        include/ORBmatcher.h:44,       src/ORBmatcher.cc:1647
 *   TemplatedVocabulary::transform (feeder) Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1127
 *   Frame::AssignFeaturesToGrid / GetFeaturesInArea  src/Frame.cc:230-245, 327-380
 * The reference has no FFI layer; these entry points are what the C++ adapters in
 * include/borb_adapters.hpp (same class signatures as the reference) forward to.
 *
 * Conventions: plain pointers and sizes only; every function returns a borb_status; no exception
 * or process exit crosses the boundary; no CPU fallback exists — without a CUDA device every
 * compute entry point returns BORB_ERR_NO_DEVICE / BORB_ERR_CUDA.  A handle owns one CUDA stream
 * and its scratch; calls on DIFFERENT handles are thread-safe and run concurrently, calls on the
 * same borb_extractor or borb_matcher must be serialised by the caller (the reference creates one
 * extractor per camera and one matcher per call site/thread, src/Tracking.cc:119-125).
 * The exceptions are the objects ORB_SLAM2's Tracking, LocalMapping and LoopClosing threads share:
 *  - a borb_voc may be used by any number of threads at once (DBoW2's transform is const): each
 *    call of borb_bow_transform / borb_compute_bow runs on the vocabulary's own stream and buffers
 *    and holds its lock until the results are copied out, and borb_frames_compute_bow runs on the
 *    matcher's and reads only the vocabulary's immutable tree;
 *  - a borb_kfdb may be added to, erased from, masked and searched by any number of threads at
 *    once, as KeyFrameDatabase's mMutex allows: every search sees each add, erase and MapPoint-mask
 *    batch whole;
 *  - a borb_frame may be read by several matchers at once; borb_frames_compute_bow rewrites its
 *    BoW, so it must not overlap any other use of the frame.
 * borb_voc_destroy and borb_kfdb_destroy must not race with any use of the handle.
 */
#ifndef BORB_H
#define BORB_H

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define BORB_API __attribute__((visibility("default")))
#else
#define BORB_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define BORB_VERSION 2
#define BORB_MAX_LEVELS 16
#define BORB_MAX_DIM 4095 /* image width/height limit (candidates pack x,y in 12 bits) */

typedef enum borb_status {
    BORB_OK = 0,
    BORB_ERR_INVALID_ARG = 1,
    BORB_ERR_NO_DEVICE = 2,   /* no CUDA device / driver: there is no CPU path */
    BORB_ERR_CUDA = 3,        /* a CUDA call failed; see borb_last_error() */
    BORB_ERR_UNSUPPORTED = 4, /* shape / quota outside the supported envelope */
    BORB_ERR_CAPACITY = 5,    /* caller buffer too small; *n_out still holds the required count */
    BORB_ERR_STATE = 6        /* call order violated (e.g. stereo match before extract) */
} borb_status;

/* Layout-identical to cv::KeyPoint (28 bytes) so adapters can memcpy (src/ORBextractor.cc:1103). */
typedef struct borb_keypoint {
    float x, y;      /* pt, level-0 pixel units (level px * mvScaleFactor[octave], :1095-1101) */
    float size;      /* PATCH_SIZE * mvScaleFactor[octave], int-truncated (:837,:846) */
    float angle;     /* degrees [0,360), IC_Angle (:77-104) */
    float response;  /* FAST score */
    int32_t octave;  /* pyramid level */
    int32_t class_id;/* -1 */
} borb_keypoint;

/* ORBextractor ctor arguments (include/ORBextractor.h:53-54; YAML keys ORBextractor.*). */
typedef struct borb_extractor_cfg {
    int32_t n_features;   /* ORBextractor.nFeatures  */
    float scale_factor;   /* ORBextractor.scaleFactor */
    int32_t n_levels;     /* ORBextractor.nLevels (<= BORB_MAX_LEVELS) */
    int32_t ini_th_fast;  /* ORBextractor.iniThFAST, 0..255 */
    int32_t min_th_fast;  /* ORBextractor.minThFAST, 0..255 */
} borb_extractor_cfg;

typedef struct borb_extractor borb_extractor;

BORB_API const char* borb_last_error(void);     /* thread-local description of the last failure */
BORB_API const char* borb_status_str(borb_status s);
BORB_API int borb_version(void);
BORB_API borb_status borb_device_count(int* n);

/* Pinned host memory for asynchronous / overlapped transfers. */
BORB_API borb_status borb_host_alloc(void** p, size_t bytes);
BORB_API borb_status borb_host_free(void* p);

/* ---------------------------------------------------------------- extractor ------------------ */
/* Replaces ORBextractor::ORBextractor (src/ORBextractor.cc:410-470).  Returns BORB_ERR_INVALID_ARG, and leaves *out NULL,
 * for n_levels outside [1, BORB_MAX_LEVELS], n_features < 1, scale_factor not above 1 (or NaN), and FAST thresholds outside
 * [0, 255], where cv::FAST's result depends on the OpenCV build; borb_last_error() names the field. */
BORB_API borb_status borb_extractor_create(const borb_extractor_cfg* cfg, int device, borb_extractor** out);
BORB_API borb_status borb_extractor_destroy(borb_extractor* e);
/* Getters of include/ORBextractor.h:63-83; arrays hold n_levels entries. */
BORB_API borb_status borb_extractor_tables(const borb_extractor* e, float* scale, float* inv_scale, float* sigma2,
                                  float* inv_sigma2, int32_t* features_per_level);
/* Upper bound of keypoints one image can return for this cfg and image size (quota may be
 * exceeded by <=3 per level and is never trimmed, src/ORBextractor.cc:730; SURVEY §8 a4). */
BORB_API borb_status borb_extractor_capacity(const borb_extractor* e, int width, int height, int* cap);
/* Pre-allocates device scratch for batches of up to max_images images of width x height. */
BORB_API borb_status borb_extractor_reserve(borb_extractor* e, int width, int height, int max_images);

/* ORBextractor::operator() (src/ORBextractor.cc:1043) for ONE host image.  gray: 8-bit, `stride`
 * bytes per row.  kps/desc: caller buffers of `cap` entries (desc: cap x 32 bytes, row-major like the
 * reference's N x 32 CV_8U Mat).  Empty image => BORB_OK with *n_out = 0 (:1046-1047). */
BORB_API borb_status borb_extract(borb_extractor* e, const uint8_t* gray, int width, int height, int stride,
                         borb_keypoint* kps, uint8_t* desc, int cap, int* n_out);

/* The same for n images of identical size in one launch sequence (the throughput path: independent
 * frames / camera streams batched per launch).  gray[i] are host pointers; image i writes
 * kps + i*cap, desc + i*cap*32 and n_out[i]. */
BORB_API borb_status borb_extract_batch(borb_extractor* e, const uint8_t* const* gray, int n_images, int width, int height,
                               int stride, borb_keypoint* kps, uint8_t* desc, int cap, int* n_out);

/* Asynchronous halves of the batch call: `_enqueue` returns once the work is queued on the handle's
 * stream (host buffers must stay valid and should be pinned); `borb_sync` waits for it.  Results of
 * the last batch stay resident in HBM until the next enqueue on this handle. */
BORB_API borb_status borb_extract_batch_enqueue(borb_extractor* e, const uint8_t* const* gray, int n_images, int width,
                                       int height, int stride, borb_keypoint* kps, uint8_t* desc, int cap, int* n_out);
BORB_API borb_status borb_sync(borb_extractor* e);

/* Device-resident input variant: d_gray points to n_images images already in HBM on the handle's
 * device (image i at d_gray + i*image_stride, rows `pitch` bytes apart).  No host copies unless the
 * output pointers are non-NULL.  Used for the HBM-resident throughput measurement.  With rectification maps installed
 * (borb_extractor_set_rectify_maps) the images are RAW width x height frames, rectified while they are read; the input
 * format of borb_extractor_set_input_format does not apply: device images are always CV_8UC1. */
BORB_API borb_status borb_extract_batch_device(borb_extractor* e, const uint8_t* d_gray, int n_images, int width, int height,
                                      size_t pitch, size_t image_stride, borb_keypoint* kps, uint8_t* desc, int cap,
                                      int* n_out);

/* Pixel format of the HOST images given to the extract / stereo entry points of this handle (default 1 = CV_8UC1).
 * With 3 or 4 channels the conversion Tracking::GrabImageStereo/RGBD/Monocular performs before calling the extractor —
 * cv::cvtColor(RGB2GRAY | BGR2GRAY | RGBA2GRAY | BGRA2GRAY), src/Tracking.cc:172-197,211-223,243-255 — is fused into the
 * upload: only the raw camera frame crosses PCIe.  rgb_order = Tracking::mbRGB (1: R first, 0: B first).
 * `stride` arguments are then bytes per row of the interleaved image. */
BORB_API borb_status borb_extractor_set_input_format(borb_extractor* e, int channels, int rgb_order);

/* Stereo rectification fused into the upload: cv::remap(imLeft, imLeftRect, M1l, M2l, cv::INTER_LINEAR) /
 * (imRight, ..., M1r, M2r, ...) of Examples/Stereo/stereo_euroc.cc:136-137 with the CV_32FC1 maps the caller built once
 * with cv::initUndistortRectifyMap (:96-98).  which = 0: mono / left, 1: right (install 0 first; in the stereo entry
 * points even images use set 0 and odd images set 1).  map_x / map_y: dst_h x dst_w floats; NULL removes the set(s).
 * Afterwards the extract / stereo entry points take RAW src_w x src_h CV_8UC1 frames and work on dst_w x dst_h. */
BORB_API borb_status borb_extractor_set_rectify_maps(borb_extractor* e, int which, const float* map_x, const float* map_y, int src_w,
                                                     int src_h, int dst_w, int dst_h);

/* mvImagePyramid[level] of image `image` of the last batch (include/ORBextractor.h:85), copied to
 * a caller buffer of at least h*w bytes (tight rows).  Pass dst=NULL to query w/h only. */
BORB_API borb_status borb_extractor_pyramid(borb_extractor* e, int image, int level, uint8_t* dst, int* w, int* h);

/* ---------------------------------------------------------------- stereo --------------------- */
/* Frame::ComputeStereoMatches (src/Frame.cc:466-640) for the images of the LAST batch of `e`:
 * pair p uses image left_idx[p] as left and right_idx[p] as right (NULL index arrays mean
 * left=2p, right=2p+1).  bf = Camera.bf, b = mb = bf/fx (src/Frame.cc:114; the reference reads mb
 * before initialising it, :496 — the intended value is used here).  Outputs per pair p at
 * u_right + p*cap and depth + p*cap, entries [0, n_left): -1.0f means "no match" (:468-469). */
BORB_API borb_status borb_stereo_match(borb_extractor* e, int n_pairs, const int* left_idx, const int* right_idx, float bf,
                              float b, float* u_right, float* depth, int cap);

/* Same, when the left and right images were extracted by two different handles on the same device
 * (the reference's mpORBextractorLeft / mpORBextractorRight, src/Frame.cc:78-81): image 0 of each.
 * The two handles must have the same image size, number of levels and scale factor (BORB_ERR_INVALID_ARG
 * otherwise); nfeatures may differ, either way round. */
BORB_API borb_status borb_stereo_match2(borb_extractor* left, borb_extractor* right, float bf, float b, float* u_right,
                               float* depth, int cap);

/* Frame::Frame stereo constructor hot path in one call (src/Frame.cc:61-117): extract L+R for
 * n_pairs frames and associate them; one H2D (images) and one D2H (results) per call.
 * Any output pointer may be NULL to skip its copy. */
BORB_API borb_status borb_stereo_frames(borb_extractor* e, const uint8_t* const* left, const uint8_t* const* right, int n_pairs,
                               int width, int height, int stride, float bf, float b, borb_keypoint* kps_left,
                               uint8_t* desc_left, int* n_left, borb_keypoint* kps_right, uint8_t* desc_right,
                               int* n_right, float* u_right, float* depth, int cap);
BORB_API borb_status borb_stereo_frames_enqueue(borb_extractor* e, const uint8_t* const* left, const uint8_t* const* right,
                                       int n_pairs, int width, int height, int stride, float bf, float b,
                                       borb_keypoint* kps_left, uint8_t* desc_left, int* n_left,
                                       borb_keypoint* kps_right, uint8_t* desc_right, int* n_right, float* u_right,
                                       float* depth, int cap);
/* HBM-resident variants (inputs as in borb_extract_batch_device: image 2p = left, 2p+1 = right). */
BORB_API borb_status borb_stereo_frames_device_enqueue(borb_extractor* e, const uint8_t* d_gray, int n_pairs, int width,
                                              int height, size_t pitch, size_t image_stride, float bf, float b,
                                              int* n_left, int* n_right, float* u_right, float* depth, int cap);
BORB_API borb_status borb_stereo_frames_device(borb_extractor* e, const uint8_t* d_gray, int n_pairs, int width, int height,
                                      size_t pitch, size_t image_stride, float bf, float b, int* n_left, int* n_right,
                                      float* u_right, float* depth, int cap);
/* Copies what the last stereo call on `e` left resident in HBM — keypoints, descriptors and counts of both images and
 * mvuRight / mvDepth of its first n_pairs pairs — into host buffers laid out as in borb_stereo_frames (any pointer may be
 * NULL), e.g. to inspect the results of the device-resident variants.  Waits for the handle's stream.  BORB_ERR_STATE unless
 * the last call on `e` was a stereo call over at least n_pairs pairs in the default layout (left 2p, right 2p+1: the
 * borb_stereo_frames* calls, or borb_stereo_match without index arrays); BORB_ERR_CAPACITY, after the copies, when an image
 * has more than `cap` keypoints. */
BORB_API borb_status borb_stereo_frames_results(borb_extractor* e, int n_pairs, borb_keypoint* kps_left, uint8_t* desc_left,
                                                int* n_left, borb_keypoint* kps_right, uint8_t* desc_right, int* n_right,
                                                float* u_right, float* depth, int cap);

/* ---------------------------------------------------------------- matchers ------------------- */
/* ORB_SLAM2::ORBmatcher is a stateless stack object created at every call site on three threads
 * (include/ORBmatcher.h:37-102; src/Tracking.cc:599,764,869,1184,1357,1396, src/LocalMapping.cc:215,483,
 * src/LoopClosing.cc:239,589).  A borb_matcher handle owns a CUDA stream and scratch: keep one per thread.
 * The pointer graphs the reference walks (Frame, KeyFrame, MapPoint) are snapshotted by the adapter into the
 * plain views below on the calling thread; results come back as indices. */
typedef struct borb_matcher borb_matcher;
/* Size envelope of every matcher / database call (the reference has no limits; these return BORB_ERR_INVALID_ARG instead of
 * failing inside a launch): at most BORB_MATCH_MAX_FEATURES features per frame or keyframe, and at most that many VALID query
 * points per call (MapPoints of SearchByProjection, last-frame features, world points).  The feature grid sort, the claim
 * bitsets and the resolve kernel's per-query lists live in shared memory, which is what bounds them.  borb_search_local_points
 * compacts the valid points before the check, so the limit applies to the points that reach Frame::isInFrustum, not to the
 * length of Tracking::mvpLocalMapPoints (a KITTI-scale local map of 10^4+ points with a few hundred candidates is fine). */
#define BORB_MATCH_MAX_FEATURES 8192
BORB_API borb_status borb_matcher_create(int device, borb_matcher** out);
BORB_API borb_status borb_matcher_destroy(borb_matcher* m);

/* Frame snapshot for SearchByProjection (include/Frame.h): undistorted keypoints, descriptors, stereo
 * coordinate, image bounds of the 64x48 feature grid (mnMinX.. / src/Frame.cc:97-102), scale factors. */
typedef struct borb_frame borb_frame;   /* device-resident Frame, see borb_frame_create below */
typedef struct borb_frame_view {
    int32_t n;                     /* N */
    const borb_keypoint* keys_un;  /* mvKeysUn */
    const uint8_t* desc;           /* mDescriptors, N x 32 */
    const float* u_right;          /* mvuRight (NULL: monocular, no stereo check) */
    const uint8_t* occupied;       /* 1 if mvpMapPoints[i] && Observations()>0 (src/ORBmatcher.cc:87-89); NULL: none */
    float min_x, min_y, max_x, max_y;
    int32_t n_levels;
    const float* scale_factors;    /* mvScaleFactors */
    const borb_frame* resident;    /* NULL, or a device-resident copy of this frame: then n, keys_un, desc, u_right, the bounds and
                                      scale_factors above are ignored (taken from the resident frame, whose feature grid is already
                                      built) and only `occupied` is read from the host */
} borb_frame_view;

/* Device-resident Frame: uploads the view once (keypoints, descriptors, mvuRight, scale factors) and builds the 64x48 feature
 * grid of Frame::AssignFeaturesToGrid (src/Frame.cc:230-245) ONCE, so that the matcher calls of one Track() — SearchLocalPoints
 * (src/Tracking.cc:1148-1194), SearchByProjection(CurrentFrame, LastFrame) (:867-898), relocalisation — stop re-uploading
 * ~100 KB and re-sorting the grid per call: put the handle into borb_frame_view::resident.  The frame may be used by any
 * matcher on the same device (creation records an event the users wait on).  Destroyed frames are recycled. */
BORB_API borb_status borb_frame_create(borb_matcher* m, const borb_frame_view* view, borb_frame** out);
BORB_API borb_status borb_frame_destroy(borb_frame* f);

/* Camera.* of the settings file as Tracking builds mK / mDistCoef / mbf (src/Tracking.cc:54-90). */
typedef struct borb_camera {
    float fx, fy, cx, cy;
    float k1, k2, p1, p2, k3;      /* k1 == 0 => mvKeysUn = mvKeys (src/Frame.cc:406-410) */
    float bf;                      /* Camera.bf */
} borb_camera;

/* The tail of the Frame constructors (src/Frame.cc:61-117 stereo, :119-178 RGB-D, :180-233 monocular) ON THE DEVICE for images
 * of the LAST batch of extractor `e` — keypoints and descriptors go from the extractor's workspace into resident frames without
 * crossing PCIe:  Frame::UndistortKeyPoints (:404-434, cv::undistortPoints restated: double arithmetic, 5 iterations),
 * Frame::ComputeStereoFromRGBD (:643-664) and Frame::AssignFeaturesToGrid (:230-245).
 *   images[i], n_keys[i]   image index inside the batch and its keypoint count (n_out of the extract call)
 *   mode 0 monocular; 1 stereo: mvuRight / mvDepth are the association borb_stereo_frames computed for pair images[i]/2
 *        (images[i] must be the LEFT image, an even index); 2 RGB-D: depth[i] = host depth map of that frame, registered to
 *        the image (same width x height), depth_type 0 = CV_32F metres, 1 = CV_16U raw with depth_factor = mDepthMapFactor
 *        (+4: depth[i] are DEVICE pointers to tightly packed maps, no copy)
 *        (the convertTo of Tracking::GrabImageRGBD, src/Tracking.cc:227-228, is fused into the lookup)
 *   keys_un / u_right / depth_out   optional host copies (mvKeysUn, mvuRight, mvDepth), n_frames x cap entries
 *   bounds4   mnMinX, mnMinY, mnMaxX, mnMaxY (Frame::ComputeImageBounds, :436-464)
 *   frames    n_frames resident frames; use them through borb_frame_view::resident, release with borb_frame_destroy. */
BORB_API borb_status borb_frames_from_extractor(borb_matcher* m, borb_extractor* e, const int32_t* images, int n_frames,
                                                const int32_t* n_keys, const borb_camera* cam, int mode, const void* const* depth,
                                                int depth_type, float depth_factor, int depth_stride_bytes, borb_keypoint* keys_un,
                                                float* u_right, float* depth_out, int cap, float* bounds4, borb_frame** frames);

/* The host members of one Frame (include/Frame.h:120-176) as its constructor fills them, written by borb_frame_from_extractors.
 * Every array may be NULL (not copied); the per-feature arrays hold `cap` entries.  `n`, `n_right` and `bounds` are outputs. */
typedef struct borb_frame_host {
    int32_t cap;
    borb_keypoint* keys;           /* mvKeys */
    uint8_t* desc;                 /* mDescriptors, N x 32 */
    borb_keypoint* keys_right;     /* mvKeysRight (stereo) */
    uint8_t* desc_right;           /* mDescriptorsRight (stereo), n_right x 32 */
    borb_keypoint* keys_un;        /* mvKeysUn */
    float* u_right;                /* mvuRight (stereo and RGB-D) */
    float* depth;                  /* mvDepth (stereo and RGB-D) */
    int32_t* cell_start;           /* mGrid flattened as in borb_debug_frame_read: 64*48 + 1 entries, cell c = x*48 + y */
    int32_t* cell_idx;             /* cell_start[64*48] entries (at most N) */
    int32_t n;                     /* N */
    int32_t n_right;               /* mvKeysRight.size() (stereo; 0 otherwise) */
    float bounds[4];               /* mnMinX, mnMinY, mnMaxX, mnMaxY (Frame::ComputeImageBounds, src/Frame.cc:436-464) */
} borb_frame_host;

/* One Frame constructor (src/Frame.cc:61-117 stereo, :119-178 RGB-D, :180-233 monocular) after its extractions were enqueued on
 * the frame's extractor handles, image 0 of each handle's last batch (borb_extract_batch_enqueue of one image per handle, no
 * synchronisation needed; two handles' streams overlap):
 *   mode 0 monocular (right = NULL); 1 stereo: `left` / `right` are mpORBextractorLeft / mpORBextractorRight, nfeatures may
 *   differ, and the call runs Frame::ComputeStereoMatches (:466-640) with bf = cam->bf and b = mb = mbf/fx > 0 on the left handle,
 *   as borb_stereo_match2 does; 2 RGB-D (right = NULL): depth = one depth map as in borb_frames_from_extractor.
 * Then UndistortKeyPoints, ComputeStereoFromRGBD and AssignFeaturesToGrid run on the device into the resident frame *out.  The
 * keypoint counts stay on the device until the end: the work is sized by the handles' capacities, and the kernels write every
 * host member `host` asks for, only the N (or N_right) elements the counts give, straight into pinned memory.  So the call waits
 * for the device once, for its results.  (The first stereo call on a left handle also waits once to install its pair table.)
 * Refused before any launch: BORB_ERR_STATE when a handle has no extracted batch; BORB_ERR_INVALID_ARG for bad arguments, a
 * handle pair that borb_stereo_match2 refuses, or a handle whose capacity (borb_extractor_capacity) exceeds
 * BORB_MATCH_MAX_FEATURES; BORB_ERR_CAPACITY when host->cap is below a handle's capacity. */
BORB_API borb_status borb_frame_from_extractors(borb_matcher* m, borb_extractor* left, borb_extractor* right, const borb_camera* cam,
                                                int mode, float b, const void* depth, int depth_type, float depth_factor,
                                                int depth_stride_bytes, borb_frame_host* host, borb_frame** out);
BORB_API borb_status borb_frame_info(const borb_frame* f, int32_t* n, int32_t* n_levels, int32_t* has_u_right);
/* Read-only introspection of a resident frame (tests, debugging): waits for the frame to be complete and copies mvKeysUn (n),
 * mDescriptors (n x 32), mvuRight / mvDepth (n; BORB_ERR_INVALID_ARG on a monocular frame, and for mvDepth on a frame made by
 * borb_frame_create, whose view carries no depth) and the feature grid of
 * Frame::AssignFeaturesToGrid flattened: cell_start[64*48 + 1], cell c = x*48 + y holding cell_idx[cell_start[c] ..
 * cell_start[c+1]) in insertion order; cell_idx needs room for n entries (cell_start[64*48] are written: features whose
 * PosInGrid fails are in no cell).  Any pointer may be NULL. */
BORB_API borb_status borb_debug_frame_read(const borb_frame* f, borb_keypoint* keys, uint8_t* desc, float* u_right, float* depth,
                                           int32_t* cell_start, int32_t* cell_idx);

/* Local map points that passed Frame::isInFrustum (src/Frame.cc:269-325), in vpMapPoints order. */
typedef struct borb_mappoint_view {
    int32_t n;
    const float* proj_x;           /* mTrackProjX */
    const float* proj_y;           /* mTrackProjY */
    const float* proj_xr;          /* mTrackProjXR */
    const int32_t* level;          /* mnTrackScaleLevel */
    const float* view_cos;         /* mTrackViewCos */
    const uint8_t* desc;           /* GetDescriptor(), n x 32 */
    const uint8_t* valid;          /* mbTrackInView && !isBad() (NULL: all valid) */
    const uint8_t* has_obs;        /* Observations()>0 (NULL: all) */
} borb_mappoint_view;

/* ORBmatcher::SearchByProjection(Frame&, const vector<MapPoint*>&, th) — src/ORBmatcher.cc:45-129.
 * match_feat[i] = index of the frame feature that received map point i (F.mvpMapPoints[idx]=pMP), or -1. */
BORB_API borb_status borb_search_by_projection(borb_matcher* m, const borb_frame_view* frame, const borb_mappoint_view* mps,
                                               float th, float nnratio, int32_t* match_feat, int32_t* n_matches);
/* The same search for n_jobs INDEPENDENT (frame, MapPoint list) pairs — e.g. the current frames of n camera streams — in one
 * launch pair and one synchronisation: frames[j] (must be device-resident: borb_frame_view::resident) is searched with points[j],
 * results go to match_feat[j][0 .. points[j].n) and n_matches[j], each identical to what the single call returns.  A single call
 * is ~6 us of kernels behind ~30 us of launch and synchronisation latency; the batch amortises the latter over the streams, the
 * way borb_extract_batch does for the images (no reference counterpart: the reference tracks one camera on one thread). */
BORB_API borb_status borb_search_by_projection_batch(borb_matcher* m, const borb_frame_view* frames, const borb_mappoint_view* points,
                                                     int n_jobs, float th, float nnratio, int32_t* const* match_feat, int32_t* n_matches);

/* LastFrame snapshot for the motion-model search: per last-frame feature i the keypoint (octave, angle of mvKeysUn), the
 * world position and representative descriptor of its MapPoint, valid[i] = mvpMapPoints[i] && !mvbOutlier[i],
 * has_obs[i] = mvpMapPoints[i]->Observations()>0. */
typedef struct borb_lastframe_view {
    int32_t n;
    const borb_keypoint* keys_un;  /* LastFrame.mvKeysUn (octave == mvKeys[i].octave) */
    const float* world_pos;        /* n x 3, pMP->GetWorldPos() */
    const uint8_t* desc;           /* n x 32, pMP->GetDescriptor() */
    const uint8_t* valid;          /* NULL: all valid */
    const uint8_t* has_obs;        /* NULL: all */
} borb_lastframe_view;

/* ORBmatcher::SearchByProjection(Frame &CurrentFrame, const Frame &LastFrame, th, bMono) — src/ORBmatcher.cc:1328-1470
 * (Tracking::TrackWithMotionModel, src/Tracking.cc:885,891).  Tcw = CurrentFrame.mTcw rows 0..2 (3x4 row-major);
 * forward/backward = the bForward/bBackward flags of :1348-1349 (a few float ops on the two poses, computed by the caller).
 * state_cur[i2] (cur->n entries): >=0 = index of the LastFrame feature whose MapPoint now sits in
 * CurrentFrame.mvpMapPoints[i2]; -1 = untouched; -2 = set to NULL by the rotation-consistency cull (:1456-1466). */
BORB_API borb_status borb_search_by_projection_last(borb_matcher* m, const borb_frame_view* cur, const borb_lastframe_view* last,
                                                    const float* Tcw, float fx, float fy, float cx, float cy, float bf, float th,
                                                    int forward, int backward, int check_orientation, int32_t* state_cur,
                                                    int32_t* n_matches);

/* A list of MapPoints with their world-frame data, for the two pose-projection searches below. */
typedef struct borb_worldpoints_view {
    int32_t n;
    const float* world_pos;        /* n x 3, pMP->GetWorldPos() */
    const uint8_t* desc;           /* n x 32, pMP->GetDescriptor() */
    const float* max_distance;     /* n, MapPoint::mfMaxDistance (GetMaxDistanceInvariance() = 1.2f * this, src/MapPoint.cc:379-383) */
    const float* min_distance;     /* n, MapPoint::mfMinDistance (GetMinDistanceInvariance() = 0.8f * this, :373-377) */
    const float* normal;           /* n x 3, pMP->GetNormal(); only read by borb_search_by_projection_sim3 */
    const float* angle;            /* n, pKF->mvKeysUn[i].angle of the keyframe feature that observes the point; only read
                                      by borb_search_by_projection_kf with check_orientation */
    const uint8_t* valid;          /* NULL: all valid */
} borb_worldpoints_view;

/* ORBmatcher::SearchByProjection(Frame &CurrentFrame, KeyFrame *pKF, const set<MapPoint*> &sAlreadyFound, th, ORBdist)
 * — src/ORBmatcher.cc:1472-1599 (Tracking::Relocalization, src/Tracking.cc:1396,1410).
 * pts[i] = pKF->GetMapPointMatches()[i] with valid[i] = pMP && !pMP->isBad() && !sAlreadyFound.count(pMP);
 * cur->occupied[i2] = CurrentFrame.mvpMapPoints[i2] != NULL.  Tcw = CurrentFrame.mTcw rows 0..2, Ow = -Rcw.t()*tcw
 * (:1476-1478, the caller's cv::Mat lines); log_scale_factor = CurrentFrame.mfLogScaleFactor (PredictScale,
 * src/MapPoint.cc:402-417).  state_cur as in borb_search_by_projection_last (index into pts, -1, -2). */
BORB_API borb_status borb_search_by_projection_kf(borb_matcher* m, const borb_frame_view* cur, const borb_worldpoints_view* pts,
                                                  const float* Tcw, const float* Ow, float fx, float fy, float cx, float cy,
                                                  float log_scale_factor, float th, int orb_dist, int check_orientation,
                                                  int32_t* state_cur, int32_t* n_matches);

/* ORBmatcher::SearchByProjection(KeyFrame* pKF, cv::Mat Scw, const vector<MapPoint*> &vpPoints, vector<MapPoint*> &vpMatched, int th)
 * — src/ORBmatcher.cc:290-403 (LoopClosing::ComputeSim3, src/LoopClosing.cc:391).
 * kf: the keyframe's features; kf->occupied[idx] = vpMatched[idx] != NULL on entry.  Tcw = [Rcw | tcw] after the
 * Sim3 scale has been divided out and Ow = -Rcw.t()*tcw (:298-303, the caller's cv::Mat lines).
 * pts->valid[i] = !vpPoints[i]->isBad() && !spAlreadyFound.count(vpPoints[i]).
 * state_kf[idx] = index into pts of the point now in vpMatched[idx], -1 = vpMatched[idx] untouched. */
BORB_API borb_status borb_search_by_projection_sim3(borb_matcher* m, const borb_frame_view* kf, const borb_worldpoints_view* pts,
                                                    const float* Tcw, const float* Ow, float fx, float fy, float cx, float cy,
                                                    float log_scale_factor, int th, int32_t* state_kf, int32_t* n_matches);

/* The search part of ORBmatcher::Fuse(KeyFrame *pKF, const vector<MapPoint *> &vpMapPoints, const float th)
 * — src/ORBmatcher.cc:825-970 (LocalMapping::SearchInNeighbors, src/LocalMapping.cc:483-511) — with scw_variant = 0, and of
 * ORBmatcher::Fuse(KeyFrame *pKF, cv::Mat Scw, vpPoints, th, vpReplacePoint) — :972-1100 (LoopClosing::SearchAndFuse,
 * src/LoopClosing.cc:589) — with scw_variant = 1 (Tcw = [Rcw|tcw] with the scale divided out, :983-987).
 * best_idx[i] = feature of pKF selected for point i (bestDist <= TH_LOW), else -1; n_found = how many.  The MapPoint
 * bookkeeping that follows in the reference (:947-966 / :1077-1090: Replace, AddObservation, AddMapPoint, vpReplacePoint)
 * stays with the caller, applied in order; it feeds back into the search only through isBad()/IsInKeyFrame() of a
 * point listed twice, which the caller re-tests when it applies best_idx.
 * kf->u_right = pKF->mvuRight (scw_variant 0; NULL = monocular), inv_level_sigma2 = pKF->mvInvLevelSigma2 (scw_variant 0),
 * pts->valid[i] = pMP && !isBad() && !IsInKeyFrame(pKF) (resp. !spAlreadyFound.count(pMP)). kf->occupied is ignored. */
BORB_API borb_status borb_fuse(borb_matcher* m, const borb_frame_view* kf, const float* inv_level_sigma2,
                               const borb_worldpoints_view* pts, const float* Tcw, const float* Ow, float fx, float fy, float cx,
                               float cy, float bf, float log_scale_factor, float th, int scw_variant, int32_t* best_idx,
                               int32_t* n_found);

/* The search part of one Fuse call, either overload: the arguments of borb_fuse. */
typedef struct borb_fuse_job {
    borb_frame_view kf;            /* kf.resident must be set; kf.occupied is ignored */
    const float* inv_level_sigma2; /* mvInvLevelSigma2; required when scw_variant == 0 */
    borb_worldpoints_view pts;     /* valid[i] as for borb_fuse */
    float Tcw[12];
    float Ow[3];
    float fx, fy, cx, cy, bf, log_scale_factor, th;
    int32_t scw_variant;           /* 0: Fuse(pKF, vpMapPoints, th)  1: Fuse(pKF, Scw, vpPoints, th, vpReplacePoint) */
    int32_t* best_idx;             /* output, pts.n entries */
} borb_fuse_job;
/* borb_fuse for n_jobs jobs in two launches (projection, then a warp per point that walks its window's grid cells and keeps the
 * first minimum: no candidate lists, so the scratch is the projections only) and one synchronisation.  Every job's best_idx and
 * n_found[j] are bit-identical to what borb_fuse returns for the same inputs; both overloads may be mixed, and a keyframe may appear
 * in several jobs.  Keyframes must be device-resident.  A host view, a frame on another device, more than BORB_MATCH_MAX_FEATURES
 * points, log_scale_factor <= 0, an incomplete points view and scw_variant == 0 without inv_level_sigma2 are refused with
 * BORB_ERR_INVALID_ARG before anything is launched, the error text starting with "job j:".  A job with no points or a keyframe with
 * 0 features gives best_idx -1 and n_found 0.
 * The Fuse calls of LocalMapping::SearchInNeighbors (src/LocalMapping.cc:483-511) for ONE keyframe are NOT independent:
 * MapPoint::Replace recomputes the surviving point's descriptor and moves observations, and later targets see that.  Batch them
 * ACROSS camera streams instead: one call per target index with one job per stream, then one call for the
 * Fuse(mpCurrentKeyFrame, vpFuseCandidates) of every stream.  The same holds for LoopClosing::SearchAndFuse (scw_variant 1). */
BORB_API borb_status borb_fuse_batch(borb_matcher* m, const borb_fuse_job* jobs, int n_jobs, int32_t* n_found);

/* ORBmatcher::SearchBySim3(pKF1, pKF2, vpMatches12, s12, R12, t12, th) — src/ORBmatcher.cc:1102-1326
 * (LoopClosing::ComputeSim3, src/LoopClosing.cc:375-378).  pts1 / pts2 = GetMapPointMatches() of the two keyframes
 * (one slot per feature: pts->n == kf->n) with valid[i] = pMP && !vbAlreadyMatched[i] && !isBad() (:1130-1141,:1151-1155).
 * T1w / T2w = the keyframe poses (3x4); S12 = [s12*R12 | t12], S21 = [(1/s12)*R12^T | -sR21*t12] as the reference's
 * cv::Mat lines produce them (:1119-1122).  (fx,fy,cx,cy) = pKF1's intrinsics, used for both directions (:1105-1108).
 * match12[i1] = index in KF2 whose MapPoint goes to vpMatches12[i1], or -1; n_found = return value. */
BORB_API borb_status borb_search_by_sim3(borb_matcher* m, const borb_frame_view* kf1, const borb_frame_view* kf2,
                                         const borb_worldpoints_view* pts1, const borb_worldpoints_view* pts2, const float* T1w,
                                         const float* T2w, const float* S12, const float* S21, float fx, float fy, float cx, float cy,
                                         float log_scale_factor1, float log_scale_factor2, float th, int32_t* match12,
                                         int32_t* n_found);

/* Tracking::SearchLocalPoints (src/Tracking.cc:1148-1194) in one call: Frame::isInFrustum (src/Frame.cc:269-325) for every
 * candidate MapPoint, then ORBmatcher::SearchByProjection(F, vpMapPoints, th) (src/ORBmatcher.cc:45-129) on those in view —
 * the projections never leave the device.  pts->valid[i] = the point reaches isInFrustum (:1171-1175: not already matched
 * in this frame, not bad); has_obs[i] = Observations()>0 (NULL: all).  Tcw = [mRcw | mtcw], Ow = mOw, mbf, log_scale_factor =
 * Frame members; viewing_cos_limit = 0.5 at the call site.  in_view[i] = mbTrackInView (the caller runs IncreaseVisible on
 * it); proj_x/proj_y/proj_xr/level/view_cos (each may be NULL) = mTrackProjX/Y/XR, mnTrackScaleLevel, mTrackViewCos
 * (0 where not in view); match_feat / n_matches as in borb_search_by_projection.  As in the reference, a point at the camera
 * centre (PcZ == 0) is in view when its min distance is 0: its projection and viewCos are NaN (the NaN payload is not
 * specified), its level is 0, and it gets no match. */
BORB_API borb_status borb_search_local_points(borb_matcher* m, const borb_frame_view* frame, const borb_worldpoints_view* pts,
                                              const uint8_t* has_obs, const float* Tcw, const float* Ow, float fx, float fy, float cx,
                                              float cy, float mbf, float viewing_cos_limit, float log_scale_factor, float th,
                                              float nnratio, uint8_t* in_view, float* proj_x, float* proj_y, float* proj_xr,
                                              int32_t* level, float* view_cos, int32_t* match_feat, int32_t* n_matches);

/* One camera stream's Tracking::SearchLocalPoints (src/Tracking.cc:1148-1194): the per-frame arguments of
 * borb_search_local_points. */
typedef struct borb_local_points_job {
    borb_frame_view frame;         /* frame.resident must be set; frame.occupied is read per job (NULL: none) */
    borb_worldpoints_view pts;     /* as for borb_search_local_points: valid[i] = the point reaches isInFrustum (:1171-1175) */
    const uint8_t* has_obs;        /* Observations()>0 (NULL: all) */
    float Tcw[12];                 /* mCurrentFrame.mTcw rows 0..2 = [mRcw | mtcw] */
    float Ow[3];                   /* mCurrentFrame.mOw = -mRcw.t()*mtcw (src/Frame.cc:266) */
    float fx, fy, cx, cy, mbf;     /* Frame::fx, fy, cx, cy, mbf (isInFrustum, src/Frame.cc:288,319) */
    float log_scale_factor;        /* mfLogScaleFactor (PredictScale, src/MapPoint.cc:402-417) */
    float th;                      /* 1, 3 (RGB-D) or 5 (just relocalised) at the call site, src/Tracking.cc:1185-1191 */
    uint8_t* in_view;              /* outputs, pts.n entries each, as in borb_search_local_points; proj_* / level / view_cos may be NULL */
    float* proj_x;
    float* proj_y;
    float* proj_xr;
    int32_t* level;
    float* view_cos;
    int32_t* match_feat;
} borb_local_points_job;
/* borb_search_local_points for n_jobs independent camera streams in one launch sequence (projection, candidates, resolve) and one
 * synchronisation.  Every job's outputs and n_matches[j] are bit-identical to what the single call returns for the same inputs.
 * Frames must be device-resident; a host view, and every per-job argument error (more than BORB_MATCH_MAX_FEATURES valid points,
 * log_scale_factor <= 0, incomplete views), is refused with BORB_ERR_INVALID_ARG before anything is launched, the error text naming
 * the job.  A job with no points or no valid points gets the single call's defaults (in_view and track fields 0, match_feat -1,
 * n_matches 0); a frame with 0 features still gets isInFrustum's in_view and track fields, with every match_feat -1. */
BORB_API borb_status borb_search_local_points_batch(borb_matcher* m, const borb_local_points_job* jobs, int n_jobs, float viewing_cos_limit,
                                                    float nnratio, int32_t* n_matches);

/* One camera stream's ORBmatcher::SearchByProjection(CurrentFrame, LastFrame, th, bMono) (src/ORBmatcher.cc:1328-1470): the
 * per-frame arguments of borb_search_by_projection_last. */
typedef struct borb_last_frame_job {
    borb_frame_view cur;           /* cur.resident must be set; cur.occupied is read per job (NULL: none) */
    borb_lastframe_view last;
    float Tcw[12];                 /* CurrentFrame.mTcw rows 0..2 = mVelocity*mLastFrame.mTcw (src/Tracking.cc:874) */
    float fx, fy, cx, cy, bf;      /* CurrentFrame.fx, fy, cx, cy, mbf (src/ORBmatcher.cc:1370-1371,1409) */
    float th;                      /* 15 (monocular / RGB-D) or 7 (stereo), doubled on the retry, src/Tracking.cc:880-891 */
    int32_t forward, backward;     /* bForward / bBackward (src/ORBmatcher.cc:1348-1349) */
    int32_t* state_cur;            /* output, cur n entries, as in borb_search_by_projection_last */
} borb_last_frame_job;
/* borb_search_by_projection_last for n_jobs independent camera streams in one launch sequence (projection, candidates, resolve
 * with a rotation histogram per job) and one synchronisation.  check_orientation applies to every job.  Every job's state_cur and
 * n_matches[j] are bit-identical to the single call's.  Frames must be device-resident; a host view and every per-job argument
 * error (more than BORB_MATCH_MAX_FEATURES last-frame points, last-frame octaves outside the frame's levels, incomplete views) are
 * refused with BORB_ERR_INVALID_ARG before anything is launched, the error text naming the job.  A job with an empty last frame or
 * a frame with 0 features gets state_cur -1 and n_matches 0. */
BORB_API borb_status borb_search_by_projection_last_batch(borb_matcher* m, const borb_last_frame_job* jobs, int n_jobs, int check_orientation,
                                                          int32_t* n_matches);

/* ORBmatcher::SearchForInitialization(Frame &F1, Frame &F2, vector<cv::Point2f> &vbPrevMatched, vector<int> &vnMatches12,
 * int windowSize) — src/ORBmatcher.cc:405-520 (Tracking::MonocularInitialization, src/Tracking.cc:599).
 * f1/f2: keys_un, desc (and f2's grid bounds) are read; prev_matched = vbPrevMatched as f1->n x 2 floats, updated in
 * place (:513-517); matches12[i1] = index in F2 or -1; n_matches = return value.  The one-job case of
 * borb_search_for_initialization_batch on host views: the device scratch is f1->n x 36 bytes plus f2's feature grid, with no
 * f1->n x f2->n candidate list. */
BORB_API borb_status borb_search_for_initialization(borb_matcher* m, const borb_frame_view* f1, const borb_frame_view* f2,
                                                    float* prev_matched, int window_size, float nnratio, int check_orientation,
                                                    int32_t* matches12, int32_t* n_matches);

/* One camera stream's ORBmatcher::SearchForInitialization(mInitialFrame, mCurrentFrame, mvbPrevMatched, mvIniMatches, windowSize)
 * (src/ORBmatcher.cc:405-520, src/Tracking.cc:600). */
typedef struct borb_init_job {
    const borb_frame* initial;     /* F1 = mInitialFrame, resident */
    const borb_frame* current;     /* F2 = mCurrentFrame, resident (its feature grid is used as built) */
    float* prev_matched;           /* in/out, initial->n x 2: vbPrevMatched, updated as the single call does (:513-517) */
    int32_t window_size;           /* 100 at the call site */
    int32_t* matches12;            /* output, initial->n entries: vnMatches12 */
} borb_init_job;
/* borb_search_for_initialization for n_jobs camera streams on resident frames in two launches and one synchronisation, whatever
 * n_jobs is.  nnratio and check_orientation apply to every job.  Every job's matches12, prev_matched and n_matches[j] are
 * bit-identical to what borb_search_for_initialization returns on host views of the same two frames.  A frame may appear in several
 * jobs (one initial frame against several current frames), and initial == current is allowed.  A NULL frame, a frame on another
 * device, a NULL prev_matched or matches12 for an initial frame with features, and a NULL jobs or n_matches when n_jobs > 0 are
 * refused with BORB_ERR_INVALID_ARG before anything is launched, the error text starting with "job j:".  A job whose initial or
 * current frame has 0 features gets matches12 -1 and 0 matches, its prev_matched untouched.
 * Per job, only prev_matched crosses PCIe (initial->n x 8 bytes each way, plus initial->n x 4 + 4 bytes of results); the device
 * scratch is initial->n x 36 bytes (the 8 smallest window entries and the window size of each initial-frame feature), with no
 * initial->n x current->n candidate list. */
BORB_API borb_status borb_search_for_initialization_batch(borb_matcher* m, const borb_init_job* jobs, int n_jobs,
                                                          float nnratio, int check_orientation, int32_t* n_matches);

/* One lost camera stream's ORBmatcher::SearchByProjection(CurrentFrame, pKF, sFound, th, ORBdist) after PnP in
 * Tracking::Relocalization (src/Tracking.cc:1452 with th 10, ORBdist 100, and :1466 with th 3, ORBdist 64; src/ORBmatcher.cc:1472-1599):
 * the per-frame arguments of borb_search_by_projection_kf. */
typedef struct borb_kf_projection_job {
    borb_frame_view cur;           /* cur.resident must be set; cur.occupied[i2] = CurrentFrame.mvpMapPoints[i2] != NULL, read per job */
    borb_worldpoints_view pts;     /* pKF->GetMapPointMatches(), valid[i] = pMP && !isBad() && !sFound.count(pMP) */
    float Tcw[12];                 /* CurrentFrame.mTcw rows 0..2 (the PnP pose) */
    float Ow[3];                   /* -Rcw.t()*tcw (:1476-1478) */
    float fx, fy, cx, cy;          /* CurrentFrame.fx, fy, cx, cy */
    float log_scale_factor;        /* CurrentFrame.mfLogScaleFactor */
    float th;                      /* 10 or 3 */
    int32_t orb_dist;              /* 100 or 64 */
    int32_t* state_cur;            /* output, cur n entries, as in borb_search_by_projection_kf */
} borb_kf_projection_job;
/* borb_search_by_projection_kf for n_jobs camera streams in one launch sequence (projection, candidates, resolve with a rotation
 * histogram per job) and one synchronisation.  check_orientation applies to every job (the relocalisation matcher is
 * ORBmatcher(0.9, true), src/Tracking.cc:1396).  Every job's state_cur and n_matches[j] are bit-identical to the single call's.
 * Frames must be device-resident; a host view, a frame on another device, more than BORB_MATCH_MAX_FEATURES points,
 * log_scale_factor <= 0, an incomplete points view and a NULL state_cur are refused with BORB_ERR_INVALID_ARG before anything is
 * launched, the error text starting with "job j:".  A job with no points or a frame with 0 features gets state_cur -1 and 0 matches.
 * The device scratch of a job includes a candidate list of pts.n x cur n x 4 bytes, as for borb_search_by_projection_last_batch. */
BORB_API borb_status borb_search_by_projection_kf_batch(borb_matcher* m, const borb_kf_projection_job* jobs, int n_jobs,
                                                        int check_orientation, int32_t* n_matches);

/* One loop-closing stream's final ORBmatcher::SearchByProjection(mpCurrentKF, mScw, mvpLoopMapPoints, mvpCurrentMatchedPoints, 10)
 * in LoopClosing::ComputeSim3 (src/LoopClosing.cc:375; src/ORBmatcher.cc:290-403): the arguments of borb_search_by_projection_sim3. */
typedef struct borb_sim3_projection_job {
    borb_frame_view kf;            /* kf.resident must be set; kf.occupied[idx] = vpMatched[idx] != NULL on entry, read per job */
    borb_worldpoints_view pts;     /* mvpLoopMapPoints, valid[i] = !isBad() && !spAlreadyFound.count(pMP) */
    float Tcw[12];                 /* [Rcw | tcw] with the Sim3 scale divided out (:298-303) */
    float Ow[3];                   /* -Rcw.t()*tcw */
    float fx, fy, cx, cy;          /* pKF->fx, fy, cx, cy */
    float log_scale_factor;        /* pKF->mfLogScaleFactor */
    int32_t th;                    /* 10 */
    int32_t* state_kf;             /* output, kf n entries, as in borb_search_by_projection_sim3 */
} borb_sim3_projection_job;
/* borb_search_by_projection_sim3 for n_jobs streams in one launch sequence (projection, candidates, resolve) and one
 * synchronisation.  Every job's state_kf and n_matches[j] are bit-identical to the single call's.  Keyframes must be
 * device-resident; refusals, defaults and scratch as for borb_search_by_projection_kf_batch. */
BORB_API borb_status borb_search_by_projection_sim3_batch(borb_matcher* m, const borb_sim3_projection_job* jobs, int n_jobs,
                                                          int32_t* n_matches);

/* One ORBmatcher::SearchBySim3(mpCurrentKF, pKF, vpMapPointMatches, s, R, t, 7.5) of LoopClosing::ComputeSim3
 * (src/LoopClosing.cc:323; src/ORBmatcher.cc:1102-1326): the arguments of borb_search_by_sim3. */
typedef struct borb_sim3_job {
    borb_frame_view kf1;           /* pKF1 = mpCurrentKF, kf1.resident must be set; kf1.occupied is ignored */
    borb_frame_view kf2;           /* pKF2 = the loop candidate, resident; kf2.occupied is ignored */
    borb_worldpoints_view pts1;    /* kf1's GetMapPointMatches(), one slot per feature (pts1.n == kf1's n), valid as for the single call */
    borb_worldpoints_view pts2;    /* kf2's, pts2.n == kf2's n */
    float T1w[12];                 /* the keyframe poses (3x4) */
    float T2w[12];
    float S12[12];                 /* [s12*R12 | t12] and [(1/s12)*R12^T | -sR21*t12] (:1119-1122) */
    float S21[12];
    float fx, fy, cx, cy;          /* pKF1's intrinsics, used for both directions (:1105-1108) */
    float log_scale_factor1, log_scale_factor2;
    float th;                      /* 7.5 */
    int32_t* match12;              /* output, kf1 n entries, as in borb_search_by_sim3 */
} borb_sim3_job;
/* borb_search_by_sim3 for n_jobs (keyframe, candidate) pairs in three launches (projection of both directions of every job, a warp
 * per point that walks its window's grid cells and keeps the first minimum, then the agreement test) and one synchronisation,
 * whatever n_jobs is.  Every job's match12 and n_found[j] are bit-identical to what borb_search_by_sim3 returns; kf1 == kf2 is
 * allowed and a keyframe may appear in several jobs.  Keyframes must be device-resident; a host view, a frame on another device,
 * more than BORB_MATCH_MAX_FEATURES points, pts1.n / pts2.n different from the keyframe's n, log_scale_factor <= 0, an incomplete
 * points view and a NULL match12 are refused with BORB_ERR_INVALID_ARG before anything is launched, the error text starting with
 * "job j:".  A job whose keyframes have 0 features gets match12 -1 and n_found 0.  The device scratch of a job is the projections
 * of its pts1.n + pts2.n points and (pts1.n + pts2.n) x 4 bytes of per-direction matches, with no candidate list. */
BORB_API borb_status borb_search_by_sim3_batch(borb_matcher* m, const borb_sim3_job* jobs, int n_jobs, int32_t* n_found);

/* MapPoint::ComputeDistinctiveDescriptors — src/MapPoint.cc:242-307, for n_points MapPoints in one launch.
 * desc: the observing keyframes' descriptors (pKF->mDescriptors.row(idx) of every non-bad observation, in
 * mObservations order), MapPoint p owning rows offsets[p] .. offsets[p+1]-1.  best_idx[p] = row (relative to
 * offsets[p]) of the descriptor with the least median distance to the others, -1 if the point has none. */
BORB_API borb_status borb_distinctive_descriptors(borb_matcher* m, const uint8_t* desc, const int32_t* offsets, int n_points,
                                                  int32_t* best_idx);

/* MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:242-307) for n_points MapPoints, read from resident keyframes.
 * frames[0..n_frames)        resident frames of the observing keyframes: any stream, any matcher on this device, repeats allowed
 * offsets[n_points + 1]      MapPoint p owns observations offsets[p] .. offsets[p+1]-1, in mObservations order, bad keyframes dropped
 * obs_frame[o], obs_idx[o]   observation o = row obs_idx[o] of frames[obs_frame[o]]
 * best_idx[p]                as borb_distinctive_descriptors (relative to offsets[p]; -1 when the point has no observation)
 * desc_out[p*32 .. +32)      that row: the new mDescriptor; left unchanged where best_idx[p] == -1
 * Many streams concatenate their points and frames into one call.  best_idx and desc_out are bit-identical to
 * borb_distinctive_descriptors on the same rows gathered on the host (first minimal median wins, median = sorted_row[(int)(0.5*(N-1))],
 * self-distance included).  One launch and one synchronisation when any observation exists, none otherwise; the call waits for every
 * distinct frame of the table.  Only obs_frame / obs_idx (8 bytes per observation), the offsets and the frame table (8 bytes per entry)
 * go up, and only best_idx and 32 bytes per point come down: a host keeps no copy of a keyframe's descriptors.  A NULL frame, a frame
 * on another device, obs_frame[o] outside [0, n_frames), obs_idx[o] outside [0, that frame's n), offsets that do not ascend from 0,
 * more than 65535 observations on one point and NULL outputs with n_points > 0 are refused with BORB_ERR_INVALID_ARG before anything
 * is uploaded or launched, the error text naming the point ("point p:") or the frame-table entry ("frame f"). */
BORB_API borb_status borb_distinctive_descriptors_frames(borb_matcher* m, const borb_frame* const* frames, int n_frames,
                                                         const int32_t* obs_frame, const int32_t* obs_idx, const int32_t* offsets,
                                                         int n_points, int32_t* best_idx, uint8_t* desc_out);

/* DBoW2::FeatureVector (ordered map NodeId -> feature indices) as CSR: node_id strictly ascending, 0 <= start[0] <=
 * start[1] <= ... <= start[n_nodes], and every feat_idx[r], r < start[n_nodes], below the view's n.  Every entry point that takes a
 * borb_keyframe_view as a host view checks this and refuses a violator with BORB_ERR_INVALID_ARG before anything is launched. */
typedef struct borb_featvec_view {
    int32_t n_nodes;
    const uint32_t* node_id;
    const int32_t* start;          /* n_nodes + 1 */
    const uint32_t* feat_idx;
} borb_featvec_view;

/* KeyFrame (or Frame) snapshot for the BoW-guided searches. */
typedef struct borb_keyframe_view {
    int32_t n;
    const borb_keypoint* keys_un;  /* mvKeysUn (angle, octave, pt) */
    const uint8_t* desc;           /* mDescriptors */
    const uint8_t* has_mp;         /* per feature: MapPoint present && !isBad() (NULL: none) */
    const float* u_right;          /* mvuRight (NULL: all -1) */
    borb_featvec_view fv;          /* mFeatVec */
    int32_t n_levels;
    const float* scale_factors;    /* mvScaleFactors */
    const float* level_sigma2;     /* mvLevelSigma2 */
} borb_keyframe_view;

/* ORBmatcher::SearchByBoW(KeyFrame*, Frame&, vector<MapPoint*>&) — src/ORBmatcher.cc:159-288, for n_kf keyframes
 * against one frame in one launch (relocalisation / loop candidates).  match[k*frame->n + j] = index of the
 * feature of keyframe k whose MapPoint frame feature j received, or -1; n_matches[k] = return value. */
BORB_API borb_status borb_search_by_bow(borb_matcher* m, const borb_keyframe_view* kfs, int n_kf, const borb_keyframe_view* frame,
                                        float nnratio, int check_orientation, int32_t* match, int32_t* n_matches);
/* ORBmatcher::SearchByBoW(KeyFrame*, KeyFrame*, vector<MapPoint*>&) — src/ORBmatcher.cc:522-655.
 * match12[i] = index in kf2 of the MapPoint matched to feature i of kf1, or -1. */
BORB_API borb_status borb_search_by_bow_kf(borb_matcher* m, const borb_keyframe_view* kf1, const borb_keyframe_view* kf2,
                                           float nnratio, int check_orientation, int32_t* match12, int32_t* n_matches);

/* One camera stream's TrackReferenceKeyFrame search, ORBmatcher::SearchByBoW(KeyFrame*, Frame&) (src/ORBmatcher.cc:159-288). */
typedef struct borb_bow_job {
    const borb_frame* frame;       /* current frame: resident, BoW computed */
    borb_keyframe_view kf;         /* reference keyframe as a host view; kf.has_mp is always read from here */
    const borb_frame* kf_frame;    /* NULL, or the resident frame the keyframe was made from (BoW computed): then kf.n, keys_un,
                                      desc and fv are taken from it and only kf.has_mp crosses PCIe */
    int32_t* match;                /* output, frame n entries: as borb_search_by_bow */
} borb_bow_job;
/* borb_search_by_bow (one keyframe against one frame) for n_jobs independent camera streams in one launch and one synchronisation
 * (Tracking::TrackReferenceKeyFrame, src/Tracking.cc:757-799, runs it whenever the motion model has no velocity or finds too few
 * matches).  Frames come with the BoW of borb_frames_compute_bow, so nothing of the current frame crosses PCIe.  match and n_matches[j]
 * are bit-identical to borb_search_by_bow on host views of the same data.  A NULL frame, a frame without BoW (every frame comes from
 * borb_frame_create / borb_frames_from_extractor without one, recycled ones included), a frame on another device and an incomplete
 * host view are refused with BORB_ERR_INVALID_ARG before anything is launched, the error text naming the job.  A frame with 0 features
 * or a keyframe with an empty FeatureVector gives 0 matches (match all -1). */
BORB_API borb_status borb_search_by_bow_batch(borb_matcher* m, const borb_bow_job* jobs, int n_jobs, float nnratio,
                                              int check_orientation, int32_t* n_matches);
/* ORBmatcher::SearchForTriangulation — src/ORBmatcher.cc:657-823.  F12 row-major 3x3; (ex,ey) = projection of
 * kf1's camera centre into kf2 (:663-670, computed by the caller).  pairs: 2*cap ints (idx1, idx2), ascending idx1. */
BORB_API borb_status borb_search_for_triangulation(borb_matcher* m, const borb_keyframe_view* kf1, const borb_keyframe_view* kf2,
                                                   const float* F12, float ex, float ey, int only_stereo, int check_orientation,
                                                   int32_t* pairs, int cap, int32_t* n_pairs);

/* One SearchForTriangulation(pKF1, pKF2, F12, vMatchedPairs, bOnlyStereo) (src/ORBmatcher.cc:657-823). */
typedef struct borb_triangulation_job {
    borb_keyframe_view kf1;        /* has_mp = GetMapPoint(i) != NULL (:697-703) is always read from here */
    const borb_frame* kf1_frame;   /* NULL, or the resident frame kf1 was made from, BoW computed: then n, keys_un, desc, u_right, fv,
                                      scale_factors come from it (exactly borb_bow_job::kf_frame) */
    borb_keyframe_view kf2;        /* has_mp and level_sigma2 (mvLevelSigma2) always read from here */
    const borb_frame* kf2_frame;
    float F12[9];                  /* row-major, LocalMapping::ComputeF12 */
    float ex, ey;                  /* epipole of kf1 in kf2 (:663-670) */
    int32_t only_stereo;
    int32_t* pairs;                /* output: 2*cap ints (idx1, idx2), ascending idx1 */
    int32_t cap;
    int32_t* n_pairs;
} borb_triangulation_job;
/* borb_search_for_triangulation for n_jobs jobs in ONE launch (a CTA per job) and one synchronisation; every job's pairs and n_pairs
 * are bit-identical to the single call's.  A keyframe may appear in several jobs (one keyframe against all its neighbours is the
 * main use).  A NULL/foreign-device/BoW-less kf*_frame, more than BORB_MATCH_MAX_FEATURES features, an incomplete view and a kf2
 * without level_sigma2 are refused with BORB_ERR_INVALID_ARG before anything is launched, the error text starting with "job j:".
 * Pairs beyond a job's cap give BORB_ERR_CAPACITY after the run (every n_pairs stays valid; the error names the first such job).
 * A job with 0 features or an empty FeatureVector on either side gives 0 pairs and no work.
 * LocalMapping::CreateNewMapPoints (src/LocalMapping.cc:207-268) from one call: submit every neighbour that passes the baseline
 * test, with kf1's has_mp as it is on entry and check_orientation = 0 (the reference's ORBmatcher matcher(0.6,false)), then
 * triangulate the neighbours IN ORDER, dropping from neighbour i's pairs every idx1 that an earlier neighbour gave a MapPoint.
 * Without the orientation check each row's result depends only on its own idx1 and on has_mp, so this replays the sequential calls
 * exactly (the CheckNewKeyFrames() early return is the caller stopping the replay).  With check_orientation = 1 the rotation
 * histogram couples the rows and the replay is NOT exact. */
BORB_API borb_status borb_search_for_triangulation_batch(borb_matcher* m, const borb_triangulation_job* jobs, int n_jobs,
                                                         int check_orientation);

/* ---- device-resident keyframe database -------------------------------------------------------------------------
 * KeyFrameDatabase (include/KeyFrameDatabase.h, src/KeyFrameDatabase.cc) re-designed for the GPU: instead of an inverted
 * file walked per query word, every keyframe's BowVector (and the keyframe-side inputs of SearchByBoW: keypoints,
 * descriptors, FeatureVector, MapPoint mask) stays in HBM, and one launch computes for ALL keyframes what the walk and
 * the scoring loop produce: the number of words shared with the query (mnRelocWords / mnLoopWords, :91-108,:211-224) and
 * DBoW2's L1 score (:127,:240; Thirdparty/DBoW2/DBoW2/ScoringObject.cpp:23-71), bit-identical (terms added in word
 * order).  The covisibility accumulation that follows (:134-190,:251-307) walks the keyframe graph and stays with the
 * caller; first_word gives it the reference's list order (keyframes are met in order of their first shared word,
 * then of insertion into that word's list). */
typedef struct borb_kfdb borb_kfdb;
BORB_API borb_status borb_kfdb_create(int device, borb_kfdb** out);
BORB_API borb_status borb_kfdb_destroy(borb_kfdb* db);
BORB_API borb_status borb_kfdb_clear(borb_kfdb* db);                                   /* KeyFrameDatabase::clear :68-73 */
/* KeyFrameDatabase::add (:41-47).  bow_word ascending (std::map order), bow_value = BowVector weights (double).
 * *slot_out identifies the keyframe from now on (slots are never reused). */
BORB_API borb_status borb_kfdb_add(borb_kfdb* db, const borb_keyframe_view* kf, const uint32_t* bow_word, const double* bow_value,
                                   int n_bow, int32_t* slot_out);
BORB_API borb_status borb_kfdb_erase(borb_kfdb* db, int32_t slot);                     /* KeyFrameDatabase::erase :49-66 */
BORB_API borb_status borb_kfdb_set_has_mp(borb_kfdb* db, int32_t slot, const uint8_t* has_mp);   /* MapPoints culled / added since add() */
/* borb_kfdb_set_has_mp for n slots (repeats allowed, the last mask wins) with one device synchronisation; every slot is checked
 * before any mask changes. */
BORB_API borb_status borb_kfdb_set_has_mp_batch(borb_kfdb* db, int n, const int32_t* slots, const uint8_t* const* has_mp);
BORB_API borb_status borb_kfdb_size(const borb_kfdb* db, int32_t* n_slots, uint64_t* device_bytes);
/* One query BowVector against every keyframe.  Outputs have one entry per slot (erased slots: 0 common words):
 * common_words[s], score[s] = (float)L1 score, first_word[s] = smallest shared word id (0xFFFFFFFF if none). */
BORB_API borb_status borb_kfdb_query(borb_matcher* m, borb_kfdb* db, const uint32_t* bow_word, const double* bow_value, int n_bow,
                                     int32_t* common_words, float* score, uint32_t* first_word, int cap, int32_t* n_slots);
/* borb_search_by_bow with the keyframes taken from the database (only the frame is uploaded). */
BORB_API borb_status borb_search_by_bow_db(borb_matcher* m, borb_kfdb* db, const int32_t* slots, int n_kf,
                                           const borb_keyframe_view* frame, float nnratio, int check_orientation, int32_t* match,
                                           int32_t* n_matches);

/* The same search returning COMPACT results — the form to use against many keyframes (BASELINE configs[4]: one frame
 * against a 2000-keyframe database; the dense matrix above would be 9.7 MB of D2H per query).  slots == NULL searches
 * slots 0..n_kf-1 (n_kf must equal the slot count; erased slots give 0 matches).  n_matches[k] = return value of
 * SearchByBoW for keyframe k.  If pairs != NULL: keyframe k's matches are pairs[pair_offset[k] .. + n_matches[k]), each
 * (frame feature index) | (keyframe feature index) << 16, in FeatureVector order of the frame (node id, then feature index);
 * the blocks of different keyframes are packed in no particular order.  *n_pairs_total = sum of n_matches; more than pairs_cap
 * => BORB_ERR_CAPACITY (counts and offsets are still valid). */
BORB_API borb_status borb_search_by_bow_db_pairs(borb_matcher* m, borb_kfdb* db, const int32_t* slots, int n_kf,
                                                 const borb_keyframe_view* frame, float nnratio, int check_orientation,
                                                 int32_t* n_matches, int32_t* pair_offset, uint32_t* pairs, int pairs_cap,
                                                 int32_t* n_pairs_total);

/* Relocalisation (Tracking::Relocalization, src/Tracking.cc:1341-1470) and loop-closure queries of many camera streams on resident
 * frames: the database query and the SearchByBoW of every lost stream, one call each, with nothing of the frames crossing PCIe.
 * Frames come with the BoW of borb_frames_compute_bow.  Each job names its own database: many streams with their own maps, or many
 * queries on one.  Every distinct database is locked for the table sync and the enqueue, in address order, so two concurrent
 * batches cannot deadlock; borb_kfdb_erase and borb_kfdb_set_has_mp keep their guarantees.  Argument errors are refused with
 * BORB_ERR_INVALID_ARG before anything is launched, the error text starting "job j:": a NULL database or frame, a frame without BoW
 * (recycled frames included), a frame, database and matcher on different devices, a slot that is not a live keyframe, slots == NULL
 * with n_kf different from the slot count, pairs without pair_offset.  A job with n_kf == 0, a database without slots, or a frame
 * with 0 features or only stop words gives zeros. */
typedef struct borb_kfdb_query_job {
    borb_kfdb* db;
    const borb_frame* frame;       /* resident, BoW computed by borb_frames_compute_bow */
    int32_t* common_words;         /* outputs, one entry per slot, as borb_kfdb_query */
    float* score;
    uint32_t* first_word;
    int32_t cap;                   /* entries of each output; fewer than the database's slots => BORB_ERR_CAPACITY before any launch */
    int32_t* n_slots;
} borb_kfdb_query_job;
/* borb_kfdb_query for n_jobs frames: job j returns exactly what borb_kfdb_query returns for the frame's BowVector.
 * 1 launch whatever n_jobs (0 when no database has a slot), one synchronisation. */
BORB_API borb_status borb_kfdb_query_batch(borb_matcher* m, const borb_kfdb_query_job* jobs, int n_jobs);

/* KeyFrameDatabase::add (:41-47) of many keyframes straight from their resident frames: LoopClosing::DetectLoop of many camera
 * streams adds each stream's keyframe with nothing of it crossing PCIe but the MapPoint mask.  Job j leaves its database exactly as
 * borb_kfdb_add, called in job order, leaves it for a host view of the frame (its mvKeysUn, mDescriptors and FeatureVector, and
 * has_mp) with the frame's BowVector: the same block bytes, the same slot (jobs on one database get ascending slots in job order),
 * the same borb_kfdb_size bytes, the same host copy of the row records that borb_kfdb_set_has_mp rewrites later.  The caller's duty,
 * as for borb_search_by_bow_db_batch: the frame's FeatureVector level (borb_frames_compute_bow's levelsup) must be the database's.
 * The new slot does not refer to the frame: destroying or recycling the frame afterwards changes nothing.  Argument errors are
 * refused with BORB_ERR_INVALID_ARG before anything is allocated or launched, the error text starting "job j:": a NULL database,
 * frame or slot_out, a frame without BoW (recycled frames included), a frame, database and matcher on different devices.  A CUDA
 * failure frees every block the call allocated and appends no slot.  A frame with 0 features or only stop words is added as
 * borb_kfdb_add adds empty vectors.  1 launch whatever n_jobs, one synchronisation; the blocks are complete when the call returns.
 * Every distinct database is locked, in address order, while the slots are appended. */
typedef struct borb_kfdb_add_job {
    borb_kfdb* db;
    const borb_frame* frame;       /* resident, BoW computed by borb_frames_compute_bow */
    const uint8_t* has_mp;         /* host, frame n entries: MapPoint present && !isBad(); NULL: none */
    int32_t* slot_out;
} borb_kfdb_add_job;
BORB_API borb_status borb_kfdb_add_frames(borb_matcher* m, const borb_kfdb_add_job* jobs, int n_jobs);

/* TemplatedVocabulary::score (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h; ScoringObject.cpp:23-71) between BowVectors that are
 * already on the device: LoopClosing::DetectLoop's minScore (src/LoopClosing.cc:121-140) of many camera streams with no host
 * BowVector.  A BowVector is a resident frame's (borb_frames_compute_bow) or a database slot's, whether or not the keyframe has
 * been added to a database yet.  score[t] = (float)score(query, targets[t]), bit-identical to DBoW2's L1 score cast to float: v1 is
 * the query, v2 the target, the terms are added in ascending word order, and two vectors that share no word give -0.0f.  Frames and
 * slots mix freely on either side, from any number of databases; repeats are allowed, and so is a query that is also one of its own
 * targets.  Argument errors are refused with BORB_ERR_INVALID_ARG before anything is uploaded, the error text starting "job j:" or,
 * for a reference, "job j query:" / "job j target t:": NULL pointers, n_targets < 0, a reference with neither frame nor database,
 * a frame without BoW (recycled frames included), a frame or database on another device than the matcher, a slot that is out of
 * range or erased.  The slots are resolved and read under the databases' locks (taken in address order), so a concurrent
 * borb_kfdb_add, _erase or _set_has_mp is seen whole.  1 launch whatever n_jobs (0 when no job has a target), one
 * synchronisation. */
typedef struct borb_bow_ref {           /* one BowVector resident on the device */
    const borb_frame* frame;            /* a resident frame whose BoW borb_frames_compute_bow computed, or NULL ... */
    borb_kfdb* db; int32_t slot;        /* ... then a live slot of a database */
} borb_bow_ref;
typedef struct borb_bow_score_job {
    borb_bow_ref query;                 /* v1 of score(): LoopClosing's mpCurrentKF->mBowVec */
    const borb_bow_ref* targets;        /* v2 of each score(): the covisible keyframes */
    int32_t n_targets;
    float* score;                       /* n_targets: float score = mpVoc->score(v1, v2) (LoopClosing.cc:133) */
} borb_bow_score_job;
BORB_API borb_status borb_bow_score_batch(borb_matcher* m, const borb_bow_score_job* jobs, int n_jobs);

typedef struct borb_bow_db_job {
    borb_kfdb* db;
    const borb_frame* frame;       /* resident, BoW computed */
    const int32_t* slots;          /* candidate keyframes (repeats allowed); NULL: every slot, n_kf must be the slot count */
    int32_t n_kf;
    int32_t* n_matches;            /* outputs as borb_search_by_bow_db_pairs; pair_offset indexes this job's own pairs */
    int32_t* pair_offset;
    uint32_t* pairs;
    int32_t pairs_cap;
    int32_t* n_pairs_total;
} borb_bow_db_job;
/* borb_search_by_bow_db_pairs for n_jobs frames: job j returns for every keyframe the same count and the same pair block as
 * borb_search_by_bow_db_pairs on a host view of the frame; only the placement of the blocks inside the job's pairs differs.  The
 * caller's duty, as for the single call: the frame's FeatureVector (borb_frames_compute_bow's levelsup) must be at the same level
 * as the FeatureVectors of the database's keyframes.  Pairs beyond a job's pairs_cap give BORB_ERR_CAPACITY after the run; counts
 * and offsets are still valid for every job, and the error names the first job that overflowed.  3 launches whatever n_jobs (the
 * device packer of the frame blocks, the match kernel, the rotation cull; 0 when no job has work), one synchronisation.  The
 * single calls are the one-job case of the same launches. */
BORB_API borb_status borb_search_by_bow_db_batch(borb_matcher* m, const borb_bow_db_job* jobs, int n_jobs, float nnratio,
                                                 int check_orientation);

/* Loop closure: ORBmatcher::SearchByBoW(KeyFrame* pKF1, KeyFrame* pKF2, vector<MapPoint*>&) (src/ORBmatcher.cc:522-655) of the
 * loop-closing keyframe against its candidates (LoopClosing::ComputeSim3, src/LoopClosing.cc:251-280), both sides read from the
 * database: nothing crosses PCIe but the slot list and the results.  Both MapPoint masks are the database's (the caller keeps them
 * current with borb_kfdb_set_has_mp).  Job j returns for candidate k the count and, in pairs[pair_offset[k] .. + n_matches[k]),
 * (query feature) | (candidate feature) << 16 in the query's FeatureVector order: exactly borb_search_by_bow_kf(query, candidate).
 * A query slot that is also a candidate is searched like any other.  Locks, outputs and errors as borb_search_by_bow_db_batch; the
 * argument errors (text "job j:") are a NULL database or one on another device, a query slot that is erased, out of range or was
 * added without features, a candidate that is not a live slot, slots == NULL with n_kf different from the slot count, pairs without
 * pair_offset.  3 launches whatever n_jobs, one synchronisation; the single call is the one-job case. */
typedef struct borb_bow_kf_db_job {
    borb_kfdb* db;
    int32_t query_slot;            /* KF1: the loop-closing keyframe, a live slot of db added with features */
    const int32_t* slots;          /* KF2 candidates (repeats allowed); NULL: every slot, n_kf must be the slot count */
    int32_t n_kf;
    int32_t* n_matches;            /* outputs as borb_search_by_bow_db_pairs, pairs = query feature | candidate feature << 16, */
    int32_t* pair_offset;          /*   each candidate's block in the query's FeatureVector order */
    uint32_t* pairs;
    int32_t pairs_cap;
    int32_t* n_pairs_total;
} borb_bow_kf_db_job;
BORB_API borb_status borb_search_by_bow_kf_db_batch(borb_matcher* m, const borb_bow_kf_db_job* jobs, int n_jobs, float nnratio,
                                                    int check_orientation);
BORB_API borb_status borb_search_by_bow_kf_db_pairs(borb_matcher* m, borb_kfdb* db, int32_t query_slot, const int32_t* slots, int n_kf,
                                                    float nnratio, int check_orientation, int32_t* n_matches, int32_t* pair_offset,
                                                    uint32_t* pairs, int pairs_cap, int32_t* n_pairs_total);

/* ---------------------------------------------------------------- vocabulary (BoW feeder) ---- */
/* ORBVocabulary = DBoW2::TemplatedVocabulary<FORB> (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h).  The tree lives
 * in HBM as one packed blob (so it can be broadcast over NCCL once and shared by every stream of a GPU).  One handle may be
 * used by several threads at once (see the top of this file). */
typedef struct borb_voc borb_voc;
/* Nodes in id order, node 0 = root; children keep the order in which they appear (loadFromTextFile :1378-1420). */
BORB_API borb_status borb_voc_create(const int32_t* parent, const uint8_t* is_leaf, const uint8_t* desc, const double* weight,
                                     int n_nodes, int k, int L, int device, borb_voc** out);
/* "k L scoring weighting" + one "parent isLeaf d0..d31 weight" line per node (ORBvoc.txt, :1338-1424). */
BORB_API borb_status borb_voc_load_text(const char* path, int device, borb_voc** out);
BORB_API borb_status borb_voc_destroy(borb_voc* v);
/* Device address and size of the packed blob (root rank: source of the NCCL broadcast). */
BORB_API borb_status borb_voc_blob(const borb_voc* v, void** d_blob, size_t* bytes);
/* Adopt a packed blob that already sits in this device's memory (receiver side of the broadcast). */
BORB_API borb_status borb_voc_from_blob(void* d_blob, size_t bytes, int device, borb_voc** out);
/* NCCL without torch, for a C++ Tracking host (SURVEY §8e): the vocabulary is parsed by ONE rank (src/System.cc:65 loads the 145 MB
 * text on every process) and broadcast over NVLink into every GPU's HBM.  libnccl.so.2 is resolved with dlopen at the first call
 * (BORB_ERR_UNSUPPORTED if absent); libborb.so itself does not link NCCL.
 *   borb_nccl_unique_id: ncclGetUniqueId (128 bytes) on one rank, handed to the others by the host's own means;
 *   borb_nccl_comm_create / _destroy: ncclCommInitRank / ncclCommDestroy — or pass an ncclComm_t the host already owns;
 *   borb_voc_broadcast: two ncclBroadcast calls (size, blob).  On `root` pass the loaded vocabulary and get it back in *out;
 *   elsewhere pass NULL and receive a vocabulary backed by the received blob.  nccl_comm = the rank's ncclComm_t. */
BORB_API borb_status borb_nccl_unique_id(uint8_t* id128);
BORB_API borb_status borb_nccl_comm_create(const uint8_t* id128, int world_size, int rank, int device, void** nccl_comm);
BORB_API borb_status borb_nccl_comm_destroy(void* nccl_comm);
BORB_API borb_status borb_voc_broadcast(borb_voc* root_voc, void* nccl_comm, int root, int rank, int device, borb_voc** out);

/* TemplatedVocabulary::transform(feature, id, weight, nid, levelsup) for n descriptors (:1218-1259): word id,
 * word weight and the node id at level L-levelsup per feature — the descent of borb_frames_compute_bow alone, on one frame of
 * host descriptors, any n.  One launch, one synchronisation. */
BORB_API borb_status borb_bow_transform(borb_voc* v, const uint8_t* desc, int n, int levelsup, int32_t* word, double* weight,
                                        int32_t* node);

/* Frame::ComputeBoW / KeyFrame::ComputeBoW (src/Frame.cc:395-402, src/KeyFrame.cc:59-68): mBowVec and mFeatVec of n descriptors in
 * one call — the one-frame case of borb_frames_compute_bow on host descriptors: the tree descent and the ordered-map bookkeeping
 * of TemplatedVocabulary::transform (:1150-1194) both on the device, 2 launches and one synchronisation.
 * bow_word / bow_value: BowVector in word order (capacity n), *n_bow entries; fv_node / fv_start / fv_idx: FeatureVector as CSR
 * (capacities n, n + 1, n), *n_nodes nodes — the layout borb_featvec_view and borb_kfdb_add take.  n > BORB_MATCH_MAX_FEATURES is
 * refused (BORB_ERR_INVALID_ARG), as every consumer of a FeatureVector refuses such a frame. */
BORB_API borb_status borb_compute_bow(borb_voc* v, const uint8_t* desc, int n, int levelsup, uint32_t* bow_word, double* bow_value,
                                      int32_t* n_bow, uint32_t* fv_node, int32_t* fv_start, uint32_t* fv_idx, int32_t* n_nodes);

/* Frame::ComputeBoW (src/Frame.cc:395-402) for n_frames resident frames: tree descent and the BowVector / FeatureVector
 * bookkeeping of TemplatedVocabulary::transform (:1127-1194) on the device, kept with the frame (borb_search_by_bow_batch reads
 * it).  borb_compute_bow is its one-frame case on host descriptors.  Host copies are optional (NULL tables: device only; a NULL
 * entry skips that frame's copy; n_bow / n_nodes may be NULL); capacities per frame as borb_compute_bow (n, n, n, n + 1, n).
 * 2 launches whatever n_frames, one synchronisation.  The vocabulary, the frames and the matcher must live on the same device; a
 * frame with 0 features or only stop words gets empty vectors (fv_start[0] = 0). */
BORB_API borb_status borb_frames_compute_bow(borb_matcher* m, borb_voc* v, borb_frame* const* frames, int n_frames, int levelsup,
                                             uint32_t* const* bow_word, double* const* bow_value, int32_t* n_bow,
                                             uint32_t* const* fv_node, int32_t* const* fv_start, uint32_t* const* fv_idx,
                                             int32_t* n_nodes);

/* ---------------------------------------------------------------- introspection -------------- */
/* Device time (CUDA events on the matcher's stream) of the kernels of the last borb_search_by_bow_db* call on this handle. */
BORB_API borb_status borb_matcher_set_timing(borb_matcher* m, int enable);
BORB_API borb_status borb_matcher_last_kernel_ms(borb_matcher* m, float* ms);
BORB_API borb_status borb_matcher_launch_count(const borb_matcher* m, uint64_t* n);
/* What the database holds for a live slot (read-only; tests compare blocks byte for byte).  counts4 = {nn FeatureVector nodes, m rows
 * (features inside the nodes), n features, n_bow BowVector words}; *block_bytes = the slot's device bytes.  Each non-NULL array gets:
 * node[nn], start[nn + 1], meta[2 m] (row records in FeatureVector order: feature | good-MapPoint flag << 16 | node index << 17, then
 * the bits of mvKeysUn[feature].angle), desc[m x 32] (row order), bow_word[n_bow], bow_value[n_bow], host_meta[2 m] (the host copy of
 * the row records), block[*block_bytes] (the whole device block, padding included).  Call with NULL arrays first to size them. */
BORB_API borb_status borb_debug_kfdb_read(borb_kfdb* db, int32_t slot, int32_t* counts4, uint64_t* block_bytes, uint32_t* node,
                                          int32_t* start, uint32_t* meta, uint8_t* desc, uint32_t* bow_word, double* bow_value,
                                          uint32_t* host_meta, uint8_t* block);
/* Per-stage intermediates of the last batch, for parity tests (tests/ compare each stage with the
 * oracle).  xys: (x, y, score) int32 triples in level pixel coordinates. */
BORB_API borb_status borb_debug_candidates(borb_extractor* e, int image, int level, int32_t* xys, int cap, int* n_out);
BORB_API borb_status borb_debug_selected(borb_extractor* e, int image, int level, int32_t* xys, int cap, int* n_out);
BORB_API borb_status borb_debug_blurred(borb_extractor* e, int image, int level, uint8_t* dst, int* w, int* h);
/* Ablation of fast_kernel for speed-of-light measurements (tools/fast_ablation.py; 0 = full kernel, the only mode that produces
 * keypoints; 1 = TMA tile load only, 2 = + packed reject pass, 3 = + exact scores without NMS / emit). */
BORB_API borb_status borb_debug_set_fast_mode(borb_extractor* e, int mode);
/* The rBRIEF tap order of the descriptor kernel (host table, no device needed): *n_bins orientation bins of 512 entries each,
 * entry = (x + 128) | (y + 128) << 8 | point << 16 for pattern point `point` (= 2 * test + 0/1) at (x, y); the first
 * min(cap, 512 * *n_bins) entries go to dst (may be NULL). */
BORB_API borb_status borb_debug_brief_slots(uint32_t* dst, int cap, int* n_bins);
/* Evaluates a device maths function on n host inputs (tests only): fn 0 sinf(a), 1 cosf(a), 2 fastAtan2(a = y, b = x) in degrees,
 * 3 logf(a), 4 PredictScale(a = max_distance, b = dist, log_scale, n_levels) -> int32.  out: n floats (int32 for fn 4).
 * These are the functions the descriptor kernel (0-2) and the projection searches (3-4) inline, compiled with them.  sinf/cosf
 * are defined for 0 <= a < 120 and logf for positive normal a (the inputs those kernels form).  Runs on the current device
 * on a stream of its own and returns when out is written; b may be NULL for fn 0, 1 and 3. */
BORB_API borb_status borb_debug_eval_math(int fn, const float* a, const float* b, int n, float log_scale, int n_levels, void* out);
/* Fills every buffer the library reuses or recycles with `byte` (0..255) before a call writes it, -1 (the default) stops: matcher
 * and vocabulary staging, arena and landing buffers, resident frame and keyframe blocks, the extractor workspace (DESIGN.md, "Buffer
 * reuse").  Process-wide; for tests that pin results to the unpoisoned run.  Other values give BORB_ERR_INVALID_ARG. */
BORB_API borb_status borb_debug_set_poison(int byte);
/* Kernel launches issued by this handle since creation (bench.py's gpu_launches). */
BORB_API borb_status borb_launch_count(const borb_extractor* e, uint64_t* n);
/* Device time (ms, CUDA events on the handle's stream) of each stage of the last batch:
 * [0] upload, [1] pyramid, [2] FAST/NMS, [3] quadtree, [4] blur, [5] orient+rBRIEF, [6] stereo, [7] download. */
BORB_API borb_status borb_stage_times(borb_extractor* e, float* ms8);
BORB_API borb_status borb_set_timing(borb_extractor* e, int enable);   /* also resets the accumulators */
/* Per-stage device time summed over every step completed (synced) since borb_set_timing(e,1); steps may
 * be queued back to back without host syncs (a ring of CUDA events on the handle's stream). */
BORB_API borb_status borb_stage_times_total(borb_extractor* e, double* ms8, uint64_t* steps);
/* The handle's cudaStream_t, so callers can bracket work with their own CUDA events. */
BORB_API borb_status borb_extractor_stream(borb_extractor* e, void** stream);

#ifdef __cplusplus
}
#endif
#endif /* BORB_H */
