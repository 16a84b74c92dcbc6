// A C++ host for N independent monocular camera streams on one GPU, written against the C ABI only (include/borb.h) — what a
// multi-camera / multi-agent front-end looks like once the per-frame work of ORB_SLAM2's Tracking thread (Frame::Frame:
// ExtractORB + UndistortKeyPoints + AssignFeaturesToGrid, then ORBmatcher::SearchByProjection against the local map) is batched
// over the streams the way libborb batches everything:
//
//   per tick:  borb_extract_batch            one launch sequence for the N images            (ORBextractor::operator() x N)
//              borb_frames_from_extractor    N device-resident frames, keypoints stay in HBM  (Frame constructor tail x N)
//              borb_search_by_projection_batch   one launch pair for the N matcher calls      (SearchByProjection x N)
//              borb_search_by_projection_last_batch   motion-model search of the N streams    (TrackWithMotionModel x N)
//              borb_frames_compute_bow       BowVector / FeatureVector of the N frames, kept in HBM   (Frame::ComputeBoW x N)
//              borb_search_by_bow_batch      reference-keyframe search of the N streams   (TrackReferenceKeyFrame x N)
//              (pose optimisation on the host)
//              borb_search_local_points_batch    isInFrustum + local-map search of the N streams   (SearchLocalPoints x N)
//   LocalMapping, per new keyframe:
//              borb_fuse_batch               the search part of Fuse(pKF, vpMapPoints) of the N streams (SearchInNeighbors x N)
//
// The program self-checks: the "local map" of every stream is made of that stream's own keypoints (projected where they were
// seen, with their own descriptors, predicted at their own octave), so SearchByProjection must give (almost) every point back to
// a feature — bar the few points whose twin at a neighbouring level wins the ratio test.  For the two Tracking-thread searches
// the keypoints are back-projected to a per-point depth with the identity pose: as the last frame's MapPoints they must land on
// their own features, and as world points (normal = viewing ray, distances that predict the keypoint's octave) as well.  For the
// reference-keyframe search every stream's frame is its own reference keyframe, every feature with a MapPoint: a feature can only
// match itself (a duplicate descriptor fails the ratio test), so every match[j] is j or -1.  The vocabulary is a small seeded tree.
// Each frame is also a keyframe into which the same back-projected points are fused: they must land on their own features.
// Build:  g++ -std=c++14 -Iinclude integration/example_multistream_host.cc orb_slam2_b200/libborb.so -Wl,-rpath,$PWD/orb_slam2_b200
// Exit code 0 = ran and checked, 3 = the library reported an error (e.g. no CUDA device: there is no CPU fallback).
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "borb.h"

#define CHECK(call)                                                                                     \
    do {                                                                                                \
        borb_status s_ = (call);                                                                        \
        if (s_ != BORB_OK) { std::printf("%s: %s (%s)\n", #call, borb_status_str(s_), borb_last_error()); return 3; } \
    } while (0)

// a textured synthetic frame: blobs and edges at several scales, different per stream
static void make_image(std::vector<uint8_t>& img, int w, int h, int stream) {
    img.resize((size_t)w * h);
    uint32_t rng = 1234567u + 7919u * (uint32_t)stream;
    auto next = [&]() { rng = rng * 1664525u + 1013904223u; return rng >> 8; };
    for (auto& p : img) p = 100;
    for (int k = 0; k < 900; k++) {
        const int cx = (int)(next() % (uint32_t)w), cy = (int)(next() % (uint32_t)h), r = 3 + (int)(next() % 14), v = (int)(next() % 256);
        const bool box = next() & 1;
        for (int y = cy - r; y <= cy + r; y++)
            for (int x = cx - r; x <= cx + r; x++) {
                if (x < 0 || y < 0 || x >= w || y >= h) continue;
                if (box || (x - cx) * (x - cx) + (y - cy) * (y - cy) <= r * r) img[(size_t)y * w + x] = (uint8_t)v;
            }
    }
}

// a seeded vocabulary (k = 10, depth 3: 1000 words, idf weights in [1, 2)); with levelsup 2 the FeatureVector has the 10 nodes of
// level 1, so every bucket holds many features
static borb_status make_vocabulary(borb_voc** out) {
    const int k = 10, L = 3;
    std::vector<int32_t> parent(1, 0);
    std::vector<uint8_t> leaf(1, 0), desc(32, 0);
    std::vector<double> weight(1, 0.0);
    uint32_t rng = 424242u;
    int first = 0, count = 1;                                // the nodes of the level above
    for (int l = 1; l <= L; l++) {
        const int start = (int)parent.size();
        for (int p = first; p < first + count; p++)
            for (int c = 0; c < k; c++) {
                parent.push_back(p);
                leaf.push_back(l == L ? 1 : 0);
                for (int b = 0; b < 32; b++) { rng = rng * 1664525u + 1013904223u; desc.push_back((uint8_t)(rng >> 24)); }
                weight.push_back(l == L ? 1.0 + (double)(parent.size() % 7) / 7.0 : 0.0);
            }
        first = start;
        count *= k;
    }
    return borb_voc_create(parent.data(), leaf.data(), desc.data(), weight.data(), (int)parent.size(), k, L, 0, out);
}

int main(int argc, char** argv) {
    const int N = argc > 1 ? std::atoi(argv[1]) : 8, W = 640, H = 480, ticks = 3;
    int ndev = 0;
    CHECK(borb_device_count(&ndev));
    borb_extractor_cfg cfg = {1000, 1.2f, 8, 20, 7};
    borb_extractor* ext = nullptr;
    borb_matcher* mat = nullptr;
    CHECK(borb_extractor_create(&cfg, 0, &ext));
    CHECK(borb_matcher_create(0, &mat));
    borb_voc* voc = nullptr;
    CHECK(make_vocabulary(&voc));
    int cap = 0;
    CHECK(borb_extractor_capacity(ext, W, H, &cap));
    std::vector<float> scale(cfg.n_levels);
    CHECK(borb_extractor_tables(ext, scale.data(), nullptr, nullptr, nullptr, nullptr));

    std::vector<std::vector<uint8_t> > imgs(N);
    std::vector<const uint8_t*> img_ptr(N);
    std::vector<borb_keypoint> kps((size_t)N * cap);
    std::vector<uint8_t> desc((size_t)N * cap * 32);
    std::vector<int> n_out(N);
    std::vector<int32_t> image_idx(N), n_keys(N);
    std::vector<borb_frame*> frames(N, nullptr);
    const borb_camera cam = {517.3f, 516.5f, 318.6f, 255.3f, 0.f, 0.f, 0.f, 0.f, 0.f, 40.f};      // k1 = 0: mvKeysUn = mvKeys
    float bounds[4];
    long total_points = 0, total_matches = 0, last_self = 0, local_self = 0, ref_self = 0, ref_other = 0, fuse_self = 0;
    const float log_scale = std::log(cfg.scale_factor);     // Frame::mfLogScaleFactor
    std::vector<float> inv_sigma2(cfg.n_levels);            // KeyFrame::mvInvLevelSigma2
    for (int l = 0; l < cfg.n_levels; l++) inv_sigma2[l] = 1.0f / (scale[l] * scale[l]);

    for (int t = 0; t < ticks; t++) {
        for (int i = 0; i < N; i++) { make_image(imgs[i], W, H, i + 100 * t); img_ptr[i] = imgs[i].data(); image_idx[i] = i; }
        // ---- N x ORBextractor::operator()
        CHECK(borb_extract_batch(ext, img_ptr.data(), N, W, H, W, kps.data(), desc.data(), cap, n_out.data()));
        for (int i = 0; i < N; i++) n_keys[i] = n_out[i];
        // ---- N x Frame constructor tail, resident
        CHECK(borb_frames_from_extractor(mat, ext, image_idx.data(), N, n_keys.data(), &cam, /*mode*/ 0, nullptr, 0, 1.f, 0, nullptr, nullptr,
                                         nullptr, 0, bounds, frames.data()));
        // ---- the streams' local maps (here: their own keypoints) and N x SearchByProjection in one call
        std::vector<std::vector<float> > px(N), py(N), pxr(N), vc(N);
        std::vector<std::vector<int32_t> > lvl(N), match(N);
        std::vector<borb_mappoint_view> mps(N);
        std::vector<borb_frame_view> fv(N);
        std::vector<int32_t*> match_ptr(N);
        std::vector<int32_t> n_matches(N);
        for (int i = 0; i < N; i++) {
            const int n = n_out[i];
            px[i].resize(n); py[i].resize(n); pxr[i].assign(n, -1.f); vc[i].assign(n, 1.f); lvl[i].resize(n); match[i].assign(n > 0 ? n : 1, -1);
            const borb_keypoint* k = &kps[(size_t)i * cap];
            for (int j = 0; j < n; j++) { px[i][j] = k[j].x; py[i][j] = k[j].y; lvl[i][j] = k[j].octave; }
            borb_mappoint_view& P = mps[i];
            P.n = n; P.proj_x = px[i].data(); P.proj_y = py[i].data(); P.proj_xr = pxr[i].data(); P.level = lvl[i].data();
            P.view_cos = vc[i].data(); P.desc = &desc[(size_t)i * cap * 32]; P.valid = nullptr; P.has_obs = nullptr;
            borb_frame_view& F = fv[i];
            F = borb_frame_view();
            F.resident = frames[i];                       // everything else of the view is taken from the resident frame
            match_ptr[i] = match[i].data();
        }
        CHECK(borb_search_by_projection_batch(mat, fv.data(), mps.data(), N, 3.0f, 0.8f, match_ptr.data(), n_matches.data()));
        // ---- the Tracking thread's two per-frame searches on the same resident frames: every keypoint back-projected to a
        //      depth z with the identity pose is the "last frame"'s MapPoint of that feature, and a local MapPoint as well
        std::vector<std::vector<float> > wpos(N), maxd(N), mind(N), nrm(N);
        std::vector<std::vector<int32_t> > state(N), lmatch(N);
        std::vector<std::vector<uint8_t> > in_view(N);
        std::vector<borb_last_frame_job> ljobs(N);
        std::vector<borb_local_points_job> pjobs(N);
        std::vector<int32_t> n_last(N), n_local(N);
        for (int i = 0; i < N; i++) {
            const int n = n_out[i];
            const borb_keypoint* k = &kps[(size_t)i * cap];
            wpos[i].resize((size_t)n * 3); maxd[i].resize(n); mind[i].resize(n); nrm[i].resize((size_t)n * 3);
            state[i].assign(n > 0 ? n : 1, -1); lmatch[i].assign(n > 0 ? n : 1, -1); in_view[i].assign(n > 0 ? n : 1, 0);
            for (int j = 0; j < n; j++) {
                const float z = 2.0f + 0.5f * (float)(j % 17);
                float* P = &wpos[i][(size_t)j * 3];
                P[0] = (k[j].x - cam.cx) * z / cam.fx; P[1] = (k[j].y - cam.cy) * z / cam.fy; P[2] = z;
                const float d = std::sqrt(P[0] * P[0] + P[1] * P[1] + P[2] * P[2]);
                for (int c = 0; c < 3; c++) nrm[i][(size_t)j * 3 + c] = P[c] / d;
                maxd[i][j] = d * scale[k[j].octave] * 0.95f;          // PredictScale: ceil(octave - 0.28) = octave
                mind[i][j] = maxd[i][j] / scale[cfg.n_levels - 1];
            }
            const float I34[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
            borb_last_frame_job& L = ljobs[i];
            L = borb_last_frame_job();
            L.cur.resident = frames[i];
            L.last.n = n; L.last.keys_un = k; L.last.world_pos = wpos[i].data(); L.last.desc = &desc[(size_t)i * cap * 32];
            for (int c = 0; c < 12; c++) L.Tcw[c] = I34[c];
            L.fx = cam.fx; L.fy = cam.fy; L.cx = cam.cx; L.cy = cam.cy; L.bf = cam.bf; L.th = 15.0f;
            L.state_cur = state[i].data();
            borb_local_points_job& J = pjobs[i];
            J = borb_local_points_job();
            J.frame.resident = frames[i];
            J.pts.n = n; J.pts.world_pos = wpos[i].data(); J.pts.desc = &desc[(size_t)i * cap * 32];
            J.pts.max_distance = maxd[i].data(); J.pts.min_distance = mind[i].data(); J.pts.normal = nrm[i].data();
            for (int c = 0; c < 12; c++) J.Tcw[c] = I34[c];
            J.fx = cam.fx; J.fy = cam.fy; J.cx = cam.cx; J.cy = cam.cy; J.mbf = cam.bf; J.log_scale_factor = log_scale; J.th = 1.0f;
            J.in_view = in_view[i].data(); J.match_feat = lmatch[i].data();
        }
        CHECK(borb_search_by_projection_last_batch(mat, ljobs.data(), N, 1, n_last.data()));
        // ---- the reference-keyframe search (Tracking::TrackReferenceKeyFrame, the fallback of a motion-model search that finds too
        //      few matches): the frames' BoW on the device, then SearchByBoW with each frame as its own reference keyframe (kf_frame:
        //      only has_mp crosses PCIe)
        CHECK(borb_frames_compute_bow(mat, voc, frames.data(), N, 2, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr));
        std::vector<borb_bow_job> bjobs(N);
        std::vector<std::vector<uint8_t> > has_mp(N);
        std::vector<std::vector<int32_t> > bmatch(N);
        std::vector<int32_t> n_ref(N);
        for (int i = 0; i < N; i++) {
            const int n = n_out[i];
            has_mp[i].assign(n > 0 ? n : 1, 1);
            bmatch[i].assign(n > 0 ? n : 1, -1);
            borb_bow_job& B = bjobs[i];
            B = borb_bow_job();
            B.frame = frames[i];
            B.kf_frame = frames[i];
            B.kf.has_mp = has_mp[i].data();
            B.match = bmatch[i].data();
        }
        CHECK(borb_search_by_bow_batch(mat, bjobs.data(), N, 0.7f, 1, n_ref.data()));
        CHECK(borb_search_local_points_batch(mat, pjobs.data(), N, 0.5f, 0.8f, n_local.data()));
        // ---- LocalMapping::SearchInNeighbors: the frame as a keyframe, its back-projected keypoints as the MapPoints to fuse.  The
        //      Fuse calls of one keyframe's targets depend on each other (MapPoint::Replace); those of different streams do not
        std::vector<borb_fuse_job> fjobs(N);
        std::vector<std::vector<int32_t> > fbest(N);
        std::vector<int32_t> n_fused(N);
        for (int i = 0; i < N; i++) {
            fbest[i].assign(n_out[i] > 0 ? n_out[i] : 1, -1);
            borb_fuse_job& Fj = fjobs[i];
            Fj = borb_fuse_job();
            Fj.kf.resident = frames[i];
            Fj.inv_level_sigma2 = inv_sigma2.data();
            Fj.pts = pjobs[i].pts;
            for (int c = 0; c < 12; c++) Fj.Tcw[c] = pjobs[i].Tcw[c];
            Fj.fx = cam.fx; Fj.fy = cam.fy; Fj.cx = cam.cx; Fj.cy = cam.cy; Fj.bf = cam.bf; Fj.log_scale_factor = log_scale; Fj.th = 3.0f;
            Fj.best_idx = fbest[i].data();
        }
        CHECK(borb_fuse_batch(mat, fjobs.data(), N, n_fused.data()));
        for (int i = 0; i < N; i++) {
            total_points += n_out[i]; total_matches += n_matches[i];
            int self = 0, sl = 0, sp = 0, sr = 0, sf = 0;
            for (int j = 0; j < n_out[i]; j++) {
                self += match[i][j] == j; sl += state[i][j] == j; sp += lmatch[i][j] == j; sr += bmatch[i][j] == j; sf += fbest[i][j] == j;
                ref_other += bmatch[i][j] != j && bmatch[i][j] != -1;
            }
            last_self += sl; local_self += sp; ref_self += sr; fuse_self += sf;
            std::printf("tick %d stream %d: %d keypoints, %d matches (%d to themselves); motion model %d (%d); reference keyframe %d (%d); "
                        "local map %d (%d); fuse %d (%d)\n", t, i, n_out[i], n_matches[i], self, n_last[i], sl, n_ref[i], sr, n_local[i], sp,
                        n_fused[i], sf);
            CHECK(borb_frame_destroy(frames[i]));
            frames[i] = nullptr;
        }
    }
    CHECK(borb_voc_destroy(voc));
    CHECK(borb_matcher_destroy(mat));
    CHECK(borb_extractor_destroy(ext));
    std::printf("%ld points, %ld matched\n", total_points, total_matches);
    std::printf("motion-model search: %ld of %ld features matched to their own last-frame point\n", last_self, total_points);
    std::printf("reference-keyframe search: %ld of %ld features matched to themselves, %ld elsewhere\n", ref_self, total_points, ref_other);
    std::printf("local-map search: %ld of %ld points matched to their own feature\n", local_self, total_points);
    std::printf("fuse: %ld of %ld points fused onto their own feature\n", fuse_self, total_points);
    if (total_points < 100L * N * ticks || total_matches < total_points * 8 / 10 || last_self < total_points * 8 / 10 ||
        ref_self < total_points * 8 / 10 || ref_other != 0 || local_self < total_points * 8 / 10 || fuse_self < total_points * 8 / 10) {
        std::printf("self-check failed\n");
        return 1;
    }
    std::printf("ok\n");
    return 0;
}
