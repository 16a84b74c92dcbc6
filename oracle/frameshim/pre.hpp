// TEST INFRASTRUCTURE ONLY (oracle/).  Force-included (-include) ahead of /root/reference/src/Frame.cc so that it compiles
// VERBATIM against the reference's REAL include/Frame.h (oracle/Makefile target `ref`, libraries _ref/libframeref.so and _ref/libframector.so): the include
// guards of the headers Frame.h pulls in are pre-defined, and plain-data stand-ins with the members Frame.cc touches take
// their place.  Frame.cc then provides, unmodified: the three constructors (:61-228), ComputeStereoMatches (:466-640),
// AssignFeaturesToGrid / PosInGrid / GetFeaturesInArea (:230-245, :327-392) and isInFrustum (:269-325).
#pragma once
#define MAPPOINT_H
#define KEYFRAME_H
#define ORBVOCABULARY_H
#define ORBEXTRACTOR_H
#define CONVERTER_H
#define ORBMATCHER_H

#include <algorithm>
#include <cassert>
#include <climits>
#include <cmath>
#include <list>
#include <map>
#include <mutex>
#include <set>
#include <sstream>
#include <thread>
#include <vector>

#include <opencv2/core/core.hpp>

using namespace std;        // the reference's headers rely on it (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:36)

namespace DBoW2 { class BowVector; class FeatureVector; }

namespace ORB_SLAM2 {

class Frame;
class KeyFrame {};

class MapPoint {
public:
    cv::Mat mWorldPos, mNormalVector;
    float mfMaxDistance = 0, mfMinDistance = 0;
    float mTrackProjX = 0, mTrackProjY = 0, mTrackProjXR = 0, mTrackViewCos = 0;
    bool mbTrackInView = false;
    int mnTrackScaleLevel = 0;
    cv::Mat GetWorldPos() { return mWorldPos.clone(); }
    cv::Mat GetNormal() { return mNormalVector.clone(); }
    float GetMinDistanceInvariance() { return 0.8f * mfMinDistance; }      // src/MapPoint.cc:373-377
    float GetMaxDistanceInvariance() { return 1.2f * mfMaxDistance; }      // :379-383
    int PredictScale(const float& currentDist, Frame* pF);                 // :402-417, defined in frameref_wrap.cpp
};

// The extractor of a Frame constructor (framector_run in framector_wrap.cpp): operator() replays the keypoints and descriptors
// that the verbatim src/ORBextractor.cc (liborbref.so) found on the same image, and the pyramid and scale tables are that run's.  As the real
// extractor does (ORBextractor.cc:1065-1068), an image without keypoints gives an empty descriptor matrix.
class ORBextractor {
public:
    std::vector<cv::Mat> mvImagePyramid;
    std::vector<float> mvScaleFactor, mvInvScaleFactor, mvLevelSigma2, mvInvLevelSigma2;
    float scaleFactor = 1.2f;                       // ORBextractor::scaleFactor (a double set from the float argument)
    std::vector<cv::KeyPoint> replayKeys;
    cv::Mat replayDesc;
    void operator()(const cv::Mat&, const cv::Mat&, std::vector<cv::KeyPoint>& keys, cv::Mat& desc) {
        keys = replayKeys;
        if (replayKeys.empty()) desc.release(); else desc = replayDesc.clone();
    }
    int GetLevels() { return (int)mvScaleFactor.size(); }
    float GetScaleFactor() { return scaleFactor; }
    std::vector<float> GetScaleFactors() { return mvScaleFactor; }
    std::vector<float> GetInverseScaleFactors() { return mvInvScaleFactor; }
    std::vector<float> GetScaleSigmaSquares() { return mvLevelSigma2; }
    std::vector<float> GetInverseScaleSigmaSquares() { return mvInvLevelSigma2; }
};

class ORBVocabulary {
public:
    template <class B, class Fv> void transform(const std::vector<cv::Mat>&, B&, Fv&, int) {}   // never run by the oracle
};

class Converter {
public:
    static std::vector<cv::Mat> toDescriptorVector(const cv::Mat&) { return std::vector<cv::Mat>(); }
};

class ORBmatcher {        // Frame::ComputeStereoMatches uses the two thresholds and the distance (src/Frame.cc:471,522)
public:
    static const int TH_LOW = 50, TH_HIGH = 100;                          // src/ORBmatcher.cc:37-38
    static int DescriptorDistance(const cv::Mat& a, const cv::Mat& b) {   // a10, pinned on its own in libmatchref
        const uint32_t* pa = a.ptr<uint32_t>();
        const uint32_t* pb = b.ptr<uint32_t>();
        int d = 0;
        for (int i = 0; i < 8; i++) d += __builtin_popcount(pa[i] ^ pb[i]);
        return d;
    }
};

}  // namespace ORB_SLAM2

// AssignFeaturesToGrid is a private member of the reference's Frame; the wrapper has to call it.  Defined here, after every
// standard header has been seen (libstdc++ does not survive the redefinition), and before Frame.h is.
#define private public
