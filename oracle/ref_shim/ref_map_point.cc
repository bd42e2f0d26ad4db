// oracle/ref_shim/ref_map_point.cc -- extern "C" driver of the reference's OWN MapPoint::UpdateNormalAndDepth
// (src/MapPoint.cc:273-312) on scripted maps (TEST INFRASTRUCTURE ONLY).
//
// Built by oracle/normal_depth.py into oracle/_ref/libref_map_point.so next to, and linked against, libref_orbslam.so: the
// MapPoint / KeyFrame / Frame code that runs is the reference's, compiled unmodified there.  A handle owns one map: keyframes
// built from a pose and keypoint octaves, map points with a reference keyframe and observations.  Scripts set a point's
// position with SetWorldPos, call UpdateNormalAndDepth, and read back GetNormal / GetMin/MaxDistanceInvariance and every
// keyframe's GetCameraCenter -- the centres are the inputs the oracle and the device entries take.
// Also the shim self-test hook of `x + y*beta` (the MatExpr the reference's `normal + normali/cv::norm(normali)` builds).
#include <opencv2/core/core.hpp>   // every standard header first: the access hack below must not reach libstdc++
#include <boost/thread.hpp>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <new>
#include <vector>
#define protected public   // the driver reads the scale table and marks keyframes bad directly
#define private public
#include "Frame.h"
#include "KeyFrame.h"
#include "KeyFrameDatabase.h"
#include "Map.h"
#include "MapPoint.h"
#undef protected
#undef private

using namespace ORB_SLAM;

namespace {

// KeyFrames and MapPoints in one arena in creation order: mObservations is a std::map keyed by KeyFrame*, so with
// addresses ascending in creation order its iteration order is the order the script created the keyframes in.
struct NdMap {
    ORBVocabulary voc;
    Map map;
    KeyFrameDatabase db;
    std::vector<KeyFrame *> kfs;
    std::vector<MapPoint *> mps;
    char *arena;
    size_t used, cap;
    NdMap() : db(voc), arena(NULL), used(0), cap((size_t)1 << 30) { arena = static_cast<char *>(std::malloc(cap)); }
    void *alloc(size_t bytes) {
        used = (used + 63) / 64 * 64;
        if (!arena || used + bytes > cap) { std::fprintf(stderr, "ref_map_point: arena exhausted\n"); std::abort(); }
        void *p = arena + used;
        used += bytes;
        return p;
    }
    ~NdMap() {
        for (size_t i = 0; i < mps.size(); i++) mps[i]->~MapPoint();
        for (size_t i = 0; i < kfs.size(); i++) kfs[i]->~KeyFrame();
        std::free(arena);
    }
};

cv::Mat point3(const float *p) {
    cv::Mat m(3, 1, CV_32F);
    for (int k = 0; k < 3; k++) m.at<float>(k) = p[k];
    return m;
}

}  // namespace

extern "C" {

void *ref_nd_create() { return new NdMap(); }
void ref_nd_free(void *h) { delete static_cast<NdMap *>(h); }

// KeyFrame(Frame&, Map*, KeyFrameDatabase*) (KeyFrame.cc:30-54) from a Frame holding n keypoints with the given octaves,
// the scale table of Frame.cc:90-103 (mvScaleFactors[i] = mvScaleFactors[i-1]*mfScaleFactor) and pose Tcw = [R|t] (3x4
// row-major).  bad != 0 marks the keyframe isBad().  With nlevels == 1 the reference's GetScaleFactor() reads
// mvScaleFactors[1], one past the table: the table's storage is given a second element holding scale_factor, so that read
// is defined and returns what GetScaleFactor() returns for nlevels >= 2.  Returns the keyframe's id in this map.
int ref_nd_add_keyframe(void *h, const float *Tcw12, const int *octaves, int n, float scale_factor, int nlevels, int bad) {
    NdMap &M = *static_cast<NdMap *>(h);
    Frame F;
    F.mpORBvocabulary = &M.voc;
    F.mpORBextractor = NULL;
    F.mTimeStamp = 0;
    F.mK = cv::Mat::eye(3, 3, CV_32F);
    F.N = n;
    F.mvKeys.resize(n);
    for (int i = 0; i < n; i++) F.mvKeys[i].octave = octaves[i];
    F.mvKeysUn = F.mvKeys;
    F.mvpMapPoints = std::vector<MapPoint *>(n, static_cast<MapPoint *>(NULL));
    F.mvbOutlier = std::vector<bool>(n, false);
    F.mnId = Frame::nNextId++;
    F.mnScaleLevels = nlevels;
    F.mfScaleFactor = scale_factor;
    F.mvScaleFactors.resize(nlevels);
    F.mvLevelSigma2.resize(nlevels);
    F.mvInvLevelSigma2.resize(nlevels);
    F.mvScaleFactors[0] = 1.0f;
    for (int i = 1; i < nlevels; i++) F.mvScaleFactors[i] = F.mvScaleFactors[i - 1] * F.mfScaleFactor;
    for (int i = 0; i < nlevels; i++) {
        F.mvLevelSigma2[i] = F.mvScaleFactors[i] * F.mvScaleFactors[i];
        F.mvInvLevelSigma2[i] = 1 / F.mvLevelSigma2[i];
    }
    F.mTcw = cv::Mat::eye(4, 4, CV_32F);
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 4; c++) F.mTcw.at<float>(r, c) = Tcw12[4 * r + c];
    KeyFrame *kf = new (M.alloc(sizeof(KeyFrame))) KeyFrame(F, &M.map, &M.db);
    if (nlevels == 1) {
        std::vector<float> t(2);
        t[0] = kf->mvScaleFactors[0];
        t[1] = scale_factor;
        t.resize(1);   // size 1, storage for 2
        kf->mvScaleFactors.swap(t);
    }
    kf->mbBad = bad != 0;
    M.kfs.push_back(kf);
    return (int)M.kfs.size() - 1;
}

// GetCameraCenter(), GetScaleFactor() and GetScaleFactor(l) for l < GetScaleLevels() of keyframe kf
void ref_nd_keyframe(void *h, int kf, float *center3, float *scale_factor, float *scale_factors) {
    KeyFrame *K = static_cast<NdMap *>(h)->kfs[(size_t)kf];
    cv::Mat c = K->GetCameraCenter();
    for (int k = 0; k < 3; k++) center3[k] = c.at<float>(k);
    *scale_factor = K->GetScaleFactor();
    for (int l = 0; l < K->GetScaleLevels(); l++) scale_factors[l] = K->GetScaleFactor(l);
}

// MapPoint(Pos, pRefKF, pMap) (MapPoint.cc:31-39); returns the point's id in this map
int ref_nd_add_point(void *h, const float *pos3, int ref_kf) {
    NdMap &M = *static_cast<NdMap *>(h);
    MapPoint *p = new (M.alloc(sizeof(MapPoint))) MapPoint(point3(pos3), M.kfs[(size_t)ref_kf], &M.map);
    M.mps.push_back(p);
    return (int)M.mps.size() - 1;
}
void ref_nd_add_observation(void *h, int mp, int kf, int idx) {
    NdMap &M = *static_cast<NdMap *>(h);
    M.mps[(size_t)mp]->AddObservation(M.kfs[(size_t)kf], (size_t)idx);
}
void ref_nd_set_point_bad(void *h, int mp) { static_cast<NdMap *>(h)->mps[(size_t)mp]->mbBad = true; }
void ref_nd_set_world_pos(void *h, int mp, const float *pos3) { static_cast<NdMap *>(h)->mps[(size_t)mp]->SetWorldPos(point3(pos3)); }

// the reference's own call, then its getters
void ref_nd_update(void *h, int mp) { static_cast<NdMap *>(h)->mps[(size_t)mp]->UpdateNormalAndDepth(); }
void ref_nd_get(void *h, int mp, float *normal3, float *min_dist, float *max_dist) {
    MapPoint *p = static_cast<NdMap *>(h)->mps[(size_t)mp];
    cv::Mat n = p->GetNormal();
    for (int k = 0; k < 3; k++) normal3[k] = n.at<float>(k);
    *min_dist = p->GetMinDistanceInvariance();
    *max_dist = p->GetMaxDistanceInvariance();
}

// the point's observations in mObservations iteration order as (keyframe id, feature index); returns their number
int ref_nd_observations(void *h, int mp, int *kf_ids, int *idx, int cap) {
    NdMap &M = *static_cast<NdMap *>(h);
    const std::map<KeyFrame *, size_t> obs = M.mps[(size_t)mp]->GetObservations();
    int n = 0;
    for (std::map<KeyFrame *, size_t>::const_iterator it = obs.begin(); it != obs.end(); ++it, ++n) {
        if (n >= cap) continue;
        kf_ids[n] = -1;
        for (size_t k = 0; k < M.kfs.size(); k++) if (M.kfs[k] == it->first) kf_ids[n] = (int)k;
        idx[n] = (int)it->second;
    }
    return n;
}

// shim self-test hook: out = x + y*beta for n x 1 float columns, the MatExpr (MatOp_AddEx with beta) the shim evaluates for
// `normal + normali/cv::norm(normali)`; tests pin it against cv2.scaleAdd(y, beta, x)
void ref_shim_scale_add(const float *x, const float *y, double beta, int n, float *out) {
    cv::Mat X(n, 1, CV_32F, const_cast<float *>(x)), Y(n, 1, CV_32F, const_cast<float *>(y));
    cv::Mat r = X + Y * beta;
    for (int i = 0; i < n; i++) out[i] = r.at<float>(i);
}

}  // extern "C"
