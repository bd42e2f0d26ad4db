// oracle/ref_shim/ref_covis.cc -- extern "C" driver of the reference's OWN covisibility graph (KeyFrame::UpdateConnections,
// AddConnection, UpdateBestCovisibles, EraseConnection, SetBadFlag; src/KeyFrame.cc) on scripted maps (TEST INFRASTRUCTURE
// ONLY).
//
// Included by ref_observations.cc (oracle/_ref/libref_drivers.so, linked against libref_orbslam.so): the KeyFrame /
// MapPoint / Map code that runs is the reference's, compiled unmodified there.  A handle owns one map whose keyframes and
// points sit in one arena in creation order, so every std::map keyed by KeyFrame* iterates in creation order and every
// pointer tie falls the way creation order does: the creation index is the order key the oracle and the device take.
// ref_cv_set_kf_order places the keyframes in a given order instead, so that any key map the oracle and the device take
// has the reference's decision beside it: the key of keyframe k ranks rank[k] among the keys.
// Observations are made with MapPoint::AddObservation + KeyFrame::AddMapPoint.  The getters read back the graph and the
// inputs of the next call (every keyframe's mvpMapPoints, every point's observations and isBad()).
#include <opencv2/core/core.hpp>   // every standard header first: the access hack below must not reach libstdc++
#include <boost/thread.hpp>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <new>
#include <set>
#include <vector>
#define protected public   // the driver resets the id counter and reads mpParent directly
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

struct CvMap {
    ORBVocabulary voc;
    Map map;
    KeyFrameDatabase db;
    std::vector<KeyFrame *> kfs;
    std::vector<MapPoint *> mps;
    std::map<const KeyFrame *, int> kf_index;
    std::map<const MapPoint *, int> mp_index;
    char *arena;
    size_t used, cap;
    // ref_cv_set_kf_order: keyframe k goes to kf_region + kf_rank[k] * sizeof(KeyFrame); empty: the arena in creation order
    char *kf_region;
    std::vector<int> kf_rank;
    CvMap() : db(voc), arena(NULL), used(0), cap((size_t)4 << 30), kf_region(NULL) { arena = static_cast<char *>(std::malloc(cap)); }
    void *alloc(size_t bytes) {
        used = (used + 63) / 64 * 64;
        if (!arena || used + bytes > cap) { std::fprintf(stderr, "ref_covis: arena exhausted\n"); std::abort(); }
        void *p = arena + used;
        used += bytes;
        return p;
    }
    int kf_id(const KeyFrame *k) const {
        std::map<const KeyFrame *, int>::const_iterator it = kf_index.find(k);
        return it == kf_index.end() ? -2 : it->second;
    }
    ~CvMap() {
        for (size_t i = 0; i < mps.size(); i++) mps[i]->~MapPoint();
        for (size_t i = 0; i < kfs.size(); i++) kfs[i]->~KeyFrame();
        std::free(arena);
    }
};

}  // namespace

extern "C" {

// a new map; its first keyframe gets mnId 0
void *ref_cv_create() {
    KeyFrame::nNextId = 0;
    return new CvMap();
}
void ref_cv_free(void *h) { delete static_cast<CvMap *>(h); }

// Before the first keyframe: keyframe k (k < n) is placed at rank[k] in one region of n KeyFrames, so pointer order, and
// with it every std::map keyed by KeyFrame* and every pointer tie, is rank order instead of creation order.  rank is a
// permutation of 0 .. n-1.  Returns 0, or -1 (nothing changed) when a keyframe exists or rank is not a permutation.
int ref_cv_set_kf_order(void *h, int n, const int *rank) {
    CvMap &M = *static_cast<CvMap *>(h);
    if (!M.kfs.empty() || n < 1) return -1;
    std::vector<char> seen((size_t)n, 0);
    for (int k = 0; k < n; k++) {
        if (rank[k] < 0 || rank[k] >= n || seen[(size_t)rank[k]]) return -1;
        seen[(size_t)rank[k]] = 1;
    }
    M.kf_rank.assign(rank, rank + n);
    M.kf_region = static_cast<char *>(M.alloc(sizeof(KeyFrame) * (size_t)n));
    return 0;
}

// KeyFrame(Frame&, Map*, KeyFrameDatabase*) from a Frame of n features without map points, identity pose
int ref_cv_add_keyframe(void *h, int n) {
    CvMap &M = *static_cast<CvMap *>(h);
    Frame F;
    F.mpORBvocabulary = &M.voc;
    F.mpORBextractor = NULL;
    F.mTimeStamp = 0;
    F.mK = cv::Mat::eye(3, 3, CV_32F);
    F.N = n;
    F.mvKeys.resize(n);
    F.mvKeysUn = F.mvKeys;
    F.mvpMapPoints = std::vector<MapPoint *>(n, static_cast<MapPoint *>(NULL));
    F.mvbOutlier = std::vector<bool>(n, false);
    F.mnId = Frame::nNextId++;
    F.mnScaleLevels = 1;
    F.mfScaleFactor = 1.2f;
    F.mvScaleFactors.assign(1, 1.0f);
    F.mvLevelSigma2.assign(1, 1.0f);
    F.mvInvLevelSigma2.assign(1, 1.0f);
    F.mTcw = cv::Mat::eye(4, 4, CV_32F);
    const size_t k = M.kfs.size();
    if (M.kf_region && k >= M.kf_rank.size()) {
        std::fprintf(stderr, "ref_covis: keyframe %zu has no place in the order of ref_cv_set_kf_order\n", k);
        std::abort();
    }
    void *at = M.kf_region ? M.kf_region + (size_t)M.kf_rank[k] * sizeof(KeyFrame) : M.alloc(sizeof(KeyFrame));
    KeyFrame *kf = new (at) KeyFrame(F, &M.map, &M.db);
    M.kf_index[kf] = (int)M.kfs.size();
    M.kfs.push_back(kf);
    return (int)M.kfs.size() - 1;
}

// MapPoint(Pos, pRefKF, pMap) at (0, 0, 1)
int ref_cv_add_point(void *h, int ref_kf) {
    CvMap &M = *static_cast<CvMap *>(h);
    cv::Mat pos = cv::Mat::zeros(3, 1, CV_32F);
    pos.at<float>(2) = 1.f;
    MapPoint *p = new (M.alloc(sizeof(MapPoint))) MapPoint(pos, M.kfs[(size_t)ref_kf], &M.map);
    M.mp_index[p] = (int)M.mps.size();
    M.mps.push_back(p);
    return (int)M.mps.size() - 1;
}

// pMP->AddObservation(pKF, idx); pKF->AddMapPoint(pMP, idx)
void ref_cv_observe(void *h, int mp, int kf, int idx) {
    CvMap &M = *static_cast<CvMap *>(h);
    M.mps[(size_t)mp]->AddObservation(M.kfs[(size_t)kf], (size_t)idx);
    M.kfs[(size_t)kf]->AddMapPoint(M.mps[(size_t)mp], (size_t)idx);
}

// ref_cv_observe for n (point, keyframe, feature) triples in order
void ref_cv_observe_many(void *h, int n, const int *mp, const int *kf, const int *idx) {
    for (int i = 0; i < n; i++) ref_cv_observe(h, mp[i], kf[i], idx[i]);
}
// n points at once (ref_cv_add_point), reference keyframes ref_kf[i]; returns the first one's index
int ref_cv_add_points(void *h, int n, const int *ref_kf) {
    const int first = (int)static_cast<CvMap *>(h)->mps.size();
    for (int i = 0; i < n; i++) ref_cv_add_point(h, ref_kf[i]);
    return first;
}

// the reference's own calls
void ref_cv_update(void *h, int kf) { static_cast<CvMap *>(h)->kfs[(size_t)kf]->UpdateConnections(); }
void ref_cv_set_bad_keyframe(void *h, int kf) { static_cast<CvMap *>(h)->kfs[(size_t)kf]->SetBadFlag(); }
void ref_cv_set_bad_point(void *h, int mp) { static_cast<CvMap *>(h)->mps[(size_t)mp]->SetBadFlag(); }
void ref_cv_erase_match(void *h, int kf, int idx) { static_cast<CvMap *>(h)->kfs[(size_t)kf]->EraseMapPointMatch((size_t)idx); }

// GetVectorCovisibleKeyFrames() and mvOrderedWeights (creation indices); returns the list's length
int ref_cv_ordered(void *h, int kf, int *ids, int *weights, int cap) {
    CvMap &M = *static_cast<CvMap *>(h);
    KeyFrame *K = M.kfs[(size_t)kf];
    const std::vector<KeyFrame *> v = K->GetVectorCovisibleKeyFrames();
    const int n = (int)v.size();
    for (int i = 0; i < n && i < cap; i++) {
        ids[i] = M.kf_id(v[i]);
        weights[i] = i < (int)K->mvOrderedWeights.size() ? K->mvOrderedWeights[i] : -1;
    }
    return n;
}

// mConnectedKeyFrameWeights in map order; returns its size
int ref_cv_weights(void *h, int kf, int *ids, int *weights, int cap) {
    CvMap &M = *static_cast<CvMap *>(h);
    KeyFrame *K = M.kfs[(size_t)kf];
    int n = 0;
    for (std::map<KeyFrame *, int>::const_iterator it = K->mConnectedKeyFrameWeights.begin(); it != K->mConnectedKeyFrameWeights.end();
         ++it, ++n)
        if (n < cap) { ids[n] = M.kf_id(it->first); weights[n] = it->second; }
    return n;
}

// GetParent() as a creation index, -1 for NULL
int ref_cv_parent(void *h, int kf) {
    CvMap &M = *static_cast<CvMap *>(h);
    KeyFrame *p = M.kfs[(size_t)kf]->GetParent();
    return p ? M.kf_id(p) : -1;
}
int ref_cv_keyframe_bad(void *h, int kf) { return static_cast<CvMap *>(h)->kfs[(size_t)kf]->isBad() ? 1 : 0; }
long ref_cv_keyframe_mnid(void *h, int kf) { return (long)static_cast<CvMap *>(h)->kfs[(size_t)kf]->mnId; }

// GetMapPointMatches() of keyframe kf as point indices: -1 where NULL or isBad(); returns the number of features
int ref_cv_matches(void *h, int kf, int *mp, int cap) {
    CvMap &M = *static_cast<CvMap *>(h);
    const std::vector<MapPoint *> v = M.kfs[(size_t)kf]->GetMapPointMatches();
    const int n = (int)v.size();
    for (int i = 0; i < n && i < cap; i++) {
        if (!v[i] || v[i]->isBad()) { mp[i] = -1; continue; }
        std::map<const MapPoint *, int>::const_iterator it = M.mp_index.find(v[i]);
        mp[i] = it == M.mp_index.end() ? -2 : it->second;
    }
    return n;
}

// the point's observations in mObservations order as (keyframe creation index, feature index); returns their number
int ref_cv_observations(void *h, int mp, int *kf_ids, int *idx, int cap) {
    CvMap &M = *static_cast<CvMap *>(h);
    const std::map<KeyFrame *, size_t> obs = M.mps[(size_t)mp]->GetObservations();
    int n = 0;
    for (std::map<KeyFrame *, size_t>::const_iterator it = obs.begin(); it != obs.end(); ++it, ++n)
        if (n < cap) { kf_ids[n] = M.kf_id(it->first); idx[n] = (int)it->second; }
    return n;
}
int ref_cv_point_bad(void *h, int mp) { return static_cast<CvMap *>(h)->mps[(size_t)mp]->isBad() ? 1 : 0; }

}  // extern "C"
