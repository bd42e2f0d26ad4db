// oracle/ref_shim/ref_local_map.cc -- the driver of ref_observations.cc with the reference's own, unmodified
// Tracking::UpdateReference (src/Tracking.cc:728-839: UpdateReferenceKeyFrames and UpdateReferencePoints) on scripted maps
// (TEST INFRASTRUCTURE ONLY).
//
// Built by oracle/local_map.py into oracle/_ref/libref_local_map.so together with the reference's src/Tracking.cc, both
// against the stand-in headers of oracle/ref_shim_tr/ and oracle/ref_shim_lm/ (ROS, tf, cv_bridge and g2o names that
// Tracking.h and Tracking.cc pull in), linked against libref_orbslam.so.  One Tracking per map is made by the reference's
// constructor (its settings file is the fixed table of ref_tr_prelude.h).  A call builds mCurrentFrame as
// ref_cv_add_keyframe builds its Frames, with a fresh Frame::nNextId (so no stamp of an earlier call matches) and the
// scripted mvpMapPoints, calls UpdateReference() and reads back mvpLocalKeyFrames, mpReferenceKF, mvpLocalMapPoints and the
// frame's cells.  The Tracking methods the driver never calls reach the bodies below, which abort.
#include <chrono>

#include "ref_observations.cc"

typedef struct RefTrCvMat CvMat;   // as in ref_tr_prelude.h: PnPsolver.h's private members name the OpenCV 1 C matrix

#define protected public   // mCurrentFrame, the local map and UpdateReference() are protected
#include "Tracking.h"
#include "Optimizer.h"
#include "PnPsolver.h"
#undef protected

namespace ORB_SLAM {
namespace {
[[noreturn]] void ref_lm_not_linked(const char *what) {
    std::fprintf(stderr, "ref_local_map: %s is not linked\n", what);
    std::abort();
}
}  // namespace
Initializer::Initializer(const Frame &, float, int) { ref_lm_not_linked("Initializer"); }
bool Initializer::Initialize(const Frame &, const std::vector<int> &, cv::Mat &, cv::Mat &, std::vector<cv::Point3f> &,
                             std::vector<bool> &) {
    ref_lm_not_linked("Initializer::Initialize");
}
bool LocalMapping::AcceptKeyFrames() { ref_lm_not_linked("LocalMapping"); }
void LocalMapping::InsertKeyFrame(KeyFrame *) { ref_lm_not_linked("LocalMapping"); }
void LocalMapping::InterruptBA() { ref_lm_not_linked("LocalMapping"); }
void LocalMapping::RequestReset() { ref_lm_not_linked("LocalMapping"); }
bool LocalMapping::isStopped() { ref_lm_not_linked("LocalMapping"); }
bool LocalMapping::stopRequested() { ref_lm_not_linked("LocalMapping"); }
void LoopClosing::RequestReset() { ref_lm_not_linked("LoopClosing"); }
void MapPublisher::SetCurrentCameraPose(const cv::Mat &) { ref_lm_not_linked("MapPublisher"); }
void Optimizer::GlobalBundleAdjustemnt(Map *, int, bool *) { ref_lm_not_linked("Optimizer::GlobalBundleAdjustemnt"); }
int Optimizer::PoseOptimization(Frame *) { ref_lm_not_linked("Optimizer::PoseOptimization"); }
PnPsolver::PnPsolver(const Frame &, const std::vector<MapPoint *> &) { ref_lm_not_linked("PnPsolver"); }
void PnPsolver::SetRansacParameters(double, int, int, int, float, float) { ref_lm_not_linked("PnPsolver"); }
cv::Mat PnPsolver::iterate(int, bool &, std::vector<bool> &, int &) { ref_lm_not_linked("PnPsolver"); }
}  // namespace ORB_SLAM

namespace {
std::map<void *, Tracking *> g_tracking;   // one Tracking per map handle
}

extern "C" {

// the map and its Tracking
void ref_lm_free(void *h) {
    std::map<void *, Tracking *>::iterator it = g_tracking.find(h);
    if (it != g_tracking.end()) {
        delete it->second->mpORBextractor;
        delete it->second->mpIniORBextractor;
        delete it->second;
        g_tracking.erase(it);
    }
    ref_cv_free(h);
}

// SetNotErase() then SetBadFlag(): the keyframe keeps mbNotErase and gets mbToBeErased, and is not bad (KeyFrame.cc:503-510)
void ref_lm_to_be_erased(void *h, int kf) {
    KeyFrame *K = static_cast<CvMap *>(h)->kfs[(size_t)kf];
    K->SetNotErase();
    K->SetBadFlag();
}

// UpdateReference() for a frame of n features whose mvpMapPoints are frame_mp (point indices, -1 = NULL).  Outputs:
// frame_mp the frame's cells afterwards; kf_ids[0 .. return value) mvpLocalKeyFrames as creation indices (at most cap_kf
// written); *ref_kf mpReferenceKF (-1 for NULL); points[0 .. *npoints) mvpLocalMapPoints (at most cap_pts written);
// *ns the call's wall time in nanoseconds.
int ref_lm_update_reference(void *h, int n, int *frame_mp, int *kf_ids, int cap_kf, int *ref_kf, int *points, int cap_pts,
                            int *npoints, long long *ns) {
    CvMap &M = *static_cast<CvMap *>(h);
    Tracking *&T = g_tracking[h];
    if (!T) T = new Tracking(&M.voc, NULL, NULL, &M.map, std::string());
    Frame F;
    F.mpORBvocabulary = &M.voc;
    F.mpORBextractor = NULL;
    F.mTimeStamp = 0;
    F.mK = cv::Mat::eye(3, 3, CV_32F);
    F.N = n;
    F.mvKeys.resize(n);
    F.mvKeysUn = F.mvKeys;
    F.mvpMapPoints = std::vector<MapPoint *>(n, static_cast<MapPoint *>(NULL));
    for (int i = 0; i < n; i++)
        if (frame_mp[i] >= 0) F.mvpMapPoints[(size_t)i] = M.mps[(size_t)frame_mp[i]];
    F.mvbOutlier = std::vector<bool>(n, false);
    F.mnId = Frame::nNextId++;
    F.mnScaleLevels = 1;
    F.mfScaleFactor = 1.2f;
    F.mvScaleFactors.assign(1, 1.0f);
    F.mvLevelSigma2.assign(1, 1.0f);
    F.mvInvLevelSigma2.assign(1, 1.0f);
    F.mTcw = cv::Mat::eye(4, 4, CV_32F);
    T->mCurrentFrame = F;
    const std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    T->UpdateReference();
    const std::chrono::steady_clock::time_point t1 = std::chrono::steady_clock::now();
    if (ns) *ns = (long long)std::chrono::duration_cast<std::chrono::nanoseconds>(t1 - t0).count();
    for (int i = 0; i < n; i++) {
        MapPoint *p = T->mCurrentFrame.mvpMapPoints[(size_t)i];
        frame_mp[i] = p ? M.mp_index[p] : -1;
    }
    const std::vector<KeyFrame *> &lk = T->mvpLocalKeyFrames;
    for (size_t t = 0; t < lk.size() && (int)t < cap_kf; t++) kf_ids[t] = M.kf_id(lk[t]);
    *ref_kf = T->mpReferenceKF ? M.kf_id(T->mpReferenceKF) : -1;
    const std::vector<MapPoint *> &lp = T->mvpLocalMapPoints;
    for (size_t j = 0; j < lp.size() && (int)j < cap_pts; j++) points[j] = M.mp_index[lp[j]];
    *npoints = (int)lp.size();
    return (int)lk.size();
}

}  // extern "C"
