// oracle/ref_shim/ref_kf_culling.cc -- the driver of ref_observations.cc with the reference's own, unmodified
// LocalMapping::KeyFrameCulling (src/LocalMapping.cc:524-578) on scripted maps (TEST INFRASTRUCTURE ONLY).
//
// Built by oracle/kf_culling.py into oracle/_ref/libref_kf_culling.so together with the reference's src/LocalMapping.cc,
// both against the stand-in headers of oracle/ref_shim_lm/ (ROS, tf and g2o names that LocalMapping.h pulls in), linked
// against libref_orbslam.so.  A culling call sets mpCurrentKeyFrame and calls KeyFrameCulling(); the verdict of each entry
// of the current keyframe's GetVectorCovisibleKeyFrames() is read from what SetBadFlag left behind: every listed keyframe
// is put into the Map just before the call, and SetBadFlag removes it (Map::EraseKeyFrame) only when it runs past its
// mnId == 0 and mbNotErase returns; mbNotErase's return sets mbToBeErased.
#include <chrono>
#include <fstream>
#include <list>
#include <sstream>
#include <string>

#include "ref_observations.cc"

#define protected public   // mpCurrentKeyFrame and KeyFrameCulling() are protected
#include "LocalMapping.h"
#include "LoopClosing.h"
#include "Optimizer.h"
#undef protected

namespace ORB_SLAM {
// LocalMapping::Run's callees outside the compiled sources; the driver never runs Run
void Optimizer::LocalBundleAdjustment(KeyFrame *, bool *) {
    std::fprintf(stderr, "ref_kf_culling: LocalBundleAdjustment is not linked\n");
    std::abort();
}
void LoopClosing::InsertKeyFrame(KeyFrame *) {
    std::fprintf(stderr, "ref_kf_culling: LoopClosing is not linked\n");
    std::abort();
}
}  // namespace ORB_SLAM

extern "C" {

// GetKeyPointUn(i).octave = oct[i] for the keyframe's first n features
void ref_kc_set_octaves(void *h, int kf, int n, const int *oct) {
    KeyFrame *K = static_cast<CvMap *>(h)->kfs[(size_t)kf];
    for (int i = 0; i < n && i < (int)K->mvKeysUn.size(); i++) K->mvKeysUn[(size_t)i].octave = oct[i];
}

void ref_kc_set_not_erase(void *h, int kf) { static_cast<CvMap *>(h)->kfs[(size_t)kf]->SetNotErase(); }

// KeyFrameCulling() with keyframe `current` as mpCurrentKeyFrame.  ids / verdicts (cap entries): the creation index and the
// ORBFE_CULL_* code of every entry of its GetVectorCovisibleKeyFrames(); *ns = the call's wall time in nanoseconds.
// Returns the list's length.
int ref_kc_cull(void *h, int current, int *ids, int *verdicts, int cap, long long *ns) {
    CvMap &M = *static_cast<CvMap *>(h);
    const std::vector<KeyFrame *> v = M.kfs[(size_t)current]->GetVectorCovisibleKeyFrames();
    std::vector<char> was_bad(v.size());
    for (size_t t = 0; t < v.size(); t++) {
        was_bad[t] = v[t]->isBad();
        v[t]->mbToBeErased = false;
        M.map.AddKeyFrame(v[t]);
    }
    LocalMapping lm(&M.map);
    lm.mpCurrentKeyFrame = M.kfs[(size_t)current];
    const std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    lm.KeyFrameCulling();
    const std::chrono::steady_clock::time_point t1 = std::chrono::steady_clock::now();
    if (ns) *ns = (long long)std::chrono::duration_cast<std::chrono::nanoseconds>(t1 - t0).count();
    const int n = (int)v.size();
    for (int t = 0; t < n && t < cap; t++) {
        ids[t] = M.kf_id(v[t]);
        const bool erased = M.map.mspKeyFrames.count(v[t]) == 0;
        if (v[t]->mnId == 0) verdicts[t] = 1;            // skipped
        else if (erased) verdicts[t] = was_bad[t] ? 4 : 2;   // a repeat on a retired keyframe, or erased
        else if (v[t]->mbToBeErased) verdicts[t] = 3;    // mbNotErase
        else verdicts[t] = 0;                            // kept
    }
    for (int t = 0; t < n; t++) M.map.mspKeyFrames.erase(v[t]);
    return n;
}

}  // extern "C"
