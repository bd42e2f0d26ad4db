// oracle/ref_shim/ref_observations.cc -- the driver of ref_covis.cc with the map edits that change a point's observations
// besides AddObservation / SetBadFlag / EraseMapPointMatch (TEST INFRASTRUCTURE ONLY): MapPoint::Replace (LocalMapping's
// Fuse), the local-BA outlier pair EraseMapPointMatch + EraseObservation (Optimizer.cc:464-465, :512-513), the two halves of
// an observation on their own (Tracking fills a new keyframe's mvpMapPoints before ProcessNewKeyFrame adds the
// observations), and the readback of GetReferenceKeyFrame().
//
// Built by oracle/Makefile into oracle/_ref/libref_drivers.so, linked against libref_orbslam.so; the culling and local-map
// drivers include it.  Keyframes made here carry zero descriptors, so Replace's ComputeDistinctiveDescriptors has rows to read.
#include "ref_covis.cc"

extern "C" {

// ref_cv_add_keyframe with an n x 32 descriptor matrix
int ref_ob_add_keyframe(void *h, int n) {
    const int k = ref_cv_add_keyframe(h, n);
    static_cast<CvMap *>(h)->kfs[(size_t)k]->mDescriptors = cv::Mat::zeros(n, 32, CV_8U);
    return k;
}

// pKF->AddMapPoint(pMP, idx) alone
void ref_ob_add_map_point(void *h, int kf, int idx, int mp) {
    CvMap &M = *static_cast<CvMap *>(h);
    M.kfs[(size_t)kf]->AddMapPoint(M.mps[(size_t)mp], (size_t)idx);
}

// pMP->AddObservation(pKF, idx) alone
void ref_ob_add_observation(void *h, int mp, int kf, int idx) {
    CvMap &M = *static_cast<CvMap *>(h);
    M.mps[(size_t)mp]->AddObservation(M.kfs[(size_t)kf], (size_t)idx);
}

// mps[from]->Replace(mps[to])
void ref_ob_replace(void *h, int from, int to) {
    CvMap &M = *static_cast<CvMap *>(h);
    M.mps[(size_t)from]->Replace(M.mps[(size_t)to]);
}

// pKF->EraseMapPointMatch(pMP); pMP->EraseObservation(pKF)
void ref_ob_ba_erase(void *h, int kf, int mp) {
    CvMap &M = *static_cast<CvMap *>(h);
    M.kfs[(size_t)kf]->EraseMapPointMatch(M.mps[(size_t)mp]);
    M.mps[(size_t)mp]->EraseObservation(M.kfs[(size_t)kf]);
}

// GetReferenceKeyFrame() as a creation index (-2 for a pointer that is no keyframe of the map)
int ref_ob_reference(void *h, int mp) {
    CvMap &M = *static_cast<CvMap *>(h);
    return M.kf_id(M.mps[(size_t)mp]->GetReferenceKeyFrame());
}

// the host build of the observation lists an integration makes without the device entry: per named point a copy of
// GetObservations(), walked in pointer order, each entry written slot_of[pKF->mnId]*cap + idx; returns the total
int ref_ob_flatten(void *h, int n, const int *points, const int *slot_of, int cap, int *ptr, int *obs) {
    CvMap &M = *static_cast<CvMap *>(h);
    int t = 0;
    ptr[0] = 0;
    for (int j = 0; j < n; j++) {
        const std::map<KeyFrame *, size_t> o = M.mps[(size_t)points[j]]->GetObservations();
        for (std::map<KeyFrame *, size_t>::const_iterator it = o.begin(); it != o.end(); ++it)
            obs[t++] = slot_of[it->first->mnId] * cap + (int)it->second;
        ptr[j + 1] = t;
    }
    return t;
}

}  // extern "C"
