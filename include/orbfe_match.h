/*
 * orbfe_match.h -- C-ABI of the windowed matchers of liborbfe.so on plain arrays.
 *
 * Each function is the array-level equivalent of one ORB_SLAM::ORBmatcher method (reference
 * src/ORBmatcher.cc); the C++ facade orb_slam_b200/host/ORBmatcher.cc converts Frame / MapPoint objects
 * into these views.  Every matcher runs on the GPU.  The windowed matchers (SearchByProjection, WindowSearch,
 * SearchForInitialization and the guided search) run on one fused kernel: Frame's grid, GetFeaturesInArea order, the
 * distances, the accept loop and the rotation histogram, one thread block per frame pair.  Their host-array forms stage the
 * arrays, launch once per call and synchronise.  Calls on one matcher run in call order, whichever streams they are
 * enqueued on: a device entry's stream first waits for the matcher's previous call (they share its candidate scratch and
 * error flags), and orbfe_matcher_sync reports the flags of every call made before it.
 *
 * Accepted domain of the host-array windowed matchers: a call is accepted when the kernel's per-block shared memory,
 * sbp_smem_fixed_bytes(cap, qcap) + 16 KB, is at most 220 KB, where sbp_smem_fixed_bytes(cap, qcap) is about 24,584 +
 * 16.125 * cap + 6.125 * qcap bytes.  For orbfe_search_by_projection_frames (cap = qcap = the most features of any view of the call) and
 * orbfe_search_for_initialization (cap = qcap = max(F1 features, F2 features)) that is at most 8283 features.  For
 * orbfe_window_search, orbfe_search_local_points, orbfe_search_by_projection_kf, orbfe_search_by_projection_f1f2 and
 * orbfe_guided_search, cap = the searched frame's feature count and qcap = the number of queries (the features or map points
 * that pass the routine's own filters): 2000 features allow about 24,800 queries per launch.  A call with more queries runs
 * them in consecutive launches on the matcher's stream, with the same result, unless it applies the rotation histogram
 * (check_orientation, hist_mode 1): such a call, like one whose features alone exceed the limit, returns
 * ORBFE_ERR_UNSUPPORTED with a message (orbfe_last_error).  orbfe_guided_best takes any number of queries the same way.
 * Every rejection sets orbfe_last_error.
 */
#ifndef ORBFE_MATCH_H
#define ORBFE_MATCH_H

#include "orbfe.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The slice of ORB_SLAM::Frame the matchers read (include/Frame.h): mvKeysUn, mDescriptors, the image
 * bounds mnMinX.. (Frame.cc:321-350), mfGridElementWidthInv/HeightInv (Frame.cc:77-78) and mvScaleFactors
 * (Frame.cc:95-103).  The 64x48 lookup grid (Frame.cc:109-123) is rebuilt from keys_un on each call. */
typedef struct {
    int n;
    const OrbfeKeyPoint *keys_un;
    const uint8_t *desc; /* n x 32 */
    float min_x, min_y, max_x, max_y;
    float grid_inv_w, grid_inv_h;
    int nlevels;
    const float *scale_factors;
} OrbfeFrameView;

/* Frame::mvScaleFactors as Frame.cc:95-103 derives them from ORBextractor::GetScaleFactor() */
void orbfe_frame_scale_factors(float scale_factor, int nlevels, float *out);

/* int ORBmatcher::SearchByProjection(Frame &CurrentFrame, const Frame &LastFrame, float th)
 * (ORBmatcher.cc:1507-1620) for `npairs` independent (Current, Last) pairs per call.
 * Per pair j: last_has_mp[j][i] != 0 <=> LastFrame.mvpMapPoints[i] != NULL; last_outlier[j][i] =
 * LastFrame.mvbOutlier[i]; last_world[j] = 3 floats per Last feature (MapPoint::GetWorldPos);
 * Tcw[j] = CurrentFrame.mTcw as 3x4 row-major floats; fx..cy = Frame::fx.. (static camera intrinsics).
 * cur_mp_inout[j][i2] = index of the Last feature whose map point got assigned to Current feature i2, or -1
 * (entries >= 0 on input are treated as already-occupied slots, CurrentFrame.mvpMapPoints[i2] != NULL).
 * nmatches_out[j] = the method's return value.  Pairs whose Current views share bounds, grid_inv_w/h, nlevels and
 * scale_factors run in one launch.  ORBFE_ERR_ARG when a Last map point's octave is >= its Current view's nlevels. */
int orbfe_search_by_projection_frames(OrbfeMatcher *m, int npairs, const OrbfeFrameView *cur,
                                      const OrbfeFrameView *last, const uint8_t *const *last_has_mp,
                                      const uint8_t *const *last_outlier, const float *const *last_world,
                                      const float *const *Tcw, float fx, float fy, float cx, float cy, float th,
                                      int check_orientation, int *const *cur_mp_inout, int *nmatches_out);

/* The same routine with EVERYTHING device-resident (no host round trip between extract and match):
 * d_kps / d_desc / d_counts are the outputs of orbfe_extract_batch_device (frame f at f*cap); pair j matches
 * frame d_cur_idx[j] (Current) against frame d_last_idx[j] (Last).  d_world = 3 floats per feature of every
 * frame (position of the feature's map point), d_flags[f*cap+i] != 0 <=> feature i of frame f has a map point and is
 * not an outlier, d_Tcw = 12 floats per pair.  d_cur_mp (npairs x cap ints) must be initialised by the caller
 * (-1 = free slot, >= 0 = occupied) and receives the Last index matched to each Current feature; d_nmatches[j] =
 * return value (-1 if the pair overflowed the candidate scratch: orbfe_matcher_sync then reports ORBFE_ERR_CAPACITY).
 * Frame's 64x48 grid, GetFeaturesInArea order, the greedy accept loop and the rotation histogram all run in one
 * kernel (one CTA per pair) with results identical to orbfe_search_by_projection_frames.  Enqueued on `stream`
 * (NULL = the matcher's stream), not synchronised. */
int orbfe_search_by_projection_device(OrbfeMatcher *m, int npairs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                      const int *d_counts, int cap, const int *d_cur_idx, const int *d_last_idx,
                                      const float *d_world, const uint8_t *d_flags, const float *d_Tcw,
                                      float min_x, float min_y, float max_x, float max_y, float scale_factor, int nlevels,
                                      float fx, float fy, float cx, float cy, float th, int check_orientation,
                                      int *d_cur_mp, int *d_nmatches, void *stream);

/* ORBmatcher::SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize) (ORBmatcher.cc:598-713; call
 * pattern Tracking.cc:352-353 and, across cameras of a rig, BASELINE config 4) with everything device-resident: pair j
 * searches the level-0 features of frame d_f1_idx[j] in frame d_f2_idx[j] (frames as laid out by
 * orbfe_extract_batch_device / the rig exchange: frame f at f*cap).  d_prev_matched: npairs x cap x 2 floats, the
 * vbPrevMatched vector of each pair (x, y per F1 feature), updated in place for the matched features (:706-710).
 * d_match12 (npairs x cap ints) receives vnMatches12, d_nmatches[j] the return value.  The candidate walk
 * (Frame::GetFeaturesInArea order), the skip of candidates whose current match is at least as close (:637), the
 * re-assignment of an already matched F2 feature (:656-663) and the rotation histogram (entries of features that were
 * unmatched later still count, as in the reference) run in one kernel, one thread block per pair.  Not synchronised. */
int orbfe_search_for_initialization_device(OrbfeMatcher *m, int npairs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                           const int *d_counts, int cap, const int *d_f1_idx, const int *d_f2_idx,
                                           float *d_prev_matched, float min_x, float min_y, float max_x, float max_y, int window,
                                           float nnratio, int check_orientation, int *d_match12, int *d_nmatches, void *stream);

/* Guided search (the skeleton shared by ORBmatcher.cc:49-125, :519-594, :1622-1746 and WindowSearch-style loops) with
 * EVERYTHING device-resident: job j searches frame d_frame_idx[j] (layout as above) with the explicit query windows
 * [d_q_base[j], d_q_base[j] + d_q_cnt[j]) of the concatenated arrays: centre (qu, qv), half-size qr, octave filter
 * [qlo, qhi] ((-1,-1) = none), 32-byte descriptor, angle (only read when check_orientation).  qcap >= every d_q_cnt[j].
 * rule 0: best <= th_dist; rule 1: best <= second*nnratio && best <= TH_HIGH (:469, :586); rule 2: best <= TH_HIGH &&
 * !(bestLevel == secondLevel && best > nnratio*second) (:113-121).  d_slot_owner (njobs x cap, in/out): >= 0 on entry =
 * occupied slot (never reassigned); free slots matched in this call receive the job-local query index.
 * d_nmatches[j] = number of matches kept (-1: candidate scratch overflow -> ORBFE_ERR_CAPACITY at sync). */
int orbfe_guided_search_device(OrbfeMatcher *m, int njobs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                               const int *d_counts, int cap, const int *d_frame_idx, const float *d_qu, const float *d_qv,
                               const float *d_qr, const int *d_qlo, const int *d_qhi, const uint8_t *d_qdesc,
                               const float *d_qangle, const int *d_q_base, const int *d_q_cnt, int qcap, float min_x,
                               float min_y, float max_x, float max_y, int rule, float nnratio, int th_dist,
                               int check_orientation, int *d_slot_owner, int *d_nmatches, void *stream);

/* ---- Camera rigs: the three device entries above over frames of several cameras in one launch ----
 *
 * A frame store filled by orbfe_extract_multi_device holds frames of up to ORBFE_MULTI_MAX_GROUPS image geometries.  The
 * *_cams_device entries below are the device entries above with the per-call geometry replaced by a camera table: `cams`
 * is a HOST array of 1 <= ncams <= ORBFE_MULTI_MAX_GROUPS cameras, d_frame_cam a DEVICE array with one camera index per
 * frame of the store.  A pair or job takes the camera of the frame it searches: the Current frame d_cur_idx[j] (its
 * bounds, grid and intrinsics), F2 = d_f2_idx[j] (its bounds; F1 may belong to another camera) or d_frame_idx[j].
 * scale_factor, nlevels, cap, qcap, thresholds and rules stay per call: one extractor made the store.  Every output of a
 * pair equals what the single-geometry entry writes when called with that pair's camera, bit for bit, in one launch.
 * The table travels in the kernel's parameters: the calls stay enqueue-only, with the matcher's stream-order rule.
 * ORBFE_ERR_ARG before anything is enqueued: ncams outside [1, ORBFE_MULTI_MAX_GROUPS], cams or d_frame_cam NULL, a
 * camera without max_x > min_x and max_y > min_y, and every check of the single-geometry entry.  A pair whose searched
 * frame has a camera index outside [0, ncams) gets d_nmatches[j] = -1 and its other outputs untouched;
 * orbfe_matcher_sync then reports ORBFE_ERR_ARG, even when another pair of the launch overflowed the candidate scratch.
 * The other pairs are unaffected.  Frame indices are not checked. */
typedef struct {
    float min_x, min_y, max_x, max_y; /* Frame::mnMinX.. of this camera (e.g. from orbfe_image_bounds) */
    float fx, fy, cx, cy;             /* read only by the projection search */
} OrbfeCamera;

int orbfe_search_by_projection_cams_device(OrbfeMatcher *m, int npairs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                           const int *d_counts, int cap, const int *d_cur_idx, const int *d_last_idx,
                                           const float *d_world, const uint8_t *d_flags, const float *d_Tcw, int ncams,
                                           const OrbfeCamera *cams, const int *d_frame_cam, float scale_factor, int nlevels,
                                           float th, int check_orientation, int *d_cur_mp, int *d_nmatches, void *stream);
int orbfe_search_for_initialization_cams_device(OrbfeMatcher *m, int npairs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                                const int *d_counts, int cap, const int *d_f1_idx, const int *d_f2_idx,
                                                float *d_prev_matched, int ncams, const OrbfeCamera *cams, const int *d_frame_cam,
                                                int window, float nnratio, int check_orientation, int *d_match12, int *d_nmatches,
                                                void *stream);
int orbfe_guided_search_cams_device(OrbfeMatcher *m, int njobs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                    const int *d_counts, int cap, const int *d_frame_idx, const float *d_qu, const float *d_qv,
                                    const float *d_qr, const int *d_qlo, const int *d_qhi, const uint8_t *d_qdesc,
                                    const float *d_qangle, const int *d_q_base, const int *d_q_cnt, int qcap, int ncams,
                                    const OrbfeCamera *cams, const int *d_frame_cam, int rule, float nnratio, int th_dist,
                                    int check_orientation, int *d_slot_owner, int *d_nmatches, void *stream);

/* int ORBmatcher::SearchByProjection(Frame &F, const vector<MapPoint*>&, float th) (ORBmatcher.cc:49-125), local-map
 * tracking.  Per map point: in_view = mbTrackInView && !isBad(); proj_xy = (mTrackProjX, mTrackProjY); level =
 * mnTrackScaleLevel; view_cos = mTrackViewCos; desc = GetDescriptor().  f_mp_inout[i2] >= 0 <=> F.mvpMapPoints[i2] set
 * on entry; on exit it holds the index of the map point assigned to feature i2. */
int orbfe_search_local_points(OrbfeMatcher *m, const OrbfeFrameView *f, int npts, const uint8_t *in_view,
                              const float *proj_xy, const int *level, const float *view_cos, const uint8_t *desc, float th,
                              float nnratio, int *f_mp_inout, int *nmatches_out);

/* int ORBmatcher::SearchByProjection(Frame &CurrentFrame, KeyFrame *pKF, const set<MapPoint*> &sAlreadyFound, float th,
 * int ORBdist) (ORBmatcher.cc:1622-1746), relocalisation refinement.  Per keyframe feature i: valid[i] = has a map point,
 * not bad, not in sAlreadyFound; world / min_dist (GetMinDistanceInvariance) / desc of that point; kf_angle[i] =
 * pKF->GetKeyPointUn(i).angle.  Tcw = CurrentFrame.mTcw (3x4). */
int orbfe_search_by_projection_kf(OrbfeMatcher *m, const OrbfeFrameView *cur, int npts, const uint8_t *valid, const float *world,
                                  const float *min_dist, const uint8_t *desc, const float *kf_angle, const float *Tcw, float fx,
                                  float fy, float cx, float cy, float th, int orb_dist, int check_orientation, int *cur_mp_inout,
                                  int *nmatches_out);

/* int ORBmatcher::SearchByProjection(Frame &F1, Frame &F2, int windowSize, vector<MapPoint*> &vpMapPointMatches2)
 * (ORBmatcher.cc:519-594).  valid1[i1] = F1 has a map point there, not bad, not already among F2's matches (:533-537);
 * world1 = its position; Tc2w = F2.mTcw; f2_mp_inout = F2's slots (>= 0 occupied), receives i1 for new matches. */
int orbfe_search_by_projection_f1f2(OrbfeMatcher *m, const OrbfeFrameView *f1, const OrbfeFrameView *f2, const uint8_t *valid1,
                                    const float *world1, const float *Tc2w, float fx, float fy, float cx, float cy, int window,
                                    float nnratio, int *f2_mp_inout, int *nmatches_out);

/* The skeleton shared by ORBmatcher's projection routines, for callers that project themselves (the facade's
 * KeyFrame-level methods: SearchByProjection(KeyFrame*,Scw,...) :286-407, SearchBySim3 :1267-1505, Fuse :1016-1265).
 * Query q searches window (qu,qv) +- qr with octave filter [qlo,qhi] (-1,-1 = none, like KeyFrame::GetFeaturesInArea)
 * among the features of `f` whose slot is still free; rule 0: best <= th_dist; rule 1: best <= second*nnratio and best <=
 * TH_HIGH; rule 2: best <= TH_HIGH unless best and second are on the same level and best > nnratio*second.
 * hist_mode 0: none, 1: rotation histogram + three-maxima filter (qangle needed), 2: filled but not applied.
 * slot_owner_inout[i2] >= 0 = occupied on entry; accepted queries store their index q there. */
int orbfe_guided_search(OrbfeMatcher *m, const OrbfeFrameView *f, int nq, const float *qu, const float *qv, const float *qr,
                        const int32_t *qlo, const int32_t *qhi, const uint8_t *qdesc, const float *qangle, int rule,
                        float nnratio, int th_dist, int hist_mode, int32_t *slot_owner_inout, int *nmatches_out);

/* Guided search without slot bookkeeping: best candidate of every query, kept iff best <= th_dist (first minimum in
 * GetFeaturesInArea order wins).  The inner loops of Fuse (ORBmatcher.cc:1090-1107, :1222-1239) and SearchBySim3
 * (:1356-1378, :1436-1458); runs on the same fused kernel as orbfe_guided_search.  best_idx_out[q] = feature index in `f`
 * or -1. */
int orbfe_guided_best(OrbfeMatcher *m, const OrbfeFrameView *f, int nq, const float *qu, const float *qv, const float *qr,
                      const int32_t *qlo, const int32_t *qhi, const uint8_t *qdesc, int th_dist, int32_t *best_idx_out);

/* int ORBmatcher::SearchByBoW(KeyFrame*, Frame&, matches) (variant 0, ORBmatcher.cc:155-284) and
 * SearchByBoW(KeyFrame*, KeyFrame*, matches12) (variant 1, :715-850): brute force inside equal vocabulary nodes.
 * A DBoW2::FeatureVector is passed as ascending node ids + CSR (ptr, items = feature indices in insertion order).
 * valid1[i] / valid2[i]: the feature has a map point that is not bad (valid2 is ignored by variant 0).
 * angle1 / angle2: mvKeysUn[i].angle of each side.  variant 0: out has n2 entries, out[i2] = matched side-1 index;
 * variant 1: out has n1 entries, out[i1] = matched side-2 index; -1 = no match.
 * items holds ptr[nn] entries, and every feature index appears in at most one node (true of any DBoW2 FeatureVector).
 * Runs as one job of orbfe_search_by_bow_device (staging, one launch, synchronised), so it rejects the same FeatureVectors:
 * a common node whose row reaches outside [0, ptr[nn]] or holds a feature index outside [0, n) gives ORBFE_ERR_ARG, and out
 * is then not meaningful.  At most 65535 features and 65535 FeatureVector nodes per side (ORBFE_ERR_UNSUPPORTED). */
int orbfe_search_by_bow(OrbfeMatcher *m, int variant, int n1, const uint8_t *desc1, const uint8_t *valid1, const float *angle1,
                        int nn1, const int32_t *ids1, const int32_t *ptr1, const int32_t *items1, int n2, const uint8_t *desc2,
                        const uint8_t *valid2, const float *angle2, int nn2, const int32_t *ids2, const int32_t *ptr2,
                        const int32_t *items2, float nnratio, int check_orientation, int32_t *out, int *nmatches_out);

/* SearchByBoW (both overloads, as orbfe_search_by_bow) with EVERYTHING device-resident, for `njobs` frame pairs per call:
 * job j matches side-1 frame d_idx1[j] against side-2 frame d_idx2[j] of the frame store d_kps / d_desc / d_counts (frame f
 * at f*cap, as orbfe_extract_batch_device lays it out).  Many jobs may share a frame: relocalisation matches one frame
 * against every candidate keyframe (Tracking.cc:841-901), loop closing one keyframe against every loop candidate.
 * FeatureVectors in the layout orbfe_feature_vector_device writes (include/orbfe_bow.h): node ids d_fv_ids[f*cap + k]
 * (strictly ascending), row starts d_fv_ptr[f*(cap+1) + k], feature indices d_fv_items[f*cap + ...], d_fv_n[f] nodes; every
 * feature index appears in at most one node (true of any DBoW2 FeatureVector).  FeatureVectors built on the host (keyframes
 * whose BoW was computed earlier) may be uploaded into the same layout.
 * d_valid[f*cap + i] != 0: feature i of frame f has a map point that is not bad (side 2 of variant 0 ignores it).
 * Angles are d_kps[].angle.  variant 0: row j of d_out (njobs x cap) is indexed by side-2 feature and holds the matched
 * side-1 index; variant 1: indexed by side-1 feature, holding the side-2 index; -1 = no match; the first count entries of
 * each row are written.  d_nmatches[j] = the method's return value.
 * One thread block per job, no global scratch.  A FeatureVector entry outside the frame's slots (node count > cap, a row
 * outside [0, cap], a feature index >= the frame's count) is never followed: that job's d_nmatches is -1 and
 * orbfe_matcher_sync reports ORBFE_ERR_ARG; the other jobs of the launch are unaffected.  Frame indices are not checked.
 * 1 <= cap <= 65535.  Enqueued on `stream` (NULL = the matcher's stream), not synchronised. */
int orbfe_search_by_bow_device(OrbfeMatcher *m, int variant, int njobs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                               const int *d_counts, int cap, const int32_t *d_fv_ids, const int32_t *d_fv_ptr,
                               const int32_t *d_fv_items, const int *d_fv_n, const uint8_t *d_valid, const int *d_idx1,
                               const int *d_idx2, float nnratio, int check_orientation, int32_t *d_out, int *d_nmatches,
                               void *stream);

/* int ORBmatcher::SearchForTriangulation(pKF1, pKF2, F12, ...) (ORBmatcher.cc:852-1014) with CheckDistEpipolarLine
 * (:136-153).  keys1/keys2 = GetKeyPointsUn(); has_mp1/2[i] != 0 <=> the feature already has a map point (skipped);
 * FeatureVectors as in orbfe_search_by_bow; F12 = 3x3 row-major floats; sigma2_kf2[level] = pKF2->GetSigma2(level), with an
 * entry for every octave that occurs in keys2 (GetScaleLevels() entries do).
 * match12_out[i1] = matched index in keyframe 2 or -1 (the caller builds vMatchedKeys1/2 and vMatchedPairs from it).
 * Runs as one job of orbfe_search_for_triangulation_device, with nlevels = 1 + the largest octave of keys2 (at most
 * ORBFE_MAX_LEVELS).  ORBFE_ERR_ARG for the FeatureVectors orbfe_search_by_bow rejects and for a side-2 feature without a map
 * point, in a common node, whose octave is negative or >= ORBFE_MAX_LEVELS; match12_out is then not meaningful.  At most
 * 65535 features and 65535 FeatureVector nodes per side (ORBFE_ERR_UNSUPPORTED). */
int orbfe_search_for_triangulation(OrbfeMatcher *m, int n1, const OrbfeKeyPoint *keys1, const uint8_t *desc1,
                                   const uint8_t *has_mp1, int nn1, const int32_t *ids1, const int32_t *ptr1, const int32_t *items1,
                                   int n2, const OrbfeKeyPoint *keys2, const uint8_t *desc2, const uint8_t *has_mp2, int nn2,
                                   const int32_t *ids2, const int32_t *ptr2, const int32_t *items2, const float *F12,
                                   const float *sigma2_kf2, int check_orientation, int32_t *match12_out, int *nmatches_out);

/* SearchForTriangulation (as orbfe_search_for_triangulation) with the keyframes device-resident, for `njobs` keyframe pairs
 * per call: job j matches pKF1 = frame d_idx1[j] against pKF2 = frame d_idx2[j] of the frame store d_kps / d_desc / d_counts
 * (frame f at f*cap, as orbfe_extract_batch_device lays it out; the keypoints are the undistorted ones, e.g. after
 * orbfe_undistort_keypoints_device in place).  Many jobs may share a frame: LocalMapping::CreateNewMapPoints
 * (LocalMapping.cc:205-252) matches the new keyframe against each of its covisible neighbours.
 * FeatureVectors in the layout orbfe_feature_vector_device writes, as in orbfe_search_by_bow_device.
 * d_has_mp[f*cap + i] != 0: feature i of frame f has a map point (GetMapPointMatches()[i] != NULL, bad points included).
 * d_F12 = njobs x 9 row-major floats (ComputeF12 of the pair); sigma2 = `nlevels` floats on the HOST (KeyFrame::GetSigma2,
 * shared by all keyframes of one extractor).  Row j of d_match12 (njobs x cap) is indexed by side-1 feature and holds the
 * matched side-2 index or -1 for the first counts[d_idx1[j]] entries; d_nmatches[j] = the method's return value.
 * One thread block per job, no global scratch.  A job whose FeatureVectors point outside the frames' slots (node count
 * outside [0, cap], a row outside [0, cap], a feature index >= the frame's count) or whose side-2 features without a map
 * point in a common node have an octave outside [0, nlevels) is never followed out of bounds: its d_nmatches is -1 and
 * orbfe_matcher_sync reports ORBFE_ERR_ARG; the other jobs of the launch are unaffected.  Frame indices are not checked.
 * 1 <= cap <= 65535, 1 <= nlevels <= ORBFE_MAX_LEVELS.  Enqueued on `stream` (NULL = the matcher's stream), not
 * synchronised. */
int orbfe_search_for_triangulation_device(OrbfeMatcher *m, int njobs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                          const int *d_counts, int cap, const int32_t *d_fv_ids, const int32_t *d_fv_ptr,
                                          const int32_t *d_fv_items, const int *d_fv_n, const uint8_t *d_has_mp, const int *d_idx1,
                                          const int *d_idx2, const float *d_F12, const float *sigma2, int nlevels,
                                          int check_orientation, int32_t *d_match12, int *d_nmatches, void *stream);

/* int ORBmatcher::WindowSearch(F1, F2, windowSize, vpMapPointMatches2, minOctave, maxOctave)
 * (ORBmatcher.cc:409-516).  f1_has_mp[i1] != 0 <=> F1.mvpMapPoints[i1] && !isBad().
 * match21_out[i2] = i1 whose map point was matched to F2 feature i2, or -1. */
int orbfe_window_search(OrbfeMatcher *m, const OrbfeFrameView *f1, const OrbfeFrameView *f2,
                        const uint8_t *f1_has_mp, int window, int min_level, int max_level, float nnratio,
                        int check_orientation, int *match21_out, int *nmatches_out);

/* int ORBmatcher::SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize)
 * (ORBmatcher.cc:598-713).  prev_matched = 2 floats per F1 feature, updated in place (:708-710).
 * match12_out[i1] = i2 or -1. */
int orbfe_search_for_initialization(OrbfeMatcher *m, const OrbfeFrameView *f1, const OrbfeFrameView *f2,
                                    float *prev_matched, int window, float nnratio, int check_orientation,
                                    int *match12_out, int *nmatches_out);

/* ---- Frame feature post-processing (SURVEY.md section 8(f) row N1) ---- */

/* Frame::UndistortKeyPoints (reference src/Frame.cc:289-319): cv::undistortPoints(pts, mK, mDistCoef, cv::Mat(), mK) on
 * the (x, y) of n keypoints, every other field copied.  dist5 = (k1, k2, p1, p2, k3) on the HOST (the reference's
 * mDistCoef has the first four; pass k3 = 0).  k1 == 0 copies the keypoints (:291-295).  Double-precision arithmetic
 * in OpenCV's evaluation order: bit-exact against OpenCV.  In-place (d_in == d_out) is allowed.
 * Device form: enqueued on `stream` (NULL = the matcher's stream), not synchronised; it chains after
 * orbfe_extract_batch_device on all batch * capacity keypoint slots at once. */
int orbfe_undistort_keypoints_device(OrbfeMatcher *m, const OrbfeKeyPoint *d_in, OrbfeKeyPoint *d_out, int n, float fx, float fy,
                                     float cx, float cy, const float *dist5, void *stream);
int orbfe_undistort_keypoints(OrbfeMatcher *m, const OrbfeKeyPoint *in, OrbfeKeyPoint *out, int n, float fx, float fy, float cx,
                              float cy, const float *dist5);
/* Frame::ComputeImageBounds (Frame.cc:321-350): bounds4 = (mnMinX, mnMinY, mnMaxX, mnMaxY). */
int orbfe_image_bounds(OrbfeMatcher *m, int cols, int rows, float fx, float fy, float cx, float cy, const float *dist5,
                       float *bounds4);

#ifdef __cplusplus
}
#endif
#endif
