/* orbfe_bow.h -- C-ABI of the two "next" rows of SURVEY.md section 8(f) that reuse the 256-bit Hamming primitive:
 *
 *   N2  DBoW2 vocabulary-tree transform: descriptors -> BowVector + FeatureVector
 *       (reference Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1126-1262, FORB.cpp:79-99 (distance),
 *        BowVector.cpp:34-84, FeatureVector.cpp:32-48; callers Frame.cc:280-287, KeyFrame.cc:56-65),
 *       and ORBVocabulary::score on the BowVectors it builds (TemplatedVocabulary.h score(), ScoringObject.cpp:23-67;
 *        caller LoopClosing.cc:117-131)
 *   N3  KeyFrameDatabase::DetectLoopCandidates / DetectRelocalisationCandidates on arrays
 *       (reference src/KeyFrameDatabase.cc:73-308, L1Scoring::score Thirdparty/DBoW2/DBoW2/ScoringObject.cpp:23-67)
 *   N4  MapPoint::ComputeDistinctiveDescriptors, batched over map points (reference src/MapPoint.cc:185-250),
 *       and MapPoint::UpdateNormalAndDepth on the same observation lists (reference src/MapPoint.cc:273-312),
 *       and the covisibility graph KeyFrame::UpdateConnections builds from them (reference src/KeyFrame.cc:126-185, 332-421)
 *
 * Plain pointers and sizes; host arrays unless a parameter is named d_*.  Return values: OrbfeStatus (orbfe.h).
 */
#ifndef ORBFE_BOW_H
#define ORBFE_BOW_H

#include <stdint.h>

#include "orbfe.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct OrbfeVocabulary OrbfeVocabulary;

/* DBoW2::WeightingType / the LNorm a scoring object asks for (ORB-SLAM: TF_IDF + L1, ORBVocabulary.h). */
enum { ORBFE_BOW_TF_IDF = 0, ORBFE_BOW_TF = 1, ORBFE_BOW_IDF = 2, ORBFE_BOW_BINARY = 3 };
enum { ORBFE_BOW_NORM_NONE = 0, ORBFE_BOW_NORM_L1 = 1, ORBFE_BOW_NORM_L2 = 2 };

/* The vocabulary tree as flat arrays (what TemplatedVocabulary::m_nodes holds after load()):
 *   node 0 is the root; the children of node i are children[child_ptr[i] .. child_ptr[i+1]) in the order of
 *   m_nodes[i].children (the descent keeps the FIRST child of minimum distance); a node without children is a leaf
 *   (a word) with word_id[i] >= 0 and weight[i]; node_desc holds 32 bytes per node (the root's are ignored).
 * depth_L = m_L.  The arrays are copied; the node table lives in device memory of `device`. */
OrbfeVocabulary *orbfe_vocabulary_create(int device, int nnodes, int depth_L, const uint8_t *node_desc, const int32_t *child_ptr,
                                         const int32_t *children, const int32_t *word_id, const double *weight, int weighting,
                                         int norm);
void orbfe_vocabulary_destroy(OrbfeVocabulary *v);

/* TemplatedVocabulary::loadFromTextFile (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1338-1424) on the device: the file is
 * read in chunks through a double-buffered pinned staging area into device memory and the node table is parsed there; it
 * never passes through host arrays.  The result equals the reference's m_nodes field for field:
 *   header `k L scoring weighting` (any tokens after them ignored), k in [0,20], L in [1,10], scoring in [0,5],
 *   weighting in [0,3]; norm = what the scoring object's mustNormalize gives (L1 for L1 / chi-square / KL / Bhattacharyya,
 *   L2 for L2, none for dot product);
 *   line n of the body is node n (node 0 is the root), `parent isLeaf b0 .. b31 weight`, any whitespace between tokens,
 *   tokens after the weight ignored; the children of a node are in line order; a node whose isLeaf is > 0 gets the next
 *   word id in line order, every other node word id 0; byte bi = (unsigned char)bi; the weight is the double
 *   `istream >> double` gives (decimal tokens of at most 15 significant digits and a decimal exponent within +-22 are
 *   converted on the device, exactly; any other token, or a missing weight, by that very extraction on the host).
 * A final empty line (the file ends with a newline) adds no node; the reference creates one from uninitialised values.
 * Rejected with ORBFE_ERR_ARG, the 1-based line number in orbfe_last_error: a missing or unreadable file, a bad header, an
 * empty or blank line before the last, fewer than 34 tokens before the weight, a parent / isLeaf / descriptor token that is
 * not a plain decimal int, a parent < 0 or >= the line's node id, a body of 2^31 bytes or more.  No device:
 * ORBFE_ERR_NO_DEVICE.  The header is checked before any device is used.  *out is NULL on every error. */
int orbfe_vocabulary_load_text(int device, const char *path, OrbfeVocabulary **out);
/* Header fields and sizes of any vocabulary (any pointer may be NULL).  k and scoring are -1 for orbfe_vocabulary_create,
 * which never receives them; nwords = the largest word id + 1. */
int orbfe_vocabulary_info(const OrbfeVocabulary *v, int *k, int *L, int *scoring, int *weighting, int *nnodes, int *nwords);
/* Copies the node table back in orbfe_vocabulary_create's layout (node_desc nnodes x 32, child_ptr nnodes + 1, children
 * child_ptr[nnodes] entries -- nnodes - 1 for a loaded text --, word_id and weight nnodes each) and the parent of every node
 * (the root's is 0).  Any pointer may be NULL.  Synchronous. */
int orbfe_vocabulary_export(OrbfeVocabulary *v, uint8_t *node_desc, int32_t *child_ptr, int32_t *children, int32_t *word_id,
                            double *weight, int32_t *parent);

/* transform(feature, word_id, weight, &nid, levelsup) for n descriptors (TemplatedVocabulary.h:1216-1260):
 * leaf_out[i] = node id of the leaf reached, node_out[i] = id of the ancestor at level depth_L - levelsup (0 = root when
 * that level is <= 0, and also when the leaf is shallower than that level, where the reference leaves *nid unset).
 * Device-pointer form: enqueued on `stream` (NULL = the vocabulary's stream), not synchronised -- it chains directly
 * after orbfe_extract_batch_device on the descriptors that call produced. */
int orbfe_bow_descend_device(OrbfeVocabulary *v, const uint8_t *d_desc, int n, int levelsup, int32_t *d_leaf_out,
                             int32_t *d_node_out, void *stream);
int orbfe_bow_descend(OrbfeVocabulary *v, const uint8_t *desc, int n, int levelsup, int32_t *leaf_out, int32_t *node_out);

/* The host-array entries (orbfe_bow_descend, orbfe_bow_transform) are synchronous and may be called from several threads on
 * one vocabulary, as DBoW2's const transform() is (Tracking and LocalMapping both compute BoW): they stage through one
 * block of the vocabulary, one call at a time, on its stream.  The device-pointer entries take no lock. */

/* transform(features, BowVector&, FeatureVector&, levelsup) (TemplatedVocabulary.h:1126-1196): the descent and both
 * std::map builds on the device, as one frame of orbfe_bow_descend_device, orbfe_bow_vector_device and
 * orbfe_feature_vector_device with cap = n.
 *   BowVector:     *nwords_out entries (word id ascending) in bow_ids / bow_vals            (capacity n each)
 *   FeatureVector: *nnodes_out entries (node id ascending) in fv_ids, rows fv_ptr[k]..fv_ptr[k+1] of fv_feats
 *                  (feature indices ascending; capacities n, n+1, n) -- the CSR form orbfe_search_by_bow takes.
 * Nothing is written past bow_ids / bow_vals[*nwords_out - 1], fv_ids[*nnodes_out - 1], fv_ptr[*nnodes_out] and
 * fv_feats[fv_ptr[*nnodes_out] - 1].  The two counts and fv_ptr[0] are set to 0 before any other work, so they stay 0 on a
 * later error; n = 0 returns there without touching the handle.  n <= ORBFE_FV_MAX_CAP, else ORBFE_ERR_UNSUPPORTED (the
 * kernels sort a frame's keys in shared memory). */
int orbfe_bow_transform(OrbfeVocabulary *v, const uint8_t *desc, int n, int levelsup, int *nwords_out, int32_t *bow_ids,
                        double *bow_vals, int *nnodes_out, int32_t *fv_ids, int32_t *fv_ptr, int32_t *fv_feats);

/* The FeatureVector half of transform() on the device, for `nframes` frames at once: d_leaf / d_node hold what
 * orbfe_bow_descend_device wrote (frame f at f*cap, d_counts[f] valid entries -- the frame layout of
 * orbfe_extract_batch_device).  Frame f receives the FeatureVector orbfe_bow_transform returns: d_fv_n[f] nodes, node ids
 * d_fv_ids[f*cap + k] ascending, row starts d_fv_ptr[f*(cap+1) + k] (k = 0..d_fv_n[f]), feature indices d_fv_items[f*cap + ...]
 * ascending inside a node.  As in DBoW2, a feature whose word has weight 0 (a stopped word; the leaf d_leaf names it) is
 * in no node; a leaf id outside the vocabulary counts as stopped.  A frame without features gets 0 nodes and
 * d_fv_ptr[f*(cap+1)] = 0.  One thread block per frame sorts the frame's (node id, feature index) pairs in shared memory:
 * cap <= ORBFE_FV_MAX_CAP, else ORBFE_ERR_UNSUPPORTED.  The output is the input of orbfe_search_by_bow_device
 * (include/orbfe_match.h).  Enqueued on `stream` (NULL = the vocabulary's stream), not synchronised. */
#define ORBFE_FV_MAX_CAP 16384
int orbfe_feature_vector_device(OrbfeVocabulary *v, int nframes, const int32_t *d_leaf, const int32_t *d_node, const int *d_counts,
                                int cap, int32_t *d_fv_ids, int32_t *d_fv_ptr, int32_t *d_fv_items, int *d_fv_n, void *stream);

/* The BowVector half of transform() on the device, in the frame layout of orbfe_feature_vector_device: d_leaf holds what
 * orbfe_bow_descend_device wrote (frame f at f*cap), frame f has min(max(d_counts[f], 0), cap) features.  Frame f receives
 * the BowVector orbfe_bow_transform returns, bit for bit: d_bow_n[f] words, word ids d_bow_ids[f*cap + k] ascending and
 * their values d_bow_vals[f*cap + k]; entries d_bow_n[f] .. cap-1 of the row hold id INT32_MAX and value 0.0, so a whole
 * row can be passed to orbfe_kfdb_detect_device with nq = cap.  The same features are stopped as in the FeatureVector
 * (weight not > 0, or a leaf id outside the vocabulary).  Values follow the vocabulary's weighting and norm: per word in
 * feature order, TF / TF_IDF add every value, IDF / BINARY keep the first; without a norm TF / TF_IDF values are divided by
 * the number of words; with one, the norm is a single sum in ascending word order.  One thread block per frame:
 * cap <= ORBFE_FV_MAX_CAP, else ORBFE_ERR_UNSUPPORTED.  Arguments are checked before the handle is used.  Enqueued on
 * `stream` (NULL = the vocabulary's stream), not synchronised. */
int orbfe_bow_vector_device(OrbfeVocabulary *v, int nframes, const int32_t *d_leaf, const int *d_counts, int cap, int32_t *d_bow_ids,
                            double *d_bow_vals, int *d_bow_n, void *stream);

/* LoopClosing::DetectLoop's minScore (LoopClosing.cc:117-131) for nqueries keyframes at once, and the ORBVocabulary::score
 * values it is the minimum of (L1Scoring::score, ScoringObject.cpp:23-67).  BowVector rows in the layout
 * orbfe_bow_vector_device writes: row f at f*cap holds min(max(d_bow_n[f], 0), cap) words, ids ascending; nothing past that
 * count is read.
 *   Query b is row d_query_row[b]; its connected keyframes are rows d_cov_row[d_cov_ptr[b] .. d_cov_ptr[b+1]) in the order of
 *   GetVectorCovisibleKeyFrames() (nqueries + 1 offsets, read as given).  A connected keyframe with isBad() is passed as a
 *   negative entry and skipped.  A row index outside [0, nframes) is never followed: as a connected keyframe it is skipped
 *   too, as a query it is an empty BowVector.
 *   d_scores (may be NULL; d_cov_ptr[nqueries] entries): d_scores[k] = the double score(query, row d_cov_row[k]), the sum
 *   over the shared words taken in ascending word order, so (float)d_scores[k] is the d_score the resident database reports
 *   for that pair in a loop query; no shared word gives -0.0; nothing is clamped, whatever the vocabulary's norm.  Entries of
 *   skipped keyframes are left untouched.
 *   d_min_score[b]: `float minScore = 1`, then (float)score wherever that is smaller, in list order: the argument of
 *   DetectLoopCandidates and entry b of orbfe_kfdb_detect_batch_device's d_min_score.  1.0f when nothing was scored.
 * One thread block per query, one warp per pair, the query's words staged in shared memory: 1 <= cap <= ORBFE_FV_MAX_CAP,
 * else ORBFE_ERR_UNSUPPORTED.  nqueries >= 0 (0 does nothing), nframes >= 1, nframes*cap < 2^31, else ORBFE_ERR_ARG.
 * Arguments are checked before the handle is used.  Enqueued on `stream` (NULL = the vocabulary's stream), not
 * synchronised, one launch whatever nqueries, no host round trip. */
int orbfe_bow_min_score_device(OrbfeVocabulary *v, int nqueries, int nframes, int cap, const int32_t *d_bow_ids, const double *d_bow_vals,
                               const int *d_bow_n, const int32_t *d_query_row, const int32_t *d_cov_ptr, const int32_t *d_cov_row,
                               double *d_scores, float *d_min_score, void *stream);

/* ORBVocabulary::score(v1, v2) of two host BowVectors (ids ascending; n = 0 may pass NULL), on the kernel of
 * orbfe_bow_min_score_device: one query with one connected keyframe, so *score_out is the d_scores entry of that pair.
 * 0 <= n1, n2 <= ORBFE_FV_MAX_CAP, else ORBFE_ERR_UNSUPPORTED.  Synchronous; may be called from several threads on one
 * vocabulary, like orbfe_bow_transform. */
int orbfe_bow_score(OrbfeVocabulary *v, int n1, const int32_t *ids1, const double *vals1, int n2, const int32_t *ids2,
                    const double *vals2, double *score_out);

/* MapPoint::ComputeDistinctiveDescriptors for ngroups map points at once: group g owns the descriptors
 * desc[group_ptr[g] .. group_ptr[g+1]) (its observations, in the order of the reference's vDescriptors);
 * best_out[g] = index inside the group of the descriptor with the least median distance to the group
 * (median = sorted[(int)(0.5*(N-1))], first minimum wins, MapPoint.cc:228-243), -1 for an empty group.
 * All N x N distances and the medians are computed on the device (one warp per map point). */
int orbfe_distinctive_descriptors(OrbfeMatcher *m, const uint8_t *desc, const int32_t *group_ptr, int ngroups, int32_t *best_out);

/* orbfe_distinctive_descriptors with the descriptors read where they already live: the frame store d_desc / d_counts
 * in the layout orbfe_extract_batch_device writes (frame f at f*cap, `nframes` frames).  Nothing passes through the host.
 *   Group g (one map point) owns the observations d_obs[d_group_ptr[g] .. d_group_ptr[g+1]) (ngroups + 1 pointers,
 *   `nobs` observations).  An observation is the flat slot f*cap + i (feature i of frame f, the index d_valid / d_has_mp
 *   use), and a group lists them in the order of the reference's vDescriptors: mObservations iteration order, with the
 *   observations in bad keyframes left out (MapPoint.cc:204-210).
 *   d_best[g] = position inside the group of the descriptor with the least median distance to the group (median =
 *   sorted[(int)(0.5*(N-1))], first minimum wins, MapPoint.cc:230-244); row g of d_mp_desc (ngroups x 32 bytes)
 *   receives that descriptor -- MapPoint::mDescriptor, and the d_qdesc row orbfe_guided_search_device reads.
 *   An empty group gets d_best[g] = -1 and its row is left untouched (the reference returns early and keeps mDescriptor);
 *   pass a bad map point as an empty group or leave it out.
 * Bad input is never followed: a group with d_group_ptr[g] < 0, d_group_ptr[g] > d_group_ptr[g+1],
 * d_group_ptr[g+1] > nobs, or an observation whose frame is >= nframes or whose feature index is >= d_counts[f], gets
 * d_best[g] = -1 with its row untouched, and orbfe_matcher_sync then reports ORBFE_ERR_ARG; the other groups of the launch
 * are unaffected.  One warp per map point, N x N distances: a group of hundreds of observations takes longest.
 * ngroups >= 0, nobs >= 0, 1 <= cap <= 65535, nframes >= 1, nframes*cap < 2^31; d_desc and d_mp_desc 16-byte aligned.
 * Arguments are checked before the handle is used; ngroups == 0 does nothing.  Enqueued on `stream` (NULL = the
 * matcher's stream), not synchronised. */
int orbfe_distinctive_descriptors_device(OrbfeMatcher *m, int ngroups, const uint8_t *d_desc, const int *d_counts,
                                         int nframes, int cap, const int32_t *d_group_ptr, const int32_t *d_obs, int nobs,
                                         int32_t *d_best, uint8_t *d_mp_desc, void *stream);

/* MapPoint::UpdateNormalAndDepth (MapPoint.cc:273-312) for npoints map points at once, on the observation lists of
 * orbfe_distinctive_descriptors_device: the frame store d_kps / d_counts (frame f at f*cap, `nframes` frames), point g owns
 * the slots d_obs[d_group_ptr[g] .. d_group_ptr[g+1]) (npoints + 1 pointers, `nobs` observations) in mObservations
 * iteration order.  Unlike ComputeDistinctiveDescriptors the reference counts EVERY observation, those in bad keyframes
 * included, so the same list serves both only when it has none of those.
 *   d_centers: 3 floats per frame row, KeyFrame::GetCameraCenter() of the keyframe in that row.
 *   d_world:   3 floats per point, MapPoint::GetWorldPos().
 *   d_ref_obs: per point the slot of its reference keyframe's observation, slot(mpRefKF)*cap + observations[mpRefKF].  Where
 *              mpRefKF is not among the observations the reference's map lookup reads index 0: pass slot(mpRefKF)*cap + 0.
 *   scale_factor = KeyFrame::GetScaleFactor(), scale_factors = the nlevels floats of GetScaleFactor(l) (host arrays, shared
 *   by the keyframes of one extractor, as sigma2 is in orbfe_search_for_triangulation_device).
 * Outputs, per point g: d_normal[3g..3g+2] = mNormalVector, d_min_dist[g] = mfMinDistance, d_max_dist[g] = mfMaxDistance,
 * bit for bit the values the reference computes with OpenCV 2.4 (the rule is in DESIGN.md §2: a float scaleAdd chain in list
 * order, (float)(1.0/n) for the mean, cv::norm in double).  A point on an observer's camera centre has a NaN normal, as in
 * the reference (its NaN payload may differ); a point on its reference centre has both distances 0.
 * An empty group is left untouched (the reference returns early for a bad map point and keeps its values): pass a bad map
 * point as an empty group or leave it out.  Bad input is never followed: a point with d_group_ptr[g] < 0,
 * d_group_ptr[g] > d_group_ptr[g+1], d_group_ptr[g+1] > nobs, an observation or reference slot whose frame is >= nframes or
 * whose feature index is >= d_counts[f], or a reference octave outside [0, nlevels), keeps its outputs untouched, and
 * orbfe_matcher_sync then reports ORBFE_ERR_ARG; the other points of the launch are unaffected.  One warp per map point.
 * npoints >= 0, nobs >= 0, 1 <= cap <= 65535, nframes >= 1, nframes*cap < 2^31, 1 <= nlevels <= ORBFE_MAX_LEVELS.
 * Arguments are checked before the handle is used; npoints == 0 does nothing.  Enqueued on `stream` (NULL = the matcher's
 * stream), not synchronised. */
int orbfe_normal_and_depth_device(OrbfeMatcher *m, int npoints, const OrbfeKeyPoint *d_kps, const int *d_counts, int nframes, int cap,
                                  const float *d_centers, const int32_t *d_group_ptr, const int32_t *d_obs, int nobs,
                                  const float *d_world, const int32_t *d_ref_obs, float scale_factor, int nlevels,
                                  const float *scale_factors, float *d_normal, float *d_min_dist, float *d_max_dist, void *stream);

/* orbfe_normal_and_depth_device for callers without a frame store (e.g. the recovery loops after a bundle adjustment), all
 * host arrays: per point g its world position world[3g..], its reference keyframe's camera centre ref_centers[3g..] and the
 * octave of the reference keyframe's observed keypoint ref_octave[g]; the camera centres of its observers are rows
 * group_ptr[g] .. group_ptr[g+1] of obs_centers (3 floats each, mObservations order; group_ptr[0] = 0, non-decreasing).
 * The outputs and the rule are those of the device form; the rows of an empty group are returned as passed.  ORBFE_ERR_ARG,
 * before the handle is used, for a bad group_ptr or a non-empty point whose ref_octave is outside [0, nlevels).  Staged
 * through the matcher's block, one launch of the same kernel, synchronous. */
int orbfe_normal_and_depth(OrbfeMatcher *m, int npoints, const float *world, const float *ref_centers, const int32_t *ref_octave,
                           const int32_t *group_ptr, const float *obs_centers, float scale_factor, int nlevels, const float *scale_factors,
                           float *normal_out, float *min_dist_out, float *max_dist_out);

/* KeyFrameDatabase::DetectLoopCandidates (mode 0, KeyFrameDatabase.cc:73-195) / DetectRelocalisationCandidates (mode 1,
 * :197-308) with the database as arrays.  Keyframe k (k = 0..nkf-1, in the order the keyframes were add()ed: that is
 * the order inside every inverted-file list) owns the BowVector db_ids/db_vals[kf_ptr[k] .. kf_ptr[k+1]) (word ids
 * ascending); the query BowVector is q_ids/q_vals (ascending).  connected[k] != 0 marks the query keyframe's
 * GetConnectedKeyFrames() (mode 0 only, may be NULL); covis/covis_ptr hold GetBestCovisibilityKeyFrames(10) of every
 * keyframe in the order that call returns them.  min_score: the minScore argument (mode 0 only).
 * One device thread per keyframe walks the two sorted word lists (shared-word count, first shared word, and the L1
 * score accumulated in ascending word order exactly as L1Scoring::score does); thresholds, the covisibility
 * accumulation and the candidate list are replayed on the host in the reference's list order.
 * cand_out (capacity nkf) receives *ncand_out keyframe indices in the order of the returned vector.  common_out /
 * score_out (capacity nkf each, may be NULL) receive mnLoopWords / the float score of every keyframe that shares a word
 * (score = -1 where the reference does not compute one). */
int orbfe_bow_db_detect(OrbfeMatcher *m, int mode, int nq, const int32_t *q_ids, const double *q_vals, int nkf,
                        const int32_t *kf_ptr, const int32_t *db_ids, const double *db_vals, const uint8_t *connected,
                        const int32_t *covis_ptr, const int32_t *covis, float min_score, int *ncand_out, int32_t *cand_out,
                        int32_t *common_out, float *score_out);

/* KeyFrameDatabase (reference src/KeyFrameDatabase.cc) as a long-lived object resident in device memory: the inverted file,
 * the keyframes' BowVectors, their best-covisibility lists and their query fields (mnLoopQuery, mnLoopWords, mLoopScore,
 * mnRelocQuery, mnRelocWords, mRelocScore; KeyFrame.h:160-165) live on the device, so a query costs the postings of its
 * words and its results equal the reference's over any sequence of calls (mRelocScore of a keyframe that shares too few
 * words with this frame is the one an earlier query left, :272-281).  A keyframe is a caller-chosen slot
 * 0 <= slot < max_keyframes (e.g. its frame-store index, so candidates go straight to orbfe_search_by_bow_device as d_idx).
 * Arguments are checked before the handle is used.  One call at a time per handle (the reference serialises these calls
 * with mMutex); every call is ordered after the handle's previous work whatever stream that was enqueued on. */
typedef struct OrbfeKeyFrameDB OrbfeKeyFrameDB;

/* KeyFrameDatabase(voc) (:32-36).  Word ids are checked against the vocabulary's word count (largest word id + 1); the
 * device is the vocabulary's.  Every buffer is allocated here (about 44 bytes per posting, 8 per vocabulary word and
 * 150 per slot); no later call allocates device memory. */
int orbfe_kfdb_create(OrbfeVocabulary *v, int max_keyframes, long long max_postings, OrbfeKeyFrameDB **out);
/* orbfe_kfdb_create with room for batches of up to max_queries queries (1 <= max_queries <= 1024, else ORBFE_ERR_ARG);
 * orbfe_kfdb_create is this call with max_queries = 1.  Every buffer is still allocated here: each query slot adds
 * 40 * max_keyframes + 12 * S + 16 bytes of device memory, S = max_keyframes rounded up to a power of two (per query: the
 * query state, connected stamps, touched list, scores, accumulations, best covisibles and first-entry tags of every slot,
 * and the sorted sharing list). */
int orbfe_kfdb_create_batched(OrbfeVocabulary *v, int max_keyframes, long long max_postings, int max_queries, OrbfeKeyFrameDB **out);
void orbfe_kfdb_destroy(OrbfeKeyFrameDB *db);

/* add(pKF) (:39-45): the BowVector ids/vals[0, nw) (word ids strictly ascending, < the vocabulary's word count) of a NEW
 * keyframe in an empty slot; it goes to the end of every word's list.  Its query fields start as a fresh KeyFrame's:
 * stamps 0, scores 0.  An occupied slot gives ORBFE_ERR_ARG; more than max_postings words in the database gives
 * ORBFE_ERR_CAPACITY; in both cases the database is unchanged.  The covisibility list of the slot is left as it is.
 * Synchronous. */
int orbfe_kfdb_add(OrbfeKeyFrameDB *db, int slot, int nw, const int32_t *ids, const double *vals);
/* n calls of orbfe_kfdb_add, in order i, with the BowVectors read where orbfe_bow_vector_device left them: keyframe slots[i]
 * gets the d_bow_n[f] words of row f = frames[i] of d_bow_ids / d_bow_vals (row f at f*cap).  slots and frames are host
 * arrays; the rows are on the database's device and frame indices are not bounds-checked.  All or nothing: slots out of
 * range, repeated or occupied, a negative frame, cap outside 1 .. ORBFE_FV_MAX_CAP, or a named row whose count is outside
 * 0 .. cap or whose ids are not strictly ascending below the vocabulary's word count give ORBFE_ERR_ARG; more than
 * max_postings words in the database gives ORBFE_ERR_CAPACITY; in every case the database is unchanged.  The rows are
 * checked on the device and only their counts come back to the host.  Ordered after the work already on `stream`
 * (NULL = the handle's stream); synchronous. */
int orbfe_kfdb_add_device(OrbfeKeyFrameDB *db, int n, const int32_t *slots, const int32_t *frames, int cap, const int32_t *d_bow_ids,
                          const double *d_bow_vals, const int *d_bow_n, void *stream);
/* erase(pKF) (:47-66): the keyframe leaves every word's list, its postings become free for later adds, and its covisibility
 * list is emptied.  Erasing an empty slot does nothing, as in the reference.  Synchronous. */
int orbfe_kfdb_erase(OrbfeKeyFrameDB *db, int slot);
/* clear() (:68-72): every slot becomes empty. Synchronous. */
int orbfe_kfdb_clear(OrbfeKeyFrameDB *db);
/* Replaces the best-covisibility lists (GetBestCovisibilityKeyFrames(10), read at :150 and :264) of n distinct slots: slot
 * slots[i] gets lists[ptr[i] .. ptr[i+1]) (ptr[0] = 0, at most 10 slot ids each, in the order that call returns).  Refresh
 * the new keyframe and its neighbours after KeyFrame::UpdateConnections.  An entry that names an empty slot contributes
 * nothing (an empty slot is never touched by a query).  Synchronous. */
int orbfe_kfdb_set_covisibles(OrbfeKeyFrameDB *db, int n, const int32_t *slots, const int32_t *ptr, const int32_t *lists);
/* orbfe_kfdb_set_covisibles with the lists read where orbfe_covis_lists_device (which = 0) wrote them: slot slots[i] (a host
 * array, checked as in the host form) gets the first 10 entries of d_lists[d_ptr[i] .. d_ptr[i+1]), so a whole export with
 * any nbest passes as it is.  A negative entry, or one >= max_keyframes, keeps its place among the 10 and contributes
 * nothing: it is the reference's bad keyframe, still in the list but never touched by a query.  A row whose range is
 * negative is empty.  Enqueued on `stream` (NULL = the handle's stream), ordered after the handle's previous work, not
 * synchronised; one launch. */
int orbfe_kfdb_set_covisibles_device(OrbfeKeyFrameDB *db, int n, const int32_t *slots, const int32_t *d_ptr, const int32_t *d_lists,
                                     void *stream);
/* Number of occupied slots and of postings held (either pointer may be NULL). */
int orbfe_kfdb_size(OrbfeKeyFrameDB *db, int *nkeyframes, long long *npostings);

/* DetectLoopCandidates (mode 0, :75-196; `connected` = the query keyframe's GetConnectedKeyFrames() as slots, min_score =
 * minScore) / DetectRelocalisationCandidates (mode 1, :198-308; connected and min_score unused).  Every call is a new query
 * id.  The query BowVector q_ids/q_vals[0, nq) has word ids strictly ascending, nq <= 65535.  cand_out receives the
 * candidate slots in the order of the returned vector.  words_out / score_out (max_keyframes entries each, may be NULL)
 * receive mnLoopWords / mnRelocWords and mLoopScore / mRelocScore of every slot this query touched (shares a word with it),
 * -1 elsewhere.  More than `cap` candidates: ORBFE_ERR_CAPACITY with the number needed in *ncand_out.
 * Host pointers, synchronous; a thin wrapper over orbfe_kfdb_detect_device. */
int orbfe_kfdb_detect(OrbfeKeyFrameDB *db, int mode, int nq, const int32_t *q_ids, const double *q_vals, int nconn, const int32_t *connected,
                      float min_score, int cap, int32_t *cand_out, int *ncand_out, int32_t *words_out, float *score_out);
/* The same query with device arrays: d_q_ids / d_q_vals / d_connected in, d_cand (cap entries), *d_ncand (the number of
 * candidates; when it exceeds cap only the first cap were written), d_words / d_score (max_keyframes entries each, may
 * be NULL) out.  Word ids out of the vocabulary's range are skipped.  In particular, entries after the last real word whose
 * id is >= the vocabulary's word count are ignored: a padded row of orbfe_bow_vector_device passed whole (nq = cap) gives
 * the same candidates, words and scores, and leaves the same mLoopScore / mRelocScore, as its d_bow_n[f] real words, so
 * the host never needs the word count.  Enqueued on `stream` (NULL = the handle's stream), not synchronised: five
 * kernels, no host round trip. */
int orbfe_kfdb_detect_device(OrbfeKeyFrameDB *db, int mode, int nq, const int32_t *d_q_ids, const double *d_q_vals, int nconn,
                             const int32_t *d_connected, float min_score, int cap, int32_t *d_cand, int *d_ncand, int32_t *d_words,
                             float *d_score, void *stream);

/* nqueries queries of one mode in one launch chain, with the results of nqueries consecutive orbfe_kfdb_detect_device
 * calls made in order b = 0 .. nqueries-1, bit for bit: query b gets the b-th of nqueries consecutive query ids, and its
 * candidates, counts, words and scores, and the mLoopScore / mRelocScore left for later calls, are those calls'.  In
 * particular, a slot query b touched but did not score (too few shared words, or connected in loop mode) keeps the score
 * the last query a < b of the batch that scored it computed, or the score from before the batch when none did; that is
 * the value query b reports in d_score and, in relocalisation mode, adds into its covisibility accumulation
 * (KeyFrameDatabase.cc:272-281).  No query sees a score of a later query of its batch.  After the batch, every slot
 * scored in it holds the score of the last query that scored it.
 *   Query b is row b of d_q_ids / d_q_vals (entries b*qcap .. b*qcap+qcap-1, ids ascending); entries after the real words
 *   with ids >= the vocabulary's word count are ignored, so a block of orbfe_bow_vector_device rows is passed as it is with
 *   qcap = its cap.  Loop mode (0): query b's connected slots are d_connected[d_conn_ptr[b] .. d_conn_ptr[b+1])
 *   (nqueries + 1 non-decreasing offsets; d_connected may be NULL when every range is empty) and its minScore is
 *   d_min_score[b]; these are device arrays, so a minimum computed on the device can feed them.  Relocalisation mode (1):
 *   all three unused, may be NULL.
 *   Out: row b of d_cand at b*cap (cap entries), d_ncand[b] (the number of candidates; when it exceeds cap only the first
 *   cap were written), and rows b of d_words / d_score at b*max_keyframes (may be NULL), as orbfe_kfdb_detect_device.
 * 1 <= nqueries <= the handle's max_queries, 0 <= qcap <= 65535, cap >= 0; anything else is ORBFE_ERR_ARG and leaves the
 * database unchanged.  Enqueued on `stream` (NULL = the handle's stream), ordered after the handle's previous work like
 * every orbfe_kfdb_* call, not synchronised: six kernels whatever nqueries, no host round trip.
 * A batch of loop queries equals the reference only when no add() falls between them: LoopClosing::DetectLoop adds each
 * keyframe to the database after its own query (LoopClosing.cc:134,209), so consecutive loop queries of the reference
 * see one more keyframe each. */
int orbfe_kfdb_detect_batch_device(OrbfeKeyFrameDB *db, int mode, int nqueries, int qcap, const int32_t *d_q_ids, const double *d_q_vals,
                                   const int32_t *d_conn_ptr, const int32_t *d_connected, const float *d_min_score, int cap,
                                   int32_t *d_cand, int *d_ncand, int32_t *d_words, float *d_score, void *stream);

/* The covisibility graph of one map (KeyFrame::UpdateConnections, AddConnection, UpdateBestCovisibles, EraseConnection and
 * the connection half of SetBadFlag; reference src/KeyFrame.cc:126-185, 332-421, 497-521, 596-610) resident in device
 * memory, so the loop and relocalisation queries read their covisibility lists without host lists.
 *   A keyframe is a slot 0 <= slot < max_keyframes equal to its frame-store row: the slot convention of orbfe_kfdb_* and
 *   orbfe_bow_min_score_device, so exported lists go straight into those calls.
 *   Each slot carries a caller-given 64-bit order key, (uintptr_t)pKF in an integration: every std::map iteration and every
 *   tie of the reference (pointer order) is taken in key order.
 * Arguments are checked before the handle is used.  One call at a time per handle; every call is ordered after the
 * handle's previous work whatever stream that was enqueued on. */
typedef struct OrbfeCovisGraph OrbfeCovisGraph;

/* Every buffer is allocated here; no later call allocates.  max_connections: the capacity of one keyframe's weight map,
 * 1 .. 2048; max_batch: the most keyframes per update call, 1 .. 1024; 1 <= max_keyframes <= 2^24 and
 * max_keyframes * max_connections < 2^31.  About 16 * max_connections + 60 bytes of device memory per slot and
 * 24 * max_connections per batch entry. */
int orbfe_covis_create(int device, int max_keyframes, int max_connections, int max_batch, OrbfeCovisGraph **out);
void orbfe_covis_destroy(OrbfeCovisGraph *g);

/* n new keyframes (host arrays): slot slots[i], mnId ids[i] (only ids[i] == 0 matters: such a keyframe gets no parent and
 * is never erased) and order key keys[i].  Every uint64_t is a valid key, 0 and 2^64 - 1 included.  Each starts as a fresh
 * KeyFrame: no weights, empty lists, mbFirstConnection.
 * All or nothing, ORBFE_ERR_ARG: a slot out of range, live or listed twice, a key equal to a live slot's key or repeated,
 * a retired slot that some weight map still names (re-adding it would alias the reference's stale pointer), or a key equal
 * to the key of such a retired slot (the reference never reuses a bad KeyFrame's pointer; the new keyframe would merge
 * onto the stale entry).  The check reads the host's copy of the keys and the same copy of the name counts as the check
 * before it.  Synchronous. */
int orbfe_covis_add(OrbfeCovisGraph *g, int n, const int32_t *slots, const int32_t *ids, const uint64_t *keys);

/* UpdateConnections() of the keyframes slots[0..n) (a host array of distinct live slots, 1 <= n <= max_batch; n = 0 does
 * nothing): the graph afterwards equals n consecutive reference calls in that order, bit for bit.
 *   d_kf_mp[s*cap + i] (i < d_counts[s]) is the map-point index at feature i of keyframe s: -1 (any negative) where
 *   mvpMapPoints[i] is NULL or isBad().  A point at two features counts twice, as in the reference.
 *   Point g's observations are d_obs[d_group_ptr[g] .. d_group_ptr[g+1]): the flat slots f*cap + i of
 *   orbfe_normal_and_depth_device (every observation counts; the frame f is the observing keyframe's slot).
 *   parent_out (device, n entries, may be NULL): parent_out[i] = the slot call i made mpParent (its first non-empty call,
 *   mnId != 0: the front of its ordered list), else -1.
 * Bad input rejects the whole batch and leaves the graph unchanged: d_counts[s] outside 0 .. cap, a point index >= npoints,
 * a group with d_group_ptr[g] < 0, d_group_ptr[g] > d_group_ptr[g+1] or d_group_ptr[g+1] > nobs, or an observation whose
 * frame is >= nframes or not a live slot; orbfe_covis_sync then reports ORBFE_ERR_ARG.  A weight map that would exceed
 * max_connections also rejects the whole batch unchanged; orbfe_covis_sync then reports ORBFE_ERR_CAPACITY.  Both are
 * decided on the device.  Host-side ORBFE_ERR_ARG: a slot not live, >= nframes or repeated, nframes < 1, cap < 1,
 * nframes*cap >= 2^31, npoints < 0, nobs < 0, a NULL array.
 * Enqueued on `stream` (NULL = the handle's stream), not synchronised: three launches, no host round trip.
 * A batch is n reference calls with nothing read in between: LoopClosing.cc:484-490's loop and the initial map's pair
 * (Tracking.cc:430-431).  Where the reference reads the graph between calls (CorrectLoop's second loop, :521-536), run
 * batches of one. */
int orbfe_covis_update_connections_device(OrbfeCovisGraph *g, int n, const int32_t *slots, const int32_t *d_kf_mp, const int *d_counts,
                                          int nframes, int cap, const int32_t *d_group_ptr, const int32_t *d_obs, int npoints, int nobs,
                                          int32_t *parent_out, void *stream);

/* SetBadFlag's connection half (KeyFrame.cc:497-521): every keyframe in the slot's own weight map gets EraseConnection
 * (:596-610: the entry erased, then all its weights re-sorted); the slot's weights and lists are cleared and the slot is
 * retired.  mnId == 0, or a slot that is not live, does nothing.  A weight map naming the slot that the slot's own map
 * does not name keeps its stale entry, as in the reference.  The spanning tree is not kept here.  Synchronous. */
int orbfe_covis_erase(OrbfeCovisGraph *g, int slot);
/* Every slot becomes empty (Tracking's reset).  Synchronous. */
int orbfe_covis_clear(OrbfeCovisGraph *g);

/* CSR lists of the n host-named slots (0 <= slots[i] < max_keyframes, repeats allowed):
 *   which = 0: GetBestCovisibilityKeyFrames(nbest), or the whole GetVectorCovisibleKeyFrames() when nbest <= 0, with
 *              mvOrderedWeights;
 *   which = 1: GetConnectedKeyFrames() in key order, with the weights of mConnectedKeyFrameWeights (nbest unused).
 * d_ptr (n + 1 entries) is an exclusive scan computed on the device; d_list and d_weights (may be NULL) hold up to
 * n x the row limit entries, the limit being min(nbest, max_connections) for which = 0 with nbest > 0, else
 * max_connections.  A retired slot in a list is written as -1 (the isBad -> negative convention of
 * orbfe_bow_min_score_device; orbfe_kfdb_detect_* ignore entries outside [0, max_keyframes)).  Enqueued on `stream` (NULL
 * = the handle's stream), not synchronised; two launches. */
int orbfe_covis_lists_device(OrbfeCovisGraph *g, int which, int n, const int32_t *slots, int nbest, int32_t *d_ptr, int32_t *d_list,
                             int32_t *d_weights, void *stream);

/* MapPoint::GetObservations() (reference src/MapPoint.cc:93-97) of the n named points d_points[0..n), built on the device as
 * the inverse of the live slots' map-point rows.  The reference keeps mObservations and mvpMapPoints in step (AddMapPoint /
 * AddObservation, EraseMapPointMatch / EraseObservation, Replace, both SetBadFlags), so at every call boundary a point's
 * observations are the live keyframes whose row names it.
 *   Observers: the live slots (added, not erased).  Slot s's row is d_kf_mp[s*cap + i], i < d_counts[s], as in
 *   orbfe_covis_update_connections_device: a negative value is NULL or isBad().  A keyframe is an observer from its
 *   orbfe_covis_add on, so add it when its observations are added (Tracking's initial pair, the start of ProcessNewKeyFrame),
 *   not while it waits in LocalMapping's queue.
 *   List of p = d_points[j]: one entry per live slot whose row names p, written s*cap + i.  A row naming p at several
 *   features gives the largest i (ProcessNewKeyFrame's mObservations[pKF] = i runs in ascending i).  Entries are in key
 *   order, ascending: the std::map order.  Point j's entries are d_obs[d_ptr[j] .. d_ptr[j+1]); d_ptr (n + 1 entries) is an
 *   exclusive scan and *d_nobs the total, so (d_ptr, d_obs) is exactly the d_group_ptr / d_obs of
 *   orbfe_distinctive_descriptors_device, orbfe_normal_and_depth_device and orbfe_covis_update_connections_device.
 *   d_ref_slot / d_ref_obs (n entries each, both or neither when n > 0): d_ref_obs[j] = ref*cap + i for ref = d_ref_slot[j] (the slot of
 *   mpRefKF) and i its entry in the list, else ref*cap + 0 (observations[pRefKF] inserts 0): the d_ref_obs of
 *   orbfe_normal_and_depth_device.
 * A total over obs_cap writes d_ptr and *d_nobs (the size needed) and nothing else; orbfe_covis_sync then reports
 * ORBFE_ERR_CAPACITY.  Decided on the device, with only d_ptr written and ORBFE_ERR_ARG from orbfe_covis_sync: a named point
 * outside [0, npoints) or named twice, a live slot's d_counts[s] outside 0 .. cap, a row value >= npoints, a reference slot
 * outside [0, nframes).  Host-side ORBFE_ERR_ARG: n < 0, n > npoints, nframes < 1, cap < 1, nframes*cap >= 2^31, obs_cap < 0,
 * a live slot >= nframes, a NULL array (d_points may be NULL when n = 0, d_obs when obs_cap = 0) or one of d_ref_slot /
 * d_ref_obs without the other when n > 0, d_scratch not 4-byte aligned;
 * cap > ORBFE_COVIS_OBS_MAX_CAP is ORBFE_ERR_UNSUPPORTED.
 * d_scratch: ORBFE_COVIS_OBS_SCRATCH_BYTES(npoints, nframes, cap, obs_cap) bytes of device memory, contents ignored; the call
 * allocates nothing.  The graph is only read.  Enqueued on `stream` (NULL = the handle's stream) after the handle's previous
 * work, not synchronised: five launches, no host round trip. */
#define ORBFE_COVIS_OBS_MAX_CAP 8192
#define ORBFE_COVIS_OBS_SCRATCH_BYTES(npoints, nframes, cap, obs_cap) (4 * (2 * (size_t)(npoints) + (size_t)(obs_cap)))
int orbfe_covis_observations_device(OrbfeCovisGraph *g, int n, const int32_t *d_points, int npoints, const int32_t *d_kf_mp,
                                    const int *d_counts, int nframes, int cap, const int32_t *d_ref_slot, int obs_cap, int32_t *d_ptr,
                                    int32_t *d_obs, int *d_nobs, int32_t *d_ref_obs, void *d_scratch, void *stream);

/* LocalMapping::KeyFrameCulling() (reference src/LocalMapping.cc:524-578) for the current keyframe `current_slot`, with the
 * map-point half of every KeyFrame::SetBadFlag it calls (EraseObservation and MapPoint::SetBadFlag, MapPoint.cc:71-122).
 *   The list is current_slot's GetVectorCovisibleKeyFrames() as the graph holds it, taken once; entry t is decided after
 *   the erases of entries 0 .. t-1, as in the reference.  A stale entry (a retired slot the list still names, -1 in
 *   orbfe_covis_lists_device) is evaluated on its unchanged row.  Rows, d_counts and d_kps (frame-store rows of cap
 *   OrbfeKeyPoint, octave = GetKeyPointUn(i).octave) are those of orbfe_covis_observations_device; a point's observers are
 *   the live slots whose rows name it, each at its largest feature index.
 *   d_point_bad[npoints] (in/out): MapPoint::isBad(); d_ref_slot[npoints] (in/out): the slot of mpRefKF.
 *   not_erase_slots (host, n_not_erase entries): the keyframes with mbNotErase.
 * Outputs, one entry per list position t < *d_ncand (at most max_connections): d_verdict_slot[t] the entry's slot (the
 * true slot for a stale entry), d_verdict[t] one of ORBFE_CULL_*, d_nmps[t] / d_nredundant[t] (both may be NULL) nMPs and
 * nRedundantObservations (0 for a skipped entry).  d_bad_points[0 .. *d_nbad) are the points this call made bad, ascending.
 * Writes on success: d_point_bad and d_ref_slot of the points the erases touched (a point left without observers goes bad
 * with its d_ref_slot unwritten: the reference's read there is undefined); in the rows of the slots live at the call, every
 * cell that names a point made bad while the slot was its observer becomes -1, duplicate cells included (the reference
 * NULLs only the observation's cell; DESIGN.md §2).  An erased keyframe's row and the rows of slots that are not live stay
 * as they are.  The graph is only read: replay orbfe_covis_erase for the ERASED verdicts, in order, on the host.
 * All or nothing, decided on the device and reported by orbfe_covis_sync, with nothing written but *d_nobs: more than
 * obs_cap observation entries over all points (ORBFE_ERR_CAPACITY, *d_nobs = the number needed); a live slot's or a listed
 * slot's count outside 0 .. cap, a row value >= npoints, a listed slot >= nframes, an octave outside 0 .. ORBFE_MAX_LEVELS-1
 * of a listed keyframe's cell or of an observer of a point it names, or such a point's d_ref_slot outside [0, nframes)
 * (ORBFE_ERR_ARG).  Host-side ORBFE_ERR_ARG before the handle is used: current_slot not live or >= nframes, npoints < 0,
 * nframes < 1, cap < 1, nframes*cap >= 2^31, obs_cap < 0, n_not_erase < 0 or > max_keyframes, an mbNotErase slot outside
 * [0, nframes), a live slot >= nframes, a NULL array (d_point_bad, d_ref_slot, d_bad_points may be NULL when npoints = 0),
 * d_scratch not 4-byte aligned; cap > ORBFE_COVIS_OBS_MAX_CAP is ORBFE_ERR_UNSUPPORTED.
 * obs_cap: the call builds the observation lists of every point 0 .. npoints-1, not only of the points the listed keyframes
 * name (so it needs no host count of those points), and obs_cap bounds their total: the number of distinct (live slot,
 * point) pairs in the live rows, at most the number of non-negative cells in the live rows.  Size it for the whole map.
 * That build reads every live row twice and is most of a call with a short list (about 0.8 ms of 1.0 ms at 20 covisible
 * keyframes on a 2000-keyframe x 2000-feature map, DESIGN.md §4.8).
 * d_scratch: ORBFE_COVIS_CULL_SCRATCH_BYTES(npoints, nframes, cap, obs_cap) bytes of device memory, contents ignored.
 * Enqueued on `stream` (NULL = the handle's stream) after the handle's previous work, not synchronised: nine launches and
 * three memsets (and the upload of not_erase_slots), no host round trip. */
#define ORBFE_CULL_KEPT 0        /* not redundant */
#define ORBFE_CULL_SKIP_ID0 1    /* mnId == 0: skipped */
#define ORBFE_CULL_ERASED 2      /* redundant: SetBadFlag erased it (its point half is done) */
#define ORBFE_CULL_NOT_ERASE 3   /* redundant, mbNotErase: SetBadFlag only sets mbToBeErased */
#define ORBFE_CULL_RETIRED 4     /* redundant, already retired: SetBadFlag again changes no point */
#define ORBFE_COVIS_CULL_SCRATCH_BYTES(npoints, nframes, cap, obs_cap) \
    (4 * (6 * (size_t)(npoints) + 1 + 2 * (size_t)(obs_cap) + 2 * (size_t)(nframes) + 8) + (size_t)(obs_cap))
int orbfe_covis_keyframe_culling_device(OrbfeCovisGraph *g, int current_slot, int32_t *d_kf_mp, const int *d_counts,
                                        const OrbfeKeyPoint *d_kps, int nframes, int cap, uint8_t *d_point_bad, int32_t *d_ref_slot,
                                        int npoints, int n_not_erase, const int32_t *not_erase_slots, int obs_cap, int *d_nobs,
                                        int32_t *d_verdict_slot, int32_t *d_verdict, int *d_ncand, int32_t *d_nmps,
                                        int32_t *d_nredundant, int32_t *d_bad_points, int *d_nbad, void *d_scratch, void *stream);

/* Tracking::UpdateReference() (reference src/Tracking.cc:728-839) for one frame: UpdateReferenceKeyFrames and
 * UpdateReferencePoints on the graph and the keyframes' rows.  SetReferenceMapPoints (visualisation) stays with the caller.
 *   d_frame_mp[nf] (in/out): the frame's mvpMapPoints as point indices, -1 = NULL; a cell naming a point with d_point_bad
 *   set becomes -1.  d_point_bad[npoints]: MapPoint::isBad().  Rows, d_counts and the observers are those of
 *   orbfe_covis_observations_device: slot s's row is d_kf_mp[s*cap + i] for i < d_counts[s], a point's observers are the
 *   live slots whose rows name it, and a row that names a point twice is one observation.
 * Outputs:
 *   d_local_kf[0 .. *d_nlocal_kf) (capacity nframes): mvpLocalKeyFrames.  Every remaining frame cell adds 1 to each
 *     observer of its point (a point at k cells votes k times); the counted slots in key order; then, visiting only those
 *     entries and stopping before a visit once the list holds more than 80, each visit appends the first of the entry's
 *     first 10 ordered neighbours that is live and not yet listed.  A retired neighbour (stale) is skipped.
 *   *d_ref_kf: mpReferenceKF, the first strict maximum of the counter in key order (the smallest key on a tie); -1 when
 *     nothing was counted.
 *   d_local_points[0 .. *d_nlocal_points) (capacity npoints): mvpLocalMapPoints, the rows of the list's entries in list
 *     order, each in ascending i < d_counts[s], negative cells and bad points skipped, each point at its first occurrence.
 * The graph is only read.  Bad input found on the device writes nothing and is reported by orbfe_covis_sync as
 * ORBFE_ERR_ARG: a frame cell or a live row's value >= npoints, a live slot's count outside 0 .. cap.  Host-side
 * ORBFE_ERR_ARG before the handle is used: nf < 0, npoints < 0, nframes < 1, cap < 1, nframes*cap >= 2^31, a NULL array
 * (d_frame_mp may be NULL when nf = 0, d_point_bad and d_local_points when npoints = 0), d_scratch not 4-byte aligned, a
 * live slot >= nframes; cap > ORBFE_COVIS_OBS_MAX_CAP is ORBFE_ERR_UNSUPPORTED.
 * d_scratch: ORBFE_COVIS_LOCAL_MAP_SCRATCH_BYTES(npoints, nframes) bytes of device memory, contents ignored.
 * Enqueued on `stream` (NULL = the handle's stream) after the handle's previous work, not synchronised: six launches and
 * two memsets, no host round trip. */
#define ORBFE_COVIS_LOCAL_MAP_SCRATCH_BYTES(npoints, nframes) (4 * (2 * (size_t)(npoints) + 4 * (size_t)(nframes) + 5))
int orbfe_covis_local_map_device(OrbfeCovisGraph *g, int nf, int32_t *d_frame_mp, const uint8_t *d_point_bad, int npoints,
                                 const int32_t *d_kf_mp, const int *d_counts, int nframes, int cap, int32_t *d_local_kf,
                                 int *d_nlocal_kf, int32_t *d_ref_kf, int32_t *d_local_points, int *d_nlocal_points,
                                 void *d_scratch, void *stream);

/* Waits for the handle's work and returns the first device-side error since the last sync (ORBFE_OK when none). */
int orbfe_covis_sync(OrbfeCovisGraph *g);

#ifdef __cplusplus
}
#endif
#endif /* ORBFE_BOW_H */
