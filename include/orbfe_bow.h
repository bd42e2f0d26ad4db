/* orbfe_bow.h -- C-ABI of the two "next" rows of SURVEY.md section 8(f) that reuse the 256-bit Hamming primitive:
 *
 *   N2  DBoW2 vocabulary-tree transform: descriptors -> BowVector + FeatureVector
 *       (reference Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1126-1262, FORB.cpp:79-99 (distance),
 *        BowVector.cpp:34-84, FeatureVector.cpp:32-48; callers Frame.cc:280-287, KeyFrame.cc:56-65)
 *   N3  KeyFrameDatabase::DetectLoopCandidates / DetectRelocalisationCandidates on arrays
 *       (reference src/KeyFrameDatabase.cc:73-308, L1Scoring::score Thirdparty/DBoW2/DBoW2/ScoringObject.cpp:23-67)
 *   N4  MapPoint::ComputeDistinctiveDescriptors, batched over map points (reference src/MapPoint.cc:185-250)
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

#ifdef __cplusplus
}
#endif
#endif /* ORBFE_BOW_H */
