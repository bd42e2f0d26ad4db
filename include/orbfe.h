/*
 * orbfe.h -- C-ABI of liborbfe.so, the H100-native ORB feature front-end (extract + match).
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++/torch types.  The reference has no
 * FFI layer (its boundary is two C++ classes, include/ORBextractor.h:32-77 and include/ORBmatcher.h:37-107
 * of raulmur/ORB_SLAM); the C++ facades in orb_slam_b200/host/ re-create those classes on top of the
 * functions below, and INTEGRATION.md shows the binding a maintainer adds on the reference side.
 *
 * Conventions: every function returns an OrbfeStatus (0 = ok, negative = error); nothing throws across
 * the ABI; a handle owns all of its device memory and its CUDA stream; there is NO CPU fallback -- if
 * no CUDA device is usable the create functions fail with ORBFE_ERR_NO_DEVICE.
 * Threading: one in-flight call per extractor handle (the reference's extractor is not re-entrant either,
 * ORBextractor.h:74-75); matcher handles are independent (one per calling thread).  Calls on one handle run in call order,
 * whichever streams they are enqueued on: a call's stream waits for the handle's previous call, so two pending calls
 * never share the handle's work buffers, and the handle's sync and read-back functions see its most recent call.
 */
#ifndef ORBFE_H
#define ORBFE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ORBFE_VERSION 1
#define ORBFE_MAX_LEVELS 32

typedef enum {
    ORBFE_OK = 0,
    ORBFE_ERR_ARG = -1,         /* null pointer / non-positive size / bad enum */
    ORBFE_ERR_UNSUPPORTED = -2, /* geometry outside the supported domain (degenerate cell grid, see DESIGN.md) */
    ORBFE_ERR_CAPACITY = -3,    /* caller buffer too small; *n_out holds the needed size */
    ORBFE_ERR_CUDA = -4,        /* a CUDA call failed; orbfe_last_error() has the text */
    ORBFE_ERR_NO_DEVICE = -5,   /* no usable CUDA device: there is no CPU path */
    ORBFE_ERR_INTERNAL = -6     /* device-side overflow flag (should never happen) */
} OrbfeStatus;

/* Same field order and size (28 bytes) as cv::KeyPoint: pt.x pt.y size angle response octave class_id.
 * Filled exactly as ORBextractor.cc:689-694,705,769-775 fills them. */
typedef struct {
    float x, y, size, angle, response;
    int32_t octave, class_id;
} OrbfeKeyPoint;

typedef struct OrbfeExtractor OrbfeExtractor;
typedef struct OrbfeMatcher OrbfeMatcher;

/* thread-local text of the last failing call on this thread */
const char *orbfe_last_error(void);
int orbfe_version(void);
/* number of CUDA devices (0 if none / no driver) */
int orbfe_device_count(void);

/* ---------------------------------------------------------------------------------------------
 * Extractor -- replaces ORBextractor::ORBextractor (src/ORBextractor.cc:457-511)
 * score_type: 0 = HARRIS_SCORE, 1 = FAST_SCORE (ORBextractor.h:37).
 * ------------------------------------------------------------------------------------------- */
int orbfe_extractor_create(int nfeatures, float scale_factor, int nlevels, int score_type, int fast_th,
                           int device, OrbfeExtractor **out);
int orbfe_extractor_destroy(OrbfeExtractor *ex);

/* GetLevels / GetScaleFactor (ORBextractor.h:47-51) */
int orbfe_extractor_levels(const OrbfeExtractor *ex);
float orbfe_extractor_scale_factor(const OrbfeExtractor *ex);
/* ctor tables (mvScaleFactor, mvInvScaleFactor, mnFeaturesPerLevel), nlevels entries each; any may be NULL */
int orbfe_extractor_tables(const OrbfeExtractor *ex, float *scale, float *inv_scale, int *quota);

/* ORBextractor::operator() (src/ORBextractor.cc:718-779) on one HOST image, synchronous.
 * img: H rows of W u8 pixels, `stride` bytes apart.  kps/desc: caller buffers for `cap` keypoints
 * (desc = cap x 32 bytes).  *n_out = number of keypoints.  Empty image (NULL or W/H<=0) -> ORBFE_OK, *n_out=0,
 * like the reference's silent return (:721-722).  Keypoints come out level-ascending; inside a level in
 * cell-row-major then raster order (the canonical order, DESIGN.md). */
int orbfe_extract(OrbfeExtractor *ex, const uint8_t *img, int width, int height, size_t stride,
                  OrbfeKeyPoint *kps, uint8_t *desc, int cap, int *n_out);

/* Batched form: `batch` independent frames of identical geometry per call (frames of a stream / cameras
 * of a rig).  HOST buffers: imgs = batch images `frame_stride` bytes apart; outputs are batch blocks of
 * `cap` keypoints / cap*32 descriptor bytes; n_out[batch].  H2D, kernels and D2H are pipelined on the
 * handle's streams; returns when all outputs are in host memory. */
int orbfe_extract_batch(OrbfeExtractor *ex, const uint8_t *imgs, int width, int height, size_t stride,
                        size_t frame_stride, int batch, OrbfeKeyPoint *kps, uint8_t *desc, int cap, int *n_out);

/* Device-resident form: inputs and outputs are DEVICE pointers on the handle's device; work is enqueued
 * on `stream` (a cudaStream_t, NULL = the handle's own stream) and NOT synchronised.
 * d_kps: batch x nfeatures OrbfeKeyPoint; d_desc: batch x nfeatures x 32; d_counts: batch ints. */
int orbfe_extract_batch_device(OrbfeExtractor *ex, const uint8_t *d_imgs, int width, int height, size_t stride,
                               size_t frame_stride, int batch, OrbfeKeyPoint *d_kps, uint8_t *d_desc,
                               int *d_counts, void *stream);
/* Mixed geometries: frames of up to ORBFE_MULTI_MAX_GROUPS image geometries (a rig whose cameras differ in resolution) in
 * one launch chain, as long as one group's (nlevels + 4 kernels, whatever ngroups is).  Frames are numbered group by group
 * in the order of `groups`; frame f of the call is at f * cap (host form: kps, desc, n_out[total frames]) or
 * f * nfeatures (device form: d_kps, d_desc, d_counts), as orbfe_extract_batch* lays out a batch.  Per frame, keypoints,
 * descriptors, count and order are those of orbfe_extract_batch_device with that frame's geometry.  A group with a NULL
 * image or W/H <= 0 yields zero keypoints for its `batch` frames.  Argument errors are ORBFE_ERR_ARG; a group whose
 * geometry the single-geometry entries reject gives ORBFE_ERR_UNSUPPORTED naming the group; nothing is launched then.
 * The handle keeps one plan for the single-geometry entries and one multi plan, keyed by the ordered (W, H) list of the
 * non-empty groups, holding as many frames per group as the largest call has passed: alternating single and multi calls,
 * or multi calls with the same geometry list, re-plans neither.  The limit on ngroups sizes the multi plan's level table
 * (ORBFE_MULTI_MAX_GROUPS x ORBFE_MAX_LEVELS entries) and the group scan each kernel does to place a thread block. */
#define ORBFE_MULTI_MAX_GROUPS 8
typedef struct {
    int width, height;      /* this group's geometry */
    size_t stride;          /* row stride in bytes */
    size_t frame_stride;    /* bytes between consecutive frames of the group */
    int batch;              /* frames in this group (>= 1) */
    const uint8_t *imgs;    /* host pointer (orbfe_extract_multi) or device pointer (_device) */
} OrbfeImageGroup;
int orbfe_extract_multi(OrbfeExtractor *ex, int ngroups, const OrbfeImageGroup *groups,
                        OrbfeKeyPoint *kps, uint8_t *desc, int cap, int *n_out);
int orbfe_extract_multi_device(OrbfeExtractor *ex, int ngroups, const OrbfeImageGroup *groups,
                               OrbfeKeyPoint *d_kps, uint8_t *d_desc, int *d_counts, void *stream);

/* block until the handle's calls are done, whichever streams they were enqueued on */
int orbfe_extractor_sync(OrbfeExtractor *ex);
/* number of kernels the last extract call launched (for bench.py's gpu_launches) */
int orbfe_extractor_last_launches(const OrbfeExtractor *ex);
/* number of plans (single-geometry and multi) the handle has built since it was created */
int orbfe_extractor_plan_builds(const OrbfeExtractor *ex);

/* How orbfe_extract_batch schedules a batch (default 0).
 *   0 "chunked": the upload of chunk k+1 overlaps ALL kernels of chunk k;
 *   1 "phased":  only the pyramids follow the upload chunk by chunk, detection and description then run once over the
 *                whole batch in full-size launches (for callers whose uploads are hidden behind other GPU work).
 * Results are identical in both modes; the default is chunked. */
int orbfe_extractor_set_batch_mode(OrbfeExtractor *ex, int mode);
/* With profiling on, every extract call records CUDA events around its stages on the launching stream.
 * orbfe_extractor_stage_times returns (name, ms) of every stage interval recorded since the previous read --
 * possibly from several calls -- and clears the list; the caller must have synchronised any external stream it
 * passed to orbfe_extract_batch_device.  Returns the number of intervals written (<= cap). */
int orbfe_extractor_set_profiling(OrbfeExtractor *ex, int on);
int orbfe_extractor_stage_times(const OrbfeExtractor *ex, char (*names)[32], float *ms, int cap);

/* Test hooks: copy intermediate images of frame `frame` of the last call back to the host.
 * which: 0 = unblurred pyramid level, 1 = blurred level.  out: h_l rows of w_l bytes, out_stride apart. */
int orbfe_debug_level_size(const OrbfeExtractor *ex, int level, int *w, int *h);
int orbfe_debug_read_level(OrbfeExtractor *ex, int frame, int level, int which, uint8_t *out, size_t out_stride);

/* ---------------------------------------------------------------------------------------------
 * Matcher -- the 256-bit Hamming work behind ORBmatcher::SearchBy* (src/ORBmatcher.cc).
 * The per-pair primitive is ORBmatcher::DescriptorDistance (ORBmatcher.cc:1794-1810).
 * ------------------------------------------------------------------------------------------- */
int orbfe_matcher_create(int device, OrbfeMatcher **out);
int orbfe_matcher_destroy(OrbfeMatcher *m);

/* distances of explicit (query, train) pairs in CSR order: pair k of query row i (row_ptr[i] <= k <
 * row_ptr[i+1]) is (qdesc[i], tdesc[cols[k]]); out_dist[k] in 0..256.  HOST pointers, synchronous.
 * This is the device half of every windowed Search* loop (e.g. ORBmatcher.cc:1557-1574): the host builds
 * the candidate lists with Frame::GetFeaturesInArea and replays the greedy accept loop over out_dist. */
int orbfe_hamming_csr(OrbfeMatcher *m, const uint8_t *qdesc, int nq, const uint8_t *tdesc, int nt,
                      const int32_t *row_ptr, const int32_t *cols, uint16_t *out_dist);
/* dense nq x nt distance matrix (row-major u16), HOST pointers */
int orbfe_hamming_dense(OrbfeMatcher *m, const uint8_t *qdesc, int nq, const uint8_t *tdesc, int nt,
                        uint16_t *out_dist);
/* best / second-best sweep of nq queries against a database split in `ngroups` groups of `group_size`
 * descriptors (keyframes): per (group, query) best distance, best index inside the group (first minimum,
 * strict-< update order as ORBmatcher.cc:456-466) and second-best distance.  Outputs are
 * ngroups x nq arrays.  *_device variant takes device pointers + stream and does not synchronise. */
int orbfe_knn2_groups(OrbfeMatcher *m, const uint8_t *qdesc, int nq, const uint8_t *db, int ngroups,
                      int group_size, uint16_t *best_dist, int32_t *best_idx, uint16_t *second_dist);
int orbfe_knn2_groups_device(OrbfeMatcher *m, const uint8_t *d_qdesc, int nq, const uint8_t *d_db, int ngroups,
                             int group_size, uint16_t *d_best_dist, int32_t *d_best_idx,
                             uint16_t *d_second_dist, void *stream);
/* device-pointer CSR distances, enqueued on stream (NULL = matcher's stream), not synchronised */
int orbfe_hamming_csr_device(OrbfeMatcher *m, const uint8_t *d_qdesc, const uint8_t *d_tdesc,
                             const int32_t *d_row_ptr, const int32_t *d_cols, int nq, int npairs,
                             uint16_t *d_out_dist, void *stream);
/* block until the matcher's calls are done, whichever streams they were enqueued on, and report (then clear) the error
 * flags they raised */
int orbfe_matcher_sync(OrbfeMatcher *m);
/* cumulative host<->device traffic and kernel launches of the host-pointer entry points (bench accounting); the bytes are
 * those of the staging block's uploaded and downloaded parts, every array padded to 256 bytes */
int orbfe_matcher_counters(const OrbfeMatcher *m, unsigned long long *h2d_bytes, unsigned long long *d2h_bytes,
                           unsigned long long *launches);

#ifdef __cplusplus
}
#endif
#endif /* ORBFE_H */
