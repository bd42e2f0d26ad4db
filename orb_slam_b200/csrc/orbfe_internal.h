// orbfe_internal.h -- structures shared by the host plan code and the sm_90a kernels of liborbfe.so.
// Not part of the public ABI (that is include/orbfe.h).
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <initializer_list>
#include <utility>
#include <vector>

#include "../../include/orbfe.h"
#include "../../include/orbfe_match.h"

#define ORBFE_EDGE 16  // EDGE_THRESHOLD, reference src/ORBextractor.cc:77

// FAST/NMS tile (detect-area pixels per CTA) and blur tile
#define ORBFE_FT_W 120
#define ORBFE_FT_H 62
// resident CTAs per SM of the FAST kernel: its launch bounds, hence its register budget (80).  3 x 80 measured faster on
// H100 than 4 x 64, which spills (DESIGN.md §4.2).
#define ORBFE_FAST_BLOCKS_PER_SM 3
#define ORBFE_BT_W 120
#define ORBFE_BT_H 64

namespace orbfe {

// One pyramid level of the current plan.  All B frames of a batch live in one allocation per level:
// frame f of level l starts at pyr + f * plane (row pitch `pitch`, a multiple of 128 B so rows are
// TMA-/vector-aligned).
struct LevelDev {
    uint8_t *pyr;   // unblurred level (level 0 = the input image)
    uint8_t *blur;  // one plane: 7x7 Gaussian of one frame's level, for orbfe_debug_read_level (the descriptor kernel smooths its own patches)
    size_t plane;   // pitch * h
    int w, h, pitch;
    // cell grid (reference ORBextractor.cc:527-547); detect windows tile [16, w-16) x [16, h-16)
    int cols, rows, cw, ch, ncells, nfc, quota;
    uint32_t cw_rcp, ch_rcp;    // ceil(2^32 / cw), ceil(2^32 / ch): n / cw == __umulhi(n, cw_rcp) exactly for 0 <= n < 2^16
    int cell_base;              // global id of this level's cell 0
    int kp_base;                // sum of quotas of lower levels = first keypoint slot of this level
    int kept_base, kept_cap;    // region of the per-frame "kept" list
    int ftiles_x, ftiles_y, ftile_base;  // FAST tiles
    int btiles_x, btiles_y, btile_base;  // blur tiles
    float scale;       // mvScaleFactor[l]
    float patch_size;  // (float)(int)(31 * scale)
    // bilinear tables for producing THIS level from level l-1 (OpenCV fixed-point, computed on the host)
    const int *xofs;      // [w]  source column (already clamped)
    const short2 *xab;    // [w]  11-bit weights (a0, a1)
    const int2 *yrows;    // [h]  source rows (r0, r1), each clipped to [0, h_src-1]
    const short2 *yab;    // [h]  (b0, b1)
    int rz_fast;          // >= 1: the 4 source columns of every aligned destination quad fit three aligned words; 2: see build_plan
};

struct PlanDev {
    int nlevels, batch, nfeatures;
    int ncells_total, nftiles_total, nbtiles_total, kept_total;
    int t_lo, t_hi;      // min / max of (max(fastTh, 1), 7): threshold 0 detects what 1 does (build_plan)
    int t1_is_lo;        // fastTh <= 7
    int score_type;
    int pdl;             // host side only: launch the pipeline's kernels with programmatic stream serialization (ORBFE_PDL, default 1)
    float harris_scale4;   // (1 / (4 * 7 * 255))^4 as the reference computes it (ORBextractor.cc:90-92)
    long long cand_total;  // candidate slots per frame
    LevelDev lv[ORBFE_MAX_LEVELS];
};

// Cell geometry of one FAST tile (host-precomputed): cells overlapped and interior cell boundaries inside it
struct FTileInfo {
    short cj0, ci0, ncj, nci;    // first cell col/row overlapped, number of cell cols/rows overlapped
    short level, tx, ty, pad;    // which level / tile this is (saves a dependent scan of the plan at CTA start)
    unsigned long long hmask;    // bit r: m-tile row r (image y0-1+r) is the first row of a cell other than the top one
    unsigned int vmask[4];       // bit c of the 128: m-tile column c (image x0-4+c) is the first column of a cell other than the leftmost
};
struct BTileInfo { short level, tx, ty, pad; };  // blur tiles

// Per-batch work buffers (device).  Index [frame] strides are in the plan.
struct WorkDev {
    const long long *cell_cand_base;  // [ncells_total] first candidate slot of each cell
    const int *cell_cand_cap;         // [ncells_total]
    const FTileInfo *ftile_info;      // [nftiles_total]
    const BTileInfo *btile_info;      // [nbtiles_total]
    const CUtensorMap *tmaps;         // [nlevels] 3-D (x, y, frame) tensor maps of the unblurred levels; never NULL (build_plan fails without TMA)
    uint32_t *cand_keys;              // [batch][cand_total]   (score<<24 | 0xFFFFFF - raster)
    unsigned long long *cand_keys64;  // HARRIS_SCORE only: order(resp)<<32 | (0xFFFFFF - raster)<<8 | score; NULL otherwise
    uint32_t *kept_aux;               // HARRIS_SCORE only: low raster bits + score of each kept entry
    int *cell_cnt_lo;                 // [batch][ncells_total] candidates with m > t_lo (= all emitted)
    int *cell_cnt_hi;                 // [batch][ncells_total] candidates with m > t_hi
    int *cell_keep;                   // [batch][ncells_total] nToRetain
    uint32_t *cell_min_key;           // [batch][ncells_total] eligibility threshold key, then the cut key
    unsigned long long *kept_keys;    // [batch][kept_total]
    int *kept_cnt;                    // [batch][nlevels]
    int2 *kp_xy_score;                // [batch][nfeatures]  (x | y<<16, score) in level coordinates
    int *level_cnt;                   // [batch][nlevels]
    int *err_flag;                    // [1]
};

// Destinations of the descriptor kernel's outputs when the exchange is fused into it (include/orbfe_comm.h, OrbfeRigExchange):
// slot [rank] of every rank's gather buffer (peer pointers over NVLink, own buffer included), plus the flag words the
// kernel's last thread block publishes the epoch to.  n == 0: plain single destination (the kernel's pointer arguments).
#define ORBFE_MAX_PEERS 16
struct PeerOut {
    int n;
    unsigned epoch;
    unsigned *done;                          // local counter of finished thread blocks (reset by the last one)
    const unsigned *ack;                     // local flags: last epoch each rank finished READING (buffer-half reuse)
    unsigned ack_epoch;                      // wait until ack[r] >= ack_epoch for all r before the first remote store (0 = no wait)
    int *err;                                // device error flag (a wait timed out)
    OrbfeKeyPoint *kps[ORBFE_MAX_PEERS];     // [nslots x nfeatures] of this rank inside peer p's buffer
    uint8_t *desc[ORBFE_MAX_PEERS];
    int *counts[ORBFE_MAX_PEERS];
    unsigned *flag[ORBFE_MAX_PEERS];         // &flags[rank] in peer p's memory
};

// ---- launchers (extract_kernels.cu): every launch covers frames [f0, f0 + nf) of the batch ----
void launch_resize_level(const PlanDev *d_plan, const PlanDev &h_plan, int level, int f0, int nf, cudaStream_t s);
void launch_fast_nms(const PlanDev *d_plan, const PlanDev &h_plan, WorkDev w, int f0, int nf, cudaStream_t s);
void launch_cell_quota(const PlanDev *d_plan, const PlanDev &h_plan, WorkDev w, int f0, int nf, cudaStream_t s);
void launch_cell_select(const PlanDev *d_plan, const PlanDev &h_plan, WorkDev w, int f0, int nf, cudaStream_t s);
void launch_level_select(const PlanDev *d_plan, const PlanDev &h_plan, WorkDev w, size_t smem_bytes, int f0, int nf, cudaStream_t s);
void launch_blur(const PlanDev *d_plan, const PlanDev &h_plan, WorkDev w, int f0, int nf, cudaStream_t s);
void launch_describe_fused(const PlanDev *d_plan, const PlanDev &h_plan, WorkDev w, const int8_t *d_pattern,
                     OrbfeKeyPoint *d_kps, uint8_t *d_desc, int *d_counts, int f0, int nf, cudaStream_t s, const PeerOut *peers = nullptr);
int fast_tma_setup();
int level_select_smem_bytes(int max_kept);
int level_select_harris_smem_bytes(int max_kept);
int set_level_select_harris_smem(int bytes);
int set_level_select_smem(int bytes);

// parameters of the device-resident SearchByProjection(Frame,Frame) kernel
struct SbpParams {
    float min_x, min_y, max_x, max_y, gw, gh;  // Frame::mnMinX.., mfGridElementWidthInv/HeightInv
    float fx, fy, cx, cy, th;
    float scale[ORBFE_MAX_LEVELS];             // Frame::mvScaleFactors
    int nlevels, cap, check_ori;
    int qcap;                                  // queries per job the shared-memory offset table is sized for
    int rule, th_dist;                         // accept rule 0/1/2/SBP_RULE_BEST and distance threshold (guided search); projection mode: 0, TH_HIGH
    float nnratio;
    int scratch_per_pair;                      // global scratch entries per pair
    int smem_entries;                          // entries that fit in the dynamic shared-memory staging area
    int smem_fixed;                            // bytes of the fixed shared-memory part
    // rig exchange hooks (include/orbfe_comm.h): wait for every rank's data of `xw_epoch` before the first read of the
    // gathered arrays, and let the last thread block tell every rank that this one is done reading (0 / NULL = unused)
    const unsigned *xw_flags;
    unsigned *xw_ack[16];
    unsigned *xw_done;
    int *xw_err;
    int xw_n;
    unsigned xw_epoch;
    int owner_base;                            // guided search: added to the job-local query index a matched slot receives
};
// Guided-search accept rule without slots (orbfe_guided_best): each query keeps the first minimum of its whole candidate
// list iff best <= th_dist, written to best_out; slot_owner is read but never written.  Internal: the exported guided searches
// take rules 0..2 (3 is SearchForInitialization's).
#define SBP_RULE_BEST 4
size_t sbp_smem_fixed_bytes(int cap, int qcap);
int launch_guided_device(const SbpParams &P, size_t smem_bytes, int njobs, const OrbfeKeyPoint *kps, const uint8_t *desc,
                         const int *counts, const int *frame_idx, const float *qu, const float *qv, const float *qr,
                         const int *qlo, const int *qhi, const uint8_t *qdesc, const float *qangle, const int *q_base,
                         const int *q_cnt, uint32_t *scratch, int *slot_owner, int *best_out, int *nmatches, int *err,
                         cudaStream_t s);
int launch_init_device(const SbpParams &P, size_t smem_bytes, int npairs, const OrbfeKeyPoint *kps, const uint8_t *desc,
                       const int *counts, const int *f1_idx, const int *f2_idx, float *prev_matched, uint32_t *scratch, int *match12,
                       int *nmatches, int *err, cudaStream_t s);
int launch_sbp_device(const SbpParams &P, size_t smem_bytes, int npairs, const OrbfeKeyPoint *kps, const uint8_t *desc,
                      const int *counts, const int *cur_idx, const int *last_idx, const float *world, const uint8_t *flags,
                      const float *Tcw, uint32_t *scratch, int *cur_mp, int *nmatches, int *err, cudaStream_t s);

// One query window of the guided search: candidates = GetFeaturesInArea(u, v, r, lo, hi) of the searched frame; a match
// writes `owner` into the frame's slot
struct GuidedQuery { float u, v, r; int lo, hi; const uint8_t *desc; float angle; int owner; };

// Host-array forms of the windowed matchers (orbfe_api.cu).  host/match_host.cpp checks the arguments and builds the
// queries; these stage everything in the matcher's pinned block, run sbp_device_kernel, copy the results back and
// synchronise.  The views' own bounds, grid_inv_w/h and scale_factors are what the kernel reads.
// guided_host: best_out (nq ints, rule SBP_RULE_BEST only, else NULL) receives each query's kept candidate or -1; slot_owner
// may then be NULL (no occupied slots).  A call too large for one launch runs its queries in consecutive chunks unless it
// applies the rotation histogram.
int sbp_frames_host(OrbfeMatcher *m, int npairs, const OrbfeFrameView *cur, const OrbfeFrameView *last,
                    const uint8_t *const *last_has_mp, const uint8_t *const *last_outlier, const float *const *last_world,
                    const float *const *Tcw, float fx, float fy, float cx, float cy, float th, int check_orientation,
                    int *const *cur_mp_inout, int *nmatches_out);
int guided_host(OrbfeMatcher *m, const OrbfeFrameView &f, int nq, const GuidedQuery *Q, int rule, float nnratio, int th_dist,
                int check_orientation, int *slot_owner, int *best_out, int *nmatches_out);
int init_host(OrbfeMatcher *m, const OrbfeFrameView &f1, const OrbfeFrameView &f2, float *prev_matched, int window,
              float nnratio, int check_orientation, int *match12_out, int *nmatches_out);

// SearchByBoW for `njobs` (side 1, side 2) frame pairs (match_kernels.cu); out-of-range FeatureVector entries set bit 2 of *err
int launch_search_by_bow(int variant, int njobs, const OrbfeKeyPoint *kps, const uint8_t *desc, const int *counts, int cap,
                         const int *fv_ids, const int *fv_ptr, const int *fv_items, const int *fv_n, const uint8_t *valid,
                         const int *idx1, const int *idx2, float nnratio, int check_ori, int *out, int *nmatches, int *err,
                         cudaStream_t s);

// SearchForTriangulation for `njobs` (pKF1, pKF2) frame pairs (match_kernels.cu); sigma2 = nlevels floats on the host;
// out-of-range FeatureVector entries or side-2 octaves set bit 4 of *err
int launch_search_for_triangulation(int njobs, const OrbfeKeyPoint *kps, const uint8_t *desc, const int *counts, int cap,
                                    const int *fv_ids, const int *fv_ptr, const int *fv_items, const int *fv_n, const uint8_t *has_mp,
                                    const int *idx1, const int *idx2, const float *F12, const float *sigma2, int nlevels,
                                    int check_ori, int *match12, int *nmatches, int *err, cudaStream_t s);

void launch_undistort(float fx, float fy, float cx, float cy, const float *dist5, const OrbfeKeyPoint *d_in, OrbfeKeyPoint *d_out,
                      int n, cudaStream_t s);

// records the thread's last-error string (orbfe_last_error) and returns `code`
int set_error(int code, const char *fmt, ...);

// returns ORBFE_ERR_CUDA from the enclosing function, naming the failed call in orbfe_last_error, when `expr` is not cudaSuccess
#define ORBFE_CUDA_TRY(expr)                                                                                                   \
    do {                                                                                                                       \
        cudaError_t e__ = (expr);                                                                                              \
        if (e__ != cudaSuccess)                                                                                                \
            return orbfe::set_error(ORBFE_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
    } while (0)

// The device arrays a handle owns: every alloc is recorded (at least 256 bytes each) and release() frees them all, so an
// array is named once, where it is allocated.  Pinned host memory, streams and events are not kept here.
struct DeviceBuffers {
    std::vector<void *> ptrs;
    template <class T>
    cudaError_t alloc(T **p, size_t count) {
        void *q = nullptr;
        const cudaError_t e = cudaMalloc(&q, std::max<size_t>(count * sizeof(T), 256));
        if (e == cudaSuccess) { ptrs.push_back(q); *p = (T *)q; }
        return e;
    }
    void release() {
        for (void *q : ptrs) cudaFree(q);
        ptrs.clear();
    }
};

// The own stream of a handle whose entries may also run on caller streams, and the rule that makes that safe: every call
// enters (its stream waits for the handle's last work) and leaves (records its own), so the handle's calls run in call order
// whichever streams they were enqueued on.  Whatever reads or frees the handle's device state from the host (a sync, a
// buffer that grows) first waits for `last`.
struct HandleStream {
    int device = 0;
    cudaStream_t stream = nullptr;   // non-blocking
    cudaEvent_t last = nullptr;      // the handle's most recent work
    cudaError_t create(int dev, int priority = 0) {
        device = dev;
        cudaError_t e = cudaSetDevice(dev);
        if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&stream, cudaStreamNonBlocking, priority);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&last, cudaEventDisableTiming);
        return e;
    }
    void destroy() {
        if (last) cudaEventDestroy(last);
        if (stream) cudaStreamDestroy(stream);
        last = nullptr;
        stream = nullptr;
    }
    // the caller's stream if one was given, else the handle's own
    cudaStream_t pick(void *caller) const { return caller ? (cudaStream_t)caller : stream; }
    int enter(cudaStream_t s) {
        ORBFE_CUDA_TRY(cudaSetDevice(device));
        ORBFE_CUDA_TRY(cudaStreamWaitEvent(s, last, 0));
        return ORBFE_OK;
    }
    int leave(cudaStream_t s, bool sync) {
        ORBFE_CUDA_TRY(cudaGetLastError());
        ORBFE_CUDA_TRY(cudaEventRecord(last, s));
        if (sync) ORBFE_CUDA_TRY(cudaStreamSynchronize(s));
        return ORBFE_OK;
    }
};

// Staging block of every host-array entry of a matcher or vocabulary handle: a grow-only pinned host block h and its device
// twin d.  The entry lays out and packs h, moves it with round_trip and synchronises before it reads the results.  Both keep
// the size (times 1.25) of the largest call the handle has seen.  The block serves one call at a time: the vocabulary holds
// its mutex across each call.
struct Stage {
    unsigned char *h = nullptr;
    unsigned char *d = nullptr;
    size_t cap = 0;
    // places arrays of `second` bytes at 256-byte aligned offsets (*first), sets *total to the block's size and grows the
    // block to hold it (ORBFE_ERR_CUDA on a failed allocation)
    int layout(std::initializer_list<std::pair<size_t *, size_t>> arrays, size_t *total);
    void release();
    // on stream s: the inputs [0, up) to the device, enqueue() (the call's kernels; returns an orbfe code), the outputs
    // [down, total) back.  Returns the first error; the caller synchronises s before it reads h.
    template <class Enqueue>
    int round_trip(cudaStream_t s, size_t up, size_t down, size_t total, Enqueue enqueue) {
        ORBFE_CUDA_TRY(cudaMemcpyAsync(d, h, up, cudaMemcpyHostToDevice, s));
        if (int rc = enqueue()) return rc;
        ORBFE_CUDA_TRY(cudaMemcpyAsync(h + down, d + down, total - down, cudaMemcpyDeviceToHost, s));
        return ORBFE_OK;
    }
};

// ---- launchers (match_kernels.cu) ----
void launch_hamming_csr(const uint8_t *q, const uint8_t *t, const int32_t *row_ptr, const int32_t *cols, int nq,
                        int npairs, uint16_t *out, cudaStream_t s);
void launch_hamming_dense(const uint8_t *q, int nq, const uint8_t *t, int nt, uint16_t *out, cudaStream_t s);
void launch_knn2_groups(const uint8_t *q, int nq, const uint8_t *db, int ngroups, int group_size,
                        uint16_t *best, int32_t *best_idx, uint16_t *second, cudaStream_t s);

// ---- launchers (bow_kernels.cu) ----
void launch_distinctive(const uint8_t *d_desc, const int *d_group_ptr, int ngroups, int *d_best, cudaStream_t s);
// an out-of-range group pointer or observation sets bit 8 of *d_err
void launch_distinctive_obs(const uint8_t *d_desc, const int *d_counts, int nframes, int cap, const int *d_group_ptr,
                            const int *d_obs, int nobs, int ngroups, int *d_best, uint8_t *d_mp_desc, int *d_err, cudaStream_t s);
// MapPoint::UpdateNormalAndDepth on the frame store; an out-of-range group pointer, slot or reference octave sets bit 16 of
// *d_err.  scale_factors: nlevels floats on the host.
void launch_normal_depth_obs(const OrbfeKeyPoint *d_kps, const int *d_counts, int nframes, int cap, const float *d_centers,
                             const int *d_group_ptr, const int *d_obs, int nobs, const float *d_world, const int *d_ref_obs,
                             float scale_factor, int nlevels, const float *scale_factors, int npoints, float *d_normal,
                             float *d_min_dist, float *d_max_dist, int *d_err, cudaStream_t s);
// the same on host-checked contiguous rows: observation centres by group, one reference centre and octave per point
void launch_normal_depth(const float *d_obs_centers, const int *d_group_ptr, const float *d_world, const float *d_ref_centers,
                         const int *d_ref_octave, float scale_factor, int nlevels, const float *scale_factors, int npoints,
                         float *d_normal, float *d_min_dist, float *d_max_dist, cudaStream_t s);
void launch_bow_db_score(int nq, const int *q_ids, const double *q_vals, int nkf, const int *kf_ptr, const int *db_ids,
                         const double *db_vals, int *common, int *first, double *score, cudaStream_t s);

// Device half of orbfe_bow_db_detect (orbfe_api.cu; the host half is host/bow_host.cpp): per keyframe, the shared-word count,
// the first shared word and the L1 score, staged through the matcher's block and synchronised
int bow_db_score(OrbfeMatcher *m, int nq, const int32_t *q_ids, const double *q_vals, int nkf, const int32_t *kf_ptr,
                 const int32_t *db_ids, const double *db_vals, int32_t *common, int32_t *first, double *score);

}  // namespace orbfe
