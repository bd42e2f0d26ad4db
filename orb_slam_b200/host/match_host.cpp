// match_host.cpp -- host half of the windowed matchers of ORB_SLAM::ORBmatcher (reference src/ORBmatcher.cc), on plain
// arrays, compiled into liborbfe.so.
//
// Each entry checks its arguments and turns its routine's inputs into query windows: the projections of map points, the
// predicted levels and search radii.  Frame's 64x48 grid, GetFeaturesInArea, the distances, the accept loop and the rotation
// histogram run once, in the fused kernel (sbp_device_kernel, match_kernels.cu), staged by orbfe_api.cu.
// orbfe_guided_best, a slot-free argmin, enumerates its candidates here and computes the distances with orbfe_hamming_csr.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include "../csrc/orbfe_internal.h"

using orbfe::GuidedQuery;
using orbfe::set_error;

namespace {

constexpr int kGridCols = 64;  // FRAME_GRID_COLS, Frame.h:36
constexpr int kGridRows = 48;  // FRAME_GRID_ROWS, Frame.h:35
constexpr int kThHigh = 100;   // TH_HIGH, ORBmatcher.cc:40

// A view is well formed when its arrays are present and every keypoint octave indexes scale_factors (a malformed
// view is rejected with ORBFE_ERR_ARG instead of being read out of bounds; octave < 0 never occurs in extractor output).
bool view_ok(const OrbfeFrameView &v) {
    if (v.n < 0 || v.nlevels < 1 || v.nlevels > ORBFE_MAX_LEVELS || !v.scale_factors) return false;
    if (v.n > 0 && (!v.keys_un || !v.desc)) return false;
    for (int i = 0; i < v.n; i++)
        if ((unsigned)v.keys_un[i].octave >= (unsigned)v.nlevels) return false;
    return true;
}

// cv::Mat `R*x + t` of the reference's projections (CV_32F, 3x3 * 3x1, one cv::gemm with flags 0): OpenCV's unrolled
// small-matrix branch sums the three products in FLOAT, left to right, then (float)(sum*alpha + t*beta) in double.
// Verified against python-cv2 (tests/golden/opencv_gemm.npz); this file is compiled with -ffp-contract=off.
inline void Rx_plus_t(const float *T, const float *X, float out[3]) {
    for (int k = 0; k < 3; k++) {
        float s = T[4 * k] * X[0];
        s = s + T[4 * k + 1] * X[1];
        s = s + T[4 * k + 2] * X[2];
        out[k] = (float)((double)s + (double)T[4 * k + 3]);
    }
}

struct Grid {
    std::vector<int> start;  // kGridCols*kGridRows + 1, cell id = ix*kGridRows + iy
    std::vector<int> items;
};

// Frame.cc:116-123 + PosInGrid :267-277
void build_grid(const OrbfeFrameView &f, Grid &g) {
    const int nc = kGridCols * kGridRows;
    g.start.assign(nc + 1, 0);
    std::vector<int> cell(f.n);
    for (int i = 0; i < f.n; i++) {
        const OrbfeKeyPoint &kp = f.keys_un[i];
        const int px = (int)std::round((kp.x - f.min_x) * f.grid_inv_w);
        const int py = (int)std::round((kp.y - f.min_y) * f.grid_inv_h);
        if (px < 0 || px >= kGridCols || py < 0 || py >= kGridRows) { cell[i] = -1; continue; }
        cell[i] = px * kGridRows + py;
        g.start[cell[i] + 1]++;
    }
    for (int c = 0; c < nc; c++) g.start[c + 1] += g.start[c];
    g.items.assign(std::max(f.n, 1), 0);
    std::vector<int> fill(g.start.begin(), g.start.end() - 1);
    for (int i = 0; i < f.n; i++)
        if (cell[i] >= 0) g.items[fill[cell[i]]++] = i;  // ascending index inside a cell (push_back order)
}

// Frame::GetFeaturesInArea, Frame.cc:200-265: appends to `out`
void features_in_area(const OrbfeFrameView &f, const Grid &g, float x, float y, float r, int minLevel, int maxLevel,
                      std::vector<int> &out) {
    int x0 = (int)std::floor((x - f.min_x - r) * f.grid_inv_w);
    x0 = std::max(0, x0);
    if (x0 >= kGridCols) return;
    int x1 = (int)std::ceil((x - f.min_x + r) * f.grid_inv_w);
    x1 = std::min(kGridCols - 1, x1);
    if (x1 < 0) return;
    int y0 = (int)std::floor((y - f.min_y - r) * f.grid_inv_h);
    y0 = std::max(0, y0);
    if (y0 >= kGridRows) return;
    int y1 = (int)std::ceil((y - f.min_y + r) * f.grid_inv_h);
    y1 = std::min(kGridRows - 1, y1);
    if (y1 < 0) return;
    bool check = true, same = false;
    if (minLevel == -1 && maxLevel == -1) check = false;
    else if (minLevel == maxLevel) same = true;
    for (int ix = x0; ix <= x1; ix++)
        for (int iy = y0; iy <= y1; iy++) {
            const int c = ix * kGridRows + iy;
            for (int k = g.start[c]; k < g.start[c + 1]; k++) {
                const int idx = g.items[k];
                const OrbfeKeyPoint &kp = f.keys_un[idx];
                if (check && !same) { if (kp.octave < minLevel || kp.octave > maxLevel) continue; }
                else if (same) { if (kp.octave != minLevel) continue; }
                if (std::fabs(kp.x - x) > r || std::fabs(kp.y - y) > r) continue;
                out.push_back(idx);
            }
        }
}

}  // namespace

// SearchByProjection(Frame &CurrentFrame, const Frame &LastFrame, float th), ORBmatcher.cc:1507-1620
extern "C" int orbfe_search_by_projection_frames(OrbfeMatcher *m, int npairs, const OrbfeFrameView *cur,
                                                 const OrbfeFrameView *last, const uint8_t *const *last_has_mp,
                                                 const uint8_t *const *last_outlier, const float *const *last_world,
                                                 const float *const *Tcw, float fx, float fy, float cx, float cy, float th,
                                                 int check_orientation, int *const *cur_mp_inout, int *nmatches_out) {
    if (!m || npairs < 0 || (npairs > 0 && (!cur || !last || !last_has_mp || !last_outlier || !last_world || !Tcw ||
                                            !cur_mp_inout || !nmatches_out)))
        return set_error(ORBFE_ERR_ARG, "orbfe_search_by_projection_frames: bad arguments");
    for (int j = 0; j < npairs; j++) {
        if (!view_ok(cur[j]) || !view_ok(last[j]))
            return set_error(ORBFE_ERR_ARG, "orbfe_search_by_projection_frames: pair %d has a malformed view", j);
        // a Last map point's search radius is th * the CURRENT frame's scale factor of its octave (:1547)
        for (int i = 0; i < last[j].n; i++)
            if (last_has_mp[j][i] && !last_outlier[j][i] && last[j].keys_un[i].octave >= cur[j].nlevels)
                return set_error(ORBFE_ERR_ARG, "orbfe_search_by_projection_frames: pair %d: Last feature %d has octave %d, the "
                                 "Current view %d levels", j, i, last[j].keys_un[i].octave, cur[j].nlevels);
    }
    return orbfe::sbp_frames_host(m, npairs, cur, last, last_has_mp, last_outlier, last_world, Tcw, fx, fy, cx, cy, th,
                                  check_orientation, cur_mp_inout, nmatches_out);
}

// SearchForInitialization, ORBmatcher.cc:598-713
extern "C" int orbfe_search_for_initialization(OrbfeMatcher *m, const OrbfeFrameView *f1, const OrbfeFrameView *f2,
                                               float *prev_matched, int window, float nnratio, int check_orientation,
                                               int *match12_out, int *nmatches_out) {
    if (!m || !f1 || !f2 || !prev_matched || !match12_out || !nmatches_out)
        return set_error(ORBFE_ERR_ARG, "orbfe_search_for_initialization: NULL argument");
    if (!view_ok(*f1) || !view_ok(*f2)) return set_error(ORBFE_ERR_ARG, "orbfe_search_for_initialization: malformed view");
    return orbfe::init_host(m, *f1, *f2, prev_matched, window, nnratio, check_orientation, match12_out, nmatches_out);
}

// Frame.cc:95-103: mvScaleFactors from GetScaleFactor()
extern "C" void orbfe_frame_scale_factors(float scale_factor, int nlevels, float *out) {
    if (!out || nlevels < 1) return;
    out[0] = 1.0f;
    for (int i = 1; i < nlevels; i++) out[i] = out[i - 1] * scale_factor;
}

// The guided search shared by ORBmatcher's projection and window routines: for each query (ascending), candidates =
// GetFeaturesInArea(u, v, r, lo, hi) of frame `f` whose slot is still free, best and second-best distance, accepted by `rule`,
// optional rotation histogram.
// rule 0: best <= th_dist                                   (ORBmatcher.cc:1576, :1693)
// rule 1: best <= second*nnratio && best <= TH_HIGH          (:469, :586)
// rule 2: best <= TH_HIGH && !(bestLevel==secondLevel && best > nnratio*second)   (:113-121)

// WindowSearch(F1, F2, windowSize, matches, minLevel, maxLevel), ORBmatcher.cc:393-517: the guided search with the
// F1 keypoint as window centre, same-octave filter, accept rule 1 (:469) and the rotation histogram of :472-489.
extern "C" int orbfe_window_search(OrbfeMatcher *m, const OrbfeFrameView *f1, const OrbfeFrameView *f2,
                                   const uint8_t *f1_has_mp, int window, int min_level, int max_level, float nnratio,
                                   int check_orientation, int *match21_out, int *nmatches_out) {
    if (!m || !f1 || !f2 || !f1_has_mp || !match21_out || !nmatches_out)
        return set_error(ORBFE_ERR_ARG, "orbfe_window_search: NULL argument");
    if (!view_ok(*f1) || !view_ok(*f2)) return set_error(ORBFE_ERR_ARG, "orbfe_window_search: malformed view");
    const bool bMin = min_level > 0, bMax = max_level < INT_MAX;
    std::vector<GuidedQuery> Q;
    for (int i1 = 0; i1 < f1->n; i1++) {
        if (!f1_has_mp[i1]) continue;
        const OrbfeKeyPoint &kp1 = f1->keys_un[i1];
        const int level1 = kp1.octave;
        if (bMin && level1 < min_level) continue;
        if (bMax && level1 > max_level) continue;
        Q.push_back({kp1.x, kp1.y, (float)window, level1, level1, f1->desc + (size_t)i1 * 32, kp1.angle, i1});
    }
    for (int i = 0; i < f2->n; i++) match21_out[i] = -1;
    return orbfe::guided_host(m, *f2, (int)Q.size(), Q.data(), 1, nnratio, kThHigh, check_orientation, match21_out, nmatches_out);
}

// SearchByProjection(Frame &F, const vector<MapPoint*>&, th), ORBmatcher.cc:49-125
extern "C" int orbfe_search_local_points(OrbfeMatcher *m, const OrbfeFrameView *f, int npts, const uint8_t *in_view,
                                         const float *proj_xy, const int *level, const float *view_cos, const uint8_t *desc,
                                         float th, float nnratio, int *f_mp_inout, int *nmatches_out) {
    if (!m || !f || npts < 0 || !f_mp_inout || !nmatches_out || (npts > 0 && (!in_view || !proj_xy || !level || !view_cos || !desc)))
        return set_error(ORBFE_ERR_ARG, "orbfe_search_local_points: bad arguments");
    if (!view_ok(*f)) return set_error(ORBFE_ERR_ARG, "orbfe_search_local_points: malformed view");
    for (int i = 0; i < npts; i++)
        if (in_view[i] && (unsigned)level[i] >= (unsigned)f->nlevels)  // level indexes scale_factors
            return set_error(ORBFE_ERR_ARG, "orbfe_search_local_points: point %d has level %d, the view %d levels", i, level[i], f->nlevels);
    const bool bFactor = th != 1.0f;
    std::vector<GuidedQuery> Q;
    for (int i = 0; i < npts; i++) {
        if (!in_view[i]) continue;
        float r = view_cos[i] > 0.998 ? 2.5f : 4.0f;  // RadiusByViewingCos :127-133
        if (bFactor) r *= th;
        const int lv = level[i];
        Q.push_back({proj_xy[2 * i], proj_xy[2 * i + 1], r * f->scale_factors[lv], lv - 1, lv, desc + (size_t)i * 32, 0.f, i});
    }
    return orbfe::guided_host(m, *f, (int)Q.size(), Q.data(), 2, nnratio, kThHigh, 0, f_mp_inout, nmatches_out);
}

// SearchByProjection(Frame &CurrentFrame, KeyFrame *pKF, sAlreadyFound, th, ORBdist), ORBmatcher.cc:1622-1746
extern "C" int orbfe_search_by_projection_kf(OrbfeMatcher *m, const OrbfeFrameView *cur, int npts, const uint8_t *valid,
                                             const float *world, const float *min_dist, const uint8_t *desc,
                                             const float *kf_angle, const float *Tcw, float fx, float fy, float cx, float cy,
                                             float th, int orb_dist, int check_orientation, int *cur_mp_inout, int *nmatches_out) {
    if (!m || !cur || npts < 0 || !Tcw || !cur_mp_inout || !nmatches_out ||
        (npts > 0 && (!valid || !world || !min_dist || !desc || !kf_angle)))
        return set_error(ORBFE_ERR_ARG, "orbfe_search_by_projection_kf: bad arguments");
    if (!view_ok(*cur)) return set_error(ORBFE_ERR_ARG, "orbfe_search_by_projection_kf: malformed view");
    float Ow[3];  // Ow = -Rcw.t()*tcw (:1628): gemm, double accumulation, alpha = -1
    for (int k = 0; k < 3; k++) {
        const double s = (double)Tcw[k] * (double)Tcw[3] + (double)Tcw[4 + k] * (double)Tcw[7] + (double)Tcw[8 + k] * (double)Tcw[11];
        Ow[k] = (float)(s * -1.0);
    }
    std::vector<GuidedQuery> Q;
    for (int i = 0; i < npts; i++) {
        if (!valid[i]) continue;
        const float *X = world + 3 * (size_t)i;
        float xc[3];
        Rx_plus_t(Tcw, X, xc);
        const float invzc = (float)(1.0 / (double)xc[2]);
        const float u = fx * xc[0] * invzc + cx, v = fy * xc[1] * invzc + cy;
        if (u < cur->min_x || u > cur->max_x) continue;
        if (v < cur->min_y || v > cur->max_y) continue;
        const float PO[3] = {X[0] - Ow[0], X[1] - Ow[1], X[2] - Ow[2]};
        const float dist3D = (float)std::sqrt((double)PO[0] * PO[0] + (double)PO[1] * PO[1] + (double)PO[2] * PO[2]);  // cv::norm
        const float ratio = dist3D / min_dist[i];
        const float *sf = cur->scale_factors;
        const int it = (int)(std::lower_bound(sf, sf + cur->nlevels, ratio) - sf);
        const int lv = std::min(it, cur->nlevels - 1);
        Q.push_back({u, v, th * sf[lv], lv - 1, lv + 1, desc + (size_t)i * 32, kf_angle[i], i});
    }
    return orbfe::guided_host(m, *cur, (int)Q.size(), Q.data(), 0, 0.f, orb_dist, check_orientation, cur_mp_inout, nmatches_out);
}

// SearchByProjection(Frame &F1, Frame &F2, int windowSize, vpMapPointMatches2), ORBmatcher.cc:519-594
extern "C" int orbfe_search_by_projection_f1f2(OrbfeMatcher *m, const OrbfeFrameView *f1, const OrbfeFrameView *f2,
                                               const uint8_t *valid1, const float *world1, const float *Tc2w, float fx, float fy,
                                               float cx, float cy, int window, float nnratio, int *f2_mp_inout, int *nmatches_out) {
    if (!m || !f1 || !f2 || !Tc2w || !f2_mp_inout || !nmatches_out || (f1->n > 0 && (!valid1 || !world1)))
        return set_error(ORBFE_ERR_ARG, "orbfe_search_by_projection_f1f2: bad arguments");
    if (!view_ok(*f1) || !view_ok(*f2)) return set_error(ORBFE_ERR_ARG, "orbfe_search_by_projection_f1f2: malformed view");
    std::vector<GuidedQuery> Q;
    for (int i1 = 0; i1 < f1->n; i1++) {
        if (!valid1[i1]) continue;
        const int level1 = f1->keys_un[i1].octave;
        float xc[3];
        Rx_plus_t(Tc2w, world1 + 3 * (size_t)i1, xc);
        const float invz = (float)(1.0 / (double)xc[2]);
        Q.push_back({fx * xc[0] * invz + cx, fy * xc[1] * invz + cy, (float)window, level1, level1, f1->desc + (size_t)i1 * 32, 0.f, i1});
    }
    return orbfe::guided_host(m, *f2, (int)Q.size(), Q.data(), 1, nnratio, kThHigh, 0, f2_mp_inout, nmatches_out);
}

// Exported form of the guided search for callers that do their own projection (the KeyFrame-level routines
// of the facade: Sim3 projection :286-407, SearchBySim3 :1267-1505, Fuse :1016-1265).
extern "C" int orbfe_guided_search(OrbfeMatcher *m, const OrbfeFrameView *f, int nq, const float *qu, const float *qv,
                                   const float *qr, const int32_t *qlo, const int32_t *qhi, const uint8_t *qdesc,
                                   const float *qangle, int rule, float nnratio, int th_dist, int hist_mode,
                                   int32_t *slot_owner_inout, int *nmatches_out) {
    if (!m || !f || nq < 0 || rule < 0 || rule > 2 || hist_mode < 0 || hist_mode > 2 || !slot_owner_inout || !nmatches_out ||
        f->n < 0 || (f->n > 0 && (!f->keys_un || !f->desc)))
        return set_error(ORBFE_ERR_ARG, "orbfe_guided_search: bad arguments");
    if (nq > 0 && (!qu || !qv || !qr || !qlo || !qhi || !qdesc || (hist_mode && !qangle)))
        return set_error(ORBFE_ERR_ARG, "orbfe_guided_search: NULL argument");
    std::vector<GuidedQuery> Q(nq);
    for (int q = 0; q < nq; q++) Q[q] = {qu[q], qv[q], qr[q], qlo[q], qhi[q], qdesc + (size_t)q * 32, qangle ? qangle[q] : 0.f, q};
    // hist_mode 2 fills the histogram without applying it: the same matches as 0
    return orbfe::guided_host(m, *f, nq, Q.data(), rule, nnratio, th_dist, hist_mode == 1, slot_owner_inout, nmatches_out);
}

// Guided search without slot bookkeeping (Fuse :1090-1107 / :1222-1239, SearchBySim3 :1356-1378 / :1436-1458):
// best candidate per query, kept iff best <= th_dist.  One distance launch for all queries.
extern "C" int orbfe_guided_best(OrbfeMatcher *m, const OrbfeFrameView *f, int nq, const float *qu, const float *qv, const float *qr,
                                 const int32_t *qlo, const int32_t *qhi, const uint8_t *qdesc, int th_dist, int32_t *best_idx_out) {
    if (!m || !f || nq < 0 || !best_idx_out) return ORBFE_ERR_ARG;
    if (nq > 0 && (!qu || !qv || !qr || !qlo || !qhi || !qdesc)) return ORBFE_ERR_ARG;
    Grid grid;
    build_grid(*f, grid);
    std::vector<int32_t> row_ptr(1, 0), cols;
    std::vector<int> tmp;
    for (int q = 0; q < nq; q++) {
        tmp.clear();
        features_in_area(*f, grid, qu[q], qv[q], qr[q], qlo[q], qhi[q], tmp);
        cols.insert(cols.end(), tmp.begin(), tmp.end());
        row_ptr.push_back((int32_t)cols.size());
        best_idx_out[q] = -1;
    }
    if (cols.empty()) return ORBFE_OK;
    std::vector<uint16_t> dist(cols.size());
    const int rc = orbfe_hamming_csr(m, qdesc, nq, f->desc, f->n, row_ptr.data(), cols.data(), dist.data());
    if (rc) return rc;
    for (int q = 0; q < nq; q++) {
        int bestDist = INT_MAX, bestIdx = -1;
        for (int c = row_ptr[q]; c < row_ptr[q + 1]; c++)
            if (dist[c] < bestDist) { bestDist = dist[c]; bestIdx = cols[c]; }
        if (bestDist <= th_dist) best_idx_out[q] = bestIdx;
    }
    return ORBFE_OK;
}
