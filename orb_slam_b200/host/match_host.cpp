// match_host.cpp -- host half of the windowed matchers of ORB_SLAM::ORBmatcher (reference
// src/ORBmatcher.cc), on plain arrays, compiled into liborbfe.so.
//
// Division of labour (SURVEY.md 8a, rows M2/M7/M8/M14):
//   host   : Frame's 64x48 lookup grid and GetFeaturesInArea candidate enumeration (src/Frame.cc:109-123,
//            :200-277) -- it defines the candidate ORDER and therefore every distance tie-break;
//   device : all (query, candidate) 256-bit Hamming distances in CSR order, one launch per call
//            (hamming_csr_kernel) -- ORBmatcher::DescriptorDistance, ORBmatcher.cc:1794-1810;
//   host   : the sequential accept/skip loop of each Search* routine replayed over the distances,
//            rotation histogram and ComputeThreeMaxima (ORBmatcher.cc:1748-1789).
// Several frame pairs can be processed per call: candidate generation and the greedy replay run on a
// small thread pool (one pair per task), the distances of ALL pairs go to the GPU in one launch.
//
// There is no CPU path for the distances: every entry point needs an OrbfeMatcher (a CUDA device).
#include <algorithm>
#include <atomic>
#include <climits>
#include <cmath>
#include <cstring>
#include <thread>
#include <vector>

#include "../../include/orbfe.h"
#include "../../include/orbfe_match.h"

extern "C" int orbfe_sbp_frames_via_device(OrbfeMatcher *m, int npairs, const OrbfeFrameView *cur, const OrbfeFrameView *last,
                                           const uint8_t *const *last_has_mp, const uint8_t *const *last_outlier,
                                           const float *const *last_world, const float *const *Tcw, float fx, float fy,
                                           float cx, float cy, float th, int check_orientation, int *const *cur_mp_inout,
                                           int *nmatches_out);
extern "C" int orbfe_guided_via_device(OrbfeMatcher *m, const OrbfeFrameView *f, int nq, const float *qu, const float *qv,
                                       const float *qr, const int *qlo, const int *qhi, const uint8_t *const *qdesc,
                                       const float *qangle, int rule, float nnratio, int th_dist, int check_orientation,
                                       const int *slot_owner, int *slot_new, int *nmatches_out);
static std::atomic<bool> g_force_host_replay(false);  // test hook, read from several matcher threads
// test hook: 1 = always use host candidate lists + device distances + host greedy replay
extern "C" void orbfe_matcher_force_host_replay(int on) { g_force_host_replay.store(on != 0); }

namespace {

constexpr int kGridCols = 64;  // FRAME_GRID_COLS, Frame.h:36
constexpr int kGridRows = 48;  // FRAME_GRID_ROWS, Frame.h:35
constexpr int kThHigh = 100, kThLow = 50, kHisto = 30;  // ORBmatcher.cc:40-42

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

// ComputeThreeMaxima, ORBmatcher.cc:1748-1789
void three_maxima(const std::vector<int> *histo, int L, int &ind1, int &ind2, int &ind3) {
    int max1 = 0, max2 = 0, max3 = 0;
    for (int i = 0; i < L; i++) {
        const int s = (int)histo[i].size();
        if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }
        else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }
        else if (s > max3) { max3 = s; ind3 = i; }
    }
    if ((float)max2 < 0.1f * (float)max1) { ind2 = -1; ind3 = -1; }
    else if ((float)max3 < 0.1f * (float)max1) { ind3 = -1; }
}

inline int rot_bin(float a1, float a2) {
    const float factor = 1.0f / kHisto;
    float rot = a1 - a2;
    if (rot < 0.0f) rot += 360.0f;
    int bin = (int)std::round(rot * factor);
    if (bin == kHisto) bin = 0;
    return bin;
}

template <typename F>
void parallel_for(int n, F fn) {
    unsigned hw = std::thread::hardware_concurrency();
    int nt = (int)std::min<unsigned>(hw ? hw : 4, (unsigned)std::max(n, 1));
    if (nt <= 1) { for (int i = 0; i < n; i++) fn(i); return; }
    std::atomic<int> next(0);
    std::vector<std::thread> th;
    for (int t = 0; t < nt; t++)
        th.emplace_back([&]() { for (int i = next++; i < n; i = next++) fn(i); });
    for (auto &t : th) t.join();
}

// One matching job = one (query frame, train frame) pair with its candidate lists.
struct Job {
    Grid grid;
    std::vector<int> row_ptr;   // per query row (nq+1), local
    std::vector<int> cols;      // candidate indices into the train frame
    std::vector<int> qidx;      // query feature index of each row
    size_t pair_base = 0;       // offset of this job's pairs in the global pair array
};

// Runs all jobs' distances in ONE device launch.  q/t views give each job's descriptor arrays.
int run_distances(OrbfeMatcher *m, std::vector<Job> &jobs, const std::vector<const OrbfeFrameView *> &qf,
                  const std::vector<const OrbfeFrameView *> &tf, std::vector<uint16_t> &dist) {
    size_t nq = 0, nt = 0, np = 0, nrows = 0;
    for (size_t j = 0; j < jobs.size(); j++) { nq += qf[j]->n; nt += tf[j]->n; np += jobs[j].cols.size(); nrows += jobs[j].qidx.size(); }
    dist.assign(np, 0);
    if (np == 0) return ORBFE_OK;
    if (nq > (size_t)INT_MAX || nt > (size_t)INT_MAX || np > (size_t)INT_MAX) return ORBFE_ERR_ARG;
    // concatenated CSR: one row per (job, query row); qdesc rows are gathered so that row r <-> qrow[r]
    std::vector<uint8_t> qd(nrows * 32), td(nt * 32);
    std::vector<int32_t> row_ptr(nrows + 1, 0), cols(np);
    size_t r = 0, p = 0, tbase = 0;
    for (size_t j = 0; j < jobs.size(); j++) {
        Job &J = jobs[j];
        J.pair_base = p;
        if (tf[j]->n) memcpy(&td[tbase * 32], tf[j]->desc, (size_t)tf[j]->n * 32);
        for (size_t k = 0; k < J.qidx.size(); k++) {
            memcpy(&qd[r * 32], qf[j]->desc + (size_t)J.qidx[k] * 32, 32);
            for (int c = J.row_ptr[k]; c < J.row_ptr[k + 1]; c++) cols[p++] = (int32_t)(tbase + J.cols[c]);
            row_ptr[++r] = (int32_t)p;
        }
        tbase += tf[j]->n;
    }
    return orbfe_hamming_csr(m, qd.data(), (int)nrows, td.data(), (int)nt, row_ptr.data(), cols.data(), dist.data());
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// SearchByProjection(Frame &CurrentFrame, const Frame &LastFrame, float th), ORBmatcher.cc:1507-1620
// ------------------------------------------------------------------------------------------------
extern "C" int orbfe_search_by_projection_frames(OrbfeMatcher *m, int npairs, const OrbfeFrameView *cur,
                                                 const OrbfeFrameView *last, const uint8_t *const *last_has_mp,
                                                 const uint8_t *const *last_outlier, const float *const *last_world,
                                                 const float *const *Tcw, float fx, float fy, float cx, float cy, float th,
                                                 int check_orientation, int *const *cur_mp_inout, int *nmatches_out) {
    if (!m || npairs < 0 || (npairs > 0 && (!cur || !last || !last_has_mp || !last_outlier || !last_world || !Tcw ||
                                            !cur_mp_inout || !nmatches_out)))
        return ORBFE_ERR_ARG;
    for (int j = 0; j < npairs; j++)
        if (!view_ok(cur[j]) || !view_ok(last[j])) return ORBFE_ERR_ARG;
    // fast path: everything (grid, candidates, distances, greedy, rotation filter) in ONE device kernel
    if (!g_force_host_replay.load()) {
        const int rc = orbfe_sbp_frames_via_device(m, npairs, cur, last, last_has_mp, last_outlier, last_world, Tcw, fx, fy, cx,
                                                   cy, th, check_orientation, cur_mp_inout, nmatches_out);
        if (rc != 1) return rc;  // 1 = not applicable (mixed geometry / overflow): exact host replay below
    }
    std::vector<Job> jobs(npairs);
    std::vector<const OrbfeFrameView *> qf(npairs), tf(npairs);
    parallel_for(npairs, [&](int j) {
        const OrbfeFrameView &C = cur[j], &L = last[j];
        qf[j] = &L; tf[j] = &C;
        Job &J = jobs[j];
        build_grid(C, J.grid);
        J.row_ptr.push_back(0);
        const float *T = Tcw[j];
        for (int i = 0; i < L.n; i++) {
            if (!last_has_mp[j][i] || last_outlier[j][i]) continue;
            // x3Dc = Rcw*x3Dw + tcw (:1527-1528): one cv::gemm on CV_32F 3x3 * 3x1 -> OpenCV's small-matrix path (Rx_plus_t)
            const float *X = last_world[j] + 3 * (size_t)i;
            float xc3[3];
            Rx_plus_t(T, X, xc3);
            const float invzc = (float)(1.0 / (double)xc3[2]);
            const float u = fx * xc3[0] * invzc + cx;
            const float v = fy * xc3[1] * invzc + cy;
            if (u < C.min_x || u > C.max_x) continue;
            if (v < C.min_y || v > C.max_y) continue;
            const int oct = L.keys_un[i].octave;
            const float radius = th * C.scale_factors[oct];
            const size_t before = J.cols.size();
            features_in_area(C, J.grid, u, v, radius, oct - 1, oct + 1, J.cols);
            if (J.cols.size() == before) continue;
            J.qidx.push_back(i);
            J.row_ptr.push_back((int)J.cols.size());
        }
    });
    std::vector<uint16_t> dist;
    int rc = run_distances(m, jobs, qf, tf, dist);
    if (rc) return rc;
    parallel_for(npairs, [&](int j) {
        const OrbfeFrameView &C = cur[j], &L = last[j];
        const Job &J = jobs[j];
        int *mp = cur_mp_inout[j];
        int nmatches = 0;
        std::vector<int> rotHist[kHisto];
        for (size_t k = 0; k < J.qidx.size(); k++) {
            const int i = J.qidx[k];
            int bestDist = INT_MAX, bestIdx2 = -1;
            for (int c = J.row_ptr[k]; c < J.row_ptr[k + 1]; c++) {
                const int i2 = J.cols[c];
                if (mp[i2] >= 0) continue;  // :1562 already matched
                const int d = dist[J.pair_base + c];
                if (d < bestDist) { bestDist = d; bestIdx2 = i2; }
            }
            if (bestDist <= kThHigh) {
                mp[bestIdx2] = i;
                nmatches++;
                if (check_orientation) rotHist[rot_bin(L.keys_un[i].angle, C.keys_un[bestIdx2].angle)].push_back(bestIdx2);
            }
        }
        if (check_orientation) {
            int i1 = -1, i2 = -1, i3 = -1;
            three_maxima(rotHist, kHisto, i1, i2, i3);
            for (int b = 0; b < kHisto; b++) {
                if (b == i1 || b == i2 || b == i3) continue;
                for (int idx : rotHist[b]) { mp[idx] = -1; nmatches--; }
            }
        }
        nmatches_out[j] = nmatches;
    });
    return ORBFE_OK;
}

// ------------------------------------------------------------------------------------------------
// WindowSearch, ORBmatcher.cc:409-516
// ------------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------------
// SearchForInitialization, ORBmatcher.cc:598-713
// ------------------------------------------------------------------------------------------------
extern "C" int orbfe_search_for_initialization(OrbfeMatcher *m, const OrbfeFrameView *f1, const OrbfeFrameView *f2,
                                               float *prev_matched, int window, float nnratio, int check_orientation,
                                               int *match12_out, int *nmatches_out) {
    if (!m || !f1 || !f2 || !prev_matched || !match12_out || !nmatches_out) return ORBFE_ERR_ARG;
    if (!view_ok(*f1) || !view_ok(*f2)) return ORBFE_ERR_ARG;
    std::vector<Job> jobs(1);
    Job &J = jobs[0];
    build_grid(*f2, J.grid);
    J.row_ptr.push_back(0);
    for (int i1 = 0; i1 < f1->n; i1++) {
        const int level1 = f1->keys_un[i1].octave;
        if (level1 > 0) continue;  // :615-616
        const size_t before = J.cols.size();
        features_in_area(*f2, J.grid, prev_matched[2 * i1], prev_matched[2 * i1 + 1], (float)window, level1, level1, J.cols);
        if (J.cols.size() == before) continue;
        J.qidx.push_back(i1);
        J.row_ptr.push_back((int)J.cols.size());
    }
    std::vector<uint16_t> dist;
    std::vector<const OrbfeFrameView *> qf{f1}, tf{f2};
    int rc = run_distances(m, jobs, qf, tf, dist);
    if (rc) return rc;
    for (int i = 0; i < f1->n; i++) match12_out[i] = -1;
    std::vector<int> mdist(std::max(f2->n, 1), INT_MAX), m21(std::max(f2->n, 1), -1);
    int nmatches = 0;
    std::vector<int> rotHist[kHisto];
    for (size_t k = 0; k < J.qidx.size(); k++) {
        const int i1 = J.qidx[k];
        int bestDist = INT_MAX, bestDist2 = INT_MAX, bestIdx2 = -1;
        for (int c = J.row_ptr[k]; c < J.row_ptr[k + 1]; c++) {
            const int i2 = J.cols[c];
            const int d = dist[c];
            if (mdist[i2] <= d) continue;  // :637
            if (d < bestDist) { bestDist2 = bestDist; bestDist = d; bestIdx2 = i2; }
            else if (d < bestDist2) bestDist2 = d;
        }
        if (bestDist <= kThLow && (float)bestDist < (float)bestDist2 * nnratio) {  // :652-654
            if (m21[bestIdx2] >= 0) { match12_out[m21[bestIdx2]] = -1; nmatches--; }
            match12_out[i1] = bestIdx2;
            m21[bestIdx2] = i1;
            mdist[bestIdx2] = bestDist;
            nmatches++;
            if (check_orientation) rotHist[rot_bin(f1->keys_un[i1].angle, f2->keys_un[bestIdx2].angle)].push_back(i1);
        }
    }
    if (check_orientation) {
        int a = -1, b2 = -1, c3 = -1;
        three_maxima(rotHist, kHisto, a, b2, c3);
        for (int b = 0; b < kHisto; b++) {
            if (b == a || b == b2 || b == c3) continue;
            for (int idx1 : rotHist[b])
                if (match12_out[idx1] >= 0) { match12_out[idx1] = -1; nmatches--; }  // :697-701
        }
    }
    for (int i1 = 0; i1 < f1->n; i1++)  // :708-710
        if (match12_out[i1] >= 0) {
            prev_matched[2 * i1] = f2->keys_un[match12_out[i1]].x;
            prev_matched[2 * i1 + 1] = f2->keys_un[match12_out[i1]].y;
        }
    *nmatches_out = nmatches;
    return ORBFE_OK;
}

// Frame.cc:95-103: mvScaleFactors from GetScaleFactor()
extern "C" void orbfe_frame_scale_factors(float scale_factor, int nlevels, float *out) {
    if (!out || nlevels < 1) return;
    out[0] = 1.0f;
    for (int i = 1; i < nlevels; i++) out[i] = out[i - 1] * scale_factor;
}

// ================================================================================================
// Generic guided search: the common skeleton of ORBmatcher's projection/window routines.
//   for each query q (ascending): candidates = GetFeaturesInArea(u_q, v_q, r_q, lo_q, hi_q) on frame `f`;
//   best (and second best) distance over the candidates whose slot is still free; accept by `rule`;
//   optional rotation histogram.  Candidate lists on the host, ALL distances in one GPU launch, replay on the host.
// rule 0: best <= th_dist                                   (ORBmatcher.cc:1576, :1693)
// rule 1: best <= second*nnratio && best <= TH_HIGH          (:469, :586)
// rule 2: best <= TH_HIGH && !(bestLevel==secondLevel && best > nnratio*second)   (:113-121)
// hist 0: none; 1: push + filter (checkOrientation); 2: push only
// ================================================================================================
namespace {

struct GuidedQuery { float u, v, r; int lo, hi; const uint8_t *desc; float angle; };

int guided_search(OrbfeMatcher *m, const OrbfeFrameView &f, const std::vector<GuidedQuery> &Q, int rule, float nnratio,
                  int th_dist, int hist_mode, int *slot_owner, const std::vector<int> &owner_id, int *nmatches_out) {
    if (!g_force_host_replay.load() && !Q.empty() && f.n > 0) {
        // fused device kernel (grid, candidates, distances, greedy accept loop, rotation histogram in one launch)
        const size_t nq = Q.size();
        std::vector<float> qu(nq), qv(nq), qr(nq), qa(nq);
        std::vector<int> qlo(nq), qhi(nq), slot_new(f.n);
        std::vector<const uint8_t *> qd(nq);
        for (size_t q = 0; q < nq; q++) {
            qu[q] = Q[q].u; qv[q] = Q[q].v; qr[q] = Q[q].r; qa[q] = Q[q].angle;
            qlo[q] = Q[q].lo; qhi[q] = Q[q].hi; qd[q] = Q[q].desc;
        }
        const int rc = orbfe_guided_via_device(m, &f, (int)nq, qu.data(), qv.data(), qr.data(), qlo.data(), qhi.data(), qd.data(),
                                               qa.data(), rule, nnratio, th_dist, hist_mode == 1, slot_owner, slot_new.data(),
                                               nmatches_out);
        if (rc == ORBFE_OK) {
            for (int i = 0; i < f.n; i++)
                if (slot_new[i] >= 0) slot_owner[i] = owner_id[slot_new[i]];
            return ORBFE_OK;
        }
        if (rc != 1) return rc;  // 1 = does not fit the kernel: CSR distances + host replay below
    }
    std::vector<Job> jobs(1);
    Job &J = jobs[0];
    build_grid(f, J.grid);
    J.row_ptr.push_back(0);
    std::vector<uint8_t> qd;
    for (size_t q = 0; q < Q.size(); q++) {
        const size_t before = J.cols.size();
        features_in_area(f, J.grid, Q[q].u, Q[q].v, Q[q].r, Q[q].lo, Q[q].hi, J.cols);
        if (J.cols.size() == before) continue;
        J.qidx.push_back((int)q);
        J.row_ptr.push_back((int)J.cols.size());
        qd.insert(qd.end(), Q[q].desc, Q[q].desc + 32);
    }
    std::vector<uint16_t> dist(std::max<size_t>(J.cols.size(), 1));
    if (!J.cols.empty()) {
        const int rc = orbfe_hamming_csr(m, qd.data(), (int)J.qidx.size(), f.desc, f.n, J.row_ptr.data(), J.cols.data(), dist.data());
        if (rc) return rc;
    }
    int nmatches = 0;
    std::vector<int> rotHist[kHisto];
    for (size_t k = 0; k < J.qidx.size(); k++) {
        const int q = J.qidx[k];
        int bestDist = INT_MAX, bestDist2 = INT_MAX, bestIdx = -1, bestLevel = -1, bestLevel2 = -1;
        for (int c = J.row_ptr[k]; c < J.row_ptr[k + 1]; c++) {
            const int i2 = J.cols[c];
            if (slot_owner[i2] >= 0) continue;
            const int d = dist[c];
            if (d < bestDist) { bestDist2 = bestDist; bestDist = d; bestLevel2 = bestLevel; bestLevel = f.keys_un[i2].octave; bestIdx = i2; }
            else if (d < bestDist2) { bestLevel2 = f.keys_un[i2].octave; bestDist2 = d; }
        }
        bool accept;
        if (rule == 0) accept = bestDist <= th_dist;
        else if (rule == 1) accept = (float)bestDist <= (float)bestDist2 * nnratio && bestDist <= kThHigh;
        else accept = bestDist <= kThHigh && !(bestLevel == bestLevel2 && (float)bestDist > nnratio * (float)bestDist2);
        if (!accept) continue;
        slot_owner[bestIdx] = owner_id[q];
        nmatches++;
        if (hist_mode) rotHist[rot_bin(Q[q].angle, f.keys_un[bestIdx].angle)].push_back(bestIdx);
    }
    if (hist_mode == 1) {
        int i1 = -1, i2 = -1, i3 = -1;
        three_maxima(rotHist, kHisto, i1, i2, i3);
        for (int b = 0; b < kHisto; b++) {
            if (b == i1 || b == i2 || b == i3) continue;
            for (int idx : rotHist[b]) { slot_owner[idx] = -1; nmatches--; }
        }
    }
    *nmatches_out = nmatches;
    return ORBFE_OK;
}

}  // namespace

// WindowSearch(F1, F2, windowSize, matches, minLevel, maxLevel), ORBmatcher.cc:393-517: the guided skeleton with the
// F1 keypoint as window centre, same-octave filter, accept rule 1 (:469) and the rotation histogram of :472-489.
extern "C" int orbfe_window_search(OrbfeMatcher *m, const OrbfeFrameView *f1, const OrbfeFrameView *f2,
                                   const uint8_t *f1_has_mp, int window, int min_level, int max_level, float nnratio,
                                   int check_orientation, int *match21_out, int *nmatches_out) {
    if (!m || !f1 || !f2 || !f1_has_mp || !match21_out || !nmatches_out) return ORBFE_ERR_ARG;
    if (!view_ok(*f1) || !view_ok(*f2)) return ORBFE_ERR_ARG;
    const bool bMin = min_level > 0, bMax = max_level < INT_MAX;
    std::vector<GuidedQuery> Q;
    std::vector<int> id;
    for (int i1 = 0; i1 < f1->n; i1++) {
        if (!f1_has_mp[i1]) continue;
        const OrbfeKeyPoint &kp1 = f1->keys_un[i1];
        const int level1 = kp1.octave;
        if (bMin && level1 < min_level) continue;
        if (bMax && level1 > max_level) continue;
        Q.push_back({kp1.x, kp1.y, (float)window, level1, level1, f1->desc + (size_t)i1 * 32, kp1.angle});
        id.push_back(i1);
    }
    for (int i = 0; i < f2->n; i++) match21_out[i] = -1;
    *nmatches_out = 0;
    if (Q.empty() || f2->n == 0) return ORBFE_OK;
    return guided_search(m, *f2, Q, 1, nnratio, kThHigh, check_orientation ? 1 : 2, match21_out, id, nmatches_out);
}

// SearchByProjection(Frame &F, const vector<MapPoint*>&, th), ORBmatcher.cc:49-125
extern "C" int orbfe_search_local_points(OrbfeMatcher *m, const OrbfeFrameView *f, int npts, const uint8_t *in_view,
                                         const float *proj_xy, const int *level, const float *view_cos, const uint8_t *desc,
                                         float th, float nnratio, int *f_mp_inout, int *nmatches_out) {
    if (!m || !f || npts < 0 || !f_mp_inout || !nmatches_out || (npts > 0 && (!in_view || !proj_xy || !level || !view_cos || !desc)))
        return ORBFE_ERR_ARG;
    if (!view_ok(*f)) return ORBFE_ERR_ARG;
    for (int i = 0; i < npts; i++)
        if (in_view[i] && (unsigned)level[i] >= (unsigned)f->nlevels) return ORBFE_ERR_ARG;  // level indexes scale_factors
    const bool bFactor = th != 1.0f;
    std::vector<GuidedQuery> Q;
    std::vector<int> id;
    for (int i = 0; i < npts; i++) {
        if (!in_view[i]) continue;
        float r = view_cos[i] > 0.998 ? 2.5f : 4.0f;  // RadiusByViewingCos :127-133
        if (bFactor) r *= th;
        const int lv = level[i];
        Q.push_back({proj_xy[2 * i], proj_xy[2 * i + 1], r * f->scale_factors[lv], lv - 1, lv, desc + (size_t)i * 32, 0.f});
        id.push_back(i);
    }
    std::vector<int> owner(Q.size());
    for (size_t q = 0; q < Q.size(); q++) owner[q] = id[q];
    return guided_search(m, *f, Q, 2, nnratio, kThHigh, 0, f_mp_inout, owner, nmatches_out);
}

// SearchByProjection(Frame &CurrentFrame, KeyFrame *pKF, sAlreadyFound, th, ORBdist), ORBmatcher.cc:1622-1746
extern "C" int orbfe_search_by_projection_kf(OrbfeMatcher *m, const OrbfeFrameView *cur, int npts, const uint8_t *valid,
                                             const float *world, const float *min_dist, const uint8_t *desc,
                                             const float *kf_angle, const float *Tcw, float fx, float fy, float cx, float cy,
                                             float th, int orb_dist, int check_orientation, int *cur_mp_inout, int *nmatches_out) {
    if (!m || !cur || npts < 0 || !Tcw || !cur_mp_inout || !nmatches_out ||
        (npts > 0 && (!valid || !world || !min_dist || !desc || !kf_angle)))
        return ORBFE_ERR_ARG;
    if (!view_ok(*cur)) return ORBFE_ERR_ARG;
    float Ow[3];  // Ow = -Rcw.t()*tcw (:1628): gemm, double accumulation, alpha = -1
    for (int k = 0; k < 3; k++) {
        const double s = (double)Tcw[k] * (double)Tcw[3] + (double)Tcw[4 + k] * (double)Tcw[7] + (double)Tcw[8 + k] * (double)Tcw[11];
        Ow[k] = (float)(s * -1.0);
    }
    std::vector<GuidedQuery> Q;
    std::vector<int> id;
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
        Q.push_back({u, v, th * sf[lv], lv - 1, lv + 1, desc + (size_t)i * 32, kf_angle[i]});
        id.push_back(i);
    }
    return guided_search(m, *cur, Q, 0, 0.f, orb_dist, check_orientation ? 1 : 0, cur_mp_inout, id, nmatches_out);
}

// SearchByProjection(Frame &F1, Frame &F2, int windowSize, vpMapPointMatches2), ORBmatcher.cc:519-594
extern "C" int orbfe_search_by_projection_f1f2(OrbfeMatcher *m, const OrbfeFrameView *f1, const OrbfeFrameView *f2,
                                               const uint8_t *valid1, const float *world1, const float *Tc2w, float fx, float fy,
                                               float cx, float cy, int window, float nnratio, int *f2_mp_inout, int *nmatches_out) {
    if (!m || !f1 || !f2 || !Tc2w || !f2_mp_inout || !nmatches_out || (f1->n > 0 && (!valid1 || !world1))) return ORBFE_ERR_ARG;
    if (!view_ok(*f1) || !view_ok(*f2)) return ORBFE_ERR_ARG;
    std::vector<GuidedQuery> Q;
    std::vector<int> id;
    for (int i1 = 0; i1 < f1->n; i1++) {
        if (!valid1[i1]) continue;
        const int level1 = f1->keys_un[i1].octave;
        float xc[3];
        Rx_plus_t(Tc2w, world1 + 3 * (size_t)i1, xc);
        const float invz = (float)(1.0 / (double)xc[2]);
        Q.push_back({fx * xc[0] * invz + cx, fy * xc[1] * invz + cy, (float)window, level1, level1, f1->desc + (size_t)i1 * 32, 0.f});
        id.push_back(i1);
    }
    return guided_search(m, *f2, Q, 1, nnratio, kThHigh, 0, f2_mp_inout, id, nmatches_out);
}

// Exported form of the guided search for callers that do their own projection (the KeyFrame-level routines
// of the facade: Sim3 projection :286-407, SearchBySim3 :1267-1505, Fuse :1016-1265).
extern "C" int orbfe_guided_search(OrbfeMatcher *m, const OrbfeFrameView *f, int nq, const float *qu, const float *qv,
                                   const float *qr, const int32_t *qlo, const int32_t *qhi, const uint8_t *qdesc,
                                   const float *qangle, int rule, float nnratio, int th_dist, int hist_mode,
                                   int32_t *slot_owner_inout, int *nmatches_out) {
    if (!m || !f || nq < 0 || rule < 0 || rule > 2 || hist_mode < 0 || hist_mode > 2 || !slot_owner_inout || !nmatches_out)
        return ORBFE_ERR_ARG;
    if (nq > 0 && (!qu || !qv || !qr || !qlo || !qhi || !qdesc || (hist_mode && !qangle))) return ORBFE_ERR_ARG;
    std::vector<GuidedQuery> Q(nq);
    std::vector<int> id(nq);
    for (int q = 0; q < nq; q++) {
        Q[q] = {qu[q], qv[q], qr[q], qlo[q], qhi[q], qdesc + (size_t)q * 32, qangle ? qangle[q] : 0.f};
        id[q] = q;
    }
    return guided_search(m, *f, Q, rule, nnratio, th_dist, hist_mode, slot_owner_inout, id, nmatches_out);
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
