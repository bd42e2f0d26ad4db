/*
 * orb_oracle_match.c -- CPU ORACLE (matcher half).  TEST INFRASTRUCTURE ONLY -- see orb_oracle.h.
 *
 * Restates reference src/ORBmatcher.cc (DescriptorDistance, SearchByProjection(Frame,Frame),
 * WindowSearch, SearchForInitialization, ComputeThreeMaxima) and the candidate generator
 * src/Frame.cc (grid fill, PosInGrid, GetFeaturesInArea) on plain arrays.
 */
#include "orb_oracle.h"

#include <limits.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define TH_HIGH 100      /* ORBmatcher.cc:40 */
#define TH_LOW 50        /* ORBmatcher.cc:41 */
#define HISTO_LENGTH 30  /* ORBmatcher.cc:42 */

/* ORBmatcher::DescriptorDistance, ORBmatcher.cc:1794-1810 (SWAR popcount over 8 x 32-bit words) */
int orb_oracle_hamming(const uint8_t *a, const uint8_t *b) {
    int dist = 0;
    for (int i = 0; i < 8; i++) {
        uint32_t wa, wb;
        memcpy(&wa, a + 4 * i, 4);
        memcpy(&wb, b + 4 * i, 4);
        uint32_t v = wa ^ wb;
        v = v - ((v >> 1) & 0x55555555u);
        v = (v & 0x33333333u) + ((v >> 2) & 0x33333333u);
        dist += (int)((((v + (v >> 4)) & 0xF0F0F0Fu) * 0x1010101u) >> 24);
    }
    return dist;
}

/* Frame.cc:95-103: mvScaleFactors[i] = mvScaleFactors[i-1]*mfScaleFactor (float*float) where
 * mfScaleFactor = GetScaleFactor() = (float)(double member) == the ctor's float argument. */
void orb_oracle_frame_scale_factors(float sf, int nlevels, float *out) {
    out[0] = 1.0f;
    for (int i = 1; i < nlevels; i++) out[i] = out[i - 1] * sf;
}

/* Frame::PosInGrid, Frame.cc:267-277: round() (half away from zero) of a float expression */
static int pos_in_grid(const OrbOracleFrame *f, const OrbOracleKeyPoint *kp, int *px, int *py) {
    *px = (int)round((double)((kp->x - f->min_x) * f->grid_inv_w));
    *py = (int)round((double)((kp->y - f->min_y) * f->grid_inv_h));
    if (*px < 0 || *px >= ORB_ORACLE_GRID_COLS || *py < 0 || *py >= ORB_ORACLE_GRID_ROWS) return 0;
    return 1;
}

/* Frame.cc:116-123: features pushed to their cell in ascending index order */
void orb_oracle_frame_grid(OrbOracleFrame *f) {
    const int NC = ORB_ORACLE_GRID_COLS * ORB_ORACLE_GRID_ROWS;
    int *cnt = (int *)calloc((size_t)NC + 1, sizeof(int));
    int *cell = (int *)malloc(sizeof(int) * (size_t)(f->n > 0 ? f->n : 1));
    for (int i = 0; i < f->n; i++) {
        int px, py;
        cell[i] = pos_in_grid(f, &f->keys_un[i], &px, &py) ? px * ORB_ORACLE_GRID_ROWS + py : -1;
        if (cell[i] >= 0) cnt[cell[i]]++;
    }
    f->cell_start[0] = 0;
    for (int c = 0; c < NC; c++) f->cell_start[c + 1] = f->cell_start[c] + cnt[c];
    memset(cnt, 0, sizeof(int) * (size_t)NC);
    for (int i = 0; i < f->n; i++)
        if (cell[i] >= 0) f->cell_items[f->cell_start[cell[i]] + cnt[cell[i]]++] = i;
    free(cnt);
    free(cell);
}

/* Frame::GetFeaturesInArea, Frame.cc:200-265 */
int orb_oracle_features_in_area(const OrbOracleFrame *f, float x, float y, float r, int minLevel,
                                int maxLevel, int *out, int cap) {
    int n = 0;
    int nMinCellX = (int)floor((double)((x - f->min_x - r) * f->grid_inv_w)); /* :205 */
    if (nMinCellX < 0) nMinCellX = 0;
    if (nMinCellX >= ORB_ORACLE_GRID_COLS) return 0;
    int nMaxCellX = (int)ceil((double)((x - f->min_x + r) * f->grid_inv_w)); /* :210 */
    if (nMaxCellX > ORB_ORACLE_GRID_COLS - 1) nMaxCellX = ORB_ORACLE_GRID_COLS - 1;
    if (nMaxCellX < 0) return 0;
    int nMinCellY = (int)floor((double)((y - f->min_y - r) * f->grid_inv_h)); /* :215 */
    if (nMinCellY < 0) nMinCellY = 0;
    if (nMinCellY >= ORB_ORACLE_GRID_ROWS) return 0;
    int nMaxCellY = (int)ceil((double)((y - f->min_y + r) * f->grid_inv_h)); /* :220 */
    if (nMaxCellY > ORB_ORACLE_GRID_ROWS - 1) nMaxCellY = ORB_ORACLE_GRID_ROWS - 1;
    if (nMaxCellY < 0) return 0;

    int bCheckLevels = 1, bSameLevel = 0; /* :225-231 */
    if (minLevel == -1 && maxLevel == -1) bCheckLevels = 0;
    else if (minLevel == maxLevel) bSameLevel = 1;

    for (int ix = nMinCellX; ix <= nMaxCellX; ix++)
        for (int iy = nMinCellY; iy <= nMaxCellY; iy++) {
            const int c = ix * ORB_ORACLE_GRID_ROWS + iy;
            for (int j = f->cell_start[c]; j < f->cell_start[c + 1]; j++) {
                const int idx = f->cell_items[j];
                const OrbOracleKeyPoint *kp = &f->keys_un[idx];
                if (bCheckLevels && !bSameLevel) {
                    if (kp->octave < minLevel || kp->octave > maxLevel) continue;
                } else if (bSameLevel) {
                    if (kp->octave != minLevel) continue;
                }
                if (fabsf(kp->x - x) > r || fabsf(kp->y - y) > r) continue; /* :254 */
                if (n < cap) out[n] = idx;
                n++;
            }
        }
    return n;
}

/* ComputeThreeMaxima, ORBmatcher.cc:1748-1789 */
void orb_oracle_three_maxima(const int *counts, int L, int *ind1, int *ind2, int *ind3) {
    int max1 = 0, max2 = 0, max3 = 0;
    *ind1 = *ind2 = *ind3 = -1;
    for (int i = 0; i < L; i++) {
        const int s = counts[i];
        if (s > max1) {
            max3 = max2; max2 = max1; max1 = s;
            *ind3 = *ind2; *ind2 = *ind1; *ind1 = i;
        } else if (s > max2) {
            max3 = max2; max2 = s;
            *ind3 = *ind2; *ind2 = i;
        } else if (s > max3) {
            max3 = s; *ind3 = i;
        }
    }
    if ((float)max2 < 0.1f * (float)max1) { *ind2 = -1; *ind3 = -1; }
    else if ((float)max3 < 0.1f * (float)max1) { *ind3 = -1; }
}

/* rotation-histogram bin, e.g. ORBmatcher.cc:1583-1590 */
static int rot_bin(float a1, float a2) {
    const float factor = 1.0f / HISTO_LENGTH;
    float rot = a1 - a2;
    if (rot < 0.0) rot += 360.0f;
    int bin = (int)roundf(rot * factor); /* round(float) -> half away from zero */
    if (bin == HISTO_LENGTH) bin = 0;
    return bin;
}

typedef struct { int *v; int n, cap; } IVec;
static void ivec_push(IVec *a, int x) {
    if (a->n == a->cap) { a->cap = a->cap ? a->cap * 2 : 64; a->v = (int *)realloc(a->v, sizeof(int) * (size_t)a->cap); }
    a->v[a->n++] = x;
}

/* SearchByProjection(Frame &CurrentFrame, const Frame &LastFrame, float th), ORBmatcher.cc:1507-1620 */
int orb_oracle_search_by_projection_ff(const OrbOracleFrame *cur, const OrbOracleFrame *last,
                                       const uint8_t *last_has_mp, const uint8_t *last_outlier,
                                       const float *last_world, const float *Tcw,
                                       float fx, float fy, float cx, float cy, float th,
                                       int check_orientation, int *cur_mp) {
    int nmatches = 0;
    IVec hist[HISTO_LENGTH];
    memset(hist, 0, sizeof(hist));
    int *cand = (int *)malloc(sizeof(int) * (size_t)(cur->n > 0 ? cur->n : 1));
    for (int i = 0; i < last->n; i++) {
        if (!last_has_mp[i] || last_outlier[i]) continue;
        /* :1527-1528: x3Dc = Rcw*x3Dw+tcw -- one cv::gemm(Rcw, x3Dw, 1, tcw, 1) on CV_32F 3x3 * 3x1 (see cv_Rx_plus_t) */
        const float *X = last_world + 3 * i;
        float xc3[3];
        orb_oracle_cv_Rx_plus_t(Tcw, X, xc3);
        const float xc = xc3[0], yc = xc3[1];
        const float invzc = (float)(1.0 / (double)xc3[2]); /* :1532 */
        const float u = fx * xc * invzc + cx;              /* :1534-1535 */
        const float v = fy * yc * invzc + cy;
        if (u < cur->min_x || u > cur->max_x) continue;
        if (v < cur->min_y || v > cur->max_y) continue;
        const int oct = last->keys_un[i].octave; /* LastFrame.mvKeys[i].octave */
        const float radius = th * cur->scale_factors[oct]; /* :1547 */
        const int nc = orb_oracle_features_in_area(cur, u, v, radius, oct - 1, oct + 1, cand, cur->n);
        if (nc == 0) continue;
        const uint8_t *dMP = last->desc + (size_t)i * 32;
        int bestDist = INT_MAX, bestIdx2 = -1;
        for (int c = 0; c < nc; c++) {
            const int i2 = cand[c];
            if (cur_mp[i2] >= 0) continue; /* :1562 */
            const int dist = orb_oracle_hamming(dMP, cur->desc + (size_t)i2 * 32);
            if (dist < bestDist) { bestDist = dist; bestIdx2 = i2; }
        }
        if (bestDist <= TH_HIGH) {
            cur_mp[bestIdx2] = i;
            nmatches++;
            if (check_orientation)
                ivec_push(&hist[rot_bin(last->keys_un[i].angle, cur->keys_un[bestIdx2].angle)], bestIdx2);
        }
    }
    if (check_orientation) {
        int counts[HISTO_LENGTH], i1, i2, i3;
        for (int b = 0; b < HISTO_LENGTH; b++) counts[b] = hist[b].n;
        orb_oracle_three_maxima(counts, HISTO_LENGTH, &i1, &i2, &i3);
        for (int b = 0; b < HISTO_LENGTH; b++) {
            if (b == i1 || b == i2 || b == i3) continue;
            for (int j = 0; j < hist[b].n; j++) { cur_mp[hist[b].v[j]] = -1; nmatches--; }
        }
    }
    for (int b = 0; b < HISTO_LENGTH; b++) free(hist[b].v);
    free(cand);
    return nmatches;
}

/* WindowSearch, ORBmatcher.cc:409-516 */
int orb_oracle_window_search(const OrbOracleFrame *f1, const OrbOracleFrame *f2, const uint8_t *f1_has_mp,
                             int window, int minLevel, int maxLevel, float nnratio,
                             int check_orientation, int *m21) {
    int nmatches = 0;
    for (int i = 0; i < f2->n; i++) m21[i] = -1;
    IVec hist[HISTO_LENGTH];
    memset(hist, 0, sizeof(hist));
    const int bMin = minLevel > 0, bMax = maxLevel < INT_MAX;
    int *cand = (int *)malloc(sizeof(int) * (size_t)(f2->n > 0 ? f2->n : 1));
    for (int i1 = 0; i1 < f1->n; i1++) {
        if (!f1_has_mp[i1]) continue;
        const OrbOracleKeyPoint *kp1 = &f1->keys_un[i1];
        const int level1 = kp1->octave;
        if (bMin && level1 < minLevel) continue;
        if (bMax && level1 > maxLevel) continue;
        const int nc = orb_oracle_features_in_area(f2, kp1->x, kp1->y, (float)window, level1, level1, cand, f2->n);
        if (nc == 0) continue;
        const uint8_t *d1 = f1->desc + (size_t)i1 * 32;
        int bestDist = INT_MAX, bestDist2 = INT_MAX, bestIdx2 = -1;
        for (int c = 0; c < nc; c++) {
            const int i2 = cand[c];
            if (m21[i2] >= 0) continue; /* :451 */
            const int dist = orb_oracle_hamming(d1, f2->desc + (size_t)i2 * 32);
            if (dist < bestDist) { bestDist2 = bestDist; bestDist = dist; bestIdx2 = i2; }
            else if (dist < bestDist2) bestDist2 = dist;
        }
        /* :469  int <= int*float  (bestDist2 may be INT_MAX -> float) */
        if ((float)bestDist <= (float)bestDist2 * nnratio && bestDist <= TH_HIGH) {
            m21[bestIdx2] = i1;
            nmatches++;
            ivec_push(&hist[rot_bin(kp1->angle, f2->keys_un[bestIdx2].angle)], bestIdx2);
        }
    }
    if (check_orientation) {
        int counts[HISTO_LENGTH], i1, i2, i3;
        for (int b = 0; b < HISTO_LENGTH; b++) counts[b] = hist[b].n;
        orb_oracle_three_maxima(counts, HISTO_LENGTH, &i1, &i2, &i3);
        for (int b = 0; b < HISTO_LENGTH; b++) {
            if (b == i1 || b == i2 || b == i3) continue;
            for (int j = 0; j < hist[b].n; j++) { m21[hist[b].v[j]] = -1; nmatches--; }
        }
    }
    for (int b = 0; b < HISTO_LENGTH; b++) free(hist[b].v);
    free(cand);
    return nmatches;
}

/* SearchForInitialization, ORBmatcher.cc:598-713 */
int orb_oracle_search_for_initialization(const OrbOracleFrame *f1, const OrbOracleFrame *f2,
                                         float *prev, int window, float nnratio,
                                         int check_orientation, int *m12) {
    int nmatches = 0;
    for (int i = 0; i < f1->n; i++) m12[i] = -1;
    IVec hist[HISTO_LENGTH];
    memset(hist, 0, sizeof(hist));
    int *mdist = (int *)malloc(sizeof(int) * (size_t)(f2->n > 0 ? f2->n : 1));
    int *m21 = (int *)malloc(sizeof(int) * (size_t)(f2->n > 0 ? f2->n : 1));
    for (int i = 0; i < f2->n; i++) { mdist[i] = INT_MAX; m21[i] = -1; }
    int *cand = (int *)malloc(sizeof(int) * (size_t)(f2->n > 0 ? f2->n : 1));
    for (int i1 = 0; i1 < f1->n; i1++) {
        const OrbOracleKeyPoint *kp1 = &f1->keys_un[i1];
        const int level1 = kp1->octave;
        if (level1 > 0) continue; /* :615-616 */
        const int nc = orb_oracle_features_in_area(f2, prev[2 * i1], prev[2 * i1 + 1], (float)window, level1, level1, cand, f2->n);
        if (nc == 0) continue;
        const uint8_t *d1 = f1->desc + (size_t)i1 * 32;
        int bestDist = INT_MAX, bestDist2 = INT_MAX, bestIdx2 = -1;
        for (int c = 0; c < nc; c++) {
            const int i2 = cand[c];
            const int dist = orb_oracle_hamming(d1, f2->desc + (size_t)i2 * 32);
            if (mdist[i2] <= dist) continue; /* :637 */
            if (dist < bestDist) { bestDist2 = bestDist; bestDist = dist; bestIdx2 = i2; }
            else if (dist < bestDist2) bestDist2 = dist;
        }
        if (bestDist <= TH_LOW) {
            if ((float)bestDist < (float)bestDist2 * nnratio) { /* :654 */
                if (m21[bestIdx2] >= 0) { m12[m21[bestIdx2]] = -1; nmatches--; }
                m12[i1] = bestIdx2;
                m21[bestIdx2] = i1;
                mdist[bestIdx2] = bestDist;
                nmatches++;
                if (check_orientation)
                    ivec_push(&hist[rot_bin(kp1->angle, f2->keys_un[bestIdx2].angle)], i1);
            }
        }
    }
    if (check_orientation) {
        int counts[HISTO_LENGTH], a, b2, c3;
        for (int b = 0; b < HISTO_LENGTH; b++) counts[b] = hist[b].n;
        orb_oracle_three_maxima(counts, HISTO_LENGTH, &a, &b2, &c3);
        for (int b = 0; b < HISTO_LENGTH; b++) {
            if (b == a || b == b2 || b == c3) continue;
            for (int j = 0; j < hist[b].n; j++) {
                const int idx1 = hist[b].v[j];
                if (m12[idx1] >= 0) { m12[idx1] = -1; nmatches--; } /* :697-701 */
            }
        }
    }
    for (int i1 = 0; i1 < f1->n; i1++) /* :708-710 */
        if (m12[i1] >= 0) {
            prev[2 * i1] = f2->keys_un[m12[i1]].x;
            prev[2 * i1 + 1] = f2->keys_un[m12[i1]].y;
        }
    for (int b = 0; b < HISTO_LENGTH; b++) free(hist[b].v);
    free(mdist); free(m21); free(cand);
    return nmatches;
}

/* dense best/second-best sweep (config 5 primitive): strict-< update in ascending db order */
void orb_oracle_knn2(const uint8_t *q, int nq, const uint8_t *db, long ndb,
                     int *best_dist, int *best_idx, int *second_dist) {
    for (int i = 0; i < nq; i++) {
        const uint64_t *a = (const uint64_t *)(const void *)(q + (size_t)i * 32);
        uint64_t a0, a1, a2, a3;
        memcpy(&a0, a, 8); memcpy(&a1, a + 1, 8); memcpy(&a2, a + 2, 8); memcpy(&a3, a + 3, 8);
        int b1 = INT_MAX, b2 = INT_MAX, bi = -1;
        for (long j = 0; j < ndb; j++) {
            uint64_t w[4];
            memcpy(w, db + (size_t)j * 32, 32);
            int d = __builtin_popcountll(a0 ^ w[0]) + __builtin_popcountll(a1 ^ w[1]) +
                    __builtin_popcountll(a2 ^ w[2]) + __builtin_popcountll(a3 ^ w[3]);
            if (d < b1) { b2 = b1; b1 = d; bi = (int)j; }
            else if (d < b2) b2 = d;
        }
        best_dist[i] = b1; best_idx[i] = bi; second_dist[i] = b2;
    }
}

/* ------------------------------------------------------------------------------------------------
 * cv::Mat float algebra used by the projecting matchers (OpenCV 2.4 core semantics):
 *   A*x + t  (MatExpr -> ONE cv::gemm(A, x, 1, t, 1), CV_32F, 3x3 * 3x1, flags 0): matmul.cpp takes its unrolled
 *            small-matrix branch (inner length 2..4, result as wide or as high as that length): the three products
 *            are summed in FLOAT, left to right, and the result is (float)((double)sum*alpha + (double)t*beta).
 *            Pinned to python-cv2's cv2.gemm by tests/test_oracle_vs_ref.py (golden vectors tests/golden/opencv_gemm.npz);
 *            round 1 restated this from memory as a double accumulation, which cv2 contradicts on ~85 % of random inputs;
 *   -R.t()*t (gemm with GEMM_1_T, alpha = -1): the general path, double accumulation, * alpha, round (also pinned);
 *   cv::norm(v) for CV_32F: sqrt of the double sum of squares (also pinned).
 * ---------------------------------------------------------------------------------------------- */
void orb_oracle_cv_Rx_plus_t(const float *T /*3x4 row-major [R|t]*/, const float *X, float out[3]) {
    for (int k = 0; k < 3; k++) {
        float s = T[4 * k + 0] * X[0];       /* -ffp-contract=off: every product and sum individually rounded */
        s = s + T[4 * k + 1] * X[1];
        s = s + T[4 * k + 2] * X[2];
        out[k] = (float)((double)s * 1.0 + (double)T[4 * k + 3] * 1.0);
    }
}
static void cv_Rx_plus_t(const float *T, const float *X, float out[3]) { orb_oracle_cv_Rx_plus_t(T, X, out); }
static void cv_camera_centre(const float *T, float Ow[3]) { /* Ow = -Rcw.t()*tcw */
    for (int k = 0; k < 3; k++) {
        double s = (double)T[0 * 4 + k] * (double)T[3] + (double)T[1 * 4 + k] * (double)T[7] + (double)T[2 * 4 + k] * (double)T[11];
        Ow[k] = (float)(s * -1.0);
    }
}
static float cv_norm3(const float *v) {
    return (float)sqrt((double)v[0] * (double)v[0] + (double)v[1] * (double)v[1] + (double)v[2] * (double)v[2]);
}

/* SearchByProjection(Frame &F, const vector<MapPoint*>&, th), ORBmatcher.cc:49-125.
 * Per map point: in_view = mbTrackInView && !isBad(); proj = (mTrackProjX, mTrackProjY); level = mnTrackScaleLevel;
 * view_cos = mTrackViewCos; desc = GetDescriptor().  f_mp[i2] >= 0 <=> F.mvpMapPoints[i2] != NULL on entry;
 * on exit f_mp[i2] = index of the map point assigned.  Returns nmatches. */
int orb_oracle_search_local_points(const OrbOracleFrame *f, int npts, const uint8_t *in_view, const float *proj_xy,
                                   const int *level, const float *view_cos, const uint8_t *desc, float th,
                                   float nnratio, int *f_mp) {
    int nmatches = 0;
    const int bFactor = th != 1.0f;
    int *cand = (int *)malloc(sizeof(int) * (size_t)(f->n > 0 ? f->n : 1));
    for (int iMP = 0; iMP < npts; iMP++) {
        if (!in_view[iMP]) continue;
        const int nPredictedLevel = level[iMP];
        float r = view_cos[iMP] > 0.998 ? 2.5f : 4.0f; /* RadiusByViewingCos :127-133 (float compared to a double literal) */
        if (bFactor) r *= th;
        const int nc = orb_oracle_features_in_area(f, proj_xy[2 * iMP], proj_xy[2 * iMP + 1], r * f->scale_factors[nPredictedLevel],
                                                   nPredictedLevel - 1, nPredictedLevel, cand, f->n);
        if (nc == 0) continue;
        const uint8_t *d = desc + (size_t)iMP * 32;
        int bestDist = INT_MAX, bestLevel = -1, bestDist2 = INT_MAX, bestLevel2 = -1, bestIdx = -1;
        for (int c = 0; c < nc; c++) {
            const int idx = cand[c];
            if (f_mp[idx] >= 0) continue;
            const int dist = orb_oracle_hamming(d, f->desc + (size_t)idx * 32);
            if (dist < bestDist) { bestDist2 = bestDist; bestDist = dist; bestLevel2 = bestLevel; bestLevel = f->keys_un[idx].octave; bestIdx = idx; }
            else if (dist < bestDist2) { bestLevel2 = f->keys_un[idx].octave; bestDist2 = dist; }
        }
        if (bestDist <= TH_HIGH) {
            if (bestLevel == bestLevel2 && (float)bestDist > nnratio * (float)bestDist2) continue;
            f_mp[bestIdx] = iMP;
            nmatches++;
        }
    }
    free(cand);
    return nmatches;
}

/* SearchByProjection(Frame &CurrentFrame, KeyFrame *pKF, sAlreadyFound, th, ORBdist), ORBmatcher.cc:1622-1746.
 * Per keyframe feature i: valid[i] = has a map point && !isBad() && not in sAlreadyFound; world/min_dist/desc of that
 * point; kf_angle[i] = pKF->GetKeyPointUn(i).angle.  cur_mp as in orb_oracle_search_by_projection_ff. */
int orb_oracle_search_by_projection_kf(const OrbOracleFrame *cur, int npts, const uint8_t *valid, const float *world,
                                       const float *min_dist, const uint8_t *desc, const float *kf_angle,
                                       const float *Tcw, float fx, float fy, float cx, float cy, float th, int orb_dist,
                                       int check_orientation, int *cur_mp) {
    int nmatches = 0;
    IVec hist[HISTO_LENGTH];
    memset(hist, 0, sizeof(hist));
    float Ow[3];
    cv_camera_centre(Tcw, Ow); /* :1628 */
    int *cand = (int *)malloc(sizeof(int) * (size_t)(cur->n > 0 ? cur->n : 1));
    for (int i = 0; i < npts; i++) {
        if (!valid[i]) continue;
        const float *X = world + 3 * i;
        float xc3[3];
        cv_Rx_plus_t(Tcw, X, xc3);
        const float invzc = (float)(1.0 / (double)xc3[2]);
        const float u = fx * xc3[0] * invzc + cx;
        const float v = fy * xc3[1] * invzc + cy;
        if (u < cur->min_x || u > cur->max_x) continue;
        if (v < cur->min_y || v > cur->max_y) continue;
        /* :1664-1670 predicted scale level */
        const float PO[3] = {X[0] - Ow[0], X[1] - Ow[1], X[2] - Ow[2]};
        const float dist3D = cv_norm3(PO);
        const float ratio = dist3D / min_dist[i];
        int it = 0; /* lower_bound: first scale factor >= ratio */
        while (it < cur->nlevels && cur->scale_factors[it] < ratio) it++;
        const int nPredictedLevel = it < cur->nlevels - 1 ? it : cur->nlevels - 1;
        const float radius = th * cur->scale_factors[nPredictedLevel];
        const int nc = orb_oracle_features_in_area(cur, u, v, radius, nPredictedLevel - 1, nPredictedLevel + 1, cand, cur->n);
        if (nc == 0) continue;
        const uint8_t *dMP = desc + (size_t)i * 32;
        int bestDist = INT_MAX, bestIdx2 = -1;
        for (int c = 0; c < nc; c++) {
            const int i2 = cand[c];
            if (cur_mp[i2] >= 0) continue;
            const int dist = orb_oracle_hamming(dMP, cur->desc + (size_t)i2 * 32);
            if (dist < bestDist) { bestDist = dist; bestIdx2 = i2; }
        }
        if (bestDist <= orb_dist) {
            cur_mp[bestIdx2] = i;
            nmatches++;
            if (check_orientation) ivec_push(&hist[rot_bin(kf_angle[i], cur->keys_un[bestIdx2].angle)], bestIdx2);
        }
    }
    if (check_orientation) {
        int counts[HISTO_LENGTH], i1, i2, i3;
        for (int b = 0; b < HISTO_LENGTH; b++) counts[b] = hist[b].n;
        orb_oracle_three_maxima(counts, HISTO_LENGTH, &i1, &i2, &i3);
        for (int b = 0; b < HISTO_LENGTH; b++) {
            if (b == i1 || b == i2 || b == i3) continue;
            for (int j = 0; j < hist[b].n; j++) { cur_mp[hist[b].v[j]] = -1; nmatches--; }
        }
    }
    for (int b = 0; b < HISTO_LENGTH; b++) free(hist[b].v);
    free(cand);
    return nmatches;
}

/* SearchByProjection(Frame &F1, Frame &F2, int windowSize, vpMapPointMatches2), ORBmatcher.cc:519-594.
 * valid1[i1] = F1 has a map point there && !isBad() && the point is not already among F2's matches (:533-537).
 * f2_mp: copy of F2.mvpMapPoints occupancy on entry (>=0 occupied), on exit index i1 for new matches. */
int orb_oracle_search_by_projection_f1f2(const OrbOracleFrame *f1, const OrbOracleFrame *f2, const uint8_t *valid1,
                                         const float *world1, const float *Tc2w, float fx, float fy, float cx, float cy,
                                         int window, float nnratio, int *f2_mp) {
    int nmatches = 0;
    int *cand = (int *)malloc(sizeof(int) * (size_t)(f2->n > 0 ? f2->n : 1));
    for (int i1 = 0; i1 < f1->n; i1++) {
        if (!valid1[i1]) continue;
        const int level1 = f1->keys_un[i1].octave;
        float xc3[3];
        cv_Rx_plus_t(Tc2w, world1 + 3 * i1, xc3);
        const float invzc2 = (float)(1.0 / (double)xc3[2]);
        const float u2 = fx * xc3[0] * invzc2 + cx;
        const float v2 = fy * xc3[1] * invzc2 + cy;
        const int nc = orb_oracle_features_in_area(f2, u2, v2, (float)window, level1, level1, cand, f2->n);
        if (nc == 0) continue;
        const uint8_t *d1 = f1->desc + (size_t)i1 * 32;
        int bestDist = INT_MAX, bestDist2 = INT_MAX, bestIdx2 = -1;
        for (int c = 0; c < nc; c++) {
            const int i2 = cand[c];
            if (f2_mp[i2] >= 0) continue;
            const int dist = orb_oracle_hamming(d1, f2->desc + (size_t)i2 * 32);
            if (dist < bestDist) { bestDist2 = bestDist; bestDist = dist; bestIdx2 = i2; }
            else if (dist < bestDist2) bestDist2 = dist;
        }
        if ((float)bestDist <= (float)bestDist2 * nnratio && bestDist <= TH_HIGH) { /* :586 */
            f2_mp[bestIdx2] = i1;
            nmatches++;
        }
    }
    free(cand);
    return nmatches;
}

/* ------------------------------------------------------------------------------------------------
 * SearchByBoW -- brute force restricted to features of the same vocabulary node.
 * A DBoW2::FeatureVector (std::map<NodeId, vector<unsigned>>) is given as: ascending node ids, CSR pointer,
 * feature indices in insertion order.
 * variant 0: SearchByBoW(KeyFrame*, Frame&, matches)   ORBmatcher.cc:155-284   (out[i2] = idx1, F slots)
 * variant 1: SearchByBoW(KeyFrame*, KeyFrame*, matches12) ORBmatcher.cc:715-850 (out[idx1] = idx2)
 * valid1[i] = KF1 feature has a map point && !isBad(); valid2 likewise (variant 1 only; variant 0 ignores it).
 * ---------------------------------------------------------------------------------------------- */
int orb_oracle_search_by_bow(int variant, int n1, const uint8_t *desc1, const uint8_t *valid1, const float *angle1,
                             int nn1, const int *ids1, const int *ptr1, const int *items1,
                             int n2, const uint8_t *desc2, const uint8_t *valid2, const float *angle2,
                             int nn2, const int *ids2, const int *ptr2, const int *items2,
                             float nnratio, int check_orientation, int *out) {
    int nmatches = 0;
    const int nout = variant == 0 ? n2 : n1;
    for (int i = 0; i < nout; i++) out[i] = -1;
    uint8_t *matched2 = (uint8_t *)calloc((size_t)(n2 > 0 ? n2 : 1), 1);
    IVec hist[HISTO_LENGTH];
    memset(hist, 0, sizeof(hist));
    int a = 0, b = 0;
    while (a < nn1 && b < nn2) {
        if (ids1[a] == ids2[b]) {
            for (int p1 = ptr1[a]; p1 < ptr1[a + 1]; p1++) {
                const int idx1 = items1[p1];
                if (!valid1[idx1]) continue;
                const uint8_t *d1 = desc1 + (size_t)idx1 * 32;
                int bestDist1 = INT_MAX, bestIdx2 = -1, bestDist2 = INT_MAX;
                for (int p2 = ptr2[b]; p2 < ptr2[b + 1]; p2++) {
                    const int idx2 = items2[p2];
                    if (variant == 0) { if (out[idx2] >= 0) continue; }          /* :204 */
                    else { if (matched2[idx2] || !valid2[idx2]) continue; }      /* :773-778 */
                    const int dist = orb_oracle_hamming(d1, desc2 + (size_t)idx2 * 32);
                    if (dist < bestDist1) { bestDist2 = bestDist1; bestDist1 = dist; bestIdx2 = idx2; }
                    else if (dist < bestDist2) bestDist2 = dist;
                }
                const int pass = variant == 0 ? (bestDist1 <= TH_LOW) : (bestDist1 < TH_LOW); /* :224 vs :797 */
                if (pass && (float)bestDist1 < nnratio * (float)bestDist2) {
                    if (variant == 0) out[bestIdx2] = idx1;
                    else { out[idx1] = bestIdx2; matched2[bestIdx2] = 1; }
                    if (check_orientation)
                        ivec_push(&hist[rot_bin(angle1[idx1], angle2[bestIdx2])], variant == 0 ? bestIdx2 : idx1);
                    nmatches++;
                }
            }
            a++; b++;
        } else if (ids1[a] < ids2[b]) {
            while (a < nn1 && ids1[a] < ids2[b]) a++;   /* lower_bound */
        } else {
            while (b < nn2 && ids2[b] < ids1[a]) b++;
        }
    }
    if (check_orientation) {
        int counts[HISTO_LENGTH], i1, i2, i3;
        for (int k = 0; k < HISTO_LENGTH; k++) counts[k] = hist[k].n;
        orb_oracle_three_maxima(counts, HISTO_LENGTH, &i1, &i2, &i3);
        for (int k = 0; k < HISTO_LENGTH; k++) {
            if (k == i1 || k == i2 || k == i3) continue;
            for (int j = 0; j < hist[k].n; j++) { out[hist[k].v[j]] = -1; nmatches--; }
        }
    }
    for (int k = 0; k < HISTO_LENGTH; k++) free(hist[k].v);
    free(matched2);
    return nmatches;
}

/* ------------------------------------------------------------------------------------------------
 * The inner "guided search" skeleton shared by ORBmatcher's projection routines, on explicit queries:
 * for each query q (ascending): candidates = GetFeaturesInArea(u, v, r, lo, hi); best / second best over the
 * candidates whose slot is free; accept by rule:
 *   0: best <= th_dist                                           (ORBmatcher.cc:394, :1107, :1239, :1576, :1693)
 *   1: best <= second*nnratio && best <= TH_HIGH                 (:469, :586)
 *   2: best <= TH_HIGH && !(bestLevel==secondLevel && best > nnratio*second)   (:113-121)
 * hist_mode 0: none; 1: rotation histogram + three-maxima filter; 2: histogram filled but not applied.
 * slot_owner[i2] >= 0 on entry = occupied; on exit = owner_id of the accepted query.
 * ---------------------------------------------------------------------------------------------- */
int orb_oracle_guided_search(const OrbOracleFrame *f, int nq, const float *qu, const float *qv, const float *qr,
                             const int *qlo, const int *qhi, const uint8_t *qdesc, const float *qangle, int rule,
                             float nnratio, int th_dist, int hist_mode, int *slot_owner) {
    int nmatches = 0;
    IVec hist[HISTO_LENGTH];
    memset(hist, 0, sizeof(hist));
    int *cand = (int *)malloc(sizeof(int) * (size_t)(f->n > 0 ? f->n : 1));
    for (int q = 0; q < nq; q++) {
        const int nc = orb_oracle_features_in_area(f, qu[q], qv[q], qr[q], qlo[q], qhi[q], cand, f->n);
        if (nc == 0) continue;
        const uint8_t *d = qdesc + (size_t)q * 32;
        int bestDist = INT_MAX, bestDist2 = INT_MAX, bestIdx = -1, bestLevel = -1, bestLevel2 = -1;
        for (int c = 0; c < nc; c++) {
            const int i2 = cand[c];
            if (slot_owner[i2] >= 0) continue;
            const int dist = orb_oracle_hamming(d, f->desc + (size_t)i2 * 32);
            if (dist < bestDist) { bestDist2 = bestDist; bestDist = dist; bestLevel2 = bestLevel; bestLevel = f->keys_un[i2].octave; bestIdx = i2; }
            else if (dist < bestDist2) { bestLevel2 = f->keys_un[i2].octave; bestDist2 = dist; }
        }
        int accept;
        if (rule == 0) accept = bestDist <= th_dist;
        else if (rule == 1) accept = (float)bestDist <= (float)bestDist2 * nnratio && bestDist <= TH_HIGH;
        else accept = bestDist <= TH_HIGH && !(bestLevel == bestLevel2 && (float)bestDist > nnratio * (float)bestDist2);
        if (!accept) continue;
        slot_owner[bestIdx] = q;
        nmatches++;
        if (hist_mode) ivec_push(&hist[rot_bin(qangle[q], f->keys_un[bestIdx].angle)], bestIdx);
    }
    if (hist_mode == 1) {
        int counts[HISTO_LENGTH], i1, i2, i3;
        for (int b = 0; b < HISTO_LENGTH; b++) counts[b] = hist[b].n;
        orb_oracle_three_maxima(counts, HISTO_LENGTH, &i1, &i2, &i3);
        for (int b = 0; b < HISTO_LENGTH; b++) {
            if (b == i1 || b == i2 || b == i3) continue;
            for (int j = 0; j < hist[b].n; j++) { slot_owner[hist[b].v[j]] = -1; nmatches--; }
        }
    }
    for (int b = 0; b < HISTO_LENGTH; b++) free(hist[b].v);
    free(cand);
    return nmatches;
}

/* CheckDistEpipolarLine, ORBmatcher.cc:136-153 (F12 = 3x3 row-major float; sigma2 = pKF2->GetSigma2(kp2.octave)) */
static int check_dist_epipolar(const OrbOracleKeyPoint *kp1, const OrbOracleKeyPoint *kp2, const float *F12, const float *sigma2) {
    const float a = kp1->x * F12[0] + kp1->y * F12[3] + F12[6];
    const float b = kp1->x * F12[1] + kp1->y * F12[4] + F12[7];
    const float c = kp1->x * F12[2] + kp1->y * F12[5] + F12[8];
    const float num = a * kp2->x + b * kp2->y + c;
    const float den = a * a + b * b;
    if (den == 0) return 0;
    const float dsqr = num * num / den;
    return (double)dsqr < 3.84 * (double)sigma2[kp2->octave];
}

typedef struct { int dist, idx; } DistIdx;
static int cmp_distidx(const void *x, const void *y) {
    const DistIdx *a = (const DistIdx *)x, *b = (const DistIdx *)y;
    if (a->dist != b->dist) return a->dist < b->dist ? -1 : 1;
    return a->idx < b->idx ? -1 : a->idx > b->idx;
}

/* SearchForTriangulation, ORBmatcher.cc:852-1014.  has_mp1/2[i] != 0 <=> the keyframe feature already has a map point.
 * match12[i1] = i2 or -1; returns nmatches. */
int orb_oracle_search_for_triangulation(int n1, const OrbOracleKeyPoint *keys1, const uint8_t *desc1, const uint8_t *has_mp1,
                                        int nn1, const int *ids1, const int *ptr1, const int *items1,
                                        int n2, const OrbOracleKeyPoint *keys2, const uint8_t *desc2, const uint8_t *has_mp2,
                                        int nn2, const int *ids2, const int *ptr2, const int *items2,
                                        const float *F12, const float *sigma2_kf2, int check_orientation, int *match12) {
    int nmatches = 0;
    for (int i = 0; i < n1; i++) match12[i] = -1;
    uint8_t *matched2 = (uint8_t *)calloc((size_t)(n2 > 0 ? n2 : 1), 1);
    DistIdx *vd = (DistIdx *)malloc(sizeof(DistIdx) * (size_t)(n2 > 0 ? n2 : 1));
    IVec hist[HISTO_LENGTH];
    memset(hist, 0, sizeof(hist));
    int a = 0, b = 0;
    while (a < nn1 && b < nn2) {
        if (ids1[a] == ids2[b]) {
            for (int p1 = ptr1[a]; p1 < ptr1[a + 1]; p1++) {
                const int idx1 = items1[p1];
                if (has_mp1[idx1]) continue; /* :896-897 */
                const OrbOracleKeyPoint *kp1 = &keys1[idx1];
                const uint8_t *d1 = desc1 + (size_t)idx1 * 32;
                int nv = 0;
                for (int p2 = ptr2[b]; p2 < ptr2[b + 1]; p2++) {
                    const int idx2 = items2[p2];
                    if (matched2[idx2] || has_mp2[idx2]) continue;
                    const int dist = orb_oracle_hamming(d1, desc2 + (size_t)idx2 * 32);
                    if (dist > TH_LOW) continue;
                    vd[nv].dist = dist; vd[nv].idx = idx2; nv++;
                }
                if (nv == 0) continue;
                qsort(vd, (size_t)nv, sizeof(DistIdx), cmp_distidx); /* sort of pair<int,size_t> */
                const int DistTh = (int)round(2.0 * vd[0].dist);
                for (int id = 0; id < nv; id++) {
                    if (vd[id].dist > DistTh) break;
                    const int cur2 = vd[id].idx;
                    if (check_dist_epipolar(kp1, &keys2[cur2], F12, sigma2_kf2)) {
                        matched2[cur2] = 1;
                        match12[idx1] = cur2;
                        nmatches++;
                        if (check_orientation) ivec_push(&hist[rot_bin(kp1->angle, keys2[cur2].angle)], idx1);
                        break;
                    }
                }
            }
            a++; b++;
        } else if (ids1[a] < ids2[b]) {
            while (a < nn1 && ids1[a] < ids2[b]) a++;
        } else {
            while (b < nn2 && ids2[b] < ids1[a]) b++;
        }
    }
    if (check_orientation) {
        int counts[HISTO_LENGTH], i1, i2, i3;
        for (int k = 0; k < HISTO_LENGTH; k++) counts[k] = hist[k].n;
        orb_oracle_three_maxima(counts, HISTO_LENGTH, &i1, &i2, &i3);
        for (int k = 0; k < HISTO_LENGTH; k++) {
            if (k == i1 || k == i2 || k == i3) continue;
            for (int j = 0; j < hist[k].n; j++) { match12[hist[k].v[j]] = -1; nmatches--; }
        }
    }
    for (int k = 0; k < HISTO_LENGTH; k++) free(hist[k].v);
    free(matched2); free(vd);
    return nmatches;
}

/* Guided search without slot bookkeeping: every query independently takes its best candidate (strict-<, first minimum)
 * and keeps it iff best <= th_dist -- the inner loops of Fuse (:1090-1107, :1222-1239) and SearchBySim3 (:1356-1378,
 * :1436-1458), whose candidates are never skipped because of earlier matches. */
void orb_oracle_guided_best(const OrbOracleFrame *f, int nq, const float *qu, const float *qv, const float *qr,
                            const int *qlo, const int *qhi, const uint8_t *qdesc, int th_dist, int *best_idx) {
    int *cand = (int *)malloc(sizeof(int) * (size_t)(f->n > 0 ? f->n : 1));
    for (int q = 0; q < nq; q++) {
        best_idx[q] = -1;
        const int nc = orb_oracle_features_in_area(f, qu[q], qv[q], qr[q], qlo[q], qhi[q], cand, f->n);
        int bestDist = INT_MAX, bestIdx = -1;
        for (int c = 0; c < nc; c++) {
            const int dist = orb_oracle_hamming(qdesc + (size_t)q * 32, f->desc + (size_t)cand[c] * 32);
            if (dist < bestDist) { bestDist = dist; bestIdx = cand[c]; }
        }
        if (bestDist <= th_dist) best_idx[q] = bestIdx;
    }
    free(cand);
}

/* ------------------------------------------------------------------------------------------------
 * Frame::UndistortKeyPoints / ComputeImageBounds (reference src/Frame.cc:289-350): cv::undistortPoints(mat, mat, mK,
 * mDistCoef, cv::Mat(), mK) = OpenCV's cvUndistortPoints with R = I, P = K: 5 fixed-point iterations of the inverse
 * distortion model in double, then the re-projection with P.  Pinned bit-exactly against python-cv2
 * (tests/golden/opencv_undistort.npz).  dist = (k1, k2, p1, p2, k3); k4..k6 = 0 as in the reference's settings.
 * These are OpenCV 2.4's semantics: the five iterations always run.  OpenCV 4.x stops at the first iteration whose
 * denominator 1 + k1 r^2 + k2 r^4 + k3 r^6 is below 0 and returns the distorted point; the two agree on every point where no
 * iteration meets such a denominator and differ on most points where one does (strong barrel distortion near the image
 * corners: tests/golden/opencv_undistort_models.npz, test_oracle_camera_domain.py).
 * ------------------------------------------------------------------------------------------------ */
void orb_oracle_undistort_points(const float *pts, int n, float fx, float fy, float cx, float cy, const float *dist, float *out) {
    const double k0 = dist[0], k1 = dist[1], k2 = dist[2], k3 = dist[3], k4 = dist[4];
    const double fxd = fx, fyd = fy, cxd = cx, cyd = cy;
    const double ifx = 1. / fxd, ify = 1. / fyd;
    for (int i = 0; i < n; i++) {
        double x = pts[2 * i], y = pts[2 * i + 1];
        double x0 = x = (x - cxd) * ifx;
        double y0 = y = (y - cyd) * ify;
        for (int j = 0; j < 5; j++) {
            const double r2 = x * x + y * y;
            const double icdist = (1 + ((0.0 * r2 + 0.0) * r2 + 0.0) * r2) / (1 + ((k4 * r2 + k1) * r2 + k0) * r2);
            const double deltaX = 2 * k2 * x * y + k3 * (r2 + 2 * x * x);
            const double deltaY = k2 * (r2 + 2 * y * y) + 2 * k3 * x * y;
            x = (x0 - deltaX) * icdist;
            y = (y0 - deltaY) * icdist;
        }
        const double xx = fxd * x + 0.0 * y + cxd;
        const double yy = 0.0 * x + fyd * y + cyd;
        const double ww = 1. / (0.0 * x + 0.0 * y + 1.0);
        out[2 * i] = (float)(xx * ww);
        out[2 * i + 1] = (float)(yy * ww);
    }
}

/* UndistortKeyPoints on the 28-byte keypoints: mvKeysUn = mvKeys when k1 == 0 (:291-295) */
void orb_oracle_undistort_keypoints(const OrbOracleKeyPoint *in, int n, float fx, float fy, float cx, float cy, const float *dist,
                                    OrbOracleKeyPoint *out) {
    for (int i = 0; i < n; i++) out[i] = in[i];
    if (dist[0] == 0.0f) return;
    for (int i = 0; i < n; i++) {
        const float p[2] = {in[i].x, in[i].y};
        float q[2];
        orb_oracle_undistort_points(p, 1, fx, fy, cx, cy, dist, q);
        out[i].x = q[0];
        out[i].y = q[1];
    }
}

/* std::min / std::max as Frame.cc:336-339 calls them: (b < a) ? b : a and (a < b) ? b : a.  Unlike fminf / fmaxf they keep a
 * NaN first argument (a corner whose undistortion meets a zero denominator) and drop a NaN second one. */
static float std_min(float a, float b) { return (b < a) ? b : a; }
static float std_max(float a, float b) { return (a < b) ? b : a; }
/* Frame's bounds are `static int` (Frame.h:121-124): the float is converted as x86-64 does, NaN and values outside
 * [-2^31, 2^31) becoming INT_MIN */
static float frame_int(float f) { return (f >= -2147483648.0f && f < 2147483648.0f) ? (float)(int)f : -2147483648.0f; }

/* ComputeImageBounds, Frame.cc:321-350: bounds = (mnMinX, mnMinY, mnMaxX, mnMaxY) */
void orb_oracle_image_bounds(int cols, int rows, float fx, float fy, float cx, float cy, const float *dist, float *bounds) {
    if (dist[0] != 0.0f) {
        const float c[8] = {0.f, 0.f, (float)cols, 0.f, 0.f, (float)rows, (float)cols, (float)rows};
        float u[8];
        orb_oracle_undistort_points(c, 4, fx, fy, cx, cy, dist, u);
        bounds[0] = frame_int(std_min(floorf(u[0]), floorf(u[4])));
        bounds[2] = frame_int(std_max(ceilf(u[2]), ceilf(u[6])));
        bounds[1] = frame_int(std_min(floorf(u[1]), floorf(u[3])));
        bounds[3] = frame_int(std_max(ceilf(u[5]), ceilf(u[7])));
    } else {
        bounds[0] = 0; bounds[2] = (float)cols; bounds[1] = 0; bounds[3] = (float)rows;
    }
}
