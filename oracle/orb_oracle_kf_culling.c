/* oracle/orb_oracle_kf_culling.c -- LocalMapping::KeyFrameCulling with KeyFrame::SetBadFlag's map-point half, restated on
 * the keyframes' map-point rows: the oracle of orbfe_covis_keyframe_culling_device (TEST INFRASTRUCTURE ONLY).
 *
 * The observations are built as orb_oracle_observations.c builds them (live slots in key order, rows in ascending feature
 * order, the last feature of a row wins).  Then the list is walked as the reference walks it: per entry the counts of
 * LocalMapping.cc:533-571 in ascending feature order, the comparison `nRedundant > 0.9 * nMPs` in double, and on an erase
 * MapPoint::EraseObservation for each non-negative cell in ascending order (the observation leaves, mpRefKF moves to the
 * smallest remaining key, a point left with at most two observations goes bad and every cell of its remaining observers'
 * rows that names it becomes -1).  Statuses are those of the device entry: 0, -1 (ORBFE_ERR_ARG: nothing written),
 * -3 (ORBFE_ERR_CAPACITY: only *nobs written). */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MAX_LEVELS 32   /* ORBFE_MAX_LEVELS */

static const uint64_t *g_keys;
static int by_key(const void *a, const void *b) {
    const uint64_t x = g_keys[*(const int *)a], y = g_keys[*(const int *)b];
    return x < y ? -1 : x > y;
}

static int octave_ok(int o) { return o >= 0 && o < MAX_LEVELS; }

/* list[ncand]: the current keyframe's ordered list (slots); live / id0 / keys / not_erase per slot [nframes];
 * octave[nframes*cap]; kf_mp, point_bad, ref_slot in/out */
int kfc_oracle(int ncand, const int *list, const uint8_t *live, const uint8_t *id0, const uint64_t *keys, const uint8_t *not_erase,
               int *kf_mp, const int *counts, const int *octave, int nframes, int cap, uint8_t *point_bad, int *ref_slot, int npoints,
               int obs_cap, int *nobs, int *verdict_slot, int *verdict, int *nmps, int *nred, int *bad_points, int *nbad) {
    int bad = 0, rc = 0;
    const size_t np = (size_t)(npoints > 0 ? npoints : 1);
    int *cnt = calloc(np, sizeof(int)), *last = malloc(sizeof(int) * np), *ptr = malloc(sizeof(int) * (np + 1));
    int *order = malloc(sizeof(int) * (size_t)nframes);
    int *obs = NULL;
    uint8_t *alive = NULL, *made_bad = calloc(np, 1);
    int nlive = 0;
    for (int s = 0; s < nframes; s++)
        if (live[s]) order[nlive++] = s;
    g_keys = keys;
    qsort(order, (size_t)nlive, sizeof(int), by_key);
    for (int p = 0; p < npoints; p++) last[p] = -1;
    for (int q = 0; q < nlive; q++) {
        const int s = order[q], c = counts[s];
        if (c < 0 || c > cap) { bad = 1; continue; }
        for (int i = 0; i < c; i++) {
            const int v = kf_mp[(size_t)s * cap + i];
            if (v < 0) continue;
            if (v >= npoints) { bad = 1; continue; }
            if (last[v] != s) { last[v] = s; cnt[v]++; }
        }
    }
    if (bad) { rc = -1; goto out; }
    ptr[0] = 0;
    for (int p = 0; p < npoints; p++) ptr[p + 1] = ptr[p] + cnt[p];
    *nobs = ptr[npoints > 0 ? npoints : 0];
    if (*nobs > obs_cap) { rc = -3; goto out; }
    obs = malloc(sizeof(int) * (size_t)(*nobs > 0 ? *nobs : 1));
    alive = malloc((size_t)(*nobs > 0 ? *nobs : 1));
    for (int p = 0; p < npoints; p++) { cnt[p] = ptr[p]; last[p] = -1; }
    for (int q = 0; q < nlive; q++) {
        const int s = order[q], c = counts[s];
        for (int i = 0; i < c; i++) {
            const int v = kf_mp[(size_t)s * cap + i];
            if (v < 0) continue;
            if (last[v] == s) { obs[cnt[v] - 1] = s * cap + i; continue; }
            last[v] = s;
            obs[cnt[v]++] = s * cap + i;
        }
    }
    for (int e = 0; e < *nobs; e++) alive[e] = 1;
    /* the listed keyframes' checks */
    for (int t = 0; t < ncand && !bad; t++) {
        const int v = list[t];
        const int c = v < nframes ? counts[v] : -1;
        if (c < 0 || c > cap) { bad = 1; break; }
        for (int i = 0; i < c; i++) {
            const int p = kf_mp[(size_t)v * cap + i];
            if (p < 0) continue;
            if (p >= npoints) { bad = 1; break; }
            if (point_bad[p]) continue;
            if (!octave_ok(octave[(size_t)v * cap + i]) || ref_slot[p] < 0 || ref_slot[p] >= nframes) { bad = 1; break; }
            for (int e = ptr[p]; e < ptr[p + 1]; e++)
                if (!octave_ok(octave[obs[e]])) bad = 1;
        }
    }
    if (bad) { rc = -1; goto out; }
    for (int t = 0; t < ncand; t++) {
        const int v = list[t], c = counts[v];
        int *row = kf_mp + (size_t)v * cap;
        verdict_slot[t] = v;
        if (id0[v]) {   /* if(pKF->mnId==0) continue; */
            verdict[t] = 1;
            nmps[t] = nred[t] = 0;
            continue;
        }
        int nm = 0, nr = 0;
        for (int i = 0; i < c; i++) {
            const int p = row[i];
            if (p < 0 || point_bad[p]) continue;
            nm++;
            int n_alive = 0;
            for (int e = ptr[p]; e < ptr[p + 1]; e++) n_alive += alive[e];
            if (n_alive > 3) {   /* pMP->Observations() > 3 */
                const int level = octave[(size_t)v * cap + i];
                int n = 0;
                for (int e = ptr[p]; e < ptr[p + 1]; e++) {
                    if (!alive[e] || obs[e] / cap == v) continue;
                    if (octave[obs[e]] <= level + 1) {
                        n++;
                        if (n >= 3) break;
                    }
                }
                if (n >= 3) nr++;
            }
        }
        nmps[t] = nm;
        nred[t] = nr;
        if (!(nr > 0.9 * nm)) { verdict[t] = 0; continue; }
        if (not_erase[v]) { verdict[t] = 3; continue; }
        if (!live[v]) { verdict[t] = 4; continue; }   /* already retired: its observations are gone */
        verdict[t] = 2;
        for (int i = 0; i < c; i++) {   /* mvpMapPoints[i]->EraseObservation(this) */
            const int p = row[i];
            if (p < 0) continue;
            int at = -1, left = 0;
            for (int e = ptr[p]; e < ptr[p + 1]; e++) {
                if (!alive[e]) continue;
                if (obs[e] / cap == v) at = e;
                else left++;
            }
            if (at < 0) continue;   /* not an observer (any more) */
            alive[at] = 0;
            if (ref_slot[p] == v)
                for (int e = ptr[p]; e < ptr[p + 1]; e++)
                    if (alive[e]) { ref_slot[p] = obs[e] / cap; break; }
            if (left <= 2) {   /* MapPoint::SetBadFlag: the remaining observers' cells, duplicates included */
                point_bad[p] = 1;
                made_bad[p] = 1;
                for (int e = ptr[p]; e < ptr[p + 1]; e++) {
                    if (!alive[e]) continue;
                    alive[e] = 0;
                    int *r = kf_mp + (size_t)(obs[e] / cap) * cap;
                    for (int k = 0; k < counts[obs[e] / cap]; k++)
                        if (r[k] == p) r[k] = -1;
                }
            }
        }
    }
    *nbad = 0;
    for (int p = 0; p < npoints; p++)
        if (made_bad[p]) bad_points[(*nbad)++] = p;
out:
    free(cnt);
    free(last);
    free(ptr);
    free(order);
    free(obs);
    free(alive);
    free(made_bad);
    return rc;
}
