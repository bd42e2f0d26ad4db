/* oracle/orb_oracle_observations.c -- MapPoint::GetObservations() of named points restated as the inverse of the live
 * keyframes' map-point rows: the oracle of orbfe_covis_observations_device (TEST INFRASTRUCTURE ONLY).
 *
 * Walks the live slots in key order and each row in ascending feature order, as the reference's std::map<KeyFrame*, size_t>
 * and ProcessNewKeyFrame's mObservations[pKF] = i do: a point's list gains one entry per slot, and a later feature of the
 * same row overwrites that entry's index.  Statuses are those of the device entry: 0, -1 (ORBFE_ERR_ARG: only ptr written),
 * -3 (ORBFE_ERR_CAPACITY: ptr and *nobs written). */
#include <stdint.h>
#include <stdlib.h>

static const uint64_t *g_keys;
static int by_key(const void *a, const void *b) {
    const uint64_t x = g_keys[*(const int *)a], y = g_keys[*(const int *)b];
    return x < y ? -1 : x > y;
}

int obs_oracle(int n, const int *points, int npoints, const int *kf_mp, const int *counts, int nframes, int cap, const uint8_t *live,
               const uint64_t *keys, const int *ref_slot, int obs_cap, int *ptr, int *obs, int *nobs, int *ref_obs) {
    int bad = 0, rc = 0;
    int *pos = malloc(sizeof(int) * (size_t)(npoints > 0 ? npoints : 1));
    int *cnt = calloc((size_t)(n > 0 ? n : 1), sizeof(int));
    int *last = malloc(sizeof(int) * (size_t)(n > 0 ? n : 1));   /* the slot of a list's newest entry */
    int *order = malloc(sizeof(int) * (size_t)nframes);
    int nlive = 0;
    for (int p = 0; p < npoints; p++) pos[p] = -1;
    for (int j = 0; j < n; j++) {
        const int p = points[j];
        if (p < 0 || p >= npoints || pos[p] >= 0) bad = 1;
        else pos[p] = j;
        last[j] = -1;
    }
    for (int s = 0; s < nframes; s++)
        if (live[s]) order[nlive++] = s;
    g_keys = keys;
    qsort(order, (size_t)nlive, sizeof(int), by_key);
    for (int q = 0; q < nlive; q++) {
        const int s = order[q], c = counts[s];
        if (c < 0 || c > cap) { bad = 1; continue; }
        for (int i = 0; i < c; i++) {
            const int v = kf_mp[(size_t)s * cap + i];
            if (v < 0) continue;
            if (v >= npoints) { bad = 1; continue; }
            const int j = pos[v];
            if (j < 0 || last[j] == s) continue;
            last[j] = s;
            cnt[j]++;
        }
    }
    for (int j = 0; ref_slot && j < n; j++)
        if (ref_slot[j] < 0 || ref_slot[j] >= nframes) bad = 1;
    ptr[0] = 0;
    for (int j = 0; j < n; j++) ptr[j + 1] = ptr[j] + cnt[j];
    if (bad) { rc = -1; goto out; }
    *nobs = ptr[n];
    if (ptr[n] > obs_cap) { rc = -3; goto out; }
    for (int j = 0; j < n; j++) { cnt[j] = ptr[j]; last[j] = -1; }
    for (int q = 0; q < nlive; q++) {
        const int s = order[q], c = counts[s];
        for (int i = 0; i < c; i++) {
            const int v = kf_mp[(size_t)s * cap + i];
            const int j = v >= 0 ? pos[v] : -1;
            if (j < 0) continue;
            if (last[j] == s) { obs[cnt[j] - 1] = s * cap + i; continue; }   /* mObservations[pKF] = i again: the later i stays */
            last[j] = s;
            obs[cnt[j]++] = s * cap + i;
        }
    }
    for (int j = 0; ref_obs && j < n; j++) {   /* observations[pRefKF]: operator[] inserts 0 when absent */
        const int ref = ref_slot[j];
        ref_obs[j] = ref * cap;
        for (int e = ptr[j]; e < ptr[j + 1]; e++)
            if (obs[e] / cap == ref) ref_obs[j] = obs[e];
    }
out:
    free(pos);
    free(cnt);
    free(last);
    free(order);
    return rc;
}
