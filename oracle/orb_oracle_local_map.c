/* oracle/orb_oracle_local_map.c -- Tracking::UpdateReference (UpdateReferenceKeyFrames and UpdateReferencePoints) restated
 * on the keyframes' map-point rows and the covisibility graph's ordered lists: the oracle of orbfe_covis_local_map_device
 * (TEST INFRASTRUCTURE ONLY).
 *
 * A point's observers are the live slots whose rows name it, once per slot (orb_oracle_observations.c).  The frame's cells
 * are walked as Tracking.cc:768-784 walks them: a bad point's cell becomes -1, every other cell adds 1 to each observer of
 * its point.  The counted slots are listed in key order with the first strict maximum as the reference keyframe
 * (:793-808); the extension visits only those entries, stops before a visit once more than 80 are listed and appends the
 * first live, unlisted one of each visited entry's first 10 ordered neighbours (:812-836); the points are the rows of the
 * list in order, each point at its first occurrence, bad points skipped (:740-760).  Statuses are those of the device
 * entry: 0, -1 (ORBFE_ERR_ARG: nothing written). */
#include <stdint.h>
#include <stdlib.h>

#define NEIGH 10
#define MAX_KF 80

static const uint64_t *g_keys;
static int by_key(const void *a, const void *b) {
    const uint64_t x = g_keys[*(const int *)a], y = g_keys[*(const int *)b];
    return x < y ? -1 : x > y;
}

/* frame_mp[nf] in/out; rows kf_mp[nframes*cap], counts / live / keys [nframes]; nb[nframes*NEIGH] the first NEIGH entries of
 * each slot's ordered list (slots as the graph holds them, retired ones included), nnb[nframes] how many there are;
 * local_kf[nframes], local_points[npoints] */
int lm_oracle(int nf, int *frame_mp, const uint8_t *point_bad, int npoints, const int *kf_mp, const int *counts, int nframes, int cap,
              const uint8_t *live, const uint64_t *keys, const int *nb, const int *nnb, int *local_kf, int *nlocal_kf, int *ref_kf,
              int *local_points, int *nlocal_points) {
    int bad = 0, rc = 0;
    const size_t np = (size_t)(npoints > 0 ? npoints : 1);
    int *ptr = calloc(np + 1, sizeof(int)), *last = malloc(sizeof(int) * np), *obs = NULL;
    int *cnt = calloc((size_t)nframes, sizeof(int)), *order = malloc(sizeof(int) * (size_t)nframes);
    uint8_t *listed = calloc((size_t)nframes, 1), *seen = calloc(np, 1);
    for (int i = 0; i < nf; i++)
        if (frame_mp[i] >= npoints) bad = 1;
    for (int p = 0; p < npoints; p++) last[p] = -1;
    for (int s = 0; s < nframes; s++) {   /* observers per point: one per live slot */
        if (!live[s]) continue;
        if (counts[s] < 0 || counts[s] > cap) { bad = 1; continue; }
        for (int i = 0; i < counts[s]; i++) {
            const int v = kf_mp[(size_t)s * cap + i];
            if (v < 0) continue;
            if (v >= npoints) { bad = 1; continue; }
            if (last[v] != s) { last[v] = s; ptr[v + 1]++; }
        }
    }
    if (bad) { rc = -1; goto out; }
    for (int p = 0; p < npoints; p++) { ptr[p + 1] += ptr[p]; last[p] = -1; }
    obs = malloc(sizeof(int) * (size_t)(ptr[npoints > 0 ? npoints : 0] + 1));
    {
        int *fill = malloc(sizeof(int) * np);
        for (int p = 0; p < npoints; p++) fill[p] = ptr[p];
        for (int s = 0; s < nframes; s++) {
            if (!live[s]) continue;
            for (int i = 0; i < counts[s]; i++) {
                const int v = kf_mp[(size_t)s * cap + i];
                if (v >= 0 && last[v] != s) { last[v] = s; obs[fill[v]++] = s; }
            }
        }
        free(fill);
    }
    /* the counter */
    for (int i = 0; i < nf; i++) {
        const int p = frame_mp[i];
        if (p < 0) continue;
        if (point_bad[p]) { frame_mp[i] = -1; continue; }
        for (int e = ptr[p]; e < ptr[p + 1]; e++) cnt[obs[e]]++;
    }
    /* the counted keyframes in key order, the first strict maximum */
    int n0 = 0, mx = 0, ref = -1;
    for (int s = 0; s < nframes; s++)
        if (cnt[s] > 0) order[n0++] = s;
    g_keys = keys;
    qsort(order, (size_t)n0, sizeof(int), by_key);
    for (int t = 0; t < n0; t++) {
        const int s = order[t];
        if (cnt[s] > mx) { mx = cnt[s]; ref = s; }
        local_kf[t] = s;
        listed[s] = 1;
    }
    /* the extension: the end is fixed at n0 */
    int n = n0;
    for (int t = 0; t < n0; t++) {
        if (n > MAX_KF) break;
        const int v = local_kf[t], m = nnb[v] < NEIGH ? nnb[v] : NEIGH;
        for (int q = 0; q < m; q++) {
            const int u = nb[(size_t)v * NEIGH + q];
            if (u < 0 || u >= nframes || !live[u]) continue;   /* isBad(): a stale entry */
            if (!listed[u]) {
                local_kf[n++] = u;
                listed[u] = 1;
                break;
            }
        }
    }
    *nlocal_kf = n;
    *ref_kf = ref;
    /* the points */
    int k = 0;
    for (int t = 0; t < n; t++) {
        const int s = local_kf[t];
        for (int i = 0; i < counts[s]; i++) {
            const int p = kf_mp[(size_t)s * cap + i];
            if (p < 0 || seen[p] || point_bad[p]) continue;
            seen[p] = 1;
            local_points[k++] = p;
        }
    }
    *nlocal_points = k;
out:
    free(ptr);
    free(last);
    free(obs);
    free(cnt);
    free(order);
    free(listed);
    free(seen);
    return rc;
}
