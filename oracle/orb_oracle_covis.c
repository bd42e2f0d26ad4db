/* orb_oracle_covis.c -- the covisibility graph (reference src/KeyFrame.cc:126-185 AddConnection / UpdateBestCovisibles,
 * :332-421 UpdateConnections, :497-521 SetBadFlag's connection half, :596-610 EraseConnection) restated as a slot-indexed
 * state machine, one reference call at a time (TEST INFRASTRUCTURE ONLY).
 *
 * A keyframe is a slot; its 64-bit key stands for the KeyFrame* that orders every std::map and breaks every tie.  Weight
 * maps are dense rows (weight 0 = absent; a count is never 0).  Inputs are those of orbfe_covis_update_connections_device:
 * kf_mp[s*cap + i] (negative = no point), counts[s], and the observations obs[gp[g] .. gp[g+1]) of point g as flat slots
 * f*cap + i. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    int K;
    uint64_t *key;
    uint8_t *live, *id0, *first;
    int *w;               /* K x K: w[s*K + t] = mConnectedKeyFrameWeights[t] of s, 0 = absent */
    int *on, *oslot, *ow; /* K, K x K, K x K: the ordered list and its weights */
    int *parent;          /* mpParent, -1 = NULL */
    int *cnt;             /* counter scratch */
} CovisOracle;

typedef struct {
    int w;
    uint64_t k;
    int s;
} Pair;

/* sort() of (weight, KeyFrame*) pairs ascending */
static int pair_cmp(const void *a, const void *b) {
    const Pair *x = (const Pair *)a, *y = (const Pair *)b;
    if (x->w != y->w) return x->w < y->w ? -1 : 1;
    if (x->k != y->k) return x->k < y->k ? -1 : 1;
    return 0;
}

static const uint64_t *g_keys;
static int slot_key_cmp(const void *a, const void *b) {
    const uint64_t x = g_keys[*(const int *)a], y = g_keys[*(const int *)b];
    return x < y ? -1 : x > y;
}

void *covis_oracle_create(int K) {
    CovisOracle *o = (CovisOracle *)calloc(1, sizeof(CovisOracle));
    o->K = K;
    o->key = (uint64_t *)calloc(K, sizeof(uint64_t));
    o->live = (uint8_t *)calloc(K, 1);
    o->id0 = (uint8_t *)calloc(K, 1);
    o->first = (uint8_t *)calloc(K, 1);
    o->w = (int *)calloc((size_t)K * K, sizeof(int));
    o->on = (int *)calloc(K, sizeof(int));
    o->oslot = (int *)calloc((size_t)K * K, sizeof(int));
    o->ow = (int *)calloc((size_t)K * K, sizeof(int));
    o->parent = (int *)malloc(K * sizeof(int));
    o->cnt = (int *)calloc(K, sizeof(int));
    for (int i = 0; i < K; i++) o->parent[i] = -1;
    return o;
}

void covis_oracle_free(void *h) {
    CovisOracle *o = (CovisOracle *)h;
    if (!o) return;
    free(o->key); free(o->live); free(o->id0); free(o->first); free(o->w); free(o->on); free(o->oslot); free(o->ow);
    free(o->parent); free(o->cnt);
    free(o);
}

/* a fresh KeyFrame in `slot` */
void covis_oracle_add(void *h, int slot, int id, uint64_t key) {
    CovisOracle *o = (CovisOracle *)h;
    o->key[slot] = key;
    o->live[slot] = 1;
    o->id0[slot] = id == 0;
    o->first[slot] = 1;
    o->on[slot] = 0;
    o->parent[slot] = -1;
    memset(o->w + (size_t)slot * o->K, 0, sizeof(int) * o->K);
}

/* UpdateBestCovisibles (:141-160): every weight, sorted, pushed to the front */
static void update_best(CovisOracle *o, int s) {
    const int K = o->K;
    Pair *v = (Pair *)malloc(sizeof(Pair) * (K > 0 ? K : 1));
    int n = 0;
    for (int t = 0; t < K; t++)
        if (o->w[(size_t)s * K + t]) { v[n].w = o->w[(size_t)s * K + t]; v[n].k = o->key[t]; v[n].s = t; n++; }
    qsort(v, n, sizeof(Pair), pair_cmp);
    for (int i = 0; i < n; i++) { o->oslot[(size_t)s * K + i] = v[n - 1 - i].s; o->ow[(size_t)s * K + i] = v[n - 1 - i].w; }
    o->on[s] = n;
    free(v);
}

/* AddConnection (:126-139): nothing happens when the weight is already there */
static void add_connection(CovisOracle *o, int s, int t, int weight) {
    int *e = &o->w[(size_t)s * o->K + t];
    if (*e == weight) return;
    *e = weight;
    update_best(o, s);
}

/* UpdateConnections (:332-421) of `slot`.  Returns the parent set by this call, else -1. */
int covis_oracle_update(void *h, int slot, const int *kf_mp, const int *counts, int cap, const int *gp, const int *obs) {
    CovisOracle *o = (CovisOracle *)h;
    const int K = o->K;
    int *touched = (int *)malloc(sizeof(int) * K), nt = 0;
    for (int i = 0; i < counts[slot]; i++) {
        const int mp = kf_mp[(size_t)slot * cap + i];
        if (mp < 0) continue;
        for (int j = gp[mp]; j < gp[mp + 1]; j++) {
            const int f = obs[j] / cap;
            if (f == slot) continue;
            if (o->cnt[f]++ == 0) touched[nt++] = f;
        }
    }
    if (nt == 0) { free(touched); return -1; }   /* KFcounter.empty(): return */
    g_keys = o->key;
    qsort(touched, nt, sizeof(int), slot_key_cmp);   /* std::map<KeyFrame*, int> order */
    int nmax = 0, pmax = -1, np = 0;
    Pair *v = (Pair *)malloc(sizeof(Pair) * nt);
    for (int i = 0; i < nt; i++) {
        const int t = touched[i], c = o->cnt[t];
        if (c > nmax) { nmax = c; pmax = t; }
        if (c >= 15) {
            v[np].w = c; v[np].k = o->key[t]; v[np].s = t; np++;
            add_connection(o, t, slot, c);
        }
    }
    if (np == 0) {
        v[0].w = nmax; v[0].k = o->key[pmax]; v[0].s = pmax; np = 1;
        add_connection(o, pmax, slot, nmax);
    }
    qsort(v, np, sizeof(Pair), pair_cmp);
    memset(o->w + (size_t)slot * K, 0, sizeof(int) * K);
    for (int i = 0; i < nt; i++) { o->w[(size_t)slot * K + touched[i]] = o->cnt[touched[i]]; o->cnt[touched[i]] = 0; }
    for (int i = 0; i < np; i++) { o->oslot[(size_t)slot * K + i] = v[np - 1 - i].s; o->ow[(size_t)slot * K + i] = v[np - 1 - i].w; }
    o->on[slot] = np;
    int parent = -1;
    if (o->first[slot] && !o->id0[slot]) {
        parent = o->parent[slot] = o->oslot[(size_t)slot * K];
        o->first[slot] = 0;
    }
    free(v);
    free(touched);
    return parent;
}

/* SetBadFlag's connection half (:497-521) with EraseConnection (:596-610) */
void covis_oracle_erase(void *h, int slot) {
    CovisOracle *o = (CovisOracle *)h;
    const int K = o->K;
    if (!o->live[slot] || o->id0[slot]) return;
    int *order = (int *)malloc(sizeof(int) * K), n = 0;
    for (int t = 0; t < K; t++)
        if (o->w[(size_t)slot * K + t]) order[n++] = t;
    g_keys = o->key;
    qsort(order, n, sizeof(int), slot_key_cmp);
    for (int i = 0; i < n; i++) {
        const int t = order[i];
        if (o->w[(size_t)t * K + slot]) {
            o->w[(size_t)t * K + slot] = 0;
            update_best(o, t);
        }
    }
    memset(o->w + (size_t)slot * K, 0, sizeof(int) * K);
    o->on[slot] = 0;
    o->live[slot] = 0;
    free(order);
}

void covis_oracle_clear(void *h) {
    CovisOracle *o = (CovisOracle *)h;
    const int K = o->K;
    memset(o->live, 0, K);
    memset(o->w, 0, sizeof(int) * (size_t)K * K);
    memset(o->on, 0, sizeof(int) * K);
    for (int i = 0; i < K; i++) o->parent[i] = -1;
}

/* the ordered list and its weights; returns its length */
int covis_oracle_ordered(void *h, int slot, int *slots, int *weights) {
    CovisOracle *o = (CovisOracle *)h;
    const int n = o->on[slot];
    memcpy(slots, o->oslot + (size_t)slot * o->K, sizeof(int) * n);
    memcpy(weights, o->ow + (size_t)slot * o->K, sizeof(int) * n);
    return n;
}

/* the weight map in key order; returns its size */
int covis_oracle_weights(void *h, int slot, int *slots, int *weights) {
    CovisOracle *o = (CovisOracle *)h;
    const int K = o->K;
    int n = 0;
    for (int t = 0; t < K; t++)
        if (o->w[(size_t)slot * K + t]) slots[n++] = t;
    g_keys = o->key;
    qsort(slots, n, sizeof(int), slot_key_cmp);
    for (int i = 0; i < n; i++) weights[i] = o->w[(size_t)slot * K + slots[i]];
    return n;
}

int covis_oracle_parent(void *h, int slot) { return ((CovisOracle *)h)->parent[slot]; }
int covis_oracle_live(void *h, int slot) { return ((CovisOracle *)h)->live[slot]; }
