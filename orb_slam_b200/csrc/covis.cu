// covis.cu -- the covisibility graph of one map (reference src/KeyFrame.cc:126-185, 332-421, 497-521, 596-610) resident in
// device memory: KeyFrame::UpdateConnections for batches of keyframes, the connection half of SetBadFlag, and the lists
// the loop and relocalisation queries read.  C-ABI in include/orbfe_bow.h (orbfe_covis_*).
//
// Layout (all allocated by orbfe_covis_create), per slot s:
//   key[s]                 the caller's order key: it stands for the KeyFrame* every std::map of the reference is ordered by
//   state[s]               live, mnId == 0, mbFirstConnection
//   wn / wslot / ww        mConnectedKeyFrameWeights as rows of max_connections (slot, weight), key ascending
//   on / oslot / ow        mvpOrderedConnectedKeyFrames / mvOrderedWeights, (weight, key) descending
//   named[s]               how many weight maps hold s as a key (a retired slot may be re-added only when this is 0)
// Batch scratch: the counter and filtered list of every entry (rows of max_connections), and per slot the batch position,
// a touched mark and the AddConnection events bucketed by target.  pos / tmark / evcnt / efill are -1 / 0 between batches:
// the apply kernel restores them for every slot the batch touched.
//
// A batch of n UpdateConnections calls is three launches, no host round trip:
//   covis_count_kernel  one block per entry: KFcounter in a shared-memory open-addressed table keyed by slot (the entry's
//                       own slot skipped), sorted by key; the first strict maximum in key order; the filtered ordered list
//                       (weights >= 15, else the maximum alone) sorted by (weight, key) descending.  Its entries are the
//                       entry's AddConnection(target, entry, weight) events.  Bad input or an overflowing counter flags the
//                       batch.
//   covis_plan_kernel   one block: marks the touched slots (entries and event targets), buckets the events by target and
//                       computes every touched weight map's final size; a flag or an oversized map rejects the batch.
//   covis_apply_kernel  one block per touched slot writes its final state in closed form (DESIGN.md §4.6): the start map is
//                       the slot's own counter (when it had a non-empty call) or its old map, the events of later entries
//                       (all events without an own call) are applied to it; the ordered list is the full sort when one of
//                       those events changed a weight, else the own call's filtered list, else unchanged.  One call's
//                       counter reads only the observations, which a batch does not change, and an entry sends at most one
//                       event to each target, so the result does not depend on scheduling.
//
// MapPoint::GetObservations() for named points (orbfe_covis_observations_device) is five launches, no host round trip: stamp
// the named points, count per (live slot, point) with the row's last feature index, scan, scatter, rank each list by key.
//
// LocalMapping::KeyFrameCulling (orbfe_covis_keyframe_culling_device) is those five launches over every point, then the
// candidates' checks, one block that walks the current keyframe's list in order, and the NULLing of made-bad points' cells.
//
// Tracking::UpdateReference (orbfe_covis_local_map_device) is six launches: the frame's point multiplicities, the keyframe
// counter from the live rows, one block that builds the local keyframe list, and three that collect the list's points.
#include <algorithm>
#include <climits>
#include <unordered_set>
#include <vector>

#include "../../include/orbfe_bow.h"
#include "orbfe_internal.h"

namespace orbfe {

#define COVIS_TH 15              // KeyFrame.cc:372
#define COVIS_MAX_CONN 2048      // the count and apply blocks hold a weight map in shared memory
#define COVIS_MAX_BATCH 1024
#define COVIS_COUNT_BLOCK 512
#define COVIS_APPLY_BLOCK 256
enum { ST_LIVE = 1, ST_ID0 = 2, ST_FIRST = 4 };
// flags: [0] bad input in this batch, [1] overflow in this batch, [2] batch accepted, [3] first error since the last sync,
//        [4] touched slots of this batch
enum { F_BAD = 0, F_OVER = 1, F_OK = 2, F_ERR = 3, F_NT = 4, F_COUNT = 8 };

struct CvEnt {
    unsigned long long k;
    int s, w;
};

static __host__ __device__ int pow2ge(int n) {
    int p = 1;
    while (p < n) p <<= 1;
    return p;
}

// bitonic sort of n2 (a power of two) entries by the whole block: ByWeight = (weight, key) descending, else key ascending
template <bool ByWeight>
__device__ __forceinline__ bool cv_before(const CvEnt &a, const CvEnt &b) {
    if (ByWeight) return a.w > b.w || (a.w == b.w && a.k > b.k);
    return a.k < b.k;
}
template <bool ByWeight>
__device__ void cv_sort(CvEnt *e, int n2) {
    for (int k = 2; k <= n2; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n2; i += blockDim.x) {
                const int l = i ^ j;
                if (l > i) {
                    const CvEnt a = e[i], b = e[l];
                    if ((i & k) == 0 ? cv_before<ByWeight>(b, a) : cv_before<ByWeight>(a, b)) { e[i] = b; e[l] = a; }
                }
            }
            __syncthreads();
        }
}
// padding that sorts last in either order
__device__ __forceinline__ CvEnt cv_pad(bool by_weight) { return by_weight ? CvEnt{0ull, -1, INT_MIN} : CvEnt{~0ull, -1, 0}; }

// index of `k` in the key-ascending slot row, or -1
__device__ __forceinline__ int cv_find(const int *row, int n, const unsigned long long *key, unsigned long long k) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (key[row[mid]] < k) lo = mid + 1; else hi = mid;
    }
    return lo < n && key[row[lo]] == k ? lo : -1;
}

// exclusive scan of one value per thread over a block of 1024; returns the prefix and adds the block total to *carry
__device__ int cv_block_scan(int v, int *s_warp, int *carry) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[wid] = x;
    __syncthreads();
    if (wid == 0) {
        int w = s_warp[lane];
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        s_warp[lane] = w;
    }
    __syncthreads();
    const int base = *carry;
    const int r = base + (wid > 0 ? s_warp[wid - 1] : 0) + x - v;
    __syncthreads();
    if (threadIdx.x == 0) *carry = base + s_warp[31];
    __syncthreads();
    return r;
}

// ---- UpdateConnections, launch 1: one block per batch entry
__global__ void __launch_bounds__(COVIS_COUNT_BLOCK) covis_count_kernel(
    const int *__restrict__ slots, int C, int Cp, int P, const int *__restrict__ kf_mp, const int *__restrict__ counts, int nframes,
    int cap, const int *__restrict__ gp, const int *__restrict__ obs, int npoints, int nobs, int K, const int *__restrict__ state,
    const unsigned long long *__restrict__ key, int *__restrict__ cn, int *__restrict__ cslot, int *__restrict__ cw, int *__restrict__ fn,
    int *__restrict__ fslot, int *__restrict__ fw, int *__restrict__ flags) {
    extern __shared__ unsigned long long cv_smem[];
    CvEnt *buf = reinterpret_cast<CvEnt *>(cv_smem);   // Cp entries: the counter, key ascending
    int *tkey = reinterpret_cast<int *>(buf + Cp);       // P slots, then P counts; reused as Cp entries of the filtered list
    int *tcnt = tkey + P;
    CvEnt *flt = reinterpret_cast<CvEnt *>(tkey);
    __shared__ int s_bad, s_full, s_n, s_c, s_nmax, s_imax, s_nth, s_f;
    const int p = blockIdx.x, s = slots[p];
    for (int i = threadIdx.x; i < P; i += blockDim.x) { tkey[i] = -1; tcnt[i] = 0; }
    if (threadIdx.x == 0) { s_bad = 0; s_full = 0; s_n = 0; s_c = 0; s_nmax = 0; s_imax = INT_MAX; s_nth = 0; s_f = 0; }
    __syncthreads();
    const int nf = counts[s];
    if (nf < 0 || nf > cap) {
        if (threadIdx.x == 0) s_bad = 1;
    } else {
        for (int i = threadIdx.x; i < nf; i += blockDim.x) {
            const int mp = kf_mp[(size_t)s * cap + i];
            if (mp < 0) continue;   // NULL or isBad()
            if (mp >= npoints) { s_bad = 1; break; }
            const int lo = gp[mp], hi = gp[mp + 1];
            if (lo < 0 || lo > hi || hi > nobs) { s_bad = 1; break; }
            for (int o = lo; o < hi; o++) {
                const int ob = obs[o];
                const int f = ob < 0 ? -1 : ob / cap;
                if (f < 0 || f >= nframes || f >= K || !(state[f] & ST_LIVE)) { s_bad = 1; break; }
                if (f == s) continue;   // mit->first->mnId == mnId
                unsigned h = ((unsigned)f * 2654435761u) & (unsigned)(P - 1);
                for (int probe = 0;; probe++) {
                    if (probe == P) { s_full = 1; break; }
                    const int old = atomicCAS(&tkey[h], -1, f);
                    if (old == -1) atomicAdd(&s_n, 1);
                    if (old == -1 || old == f) { atomicAdd(&tcnt[h], 1); break; }
                    h = (h + 1) & (unsigned)(P - 1);
                }
            }
        }
    }
    __syncthreads();
    const int n = s_n;
    if (s_bad || s_full || n > C || n == 0) {
        if (threadIdx.x == 0) {
            if (s_bad) atomicOr(&flags[F_BAD], 1);
            else if (n != 0) atomicOr(&flags[F_OVER], 1);
            cn[p] = 0;   // an empty counter: the call returns at once (KeyFrame.cc:365)
            fn[p] = 0;
        }
        return;
    }
    for (int h = threadIdx.x; h < P; h += blockDim.x) {
        const int f = tkey[h];
        if (f >= 0) buf[atomicAdd(&s_c, 1)] = CvEnt{key[f], f, tcnt[h]};
    }
    const int n2 = pow2ge(n);
    for (int j = n + threadIdx.x; j < n2; j += blockDim.x) buf[j] = cv_pad(false);
    __syncthreads();
    cv_sort<false>(buf, n2);
    int *crs = cslot + (size_t)p * C, *crw = cw + (size_t)p * C;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        crs[j] = buf[j].s;
        crw[j] = buf[j].w;
        atomicMax(&s_nmax, buf[j].w);
        if (buf[j].w >= COVIS_TH) atomicAdd(&s_nth, 1);
    }
    if (threadIdx.x == 0) cn[p] = n;
    __syncthreads();   // the table is dead from here: its storage takes the filtered list
    for (int j = threadIdx.x; j < n; j += blockDim.x)
        if (buf[j].w == s_nmax) atomicMin(&s_imax, j);   // `mit->second > nmax` in key order: the first maximum
    __syncthreads();
    const int m = s_nth > 0 ? s_nth : 1;
    if (s_nth > 0) {
        for (int j = threadIdx.x; j < n; j += blockDim.x)
            if (buf[j].w >= COVIS_TH) flt[atomicAdd(&s_f, 1)] = buf[j];
    } else if (threadIdx.x == 0) {
        flt[0] = buf[s_imax];
    }
    const int m2 = pow2ge(m);
    for (int j = m + threadIdx.x; j < m2; j += blockDim.x) flt[j] = cv_pad(true);
    __syncthreads();
    cv_sort<true>(flt, m2);   // sort() of (weight, KeyFrame*) pairs, then push_front: descending
    for (int j = threadIdx.x; j < m; j += blockDim.x) {
        fslot[(size_t)p * C + j] = flt[j].s;
        fw[(size_t)p * C + j] = flt[j].w;
    }
    if (threadIdx.x == 0) fn[p] = m;
}

// ---- launch 2: one block of 1024
__global__ void __launch_bounds__(1024) covis_plan_kernel(
    int n, const int *__restrict__ slots, int C, const int *__restrict__ cn, const int *__restrict__ cslot, const int *__restrict__ fn,
    const int *__restrict__ fslot, const int *__restrict__ fw, const int *__restrict__ state, const unsigned long long *__restrict__ key,
    const int *__restrict__ wn, const int *__restrict__ wslot, int *__restrict__ pos, int *__restrict__ tmark, int *__restrict__ evcnt,
    int *__restrict__ efill, int *__restrict__ ebase, int *__restrict__ touched, int *__restrict__ ev_p, int *__restrict__ ev_w,
    int *__restrict__ parent_out, int *__restrict__ flags) {
    __shared__ int s_nt, s_over, s_carry, s_warp[32];
    const int bad = flags[F_BAD], over = flags[F_OVER];
    if (threadIdx.x == 0) { s_nt = 0; s_over = 0; s_carry = 0; }
    __syncthreads();
    if (bad || over) {   // rejected before anything was marked
        if (threadIdx.x == 0) {
            flags[F_BAD] = 0;
            flags[F_OVER] = 0;
            flags[F_OK] = 0;
            flags[F_NT] = 0;
            atomicCAS(&flags[F_ERR], 0, bad ? ORBFE_ERR_ARG : ORBFE_ERR_CAPACITY);
        }
        if (parent_out)
            for (int p = threadIdx.x; p < n; p += blockDim.x) parent_out[p] = -1;
        return;
    }
    for (int p = threadIdx.x; p < n; p += blockDim.x) {
        const int s = slots[p];
        pos[s] = p;
        if (atomicExch(&tmark[s], 1) == 0) touched[atomicAdd(&s_nt, 1)] = s;
    }
    for (int p = 0; p < n; p++) {
        const int m = fn[p];
        for (int j = threadIdx.x; j < m; j += blockDim.x) {
            const int t = fslot[(size_t)p * C + j];
            atomicAdd(&evcnt[t], 1);
            if (atomicExch(&tmark[t], 1) == 0) touched[atomicAdd(&s_nt, 1)] = t;
        }
    }
    __syncthreads();
    const int nt = s_nt;
    for (int b = 0; b < nt; b += blockDim.x) {
        const int i = b + threadIdx.x;
        const int v = i < nt ? evcnt[touched[i]] : 0;
        const int e = cv_block_scan(v, s_warp, &s_carry);
        if (i < nt) ebase[touched[i]] = e;
    }
    __syncthreads();
    for (int p = 0; p < n; p++) {
        const int m = fn[p];
        for (int j = threadIdx.x; j < m; j += blockDim.x) {
            const int t = fslot[(size_t)p * C + j];
            const int e = ebase[t] + atomicAdd(&efill[t], 1);
            ev_p[e] = p;
            ev_w[e] = fw[(size_t)p * C + j];
        }
    }
    __syncthreads();
    // final size of every touched weight map: its start map plus the keys the applied events add
    for (int i = threadIdx.x; i < nt; i += blockDim.x) {
        const int t = touched[i], pt = pos[t];
        const bool own = pt >= 0 && cn[pt] > 0;
        const int *row = own ? cslot + (size_t)pt * C : wslot + (size_t)t * C;
        const int n0 = own ? cn[pt] : wn[t];
        int extra = 0;
        for (int e = ebase[t], e1 = e + evcnt[t]; e < e1; e++) {
            const int q = ev_p[e];
            if (own && q <= pt) continue;
            if (cv_find(row, n0, key, key[slots[q]]) < 0) extra++;
        }
        if (n0 + extra > C) s_over = 1;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        flags[F_OK] = !s_over;
        flags[F_NT] = nt;
        if (s_over) atomicCAS(&flags[F_ERR], 0, ORBFE_ERR_CAPACITY);
    }
    if (parent_out)
        for (int p = threadIdx.x; p < n; p += blockDim.x) {
            const int st = state[slots[p]];
            parent_out[p] = !s_over && cn[p] > 0 && (st & ST_FIRST) && !(st & ST_ID0) ? fslot[(size_t)p * C] : -1;
        }
}

// ---- launch 3: blocks stride over the touched slots
__global__ void __launch_bounds__(COVIS_APPLY_BLOCK) covis_apply_kernel(
    const int *__restrict__ slots, int C, int Cp, int Bp, const int *__restrict__ cn, const int *__restrict__ cslot,
    const int *__restrict__ cw, const int *__restrict__ fn, const int *__restrict__ fslot, const int *__restrict__ fw,
    const unsigned long long *__restrict__ key, int *__restrict__ state, int *__restrict__ wn, int *__restrict__ wslot,
    int *__restrict__ ww, int *__restrict__ on, int *__restrict__ oslot, int *__restrict__ ow, int *__restrict__ named,
    int *__restrict__ pos, int *__restrict__ tmark, int *__restrict__ evcnt, int *__restrict__ efill, const int *__restrict__ ebase,
    const int *__restrict__ touched, const int *__restrict__ ev_p, const int *__restrict__ ev_w, const int *__restrict__ flags) {
    extern __shared__ unsigned long long cv_smem[];
    CvEnt *A = reinterpret_cast<CvEnt *>(cv_smem);   // Cp: the start map, later the full sort
    CvEnt *E = A + Cp;                                // Bp: the applied events
    CvEnt *F = E + Bp;                                // Cp: the final map, key ascending
    __shared__ int s_ne, s_nf, s_changed;
    const int nt = flags[F_NT];
    const bool ok = flags[F_OK] != 0;
    for (int i = blockIdx.x; i < nt; i += gridDim.x) {
        const int t = touched[i], pt = pos[t];
        if (ok) {
            const bool own = pt >= 0 && cn[pt] > 0;
            const int *rs = own ? cslot + (size_t)pt * C : wslot + (size_t)t * C;
            const int *rw = own ? cw + (size_t)pt * C : ww + (size_t)t * C;
            const int na = own ? cn[pt] : wn[t];
            const int nold = wn[t];
            if (threadIdx.x == 0) { s_ne = 0; s_changed = 0; }
            for (int j = threadIdx.x; j < na; j += blockDim.x) A[j] = CvEnt{key[rs[j]], rs[j], rw[j]};
            __syncthreads();
            for (int e = ebase[t] + threadIdx.x, e1 = ebase[t] + evcnt[t]; e < e1; e += blockDim.x) {
                const int q = ev_p[e];
                if (own && q <= pt) continue;   // overwritten by the slot's own mConnectedKeyFrameWeights = KFcounter
                const int src = slots[q];
                E[atomicAdd(&s_ne, 1)] = CvEnt{key[src], src, ev_w[e]};
            }
            __syncthreads();
            const int ne = s_ne, ne2 = pow2ge(max(ne, 1));
            for (int j = ne + threadIdx.x; j < ne2; j += blockDim.x) E[j] = cv_pad(false);
            __syncthreads();
            cv_sort<false>(E, ne2);
            // an event changes the map when its key is absent or holds another weight (AddConnection, KeyFrame.cc:130-135)
            for (int j = threadIdx.x; j < ne; j += blockDim.x) {
                int lo = 0, hi = na;
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (A[mid].k < E[j].k) lo = mid + 1; else hi = mid;
                }
                if (lo == na || A[lo].k != E[j].k || A[lo].w != E[j].w) s_changed = 1;
            }
            if (threadIdx.x == 0) {   // merge by key; an event's weight replaces the start map's
                int a = 0, b = 0, f = 0;
                while (a < na || b < ne) {
                    if (b == ne || (a < na && A[a].k < E[b].k)) F[f++] = A[a++];
                    else {
                        if (a < na && A[a].k == E[b].k) a++;
                        F[f++] = E[b++];
                    }
                }
                s_nf = f;
            }
            __syncthreads();
            const int nf = s_nf;
            int *ws = wslot + (size_t)t * C, *wv = ww + (size_t)t * C;
            // keys that leave or enter the map
            for (int j = threadIdx.x; j < nold; j += blockDim.x) {
                const unsigned long long k = key[ws[j]];
                int lo = 0, hi = nf;
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (F[mid].k < k) lo = mid + 1; else hi = mid;
                }
                if (lo == nf || F[lo].k != k) atomicSub(&named[ws[j]], 1);
            }
            for (int j = threadIdx.x; j < nf; j += blockDim.x)
                if (cv_find(ws, nold, key, F[j].k) < 0) atomicAdd(&named[F[j].s], 1);
            __syncthreads();
            for (int j = threadIdx.x; j < nf; j += blockDim.x) { ws[j] = F[j].s; wv[j] = F[j].w; }
            const bool changed = s_changed != 0;
            int *os = oslot + (size_t)t * C, *ov = ow + (size_t)t * C;
            if (changed) {   // UpdateBestCovisibles over the whole map
                const int nf2 = pow2ge(nf);
                for (int j = threadIdx.x; j < nf2; j += blockDim.x) A[j] = j < nf ? F[j] : cv_pad(true);
                __syncthreads();
                cv_sort<true>(A, nf2);
                for (int j = threadIdx.x; j < nf; j += blockDim.x) { os[j] = A[j].s; ov[j] = A[j].w; }
            } else if (own) {
                const int m = fn[pt];
                for (int j = threadIdx.x; j < m; j += blockDim.x) { os[j] = fslot[(size_t)pt * C + j]; ov[j] = fw[(size_t)pt * C + j]; }
            }
            if (threadIdx.x == 0) {
                wn[t] = nf;
                if (changed) on[t] = nf;
                else if (own) on[t] = fn[pt];
                if (own && (state[t] & ST_FIRST) && !(state[t] & ST_ID0)) state[t] &= ~ST_FIRST;
            }
        }
        if (threadIdx.x == 0) {
            tmark[t] = 0;
            evcnt[t] = 0;
            efill[t] = 0;
            pos[t] = -1;
        }
        __syncthreads();
    }
}

// ---- SetBadFlag's connection half: block j handles the j-th key of the slot's own map (EraseConnection on that neighbour)
__global__ void __launch_bounds__(COVIS_APPLY_BLOCK) covis_erase_kernel(int slot, int C, const unsigned long long *__restrict__ key,
                                                                         int *__restrict__ wn, int *__restrict__ wslot, int *__restrict__ ww,
                                                                         int *__restrict__ on, int *__restrict__ oslot, int *__restrict__ ow,
                                                                         int *__restrict__ named) {
    extern __shared__ unsigned long long cv_smem[];
    CvEnt *A = reinterpret_cast<CvEnt *>(cv_smem);
    __shared__ int s_at;
    const int j = blockIdx.x;
    if (j >= wn[slot]) return;
    const int nb = wslot[(size_t)slot * C + j];
    int *ws = wslot + (size_t)nb * C, *wv = ww + (size_t)nb * C;
    const int n = wn[nb];
    if (threadIdx.x == 0) {
        atomicSub(&named[nb], 1);   // the slot's own map is cleared
        s_at = cv_find(ws, n, key, key[slot]);
    }
    __syncthreads();
    const int at = s_at;
    if (at < 0) return;   // a map that does not name the slot is left as it is (KeyFrame.cc:601)
    const int m = n - 1, m2 = pow2ge(max(m, 1));
    for (int i = threadIdx.x; i < m2; i += blockDim.x) {
        if (i < m) {
            const int src = i < at ? i : i + 1;
            A[i] = CvEnt{key[ws[src]], ws[src], wv[src]};
        } else {
            A[i] = cv_pad(true);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += blockDim.x) { ws[i] = A[i].s; wv[i] = A[i].w; }   // key order, the entry removed
    __syncthreads();
    cv_sort<true>(A, m2);
    int *os = oslot + (size_t)nb * C, *ov = ow + (size_t)nb * C;
    for (int i = threadIdx.x; i < m; i += blockDim.x) { os[i] = A[i].s; ov[i] = A[i].w; }
    if (threadIdx.x == 0) {
        wn[nb] = m;
        on[nb] = m;
        atomicSub(&named[slot], 1);
    }
}

__global__ void covis_retire_kernel(int slot, int *__restrict__ state, int *__restrict__ wn, int *__restrict__ on) {
    state[slot] = 0;
    wn[slot] = 0;
    on[slot] = 0;
}

// rows: slot, mnId == 0, key (two ints)
__global__ void covis_add_kernel(int n, const int *__restrict__ rows, unsigned long long *__restrict__ key, int *__restrict__ state,
                                 int *__restrict__ wn, int *__restrict__ on) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int *r = rows + 4 * i;
    const int s = r[0];
    key[s] = (unsigned long long)(unsigned)r[2] | (unsigned long long)(unsigned)r[3] << 32;
    state[s] = ST_LIVE | ST_FIRST | (r[1] ? ST_ID0 : 0);
    wn[s] = 0;
    on[s] = 0;
}

// ---- the exported lists: row lengths and their exclusive scan (one block of 1024), then one block per row
__global__ void __launch_bounds__(1024) covis_lens_kernel(int n, const int *__restrict__ slots, int which, int limit,
                                                          const int *__restrict__ wn, const int *__restrict__ on, int *__restrict__ ptr) {
    __shared__ int s_carry, s_warp[32];
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int b = 0; b < n; b += blockDim.x) {
        const int i = b + threadIdx.x;
        const int v = i < n ? min(which ? wn[slots[i]] : on[slots[i]], limit) : 0;
        const int e = cv_block_scan(v, s_warp, &s_carry);
        if (i < n) ptr[i] = e;
    }
    if (threadIdx.x == 0) ptr[n] = s_carry;
}

__global__ void covis_lists_kernel(const int *__restrict__ slots, int which, int C, const int *__restrict__ ptr,
                                   const int *__restrict__ wslot, const int *__restrict__ ww, const int *__restrict__ oslot,
                                   const int *__restrict__ ow, const int *__restrict__ state, int *__restrict__ list,
                                   int *__restrict__ weights) {
    const int i = blockIdx.x, s = slots[i];
    const int lo = ptr[i], len = ptr[i + 1] - lo;
    const int *rs = (which ? wslot : oslot) + (size_t)s * C, *rw = (which ? ww : ow) + (size_t)s * C;
    for (int j = threadIdx.x; j < len; j += blockDim.x) {
        const int v = rs[j];
        list[lo + j] = (state[v] & ST_LIVE) ? v : -1;   // a retired keyframe still named here: isBad() -> negative
        if (weights) weights[lo + j] = rw[j];
    }
}

// ---- MapPoint::GetObservations() of named points, built as the inverse of the live slots' map-point rows (DESIGN.md §4.7).
// Five launches, no host round trip.  The scratch is the caller's: stamp[npoints], cnt[npoints], tmp[obs_cap]; none of it
// has to be initialised, because a stamp is only believed when points[stamp[v]] == v.
#define COVIS_OBS_MAX_CAP ORBFE_COVIS_OBS_MAX_CAP   // a row's table (2 * cap entries, rounded up to a power of two) is in shared memory
#define COVIS_OBS_BLOCK 512
#define COVIS_OBS_SCAN_ITEMS 8
#define COVIS_OBS_SORT_BLOCK 256
#define COVIS_OBS_TILE 1024
// flags of this entry: [5] bad input in this call, [6] this call stops after the scan, [7] the entry that set [3]
enum { F_OBS_BAD = 5, F_OBS_STOP = 6, F_ERR_SRC = 7 };

// the position of point v among the named points, or -1
__device__ __forceinline__ int obs_pos(int v, int n, const int *points, const int *stamp) {
    const int j = stamp[v];
    return j >= 0 && j < n && points[j] == v ? j : -1;
}

// launch 1: stamp[p] = j for the named point p = points[j]; the per-position counts start at 0
__global__ void covis_obs_stamp_kernel(int n, const int *__restrict__ points, int npoints, int *__restrict__ stamp, int *__restrict__ cnt,
                                       int *__restrict__ flags) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const int p = points[j];
        if (p < 0 || p >= npoints) atomicOr(&flags[F_OBS_BAD], 1);
        else stamp[p] = j;
        cnt[j] = 0;
    }
}

// launches 2 and 4: blocks stride over the live slots.  A row's named points go into a shared-memory table keyed by point
// that keeps the largest feature index (ProcessNewKeyFrame writes mObservations[pKF] = i in ascending i: the last one stays).
// Scatter = false counts one observation per (slot, point) and checks the input; Scatter = true writes s*cap + i at the
// point's next free entry of tmp, counting its count back down to 0.
template <bool Scatter>
__global__ void __launch_bounds__(COVIS_OBS_BLOCK) covis_obs_rows_kernel(
    int nslots, int T, const int *__restrict__ state, const int *__restrict__ kf_mp, const int *__restrict__ counts, int cap, int npoints,
    int n, const int *__restrict__ points, const int *__restrict__ stamp, int *__restrict__ cnt, const int *__restrict__ ptr,
    int *__restrict__ tmp, int *__restrict__ flags) {
    extern __shared__ int2 ob_tab[];
    if (Scatter && flags[F_OBS_STOP]) return;
    if (!Scatter)   // a point named twice: one of its positions lost the stamp
        for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
            const int p = points[j];
            if (p >= 0 && p < npoints && stamp[p] != j) atomicOr(&flags[F_OBS_BAD], 1);
        }
    for (int s = blockIdx.x; s < nslots; s += gridDim.x) {
        if (!(state[s] & ST_LIVE)) continue;   // not an observer: never added, or retired
        const int c = counts[s];
        if (c < 0 || c > cap) {
            if (!Scatter && threadIdx.x == 0) atomicOr(&flags[F_OBS_BAD], 1);
            continue;
        }
        for (int h = threadIdx.x; h < T; h += blockDim.x) ob_tab[h] = make_int2(-1, -1);
        __syncthreads();
        const int *row = kf_mp + (size_t)s * cap;
        for (int i = threadIdx.x; i < c; i += blockDim.x) {
            const int v = row[i];
            if (v < 0) continue;   // NULL or isBad()
            if (v >= npoints) {
                if (!Scatter) atomicOr(&flags[F_OBS_BAD], 1);
                continue;
            }
            if (obs_pos(v, n, points, stamp) < 0) continue;
            unsigned h = ((unsigned)v * 2654435761u) & (unsigned)(T - 1);
            for (;;) {   // T >= 2 * cap: never full
                const int old = atomicCAS(&ob_tab[h].x, -1, v);
                if (old == -1 || old == v) { atomicMax(&ob_tab[h].y, i); break; }
                h = (h + 1) & (unsigned)(T - 1);
            }
        }
        __syncthreads();
        for (int h = threadIdx.x; h < T; h += blockDim.x) {
            const int2 e = ob_tab[h];
            if (e.x < 0) continue;
            const int j = stamp[e.x];
            if (Scatter) tmp[ptr[j] + atomicSub(&cnt[j], 1) - 1] = s * cap + e.y;
            else atomicAdd(&cnt[j], 1);
        }
        __syncthreads();
    }
}

// launch 3: one block of 1024.  ptr = the exclusive scan of the counts (tiles of 1024 x 8), the reference slots checked, the
// call decided: bad input stops it with ptr written, a total over obs_cap stops it with ptr and *nobs_out written.
__global__ void __launch_bounds__(1024) covis_obs_scan_kernel(int n, const int *__restrict__ cnt, const int *__restrict__ ref_slot,
                                                              int nframes, int obs_cap, int *__restrict__ ptr, int *__restrict__ nobs_out,
                                                              int *__restrict__ flags) {
    __shared__ int s_carry, s_badref, s_warp[32];
    __shared__ int s_v[1024 * COVIS_OBS_SCAN_ITEMS];
    const int TN = 1024 * COVIS_OBS_SCAN_ITEMS;
    if (threadIdx.x == 0) { s_carry = 0; s_badref = 0; }
    __syncthreads();
    for (int b = 0; b < n; b += TN) {
        for (int k = threadIdx.x; k < TN; k += blockDim.x) s_v[k] = b + k < n ? cnt[b + k] : 0;
        __syncthreads();
        int *mine = s_v + threadIdx.x * COVIS_OBS_SCAN_ITEMS, loc = 0;
        for (int q = 0; q < COVIS_OBS_SCAN_ITEMS; q++) loc += mine[q];
        int run = cv_block_scan(loc, s_warp, &s_carry);
        for (int q = 0; q < COVIS_OBS_SCAN_ITEMS; q++) {
            const int v = mine[q];
            mine[q] = run;
            run += v;
        }
        __syncthreads();
        for (int k = threadIdx.x; k < TN && b + k < n; k += blockDim.x) ptr[b + k] = s_v[k];
        __syncthreads();
    }
    if (ref_slot)
        for (int j = threadIdx.x; j < n; j += blockDim.x) {
            const int r = ref_slot[j];
            if (r < 0 || r >= nframes) s_badref = 1;
        }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int total = s_carry;
        ptr[n] = total;
        const int bad = flags[F_OBS_BAD] | s_badref;
        flags[F_OBS_BAD] = 0;
        int code = ORBFE_OK;
        if (bad) {
            code = ORBFE_ERR_ARG;
        } else {
            *nobs_out = total;
            if (total > obs_cap) code = ORBFE_ERR_CAPACITY;
        }
        flags[F_OBS_STOP] = code != ORBFE_OK;
        if (code != ORBFE_OK && atomicCAS(&flags[F_ERR], 0, code) == 0) flags[F_ERR_SRC] = 1;
    }
}

// launch 5: every list in key order, and the reference observation.  Blocks stride over groups of 8 points, one warp per
// point: a list of at most 32 entries is ranked in registers; a longer one is queued and ranked by the whole block against
// its keys staged in shared memory.  A list's keys are distinct (one entry per live slot), so the ranks are a permutation.
__global__ void __launch_bounds__(COVIS_OBS_SORT_BLOCK) covis_obs_sort_kernel(
    int n, int cap, const unsigned long long *__restrict__ key, const int *__restrict__ ptr, const int *__restrict__ tmp,
    const int *__restrict__ ref_slot, int *__restrict__ obs, int *__restrict__ ref_obs, const int *__restrict__ flags) {
    __shared__ unsigned long long s_key[COVIS_OBS_TILE];
    __shared__ int s_long[COVIS_OBS_SORT_BLOCK / 32], s_nlong, s_found;
    if (flags[F_OBS_STOP]) return;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, W = COVIS_OBS_SORT_BLOCK / 32;
    for (int g0 = blockIdx.x * W; g0 < n; g0 += gridDim.x * W) {
        if (threadIdx.x == 0) s_nlong = 0;
        __syncthreads();
        const int j = g0 + wid;
        if (j < n) {
            const int lo = ptr[j], L = ptr[j + 1] - lo;
            if (L > 32) {
                if (lane == 0) s_long[atomicAdd(&s_nlong, 1)] = j;
            } else {
                const int v = lane < L ? tmp[lo + lane] : 0;
                const unsigned long long k = lane < L ? key[v / cap] : ~0ull;
                int r = 0;
                for (int o = 0; o < L; o++) r += __shfl_sync(0xffffffffu, k, o) < k;
                if (lane < L) obs[lo + r] = v;
                if (ref_obs) {   // observations[pRefKF], the map's insert-0 when absent
                    const int ref = ref_slot[j];
                    const unsigned m = __ballot_sync(0xffffffffu, lane < L && v / cap == ref);
                    if (lane == (m ? __ffs(m) - 1 : 0)) ref_obs[j] = m ? v : ref * cap;
                }
            }
        }
        __syncthreads();
        for (int q = 0; q < s_nlong; q++) {
            const int jl = s_long[q], lo = ptr[jl], L = ptr[jl + 1] - lo;
            const int ref = ref_obs ? ref_slot[jl] : -1;
            if (threadIdx.x == 0) s_found = ref * cap;
            for (int b = 0; b < L; b += blockDim.x) {
                const int e = b + threadIdx.x;
                const int v = e < L ? tmp[lo + e] : 0;
                const unsigned long long k = e < L ? key[v / cap] : 0ull;
                int r = 0;
                for (int t0 = 0; t0 < L; t0 += COVIS_OBS_TILE) {
                    const int tn = min(COVIS_OBS_TILE, L - t0);
                    __syncthreads();
                    for (int x = threadIdx.x; x < tn; x += blockDim.x) s_key[x] = key[tmp[lo + t0 + x] / cap];
                    __syncthreads();
                    if (e < L)
                        for (int x = 0; x < tn; x++) r += s_key[x] < k;
                }
                if (e < L) {
                    obs[lo + r] = v;
                    if (v / cap == ref) s_found = v;   // at most one entry per slot
                }
            }
            __syncthreads();
            if (ref_obs && threadIdx.x == 0) ref_obs[jl] = s_found;
            __syncthreads();
        }
        __syncthreads();
    }
}

// ---- LocalMapping::KeyFrameCulling (LocalMapping.cc:524-578) for the current keyframe's GetVectorCovisibleKeyFrames(), with
// KeyFrame::SetBadFlag's point half (MapPoint::EraseObservation / SetBadFlag, MapPoint.cc:71-122) applied in list order
// (DESIGN.md §4.8).  After the five observation launches (every point's list, so no host count is needed), three launches:
// the candidates' checks, one persistent block that walks the list, and the NULLing of the made-bad points' cells.
// Scratch beyond the observation kernels' (all ints, then one byte per list entry):
//   pts[npoints] = 0, 1, ..  (the named points of the observation build), ptr[npoints + 1], obs[obs_cap],
//   lcnt[npoints]   live observers of each point the candidates name
//   bad_at[npoints] the list position whose SetBadFlag made the point bad, else CULL_NEVER
//   gone_at[nframes] the list position that erased the slot, else CULL_NEVER
//   ne[nframes]     mbNotErase
//   ctl[8]          [0] bad input, [1] an error was pending before this call
//   alive[obs_cap]  the entry is still in mObservations
#define COVIS_CULL_BLOCK 1024
#define COVIS_CULL_CHECK_BLOCK 256
#define CULL_NEVER 0x7F7F7F7F   // the memset byte 0x7F: after every list position
enum { CULL_KEPT = ORBFE_CULL_KEPT, CULL_SKIP_ID0 = ORBFE_CULL_SKIP_ID0, CULL_ERASED = ORBFE_CULL_ERASED,
       CULL_NOT_ERASE = ORBFE_CULL_NOT_ERASE, CULL_RETIRED = ORBFE_CULL_RETIRED };
enum { CTL_BAD = 0, CTL_PENDING = 1, CTL_COUNT = 8 };

struct CullScratch {
    int *stamp, *cnt, *tmp, *pts, *ptr, *obs, *lcnt, *bad_at, *gone_at, *ne, *ctl;
    unsigned char *alive;
};

// the named points are all points; mbNotErase marks; whether an error was already pending
__global__ void covis_cull_prep_kernel(int npoints, int n_ne, const int *__restrict__ ne_slots, CullScratch w, const int *__restrict__ flags) {
    const int t0 = blockIdx.x * blockDim.x + threadIdx.x, T = gridDim.x * blockDim.x;
    for (int p = t0; p < npoints; p += T) w.pts[p] = p;
    for (int j = t0; j < n_ne; j += T) w.ne[ne_slots[j]] = 1;
    if (t0 == 0) w.ctl[CTL_PENDING] = flags[F_ERR] != 0;
}

__device__ __forceinline__ bool cull_octave_ok(int o) { return o >= 0 && o < ORBFE_MAX_LEVELS; }

// one block per list position: the candidate's count, row values, octaves, its points' reference slots and their observers'
// octaves are checked; the live count and entry flags of every point it names are set (several blocks may write the same
// values)
__global__ void __launch_bounds__(COVIS_CULL_CHECK_BLOCK) covis_cull_check_kernel(
    int cur, int C, const int *__restrict__ on, const int *__restrict__ oslot, const int *__restrict__ kf_mp, const int *__restrict__ counts,
    const OrbfeKeyPoint *__restrict__ kps, int nframes, int cap, const unsigned char *__restrict__ point_bad,
    const int *__restrict__ ref_slot, int npoints, CullScratch w, const int *__restrict__ flags) {
    const int n = on[cur];
    if (flags[F_OBS_STOP]) return;
    for (int t = blockIdx.x; t < n; t += gridDim.x) {
        const int v = oslot[(size_t)cur * C + t];
        const int c = v < nframes ? counts[v] : -1;
        if (c < 0 || c > cap) {
            if (threadIdx.x == 0) atomicOr(&w.ctl[CTL_BAD], 1);
            continue;
        }
        for (int i = threadIdx.x; i < c; i += blockDim.x) {
            const int p = kf_mp[(size_t)v * cap + i];
            if (p < 0) continue;
            if (p >= npoints) { atomicOr(&w.ctl[CTL_BAD], 1); continue; }
            if (point_bad[p]) continue;
            bool ok = cull_octave_ok(kps[(size_t)v * cap + i].octave);
            const int r = ref_slot[p];
            ok &= r >= 0 && r < nframes;
            const int lo = w.ptr[p], hi = w.ptr[p + 1];
            for (int e = lo; e < hi; e++) {
                ok &= cull_octave_ok(kps[w.obs[e]].octave);
                w.alive[e] = 1;
            }
            w.lcnt[p] = hi - lo;
            if (!ok) atomicOr(&w.ctl[CTL_BAD], 1);
        }
    }
}

// the sum of v over the block, returned to every thread
__device__ int cull_block_sum(int v, int *s_warp) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
    __syncthreads();
    int s = 0;
    for (int k = 0; k < COVIS_CULL_BLOCK / 32; k++) s += s_warp[k];
    __syncthreads();
    return s;
}

// one block of 1024 walks the list in order; each step's cells are spread over the block, and an erase's cascade runs on
// the row's cells in parallel (one point per cell that holds the point's observation of the keyframe: its largest index)
__global__ void __launch_bounds__(COVIS_CULL_BLOCK) covis_cull_kernel(
    int cur, int C, const int *__restrict__ on, const int *__restrict__ oslot, const int *__restrict__ state, const unsigned long long *__restrict__ key,
    const int *__restrict__ kf_mp, const int *__restrict__ counts, const OrbfeKeyPoint *__restrict__ kps, int cap,
    unsigned char *__restrict__ point_bad, int *__restrict__ ref_slot, int npoints, int *__restrict__ verdict_slot, int *__restrict__ verdict,
    int *__restrict__ ncand, int *__restrict__ nmps_out, int *__restrict__ nred_out, int *__restrict__ bad_points, int *__restrict__ nbad,
    CullScratch w, int *__restrict__ flags) {
    __shared__ int s_warp[COVIS_CULL_BLOCK / 32], s_carry;
    if (flags[F_OBS_STOP] || w.ctl[CTL_BAD]) {   // nothing written
        if (threadIdx.x == 0) {
            if (w.ctl[CTL_BAD] && !flags[F_OBS_STOP]) atomicCAS(&flags[F_ERR], 0, ORBFE_ERR_ARG);
            if (!w.ctl[CTL_PENDING]) flags[F_ERR_SRC] = 2;
        }
        return;
    }
    const int n = on[cur];
    for (int t = 0; t < n; t++) {
        const int v = oslot[(size_t)cur * C + t];
        const int st = state[v];
        if (st & ST_ID0) {   // pKF->mnId == 0: skipped before anything is counted
            if (threadIdx.x == 0) {
                verdict_slot[t] = v;
                verdict[t] = CULL_SKIP_ID0;
                if (nmps_out) nmps_out[t] = 0;
                if (nred_out) nred_out[t] = 0;
            }
            continue;
        }
        const int c = counts[v];
        const int *row = kf_mp + (size_t)v * cap;
        const OrbfeKeyPoint *kp = kps + (size_t)v * cap;
        int nm = 0, nr = 0;
        for (int i = threadIdx.x; i < c; i += blockDim.x) {
            const int p = row[i];
            if (p < 0 || point_bad[p]) continue;
            nm++;
            if (w.lcnt[p] <= 3) continue;   // Observations() counts pKF itself when it observes p
            const int lvl = kp[i].octave;
            int m = 0;
            for (int e = w.ptr[p], e1 = w.ptr[p + 1]; e < e1 && m < 3; e++) {
                const int o = w.obs[e];
                if (!w.alive[e] || o / cap == v) continue;
                if (kps[o].octave <= lvl + 1) m++;
            }
            nr += m >= 3;
        }
        const int NM = cull_block_sum(nm, s_warp), NR = cull_block_sum(nr, s_warp);
        const bool redundant = 10 * (long long)NR > 9 * (long long)NM;   // == (double)NR > 0.9 * NM for every int (DESIGN §2)
        const int code = !redundant ? CULL_KEPT : w.ne[v] ? CULL_NOT_ERASE : !(st & ST_LIVE) ? CULL_RETIRED : CULL_ERASED;
        if (threadIdx.x == 0) {
            verdict_slot[t] = v;
            verdict[t] = code;
            if (nmps_out) nmps_out[t] = NM;
            if (nred_out) nred_out[t] = NR;
            if (code == CULL_ERASED) w.gone_at[v] = t;
        }
        if (code == CULL_ERASED) {
            const unsigned long long kv = key[v];
            for (int i = threadIdx.x; i < c; i += blockDim.x) {
                const int p = row[i];
                if (p < 0 || point_bad[p]) continue;
                const int lo = w.ptr[p], hi = w.ptr[p + 1];
                int a = lo, b = hi;   // the list is in key order: v's entry
                while (a < b) {
                    const int mid = (a + b) >> 1;
                    if (key[w.obs[mid] / cap] < kv) a = mid + 1; else b = mid;
                }
                if (a == hi || w.obs[a] != v * cap + i || !w.alive[a]) continue;   // not an observer, or not this cell
                w.alive[a] = 0;
                const int left = --w.lcnt[p];
                if (ref_slot[p] == v) {   // mpRefKF = mObservations.begin()->first; undefined when none is left
                    for (int e = lo; e < hi; e++)
                        if (w.alive[e]) { ref_slot[p] = w.obs[e] / cap; break; }
                }
                if (left <= 2) {
                    point_bad[p] = 1;
                    w.bad_at[p] = t;
                }
            }
        }
        __syncthreads();
    }
    // the points this call made bad, ascending: tiles of 1024 x 8, each thread's 8 points consecutive
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int b = 0; b < npoints; b += COVIS_CULL_BLOCK * COVIS_OBS_SCAN_ITEMS) {
        const int p0 = b + threadIdx.x * COVIS_OBS_SCAN_ITEMS;
        unsigned mine = 0;
        for (int q = 0; q < COVIS_OBS_SCAN_ITEMS; q++)
            if (p0 + q < npoints && w.bad_at[p0 + q] != CULL_NEVER) mine |= 1u << q;
        int at = cv_block_scan(__popc(mine), s_warp, &s_carry);
        for (int q = 0; q < COVIS_OBS_SCAN_ITEMS; q++)
            if (mine >> q & 1) bad_points[at++] = p0 + q;
    }
    if (threadIdx.x == 0) {
        *nbad = s_carry;
        *ncand = n;
    }
}

// blocks stride over the slots live at the call: a cell naming a point made bad while the slot was still its observer (before
// the slot's own erase, if any) becomes NULL, duplicates included
__global__ void __launch_bounds__(256) covis_cull_null_kernel(int nslots, const int *__restrict__ state, int *__restrict__ kf_mp,
                                                              const int *__restrict__ counts, int cap, CullScratch w,
                                                              const int *__restrict__ flags) {
    if (flags[F_OBS_STOP] || w.ctl[CTL_BAD]) return;
    for (int s = blockIdx.x; s < nslots; s += gridDim.x) {
        if (!(state[s] & ST_LIVE)) continue;
        const int gone = w.gone_at[s], c = counts[s];
        int *row = kf_mp + (size_t)s * cap;
        for (int i = threadIdx.x; i < c; i += blockDim.x) {
            const int p = row[i];
            if (p >= 0 && w.bad_at[p] < gone) row[i] = -1;
        }
    }
}

// ---- Tracking::UpdateReference (Tracking.cc:728-839) for one frame: UpdateReferenceKeyFrames and UpdateReferencePoints on
// the graph and the live slots' rows (DESIGN.md §4.9).  Six launches after two memsets, no host round trip:
//   frame   mult[p] = the frame cells naming p (p not bad); cells >= npoints flag the call
//   vote    one block per live row: the row's points with mult > 0, deduplicated in a shared-memory table, add their mult
//           to the slot's counter (a point at k cells votes k times; a row naming it twice is one observation)
//   list    one block: NULL the bad frame cells, compact the counted slots, rank them by key, the first strict maximum,
//           the sequential extension by one warp, the row offsets of the list's entries
//   first   atomicMin of each point's position in the concatenated rows of the list
//   keep / scatter   the cells holding their point's first position, counted per row and written in row order
// Scratch (ints): mult[npoints], ctl[LM_CTL] (zeroed by the entry), first[npoints] (set to all ones by the entry),
// cnt[nframes], cand[nframes], rowoff[nframes + 1], kcnt[nframes].
#define COVIS_LM_BLOCK 1024
#define COVIS_LM_VOTE_BLOCK 512
#define LM_NEIGH 10       // GetBestCovisibilityKeyFrames(10), Tracking.cc:820
#define LM_MAX_KF 80      // `mvpLocalKeyFrames.size() > 80` stops the extension, Tracking.cc:815
#define LM_HASH 256       // the appended slots (at most LM_MAX_KF + 1) in shared memory
enum { LM_BAD = 0, LM_NL = 1, LM_CTL = 4 };

struct LmScratch {
    int *mult, *ctl;
    unsigned *first;
    int *cnt, *cand, *rowoff, *kcnt;
};

__global__ void covis_lm_frame_kernel(int nf, const int *__restrict__ frame_mp, const unsigned char *__restrict__ point_bad, int npoints,
                                      LmScratch w) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nf; i += gridDim.x * blockDim.x) {
        const int p = frame_mp[i];
        if (p < 0) continue;
        if (p >= npoints) atomicOr(&w.ctl[LM_BAD], 1);
        else if (!point_bad[p]) atomicAdd(&w.mult[p], 1);
    }
}

// blocks stride over the slots; a slot that is not live counts 0 (retired slots are not observers)
__global__ void __launch_bounds__(COVIS_LM_VOTE_BLOCK) covis_lm_vote_kernel(int nslots, int T, const int *__restrict__ state,
                                                                           const int *__restrict__ kf_mp, const int *__restrict__ counts,
                                                                           int cap, int npoints, LmScratch w) {
    extern __shared__ int lm_tab[];
    __shared__ int s_warp[COVIS_LM_VOTE_BLOCK / 32];
    for (int s = blockIdx.x; s < nslots; s += gridDim.x) {
        if (!(state[s] & ST_LIVE)) {
            if (threadIdx.x == 0) w.cnt[s] = 0;
            continue;
        }
        const int c = counts[s];
        if (c < 0 || c > cap) {
            if (threadIdx.x == 0) {
                atomicOr(&w.ctl[LM_BAD], 1);
                w.cnt[s] = 0;
            }
            continue;
        }
        for (int h = threadIdx.x; h < T; h += blockDim.x) lm_tab[h] = -1;
        __syncthreads();
        const int *row = kf_mp + (size_t)s * cap;
        for (int i = threadIdx.x; i < c; i += blockDim.x) {
            const int p = row[i];
            if (p < 0) continue;   // NULL or isBad()
            if (p >= npoints) {
                atomicOr(&w.ctl[LM_BAD], 1);
                continue;
            }
            if (w.mult[p] == 0) continue;   // not in the frame
            unsigned h = ((unsigned)p * 2654435761u) & (unsigned)(T - 1);
            for (;;) {   // T >= 2 * cap: never full
                const int old = atomicCAS(&lm_tab[h], -1, p);
                if (old == -1 || old == p) break;
                h = (h + 1) & (unsigned)(T - 1);
            }
        }
        __syncthreads();
        int v = 0;
        for (int h = threadIdx.x; h < T; h += blockDim.x)
            if (lm_tab[h] >= 0) v += w.mult[lm_tab[h]];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
        __syncthreads();
        if (threadIdx.x == 0) {
            int t = 0;
            for (int k = 0; k < COVIS_LM_VOTE_BLOCK / 32; k++) t += s_warp[k];
            w.cnt[s] = t;
        }
        __syncthreads();
    }
}

__device__ __forceinline__ bool lm_hash_has(const int *tab, int u) {
    for (unsigned h = ((unsigned)u * 2654435761u) & (LM_HASH - 1);; h = (h + 1) & (LM_HASH - 1)) {
        if (tab[h] == u) return true;
        if (tab[h] < 0) return false;
    }
}

__device__ __forceinline__ void lm_hash_put(int *tab, int u) {
    unsigned h = ((unsigned)u * 2654435761u) & (LM_HASH - 1);
    while (tab[h] >= 0) h = (h + 1) & (LM_HASH - 1);
    tab[h] = u;
}

__global__ void __launch_bounds__(COVIS_LM_BLOCK) covis_lm_list_kernel(
    int nslots, int C, const int *__restrict__ on, const int *__restrict__ oslot, const int *__restrict__ state,
    const unsigned long long *__restrict__ key, const int *__restrict__ counts, int nf, int *__restrict__ frame_mp,
    const unsigned char *__restrict__ point_bad, int *__restrict__ local_kf, int *__restrict__ nlocal_kf, int *__restrict__ ref_kf,
    LmScratch w, int *__restrict__ flags) {
    __shared__ unsigned long long s_key[COVIS_LM_BLOCK], s_kmin;
    __shared__ int s_warp[32], s_carry, s_max, s_ref, s_n;
    __shared__ int s_nb[LM_MAX_KF * LM_NEIGH], s_app[LM_HASH];
    if (w.ctl[LM_BAD]) {   // nothing written
        if (threadIdx.x == 0 && atomicCAS(&flags[F_ERR], 0, ORBFE_ERR_ARG) == 0) flags[F_ERR_SRC] = 3;
        return;
    }
    for (int i = threadIdx.x; i < nf; i += blockDim.x) {   // Tracking.cc:779-782
        const int p = frame_mp[i];
        if (p >= 0 && point_bad[p]) frame_mp[i] = -1;
    }
    if (threadIdx.x == 0) { s_carry = 0; s_max = 0; s_kmin = ~0ull; s_ref = -1; }
    __syncthreads();
    // the counted slots in slot order, and the largest count
    int mx = 0;
    for (int b = 0; b < nslots; b += blockDim.x) {
        const int s = b + threadIdx.x;
        const int c = s < nslots ? w.cnt[s] : 0;
        const int at = cv_block_scan(c > 0, s_warp, &s_carry);
        if (c > 0) {
            w.cand[at] = s;
            mx = max(mx, c);
        }
    }
    atomicMax(&s_max, mx);
    __syncthreads();
    const int n0 = s_carry, M = s_max;
    // `it->second > max` over the map in key order: the first maximum, the smallest key among the maxima
    for (int e = threadIdx.x; e < n0; e += blockDim.x) {
        const int s = w.cand[e];
        if (w.cnt[s] == M) atomicMin(&s_kmin, key[s]);
    }
    __syncthreads();
    // std::map<KeyFrame*, int> order: each counted slot's rank among the counted keys (distinct: one per live slot)
    for (int b = 0; b < n0; b += blockDim.x) {
        const int e = b + threadIdx.x;
        const int s = e < n0 ? w.cand[e] : -1;
        const unsigned long long k = e < n0 ? key[s] : 0ull;
        int r = 0;
        for (int t0 = 0; t0 < n0; t0 += COVIS_LM_BLOCK) {
            const int tn = min(COVIS_LM_BLOCK, n0 - t0);
            __syncthreads();
            if (threadIdx.x < tn) s_key[threadIdx.x] = key[w.cand[t0 + threadIdx.x]];
            __syncthreads();
            if (e < n0)
                for (int x = 0; x < tn; x++) r += s_key[x] < k;
        }
        if (e < n0) {
            local_kf[r] = s;
            if (k == s_kmin) s_ref = s;
        }
    }
    // the extension visits only the n0 entries above (its end iterator is fixed) and stops before a visit once the list
    // holds more than 80: with n0 > 80 nothing is visited.  Each visit's first 10 neighbours are staged with the ones that
    // cannot be taken (retired: a stale entry; or counted: listed above) already removed.
    const int V = n0 <= LM_MAX_KF ? n0 : 0;
    for (int h = threadIdx.x; h < LM_HASH; h += blockDim.x) s_app[h] = -1;
    __syncthreads();
    for (int j = threadIdx.x; j < V * LM_NEIGH; j += blockDim.x) {
        const int t = j / LM_NEIGH, q = j - t * LM_NEIGH, v = local_kf[t];
        const int u = q < on[v] ? oslot[(size_t)v * C + q] : -1;
        s_nb[j] = u >= 0 && (state[u] & ST_LIVE) && w.cnt[u] == 0 ? u : -1;   // a live slot is < nslots
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        int n = n0;
        for (int t = 0; t < V && n <= LM_MAX_KF; t++) {
            const int u = lane < LM_NEIGH ? s_nb[t * LM_NEIGH + lane] : -1;
            const unsigned m = __ballot_sync(0xffffffffu, u >= 0 && !lm_hash_has(s_app, u));
            if (m) {   // the first neighbour not yet listed is appended, and the walk of this entry's neighbours stops
                const int take = __shfl_sync(0xffffffffu, u, __ffs(m) - 1);
                if (lane == 0) {
                    lm_hash_put(s_app, take);
                    local_kf[n] = take;
                }
                n++;
            }
            __syncwarp();
        }
        if (lane == 0) s_n = n;
    }
    __syncthreads();
    const int nl = s_n;
    if (threadIdx.x == 0) {
        *nlocal_kf = nl;
        *ref_kf = s_ref;   // NULL when nothing was counted
        w.ctl[LM_NL] = nl;
        s_carry = 0;
    }
    __syncthreads();
    // where each entry's row starts in the list's concatenated rows
    for (int b = 0; b < nl; b += blockDim.x) {
        const int t = b + threadIdx.x;
        const int c = t < nl ? counts[local_kf[t]] : 0;
        const int o = cv_block_scan(c, s_warp, &s_carry);
        if (t < nl) w.rowoff[t] = o;
    }
    if (threadIdx.x == 0) w.rowoff[nl] = s_carry;
}

// blocks stride over the list's entries: each point's first position in the concatenated rows
__global__ void __launch_bounds__(256) covis_lm_first_kernel(const int *__restrict__ kf_mp, const int *__restrict__ counts, int cap,
                                                             const unsigned char *__restrict__ point_bad, const int *__restrict__ local_kf,
                                                             LmScratch w) {
    if (w.ctl[LM_BAD]) return;
    const int nl = w.ctl[LM_NL];
    for (int t = blockIdx.x; t < nl; t += gridDim.x) {
        const int v = local_kf[t], c = counts[v], base = w.rowoff[t];
        const int *row = kf_mp + (size_t)v * cap;
        for (int i = threadIdx.x; i < c; i += blockDim.x) {
            const int p = row[i];
            if (p >= 0 && !point_bad[p]) atomicMin(&w.first[p], (unsigned)(base + i));
        }
    }
}

// the cell at position pos keeps its point when it is the point's first position (so the point is not bad)
__device__ __forceinline__ bool lm_keep(int p, int pos, const LmScratch &w) { return p >= 0 && w.first[p] == (unsigned)pos; }

__global__ void __launch_bounds__(COVIS_LM_BLOCK) covis_lm_keep_kernel(const int *__restrict__ kf_mp, const int *__restrict__ counts, int cap,
                                                                      const int *__restrict__ local_kf, LmScratch w) {
    __shared__ int s_warp[COVIS_LM_BLOCK / 32];
    if (w.ctl[LM_BAD]) return;
    const int nl = w.ctl[LM_NL];
    for (int t = blockIdx.x; t < nl; t += gridDim.x) {
        const int v = local_kf[t], c = counts[v], base = w.rowoff[t];
        const int *row = kf_mp + (size_t)v * cap;
        int k = 0;
        for (int i = threadIdx.x; i < c; i += blockDim.x) k += lm_keep(row[i], base + i, w);
        k = cull_block_sum(k, s_warp);
        if (threadIdx.x == 0) w.kcnt[t] = k;
    }
}

__global__ void __launch_bounds__(COVIS_LM_BLOCK) covis_lm_scatter_kernel(const int *__restrict__ kf_mp, const int *__restrict__ counts,
                                                                         int cap, const int *__restrict__ local_kf,
                                                                         int *__restrict__ local_points, int *__restrict__ nlocal_points,
                                                                         LmScratch w) {
    __shared__ int s_warp[32], s_carry;
    if (w.ctl[LM_BAD]) return;
    const int nl = w.ctl[LM_NL];
    if (nl == 0 && blockIdx.x == 0 && threadIdx.x == 0) *nlocal_points = 0;
    for (int t = blockIdx.x; t < nl; t += gridDim.x) {
        int before = 0;
        for (int x = threadIdx.x; x < t; x += blockDim.x) before += w.kcnt[x];
        before = cull_block_sum(before, s_warp);
        if (threadIdx.x == 0) s_carry = before;
        __syncthreads();
        const int v = local_kf[t], c = counts[v], base = w.rowoff[t];
        const int *row = kf_mp + (size_t)v * cap;
        for (int b = 0; b < c; b += blockDim.x) {
            const int i = b + threadIdx.x;
            const int p = i < c ? row[i] : -1;
            const bool keep = i < c && lm_keep(p, base + i, w);
            const int at = cv_block_scan(keep, s_warp, &s_carry);
            if (keep) local_points[at] = p;
        }
        if (t == nl - 1 && threadIdx.x == 0) *nlocal_points = s_carry;
        __syncthreads();
    }
}

}  // namespace orbfe

using namespace orbfe;

struct OrbfeCovisGraph {
    int K = 0, C = 0, Cp = 1, P = 2, B = 0, Bp = 1, apply_grid = 1, obs_grid = 1;
    size_t count_smem = 0, apply_smem = 0, erase_smem = 0;
    // host mirror of what only the synchronous calls change
    std::vector<uint8_t> live, id0;
    std::vector<unsigned long long> keys;
    std::unordered_set<unsigned long long> live_keys;
    HandleStream hs;
    DeviceBuffers mem;   // every device array below
    // device
    unsigned long long *key = nullptr;
    int *state = nullptr, *wn = nullptr, *wslot = nullptr, *ww = nullptr, *on = nullptr, *oslot = nullptr, *ow = nullptr, *named = nullptr;
    int *slots = nullptr, *pos = nullptr, *tmark = nullptr, *evcnt = nullptr, *efill = nullptr, *ebase = nullptr, *touched = nullptr;
    int *cn = nullptr, *cslot = nullptr, *cw = nullptr, *fn = nullptr, *fslot = nullptr, *fw = nullptr, *ev_p = nullptr, *ev_w = nullptr;
    int *flags = nullptr;
};

extern "C" void orbfe_covis_destroy(OrbfeCovisGraph *g) {
    if (!g) return;
    cudaSetDevice(g->hs.device);
    if (g->hs.stream) cudaStreamSynchronize(g->hs.stream);
    g->mem.release();
    g->hs.destroy();
    delete g;
}

// every slot empty; the batch scratch in its between-batches state
static int covis_reset(OrbfeCovisGraph *g, cudaStream_t s) {
    const size_t K = (size_t)g->K;
    ORBFE_CUDA_TRY(cudaMemsetAsync(g->state, 0, sizeof(int) * K, s));
    ORBFE_CUDA_TRY(cudaMemsetAsync(g->wn, 0, sizeof(int) * K, s));
    ORBFE_CUDA_TRY(cudaMemsetAsync(g->on, 0, sizeof(int) * K, s));
    ORBFE_CUDA_TRY(cudaMemsetAsync(g->named, 0, sizeof(int) * K, s));
    ORBFE_CUDA_TRY(cudaMemsetAsync(g->pos, 0xFF, sizeof(int) * K, s));
    ORBFE_CUDA_TRY(cudaMemsetAsync(g->tmark, 0, sizeof(int) * K, s));
    ORBFE_CUDA_TRY(cudaMemsetAsync(g->evcnt, 0, sizeof(int) * K, s));
    ORBFE_CUDA_TRY(cudaMemsetAsync(g->efill, 0, sizeof(int) * K, s));
    g->live.assign(K, 0);
    g->id0.assign(K, 0);
    g->keys.assign(K, 0);
    g->live_keys.clear();
    return ORBFE_OK;
}

extern "C" int orbfe_covis_create(int device, int max_keyframes, int max_connections, int max_batch, OrbfeCovisGraph **out) {
    if (!out) return set_error(ORBFE_ERR_ARG, "orbfe_covis_create: NULL out");
    *out = nullptr;
    if (device < 0 || max_keyframes < 1 || max_keyframes > (1 << 24) || max_connections < 1 || max_connections > COVIS_MAX_CONN ||
        max_batch < 1 || max_batch > COVIS_MAX_BATCH)
        return set_error(ORBFE_ERR_ARG, "orbfe_covis_create: bad arguments (device >= 0, 1 <= max_keyframes <= 2^24, 1 <= max_connections <= %d, "
                         "1 <= max_batch <= %d)", COVIS_MAX_CONN, COVIS_MAX_BATCH);
    if ((long long)max_keyframes * max_connections >= (1LL << 31) || (long long)max_batch * max_connections >= (1LL << 31))
        return set_error(ORBFE_ERR_ARG, "orbfe_covis_create: max_keyframes * max_connections must be < 2^31");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device >= ndev) {
        cudaGetLastError();
        return set_error(ORBFE_ERR_NO_DEVICE, "orbfe_covis_create: no CUDA device %d", device);
    }
    OrbfeCovisGraph *g = new OrbfeCovisGraph();
    g->K = max_keyframes;
    g->C = max_connections;
    g->Cp = pow2ge(max_connections);
    g->P = 2 * g->Cp;
    g->B = max_batch;
    g->Bp = pow2ge(max_batch);
    g->count_smem = sizeof(CvEnt) * (size_t)g->Cp + 2 * sizeof(int) * (size_t)g->P;
    g->apply_smem = sizeof(CvEnt) * (2 * (size_t)g->Cp + (size_t)g->Bp);
    g->erase_smem = sizeof(CvEnt) * (size_t)g->Cp;
    const size_t K = (size_t)g->K, KC = K * g->C, BC = (size_t)g->B * g->C;
    bool ok = g->hs.create(device) == cudaSuccess;
    int nsm = 1;
    ok = ok && cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device) == cudaSuccess;
    g->apply_grid = std::max(1, std::min(g->K, 4 * nsm));
    g->obs_grid = 8 * nsm;
    ok = ok && cudaFuncSetAttribute(covis_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g->count_smem) == cudaSuccess &&
         cudaFuncSetAttribute(covis_apply_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g->apply_smem) == cudaSuccess &&
         cudaFuncSetAttribute(covis_erase_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g->erase_smem) == cudaSuccess;
    const int obs_smem = (int)(sizeof(int2) * (size_t)pow2ge(2 * COVIS_OBS_MAX_CAP));
    ok = ok && cudaFuncSetAttribute(covis_obs_rows_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, obs_smem) == cudaSuccess &&
         cudaFuncSetAttribute(covis_obs_rows_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, obs_smem) == cudaSuccess &&
         cudaFuncSetAttribute(covis_lm_vote_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, obs_smem / 2) == cudaSuccess;
    const auto alloc = [&](auto **p, size_t n) { ok = ok && g->mem.alloc(p, n) == cudaSuccess; };
    alloc(&g->key, K); alloc(&g->state, K); alloc(&g->wn, K); alloc(&g->on, K); alloc(&g->named, K);
    alloc(&g->wslot, KC); alloc(&g->ww, KC); alloc(&g->oslot, KC); alloc(&g->ow, KC);
    // add stages 4 ints per keyframe; batches and lists name at most K slots
    alloc(&g->slots, 4 * K); alloc(&g->pos, K); alloc(&g->tmark, K); alloc(&g->evcnt, K);
    alloc(&g->efill, K); alloc(&g->ebase, K); alloc(&g->touched, K);
    alloc(&g->cn, (size_t)g->B); alloc(&g->fn, (size_t)g->B); alloc(&g->cslot, BC); alloc(&g->cw, BC);
    alloc(&g->fslot, BC); alloc(&g->fw, BC); alloc(&g->ev_p, BC); alloc(&g->ev_w, BC);
    alloc(&g->flags, (size_t)F_COUNT);
    ok = ok && cudaMemset(g->flags, 0, sizeof(int) * F_COUNT) == cudaSuccess && cudaMemset(g->key, 0, sizeof(unsigned long long) * K) == cudaSuccess;
    if (!ok) {
        const int rc = set_error(ORBFE_ERR_CUDA, "orbfe_covis_create: allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
        orbfe_covis_destroy(g);
        return rc;
    }
    int rc = covis_reset(g, g->hs.stream);
    if (!rc && cudaStreamSynchronize(g->hs.stream) != cudaSuccess) rc = set_error(ORBFE_ERR_CUDA, "orbfe_covis_create: reset failed");
    if (rc) { orbfe_covis_destroy(g); return rc; }
    *out = g;
    return ORBFE_OK;
}

extern "C" int orbfe_covis_add(OrbfeCovisGraph *g, int n, const int32_t *slots, const int32_t *ids, const uint64_t *keys) {
    if (!g || n < 0 || (n > 0 && (!slots || !ids || !keys))) return set_error(ORBFE_ERR_ARG, "orbfe_covis_add: bad arguments");
    for (int i = 0; i < n; i++)
        if (slots[i] < 0) return set_error(ORBFE_ERR_ARG, "orbfe_covis_add: negative slot");
    if (n == 0) return ORBFE_OK;
    if (n > g->K) return set_error(ORBFE_ERR_ARG, "orbfe_covis_add: more keyframes than slots");
    std::unordered_set<int> seen;
    std::unordered_set<unsigned long long> new_keys;
    for (int i = 0; i < n; i++) {
        const int s = slots[i];
        if (s < 0 || s >= g->K) return set_error(ORBFE_ERR_ARG, "orbfe_covis_add: slot %d out of range (max_keyframes %d)", s, g->K);
        if (g->live[s]) return set_error(ORBFE_ERR_ARG, "orbfe_covis_add: slot %d is live", s);
        if (!seen.insert(s).second) return set_error(ORBFE_ERR_ARG, "orbfe_covis_add: slot %d listed twice", s);
        if (g->live_keys.count(keys[i]) || !new_keys.insert(keys[i]).second)
            return set_error(ORBFE_ERR_ARG, "orbfe_covis_add: key of slot %d equals a live keyframe's key", s);
    }
    cudaStream_t st = g->hs.stream;
    int rc = g->hs.enter(st);
    if (rc) return rc;
    // a retired slot that a weight map still names is the reference's stale pointer: it cannot become a new keyframe
    std::vector<int> named((size_t)g->K);
    ORBFE_CUDA_TRY(cudaMemcpyAsync(named.data(), g->named, sizeof(int) * named.size(), cudaMemcpyDeviceToHost, st));
    ORBFE_CUDA_TRY(cudaStreamSynchronize(st));
    for (int i = 0; i < n; i++)
        if (named[slots[i]] != 0)
            return set_error(ORBFE_ERR_ARG, "orbfe_covis_add: retired slot %d is still named by %d weight maps", slots[i], named[slots[i]]);
    std::vector<int> rows(4 * (size_t)n);
    for (int i = 0; i < n; i++) {
        rows[4 * i] = slots[i];
        rows[4 * i + 1] = ids[i] == 0;
        rows[4 * i + 2] = (int)(uint32_t)keys[i];
        rows[4 * i + 3] = (int)(uint32_t)(keys[i] >> 32);
    }
    ORBFE_CUDA_TRY(cudaMemcpyAsync(g->slots, rows.data(), sizeof(int) * rows.size(), cudaMemcpyHostToDevice, st));
    covis_add_kernel<<<(n + 127) / 128, 128, 0, st>>>(n, g->slots, g->key, g->state, g->wn, g->on);
    if ((rc = g->hs.leave(st, true))) return rc;
    for (int i = 0; i < n; i++) {
        g->live[slots[i]] = 1;
        g->id0[slots[i]] = ids[i] == 0;
        g->keys[slots[i]] = keys[i];
        g->live_keys.insert(keys[i]);
    }
    return ORBFE_OK;
}

extern "C" int orbfe_covis_update_connections_device(OrbfeCovisGraph *g, int n, const int32_t *slots, const int32_t *d_kf_mp,
                                                     const int *d_counts, int nframes, int cap, const int32_t *d_group_ptr,
                                                     const int32_t *d_obs, int npoints, int nobs, int32_t *parent_out, void *stream) {
    if (!g || n < 0 || nframes < 1 || cap < 1 || npoints < 0 || nobs < 0 || (long long)nframes * cap >= (1LL << 31))
        return set_error(ORBFE_ERR_ARG, "orbfe_covis_update_connections_device: bad arguments (n >= 0, nframes >= 1, cap >= 1, "
                         "nframes*cap < 2^31, npoints >= 0, nobs >= 0)");
    if (n > 0 && (!slots || !d_kf_mp || !d_counts || !d_group_ptr || (nobs > 0 && !d_obs)))
        return set_error(ORBFE_ERR_ARG, "orbfe_covis_update_connections_device: NULL argument");
    std::unordered_set<int> seen;
    for (int i = 0; i < n; i++) {
        const int s = slots[i];
        if (s < 0 || s >= nframes) return set_error(ORBFE_ERR_ARG, "orbfe_covis_update_connections_device: slot %d outside [0, nframes)", s);
        if (!seen.insert(s).second) return set_error(ORBFE_ERR_ARG, "orbfe_covis_update_connections_device: slot %d listed twice", s);
    }
    if (n == 0) return ORBFE_OK;
    if (n > g->B) return set_error(ORBFE_ERR_ARG, "orbfe_covis_update_connections_device: n %d > max_batch %d", n, g->B);
    for (int i = 0; i < n; i++)
        if (slots[i] >= g->K || !g->live[slots[i]])
            return set_error(ORBFE_ERR_ARG, "orbfe_covis_update_connections_device: slot %d is not a live keyframe", slots[i]);
    cudaStream_t st = g->hs.pick(stream);
    int rc = g->hs.enter(st);
    if (rc) return rc;
    ORBFE_CUDA_TRY(cudaMemcpyAsync(g->slots, slots, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, st));
    covis_count_kernel<<<n, COVIS_COUNT_BLOCK, g->count_smem, st>>>(g->slots, g->C, g->Cp, g->P, d_kf_mp, d_counts, nframes, cap,
                                                                  d_group_ptr, d_obs, npoints, nobs, g->K, g->state, g->key, g->cn, g->cslot,
                                                                  g->cw, g->fn, g->fslot, g->fw, g->flags);
    covis_plan_kernel<<<1, 1024, 0, st>>>(n, g->slots, g->C, g->cn, g->cslot, g->fn, g->fslot, g->fw, g->state, g->key, g->wn, g->wslot,
                                          g->pos, g->tmark, g->evcnt, g->efill, g->ebase, g->touched, g->ev_p, g->ev_w, parent_out, g->flags);
    covis_apply_kernel<<<g->apply_grid, COVIS_APPLY_BLOCK, g->apply_smem, st>>>(
        g->slots, g->C, g->Cp, g->Bp, g->cn, g->cslot, g->cw, g->fn, g->fslot, g->fw, g->key, g->state, g->wn, g->wslot, g->ww, g->on,
        g->oslot, g->ow, g->named, g->pos, g->tmark, g->evcnt, g->efill, g->ebase, g->touched, g->ev_p, g->ev_w, g->flags);
    return g->hs.leave(st, false);
}

extern "C" int orbfe_covis_erase(OrbfeCovisGraph *g, int slot) {
    if (!g || slot < 0 || slot >= g->K) return set_error(ORBFE_ERR_ARG, "orbfe_covis_erase: bad arguments");
    if (!g->live[slot] || g->id0[slot]) return ORBFE_OK;   // SetBadFlag of mnId == 0 returns at once (KeyFrame.cc:501)
    cudaStream_t st = g->hs.stream;
    int rc = g->hs.enter(st);
    if (rc) return rc;
    covis_erase_kernel<<<g->C, COVIS_APPLY_BLOCK, g->erase_smem, st>>>(slot, g->C, g->key, g->wn, g->wslot, g->ww, g->on, g->oslot, g->ow,
                                                                      g->named);
    covis_retire_kernel<<<1, 1, 0, st>>>(slot, g->state, g->wn, g->on);
    if ((rc = g->hs.leave(st, true))) return rc;
    g->live[slot] = 0;
    g->live_keys.erase(g->keys[slot]);
    return ORBFE_OK;
}

extern "C" int orbfe_covis_clear(OrbfeCovisGraph *g) {
    if (!g) return set_error(ORBFE_ERR_ARG, "orbfe_covis_clear: bad arguments");
    int rc = g->hs.enter(g->hs.stream);
    if (rc) return rc;
    if ((rc = covis_reset(g, g->hs.stream))) return rc;
    return g->hs.leave(g->hs.stream, true);
}

extern "C" int orbfe_covis_lists_device(OrbfeCovisGraph *g, int which, int n, const int32_t *slots, int nbest, int32_t *d_ptr,
                                        int32_t *d_list, int32_t *d_weights, void *stream) {
    if (!g || (which != 0 && which != 1) || n < 0 || (n > 0 && (!slots || !d_ptr || !d_list)))
        return set_error(ORBFE_ERR_ARG, "orbfe_covis_lists_device: bad arguments (which 0 or 1, n >= 0, slots / d_ptr / d_list non-NULL)");
    for (int i = 0; i < n; i++)
        if (slots[i] < 0) return set_error(ORBFE_ERR_ARG, "orbfe_covis_lists_device: negative slot");
    if (n == 0) return ORBFE_OK;
    if (n > g->K) return set_error(ORBFE_ERR_ARG, "orbfe_covis_lists_device: more rows than slots");
    for (int i = 0; i < n; i++)
        if (slots[i] >= g->K) return set_error(ORBFE_ERR_ARG, "orbfe_covis_lists_device: slot %d out of range", slots[i]);
    const int limit = which == 0 && nbest > 0 ? std::min(nbest, g->C) : g->C;
    cudaStream_t st = g->hs.pick(stream);
    int rc = g->hs.enter(st);
    if (rc) return rc;
    ORBFE_CUDA_TRY(cudaMemcpyAsync(g->slots, slots, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, st));
    covis_lens_kernel<<<1, 1024, 0, st>>>(n, g->slots, which, limit, g->wn, g->on, d_ptr);
    covis_lists_kernel<<<n, 128, 0, st>>>(g->slots, which, g->C, d_ptr, g->wslot, g->ww, g->oslot, g->ow, g->state, d_list, d_weights);
    return g->hs.leave(st, false);
}

extern "C" int orbfe_covis_observations_device(OrbfeCovisGraph *g, int n, const int32_t *d_points, int npoints, const int32_t *d_kf_mp,
                                               const int *d_counts, int nframes, int cap, const int32_t *d_ref_slot, int obs_cap,
                                               int32_t *d_ptr, int32_t *d_obs, int *d_nobs, int32_t *d_ref_obs, void *d_scratch, void *stream) {
    if (!g || n < 0 || npoints < 0 || n > npoints || nframes < 1 || cap < 1 || obs_cap < 0 || (long long)nframes * cap >= (1LL << 31))
        return set_error(ORBFE_ERR_ARG, "orbfe_covis_observations_device: bad arguments (0 <= n <= npoints, nframes >= 1, cap >= 1, "
                         "nframes*cap < 2^31, obs_cap >= 0)");
    if (!d_kf_mp || !d_counts || !d_ptr || !d_nobs || !d_scratch || (n > 0 && !d_points) || (obs_cap > 0 && !d_obs) ||
        (n > 0 && (d_ref_slot == nullptr) != (d_ref_obs == nullptr)))
        return set_error(ORBFE_ERR_ARG, "orbfe_covis_observations_device: NULL argument (d_ref_slot and d_ref_obs go together when n > 0)");
    if ((uintptr_t)d_scratch % alignof(int) != 0)
        return set_error(ORBFE_ERR_ARG, "orbfe_covis_observations_device: d_scratch is not 4-byte aligned");
    if (cap > COVIS_OBS_MAX_CAP)
        return set_error(ORBFE_ERR_UNSUPPORTED, "orbfe_covis_observations_device: cap %d > %d", cap, COVIS_OBS_MAX_CAP);
    for (int s = nframes; s < g->K; s++)
        if (g->live[s]) return set_error(ORBFE_ERR_ARG, "orbfe_covis_observations_device: live slot %d >= nframes %d", s, nframes);
    cudaStream_t st = g->hs.pick(stream);
    int rc = g->hs.enter(st);
    if (rc) return rc;
    int *stamp = static_cast<int *>(d_scratch), *cnt = stamp + npoints, *tmp = cnt + npoints;
    const int nslots = std::min(g->K, nframes), T = pow2ge(2 * cap);
    const int rows_grid = std::min(nslots, 4 * g->obs_grid);
    const size_t smem = sizeof(int2) * (size_t)T;
    const int W = COVIS_OBS_SORT_BLOCK / 32;
    covis_obs_stamp_kernel<<<std::max(1, std::min((n + 255) / 256, g->obs_grid)), 256, 0, st>>>(n, d_points, npoints, stamp, cnt, g->flags);
    covis_obs_rows_kernel<false><<<rows_grid, COVIS_OBS_BLOCK, smem, st>>>(nslots, T, g->state, d_kf_mp, d_counts, cap, npoints, n, d_points,
                                                                            stamp, cnt, d_ptr, tmp, g->flags);
    covis_obs_scan_kernel<<<1, 1024, 0, st>>>(n, cnt, d_ref_slot, nframes, obs_cap, d_ptr, d_nobs, g->flags);
    covis_obs_rows_kernel<true><<<rows_grid, COVIS_OBS_BLOCK, smem, st>>>(nslots, T, g->state, d_kf_mp, d_counts, cap, npoints, n, d_points,
                                                                           stamp, cnt, d_ptr, tmp, g->flags);
    covis_obs_sort_kernel<<<std::max(1, std::min((n + W - 1) / W, g->obs_grid)), COVIS_OBS_SORT_BLOCK, 0, st>>>(
        n, cap, g->key, d_ptr, tmp, d_ref_slot, d_obs, d_ref_obs, g->flags);
    return g->hs.leave(st, false);
}

extern "C" int orbfe_covis_keyframe_culling_device(OrbfeCovisGraph *g, int current_slot, int32_t *d_kf_mp, const int *d_counts,
                                                   const OrbfeKeyPoint *d_kps, int nframes, int cap, uint8_t *d_point_bad,
                                                   int32_t *d_ref_slot, int npoints, int n_not_erase, const int32_t *not_erase_slots,
                                                   int obs_cap, int *d_nobs, int32_t *d_verdict_slot, int32_t *d_verdict, int *d_ncand,
                                                   int32_t *d_nmps, int32_t *d_nredundant, int32_t *d_bad_points, int *d_nbad,
                                                   void *d_scratch, void *stream) {
    static const char *fn = "orbfe_covis_keyframe_culling_device";
    if (!g || npoints < 0 || nframes < 1 || cap < 1 || obs_cap < 0 || n_not_erase < 0 || (long long)nframes * cap >= (1LL << 31))
        return set_error(ORBFE_ERR_ARG, "%s: bad arguments (npoints >= 0, nframes >= 1, cap >= 1, nframes*cap < 2^31, obs_cap >= 0, "
                         "n_not_erase >= 0)", fn);
    if (!d_kf_mp || !d_counts || !d_kps || !d_nobs || !d_verdict_slot || !d_verdict || !d_ncand || !d_nbad || !d_scratch ||
        (npoints > 0 && (!d_point_bad || !d_ref_slot || !d_bad_points)) || (n_not_erase > 0 && !not_erase_slots))
        return set_error(ORBFE_ERR_ARG, "%s: NULL argument", fn);
    if ((uintptr_t)d_scratch % alignof(int) != 0) return set_error(ORBFE_ERR_ARG, "%s: d_scratch is not 4-byte aligned", fn);
    if (cap > COVIS_OBS_MAX_CAP) return set_error(ORBFE_ERR_UNSUPPORTED, "%s: cap %d > %d", fn, cap, COVIS_OBS_MAX_CAP);
    if (current_slot < 0 || current_slot >= g->K || current_slot >= nframes || !g->live[current_slot])
        return set_error(ORBFE_ERR_ARG, "%s: current slot %d is not a live keyframe below nframes", fn, current_slot);
    if (n_not_erase > g->K) return set_error(ORBFE_ERR_ARG, "%s: n_not_erase %d > max_keyframes %d", fn, n_not_erase, g->K);
    for (int j = 0; j < n_not_erase; j++)
        if (not_erase_slots[j] < 0 || not_erase_slots[j] >= nframes)
            return set_error(ORBFE_ERR_ARG, "%s: mbNotErase slot %d outside [0, nframes)", fn, not_erase_slots[j]);
    for (int s = nframes; s < g->K; s++)
        if (g->live[s]) return set_error(ORBFE_ERR_ARG, "%s: live slot %d >= nframes %d", fn, s, nframes);
    cudaStream_t st = g->hs.pick(stream);
    int rc = g->hs.enter(st);
    if (rc) return rc;
    const size_t np = (size_t)npoints, nf = (size_t)nframes;
    CullScratch w;
    w.stamp = static_cast<int *>(d_scratch);
    w.cnt = w.stamp + np;
    w.tmp = w.cnt + np;
    w.pts = w.tmp + obs_cap;
    w.ptr = w.pts + np;
    w.obs = w.ptr + np + 1;
    w.lcnt = w.obs + obs_cap;
    w.bad_at = w.lcnt + np;
    w.gone_at = w.bad_at + np;
    w.ne = w.gone_at + nf;
    w.ctl = w.ne + nf;
    w.alive = reinterpret_cast<unsigned char *>(w.ctl + CTL_COUNT);
    ORBFE_CUDA_TRY(cudaMemsetAsync(w.bad_at, 0x7F, sizeof(int) * np, st));
    ORBFE_CUDA_TRY(cudaMemsetAsync(w.gone_at, 0x7F, sizeof(int) * nf, st));
    ORBFE_CUDA_TRY(cudaMemsetAsync(w.ne, 0, sizeof(int) * (nf + CTL_COUNT), st));
    if (n_not_erase > 0)
        ORBFE_CUDA_TRY(cudaMemcpyAsync(g->slots, not_erase_slots, sizeof(int) * (size_t)n_not_erase, cudaMemcpyHostToDevice, st));
    const int T = pow2ge(2 * cap), nslots = std::min(g->K, nframes), rows_grid = std::min(nslots, 4 * g->obs_grid);
    const size_t smem = sizeof(int2) * (size_t)T;
    const int W = COVIS_OBS_SORT_BLOCK / 32;
    covis_cull_prep_kernel<<<g->obs_grid, 256, 0, st>>>(npoints, n_not_erase, g->slots, w, g->flags);
    // every point's observation list: the launches of orbfe_covis_observations_device over the points 0 .. npoints-1
    covis_obs_stamp_kernel<<<std::max(1, std::min((npoints + 255) / 256, g->obs_grid)), 256, 0, st>>>(npoints, w.pts, npoints, w.stamp, w.cnt,
                                                                                                       g->flags);
    covis_obs_rows_kernel<false><<<rows_grid, COVIS_OBS_BLOCK, smem, st>>>(nslots, T, g->state, d_kf_mp, d_counts, cap, npoints, npoints,
                                                                            w.pts, w.stamp, w.cnt, w.ptr, w.tmp, g->flags);
    covis_obs_scan_kernel<<<1, 1024, 0, st>>>(npoints, w.cnt, nullptr, nframes, obs_cap, w.ptr, d_nobs, g->flags);
    covis_obs_rows_kernel<true><<<rows_grid, COVIS_OBS_BLOCK, smem, st>>>(nslots, T, g->state, d_kf_mp, d_counts, cap, npoints, npoints,
                                                                           w.pts, w.stamp, w.cnt, w.ptr, w.tmp, g->flags);
    covis_obs_sort_kernel<<<std::max(1, std::min((npoints + W - 1) / W, g->obs_grid)), COVIS_OBS_SORT_BLOCK, 0, st>>>(
        npoints, cap, g->key, w.ptr, w.tmp, nullptr, w.obs, nullptr, g->flags);
    covis_cull_check_kernel<<<g->C, COVIS_CULL_CHECK_BLOCK, 0, st>>>(current_slot, g->C, g->on, g->oslot, d_kf_mp, d_counts, d_kps, nframes,
                                                                    cap, d_point_bad, d_ref_slot, npoints, w, g->flags);
    covis_cull_kernel<<<1, COVIS_CULL_BLOCK, 0, st>>>(current_slot, g->C, g->on, g->oslot, g->state, g->key, d_kf_mp, d_counts, d_kps, cap,
                                                      d_point_bad, d_ref_slot, npoints, d_verdict_slot, d_verdict, d_ncand, d_nmps,
                                                      d_nredundant, d_bad_points, d_nbad, w, g->flags);
    covis_cull_null_kernel<<<rows_grid, 256, 0, st>>>(nslots, g->state, d_kf_mp, d_counts, cap, w, g->flags);
    return g->hs.leave(st, false);
}

extern "C" int orbfe_covis_local_map_device(OrbfeCovisGraph *g, int nf, int32_t *d_frame_mp, const uint8_t *d_point_bad, int npoints,
                                            const int32_t *d_kf_mp, const int *d_counts, int nframes, int cap, int32_t *d_local_kf,
                                            int *d_nlocal_kf, int32_t *d_ref_kf, int32_t *d_local_points, int *d_nlocal_points,
                                            void *d_scratch, void *stream) {
    static const char *fn = "orbfe_covis_local_map_device";
    if (!g || nf < 0 || npoints < 0 || nframes < 1 || cap < 1 || (long long)nframes * cap >= (1LL << 31))
        return set_error(ORBFE_ERR_ARG, "%s: bad arguments (nf >= 0, npoints >= 0, nframes >= 1, cap >= 1, nframes*cap < 2^31)", fn);
    if (!d_kf_mp || !d_counts || !d_local_kf || !d_nlocal_kf || !d_ref_kf || !d_nlocal_points || !d_scratch || (nf > 0 && !d_frame_mp) ||
        (npoints > 0 && (!d_point_bad || !d_local_points)))
        return set_error(ORBFE_ERR_ARG, "%s: NULL argument", fn);
    if ((uintptr_t)d_scratch % alignof(int) != 0) return set_error(ORBFE_ERR_ARG, "%s: d_scratch is not 4-byte aligned", fn);
    if (cap > COVIS_OBS_MAX_CAP) return set_error(ORBFE_ERR_UNSUPPORTED, "%s: cap %d > %d", fn, cap, COVIS_OBS_MAX_CAP);
    for (int s = nframes; s < g->K; s++)
        if (g->live[s]) return set_error(ORBFE_ERR_ARG, "%s: live slot %d >= nframes %d", fn, s, nframes);
    cudaStream_t st = g->hs.pick(stream);
    int rc = g->hs.enter(st);
    if (rc) return rc;
    const size_t np = (size_t)npoints, nfr = (size_t)nframes;
    LmScratch w;
    w.mult = static_cast<int *>(d_scratch);
    w.ctl = w.mult + np;
    w.first = reinterpret_cast<unsigned *>(w.ctl + LM_CTL);
    w.cnt = reinterpret_cast<int *>(w.first + np);
    w.cand = w.cnt + nfr;
    w.rowoff = w.cand + nfr;
    w.kcnt = w.rowoff + nfr + 1;
    ORBFE_CUDA_TRY(cudaMemsetAsync(w.mult, 0, sizeof(int) * (np + LM_CTL), st));
    ORBFE_CUDA_TRY(cudaMemsetAsync(w.first, 0xFF, sizeof(unsigned) * np, st));
    const int nslots = std::min(g->K, nframes), T = pow2ge(2 * cap), grid = std::max(1, std::min(nslots, 4 * g->obs_grid));
    covis_lm_frame_kernel<<<std::max(1, std::min((nf + 255) / 256, g->obs_grid)), 256, 0, st>>>(nf, d_frame_mp, d_point_bad, npoints, w);
    covis_lm_vote_kernel<<<grid, COVIS_LM_VOTE_BLOCK, sizeof(int) * (size_t)T, st>>>(nslots, T, g->state, d_kf_mp, d_counts, cap, npoints, w);
    covis_lm_list_kernel<<<1, COVIS_LM_BLOCK, 0, st>>>(nslots, g->C, g->on, g->oslot, g->state, g->key, d_counts, nf, d_frame_mp, d_point_bad,
                                                       d_local_kf, d_nlocal_kf, d_ref_kf, w, g->flags);
    covis_lm_first_kernel<<<grid, 256, 0, st>>>(d_kf_mp, d_counts, cap, d_point_bad, d_local_kf, w);
    covis_lm_keep_kernel<<<grid, COVIS_LM_BLOCK, 0, st>>>(d_kf_mp, d_counts, cap, d_local_kf, w);
    covis_lm_scatter_kernel<<<grid, COVIS_LM_BLOCK, 0, st>>>(d_kf_mp, d_counts, cap, d_local_kf, d_local_points, d_nlocal_points, w);
    return g->hs.leave(st, false);
}

extern "C" int orbfe_covis_sync(OrbfeCovisGraph *g) {
    if (!g) return set_error(ORBFE_ERR_ARG, "orbfe_covis_sync: bad arguments");
    cudaStream_t st = g->hs.stream;
    int rc = g->hs.enter(st);
    if (rc) return rc;
    int err = 0, src = 0;
    ORBFE_CUDA_TRY(cudaMemcpyAsync(&err, g->flags + F_ERR, sizeof(int), cudaMemcpyDeviceToHost, st));
    ORBFE_CUDA_TRY(cudaMemcpyAsync(&src, g->flags + F_ERR_SRC, sizeof(int), cudaMemcpyDeviceToHost, st));
    ORBFE_CUDA_TRY(cudaMemsetAsync(g->flags + F_ERR, 0, sizeof(int), st));
    ORBFE_CUDA_TRY(cudaMemsetAsync(g->flags + F_ERR_SRC, 0, sizeof(int), st));
    if ((rc = g->hs.leave(st, true))) return rc;
    if (src == 1 && err == ORBFE_ERR_ARG)
        return set_error(ORBFE_ERR_ARG, "orbfe_covis_sync: an observations call was rejected: a named point out of range or named "
                         "twice, a count outside 0 .. cap, a row value >= npoints or a reference slot outside [0, nframes)");
    if (src == 1 && err == ORBFE_ERR_CAPACITY)
        return set_error(ORBFE_ERR_CAPACITY, "orbfe_covis_sync: an observations call needed more than obs_cap entries");
    if (src == 2 && err == ORBFE_ERR_ARG)
        return set_error(ORBFE_ERR_ARG, "orbfe_covis_sync: a keyframe culling call was rejected: a count outside 0 .. cap, a row value >= "
                         "npoints, a listed slot >= nframes, an octave outside 0 .. %d or a reference slot outside [0, nframes)",
                         ORBFE_MAX_LEVELS - 1);
    if (src == 2 && err == ORBFE_ERR_CAPACITY)
        return set_error(ORBFE_ERR_CAPACITY, "orbfe_covis_sync: a keyframe culling call needed more than obs_cap observation entries");
    if (src == 3 && err == ORBFE_ERR_ARG)
        return set_error(ORBFE_ERR_ARG, "orbfe_covis_sync: a local map call was rejected: a frame cell or row value >= npoints, or a "
                         "live slot's count outside 0 .. cap");
    if (err == ORBFE_ERR_ARG)
        return set_error(ORBFE_ERR_ARG, "orbfe_covis_sync: an update batch was rejected: a point index, group pointer or observation was "
                         "out of range or named a slot that is not live");
    if (err == ORBFE_ERR_CAPACITY)
        return set_error(ORBFE_ERR_CAPACITY, "orbfe_covis_sync: an update batch was rejected: a weight map would exceed max_connections");
    return err;
}
