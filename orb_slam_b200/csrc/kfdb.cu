// kfdb.cu -- KeyFrameDatabase (reference src/KeyFrameDatabase.cc) resident in device memory: add / erase / clear and the
// two candidate queries, with the keyframes' query fields (KeyFrame.h:160-165) kept per slot on the device.  C-ABI in
// include/orbfe_bow.h.
//
// Layout (all allocated by orbfe_kfdb_create):
//   store    the BowVector of every keyframe, contiguous per slot (word id, value, inverted-file node of that word);
//            rows are appended, erase leaves a hole, and add compacts the live rows into the second half of a double
//            buffer when the tail is full but the holes are not.
//   nodes    one node per posting: the inverted file is a doubly linked list per word (head / tail per word, nodes in
//            push_back order = add order), so add appends and erase unlinks without touching the rest of the list.  Free
//            node indices are a stack on the host (allocation only; the lists themselves live on the device).
//   slots    (begin, end) of the slot's store rows, add sequence number, the packed query state (query id << 32 |
//            lowest shared-word rank << 16 | shared-word count: the device form of mnLoopQuery/mnRelocQuery and
//            mnLoopWords/mnRelocWords, updated by CAS so no per-query clearing is needed), mLoopScore / mRelocScore
//            (persistent: the relocalisation accumulation reads scores of earlier queries, :272-281), and the best
//            covisibility list (at most 10 slots, GetBestCovisibilityKeyFrames(10)).
//   rows     one row per query of a batch (max_queries rows, row b at b * max_keyframes, or b * sortcap for the sorted list):
//            the packed query state, the connected stamps, the touched and sorted lists, the scores the query computed
//            (`scored`: query id << 32 | float bits), the accumulations, the best covisibles and the first-entry tags.
//            Every row entry is keyed on the query id of its row, so no row is ever cleared.
// A batch of B queries (B = 1 for orbfe_kfdb_detect_device) gets B consecutive query ids and is six launches on one
// stream (five when B = 1: the score kernel then writes the scores back itself), no host synchronisation:
//   kfdb_begin_kernel     stamps each query keyframe's connected slots (loop mode) and resets the touched counters;
//   kfdb_walk_kernel      one thread per (query, word) walks that word's list: counts shared words, keeps the lowest shared
//                         word rank, and the first touch appends the slot to the query's touched list (lKFsSharingWords,
//                         unordered);
//   kfdb_order_kernel     one block per query: maxCommonWords over the touched slots, the threshold, and the qualifying
//                         slots sorted by (first shared word rank, add order) -- the order of lKFsSharingWords;
//   kfdb_score_kernel     one thread per (query, qualifying slot): the L1 score (bow_l1.cuh, the walk bow_db_score_kernel
//                         uses), recorded in the query's row (and, when B = 1, in the slot's persistent score);
//   kfdb_select_kernel    one block per query: covisibility accumulation and candidate selection in list order, and the
//                         outputs.  A score read of slot s by query b is the one the last query a <= b of the batch
//                         computed, else the persistent one: what B calls in order would have read;
//   kfdb_writeback_kernel the persistent mLoopScore / mRelocScore of every slot scored in the batch, from its last scorer,
//                         after every select has read the values from before the batch.
// Every order-dependent step works on the sorted list, so results do not depend on block scheduling.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/orbfe_bow.h"
#include "bow_l1.cuh"
#include "orbfe_internal.h"

namespace orbfe {
int vocab_device(const OrbfeVocabulary *v);
int vocab_nwords(const OrbfeVocabulary *v);

#define KFDB_COVIS 10
#define KFDB_BLOCK 1024

__global__ void kfdb_link_kernel(int slot, int base, int nw, unsigned seq, const int *__restrict__ s_id, const int *__restrict__ s_node,
                                 int *__restrict__ n_slot, int *__restrict__ n_next, int *__restrict__ n_prev, int *__restrict__ w_head,
                                 int *__restrict__ w_tail, int *__restrict__ range, unsigned *__restrict__ seqs,
                                 float *__restrict__ lscore, float *__restrict__ rscore) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) {   // a fresh KeyFrame: scores 0; its stamps are older query ids than any later query's, as 0 would be
        range[2 * slot] = base;
        range[2 * slot + 1] = base + nw;
        seqs[slot] = seq;
        lscore[slot] = 0.f;
        rscore[slot] = 0.f;
    }
    if (i >= nw) return;
    // the words of one keyframe are distinct: every thread appends to a different list (mvInvertedFile[w].push_back)
    const int w = s_id[base + i], nd = s_node[base + i];
    const int t = w_tail[w];
    n_slot[nd] = slot;
    n_next[nd] = -1;
    n_prev[nd] = t;
    if (t >= 0) n_next[t] = nd; else w_head[w] = nd;
    w_tail[w] = nd;
}

__global__ void kfdb_unlink_kernel(int slot, int base, int nw, const int *__restrict__ s_id, const int *__restrict__ s_node,
                                   int *__restrict__ n_next, int *__restrict__ n_prev, int *__restrict__ w_head, int *__restrict__ w_tail,
                                   int *__restrict__ range, int *__restrict__ covn) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) {
        range[2 * slot] = 0;
        range[2 * slot + 1] = -1;   // empty
        covn[slot] = 0;
    }
    if (i >= nw) return;
    // one node per list: the unlinks of one keyframe never touch the same node
    const int w = s_id[base + i], nd = s_node[base + i];
    const int p = n_prev[nd], n = n_next[nd];
    if (p >= 0) n_next[p] = n; else w_head[w] = n;
    if (n >= 0) n_prev[n] = p; else w_tail[w] = p;
}

// move the live rows of `nmove` slots (old begin, new begin, length) from one half of the store to the other
__global__ void kfdb_compact_kernel(const int *__restrict__ moves, int nmove, const int *__restrict__ id0, const double *__restrict__ val0,
                                    const int *__restrict__ node0, int *__restrict__ id1, double *__restrict__ val1, int *__restrict__ node1) {
    for (int m = blockIdx.x; m < nmove; m += gridDim.x) {
        const int ob = moves[3 * m], nb = moves[3 * m + 1], n = moves[3 * m + 2];
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            id1[nb + i] = id0[ob + i];
            val1[nb + i] = val0[ob + i];
            node1[nb + i] = node0[ob + i];
        }
    }
}

// orbfe_kfdb_add_device: one block per named row (frame frames[r] of the caller's BowVector rows) gathers its word count into
// info[1 + r] and raises info[0] when the count is outside [0, cap] or the ids are not strictly ascending in [0, nwords).
__global__ void kfdb_check_rows_kernel(const int *__restrict__ frames, int n, int cap, int nwords, const int *__restrict__ bow_n,
                                       const int *__restrict__ bow_ids, int *__restrict__ info) {
    for (int r = blockIdx.x; r < n; r += gridDim.x) {
        const size_t f = (size_t)frames[r];
        const int c = bow_n[f];
        if (threadIdx.x == 0) info[1 + r] = c;
        const int *row = bow_ids + f * (size_t)cap;
        bool bad = c < 0 || c > cap;
        if (!bad)
            for (int k = threadIdx.x; k < c; k += blockDim.x) {
                const int w = row[k];
                bad |= (unsigned)w >= (unsigned)nwords || (k > 0 && row[k - 1] >= w);
            }
        if (__syncthreads_or(bad) && threadIdx.x == 0) info[0] = 1;
    }
}

// copy the rows (frame, store begin, length) of `n` keyframes from the caller's BowVector rows into the store
__global__ void kfdb_gather_kernel(const int *__restrict__ rows, int n, int cap, const int *__restrict__ bow_ids,
                                   const double *__restrict__ bow_vals, int *__restrict__ id1, double *__restrict__ val1) {
    for (int m = blockIdx.x; m < n; m += gridDim.x) {
        const size_t src = (size_t)rows[3 * m] * (size_t)cap;
        const int nb = rows[3 * m + 1], len = rows[3 * m + 2];
        for (int i = threadIdx.x; i < len; i += blockDim.x) {
            id1[nb + i] = bow_ids[src + i];
            val1[nb + i] = bow_vals[src + i];
        }
    }
}

__global__ void kfdb_covis_kernel(const int *__restrict__ rows, int n, int *__restrict__ covn, int *__restrict__ cov) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int *r = rows + i * (2 + KFDB_COVIS);
    const int s = r[0], c = r[1];
    covn[s] = c;
    for (int j = 0; j < c; j++) cov[s * KFDB_COVIS + j] = r[2 + j];
}

// the device form: row i of the CSR lists (ptr[i] .. ptr[i+1]) for slot rows[i]; only its first 10 entries are read, and an
// entry outside [0, K) is kept in its place as -1
__global__ void kfdb_covis_device_kernel(const int *__restrict__ rows, int n, int K, const int *__restrict__ ptr,
                                         const int *__restrict__ lists, int *__restrict__ covn, int *__restrict__ cov) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = rows[i], lo = ptr[i];
    const int c = min(max(ptr[i + 1] - lo, 0), KFDB_COVIS);
    for (int j = 0; j < c; j++) {
        const int v = lists[lo + j];
        cov[s * KFDB_COVIS + j] = (unsigned)v < (unsigned)K ? v : -1;
    }
    covn[s] = c;
}

__device__ __forceinline__ unsigned q_stamp(unsigned long long st) { return (unsigned)(st >> 32); }
__device__ __forceinline__ int q_rank(unsigned long long st) { return (int)((st >> 16) & 0xFFFFu); }
__device__ __forceinline__ int q_words(unsigned long long st) { return (int)(st & 0xFFFFu); }

// The score of slot s as query b of the batch reads it: the one the last query a <= b of the batch computed (its
// mLoopScore / mRelocScore after query a), else the one left before the batch (KeyFrameDatabase.cc:272-281).
__device__ __forceinline__ float kfdb_score_read(int b, unsigned qid0, int s, int K, const unsigned long long *__restrict__ scored,
                                                 const float *__restrict__ sc) {
    const float before = sc[s];   // loaded with the first row's entry, not after the scan
    for (int a = b; a >= 0; a--) {
        const unsigned long long v = scored[(size_t)a * K + s];
        if ((unsigned)(v >> 32) == qid0 + (unsigned)a) return __uint_as_float((unsigned)v);
    }
    return before;
}

// grid (x, queries): query b stamps d_connected[conn_ptr[b] .. conn_ptr[b+1]) into its row; without conn_ptr (one query)
// the range is [0, nconn)
__global__ void kfdb_begin_kernel(int loop, unsigned qid0, const int *__restrict__ conn_ptr, const int *__restrict__ connected, int nconn,
                                  int K, unsigned *__restrict__ conn, int *__restrict__ info) {
    const int b = blockIdx.y;
    if (blockIdx.x == 0 && threadIdx.x == 0) info[4 * b] = 0;   // touched count
    if (!loop || !connected) return;
    const int lo = conn_ptr ? conn_ptr[b] : 0, hi = conn_ptr ? conn_ptr[b + 1] : nconn;
    unsigned *cb = conn + (size_t)b * K;
    for (int i = lo + blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += gridDim.x * blockDim.x) {
        const int c = connected[i];
        if ((unsigned)c < (unsigned)K) cb[c] = qid0 + b;
    }
}

// grid (words, queries): query b's words are q_ids[b * qcap .. b * qcap + qcap)
__global__ void __launch_bounds__(128) kfdb_walk_kernel(unsigned qid0, int nq, const int *__restrict__ q_ids, int nwords,
                                                        const int *__restrict__ w_head, const int *__restrict__ n_slot,
                                                        const int *__restrict__ n_next, unsigned long long *__restrict__ state, int K,
                                                        int *__restrict__ touched, int *__restrict__ info) {
    const int qi = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (qi >= nq) return;
    const unsigned qid = qid0 + b;
    const int w = q_ids[(size_t)b * nq + qi];
    if ((unsigned)w >= (unsigned)nwords) return;
    state += (size_t)b * K;
    touched += (size_t)b * K;
    info += 4 * b;
    for (int nd = w_head[w]; nd >= 0; nd = n_next[nd]) {
        const int s = n_slot[nd];
        unsigned long long old = state[s], assumed;
        do {
            assumed = old;
            unsigned long long nv;
            if (q_stamp(assumed) == qid)
                nv = ((unsigned long long)qid << 32) | ((unsigned long long)min(q_rank(assumed), qi) << 16) | (unsigned long long)(q_words(assumed) + 1);
            else
                nv = ((unsigned long long)qid << 32) | ((unsigned long long)qi << 16) | 1ull;   // mnLoopWords = 0; ++
            old = atomicCAS(&state[s], assumed, nv);
        } while (old != assumed);
        if (q_stamp(assumed) != qid) touched[atomicAdd(&info[0], 1)] = s;
    }
}

// one block per query; info row b: [0] touched, [1] list length, [2] minCommonWords
__global__ void __launch_bounds__(KFDB_BLOCK) kfdb_order_kernel(int loop, unsigned qid0, const unsigned long long *__restrict__ state,
                                                                const unsigned *__restrict__ conn, const unsigned *__restrict__ seqs,
                                                                const int *__restrict__ touched, int *__restrict__ info,
                                                                unsigned long long *__restrict__ keys, int *__restrict__ list, int K, int S) {
    __shared__ int sh[2];   // [0] list length, [1] maxCommonWords
    const int b = blockIdx.x;
    const unsigned qid = qid0 + b;
    state += (size_t)b * K;
    conn += (size_t)b * K;
    touched += (size_t)b * K;
    info += 4 * b;
    keys += (size_t)b * S;
    list += (size_t)b * S;
    const int nt = min(info[0], K);
    if (threadIdx.x == 0) sh[0] = sh[1] = 0;
    __syncthreads();
    // maxCommonWords over lKFsSharingWords (connected keyframes are not in it in loop mode)
    int mx = 0;
    for (int i = threadIdx.x; i < nt; i += blockDim.x) {
        const int s = touched[i];
        if (!(loop && conn[s] == qid)) mx = max(mx, q_words(state[s]));
    }
    atomicMax(&sh[1], mx);
    __syncthreads();
    const int maxCommon = sh[1];
    const int minCommon = (int)((float)maxCommon * 0.8f);
    // the qualifying slots, keyed by (first shared word rank, add order)
    for (int i = threadIdx.x; i < nt; i += blockDim.x) {
        const int s = touched[i];
        const unsigned long long st = state[s];
        if (!(loop && conn[s] == qid) && q_words(st) > minCommon) {
            const int p = atomicAdd(&sh[0], 1);
            keys[p] = ((unsigned long long)q_rank(st) << 32) | seqs[s];
            list[p] = s;
        }
    }
    __syncthreads();
    const int nl = sh[0];
    int n2 = 1;
    while (n2 < nl) n2 <<= 1;
    for (int i = nl + threadIdx.x; i < n2; i += blockDim.x) { keys[i] = ~0ull; list[i] = -1; }
    __syncthreads();
    // bitonic sort of (key, slot) pairs in global memory; keys are unique (add sequence numbers are)
    for (int k = 2; k <= n2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n2; i += blockDim.x) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long x = keys[i], y = keys[ixj];
                    if (((i & k) == 0) ? (x > y) : (x < y)) {
                        keys[i] = y; keys[ixj] = x;
                        const int t = list[i]; list[i] = list[ixj]; list[ixj] = t;
                    }
                }
            }
            __syncthreads();
        }
    }
    if (threadIdx.x == 0) { info[1] = nl; info[2] = minCommon; }
}

// grid (list entries, queries): query b's entry e records pKFi->mLoopScore / mRelocScore = si in the query's row; for a
// batch of one (`persist` = the mode's persistent scores) also in the slot itself, which is then the write-back
__global__ void __launch_bounds__(128) kfdb_score_kernel(unsigned qid0, int nq, const int *__restrict__ q_ids, const double *__restrict__ q_vals,
                                                         const int *__restrict__ info, const int *__restrict__ list, int S,
                                                         const int *__restrict__ range, const int *__restrict__ s_id,
                                                         const double *__restrict__ s_val, unsigned long long *__restrict__ scored, int K,
                                                         float *__restrict__ persist) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (e >= info[4 * b + 1]) return;
    const int s = list[(size_t)b * S + e];
    int common, first;
    const size_t q0 = (size_t)b * nq;
    const float si = (float)bow_l1_walk(nq, q_ids + q0, q_vals + q0, range[2 * s], range[2 * s + 1], s_id, s_val, common, first);
    scored[(size_t)b * K + s] = ((unsigned long long)(qid0 + b) << 32) | __float_as_uint(si);
    if (persist) persist[s] = si;
}

// grid (list entries, queries): the persistent score of a slot query b scored, unless a later query of the batch scored
// it too; runs after every select of the batch
__global__ void __launch_bounds__(128) kfdb_writeback_kernel(int loop, unsigned qid0, int nb, int K, int S, const int *__restrict__ info,
                                                             const int *__restrict__ list, const unsigned long long *__restrict__ scored,
                                                             float *__restrict__ lscore, float *__restrict__ rscore) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (e >= info[4 * b + 1]) return;
    const int s = list[(size_t)b * S + e];
    for (int a = b + 1; a < nb; a++)
        if ((unsigned)(scored[(size_t)a * K + s] >> 32) == qid0 + (unsigned)a) return;
    const float si = __uint_as_float((unsigned)scored[(size_t)b * K + s]);
    if (loop) lscore[s] = si; else rscore[s] = si;
}

// one block per query
__global__ void __launch_bounds__(KFDB_BLOCK) kfdb_select_kernel(int loop, unsigned qid0, const float *__restrict__ d_min_score, float min_score0,
                                                                 int K, int S, const int *__restrict__ info, const int *__restrict__ list,
                                                                 const unsigned long long *__restrict__ scored,
                                                                 const unsigned long long *__restrict__ state, const unsigned *__restrict__ conn,
                                                                 const float *__restrict__ lscore, const float *__restrict__ rscore,
                                                                 const int *__restrict__ covn, const int *__restrict__ cov,
                                                                 const int *__restrict__ touched, float *__restrict__ acc, int *__restrict__ best,
                                                                 unsigned long long *__restrict__ firstpos, int cap, int *__restrict__ cand,
                                                                 int *__restrict__ ncand, int *__restrict__ words_out, float *__restrict__ score_out) {
    __shared__ float s_best, s_wmax[KFDB_BLOCK / 32];
    __shared__ int s_cnt[KFDB_BLOCK / 32];
    __shared__ int s_base;
    const int q = blockIdx.x;
    const unsigned qid = qid0 + q;
    const float min_score = d_min_score ? d_min_score[q] : min_score0;
    const size_t rk = (size_t)q * K;
    info += 4 * q;
    list += (size_t)q * S;
    state += rk;
    conn += rk;
    touched += rk;
    acc += rk;
    best += rk;
    firstpos += rk;
    cand += (size_t)q * cap;
    ncand += q;
    if (words_out) words_out += rk;
    if (score_out) score_out += rk;
    const int nl = info[1], minCommon = info[2], nt = min(info[0], K);
    const float *sc = loop ? lscore : rscore;
    // words_out / score_out: this query's mnLoopWords / mnRelocWords and mLoopScore / mRelocScore of every touched slot
    if (words_out || score_out) {
        for (int i = threadIdx.x; i < K; i += blockDim.x) {
            if (words_out) words_out[i] = -1;
            if (score_out) score_out[i] = -1.f;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < nt; i += blockDim.x) {
            const int s = touched[i];
            // a connected keyframe is reset at every visit and never stamped: its mnLoopWords ends at 1 (:92-101)
            if (words_out) words_out[s] = (loop && conn[s] == qid) ? 1 : q_words(state[s]);
            if (score_out) score_out[s] = kfdb_score_read(q, qid0, s, K, scored, sc);
        }
    }
    if (threadIdx.x == 0) { s_best = loop ? min_score : 0.f; s_base = 0; }
    __syncthreads();
    // lAccScoreAndMatch, one entry per lScoreAndMatch entry (loop mode keeps si >= minScore, :135)
    float mybest = -INFINITY;
    for (int e = threadIdx.x; e < nl; e += blockDim.x) {
        const int s = list[e];
        const float si = __uint_as_float((unsigned)scored[rk + s]);
        if (loop && !(si >= min_score)) { best[e] = -1; continue; }
        float bestScore = si, accScore = si;
        int b = s;
        const int nc = covn[s];
        for (int j = 0; j < nc; j++) {
            const int s2 = cov[s * KFDB_COVIS + j];
            if (s2 < 0) continue;   // a bad keyframe in a device-written list: it holds its place and contributes nothing
            const unsigned long long st = state[s2];
            // an earlier query's score when s2 was only touched; read next to the stamp, used only when s2 counts
            const float s2c = kfdb_score_read(q, qid0, s2, K, scored, sc);
            if (q_stamp(st) != qid) continue;                                              // mnLoopQuery / mnRelocQuery
            if (loop && (conn[s2] == qid || !(q_words(st) > minCommon))) continue;         // :158
            accScore += s2c;
            if (s2c > bestScore) { b = s2; bestScore = s2c; }
        }
        acc[e] = accScore;
        best[e] = b;
        mybest = fmaxf(mybest, accScore);
    }
    // bestAccScore = max(initial, every accScore): a maximum, independent of the order it is taken in
    for (int o = 16; o > 0; o >>= 1) mybest = fmaxf(mybest, __shfl_xor_sync(0xffffffffu, mybest, o));
    if ((threadIdx.x & 31) == 0) s_wmax[threadIdx.x >> 5] = mybest;
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 0; w < KFDB_BLOCK / 32; w++) s_best = fmaxf(s_best, s_wmax[w]);
    __syncthreads();
    const float minScoreToRetain = 0.75f * s_best;
    // the first entry naming a keyframe wins (spAlreadyAddedKF): the lowest entry index per keyframe; a newer query id
    // makes a smaller high word, so earlier queries' values never win
    const unsigned long long tag = (unsigned long long)(0xFFFFFFFFu - qid) << 32;
    for (int e = threadIdx.x; e < nl; e += blockDim.x)
        if (best[e] >= 0 && acc[e] > minScoreToRetain) atomicMin(&firstpos[best[e]], tag | (unsigned)e);
    __syncthreads();
    // in-order compaction of the winning entries
    for (int c0 = 0; c0 < nl; c0 += blockDim.x) {
        const int e = c0 + threadIdx.x;
        bool keep = false;
        int b = -1;
        if (e < nl) {
            b = best[e];
            keep = b >= 0 && acc[e] > minScoreToRetain && atomicAdd(&firstpos[b], 0ull) == (tag | (unsigned)e);
        }
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
        if (lane == 0) s_cnt[wid] = __popc(bal);
        __syncthreads();
        int before = s_base, total = 0;
        for (int w = 0; w < KFDB_BLOCK / 32; w++) {
            if (w < wid) before += s_cnt[w];
            total += s_cnt[w];
        }
        if (keep) {
            const int pos = before + __popc(bal & ((1u << lane) - 1u));
            if (pos < cap) cand[pos] = b;
        }
        __syncthreads();
        if (threadIdx.x == 0) s_base += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) *ncand = s_base;
}

}  // namespace orbfe

using namespace orbfe;

struct OrbfeKeyFrameDB {
    int nwords = 0, K = 0, sortcap = 1, Q = 1;   // Q: rows of per-query state (max_queries)
    long long P = 0;
    HandleStream hs;
    DeviceBuffers mem;            // every device array below
    // host side: allocation only
    std::vector<int> begin, len;   // store rows of each slot; len -1 = empty
    std::vector<std::vector<int>> nodes;
    std::vector<int> free_nodes;
    long long top = 0, live = 0;
    unsigned seq = 0, qid = 0;
    // device
    int *s_id[2] = {nullptr, nullptr}, *s_node[2] = {nullptr, nullptr};
    double *s_val[2] = {nullptr, nullptr};
    int cur = 0;
    int *n_slot = nullptr, *n_next = nullptr, *n_prev = nullptr, *w_head = nullptr, *w_tail = nullptr;
    int *range = nullptr, *covn = nullptr, *cov = nullptr, *touched = nullptr, *list = nullptr, *best = nullptr, *info = nullptr;
    int *moves = nullptr, *covrows = nullptr;
    int *a_info = nullptr;        // add_device: [0] bad-row flag, [1 + i] word count of row i
    unsigned *seqs = nullptr, *conn = nullptr;
    unsigned long long *state = nullptr, *keys = nullptr, *firstpos = nullptr, *scored = nullptr;
    float *lscore = nullptr, *rscore = nullptr, *acc = nullptr;
    // staging of the host-pointer detect
    int *q_ids = nullptr, *q_conn = nullptr, *o_cand = nullptr, *o_words = nullptr, *o_n = nullptr;
    double *q_vals = nullptr;
    float *o_score = nullptr;
};

#define KFDB_MAX_NQ 65535   // the shared-word rank and count are 16-bit fields of the query state

extern "C" void orbfe_kfdb_destroy(OrbfeKeyFrameDB *db) {
    if (!db) return;
    cudaSetDevice(db->hs.device);
    if (db->hs.stream) cudaStreamSynchronize(db->hs.stream);
    db->mem.release();
    db->hs.destroy();
    delete db;
}

static int kfdb_reset(OrbfeKeyFrameDB *db) {
    db->begin.assign(db->K, 0);
    db->len.assign(db->K, -1);
    db->nodes.assign(db->K, std::vector<int>());
    db->free_nodes.resize((size_t)db->P);
    for (long long i = 0; i < db->P; i++) db->free_nodes[(size_t)i] = (int)(db->P - 1 - i);   // pops 0, 1, 2, ...
    db->top = db->live = 0;
    cudaStream_t s = db->hs.stream;
    ORBFE_CUDA_TRY(cudaMemsetAsync(db->w_head, 0xFF, sizeof(int) * (size_t)db->nwords, s));
    ORBFE_CUDA_TRY(cudaMemsetAsync(db->w_tail, 0xFF, sizeof(int) * (size_t)db->nwords, s));
    std::vector<int> r(2 * (size_t)db->K);
    for (int k = 0; k < db->K; k++) { r[2 * k] = 0; r[2 * k + 1] = -1; }
    ORBFE_CUDA_TRY(cudaMemcpyAsync(db->range, r.data(), sizeof(int) * r.size(), cudaMemcpyHostToDevice, s));
    ORBFE_CUDA_TRY(cudaMemsetAsync(db->covn, 0, sizeof(int) * (size_t)db->K, s));
    ORBFE_CUDA_TRY(cudaStreamSynchronize(s));
    return ORBFE_OK;
}

#define KFDB_MAX_QUERIES 1024

extern "C" int orbfe_kfdb_create_batched(OrbfeVocabulary *v, int max_keyframes, long long max_postings, int max_queries,
                                         OrbfeKeyFrameDB **out) {
    if (!out) return set_error(ORBFE_ERR_ARG, "NULL out");
    *out = nullptr;
    if (!v || max_keyframes < 1 || max_keyframes > (1 << 24) || max_postings < 1 || max_postings > 0x7FFFFFFFLL || max_queries < 1 ||
        max_queries > KFDB_MAX_QUERIES)
        return set_error(ORBFE_ERR_ARG, "bad arguments (1 <= max_keyframes <= 2^24, 1 <= max_postings < 2^31, 1 <= max_queries <= %d)",
                         KFDB_MAX_QUERIES);
    OrbfeKeyFrameDB *db = new OrbfeKeyFrameDB();
    db->nwords = std::max(vocab_nwords(v), 1);
    db->K = max_keyframes;
    db->P = max_postings;
    db->Q = max_queries;
    while (db->sortcap < db->K) db->sortcap <<= 1;
    const size_t K = (size_t)db->K, P = (size_t)db->P, W = (size_t)db->nwords, S = (size_t)db->sortcap, QK = (size_t)db->Q * K,
                 QS = (size_t)db->Q * S;
    bool ok = db->hs.create(vocab_device(v)) == cudaSuccess;
    const auto alloc = [&](auto **p, size_t n) { ok = ok && db->mem.alloc(p, n) == cudaSuccess; };
    for (int h = 0; h < 2; h++) { alloc(&db->s_id[h], P); alloc(&db->s_node[h], P); alloc(&db->s_val[h], P); }
    alloc(&db->n_slot, P); alloc(&db->n_next, P); alloc(&db->n_prev, P);
    alloc(&db->w_head, W); alloc(&db->w_tail, W);
    alloc(&db->range, 2 * K); alloc(&db->covn, K); alloc(&db->cov, K * KFDB_COVIS); alloc(&db->moves, 3 * K);
    alloc(&db->covrows, K * (2 + KFDB_COVIS)); alloc(&db->seqs, K); alloc(&db->lscore, K); alloc(&db->rscore, K);
    // per-query rows (include/orbfe_bow.h states their size)
    alloc(&db->touched, QK); alloc(&db->list, QS); alloc(&db->best, QK); alloc(&db->info, 4 * (size_t)db->Q);
    alloc(&db->conn, QK); alloc(&db->state, QK); alloc(&db->keys, QS); alloc(&db->firstpos, QK);
    alloc(&db->scored, QK); alloc(&db->acc, QK);
    alloc(&db->q_ids, KFDB_MAX_NQ); alloc(&db->q_vals, KFDB_MAX_NQ); alloc(&db->q_conn, K);
    alloc(&db->o_cand, K); alloc(&db->o_words, K); alloc(&db->o_score, K); alloc(&db->o_n, 1);
    alloc(&db->a_info, K + 1);
    ok = ok && cudaMemset(db->conn, 0, sizeof(unsigned) * QK) == cudaSuccess && cudaMemset(db->state, 0, sizeof(unsigned long long) * QK) == cudaSuccess &&
         cudaMemset(db->scored, 0, sizeof(unsigned long long) * QK) == cudaSuccess &&
         cudaMemset(db->firstpos, 0xFF, sizeof(unsigned long long) * QK) == cudaSuccess;
    if (!ok) {
        const int rc = set_error(ORBFE_ERR_CUDA, "keyframe database allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
        orbfe_kfdb_destroy(db);
        return rc;
    }
    const int rc = kfdb_reset(db);
    if (rc) { orbfe_kfdb_destroy(db); return rc; }
    *out = db;
    return ORBFE_OK;
}

extern "C" int orbfe_kfdb_create(OrbfeVocabulary *v, int max_keyframes, long long max_postings, OrbfeKeyFrameDB **out) {
    return orbfe_kfdb_create_batched(v, max_keyframes, max_postings, 1, out);
}

// move every live slot's rows to the front of the other half of the store
static int kfdb_compact(OrbfeKeyFrameDB *db) {
    std::vector<int> order;
    for (int k = 0; k < db->K; k++) if (db->len[k] > 0) order.push_back(k);
    std::sort(order.begin(), order.end(), [&](int a, int b) { return db->begin[a] < db->begin[b]; });
    std::vector<int> moves;
    int pos = 0;
    for (int k : order) {
        moves.push_back(db->begin[k]); moves.push_back(pos); moves.push_back(db->len[k]);
        db->begin[k] = pos;
        pos += db->len[k];
    }
    std::vector<int> r(2 * (size_t)db->K);
    for (int k = 0; k < db->K; k++) {
        r[2 * k] = db->len[k] >= 0 ? db->begin[k] : 0;
        r[2 * k + 1] = db->len[k] >= 0 ? db->begin[k] + db->len[k] : -1;
    }
    cudaStream_t s = db->hs.stream;
    const int o = db->cur, n = 1 - db->cur;
    const int nmove = (int)order.size();
    if (nmove > 0) {
        ORBFE_CUDA_TRY(cudaMemcpyAsync(db->moves, moves.data(), sizeof(int) * moves.size(), cudaMemcpyHostToDevice, s));
        kfdb_compact_kernel<<<std::min(nmove, 1024), 256, 0, s>>>(db->moves, nmove, db->s_id[o], db->s_val[o], db->s_node[o], db->s_id[n],
                                                                  db->s_val[n], db->s_node[n]);
    }
    ORBFE_CUDA_TRY(cudaMemcpyAsync(db->range, r.data(), sizeof(int) * r.size(), cudaMemcpyHostToDevice, s));
    ORBFE_CUDA_TRY(cudaStreamSynchronize(s));   // `moves` / `r` are host locals
    db->cur = n;
    db->top = pos;
    return ORBFE_OK;
}

extern "C" int orbfe_kfdb_add(OrbfeKeyFrameDB *db, int slot, int nw, const int32_t *ids, const double *vals) {
    if (!db || slot < 0 || nw < 0 || (nw > 0 && (!ids || !vals))) return set_error(ORBFE_ERR_ARG, "bad arguments");
    for (int i = 0; i < nw; i++)
        if (ids[i] < 0 || (i > 0 && ids[i] <= ids[i - 1])) return set_error(ORBFE_ERR_ARG, "word ids must be >= 0 and strictly ascending");
    if (slot >= db->K) return set_error(ORBFE_ERR_ARG, "slot %d out of range (max_keyframes %d)", slot, db->K);
    if (nw > 0 && ids[nw - 1] >= db->nwords) return set_error(ORBFE_ERR_ARG, "word id %d >= vocabulary words %d", ids[nw - 1], db->nwords);
    if (db->len[slot] >= 0) return set_error(ORBFE_ERR_ARG, "slot %d is occupied", slot);
    if (db->live + nw > db->P)
        return set_error(ORBFE_ERR_CAPACITY, "%lld postings + %d exceed max_postings %lld", db->live, nw, db->P);
    cudaStream_t s = db->hs.stream;
    int rc = db->hs.enter(s);
    if (rc) return rc;
    if (db->top + nw > db->P && (rc = kfdb_compact(db))) return rc;
    std::vector<int> nodes(nw);
    for (int i = 0; i < nw; i++) { nodes[i] = db->free_nodes.back(); db->free_nodes.pop_back(); }
    const int base = (int)db->top, c = db->cur;
    if (nw > 0) {
        ORBFE_CUDA_TRY(cudaMemcpyAsync(db->s_id[c] + base, ids, sizeof(int) * nw, cudaMemcpyHostToDevice, s));
        ORBFE_CUDA_TRY(cudaMemcpyAsync(db->s_val[c] + base, vals, sizeof(double) * nw, cudaMemcpyHostToDevice, s));
        ORBFE_CUDA_TRY(cudaMemcpyAsync(db->s_node[c] + base, nodes.data(), sizeof(int) * nw, cudaMemcpyHostToDevice, s));
    }
    kfdb_link_kernel<<<(std::max(nw, 1) + 255) / 256, 256, 0, s>>>(slot, base, nw, ++db->seq, db->s_id[c], db->s_node[c], db->n_slot, db->n_next,
                                                                   db->n_prev, db->w_head, db->w_tail, db->range, db->seqs, db->lscore,
                                                                   db->rscore);
    if ((rc = db->hs.leave(s, true))) return rc;
    db->begin[slot] = base;
    db->len[slot] = nw;
    db->nodes[slot].swap(nodes);
    db->top += nw;
    db->live += nw;
    return ORBFE_OK;
}

extern "C" int orbfe_kfdb_add_device(OrbfeKeyFrameDB *db, int n, const int32_t *slots, const int32_t *frames, int cap,
                                     const int32_t *d_bow_ids, const double *d_bow_vals, const int *d_bow_n, void *stream) {
    if (!db || n < 0 || cap < 1 || cap > ORBFE_FV_MAX_CAP)
        return set_error(ORBFE_ERR_ARG, "bad arguments (n >= 0, 1 <= cap <= %d)", ORBFE_FV_MAX_CAP);
    if (n > 0 && (!slots || !frames || !d_bow_ids || !d_bow_vals || !d_bow_n)) return set_error(ORBFE_ERR_ARG, "NULL argument");
    for (int i = 0; i < n; i++)
        if (slots[i] < 0 || frames[i] < 0) return set_error(ORBFE_ERR_ARG, "negative slot or frame at %d", i);
    std::vector<int> sorted(slots, slots + n);
    std::sort(sorted.begin(), sorted.end());
    for (int i = 1; i < n; i++)
        if (sorted[i] == sorted[i - 1]) return set_error(ORBFE_ERR_ARG, "slot %d listed twice", sorted[i]);
    if (n == 0) return ORBFE_OK;
    for (int i = 0; i < n; i++) {
        if (slots[i] >= db->K) return set_error(ORBFE_ERR_ARG, "slot %d out of range (max_keyframes %d)", slots[i], db->K);
        if (db->len[slots[i]] >= 0) return set_error(ORBFE_ERR_ARG, "slot %d is occupied", slots[i]);
    }
    // the rows are checked on the device, after the work that wrote them; their word counts are the one readback
    cudaStream_t s = db->hs.pick(stream);
    int rc = db->hs.enter(s);
    if (rc) return rc;
    ORBFE_CUDA_TRY(cudaMemcpyAsync(db->moves, frames, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, s));
    ORBFE_CUDA_TRY(cudaMemsetAsync(db->a_info, 0, sizeof(int), s));
    kfdb_check_rows_kernel<<<std::min(n, 1024), 256, 0, s>>>(db->moves, n, cap, db->nwords, d_bow_n, d_bow_ids, db->a_info);
    ORBFE_CUDA_TRY(cudaGetLastError());
    std::vector<int> info((size_t)n + 1);
    ORBFE_CUDA_TRY(cudaMemcpyAsync(info.data(), db->a_info, sizeof(int) * info.size(), cudaMemcpyDeviceToHost, s));
    ORBFE_CUDA_TRY(cudaStreamSynchronize(s));
    if (info[0])
        return set_error(ORBFE_ERR_ARG, "a BowVector row has a word count outside 0 .. %d, or word ids that are not strictly ascending below %d",
                         cap, db->nwords);
    long long total = 0;
    for (int i = 0; i < n; i++) total += info[1 + i];
    if (db->live + total > db->P)
        return set_error(ORBFE_ERR_CAPACITY, "%lld postings + %lld exceed max_postings %lld", db->live, total, db->P);
    // `s` has drained: the handle's earlier work and the rows are complete, the rest runs on the handle's stream
    cudaStream_t hs = db->hs.stream;
    if (db->top + total > db->P && (rc = kfdb_compact(db))) return rc;
    const int c = db->cur, top = (int)db->top;
    std::vector<int> rows(3 * (size_t)n), nodes((size_t)total);
    for (int i = 0, pos = 0; i < n; i++) {
        rows[3 * i] = frames[i];
        rows[3 * i + 1] = top + pos;
        rows[3 * i + 2] = info[1 + i];
        for (int k = 0; k < info[1 + i]; k++, pos++) { nodes[pos] = db->free_nodes.back(); db->free_nodes.pop_back(); }
    }
    ORBFE_CUDA_TRY(cudaMemcpyAsync(db->moves, rows.data(), sizeof(int) * rows.size(), cudaMemcpyHostToDevice, hs));
    if (total > 0) ORBFE_CUDA_TRY(cudaMemcpyAsync(db->s_node[c] + top, nodes.data(), sizeof(int) * nodes.size(), cudaMemcpyHostToDevice, hs));
    kfdb_gather_kernel<<<std::min(n, 1024), 256, 0, hs>>>(db->moves, n, cap, d_bow_ids, d_bow_vals, db->s_id[c], db->s_val[c]);
    // one keyframe after the other: two keyframes may share a word, and every word's list is in add order
    for (int i = 0; i < n; i++) {
        const int nw = rows[3 * i + 2];
        kfdb_link_kernel<<<(std::max(nw, 1) + 255) / 256, 256, 0, hs>>>(slots[i], rows[3 * i + 1], nw, ++db->seq, db->s_id[c], db->s_node[c],
                                                                        db->n_slot, db->n_next, db->n_prev, db->w_head, db->w_tail,
                                                                        db->range, db->seqs, db->lscore, db->rscore);
    }
    if ((rc = db->hs.leave(hs, true))) return rc;
    for (int i = 0, pos = 0; i < n; i++) {
        const int sl = slots[i], nw = rows[3 * i + 2];
        db->begin[sl] = rows[3 * i + 1];
        db->len[sl] = nw;
        db->nodes[sl].assign(nodes.begin() + pos, nodes.begin() + pos + nw);
        pos += nw;
    }
    db->top += total;
    db->live += total;
    return ORBFE_OK;
}

extern "C" int orbfe_kfdb_erase(OrbfeKeyFrameDB *db, int slot) {
    if (!db || slot < 0) return set_error(ORBFE_ERR_ARG, "bad arguments");
    if (slot >= db->K) return set_error(ORBFE_ERR_ARG, "slot %d out of range (max_keyframes %d)", slot, db->K);
    if (db->len[slot] < 0) return ORBFE_OK;   // erase of a keyframe that is not in the database: nothing to unlink
    cudaStream_t s = db->hs.stream;
    int rc = db->hs.enter(s);
    if (rc) return rc;
    const int nw = db->len[slot];
    kfdb_unlink_kernel<<<(std::max(nw, 1) + 255) / 256, 256, 0, s>>>(slot, db->begin[slot], nw, db->s_id[db->cur], db->s_node[db->cur], db->n_next,
                                                                     db->n_prev, db->w_head, db->w_tail, db->range, db->covn);
    if ((rc = db->hs.leave(s, true))) return rc;
    for (int nd : db->nodes[slot]) db->free_nodes.push_back(nd);
    db->nodes[slot].clear();
    if (db->begin[slot] + nw == db->top) db->top -= nw;   // the last rows: the tail shrinks back
    db->live -= nw;
    db->len[slot] = -1;
    return ORBFE_OK;
}

extern "C" int orbfe_kfdb_clear(OrbfeKeyFrameDB *db) {
    if (!db) return set_error(ORBFE_ERR_ARG, "bad arguments");
    int rc = db->hs.enter(db->hs.stream);
    if (rc) return rc;
    if ((rc = kfdb_reset(db))) return rc;
    return db->hs.leave(db->hs.stream, true);
}

extern "C" int orbfe_kfdb_set_covisibles(OrbfeKeyFrameDB *db, int n, const int32_t *slots, const int32_t *ptr, const int32_t *lists) {
    if (!db || n < 0 || (n > 0 && (!slots || !ptr))) return set_error(ORBFE_ERR_ARG, "bad arguments");
    if (n == 0) return ORBFE_OK;
    if (ptr[0] != 0) return set_error(ORBFE_ERR_ARG, "ptr[0] must be 0");
    for (int i = 0; i < n; i++) {
        const int c = ptr[i + 1] - ptr[i];
        if (c < 0 || c > KFDB_COVIS) return set_error(ORBFE_ERR_ARG, "list %d has %d entries (0 .. %d)", i, c, KFDB_COVIS);
        if (slots[i] < 0) return set_error(ORBFE_ERR_ARG, "negative slot");
    }
    if (ptr[n] > 0 && !lists) return set_error(ORBFE_ERR_ARG, "NULL lists");
    for (int j = 0; j < ptr[n]; j++)
        if (lists[j] < 0) return set_error(ORBFE_ERR_ARG, "negative slot in a list");
    if (n > db->K) return set_error(ORBFE_ERR_ARG, "more lists than slots");
    std::vector<uint8_t> seen(db->K, 0);
    std::vector<int> rows((size_t)n * (2 + KFDB_COVIS), 0);
    for (int i = 0; i < n; i++) {
        if (slots[i] >= db->K) return set_error(ORBFE_ERR_ARG, "slot %d out of range", slots[i]);
        if (seen[slots[i]]++) return set_error(ORBFE_ERR_ARG, "slot %d listed twice", slots[i]);
        int *r = &rows[(size_t)i * (2 + KFDB_COVIS)];
        r[0] = slots[i];
        r[1] = ptr[i + 1] - ptr[i];
        for (int j = ptr[i]; j < ptr[i + 1]; j++) {
            if (lists[j] >= db->K) return set_error(ORBFE_ERR_ARG, "covisible slot %d out of range", lists[j]);
            r[2 + j - ptr[i]] = lists[j];
        }
    }
    cudaStream_t s = db->hs.stream;
    int rc = db->hs.enter(s);
    if (rc) return rc;
    ORBFE_CUDA_TRY(cudaMemcpyAsync(db->covrows, rows.data(), sizeof(int) * rows.size(), cudaMemcpyHostToDevice, s));
    kfdb_covis_kernel<<<(n + 127) / 128, 128, 0, s>>>(db->covrows, n, db->covn, db->cov);
    return db->hs.leave(s, true);
}

extern "C" int orbfe_kfdb_set_covisibles_device(OrbfeKeyFrameDB *db, int n, const int32_t *slots, const int32_t *d_ptr,
                                                const int32_t *d_lists, void *stream) {
    if (!db || n < 0 || (n > 0 && (!slots || !d_ptr || !d_lists))) return set_error(ORBFE_ERR_ARG, "bad arguments");
    for (int i = 0; i < n; i++)
        if (slots[i] < 0) return set_error(ORBFE_ERR_ARG, "negative slot");
    if (n == 0) return ORBFE_OK;
    if (n > db->K) return set_error(ORBFE_ERR_ARG, "more lists than slots");
    std::vector<uint8_t> seen(db->K, 0);
    for (int i = 0; i < n; i++) {
        if (slots[i] >= db->K) return set_error(ORBFE_ERR_ARG, "slot %d out of range", slots[i]);
        if (seen[slots[i]]++) return set_error(ORBFE_ERR_ARG, "slot %d listed twice", slots[i]);
    }
    cudaStream_t s = db->hs.pick(stream);
    int rc = db->hs.enter(s);
    if (rc) return rc;
    ORBFE_CUDA_TRY(cudaMemcpyAsync(db->covrows, slots, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, s));
    kfdb_covis_device_kernel<<<(n + 127) / 128, 128, 0, s>>>(db->covrows, n, db->K, d_ptr, d_lists, db->covn, db->cov);
    return db->hs.leave(s, false);
}

static int kfdb_check_detect(int mode, int nq, int nconn, int cap) {
    if (mode < 0 || mode > 1) return set_error(ORBFE_ERR_ARG, "mode must be 0 (loop) or 1 (relocalisation)");
    if (nq < 0 || nq > KFDB_MAX_NQ) return set_error(ORBFE_ERR_ARG, "nq %d out of range (0 .. %d)", nq, KFDB_MAX_NQ);
    if (nconn < 0) return set_error(ORBFE_ERR_ARG, "nconn < 0");
    if (cap < 0) return set_error(ORBFE_ERR_ARG, "cap < 0");
    return ORBFE_OK;
}

// nb queries of one mode on the per-query rows 0 .. nb-1, as nb consecutive query ids; enqueued on s.  Query b's words are
// row b of q_ids / q_vals (qcap entries); its connected slots are conn_ptr's range of `connected` (no conn_ptr: [0, nconn));
// its minScore is d_min_score[b] (no d_min_score: min_score).
static void kfdb_queries(OrbfeKeyFrameDB *db, int mode, int nb, int qcap, const int *q_ids, const double *q_vals, const int *conn_ptr,
                         const int *connected, int nconn, const float *d_min_score, float min_score, int cap, int *cand, int *ncand,
                         int *words, float *score, cudaStream_t s) {
    const int loop = mode == 0;
    const unsigned qid0 = db->qid + 1;
    db->qid += (unsigned)nb;
    const int K = db->K, S = db->sortcap, c = db->cur;
    const int bx = conn_ptr ? 4 : std::max(1, std::min((nconn + 255) / 256, 64));
    kfdb_begin_kernel<<<dim3(bx, nb), 256, 0, s>>>(loop, qid0, conn_ptr, connected, nconn, K, db->conn, db->info);
    if (qcap > 0)
        kfdb_walk_kernel<<<dim3((qcap + 127) / 128, nb), 128, 0, s>>>(qid0, qcap, q_ids, db->nwords, db->w_head, db->n_slot, db->n_next,
                                                                      db->state, K, db->touched, db->info);
    kfdb_order_kernel<<<nb, KFDB_BLOCK, 0, s>>>(loop, qid0, db->state, db->conn, db->seqs, db->touched, db->info, db->keys, db->list, K, S);
    const dim3 per_entry((K + 127) / 128, nb);
    kfdb_score_kernel<<<per_entry, 128, 0, s>>>(qid0, qcap, q_ids, q_vals, db->info, db->list, S, db->range, db->s_id[c], db->s_val[c],
                                                db->scored, K, nb == 1 ? (loop ? db->lscore : db->rscore) : nullptr);
    kfdb_select_kernel<<<nb, KFDB_BLOCK, 0, s>>>(loop, qid0, d_min_score, min_score, K, S, db->info, db->list, db->scored, db->state,
                                                 db->conn, db->lscore, db->rscore, db->covn, db->cov, db->touched, db->acc, db->best,
                                                 db->firstpos, cap, cand, ncand, words, score);
    if (nb > 1) kfdb_writeback_kernel<<<per_entry, 128, 0, s>>>(loop, qid0, nb, K, S, db->info, db->list, db->scored, db->lscore, db->rscore);
}

extern "C" int orbfe_kfdb_detect_device(OrbfeKeyFrameDB *db, int mode, int nq, const int32_t *d_q_ids, const double *d_q_vals, int nconn,
                                        const int32_t *d_connected, float min_score, int cap, int32_t *d_cand, int *d_ncand,
                                        int32_t *d_words, float *d_score, void *stream) {
    int rc = kfdb_check_detect(mode, nq, nconn, cap);
    if (rc) return rc;
    if (!db || !d_ncand || (nq > 0 && (!d_q_ids || !d_q_vals)) || (mode == 0 && nconn > 0 && !d_connected) || (cap > 0 && !d_cand))
        return set_error(ORBFE_ERR_ARG, "NULL argument");
    cudaStream_t s = db->hs.pick(stream);
    if ((rc = db->hs.enter(s))) return rc;
    kfdb_queries(db, mode, 1, nq, d_q_ids, d_q_vals, nullptr, d_connected, mode == 0 ? nconn : 0, nullptr, min_score, cap, d_cand, d_ncand,
                 d_words, d_score, s);
    return db->hs.leave(s, false);
}

extern "C" int orbfe_kfdb_detect_batch_device(OrbfeKeyFrameDB *db, int mode, int nqueries, int qcap, const int32_t *d_q_ids,
                                              const double *d_q_vals, const int32_t *d_conn_ptr, const int32_t *d_connected,
                                              const float *d_min_score, int cap, int32_t *d_cand, int *d_ncand, int32_t *d_words,
                                              float *d_score, void *stream) {
    int rc = kfdb_check_detect(mode, qcap, 0, cap);
    if (rc) return rc;
    if (nqueries < 1) return set_error(ORBFE_ERR_ARG, "nqueries %d < 1", nqueries);
    if (!db || !d_ncand || (qcap > 0 && (!d_q_ids || !d_q_vals)) || (mode == 0 && (!d_conn_ptr || !d_min_score)) || (cap > 0 && !d_cand))
        return set_error(ORBFE_ERR_ARG, "NULL argument");
    if (nqueries > db->Q) return set_error(ORBFE_ERR_ARG, "nqueries %d > max_queries %d", nqueries, db->Q);
    cudaStream_t s = db->hs.pick(stream);
    if ((rc = db->hs.enter(s))) return rc;
    kfdb_queries(db, mode, nqueries, qcap, d_q_ids, d_q_vals, mode == 0 ? d_conn_ptr : nullptr, mode == 0 ? d_connected : nullptr, 0,
                 mode == 0 ? d_min_score : nullptr, 0.f, cap, d_cand, d_ncand, d_words, d_score, s);
    return db->hs.leave(s, false);
}

extern "C" int orbfe_kfdb_detect(OrbfeKeyFrameDB *db, int mode, int nq, const int32_t *q_ids, const double *q_vals, int nconn,
                                 const int32_t *connected, float min_score, int cap, int32_t *cand_out, int *ncand_out, int32_t *words_out,
                                 float *score_out) {
    int rc = kfdb_check_detect(mode, nq, nconn, cap);
    if (rc) return rc;
    if (!db || !ncand_out || (nq > 0 && (!q_ids || !q_vals)) || (mode == 0 && nconn > 0 && !connected) || (cap > 0 && !cand_out))
        return set_error(ORBFE_ERR_ARG, "NULL argument");
    for (int i = 0; i < nq; i++)
        if (q_ids[i] < 0 || (i > 0 && q_ids[i] <= q_ids[i - 1])) return set_error(ORBFE_ERR_ARG, "query word ids must be >= 0 and strictly ascending");
    if (nq > 0 && q_ids[nq - 1] >= db->nwords) return set_error(ORBFE_ERR_ARG, "query word id %d >= vocabulary words %d", q_ids[nq - 1], db->nwords);
    if (mode == 0) {
        if (nconn > db->K) return set_error(ORBFE_ERR_ARG, "more connected keyframes than slots");
        for (int i = 0; i < nconn; i++)
            if (connected[i] < 0 || connected[i] >= db->K) return set_error(ORBFE_ERR_ARG, "connected slot %d out of range", connected[i]);
    }
    cudaStream_t s = db->hs.stream;
    if ((rc = db->hs.enter(s))) return rc;
    if (nq > 0) {
        ORBFE_CUDA_TRY(cudaMemcpyAsync(db->q_ids, q_ids, sizeof(int) * nq, cudaMemcpyHostToDevice, s));
        ORBFE_CUDA_TRY(cudaMemcpyAsync(db->q_vals, q_vals, sizeof(double) * nq, cudaMemcpyHostToDevice, s));
    }
    if (mode == 0 && nconn > 0) ORBFE_CUDA_TRY(cudaMemcpyAsync(db->q_conn, connected, sizeof(int) * nconn, cudaMemcpyHostToDevice, s));
    rc = orbfe_kfdb_detect_device(db, mode, nq, db->q_ids, db->q_vals, mode == 0 ? nconn : 0, db->q_conn, min_score, db->K, db->o_cand,
                                  db->o_n, db->o_words, db->o_score, s);
    if (rc) return rc;
    int n = 0;
    ORBFE_CUDA_TRY(cudaMemcpyAsync(&n, db->o_n, sizeof(int), cudaMemcpyDeviceToHost, s));
    if (words_out) ORBFE_CUDA_TRY(cudaMemcpyAsync(words_out, db->o_words, sizeof(int) * (size_t)db->K, cudaMemcpyDeviceToHost, s));
    if (score_out) ORBFE_CUDA_TRY(cudaMemcpyAsync(score_out, db->o_score, sizeof(float) * (size_t)db->K, cudaMemcpyDeviceToHost, s));
    ORBFE_CUDA_TRY(cudaStreamSynchronize(s));
    *ncand_out = n;
    if (n > cap) return set_error(ORBFE_ERR_CAPACITY, "%d candidates exceed cap %d", n, cap);
    if (n > 0) ORBFE_CUDA_TRY(cudaMemcpy(cand_out, db->o_cand, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost));
    return ORBFE_OK;
}

extern "C" int orbfe_kfdb_size(OrbfeKeyFrameDB *db, int *nkeyframes, long long *npostings) {
    if (!db) return set_error(ORBFE_ERR_ARG, "bad arguments");
    int n = 0;
    for (int k = 0; k < db->K; k++) n += db->len[k] >= 0;
    if (nkeyframes) *nkeyframes = n;
    if (npostings) *npostings = db->live;
    return ORBFE_OK;
}
