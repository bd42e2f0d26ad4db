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
// A query is five launches on one stream and no host synchronisation:
//   kfdb_begin_kernel   stamps the query keyframe's connected slots (loop mode) and resets the touched counter;
//   kfdb_walk_kernel    one thread per query word walks that word's list: counts shared words, keeps the lowest shared
//                       word rank, and the first touch appends the slot to the touched list (lKFsSharingWords, unordered);
//   kfdb_order_kernel   one block: maxCommonWords over the touched slots, the threshold, and the qualifying slots sorted by
//                       (first shared word rank, add order) -- the order of lKFsSharingWords;
//   kfdb_score_kernel   one thread per qualifying slot: the L1 score (bow_l1.cuh, the walk bow_db_score_kernel uses);
//   kfdb_select_kernel  one block: covisibility accumulation and candidate selection in list order, and the outputs.
// Every order-dependent step works on the sorted list, so results do not depend on block scheduling.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/orbfe_bow.h"
#include "bow_l1.cuh"
#include "orbfe_internal.h"

namespace orbfe {
int set_error(int code, const char *fmt, ...);
int vocab_device(const OrbfeVocabulary *v);
int vocab_nwords(const OrbfeVocabulary *v);

#define KFDB_COVIS 10
#define KFDB_BLOCK 1024

__global__ void kfdb_link_kernel(int slot, int base, int nw, unsigned seq, const int *__restrict__ s_id, const int *__restrict__ s_node,
                                 int *__restrict__ n_slot, int *__restrict__ n_next, int *__restrict__ n_prev, int *__restrict__ w_head,
                                 int *__restrict__ w_tail, int *__restrict__ range, unsigned *__restrict__ seqs,
                                 unsigned long long *__restrict__ state, float *__restrict__ lscore, float *__restrict__ rscore) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) {   // a fresh KeyFrame: stamps 0, scores 0
        range[2 * slot] = base;
        range[2 * slot + 1] = base + nw;
        seqs[slot] = seq;
        state[slot] = 0ull;
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

__device__ __forceinline__ unsigned q_stamp(unsigned long long st) { return (unsigned)(st >> 32); }
__device__ __forceinline__ int q_rank(unsigned long long st) { return (int)((st >> 16) & 0xFFFFu); }
__device__ __forceinline__ int q_words(unsigned long long st) { return (int)(st & 0xFFFFu); }

__global__ void kfdb_begin_kernel(int loop, unsigned qid, const int *__restrict__ connected, int nconn, int K, unsigned *__restrict__ conn,
                                  int *__restrict__ info) {
    if (blockIdx.x == 0 && threadIdx.x == 0) info[0] = 0;   // touched count
    if (!loop) return;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nconn; i += gridDim.x * blockDim.x) {
        const int c = connected[i];
        if ((unsigned)c < (unsigned)K) conn[c] = qid;
    }
}

__global__ void __launch_bounds__(128) kfdb_walk_kernel(unsigned qid, int nq, const int *__restrict__ q_ids, int nwords,
                                                        const int *__restrict__ w_head, const int *__restrict__ n_slot,
                                                        const int *__restrict__ n_next, unsigned long long *__restrict__ state,
                                                        int *__restrict__ touched, int *__restrict__ info) {
    const int qi = blockIdx.x * blockDim.x + threadIdx.x;
    if (qi >= nq) return;
    const int w = q_ids[qi];
    if ((unsigned)w >= (unsigned)nwords) return;
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

// info: [0] touched, [1] list length, [2] minCommonWords
__global__ void __launch_bounds__(KFDB_BLOCK) kfdb_order_kernel(int loop, unsigned qid, const unsigned long long *__restrict__ state,
                                                                const unsigned *__restrict__ conn, const unsigned *__restrict__ seqs,
                                                                const int *__restrict__ touched, int *__restrict__ info,
                                                                unsigned long long *__restrict__ keys, int *__restrict__ list, int K) {
    __shared__ int sh[2];   // [0] list length, [1] maxCommonWords
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

__global__ void __launch_bounds__(128) kfdb_score_kernel(int loop, int nq, const int *__restrict__ q_ids, const double *__restrict__ q_vals,
                                                         const int *__restrict__ info, const int *__restrict__ list, const int *__restrict__ range,
                                                         const int *__restrict__ s_id, const double *__restrict__ s_val, float *__restrict__ lsc,
                                                         float *__restrict__ lscore, float *__restrict__ rscore) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= info[1]) return;
    const int s = list[e];
    int common, first;
    const float si = (float)bow_l1_walk(nq, q_ids, q_vals, range[2 * s], range[2 * s + 1], s_id, s_val, common, first);
    lsc[e] = si;
    if (loop) lscore[s] = si; else rscore[s] = si;   // pKFi->mLoopScore / mRelocScore = si
}

__global__ void __launch_bounds__(KFDB_BLOCK) kfdb_select_kernel(int loop, unsigned qid, float min_score, int K, const int *__restrict__ info,
                                                                 const int *__restrict__ list, const float *__restrict__ lsc,
                                                                 const unsigned long long *__restrict__ state, const unsigned *__restrict__ conn,
                                                                 const float *__restrict__ lscore, const float *__restrict__ rscore,
                                                                 const int *__restrict__ covn, const int *__restrict__ cov,
                                                                 const int *__restrict__ touched, float *__restrict__ acc, int *__restrict__ best,
                                                                 unsigned long long *__restrict__ firstpos, int cap, int *__restrict__ cand,
                                                                 int *__restrict__ ncand, int *__restrict__ words_out, float *__restrict__ score_out) {
    __shared__ float s_best, s_wmax[KFDB_BLOCK / 32];
    __shared__ int s_cnt[KFDB_BLOCK / 32];
    __shared__ int s_base;
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
            if (score_out) score_out[s] = sc[s];
        }
    }
    if (threadIdx.x == 0) { s_best = loop ? min_score : 0.f; s_base = 0; }
    __syncthreads();
    // lAccScoreAndMatch, one entry per lScoreAndMatch entry (loop mode keeps si >= minScore, :135)
    float mybest = -INFINITY;
    for (int e = threadIdx.x; e < nl; e += blockDim.x) {
        const int s = list[e];
        const float si = lsc[e];
        if (loop && !(si >= min_score)) { best[e] = -1; continue; }
        float bestScore = si, accScore = si;
        int b = s;
        const int nc = covn[s];
        for (int j = 0; j < nc; j++) {
            const int s2 = cov[s * KFDB_COVIS + j];
            const unsigned long long st = state[s2];
            if (q_stamp(st) != qid) continue;                                              // mnLoopQuery / mnRelocQuery
            if (loop && (conn[s2] == qid || !(q_words(st) > minCommon))) continue;         // :158
            const float s2c = sc[s2];
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

#define KFDB_TRY(expr)                                                                                       \
    do {                                                                                                     \
        cudaError_t e__ = (expr);                                                                            \
        if (e__ != cudaSuccess)                                                                              \
            return set_error(ORBFE_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
    } while (0)

struct OrbfeKeyFrameDB {
    int device = 0, nwords = 0, K = 0, sortcap = 1;
    long long P = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t last = nullptr;   // the handle's most recent work: every call orders itself after it
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
    unsigned long long *state = nullptr, *keys = nullptr, *firstpos = nullptr;
    float *lscore = nullptr, *rscore = nullptr, *lsc = nullptr, *acc = nullptr;
    // staging of the host-pointer detect
    int *q_ids = nullptr, *q_conn = nullptr, *o_cand = nullptr, *o_words = nullptr, *o_n = nullptr;
    double *q_vals = nullptr;
    float *o_score = nullptr;
};

#define KFDB_MAX_NQ 65535   // the shared-word rank and count are 16-bit fields of the query state

extern "C" void orbfe_kfdb_destroy(OrbfeKeyFrameDB *db) {
    if (!db) return;
    cudaSetDevice(db->device);
    if (db->stream) cudaStreamSynchronize(db->stream);
    void *ptrs[] = {db->s_id[0], db->s_id[1], db->s_node[0], db->s_node[1], db->s_val[0], db->s_val[1], db->n_slot, db->n_next, db->n_prev,
                    db->w_head, db->w_tail, db->range, db->covn, db->cov, db->touched, db->list, db->best, db->info, db->moves, db->covrows,
                    db->seqs, db->conn, db->state, db->keys, db->firstpos, db->lscore, db->rscore, db->lsc, db->acc, db->q_ids, db->q_conn,
                    db->o_cand, db->o_words, db->o_n, db->q_vals, db->o_score, db->a_info};
    for (void *p : ptrs) cudaFree(p);
    if (db->last) cudaEventDestroy(db->last);
    if (db->stream) cudaStreamDestroy(db->stream);
    delete db;
}

static int kfdb_reset(OrbfeKeyFrameDB *db) {
    db->begin.assign(db->K, 0);
    db->len.assign(db->K, -1);
    db->nodes.assign(db->K, std::vector<int>());
    db->free_nodes.resize((size_t)db->P);
    for (long long i = 0; i < db->P; i++) db->free_nodes[(size_t)i] = (int)(db->P - 1 - i);   // pops 0, 1, 2, ...
    db->top = db->live = 0;
    cudaStream_t s = db->stream;
    KFDB_TRY(cudaMemsetAsync(db->w_head, 0xFF, sizeof(int) * (size_t)db->nwords, s));
    KFDB_TRY(cudaMemsetAsync(db->w_tail, 0xFF, sizeof(int) * (size_t)db->nwords, s));
    std::vector<int> r(2 * (size_t)db->K);
    for (int k = 0; k < db->K; k++) { r[2 * k] = 0; r[2 * k + 1] = -1; }
    KFDB_TRY(cudaMemcpyAsync(db->range, r.data(), sizeof(int) * r.size(), cudaMemcpyHostToDevice, s));
    KFDB_TRY(cudaMemsetAsync(db->covn, 0, sizeof(int) * (size_t)db->K, s));
    KFDB_TRY(cudaStreamSynchronize(s));
    return ORBFE_OK;
}

extern "C" int orbfe_kfdb_create(OrbfeVocabulary *v, int max_keyframes, long long max_postings, OrbfeKeyFrameDB **out) {
    if (!out) return set_error(ORBFE_ERR_ARG, "NULL out");
    *out = nullptr;
    if (!v || max_keyframes < 1 || max_keyframes > (1 << 24) || max_postings < 1 || max_postings > 0x7FFFFFFFLL)
        return set_error(ORBFE_ERR_ARG, "bad arguments (1 <= max_keyframes <= 2^24, 1 <= max_postings < 2^31)");
    OrbfeKeyFrameDB *db = new OrbfeKeyFrameDB();
    db->device = vocab_device(v);
    db->nwords = std::max(vocab_nwords(v), 1);
    db->K = max_keyframes;
    db->P = max_postings;
    while (db->sortcap < db->K) db->sortcap <<= 1;
    const size_t K = (size_t)db->K, P = (size_t)db->P, W = (size_t)db->nwords, S = (size_t)db->sortcap;
    bool ok = cudaSetDevice(db->device) == cudaSuccess && cudaStreamCreateWithFlags(&db->stream, cudaStreamNonBlocking) == cudaSuccess &&
              cudaEventCreateWithFlags(&db->last, cudaEventDisableTiming) == cudaSuccess;
#define KFDB_ALLOC(p, n) ok = ok && cudaMalloc((void **)&(p), sizeof(*(p)) * (n)) == cudaSuccess
    for (int h = 0; h < 2; h++) { KFDB_ALLOC(db->s_id[h], P); KFDB_ALLOC(db->s_node[h], P); KFDB_ALLOC(db->s_val[h], P); }
    KFDB_ALLOC(db->n_slot, P); KFDB_ALLOC(db->n_next, P); KFDB_ALLOC(db->n_prev, P);
    KFDB_ALLOC(db->w_head, W); KFDB_ALLOC(db->w_tail, W);
    KFDB_ALLOC(db->range, 2 * K); KFDB_ALLOC(db->covn, K); KFDB_ALLOC(db->cov, K * KFDB_COVIS); KFDB_ALLOC(db->touched, K);
    KFDB_ALLOC(db->list, S); KFDB_ALLOC(db->best, K); KFDB_ALLOC(db->info, 4); KFDB_ALLOC(db->moves, 3 * K);
    KFDB_ALLOC(db->covrows, K * (2 + KFDB_COVIS)); KFDB_ALLOC(db->seqs, K); KFDB_ALLOC(db->conn, K); KFDB_ALLOC(db->state, K);
    KFDB_ALLOC(db->keys, S); KFDB_ALLOC(db->firstpos, K); KFDB_ALLOC(db->lscore, K); KFDB_ALLOC(db->rscore, K); KFDB_ALLOC(db->lsc, K);
    KFDB_ALLOC(db->acc, K); KFDB_ALLOC(db->q_ids, KFDB_MAX_NQ); KFDB_ALLOC(db->q_vals, KFDB_MAX_NQ); KFDB_ALLOC(db->q_conn, K);
    KFDB_ALLOC(db->o_cand, K); KFDB_ALLOC(db->o_words, K); KFDB_ALLOC(db->o_score, K); KFDB_ALLOC(db->o_n, 1);
    KFDB_ALLOC(db->a_info, K + 1);
#undef KFDB_ALLOC
    ok = ok && cudaMemset(db->conn, 0, sizeof(unsigned) * K) == cudaSuccess && cudaMemset(db->state, 0, sizeof(unsigned long long) * K) == cudaSuccess &&
         cudaMemset(db->firstpos, 0xFF, sizeof(unsigned long long) * K) == cudaSuccess;
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

// order the handle's stream after the handle's previous work (which may have been enqueued on another stream)
static int kfdb_enter(OrbfeKeyFrameDB *db, cudaStream_t s) {
    KFDB_TRY(cudaSetDevice(db->device));
    KFDB_TRY(cudaStreamWaitEvent(s, db->last, 0));
    return ORBFE_OK;
}
static int kfdb_leave(OrbfeKeyFrameDB *db, cudaStream_t s, bool sync) {
    KFDB_TRY(cudaGetLastError());
    KFDB_TRY(cudaEventRecord(db->last, s));
    if (sync) KFDB_TRY(cudaStreamSynchronize(s));
    return ORBFE_OK;
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
    cudaStream_t s = db->stream;
    const int o = db->cur, n = 1 - db->cur;
    const int nmove = (int)order.size();
    if (nmove > 0) {
        KFDB_TRY(cudaMemcpyAsync(db->moves, moves.data(), sizeof(int) * moves.size(), cudaMemcpyHostToDevice, s));
        kfdb_compact_kernel<<<std::min(nmove, 1024), 256, 0, s>>>(db->moves, nmove, db->s_id[o], db->s_val[o], db->s_node[o], db->s_id[n],
                                                                  db->s_val[n], db->s_node[n]);
    }
    KFDB_TRY(cudaMemcpyAsync(db->range, r.data(), sizeof(int) * r.size(), cudaMemcpyHostToDevice, s));
    KFDB_TRY(cudaStreamSynchronize(s));   // `moves` / `r` are host locals
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
    cudaStream_t s = db->stream;
    int rc = kfdb_enter(db, s);
    if (rc) return rc;
    if (db->top + nw > db->P && (rc = kfdb_compact(db))) return rc;
    std::vector<int> nodes(nw);
    for (int i = 0; i < nw; i++) { nodes[i] = db->free_nodes.back(); db->free_nodes.pop_back(); }
    const int base = (int)db->top, c = db->cur;
    if (nw > 0) {
        KFDB_TRY(cudaMemcpyAsync(db->s_id[c] + base, ids, sizeof(int) * nw, cudaMemcpyHostToDevice, s));
        KFDB_TRY(cudaMemcpyAsync(db->s_val[c] + base, vals, sizeof(double) * nw, cudaMemcpyHostToDevice, s));
        KFDB_TRY(cudaMemcpyAsync(db->s_node[c] + base, nodes.data(), sizeof(int) * nw, cudaMemcpyHostToDevice, s));
    }
    kfdb_link_kernel<<<(std::max(nw, 1) + 255) / 256, 256, 0, s>>>(slot, base, nw, ++db->seq, db->s_id[c], db->s_node[c], db->n_slot, db->n_next,
                                                                   db->n_prev, db->w_head, db->w_tail, db->range, db->seqs, db->state,
                                                                   db->lscore, db->rscore);
    if ((rc = kfdb_leave(db, s, true))) return rc;
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
    cudaStream_t s = stream ? (cudaStream_t)stream : db->stream;
    int rc = kfdb_enter(db, s);
    if (rc) return rc;
    KFDB_TRY(cudaMemcpyAsync(db->moves, frames, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, s));
    KFDB_TRY(cudaMemsetAsync(db->a_info, 0, sizeof(int), s));
    kfdb_check_rows_kernel<<<std::min(n, 1024), 256, 0, s>>>(db->moves, n, cap, db->nwords, d_bow_n, d_bow_ids, db->a_info);
    KFDB_TRY(cudaGetLastError());
    std::vector<int> info((size_t)n + 1);
    KFDB_TRY(cudaMemcpyAsync(info.data(), db->a_info, sizeof(int) * info.size(), cudaMemcpyDeviceToHost, s));
    KFDB_TRY(cudaStreamSynchronize(s));
    if (info[0])
        return set_error(ORBFE_ERR_ARG, "a BowVector row has a word count outside 0 .. %d, or word ids that are not strictly ascending below %d",
                         cap, db->nwords);
    long long total = 0;
    for (int i = 0; i < n; i++) total += info[1 + i];
    if (db->live + total > db->P)
        return set_error(ORBFE_ERR_CAPACITY, "%lld postings + %lld exceed max_postings %lld", db->live, total, db->P);
    // `s` has drained: the handle's earlier work and the rows are complete, the rest runs on the handle's stream
    cudaStream_t hs = db->stream;
    if (db->top + total > db->P && (rc = kfdb_compact(db))) return rc;
    const int c = db->cur, top = (int)db->top;
    std::vector<int> rows(3 * (size_t)n), nodes((size_t)total);
    for (int i = 0, pos = 0; i < n; i++) {
        rows[3 * i] = frames[i];
        rows[3 * i + 1] = top + pos;
        rows[3 * i + 2] = info[1 + i];
        for (int k = 0; k < info[1 + i]; k++, pos++) { nodes[pos] = db->free_nodes.back(); db->free_nodes.pop_back(); }
    }
    KFDB_TRY(cudaMemcpyAsync(db->moves, rows.data(), sizeof(int) * rows.size(), cudaMemcpyHostToDevice, hs));
    if (total > 0) KFDB_TRY(cudaMemcpyAsync(db->s_node[c] + top, nodes.data(), sizeof(int) * nodes.size(), cudaMemcpyHostToDevice, hs));
    kfdb_gather_kernel<<<std::min(n, 1024), 256, 0, hs>>>(db->moves, n, cap, d_bow_ids, d_bow_vals, db->s_id[c], db->s_val[c]);
    // one keyframe after the other: two keyframes may share a word, and every word's list is in add order
    for (int i = 0; i < n; i++) {
        const int nw = rows[3 * i + 2];
        kfdb_link_kernel<<<(std::max(nw, 1) + 255) / 256, 256, 0, hs>>>(slots[i], rows[3 * i + 1], nw, ++db->seq, db->s_id[c], db->s_node[c],
                                                                        db->n_slot, db->n_next, db->n_prev, db->w_head, db->w_tail,
                                                                        db->range, db->seqs, db->state, db->lscore, db->rscore);
    }
    if ((rc = kfdb_leave(db, hs, true))) return rc;
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
    cudaStream_t s = db->stream;
    int rc = kfdb_enter(db, s);
    if (rc) return rc;
    const int nw = db->len[slot];
    kfdb_unlink_kernel<<<(std::max(nw, 1) + 255) / 256, 256, 0, s>>>(slot, db->begin[slot], nw, db->s_id[db->cur], db->s_node[db->cur], db->n_next,
                                                                     db->n_prev, db->w_head, db->w_tail, db->range, db->covn);
    if ((rc = kfdb_leave(db, s, true))) return rc;
    for (int nd : db->nodes[slot]) db->free_nodes.push_back(nd);
    db->nodes[slot].clear();
    if (db->begin[slot] + nw == db->top) db->top -= nw;   // the last rows: the tail shrinks back
    db->live -= nw;
    db->len[slot] = -1;
    return ORBFE_OK;
}

extern "C" int orbfe_kfdb_clear(OrbfeKeyFrameDB *db) {
    if (!db) return set_error(ORBFE_ERR_ARG, "bad arguments");
    int rc = kfdb_enter(db, db->stream);
    if (rc) return rc;
    if ((rc = kfdb_reset(db))) return rc;
    return kfdb_leave(db, db->stream, true);
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
    cudaStream_t s = db->stream;
    int rc = kfdb_enter(db, s);
    if (rc) return rc;
    KFDB_TRY(cudaMemcpyAsync(db->covrows, rows.data(), sizeof(int) * rows.size(), cudaMemcpyHostToDevice, s));
    kfdb_covis_kernel<<<(n + 127) / 128, 128, 0, s>>>(db->covrows, n, db->covn, db->cov);
    return kfdb_leave(db, s, true);
}

static int kfdb_check_detect(int mode, int nq, int nconn, int cap) {
    if (mode < 0 || mode > 1) return set_error(ORBFE_ERR_ARG, "mode must be 0 (loop) or 1 (relocalisation)");
    if (nq < 0 || nq > KFDB_MAX_NQ) return set_error(ORBFE_ERR_ARG, "nq %d out of range (0 .. %d)", nq, KFDB_MAX_NQ);
    if (nconn < 0) return set_error(ORBFE_ERR_ARG, "nconn < 0");
    if (cap < 0) return set_error(ORBFE_ERR_ARG, "cap < 0");
    return ORBFE_OK;
}

extern "C" int orbfe_kfdb_detect_device(OrbfeKeyFrameDB *db, int mode, int nq, const int32_t *d_q_ids, const double *d_q_vals, int nconn,
                                        const int32_t *d_connected, float min_score, int cap, int32_t *d_cand, int *d_ncand,
                                        int32_t *d_words, float *d_score, void *stream) {
    int rc = kfdb_check_detect(mode, nq, nconn, cap);
    if (rc) return rc;
    if (!db || !d_ncand || (nq > 0 && (!d_q_ids || !d_q_vals)) || (mode == 0 && nconn > 0 && !d_connected) || (cap > 0 && !d_cand))
        return set_error(ORBFE_ERR_ARG, "NULL argument");
    cudaStream_t s = stream ? (cudaStream_t)stream : db->stream;
    if ((rc = kfdb_enter(db, s))) return rc;
    const int loop = mode == 0;
    const unsigned qid = ++db->qid;
    const int K = db->K, c = db->cur;
    kfdb_begin_kernel<<<std::max(1, std::min((nconn + 255) / 256, 64)), 256, 0, s>>>(loop, qid, d_connected, loop ? nconn : 0, K, db->conn, db->info);
    if (nq > 0)
        kfdb_walk_kernel<<<(nq + 127) / 128, 128, 0, s>>>(qid, nq, d_q_ids, db->nwords, db->w_head, db->n_slot, db->n_next, db->state,
                                                          db->touched, db->info);
    kfdb_order_kernel<<<1, KFDB_BLOCK, 0, s>>>(loop, qid, db->state, db->conn, db->seqs, db->touched, db->info, db->keys, db->list, K);
    kfdb_score_kernel<<<(K + 127) / 128, 128, 0, s>>>(loop, nq, d_q_ids, d_q_vals, db->info, db->list, db->range, db->s_id[c], db->s_val[c],
                                                      db->lsc, db->lscore, db->rscore);
    kfdb_select_kernel<<<1, KFDB_BLOCK, 0, s>>>(loop, qid, min_score, K, db->info, db->list, db->lsc, db->state, db->conn, db->lscore,
                                                db->rscore, db->covn, db->cov, db->touched, db->acc, db->best, db->firstpos, cap, d_cand,
                                                d_ncand, d_words, d_score);
    return kfdb_leave(db, s, false);
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
    cudaStream_t s = db->stream;
    if ((rc = kfdb_enter(db, s))) return rc;
    if (nq > 0) {
        KFDB_TRY(cudaMemcpyAsync(db->q_ids, q_ids, sizeof(int) * nq, cudaMemcpyHostToDevice, s));
        KFDB_TRY(cudaMemcpyAsync(db->q_vals, q_vals, sizeof(double) * nq, cudaMemcpyHostToDevice, s));
    }
    if (mode == 0 && nconn > 0) KFDB_TRY(cudaMemcpyAsync(db->q_conn, connected, sizeof(int) * nconn, cudaMemcpyHostToDevice, s));
    rc = orbfe_kfdb_detect_device(db, mode, nq, db->q_ids, db->q_vals, mode == 0 ? nconn : 0, db->q_conn, min_score, db->K, db->o_cand,
                                  db->o_n, db->o_words, db->o_score, s);
    if (rc) return rc;
    int n = 0;
    KFDB_TRY(cudaMemcpyAsync(&n, db->o_n, sizeof(int), cudaMemcpyDeviceToHost, s));
    if (words_out) KFDB_TRY(cudaMemcpyAsync(words_out, db->o_words, sizeof(int) * (size_t)db->K, cudaMemcpyDeviceToHost, s));
    if (score_out) KFDB_TRY(cudaMemcpyAsync(score_out, db->o_score, sizeof(float) * (size_t)db->K, cudaMemcpyDeviceToHost, s));
    KFDB_TRY(cudaStreamSynchronize(s));
    *ncand_out = n;
    if (n > cap) return set_error(ORBFE_ERR_CAPACITY, "%d candidates exceed cap %d", n, cap);
    if (n > 0) KFDB_TRY(cudaMemcpy(cand_out, db->o_cand, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost));
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
