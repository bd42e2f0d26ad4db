// bow_kernels.cu -- the two Hamming-primitive rows of SURVEY.md section 8(f):
//   N2  DBoW2 vocabulary-tree descent (reference Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1216-1260, FORB.cpp:79-99)
//   N4  MapPoint::ComputeDistinctiveDescriptors, batched (reference src/MapPoint.cc:185-250)
// plus the device-side half of the C-ABI in include/orbfe_bow.h.  The std::map builds of transform() are restated twice:
// on the host for the host-array orbfe_bow_transform (host/bow_host.cpp), and here for batches of frames in HBM
// (feature_vector_kernel, bow_vector_kernel).  The descent is integer work only (XOR + POPC), bound by launch latency at
// SLAM sizes (2000 descriptors x 6 levels x 10 children = 120 k distances per frame).
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/orbfe_bow.h"
#include "bow_l1.cuh"
#include "orbfe_internal.h"

namespace orbfe {

__device__ __forceinline__ int bow_ham256(const uint4 a0, const uint4 a1, const uint4 b0, const uint4 b1) {
    return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
           __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

// One warp per descriptor; at every level the lanes take the children of the current node (10 in ORBvoc), the
// minimum of (distance << 16 | child position) over the warp is the reference's strict-< scan (first minimum wins).
__global__ void __launch_bounds__(256) bow_descend_kernel(const uint4 *__restrict__ node_desc, const int *__restrict__ child_ptr,
                                                          const int *__restrict__ children, const uint4 *__restrict__ desc,
                                                          int n, int nid_level, int *__restrict__ leaf_out,
                                                          int *__restrict__ node_out) {
    const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n) return;
    const int lane = threadIdx.x & 31;
    const uint4 a0 = __ldg(&desc[2 * i]), a1 = __ldg(&desc[2 * i + 1]);
    int cur = 0, level = 0, nid = 0;
    int cb = __ldg(&child_ptr[0]), ce = __ldg(&child_ptr[1]);
    // do { ... } while (!isLeaf): the root of a non-empty vocabulary has children.  The level cap only guards against a
    // malformed table with a cycle (a DBoW2 tree is a handful of levels deep): the kernel must terminate.
    while (ce > cb && level < 64) {
        level++;
        uint32_t best = 0xFFFFFFFFu;
        for (int c0 = cb; c0 < ce; c0 += 32) {
            const int c = c0 + lane;
            uint32_t key = 0xFFFFFFFFu;
            if (c < ce) {
                const int id = __ldg(&children[c]);
                const int d = bow_ham256(a0, a1, __ldg(&node_desc[2 * id]), __ldg(&node_desc[2 * id + 1]));
                key = ((uint32_t)d << 16) | (uint32_t)min(c - cb, 0xFFFF);
            }
            best = min(best, __reduce_min_sync(0xffffffffu, key));
        }
        cur = __ldg(&children[cb + (int)(best & 0xFFFF)]);
        if (level == nid_level) nid = cur;
        cb = __ldg(&child_ptr[cur]);
        ce = __ldg(&child_ptr[cur + 1]);
    }
    if (lane == 0) {
        leaf_out[i] = cur;
        node_out[i] = nid;
    }
}

// One warp per map point.  Row i of the N x N distance matrix is histogrammed (257 bins) in shared memory and the
// (int)(0.5*(N-1))-th smallest entry read off the cumulative counts; the first row with the least median wins.
// kObs = false (orbfe_distinctive_descriptors): descriptor j of group g is row group_ptr[g] + j of `desc`, and the host
// has checked group_ptr.  kObs = true (orbfe_distinctive_descriptors_device): it is row obs[group_ptr[g] + j] of the frame
// store (slot f*cap + i); a group whose pointers or observations are out of range is never followed (best -1, its
// mp_desc row untouched, bit 8 of *err), and the chosen 32 bytes are copied to row g of mp_desc.
template <bool kObs>
__global__ void __launch_bounds__(128) distinctive_kernel(const uint4 *__restrict__ desc, const int *__restrict__ group_ptr,
                                                          const int *__restrict__ obs, int nobs, const int *__restrict__ counts,
                                                          int nframes, int cap, int ngroups, int *__restrict__ best_out,
                                                          uint4 *__restrict__ mp_desc, int *__restrict__ err) {
    __shared__ int hist[4][288];
    const int wq = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = blockIdx.x * 4 + wq;
    if (g >= ngroups) return;
    const int b = __ldg(&group_ptr[g]), e = __ldg(&group_ptr[g + 1]);
    if (kObs) {
        bool bad = b < 0 || b > e || e > nobs;
        if (!bad) {
            bool mine = false;
            for (int j = b + lane; j < e; j += 32) {
                const int o = __ldg(&obs[j]);
                mine |= o < 0 || o / cap >= nframes || o % cap >= __ldg(&counts[o / cap]);
            }
            bad = __any_sync(0xffffffffu, mine);
        }
        if (bad) {
            if (lane == 0) { best_out[g] = -1; atomicOr(err, 8); }
            return;
        }
    }
    const int N = e - b;
    if (N <= 0) {
        if (lane == 0) best_out[g] = -1;
        return;
    }
    auto row = [&](int j) -> size_t { return kObs ? (size_t)__ldg(&obs[b + j]) : (size_t)(b + j); };
    const int k = (N - 1) >> 1;  // vDists[0.5*(N-1)]
    int *h = hist[wq];
    int bestMedian = 0x7FFFFFFF, bestIdx = 0;
    for (int i = 0; i < N; i++) {
        for (int t = lane; t < 288; t += 32) h[t] = 0;
        __syncwarp();
        const size_t ri = row(i);
        const uint4 a0 = __ldg(&desc[2 * ri]), a1 = __ldg(&desc[2 * ri + 1]);
        for (int j = lane; j < N; j += 32) {
            const size_t rj = row(j);
            const int d = bow_ham256(a0, a1, __ldg(&desc[2 * rj]), __ldg(&desc[2 * rj + 1]));
            atomicAdd(&h[d], 1);
        }
        __syncwarp();
        // lane L owns bins 9L .. 9L+8 (288 >= 257 bins)
        int c[9], sum = 0;
#pragma unroll
        for (int t = 0; t < 9; t++) { c[t] = h[9 * lane + t]; sum += c[t]; }
        int incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        const int fl = __ffs(__ballot_sync(0xffffffffu, incl > k)) - 1;  // lane whose bins hold the k-th smallest
        int median = 0;
        if (lane == fl) {
            int run = incl - sum;
#pragma unroll
            for (int t = 0; t < 9; t++) {
                run += c[t];
                if (run > k) { median = 9 * lane + t; break; }
            }
        }
        median = __shfl_sync(0xffffffffu, median, fl);
        if (median < bestMedian) { bestMedian = median; bestIdx = i; }
        __syncwarp();
    }
    if (lane == 0) best_out[g] = bestIdx;
    if (kObs && lane < 2) mp_desc[2 * (size_t)g + lane] = __ldg(&desc[2 * row(bestIdx) + lane]);
}

// KeyFrameDatabase scoring: one thread per keyframe, the shared L1 walk (bow_l1.cuh) over the word lists of the query and
// of the keyframe.
__global__ void __launch_bounds__(128) bow_db_score_kernel(int nq, const int *__restrict__ q_ids, const double *__restrict__ q_vals,
                                                           int nkf, const int *__restrict__ kf_ptr, const int *__restrict__ db_ids,
                                                           const double *__restrict__ db_vals, int *__restrict__ common_out,
                                                           int *__restrict__ first_out, double *__restrict__ score_out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nkf) return;
    const int b = __ldg(&kf_ptr[k]);
    const int be = __ldg(&kf_ptr[k + 1]);
    int common, first;
    const double score = bow_l1_walk(nq, q_ids, q_vals, b, be, db_ids, db_vals, common, first);
    common_out[k] = common;
    first_out[k] = first;
    score_out[k] = score;
}

void launch_bow_db_score(int nq, const int *q_ids, const double *q_vals, int nkf, const int *kf_ptr, const int *db_ids,
                         const double *db_vals, int *common, int *first, double *score, cudaStream_t s) {
    if (nkf <= 0) return;
    bow_db_score_kernel<<<(nkf + 127) / 128, 128, 0, s>>>(nq, q_ids, q_vals, nkf, kf_ptr, db_ids, db_vals, common, first, score);
}

// The two std::map builds of transform() (TemplatedVocabulary.h:1126-1196) on the device, one CTA per frame.  Both group
// a frame's kept features by a 32-bit id (the node of the FeatureVector, the word of the BowVector) in feature order:
// the (id << 32 | feature index) keys are unique, so an ascending bitonic sort in shared memory is the stable sort by id,
// and a block scan over the run heads numbers the ids.
#define FV_THREADS 1024

// Writes the keys of frame features [0, n) into keys[0, n2) (n2 = the power of two >= n): key(i) for a kept feature, ~0 (sorts
// last) otherwise; returns the number kept.  A feature whose word has weight 0 (a stopped word) is dropped
// (TemplatedVocabulary.h:1175, `if (w > 0)`); a leaf id outside the vocabulary counts as stopped.
template <class Key>
__device__ __forceinline__ int fv_fill_keys(unsigned long long *keys, int n, int n2, const int *__restrict__ lf,
                                            const uint8_t *__restrict__ live, int nnodes, Key key) {
    int nk = 0;
    for (int c0 = 0; c0 < n2; c0 += FV_THREADS) {
        const int i = c0 + threadIdx.x;
        bool keep = false;
        if (i < n2) {
            int l = -1;
            if (i < n) {
                l = lf[i];
                keep = (unsigned)l < (unsigned)nnodes && live[l];
            }
            keys[i] = keep ? ((unsigned long long)key(i, l) << 32) | (uint32_t)i : ~0ull;
        }
        nk += __syncthreads_count(keep);
    }
    return nk;
}

// Ascending block-wide bitonic sort of keys[0, n2), n2 a power of two.
__device__ __forceinline__ void fv_sort_keys(unsigned long long *keys, int n2) {
    for (int k = 2; k <= n2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n2; i += FV_THREADS) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long x = keys[i], y = keys[ixj];
                    if (((i & k) == 0) ? (x > y) : (x < y)) { keys[i] = y; keys[ixj] = x; }
                }
            }
            __syncthreads();
        }
    }
}

// Walks the sorted keys[0, nk): visit(i, key, head, r) for every position i, where head marks the first key of a run of
// equal ids and r (valid at a head) numbers the runs in ascending id order.  Returns the number of runs.
template <class Visit>
__device__ __forceinline__ int fv_scan_runs(const unsigned long long *keys, int nk, int *s_warp, Visit visit) {
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    int base = 0;   // runs started before this chunk
    for (int c0 = 0; c0 < nk; c0 += FV_THREADS) {
        const int i = c0 + tid;
        unsigned long long key = 0;
        bool head = false;
        if (i < nk) {
            key = keys[i];
            head = i == 0 || (uint32_t)(keys[i - 1] >> 32) != (uint32_t)(key >> 32);
        }
        // exclusive scan of the head flags over the block
        const unsigned bal = __ballot_sync(0xffffffffu, head);
        if (lane == 0) s_warp[wid] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
        for (int w = 0; w < FV_THREADS / 32; w++) {
            const int c = s_warp[w];
            if (w < wid) before += c;
            total += c;
        }
        if (i < nk) visit(i, key, head, base + before + __popc(bal & ((1u << lane) - 1u)));
        base += total;
        __syncthreads();   // s_warp is rewritten by the next chunk
    }
    return base;
}

// DBoW2::FeatureVector of every frame from the per-feature node ids (TemplatedVocabulary.h:1180-1190 adds feature i to
// node nid[i] in index order).
__global__ void __launch_bounds__(FV_THREADS) feature_vector_kernel(const int *__restrict__ leaf, const int *__restrict__ node,
                                                                    const uint8_t *__restrict__ live, int nnodes,
                                                                    const int *__restrict__ counts, int cap, int *__restrict__ fv_ids,
                                                                    int *__restrict__ fv_ptr, int *__restrict__ fv_items,
                                                                    int *__restrict__ fv_n) {
    extern __shared__ unsigned long long fkeys[];   // [n2]
    __shared__ int s_warp[FV_THREADS / 32];
    const int f = blockIdx.x;
    const int n = min(max(counts[f], 0), cap);
    int n2 = 1;
    while (n2 < n) n2 <<= 1;
    const int *__restrict__ nd = node + (size_t)f * cap;
    const int nk = fv_fill_keys(fkeys, n, n2, leaf + (size_t)f * cap, live, nnodes, [&](int i, int) { return (uint32_t)nd[i]; });
    fv_sort_keys(fkeys, n2);
    int *__restrict__ ids = fv_ids + (size_t)f * cap;
    int *__restrict__ ptr = fv_ptr + (size_t)f * (cap + 1);
    int *__restrict__ items = fv_items + (size_t)f * cap;
    const int nn = fv_scan_runs(fkeys, nk, s_warp, [&](int i, unsigned long long key, bool head, int r) {
        items[i] = (int)(uint32_t)key;
        if (head) {
            ids[r] = (int)(uint32_t)(key >> 32);
            ptr[r] = i;
        }
    });
    if (threadIdx.x == 0) {
        ptr[nn] = nk;
        fv_n[f] = nn;
    }
}

// DBoW2::BowVector of every frame from the per-feature leaf ids (TemplatedVocabulary.h:1126-1172, BowVector.cpp:34-84).  Word
// ids are keyed with the sign bit flipped, so that the unsigned key order is the signed word order of the std::map.  The
// thread at the head of a word's run takes that word's values in feature order (first inserted; TF / TF-IDF add the others,
// IDF / BINARY keep the first) and writes the word to the output row; the values stay out of shared memory, which holds the
// keys.  The norm is one sequential sum in ascending word order, as BowVector::normalize takes it: a tree reduction would
// round differently.
__global__ void __launch_bounds__(FV_THREADS) bow_vector_kernel(const int *__restrict__ leaf, const uint8_t *__restrict__ live,
                                                                const int *__restrict__ word_id, const double *__restrict__ weight,
                                                                int nnodes, int accumulate, int norm, const int *__restrict__ counts,
                                                                int cap, int *__restrict__ bow_ids, double *__restrict__ bow_vals,
                                                                int *__restrict__ bow_n) {
    extern __shared__ unsigned long long wkeys[];   // [n2]
    __shared__ int s_warp[FV_THREADS / 32];
    __shared__ double s_norm;
    const int f = blockIdx.x, tid = threadIdx.x;
    const int n = min(max(counts[f], 0), cap);
    int n2 = 1;
    while (n2 < n) n2 <<= 1;
    const int *__restrict__ lf = leaf + (size_t)f * cap;
    const int nk = fv_fill_keys(wkeys, n, n2, lf, live, nnodes, [&](int, int l) { return (uint32_t)__ldg(&word_id[l]) ^ 0x80000000u; });
    fv_sort_keys(wkeys, n2);
    int *__restrict__ ids = bow_ids + (size_t)f * cap;
    double *__restrict__ vals = bow_vals + (size_t)f * cap;
    const int nw = fv_scan_runs(wkeys, nk, s_warp, [&](int i, unsigned long long key, bool head, int r) {
        if (!head) return;
        const uint32_t w = (uint32_t)(key >> 32);
        double v = __ldg(&weight[lf[(uint32_t)key]]);   // insert(id, w)
        if (accumulate)
            for (int j = i + 1; j < nk && (uint32_t)(wkeys[j] >> 32) == w; j++)
                v = __dadd_rn(v, __ldg(&weight[lf[(uint32_t)wkeys[j]]]));   // addWeight
        ids[r] = (int)(w ^ 0x80000000u);
        vals[r] = v;
    });
    // fv_scan_runs ends on a barrier: every word's value is in `vals`.  The division loops stay rolled: an unrolled copy
    // spills around the calls of the division's slow path.
    if (norm == ORBFE_BOW_NORM_NONE) {
        if (accumulate && nw > 0) {
            const double d = (double)nw;
#pragma unroll 1
            for (int k = tid; k < nw; k += FV_THREADS) vals[k] = __ddiv_rn(vals[k], d);
        }
    } else {
        if (tid == 0) {
            double s = 0.0;
            if (norm == ORBFE_BOW_NORM_L1) {
                for (int k = 0; k < nw; k++) s = __dadd_rn(s, fabs(vals[k]));
            } else {
                for (int k = 0; k < nw; k++) s = __dadd_rn(s, __dmul_rn(vals[k], vals[k]));
                s = __dsqrt_rn(s);
            }
            s_norm = s;
        }
        __syncthreads();
        const double s = s_norm;
        if (s > 0.0)
#pragma unroll 1
            for (int k = tid; k < nw; k += FV_THREADS) vals[k] = __ddiv_rn(vals[k], s);
    }
    // the padding a keyframe database query skips (word id >= the word count)
    for (int k = nw + tid; k < cap; k += FV_THREADS) {
        ids[k] = INT32_MAX;
        vals[k] = 0.0;
    }
    if (tid == 0) bow_n[f] = nw;
}

// Shared memory of one frame's keys: cap <= ORBFE_FV_MAX_CAP, at most 16384 keys = 128 KB.
template <class Kernel>
static cudaError_t fv_smem(Kernel kernel, int cap, size_t *smem) {
    int n2 = 1;
    while (n2 < cap) n2 <<= 1;
    *smem = sizeof(unsigned long long) * (size_t)n2;
    if (*smem > 48 * 1024) return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*smem);
    return cudaSuccess;
}

static int launch_feature_vector(int nframes, const int *d_leaf, const int *d_node, const uint8_t *d_live, int nnodes,
                                 const int *d_counts, int cap, int *d_ids, int *d_ptr, int *d_items, int *d_n, cudaStream_t s) {
    if (nframes <= 0) return 0;
    size_t smem = 0;
    const cudaError_t e = fv_smem(feature_vector_kernel, cap, &smem);
    if (e != cudaSuccess) return (int)e;
    feature_vector_kernel<<<nframes, FV_THREADS, smem, s>>>(d_leaf, d_node, d_live, nnodes, d_counts, cap, d_ids, d_ptr, d_items, d_n);
    return 0;
}

}  // namespace orbfe

using namespace orbfe;

#define BOW_TRY(expr)                                                                                        \
    do {                                                                                                     \
        cudaError_t e__ = (expr);                                                                            \
        if (e__ != cudaSuccess)                                                                              \
            return set_error(ORBFE_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
    } while (0)

struct OrbfeVocabulary {
    int device = 0, nnodes = 0, depth = 0, weighting = 0, norm = 0;
    cudaStream_t stream = nullptr;
    uint8_t *d_desc = nullptr;
    uint8_t *d_live = nullptr;      // per node: weight > 0 (the FeatureVector skips stopped words)
    int *d_child_ptr = nullptr, *d_children = nullptr;
    int *d_word_id = nullptr;       // per node, for the BowVector kernel
    double *d_weight = nullptr;
    std::vector<int32_t> word_id;   // per node, host side (leaf -> word)
    std::vector<double> weight;
    // grow-only staging of the host-pointer entry point
    uint8_t *d_in = nullptr;
    int *d_out = nullptr;
    size_t in_cap = 0, out_cap = 0;
};

extern "C" void orbfe_vocabulary_destroy(OrbfeVocabulary *v) {
    if (!v) return;
    cudaSetDevice(v->device);
    if (v->stream) cudaStreamDestroy(v->stream);
    cudaFree(v->d_desc); cudaFree(v->d_live); cudaFree(v->d_child_ptr); cudaFree(v->d_children); cudaFree(v->d_in); cudaFree(v->d_out);
    cudaFree(v->d_word_id); cudaFree(v->d_weight);
    delete v;
}

extern "C" OrbfeVocabulary *orbfe_vocabulary_create(int device, int nnodes, int depth_L, const uint8_t *node_desc,
                                                    const int32_t *child_ptr, const int32_t *children, const int32_t *word_id,
                                                    const double *weight, int weighting, int norm) {
    if (nnodes < 1 || depth_L < 0 || !node_desc || !child_ptr || !word_id || !weight || weighting < 0 || weighting > 3 || norm < 0 ||
        norm > 2) {
        set_error(ORBFE_ERR_ARG, "bad vocabulary arguments");
        return nullptr;
    }
    const int nchild = child_ptr[nnodes];
    if (child_ptr[0] != 0 || nchild < 0 || (nchild > 0 && !children)) { set_error(ORBFE_ERR_ARG, "bad child_ptr"); return nullptr; }
    for (int i = 0; i < nnodes; i++)
        if (child_ptr[i + 1] < child_ptr[i]) { set_error(ORBFE_ERR_ARG, "child_ptr must be non-decreasing"); return nullptr; }
    for (int c = 0; c < nchild; c++)
        if (children[c] <= 0 || children[c] >= nnodes) { set_error(ORBFE_ERR_ARG, "child id out of range"); return nullptr; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        set_error(ORBFE_ERR_NO_DEVICE, "no CUDA device: this library has no CPU fallback");
        return nullptr;
    }
    if (device < 0 || device >= ndev) { set_error(ORBFE_ERR_ARG, "device %d out of range", device); return nullptr; }
    OrbfeVocabulary *v = new OrbfeVocabulary();
    v->device = device; v->nnodes = nnodes; v->depth = depth_L; v->weighting = weighting; v->norm = norm;
    v->word_id.assign(word_id, word_id + nnodes);
    v->weight.assign(weight, weight + nnodes);
    std::vector<uint8_t> live(nnodes);
    for (int i = 0; i < nnodes; i++) live[i] = weight[i] > 0 ? 1 : 0;
    bool ok = cudaSetDevice(device) == cudaSuccess && cudaStreamCreateWithFlags(&v->stream, cudaStreamNonBlocking) == cudaSuccess &&
              cudaMalloc((void **)&v->d_desc, (size_t)nnodes * 32) == cudaSuccess &&
              cudaMalloc((void **)&v->d_live, (size_t)nnodes) == cudaSuccess &&
              cudaMemcpy(v->d_live, live.data(), (size_t)nnodes, cudaMemcpyHostToDevice) == cudaSuccess &&
              cudaMalloc((void **)&v->d_word_id, sizeof(int) * (size_t)nnodes) == cudaSuccess &&
              cudaMemcpy(v->d_word_id, word_id, sizeof(int) * (size_t)nnodes, cudaMemcpyHostToDevice) == cudaSuccess &&
              cudaMalloc((void **)&v->d_weight, sizeof(double) * (size_t)nnodes) == cudaSuccess &&
              cudaMemcpy(v->d_weight, weight, sizeof(double) * (size_t)nnodes, cudaMemcpyHostToDevice) == cudaSuccess &&
              cudaMalloc((void **)&v->d_child_ptr, sizeof(int) * ((size_t)nnodes + 1)) == cudaSuccess &&
              cudaMalloc((void **)&v->d_children, sizeof(int) * (size_t)std::max(nchild, 1)) == cudaSuccess &&
              cudaMemcpy(v->d_desc, node_desc, (size_t)nnodes * 32, cudaMemcpyHostToDevice) == cudaSuccess &&
              cudaMemcpy(v->d_child_ptr, child_ptr, sizeof(int) * ((size_t)nnodes + 1), cudaMemcpyHostToDevice) == cudaSuccess &&
              (nchild == 0 || cudaMemcpy(v->d_children, children, sizeof(int) * (size_t)nchild, cudaMemcpyHostToDevice) == cudaSuccess);
    if (!ok) {
        set_error(ORBFE_ERR_CUDA, "vocabulary upload failed: %s", cudaGetErrorString(cudaGetLastError()));
        orbfe_vocabulary_destroy(v);
        return nullptr;
    }
    return v;
}

extern "C" int orbfe_bow_descend_device(OrbfeVocabulary *v, const uint8_t *d_desc, int n, int levelsup, int32_t *d_leaf_out,
                                        int32_t *d_node_out, void *stream) {
    if (!v || n < 0) return set_error(ORBFE_ERR_ARG, "bad arguments");
    if (n == 0) return ORBFE_OK;
    if (!d_desc || !d_leaf_out || !d_node_out) return set_error(ORBFE_ERR_ARG, "NULL argument");
    BOW_TRY(cudaSetDevice(v->device));
    cudaStream_t s = stream ? (cudaStream_t)stream : v->stream;
    bow_descend_kernel<<<(n + 7) / 8, 256, 0, s>>>(reinterpret_cast<const uint4 *>(v->d_desc), v->d_child_ptr, v->d_children,
                                                   reinterpret_cast<const uint4 *>(d_desc), n, v->depth - levelsup, d_leaf_out,
                                                   d_node_out);
    BOW_TRY(cudaGetLastError());
    return ORBFE_OK;
}

extern "C" int orbfe_feature_vector_device(OrbfeVocabulary *v, int nframes, const int32_t *d_leaf, const int32_t *d_node,
                                           const int *d_counts, int cap, int32_t *d_fv_ids, int32_t *d_fv_ptr, int32_t *d_fv_items,
                                           int *d_fv_n, void *stream) {
    if (!v || nframes < 0 || cap < 1) return set_error(ORBFE_ERR_ARG, "bad arguments");
    if (nframes > 0 && (!d_leaf || !d_node || !d_counts || !d_fv_ids || !d_fv_ptr || !d_fv_items || !d_fv_n))
        return set_error(ORBFE_ERR_ARG, "NULL argument");
    if (cap > ORBFE_FV_MAX_CAP)
        return set_error(ORBFE_ERR_UNSUPPORTED, "cap %d exceeds the %d features per frame the FeatureVector kernel sorts in shared memory",
                         cap, ORBFE_FV_MAX_CAP);
    if (nframes == 0) return ORBFE_OK;
    BOW_TRY(cudaSetDevice(v->device));
    cudaStream_t s = stream ? (cudaStream_t)stream : v->stream;
    BOW_TRY((cudaError_t)launch_feature_vector(nframes, d_leaf, d_node, v->d_live, v->nnodes, d_counts, cap, d_fv_ids, d_fv_ptr,
                                               d_fv_items, d_fv_n, s));
    BOW_TRY(cudaGetLastError());
    return ORBFE_OK;
}

extern "C" int orbfe_bow_vector_device(OrbfeVocabulary *v, int nframes, const int32_t *d_leaf, const int *d_counts, int cap,
                                       int32_t *d_bow_ids, double *d_bow_vals, int *d_bow_n, void *stream) {
    if (!v || nframes < 0 || cap < 1) return set_error(ORBFE_ERR_ARG, "bad arguments");
    if (nframes > 0 && (!d_leaf || !d_counts || !d_bow_ids || !d_bow_vals || !d_bow_n)) return set_error(ORBFE_ERR_ARG, "NULL argument");
    if (cap > ORBFE_FV_MAX_CAP)
        return set_error(ORBFE_ERR_UNSUPPORTED, "cap %d exceeds the %d features per frame the BowVector kernel sorts in shared memory",
                         cap, ORBFE_FV_MAX_CAP);
    if (nframes == 0) return ORBFE_OK;
    BOW_TRY(cudaSetDevice(v->device));
    cudaStream_t s = stream ? (cudaStream_t)stream : v->stream;
    size_t smem = 0;
    BOW_TRY(fv_smem(bow_vector_kernel, cap, &smem));
    const int accumulate = v->weighting == ORBFE_BOW_TF || v->weighting == ORBFE_BOW_TF_IDF;
    bow_vector_kernel<<<nframes, FV_THREADS, smem, s>>>(d_leaf, v->d_live, v->d_word_id, v->d_weight, v->nnodes, accumulate, v->norm,
                                                        d_counts, cap, d_bow_ids, d_bow_vals, d_bow_n);
    BOW_TRY(cudaGetLastError());
    return ORBFE_OK;
}

extern "C" int orbfe_bow_descend(OrbfeVocabulary *v, const uint8_t *desc, int n, int levelsup, int32_t *leaf_out, int32_t *node_out) {
    if (!v || n < 0) return set_error(ORBFE_ERR_ARG, "bad arguments");
    if (n == 0) return ORBFE_OK;
    if (!desc || !leaf_out || !node_out) return set_error(ORBFE_ERR_ARG, "NULL argument");
    BOW_TRY(cudaSetDevice(v->device));
    if (v->in_cap < (size_t)n * 32) {
        cudaFree(v->d_in); v->d_in = nullptr; v->in_cap = 0;
        BOW_TRY(cudaMalloc((void **)&v->d_in, (size_t)n * 32 * 2));
        v->in_cap = (size_t)n * 32 * 2;
    }
    if (v->out_cap < (size_t)n * 2) {
        cudaFree(v->d_out); v->d_out = nullptr; v->out_cap = 0;
        BOW_TRY(cudaMalloc((void **)&v->d_out, sizeof(int) * (size_t)n * 4));
        v->out_cap = (size_t)n * 4;
    }
    BOW_TRY(cudaMemcpyAsync(v->d_in, desc, (size_t)n * 32, cudaMemcpyHostToDevice, v->stream));
    int rc = orbfe_bow_descend_device(v, v->d_in, n, levelsup, v->d_out, v->d_out + n, v->stream);
    if (rc) return rc;
    BOW_TRY(cudaMemcpyAsync(leaf_out, v->d_out, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, v->stream));
    BOW_TRY(cudaMemcpyAsync(node_out, v->d_out + n, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, v->stream));
    BOW_TRY(cudaStreamSynchronize(v->stream));
    return ORBFE_OK;
}

// accessors for host/bow_host.cpp (the struct layout stays private to this file)
namespace orbfe {
const int32_t *vocab_word_ids(const OrbfeVocabulary *v) { return v->word_id.data(); }
const double *vocab_weights(const OrbfeVocabulary *v) { return v->weight.data(); }
void vocab_modes(const OrbfeVocabulary *v, int *weighting, int *norm) { *weighting = v->weighting; *norm = v->norm; }
// for kfdb.cu: the device of the node table, and the number of words (largest word id + 1)
int vocab_device(const OrbfeVocabulary *v) { return v->device; }
int vocab_nwords(const OrbfeVocabulary *v) {
    int n = 0;
    for (int32_t w : v->word_id) n = std::max(n, w + 1);
    return n;
}

void launch_distinctive(const uint8_t *d_desc, const int *d_group_ptr, int ngroups, int *d_best, cudaStream_t s) {
    if (ngroups <= 0) return;
    distinctive_kernel<false><<<(ngroups + 3) / 4, 128, 0, s>>>(reinterpret_cast<const uint4 *>(d_desc), d_group_ptr, nullptr, 0,
                                                                nullptr, 0, 1, ngroups, d_best, nullptr, nullptr);
}

void launch_distinctive_obs(const uint8_t *d_desc, const int *d_counts, int nframes, int cap, const int *d_group_ptr,
                            const int *d_obs, int nobs, int ngroups, int *d_best, uint8_t *d_mp_desc, int *d_err, cudaStream_t s) {
    if (ngroups <= 0) return;
    distinctive_kernel<true><<<(ngroups + 3) / 4, 128, 0, s>>>(reinterpret_cast<const uint4 *>(d_desc), d_group_ptr, d_obs, nobs,
                                                               d_counts, nframes, cap, ngroups, d_best,
                                                               reinterpret_cast<uint4 *>(d_mp_desc), d_err);
}
}  // namespace orbfe
