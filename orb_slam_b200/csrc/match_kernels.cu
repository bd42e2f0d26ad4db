// match_kernels.cu -- 256-bit Hamming kernels behind ORBmatcher::SearchBy* (reference src/ORBmatcher.cc).
//
// The per-pair primitive is ORBmatcher::DescriptorDistance (ORBmatcher.cc:1794-1810): popcount of the XOR
// of two 32-byte descriptors.  On the device that is 8 x (XOR + POPC) on 32-bit words.  These kernels are
// bound by the integer/POPC issue rate (all-pairs sweep) or by launch latency (windowed CSR lists), never
// by HBM; no tensor cores (the north star forbids reshaping Hamming into a GEMM).
#include <cstring>

#include "orbfe_internal.h"

namespace orbfe {

__device__ __forceinline__ int ham256(const uint4 a0, const uint4 a1, const uint4 b0, const uint4 b1) {
    return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
           __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

// The same distance with half the POPCs, for the all-pairs sweep (config 5), which ncu shows saturating the XU pipe
// (POPC issues at 16 lanes/clk/SM: 96.7 % busy with 8 POPC per pair).  Four carry-save adders (two LOP3 each, on the
// four-times-wider integer pipe) compress the eight XOR words x0..x7 into words of weight 1, 1, 2 and 4:
//   x0+x1+x2 = 2*t0 + s0 ; x3+x4+x5 = 2*t1 + s1 ; s0+s1+x6 = 2*t2 + s2 ; t0+t1+t2 = 2*f0 + tw
//   => popcount(x0..x7) = popc(s2) + popc(x7) + 2*popc(tw) + 4*popc(f0)           (exact: bitwise column sums)
__device__ __forceinline__ void csa(uint32_t a, uint32_t b, uint32_t c, uint32_t &carry, uint32_t &sum) {
    sum = a ^ b ^ c;                       // one LOP3
    carry = (a & b) | (c & (a ^ b));       // one LOP3 (majority)
}
__device__ __forceinline__ int ham256_csa(const uint4 a0, const uint4 a1, const uint4 b0, const uint4 b1) {
    const uint32_t x0 = a0.x ^ b0.x, x1 = a0.y ^ b0.y, x2 = a0.z ^ b0.z, x3 = a0.w ^ b0.w;
    const uint32_t x4 = a1.x ^ b1.x, x5 = a1.y ^ b1.y, x6 = a1.z ^ b1.z, x7 = a1.w ^ b1.w;
    uint32_t t0, s0, t1, s1, t2, s2, f0, tw;
    csa(x0, x1, x2, t0, s0);
    csa(x3, x4, x5, t1, s1);
    csa(s0, s1, x6, t2, s2);
    csa(t0, t1, t2, f0, tw);
    return __popc(s2) + __popc(x7) + 2 * __popc(tw) + 4 * __popc(f0);
}

// One warp per query row of the CSR candidate structure; lanes stride over that row's candidates.
__global__ void __launch_bounds__(256) hamming_csr_kernel(const uint4 *__restrict__ q, const uint4 *__restrict__ t,
                                                          const int32_t *__restrict__ row_ptr,
                                                          const int32_t *__restrict__ cols, int nq,
                                                          uint16_t *__restrict__ out) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= nq) return;
    const int lane = threadIdx.x & 31;
    const int beg = __ldg(&row_ptr[row]), end = __ldg(&row_ptr[row + 1]);
    if (beg >= end) return;
    const uint4 a0 = __ldg(&q[2 * row]), a1 = __ldg(&q[2 * row + 1]);
    for (int k = beg + lane; k < end; k += 32) {
        const int j = __ldg(&cols[k]);
        const uint4 b0 = __ldg(&t[2 * j]), b1 = __ldg(&t[2 * j + 1]);
        out[k] = (uint16_t)ham256(a0, a1, b0, b1);
    }
}

void launch_hamming_csr(const uint8_t *q, const uint8_t *t, const int32_t *row_ptr, const int32_t *cols, int nq,
                        int npairs, uint16_t *out, cudaStream_t s) {
    (void)npairs;
    if (nq <= 0) return;
    hamming_csr_kernel<<<(nq + 7) / 8, 256, 0, s>>>(reinterpret_cast<const uint4 *>(q), reinterpret_cast<const uint4 *>(t),
                                                    row_ptr, cols, nq, out);
}

// Dense nq x nt matrix: blockIdx.y strides over queries (grid.y is capped at 65535), threads stride over train descriptors.
__global__ void __launch_bounds__(256) hamming_dense_kernel(const uint4 *__restrict__ q, int nq,
                                                            const uint4 *__restrict__ t, int nt,
                                                            uint16_t *__restrict__ out) {
    for (int i = blockIdx.y; i < nq; i += gridDim.y) {
        const uint4 a0 = __ldg(&q[2 * i]), a1 = __ldg(&q[2 * i + 1]);
        for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nt; j += gridDim.x * blockDim.x) {
            const uint4 b0 = __ldg(&t[2 * j]), b1 = __ldg(&t[2 * j + 1]);
            out[(size_t)i * nt + j] = (uint16_t)ham256(a0, a1, b0, b1);
        }
    }
}

void launch_hamming_dense(const uint8_t *q, int nq, const uint8_t *t, int nt, uint16_t *out, cudaStream_t s) {
    if (nq <= 0 || nt <= 0) return;
    dim3 grid(min((nt + 255) / 256, 64), min(nq, 65535));
    hamming_dense_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const uint4 *>(q), nq, reinterpret_cast<const uint4 *>(t), nt, out);
}

// Best / second-best sweep: blockIdx.x = database group (keyframe), blockIdx.y = block of 256 queries.
// Each thread owns one query in registers; the group's descriptors stream through shared memory in
// chunks and are read by all threads at the same address (broadcast).  Update rule = the strict-<
// best/second loop of ORBmatcher.cc:456-466, in ascending database order (first minimum wins).
#define KNN_CHUNK 128
__global__ void __launch_bounds__(256) knn2_groups_kernel(const uint4 *__restrict__ q, int nq,
                                                          const uint4 *__restrict__ db, int group_size,
                                                          uint16_t *__restrict__ best, int32_t *__restrict__ best_idx,
                                                          uint16_t *__restrict__ second) {
    __shared__ uint4 chunk[KNN_CHUNK * 2];
    const int g = blockIdx.x;
    const int qi = blockIdx.y * blockDim.x + threadIdx.x;
    const bool active = qi < nq;
    uint4 a0 = make_uint4(0, 0, 0, 0), a1 = a0;
    if (active) { a0 = __ldg(&q[2 * qi]); a1 = __ldg(&q[2 * qi + 1]); }
    int b1 = 0x7fffffff, b2 = 0x7fffffff, bi = -1;
    const uint4 *__restrict__ gdb = db + (size_t)g * group_size * 2;
    for (int c0 = 0; c0 < group_size; c0 += KNN_CHUNK) {
        const int nc = min(KNN_CHUNK, group_size - c0);
        __syncthreads();
        for (int i = threadIdx.x; i < nc * 2; i += blockDim.x) chunk[i] = __ldg(&gdb[(size_t)c0 * 2 + i]);
        __syncthreads();
        if (active) {
#pragma unroll 4
            for (int j = 0; j < nc; j++) {
                const int d = ham256_csa(a0, a1, chunk[2 * j], chunk[2 * j + 1]);
                if (d < b1) { b2 = b1; b1 = d; bi = c0 + j; }
                else if (d < b2) b2 = d;
            }
        }
    }
    if (active) {
        const size_t o = (size_t)g * nq + qi;
        best[o] = (uint16_t)min(b1, 0xFFFF);
        best_idx[o] = bi;
        second[o] = (uint16_t)min(b2, 0xFFFF);
    }
}

void launch_knn2_groups(const uint8_t *q, int nq, const uint8_t *db, int ngroups, int group_size,
                        uint16_t *best, int32_t *best_idx, uint16_t *second, cudaStream_t s) {
    if (nq <= 0 || ngroups <= 0) return;
    dim3 grid(ngroups, (nq + 255) / 256);
    knn2_groups_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const uint4 *>(q), nq, reinterpret_cast<const uint4 *>(db),
                                            group_size, best, best_idx, second);
}

}  // namespace orbfe

// ================================================================================================
// Device-resident frame-to-frame matcher: ORBmatcher::SearchByProjection(Frame &Cur, const Frame &Last, th)
// (reference src/ORBmatcher.cc:1507-1620) with Frame's lookup grid (src/Frame.cc:109-123,200-277) rebuilt on
// the device.  One CTA per (Current, Last) pair:
//   A  grid of the Current frame: counting sort of the keypoints into the 64x48 cells, ascending index
//      inside a cell (= push_back order, Frame.cc:116-123; PosInGrid rounds with round(), :269-270);
//   B  one thread per Last feature: project its map point with Tcw (float accumulation: cv::gemm's small-matrix path),
//      enumerate the candidates exactly in GetFeaturesInArea order (ix outer, iy inner, cell order; octave
//      and |dx|,|dy| <= r filters) and compute every 256-bit Hamming distance (XOR + POPC);
//   C  the sequential accept loop, replayed by one warp over the precomputed (candidate, distance) lists:
//      strict-< argmin over the candidates whose Current slot is still free, accept if <= TH_HIGH;
//   D  rotation histogram + ComputeThreeMaxima (:1748-1789) and removal of the inconsistent matches.
// Bit-exact with the oracle; the only implementation of these rules (the host-array entries stage their inputs for it).
// ================================================================================================
namespace orbfe {

#define SBP_GCOLS 64
#define SBP_GROWS 48
#define SBP_NCELL (SBP_GCOLS * SBP_GROWS)

#define SBP_MAX_ROUNDS 48
#define SBP_THREADS 1024
#define SBP_WARPS (SBP_THREADS / 32)

__device__ __forceinline__ int block_excl_scan(int v, int *s_warp /*[SBP_WARPS]*/, int *total) {
    // exclusive scan of one value per thread over the CTA
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[wid] = x;
    __syncthreads();
    const int wv = s_warp[lane];  // SBP_WARPS == 32: one partial per lane
    int incl = wv;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    const int base = __shfl_sync(0xffffffffu, incl - wv, wid);
    *total = __shfl_sync(0xffffffffu, incl, 31);
    __syncthreads();
    return base + x - v;
}

struct SbpQuery {
    float u, v, r;
    int lo, hi;  // octave filter [lo, hi]; (-1, -1) = none (KeyFrame::GetFeaturesInArea has none)
    int x0, x1, y0, y1;
    bool ok;
};

// `int nMinCellX = floor(...)` and its three siblings (Frame.cc:205-223) convert a float to int the x86-64 way (cvttss2si):
// NaN and every value outside [-2^31, 2^31) give INT_MIN, so a window with a NaN or infinite centre or radius, or one reaching
// 2^31 cells, is empty.  The device's conversion saturates and turns NaN into 0, which would scan cell 0 or the whole grid.
__device__ __forceinline__ int cell_bound(float f) {
    return (f >= -2147483648.0f && f < 2147483648.0f) ? (int)f : (int)0x80000000u;
}

// cell range of Frame::GetFeaturesInArea (Frame.cc:205-223); false if the window misses the grid
__device__ __forceinline__ bool sbp_cell_range(const SbpParams &P, SbpQuery &q) {
    int x0 = cell_bound(floorf(__fmul_rn(__fsub_rn(__fsub_rn(q.u, P.min_x), q.r), P.gw)));
    x0 = max(0, x0);
    if (x0 >= SBP_GCOLS) return false;
    int x1 = cell_bound(ceilf(__fmul_rn(__fadd_rn(__fsub_rn(q.u, P.min_x), q.r), P.gw)));
    x1 = min(SBP_GCOLS - 1, x1);
    if (x1 < 0) return false;
    int y0 = cell_bound(floorf(__fmul_rn(__fsub_rn(__fsub_rn(q.v, P.min_y), q.r), P.gh)));
    y0 = max(0, y0);
    if (y0 >= SBP_GROWS) return false;
    int y1 = cell_bound(ceilf(__fmul_rn(__fadd_rn(__fsub_rn(q.v, P.min_y), q.r), P.gh)));
    y1 = min(SBP_GROWS - 1, y1);
    if (y1 < 0) return false;
    q.x0 = x0; q.x1 = x1; q.y0 = y0; q.y1 = y1;
    return true;
}

__device__ __forceinline__ SbpQuery sbp_project(const SbpParams &P, const OrbfeKeyPoint &kl, const float *X, const float *T) {
    SbpQuery q;
    q.ok = false;
    float xc3[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        // x3Dc = Rcw*x3Dw + tcw: one cv::gemm on CV_32F 3x3 * 3x1 (flags 0) = OpenCV's unrolled small-matrix path: the three
        // products summed in FLOAT left to right, then (float)((double)sum + (double)t)  (pinned to cv2.gemm golden vectors)
        const float s = __fadd_rn(__fadd_rn(__fmul_rn(T[4 * k], X[0]), __fmul_rn(T[4 * k + 1], X[1])), __fmul_rn(T[4 * k + 2], X[2]));
        xc3[k] = (float)__dadd_rn((double)s, (double)T[4 * k + 3]);
    }
    const float invzc = (float)(1.0 / (double)xc3[2]);
    q.u = __fadd_rn(__fmul_rn(__fmul_rn(P.fx, xc3[0]), invzc), P.cx);
    q.v = __fadd_rn(__fmul_rn(__fmul_rn(P.fy, xc3[1]), invzc), P.cy);
    if (q.u < P.min_x || q.u > P.max_x) return q;
    if (q.v < P.min_y || q.v > P.max_y) return q;
    q.lo = kl.octave - 1;
    q.hi = kl.octave + 1;
    q.r = __fmul_rn(P.th, P.scale[kl.octave]);
    q.ok = sbp_cell_range(P, q);
    return q;
}

// explicit queries (guided search): one job = `q_cnt` queries starting at `q_base` of the concatenated arrays
struct GuidedQueries {
    const float *qu, *qv, *qr, *qangle;
    const int *qlo, *qhi;
    const uint8_t *qdesc;
    const int *q_base, *q_cnt;
    int *best;   // rule SBP_RULE_BEST: per query (concatenated index) the kept candidate, or -1
};

__device__ __forceinline__ bool octave_ok(int o, int lo, int hi) {
    return (lo == -1 && hi == -1) || (o >= lo && o <= hi);
}

// Rotation histogram of the matchers (e.g. ORBmatcher.cc:263-281, :1583-1590): bin = round((a1 - a2 [+360]) * (1/30)), 30 -> 0.
__device__ __forceinline__ int rot_hist_bin(float a1, float a2) {
    float rot = __fsub_rn(a1, a2);
    if (rot < 0.0f) rot = __fadd_rn(rot, 360.0f);
    int bin = (int)roundf(__fmul_rn(rot, 1.0f / 30));
    if (bin == 30) bin = 0;
    return bin;
}

// ComputeThreeMaxima (ORBmatcher.cc:1748-1789) over the 30 bin counts `hist`: keep[0..2] = the bins whose matches stay (-1 =
// none).  The first maximum wins ties; the second and third are dropped when below 0.1 * max1.  For one thread.  A macro rather
// than an inline function: expanded in place it leaves the fused projection kernel's SASS exactly as it was.
#define THREE_MAXIMA_KEEP(hist, keep)                                                                    \
    {                                                                                                    \
        int max1 = 0, max2 = 0, max3 = 0, ind1 = -1, ind2 = -1, ind3 = -1;                               \
        for (int i = 0; i < 30; i++) {                                                                   \
            const int s = (hist)[i];                                                                     \
            if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }    \
            else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }                         \
            else if (s > max3) { max3 = s; ind3 = i; }                                                   \
        }                                                                                                \
        if ((float)max2 < __fmul_rn(0.1f, (float)max1)) { ind2 = -1; ind3 = -1; }                        \
        else if ((float)max3 < __fmul_rn(0.1f, (float)max1)) { ind3 = -1; }                             \
        (keep)[0] = ind1; (keep)[1] = ind2; (keep)[2] = ind3;                                            \
    }

// MODE 0: SearchByProjection(Frame, Frame) -- queries = projections of the Last frame's map points;
// MODE 1: guided search -- explicit query windows (M3, M4, M6, M7 and the KeyFrame-level routines);
// MODE 2: SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize) (ORBmatcher.cc:598-713) -- queries = the
//         level-0 features of F1 (= frame last_idx[pair]) searched in F2 (= frame cur_idx[pair]) inside a `th`-pixel window
//         around their previously matched position (`world` holds vbPrevMatched, 2 floats per F1 feature, updated in place,
//         :708-710); an F2 feature can be RE-assigned to a later, closer F1 feature (:637, :656-663); cur_mp receives
//         vnMatches12 (per F1 feature).
template <int MODE>
__global__ void __launch_bounds__(SBP_THREADS) sbp_device_kernel(SbpParams P, const OrbfeKeyPoint *__restrict__ kps,
                                                                 const uint8_t *__restrict__ desc, const int *__restrict__ counts,
                                                                 const int *__restrict__ cur_idx, const int *__restrict__ last_idx,
                                                                 const float *__restrict__ world, const uint8_t *__restrict__ flags,
                                                                 const float *__restrict__ Tcw, GuidedQueries GQ,
                                                                 uint32_t *__restrict__ scratch, int *__restrict__ cur_mp,
                                                                 int *__restrict__ nmatches, int *__restrict__ err) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int cap = P.cap;
    int *cell_start = reinterpret_cast<int *>(smem);                 // [NCELL + 1]
    int *cell_cur = cell_start + SBP_NCELL + 1;                      // [NCELL]
    int *q_off = cell_cur + SBP_NCELL;                               // [qcap + 1]
    float *kx = reinterpret_cast<float *>(q_off + P.qcap + 1);       // [cap] Current keypoint x
    float *ky = kx + cap;                                            // [cap]
    uint32_t *taken = reinterpret_cast<uint32_t *>(ky + cap);        // [(cap + 31) / 32]
    uint16_t *items = reinterpret_cast<uint16_t *>(taken + (cap + 31) / 32);  // [cap]
    uint8_t *newbin = reinterpret_cast<uint8_t *>(items + cap);      // [cap]
    uint8_t *koct = newbin + cap;                                    // [cap] Current keypoint octave
    // (items, newbin, koct together are 4 * cap bytes after a 4-byte aligned start: what follows stays 4-byte aligned)
    uint16_t *mdist = reinterpret_cast<uint16_t *>(koct + cap);      // MODE 2: [cap] vMatchedDistance (0xFFFF = INT_MAX)
    uint16_t *owner = mdist + cap;                                   // MODE 2: [cap] vnMatches21 (0xFFFF = -1)
    int *firstq = reinterpret_cast<int *>(mdist);                    // rules 0-2 (never MODE 2): [cap] lowest query holding / stamping the slot -- same bytes as mdist + owner
    uint16_t *choice = reinterpret_cast<uint16_t *>(firstq + cap);   // rule 0: [qcap] the slot a query wants this round
    uint32_t *resolved = reinterpret_cast<uint32_t *>(choice + P.qcap + (P.qcap & 1));  // [(qcap + 31) / 32] query has been decided
    constexpr bool EXPLICIT = MODE == 1;
    constexpr bool INIT = MODE == 2;
    const int qown = EXPLICIT ? P.owner_base : 0;   // a matched slot receives qown + the job-local query index
    __shared__ int s_warp[SBP_WARPS], s_hist[32], s_keep[3], s_removed, s_nm, s_unres;
    uint32_t *s_ent = reinterpret_cast<uint32_t *>(smem + P.smem_fixed);  // entry staging area

    const int pair = blockIdx.x;
    const int fc = cur_idx[pair], fl = EXPLICIT ? 0 : last_idx[pair];
    const int nc = min(counts[fc], cap);
    const int qb = EXPLICIT ? GQ.q_base[pair] : 0;
    const int nl = EXPLICIT ? min(GQ.q_cnt[pair], P.qcap) : min(counts[fl], cap);
    const OrbfeKeyPoint *__restrict__ kc = kps + (size_t)fc * cap;
    const OrbfeKeyPoint *__restrict__ kl = kps + (size_t)fl * cap;
    const uint4 *__restrict__ dc = reinterpret_cast<const uint4 *>(desc + (size_t)fc * cap * 32);
    const uint4 *__restrict__ dl = EXPLICIT ? reinterpret_cast<const uint4 *>(GQ.qdesc + (size_t)qb * 32)
                                            : reinterpret_cast<const uint4 *>(desc + (size_t)fl * cap * 32);
    const float *__restrict__ wl = EXPLICIT ? nullptr : INIT ? world + (size_t)pair * cap * 2 /* vbPrevMatched of this pair */
                                                            : world + (size_t)fl * cap * 3;
    const uint8_t *__restrict__ fll = EXPLICIT ? nullptr : flags + (size_t)fl * cap;
    const float *__restrict__ T = (EXPLICIT || INIT) ? nullptr : Tcw + (size_t)pair * 12;
    int *__restrict__ mp = cur_mp + (size_t)pair * cap;
    const int tid = threadIdx.x;
    // query q of this job (projection of a Last feature, or an explicit (u, v, r, lo, hi) window)
    auto get_query = [&](int q) -> SbpQuery {
        if (EXPLICIT) {
            SbpQuery Q;
            Q.u = GQ.qu[qb + q]; Q.v = GQ.qv[qb + q]; Q.r = GQ.qr[qb + q];
            Q.lo = GQ.qlo[qb + q]; Q.hi = GQ.qhi[qb + q];
            Q.ok = sbp_cell_range(P, Q);
            return Q;
        }
        if (INIT) {   // :609-618: level-0 features only, window around the previously matched position, same level
            SbpQuery Q;
            Q.ok = false;
            if (kl[q].octave > 0) return Q;
            Q.u = wl[2 * q]; Q.v = wl[2 * q + 1]; Q.r = P.th;
            Q.lo = 0; Q.hi = 0;
            Q.ok = sbp_cell_range(P, Q);
            return Q;
        }
        return sbp_project(P, kl[q], wl + 3 * q, T);
    };
    auto query_angle = [&](int q) -> float { return EXPLICIT ? GQ.qangle[qb + q] : kl[q].angle; };

    // rig exchange: the gathered keypoints / descriptors of the other ranks arrive by remote stores; wait for every rank's
    // epoch flag (local polling) before the first read
    if (P.xw_flags) {
        if (tid < P.xw_n) {
            const long long t0 = clock64();
            unsigned v;
            do {
                asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(P.xw_flags + tid) : "memory");
                if ((int)(v - P.xw_epoch) >= 0) break;
                if (clock64() - t0 > 4000000000ll) { atomicExch(P.xw_err, 1); break; }
                __nanosleep(100);
            } while (true);
        }
        __syncthreads();
    }
    // ... and the last thread block to finish tells every rank that this one has read the epoch (called by ALL threads)
    auto publish_ack = [&]() {
        if (!P.xw_done) return;
        __syncthreads();
        if (tid == 0) {
            unsigned prev;
            asm volatile("atom.add.release.gpu.global.u32 %0, [%1], 1;" : "=r"(prev) : "l"(P.xw_done) : "memory");
            if (prev == gridDim.x - 1) {
                asm volatile("fence.acq_rel.sys;" ::: "memory");
                *P.xw_done = 0;
                for (int r = 0; r < P.xw_n; r++)
                    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(P.xw_ack[r]), "r"(P.xw_epoch) : "memory");
            }
        }
    };
    // ---- A: grid of the Current frame ----
    for (int i = tid; i < SBP_NCELL; i += SBP_THREADS) cell_cur[i] = 0;
    for (int i = tid; i < (cap + 31) / 32; i += SBP_THREADS) taken[i] = 0;
    if (tid < 32) s_hist[tid] = 0;
    if (tid == 0) { s_removed = 0; s_nm = 0; }
    __syncthreads();
    for (int i = tid; i < nc; i += SBP_THREADS) {
        const OrbfeKeyPoint k = kc[i];
        kx[i] = k.x; ky[i] = k.y; koct[i] = (uint8_t)k.octave;
        const float px = roundf(__fmul_rn(__fsub_rn(k.x, P.min_x), P.gw));
        const float py = roundf(__fmul_rn(__fsub_rn(k.y, P.min_y), P.gh));
        int cell = -1;
        // MODE 2 asks for level-0 features only (:618): the other levels never enter the grid, so the window walks touch
        // one keypoint in five
        if (px >= 0.f && px < (float)SBP_GCOLS && py >= 0.f && py < (float)SBP_GROWS && !(INIT && k.octave != 0)) cell = (int)px * SBP_GROWS + (int)py;
        newbin[i] = 0xFF;
        if (cell >= 0) atomicAdd(&cell_cur[cell], 1);
        if (INIT) { mdist[i] = 0xFFFF; owner[i] = 0xFFFF; }
        else if (mp[i] >= 0) atomicOr(&taken[i >> 5], 1u << (i & 31));  // slot occupied on entry (:1562)
    }
    if (INIT) {
        for (int i = tid; i < cap; i += SBP_THREADS) { mp[i] = -1; if (i >= nc) newbin[i] = 0xFF; }   // vnMatches12 = -1 (:601); newbin = rotation bin per F1 feature
        for (int i = tid; i < P.qcap; i += SBP_THREADS) choice[i] = 0xFFFF;                            // slot accepted for each F1 feature
    }
    __syncthreads();
    {   // exclusive scan of the 3072 cell counts: 3 cells per thread
        int loc[3], sum = 0;
#pragma unroll
        for (int k = 0; k < 3; k++) { loc[k] = cell_cur[tid * 3 + k]; sum += loc[k]; }
        int tot;
        int base = block_excl_scan(sum, s_warp, &tot);
#pragma unroll
        for (int k = 0; k < 3; k++) { cell_start[tid * 3 + k] = base; cell_cur[tid * 3 + k] = base; base += loc[k]; }
        if (tid == SBP_THREADS - 1) cell_start[SBP_NCELL] = base;
    }
    __syncthreads();
    for (int i = tid; i < nc; i += SBP_THREADS) {
        const float px = roundf(__fmul_rn(__fsub_rn(kx[i], P.min_x), P.gw));
        const float py = roundf(__fmul_rn(__fsub_rn(ky[i], P.min_y), P.gh));
        if (px >= 0.f && px < (float)SBP_GCOLS && py >= 0.f && py < (float)SBP_GROWS && !(INIT && koct[i] != 0)) {
            const int cell = (int)px * SBP_GROWS + (int)py;
            items[atomicAdd(&cell_cur[cell], 1)] = (uint16_t)i;
        }
    }
    __syncthreads();
    for (int c = tid; c < SBP_NCELL; c += SBP_THREADS) {  // ascending index inside each cell (cells are tiny)
        const int b = cell_start[c], e = cell_start[c + 1];
        for (int i = b + 1; i < e; i++) {
            const uint16_t v = items[i];
            int j = i - 1;
            while (j >= b && items[j] > v) { items[j + 1] = items[j]; j--; }
            items[j + 1] = v;
        }
    }
    __syncthreads();

    // ---- B1: candidate counts per Last feature ----
    const int nq_iter = (nl + SBP_THREADS - 1) / SBP_THREADS;
    int run_total = 0;
    for (int it = 0; it < nq_iter; it++) {
        const int q = it * SBP_THREADS + tid;
        int cnt = 0;
        if (q < nl && (EXPLICIT || INIT || fll[q])) {
            const SbpQuery Q = get_query(q);
            if (Q.ok) {
                for (int ix = Q.x0; ix <= Q.x1; ix++) {
                    // cells (ix, y0..y1) are contiguous in the cell-major layout: one item range per column
                    const int kb = cell_start[ix * SBP_GROWS + Q.y0], ke = cell_start[ix * SBP_GROWS + Q.y1 + 1];
                    for (int k = kb; k < ke; k++) {
                        const int i2 = items[k];
                        if (!octave_ok(koct[i2], Q.lo, Q.hi)) continue;
                        if (fabsf(__fsub_rn(kx[i2], Q.u)) > Q.r || fabsf(__fsub_rn(ky[i2], Q.v)) > Q.r) continue;
                        cnt++;
                    }
                }
            }
        }
        int tot;
        const int off = block_excl_scan(cnt, s_warp, &tot);
        if (q < nl) q_off[q] = run_total + off;
        run_total += tot;
    }
    if (tid == 0) q_off[nl] = run_total;
    __syncthreads();
    const int T_total = run_total;
    if (T_total > P.scratch_per_pair) {   // err[1]: the most entries any overflowing job needed, for a relaunch that fits
        if (tid == 0) { atomicExch(err, 1); atomicMax(err + 1, T_total); nmatches[pair] = -1; }
        publish_ack();
        return;
    }
    uint32_t *ent = (T_total <= P.smem_entries) ? s_ent : scratch + (size_t)pair * P.scratch_per_pair;

    // ---- B2: candidate indices in enumeration order (query index in the upper half for now) ----
    for (int q = tid; q < nl; q += SBP_THREADS) {
        int o = q_off[q];
        if (q_off[q + 1] == o) continue;
        const SbpQuery Q = get_query(q);
        for (int ix = Q.x0; ix <= Q.x1; ix++) {
            const int kb = cell_start[ix * SBP_GROWS + Q.y0], ke = cell_start[ix * SBP_GROWS + Q.y1 + 1];
            for (int k = kb; k < ke; k++) {
                const int i2 = items[k];
                if (!octave_ok(koct[i2], Q.lo, Q.hi)) continue;
                if (fabsf(__fsub_rn(kx[i2], Q.u)) > Q.r || fabsf(__fsub_rn(ky[i2], Q.v)) > Q.r) continue;
                ent[o++] = (uint32_t)i2 | ((uint32_t)q << 16);
            }
        }
    }
    __threadfence_block();
    __syncthreads();
    // ---- B3: one 256-bit distance per ENTRY (balanced over the block whatever the list lengths are; the descriptor loads
    //          of independent entries overlap): entry = candidate index | distance << 16 ----
#pragma unroll 4
    for (int p = tid; p < T_total; p += SBP_THREADS) {
        const uint32_t v = ent[p];
        const int i2 = (int)(v & 0xFFFF), q = (int)(v >> 16);
        const int d = ham256(__ldg(&dl[2 * q]), __ldg(&dl[2 * q + 1]), __ldg(&dc[2 * i2]), __ldg(&dc[2 * i2 + 1]));
        ent[p] = (uint32_t)i2 | ((uint32_t)d << 16);
    }
    __threadfence_block();
    __syncthreads();

    // ---- C': best-only without slots (SBP_RULE_BEST, orbfe_guided_best): each query keeps the first minimum of its whole
    //          list iff it is <= th_dist.  No slots, no histogram, no interaction between queries. ----
    if (EXPLICIT && P.rule == SBP_RULE_BEST) {
        int kept = 0;
        for (int q = tid; q < nl; q += SBP_THREADS) {
            const int b = q_off[q], e = q_off[q + 1];
            uint32_t best = 0xFFFFFFFFu;   // dist << 16 | position: strict-< argmin in enumeration order
            for (int p = b; p < e; p++) best = min(best, (ent[p] & 0xFFFF0000u) | (uint32_t)(p - b));
            int idx = -1;
            if (best != 0xFFFFFFFFu && (int)(best >> 16) <= P.th_dist) { idx = (int)(ent[b + (int)(best & 0xFFFF)] & 0xFFFF); kept++; }
            GQ.best[qb + q] = idx;
        }
        if (kept) atomicAdd(&s_nm, kept);
        __syncthreads();
        if (tid == 0) nmatches[pair] = s_nm;
        return;
    }

    // ---- C: the accept loop.  In the reference it is sequential: query q takes the best candidate that no EARLIER query
    //         took.  Here it is resolved in parallel rounds of deterministic reservations: every undecided query picks its
    //         best free slot and stamps its index (atomicMin) on every free slot of its list.  Best-only rule (rule 0:
    //         SearchByProjection(Frame,Frame) and the best-only guided searches): a query commits iff its own stamp survived on
    //         the slot it picked -- no earlier undecided query can still take that slot, and earlier queries can only remove
    //         slots it ranks lower, so the pick is final.  Second-best rules (1, 2): the runner-up matters too, so a query
    //         decides (accept OR reject) only once its stamp survived on EVERY free slot of its list.  The outcome equals the
    //         sequential loop's; almost every query is decided in the first round, the rest within a few.  A chain longer
    //         than SBP_MAX_ROUNDS finishes in the sequential loop below, which skips decided queries.
    //         SearchForInitialization (MODE 2) re-assigns slots by distance and keeps the sequential warp. ----
    for (int i = tid; i < (P.qcap + 31) / 32; i += SBP_THREADS) resolved[i] = 0;
    __syncthreads();
    const bool par_rule0 = !INIT;   // rules 0, 1, 2 (SearchForInitialization's re-assignment rule keeps the sequential warp)
    if (par_rule0 && P.rule == 0) {
        // Best-only rule: "query q takes its best slot no earlier query took" is the serial dictatorship of the queries over
        // the slots, which is the unique stable assignment when every slot prefers the lower query index -- so deferred
        // acceptance reaches it in any proposal order.  firstq[c] = lowest query that proposed to slot c so far (it only
        // decreases, and the lowest proposer is never displaced); a query whose pick is held by a lower index moves to its
        // next best slot (distance, then list position) that no lower index holds.  The block iterates until a pass changes
        // nothing: ~half the passes of the reservation rounds below and a fraction of their work per pass.
        for (int c = tid; c < nc; c += SBP_THREADS) firstq[c] = ((taken[c >> 5] >> (c & 31)) & 1u) ? -1 : 0x7FFFFFFF;
        for (int q = tid; q < nl; q += SBP_THREADS) choice[q] = 0xFFFE;   // not started
        volatile int *holder = firstq;
        for (;;) {
            if (tid == 0) s_unres = 0;
            __syncthreads();
            bool changed = false;
            for (int q = tid; q < nl; q += SBP_THREADS) {
                int pos = choice[q];
                if (pos == 0xFFFF) continue;   // list exhausted: no match
                const int b = q_off[q], e = q_off[q + 1];
                for (;;) {
                    uint32_t lower = 0;   // keys are compared as key + 1, so 0 = "nothing picked yet"
                    if (pos != 0xFFFE) {
                        const uint32_t cur = ent[b + pos];
                        const int c = (int)(cur & 0xFFFF), h = holder[c];
                        if (h == q) break;
                        if (h > q) { atomicMin(&firstq[c], q); changed = true; break; }
                        lower = ((cur & 0xFFFF0000u) | (uint32_t)pos) + 1u;
                    }
                    uint32_t next = 0xFFFFFFFFu;
                    for (int p = b; p < e; p++) {
                        const uint32_t cur = ent[p];
                        const uint32_t key = ((cur & 0xFFFF0000u) | (uint32_t)(p - b)) + 1u;
                        if (key > lower && key < next && (int)(cur >> 16) <= P.th_dist && holder[cur & 0xFFFF] > q) next = key;
                    }
                    changed = true;
                    pos = next == 0xFFFFFFFFu ? 0xFFFF : (int)((next - 1u) & 0xFFFF);
                    choice[q] = (uint16_t)pos;
                    if (pos == 0xFFFF) break;
                }
            }
            if (changed) s_unres = 1;
            __syncthreads();
            if (!s_unres) break;
            __syncthreads();   // everybody has read s_unres before the next pass clears it
        }
        for (int q = tid; q < nl; q += SBP_THREADS) {
            const int pos = choice[q];
            if (pos == 0xFFFF) continue;
            const int i2 = (int)(ent[q_off[q] + pos] & 0xFFFF);
            if (firstq[i2] != q) continue;
            atomicOr(&taken[i2 >> 5], 1u << (i2 & 31));
            mp[i2] = qown + q;
            newbin[i2] = 0xFE;  // matched in this call; the rotation bin is filled in phase D
            atomicAdd(&s_nm, 1);
        }
        __syncthreads();
    } else if (par_rule0) {
        const bool needs_all = true;   // the second-best rules read EVERY free slot of the list, not just the pick
        for (int round = 0; round < SBP_MAX_ROUNDS; round++) {
            for (int c = tid; c < nc; c += SBP_THREADS) firstq[c] = 0x7FFFFFFF;
            if (tid == 0) s_unres = 0;
            __syncthreads();
            for (int q = tid; q < nl; q += SBP_THREADS) {
                if ((resolved[q >> 5] >> (q & 31)) & 1u) continue;
                const int b = q_off[q], e = q_off[q + 1];
                uint32_t best = 0xFFFFFFFFu;   // dist << 16 | position: strict-< argmin, first minimum wins
                for (int p = b; p < e; p++) {
                    const uint32_t cur = ent[p];
                    const int i2 = (int)(cur & 0xFFFF);
                    if (!((taken[i2 >> 5] >> (i2 & 31)) & 1u)) best = min(best, (cur & 0xFFFF0000u) | (uint32_t)(p - b));
                }
                // no free slot, or (best-only rule) a best that is already too far: final, because the free set only shrinks
                if (best == 0xFFFFFFFFu || (!needs_all && (int)(best >> 16) > P.th_dist)) {
                    atomicOr(&resolved[q >> 5], 1u << (q & 31));
                    choice[q] = 0xFFFF;
                    continue;
                }
                choice[q] = (uint16_t)(best & 0xFFFF);   // POSITION of the pick inside the list
                for (int p = b; p < e; p++) {
                    const int i2 = (int)(ent[p] & 0xFFFF);
                    if (!((taken[i2 >> 5] >> (i2 & 31)) & 1u)) atomicMin(&firstq[i2], q);
                }
            }
            __syncthreads();
            for (int q = tid; q < nl; q += SBP_THREADS) {
                if ((resolved[q >> 5] >> (q & 31)) & 1u) continue;
                const int b = q_off[q], e = q_off[q + 1];
                const int bpos = choice[q];
                const uint32_t bent = ent[b + bpos];
                const int i2 = (int)(bent & 0xFFFF), bd = (int)(bent >> 16);
                bool mine = firstq[i2] == q, accept = true;
                if (needs_all && mine) {
                    // every free slot of the list must carry this query's stamp: then no earlier undecided query can change the
                    // second best either, and the decision -- accept OR reject -- is final
                    uint32_t second = 0xFFFFFFFFu;
                    for (int p = b; p < e; p++) {
                        const uint32_t c2 = ent[p];
                        const int j2 = (int)(c2 & 0xFFFF);
                        if ((taken[j2 >> 5] >> (j2 & 31)) & 1u) continue;
                        if (firstq[j2] != q) { mine = false; break; }
                        if (p - b != bpos) second = min(second, (c2 & 0xFFFF0000u) | (uint32_t)(p - b));
                    }
                    if (mine) {
                        // INT_MAX stands for "no second candidate": (float)INT_MAX in the reference's comparisons
                        const float sd = second == 0xFFFFFFFFu ? 2147483648.0f : (float)(int)(second >> 16);
                        if (P.rule == 1) {
                            accept = (float)bd <= __fmul_rn(sd, P.nnratio) && bd <= 100;
                        } else {
                            const int lb = koct[i2];
                            const int ls = second == 0xFFFFFFFFu ? -1 : (int)koct[ent[b + (int)(second & 0xFFFF)] & 0xFFFF];
                            accept = bd <= 100 && !(lb == ls && (float)bd > __fmul_rn(P.nnratio, sd));
                        }
                    }
                }
                if (!mine) { s_unres = 1; continue; }
                atomicOr(&resolved[q >> 5], 1u << (q & 31));
                if (accept) {
                    atomicOr(&taken[i2 >> 5], 1u << (i2 & 31));
                    mp[i2] = qown + q;
                    newbin[i2] = 0xFE;  // matched in this call; the rotation bin is filled in phase D
                    atomicAdd(&s_nm, 1);
                }
            }
            __syncthreads();
            if (!s_unres) break;
            __syncthreads();   // everybody has read s_unres before the next round clears it
        }
    }
    if (tid < 32 && !(par_rule0 && !s_unres)) {
        const int lane = tid;
        int nm = 0;
        // 32 queries per step: one ballot finds the queries that have candidates and are still undecided, so the empty
        // ones (4 of 5 in SearchForInitialization: only level-0 features ask) cost no dependent shared-memory round trip
        for (int q0 = 0; q0 < nl; q0 += 32) {
            const int ql = q0 + lane;
            int bb = 0, ee = 0;
            if (ql < nl) { bb = q_off[ql]; ee = q_off[ql + 1]; }
            if (par_rule0 && ql < nl && ((resolved[ql >> 5] >> (ql & 31)) & 1u)) ee = bb;   // decided in the parallel rounds
            unsigned todo = __ballot_sync(0xffffffffu, ee != bb);
            int jn = todo ? __ffs(todo) - 1 : 0;
            int nb = __shfl_sync(0xffffffffu, bb, jn), ne = __shfl_sync(0xffffffffu, ee, jn);
            uint32_t nen = (todo && nb + lane < ne) ? ent[nb + lane] : 0xFFFFFFFFu;
            // MODE 2: vMatchedDistance of this lane's candidate rides along with the prefetch (patched below when the query
            // in between changes that slot)
            uint32_t nmd = (INIT && todo && nb + lane < ne) ? mdist[nen & 0xFFFF] : 0;
            while (todo) {
            const int q = q0 + jn, b = nb, e = ne;
            const uint32_t en = nen, md = nmd;
            todo &= todo - 1;
            if (todo) {   // prefetch the next query that has work
                jn = __ffs(todo) - 1;
                // MODE 2 skips only empty lists, so the next list starts where this one ends
                nb = INIT ? ne : __shfl_sync(0xffffffffu, bb, jn);
                ne = __shfl_sync(0xffffffffu, ee, jn);
                nen = (nb + lane < ne) ? ent[nb + lane] : 0xFFFFFFFFu;
                if (INIT) nmd = (nb + lane < ne) ? mdist[nen & 0xFFFF] : 0;
            }
            if (INIT && b != e) {
                // best / second over the candidates whose current match is worse than this distance (:637); strict-< update
                // order = first minimum wins, the second best is the minimum over the remaining candidates
                uint32_t best = 0xFFFFFFFFu, second = 0xFFFFFFFFu;
                if (e - b <= 32) {
                    // the usual case, one candidate per lane: keys are unique (lane in the low half), so the second best is
                    // the minimum with the winner's key masked out -- two REDUX, no second trip through shared memory
                    uint32_t key = 0xFFFFFFFFu;
                    if (b + lane < e && md > (en >> 16)) key = (en & 0xFFFF0000u) | (uint32_t)lane;
                    best = __reduce_min_sync(0xffffffffu, key);
                    second = __reduce_min_sync(0xffffffffu, key == best ? 0xFFFFFFFFu : key);
                    if (second != 0xFFFFFFFFu) second >>= 16;
                } else {
                    uint32_t cur = en;
                    for (int p0 = b; p0 < e; p0 += 32) {
                        const int p = p0 + lane;
                        if (p0 != b) cur = (p < e) ? ent[p] : 0xFFFFFFFFu;
                        uint32_t key = 0xFFFFFFFFu;
                        if (p < e && (uint32_t)mdist[cur & 0xFFFF] > (cur >> 16)) key = (cur & 0xFFFF0000u) | (uint32_t)(p - b);
                        best = min(best, __reduce_min_sync(0xffffffffu, key));
                    }
                    if (best != 0xFFFFFFFFu) {
                        const int bpos = (int)(best & 0xFFFF);
                        for (int p0 = b; p0 < e; p0 += 32) {
                            const int p = p0 + lane;
                            uint32_t key = 0xFFFFFFFFu;
                            if (p < e && p - b != bpos) {
                                const uint32_t c2 = ent[p];
                                if ((uint32_t)mdist[c2 & 0xFFFF] > (c2 >> 16)) key = c2 >> 16;
                            }
                            second = min(second, __reduce_min_sync(0xffffffffu, key));
                        }
                    }
                }
                if (best != 0xFFFFFFFFu) {
                    const int bpos = (int)(best & 0xFFFF), bd = (int)(best >> 16);
                    const float sd = second == 0xFFFFFFFFu ? 2147483648.0f : (float)(int)second;   // (float)INT_MAX
                    if (bd <= 50 /* TH_LOW, :652 */ && (float)bd < __fmul_rn(sd, P.nnratio)) {
                        // the winner's lane still holds its entry when the list fits one pass
                        const int i2 = (e - b <= 32) ? (int)(__shfl_sync(0xffffffffu, en, bpos) & 0xFFFF) : (int)(ent[b + bpos] & 0xFFFF);
                        // :656-660 re-assignment: the slot changes owner.  Only shared memory is touched here -- which feature
                        // owns the slot at the END decides vnMatches12 (filled in parallel after the loop), and the slot
                        // accepted for q is remembered for the rotation histogram (:666-676 keeps the entries of features
                        // that get unmatched later; a query is accepted at most once)
                        if (lane == 0) {
                            owner[i2] = (uint16_t)q;
                            mdist[i2] = (uint16_t)bd;
                            choice[q] = (uint16_t)i2;
                        }
                        if (nb + lane < ne && (int)(nen & 0xFFFF) == i2) nmd = (uint32_t)bd;   // the prefetched distance of that slot is stale now
                        __syncwarp();
                    }
                }
            } else if (b != e) {
                uint32_t best = 0xFFFFFFFFu;  // dist << 16 | position: strict-< argmin, first minimum wins
                uint32_t cur = en;
                for (int p0 = b; p0 < e; p0 += 32) {
                    const int p = p0 + lane;
                    if (p0 != b) cur = (p < e) ? ent[p] : 0xFFFFFFFFu;
                    uint32_t key = 0xFFFFFFFFu;
                    if (p < e) {
                        const int i2 = (int)(cur & 0xFFFF);
                        if (!((taken[i2 >> 5] >> (i2 & 31)) & 1u)) key = (cur & 0xFFFF0000u) | (uint32_t)(p - b);
                    }
                    best = min(best, __reduce_min_sync(0xffffffffu, key));
                }
                bool accept = best != 0xFFFFFFFFu && (int)(best >> 16) <= P.th_dist;  // rule 0 (th_dist = TH_HIGH for :1576)
                if (EXPLICIT && P.rule != 0 && best != 0xFFFFFFFFu) {
                    // second best among the remaining free candidates (strict-< order does not matter for the value)
                    const int bpos = (int)(best & 0xFFFF);
                    uint32_t second = 0xFFFFFFFFu;
                    for (int p0 = b; p0 < e; p0 += 32) {
                        const int p = p0 + lane;
                        uint32_t key = 0xFFFFFFFFu;
                        if (p < e && p - b != bpos) {
                            const uint32_t c2 = ent[p];
                            const int j2 = (int)(c2 & 0xFFFF);
                            if (!((taken[j2 >> 5] >> (j2 & 31)) & 1u)) key = (c2 & 0xFFFF0000u) | (uint32_t)(p - b);
                        }
                        second = min(second, __reduce_min_sync(0xffffffffu, key));
                    }
                    const int bd = (int)(best >> 16);
                    // INT_MAX stands for "no second candidate": (float)INT_MAX in the reference's comparisons
                    const float sd = second == 0xFFFFFFFFu ? 2147483648.0f : (float)(int)(second >> 16);
                    if (P.rule == 1) {
                        accept = (float)bd <= __fmul_rn(sd, P.nnratio) && bd <= 100;
                    } else {
                        const int lb = koct[ent[b + bpos] & 0xFFFF];
                        const int ls = second == 0xFFFFFFFFu ? -1 : (int)koct[ent[b + (int)(second & 0xFFFF)] & 0xFFFF];
                        accept = bd <= 100 && !(lb == ls && (float)bd > __fmul_rn(P.nnratio, sd));
                    }
                }
                if (accept) {
                    const int i2 = (int)(ent[b + (int)(best & 0xFFFF)] & 0xFFFF);
                    if (lane == 0) {
                        taken[i2 >> 5] |= 1u << (i2 & 31);
                        mp[i2] = qown + q;
                        newbin[i2] = 0xFE;  // matched in this call; the rotation bin is filled in phase D
                    }
                    nm++;
                    __syncwarp();
                }
            }
            }
        }
        if (lane == 0) s_nm += nm;
    }
    __syncthreads();

    // ---- D: rotation consistency ----
    if (INIT) {
        {   // vnMatches12: feature q keeps its slot iff it still owns it after every re-assignment
            int matched = 0;
            for (int q = tid; q < nl; q += SBP_THREADS) {
                const int i2 = choice[q];
                if (i2 != 0xFFFF && owner[i2] == q) { mp[q] = i2; matched++; }
            }
            if (matched) atomicAdd(&s_nm, matched);
        }
        if (P.check_ori) {
            for (int q = tid; q < nl; q += SBP_THREADS) {   // :666-676, one entry per ACCEPTED feature, unmatched later or not
                const int i2 = choice[q];
                if (i2 == 0xFFFF) continue;
                const int bin = rot_hist_bin(kl[q].angle, kc[i2].angle);
                newbin[q] = (uint8_t)bin;
                atomicAdd(&s_hist[bin], 1);
            }
            __syncthreads();
            if (tid == 0) THREE_MAXIMA_KEEP(s_hist, s_keep)
            __syncthreads();
            int removed = 0;
            for (int q = tid; q < nl; q += SBP_THREADS) {   // :691-702: only features that are still matched lose their match
                const int bb = newbin[q];
                if (bb != 0xFF && bb != s_keep[0] && bb != s_keep[1] && bb != s_keep[2] && mp[q] >= 0) { mp[q] = -1; removed++; }
            }
            if (removed) atomicAdd(&s_removed, removed);
            __syncthreads();
        }
        // :706-710 vbPrevMatched[i1] = F2.mvKeysUn[vnMatches12[i1]].pt
        float *wout = const_cast<float *>(wl);
        for (int q = tid; q < nl; q += SBP_THREADS)
            if (mp[q] >= 0) { wout[2 * q] = kx[mp[q]]; wout[2 * q + 1] = ky[mp[q]]; }
        __syncthreads();
        if (tid == 0) nmatches[pair] = s_nm - s_removed;
        publish_ack();
        return;
    }
    if (P.check_ori) {
        // rotation histogram of the new matches (:1583-1590), in parallel: bin = round((aLast - aCur [+360]) / 30)
        for (int i = tid; i < nc; i += SBP_THREADS) {
            if (newbin[i] != 0xFE) continue;
            const int bin = rot_hist_bin(query_angle(mp[i] - qown), kc[i].angle);
            newbin[i] = (uint8_t)bin;
            atomicAdd(&s_hist[bin], 1);
        }
        __syncthreads();
        if (tid == 0) THREE_MAXIMA_KEEP(s_hist, s_keep)
        __syncthreads();
        int removed = 0;
        for (int i = tid; i < nc; i += SBP_THREADS) {
            const int bb = newbin[i];
            if (bb != 0xFF && bb != s_keep[0] && bb != s_keep[1] && bb != s_keep[2]) { mp[i] = -1; removed++; }
        }
        if (removed) atomicAdd(&s_removed, removed);
        __syncthreads();
    }
    if (tid == 0) nmatches[pair] = s_nm - s_removed;
}

size_t sbp_smem_fixed_bytes(int cap, int qcap) {
    size_t b = sizeof(int) * (SBP_NCELL + 1) + sizeof(int) * SBP_NCELL + sizeof(int) * ((size_t)qcap + 1) +   // cell_start, cell_cur, q_off
               2 * sizeof(float) * (size_t)cap + sizeof(uint32_t) * (((size_t)cap + 31) / 32) +              // kx, ky, taken
               sizeof(uint16_t) * (size_t)cap + 2 * (size_t)cap +                                             // items, newbin, koct
               sizeof(int) * (size_t)cap +                       // MODE 2: matched distance, owner (u16 each); otherwise the stamps (int)
               sizeof(uint16_t) * ((size_t)qcap + ((size_t)qcap & 1)) +                                       // picks
               sizeof(uint32_t) * (((size_t)qcap + 31) / 32);                                                 // rule 0: decided bits
    return (b + 15) / 16 * 16;
}

int launch_sbp_device(const SbpParams &P, size_t smem_bytes, int npairs, const OrbfeKeyPoint *kps, const uint8_t *desc,
                      const int *counts, const int *cur_idx, const int *last_idx, const float *world, const uint8_t *flags,
                      const float *Tcw, uint32_t *scratch, int *cur_mp, int *nmatches, int *err, cudaStream_t s) {
    if (smem_bytes > 48 * 1024) {  // per device/context attribute: set on every call (cheap), never cached process-wide
        cudaError_t e = cudaFuncSetAttribute(sbp_device_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
        if (e != cudaSuccess) return (int)e;
    }
    GuidedQueries none;
    memset(&none, 0, sizeof(none));
    sbp_device_kernel<0><<<npairs, SBP_THREADS, smem_bytes, s>>>(P, kps, desc, counts, cur_idx, last_idx, world, flags, Tcw, none,
                                                             scratch, cur_mp, nmatches, err);
    return 0;
}

int launch_init_device(const SbpParams &P, size_t smem_bytes, int npairs, const OrbfeKeyPoint *kps, const uint8_t *desc,
                       const int *counts, const int *f1_idx, const int *f2_idx, float *prev_matched, uint32_t *scratch, int *match12,
                       int *nmatches, int *err, cudaStream_t s) {
    if (smem_bytes > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(sbp_device_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
        if (e != cudaSuccess) return (int)e;
    }
    GuidedQueries none;
    memset(&none, 0, sizeof(none));
    // cur = F2 (the searched frame), last = F1 (the querying frame)
    sbp_device_kernel<2><<<npairs, SBP_THREADS, smem_bytes, s>>>(P, kps, desc, counts, f2_idx, f1_idx, prev_matched, nullptr, nullptr, none,
                                                            scratch, match12, nmatches, err);
    return 0;
}

int launch_guided_device(const SbpParams &P, size_t smem_bytes, int njobs, const OrbfeKeyPoint *kps, const uint8_t *desc,
                         const int *counts, const int *frame_idx, const float *qu, const float *qv, const float *qr,
                         const int *qlo, const int *qhi, const uint8_t *qdesc, const float *qangle, const int *q_base,
                         const int *q_cnt, uint32_t *scratch, int *slot_owner, int *best_out, int *nmatches, int *err,
                         cudaStream_t s) {
    if (smem_bytes > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(sbp_device_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
        if (e != cudaSuccess) return (int)e;
    }
    GuidedQueries G;
    G.qu = qu; G.qv = qv; G.qr = qr; G.qangle = qangle; G.qlo = qlo; G.qhi = qhi; G.qdesc = qdesc; G.q_base = q_base; G.q_cnt = q_cnt;
    G.best = best_out;
    sbp_device_kernel<1><<<njobs, SBP_THREADS, smem_bytes, s>>>(P, kps, desc, counts, frame_idx, nullptr, nullptr, nullptr, nullptr, G,
                                                            scratch, slot_owner, nmatches, err);
    return 0;
}

// ------------------------------------------------------------------------------------------------
// SearchByBoW, both overloads (ORBmatcher.cc:155-284 KeyFrame vs Frame, :715-850 KeyFrame vs KeyFrame), one CTA per job.
// A FeatureVector holds every feature in exactly one node, so the "already matched" skip (:204 / :773) only ever sees
// candidates of the node being processed: the common nodes are independent and each one is replayed sequentially, in list
// order, by one warp -- the reference's result whatever order the warps take the nodes in.  The rotation histogram only
// needs the bin counts (shared-memory atomics) and each match's bin, recomputed in the final pass.
// Per side-1 feature the lanes take the free candidates in list order and keep their own two smallest
// (distance << 16 | list position) keys; the warp minimum is the first minimum of the strict-< scan, and the minimum with
// the winner's key replaced by its lane's runner-up is the reference's second best.
// ------------------------------------------------------------------------------------------------
#define BOW_THREADS 512
__global__ void __launch_bounds__(BOW_THREADS) search_by_bow_kernel(int variant, const OrbfeKeyPoint *__restrict__ kps,
                                                                    const uint8_t *__restrict__ desc, const int *__restrict__ counts,
                                                                    int cap, const int *__restrict__ fv_ids,
                                                                    const int *__restrict__ fv_ptr, const int *__restrict__ fv_items,
                                                                    const int *__restrict__ fv_n, const uint8_t *__restrict__ valid,
                                                                    const int *__restrict__ idx1, const int *__restrict__ idx2,
                                                                    float nnratio, int check_ori, int *__restrict__ out,
                                                                    int *__restrict__ nmatches, int *__restrict__ err) {
    extern __shared__ uint32_t matched2[];   // [(cap + 31) / 32] side-2 feature already matched in this job
    __shared__ int s_hist[32], s_keep[3], s_nm, s_removed, s_bad;
    const int job = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int f1 = idx1[job], f2 = idx2[job];
    const int n1 = min(max(counts[f1], 0), cap), n2 = min(max(counts[f2], 0), cap);
    const int nn1 = fv_n[f1], nn2 = fv_n[f2];
    const int nout = variant == 0 ? n2 : n1;
    int *__restrict__ row = out + (size_t)job * cap;
    const OrbfeKeyPoint *__restrict__ k1 = kps + (size_t)f1 * cap;
    const OrbfeKeyPoint *__restrict__ k2 = kps + (size_t)f2 * cap;
    const uint4 *__restrict__ d1 = reinterpret_cast<const uint4 *>(desc + (size_t)f1 * cap * 32);
    const uint4 *__restrict__ d2 = reinterpret_cast<const uint4 *>(desc + (size_t)f2 * cap * 32);
    const uint8_t *__restrict__ v1 = valid + (size_t)f1 * cap;
    const uint8_t *__restrict__ v2 = valid + (size_t)f2 * cap;
    const int *__restrict__ ids1 = fv_ids + (size_t)f1 * cap, *__restrict__ ids2 = fv_ids + (size_t)f2 * cap;
    const int *__restrict__ ptr1 = fv_ptr + (size_t)f1 * (cap + 1), *__restrict__ ptr2 = fv_ptr + (size_t)f2 * (cap + 1);
    const int *__restrict__ it1 = fv_items + (size_t)f1 * cap, *__restrict__ it2 = fv_items + (size_t)f2 * cap;

    for (int i = tid; i < (cap + 31) / 32; i += BOW_THREADS) matched2[i] = 0;
    for (int i = tid; i < nout; i += BOW_THREADS) row[i] = -1;
    if (tid < 32) s_hist[tid] = 0;
    if (tid == 0) { s_nm = 0; s_removed = 0; s_bad = (nn1 < 0 || nn1 > cap || nn2 < 0 || nn2 > cap) ? 1 : 0; }
    __syncthreads();
    const bool bad_n = s_bad != 0;
    bool bad = false;   // warp-uniform: this warp met an out-of-range node row or item index
    int nm = 0;
    for (int a = warp; a < nn1 && !bad_n && !bad; a += BOW_THREADS / 32) {
        // the side-2 node with the same id (ids ascending): lower_bound
        const int id = ids1[a];
        int lo = 0, hi = nn2;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (ids2[mid] < id) lo = mid + 1; else hi = mid;
        }
        if (lo == nn2 || ids2[lo] != id) continue;
        const int b1 = ptr1[a], e1 = ptr1[a + 1], b2 = ptr2[lo], e2 = ptr2[lo + 1];
        if (b1 < 0 || b1 > e1 || e1 > cap || b2 < 0 || b2 > e2 || e2 > cap) { bad = true; break; }
        // the first 32 candidates stay in registers for all side-1 features of the node
        int c_i2 = -1;
        uint4 c0 = make_uint4(0, 0, 0, 0), c1 = c0;
        bool c_bad = false;
        if (b2 + lane < e2) {
            c_i2 = it2[b2 + lane];
            if ((unsigned)c_i2 >= (unsigned)n2) c_bad = true;
            else if (variant == 1 && !v2[c_i2]) c_i2 = -1;   // :777 (variant 0 does not look at the Frame's map points)
            else { c0 = __ldg(&d2[2 * c_i2]); c1 = __ldg(&d2[2 * c_i2 + 1]); }
        }
        if (__any_sync(0xffffffffu, c_bad)) { bad = true; break; }
        for (int p1 = b1; p1 < e1; p1++) {
            const int i1 = it1[p1];
            if ((unsigned)i1 >= (unsigned)n1) { bad = true; break; }
            if (!v1[i1]) continue;
            const uint4 a0 = __ldg(&d1[2 * i1]), a1 = __ldg(&d1[2 * i1 + 1]);
            uint32_t m1 = 0xFFFFFFFFu, m2 = 0xFFFFFFFFu;   // this lane's two smallest keys
            if (c_i2 >= 0 && !((matched2[c_i2 >> 5] >> (c_i2 & 31)) & 1u))
                m1 = ((uint32_t)ham256(a0, a1, c0, c1) << 16) | (uint32_t)lane;
            for (int p = b2 + 32 + lane; p - lane < e2; p += 32) {
                bool lbad = false;
                if (p < e2) {
                    const int i2 = it2[p];
                    if ((unsigned)i2 >= (unsigned)n2) lbad = true;
                    else if ((variant == 0 || v2[i2]) && !((matched2[i2 >> 5] >> (i2 & 31)) & 1u)) {
                        const uint32_t key = ((uint32_t)ham256(a0, a1, __ldg(&d2[2 * i2]), __ldg(&d2[2 * i2 + 1])) << 16) | (uint32_t)(p - b2);
                        if (key < m1) { m2 = m1; m1 = key; }
                        else if (key < m2) m2 = key;
                    }
                }
                if (__any_sync(0xffffffffu, lbad)) { bad = true; break; }
            }
            if (bad) break;
            const uint32_t best = __reduce_min_sync(0xffffffffu, m1);
            if (best == 0xFFFFFFFFu) continue;
            const uint32_t second = __reduce_min_sync(0xffffffffu, m1 == best ? m2 : m1);
            const int bd = (int)(best >> 16);
            // INT_MAX stands for "no second candidate": (float)INT_MAX in the reference's comparison
            const float sd = second == 0xFFFFFFFFu ? 2147483648.0f : (float)(int)(second >> 16);
            const bool pass = variant == 0 ? bd <= 50 : bd < 50;   // TH_LOW, :224 vs :797
            if (pass && (float)bd < __fmul_rn(nnratio, sd)) {
                const int i2 = it2[b2 + (int)(best & 0xFFFF)];
                if (lane == 0) {
                    atomicOr(&matched2[i2 >> 5], 1u << (i2 & 31));
                    if (variant == 0) row[i2] = i1; else row[i1] = i2;
                    if (check_ori) atomicAdd(&s_hist[rot_hist_bin(k1[i1].angle, k2[i2].angle)], 1);
                }
                nm++;
                __syncwarp();
            }
        }
    }
    if (lane == 0) {
        if (bad) s_bad = 1;
        if (nm) atomicAdd(&s_nm, nm);
    }
    __syncthreads();
    if (s_bad) {   // malformed FeatureVector: nothing outside the frames' slots was read; the row is not meaningful
        if (tid == 0) { nmatches[job] = -1; atomicOr(err, 2); }
        return;
    }
    if (check_ori) {
        if (tid == 0) THREE_MAXIMA_KEEP(s_hist, s_keep)
        __syncthreads();
        int removed = 0;
        for (int r = tid; r < nout; r += BOW_THREADS) {
            const int o = row[r];
            if (o < 0) continue;
            const int bin = variant == 0 ? rot_hist_bin(k1[o].angle, k2[r].angle) : rot_hist_bin(k1[r].angle, k2[o].angle);
            if (bin != s_keep[0] && bin != s_keep[1] && bin != s_keep[2]) { row[r] = -1; removed++; }
        }
        if (removed) atomicAdd(&s_removed, removed);
        __syncthreads();
    }
    if (tid == 0) nmatches[job] = s_nm - s_removed;
}

int launch_search_by_bow(int variant, int njobs, const OrbfeKeyPoint *kps, const uint8_t *desc, const int *counts, int cap,
                         const int *fv_ids, const int *fv_ptr, const int *fv_items, const int *fv_n, const uint8_t *valid,
                         const int *idx1, const int *idx2, float nnratio, int check_ori, int *out, int *nmatches, int *err,
                         cudaStream_t s) {
    if (njobs <= 0) return 0;
    const size_t smem = sizeof(uint32_t) * (((size_t)cap + 31) / 32);
    search_by_bow_kernel<<<njobs, BOW_THREADS, smem, s>>>(variant, kps, desc, counts, cap, fv_ids, fv_ptr, fv_items, fv_n, valid,
                                                          idx1, idx2, nnratio, check_ori, out, nmatches, err);
    return 0;
}

// ------------------------------------------------------------------------------------------------
// SearchForTriangulation (ORBmatcher.cc:852-1014) with CheckDistEpipolarLine (:136-153), one CTA per (pKF1, pKF2) job.
// The node-disjointness argument of search_by_bow_kernel holds unchanged: vbMatched2 (:911, :940) only ever meets candidates
// of the node being processed, so warps take the common nodes in any order and each one is replayed sequentially, in list
// order, by one warp.
// Per side-1 feature the reference sorts the free candidates with distance <= TH_LOW by (distance, side-2 index) and takes
// the first one, up to 2 * best distance, that passes the epipolar test: the minimum (distance << 16 | idx2) key among the
// candidates that pass, kept iff its distance <= 2 * the minimum distance of all of them (cap <= 65535 keeps idx2 in 16
// bits).  Each lane keeps its own two minima and the warp reduces both.  Ties break by feature index, whatever order the
// node lists its items in.
// Every item of a common node is checked (index < count; octave in [0, nlevels) for side-2 features without a map point)
// before the node is matched, so whether a job is rejected does not depend on the distances.
// ------------------------------------------------------------------------------------------------
#define TRI_THREADS 512
struct TriParams { double thr[ORBFE_MAX_LEVELS]; };   // 3.84 * (double)GetSigma2(level), as in :152

// CheckDistEpipolarLine after the line l = x1' F12 = (la, lb, lc) and den = la^2 + lb^2: individually rounded, in the
// reference's order
__device__ __forceinline__ bool epipolar_ok(float la, float lb, float lc, float den, float x2, float y2, double thr) {
    const float num = __fadd_rn(__fadd_rn(__fmul_rn(la, x2), __fmul_rn(lb, y2)), lc);
    if (den == 0.0f) return false;
    const float dsqr = __fdiv_rn(__fmul_rn(num, num), den);
    return (double)dsqr < thr;
}

__global__ void __launch_bounds__(TRI_THREADS) search_for_triangulation_kernel(
    const OrbfeKeyPoint *__restrict__ kps, const uint8_t *__restrict__ desc, const int *__restrict__ counts, int cap,
    const int *__restrict__ fv_ids, const int *__restrict__ fv_ptr, const int *__restrict__ fv_items, const int *__restrict__ fv_n,
    const uint8_t *__restrict__ has_mp, const int *__restrict__ idx1, const int *__restrict__ idx2, const float *__restrict__ F12,
    const TriParams T, int nlevels, int check_ori, int *__restrict__ match12, int *__restrict__ nmatches, int *__restrict__ err) {
    extern __shared__ uint32_t matched2[];   // [(cap + 31) / 32] side-2 feature already matched in this job
    __shared__ int s_hist[32], s_keep[3], s_nm, s_removed, s_bad;
    const int job = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int f1 = idx1[job], f2 = idx2[job];
    const int n1 = min(max(counts[f1], 0), cap), n2 = min(max(counts[f2], 0), cap);
    const int nn1 = fv_n[f1], nn2 = fv_n[f2];
    int *__restrict__ row = match12 + (size_t)job * cap;
    const OrbfeKeyPoint *__restrict__ k1 = kps + (size_t)f1 * cap;
    const OrbfeKeyPoint *__restrict__ k2 = kps + (size_t)f2 * cap;
    const uint4 *__restrict__ d1 = reinterpret_cast<const uint4 *>(desc + (size_t)f1 * cap * 32);
    const uint4 *__restrict__ d2 = reinterpret_cast<const uint4 *>(desc + (size_t)f2 * cap * 32);
    const uint8_t *__restrict__ mp1 = has_mp + (size_t)f1 * cap;
    const uint8_t *__restrict__ mp2 = has_mp + (size_t)f2 * cap;
    const int *__restrict__ ids1 = fv_ids + (size_t)f1 * cap, *__restrict__ ids2 = fv_ids + (size_t)f2 * cap;
    const int *__restrict__ ptr1 = fv_ptr + (size_t)f1 * (cap + 1), *__restrict__ ptr2 = fv_ptr + (size_t)f2 * (cap + 1);
    const int *__restrict__ it1 = fv_items + (size_t)f1 * cap, *__restrict__ it2 = fv_items + (size_t)f2 * cap;
    const float *__restrict__ F = F12 + (size_t)job * 9;
    const float F0 = F[0], F1 = F[1], F2 = F[2], F3 = F[3], F4 = F[4], F5 = F[5], F6 = F[6], F7 = F[7], F8 = F[8];

    for (int i = tid; i < (cap + 31) / 32; i += TRI_THREADS) matched2[i] = 0;
    for (int i = tid; i < n1; i += TRI_THREADS) row[i] = -1;
    if (tid < 32) s_hist[tid] = 0;
    if (tid == 0) { s_nm = 0; s_removed = 0; s_bad = (nn1 < 0 || nn1 > cap || nn2 < 0 || nn2 > cap) ? 1 : 0; }
    __syncthreads();
    const bool bad_n = s_bad != 0;
    bool bad = false;   // warp-uniform: this warp met an out-of-range node row, item index or octave
    int nm = 0;
    for (int a = warp; a < nn1 && !bad_n && !bad; a += TRI_THREADS / 32) {
        // the side-2 node with the same id (ids ascending): lower_bound
        const int id = ids1[a];
        int lo = 0, hi = nn2;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (ids2[mid] < id) lo = mid + 1; else hi = mid;
        }
        if (lo == nn2 || ids2[lo] != id) continue;
        const int b1 = ptr1[a], e1 = ptr1[a + 1], b2 = ptr2[lo], e2 = ptr2[lo + 1];
        if (b1 < 0 || b1 > e1 || e1 > cap || b2 < 0 || b2 > e2 || e2 > cap) { bad = true; break; }
        bool lbad = false;
        for (int p = b1 + lane; p < e1; p += 32) lbad |= (unsigned)it1[p] >= (unsigned)n1;
        for (int p = b2 + lane; p < e2; p += 32) {
            const int i2 = it2[p];
            if ((unsigned)i2 >= (unsigned)n2) lbad = true;
            else if (!mp2[i2] && (unsigned)k2[i2].octave >= (unsigned)nlevels) lbad = true;
        }
        if (__any_sync(0xffffffffu, lbad)) { bad = true; break; }
        // the first 32 candidates stay in registers for all side-1 features of the node
        int c_i2 = -1;
        uint4 c0 = make_uint4(0, 0, 0, 0), c1 = c0;
        float c_x = 0.0f, c_y = 0.0f;
        double c_thr = 0.0;
        if (b2 + lane < e2) {
            c_i2 = it2[b2 + lane];
            if (mp2[c_i2]) c_i2 = -1;   // :911
            else {
                c0 = __ldg(&d2[2 * c_i2]); c1 = __ldg(&d2[2 * c_i2 + 1]);
                c_x = k2[c_i2].x; c_y = k2[c_i2].y; c_thr = T.thr[k2[c_i2].octave];
            }
        }
        for (int p1 = b1; p1 < e1; p1++) {
            const int i1 = it1[p1];
            if (mp1[i1]) continue;   // :895
            const uint4 a0 = __ldg(&d1[2 * i1]), a1 = __ldg(&d1[2 * i1 + 1]);
            const float x1 = k1[i1].x, y1 = k1[i1].y;
            const float la = __fadd_rn(__fadd_rn(__fmul_rn(x1, F0), __fmul_rn(y1, F3)), F6);
            const float lb = __fadd_rn(__fadd_rn(__fmul_rn(x1, F1), __fmul_rn(y1, F4)), F7);
            const float lc = __fadd_rn(__fadd_rn(__fmul_rn(x1, F2), __fmul_rn(y1, F5)), F8);
            const float den = __fadd_rn(__fmul_rn(la, la), __fmul_rn(lb, lb));
            uint32_t dmin = 0xFFFFFFFFu, kmin = 0xFFFFFFFFu;   // this lane's minimum distance / minimum passing key
            if (c_i2 >= 0 && !((matched2[c_i2 >> 5] >> (c_i2 & 31)) & 1u)) {
                const uint32_t d = (uint32_t)ham256(a0, a1, c0, c1);
                if (d <= 50) {   // TH_LOW, :918
                    dmin = d;
                    if (epipolar_ok(la, lb, lc, den, c_x, c_y, c_thr)) kmin = (d << 16) | (uint32_t)c_i2;
                }
            }
            for (int p = b2 + 32 + lane; p < e2; p += 32) {
                const int i2 = it2[p];
                if (mp2[i2] || ((matched2[i2 >> 5] >> (i2 & 31)) & 1u)) continue;
                const uint32_t d = (uint32_t)ham256(a0, a1, __ldg(&d2[2 * i2]), __ldg(&d2[2 * i2 + 1]));
                if (d > 50) continue;
                dmin = min(dmin, d);
                const uint32_t key = (d << 16) | (uint32_t)i2;
                if (key < kmin && epipolar_ok(la, lb, lc, den, k2[i2].x, k2[i2].y, T.thr[k2[i2].octave])) kmin = key;
            }
            const uint32_t best = __reduce_min_sync(0xffffffffu, dmin);
            if (best == 0xFFFFFFFFu) continue;
            const uint32_t win = __reduce_min_sync(0xffffffffu, kmin);
            if (win == 0xFFFFFFFFu || (win >> 16) > 2 * best) continue;   // DistTh = round(2 * BestDist), :929-934
            if (lane == 0) {
                const int i2 = (int)(win & 0xFFFF);
                atomicOr(&matched2[i2 >> 5], 1u << (i2 & 31));
                row[i1] = i2;
                if (check_ori) atomicAdd(&s_hist[rot_hist_bin(k1[i1].angle, k2[i2].angle)], 1);
            }
            nm++;
            __syncwarp();
        }
    }
    if (lane == 0) {
        if (bad) s_bad = 1;
        if (nm) atomicAdd(&s_nm, nm);
    }
    __syncthreads();
    if (s_bad) {   // malformed input: nothing outside the frames' slots was read; the row is not meaningful
        if (tid == 0) { nmatches[job] = -1; atomicOr(err, 4); }
        return;
    }
    if (check_ori) {   // :975-994
        if (tid == 0) THREE_MAXIMA_KEEP(s_hist, s_keep)
        __syncthreads();
        int removed = 0;
        for (int r = tid; r < n1; r += TRI_THREADS) {
            const int o = row[r];
            if (o < 0) continue;
            const int bin = rot_hist_bin(k1[r].angle, k2[o].angle);
            if (bin != s_keep[0] && bin != s_keep[1] && bin != s_keep[2]) { row[r] = -1; removed++; }
        }
        if (removed) atomicAdd(&s_removed, removed);
        __syncthreads();
    }
    if (tid == 0) nmatches[job] = s_nm - s_removed;
}

int launch_search_for_triangulation(int njobs, const OrbfeKeyPoint *kps, const uint8_t *desc, const int *counts, int cap,
                                    const int *fv_ids, const int *fv_ptr, const int *fv_items, const int *fv_n, const uint8_t *has_mp,
                                    const int *idx1, const int *idx2, const float *F12, const float *sigma2, int nlevels,
                                    int check_ori, int *match12, int *nmatches, int *err, cudaStream_t s) {
    if (njobs <= 0) return 0;
    TriParams T;
    for (int l = 0; l < ORBFE_MAX_LEVELS; l++) T.thr[l] = l < nlevels ? 3.84 * (double)sigma2[l] : 0.0;
    const size_t smem = sizeof(uint32_t) * (((size_t)cap + 31) / 32);
    search_for_triangulation_kernel<<<njobs, TRI_THREADS, smem, s>>>(kps, desc, counts, cap, fv_ids, fv_ptr, fv_items, fv_n, has_mp,
                                                                     idx1, idx2, F12, T, nlevels, check_ori, match12, nmatches, err);
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Frame::UndistortKeyPoints (reference src/Frame.cc:289-319) = cv::undistortPoints(pts, K, D, R = I, P = K): five
// fixed-point iterations of the inverse distortion model in double, then the re-projection; every operation
// individually rounded (no FMA), in the order OpenCV evaluates them -- bit-exact against python-cv2
// (tests/golden/opencv_undistort.npz).  One thread per keypoint; the other keypoint fields are copied.
// ------------------------------------------------------------------------------------------------
struct UndistortParams { double fx, fy, cx, cy, ifx, ify, k0, k1, k2, k3, k4; };

__device__ __forceinline__ void undistort_point(const UndistortParams &U, float px, float py, float &ox, float &oy) {
    double x = __dmul_rn(__dsub_rn((double)px, U.cx), U.ifx), y = __dmul_rn(__dsub_rn((double)py, U.cy), U.ify);
    const double x0 = x, y0 = y;
#pragma unroll 1
    for (int j = 0; j < 5; j++) {
        const double r2 = __dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y));
        // (1 + ((k7*r2 + k6)*r2 + k5)*r2) / (1 + ((k4*r2 + k1)*r2 + k0)*r2) with k5..k7 = 0: the numerator is exactly 1
        const double den = __dadd_rn(1.0, __dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(U.k4, r2), U.k1), r2), U.k0), r2));
        const double icdist = __ddiv_rn(1.0, den);
        const double twoxy_k2 = __dmul_rn(__dmul_rn(__dmul_rn(2.0, U.k2), x), y);                          // 2*k2*x*y
        const double dX = __dadd_rn(twoxy_k2, __dmul_rn(U.k3, __dadd_rn(r2, __dmul_rn(__dmul_rn(2.0, x), x))));  // + k3*(r2 + 2*x*x)
        const double dY = __dadd_rn(__dmul_rn(U.k2, __dadd_rn(r2, __dmul_rn(__dmul_rn(2.0, y), y))),
                                    __dmul_rn(__dmul_rn(__dmul_rn(2.0, U.k3), x), y));                      // k2*(r2 + 2*y*y) + 2*k3*x*y
        x = __dmul_rn(__dsub_rn(x0, dX), icdist);
        y = __dmul_rn(__dsub_rn(y0, dY), icdist);
    }
    // xx = fx*x + 0*y + cx, yy = 0*x + fy*y + cy, ww = 1/(0*x + 0*y + 1) = 1 (the zero products add exactly)
    ox = (float)__dadd_rn(__dmul_rn(U.fx, x), U.cx);
    oy = (float)__dadd_rn(__dmul_rn(U.fy, y), U.cy);
}

__global__ void __launch_bounds__(256) undistort_kernel(UndistortParams U, const OrbfeKeyPoint *__restrict__ in,
                                                        OrbfeKeyPoint *__restrict__ out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    OrbfeKeyPoint k = in[i];
    float ox, oy;
    undistort_point(U, k.x, k.y, ox, oy);
    k.x = ox;
    k.y = oy;
    out[i] = k;
}

void launch_undistort(float fx, float fy, float cx, float cy, const float *dist5, const OrbfeKeyPoint *d_in, OrbfeKeyPoint *d_out,
                      int n, cudaStream_t s) {
    if (n <= 0) return;
    UndistortParams U;
    U.fx = fx; U.fy = fy; U.cx = cx; U.cy = cy;
    U.ifx = 1. / U.fx; U.ify = 1. / U.fy;
    U.k0 = dist5[0]; U.k1 = dist5[1]; U.k2 = dist5[2]; U.k3 = dist5[3]; U.k4 = dist5[4];
    undistort_kernel<<<(n + 255) / 256, 256, 0, s>>>(U, d_in, d_out, n);
}

}  // namespace orbfe
