// vocab_text.cu -- orbfe_vocabulary_load_text: DBoW2's TemplatedVocabulary::loadFromTextFile (reference
// Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1338-1424) with the node table parsed in device memory.
//
// The header line is read and checked on the host (four integers).  The body goes up in chunks through two pinned staging
// buffers, then:
//   nl_count_kernel / nl_starts_kernel   newline count per 8 KB tile, exclusive scan, line starts (one thread per 32 bytes,
//                                        __vcmpeq4 over the 8 words)
//   parse_kernel                         one thread per line: parent, isLeaf, 32 descriptor bytes, the weight (exact fast
//                                        path or a fallback slot) and the first failing line (atomicMin)
//   fallback on the host                 the slots come back through the staging area; `istream >> double` on each token
//   CSR                                  child counts (atomics on the parent) + scan = child_ptr; children = node ids
//                                        stably radix-sorted by parent (LSD, 8 bits a pass), so line order within a parent
//                                        for any input; word ids = exclusive scan of the leaf flags
// The vocabulary adopts the node table the kernels wrote; the text and every scratch buffer are freed before returning.
#include <cooperative_groups.h>
#include <sys/stat.h>

#include <algorithm>
#include <cerrno>
#include <climits>
#include <cstdio>
#include <cstring>
#include <sstream>
#include <string>

#include "vocab.h"

namespace cg = cooperative_groups;

namespace orbfe {
namespace {

constexpr size_t kChunk = 8u << 20;     // bytes per staging buffer
constexpr int kNlThreads = 256;         // newline kernels: 32 bytes per thread
constexpr int kNlTile = kNlThreads * 32;
constexpr int kScThreads = 1024, kScItems = 4, kScTile = kScThreads * kScItems;
constexpr int kRsThreads = 256, kRsTile = 4096;
constexpr int kFbText = 32;             // token bytes a fallback slot carries (NUL included); longer tokens are fetched

// What parse_kernel rejects (the low byte of the error key; the line is above it)
enum { E_BLANK = 1, E_FEW = 2, E_PARENT_TOK = 3, E_LEAF_TOK = 4, E_DESC_TOK = 5, E_PARENT_RANGE = 6 };

struct FbSlot {                         // a weight for the host: node, token [start, start + len) of the body
    int node, len, start, pad;
    char text[kFbText];
};

__host__ __device__ __forceinline__ bool vt_space(unsigned c) { return c == ' ' || (c >= '\t' && c <= '\r'); }

// `>> int` on a whitespace-delimited token that must be a plain decimal int: [+-]?[0-9]+ within int's range.
// 0: ok, 1: no token before the end, 2: not a plain int.
__host__ __device__ __forceinline__ int vt_int(const uint8_t *t, int &p, int e, int &v) {
    while (p < e && vt_space(t[p])) p++;
    if (p == e) return 1;
    bool neg = false;
    unsigned c = t[p];
    if (c == '+' || c == '-') { neg = c == '-'; p++; }
    long long a = 0;
    int nd = 0;
    for (; p < e; p++) {
        c = t[p];
        if (vt_space(c)) break;
        if (c < '0' || c > '9') return 2;
        a = a < 10000000000ll ? a * 10 + (c - '0') : a;
        nd++;
    }
    if (nd == 0) return 2;
    if (neg) a = -a;
    if (a > INT_MAX || a < INT_MIN) return 2;
    v = (int)a;
    return 0;
}

__constant__ double c_p10[23] = {1e0,  1e1,  1e2,  1e3,  1e4,  1e5,  1e6,  1e7,  1e8,  1e9,  1e10, 1e11,
                                 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};

// Clinger's exact fast path: [+-]?digits[.digits]([eE][+-]?digits)? (either digit run may be empty, not both) with at most
// 15 significant digits (the mantissa is an exact double) and a decimal exponent within +-22 (10^|e| is an exact double):
// one correctly rounded multiplication or division gives strtod's result.  false: the host converts the token.
__device__ __forceinline__ bool vt_weight_fast(const uint8_t *t, int len, double *out) {
    int i = 0;
    bool neg = false;
    if (i < len && (t[i] == '+' || t[i] == '-')) { neg = t[i] == '-'; i++; }
    unsigned long long m = 0;
    int nd = 0, e10 = 0;
    bool any = false;
    for (; i < len && t[i] >= '0' && t[i] <= '9'; i++) {
        any = true;
        const int d = t[i] - '0';
        if (nd || d) {
            if (nd == 15) return false;
            m = m * 10 + d;
            nd++;
        }
    }
    if (i < len && t[i] == '.') {
        for (i++; i < len && t[i] >= '0' && t[i] <= '9'; i++) {
            any = true;
            const int d = t[i] - '0';
            if (nd || d) {
                if (nd == 15) return false;
                m = m * 10 + d;
                nd++;
            }
            e10--;
        }
    }
    if (!any) return false;
    if (i < len && (t[i] == 'e' || t[i] == 'E')) {
        i++;
        bool eneg = false;
        if (i < len && (t[i] == '+' || t[i] == '-')) { eneg = t[i] == '-'; i++; }
        int x = 0, xd = 0;
        for (; i < len && t[i] >= '0' && t[i] <= '9'; i++, xd++) x = x < 100000 ? x * 10 + (t[i] - '0') : x;
        if (xd == 0) return false;
        e10 += eneg ? -x : x;
    }
    if (i != len) return false;
    double v = 0.0;
    if (m != 0) {
        if (e10 < -22 || e10 > 22) return false;
        v = e10 >= 0 ? __dmul_rn((double)m, c_p10[e10]) : __ddiv_rn((double)m, c_p10[-e10]);
    }
    *out = neg ? -v : v;
    return true;
}

__device__ __forceinline__ int nl_in_word(uint32_t w) { return __popc(__vcmpeq4(w, 0x0A0A0A0Au)) >> 3; }

// Exclusive scan of x over the block (blockDim.x a multiple of 32, <= 1024); *total = the block's sum.  Ends on a barrier.
__device__ __forceinline__ int block_excl_scan(int x, int *total) {
    __shared__ int s_w[33];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) s_w[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        const int t = lane < nw ? s_w[lane] : 0;
        int ti = t;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, ti, o);
            if (lane >= o) ti += y;
        }
        s_w[lane] = ti - t;
        if (lane == 31) s_w[32] = ti;
    }
    __syncthreads();
    const int r = s_w[wid] + inc - x;
    *total = s_w[32];
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(kNlThreads) nl_count_kernel(const uint8_t *__restrict__ text, int T, int *__restrict__ tile_cnt) {
    const long long p = (long long)blockIdx.x * kNlTile + threadIdx.x * 32;
    int c = 0;
    if (p + 32 <= T) {
        const uint4 a = __ldg(reinterpret_cast<const uint4 *>(text + p)), b = __ldg(reinterpret_cast<const uint4 *>(text + p) + 1);
        c = nl_in_word(a.x) + nl_in_word(a.y) + nl_in_word(a.z) + nl_in_word(a.w) + nl_in_word(b.x) + nl_in_word(b.y) +
            nl_in_word(b.z) + nl_in_word(b.w);
    } else {
        for (long long i = p; i < T; i++) c += text[i] == '\n';
    }
    int total;
    block_excl_scan(c, &total);
    if (threadIdx.x == 0) tile_cnt[blockIdx.x] = total;
}

// starts[k + 1] = 1 + position of the k-th newline (starts[0] = 0 is set by the host)
__global__ void __launch_bounds__(kNlThreads) nl_starts_kernel(const uint8_t *__restrict__ text, int T, const int *__restrict__ tile_off,
                                                               int *__restrict__ starts) {
    const long long p = (long long)blockIdx.x * kNlTile + threadIdx.x * 32;
    const bool full = p + 32 <= T;
    uint4 a = make_uint4(0, 0, 0, 0), b = a;
    int c = 0;
    if (full) {
        a = __ldg(reinterpret_cast<const uint4 *>(text + p));
        b = __ldg(reinterpret_cast<const uint4 *>(text + p) + 1);
        c = nl_in_word(a.x) + nl_in_word(a.y) + nl_in_word(a.z) + nl_in_word(a.w) + nl_in_word(b.x) + nl_in_word(b.y) +
            nl_in_word(b.z) + nl_in_word(b.w);
    } else {
        for (long long i = p; i < T; i++) c += text[i] == '\n';
    }
    int total;
    int k = tile_off[blockIdx.x] + block_excl_scan(c, &total);
    if (!full) {
        for (long long i = p; i < T; i++)
            if (text[i] == '\n') starts[++k] = (int)(i + 1);
        return;
    }
    const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int j = 0; j < 8; j++) {
        uint32_t m = __vcmpeq4(w[j], 0x0A0A0A0Au);
        while (m) {
            const int byte = (__ffs(m) - 1) >> 3;
            starts[++k] = (int)(p + 4 * j + byte + 1);
            m &= ~(0xFFu << (8 * byte));
        }
    }
}

// Line i (0-based in the body, node i + 1, file line i + 2) spans [starts[i], starts[i + 1] - 1), the last one [starts[nl], T).
__global__ void __launch_bounds__(256) parse_kernel(const uint8_t *__restrict__ text, int T, const int *__restrict__ starts, int nl,
                                                    int *__restrict__ parent, int *__restrict__ leaf, uint32_t *__restrict__ desc,
                                                    double *__restrict__ weight, FbSlot *__restrict__ fb, int *__restrict__ nfb,
                                                    unsigned long long *__restrict__ err, int *__restrict__ last_blank) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > nl) return;
    const int e = i < nl ? starts[i + 1] - 1 : T;
    const int n = i + 1;
    const unsigned long long line = (unsigned long long)i + 2;
    auto fail = [&](int code) { atomicMin(err, line << 8 | (unsigned long long)code); };
    int p = starts[i];
    while (p < e && vt_space(text[p])) p++;
    if (p == e) {
        if (i == nl) *last_blank = 1;   // the text after the final newline: no node
        else fail(E_BLANK);
        return;
    }
    int v = 0;
    int r = vt_int(text, p, e, v);
    if (r) { fail(E_PARENT_TOK); return; }
    if (v < 0 || v >= n) { fail(E_PARENT_RANGE); return; }
    parent[n] = v;
    r = vt_int(text, p, e, v);
    if (r) { fail(r == 1 ? E_FEW : E_LEAF_TOK); return; }
    leaf[n] = v > 0;
    uint32_t word = 0;
    for (int j = 0; j < 32; j++) {
        r = vt_int(text, p, e, v);
        if (r) { fail(r == 1 ? E_FEW : E_DESC_TOK); return; }
        word |= (uint32_t)(v & 0xFF) << (8 * (j & 3));
        if ((j & 3) == 3) {
            desc[(size_t)n * 8 + (j >> 2)] = word;
            word = 0;
        }
    }
    while (p < e && vt_space(text[p])) p++;
    const int ws = p;
    while (p < e && !vt_space(text[p])) p++;
    double w = 0.0;
    if (p > ws && vt_weight_fast(text + ws, p - ws, &w)) {
        weight[n] = w;
        return;
    }
    weight[n] = 0.0;
    cg::coalesced_group g = cg::coalesced_threads();
    int base = 0;
    if (g.thread_rank() == 0) base = atomicAdd(nfb, (int)g.size());
    base = g.shfl(base, 0);
    FbSlot *s = fb + base + g.thread_rank();
    s->node = n;
    s->len = p - ws;
    s->start = ws;
    const int c = min(p - ws, kFbText - 1);
    for (int q = 0; q < c; q++) s->text[q] = (char)text[ws + q];
    s->text[c] = 0;
}

__global__ void fallback_scatter_kernel(const FbSlot *__restrict__ fb, const double *__restrict__ w, int nfb, double *__restrict__ weight) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < nfb) weight[fb[k].node] = w[k];
}

__global__ void child_count_kernel(const int *__restrict__ parent, int nnodes, int *__restrict__ cnt) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= 1 && n < nnodes) atomicAdd(&cnt[parent[n]], 1);
}

// word_id holds the exclusive scan of the leaf flags: keep it where the flag is set, 0 (Node()'s default) elsewhere
__global__ void finalize_kernel(const int *__restrict__ leaf, const double *__restrict__ weight, int nnodes, int *__restrict__ word_id,
                                uint8_t *__restrict__ live) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= nnodes) return;
    if (!leaf[n]) word_id[n] = 0;
    live[n] = weight[n] > 0 ? 1 : 0;
}

// ---- exclusive scan of n ints (in == out allowed): tile sums, one block scans them, tiles apply their offset ----------
__global__ void __launch_bounds__(kScThreads) sc_reduce_kernel(const int *__restrict__ in, int n, int *__restrict__ sums) {
    const long long i0 = (long long)blockIdx.x * kScTile + threadIdx.x * kScItems;
    int s = 0;
#pragma unroll
    for (int j = 0; j < kScItems; j++)
        if (i0 + j < n) s += in[i0 + j];
    int total;
    block_excl_scan(s, &total);
    if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScThreads) sc_sums_kernel(int *sums, int nb, int *total_out) {
    int carry = 0;
    for (int c0 = 0; c0 < nb; c0 += kScThreads) {
        const int i = c0 + threadIdx.x;
        const int x = i < nb ? sums[i] : 0;
        int total;
        const int ex = block_excl_scan(x, &total);
        if (i < nb) sums[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0 && total_out) *total_out = carry;
}

__global__ void __launch_bounds__(kScThreads) sc_apply_kernel(const int *in, int *out, int n, const int *__restrict__ sums) {
    const long long i0 = (long long)blockIdx.x * kScTile + threadIdx.x * kScItems;
    int x[kScItems], s = 0;
#pragma unroll
    for (int j = 0; j < kScItems; j++) {
        x[j] = i0 + j < n ? in[i0 + j] : 0;
        s += x[j];
    }
    int total;
    int run = sums[blockIdx.x] + block_excl_scan(s, &total);
#pragma unroll
    for (int j = 0; j < kScItems; j++)
        if (i0 + j < n) {
            out[i0 + j] = run;
            run += x[j];
        }
}

// ---- one stable LSD radix pass over 8 bits of the keys (parents); values are node ids, identity when vals_in is NULL ----
__global__ void __launch_bounds__(kRsThreads) rs_hist_kernel(const int *__restrict__ keys, int n, int shift, int ntiles,
                                                             int *__restrict__ hist) {
    __shared__ int h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int end = min(n, (blockIdx.x + 1) * kRsTile);
    for (int i = blockIdx.x * kRsTile + threadIdx.x; i < end; i += kRsThreads) atomicAdd(&h[(keys[i] >> shift) & 255], 1);
    __syncthreads();
    hist[threadIdx.x * ntiles + blockIdx.x] = h[threadIdx.x];
}

// Items of a tile are placed 256 at a time in index order: the rank of an item among the equal digits before it is its rank
// inside its warp (__match_any_sync) plus the counts of the earlier warps and of the earlier rounds, so the pass is stable.
__global__ void __launch_bounds__(kRsThreads) rs_scatter_kernel(const int *__restrict__ keys_in, const int *__restrict__ vals_in,
                                                                int *__restrict__ keys_out, int *__restrict__ vals_out, int n, int shift,
                                                                int ntiles, const int *__restrict__ off) {
    __shared__ int s_base[256];
    __shared__ int s_wc[kRsThreads / 32][256];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    s_base[tid] = off[tid * ntiles + blockIdx.x];
    const int end = min(n, (blockIdx.x + 1) * kRsTile);
    for (int c0 = blockIdx.x * kRsTile; c0 < end; c0 += kRsThreads) {
#pragma unroll
        for (int w = 0; w < kRsThreads / 32; w++) s_wc[w][tid] = 0;
        __syncthreads();
        const int i = c0 + tid;
        const bool ok = i < end;
        const int key = ok ? keys_in[i] : 0;
        const int d = ok ? (key >> shift) & 255 : 256;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int rank = __popc(peers & ((1u << lane) - 1u));
        if (ok && rank == 0) s_wc[wid][d] = __popc(peers);
        __syncthreads();
        int run = 0;
#pragma unroll
        for (int w = 0; w < kRsThreads / 32; w++) {
            const int c = s_wc[w][tid];
            s_wc[w][tid] = run;
            run += c;
        }
        __syncthreads();
        if (ok) {
            const int pos = s_base[d] + s_wc[wid][d] + rank;
            vals_out[pos] = vals_in ? vals_in[i] : i + 1;
            if (keys_out) keys_out[pos] = key;
        }
        __syncthreads();
        s_base[tid] += run;
    }
}

// Everything load_text allocates besides the vocabulary itself; released on every return.
struct Scratch {
    FILE *f = nullptr;
    unsigned char *h_stage[2] = {nullptr, nullptr};
    cudaEvent_t ev[2] = {nullptr, nullptr};
    cudaStream_t s0 = nullptr;
    DeviceBuffers mem;                 // the device arrays below
    uint8_t *d_text = nullptr;
    int *d_tiles = nullptr, *d_sums = nullptr, *d_starts = nullptr, *d_parent = nullptr, *d_leaf = nullptr, *d_cnt = nullptr;
    int *d_keys[2] = {nullptr, nullptr}, *d_vals = nullptr, *d_hist = nullptr, *d_scal = nullptr;
    unsigned long long *d_err = nullptr;
    FbSlot *d_fb = nullptr;
    double *d_fbw = nullptr;
    OrbfeVocabulary *v = nullptr;      // until it is handed out
    ~Scratch() {
        if (f) fclose(f);
        for (int b = 0; b < 2; b++) {
            if (h_stage[b]) cudaFreeHost(h_stage[b]);
            if (ev[b]) cudaEventDestroy(ev[b]);
        }
        if (s0) cudaStreamDestroy(s0);
        mem.release();
        if (v) orbfe_vocabulary_destroy(v);
    }
};

int div_up(long long a, int b) { return (int)((a + b - 1) / b); }

// exclusive scan of n ints; *d_total (may be NULL) receives the sum.  d_sums holds div_up(n, kScTile) ints.
void scan_excl(const int *in, int *out, int n, int *d_sums, int *d_total, cudaStream_t s) {
    const int nb = std::max(div_up(n, kScTile), 1);
    sc_reduce_kernel<<<nb, kScThreads, 0, s>>>(in, n, d_sums);
    sc_sums_kernel<<<1, kScThreads, 0, s>>>(d_sums, nb, d_total);
    sc_apply_kernel<<<nb, kScThreads, 0, s>>>(in, out, n, d_sums);
}

// The header `k L scoring weighting` as `>> m_k >> m_L >> n1 >> n2` reads it, each a plain int
int parse_header(const std::string &h, int hv[4]) {
    int p = 0;
    for (int j = 0; j < 4; j++)
        if (vt_int(reinterpret_cast<const uint8_t *>(h.data()), p, (int)h.size(), hv[j]))
            return set_error(ORBFE_ERR_ARG, "line 1: the header needs four integers `k L scoring weighting`");
    if (hv[0] < 0 || hv[0] > 20) return set_error(ORBFE_ERR_ARG, "line 1: header k = %d outside [0, 20]", hv[0]);
    if (hv[1] < 1 || hv[1] > 10) return set_error(ORBFE_ERR_ARG, "line 1: header L = %d outside [1, 10]", hv[1]);
    if (hv[2] < 0 || hv[2] > 5) return set_error(ORBFE_ERR_ARG, "line 1: header scoring = %d outside [0, 5]", hv[2]);
    if (hv[3] < 0 || hv[3] > 3) return set_error(ORBFE_ERR_ARG, "line 1: header weighting = %d outside [0, 3]", hv[3]);
    return ORBFE_OK;
}

// GeneralScoring::mustNormalize of scoring objects 0..5 (ScoringObject.h): L1, L2, chi-square, KL, Bhattacharyya, dot product
const int kScoringNorm[6] = {ORBFE_BOW_NORM_L1, ORBFE_BOW_NORM_L2, ORBFE_BOW_NORM_L1, ORBFE_BOW_NORM_L1, ORBFE_BOW_NORM_L1,
                             ORBFE_BOW_NORM_NONE};

const char *error_text(int code) {
    switch (code) {
        case E_BLANK: return "empty or blank line before the last line";
        case E_FEW: return "fewer than 34 tokens before the weight";
        case E_PARENT_TOK: return "the parent is not a plain decimal int";
        case E_LEAF_TOK: return "isLeaf is not a plain decimal int";
        case E_DESC_TOK: return "a descriptor byte is not a plain decimal int";
        default: return "the parent is negative or not an earlier node";
    }
}

}  // namespace
}  // namespace orbfe

using namespace orbfe;

extern "C" int orbfe_vocabulary_load_text(int device, const char *path, OrbfeVocabulary **out) {
    if (!out) return set_error(ORBFE_ERR_ARG, "out is NULL");
    *out = nullptr;
    if (!path) return set_error(ORBFE_ERR_ARG, "NULL path");
    Scratch S;
    S.f = fopen(path, "rb");
    if (!S.f) return set_error(ORBFE_ERR_ARG, "cannot open %s: %s", path, strerror(errno));
    struct stat st;
    if (fstat(fileno(S.f), &st) != 0 || !S_ISREG(st.st_mode)) return set_error(ORBFE_ERR_ARG, "%s is not a readable regular file", path);
    std::string hdr;
    int ch;
    while ((ch = fgetc(S.f)) != EOF && ch != '\n') hdr.push_back((char)ch);
    if (ferror(S.f)) return set_error(ORBFE_ERR_ARG, "cannot read %s: %s", path, strerror(errno));
    int hv[4];
    if (int rc = parse_header(hdr, hv)) return rc;
    const long long hdr_len = (long long)hdr.size() + (ch == '\n' ? 1 : 0);
    const long long body = (long long)st.st_size - hdr_len;
    if (body >= INT_MAX) return set_error(ORBFE_ERR_ARG, "%s: a body of %lld bytes; at most %d are supported", path, body, INT_MAX - 1);
    const int T = (int)std::max(body, 0ll);

    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return set_error(ORBFE_ERR_NO_DEVICE, "no CUDA device: this library has no CPU fallback");
    }
    if (device < 0 || device >= ndev) return set_error(ORBFE_ERR_ARG, "device %d out of range", device);
    ORBFE_CUDA_TRY(cudaSetDevice(device));

    // ---- the body into device memory, chunk by chunk through two pinned buffers ----
    ORBFE_CUDA_TRY(cudaStreamCreateWithFlags(&S.s0, cudaStreamNonBlocking));
    cudaStream_t s = S.s0;
    const int ntl = std::max(div_up(T, kNlTile), 1);
    ORBFE_CUDA_TRY(S.mem.alloc(&S.d_text, (size_t)T + 32));
    ORBFE_CUDA_TRY(S.mem.alloc(&S.d_tiles, (size_t)ntl));
    ORBFE_CUDA_TRY(S.mem.alloc(&S.d_sums, (size_t)(div_up(std::max<long long>(ntl, 2ll * T + 1024), kScTile) + 1)));
    ORBFE_CUDA_TRY(S.mem.alloc(&S.d_scal, 8));
    ORBFE_CUDA_TRY(S.mem.alloc(&S.d_err, 1));
    for (int b = 0; b < 2; b++) {
        ORBFE_CUDA_TRY(cudaHostAlloc((void **)&S.h_stage[b], kChunk, cudaHostAllocDefault));
        ORBFE_CUDA_TRY(cudaEventCreateWithFlags(&S.ev[b], cudaEventDisableTiming));
    }
    for (long long off = 0, k = 0; off < T; k++) {
        const int b = (int)(k & 1);
        if (k >= 2) ORBFE_CUDA_TRY(cudaEventSynchronize(S.ev[b]));
        const size_t len = (size_t)std::min<long long>(kChunk, T - off);
        if (fread(S.h_stage[b], 1, len, S.f) != len) return set_error(ORBFE_ERR_ARG, "cannot read %s: short read", path);
        ORBFE_CUDA_TRY(cudaMemcpyAsync(S.d_text + off, S.h_stage[b], len, cudaMemcpyHostToDevice, s));
        ORBFE_CUDA_TRY(cudaEventRecord(S.ev[b], s));
        off += (long long)len;
    }
    fclose(S.f);
    S.f = nullptr;

    // ---- line starts ----
    int *d_nl = S.d_scal;           // scalars: [0] newlines, [1] fallbacks, [2] last line blank, [3] leaf flags
    ORBFE_CUDA_TRY(cudaMemsetAsync(S.d_scal, 0, sizeof(int) * 8, s));
    if (T > 0) {
        nl_count_kernel<<<ntl, kNlThreads, 0, s>>>(S.d_text, T, S.d_tiles);
        scan_excl(S.d_tiles, S.d_tiles, ntl, S.d_sums, d_nl, s);
    }
    int nl = 0;
    ORBFE_CUDA_TRY(cudaMemcpyAsync(&nl, d_nl, sizeof(int), cudaMemcpyDeviceToHost, s));
    ORBFE_CUDA_TRY(cudaStreamSynchronize(s));
    ORBFE_CUDA_TRY(cudaGetLastError());
    if ((long long)nl + 2 > INT_MAX) return set_error(ORBFE_ERR_ARG, "%s: more than %d nodes", path, INT_MAX);
    const int cap = nl + 2;         // nodes if the text after the last newline is a node line
    ORBFE_CUDA_TRY(S.mem.alloc(&S.d_starts, (size_t)nl + 1));
    ORBFE_CUDA_TRY(cudaMemsetAsync(S.d_starts, 0, sizeof(int), s));
    if (nl > 0) nl_starts_kernel<<<ntl, kNlThreads, 0, s>>>(S.d_text, T, S.d_tiles, S.d_starts);

    // ---- parse into the vocabulary's own table ----
    OrbfeVocabulary *v = S.v = new OrbfeVocabulary();
    v->device = device;
    ORBFE_CUDA_TRY(vocab_alloc(v, cap, cap - 1));
    ORBFE_CUDA_TRY(S.mem.alloc(&S.d_parent, (size_t)cap));
    ORBFE_CUDA_TRY(S.mem.alloc(&S.d_leaf, (size_t)cap));
    ORBFE_CUDA_TRY(S.mem.alloc(&S.d_fb, (size_t)nl + 1));
    ORBFE_CUDA_TRY(cudaMemsetAsync(S.d_parent, 0, sizeof(int), s));
    ORBFE_CUDA_TRY(cudaMemsetAsync(S.d_leaf, 0, sizeof(int), s));
    ORBFE_CUDA_TRY(cudaMemsetAsync(v->d_weight, 0, sizeof(double), s));
    ORBFE_CUDA_TRY(cudaMemsetAsync(v->d_desc, 0, 32, s));
    ORBFE_CUDA_TRY(cudaMemsetAsync(S.d_err, 0xFF, sizeof(unsigned long long), s));
    parse_kernel<<<div_up((long long)nl + 1, 256), 256, 0, s>>>(S.d_text, T, S.d_starts, nl, S.d_parent, S.d_leaf,
                                                                reinterpret_cast<uint32_t *>(v->d_desc), v->d_weight, S.d_fb,
                                                                S.d_scal + 1, S.d_err, S.d_scal + 2);
    int scal[3];
    unsigned long long err = 0;
    ORBFE_CUDA_TRY(cudaMemcpyAsync(scal, S.d_scal, sizeof(scal), cudaMemcpyDeviceToHost, s));
    ORBFE_CUDA_TRY(cudaMemcpyAsync(&err, S.d_err, sizeof(err), cudaMemcpyDeviceToHost, s));
    ORBFE_CUDA_TRY(cudaStreamSynchronize(s));
    ORBFE_CUDA_TRY(cudaGetLastError());
    if (err != ~0ull) return set_error(ORBFE_ERR_ARG, "%s: line %llu: %s", path, err >> 8, error_text((int)(err & 0xFF)));
    const int nfb = scal[1];
    const int nnodes = 1 + nl + (scal[2] ? 0 : 1);

    // ---- weights the device did not convert: `>> double` on their tokens, in batches through the staging buffers ----
    if (nfb > 0) {
        ORBFE_CUDA_TRY(S.mem.alloc(&S.d_fbw, (size_t)nfb));
        const int batch = (int)(kChunk / sizeof(FbSlot));
        const FbSlot *slots = reinterpret_cast<const FbSlot *>(S.h_stage[0]);
        double *w = reinterpret_cast<double *>(S.h_stage[1]);
        std::string tok;
        for (int b0 = 0; b0 < nfb; b0 += batch) {
            const int nb = std::min(batch, nfb - b0);
            ORBFE_CUDA_TRY(cudaMemcpyAsync(S.h_stage[0], S.d_fb + b0, sizeof(FbSlot) * (size_t)nb, cudaMemcpyDeviceToHost, s));
            ORBFE_CUDA_TRY(cudaStreamSynchronize(s));   // also: the previous batch's weights have left h_stage[1]
            for (int k = 0; k < nb; k++) {
                const FbSlot &sl = slots[k];
                if (sl.len < kFbText) {
                    tok.assign(sl.text, (size_t)sl.len);
                } else {
                    tok.resize((size_t)sl.len);
                    ORBFE_CUDA_TRY(cudaMemcpy(&tok[0], S.d_text + sl.start, (size_t)sl.len, cudaMemcpyDeviceToHost));
                }
                std::istringstream is(tok);
                double x = 0.0;                 // Node()'s weight: kept when nothing is extracted
                is >> x;
                w[k] = x;
            }
            ORBFE_CUDA_TRY(cudaMemcpyAsync(S.d_fbw + b0, w, sizeof(double) * (size_t)nb, cudaMemcpyHostToDevice, s));
        }
        fallback_scatter_kernel<<<div_up(nfb, 256), 256, 0, s>>>(S.d_fb, S.d_fbw, nfb, v->d_weight);
    }

    // ---- CSR, word ids, live flags ----
    ORBFE_CUDA_TRY(S.mem.alloc(&S.d_cnt, (size_t)nnodes + 1));
    ORBFE_CUDA_TRY(cudaMemsetAsync(S.d_cnt, 0, sizeof(int) * ((size_t)nnodes + 1), s));
    child_count_kernel<<<div_up(nnodes, 256), 256, 0, s>>>(S.d_parent, nnodes, S.d_cnt);
    scan_excl(S.d_cnt, v->d_child_ptr, nnodes + 1, S.d_sums, nullptr, s);
    scan_excl(S.d_leaf, v->d_word_id, nnodes, S.d_sums, S.d_scal + 3, s);
    finalize_kernel<<<div_up(nnodes, 256), 256, 0, s>>>(S.d_leaf, v->d_weight, nnodes, v->d_word_id, v->d_live);
    const int nitems = nnodes - 1;  // nodes 1 .. nnodes-1, keyed by parent
    if (nitems > 0) {
        int bits = 1;
        while (bits < 31 && (1 << bits) <= nnodes - 1) bits++;
        const int npass = (bits + 7) / 8, ntiles = div_up(nitems, kRsTile);
        ORBFE_CUDA_TRY(S.mem.alloc(&S.d_hist, 256 * (size_t)ntiles));
        ORBFE_CUDA_TRY(S.mem.alloc(&S.d_vals, (size_t)nitems));
        for (int b = 0; b < 2 && npass > 1; b++) ORBFE_CUDA_TRY(S.mem.alloc(&S.d_keys[b], (size_t)nitems));
        const int *keys = S.d_parent + 1, *vals = nullptr;
        for (int ps = 0; ps < npass; ps++) {
            const bool last = ps == npass - 1;
            // the last pass writes the children; the values ping-pong between d_vals and d_children before it
            int *vals_out = last ? v->d_children : ((npass - 1 - ps) & 1 ? S.d_vals : v->d_children);
            int *keys_out = last ? nullptr : S.d_keys[ps & 1];
            rs_hist_kernel<<<ntiles, kRsThreads, 0, s>>>(keys, nitems, 8 * ps, ntiles, S.d_hist);
            scan_excl(S.d_hist, S.d_hist, 256 * ntiles, S.d_sums, nullptr, s);
            rs_scatter_kernel<<<ntiles, kRsThreads, 0, s>>>(keys, vals, keys_out, vals_out, nitems, 8 * ps, ntiles, S.d_hist);
            keys = keys_out;
            vals = vals_out;
        }
    }
    int nleaf = 0;
    ORBFE_CUDA_TRY(cudaMemcpyAsync(&nleaf, S.d_scal + 3, sizeof(int), cudaMemcpyDeviceToHost, s));
    ORBFE_CUDA_TRY(cudaStreamSynchronize(s));
    ORBFE_CUDA_TRY(cudaGetLastError());

    v->nnodes = nnodes;
    v->nchild = nitems;
    v->k = hv[0];
    v->depth = hv[1];
    v->scoring = hv[2];
    v->weighting = hv[3];
    v->norm = kScoringNorm[hv[2]];
    v->nwords = std::max(nleaf, 1);     // as create() counts: the largest word id + 1, every node's word id >= 0
    *out = v;
    S.v = nullptr;
    return ORBFE_OK;
}
