// orbfe_api.cu -- host side of liborbfe.so: the extractor/matcher handles, the per-geometry plan and the
// extern "C" entry points declared in include/orbfe.h.
//
// Host float arithmetic here reproduces the reference constructor and OpenCV's resize tables
// (src/ORBextractor.cc:457-511, :785-786, :527-547); this translation unit is compiled with
// -ffp-contract=off so that every float operation is individually rounded, as the canonical
// semantics require (DESIGN.md).
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <string>
#include <utility>
#include <vector>
#include <atomic>
#include <climits>
#include <memory>
#include <thread>
#include <unordered_map>

#include "../../include/orbfe_bow.h"
#include "../../include/orbfe_match.h"
#include "orbfe_internal.h"

using namespace orbfe;

// ------------------------------------------------------------------------------------------------
// error plumbing
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";

int orbfe::set_error(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
static int (*const fail)(int, const char *, ...) = orbfe::set_error;  // this file's spelling

extern "C" const char *orbfe_last_error(void) { return g_err; }
extern "C" int orbfe_version(void) { return ORBFE_VERSION; }
extern "C" int orbfe_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

static const int8_t kBriefPattern[1024] = {
#include "../../include/orbfe_brief_pattern.inc"
};

// OpenCV rounding helpers: cvRound = round-half-even of the double value
static inline int cv_round(double v) { return (int)std::lrint(v); }
static inline int cv_floor(double v) { int i = (int)v; return i - (i > v); }

// ------------------------------------------------------------------------------------------------
// Extractor
// ------------------------------------------------------------------------------------------------
struct StageTimer {
    std::vector<std::string> names;
    std::vector<cudaEvent_t> ev;  // names.size()+1 events
    bool origin_pending = true;
};

// One plan of a handle: a level table (PlanDev: one geometry; MultiPlanDev: up to ORBFE_MULTI_MAX_GROUPS) with its level
// planes, work buffers and the outputs of the host-array entries.  Keyed by the (W, H) list of its groups and the frames
// each group holds; an empty key means no plan.
template <class PD>
struct Plan {
    std::vector<int> geom, cap;   // key: (W, H) of group g at geom[2g], geom[2g + 1]; cap[g] frames of group g
    std::unique_ptr<PD> hp;       // host copy (a MultiPlanDev is large: on the heap)
    PD *dp = nullptr;             // device copy
    WorkDev work;
    DeviceBuffers mem;            // every device allocation of the plan
    void *counters = nullptr;     // cell_cnt_lo | cell_cnt_hi | kept_cnt (zeroed per call)
    size_t counters_bytes = 0, ls_smem = 0;
    // level 0 of a group either lives in the plan's own pitched planes or IS the caller's device buffer (no ingest copy)
    LevelDev own0[ORBFE_MULTI_MAX_GROUPS];
    OrbfeKeyPoint *d_kps = nullptr;   // outputs of the host-array entries, [sum of cap] frames
    uint8_t *d_desc = nullptr;
    int *d_counts = nullptr;

    void release() {
        mem.release();
        geom.clear();
        cap.clear();
    }
};

struct OrbfeExtractor {
    int nfeatures = 0, nlevels = 0, score_type = 1, fast_th = 20, device = 0;
    int batch_mode = 0;         // orbfe_extractor_set_batch_mode
    double scale_factor = 1.2;  // double member initialised from a float (ORBextractor.h:62, .cc:459)
    float scale[ORBFE_MAX_LEVELS], inv_scale[ORBFE_MAX_LEVELS];
    int quota[ORBFE_MAX_LEVELS];

    Plan<PlanDev> single;        // orbfe_extract, orbfe_extract_batch*
    Plan<MultiPlanDev> multi;    // orbfe_extract_multi*
    int8_t *d_pattern = nullptr;
    void *tma_encode = nullptr;  // cuTensorMapEncodeTiled
    int *h_counts = nullptr;     // pinned
    int *h_err = nullptr;        // pinned
    size_t h_counts_cap = 0;

    HandleStream hs;            // every call enters and leaves it, whichever stream it is enqueued on
    cudaStream_t copy_stream = nullptr;
    std::vector<cudaEvent_t> chunk_ev;
    int last_launches = 0;
    int plan_builds = 0;
    bool profiling = false;
    StageTimer timer;
    std::vector<float> stage_ms;
    std::vector<std::string> stage_names;
};

// the pinned block the host-array entries read the counts back into
static int grow_host_counts(OrbfeExtractor *ex, int n) {
    if (ex->h_counts_cap < (size_t)n) {
        if (ex->h_counts) cudaFreeHost(ex->h_counts);
        ex->h_counts = nullptr;
        ex->h_counts_cap = 0;
        ORBFE_CUDA_TRY(cudaHostAlloc((void **)&ex->h_counts, sizeof(int) * n, cudaHostAllocDefault));
        ex->h_counts_cap = n;
    }
    return ORBFE_OK;
}

// cv::resize INTER_LINEAR tap tables for one axis (OpenCV imgproc resize.cpp semantics, see SURVEY 8c)
static void resize_axis(int dn, int sn, bool clamp_weights, std::vector<int> &ofs, std::vector<short2> &ab) {
    ofs.resize(dn);
    ab.resize(dn);
    const double scale = 1.0 / ((double)dn / (double)sn);
    for (int d = 0; d < dn; d++) {
        float f = (float)(((double)d + 0.5) * scale - 0.5);
        int s = cv_floor((double)f);
        f -= (float)s;
        if (clamp_weights) {  // horizontal: sx<0 -> (0,f=0); sx>=sn-1 -> (sn-1,f=0)
            if (s < 0) { s = 0; f = 0.f; }
            if (s >= sn - 1) { s = sn - 1; f = 0.f; }
        }
        ofs[d] = s;
        ab[d].x = (short)cv_round((double)((1.f - f) * 2048.f));
        ab[d].y = (short)cv_round((double)(f * 2048.f));
    }
}

// The 3-D (x, y, frame) tensor map of one unblurred level, as fast_nms_tma_kernel loads its pixel tiles: a box of
// F2_TW x F2_PH x 1 bytes.  `encode` is the driver's cuTensorMapEncodeTiled; pitch and plane are the byte strides of y and frame.
static CUresult encode_level_map(void *encode, CUtensorMap *map, uint8_t *ptr, int w, int h, int frames, int pitch, size_t plane) {
    typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                 const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    const cuuint64_t dims[3] = {(cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)frames};
    const cuuint64_t strides[2] = {(cuuint64_t)pitch, (cuuint64_t)plane};
    const cuuint32_t box[3] = {160, ORBFE_FT_H + 8, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    return ((EncodeFn)encode)(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

// Running totals of a level table being laid out.  Cell ids and FAST / blur tiles run on across the geometries of a multi
// plan; candidate slots, kept lists and keypoint slots restart at 0 in each geometry, so the per-frame strides are the
// largest geometry's.
struct PlanLayout {
    int cell_base = 0, ft_base = 0, bt_base = 0, max_kept = 0, kept_total = 0, kp_total = 0;
    long long cand_total = 0;
    std::vector<long long> cand_base;   // [cells] first candidate slot of each cell inside its frame
    std::vector<int> cand_cap;          // [cells]
};

// The levels of one W x H geometry in lv[0, nlevels): sizes, cell grid, bases, tile counts and candidate slots.  Host only:
// nothing is allocated or launched.  ORBFE_ERR_UNSUPPORTED for a geometry outside the supported domain.
static int layout_geometry(const OrbfeExtractor *ex, int W, int H, LevelDev *lv, PlanLayout &A) {
    const float ratio = (float)W / (float)H;  // :527 (level-0 dims)
    int kp_base = 0, kept_base = 0;
    long long cand_total = 0;
    for (int l = 0; l < ex->nlevels; l++) {
        LevelDev &L = lv[l];
        L.w = cv_round((double)((float)W * ex->inv_scale[l]));  // :785-786
        L.h = cv_round((double)((float)H * ex->inv_scale[l]));
        if (L.w < 1 || L.h < 1 || L.w > 65535 || L.h > 32767)
            return fail(ORBFE_ERR_UNSUPPORTED, "level %d size %dx%d outside the supported domain", l, L.w, L.h);
        L.pitch = (L.w + 127) / 128 * 128;
        L.plane = (size_t)L.pitch * L.h;
        L.quota = ex->quota[l];
        L.scale = ex->scale[l];
        L.patch_size = (float)(int)(31.0f * ex->scale[l]);  // :675
        // cell grid, :533-547
        L.cols = (int)std::sqrt((float)L.quota / (5.0f * ratio));
        L.rows = (int)(ratio * (float)L.cols);
        const int Wd = L.w - 2 * ORBFE_EDGE, Hd = L.h - 2 * ORBFE_EDGE;
        // levelCols == 0 (a quota below 5*ratio) or levelRows == 0 (portrait images): the reference's cell vectors are
        // empty, its loops over the rows do nothing and the level yields no keypoints while the others run (:549-703)
        const bool empty_level = L.cols < 1 || L.rows < 1;
        if (empty_level) {
            L.cols = L.rows = 0;
            L.cw = L.ch = 1;
            L.cw_rcp = L.ch_rcp = 1;
            L.ncells = 0;
            L.nfc = 0;
        } else {
            if (Wd < 1 || Hd < 1)
                return fail(ORBFE_ERR_UNSUPPORTED, "level %d (%dx%d): no pixels inside the 16-px detection border", l, L.w, L.h);
            L.cw = (int)std::ceil((float)Wd / (float)L.cols);
            L.ch = (int)std::ceil((float)Hd / (float)L.rows);
            if (L.cw < 2 || L.ch < 2)
                return fail(ORBFE_ERR_UNSUPPORTED, "level %d: %dx%d-pixel cells (image too small for %d features)", l, L.cw, L.ch, L.quota);
            L.cw_rcp = (uint32_t)((0x100000000ull + (unsigned)L.cw - 1) / (unsigned)L.cw);
            L.ch_rcp = (uint32_t)((0x100000000ull + (unsigned)L.ch - 1) / (unsigned)L.ch);
            L.ncells = L.rows * L.cols;
            L.nfc = (int)std::ceil((float)L.quota / (float)L.ncells);
            if ((L.cols - 1) * L.cw > Wd || (L.rows - 1) * L.ch > Hd)
                return fail(ORBFE_ERR_UNSUPPORTED, "level %d: cell grid does not tile the detect area (image too small)", l);
            // a FAST tile (ORBFE_FT_W x ORBFE_FT_H) may overlap at most 64 cells (shared-memory counters)
            if (((ORBFE_FT_W + L.cw - 2) / L.cw + 1) * ((ORBFE_FT_H + L.ch - 2) / L.ch + 1) > 64)
                return fail(ORBFE_ERR_UNSUPPORTED, "level %d: cells of %dx%d are too small for the FAST tile", l, L.cw, L.ch);
            if (L.ncells > 4096 || (long long)L.cw * L.ch > (1 << 24))
                return fail(ORBFE_ERR_UNSUPPORTED, "level %d: %d cells of %dx%d exceed the key layout", l, L.ncells, L.cw, L.ch);
        }
        L.cell_base = A.cell_base;
        A.cell_base += L.ncells;
        L.kp_base = kp_base;
        kp_base += L.quota;
        L.kept_base = kept_base;
        L.kept_cap = L.quota + 2 * L.ncells + 64;
        kept_base += L.kept_cap;
        A.max_kept = std::max(A.max_kept, L.kept_cap);
        L.ftiles_x = empty_level ? 0 : (Wd + ORBFE_FT_W - 1) / ORBFE_FT_W;
        L.ftiles_y = empty_level ? 0 : (Hd + ORBFE_FT_H - 1) / ORBFE_FT_H;
        L.ftile_base = A.ft_base;
        A.ft_base += L.ftiles_x * L.ftiles_y;
        L.btiles_x = (L.w + ORBFE_BT_W - 1) / ORBFE_BT_W;
        L.btiles_y = (L.h + ORBFE_BT_H - 1) / ORBFE_BT_H;
        L.btile_base = A.bt_base;
        A.bt_base += L.btiles_x * L.btiles_y;
        for (int i = 0; i < L.rows; i++)
            for (int j = 0; j < L.cols; j++) {
                const int ww = (j == L.cols - 1) ? Wd - j * L.cw : L.cw;
                const int hh = (i == L.rows - 1) ? Hd - i * L.ch : L.ch;
                const int cap = std::max(1, ((ww + 1) / 2) * ((hh + 1) / 2));  // strict 8-neighbour maxima bound
                A.cand_base.push_back(cand_total);
                A.cand_cap.push_back(cap);
                cand_total += cap;
            }
    }
    A.cand_total = std::max(A.cand_total, cand_total);
    A.kept_total = std::max(A.kept_total, kept_base);
    // keypoint slots = sum of the per-level quotas; equals nfeatures whenever the last-level remainder
    // max(nfeatures - sum, 0) is not clipped (:487)
    A.kp_total = kp_base;
    return ORBFE_OK;
}

// Shared memory of the level-select kernels for a plan whose largest kept list is max_kept; the kernels' attribute only ever
// grows (it is per process, and another plan may need more)
static int level_select_smem(const OrbfeExtractor *ex, int max_kept, size_t *bytes) {
    *bytes = ex->score_type == 0 ? (size_t)level_select_harris_smem_bytes(max_kept) : (size_t)level_select_smem_bytes(max_kept);
    if (*bytes > 200 * 1024)
        return fail(ORBFE_ERR_UNSUPPORTED, "nfeatures too large for the level-select kernel (%zu B smem)", *bytes);
    return ORBFE_OK;
}

static int set_level_select_attr(const OrbfeExtractor *ex, size_t bytes) {
    if (bytes > 48 * 1024) {
        cudaError_t e = (cudaError_t)(ex->score_type == 0 ? set_level_select_harris_smem((int)bytes) : set_level_select_smem((int)bytes));
        if (e != cudaSuccess) return fail(ORBFE_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    }
    return ORBFE_OK;
}

// Device part of one geometry laid out in lv[0, nlevels) (entries v0 .. v0 + nlevels - 1 of the level table): the level
// planes for B frames (level 0 too: it serves callers whose frames cannot be read in place), the resize tables, and the
// geometry's FAST and blur tile entries and tensor maps, written into the plan's tables.
static int alloc_geometry(OrbfeExtractor *ex, DeviceBuffers &mem, LevelDev *lv, int B, int v0, void *encode,
                          std::vector<FTileInfo> &info, std::vector<BTileInfo> &binfo, std::vector<CUtensorMap> &maps) {
    for (int l = 0; l < ex->nlevels; l++) {
        LevelDev &L = lv[l];
        ORBFE_CUDA_TRY(mem.alloc(&L.pyr, L.plane * B + 256));
        ORBFE_CUDA_TRY(mem.alloc(&L.blur, L.plane + 256));  // one plane, for orbfe_debug_read_level
        ORBFE_CUDA_TRY(cudaMemsetAsync(L.pyr, 0, L.plane * B + 256, ex->hs.stream));
        if (l > 0) {
            const LevelDev &S = lv[l - 1];
            std::vector<int> xo, yo;
            std::vector<short2> xab, yab;
            resize_axis(L.w, S.w, true, xo, xab);
            resize_axis(L.h, S.h, false, yo, yab);
            std::vector<int2> yr(L.h);
            for (int y = 0; y < L.h; y++) {  // rows sy, sy+1 clipped to [0, sh-1]; weights not reset at the clip
                yr[y].x = std::min(std::max(yo[y], 0), S.h - 1);
                yr[y].y = std::min(std::max(yo[y] + 1, 0), S.h - 1);
            }
            // the kernel reads the x tables four entries at a time: pad with copies of the last entry
            while (xo.size() % 4 || xo.size() < (size_t)L.w + 4) { xo.push_back(xo[L.w - 1]); xab.push_back(xab[L.w - 1]); }
            L.rz_fast = 1;
            for (size_t x4 = 0; x4 + 3 < xo.size(); x4 += 4)
                if (xo[x4 + 3] - (xo[x4] & ~3) > 7) L.rz_fast = 0;
            if (L.rz_fast) {  // 2: the first three columns of every quad start within 6 bytes (single-PRMT extraction)
                L.rz_fast = 2;
                for (size_t x4 = 0; x4 + 3 < xo.size(); x4 += 4)
                    if (xo[x4 + 2] - (xo[x4] & ~3) > 6) L.rz_fast = 1;
            }
            int *dxo; short2 *dxab; int2 *dyr; short2 *dyab;
            ORBFE_CUDA_TRY(mem.alloc(&dxo, xo.size()));
            ORBFE_CUDA_TRY(mem.alloc(&dxab, xab.size()));
            ORBFE_CUDA_TRY(mem.alloc(&dyr, (size_t)L.h));
            ORBFE_CUDA_TRY(mem.alloc(&dyab, (size_t)L.h));
            ORBFE_CUDA_TRY(cudaMemcpy(dxo, xo.data(), sizeof(int) * xo.size(), cudaMemcpyHostToDevice));
            ORBFE_CUDA_TRY(cudaMemcpy(dxab, xab.data(), sizeof(short2) * xab.size(), cudaMemcpyHostToDevice));
            ORBFE_CUDA_TRY(cudaMemcpy(dyr, yr.data(), sizeof(int2) * L.h, cudaMemcpyHostToDevice));
            ORBFE_CUDA_TRY(cudaMemcpy(dyab, yab.data(), sizeof(short2) * L.h, cudaMemcpyHostToDevice));
            L.xofs = dxo; L.xab = dxab; L.yrows = dyr; L.yab = dyab;
        }
    }
    // per-tile cell geometry for the FAST kernel
    for (int l = 0; l < ex->nlevels; l++) {
        const LevelDev &L = lv[l];
        const int xmax = L.w - ORBFE_EDGE, ymax = L.h - ORBFE_EDGE;
        for (int ty = 0; ty < L.ftiles_y; ty++)
            for (int tx = 0; tx < L.ftiles_x; tx++) {
                FTileInfo &T = info[(size_t)L.ftile_base + ty * L.ftiles_x + tx];
                const int x0 = ORBFE_EDGE + tx * ORBFE_FT_W, y0 = ORBFE_EDGE + ty * ORBFE_FT_H;
                const int x1 = std::min(x0 + ORBFE_FT_W, xmax) - 1, y1 = std::min(y0 + ORBFE_FT_H, ymax) - 1;
                const int cj0 = std::min((x0 - ORBFE_EDGE) / L.cw, L.cols - 1), cj1 = std::min((x1 - ORBFE_EDGE) / L.cw, L.cols - 1);
                const int ci0 = std::min((y0 - ORBFE_EDGE) / L.ch, L.rows - 1), ci1 = std::min((y1 - ORBFE_EDGE) / L.ch, L.rows - 1);
                T.cj0 = (short)cj0; T.ci0 = (short)ci0; T.ncj = (short)(cj1 - cj0 + 1); T.nci = (short)(ci1 - ci0 + 1);
                T.level = (short)(v0 + l); T.tx = (short)tx; T.ty = (short)ty; T.pad = 0;
                // interior cell boundaries: y = 16 + ci*ch (ci >= 1) and x = 16 + cj*cw (cj >= 1)
                T.hmask = 0;
                for (int r = 0; r < ORBFE_FT_H + 2; r++) {
                    const int y = y0 - 1 + r;
                    const int d = y - ORBFE_EDGE;
                    if (d >= L.ch && d % L.ch == 0 && d / L.ch <= L.rows - 1) T.hmask |= 1ull << r;
                }
                for (int w = 0; w < 4; w++) T.vmask[w] = 0;
                for (int c = 0; c < 128; c++) {
                    const int d = x0 - 4 + c - ORBFE_EDGE;
                    if (d >= L.cw && d % L.cw == 0 && d / L.cw <= L.cols - 1) T.vmask[c >> 5] |= 1u << (c & 31);
                }
                if (T.ncj * T.nci > 64) return fail(ORBFE_ERR_UNSUPPORTED, "level %d: a FAST tile overlaps %d cells", l, T.ncj * T.nci);
            }
        for (int ty = 0; ty < L.btiles_y; ty++)
            for (int tx = 0; tx < L.btiles_x; tx++) {
                BTileInfo &T = binfo[(size_t)L.btile_base + ty * L.btiles_x + tx];
                T.level = (short)(v0 + l); T.tx = (short)tx; T.ty = (short)ty; T.pad = 0;
            }
        // the 3-D (x, y, frame) tensor map of the level for the FAST kernel's pixel tiles
        const CUresult r = encode_level_map(encode, &maps[v0 + l], L.pyr, L.w, L.h, B, L.pitch, L.plane);
        if (r != CUDA_SUCCESS) return fail(ORBFE_ERR_CUDA, "cuTensorMapEncodeTiled(level %d) failed: %d", l, (int)r);
    }
    return ORBFE_OK;
}

static int tensor_map_encoder(void **fn) {
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", fn, cudaEnableDefault, &qres) != cudaSuccess || !*fn ||
        qres != cudaDriverEntryPointSuccess)
        return fail(ORBFE_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
    return ORBFE_OK;
}

// The tile and candidate tables, the tensor maps and the per-frame work buffers for B frames at P's strides.  The counters
// (cell_cnt_lo | cell_cnt_hi | kept_cnt, zeroed per call) are one allocation: *counters, *counters_bytes.
template <class T>
static int upload(DeviceBuffers &mem, const std::vector<T> &v, const T **out) {
    T *d;
    ORBFE_CUDA_TRY(mem.alloc(&d, v.size()));
    ORBFE_CUDA_TRY(cudaMemcpy(d, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice));
    *out = d;
    return ORBFE_OK;
}

static int alloc_work(OrbfeExtractor *ex, DeviceBuffers &mem, const PlanHead &P, int B, const PlanLayout &A,
                      const std::vector<FTileInfo> &info, const std::vector<BTileInfo> &binfo, const std::vector<CUtensorMap> &maps,
                      WorkDev &Wk, void **counters, size_t *counters_bytes) {
    memset(&Wk, 0, sizeof(Wk));
    if (int rc = upload(mem, info, &Wk.ftile_info)) return rc;
    if (int rc = upload(mem, binfo, &Wk.btile_info)) return rc;
    if (int rc = upload(mem, A.cand_base, &Wk.cell_cand_base)) return rc;
    if (int rc = upload(mem, A.cand_cap, &Wk.cell_cand_cap)) return rc;
    if (int rc = upload(mem, maps, &Wk.tmaps)) return rc;
    cudaError_t e = (cudaError_t)fast_tma_setup();
    if (e != cudaSuccess) return fail(ORBFE_ERR_CUDA, "cudaFuncSetAttribute(fast_nms_tma_kernel): %s", cudaGetErrorString(e));
    ORBFE_CUDA_TRY(mem.alloc(&Wk.cand_keys, (size_t)P.cand_total * B));
    if (ex->score_type == 0) {
        ORBFE_CUDA_TRY(mem.alloc(&Wk.cand_keys64, (size_t)P.cand_total * B));
        ORBFE_CUDA_TRY(mem.alloc(&Wk.kept_aux, (size_t)P.kept_total * B));
    }
    const size_t nc = (size_t)P.ncells_total * B, nl = (size_t)P.nlevels * B;
    int *cnt;
    *counters_bytes = sizeof(int) * (2 * nc + nl);
    ORBFE_CUDA_TRY(mem.alloc(&cnt, 2 * nc + nl));
    *counters = cnt;
    Wk.cell_cnt_lo = cnt;
    Wk.cell_cnt_hi = cnt + nc;
    Wk.kept_cnt = cnt + 2 * nc;
    ORBFE_CUDA_TRY(mem.alloc(&Wk.cell_keep, nc));
    ORBFE_CUDA_TRY(mem.alloc(&Wk.cell_min_key, nc));
    ORBFE_CUDA_TRY(mem.alloc(&Wk.kept_keys, (size_t)P.kept_total * B));
    ORBFE_CUDA_TRY(mem.alloc(&Wk.kp_xy_score, (size_t)std::max(P.nfeatures, 1) * B));
    ORBFE_CUDA_TRY(mem.alloc(&Wk.level_cnt, nl));
    ORBFE_CUDA_TRY(mem.alloc(&Wk.err_flag, 1));
    ORBFE_CUDA_TRY(cudaMemsetAsync(Wk.err_flag, 0, sizeof(int), ex->hs.stream));
    return ORBFE_OK;
}

// The head of a plan for this handle: thresholds, score type, PDL switch
static void plan_head(const OrbfeExtractor *ex, PlanHead &P, int B) {
    P.nlevels = ex->nlevels;
    P.batch = B;
    // cv::FAST keeps a pixel only if its score is strictly above all 8 neighbours', and a non-corner scores 0: a corner of
    // score 0 (a pixel that is a corner at threshold 0 only) is never kept and suppresses nothing.  Threshold 0 therefore
    // detects exactly what threshold 1 detects; the kernel, whose NMS input is m - t_lo, runs it as 1.
    const int th = std::max(ex->fast_th, 1);
    P.t_lo = std::min(th, 7);
    P.t_hi = std::max(th, 7);
    P.t1_is_lo = th <= 7;
    P.score_type = ex->score_type;
    {   // programmatic dependent launch of the pipeline's kernels (extract_kernels.cu, pdl_prologue); ORBFE_PDL=0 turns it off
        const char *e = getenv("ORBFE_PDL");
        P.pdl = !(e && *e == '0');
    }
    {   // HarrisResponses scale (ORBextractor.cc:90-92)
        float scale = (float)(1 << 2) * (float)7 * 255.0f;
        scale = 1.0f / scale;
        P.harris_scale4 = scale * scale * scale * scale;
    }
}

// Builds `plan` for the groups of the (W, H) list `geom`, cap[g] frames of group g, unless it already holds them: it is
// rebuilt only when the list changes or a group outgrows its capacity, and a rebuild for the same list keeps every group's
// old capacity.  All geometries are laid out, on the host, before anything is freed: a refused call leaves the handle's
// plans as they were.  gidx: the call's index of each group, named in a refusal (NULL: the message names no group).
template <class PD>
static int build(OrbfeExtractor *ex, Plan<PD> &plan, const std::vector<int> &geom, std::vector<int> cap, const int *gidx) {
    const int n = (int)cap.size(), nl = ex->nlevels;
    if (geom == plan.geom) {
        bool fits = true;
        for (int i = 0; i < n; i++) fits = fits && cap[i] <= plan.cap[i];
        if (fits) return ORBFE_OK;
        for (int i = 0; i < n; i++) cap[i] = std::max(cap[i], plan.cap[i]);
    }
    std::unique_ptr<PD> hp(new PD());
    PD &P = *hp;
    int frames = 0;
    for (int c : cap) frames += c;
    plan_head(ex, P, frames);
    PlanLayout A;
    for (int i = 0; i < n; i++) {
        // a geometry's kept lists (quota + 2 * cells + 64) decide its level-select footprint, so that refusal names the group too
        int rc = layout_geometry(ex, geom[2 * i], geom[2 * i + 1], &P.lv[i * nl], A);
        if (!rc) {
            int kept = 0;
            size_t bytes = 0;
            for (int l = 0; l < nl; l++) kept = std::max(kept, P.lv[i * nl + l].kept_cap);
            rc = level_select_smem(ex, kept, &bytes);
        }
        if (rc && gidx) {
            const std::string why = g_err;
            return fail(rc, "group %d (%dx%d): %s", gidx[i], geom[2 * i], geom[2 * i + 1], why.c_str());
        }
        if (rc) return rc;
        if constexpr (std::is_same<PD, MultiPlanDev>::value) {   // the group table (a PlanDev is one group and has none)
            GroupDev &G = P.grp[P.ngroups++];
            G.ftile0 = P.lv[i * nl].ftile_base;
            G.nftiles = A.ft_base - G.ftile0;
            G.cell0 = P.lv[i * nl].cell_base;
            G.ncells = A.cell_base - G.cell0;
        }
    }
    size_t ls = 0;
    if (int rc = level_select_smem(ex, A.max_kept, &ls)) return rc;
    P.ncells_total = A.cell_base;
    P.nftiles_total = A.ft_base;
    P.nbtiles_total = A.bt_base;
    P.kept_total = A.kept_total;
    P.cand_total = A.cand_total;
    P.nfeatures = A.kp_total;

    ORBFE_CUDA_TRY(cudaSetDevice(ex->device));
    ORBFE_CUDA_TRY(cudaEventSynchronize(ex->hs.last));   // the handle's pending calls still use the plan
    plan.release();
    plan.hp = std::move(hp);
    if (int rc = set_level_select_attr(ex, ls)) return rc;
    plan.ls_smem = ls;
    void *fn = nullptr;
    if (int rc = tensor_map_encoder(&fn)) return rc;
    std::vector<FTileInfo> info((size_t)P.nftiles_total);
    std::vector<BTileInfo> binfo((size_t)P.nbtiles_total);
    std::vector<CUtensorMap> maps((size_t)n * nl);
    for (int i = 0; i < n; i++) {
        if (int rc = alloc_geometry(ex, plan.mem, &P.lv[i * nl], cap[i], i * nl, fn, info, binfo, maps)) return rc;
        plan.own0[i] = P.lv[i * nl];
    }
    if (int rc = alloc_work(ex, plan.mem, P, frames, A, info, binfo, maps, plan.work, &plan.counters, &plan.counters_bytes))
        return rc;
    ex->tma_encode = fn;
    ORBFE_CUDA_TRY(plan.mem.alloc(&plan.d_kps, (size_t)std::max(P.nfeatures, 1) * frames));
    ORBFE_CUDA_TRY(plan.mem.alloc(&plan.d_desc, (size_t)std::max(P.nfeatures, 1) * frames * 32));
    ORBFE_CUDA_TRY(plan.mem.alloc(&plan.d_counts, (size_t)frames));
    ORBFE_CUDA_TRY(plan.mem.alloc(&plan.dp, 1));
    ORBFE_CUDA_TRY(cudaMemcpyAsync(plan.dp, &P, sizeof(P), cudaMemcpyHostToDevice, ex->hs.stream));
    if (int rc = grow_host_counts(ex, frames)) return rc;
    ORBFE_CUDA_TRY(cudaStreamSynchronize(ex->hs.stream));
    plan.geom = geom;
    plan.cap = cap;
    ex->plan_builds++;
    return ORBFE_OK;
}

// Point level 0 of group g of `plan` at `ptr` (the plan's own planes, or the caller's device frames read in place).
// Stream-ordered: the device copy of the level descriptor and the level-0 tensor map are rewritten on `s` before the
// kernels that read them.
template <class PD>
static int bind_level0(OrbfeExtractor *ex, Plan<PD> &plan, int g, uint8_t *ptr, int pitch, size_t plane, cudaStream_t s) {
    const int v = g * ex->nlevels;
    LevelDev &L0 = plan.hp->lv[v];
    if (L0.pyr == ptr && L0.pitch == pitch && L0.plane == plane) return ORBFE_OK;
    L0.pyr = ptr; L0.pitch = pitch; L0.plane = plane;
    ORBFE_CUDA_TRY(cudaMemcpyAsync(&plan.dp->lv[v], &L0, sizeof(LevelDev), cudaMemcpyHostToDevice, s));
    CUtensorMap m;
    const CUresult r = encode_level_map(ex->tma_encode, &m, ptr, L0.w, L0.h, plan.cap[g], pitch, plane);
    if (r != CUDA_SUCCESS) return fail(ORBFE_ERR_CUDA, "cuTensorMapEncodeTiled(group %d level 0) failed: %d", g, (int)r);
    ORBFE_CUDA_TRY(cudaMemcpyAsync(const_cast<CUtensorMap *>(plan.work.tmaps) + v, &m, sizeof(m), cudaMemcpyHostToDevice, s));
    return ORBFE_OK;
}

// Device frames can be level 0 as they are (no copy) when the level-0 tensor map takes them: 16-byte aligned base and
// strides, a row stride that fits an int, frames that do not overlap.  ORBFE_INGEST_COPY=1 copies them always.
static bool readable_in_place(const uint8_t *imgs, int height, size_t stride, size_t frame_stride) {
    return !getenv("ORBFE_INGEST_COPY") && (uintptr_t)imgs % 16 == 0 && stride % 16 == 0 && frame_stride % 16 == 0 &&
           stride <= (size_t)INT_MAX && frame_stride >= stride * (size_t)height;
}

// Frames [f0, f1) of the caller's frames into the same frames of level 0 L0: one linear copy when both sides are fully
// contiguous, one 2-D copy when the frames of each side follow each other row after row, else one 2-D copy per frame.
static int copy_frames(const LevelDev &L0, const uint8_t *src, int width, int height, size_t stride, size_t frame_stride, int f0,
                       int f1, cudaMemcpyKind kind, cudaStream_t s) {
    uint8_t *dst = L0.pyr + (size_t)f0 * L0.plane;
    src += (size_t)f0 * frame_stride;
    const bool rows = frame_stride == stride * (size_t)height && L0.plane == (size_t)L0.pitch * height;
    if (rows && stride == (size_t)width && L0.pitch == width) {
        ORBFE_CUDA_TRY(cudaMemcpyAsync(dst, src, (size_t)width * height * (f1 - f0), kind, s));
    } else if (rows) {
        ORBFE_CUDA_TRY(cudaMemcpy2DAsync(dst, L0.pitch, src, stride, width, (size_t)height * (f1 - f0), kind, s));
    } else {
        for (int f = 0; f < f1 - f0; f++)
            ORBFE_CUDA_TRY(cudaMemcpy2DAsync(dst + f * L0.plane, L0.pitch, src + f * frame_stride, stride, width, height, kind, s));
    }
    return ORBFE_OK;
}

// Level 0 of group g for `nframes` frames on s: the caller's device frames read in place when they can be, else copied
// (host frames: uploaded) into the plan's own planes
template <class PD>
static int ingest(OrbfeExtractor *ex, Plan<PD> &plan, int g, const uint8_t *imgs, int width, int height, size_t stride,
                  size_t frame_stride, int nframes, cudaMemcpyKind kind, cudaStream_t s) {
    if (kind == cudaMemcpyDeviceToDevice && readable_in_place(imgs, height, stride, frame_stride))
        return bind_level0(ex, plan, g, const_cast<uint8_t *>(imgs), (int)stride, frame_stride, s);
    const LevelDev &own = plan.own0[g];
    if (int rc = bind_level0(ex, plan, g, own.pyr, own.pitch, own.plane, s)) return rc;
    return copy_frames(own, imgs, width, height, stride, frame_stride, 0, nframes, kind, s);
}

extern "C" int orbfe_extractor_create(int nfeatures, float scale_factor, int nlevels, int score_type, int fast_th,
                                      int device, OrbfeExtractor **out) {
    if (!out) return fail(ORBFE_ERR_ARG, "out is NULL");
    *out = nullptr;
    if (nfeatures < 0 || nlevels < 1 || nlevels > ORBFE_MAX_LEVELS || !(scale_factor > 1.0f) || fast_th < 0 || fast_th > 254)
        return fail(ORBFE_ERR_ARG, "bad extractor parameters (nfeatures=%d scale=%g nlevels=%d fastTh=%d)", nfeatures,
                    (double)scale_factor, nlevels, fast_th);
    if (score_type != 0 && score_type != 1) return fail(ORBFE_ERR_ARG, "score_type must be 0 (HARRIS) or 1 (FAST)");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(ORBFE_ERR_NO_DEVICE, "no CUDA device available: liborbfe has no CPU path");
    }
    if (device < 0 || device >= ndev) return fail(ORBFE_ERR_ARG, "device %d out of range (%d devices)", device, ndev);
    OrbfeExtractor *ex = new OrbfeExtractor();
    ex->nfeatures = nfeatures;
    ex->nlevels = nlevels;
    ex->score_type = score_type;
    ex->fast_th = fast_th;
    ex->device = device;
    ex->scale_factor = (double)scale_factor;
    const double sf = ex->scale_factor;
    // mvScaleFactor / mvInvScaleFactor, :461-471
    ex->scale[0] = 1.0f;
    for (int i = 1; i < nlevels; i++) ex->scale[i] = (float)((double)ex->scale[i - 1] * sf);
    const float inv = (float)(1.0f / sf);
    ex->inv_scale[0] = 1.0f;
    for (int i = 1; i < nlevels; i++) ex->inv_scale[i] = ex->inv_scale[i - 1] * inv;
    // mnFeaturesPerLevel, :476-487
    const float factor = (float)(1.0 / sf);
    float nd = (float)nfeatures * (1.0f - factor) / (1.0f - (float)std::pow((double)factor, (double)nlevels));
    int sum = 0;
    for (int l = 0; l < nlevels - 1; l++) {
        ex->quota[l] = cv_round((double)nd);
        sum += ex->quota[l];
        nd *= factor;
    }
    ex->quota[nlevels - 1] = std::max(nfeatures - sum, 0);

    cudaError_t e = ex->hs.create(device);
    if (e == cudaSuccess) e = cudaMalloc((void **)&ex->d_pattern, 1024);
    if (e == cudaSuccess) e = cudaMemcpy(ex->d_pattern, kBriefPattern, 1024, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaHostAlloc((void **)&ex->h_err, sizeof(int), cudaHostAllocDefault);
    if (e != cudaSuccess) {
        orbfe_extractor_destroy(ex);
        return fail(ORBFE_ERR_CUDA, "extractor setup failed: %s", cudaGetErrorString(e));
    }
    *out = ex;
    return ORBFE_OK;
}

extern "C" int orbfe_extractor_destroy(OrbfeExtractor *ex) {
    if (!ex) return ORBFE_OK;
    cudaSetDevice(ex->device);
    if (ex->hs.last) cudaEventSynchronize(ex->hs.last);
    if (ex->hs.stream) cudaStreamSynchronize(ex->hs.stream);
    ex->single.release();
    ex->multi.release();
    if (ex->d_pattern) cudaFree(ex->d_pattern);
    if (ex->h_counts) cudaFreeHost(ex->h_counts);
    if (ex->h_err) cudaFreeHost(ex->h_err);
    for (cudaEvent_t ev : ex->timer.ev) cudaEventDestroy(ev);
    for (cudaEvent_t ev : ex->chunk_ev) cudaEventDestroy(ev);
    if (ex->copy_stream) cudaStreamDestroy(ex->copy_stream);
    ex->hs.destroy();
    delete ex;
    return ORBFE_OK;
}

extern "C" int orbfe_extractor_levels(const OrbfeExtractor *ex) { return ex ? ex->nlevels : 0; }
extern "C" float orbfe_extractor_scale_factor(const OrbfeExtractor *ex) { return ex ? (float)ex->scale_factor : 0.f; }
extern "C" int orbfe_extractor_tables(const OrbfeExtractor *ex, float *scale, float *inv_scale, int *quota) {
    if (!ex) return fail(ORBFE_ERR_ARG, "ex is NULL");
    for (int l = 0; l < ex->nlevels; l++) {
        if (scale) scale[l] = ex->scale[l];
        if (inv_scale) inv_scale[l] = ex->inv_scale[l];
        if (quota) quota[l] = ex->quota[l];
    }
    return ORBFE_OK;
}

// Stage timing: a flat list of events; entry i of `names` labels the interval ev[i] -> ev[i+1]; the marker
// name "" opens a new call (its interval, the gap since the previous call, is dropped when reading).
// The list accumulates over calls until orbfe_extractor_stage_times() is read, so several calls can be in
// flight on the stream (chunked pipelines) without a host synchronisation in between.
static void stage_mark(OrbfeExtractor *ex, cudaStream_t s, const char *name) {
    if (!ex->profiling) return;
    StageTimer &T = ex->timer;
    const size_t i = T.names.size();  // ev[0] is the origin; names[i] labels ev[i] -> ev[i+1]
    while (T.ev.size() < i + 2) { cudaEvent_t e; cudaEventCreate(&e); T.ev.push_back(e); }
    if (i == 0 && T.origin_pending) { cudaEventRecord(T.ev[0], s); T.origin_pending = false; }
    T.names.push_back(name ? name : "");
    cudaEventRecord(T.ev[i + 1], s);
}

// The per-call counters of a plan, zeroed on s before the call's first launch
template <class PD>
static int zero_counters(const Plan<PD> &plan, cudaStream_t s) {
    ORBFE_CUDA_TRY(cudaMemsetAsync(plan.counters, 0, plan.counters_bytes, s));
    return ORBFE_OK;
}

static void enqueue_pyramid(OrbfeExtractor *ex, int f0, int nf, cudaStream_t s) {
    const PlanDev &hp = *ex->single.hp;
    for (int l = 1; l < hp.nlevels; l++) launch_resize_level(ex->single.dp, hp, l, f0, nf, s);
    ex->last_launches += hp.nlevels - 1;
    stage_mark(ex, s, "pyramid");
}

// Enqueue the device pipeline for frames [f0, f0+nf) whose level-0 images are already in lv[0].pyr.
// The per-call counters must have been zeroed (zero_counters) before the first chunk.
static int enqueue_pipeline(OrbfeExtractor *ex, int f0, int nf, OrbfeKeyPoint *d_kps, uint8_t *d_desc, int *d_counts,
                            cudaStream_t s, bool with_pyramid = true, const PeerOut *peers = nullptr) {
    const Plan<PlanDev> &P = ex->single;
    const PlanDev &hp = *P.hp;
    int launches = 0;
    if (with_pyramid) enqueue_pyramid(ex, f0, nf, s);
    launch_fast_nms(P.dp, hp, P.work, f0, nf, s); launches++;
    stage_mark(ex, s, "fast_nms");
    launch_cell_quota(P.dp, hp, P.work, f0, nf, s); launches++;
    stage_mark(ex, s, "cell_quota");
    launch_cell_select(P.dp, hp, P.work, f0, nf, s); launches++;
    stage_mark(ex, s, "cell_select");
    launch_level_select(P.dp, hp, P.work, P.ls_smem, f0, nf, s); launches++;
    stage_mark(ex, s, "level_select");
    launch_describe_fused(P.dp, hp, P.work, ex->d_pattern, d_kps, d_desc, d_counts, f0, nf, s, peers); launches++;
    stage_mark(ex, s, "describe");
    ORBFE_CUDA_TRY(cudaGetLastError());
    ex->last_launches += launches;
    return ORBFE_OK;
}

static void profiling_begin(OrbfeExtractor *ex, cudaStream_t s) {
    if (!ex->profiling) return;
    if (ex->timer.names.size() > 16384) { ex->timer.names.clear(); ex->timer.origin_pending = true; }  // never read: recycle
    stage_mark(ex, s, nullptr);  // call marker (its interval is ignored)
}

// reads and clears the accumulated list; the caller must have synchronised the stream(s) used
static void profiling_collect(OrbfeExtractor *ex) {
    ex->stage_names.clear();
    ex->stage_ms.clear();
    StageTimer &T = ex->timer;
    for (size_t i = 0; i < T.names.size(); i++) {
        if (T.names[i].empty()) continue;
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, T.ev[i], T.ev[i + 1]) != cudaSuccess) { cudaGetLastError(); continue; }
        ex->stage_names.push_back(T.names[i]);
        ex->stage_ms.push_back(ms);
    }
    T.names.clear();
    T.origin_pending = true;
}

// Frames [frame0, frame0 + n) of a plan's outputs: the caller's frames from `out` on
struct FrameRun { int frame0, n, out; };

// The end of both host-array entries, enqueued on s after their launches: the counts, the overflow flag and each run's
// keypoints and descriptors (one 2-D copy each, `cap` slots per caller frame) back to the host; then the wait for them and
// the caller's counts.
template <class PD>
static int read_back(OrbfeExtractor *ex, const Plan<PD> &plan, const std::vector<FrameRun> &runs, OrbfeKeyPoint *kps, uint8_t *desc,
                     int cap, int *n_out, cudaStream_t s) {
    const int nf = plan.hp->nfeatures, ncopy = std::min(cap, nf);
    int frames = 0;
    for (const FrameRun &r : runs) frames += r.n;
    ORBFE_CUDA_TRY(cudaMemcpyAsync(ex->h_counts, plan.d_counts, sizeof(int) * frames, cudaMemcpyDeviceToHost, s));
    ORBFE_CUDA_TRY(cudaMemcpyAsync(ex->h_err, plan.work.err_flag, sizeof(int), cudaMemcpyDeviceToHost, s));
    for (size_t i = 0; ncopy > 0 && i < runs.size(); i++) {
        const FrameRun &r = runs[i];
        ORBFE_CUDA_TRY(cudaMemcpy2DAsync(kps + (size_t)r.out * cap, sizeof(OrbfeKeyPoint) * cap, plan.d_kps + (size_t)r.frame0 * nf,
                                         sizeof(OrbfeKeyPoint) * nf, sizeof(OrbfeKeyPoint) * ncopy, r.n, cudaMemcpyDeviceToHost, s));
        ORBFE_CUDA_TRY(cudaMemcpy2DAsync(desc + (size_t)r.out * cap * 32, (size_t)32 * cap, plan.d_desc + (size_t)r.frame0 * nf * 32,
                                         (size_t)32 * nf, (size_t)32 * ncopy, r.n, cudaMemcpyDeviceToHost, s));
    }
    stage_mark(ex, s, "d2h");
    if (int rc = ex->hs.leave(s, true)) return rc;
    if (*ex->h_err) {
        const int code = *ex->h_err;
        cudaMemsetAsync(plan.work.err_flag, 0, sizeof(int), s);
        ex->hs.leave(s, false);
        return fail(ORBFE_ERR_INTERNAL, "device overflow flag %d", code);
    }
    int status = ORBFE_OK;
    for (const FrameRun &r : runs)
        for (int f = 0; f < r.n; f++) {
            n_out[r.out + f] = ex->h_counts[r.frame0 + f];
            if (n_out[r.out + f] > cap) status = ORBFE_ERR_CAPACITY;
        }
    if (status) return fail(status, "caller capacity %d too small", cap);
    return ORBFE_OK;
}

// Head of both device-resident extract entries: the plan for this geometry, then on *s (the caller's stream, or the handle's),
// behind the handle's earlier calls, level 0 taken from the caller's device frames and the per-call counters zeroed.  The
// entry leaves the handle's stream after its last launch.
static int begin_device_extract(OrbfeExtractor *ex, const uint8_t *d_imgs, int width, int height, size_t stride, size_t frame_stride,
                                int batch, void *stream, cudaStream_t *s) {
    if (width <= 0 || height <= 0 || batch <= 0 || stride < (size_t)width) return fail(ORBFE_ERR_ARG, "bad geometry");
    ORBFE_CUDA_TRY(cudaSetDevice(ex->device));
    int rc = build(ex, ex->single, {width, height}, {batch}, nullptr);
    if (rc) return rc;
    *s = ex->hs.pick(stream);
    if ((rc = ex->hs.enter(*s))) return rc;
    profiling_begin(ex, *s);
    rc = ingest(ex, ex->single, 0, d_imgs, width, height, stride, frame_stride, batch, cudaMemcpyDeviceToDevice, *s);
    if (rc) return rc;
    stage_mark(ex, *s, "ingest");
    ex->last_launches = 0;
    return zero_counters(ex->single, *s);
}

extern "C" int orbfe_extract_batch_device(OrbfeExtractor *ex, const uint8_t *d_imgs, int width, int height,
                                          size_t stride, size_t frame_stride, int batch, OrbfeKeyPoint *d_kps,
                                          uint8_t *d_desc, int *d_counts, void *stream) {
    if (!ex || !d_imgs || !d_kps || !d_desc || !d_counts) return fail(ORBFE_ERR_ARG, "NULL argument");
    cudaStream_t s;
    if (int rc = begin_device_extract(ex, d_imgs, width, height, stride, frame_stride, batch, stream, &s)) return rc;
    if (int rc = enqueue_pipeline(ex, 0, batch, d_kps, d_desc, d_counts, s)) return rc;
    return ex->hs.leave(s, false);
}

// The device-resident extract with the descriptor kernel's outputs redirected into the gather buffers of a rig exchange
// (include/orbfe_comm.h; called by orbfe_extract_batch_device_exchange in comm.cu)
int orbfe_extract_batch_device_peers(OrbfeExtractor *ex, const uint8_t *d_imgs, int width, int height, size_t stride, size_t frame_stride,
                                     int batch, const PeerOut &po, int cap, void *stream) {
    if (!ex || !d_imgs) return fail(ORBFE_ERR_ARG, "NULL argument");
    cudaStream_t s;
    if (int rc = begin_device_extract(ex, d_imgs, width, height, stride, frame_stride, batch, stream, &s)) return rc;
    if (cap != ex->single.hp->nfeatures) {
        ex->hs.leave(s, false);   // the ingest is enqueued
        return fail(ORBFE_ERR_ARG, "exchange capacity %d != keypoint slots per frame %d", cap, ex->single.hp->nfeatures);
    }
    if (int rc = enqueue_pipeline(ex, 0, batch, nullptr, nullptr, nullptr, s, true, &po)) return rc;
    return ex->hs.leave(s, false);
}

extern "C" int orbfe_extract_batch(OrbfeExtractor *ex, const uint8_t *imgs, int width, int height, size_t stride,
                                   size_t frame_stride, int batch, OrbfeKeyPoint *kps, uint8_t *desc, int cap,
                                   int *n_out) {
    if (!ex || !n_out) return fail(ORBFE_ERR_ARG, "NULL argument");
    for (int f = 0; f < std::max(batch, 0); f++) n_out[f] = 0;
    if (!imgs || width <= 0 || height <= 0) return ORBFE_OK;  // empty image: silent return (ORBextractor.cc:721-722)
    if (batch <= 0 || stride < (size_t)width || cap < 0 || (cap > 0 && (!kps || !desc))) return fail(ORBFE_ERR_ARG, "bad arguments");
    ORBFE_CUDA_TRY(cudaSetDevice(ex->device));
    Plan<PlanDev> &P = ex->single;
    int rc = build(ex, P, {width, height}, {batch}, nullptr);
    if (rc) return rc;
    cudaStream_t s = ex->hs.stream;
    if ((rc = ex->hs.enter(s))) return rc;
    const LevelDev &own = P.own0[0];
    rc = bind_level0(ex, P, 0, own.pyr, own.pitch, own.plane, s);   // the uploads land in the plan's own planes
    if (rc) return rc;
    profiling_begin(ex, s);
    ex->last_launches = 0;
    rc = zero_counters(P, s);
    if (rc) return rc;
    // H2D of chunk k+1 (copy stream) overlaps the kernels of chunk k (compute stream)
    int nchunks = batch >= 8 ? 4 : 1;   // H100, 400 W (64 x 1080p, bench.py's three handles): 1, 2 and 4 chunks within 2 % (37.4-38.1 Mkp/s end to end)
    if (const char *e = getenv("ORBFE_CHUNKS")) nchunks = std::max(1, std::min(batch, atoi(e)));  // tuning knob
    if (!ex->copy_stream) ORBFE_CUDA_TRY(cudaStreamCreateWithFlags(&ex->copy_stream, cudaStreamNonBlocking));
    while ((int)ex->chunk_ev.size() < nchunks + 1) {
        cudaEvent_t e;
        ORBFE_CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        ex->chunk_ev.push_back(e);
    }
    // the copy stream must not overwrite level 0 before earlier work of this handle has drained: s has entered (it waits for
    // the handle's last call, whichever stream that ran on), so an event recorded on it now covers that call too
    ORBFE_CUDA_TRY(cudaEventRecord(ex->chunk_ev[nchunks], s));
    ORBFE_CUDA_TRY(cudaStreamWaitEvent(ex->copy_stream, ex->chunk_ev[nchunks], 0));
    for (int k = 0; k < nchunks; k++) {
        const int f0 = (int)((long long)batch * k / nchunks), f1 = (int)((long long)batch * (k + 1) / nchunks);
        if (f1 <= f0) continue;
        if ((rc = copy_frames(own, imgs, width, height, stride, frame_stride, f0, f1, cudaMemcpyHostToDevice, ex->copy_stream))) return rc;
        ORBFE_CUDA_TRY(cudaEventRecord(ex->chunk_ev[k], ex->copy_stream));
        ORBFE_CUDA_TRY(cudaStreamWaitEvent(s, ex->chunk_ev[k], 0));
        if (ex->batch_mode == 1) {
            enqueue_pyramid(ex, f0, f1 - f0, s);   // phased: only the pyramids follow the upload chunk by chunk
        } else {
            rc = enqueue_pipeline(ex, f0, f1 - f0, P.d_kps, P.d_desc, P.d_counts, s);
            if (rc) return rc;
        }
    }
    if (ex->batch_mode == 1) {   // ... detection and description run once over the whole batch (full-size launches)
        rc = enqueue_pipeline(ex, 0, batch, P.d_kps, P.d_desc, P.d_counts, s, false);
        if (rc) return rc;
    }
    return read_back(ex, P, {{0, batch, 0}}, kps, desc, cap, n_out, s);
}

extern "C" int orbfe_extract(OrbfeExtractor *ex, const uint8_t *img, int width, int height, size_t stride,
                             OrbfeKeyPoint *kps, uint8_t *desc, int cap, int *n_out) {
    return orbfe_extract_batch(ex, img, width, height, stride, stride * (size_t)std::max(height, 0), 1, kps, desc, cap, n_out);
}

// ------------------------------------------------------------------------------------------------
// Mixed geometries (orbfe_extract_multi*): the groups of a call run as one chain on the multi plan
// ------------------------------------------------------------------------------------------------
static bool group_empty(const OrbfeImageGroup &G) { return !G.imgs || G.width <= 0 || G.height <= 0; }

// The argument checks of both entries, made before the handle is used; *frames = the call's frames
static int check_groups(const OrbfeExtractor *ex, int ngroups, const OrbfeImageGroup *groups, int *frames) {
    if (!ex) return fail(ORBFE_ERR_ARG, "ex is NULL");
    if (ngroups < 1 || ngroups > ORBFE_MULTI_MAX_GROUPS)
        return fail(ORBFE_ERR_ARG, "ngroups %d outside 1..%d", ngroups, ORBFE_MULTI_MAX_GROUPS);
    if (!groups) return fail(ORBFE_ERR_ARG, "groups is NULL");
    long long n = 0;
    for (int g = 0; g < ngroups; g++) {
        const OrbfeImageGroup &G = groups[g];
        if (G.batch < 1) return fail(ORBFE_ERR_ARG, "group %d: batch %d", g, G.batch);
        if (!group_empty(G) && G.stride < (size_t)G.width) return fail(ORBFE_ERR_ARG, "group %d: stride %zu < width %d", g, G.stride, G.width);
        n += G.batch;
    }
    if (n > 65535) return fail(ORBFE_ERR_ARG, "%lld frames in one call (at most 65535: one grid row per frame)", n);
    *frames = (int)n;
    return ORBFE_OK;
}

// The multi plan for the non-empty groups of a call, keyed by their (W, H) list (a call without one plans nothing)
static int build_multi(OrbfeExtractor *ex, int ngroups, const OrbfeImageGroup *groups) {
    std::vector<int> geom, cap, gidx;
    for (int g = 0; g < ngroups; g++) {
        if (group_empty(groups[g])) continue;
        geom.push_back(groups[g].width);
        geom.push_back(groups[g].height);
        cap.push_back(groups[g].batch);
        gidx.push_back(g);
    }
    return cap.empty() ? ORBFE_OK : build(ex, ex->multi, geom, cap, gidx.data());
}

// On s, after the handle's earlier calls: this call's frame and work ranges of the planned groups, their level 0 (ingest)
// and the zeroed counters.  Device outputs (d_counts != NULL): a group's frames are written at their place in the call, and
// the counts of empty groups are zeroed here; host outputs: the planned frames are written packed.  runs[i]: planned group
// i's frames in the plan's outputs and the call's frame of its first frame.
static int begin_multi(OrbfeExtractor *ex, int ngroups, const OrbfeImageGroup *groups, bool host, int *d_counts, cudaStream_t s,
                       std::vector<FrameRun> &runs) {
    Plan<MultiPlanDev> &P = ex->multi;
    int i = 0, frame = 0, out = 0, fw = 0, cw = 0;
    runs.clear();
    for (int g = 0; g < ngroups; g++) {
        const OrbfeImageGroup &Gi = groups[g];
        if (group_empty(Gi)) {
            if (d_counts) ORBFE_CUDA_TRY(cudaMemsetAsync(d_counts + out, 0, sizeof(int) * Gi.batch, s));
            out += Gi.batch;
            continue;
        }
        GroupDev &G = P.hp->grp[i];
        G.frame0 = frame;
        G.nframes = Gi.batch;
        G.out0 = host ? frame : out;
        G.fwork0 = fw;
        G.cwork0 = cw;
        fw += G.nftiles * Gi.batch;
        cw += G.ncells * Gi.batch;
        runs.push_back({frame, Gi.batch, out});
        if (int rc = ingest(ex, P, i, Gi.imgs, Gi.width, Gi.height, Gi.stride, Gi.frame_stride, Gi.batch,
                            host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, s))
            return rc;
        frame += Gi.batch;
        out += Gi.batch;
        i++;
    }
    if (frame == 0) return ORBFE_OK;
    MultiPlanDev &M = *P.hp;
    M.nframes = frame;
    M.nfwork = fw;
    M.ncwork = cw;
    ORBFE_CUDA_TRY(cudaMemcpyAsync(P.dp->grp, M.grp, sizeof(M.grp), cudaMemcpyHostToDevice, s));
    stage_mark(ex, s, "ingest");
    return zero_counters(P, s);
}

// One launch per stage for all groups: nlevels - 1 resizes, then FAST, quota, cell select, level select, describe
static int enqueue_multi(OrbfeExtractor *ex, OrbfeKeyPoint *d_kps, uint8_t *d_desc, int *d_counts, cudaStream_t s) {
    const Plan<MultiPlanDev> &P = ex->multi;
    const MultiPlanDev &M = *P.hp;
    for (int l = 1; l < M.nlevels; l++) launch_resize_level_multi(P.dp, M, l, s);
    stage_mark(ex, s, "pyramid");
    launch_fast_nms_multi(P.dp, M, P.work, s);
    stage_mark(ex, s, "fast_nms");
    launch_cell_quota_multi(P.dp, M, P.work, s);
    stage_mark(ex, s, "cell_quota");
    launch_cell_select_multi(P.dp, M, P.work, s);
    stage_mark(ex, s, "cell_select");
    launch_level_select_multi(P.dp, M, P.work, P.ls_smem, s);
    stage_mark(ex, s, "level_select");
    launch_describe_multi(P.dp, M, P.work, ex->d_pattern, d_kps, d_desc, d_counts, s);
    stage_mark(ex, s, "describe");
    ORBFE_CUDA_TRY(cudaGetLastError());
    ex->last_launches += M.nlevels + 4;
    return ORBFE_OK;
}

extern "C" int orbfe_extract_multi_device(OrbfeExtractor *ex, int ngroups, const OrbfeImageGroup *groups, OrbfeKeyPoint *d_kps,
                                          uint8_t *d_desc, int *d_counts, void *stream) {
    int frames = 0;
    if (int rc = check_groups(ex, ngroups, groups, &frames)) return rc;
    if (!d_kps || !d_desc || !d_counts) return fail(ORBFE_ERR_ARG, "NULL output");
    ORBFE_CUDA_TRY(cudaSetDevice(ex->device));
    if (int rc = build_multi(ex, ngroups, groups)) return rc;
    const cudaStream_t s = ex->hs.pick(stream);
    if (int rc = ex->hs.enter(s)) return rc;
    profiling_begin(ex, s);
    ex->last_launches = 0;
    std::vector<FrameRun> runs;
    if (int rc = begin_multi(ex, ngroups, groups, false, d_counts, s, runs)) return rc;
    if (!runs.empty())
        if (int rc = enqueue_multi(ex, d_kps, d_desc, d_counts, s)) return rc;
    return ex->hs.leave(s, false);
}

extern "C" int orbfe_extract_multi(OrbfeExtractor *ex, int ngroups, const OrbfeImageGroup *groups, OrbfeKeyPoint *kps,
                                   uint8_t *desc, int cap, int *n_out) {
    int frames = 0;
    if (int rc = check_groups(ex, ngroups, groups, &frames)) return rc;
    if (!n_out || cap < 0 || (cap > 0 && (!kps || !desc))) return fail(ORBFE_ERR_ARG, "bad output arguments");
    for (int f = 0; f < frames; f++) n_out[f] = 0;
    ORBFE_CUDA_TRY(cudaSetDevice(ex->device));
    if (int rc = build_multi(ex, ngroups, groups)) return rc;
    const cudaStream_t s = ex->hs.stream;
    if (int rc = ex->hs.enter(s)) return rc;
    profiling_begin(ex, s);
    ex->last_launches = 0;
    std::vector<FrameRun> runs;
    if (int rc = begin_multi(ex, ngroups, groups, true, nullptr, s, runs)) return rc;
    if (runs.empty()) return ex->hs.leave(s, false);
    const Plan<MultiPlanDev> &P = ex->multi;
    if (int rc = enqueue_multi(ex, P.d_kps, P.d_desc, P.d_counts, s)) return rc;
    return read_back(ex, P, runs, kps, desc, cap, n_out, s);
}

extern "C" int orbfe_extractor_sync(OrbfeExtractor *ex) {
    if (!ex) return fail(ORBFE_ERR_ARG, "ex is NULL");
    if (int rc = ex->hs.enter(ex->hs.stream)) return rc;   // the handle's last call may have run on a caller's stream
    ORBFE_CUDA_TRY(cudaStreamSynchronize(ex->hs.stream));
    return ORBFE_OK;
}

extern "C" int orbfe_extractor_last_launches(const OrbfeExtractor *ex) { return ex ? ex->last_launches : 0; }
extern "C" int orbfe_extractor_plan_builds(const OrbfeExtractor *ex) { return ex ? ex->plan_builds : 0; }

extern "C" int orbfe_extractor_set_batch_mode(OrbfeExtractor *ex, int mode) {
    if (!ex || mode < 0 || mode > 1) return fail(ORBFE_ERR_ARG, "bad arguments");
    ex->batch_mode = mode;
    return ORBFE_OK;
}

extern "C" int orbfe_extractor_set_profiling(OrbfeExtractor *ex, int on) {
    if (!ex) return fail(ORBFE_ERR_ARG, "ex is NULL");
    ex->profiling = on != 0;
    return ORBFE_OK;
}

extern "C" int orbfe_extractor_stage_times(const OrbfeExtractor *ex_c, char (*names)[32], float *ms, int cap) {
    if (!ex_c) return 0;
    OrbfeExtractor *ex = const_cast<OrbfeExtractor *>(ex_c);
    if (!ex->profiling) return 0;
    if (ex->hs.enter(ex->hs.stream) || cudaStreamSynchronize(ex->hs.stream) != cudaSuccess) return 0;   // every timed call has ended
    profiling_collect(ex);
    int n = (int)std::min<size_t>(ex->stage_ms.size(), (size_t)std::max(cap, 0));
    for (int i = 0; i < n; i++) {
        if (names) { strncpy(names[i], ex->stage_names[i].c_str(), 31); names[i][31] = 0; }
        if (ms) ms[i] = ex->stage_ms[i];
    }
    return n;
}

extern "C" int orbfe_debug_level_size(const OrbfeExtractor *ex, int level, int *w, int *h) {
    if (!ex || level < 0 || level >= ex->nlevels || ex->single.geom.empty()) return fail(ORBFE_ERR_ARG, "no plan / bad level");
    if (w) *w = ex->single.hp->lv[level].w;
    if (h) *h = ex->single.hp->lv[level].h;
    return ORBFE_OK;
}

extern "C" int orbfe_debug_read_level(OrbfeExtractor *ex, int frame, int level, int which, uint8_t *out, size_t out_stride) {
    if (!ex || !out || level < 0 || level >= ex->nlevels || frame < 0 || ex->single.geom.empty() || frame >= ex->single.cap[0])
        return fail(ORBFE_ERR_ARG, "bad arguments");
    const Plan<PlanDev> &P = ex->single;
    // the levels of the handle's last call, whichever stream it ran on
    cudaStream_t s = ex->hs.stream;
    if (int rc = ex->hs.enter(s)) return rc;
    const LevelDev &L = P.hp->lv[level];
    const uint8_t *src = which ? L.blur : L.pyr + (size_t)frame * L.plane;
    // the pipeline smooths only descriptor patches; materialise the smoothed level of this frame on demand
    if (which) launch_blur(P.dp, *P.hp, P.work, frame, 1, s);
    if (int rc = ex->hs.leave(s, true)) return rc;
    ORBFE_CUDA_TRY(cudaMemcpy2D(out, out_stride, src, L.pitch, L.w, L.h, cudaMemcpyDeviceToHost));
    return ORBFE_OK;
}

// ------------------------------------------------------------------------------------------------
// Matcher
// ------------------------------------------------------------------------------------------------
struct OrbfeMatcher {
    int device = 0;
    int nsm = 132;
    HandleStream hs;       // every entry enters and leaves it, whichever stream it is enqueued on
    unsigned long long h2d_bytes = 0, d2h_bytes = 0, launches = 0;  // cumulative, for bench.py
    uint32_t *scratch = nullptr;  // candidate entries of the device-resident matcher
    size_t scratch_entries = 0;
    int *d_err = nullptr;  // [0]: error flags of the last launches; [1]: candidate entries an overflowing fused-matcher job needed
    int *h_err = nullptr;  // pinned
    Stage stage;           // every host-array entry of the handle; with `scratch`, the only device memory it grows
};

// Dynamic shared memory of the fused matcher (one thread block per pair / job).  What is left after the fixed arrays
// holds the candidate entries; lists that do not fit go to the global scratch, which costs the accept loop an L2 round
// trip per list.  Up to one block per SM nothing else of this launch could use the space, so the block takes most of the
// carve-out; larger launches keep 100 KB so that two blocks share an SM.  ORBFE_SBP_SMEM_KB overrides (measurement knob).
static size_t sbp_smem_total(const OrbfeMatcher *m, size_t fixed, int nblocks) {
    size_t total = nblocks <= m->nsm ? 200 * 1024 : 100 * 1024;
    if (const char *e = getenv("ORBFE_SBP_SMEM_KB")) total = (size_t)std::max(0, atoi(e)) * 1024;
    total = std::max(total, fixed + 16 * 1024);
    return total;
}

extern "C" int orbfe_matcher_create(int device, OrbfeMatcher **out) {
    if (!out) return fail(ORBFE_ERR_ARG, "out is NULL");
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(ORBFE_ERR_NO_DEVICE, "no CUDA device available: liborbfe has no CPU path");
    }
    if (device < 0 || device >= ndev) return fail(ORBFE_ERR_ARG, "device %d out of range", device);
    OrbfeMatcher *m = new OrbfeMatcher();
    m->device = device;
    cudaError_t e = cudaSetDevice(device);
    if (e == cudaSuccess) {
        // matching is a short, latency-critical job that usually shares the GPU with an extractor's long kernels: its
        // thread blocks go first whenever an SM frees up
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        e = m->hs.create(device, hi);
    }
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&m->nsm, cudaDevAttrMultiProcessorCount, device);
    if (e == cudaSuccess) e = cudaMalloc((void **)&m->d_err, 2 * sizeof(int));
    if (e == cudaSuccess) e = cudaMemset(m->d_err, 0, 2 * sizeof(int));
    if (e == cudaSuccess) e = cudaHostAlloc((void **)&m->h_err, 2 * sizeof(int), cudaHostAllocDefault);
    if (e != cudaSuccess) { orbfe_matcher_destroy(m); return fail(ORBFE_ERR_CUDA, "matcher setup failed: %s", cudaGetErrorString(e)); }
    *out = m;
    return ORBFE_OK;
}

extern "C" int orbfe_matcher_destroy(OrbfeMatcher *m) {
    if (!m) return ORBFE_OK;
    cudaSetDevice(m->device);
    if (m->hs.last) cudaEventSynchronize(m->hs.last);
    if (m->hs.stream) cudaStreamSynchronize(m->hs.stream);
    if (m->scratch) cudaFree(m->scratch);
    m->stage.release();
    if (m->d_err) cudaFree(m->d_err);
    if (m->h_err) cudaFreeHost(m->h_err);
    m->hs.destroy();
    delete m;
    return ORBFE_OK;
}

extern "C" int orbfe_matcher_counters(const OrbfeMatcher *m, unsigned long long *h2d_bytes,
                                      unsigned long long *d2h_bytes, unsigned long long *launches) {
    if (!m) return fail(ORBFE_ERR_ARG, "m is NULL");
    if (h2d_bytes) *h2d_bytes = m->h2d_bytes;
    if (d2h_bytes) *d2h_bytes = m->d2h_bytes;
    if (launches) *launches = m->launches;
    return ORBFE_OK;
}

// Reads the flags the handle's calls so far have raised, whichever streams they ran on, and clears them
extern "C" int orbfe_matcher_sync(OrbfeMatcher *m) {
    if (!m) return fail(ORBFE_ERR_ARG, "m is NULL");
    cudaStream_t s = m->hs.stream;
    if (int rc = m->hs.enter(s)) return rc;
    ORBFE_CUDA_TRY(cudaMemcpyAsync(m->h_err, m->d_err, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (int rc = m->hs.leave(s, true)) return rc;
    if (*m->h_err) {
        const int flags = *m->h_err;
        ORBFE_CUDA_TRY(cudaMemsetAsync(m->d_err, 0, 2 * sizeof(int), s));
        if (int rc = m->hs.leave(s, false)) return rc;   // the next call's flags land after the clear
        if (flags & 2)
            return fail(ORBFE_ERR_ARG, "orbfe_search_by_bow_device: a job's FeatureVector has an out-of-range node row or feature "
                                       "index (its nmatches is -1)");
        if (flags & 4)
            return fail(ORBFE_ERR_ARG, "orbfe_search_for_triangulation_device: a job's FeatureVector has an out-of-range node row or "
                                       "feature index, or a side-2 feature without a map point has an octave outside [0, nlevels) "
                                       "(its nmatches is -1)");
        if (flags & 8)
            return fail(ORBFE_ERR_ARG, "orbfe_distinctive_descriptors_device: a group's pointers or an observation's frame or "
                                       "feature index are out of range (its best index is -1)");
        if (flags & 16)
            return fail(ORBFE_ERR_ARG, "orbfe_normal_and_depth_device: a point's group pointers, an observation or reference slot, "
                                       "or its reference octave are out of range (its outputs are untouched)");
        if (flags & 32)
            return fail(ORBFE_ERR_ARG, "device matcher (*_cams_device): a pair's searched frame has a camera index outside "
                                       "[0, ncams) (its nmatches is -1, its other outputs are untouched)");
        return fail(ORBFE_ERR_CAPACITY, "device matcher: a job's candidate entries exceeded its global scratch (its nmatches is -1; "
                                        "%d entries were needed)", m->h_err[1]);
    }
    return ORBFE_OK;
}

static constexpr size_t kSbpSmemMax = 220 * 1024;   // shared memory per block sbp_prepare grants the fused kernel

// mfGridElementWidthInv / HeightInv (Frame.cc:77-78): `cells` grid cells over [lo, hi]
static float grid_inv(int cells, float lo, float hi) { return (float)cells / (float)(hi - lo); }

// Prepares one launch of sbp_device_kernel over `njobs` jobs of at most `cap` features and `qcap` queries each: the image
// bounds and their grid cell sizes (Frame.cc:77-78) in P, the split of the dynamic shared memory (returned in *smem) and
// `per_job` global scratch entries per job.  The one place that decides whether a job fits the kernel.
static int sbp_prepare(OrbfeMatcher *m, SbpParams &P, float min_x, float min_y, float max_x, float max_y, int cap, int qcap,
                       int njobs, size_t per_job, size_t *smem) {
    P.min_x = min_x; P.min_y = min_y; P.max_x = max_x; P.max_y = max_y;
    P.gw = grid_inv(64, min_x, max_x);
    P.gh = grid_inv(48, min_y, max_y);
    P.cap = cap; P.qcap = qcap;
    const size_t fixed = sbp_smem_fixed_bytes(cap, qcap);
    const size_t total = sbp_smem_total(m, fixed, njobs);
    if (total > kSbpSmemMax)
        return fail(ORBFE_ERR_UNSUPPORTED, "fused matcher: %d features and %d queries per job need %zu bytes of shared memory, more "
                    "than 220 KB (sbp_smem_fixed_bytes(cap, qcap) + 16 KB <= 220 KB: at most 8283 features when every feature is a "
                    "query)", cap, qcap, fixed + 16 * 1024);
    if (per_job > (size_t)INT_MAX) return fail(ORBFE_ERR_UNSUPPORTED, "fused matcher: %zu candidate entries per job", per_job);
    P.smem_fixed = (int)fixed;
    P.smem_entries = (int)((total - fixed) / sizeof(uint32_t));
    if (getenv("ORBFE_SBP_FORCE_SCRATCH")) P.smem_entries = 0;  // test knob: candidate entries always in the global scratch
    P.scratch_per_pair = (int)per_job;
    const size_t need = (size_t)njobs * per_job;
    if (m->scratch_entries < need) {
        ORBFE_CUDA_TRY(cudaEventSynchronize(m->hs.last));   // the handle's pending launches still use the scratch
        if (m->scratch) cudaFree(m->scratch);
        m->scratch = nullptr; m->scratch_entries = 0;
        ORBFE_CUDA_TRY(cudaMalloc((void **)&m->scratch, need * sizeof(uint32_t)));
        m->scratch_entries = need;
    }
    *smem = total;
    return ORBFE_OK;
}

// the launchers' cudaFuncSetAttribute result, then the launch itself
static int sbp_launched(OrbfeMatcher *m, int rc) {
    if (rc) return fail(ORBFE_ERR_CUDA, "cudaFuncSetAttribute failed: %s", cudaGetErrorString((cudaError_t)rc));
    ORBFE_CUDA_TRY(cudaGetLastError());
    m->launches += 1;
    return ORBFE_OK;
}

// The camera table of a *_cams_device call: each camera's bounds checked and its grid cell sizes computed as sbp_prepare
// computes them.  Host-side only.
static int cams_table(int ncams, const OrbfeCamera *cams, const int *d_frame_cam, SbpCams &T) {
    if (ncams < 1 || ncams > ORBFE_MULTI_MAX_GROUPS) return fail(ORBFE_ERR_ARG, "ncams %d outside 1..%d", ncams, ORBFE_MULTI_MAX_GROUPS);
    if (!cams || !d_frame_cam) return fail(ORBFE_ERR_ARG, "NULL camera table or frame-camera array");
    memset(&T, 0, sizeof(T));
    T.n = ncams;
    for (int c = 0; c < ncams; c++) {
        const OrbfeCamera &k = cams[c];
        if (!(k.max_x > k.min_x) || !(k.max_y > k.min_y)) return fail(ORBFE_ERR_ARG, "bad image bounds of camera %d", c);
        SbpCam &t = T.cam[c];
        t.min_x = k.min_x; t.min_y = k.min_y; t.max_x = k.max_x; t.max_y = k.max_y;
        t.gw = grid_inv(64, k.min_x, k.max_x);
        t.gh = grid_inv(48, k.min_y, k.max_y);
        t.fx = k.fx; t.fy = k.fy; t.cx = k.cx; t.cy = k.cy;
    }
    return ORBFE_OK;
}

// SearchByProjection(Frame &Current, const Frame &Last, th) for `npairs` pairs, everything device-resident.  T: NULL, or the
// camera table the kernel takes each pair's geometry from (the geometry arguments are then camera 0's, for the checks only).
static int sbp_projection(OrbfeMatcher *m, int npairs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc, const int *d_counts,
                          int cap, const int *d_cur_idx, const int *d_last_idx, const float *d_world, const uint8_t *d_flags,
                          const float *d_Tcw, float min_x, float min_y, float max_x, float max_y, float scale_factor, int nlevels,
                          float fx, float fy, float cx, float cy, float th, int check_orientation, int *d_cur_mp, int *d_nmatches,
                          void *stream, const SbpCams *T, const int *d_frame_cam) {
    if (!m || npairs < 0 || cap < 1 || cap > 65535 || nlevels < 1 || nlevels > ORBFE_MAX_LEVELS) return fail(ORBFE_ERR_ARG, "bad arguments");
    if (npairs == 0) return ORBFE_OK;
    if (!d_kps || !d_desc || !d_counts || !d_cur_idx || !d_last_idx || !d_world || !d_flags || !d_Tcw || !d_cur_mp || !d_nmatches)
        return fail(ORBFE_ERR_ARG, "NULL argument");
    if (!(max_x > min_x) || !(max_y > min_y)) return fail(ORBFE_ERR_ARG, "bad image bounds");
    cudaStream_t s = m->hs.pick(stream);
    if (int rc = m->hs.enter(s)) return rc;
    SbpParams P;
    memset(&P, 0, sizeof(P));
    P.fx = fx; P.fy = fy; P.cx = cx; P.cy = cy; P.th = th;
    P.scale[0] = 1.0f;                           // Frame.cc:95-103
    for (int i = 1; i < nlevels; i++) P.scale[i] = P.scale[i - 1] * scale_factor;
    P.nlevels = nlevels; P.check_ori = check_orientation ? 1 : 0;
    P.rule = 0; P.th_dist = 100 /* TH_HIGH, ORBmatcher.cc:1576 */; P.nnratio = 0.f;
    size_t smem;
    if (int rc = sbp_prepare(m, P, min_x, min_y, max_x, max_y, cap, cap, npairs, (size_t)64 * cap, &smem)) return rc;
    if (int rc = sbp_launched(m, launch_sbp_device(P, smem, npairs, d_kps, d_desc, d_counts, d_cur_idx, d_last_idx, d_world, d_flags, d_Tcw,
                                                   m->scratch, d_cur_mp, d_nmatches, m->d_err, s, T, d_frame_cam)))
        return rc;
    return m->hs.leave(s, false);
}

extern "C" int orbfe_search_by_projection_device(OrbfeMatcher *m, int npairs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                                 const int *d_counts, int cap, const int *d_cur_idx, const int *d_last_idx,
                                                 const float *d_world, const uint8_t *d_flags, const float *d_Tcw,
                                                 float min_x, float min_y, float max_x, float max_y, float scale_factor,
                                                 int nlevels, float fx, float fy, float cx, float cy, float th,
                                                 int check_orientation, int *d_cur_mp, int *d_nmatches, void *stream) {
    return sbp_projection(m, npairs, d_kps, d_desc, d_counts, cap, d_cur_idx, d_last_idx, d_world, d_flags, d_Tcw, min_x, min_y, max_x,
                          max_y, scale_factor, nlevels, fx, fy, cx, cy, th, check_orientation, d_cur_mp, d_nmatches, stream, nullptr,
                          nullptr);
}

extern "C" int orbfe_search_by_projection_cams_device(OrbfeMatcher *m, int npairs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                                      const int *d_counts, int cap, const int *d_cur_idx, const int *d_last_idx,
                                                      const float *d_world, const uint8_t *d_flags, const float *d_Tcw, int ncams,
                                                      const OrbfeCamera *cams, const int *d_frame_cam, float scale_factor,
                                                      int nlevels, float th, int check_orientation, int *d_cur_mp, int *d_nmatches,
                                                      void *stream) {
    SbpCams T;
    if (int rc = cams_table(ncams, cams, d_frame_cam, T)) return rc;
    const SbpCam &c = T.cam[0];
    return sbp_projection(m, npairs, d_kps, d_desc, d_counts, cap, d_cur_idx, d_last_idx, d_world, d_flags, d_Tcw, c.min_x, c.min_y,
                          c.max_x, c.max_y, scale_factor, nlevels, c.fx, c.fy, c.cx, c.cy, th, check_orientation, d_cur_mp, d_nmatches,
                          stream, &T, d_frame_cam);
}

// SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize) for `npairs` (F1, F2) pairs, device-resident
// (ORBmatcher.cc:598-713; the fused kernel's MODE 2).  d_prev_matched: npairs x cap x 2 floats, in/out.
int orbfe_search_for_initialization_hooked(OrbfeMatcher *m, int npairs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                           const int *d_counts, int cap, const int *d_f1_idx, const int *d_f2_idx,
                                           float *d_prev_matched, float min_x, float min_y, float max_x, float max_y,
                                           int window, float nnratio, int check_orientation, int *d_match12,
                                           int *d_nmatches, void *stream, const SbpParams *hooks);

extern "C" int orbfe_search_for_initialization_device(OrbfeMatcher *m, int npairs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                                      const int *d_counts, int cap, const int *d_f1_idx, const int *d_f2_idx,
                                                      float *d_prev_matched, float min_x, float min_y, float max_x, float max_y,
                                                      int window, float nnratio, int check_orientation, int *d_match12,
                                                      int *d_nmatches, void *stream) {
    return orbfe_search_for_initialization_hooked(m, npairs, d_kps, d_desc, d_counts, cap, d_f1_idx, d_f2_idx, d_prev_matched, min_x, min_y,
                                                  max_x, max_y, window, nnratio, check_orientation, d_match12, d_nmatches, stream, nullptr);
}

// MODE 2 parameters of SearchForInitialization with a `window`-pixel search window (GetFeaturesInArea(x, y, windowSize, 0, 0), :618)
static SbpParams init_params(int window, float nnratio, int check_orientation) {
    SbpParams P;
    memset(&P, 0, sizeof(P));
    P.th = (float)window;
    P.nlevels = 1; P.check_ori = check_orientation ? 1 : 0;
    P.rule = 3; P.th_dist = 50 /* TH_LOW, :652 */; P.nnratio = nnratio;
    return P;
}

// a 100-px window at 720p holds a few hundred level-0 candidates per query: entries live in the global scratch
static size_t init_scratch_per_pair(int cap) { return (size_t)256 * cap; }

// `hooks`: only the xw_* fields are read (rig exchange: wait for the epoch's data at kernel start, publish the release at its end).
// T: camera table (see sbp_projection), or NULL.
static int init_device(OrbfeMatcher *m, int npairs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc, const int *d_counts, int cap,
                       const int *d_f1_idx, const int *d_f2_idx, float *d_prev_matched, float min_x, float min_y, float max_x,
                       float max_y, int window, float nnratio, int check_orientation, int *d_match12, int *d_nmatches, void *stream,
                       const SbpParams *hooks, const SbpCams *T, const int *d_frame_cam) {
    if (!m || npairs < 0 || cap < 1 || cap > 65534 || window < 0) return fail(ORBFE_ERR_ARG, "bad arguments");
    if (npairs == 0) return ORBFE_OK;
    if (!d_kps || !d_desc || !d_counts || !d_f1_idx || !d_f2_idx || !d_prev_matched || !d_match12 || !d_nmatches)
        return fail(ORBFE_ERR_ARG, "NULL argument");
    if (!(max_x > min_x) || !(max_y > min_y)) return fail(ORBFE_ERR_ARG, "bad image bounds");
    cudaStream_t s = m->hs.pick(stream);
    if (int rc = m->hs.enter(s)) return rc;
    SbpParams P = init_params(window, nnratio, check_orientation);
    if (hooks) {
        P.xw_flags = hooks->xw_flags; P.xw_done = hooks->xw_done; P.xw_err = hooks->xw_err; P.xw_n = hooks->xw_n; P.xw_epoch = hooks->xw_epoch;
        for (int r = 0; r < 16; r++) P.xw_ack[r] = hooks->xw_ack[r];
    }
    size_t smem;
    if (int rc = sbp_prepare(m, P, min_x, min_y, max_x, max_y, cap, cap, npairs, init_scratch_per_pair(cap), &smem)) return rc;
    if (int rc = sbp_launched(m, launch_init_device(P, smem, npairs, d_kps, d_desc, d_counts, d_f1_idx, d_f2_idx, d_prev_matched, m->scratch,
                                                    d_match12, d_nmatches, m->d_err, s, T, d_frame_cam)))
        return rc;
    return m->hs.leave(s, false);
}

int orbfe_search_for_initialization_hooked(OrbfeMatcher *m, int npairs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                           const int *d_counts, int cap, const int *d_f1_idx, const int *d_f2_idx,
                                           float *d_prev_matched, float min_x, float min_y, float max_x, float max_y,
                                           int window, float nnratio, int check_orientation, int *d_match12,
                                           int *d_nmatches, void *stream, const SbpParams *hooks) {
    return init_device(m, npairs, d_kps, d_desc, d_counts, cap, d_f1_idx, d_f2_idx, d_prev_matched, min_x, min_y, max_x, max_y, window,
                       nnratio, check_orientation, d_match12, d_nmatches, stream, hooks, nullptr, nullptr);
}

extern "C" int orbfe_search_for_initialization_cams_device(OrbfeMatcher *m, int npairs, const OrbfeKeyPoint *d_kps,
                                                           const uint8_t *d_desc, const int *d_counts, int cap, const int *d_f1_idx,
                                                           const int *d_f2_idx, float *d_prev_matched, int ncams,
                                                           const OrbfeCamera *cams, const int *d_frame_cam, int window, float nnratio,
                                                           int check_orientation, int *d_match12, int *d_nmatches, void *stream) {
    SbpCams T;
    if (int rc = cams_table(ncams, cams, d_frame_cam, T)) return rc;
    const SbpCam &c = T.cam[0];
    return init_device(m, npairs, d_kps, d_desc, d_counts, cap, d_f1_idx, d_f2_idx, d_prev_matched, c.min_x, c.min_y, c.max_x, c.max_y,
                       window, nnratio, check_orientation, d_match12, d_nmatches, stream, nullptr, &T, d_frame_cam);
}

// Guided search with explicit query windows, device-resident (same kernel, EXPLICIT query source).  T: camera table (see
// sbp_projection), or NULL.
static int guided_device(OrbfeMatcher *m, int njobs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc, const int *d_counts, int cap,
                         const int *d_frame_idx, const float *d_qu, const float *d_qv, const float *d_qr, const int *d_qlo,
                         const int *d_qhi, const uint8_t *d_qdesc, const float *d_qangle, const int *d_q_base, const int *d_q_cnt,
                         int qcap, float min_x, float min_y, float max_x, float max_y, int rule, float nnratio, int th_dist,
                         int check_orientation, int *d_slot_owner, int *d_nmatches, void *stream, const SbpCams *T,
                         const int *d_frame_cam) {
    if (!m || njobs < 0 || cap < 1 || cap > 65535 || qcap < 1 || qcap > 65535 || rule < 0 || rule > 2) return fail(ORBFE_ERR_ARG, "bad arguments");
    if (njobs == 0) return ORBFE_OK;
    if (!d_kps || !d_desc || !d_counts || !d_frame_idx || !d_qu || !d_qv || !d_qr || !d_qlo || !d_qhi || !d_qdesc || !d_q_base ||
        !d_q_cnt || !d_slot_owner || !d_nmatches || (check_orientation && !d_qangle))
        return fail(ORBFE_ERR_ARG, "NULL argument");
    if (!(max_x > min_x) || !(max_y > min_y)) return fail(ORBFE_ERR_ARG, "bad image bounds");
    cudaStream_t s = m->hs.pick(stream);
    if (int rc = m->hs.enter(s)) return rc;
    SbpParams P;
    memset(&P, 0, sizeof(P));
    P.nlevels = 1; P.check_ori = check_orientation ? 1 : 0;
    P.rule = rule; P.th_dist = th_dist; P.nnratio = nnratio;
    size_t smem;
    if (int rc = sbp_prepare(m, P, min_x, min_y, max_x, max_y, cap, qcap, njobs, (size_t)64 * std::max(cap, qcap), &smem)) return rc;
    if (int rc = sbp_launched(m, launch_guided_device(P, smem, njobs, d_kps, d_desc, d_counts, d_frame_idx, d_qu, d_qv, d_qr, d_qlo, d_qhi,
                                                      d_qdesc, d_qangle, d_q_base, d_q_cnt, m->scratch, d_slot_owner, nullptr, d_nmatches,
                                                      m->d_err, s, T, d_frame_cam)))
        return rc;
    return m->hs.leave(s, false);
}

extern "C" int orbfe_guided_search_device(OrbfeMatcher *m, int njobs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                          const int *d_counts, int cap, const int *d_frame_idx, const float *d_qu,
                                          const float *d_qv, const float *d_qr, const int *d_qlo, const int *d_qhi,
                                          const uint8_t *d_qdesc, const float *d_qangle, const int *d_q_base,
                                          const int *d_q_cnt, int qcap, float min_x, float min_y, float max_x, float max_y,
                                          int rule, float nnratio, int th_dist, int check_orientation, int *d_slot_owner,
                                          int *d_nmatches, void *stream) {
    return guided_device(m, njobs, d_kps, d_desc, d_counts, cap, d_frame_idx, d_qu, d_qv, d_qr, d_qlo, d_qhi, d_qdesc, d_qangle, d_q_base,
                         d_q_cnt, qcap, min_x, min_y, max_x, max_y, rule, nnratio, th_dist, check_orientation, d_slot_owner, d_nmatches,
                         stream, nullptr, nullptr);
}

extern "C" int orbfe_guided_search_cams_device(OrbfeMatcher *m, int njobs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                               const int *d_counts, int cap, const int *d_frame_idx, const float *d_qu,
                                               const float *d_qv, const float *d_qr, const int *d_qlo, const int *d_qhi,
                                               const uint8_t *d_qdesc, const float *d_qangle, const int *d_q_base,
                                               const int *d_q_cnt, int qcap, int ncams, const OrbfeCamera *cams,
                                               const int *d_frame_cam, int rule, float nnratio, int th_dist, int check_orientation,
                                               int *d_slot_owner, int *d_nmatches, void *stream) {
    SbpCams T;
    if (int rc = cams_table(ncams, cams, d_frame_cam, T)) return rc;
    const SbpCam &c = T.cam[0];
    return guided_device(m, njobs, d_kps, d_desc, d_counts, cap, d_frame_idx, d_qu, d_qv, d_qr, d_qlo, d_qhi, d_qdesc, d_qangle, d_q_base,
                         d_q_cnt, qcap, c.min_x, c.min_y, c.max_x, c.max_y, rule, nnratio, th_dist, check_orientation, d_slot_owner,
                         d_nmatches, stream, &T, d_frame_cam);
}

int orbfe::Stage::layout(std::initializer_list<std::pair<size_t *, size_t>> arrays, size_t *total) {
    size_t off = 0;
    for (const auto &a : arrays) {
        *a.first = off;
        off += (a.second + 255) / 256 * 256;
    }
    *total = off;
    if (cap < off) {
        release();
        const size_t want = off + off / 4;
        ORBFE_CUDA_TRY(cudaHostAlloc((void **)&h, want, cudaHostAllocDefault));
        ORBFE_CUDA_TRY(cudaMalloc((void **)&d, want));
        cap = want;
    }
    return ORBFE_OK;
}

void orbfe::Stage::release() {
    if (h) cudaFreeHost(h);
    if (d) cudaFree(d);
    h = nullptr; d = nullptr; cap = 0;
}

// One host-array matcher call on the staged block: the round trip on the matcher's stream behind the handle's earlier calls,
// its bytes counted, then either orbfe_matcher_sync (`read_flags`: the call's kernels report through d_err) or a plain
// synchronise.  The enqueued device entries enter and leave the same stream again, which orders nothing new.
template <class Enqueue>
static int matcher_round_trip(OrbfeMatcher *m, bool read_flags, size_t up, size_t down, size_t total, Enqueue enqueue) {
    cudaStream_t s = m->hs.stream;
    if (int rc = m->hs.enter(s)) return rc;
    if (int rc = m->stage.round_trip(s, up, down, total, enqueue)) return rc;
    m->h2d_bytes += up;
    m->d2h_bytes += total - down;
    if (int rc = m->hs.leave(s, !read_flags)) return rc;
    return read_flags ? orbfe_matcher_sync(m) : ORBFE_OK;
}

// SearchByBoW (both overloads) for `njobs` frame pairs, device-resident (include/orbfe_match.h).  Arguments are checked before
// the handle is used.
extern "C" int orbfe_search_by_bow_device(OrbfeMatcher *m, int variant, int njobs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                          const int *d_counts, int cap, const int32_t *d_fv_ids, const int32_t *d_fv_ptr,
                                          const int32_t *d_fv_items, const int *d_fv_n, const uint8_t *d_valid, const int *d_idx1,
                                          const int *d_idx2, float nnratio, int check_orientation, int32_t *d_out, int *d_nmatches,
                                          void *stream) {
    if (!m || (variant != 0 && variant != 1) || njobs < 0 || cap < 1 || cap > 65535) return fail(ORBFE_ERR_ARG, "bad arguments");
    if (njobs == 0) return ORBFE_OK;
    if (!d_kps || !d_desc || !d_counts || !d_fv_ids || !d_fv_ptr || !d_fv_items || !d_fv_n || !d_valid || !d_idx1 || !d_idx2 ||
        !d_out || !d_nmatches)
        return fail(ORBFE_ERR_ARG, "NULL argument");
    cudaStream_t s = m->hs.pick(stream);
    if (int rc = m->hs.enter(s)) return rc;
    launch_search_by_bow(variant, njobs, d_kps, d_desc, d_counts, cap, d_fv_ids, d_fv_ptr, d_fv_items, d_fv_n, d_valid, d_idx1, d_idx2,
                         nnratio, check_orientation ? 1 : 0, d_out, d_nmatches, m->d_err, s);
    m->launches += 1;
    return m->hs.leave(s, false);
}

// Offsets, in the staging block, of the two-frame store (frame 0 = side 1, frame 1 = side 2, `cap` slots each) that the
// host-array SearchByBoW and SearchForTriangulation run as one job
struct PairStore { size_t kps, desc, cnt, ids, ptr, items, nn, flags, idx; };

// Packs side f of the store: its counts, frame index, descriptors and FeatureVector (nn nodes: ids, ptr, items).  Item slots
// past ptr[nn] hold -1, so a row that reaches beyond the caller's items is rejected by the kernel instead of being read.
static void pack_pair_side(unsigned char *H, const PairStore &o, int f, int cap, int n, const uint8_t *desc, int nn, const int32_t *ids,
                           const int32_t *ptr, const int32_t *items) {
    const size_t C = (size_t)cap;
    ((int *)(H + o.cnt))[f] = n;
    ((int *)(H + o.nn))[f] = nn;
    ((int *)(H + o.idx))[f] = f;
    if (n) memcpy(H + o.desc + f * C * 32, desc, (size_t)n * 32);
    int *fptr = (int *)(H + o.ptr) + f * (C + 1), *fitems = (int *)(H + o.items) + f * C;
    fptr[0] = 0;
    if (nn) {
        memcpy((int *)(H + o.ids) + f * C, ids, (size_t)nn * 4);
        memcpy(fptr, ptr, ((size_t)nn + 1) * 4);
    }
    const int ni = nn ? std::min(std::max(ptr[nn], 0), cap) : 0;
    if (ni) memcpy(fitems, items, (size_t)ni * 4);
    std::fill(fitems + ni, fitems + C, -1);
}

// SearchByBoW on host arrays: both sides staged as a two-frame store, one H2D, one job of orbfe_search_by_bow_device, one D2H.
extern "C" int orbfe_search_by_bow(OrbfeMatcher *m, int variant, int n1, const uint8_t *desc1, const uint8_t *valid1,
                                   const float *angle1, int nn1, const int32_t *ids1, const int32_t *ptr1, const int32_t *items1,
                                   int n2, const uint8_t *desc2, const uint8_t *valid2, const float *angle2, int nn2,
                                   const int32_t *ids2, const int32_t *ptr2, const int32_t *items2, float nnratio,
                                   int check_orientation, int32_t *out, int *nmatches_out) {
    if (!m || (variant != 0 && variant != 1) || n1 < 0 || n2 < 0 || nn1 < 0 || nn2 < 0 || !out || !nmatches_out)
        return fail(ORBFE_ERR_ARG, "bad arguments");
    if ((n1 > 0 && (!desc1 || !valid1 || !angle1)) || (n2 > 0 && (!desc2 || !angle2 || (variant == 1 && !valid2))) ||
        (nn1 > 0 && (!ids1 || !ptr1 || !items1)) || (nn2 > 0 && (!ids2 || !ptr2 || !items2)))
        return fail(ORBFE_ERR_ARG, "NULL argument");
    const int cap = std::max({n1, n2, nn1, nn2, 1});
    if (cap > 65535) return fail(ORBFE_ERR_UNSUPPORTED, "%d features or FeatureVector nodes on one side: at most 65535", cap);
    ORBFE_CUDA_TRY(cudaSetDevice(m->device));
    const size_t C = (size_t)cap;
    PairStore o;
    size_t o_out, o_nm, total;
    if (int rc = m->stage.layout({{&o.kps, 2 * C * sizeof(OrbfeKeyPoint)}, {&o.desc, 2 * C * 32}, {&o.cnt, 2 * sizeof(int)},
                                  {&o.ids, 2 * C * 4}, {&o.ptr, 2 * (C + 1) * 4}, {&o.items, 2 * C * 4}, {&o.nn, 2 * sizeof(int)},
                                  {&o.flags, 2 * C}, {&o.idx, 2 * sizeof(int)}, {&o_out, C * 4}, {&o_nm, sizeof(int)}},
                              &total))
        return rc;
    unsigned char *H = m->stage.h, *D = m->stage.d;
    pack_pair_side(H, o, 0, cap, n1, desc1, nn1, ids1, ptr1, items1);
    pack_pair_side(H, o, 1, cap, n2, desc2, nn2, ids2, ptr2, items2);
    const int n[2] = {n1, n2};
    const uint8_t *valid[2] = {valid1, variant == 1 ? valid2 : nullptr};
    const float *angle[2] = {angle1, angle2};
    for (int f = 0; f < 2; f++) {
        // search_by_bow_kernel reads no keypoint field but .angle
        OrbfeKeyPoint *kp = (OrbfeKeyPoint *)(H + o.kps) + f * C;
        for (int i = 0; i < n[f]; i++) kp[i].angle = angle[f][i];
        if (valid[f]) memcpy(H + o.flags + f * C, valid[f], (size_t)n[f]);
        else memset(H + o.flags + f * C, 0, (size_t)n[f]);   // variant 0 ignores side 2's flags
    }
    const int *d_idx = (const int *)(D + o.idx);
    if (int rc = matcher_round_trip(m, true, o_out, o_out, total, [&] {
            return orbfe_search_by_bow_device(m, variant, 1, (const OrbfeKeyPoint *)(D + o.kps), D + o.desc, (const int *)(D + o.cnt),
                                              cap, (const int32_t *)(D + o.ids), (const int32_t *)(D + o.ptr),
                                              (const int32_t *)(D + o.items), (const int *)(D + o.nn), D + o.flags, d_idx, d_idx + 1,
                                              nnratio, check_orientation, (int32_t *)(D + o_out), (int *)(D + o_nm), m->hs.stream);
        }))
        return rc;
    const int nout = variant == 0 ? n2 : n1;
    if (nout) memcpy(out, H + o_out, (size_t)nout * 4);
    *nmatches_out = *(const int *)(H + o_nm);
    return ORBFE_OK;
}

// SearchForTriangulation for `njobs` keyframe pairs, device-resident (include/orbfe_match.h).  Arguments are checked before
// the handle is used.
extern "C" int orbfe_search_for_triangulation_device(OrbfeMatcher *m, int njobs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                                     const int *d_counts, int cap, const int32_t *d_fv_ids, const int32_t *d_fv_ptr,
                                                     const int32_t *d_fv_items, const int *d_fv_n, const uint8_t *d_has_mp,
                                                     const int *d_idx1, const int *d_idx2, const float *d_F12, const float *sigma2,
                                                     int nlevels, int check_orientation, int32_t *d_match12, int *d_nmatches,
                                                     void *stream) {
    if (!m || njobs < 0 || cap < 1 || cap > 65535 || nlevels < 1 || nlevels > ORBFE_MAX_LEVELS) return fail(ORBFE_ERR_ARG, "bad arguments");
    if (njobs == 0) return ORBFE_OK;
    if (!d_kps || !d_desc || !d_counts || !d_fv_ids || !d_fv_ptr || !d_fv_items || !d_fv_n || !d_has_mp || !d_idx1 || !d_idx2 ||
        !d_F12 || !sigma2 || !d_match12 || !d_nmatches)
        return fail(ORBFE_ERR_ARG, "NULL argument");
    cudaStream_t s = m->hs.pick(stream);
    if (int rc = m->hs.enter(s)) return rc;
    launch_search_for_triangulation(njobs, d_kps, d_desc, d_counts, cap, d_fv_ids, d_fv_ptr, d_fv_items, d_fv_n, d_has_mp, d_idx1, d_idx2,
                                    d_F12, sigma2, nlevels, check_orientation ? 1 : 0, d_match12, d_nmatches, m->d_err, s);
    m->launches += 1;
    return m->hs.leave(s, false);
}

// SearchForTriangulation on host arrays: staged and run as orbfe_search_by_bow stages and runs SearchByBoW, with F12 as the
// job's 9 floats and as many levels as the octaves of keys2 need.
extern "C" int orbfe_search_for_triangulation(OrbfeMatcher *m, int n1, const OrbfeKeyPoint *keys1, const uint8_t *desc1,
                                              const uint8_t *has_mp1, int nn1, const int32_t *ids1, const int32_t *ptr1,
                                              const int32_t *items1, int n2, const OrbfeKeyPoint *keys2, const uint8_t *desc2,
                                              const uint8_t *has_mp2, int nn2, const int32_t *ids2, const int32_t *ptr2,
                                              const int32_t *items2, const float *F12, const float *sigma2_kf2,
                                              int check_orientation, int32_t *match12_out, int *nmatches_out) {
    if (!m || n1 < 0 || n2 < 0 || nn1 < 0 || nn2 < 0 || !F12 || !sigma2_kf2 || !match12_out || !nmatches_out)
        return fail(ORBFE_ERR_ARG, "bad arguments");
    if ((n1 > 0 && (!keys1 || !desc1 || !has_mp1)) || (n2 > 0 && (!keys2 || !desc2 || !has_mp2)) ||
        (nn1 > 0 && (!ids1 || !ptr1 || !items1)) || (nn2 > 0 && (!ids2 || !ptr2 || !items2)))
        return fail(ORBFE_ERR_ARG, "NULL argument");
    const int cap = std::max({n1, n2, nn1, nn2, 1});
    if (cap > 65535) return fail(ORBFE_ERR_UNSUPPORTED, "%d features or FeatureVector nodes on one side: at most 65535", cap);
    // sigma2_kf2 holds an entry for every octave of keys2; an octave outside [0, nlevels) of a feature the kernel would test
    // rejects the job
    int nlevels = 1;
    for (int i = 0; i < n2; i++) nlevels = std::max(nlevels, std::min(keys2[i].octave, ORBFE_MAX_LEVELS - 1) + 1);
    ORBFE_CUDA_TRY(cudaSetDevice(m->device));
    const size_t C = (size_t)cap;
    PairStore o;
    size_t o_F, o_out, o_nm, total;
    if (int rc = m->stage.layout({{&o.kps, 2 * C * sizeof(OrbfeKeyPoint)}, {&o.desc, 2 * C * 32}, {&o.cnt, 2 * sizeof(int)},
                                  {&o.ids, 2 * C * 4}, {&o.ptr, 2 * (C + 1) * 4}, {&o.items, 2 * C * 4}, {&o.nn, 2 * sizeof(int)},
                                  {&o.flags, 2 * C}, {&o.idx, 2 * sizeof(int)}, {&o_F, 9 * sizeof(float)}, {&o_out, C * 4},
                                  {&o_nm, sizeof(int)}},
                              &total))
        return rc;
    unsigned char *H = m->stage.h, *D = m->stage.d;
    pack_pair_side(H, o, 0, cap, n1, desc1, nn1, ids1, ptr1, items1);
    pack_pair_side(H, o, 1, cap, n2, desc2, nn2, ids2, ptr2, items2);
    const int n[2] = {n1, n2};
    const OrbfeKeyPoint *keys[2] = {keys1, keys2};
    const uint8_t *has_mp[2] = {has_mp1, has_mp2};
    for (int f = 0; f < 2; f++) {
        if (!n[f]) continue;
        memcpy(H + o.kps + f * C * sizeof(OrbfeKeyPoint), keys[f], (size_t)n[f] * sizeof(OrbfeKeyPoint));
        memcpy(H + o.flags + f * C, has_mp[f], (size_t)n[f]);
    }
    memcpy(H + o_F, F12, 9 * sizeof(float));
    const int *d_idx = (const int *)(D + o.idx);
    if (int rc = matcher_round_trip(m, true, o_out, o_out, total, [&] {
            return orbfe_search_for_triangulation_device(m, 1, (const OrbfeKeyPoint *)(D + o.kps), D + o.desc, (const int *)(D + o.cnt),
                                                         cap, (const int32_t *)(D + o.ids), (const int32_t *)(D + o.ptr),
                                                         (const int32_t *)(D + o.items), (const int *)(D + o.nn), D + o.flags, d_idx,
                                                         d_idx + 1, (const float *)(D + o_F), sigma2_kf2, nlevels, check_orientation,
                                                         (int32_t *)(D + o_out), (int *)(D + o_nm), m->hs.stream);
        }))
        return rc;
    if (n1) memcpy(match12_out, H + o_out, (size_t)n1 * 4);
    *nmatches_out = *(const int *)(H + o_nm);
    return ORBFE_OK;
}

extern "C" int orbfe_hamming_csr_device(OrbfeMatcher *m, const uint8_t *d_q, const uint8_t *d_t, const int32_t *d_row_ptr,
                                        const int32_t *d_cols, int nq, int npairs, uint16_t *d_out, void *stream) {
    if (!m || (nq > 0 && (!d_q || !d_t || !d_row_ptr))) return fail(ORBFE_ERR_ARG, "NULL argument");
    ORBFE_CUDA_TRY(cudaSetDevice(m->device));
    if (nq <= 0 || npairs <= 0) return ORBFE_OK;
    cudaStream_t s = m->hs.pick(stream);
    if (int rc = m->hs.enter(s)) return rc;
    launch_hamming_csr(d_q, d_t, d_row_ptr, d_cols, nq, npairs, d_out, s);
    return m->hs.leave(s, false);
}

extern "C" int orbfe_hamming_csr(OrbfeMatcher *m, const uint8_t *q, int nq, const uint8_t *t, int nt,
                                 const int32_t *row_ptr, const int32_t *cols, uint16_t *out) {
    if (!m || nq < 0 || nt < 0) return fail(ORBFE_ERR_ARG, "bad arguments");
    if (nq == 0) return ORBFE_OK;
    if (!q || !row_ptr) return fail(ORBFE_ERR_ARG, "NULL argument");
    const int np = row_ptr[nq];
    if (np == 0) return ORBFE_OK;
    if (np < 0) return fail(ORBFE_ERR_ARG, "row_ptr[nq]=%d is negative", np);
    if (!t || !cols || !out || nt == 0) return fail(ORBFE_ERR_ARG, "NULL argument");
    for (int k = 0; k < np; k++)
        if (cols[k] < 0 || cols[k] >= nt) return fail(ORBFE_ERR_ARG, "cols[%d]=%d out of range", k, cols[k]);
    ORBFE_CUDA_TRY(cudaSetDevice(m->device));
    const size_t b_q = (size_t)nq * 32, b_t = (size_t)nt * 32, b_row = sizeof(int32_t) * ((size_t)nq + 1);
    const size_t b_cols = sizeof(int32_t) * (size_t)np, b_out = sizeof(uint16_t) * (size_t)np;
    size_t o_q, o_t, o_row, o_cols, o_out, total;
    if (int rc = m->stage.layout({{&o_q, b_q}, {&o_t, b_t}, {&o_row, b_row}, {&o_cols, b_cols}, {&o_out, b_out}}, &total)) return rc;
    unsigned char *H = m->stage.h, *D = m->stage.d;
    memcpy(H + o_q, q, b_q);
    memcpy(H + o_t, t, b_t);
    memcpy(H + o_row, row_ptr, b_row);
    memcpy(H + o_cols, cols, b_cols);
    if (int rc = matcher_round_trip(m, false, o_out, o_out, total, [&]() -> int {
            if (int rc = orbfe_hamming_csr_device(m, D + o_q, D + o_t, (const int32_t *)(D + o_row), (const int32_t *)(D + o_cols), nq,
                                                  np, (uint16_t *)(D + o_out), m->hs.stream))
                return rc;
            m->launches += 1;
            return ORBFE_OK;
        }))
        return rc;
    memcpy(out, H + o_out, b_out);
    return ORBFE_OK;
}

// The staging block is pinned and sized by the largest call the handle has seen: an nq x nt output this large stays pinned
// for the handle's lifetime.
extern "C" int orbfe_hamming_dense(OrbfeMatcher *m, const uint8_t *q, int nq, const uint8_t *t, int nt, uint16_t *out) {
    if (!m || nq < 0 || nt < 0) return fail(ORBFE_ERR_ARG, "bad arguments");
    if (nq == 0 || nt == 0) return ORBFE_OK;
    if (!q || !t || !out) return fail(ORBFE_ERR_ARG, "NULL argument");
    ORBFE_CUDA_TRY(cudaSetDevice(m->device));
    const size_t b_q = (size_t)nq * 32, b_t = (size_t)nt * 32, b_out = sizeof(uint16_t) * (size_t)nq * nt;
    size_t o_q, o_t, o_out, total;
    if (int rc = m->stage.layout({{&o_q, b_q}, {&o_t, b_t}, {&o_out, b_out}}, &total)) return rc;
    unsigned char *H = m->stage.h, *D = m->stage.d;
    memcpy(H + o_q, q, b_q);
    memcpy(H + o_t, t, b_t);
    if (int rc = matcher_round_trip(m, false, o_out, o_out, total, [&]() -> int {
            launch_hamming_dense(D + o_q, nq, D + o_t, nt, (uint16_t *)(D + o_out), m->hs.stream);
            ORBFE_CUDA_TRY(cudaGetLastError());
            return ORBFE_OK;
        }))
        return rc;
    memcpy(out, H + o_out, b_out);
    return ORBFE_OK;
}

// Frame::UndistortKeyPoints / ComputeImageBounds (include/orbfe_match.h)
extern "C" int orbfe_undistort_keypoints_device(OrbfeMatcher *m, const OrbfeKeyPoint *d_in, OrbfeKeyPoint *d_out, int n, float fx,
                                                float fy, float cx, float cy, const float *dist5, void *stream) {
    if (!m || n < 0 || !dist5 || !(fx != 0.f) || !(fy != 0.f)) return fail(ORBFE_ERR_ARG, "bad arguments");
    if (n == 0) return ORBFE_OK;
    if (!d_in || !d_out) return fail(ORBFE_ERR_ARG, "NULL argument");
    cudaStream_t s = m->hs.pick(stream);
    if (int rc = m->hs.enter(s)) return rc;
    if (dist5[0] == 0.0f) {  // mvKeysUn = mvKeys (Frame.cc:291-295)
        if (d_in != d_out) ORBFE_CUDA_TRY(cudaMemcpyAsync(d_out, d_in, sizeof(OrbfeKeyPoint) * (size_t)n, cudaMemcpyDeviceToDevice, s));
        return m->hs.leave(s, false);
    }
    launch_undistort(fx, fy, cx, cy, dist5, d_in, d_out, n, s);
    m->launches += 1;
    return m->hs.leave(s, false);
}

extern "C" int orbfe_undistort_keypoints(OrbfeMatcher *m, const OrbfeKeyPoint *in, OrbfeKeyPoint *out, int n, float fx, float fy,
                                         float cx, float cy, const float *dist5) {
    if (!m || n < 0 || !dist5) return fail(ORBFE_ERR_ARG, "bad arguments");
    if (n == 0) return ORBFE_OK;
    if (!in || !out) return fail(ORBFE_ERR_ARG, "NULL argument");
    if (dist5[0] == 0.0f) {
        if (in != out) memcpy(out, in, sizeof(OrbfeKeyPoint) * (size_t)n);
        return ORBFE_OK;
    }
    ORBFE_CUDA_TRY(cudaSetDevice(m->device));
    // one array, undistorted in place on the device: input and output of the block at once
    size_t o_kps, total;
    if (int rc = m->stage.layout({{&o_kps, sizeof(OrbfeKeyPoint) * (size_t)n}}, &total)) return rc;
    OrbfeKeyPoint *h_kps = (OrbfeKeyPoint *)m->stage.h, *d_kps = (OrbfeKeyPoint *)m->stage.d;
    memcpy(h_kps, in, sizeof(OrbfeKeyPoint) * (size_t)n);
    if (int rc = matcher_round_trip(m, false, total, 0, total, [&] {
            return orbfe_undistort_keypoints_device(m, d_kps, d_kps, n, fx, fy, cx, cy, dist5, m->hs.stream);
        }))
        return rc;
    memcpy(out, h_kps, sizeof(OrbfeKeyPoint) * (size_t)n);
    return ORBFE_OK;
}

extern "C" int orbfe_image_bounds(OrbfeMatcher *m, int cols, int rows, float fx, float fy, float cx, float cy, const float *dist5,
                                  float *bounds4) {
    if (!m || !dist5 || !bounds4 || cols < 1 || rows < 1) return fail(ORBFE_ERR_ARG, "bad arguments");
    if (dist5[0] == 0.0f) {  // Frame.cc:343-348
        bounds4[0] = 0.f; bounds4[1] = 0.f; bounds4[2] = (float)cols; bounds4[3] = (float)rows;
        return ORBFE_OK;
    }
    OrbfeKeyPoint c[4];
    memset(c, 0, sizeof(c));
    c[1].x = (float)cols; c[2].y = (float)rows; c[3].x = (float)cols; c[3].y = (float)rows;   // Frame.cc:325-329
    const int rc = orbfe_undistort_keypoints(m, c, c, 4, fx, fy, cx, cy, dist5);
    if (rc) return rc;
    // Frame's bounds are `static int` (Frame.h:121-124), converted as x86-64 does: NaN (a corner whose undistortion meets a zero
    // denominator) and values outside [-2^31, 2^31) become INT_MIN
    auto frame_int = [](float f) { return (f >= -2147483648.0f && f < 2147483648.0f) ? (float)(int)f : -2147483648.0f; };
    bounds4[0] = frame_int(std::min(std::floor(c[0].x), std::floor(c[2].x)));   // :336-339
    bounds4[2] = frame_int(std::max(std::ceil(c[1].x), std::ceil(c[3].x)));
    bounds4[1] = frame_int(std::min(std::floor(c[0].y), std::floor(c[1].y)));
    bounds4[3] = frame_int(std::max(std::ceil(c[2].y), std::ceil(c[3].y)));
    return ORBFE_OK;
}

// MapPoint::ComputeDistinctiveDescriptors for many map points in one launch (include/orbfe_bow.h)
extern "C" int orbfe_distinctive_descriptors(OrbfeMatcher *m, const uint8_t *desc, const int32_t *group_ptr, int ngroups,
                                             int32_t *best_out) {
    if (!m || ngroups < 0) return fail(ORBFE_ERR_ARG, "bad arguments");
    if (ngroups == 0) return ORBFE_OK;
    if (!group_ptr || !best_out) return fail(ORBFE_ERR_ARG, "NULL argument");
    const int total = group_ptr[ngroups];
    if (group_ptr[0] != 0 || total < 0 || (total > 0 && !desc)) return fail(ORBFE_ERR_ARG, "bad group_ptr");
    for (int g = 0; g < ngroups; g++)
        if (group_ptr[g + 1] < group_ptr[g]) return fail(ORBFE_ERR_ARG, "group_ptr must be non-decreasing");
    ORBFE_CUDA_TRY(cudaSetDevice(m->device));
    const size_t b_desc = (size_t)total * 32, b_ptr = sizeof(int) * ((size_t)ngroups + 1), b_best = sizeof(int) * (size_t)ngroups;
    size_t o_desc, o_ptr, o_best, nbytes;
    if (int rc = m->stage.layout({{&o_desc, b_desc}, {&o_ptr, b_ptr}, {&o_best, b_best}}, &nbytes)) return rc;
    unsigned char *H = m->stage.h, *D = m->stage.d;
    if (total > 0) memcpy(H + o_desc, desc, b_desc);   // all groups empty: nothing to upload, the launch still writes every -1
    memcpy(H + o_ptr, group_ptr, b_ptr);
    if (int rc = matcher_round_trip(m, false, o_best, o_best, nbytes, [&]() -> int {
            launch_distinctive(D + o_desc, (const int *)(D + o_ptr), ngroups, (int *)(D + o_best), m->hs.stream);
            ORBFE_CUDA_TRY(cudaGetLastError());
            return ORBFE_OK;
        }))
        return rc;
    m->launches += 1;
    memcpy(best_out, H + o_best, b_best);
    return ORBFE_OK;
}

// The same on the frame store, every map point's descriptors addressed through its observation list
// (include/orbfe_bow.h).  Arguments are checked before the handle is used.
extern "C" int orbfe_distinctive_descriptors_device(OrbfeMatcher *m, int ngroups, const uint8_t *d_desc, const int *d_counts,
                                                    int nframes, int cap, const int32_t *d_group_ptr, const int32_t *d_obs, int nobs,
                                                    int32_t *d_best, uint8_t *d_mp_desc, void *stream) {
    if (!m || ngroups < 0 || nobs < 0 || cap < 1 || cap > 65535 || nframes < 1 || (long long)nframes * cap > INT32_MAX)
        return fail(ORBFE_ERR_ARG, "orbfe_distinctive_descriptors_device: bad arguments");
    if (ngroups == 0) return ORBFE_OK;
    if (!d_desc || !d_counts || !d_group_ptr || !d_obs || !d_best || !d_mp_desc)
        return fail(ORBFE_ERR_ARG, "orbfe_distinctive_descriptors_device: NULL argument");
    if (((uintptr_t)d_desc | (uintptr_t)d_mp_desc) % 16)
        return fail(ORBFE_ERR_ARG, "orbfe_distinctive_descriptors_device: d_desc and d_mp_desc must be 16-byte aligned");
    cudaStream_t s = m->hs.pick(stream);
    if (int rc = m->hs.enter(s)) return rc;
    launch_distinctive_obs(d_desc, d_counts, nframes, cap, d_group_ptr, d_obs, nobs, ngroups, d_best, d_mp_desc, m->d_err, s);
    m->launches += 1;
    return m->hs.leave(s, false);
}

// MapPoint::UpdateNormalAndDepth for many map points in one launch, on the frame store (include/orbfe_bow.h).  Arguments
// are checked before the handle is used.
extern "C" int orbfe_normal_and_depth_device(OrbfeMatcher *m, int npoints, const OrbfeKeyPoint *d_kps, const int *d_counts, int nframes,
                                             int cap, const float *d_centers, const int32_t *d_group_ptr, const int32_t *d_obs, int nobs,
                                             const float *d_world, const int32_t *d_ref_obs, float scale_factor, int nlevels,
                                             const float *scale_factors, float *d_normal, float *d_min_dist, float *d_max_dist,
                                             void *stream) {
    if (!m || npoints < 0 || nobs < 0 || cap < 1 || cap > 65535 || nframes < 1 || (long long)nframes * cap > INT32_MAX || nlevels < 1 ||
        nlevels > ORBFE_MAX_LEVELS)
        return fail(ORBFE_ERR_ARG, "orbfe_normal_and_depth_device: bad arguments");
    if (npoints == 0) return ORBFE_OK;
    if (!d_kps || !d_counts || !d_centers || !d_group_ptr || !d_obs || !d_world || !d_ref_obs || !scale_factors || !d_normal ||
        !d_min_dist || !d_max_dist)
        return fail(ORBFE_ERR_ARG, "orbfe_normal_and_depth_device: NULL argument");
    cudaStream_t s = m->hs.pick(stream);
    if (int rc = m->hs.enter(s)) return rc;
    launch_normal_depth_obs(d_kps, d_counts, nframes, cap, d_centers, d_group_ptr, d_obs, nobs, d_world, d_ref_obs, scale_factor, nlevels,
                            scale_factors, npoints, d_normal, d_min_dist, d_max_dist, m->d_err, s);
    m->launches += 1;
    return m->hs.leave(s, false);
}

// The same for callers without a frame store: every centre given on the host, staged through the matcher's block and run
// as one launch of the same kernel (include/orbfe_bow.h)
extern "C" int orbfe_normal_and_depth(OrbfeMatcher *m, int npoints, const float *world, const float *ref_centers, const int32_t *ref_octave,
                                      const int32_t *group_ptr, const float *obs_centers, float scale_factor, int nlevels,
                                      const float *scale_factors, float *normal_out, float *min_dist_out, float *max_dist_out) {
    if (!m || npoints < 0 || nlevels < 1 || nlevels > ORBFE_MAX_LEVELS) return fail(ORBFE_ERR_ARG, "orbfe_normal_and_depth: bad arguments");
    if (npoints == 0) return ORBFE_OK;
    if (!world || !ref_centers || !ref_octave || !group_ptr || !scale_factors || !normal_out || !min_dist_out || !max_dist_out)
        return fail(ORBFE_ERR_ARG, "orbfe_normal_and_depth: NULL argument");
    const int total = group_ptr[npoints];
    if (group_ptr[0] != 0 || total < 0 || (total > 0 && !obs_centers)) return fail(ORBFE_ERR_ARG, "orbfe_normal_and_depth: bad group_ptr");
    for (int g = 0; g < npoints; g++) {
        if (group_ptr[g + 1] < group_ptr[g]) return fail(ORBFE_ERR_ARG, "orbfe_normal_and_depth: group_ptr must be non-decreasing");
        if (group_ptr[g + 1] > group_ptr[g] && (ref_octave[g] < 0 || ref_octave[g] >= nlevels))
            return fail(ORBFE_ERR_ARG, "orbfe_normal_and_depth: point %d has reference octave %d outside [0, %d)", g, ref_octave[g], nlevels);
    }
    ORBFE_CUDA_TRY(cudaSetDevice(m->device));
    const size_t NP = (size_t)npoints, b3 = 3 * sizeof(float) * NP, b1 = sizeof(float) * NP;
    size_t o_world, o_ref, o_oct, o_ptr, o_obs, o_normal, o_min, o_max, nbytes;
    if (int rc = m->stage.layout({{&o_world, b3}, {&o_ref, b3}, {&o_oct, sizeof(int) * NP}, {&o_ptr, sizeof(int) * (NP + 1)},
                                  {&o_obs, 3 * sizeof(float) * (size_t)total}, {&o_normal, b3}, {&o_min, b1}, {&o_max, b1}},
                                 &nbytes))
        return rc;
    unsigned char *H = m->stage.h, *D = m->stage.d;
    memcpy(H + o_world, world, b3);
    memcpy(H + o_ref, ref_centers, b3);
    memcpy(H + o_oct, ref_octave, sizeof(int) * NP);
    memcpy(H + o_ptr, group_ptr, sizeof(int) * (NP + 1));
    if (total > 0) memcpy(H + o_obs, obs_centers, 3 * sizeof(float) * (size_t)total);
    // the outputs go up too: the rows of empty groups come back as the caller passed them
    memcpy(H + o_normal, normal_out, b3);
    memcpy(H + o_min, min_dist_out, b1);
    memcpy(H + o_max, max_dist_out, b1);
    if (int rc = matcher_round_trip(m, false, nbytes, o_normal, nbytes, [&]() -> int {
            launch_normal_depth((const float *)(D + o_obs), (const int *)(D + o_ptr), (const float *)(D + o_world),
                                (const float *)(D + o_ref), (const int *)(D + o_oct), scale_factor, nlevels, scale_factors, npoints,
                                (float *)(D + o_normal), (float *)(D + o_min), (float *)(D + o_max), m->hs.stream);
            ORBFE_CUDA_TRY(cudaGetLastError());
            return ORBFE_OK;
        }))
        return rc;
    m->launches += 1;
    memcpy(normal_out, H + o_normal, b3);
    memcpy(min_dist_out, H + o_min, b1);
    memcpy(max_dist_out, H + o_max, b1);
    return ORBFE_OK;
}

// Device half of orbfe_bow_db_detect (host/bow_host.cpp): per-keyframe shared-word count, first shared word, L1 score.
int orbfe::bow_db_score(OrbfeMatcher *m, int nq, const int32_t *q_ids, const double *q_vals, int nkf, const int32_t *kf_ptr,
                        const int32_t *db_ids, const double *db_vals, int32_t *common, int32_t *first, double *score) {
    const size_t NQ = (size_t)nq, NK = (size_t)nkf, nw = (size_t)kf_ptr[nkf];
    ORBFE_CUDA_TRY(cudaSetDevice(m->device));
    size_t o_qi, o_qv, o_kp, o_di, o_dv, o_c, o_f, o_s, total;
    if (int rc = m->stage.layout({{&o_qi, NQ * sizeof(int)}, {&o_qv, NQ * sizeof(double)}, {&o_kp, (NK + 1) * sizeof(int)},
                                  {&o_di, nw * sizeof(int)}, {&o_dv, nw * sizeof(double)}, {&o_c, NK * sizeof(int)},
                                  {&o_f, NK * sizeof(int)}, {&o_s, NK * sizeof(double)}},
                              &total))
        return rc;
    unsigned char *H = m->stage.h, *D = m->stage.d;
    if (nq > 0) {
        memcpy(H + o_qi, q_ids, NQ * sizeof(int));
        memcpy(H + o_qv, q_vals, NQ * sizeof(double));
    }
    memcpy(H + o_kp, kf_ptr, (NK + 1) * sizeof(int));
    if (nw > 0) {
        memcpy(H + o_di, db_ids, nw * sizeof(int));
        memcpy(H + o_dv, db_vals, nw * sizeof(double));
    }
    if (int rc = matcher_round_trip(m, false, o_c, o_c, total, [&]() -> int {
            launch_bow_db_score(nq, (const int *)(D + o_qi), (const double *)(D + o_qv), nkf, (const int *)(D + o_kp),
                                (const int *)(D + o_di), (const double *)(D + o_dv), (int *)(D + o_c), (int *)(D + o_f),
                                (double *)(D + o_s), m->hs.stream);
            ORBFE_CUDA_TRY(cudaGetLastError());
            return ORBFE_OK;
        }))
        return rc;
    m->launches += 1;
    memcpy(common, H + o_c, NK * sizeof(int));
    memcpy(first, H + o_f, NK * sizeof(int));
    memcpy(score, H + o_s, NK * sizeof(double));
    return ORBFE_OK;
}

extern "C" int orbfe_knn2_groups_device(OrbfeMatcher *m, const uint8_t *d_q, int nq, const uint8_t *d_db, int ngroups,
                                        int group_size, uint16_t *d_best, int32_t *d_best_idx, uint16_t *d_second,
                                        void *stream) {
    if (!m || nq < 0 || ngroups < 0 || group_size < 0) return fail(ORBFE_ERR_ARG, "bad arguments");
    if (nq == 0 || ngroups == 0) return ORBFE_OK;
    if (!d_q || !d_db || !d_best || !d_best_idx || !d_second) return fail(ORBFE_ERR_ARG, "NULL argument");
    cudaStream_t s = m->hs.pick(stream);
    if (int rc = m->hs.enter(s)) return rc;
    launch_knn2_groups(d_q, nq, d_db, ngroups, group_size, d_best, d_best_idx, d_second, s);
    return m->hs.leave(s, false);
}

// The database is staged through the handle's pinned block, which keeps the size of the largest call; a bulk sweep belongs on
// orbfe_knn2_groups_device.
extern "C" int orbfe_knn2_groups(OrbfeMatcher *m, const uint8_t *q, int nq, const uint8_t *db, int ngroups,
                                 int group_size, uint16_t *best, int32_t *best_idx, uint16_t *second) {
    if (!m || nq < 0 || ngroups < 0 || group_size < 0) return fail(ORBFE_ERR_ARG, "bad arguments");
    if (nq == 0 || ngroups == 0) return ORBFE_OK;
    if (!q || !db || !best || !best_idx || !second) return fail(ORBFE_ERR_ARG, "NULL argument");
    ORBFE_CUDA_TRY(cudaSetDevice(m->device));
    const size_t no = (size_t)ngroups * nq;
    const size_t b_q = (size_t)nq * 32, b_db = (size_t)ngroups * group_size * 32;
    size_t o_q, o_db, o_best, o_idx, o_second, total;
    if (int rc = m->stage.layout({{&o_q, b_q}, {&o_db, b_db}, {&o_best, sizeof(uint16_t) * no}, {&o_idx, sizeof(int32_t) * no},
                                  {&o_second, sizeof(uint16_t) * no}},
                              &total))
        return rc;
    unsigned char *H = m->stage.h, *D = m->stage.d;
    memcpy(H + o_q, q, b_q);
    memcpy(H + o_db, db, b_db);
    if (int rc = matcher_round_trip(m, false, o_best, o_best, total, [&] {
            return orbfe_knn2_groups_device(m, D + o_q, nq, D + o_db, ngroups, group_size, (uint16_t *)(D + o_best),
                                            (int32_t *)(D + o_idx), (uint16_t *)(D + o_second), m->hs.stream);
        }))
        return rc;
    memcpy(best, H + o_best, sizeof(uint16_t) * no);
    memcpy(best_idx, H + o_idx, sizeof(int32_t) * no);
    memcpy(second, H + o_second, sizeof(uint16_t) * no);
    return ORBFE_OK;
}

// ------------------------------------------------------------------------------------------------
// Host-array windowed matchers (orbfe_internal.h) on the fused kernel: the caller's arrays are packed into the pinned staging
// block, inputs go up in one H2D, the kernel runs, results come back in one D2H.
// ------------------------------------------------------------------------------------------------

// The block holds inputs [0, inout), arrays the kernel updates in place [inout, out) and outputs [out, total).  `pack_inout`
// writes the in-place arrays from the caller's, `launch(per_job)` enqueues the kernel with `per_job` scratch entries per job.
// A job whose candidates overflow its scratch leaves its outputs unwritten and reports the entries it needed
// (sbp_device_kernel, d_err[1]); the call then runs once more from the caller's arrays with exactly that scratch.
template <class Pack, class Launch>
static int run_staged(OrbfeMatcher *m, size_t inout, size_t out, size_t total, size_t per_job, Pack pack_inout, Launch launch) {
    for (bool grown = false;; grown = true) {
        pack_inout();
        const int rc = matcher_round_trip(m, true, out, inout, total, [&] { return launch(per_job); });
        if (rc != ORBFE_ERR_CAPACITY || grown) return rc;
        per_job = (size_t)m->h_err[1];
    }
}

static bool same_geometry(const OrbfeFrameView &a, const OrbfeFrameView &b) {
    if (a.min_x != b.min_x || a.min_y != b.min_y || a.max_x != b.max_x || a.max_y != b.max_y || a.grid_inv_w != b.grid_inv_w ||
        a.grid_inv_h != b.grid_inv_h || a.nlevels != b.nlevels)
        return false;
    for (int l = 0; l < a.nlevels; l++)
        if (a.scale_factors[l] != b.scale_factors[l]) return false;
    return true;
}

// SearchByProjection(Frame &Current, const Frame &Last, th) for `npairs` pairs.  The kernel reads only the Current view's
// geometry, so pairs are launched in groups whose Current views share it (usually one group, one launch).
int orbfe::sbp_frames_host(OrbfeMatcher *m, int npairs, const OrbfeFrameView *cur, const OrbfeFrameView *last,
                           const uint8_t *const *last_has_mp, const uint8_t *const *last_outlier, const float *const *last_world,
                           const float *const *Tcw, float fx, float fy, float cx, float cy, float th, int check_orientation,
                           int *const *cur_mp_inout, int *nmatches_out) {
    if (npairs == 0) return ORBFE_OK;
    // groups of pairs, staged in group order: pair order[k] is staged at position k; group g is [gbeg[g], gbeg[g + 1])
    std::vector<int> group(npairs), order, gbeg;
    std::vector<const OrbfeFrameView *> rep;
    int cap = 1;
    for (int j = 0; j < npairs; j++) {
        int g = 0;
        while (g < (int)rep.size() && !same_geometry(*rep[g], cur[j])) g++;
        if (g == (int)rep.size()) rep.push_back(&cur[j]);
        group[j] = g;
        cap = std::max({cap, cur[j].n, last[j].n});
    }
    for (int g = 0; g < (int)rep.size(); g++) {
        gbeg.push_back((int)order.size());
        for (int j = 0; j < npairs; j++)
            if (group[j] == g) order.push_back(j);
    }
    gbeg.push_back(npairs);
    ORBFE_CUDA_TRY(cudaSetDevice(m->device));
    // frame slots: a frame that appears several times (in a video stream the Last frame of pair j is the Current
    // frame of pair j-1) is staged and uploaded once.  Identity = same keypoint and descriptor arrays.
    // A frame used as Last carries that pair's world/flags arrays; two pairs that share a Last frame but pass
    // different world/flags arrays get separate slots.
    struct Slot { const OrbfeFrameView *v; const float *world; const uint8_t *has, *outl; };
    std::vector<Slot> slots;
    std::vector<int> ci(npairs), li(npairs);
    {
        std::unordered_map<const void *, std::vector<int>> by_keys;
        auto find_slot = [&](const OrbfeFrameView &v, const float *world, const uint8_t *has, const uint8_t *outl, bool as_last) {
            auto &cand = by_keys[(const void *)v.keys_un];
            for (int sidx : cand) {
                Slot &S = slots[sidx];
                if (S.v->desc != v.desc || S.v->n != v.n) continue;
                if (as_last) {
                    if (S.world && (S.world != world || S.has != has || S.outl != outl)) continue;
                    S.world = world; S.has = has; S.outl = outl;
                }
                return sidx;
            }
            slots.push_back({&v, as_last ? world : nullptr, as_last ? has : nullptr, as_last ? outl : nullptr});
            cand.push_back((int)slots.size() - 1);
            return (int)slots.size() - 1;
        };
        for (int j = 0; j < npairs; j++) {
            ci[j] = find_slot(cur[j], nullptr, nullptr, nullptr, false);
            li[j] = find_slot(last[j], last_world[j], last_has_mp[j], last_outlier[j], true);
        }
    }
    const size_t nf = slots.size();
    size_t o_kps, o_desc, o_cnt, o_world, o_flags, o_T, o_ci, o_li, o_mp, o_nm, total;
    if (int rc = m->stage.layout({{&o_kps, nf * cap * sizeof(OrbfeKeyPoint)}, {&o_desc, nf * cap * 32}, {&o_cnt, nf * sizeof(int)},
                                  {&o_world, nf * cap * 3 * sizeof(float)}, {&o_flags, nf * cap},
                                  {&o_T, (size_t)npairs * 12 * sizeof(float)}, {&o_ci, (size_t)npairs * sizeof(int)},
                                  {&o_li, (size_t)npairs * sizeof(int)}, {&o_mp, (size_t)npairs * cap * sizeof(int)},
                                  {&o_nm, (size_t)npairs * sizeof(int)}},
                              &total))
        return rc;
    unsigned char *H = m->stage.h, *D = m->stage.d;
    int *h_cnt = (int *)(H + o_cnt), *h_ci = (int *)(H + o_ci), *h_li = (int *)(H + o_li);
    auto pack_slot = [&](int sidx) {
        const Slot &S = slots[sidx];
        const OrbfeFrameView &V = *S.v;
        h_cnt[sidx] = V.n;
        if (!V.n) return;
        memcpy(H + o_kps + (size_t)sidx * cap * sizeof(OrbfeKeyPoint), V.keys_un, (size_t)V.n * sizeof(OrbfeKeyPoint));
        memcpy(H + o_desc + (size_t)sidx * cap * 32, V.desc, (size_t)V.n * 32);
        if (S.world) {
            memcpy(H + o_world + (size_t)sidx * cap * 3 * sizeof(float), S.world, (size_t)V.n * 3 * sizeof(float));
            unsigned char *fl = H + o_flags + (size_t)sidx * cap;
            for (int i = 0; i < V.n; i++) fl[i] = (S.has[i] && !S.outl[i]) ? 1 : 0;
        }
    };
    {   // staging is a plain memory copy of ~150 KB per frame: spread it over a few host threads
        const int nt = (int)std::min<size_t>(8, nf);
        if (nt <= 1) {
            for (size_t k = 0; k < nf; k++) pack_slot((int)k);
        } else {
            std::atomic<int> next(0);
            std::vector<std::thread> th;
            for (int w = 0; w < nt; w++)
                th.emplace_back([&]() { for (int k = next++; k < (int)nf; k = next++) pack_slot(k); });
            for (auto &w : th) w.join();
        }
    }
    for (int k = 0; k < npairs; k++) {
        const int j = order[k];
        h_ci[k] = ci[j]; h_li[k] = li[j];
        memcpy(H + o_T + (size_t)k * 12 * sizeof(float), Tcw[j], 12 * sizeof(float));
    }
    auto pack_mp = [&]() {
        for (int k = 0; k < npairs; k++)
            if (cur[order[k]].n) memcpy(H + o_mp + (size_t)k * cap * sizeof(int), cur_mp_inout[order[k]], (size_t)cur[order[k]].n * sizeof(int));
    };
    auto launch = [&](size_t per_pair) -> int {
        for (size_t g = 0; g + 1 < gbeg.size(); g++) {
            const OrbfeFrameView &C = *rep[g];
            const int k0 = gbeg[g], n = gbeg[g + 1] - k0;
            SbpParams P;
            memset(&P, 0, sizeof(P));
            P.fx = fx; P.fy = fy; P.cx = cx; P.cy = cy; P.th = th;
            for (int l = 0; l < C.nlevels; l++) P.scale[l] = C.scale_factors[l];
            P.nlevels = C.nlevels; P.check_ori = check_orientation ? 1 : 0;
            P.rule = 0; P.th_dist = 100 /* TH_HIGH, ORBmatcher.cc:1576 */; P.nnratio = 0.f;
            size_t smem;
            if (int rc = sbp_prepare(m, P, C.min_x, C.min_y, C.max_x, C.max_y, cap, cap, n, per_pair, &smem)) return rc;
            P.gw = C.grid_inv_w; P.gh = C.grid_inv_h;
            const int rc = launch_sbp_device(P, smem, n, (const OrbfeKeyPoint *)(D + o_kps), D + o_desc, (const int *)(D + o_cnt),
                                             (const int *)(D + o_ci) + k0, (const int *)(D + o_li) + k0, (const float *)(D + o_world),
                                             D + o_flags, (const float *)(D + o_T) + (size_t)k0 * 12, m->scratch,
                                             (int *)(D + o_mp) + (size_t)k0 * cap, (int *)(D + o_nm) + k0, m->d_err, m->hs.stream);
            if (int e = sbp_launched(m, rc)) return e;
        }
        return ORBFE_OK;
    };
    if (int rc = run_staged(m, o_mp, o_nm, total, (size_t)64 * cap, pack_mp, launch)) return rc;
    const int *h_nm = (const int *)(H + o_nm);
    for (int k = 0; k < npairs; k++) {
        const int j = order[k];
        if (cur[j].n) memcpy(cur_mp_inout[j], H + o_mp + (size_t)k * cap * sizeof(int), (size_t)cur[j].n * sizeof(int));
        nmatches_out[j] = h_nm[k];
    }
    return ORBFE_OK;
}

// the most queries (at most nq, at least 1) that one guided job over `cap` features holds in sbp_prepare's shared memory
static int sbp_fit_qcap(int cap, int nq) {
    int lo = 1, hi = nq;
    while (lo < hi) {
        const int mid = lo + (hi - lo + 1) / 2;
        if (sbp_smem_fixed_bytes(cap, mid) + 16 * 1024 <= kSbpSmemMax) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// Guided search of `nq` query windows in frame f: one job, cap = f.n.  Without the rotation histogram, a call whose queries
// do not fit one launch runs them in consecutive chunks, launched in order on the matcher's stream against the same slot
// array: under rules 0-2 query q's outcome depends only on the slots earlier queries took, under SBP_RULE_BEST on nothing
// else, so the chunks give the one-launch result.  The histogram spans the whole call, so with it the call must fit one launch.
int orbfe::guided_host(OrbfeMatcher *m, const OrbfeFrameView &f, int nq, const GuidedQuery *Q, int rule, float nnratio, int th_dist,
                       int check_orientation, int *slot_owner, int *best_out, int *nmatches_out) {
    *nmatches_out = 0;
    if (best_out) std::fill(best_out, best_out + nq, -1);
    if (f.n == 0 || nq == 0) return ORBFE_OK;   // no candidates: nothing is matched, the slots stay as they are
    const int cap = f.n;
    const int qcap = check_orientation ? nq : sbp_fit_qcap(cap, nq);   // queries per launch
    const int nchunks = (nq + qcap - 1) / qcap;
    ORBFE_CUDA_TRY(cudaSetDevice(m->device));
    size_t o_kps, o_desc, o_cnt, o_fi, o_qb, o_qc, o_qu, o_qv, o_qr, o_qa, o_lo, o_hi, o_qd, o_mp, o_nm, o_best, total;
    const size_t nc4 = (size_t)nchunks * sizeof(int);
    if (int rc = m->stage.layout({{&o_kps, (size_t)cap * sizeof(OrbfeKeyPoint)}, {&o_desc, (size_t)cap * 32}, {&o_cnt, sizeof(int)},
                                  {&o_fi, sizeof(int)}, {&o_qb, nc4}, {&o_qc, nc4}, {&o_qu, (size_t)nq * 4},
                                  {&o_qv, (size_t)nq * 4}, {&o_qr, (size_t)nq * 4}, {&o_qa, (size_t)nq * 4}, {&o_lo, (size_t)nq * 4},
                                  {&o_hi, (size_t)nq * 4}, {&o_qd, (size_t)nq * 32}, {&o_mp, (size_t)cap * sizeof(int)},
                                  {&o_nm, nc4}, {&o_best, best_out ? (size_t)nq * sizeof(int) : 0}},
                              &total))
        return rc;
    unsigned char *H = m->stage.h, *D = m->stage.d;
    memcpy(H + o_kps, f.keys_un, (size_t)cap * sizeof(OrbfeKeyPoint));
    memcpy(H + o_desc, f.desc, (size_t)cap * 32);
    *(int *)(H + o_cnt) = cap; *(int *)(H + o_fi) = 0;
    for (int c = 0; c < nchunks; c++) {
        ((int *)(H + o_qb))[c] = c * qcap;
        ((int *)(H + o_qc))[c] = std::min(qcap, nq - c * qcap);
    }
    float *qu = (float *)(H + o_qu), *qv = (float *)(H + o_qv), *qr = (float *)(H + o_qr), *qa = (float *)(H + o_qa);
    int *lo = (int *)(H + o_lo), *hi = (int *)(H + o_hi);
    for (int q = 0; q < nq; q++) {
        qu[q] = Q[q].u; qv[q] = Q[q].v; qr[q] = Q[q].r; qa[q] = Q[q].angle; lo[q] = Q[q].lo; hi[q] = Q[q].hi;
        memcpy(H + o_qd + (size_t)q * 32, Q[q].desc, 32);
    }
    auto pack_slots = [&]() {
        if (slot_owner) memcpy(H + o_mp, slot_owner, (size_t)cap * sizeof(int));
        else memset(H + o_mp, 0xFF, (size_t)cap * sizeof(int));   // every slot free
    };
    auto launch = [&](size_t per_job) -> int {
        SbpParams P;
        memset(&P, 0, sizeof(P));
        P.nlevels = 1; P.check_ori = check_orientation ? 1 : 0;
        P.rule = rule; P.th_dist = th_dist; P.nnratio = nnratio;
        size_t smem;
        if (int rc = sbp_prepare(m, P, f.min_x, f.min_y, f.max_x, f.max_y, cap, qcap, 1, per_job, &smem)) return rc;
        P.gw = f.grid_inv_w; P.gh = f.grid_inv_h;
        for (int c = 0; c < nchunks; c++) {
            P.owner_base = c * qcap;   // the slots receive call-wide query indices
            const int rc = launch_guided_device(P, smem, 1, (const OrbfeKeyPoint *)(D + o_kps), D + o_desc, (const int *)(D + o_cnt),
                                                (const int *)(D + o_fi), (const float *)(D + o_qu), (const float *)(D + o_qv),
                                                (const float *)(D + o_qr), (const int *)(D + o_lo), (const int *)(D + o_hi), D + o_qd,
                                                (const float *)(D + o_qa), (const int *)(D + o_qb) + c, (const int *)(D + o_qc) + c,
                                                m->scratch, (int *)(D + o_mp), best_out ? (int *)(D + o_best) : nullptr,
                                                (int *)(D + o_nm) + c, m->d_err, m->hs.stream);
            if (int e = sbp_launched(m, rc)) return e;
        }
        return ORBFE_OK;
    };
    if (int rc = run_staged(m, o_mp, o_nm, total, (size_t)64 * std::max(cap, qcap), pack_slots, launch)) return rc;
    // the kernel leaves occupied slots as they were and writes the query index into the slots it matched
    const int *mp = (const int *)(H + o_mp);
    if (slot_owner)
        for (int i = 0; i < cap; i++)
            if (slot_owner[i] < 0 && mp[i] >= 0) slot_owner[i] = Q[mp[i]].owner;
    if (best_out) memcpy(best_out, H + o_best, (size_t)nq * sizeof(int));
    for (int c = 0; c < nchunks; c++) *nmatches_out += ((const int *)(H + o_nm))[c];
    return ORBFE_OK;
}

// SearchForInitialization: F1 and F2 staged as a two-frame store (frame 0 = F1, frame 1 = F2), one MODE 2 pair.
int orbfe::init_host(OrbfeMatcher *m, const OrbfeFrameView &f1, const OrbfeFrameView &f2, float *prev_matched, int window,
                     float nnratio, int check_orientation, int *match12_out, int *nmatches_out) {
    const int cap = std::max({f1.n, f2.n, 1});
    const size_t C = (size_t)cap;
    ORBFE_CUDA_TRY(cudaSetDevice(m->device));
    size_t o_kps, o_desc, o_cnt, o_idx, o_prev, o_m12, o_nm, total;
    if (int rc = m->stage.layout({{&o_kps, 2 * C * sizeof(OrbfeKeyPoint)}, {&o_desc, 2 * C * 32}, {&o_cnt, 2 * sizeof(int)},
                                  {&o_idx, 2 * sizeof(int)}, {&o_prev, C * 2 * sizeof(float)}, {&o_m12, C * sizeof(int)},
                                  {&o_nm, sizeof(int)}},
                              &total))
        return rc;
    unsigned char *H = m->stage.h, *D = m->stage.d;
    const OrbfeFrameView *v[2] = {&f1, &f2};
    for (int f = 0; f < 2; f++) {
        ((int *)(H + o_cnt))[f] = v[f]->n;
        ((int *)(H + o_idx))[f] = f;
        if (!v[f]->n) continue;
        memcpy(H + o_kps + f * C * sizeof(OrbfeKeyPoint), v[f]->keys_un, (size_t)v[f]->n * sizeof(OrbfeKeyPoint));
        memcpy(H + o_desc + f * C * 32, v[f]->desc, (size_t)v[f]->n * 32);
    }
    auto pack_prev = [&]() { if (f1.n) memcpy(H + o_prev, prev_matched, (size_t)f1.n * 2 * sizeof(float)); };
    auto launch = [&](size_t per_pair) {
        SbpParams P = init_params(window, nnratio, check_orientation);
        size_t smem;
        if (int rc = sbp_prepare(m, P, f2.min_x, f2.min_y, f2.max_x, f2.max_y, cap, cap, 1, per_pair, &smem)) return rc;
        P.gw = f2.grid_inv_w; P.gh = f2.grid_inv_h;
        const int *d_idx = (const int *)(D + o_idx);
        return sbp_launched(m, launch_init_device(P, smem, 1, (const OrbfeKeyPoint *)(D + o_kps), D + o_desc, (const int *)(D + o_cnt),
                                                  d_idx, d_idx + 1, (float *)(D + o_prev), m->scratch, (int *)(D + o_m12),
                                                  (int *)(D + o_nm), m->d_err, m->hs.stream));
    };
    if (int rc = run_staged(m, o_prev, o_m12, total, init_scratch_per_pair(cap), pack_prev, launch)) return rc;
    if (f1.n) {
        memcpy(prev_matched, H + o_prev, (size_t)f1.n * 2 * sizeof(float));
        memcpy(match12_out, H + o_m12, (size_t)f1.n * sizeof(int));
    }
    *nmatches_out = *(const int *)(H + o_nm);
    return ORBFE_OK;
}
