// extract_kernels.cu -- hand-written sm_90a kernels of the ORB extractor hot path.
//
// Stage map (reference src/ORBextractor.cc; canonical algorithm = SURVEY.md Appendix A):
//   resize_level_kernel   ComputePyramid: cv::resize INTER_LINEAR u8 (:800), integer fixed point
//   fast_nms_kernel       cv::FAST per cell (:599-614) as ONE threshold-free score map + windowed NMS
//   cell_quota_kernel     per-cell quota redistribution (:622-670)
//   cell_select_kernel    per-cell retainBest (:683-685) as an exact radix select on unique keys
//   level_select_kernel   level-wide retainBest (:697-701) + canonical ordering
//   blur7_kernel          cv::GaussianBlur 7x7 sigma 2 (:760), OpenCV-2.4 integer engine
//   describe_kernel       IC_Angle (:124-151) + computeOrbDescriptor (:155-194) + output packing (:768-777)
//
// All pixel arithmetic is integer; floats appear only in IC_Angle's atan2 polynomial, the BRIEF
// rotation and the coordinate rescale, each written with explicit round-to-nearest intrinsics
// (no FMA contraction).  No tensor cores: there is no dense contraction on this path.
#include <cuda_fp16.h>

#include "orbfe_internal.h"

namespace orbfe {

__global__ void cell_select_harris_kernel(const PlanDev *__restrict__ plan, WorkDev wk, int f0);
__global__ void level_select_harris_kernel(const PlanDev *__restrict__ plan, WorkDev wk, int f0);

__device__ __forceinline__ int find_level_by(const PlanDev *plan, int idx, int which) {
    // which: 0 = ftile_base, 1 = btile_base, 2 = cell_base, 3 = kp_base
    int l = 0;
    const int n = plan->nlevels;
    for (int k = 1; k < n; k++) {
        const LevelDev &L = plan->lv[k];
        const int base = which == 0 ? L.ftile_base : which == 1 ? L.btile_base : which == 2 ? L.cell_base : L.kp_base;
        // levels with zero extent share a base with their successor: the LAST level whose base <= idx wins
        if (idx >= base) l = k;
    }
    return l;
}

// ------------------------------------------------------------------------------------------------
// Programmatic dependent launch (sm_90+): every kernel of the pipeline opens with
//     griddepcontrol.launch_dependents   -- the NEXT kernel in the stream may be launched as soon as all CTAs of this one run
//     griddepcontrol.wait                -- ... and this one touches nothing a predecessor wrote until that grid has completed
// and is launched with cudaLaunchAttributeProgrammaticStreamSerialization, so that the launch latency and prologue of kernel
// n+1 overlap the tail of kernel n.  It matters for the small batches of the reference's own call shape (one frame per call:
// twelve launches of 5-30 us); with ORBFE_PDL=0 (or for kernels launched without the attribute) both instructions are no-ops.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_prologue() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
}

template <typename... P, typename... A>
static inline void launch_k(void (*kern)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, bool pdl, A... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kern, static_cast<P>(args)...);
}

// ------------------------------------------------------------------------------------------------
// Pyramid: level l from level l-1.  One thread = 4 adjacent destination pixels (one uchar4 store).
// Horizontal/vertical tap tables were computed on the host exactly as OpenCV computes them, so the
// device part is pure integer: r = S[x0]*a0 + S[x1]*a1 ; v = (((b0*(r0>>4))>>16) + ((b1*(r1>>4))>>16) + 2) >> 2.
// ------------------------------------------------------------------------------------------------
#define RZ_ROWS 4  // destination rows per thread (the horizontal taps are loaded once and reused)

__global__ void __launch_bounds__(256) resize_level_kernel(const PlanDev *__restrict__ plan, int level, int f0) {
    pdl_prologue();
    const LevelDev &D = plan->lv[level];
    const LevelDev &S = plan->lv[level - 1];
    const int f = blockIdx.z + f0;
    const int ybase = (blockIdx.y * blockDim.y + threadIdx.y) * RZ_ROWS;
    const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int dw = D.w, dh = D.h;
    if (ybase >= dh || x4 >= dw) return;
    // taps of the thread's 4 destination columns (tables are padded to a multiple of 4 entries)
    const int4 xo = __ldg(reinterpret_cast<const int4 *>(D.xofs + x4));
    const uint4 ab = __ldg(reinterpret_cast<const uint4 *>(D.xab + x4));  // (a0 | a1 << 16) per column
    // the 4 source columns and their right neighbours lie within 9 bytes of sbase: three aligned words
    const int sbase = xo.x & ~3;
    const int o0 = xo.x - sbase, o1 = xo.y - sbase, o2 = xo.z - sbase, o3 = xo.w - sbase;
    const uint8_t *__restrict__ src = S.pyr + (size_t)f * S.plane + sbase;
    uint8_t *__restrict__ dst = D.pyr + (size_t)f * D.plane + x4;
    const int spitch = S.pitch;
    if (!D.rz_fast) {
        // generic path (scale factors > 4/3: the four source columns do not fit three words): byte loads
        const uint8_t *__restrict__ sb = S.pyr + (size_t)f * S.plane;
        const int xs[4] = {xo.x, xo.y, xo.z, xo.w};
        const uint32_t as[4] = {ab.x, ab.y, ab.z, ab.w};
        for (int ry = 0; ry < RZ_ROWS; ry++) {
            const int y = ybase + ry;
            if (y >= dh) break;
            const int2 rr = __ldg(&D.yrows[y]);
            const short2 bb = __ldg(&D.yab[y]);
            const uint8_t *s0 = sb + (size_t)rr.x * spitch, *s1 = sb + (size_t)rr.y * spitch;
            uint32_t out = 0;
            for (int i = 0; i < 4; i++) {
                const int a0 = (int)(as[i] & 0xFFFF), a1 = (int)(as[i] >> 16);
                const int xn = min(xs[i] + 1, S.w - 1);   // the right tap of the last column has weight 0: keep its address inside the row
                const int r0 = (int)__ldg(s0 + xs[i]) * a0 + (int)__ldg(s0 + xn) * a1;
                const int r1 = (int)__ldg(s1 + xs[i]) * a0 + (int)__ldg(s1 + xn) * a1;
                int v = ((((int)bb.x * (r0 >> 4)) >> 16) + (((int)bb.y * (r1 >> 4)) >> 16) + 2) >> 2;
                out |= (uint32_t)min(max(v, 0), 255) << (8 * i);
            }
            *reinterpret_cast<uint32_t *>(dst + (size_t)y * D.pitch) = out;
        }
        return;
    }
    const bool lo3 = D.rz_fast == 2;
    const uint32_t sel0 = (uint32_t)(o0 | ((o0 + 1) << 4)), sel1 = (uint32_t)(o1 | ((o1 + 1) << 4)), sel2 = (uint32_t)(o2 | ((o2 + 1) << 4));
    // all table loads, then all 24 pixel-word loads, then the arithmetic: the loads of the four rows are independent
    // and in flight together (rows past the bottom edge are clamped for the loads and skipped at the store)
    int2 rr[RZ_ROWS];
    short2 bb[RZ_ROWS];
#pragma unroll
    for (int ry = 0; ry < RZ_ROWS; ry++) {
        const int y = min(ybase + ry, dh - 1);
        rr[ry] = __ldg(&D.yrows[y]);
        bb[ry] = __ldg(&D.yab[y]);
    }
    // the three words may reach past the last pixel of the row (those bytes only meet zero weights); when level 0 is the
    // caller's buffer there is no slack behind the last row: keep the word addresses inside the row
    const int wlim = max((spitch - 4 - sbase) >> 2, 0);
    const int w1 = min(1, wlim), w2 = min(2, wlim);
    uint32_t u[RZ_ROWS][3], v[RZ_ROWS][3];
#pragma unroll
    for (int ry = 0; ry < RZ_ROWS; ry++) {
        const uint32_t *p0 = reinterpret_cast<const uint32_t *>(src + (size_t)rr[ry].x * spitch);
        const uint32_t *p1 = reinterpret_cast<const uint32_t *>(src + (size_t)rr[ry].y * spitch);
        u[ry][0] = __ldg(p0); u[ry][1] = __ldg(p0 + w1); u[ry][2] = __ldg(p0 + w2);
        v[ry][0] = __ldg(p1); v[ry][1] = __ldg(p1 + w1); v[ry][2] = __ldg(p1 + w2);
    }
#pragma unroll
    for (int ry = 0; ry < RZ_ROWS; ry++) {
        const int y = ybase + ry;
        const uint32_t u0 = u[ry][0], u1 = u[ry][1], u2 = u[ry][2], v0 = v[ry][0], v1 = v[ry][1], v2 = v[ry][2];
        const int b0 = bb[ry].x, b1 = bb[ry].y;
        uint32_t out = 0;
        // bytes S[s], S[s+1] of a column that starts o bytes into (u0 u1 u2).  With rz_fast == 2 the first three
        // columns of every quad start within 6 bytes: one PRMT on (u0,u1) with a per-thread selector; otherwise a
        // word select + funnel shift.  The weighted sum is <= 255 by construction (weights sum to 2048): no clamp.
#define RZ_MIX(i, pu, pv, abv)                                                                              \
        {                                                                                                   \
            const int r0 = (int)__dp2a_lo((abv), (pu), 0u);  /* S[s]*a0 + S[s+1]*a1 */                      \
            const int r1 = (int)__dp2a_lo((abv), (pv), 0u);                                                 \
            const int q = (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2;                   \
            out |= (uint32_t)q << (8 * (i));                                                                \
        }
#define RZ_PIX_SEL(i, o, abv)                                                                               \
        {                                                                                                   \
            const int sh = 8 * ((o) & 3);                                                                   \
            const bool hiw = (o) >= 4;                                                                      \
            RZ_MIX(i, __funnelshift_r(hiw ? u1 : u0, hiw ? u2 : u1, sh), __funnelshift_r(hiw ? v1 : v0, hiw ? v2 : v1, sh), abv) \
        }
#define RZ_PIX_LO(i, sel, abv) RZ_MIX(i, __byte_perm(u0, u1, (sel)), __byte_perm(v0, v1, (sel)), abv)
        if (lo3) {
            RZ_PIX_LO(0, sel0, ab.x)
            RZ_PIX_LO(1, sel1, ab.y)
            RZ_PIX_LO(2, sel2, ab.z)
        } else {
            RZ_PIX_SEL(0, o0, ab.x)
            RZ_PIX_SEL(1, o1, ab.y)
            RZ_PIX_SEL(2, o2, ab.z)
        }
        RZ_PIX_SEL(3, o3, ab.w)
#undef RZ_PIX_LO
#undef RZ_PIX_SEL
#undef RZ_MIX
        // pitch is a multiple of 128 and x4 a multiple of 4: aligned 32-bit store (bytes beyond w land in row padding)
        if (y < dh) *reinterpret_cast<uint32_t *>(dst + (size_t)y * D.pitch) = out;
    }
}

void launch_resize_level(const PlanDev *d_plan, const PlanDev &hp, int level, int f0, int nf, cudaStream_t s) {
    const LevelDev &D = hp.lv[level];
    dim3 block(64, 4);
    dim3 grid((D.w + 255) / 256, (D.h + 4 * RZ_ROWS - 1) / (4 * RZ_ROWS), nf);
    launch_k(resize_level_kernel, grid, block, 0, s, hp.pdl != 0, d_plan, level, f0);
}

// ------------------------------------------------------------------------------------------------
// FAST-9/16 score map + windowed 3x3 NMS + candidate emission.
//
// m(p) = max over the 16 contiguous 9-arcs of min(ring - v) and of min(v - ring)  (clamped at 0).
// p is a FAST corner at threshold t  <=>  m > t ; OpenCV's score = m - 1 (threshold independent).
// NMS: strict maximum over the 8 neighbours that lie inside the same cell's detect window
// (cv::FAST ran on the cell image, so it never saw the neighbouring cell; :599-607).
// Because any neighbour that is not a corner at t has m' <= t < m, the NMS outcome does not depend
// on t: one pass emits every local maximum with m > min(fastTh,7) and the per-cell threshold
// (fastTh, or 7 when fastTh yields <= 3 keypoints, :609-614) is applied later as a key threshold.
// ------------------------------------------------------------------------------------------------
// Geometry of one CTA: detect tile 120 x 62 px.  m is needed on a 1-px apron (122 x 64); it is computed for
// 32 column groups of 4 px (x0-4 .. x0+123) x 64 rows (y0-1 .. y0+62): lane = column group, warp = 8-row
// segment.  Each thread slides a 7-row register window down its 4-px column: per new row 3 LDS.32 + 10 PRMT
// build the eight packed pixel pairs P_j = (b_j, b_{j+2}) as u16x2; every ring pixel of the two pixel pairs
// A = (x, x+2) and B = (x+1, x+3) is then one of those registers, and the 16 arc minima / maxima are
// VIMNMX3.U16x2 (two pixels per instruction, no divergence):
//     t_k = min3(r_k, r_k+1, r_k+2) ; w_k = min3(t_k, t_k+3, t_k+6) = min of the 9-arc starting at k
//     m   = max( max_k w_k - v , v - min_k W_k , 0 )          (W_k likewise with max3)
#define F2_W ORBFE_FT_W            // 120
#define F2_H ORBFE_FT_H            // 62
#define F2_PW 144                  // staged pixel row stride (bytes): cols x0-8 .. x0+135
#define F2_PWORDS 35               // words actually loaded per row (x0-8 .. x0+131)
#define F2_PH (F2_H + 8)           // 70 staged rows: y0-4 .. y0+65
#define F2_MS 128                  // m tile row stride (32 groups x 4)
#ifndef ORBFE_FAST_ARC_DEFAULT
#define ORBFE_FAST_ARC_DEFAULT 12   // arc-network variant of the non-TMA kernel (fast_m_arc): second form, 12 (min, max) pairs on the FMA pipe
#endif
#define F2_MH (F2_H + 2)           // 64 m rows

__device__ __forceinline__ uint32_t max16_u16x2(const uint32_t *w) {
    const uint32_t a0 = __vimax3_u16x2(w[0], w[1], w[2]), a1 = __vimax3_u16x2(w[3], w[4], w[5]);
    const uint32_t a2 = __vimax3_u16x2(w[6], w[7], w[8]), a3 = __vimax3_u16x2(w[9], w[10], w[11]);
    const uint32_t a4 = __vimax3_u16x2(w[12], w[13], w[14]);
    return __vmaxu2(__vimax3_u16x2(a0, a1, a2), __vimax3_u16x2(a3, a4, w[15]));
}
__device__ __forceinline__ uint32_t min16_u16x2(const uint32_t *w) {
    const uint32_t a0 = __vimin3_u16x2(w[0], w[1], w[2]), a1 = __vimin3_u16x2(w[3], w[4], w[5]);
    const uint32_t a2 = __vimin3_u16x2(w[6], w[7], w[8]), a3 = __vimin3_u16x2(w[9], w[10], w[11]);
    const uint32_t a4 = __vimin3_u16x2(w[12], w[13], w[14]);
    return __vminu2(__vimin3_u16x2(a0, a1, a2), __vimin3_u16x2(a3, a4, w[15]));
}

// r[16]: ring pixels (two pixels per register, values 0..255 in each 16-bit half), c: the two centres
__device__ __forceinline__ uint32_t fast_m_u16x2(const uint32_t (&r)[16], uint32_t c) {
    uint32_t tmin[16], tmax[16], w[16];
#pragma unroll
    for (int k = 0; k < 16; k++) {
        tmin[k] = __vimin3_u16x2(r[k], r[(k + 1) & 15], r[(k + 2) & 15]);
        tmax[k] = __vimax3_u16x2(r[k], r[(k + 1) & 15], r[(k + 2) & 15]);
    }
#pragma unroll
    for (int k = 0; k < 16; k++) w[k] = __vimin3_u16x2(tmin[k], tmin[(k + 3) & 15], tmin[(k + 6) & 15]);
    const uint32_t mb = max16_u16x2(w);  // brightest guaranteed level of some 9-arc
#pragma unroll
    for (int k = 0; k < 16; k++) w[k] = __vimax3_u16x2(tmax[k], tmax[(k + 3) & 15], tmax[(k + 6) & 15]);
    const uint32_t md = min16_u16x2(w);  // darkest guaranteed level of some 9-arc
    const uint32_t bright = __vmaxu2(mb, c) - c;  // per half >= 0: no borrow across halves
    const uint32_t dark = c - __vminu2(md, c);
    return __vmaxu2(bright, dark);
}

// ---- arc network, second form (default).  For even k the two 9-arcs starting at k and k+1 share the 8 ring pixels
// k+1 .. k+8; with c_k their minimum,  max(min(c_k, r_k), min(c_k, r_k+9)) = min(c_k, max(r_k, r_k+9)), so
//     p_j  = min(r_2j+1, r_2j+2)              8 pair minima
//     pp_j = min(p_j, p_j+1)                  8 quad minima  (r_2j+1 .. r_2j+4)
//     e_i  = max(r_2i, r_2i+9)                8 arc-end maxima
//     v_i  = min3(pp_i, pp_i+2, e_i)          the better of arcs 2i and 2i+1
//     mb   = max(v_0 .. v_7, centre)          4 three-input maxima (the centre clamp rides in the tree)
// and the dual for the dark arcs: 36 operations per polarity instead of 40.  NPAIR of the 16 (min, max) pairs
// (p_j / P_j and e_i / E_i take the minimum AND the maximum of the same two registers) are computed on the FMA pipe
// instead of the integer ALU pipe the rest of the kernel saturates: pixel values 0..255 in a 16-bit half are fp16
// subnormals, on which HFMA2 is exact, so  t = relu(a - b), min = a - t, max = b + t  is three FMA-pipe
// instructions per pair, bit-identical to VIMNMX.U16x2.
__device__ __forceinline__ uint32_t hfma2_relu(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d;
    asm("fma.rn.relu.f16x2 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
__device__ __forceinline__ uint32_t hfma2(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d;
    asm("fma.rn.f16x2 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
// fma_pipe is a compile-time constant at every call site once the callers' loops are unrolled
__device__ __forceinline__ void minmax_u16x2(bool fma_pipe, uint32_t a, uint32_t b, uint32_t &mn, uint32_t &mx) {
    if (fma_pipe) {
        const uint32_t NEG1 = 0xBC00BC00u, ONE = 0x3C003C00u;
        const uint32_t t = hfma2_relu(b, NEG1, a);   // relu(a - b)
        mn = hfma2(t, NEG1, a);                      // a - relu(a - b)
        mx = hfma2(t, ONE, b);                       // b + relu(a - b)
    } else {
        mn = __vminu2(a, b);
        mx = __vmaxu2(a, b);
    }
}
template <int NPAIR>
__device__ __forceinline__ uint32_t fast_m2_u16x2(const uint32_t (&r)[16], uint32_t c) {
    uint32_t p[8], P[8], e[8], E[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        // pairs are handed to the FMA pipe interleaved (p_0, e_0, p_1, e_1, ...) so that any NPAIR spreads over the network
        minmax_u16x2(2 * j < NPAIR, r[2 * j + 1], r[(2 * j + 2) & 15], p[j], P[j]);
        minmax_u16x2(2 * j + 1 < NPAIR, r[2 * j], r[(2 * j + 9) & 15], E[j], e[j]);
    }
    uint32_t pp[8], PP[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        pp[j] = __vminu2(p[j], p[(j + 1) & 7]);
        PP[j] = __vmaxu2(P[j], P[(j + 1) & 7]);
    }
    uint32_t v[8], V[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        v[i] = __vimin3_u16x2(pp[i], pp[(i + 2) & 7], e[i]);
        V[i] = __vimax3_u16x2(PP[i], PP[(i + 2) & 7], E[i]);
    }
    // mb >= c and md <= c by construction: the differences need no clamp and cannot borrow across halves
    const uint32_t mb = __vimax3_u16x2(__vimax3_u16x2(v[0], v[1], v[2]), __vimax3_u16x2(v[3], v[4], v[5]), __vimax3_u16x2(v[6], v[7], c));
    const uint32_t md = __vimin3_u16x2(__vimin3_u16x2(V[0], V[1], V[2]), __vimin3_u16x2(V[3], V[4], V[5]), __vimin3_u16x2(V[6], V[7], c));
    return __vmaxu2(mb - c, c - md);
}
// ARC < 0: the first form (16 triple minima + 16 nine-arc minima per polarity); ARC >= 0: the second form with ARC pairs on the FMA pipe
template <int ARC>
__device__ __forceinline__ uint32_t fast_m_arc(const uint32_t (&r)[16], uint32_t c) {
    if (ARC < 0) return fast_m_u16x2(r, c);
    return fast_m2_u16x2<(ARC < 0 ? 0 : ARC)>(r, c);
}

__device__ __forceinline__ void fast_load_row(const uint8_t *row /* smem, word aligned at the group's b0 */, uint32_t (&P)[8]) {
    const uint32_t w0 = *reinterpret_cast<const uint32_t *>(row);
    const uint32_t w1 = *reinterpret_cast<const uint32_t *>(row + 4);
    const uint32_t w2 = *reinterpret_cast<const uint32_t *>(row + 8);
    const uint32_t E0 = __byte_perm(w0, 0, 0x4240), O0 = __byte_perm(w0, 0, 0x4341);
    const uint32_t E1 = __byte_perm(w1, 0, 0x4240), O1 = __byte_perm(w1, 0, 0x4341);
    const uint32_t E2 = __byte_perm(w2, 0, 0x4240), O2 = __byte_perm(w2, 0, 0x4341);
    P[0] = O0;                             // P_1 = (b1, b3)
    P[1] = __byte_perm(E0, E1, 0x5412);    // P_2 = (b2, b4)
    P[2] = __byte_perm(O0, O1, 0x5412);    // P_3 = (b3, b5)
    P[3] = E1;                             // P_4 = (b4, b6)   centre of pair A
    P[4] = O1;                             // P_5 = (b5, b7)   centre of pair B
    P[5] = __byte_perm(E1, E2, 0x5412);    // P_6 = (b6, b8)
    P[6] = __byte_perm(O1, O2, 0x5412);    // P_7 = (b7, b9)
    P[7] = E2;                             // P_8 = (b8, b10)
}

// m tile in shared memory, u16x2 pairs exactly as produced: row r, group g -> [mA, mB] (8 bytes) with
// mA = (m[x], m[x+2]), mB = (m[x+1], m[x+3]), x = x0-4+4g.
__device__ __forceinline__ int m_at(const uint32_t *mt, int r, int c /* tile column, 0 <-> x0-4 */) {
    const int g = c >> 2, k = c & 3;
    const uint32_t wv = mt[(r * 32 + g) * 2 + (k & 1)];
    return (k & 2) ? (int)(wv >> 16) : (int)(wv & 0xFFFF);
}

// candidates per tile: strict 8-neighbour maxima (<= one per 2x2 block) + cell-boundary pixels of pass 2
#define F2_MAXC ((F2_W / 2) * (F2_H / 2) + 4 * (F2_W + F2_H))
#define F2_MAXCELLS 64                    // cells a tile can overlap (host-checked)

// monotonic map float -> u32 (larger float <=> larger key), for selection keys
__device__ __forceinline__ uint32_t float_order_key(float v) {
    const uint32_t b = __float_as_uint(v);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float float_from_order_key(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

// HarrisResponses for one keypoint (reference ORBextractor.cc:79-120, blockSize 7, k = 0.04): integer sums of the
// 3x3 Sobel-like gradients over the 7x7 block, then a*b - c*c - k*(a+b)^2 in binary32, every operation rounded
__device__ __forceinline__ float harris_response(const uint8_t *__restrict__ img, int pitch, int x, int y, float scale4) {
    int a = 0, b = 0, c = 0;
    for (int i = -3; i <= 3; i++) {
        const uint8_t *r0 = img + (size_t)(y + i - 1) * pitch + x, *r1 = r0 + pitch, *r2 = r1 + pitch;
        for (int j = -3; j <= 3; j++) {
            const int Ix = ((int)__ldg(r1 + j + 1) - (int)__ldg(r1 + j - 1)) * 2 + ((int)__ldg(r0 + j + 1) - (int)__ldg(r0 + j - 1)) +
                           ((int)__ldg(r2 + j + 1) - (int)__ldg(r2 + j - 1));
            const int Iy = ((int)__ldg(r2 + j) - (int)__ldg(r0 + j)) * 2 + ((int)__ldg(r2 + j - 1) - (int)__ldg(r0 + j - 1)) +
                           ((int)__ldg(r2 + j + 1) - (int)__ldg(r0 + j + 1));
            a += Ix * Ix;
            b += Iy * Iy;
            c += Ix * Iy;
        }
    }
    const float fa = (float)a, fb = (float)b, fc = (float)c;
    const float s = __fadd_rn(fa, fb);
    const float t = __fsub_rn(__fsub_rn(__fmul_rn(fa, fb), __fmul_rn(fc, fc)), __fmul_rn(__fmul_rn(0.04f, s), s));
    return __fmul_rn(t, scale4);
}

// candidate queue entry (u32): x - x0 (7 bits) | y - y0 (6 bits) << 7 | m (8 bits) << 13 | slot inside (tile, cell) (11 bits) << 21
__device__ __forceinline__ void fast_push(uint32_t *q, int *q_n, int xl, int yl, int m) {
    const int n = atomicAdd(q_n, 1);
    q[n] = (uint32_t)xl | ((uint32_t)yl << 7) | ((uint32_t)m << 13);
}

// cell of (x, y) and its detect window [xa, xb] x [ya, yb]  (ORBextractor.cc:560-599)
__device__ __forceinline__ void cell_window(const LevelDev &L, int xmax, int ymax, int x, int y, int &ci, int &cj, int &xa,
                                            int &xb, int &ya, int &yb) {
    // x, y >= 16 here; division by the cell size as a multiply-high with the host-computed reciprocal (exact below 2^16)
    cj = min((int)__umulhi((uint32_t)(x - ORBFE_EDGE), L.cw_rcp), L.cols - 1);
    ci = min((int)__umulhi((uint32_t)(y - ORBFE_EDGE), L.ch_rcp), L.rows - 1);
    xa = ORBFE_EDGE + cj * L.cw;
    ya = ORBFE_EDGE + ci * L.ch;
    xb = (cj == L.cols - 1) ? xmax - 1 : xa + L.cw - 1;
    yb = (ci == L.rows - 1) ? ymax - 1 : ya + L.ch - 1;
}

// Everything after the pixel tile is staged: m map, NMS passes, candidate conversion and flush.
// pix: staged pixel rows (stride F2_PW); mt: 16 KB m tile; s_cand: candidate list (F2_MAXC entries).
template <int PSTRIDE, int ARC>
__device__ __forceinline__ void fast_tile_compute(const PlanDev *__restrict__ plan, const WorkDev &wk, const LevelDev &L,
                                                  const FTileInfo &ti, int f, int x0, int y0, const uint8_t *pix, uint32_t *mt,
                                                  uint32_t *s_cand, int &s_n, int *s_cnt_lo, int *s_cnt_hi, int *s_base) {
    const int w = L.w, h = L.h;
    const int tlo = plan->t_lo;
    const int xmax = w - ORBFE_EDGE, ymax = h - ORBFE_EDGE;  // detect area is [16, xmax) x [16, ymax)
    const int g = threadIdx.x & 31, seg = threadIdx.x >> 5;
    const int gx = x0 - 4 + 4 * g;  // image x of the group's first pixel
    // ---- m for 32 groups x 64 rows; lane = group, warp = 8-row segment ----
    {
        // halves of (mA, mB) that lie inside the detect area: A = (gx, gx+2), B = (gx+1, gx+3)
        uint32_t maskA = 0, maskB = 0;
        if (gx >= ORBFE_EDGE && gx < xmax) maskA |= 0x0000FFFFu;
        if (gx + 2 >= ORBFE_EDGE && gx + 2 < xmax) maskA |= 0xFFFF0000u;
        if (gx + 1 >= ORBFE_EDGE && gx + 1 < xmax) maskB |= 0x0000FFFFu;
        if (gx + 3 >= ORBFE_EDGE && gx + 3 < xmax) maskB |= 0xFFFF0000u;
        const uint8_t *base = &pix[(seg * 8) * PSTRIDE + 4 * g];  // b0 of the group = tile col 4g  (image x gx-4)
        uint32_t P[7][8];
#pragma unroll
        for (int r = 0; r < 6; r++) fast_load_row(base + r * PSTRIDE, P[r]);
#pragma unroll
        for (int i = 0; i < 8; i++) {
            fast_load_row(base + (6 + i) * PSTRIDE, P[(6 + i) % 7]);
#define FROW(dy) P[(i + (dy) + 3) % 7]
            // ring in circular order, (dx,dy): (0,3)(1,3)(2,2)(3,1)(3,0)(3,-1)(2,-2)(1,-3)(0,-3)(-1,-3)(-2,-2)(-3,-1)(-3,0)(-3,1)(-2,2)(-1,3)
            // pair A uses P_{4+dx} = index 3+dx ; pair B uses P_{5+dx} = index 4+dx
            uint32_t mA, mB;
            {
                const uint32_t r[16] = {FROW(3)[3], FROW(3)[4], FROW(2)[5], FROW(1)[6], FROW(0)[6], FROW(-1)[6], FROW(-2)[5], FROW(-3)[4],
                                        FROW(-3)[3], FROW(-3)[2], FROW(-2)[1], FROW(-1)[0], FROW(0)[0], FROW(1)[0], FROW(2)[1], FROW(3)[2]};
                mA = fast_m_arc<ARC>(r, FROW(0)[3]);
            }
            {
                const uint32_t r[16] = {FROW(3)[4], FROW(3)[5], FROW(2)[6], FROW(1)[7], FROW(0)[7], FROW(-1)[7], FROW(-2)[6], FROW(-3)[5],
                                        FROW(-3)[4], FROW(-3)[3], FROW(-2)[2], FROW(-1)[1], FROW(0)[1], FROW(1)[1], FROW(2)[2], FROW(3)[3]};
                mB = fast_m_arc<ARC>(r, FROW(0)[4]);
            }
#undef FROW
            const int mr = seg * 8 + i;
            const int y = y0 - 1 + mr;
            const bool yin = (y >= ORBFE_EDGE && y < ymax);
            uint2 o;
            o.x = yin ? (mA & maskA) : 0u;
            o.y = yin ? (mB & maskB) : 0u;
            *reinterpret_cast<uint2 *>(&mt[(mr * 32 + g) * 2]) = o;
        }
    }
    __syncthreads();

    const int thi = plan->t_hi;
    const uint32_t tlo2 = (uint32_t)tlo * 0x00010001u;
    // ---- windowed 3x3 NMS, two pixels per instruction.  A pixel only competes with the neighbours inside
    //      its own cell's detect window (cv::FAST ran per cell image): neighbour relations that cross an
    //      interior cell boundary are masked to 0 -- per-lane u16x2 masks for vertical boundaries (they kill
    //      the left/right/diagonal terms), per-row flags for horizontal ones (they kill the row above/below).
    //      Rows 1..62 and groups 1..30 are the detect tile.
    uint32_t fbits = 0;  // candidate flags of the lane's 4 pixels x 8 rows: bit 8k + r
    const int r0 = seg * 8;
    if (g >= 1 && g <= 30) {
        // relation (gx+d-1 <-> gx+d), d = 0..4, crosses a boundary at X = 16 + cj*cw  <=>  X == gx + d
        uint32_t mLA = 0xFFFFFFFFu, mRA = 0xFFFFFFFFu, mLB = 0xFFFFFFFFu, mRB = 0xFFFFFFFFu;
        for (int bnd = 0; bnd < ti.nv; bnd++) {
            const int d = ORBFE_EDGE + (ti.cj_lo + bnd) * L.cw - gx;
            if (d == 0) mLA &= 0xFFFF0000u;
            else if (d == 1) { mRA &= 0xFFFF0000u; mLB &= 0xFFFF0000u; }
            else if (d == 2) { mLA &= 0x0000FFFFu; mRB &= 0xFFFF0000u; }
            else if (d == 3) { mRA &= 0x0000FFFFu; mLB &= 0x0000FFFFu; }
            else if (d == 4) mRB &= 0x0000FFFFu;
        }
        // ti.hmask bit r: tile row r (image y0-1+r) is the top row of a cell (interior horizontal boundary above it)
        const unsigned long long hmask = ti.hmask;
        uint32_t A[3], B[3], lrA[3], lrB[3], fullA[3], fullB[3];
#pragma unroll
        for (int j = 0; j < 10; j++) {
            // load tile row r0 - 1 + j into slot j % 3
            const int rr = min(max(r0 - 1 + j, 0), F2_MH - 1);
            const uint32_t *rowp = &mt[(rr * 32 + g) * 2];
            const uint2 own = *reinterpret_cast<const uint2 *>(rowp);
            const uint32_t pB = rowp[-1], nA = rowp[2];
            const int sl = j % 3;
            A[sl] = own.x;
            B[sl] = own.y;
            const uint32_t leftA = __byte_perm(pB, own.y, 0x5432) & mLA;   // (m[x-1], m[x+1])
            const uint32_t rightB = __byte_perm(own.x, nA, 0x5432) & mRB;  // (m[x+2], m[x+4])
            lrA[sl] = __vmaxu2(leftA, own.y & mRA);
            fullA[sl] = __vmaxu2(lrA[sl], own.x);
            lrB[sl] = __vmaxu2(own.x & mLB, rightB);
            fullB[sl] = __vmaxu2(lrB[sl], own.y);
            if (j >= 2) {
                const int cr = r0 + j - 2;  // centre row (slot (j-1)%3), above = (j-2)%3, below = j%3
                const int c = (j - 1) % 3, u = (j - 2) % 3, d = j % 3;
                const bool no_up = (hmask >> cr) & 1ull, no_dn = (hmask >> (cr + 1)) & 1ull;
                const uint32_t upA = no_up ? 0u : fullA[u], dnA = no_dn ? 0u : fullA[d];
                const uint32_t upB = no_up ? 0u : fullB[u], dnB = no_dn ? 0u : fullB[d];
                // neighbour maximum, floored at t_lo: m must exceed both to be a candidate
                const uint32_t nbA = __vmaxu2(__vimax3_u16x2(upA, dnA, lrA[c]), tlo2);
                const uint32_t nbB = __vmaxu2(__vimax3_u16x2(upB, dnB, lrB[c]), tlo2);
                // m - nb + 0x7FFF per half (both < 0x8000: no borrow between halves): bit 15 set  <=>  m > nb
                const uint32_t tA = A[c] + 0x7FFF7FFFu - nbA;
                const uint32_t tB = B[c] + 0x7FFF7FFFu - nbB;
                // flag bytes of pixels k = 0..3 -> byte k, bit (row inside the segment); the (rare) candidates are
                // pushed after the loop, outside the unrolled code
                if (cr >= 1 && cr <= F2_H) fbits |= (__byte_perm(tA, tB, 0x7351) & 0x80808080u) >> (7 - (j - 2));
            }
        }
    }
    // warp-aggregated queue reservation (all 32 lanes; the halo lanes have no flags): one shared-memory atomic per
    // warp, then every lane writes its own candidates
    {
        {
            const int mine = __popc(fbits);
            int incl = mine;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, incl, o);
                if (g >= o) incl += v;
            }
            int wbase = 0;
            const int total = __shfl_sync(0xffffffffu, incl, 31);
            if (g == 31 && total) wbase = atomicAdd(&s_n, total);
            wbase = __shfl_sync(0xffffffffu, wbase, 31);
            int n = wbase + incl - mine;
            while (fbits) {
                const int b = __ffs(fbits) - 1;
                fbits &= fbits - 1;
                const int cr = r0 + (b & 7), k = b >> 3;
                s_cand[n++] = (uint32_t)(gx + k - x0) | ((uint32_t)(cr - 1) << 7) | ((uint32_t)m_at(mt, cr, 4 * g + k) << 13);
            }
        }
    }
    __syncthreads();
    // ---- per-(tile, cell) slots: each candidate takes a slot in its cell's local counter ----
    const int ncand = s_n;
    const int ncell_loc = ti.ncj * ti.nci;
    for (int i = threadIdx.x; i < ncand; i += blockDim.x) {
        const uint32_t q = s_cand[i];
        const int x = x0 + (int)(q & 127), y = y0 + (int)((q >> 7) & 63), m = (int)((q >> 13) & 255);
        int ci, cj, xa, xb, ya, yb;
        cell_window(L, xmax, ymax, x, y, ci, cj, xa, xb, ya, yb);
        const int lc = (ci - ti.ci0) * ti.ncj + (cj - ti.cj0);
        const int slot = atomicAdd(&s_cnt_lo[lc], 1);
        if (m > thi) atomicAdd(&s_cnt_hi[lc], 1);
        if (slot >= 2048) atomicExch(wk.err_flag, 3);  // 11-bit slot field (unreachable: <= 1860 maxima per tile)
        s_cand[i] = q | ((uint32_t)slot << 21);
    }
    // ---- flush: one global atomic per (tile, cell) reserves the range, then the keys are written ----
    __syncthreads();
    if ((int)threadIdx.x < ncell_loc) {
        const int lc = threadIdx.x;
        const int gcell = L.cell_base + (ti.ci0 + lc / ti.ncj) * L.cols + (ti.cj0 + lc % ti.ncj);
        const size_t fc = (size_t)f * plan->ncells_total + gcell;
        int base = 0;
        if (s_cnt_lo[lc] > 0) {
            base = atomicAdd(&wk.cell_cnt_lo[fc], s_cnt_lo[lc]);
            if (s_cnt_hi[lc] > 0) atomicAdd(&wk.cell_cnt_hi[fc], s_cnt_hi[lc]);
            if (base + s_cnt_lo[lc] > wk.cell_cand_cap[gcell]) atomicExch(wk.err_flag, 1);
        }
        s_base[lc] = base;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < ncand; i += blockDim.x) {
        const uint32_t q = s_cand[i];
        const int x = x0 + (int)(q & 127), y = y0 + (int)((q >> 7) & 63), m = (int)((q >> 13) & 255), slot = (int)(q >> 21);
        int ci, cj, xa, xb, ya, yb;
        cell_window(L, xmax, ymax, x, y, ci, cj, xa, xb, ya, yb);
        const int lc = (ci - ti.ci0) * ti.ncj + (cj - ti.cj0);
        const int gcell = L.cell_base + ci * L.cols + cj;
        const int pos = s_base[lc] + slot;
        const uint32_t raster = (uint32_t)((y - ya) * L.cw + (x - xa));
        if (pos < wk.cell_cand_cap[gcell]) {
            const size_t kidx = (size_t)f * plan->cand_total + wk.cell_cand_base[gcell] + pos;
            if (wk.cand_keys64) {
                // HARRIS_SCORE (:616-620): rank by the Harris response; the FAST score rides along for eligibility
                const float resp = harris_response(L.pyr + (size_t)f * L.plane, L.pitch, x, y, plan->harris_scale4);
                wk.cand_keys64[kidx] = ((unsigned long long)float_order_key(resp) << 32) |
                                       ((unsigned long long)(0xFFFFFFu - raster) << 8) | (unsigned long long)(m - 1);
            } else {
                wk.cand_keys[kidx] = ((uint32_t)(m - 1) << 24) | (0xFFFFFFu - raster);
            }
        }
    }
}

__global__ void __launch_bounds__(256, 2) fast_nms_kernel(const PlanDev *__restrict__ plan, WorkDev wk, int f0) {
    // one buffer, two lives: the staged pixel tile (until m is computed), then the candidate list
    __shared__ __align__(16) uint8_t sbuf[(F2_MAXC * 4 > F2_PH * F2_PW) ? F2_MAXC * 4 : F2_PH * F2_PW];
    __shared__ __align__(16) uint32_t mt[F2_MH * 32 * 2];  // 16 KB
    __shared__ int s_n, s_cnt_lo[F2_MAXCELLS], s_cnt_hi[F2_MAXCELLS], s_base[F2_MAXCELLS];
    uint8_t *pix = sbuf;
    uint32_t *s_cand = reinterpret_cast<uint32_t *>(sbuf);

    const int f = blockIdx.y + f0;
    const FTileInfo ti = wk.ftile_info[blockIdx.x];
    const LevelDev &L = plan->lv[ti.level];
    const int x0 = ORBFE_EDGE + ti.tx * F2_W, y0 = ORBFE_EDGE + ti.ty * F2_H;
    const int h = L.h, pitch = L.pitch;
    const uint8_t *__restrict__ img = L.pyr + (size_t)f * L.plane;

    if (threadIdx.x < F2_MAXCELLS) { s_cnt_lo[threadIdx.x] = 0; s_cnt_hi[threadIdx.x] = 0; }
    if (threadIdx.x == 0) s_n = 0;
    // ---- stage pixel rows y0-4 .. y0+65, cols x0-8 .. x0+131 (x0 is a multiple of 4) ----
    {
        const int max_word = pitch / 4 - 1;
        const int wx0 = (x0 - 8) >> 2;
        for (int i = threadIdx.x; i < F2_PH * F2_PWORDS; i += blockDim.x) {
            const int r = i / F2_PWORDS, c = i - r * F2_PWORDS;
            const int gy = min(y0 - 4 + r, h - 1);
            const int gw = min(wx0 + c, max_word);
            *reinterpret_cast<uint32_t *>(&pix[r * F2_PW + c * 4]) =
                __ldg(reinterpret_cast<const uint32_t *>(img + (size_t)gy * pitch) + gw);
        }
    }
    __syncthreads();
    fast_tile_compute<F2_PW, ORBFE_FAST_ARC_DEFAULT>(plan, wk, L, ti, f, x0, y0, pix, mt, s_cand, s_n, s_cnt_lo, s_cnt_hi, s_base);
}

// ------------------------------------------------------------------------------------------------
// TMA variant (default): persistent CTAs, the pixel tile of work item i+1 is fetched by the Tensor
// Memory Accelerator (cp.async.bulk.tensor.3d -> UTMALDG) into the second buffer while item i is
// being computed; completion is signalled on an mbarrier.  One 3-D tensor map (x, y, frame) per level;
// out-of-image parts of the box are zero-filled by the hardware (they only feed masked m positions).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void *smem_dst, const void *tmap, uint64_t *bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

// TMA needs the innermost box coordinate 16-byte aligned (measured: a misaligned start traps as an illegal
// instruction): the box starts at (x0-8) & ~15 and is 160 wide; the tile's own columns begin dx = (x0-8) & 15 in.
#define F2_TW 160
#define F2_PIXBYTES (F2_PH * F2_TW)                       // 11200 = TMA box 160 x 70 x 1
#define F2_PIXSLOT ((F2_PIXBYTES + 127) / 128 * 128)      // 11264
#define F2_TMA_SMEM (2 * F2_PIXSLOT + F2_MH * 32 * 2 * 4 + 128)
static_assert(F2_MAXC * 4 <= F2_PIXSLOT, "the candidate queue lives in the pixel slot that was just consumed");

template <int ARC, int MINB>
__global__ void __launch_bounds__(256, MINB) fast_nms_tma_kernel(const PlanDev *__restrict__ plan, WorkDev wk, int f0, int nwork) {
    extern __shared__ __align__(128) uint8_t dsm[];
    uint8_t *pixbuf0 = dsm, *pixbuf1 = dsm + F2_PIXSLOT;
    uint32_t *mt = reinterpret_cast<uint32_t *>(dsm + 2 * F2_PIXSLOT);
    __shared__ __align__(8) uint64_t bar[2];
    __shared__ int s_n, s_cnt_lo[F2_MAXCELLS], s_cnt_hi[F2_MAXCELLS], s_base[F2_MAXCELLS];

    const int ntiles = plan->nftiles_total;
    if (threadIdx.x == 0) {
        mbar_init(&bar[0], 1);
        mbar_init(&bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdl_prologue();   // the barriers above are private to the CTA; the first TMA load reads what the resize kernels wrote
    int wi = blockIdx.x;
    if (wi < nwork && threadIdx.x == 0) {
        const FTileInfo t0 = wk.ftile_info[wi % ntiles];
        mbar_expect_tx(&bar[0], F2_PIXBYTES);
        tma_load_3d(pixbuf0, &wk.tmaps[t0.level], &bar[0], (ORBFE_EDGE + t0.tx * F2_W - 8) & ~15, ORBFE_EDGE + t0.ty * F2_H - 4, f0 + wi / ntiles);
    }
    for (int it = 0; wi < nwork; it++, wi += gridDim.x) {
        const int cur = it & 1;
        const int nxt = wi + gridDim.x;
        if (nxt < nwork && threadIdx.x == 0) {  // prefetch the next tile into the other buffer
            const FTileInfo tn = wk.ftile_info[nxt % ntiles];
            mbar_expect_tx(&bar[cur ^ 1], F2_PIXBYTES);
            tma_load_3d(cur ? pixbuf0 : pixbuf1, &wk.tmaps[tn.level], &bar[cur ^ 1], (ORBFE_EDGE + tn.tx * F2_W - 8) & ~15,
                        ORBFE_EDGE + tn.ty * F2_H - 4, f0 + nxt / ntiles);
        }
        const FTileInfo ti = wk.ftile_info[wi % ntiles];
        const int f = f0 + wi / ntiles;
        const LevelDev &L = plan->lv[ti.level];
        const int x0 = ORBFE_EDGE + ti.tx * F2_W, y0 = ORBFE_EDGE + ti.ty * F2_H;
        if (threadIdx.x < F2_MAXCELLS) { s_cnt_lo[threadIdx.x] = 0; s_cnt_hi[threadIdx.x] = 0; }
        if (threadIdx.x == 0) s_n = 0;
        mbar_wait(&bar[cur], (it >> 1) & 1);
        __syncthreads();
        // the candidate queue reuses the current pixel slot (dead once m is computed; the next TMA into it is
        // only issued after the __syncthreads that ends this iteration)
        uint8_t *slot_cur = cur ? pixbuf1 : pixbuf0;
        fast_tile_compute<F2_TW, ARC>(plan, wk, L, ti, f, x0, y0, slot_cur + ((x0 - 8) & 15), mt, reinterpret_cast<uint32_t *>(slot_cur),
                                 s_n, s_cnt_lo, s_cnt_hi, s_base);
        __syncthreads();  // mt / s_cand / counters and the pixel buffer are reused by the next item
    }
}

// arc-network variants compiled in (WorkDev::fast_arc; ORBFE_FAST_ARC=n picks one, see orbfe_api.cu)
// (arc variant, resident CTAs per SM the register budget is sized for: 4 -> 64 registers, 3 -> 80)
#define FAST_ARC_VARIANTS(X) X(-1, 4) X(0, 4) X(4, 4) X(8, 4) X(12, 4) X(16, 4) X(12, 3) X(16, 3)
typedef void (*FastTmaKernel)(const PlanDev *, WorkDev, int, int);
static FastTmaKernel fast_tma_variant(int arc, int minb) {
#define X(a, b) if (arc == (a) && minb == (b)) return fast_nms_tma_kernel<(a), (b)>;
    FAST_ARC_VARIANTS(X)
#undef X
    return nullptr;
}
int fast_arc_supported(int arc, int ctas_per_sm) { return fast_tma_variant(arc, ctas_per_sm <= 3 ? 3 : 4) != nullptr; }

int fast_tma_setup() {
#define X(a, b) { cudaError_t e = cudaFuncSetAttribute(fast_nms_tma_kernel<(a), (b)>, cudaFuncAttributeMaxDynamicSharedMemorySize, F2_TMA_SMEM); if (e != cudaSuccess) return (int)e; }
    FAST_ARC_VARIANTS(X)
#undef X
    return 0;
}

void launch_fast_nms(const PlanDev *d_plan, const PlanDev &hp, WorkDev w, int f0, int nf, cudaStream_t s) {
    if (hp.nftiles_total == 0) return;  // every level has an empty cell grid: nothing to detect
    if (w.tmaps) {
        const int nwork = hp.nftiles_total * nf;
        const int grid = min(nwork, w.fast_grid);
        launch_k(fast_tma_variant(w.fast_arc, w.fast_ctas <= 3 ? 3 : 4), dim3(grid), dim3(256), F2_TMA_SMEM, s, hp.pdl != 0, d_plan, w, f0, nwork);
        return;
    }
    dim3 grid(hp.nftiles_total, nf);
    fast_nms_kernel<<<grid, 256, 0, s>>>(d_plan, w, f0);
}

// ------------------------------------------------------------------------------------------------
// Per-level quota redistribution (ORBextractor.cc:622-670).  One warp per (level, frame).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__global__ void __launch_bounds__(32) cell_quota_kernel(const PlanDev *__restrict__ plan, WorkDev wk, int f0) {
    pdl_prologue();
    __shared__ uint32_t no_more[128];  // bitmap, up to 4096 cells per level
    const int l = blockIdx.x, f = blockIdx.y + f0;
    const LevelDev &L = plan->lv[l];
    const int lane = threadIdx.x;
    const int nCells = L.ncells, nfc = L.nfc;
    const size_t fb = (size_t)f * plan->ncells_total + L.cell_base;
    const int t1_is_lo = plan->t1_is_lo;
    const int t1 = t1_is_lo ? plan->t_lo : plan->t_hi;  // fastTh
    const int t2 = t1_is_lo ? plan->t_hi : plan->t_lo;  // 7
    for (int i = lane; i < 128; i += 32) no_more[i] = 0;
    __syncwarp();

    int toDist = 0, nNoMore = 0;
    for (int c = lane; c < nCells; c += 32) {
        const int lo = wk.cell_cnt_lo[fb + c], hi = wk.cell_cnt_hi[fb + c];
        const int n1 = t1_is_lo ? lo : hi, n2 = t1_is_lo ? hi : lo;
        const bool fallback = n1 <= 3;  // :609
        const int nTotal = fallback ? n2 : n1;
        wk.cell_min_key[fb + c] = (uint32_t)(fallback ? t2 : t1) << 24;  // score = m-1 >= t  <=>  m > t
        // park nTotal in cell_cnt_lo? no: keep counts intact, recompute below
        int keep;
        if (nTotal > nfc) keep = nfc;
        else { keep = nTotal; toDist += nfc - nTotal; nNoMore++; atomicOr(&no_more[c >> 5], 1u << (c & 31)); }
        wk.cell_keep[fb + c] = keep;
    }
    toDist = warp_sum(toDist);
    nNoMore = warp_sum(nNoMore);
    __syncwarp();

    while (toDist > 0 && nNoMore < nCells) {
        const int nNew = nfc + (int)ceilf(__fdiv_rn((float)toDist, (float)(nCells - nNoMore)));  // :646
        int dist = 0, more = 0;
        for (int c = lane; c < nCells; c += 32) {
            if (no_more[c >> 5] & (1u << (c & 31))) continue;
            const int lo = wk.cell_cnt_lo[fb + c], hi = wk.cell_cnt_hi[fb + c];
            const int n1 = t1_is_lo ? lo : hi, n2 = t1_is_lo ? hi : lo;
            const int nTotal = (n1 <= 3) ? n2 : n1;
            if (nTotal > nNew) wk.cell_keep[fb + c] = nNew;
            else {
                wk.cell_keep[fb + c] = nTotal;
                dist += nNew - nTotal;
                more++;
                atomicOr(&no_more[c >> 5], 1u << (c & 31));
            }
        }
        toDist = warp_sum(dist);
        nNoMore += warp_sum(more);
        __syncwarp();
    }
}

void launch_cell_quota(const PlanDev *d_plan, const PlanDev &hp, WorkDev w, int f0, int nf, cudaStream_t s) {
    dim3 grid(hp.nlevels, nf);
    launch_k(cell_quota_kernel, grid, dim3(32), 0, s, hp.pdl != 0, d_plan, w, f0);
}

// ------------------------------------------------------------------------------------------------
// Per-cell retention: keep the `keep` largest keys among the eligible ones (key >= min_key).
// Keys are unique (score<<24 | inverted raster), so "top-n, ties at the cut broken by earlier raster
// position" (the canonical retainBest rule) is simply an exact n-th-largest-key radix select.
// Survivors are appended (order irrelevant) to the level's kept list as 64-bit selection keys
//   score(8) << 36 | (4095 - cell)(12) << 24 | (0xFFFFFF - raster)(24).
// ------------------------------------------------------------------------------------------------
#define CS_LIST 256   // candidates sharing the score at the cut that are ranked directly
__global__ void __launch_bounds__(128) cell_select_kernel(const PlanDev *__restrict__ plan, WorkDev wk, int f0) {
    pdl_prologue();
    __shared__ int hist[256];
    __shared__ uint32_t s_prefix, s_mask, s_list[CS_LIST];
    __shared__ int s_k, s_base, s_fill, s_bin_cnt, s_ln;

    const int gcell = blockIdx.x, f = blockIdx.y + f0;
    const size_t fc = (size_t)f * plan->ncells_total + gcell;
    const int keep = wk.cell_keep[fc];
    if (keep <= 0) return;
    const int l = find_level_by(plan, gcell, 2);
    const LevelDev &L = plan->lv[l];
    const int n = min(wk.cell_cnt_lo[fc], wk.cell_cand_cap[gcell]);
    const uint32_t min_key = wk.cell_min_key[fc];
    const uint32_t *__restrict__ keys = wk.cand_keys + (size_t)f * plan->cand_total + wk.cell_cand_base[gcell];
    const int tid = threadIdx.x;

    // number of eligible candidates
    const int lo = wk.cell_cnt_lo[fc], hi = wk.cell_cnt_hi[fc];
    const int n1 = plan->t1_is_lo ? lo : hi, n2 = plan->t1_is_lo ? hi : lo;
    const int n_elig = (n1 <= 3) ? n2 : n1;

    uint32_t cut = min_key;
    if (n_elig > keep) {
        if (tid == 0) { s_prefix = 0; s_mask = 0; s_k = keep; }
        for (int shift = 24; shift >= 0; shift -= 8) {
            for (int i = tid; i < 256; i += blockDim.x) hist[i] = 0;
            __syncthreads();
            const uint32_t prefix = s_prefix, mask = s_mask;
            for (int i = tid; i < n; i += blockDim.x) {
                const uint32_t k = keys[i];
                if (k >= min_key && (k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 0xFF], 1);
            }
            __syncthreads();
            if (tid < 32) {
                // bin of the k-th largest: warp 0 walks the 256 bins from the top, 8 bins per lane (lane 0 = bins 255..248)
                const int k = s_k;
                int hb[8], sum = 0;
#pragma unroll
                for (int t = 0; t < 8; t++) { hb[t] = hist[255 - 8 * tid - t]; sum += hb[t]; }
                int incl = sum;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int v = __shfl_up_sync(0xffffffffu, incl, o);
                    if (tid >= o) incl += v;
                }
                const int fl = __ffs(__ballot_sync(0xffffffffu, incl >= k)) - 1;  // the bins are known to hold >= k keys
                if (tid == fl) {
                    int cum = incl - sum, b = 255 - 8 * tid, t = 0;
#pragma unroll
                    for (; t < 8; t++) {
                        if (cum + hb[t] >= k) break;
                        cum += hb[t];
                        b--;
                    }
                    s_k = k - cum;  // rank inside bin b
                    s_bin_cnt = hb[min(t, 7)];
                    s_prefix = prefix | ((uint32_t)b << shift);
                    s_mask = mask | (0xFFu << shift);
                    s_ln = 0;
                }
            }
            __syncthreads();
            // after the score byte the cut falls inside ONE score value: when few candidates share it (the usual case), rank
            // them directly instead of three more radix passes over all keys
            if (shift == 24 && s_bin_cnt <= CS_LIST) {
                const uint32_t prefix2 = s_prefix;
                for (int i = tid; i < n; i += blockDim.x) {
                    const uint32_t k = keys[i];
                    if (k >= min_key && (k & 0xFF000000u) == prefix2) s_list[atomicAdd(&s_ln, 1)] = k;
                }
                __syncthreads();
                const int ln = s_ln, kk = s_k;
                for (int t = tid; t < ln; t += blockDim.x) {
                    const uint32_t mine = s_list[t];
                    int rank = 0;
                    for (int j = 0; j < ln; j++) rank += s_list[j] > mine;
                    if (rank == kk - 1) s_prefix = mine;   // keys are unique: exactly one thread
                }
                __syncthreads();
                break;
            }
        }
        cut = s_prefix;  // the keep-th largest eligible key
    }
    const int nk = min(keep, n_elig);
    if (tid == 0) {
        s_base = atomicAdd(&wk.kept_cnt[(size_t)f * plan->nlevels + l], nk);
        s_fill = 0;
    }
    __syncthreads();
    const int base = s_base;
    const unsigned long long cell_part = (unsigned long long)(4095 - (gcell - L.cell_base)) << 24;
    unsigned long long *__restrict__ kept = wk.kept_keys + (size_t)f * plan->kept_total + L.kept_base;
    for (int i = tid; i < n; i += blockDim.x) {
        const uint32_t k = keys[i];
        if (k >= cut) {
            const int p = base + atomicAdd(&s_fill, 1);
            if (p < L.kept_cap)
                kept[p] = ((unsigned long long)(k >> 24) << 36) | cell_part | (unsigned long long)(k & 0xFFFFFFu);
            else
                atomicExch(wk.err_flag, 2);
        }
    }
}

void launch_cell_select(const PlanDev *d_plan, const PlanDev &hp, WorkDev w, int f0, int nf, cudaStream_t s) {
    if (hp.ncells_total == 0) return;
    dim3 grid(hp.ncells_total, nf);
    if (w.cand_keys64) { cell_select_harris_kernel<<<grid, 128, 0, s>>>(d_plan, w, f0); return; }
    launch_k(cell_select_kernel, grid, dim3(128), 0, s, hp.pdl != 0, d_plan, w, f0);
}

// ------------------------------------------------------------------------------------------------
// Level-wide trim (:697-701) and canonical ordering.  One CTA per (level, frame); bitonic sorts in smem.
// ------------------------------------------------------------------------------------------------
__device__ void bitonic_sort_desc(unsigned long long *a, int n2) {
    // (warp-local stages under __syncwarp were tried: 21 instead of 55 block barriers for 1024 keys, no gain for one frame and
    // 41 -> 50 us for a 64-frame batch -- the barriers are not what this kernel waits for)
    for (int k = 2; k <= n2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n2; i += blockDim.x) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long x = a[i], y = a[ixj];
                    const bool desc = (i & k) == 0;
                    if (desc ? (x < y) : (x > y)) { a[i] = y; a[ixj] = x; }
                }
            }
            __syncthreads();
        }
    }
}

__global__ void __launch_bounds__(512) level_select_kernel(const PlanDev *__restrict__ plan, WorkDev wk, int f0) {
    pdl_prologue();
    extern __shared__ unsigned long long skeys[];
    const int l = blockIdx.x, f = blockIdx.y + f0;
    const LevelDev &L = plan->lv[l];
    int n = min(wk.kept_cnt[(size_t)f * plan->nlevels + l], L.kept_cap);
    int n2 = 1;
    while (n2 < n) n2 <<= 1;
    const unsigned long long *__restrict__ kept = wk.kept_keys + (size_t)f * plan->kept_total + L.kept_base;
    for (int i = threadIdx.x; i < n2; i += blockDim.x) skeys[i] = i < n ? kept[i] : 0ull;
    __syncthreads();
    int n_out = n;
    if (n > L.quota) {
        bitonic_sort_desc(skeys, n2);
        n_out = L.quota;
    }
    // order key: (cell asc, raster asc) == inverted fields descending; carry the score in the low byte
    const unsigned long long m36 = (1ull << 36) - 1ull;
    for (int i = threadIdx.x; i < n2; i += blockDim.x) {
        const unsigned long long k = skeys[i];
        skeys[i] = i < n_out ? (((k & m36) << 8) | (k >> 36)) : 0ull;
    }
    __syncthreads();
    int m2 = 1;
    while (m2 < n_out) m2 <<= 1;
    bitonic_sort_desc(skeys, m2);
    int2 *__restrict__ out = wk.kp_xy_score + (size_t)f * plan->nfeatures + L.kp_base;
    for (int i = threadIdx.x; i < n_out; i += blockDim.x) {
        const unsigned long long k = skeys[i];
        const int score = (int)(k & 0xFF);
        const unsigned long long inv = k >> 8;
        const int cell = 4095 - (int)(inv >> 24);
        const int raster = 0xFFFFFF - (int)(inv & 0xFFFFFF);
        const int ci = cell / L.cols, cj = cell - ci * L.cols;
        const int ly = raster / L.cw, lx = raster - ly * L.cw;
        const int x = ORBFE_EDGE + cj * L.cw + lx, y = ORBFE_EDGE + ci * L.ch + ly;
        out[i] = make_int2(x | (y << 16), score);
    }
    if (threadIdx.x == 0) wk.level_cnt[(size_t)f * plan->nlevels + l] = n_out;
}

// ------------------------------------------------------------------------------------------------
// HARRIS_SCORE variants (scoreType == 0, reference :616-620): candidates are ranked by the float Harris
// response instead of the FAST score.  64-bit candidate keys  order(resp) << 32 | (0xFFFFFF - raster) << 8 | score;
// eligibility still comes from the FAST score (low byte >= the cell's threshold).  Kept entries carry
// (order(resp), cell, raster, score); the level trim ranks by counting (n is at most a few thousand).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) cell_select_harris_kernel(const PlanDev *__restrict__ plan, WorkDev wk, int f0) {
    __shared__ int hist[256];
    __shared__ unsigned long long s_prefix, s_mask;
    __shared__ int s_k, s_base, s_fill;

    const int gcell = blockIdx.x, f = blockIdx.y + f0;
    const size_t fc = (size_t)f * plan->ncells_total + gcell;
    const int keep = wk.cell_keep[fc];
    if (keep <= 0) return;
    const int l = find_level_by(plan, gcell, 2);
    const LevelDev &L = plan->lv[l];
    const int n = min(wk.cell_cnt_lo[fc], wk.cell_cand_cap[gcell]);
    const unsigned long long min_score = wk.cell_min_key[fc] >> 24;  // threshold t: eligible <=> score >= t
    const unsigned long long *__restrict__ keys = wk.cand_keys64 + (size_t)f * plan->cand_total + wk.cell_cand_base[gcell];
    const int tid = threadIdx.x;
    const int lo = wk.cell_cnt_lo[fc], hi = wk.cell_cnt_hi[fc];
    const int n1 = plan->t1_is_lo ? lo : hi, n2 = plan->t1_is_lo ? hi : lo;
    const int n_elig = (n1 <= 3) ? n2 : n1;

    unsigned long long cut = 0;  // rank on the upper 56 bits
    if (n_elig > keep) {
        if (tid == 0) { s_prefix = 0; s_mask = 0; s_k = keep; }
        for (int shift = 56; shift >= 8; shift -= 8) {
            for (int i = tid; i < 256; i += blockDim.x) hist[i] = 0;
            __syncthreads();
            const unsigned long long prefix = s_prefix, mask = s_mask;
            for (int i = tid; i < n; i += blockDim.x) {
                const unsigned long long k = keys[i];
                if ((k & 0xFF) >= min_score && (k & mask) == prefix) atomicAdd(&hist[(int)((k >> shift) & 0xFF)], 1);
            }
            __syncthreads();
            if (tid == 0) {
                int k = s_k, cum = 0, b = 255;
                for (; b >= 0; b--) {
                    if (cum + hist[b] >= k) break;
                    cum += hist[b];
                }
                s_k = k - cum;
                s_prefix = prefix | ((unsigned long long)b << shift);
                s_mask = mask | (0xFFull << shift);
            }
            __syncthreads();
        }
        cut = s_prefix;
    }
    const int nk = min(keep, n_elig);
    if (tid == 0) {
        s_base = atomicAdd(&wk.kept_cnt[(size_t)f * plan->nlevels + l], nk);
        s_fill = 0;
    }
    __syncthreads();
    const int base = s_base;
    const unsigned long long cellinv = (unsigned long long)(4095 - (gcell - L.cell_base));
    unsigned long long *__restrict__ kept = wk.kept_keys + (size_t)f * plan->kept_total + L.kept_base;
    uint32_t *__restrict__ kept2 = wk.kept_aux + (size_t)f * plan->kept_total + L.kept_base;
    for (int i = tid; i < n; i += blockDim.x) {
        const unsigned long long k = keys[i];
        if ((k & 0xFF) >= min_score && (k & ~0xFFull) >= cut) {
            const int p = base + atomicAdd(&s_fill, 1);
            if (p < L.kept_cap) {
                kept[p] = (k & 0xFFFFFFFF00000000ull) | (cellinv << 20) | ((k >> 12) & 0xFFFFFull);  // resp | ~cell | ~raster[23:4]
                kept2[p] = (uint32_t)(((k >> 8) & 0xFull) << 8) | (uint32_t)(k & 0xFF);             // ~raster[3:0] | score
            } else {
                atomicExch(wk.err_flag, 2);
            }
        }
    }
}

__global__ void __launch_bounds__(512) level_select_harris_kernel(const PlanDev *__restrict__ plan, WorkDev wk, int f0) {
    extern __shared__ unsigned long long skeys[];  // [n] hi keys, then [n] u32 lo keys, then [n] u8 survivor flags
    const int l = blockIdx.x, f = blockIdx.y + f0;
    const LevelDev &L = plan->lv[l];
    const int n = min(wk.kept_cnt[(size_t)f * plan->nlevels + l], L.kept_cap);
    uint32_t *slo = reinterpret_cast<uint32_t *>(skeys + L.kept_cap);
    uint8_t *keepf = reinterpret_cast<uint8_t *>(slo + L.kept_cap);
    const unsigned long long *__restrict__ kept = wk.kept_keys + (size_t)f * plan->kept_total + L.kept_base;
    const uint32_t *__restrict__ kept2 = wk.kept_aux + (size_t)f * plan->kept_total + L.kept_base;
    for (int i = threadIdx.x; i < n; i += blockDim.x) { skeys[i] = kept[i]; slo[i] = kept2[i]; }
    __syncthreads();
    const int quota = L.quota;
    // rank by (resp desc, cell asc, raster asc): element i survives iff fewer than `quota` elements beat it
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const unsigned long long hi = skeys[i];
        const uint32_t lo = slo[i] >> 8;
        int rank = 0;
        if (n > quota)
            for (int j = 0; j < n; j++) {
                const unsigned long long hj = skeys[j];
                rank += (hj > hi) || (hj == hi && (slo[j] >> 8) > lo);
            }
        keepf[i] = rank < quota;
    }
    __syncthreads();
    int2 *__restrict__ out = wk.kp_xy_score + (size_t)f * plan->nfeatures + L.kp_base;
    const unsigned long long pos_mask = 0xFFFFFFFFull;  // ~cell (12) | ~raster[23:4] (20)
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        if (!keepf[i]) continue;
        const unsigned long long pi = skeys[i] & pos_mask;
        const uint32_t li = slo[i] >> 8;
        int o = 0;  // canonical position: survivors with a smaller (cell, raster) = larger inverted fields
        for (int j = 0; j < n; j++) {
            if (!keepf[j]) continue;
            const unsigned long long pj = skeys[j] & pos_mask;
            o += (pj > pi) || (pj == pi && (slo[j] >> 8) > li);
        }
        const int cell = 4095 - (int)((pi >> 20) & 0xFFF);
        const int raster = 0xFFFFFF - (int)(((pi & 0xFFFFF) << 4) | li);
        const int ci = cell / L.cols, cj = cell - ci * L.cols;
        const int ly = raster / L.cw, lx = raster - ly * L.cw;
        const int x = ORBFE_EDGE + cj * L.cw + lx, y = ORBFE_EDGE + ci * L.ch + ly;
        out[o] = make_int2(x | (y << 16), (int)__float_as_uint(float_from_order_key((uint32_t)(skeys[i] >> 32))));
    }
    if (threadIdx.x == 0) wk.level_cnt[(size_t)f * plan->nlevels + l] = min(n, quota);
}

int level_select_harris_smem_bytes(int max_kept) { return max_kept * (8 + 4 + 1) + 16; }
int set_level_select_harris_smem(int bytes) {
    return (int)cudaFuncSetAttribute(level_select_harris_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
}

int level_select_smem_bytes(int max_kept) {
    int n2 = 1;
    while (n2 < max_kept) n2 <<= 1;
    return n2 * (int)sizeof(unsigned long long);
}

int set_level_select_smem(int bytes) {
    return (int)cudaFuncSetAttribute(level_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
}

void launch_level_select(const PlanDev *d_plan, const PlanDev &hp, WorkDev w, size_t smem_bytes, int f0, int nf, cudaStream_t s) {
    dim3 grid(hp.nlevels, nf);
    if (w.cand_keys64) { level_select_harris_kernel<<<grid, 512, smem_bytes, s>>>(d_plan, w, f0); return; }
    launch_k(level_select_kernel, grid, dim3(512), smem_bytes, s, hp.pdl != 0, d_plan, w, f0);
}

// ------------------------------------------------------------------------------------------------
// 7x7 Gaussian, OpenCV-2.4 integer engine: taps [18,34,49,55,49,34,18] per pass (sum 257), exact
// int accumulation, (sum)/65536 rounded half-to-even, saturated.  BORDER_REFLECT_101 by index reflection.
// Row sums fit u16 exactly (255*257 = 65535).
// ------------------------------------------------------------------------------------------------
// Tile = 120 x 64 output pixels per CTA.  lane = 4-px column group (lanes 0 and 31 are halo columns), warp =
// 8-row segment.  Vertical pass FIRST, on packed pixel pairs (b0,b2)/(b1,b3) of the thread's own word, in a 7-row
// register window: column sums fit u16, so one IMAD/IADD handles two pixels.  The horizontal pass takes the
// three neighbours on each side from the adjacent lanes (4 shuffles) and finishes in 32-bit.
#define B2_W ORBFE_BT_W           // 120
#define B2_H ORBFE_BT_H           // 64
#define B2_PH (B2_H + 6)          // staged rows y0-3 .. y0+66
#define B2_PS 128                 // staged row stride: cols x0-4 .. x0+123

__device__ __forceinline__ int reflect101(int i, int n) {
    if (n == 1) return 0;
    while (i < 0 || i >= n) i = i < 0 ? -i : 2 * (n - 1) - i;
    return i;
}

__device__ __forceinline__ uint32_t blur_round_u8(int s) {
    int q = (s + 0x7FFF + ((s >> 16) & 1)) >> 16;  // round half to even of s / 65536
    return (uint32_t)min(q, 255);
}

__global__ void __launch_bounds__(256) blur7_kernel(const PlanDev *__restrict__ plan, const BTileInfo *__restrict__ btiles, int f0,
                                                    int dst_f0) {
    __shared__ __align__(16) uint8_t pix[B2_PH * B2_PS];

    const int f = blockIdx.y + f0;
    const BTileInfo bt = btiles[blockIdx.x];
    const LevelDev &L = plan->lv[bt.level];
    const int x0 = bt.tx * B2_W, y0 = bt.ty * B2_H;
    const int w = L.w, h = L.h, pitch = L.pitch;
    const uint8_t *__restrict__ img = L.pyr + (size_t)f * L.plane;

    const bool interior = (x0 >= 4) && (x0 + B2_W + 4 <= w) && (y0 >= 3) && (y0 + B2_H + 3 <= h);
    if (interior) {
        for (int i = threadIdx.x; i < B2_PH * 32; i += blockDim.x) {
            const int r = i >> 5, c = i & 31;
            reinterpret_cast<uint32_t *>(pix)[i] =
                __ldg(reinterpret_cast<const uint32_t *>(img + (size_t)(y0 - 3 + r) * pitch + (x0 - 4)) + c);
        }
    } else {
        for (int i = threadIdx.x; i < B2_PH * B2_PS; i += blockDim.x) {
            const int r = i >> 7, c = i & 127;
            const int gy = reflect101(y0 - 3 + r, h);
            const int gx = reflect101(x0 - 4 + c, w);
            pix[i] = __ldg(img + (size_t)gy * pitch + gx);
        }
    }
    __syncthreads();

    const int g = threadIdx.x & 31, seg = threadIdx.x >> 5;
    const uint32_t *col = reinterpret_cast<const uint32_t *>(pix) + (seg * 8) * 32 + g;
    uint32_t A[7], B[7];  // packed (b0,b2) and (b1,b3) of rows r-3 .. r+3
#pragma unroll
    for (int r = 0; r < 6; r++) {
        const uint32_t wv = col[r * 32];
        A[r] = __byte_perm(wv, 0, 0x4240);
        B[r] = __byte_perm(wv, 0, 0x4341);
    }
    uint8_t *__restrict__ dst = L.blur + (size_t)(blockIdx.y + dst_f0) * L.plane;
    const int gx = x0 - 4 + 4 * g;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        {
            const uint32_t wv = col[(6 + i) * 32];
            A[(6 + i) % 7] = __byte_perm(wv, 0, 0x4240);
            B[(6 + i) % 7] = __byte_perm(wv, 0, 0x4341);
        }
#define WR(k) ((i + (k)) % 7)
        // vertical 7-tap on packed pairs (each half <= 65535: no carry between halves)
        const uint32_t VA = 55u * A[WR(3)] + 49u * (A[WR(2)] + A[WR(4)]) + 34u * (A[WR(1)] + A[WR(5)]) + 18u * (A[WR(0)] + A[WR(6)]);
        const uint32_t VB = 55u * B[WR(3)] + 49u * (B[WR(2)] + B[WR(4)]) + 34u * (B[WR(1)] + B[WR(5)]) + 18u * (B[WR(0)] + B[WR(6)]);
#undef WR
        const uint32_t LA = __shfl_up_sync(0xffffffffu, VA, 1), LB = __shfl_up_sync(0xffffffffu, VB, 1);
        const uint32_t RA = __shfl_down_sync(0xffffffffu, VA, 1), RB = __shfl_down_sync(0xffffffffu, VB, 1);
        // column sums v[-3..6] around the group's 4 pixels
        const int vm3 = (int)(LB & 0xFFFF), vm2 = (int)(LA >> 16), vm1 = (int)(LB >> 16);
        const int v0 = (int)(VA & 0xFFFF), v1 = (int)(VB & 0xFFFF), v2 = (int)(VA >> 16), v3 = (int)(VB >> 16);
        const int v4 = (int)(RA & 0xFFFF), v5 = (int)(RB & 0xFFFF), v6 = (int)(RA >> 16);
        const int s0 = 55 * v0 + 49 * (vm1 + v1) + 34 * (vm2 + v2) + 18 * (vm3 + v3);
        const int s1 = 55 * v1 + 49 * (v0 + v2) + 34 * (vm1 + v3) + 18 * (vm2 + v4);
        const int s2 = 55 * v2 + 49 * (v1 + v3) + 34 * (v0 + v4) + 18 * (vm1 + v5);
        const int s3 = 55 * v3 + 49 * (v2 + v4) + 34 * (v1 + v5) + 18 * (v0 + v6);
        const uint32_t out = blur_round_u8(s0) | (blur_round_u8(s1) << 8) | (blur_round_u8(s2) << 16) | (blur_round_u8(s3) << 24);
        const int gy = y0 + seg * 8 + i;
        if (g >= 1 && g <= 30 && gy < h && gx < w) *reinterpret_cast<uint32_t *>(dst + (size_t)gy * pitch + gx) = out;
    }
}

// smoothed planes of frames [f0, f0+nf) are written to plane slots [dst_f0, dst_f0+nf) of lv[].blur
void launch_blur(const PlanDev *d_plan, const PlanDev &hp, WorkDev w, int f0, int nf, int dst_f0, cudaStream_t s) {
    dim3 grid(hp.nbtiles_total, nf);
    blur7_kernel<<<grid, 256, 0, s>>>(d_plan, w.btile_info, f0, dst_f0);
}

// ------------------------------------------------------------------------------------------------
// Orientation + descriptor + output packing.  One warp per keypoint slot.
// ------------------------------------------------------------------------------------------------
__constant__ int c_umax[16] = {15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3};

// cv::fastAtan2: 7th-order odd polynomial, every operation rounded to binary32, no FMA
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {
    const float scale = (float)(180.0 / 3.14159265358979323846);
    const float p1 = 0.9997878412794807f * scale, p3 = -0.3258083974640975f * scale;
    const float p5 = 0.1555786518463281f * scale, p7 = -0.04432655554792128f * scale;
    const float eps = (float)2.2204460492503131e-16;  // (float)DBL_EPSILON
    const float ax = fabsf(x), ay = fabsf(y);
    float a;
    if (ax >= ay) {
        const float c = __fdiv_rn(ay, __fadd_rn(ax, eps));
        const float c2 = __fmul_rn(c, c);
        a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
    } else {
        const float c = __fdiv_rn(ax, __fadd_rn(ay, eps));
        const float c2 = __fmul_rn(c, c);
        a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
    }
    if (x < 0) a = __fsub_rn(180.f, a);
    if (y < 0) a = __fsub_rn(360.f, a);
    return a;
}

__global__ void __launch_bounds__(256) describe_kernel(const PlanDev *__restrict__ plan, WorkDev wk,
                                                       const int8_t *__restrict__ g_pattern,
                                                       OrbfeKeyPoint *__restrict__ out_kps,
                                                       uint8_t *__restrict__ out_desc, int *__restrict__ out_counts, int f0) {
    __shared__ __align__(16) int8_t pat[1024];
    for (int i = threadIdx.x; i < 256; i += blockDim.x)
        reinterpret_cast<uint32_t *>(pat)[i] = __ldg(reinterpret_cast<const uint32_t *>(g_pattern) + i);
    __syncthreads();

    const int f = blockIdx.y + f0;
    const int lane = threadIdx.x & 31;
    const int slot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int nlev = plan->nlevels;
    const int *__restrict__ lcnt = wk.level_cnt + (size_t)f * nlev;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        int tot = 0;
        for (int k = 0; k < nlev; k++) tot += lcnt[k];
        out_counts[f] = tot;
    }
    if (slot >= plan->nfeatures) return;
    const int l = find_level_by(plan, slot, 3);
    const LevelDev &L = plan->lv[l];
    const int idx = slot - L.kp_base;
    if (idx >= lcnt[l]) return;
    int out_idx = idx;
    for (int k = 0; k < l; k++) out_idx += lcnt[k];

    const int2 kp = wk.kp_xy_score[(size_t)f * plan->nfeatures + slot];
    const int x = kp.x & 0xFFFF, y = kp.x >> 16;
    const int w = L.w, h = L.h, pitch = L.pitch;
    const uint8_t *__restrict__ img = L.pyr + (size_t)f * L.plane;
    const uint8_t *__restrict__ blr = L.blur + (size_t)f * L.plane;

    // ---- IC_Angle: lane <-> column u = lane-15, loop over rows v ----
    int m10 = 0, m01 = 0;
    {
        const int u = lane - 15;
        const int au = abs(u);
        if (lane < 31) {
            const uint8_t *c = img + (size_t)y * pitch + x + u;
            // all 31 row loads are independent: issue them back to back (fully unrolled), then reduce
            int colsum = 0;
#pragma unroll
            for (int v = -15; v <= 15; v++) {
                const int val = (au <= c_umax[v < 0 ? -v : v]) ? (int)__ldg(c + (ptrdiff_t)v * pitch) : 0;
                colsum += val;
                m01 += v * val;
            }
            m10 = u * colsum;
        }
        m10 = warp_sum(m10);
        m01 = warp_sum(m01);
    }
    const float angle = fast_atan2_deg((float)m01, (float)m10);

    // ---- rotated BRIEF: lane <-> descriptor byte ----
    const float factorPI = (float)(3.14159265358979323846 / 180.f);  // (float)(CV_PI/180.f)
    const float th = __fmul_rn(angle, factorPI);
    const float a = (float)cos((double)th), b = (float)sin((double)th);
    int val = 0;
    const int8_t *pp = pat + lane * 32;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        int t[2];
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const float px = (float)pp[4 * k + 2 * e], py = (float)pp[4 * k + 2 * e + 1];
            const int ry = __float2int_rn(__fadd_rn(__fmul_rn(px, b), __fmul_rn(py, a)));
            const int rx = __float2int_rn(__fsub_rn(__fmul_rn(px, a), __fmul_rn(py, b)));
            const int sx = x + rx, sy = y + ry;
            if (sx >= 0 && sx < w && sy >= 0 && sy < h) t[e] = __ldg(blr + (size_t)sy * pitch + sx);
            else t[e] = __ldg(img + (size_t)reflect101(sy, h) * pitch + reflect101(sx, w));  // unblurred frame
        }
        val |= (t[0] < t[1]) << k;
    }
    // pack 4 lanes' bytes into a word; lanes 0,4,8,.. store
    uint32_t word = (uint32_t)val;
    word |= __shfl_down_sync(0xffffffffu, (uint32_t)val, 1) << 8;
    word |= __shfl_down_sync(0xffffffffu, (uint32_t)val, 2) << 16;
    word |= __shfl_down_sync(0xffffffffu, (uint32_t)val, 3) << 24;
    const size_t o = (size_t)f * plan->nfeatures + out_idx;
    if ((lane & 3) == 0) reinterpret_cast<uint32_t *>(out_desc + o * 32)[lane >> 2] = word;
    if (lane == 0) {
        OrbfeKeyPoint r;
        r.x = l ? __fmul_rn((float)x, L.scale) : (float)x;  // :768-775
        r.y = l ? __fmul_rn((float)y, L.scale) : (float)y;
        r.size = L.patch_size;
        r.angle = angle;
        r.response = wk.cand_keys64 ? __int_as_float(kp.y) : (float)kp.y;  // Harris response or FAST score
        r.octave = l;
        r.class_id = -1;
        out_kps[o] = r;
    }
}

// ------------------------------------------------------------------------------------------------
// Fused variant (the one the pipeline runs): the 7x7 Gaussian is evaluated only where a descriptor reads it.
// A rotated BRIEF offset has |dx|,|dy| <= 18 (pattern radius 18.38), so every smoothed value a keypoint needs
// comes from the raw 43x43 patch around it.  Per warp: stage the patch in shared memory (reflect-101 at the image
// border, exactly the frame blur7_kernel stages), IC_Angle from the staged patch, vertical 7-tap of the 37 rows a
// sample can fall on (4x4 byte transposes, then two IDP.4A per output; u16 results: 255*257 = 65535), then the
// horizontal 7-tap (four IDP.2A on contiguous u16) + round-half-even only at the 512 sampled positions.  Integer arithmetic throughout: bit-identical to blur7_kernel + describe_kernel, without
// writing and re-reading a blurred copy of the pyramid (2 x P bytes per frame) and ~6x fewer filter taps.
// ------------------------------------------------------------------------------------------------
#define DF_R 21                 // patch radius: 18 (largest rotated offset) + 3 (filter taps)
#define DF_ROWS (2 * DF_R + 1)  // 43
#define DF_RW 13                // raw row stride in words (52 bytes >= 3 + 43 + 6)
#define DF_VR 37                // column-filtered rows: sample rows -18 .. 18
#define DF_VW 24                // their stride in words (48 u16 >= 3 + 43)
#define DF_WARP_WORDS (DF_ROWS * DF_RW + 1 + DF_VR * DF_VW)  // 559 + 1 (pad to even) + 888

// one descriptor byte (8 comparisons) of the fused kernel: vpW = column sums of the staged patch (row ry+18, u16
// index xoff + rx - 3 + tap), ctr = the patch's centre pixel
template <bool CHECK>
__device__ __forceinline__ int brief_byte_fused(const __half2 *pp, float a, float b, int x, int y, int w, int h,
                                                const uint32_t *vpW, int xoff, const uint8_t *ctr) {
    int val = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        int t[2];
#pragma unroll
        for (int e = 0; e < 2; e++) {
            // pattern pair 2k+e of this lane's descriptor byte; layout [pair / 4][lane][pair % 4]: the four LDS.128 of a warp
            // cover 512 contiguous bytes each (the byte-major layout [lane][16] put 16 lanes on the same banks)
            const float2 pf = __half22float2(pp[(k >> 1) * 128 + ((2 * k + e) & 3)]);
            const float px = pf.x, py = pf.y;
            // cvRound (round half to even) of |v| < 2^22 as one FADD: v + 1.5 * 2^23 has ulp 1
            const float fy = __fadd_rn(__fadd_rn(__fmul_rn(px, b), __fmul_rn(py, a)), 12582912.0f);
            const float fx = __fadd_rn(__fsub_rn(__fmul_rn(px, a), __fmul_rn(py, b)), 12582912.0f);
            const int ry = __float_as_int(fy) - 0x4B400000, rx = __float_as_int(fx) - 0x4B400000;
            const int sx = x + rx, sy = y + ry;
            if (!CHECK || (sx >= 0 && sx < w && sy >= 0 && sy < h)) {
                // 7 contiguous column sums starting at u16 index c0 of row ry + 18: four words from the even index
                // below c0; the taps sit on even or odd positions of those words
                const int c0 = xoff + rx;
                const uint32_t *vw = vpW + (ry + 18) * DF_VW + (c0 >> 1);
                const bool odd = c0 & 1;
                const uint32_t TX = odd ? 0x31221200u : 0x37312212u, TY = odd ? 0x12223137u : 0x00122231u;
                const int s = (int)__dp2a_lo(vw[0], TX, __dp2a_hi(vw[1], TX, __dp2a_lo(vw[2], TY, __dp2a_hi(vw[3], TY, 0u))));
                t[e] = (int)blur_round_u8(s);
            } else {
                t[e] = ctr[ry * (4 * DF_RW) + rx];  // outside the image: the reflected, unblurred frame
            }
        }
        val |= (t[0] < t[1]) << k;
    }
    return val;
}

// PEERS: the exchange of a camera rig fused into the kernel (include/orbfe_comm.h): every keypoint / descriptor / count is
// stored into slot [rank] of EVERY rank's gather buffer (st.global on peer pointers over NVLink) instead of one local
// output, and the last thread block to finish publishes the epoch to every rank's flag word (release at system scope).
template <bool PEERS>
__device__ __forceinline__ void describe_fused_body(const PlanDev *__restrict__ plan, const WorkDev &wk,
                                                    const int8_t *__restrict__ g_pattern,
                                                    OrbfeKeyPoint *__restrict__ out_kps,
                                                    uint8_t *__restrict__ out_desc, int *__restrict__ out_counts, int f0,
                                                    const PeerOut &po) {
    // the pattern as fp16 (x, y) pairs: small integers are exact, and fp16 -> fp32 is a full-rate conversion
    __shared__ __align__(16) __half2 pat[512];
    __shared__ __align__(16) uint32_t patch[8 * DF_WARP_WORDS];
    for (int i = threadIdx.x; i < 512; i += blockDim.x) {   // i = 16 * descriptor byte (= lane) + pair
        const char2 p = *reinterpret_cast<const char2 *>(g_pattern + 2 * i);
        const int ln = i >> 4, pr = i & 15;
        pat[((pr >> 2) * 32 + ln) * 4 + (pr & 3)] = __floats2half2_rn((float)p.x, (float)p.y);
    }
    __syncthreads();

    const int f = blockIdx.y + f0;
    const int lane = threadIdx.x & 31;
    const int slot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int nlev = plan->nlevels;
    const int *__restrict__ lcnt = wk.level_cnt + (size_t)f * nlev;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        int tot = 0;
        for (int k = 0; k < nlev; k++) tot += lcnt[k];
        if (PEERS) { for (int p = 0; p < po.n; p++) po.counts[p][f] = tot; }
        else out_counts[f] = tot;
    }
    if (slot >= plan->nfeatures) return;
    // level of this slot and its position in the frame's output, warp-cooperatively: lane k holds level k's slot
    // base and kept count (bases are non-decreasing: the last level whose base <= slot owns it)
    const int base_k = lane < nlev ? plan->lv[lane].kp_base : 0x7FFFFFFF;
    const int cnt_k = lane < nlev ? lcnt[lane] : 0;
    const int l = 31 - __clz(__ballot_sync(0xffffffffu, slot >= base_k));
    const LevelDev &L = plan->lv[l];
    const int idx = slot - __shfl_sync(0xffffffffu, base_k, l);
    if (idx >= __shfl_sync(0xffffffffu, cnt_k, l)) return;
    const int out_idx = idx + warp_sum(lane < l ? cnt_k : 0);

    const int2 kp = wk.kp_xy_score[(size_t)f * plan->nfeatures + slot];
    const int x = kp.x & 0xFFFF, y = kp.x >> 16;
    const int w = L.w, h = L.h, pitch = L.pitch;
    const uint8_t *__restrict__ img = L.pyr + (size_t)f * L.plane;

    uint32_t *rawW = patch + (threadIdx.x >> 5) * DF_WARP_WORDS;   // [43][13] words
    uint32_t *vpW = rawW + DF_ROWS * DF_RW + 1;                    // [37][24] words = [37][48] u16 (8-byte aligned)
    uint8_t *rawB = reinterpret_cast<uint8_t *>(rawW);

    // ---- stage the raw patch: patch column j (image column x-21+j) sits at byte off + j of its row ----
    const int xa = (x - DF_R) & ~3;
    // interior keypoints (all but a thin border band): 43 rows x 13 aligned words, two rows per step on lanes 0..25;
    // every load is issued before the first store waits on one
    const bool fast = (x >= DF_R) && (x + DF_R < w) && (y >= DF_R) && (y + DF_R < h) && (xa + 4 * DF_RW <= pitch);
    const int off = fast ? ((x - DF_R) & 3) : 0;
    if (fast) {
        const int sub = lane >= DF_RW ? 1 : 0, c = lane - sub * DF_RW;
        constexpr int NS = (DF_ROWS + 1) / 2;  // 22 steps
        uint32_t v[NS];
        const uint32_t *src = reinterpret_cast<const uint32_t *>(img + (size_t)(y - DF_R + sub) * pitch + xa) + c;
        const size_t step = (size_t)pitch >> 1;  // two rows, in words
        if (lane < 2 * DF_RW) {
#pragma unroll
            for (int q = 0; q < NS; q++)
                if (2 * q + sub < DF_ROWS) v[q] = __ldg(src + q * step);
#pragma unroll
            for (int q = 0; q < NS; q++)
                if (2 * q + sub < DF_ROWS) rawW[(2 * q) * DF_RW + lane] = v[q];  // (2q + sub) * 13 + c == 2q * 13 + lane
        }
    } else {
        for (int i = lane; i < DF_ROWS * 4 * DF_RW; i += 32) {
            const int r = i / (4 * DF_RW), j = i - r * (4 * DF_RW);
            const int gy = reflect101(y - DF_R + r, h);
            const int gx = reflect101(x - DF_R + j, w);
            rawB[i] = __ldg(img + (size_t)gy * pitch + gx);
        }
    }
    __syncwarp();
    const uint8_t *ctr = rawB + DF_R * (4 * DF_RW) + off + DF_R;   // the keypoint's own pixel

    // ---- IC_Angle: lane <-> column u = lane-15, loop over rows v ----
    int m10 = 0, m01 = 0;
    {
        const int u = lane - 15;
        const int au = abs(u);
        if (lane < 31) {
            int colsum = 0;
#pragma unroll
            for (int v = -15; v <= 15; v++) {
                const int val = (au <= c_umax[v < 0 ? -v : v]) ? (int)ctr[v * (4 * DF_RW) + u] : 0;
                colsum += val;
                m01 += v * val;
            }
            m10 = u * colsum;
        }
        m10 = warp_sum(m10);
        m01 = warp_sum(m01);
    }
    const float angle = fast_atan2_deg((float)m01, (float)m10);

    // ---- vertical 7-tap: V[o][c] = sum_k T[k] * raw[o + k][c], o = 0..36 (sample rows -18..18), all 48 staged columns.
    //      lane = (word column cw, half): 12 x 2 lanes; a lane walks down its 4 byte columns in groups of 4 rows,
    //      transposing each 4x4 byte block so that 4 vertically adjacent pixels share a register ----
    if (lane < 24) {
        const uint32_t T0 = 18u | (34u << 8) | (49u << 16) | (55u << 24), T1 = 49u | (34u << 8) | (18u << 16);
        const int half = lane >= 12 ? 1 : 0, cw = lane - 12 * half;
        // half 0: output rows 0..19 (input rows 0..27), half 1: output rows 20..36 (input rows 20..42, clamped loads)
        const int obase = 20 * half;
        const uint32_t *rw = rawW + obase * DF_RW + cw;
        uint32_t *vw = vpW + obase * DF_VW + 2 * cw;
        uint32_t col[3][4];  // transposed blocks g, g+1, g+2: col[b][j] = 4 consecutive rows of byte column j
#define DF_LOAD_BLOCK(dst, g)                                                                               \
        {                                                                                                   \
            const int rmax = DF_ROWS - 1 - obase;                                                           \
            const uint32_t q0 = rw[min(4 * (g), rmax) * DF_RW], q1 = rw[min(4 * (g) + 1, rmax) * DF_RW];     \
            const uint32_t q2 = rw[min(4 * (g) + 2, rmax) * DF_RW], q3 = rw[min(4 * (g) + 3, rmax) * DF_RW]; \
            const uint32_t t0 = __byte_perm(q0, q1, 0x5140), t1 = __byte_perm(q0, q1, 0x7362);               \
            const uint32_t t2 = __byte_perm(q2, q3, 0x5140), t3 = __byte_perm(q2, q3, 0x7362);               \
            dst[0] = __byte_perm(t0, t2, 0x5410); dst[1] = __byte_perm(t0, t2, 0x7632);                       \
            dst[2] = __byte_perm(t1, t3, 0x5410); dst[3] = __byte_perm(t1, t3, 0x7632);                       \
        }
        DF_LOAD_BLOCK(col[0], 0)
        DF_LOAD_BLOCK(col[1], 1)
#pragma unroll
        for (int g = 0; g < 5; g++) {
            DF_LOAD_BLOCK(col[(g + 2) % 3], g + 2)
#pragma unroll
            for (int sft = 0; sft < 4; sft++) {
                const int o = 4 * g + sft;  // output row inside this half
                uint32_t hv[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const uint32_t lo = __funnelshift_r(col[g % 3][j], col[(g + 1) % 3][j], 8 * sft);        // rows o .. o+3
                    const uint32_t hi = __funnelshift_r(col[(g + 1) % 3][j], col[(g + 2) % 3][j], 8 * sft);  // rows o+4 .. o+7
                    hv[j] = __dp4a(lo, T0, __dp4a(hi, T1, 0u));
                }
                if (obase + o < DF_VR)
                    *reinterpret_cast<uint2 *>(vw + o * DF_VW) = make_uint2(__byte_perm(hv[0], hv[1], 0x5410), __byte_perm(hv[2], hv[3], 0x5410));
            }
        }
#undef DF_LOAD_BLOCK
    }
    __syncwarp();

    // ---- rotated BRIEF: lane <-> descriptor byte; smoothed value = vertical 7-tap of the row sums at the sample ----
    const float factorPI = (float)(3.14159265358979323846 / 180.f);  // (float)(CV_PI/180.f)
    const float th = __fmul_rn(angle, factorPI);
    double sd, cd;
    sincos((double)th, &sd, &cd);
    const float a = (float)cd, b = (float)sd;
    // keypoints at least 18 px inside the image (all but a 2-px band behind the 16-px detection border) cannot sample
    // outside it: no per-sample bounds test
    const bool inner = (x >= 18) && (x + 18 < w) && (y >= 18) && (y + 18 < h);
    const int xoff = off + DF_R - 3;  // u16 index of the leftmost tap of a sample at rx = 0
    const int val = inner ? brief_byte_fused<false>(pat + lane * 4, a, b, x, y, w, h, vpW, xoff, ctr)
                          : brief_byte_fused<true>(pat + lane * 4, a, b, x, y, w, h, vpW, xoff, ctr);
    uint32_t word = (uint32_t)val;
    word |= __shfl_down_sync(0xffffffffu, (uint32_t)val, 1) << 8;
    word |= __shfl_down_sync(0xffffffffu, (uint32_t)val, 2) << 16;
    word |= __shfl_down_sync(0xffffffffu, (uint32_t)val, 3) << 24;
    const size_t o = (size_t)f * plan->nfeatures + out_idx;
    if (PEERS) {
        // remote stores over NVLink: 16-byte descriptor halves from lanes 0 and 16, the seven keypoint fields from lanes 0..6
        // (one coalesced 28-byte segment per destination) -- every lane holds the same keypoint values
        const uint32_t w1 = __shfl_down_sync(0xffffffffu, word, 4), w2 = __shfl_down_sync(0xffffffffu, word, 8);
        const uint32_t w3 = __shfl_down_sync(0xffffffffu, word, 12);
        const float kx = l ? __fmul_rn((float)x, L.scale) : (float)x, ky = l ? __fmul_rn((float)y, L.scale) : (float)y;  // :768-775
        const float resp = wk.cand_keys64 ? __int_as_float(kp.y) : (float)kp.y;
        const uint32_t field = lane == 0 ? __float_as_uint(kx) : lane == 1 ? __float_as_uint(ky) : lane == 2 ? __float_as_uint(L.patch_size)
                             : lane == 3 ? __float_as_uint(angle) : lane == 4 ? __float_as_uint(resp) : lane == 5 ? (uint32_t)l : 0xFFFFFFFFu;
        for (int p = 0; p < po.n; p++) {
            if ((lane & 15) == 0) reinterpret_cast<uint4 *>(po.desc[p] + o * 32)[lane >> 4] = make_uint4(word, w1, w2, w3);
            if (lane < 7) reinterpret_cast<uint32_t *>(po.kps[p] + o)[lane] = field;
        }
        return;
    }
    if ((lane & 3) == 0) reinterpret_cast<uint32_t *>(out_desc + o * 32)[lane >> 2] = word;
    if (lane == 0) {
        OrbfeKeyPoint r;
        r.x = l ? __fmul_rn((float)x, L.scale) : (float)x;  // :768-775
        r.y = l ? __fmul_rn((float)y, L.scale) : (float)y;
        r.size = L.patch_size;
        r.angle = angle;
        r.response = wk.cand_keys64 ? __int_as_float(kp.y) : (float)kp.y;  // Harris response or FAST score
        r.octave = l;
        r.class_id = -1;
        out_kps[o] = r;
    }
}

__global__ void __launch_bounds__(256) describe_fused_kernel(const PlanDev *__restrict__ plan, WorkDev wk,
                                                             const int8_t *__restrict__ g_pattern,
                                                             OrbfeKeyPoint *__restrict__ out_kps,
                                                             uint8_t *__restrict__ out_desc, int *__restrict__ out_counts, int f0) {
    pdl_prologue();
    PeerOut none;
    none.n = 0;
    describe_fused_body<false>(plan, wk, g_pattern, out_kps, out_desc, out_counts, f0, none);
}

__global__ void __launch_bounds__(256) describe_fused_exchange_kernel(const PlanDev *__restrict__ plan, WorkDev wk,
                                                                      const int8_t *__restrict__ g_pattern, int f0,
                                                                      const __grid_constant__ PeerOut po) {
    // a half of the peers' gather buffers is reused every second epoch: before the first remote store, every rank must have
    // released the epoch that last used it (their acknowledgement flags live in THIS rank's memory: local polling)
    if (po.ack_epoch && (int)threadIdx.x < po.n) {
        const long long t0 = clock64();
        unsigned v;
        do {
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(po.ack + threadIdx.x) : "memory");
            if ((int)(v - po.ack_epoch) >= 0) break;
            if (clock64() - t0 > 4000000000ll) { atomicExch(po.err, 2); break; }   // ~2 s: a peer is gone
            __nanosleep(100);
        } while (true);
    }
    __syncthreads();
    describe_fused_body<true>(plan, wk, g_pattern, nullptr, nullptr, nullptr, f0, po);
    // ---- publish.  The block barrier orders every warp's remote stores before thread 0, whose RELEASE increment of the arrival
    //      counter (gpu scope: the counter is only read by this GPU's blocks) is cumulative over them.  The last block to
    //      arrive has read the counter after all the others' releases; its acq_rel fence at SYSTEM scope then orders all of that
    //      before the epoch words it stores into every rank's flag array.  (A seq_cst system fence per block, which is what
    //      __threadfence_system() is, cost 20 us per 16 k keypoints even with a single local destination.)
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned total = gridDim.x * gridDim.y;
        unsigned prev;
        asm volatile("atom.add.release.gpu.global.u32 %0, [%1], 1;" : "=r"(prev) : "l"(po.done) : "memory");
        if (prev == total - 1) {
            asm volatile("fence.acq_rel.sys;" ::: "memory");
            *po.done = 0;   // ready for the next launch (stream order separates them)
            for (int p = 0; p < po.n; p++)
                asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(po.flag[p]), "r"(po.epoch) : "memory");   // fence above + relaxed store = release
        }
    }
}

void launch_describe_fused(const PlanDev *d_plan, const PlanDev &hp, WorkDev w, const int8_t *d_pattern,
                           OrbfeKeyPoint *d_kps, uint8_t *d_desc, int *d_counts, int f0, int nf, cudaStream_t s, const PeerOut *peers) {
    dim3 grid((hp.nfeatures + 7) / 8, nf);
    if (grid.x == 0) grid.x = 1;
    if (peers && peers->n > 0) { describe_fused_exchange_kernel<<<grid, 256, 0, s>>>(d_plan, w, d_pattern, f0, *peers); return; }
    launch_k(describe_fused_kernel, grid, dim3(256), 0, s, hp.pdl != 0, d_plan, w, d_pattern, d_kps, d_desc, d_counts, f0);
}

void launch_describe(const PlanDev *d_plan, const PlanDev &hp, WorkDev w, const int8_t *d_pattern,
                     OrbfeKeyPoint *d_kps, uint8_t *d_desc, int *d_counts, int f0, int nf, cudaStream_t s) {
    dim3 grid((hp.nfeatures + 7) / 8, nf);
    if (grid.x == 0) grid.x = 1;
    describe_kernel<<<grid, 256, 0, s>>>(d_plan, w, d_pattern, d_kps, d_desc, d_counts, f0);
}

}  // namespace orbfe
