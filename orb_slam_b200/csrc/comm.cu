// comm.cu -- multi-GPU entry points of liborbfe.so (include/orbfe_comm.h): NCCL communicator, descriptor-block all-gather,
// sharded keyframe-database sweep, and the rig exchange fused into the extractor's descriptor kernel (peer stores over
// NVLink + epoch flags, CUDA IPC for the peer pointers).  One process per GPU.  NCCL is loaded with dlopen.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>   // types only; every function is resolved at run time

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <vector>

#include "orbfe_internal.h"
#include "../../include/orbfe_comm.h"

using namespace orbfe;

namespace {

struct NcclApi {
    void *handle = nullptr;
    ncclResult_t (*GetVersion)(int *) = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Broadcast)(const void *, void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
};

NcclApi &nccl() {
    static NcclApi a;
    static bool tried = false;
    if (tried) return a;
    tried = true;
    // RTLD_NOLOAD first: if the host program already carries an NCCL (torch bundles one), use exactly that copy
    const char *names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char *n : names) { a.handle = dlopen(n, RTLD_NOW | RTLD_NOLOAD); if (a.handle) break; }
    for (const char *n : names) { if (a.handle) break; a.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL); }
    if (!a.handle) return a;
#define ORBFE_NCCL_SYM(field, name) *(void **)(&a.field) = dlsym(a.handle, name)
    ORBFE_NCCL_SYM(GetVersion, "ncclGetVersion");
    ORBFE_NCCL_SYM(GetUniqueId, "ncclGetUniqueId");
    ORBFE_NCCL_SYM(CommInitRank, "ncclCommInitRank");
    ORBFE_NCCL_SYM(CommDestroy, "ncclCommDestroy");
    ORBFE_NCCL_SYM(AllGather, "ncclAllGather");
    ORBFE_NCCL_SYM(Broadcast, "ncclBroadcast");
    ORBFE_NCCL_SYM(AllReduce, "ncclAllReduce");
    ORBFE_NCCL_SYM(GroupStart, "ncclGroupStart");
    ORBFE_NCCL_SYM(GroupEnd, "ncclGroupEnd");
    ORBFE_NCCL_SYM(GetErrorString, "ncclGetErrorString");
#undef ORBFE_NCCL_SYM
    a.ok = a.GetVersion && a.GetUniqueId && a.CommInitRank && a.CommDestroy && a.AllGather && a.Broadcast && a.AllReduce &&
           a.GroupStart && a.GroupEnd && a.GetErrorString;
    return a;
}

#define NCCL_TRY(expr)                                                                                                \
    do {                                                                                                              \
        ncclResult_t r__ = (expr);                                                                                    \
        if (r__ != ncclSuccess)                                                                                       \
            return set_error(ORBFE_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, nccl().GetErrorString(r__), __FILE__, __LINE__); \
    } while (0)

}  // namespace

struct OrbfeComm {
    ncclComm_t comm = nullptr;
    int world = 1, rank = 0, device = 0;
    cudaStream_t stream = nullptr;
    int *d_token = nullptr;
};

static_assert(sizeof(ncclUniqueId) == ORBFE_COMM_ID_BYTES, "ORBFE_COMM_ID_BYTES must be sizeof(ncclUniqueId)");

extern "C" int orbfe_comm_nccl_version(void) {
    int v = 0;
    if (nccl().ok) nccl().GetVersion(&v);
    return v;
}

extern "C" int orbfe_comm_unique_id(uint8_t id[ORBFE_COMM_ID_BYTES]) {
    if (!id) return set_error(ORBFE_ERR_ARG, "id is NULL");
    if (!nccl().ok) return set_error(ORBFE_ERR_UNSUPPORTED, "libnccl.so.2 could not be loaded: %s", dlerror() ? dlerror() : "not found");
    ncclUniqueId u;
    NCCL_TRY(nccl().GetUniqueId(&u));
    memcpy(id, &u, sizeof(u));
    return ORBFE_OK;
}

extern "C" int orbfe_comm_create(const uint8_t id[ORBFE_COMM_ID_BYTES], int world, int rank, int device, OrbfeComm **out) {
    if (!out) return set_error(ORBFE_ERR_ARG, "out is NULL");
    *out = nullptr;
    if (!id || world < 1 || world > ORBFE_MAX_RANKS || rank < 0 || rank >= world) return set_error(ORBFE_ERR_ARG, "bad communicator arguments");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return set_error(ORBFE_ERR_NO_DEVICE, "no CUDA device"); }
    if (device < 0 || device >= ndev) return set_error(ORBFE_ERR_ARG, "device %d out of range", device);
    if (!nccl().ok) return set_error(ORBFE_ERR_UNSUPPORTED, "libnccl.so.2 could not be loaded");
    ORBFE_CUDA_TRY(cudaSetDevice(device));
    OrbfeComm *c = new OrbfeComm();
    c->world = world; c->rank = rank; c->device = device;
    ncclUniqueId u;
    memcpy(&u, id, sizeof(u));
    ncclResult_t r = nccl().CommInitRank(&c->comm, world, u, rank);
    if (r != ncclSuccess) { delete c; return set_error(ORBFE_ERR_CUDA, "ncclCommInitRank failed: %s", nccl().GetErrorString(r)); }
    cudaError_t e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMalloc((void **)&c->d_token, 2 * sizeof(int));
    if (e == cudaSuccess) e = cudaMemset(c->d_token, 0, 2 * sizeof(int));
    if (e != cudaSuccess) { orbfe_comm_destroy(c); return set_error(ORBFE_ERR_CUDA, "communicator setup failed: %s", cudaGetErrorString(e)); }
    *out = c;
    return ORBFE_OK;
}

extern "C" int orbfe_comm_destroy(OrbfeComm *c) {
    if (!c) return ORBFE_OK;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->comm) nccl().CommDestroy(c->comm);
    if (c->d_token) cudaFree(c->d_token);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
    return ORBFE_OK;
}

extern "C" int orbfe_comm_world(const OrbfeComm *c) { return c ? c->world : 0; }
extern "C" int orbfe_comm_rank(const OrbfeComm *c) { return c ? c->rank : -1; }

extern "C" int orbfe_comm_sync(OrbfeComm *c) {
    if (!c) return set_error(ORBFE_ERR_ARG, "c is NULL");
    ORBFE_CUDA_TRY(cudaSetDevice(c->device));
    ORBFE_CUDA_TRY(cudaStreamSynchronize(c->stream));
    return ORBFE_OK;
}

extern "C" int orbfe_comm_barrier(OrbfeComm *c, void *stream) {
    if (!c) return set_error(ORBFE_ERR_ARG, "c is NULL");
    ORBFE_CUDA_TRY(cudaSetDevice(c->device));
    NCCL_TRY(nccl().AllReduce(c->d_token, c->d_token + 1, 1, ncclInt32, ncclSum, c->comm, stream ? (cudaStream_t)stream : c->stream));
    return ORBFE_OK;
}

extern "C" int orbfe_comm_broadcast(OrbfeComm *c, void *d_buf, size_t bytes, int root, void *stream) {
    if (!c || !d_buf || root < 0 || root >= c->world) return set_error(ORBFE_ERR_ARG, "bad arguments");
    if (bytes == 0) return ORBFE_OK;
    ORBFE_CUDA_TRY(cudaSetDevice(c->device));
    NCCL_TRY(nccl().Broadcast(d_buf, d_buf, bytes, ncclUint8, root, c->comm, stream ? (cudaStream_t)stream : c->stream));
    return ORBFE_OK;
}

extern "C" int orbfe_comm_allgather(OrbfeComm *c, const void *d_send, void *d_recv, size_t bytes_per_rank, void *stream) {
    if (!c || !d_send || !d_recv) return set_error(ORBFE_ERR_ARG, "bad arguments");
    if (bytes_per_rank == 0) return ORBFE_OK;
    ORBFE_CUDA_TRY(cudaSetDevice(c->device));
    NCCL_TRY(nccl().AllGather(d_send, d_recv, bytes_per_rank, ncclUint8, c->comm, stream ? (cudaStream_t)stream : c->stream));
    return ORBFE_OK;
}

extern "C" int orbfe_allgather_desc(OrbfeComm *c, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc, const int *d_counts, int cap, int nslots,
                                    OrbfeKeyPoint *d_all_kps, uint8_t *d_all_desc, int *d_all_counts, void *stream) {
    if (!c || !d_kps || !d_desc || !d_counts || !d_all_kps || !d_all_desc || !d_all_counts || cap < 1 || nslots < 1)
        return set_error(ORBFE_ERR_ARG, "bad arguments");
    ORBFE_CUDA_TRY(cudaSetDevice(c->device));
    cudaStream_t s = stream ? (cudaStream_t)stream : c->stream;
    const size_t n = (size_t)cap * nslots;
    NCCL_TRY(nccl().GroupStart());
    ncclResult_t r1 = nccl().AllGather(d_kps, d_all_kps, n * sizeof(OrbfeKeyPoint), ncclUint8, c->comm, s);
    ncclResult_t r2 = nccl().AllGather(d_desc, d_all_desc, n * 32, ncclUint8, c->comm, s);
    ncclResult_t r3 = nccl().AllGather(d_counts, d_all_counts, (size_t)nslots, ncclInt32, c->comm, s);
    NCCL_TRY(nccl().GroupEnd());
    NCCL_TRY(r1); NCCL_TRY(r2); NCCL_TRY(r3);
    return ORBFE_OK;
}

extern "C" int orbfe_shard_range(int n_items, int world, int rank, int *lo, int *hi) {
    if (n_items < 0 || world < 1 || rank < 0 || rank >= world || !lo || !hi) return set_error(ORBFE_ERR_ARG, "bad arguments");
    const int base = n_items / world, rem = n_items % world;
    *lo = rank * base + std::min(rank, rem);
    *hi = *lo + base + (rank < rem ? 1 : 0);
    return ORBFE_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// config 5: broadcast the query, sweep the local shard, all-gather the per-keyframe results (padded shards), compact
// ------------------------------------------------------------------------------------------------------------------
namespace {
// gathered layout: [world][gmax][nq] per array; destination: [ngroups_total][nq] in global keyframe order
__global__ void unpad_results_kernel(const uint16_t *__restrict__ gb, const int32_t *__restrict__ gi, const uint16_t *__restrict__ gs,
                                     int world, int gmax, int ngroups_total, int nq, uint16_t *__restrict__ best,
                                     int32_t *__restrict__ idx, uint16_t *__restrict__ second) {
    const size_t total = (size_t)ngroups_total * nq;
    const int base = ngroups_total / world, rem = ngroups_total % world;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(i / nq), q = (int)(i - (size_t)g * nq);
        // owner of global group g: ranks < rem hold base+1 groups
        int r, lo;
        if (g < rem * (base + 1)) { r = g / (base + 1); lo = r * (base + 1); }
        else { r = rem + (base ? (g - rem * (base + 1)) / base : 0); lo = rem * (base + 1) + (r - rem) * base; }
        const size_t src = ((size_t)r * gmax + (g - lo)) * nq + q;
        best[i] = gb[src]; idx[i] = gi[src]; second[i] = gs[src];
    }
}
}  // namespace

extern "C" int orbfe_knn2_sweep_sharded(OrbfeComm *c, OrbfeMatcher *m, uint8_t *d_query, int nq, int root, const uint8_t *d_db_shard,
                                        int ngroups_total, int group_size, uint16_t *d_best_all, int32_t *d_best_idx_all,
                                        uint16_t *d_second_all, void *d_scratch, void *stream) {
    if (!c || !m || !d_query || nq < 1 || ngroups_total < 1 || group_size < 1 || !d_best_all || !d_best_idx_all || !d_second_all || !d_scratch)
        return set_error(ORBFE_ERR_ARG, "bad arguments");
    ORBFE_CUDA_TRY(cudaSetDevice(c->device));
    cudaStream_t s = stream ? (cudaStream_t)stream : c->stream;
    int lo, hi;
    orbfe_shard_range(ngroups_total, c->world, c->rank, &lo, &hi);
    const int nloc = hi - lo, gmax = (ngroups_total + c->world - 1) / c->world;
    if (nloc > 0 && !d_db_shard) return set_error(ORBFE_ERR_ARG, "d_db_shard is NULL");
    // scratch: local results (gmax x nq x 8 B, send side) followed by the gathered copy (world x gmax x nq x 8 B)
    // -- callers size d_scratch for (world + 1) * gmax * nq * 8 bytes
    const size_t per = (size_t)gmax * nq;
    uint8_t *S = (uint8_t *)d_scratch;
    uint16_t *lb = (uint16_t *)S; int32_t *li = (int32_t *)(S + per * 2); uint16_t *ls = (uint16_t *)(S + per * 6);
    uint8_t *G = S + per * 8;
    uint16_t *gb = (uint16_t *)G; int32_t *gi = (int32_t *)(G + (size_t)c->world * per * 2); uint16_t *gs = (uint16_t *)(G + (size_t)c->world * per * 6);
    if (c->world > 1) NCCL_TRY(nccl().Broadcast(d_query, d_query, (size_t)nq * 32, ncclUint8, root, c->comm, s));
    if (c->world == 1) {
        return orbfe_knn2_groups_device(m, d_query, nq, d_db_shard, ngroups_total, group_size, d_best_all, d_best_idx_all, d_second_all, s);
    }
    if (nloc > 0) {
        int rc = orbfe_knn2_groups_device(m, d_query, nq, d_db_shard, nloc, group_size, lb, li, ls, s);
        if (rc) return rc;
    }
    NCCL_TRY(nccl().GroupStart());
    ncclResult_t r1 = nccl().AllGather(lb, gb, per * 2, ncclUint8, c->comm, s);
    ncclResult_t r2 = nccl().AllGather(li, gi, per * 4, ncclUint8, c->comm, s);
    ncclResult_t r3 = nccl().AllGather(ls, gs, per * 2, ncclUint8, c->comm, s);
    NCCL_TRY(nccl().GroupEnd());
    NCCL_TRY(r1); NCCL_TRY(r2); NCCL_TRY(r3);
    unpad_results_kernel<<<296, 256, 0, s>>>(gb, gi, gs, c->world, gmax, ngroups_total, nq, d_best_all, d_best_idx_all, d_second_all);
    ORBFE_CUDA_TRY(cudaGetLastError());
    return ORBFE_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// Rig exchange fused into the extractor (config 4)
// ------------------------------------------------------------------------------------------------------------------
struct OrbfeRigExchange {
    OrbfeComm *c = nullptr;
    int cap = 0, nslots = 0, world = 1, rank = 0;
    // one allocation per rank: [2 halves][ kps world*nslots*cap | desc | counts ] + flags
    uint8_t *base = nullptr;
    size_t half_bytes = 0, kps_off = 0, desc_off = 0, cnt_off = 0, flags_off = 0, total_bytes = 0;
    uint8_t *peer_base[ORBFE_MAX_RANKS] = {nullptr};
    unsigned *done = nullptr;   // local block counter of the publishing kernel
    unsigned *done2 = nullptr;  // local block counter of the consuming (matcher) kernel
    int *d_err = nullptr;
    int *h_err = nullptr;
    unsigned epoch = 0;         // last epoch produced
    unsigned waited = 0;        // last epoch waited for
    size_t last_bytes = 0;
};

namespace {
// flags region: data[world] (epoch published by rank r), ack[world] (last epoch rank r finished reading)
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned *p) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__global__ void wait_flags_kernel(const unsigned *__restrict__ flags, int n, unsigned epoch, int *err, int code) {
    const int r = threadIdx.x;
    if (r >= n) return;
    const long long t0 = clock64();
    while ((int)(ld_acquire_sys(flags + r) - epoch) < 0) {
        if (clock64() - t0 > 4000000000ll) { atomicExch(err, code); break; }   // ~2 s at 1.9 GHz: a peer is gone
        __nanosleep(200);
    }
}
struct AckTargets { int n; unsigned *p[ORBFE_MAX_RANKS]; };
__global__ void publish_kernel(const __grid_constant__ AckTargets t, unsigned epoch) {
    __threadfence_system();
    if ((int)threadIdx.x < t.n) asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(t.p[threadIdx.x]), "r"(epoch) : "memory");
}
}  // namespace

extern "C" int orbfe_rig_exchange_create(OrbfeComm *c, int cap, int nslots, OrbfeRigExchange **out) {
    if (!out) return set_error(ORBFE_ERR_ARG, "out is NULL");
    *out = nullptr;
    if (!c || cap < 1 || nslots < 1) return set_error(ORBFE_ERR_ARG, "bad arguments");
    ORBFE_CUDA_TRY(cudaSetDevice(c->device));
    OrbfeRigExchange *x = new OrbfeRigExchange();
    x->c = c; x->cap = cap; x->nslots = nslots; x->world = c->world; x->rank = c->rank;
    const size_t n = (size_t)c->world * nslots * cap;
    auto up = [](size_t v) { return (v + 255) / 256 * 256; };
    x->kps_off = 0;
    x->desc_off = up(n * sizeof(OrbfeKeyPoint));
    x->cnt_off = x->desc_off + up(n * 32);
    x->half_bytes = x->cnt_off + up((size_t)c->world * nslots * sizeof(int));
    x->flags_off = 2 * x->half_bytes;
    x->total_bytes = x->flags_off + up(2 * ORBFE_MAX_RANKS * sizeof(unsigned));
    cudaError_t e = cudaMalloc((void **)&x->base, x->total_bytes);
    if (e == cudaSuccess) e = cudaMemset(x->base, 0, x->total_bytes);
    if (e == cudaSuccess) e = cudaMalloc((void **)&x->done, 2 * sizeof(unsigned));
    if (e == cudaSuccess) e = cudaMemset(x->done, 0, 2 * sizeof(unsigned));
    if (e == cudaSuccess) x->done2 = x->done + 1;
    if (e == cudaSuccess) e = cudaMalloc((void **)&x->d_err, sizeof(int));
    if (e == cudaSuccess) e = cudaMemset(x->d_err, 0, sizeof(int));
    if (e == cudaSuccess) e = cudaHostAlloc((void **)&x->h_err, sizeof(int), cudaHostAllocDefault);
    if (e != cudaSuccess) { orbfe_rig_exchange_destroy(x); return set_error(ORBFE_ERR_CUDA, "rig exchange allocation failed: %s", cudaGetErrorString(e)); }
    x->peer_base[c->rank] = x->base;
    if (c->world > 1) {
        // ship the IPC handle of the allocation to every rank through the communicator itself
        cudaIpcMemHandle_t mine, *all = nullptr;
        uint8_t *d_h = nullptr;
        e = cudaIpcGetMemHandle(&mine, x->base);
        if (e == cudaSuccess) e = cudaMalloc((void **)&d_h, sizeof(mine) * (size_t)(c->world + 1));
        if (e == cudaSuccess) e = cudaMemcpy(d_h, &mine, sizeof(mine), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) { orbfe_rig_exchange_destroy(x); return set_error(ORBFE_ERR_CUDA, "cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e)); }
        ncclResult_t r = nccl().AllGather(d_h, d_h + sizeof(mine), sizeof(mine), ncclUint8, c->comm, c->stream);
        if (r != ncclSuccess) { cudaFree(d_h); orbfe_rig_exchange_destroy(x); return set_error(ORBFE_ERR_CUDA, "handle all-gather failed: %s", nccl().GetErrorString(r)); }
        std::vector<cudaIpcMemHandle_t> hs(c->world);
        all = hs.data();
        e = cudaStreamSynchronize(c->stream);
        if (e == cudaSuccess) e = cudaMemcpy(all, d_h + sizeof(mine), sizeof(mine) * (size_t)c->world, cudaMemcpyDeviceToHost);
        cudaFree(d_h);
        for (int p = 0; p < c->world && e == cudaSuccess; p++) {
            if (p == c->rank) continue;
            void *ptr = nullptr;
            e = cudaIpcOpenMemHandle(&ptr, all[p], cudaIpcMemLazyEnablePeerAccess);
            x->peer_base[p] = (uint8_t *)ptr;
        }
        if (e != cudaSuccess) { orbfe_rig_exchange_destroy(x); return set_error(ORBFE_ERR_CUDA, "cudaIpcOpenMemHandle failed: %s (peer access over NVLink is required)", cudaGetErrorString(e)); }
        int rc = orbfe_comm_barrier(c, c->stream);   // nobody writes into a peer before everybody has opened everything
        if (rc == ORBFE_OK) rc = orbfe_comm_sync(c);
        if (rc) { orbfe_rig_exchange_destroy(x); return rc; }
    }
    *out = x;
    return ORBFE_OK;
}

extern "C" int orbfe_rig_exchange_destroy(OrbfeRigExchange *x) {
    if (!x) return ORBFE_OK;
    if (x->c) {
        cudaSetDevice(x->c->device);
        cudaDeviceSynchronize();
        if (x->c->world > 1) { orbfe_comm_barrier(x->c, x->c->stream); orbfe_comm_sync(x->c); }   // peers stop writing first
    }
    for (int p = 0; p < x->world; p++)
        if (p != x->rank && x->peer_base[p]) cudaIpcCloseMemHandle(x->peer_base[p]);
    if (x->base) cudaFree(x->base);
    if (x->done) cudaFree(x->done);
    if (x->d_err) cudaFree(x->d_err);
    if (x->h_err) cudaFreeHost(x->h_err);
    delete x;
    return ORBFE_OK;
}

// declared in orbfe_api.cu: runs the extractor pipeline with the descriptor kernel's outputs redirected to `po`
int orbfe_extract_batch_device_peers(OrbfeExtractor *ex, const uint8_t *d_imgs, int width, int height, size_t stride, size_t frame_stride,
                                     int batch, const PeerOut &po, int cap, void *stream);

extern "C" int orbfe_extract_batch_device_exchange(OrbfeExtractor *ex, const uint8_t *d_imgs, int width, int height, size_t stride,
                                                   size_t frame_stride, int batch, OrbfeRigExchange *x, void *stream) {
    if (!ex || !x || !d_imgs) return set_error(ORBFE_ERR_ARG, "NULL argument");
    if (batch != x->nslots) return set_error(ORBFE_ERR_ARG, "batch %d != nslots %d of the exchange", batch, x->nslots);
    ORBFE_CUDA_TRY(cudaSetDevice(x->c->device));
    cudaStream_t s = stream ? (cudaStream_t)stream : x->c->stream;
    const unsigned epoch = x->epoch + 1;
    const int half = (int)(epoch & 1u);
    unsigned *flags = (unsigned *)(x->base + x->flags_off);
    // a buffer half is overwritten only after EVERY rank has released the epoch that last used it (epoch - 2): the
    // descriptor kernel polls the acknowledgement flags (local memory) before its first remote store
    PeerOut po;
    memset(&po, 0, sizeof(po));
    po.n = x->world;
    po.epoch = epoch;
    po.done = x->done;
    po.ack = flags + ORBFE_MAX_RANKS;
    po.ack_epoch = (epoch > 2 && x->world > 1) ? epoch - 2 : 0;
    po.err = x->d_err;
    const size_t slot = (size_t)x->rank * x->nslots * x->cap;
    for (int p = 0; p < x->world; p++) {
        uint8_t *hb = x->peer_base[p] + (size_t)half * x->half_bytes;
        po.kps[p] = (OrbfeKeyPoint *)(hb + x->kps_off) + slot;
        po.desc[p] = hb + x->desc_off + slot * 32;
        po.counts[p] = (int *)(hb + x->cnt_off) + (size_t)x->rank * x->nslots;
        po.flag[p] = (unsigned *)(x->peer_base[p] + x->flags_off) + x->rank;
    }
    int rc = orbfe_extract_batch_device_peers(ex, d_imgs, width, height, stride, frame_stride, batch, po, x->cap, s);
    if (rc) return rc;
    x->epoch = epoch;
    x->last_bytes = (size_t)x->nslots * x->cap * 60 * (size_t)(x->world - 1);
    return ORBFE_OK;
}

// declared in orbfe_api.cu
int orbfe_search_for_initialization_hooked(OrbfeMatcher *m, int npairs, const OrbfeKeyPoint *d_kps, const uint8_t *d_desc,
                                           const int *d_counts, int cap, const int *d_f1_idx, const int *d_f2_idx,
                                           float *d_prev_matched, float min_x, float min_y, float max_x, float max_y,
                                           int window, float nnratio, int check_orientation, int *d_match12,
                                           int *d_nmatches, void *stream, const SbpParams *hooks);

// Cross-camera SearchForInitialization on the epoch just produced: the matcher kernel itself waits for every rank's data
// (polling the local epoch flags) and its last thread block releases the epoch to every rank -- together with
// orbfe_extract_batch_device_exchange a rig step is two library calls and not a single extra kernel launch.
extern "C" int orbfe_search_for_initialization_exchange(OrbfeMatcher *m, OrbfeRigExchange *x, int npairs, const int *d_f1_idx,
                                                        const int *d_f2_idx, float *d_prev_matched, float min_x, float min_y, float max_x,
                                                        float max_y, int window, float nnratio, int check_orientation, int *d_match12,
                                                        int *d_nmatches, void *stream) {
    if (!m || !x) return set_error(ORBFE_ERR_ARG, "NULL argument");
    ORBFE_CUDA_TRY(cudaSetDevice(x->c->device));
    cudaStream_t s = stream ? (cudaStream_t)stream : x->c->stream;
    x->waited = x->epoch;
    uint8_t *hb = x->base + (size_t)(x->waited & 1u) * x->half_bytes;
    SbpParams H;
    memset(&H, 0, sizeof(H));
    H.xw_flags = (unsigned *)(x->base + x->flags_off);
    H.xw_done = x->done2;
    H.xw_err = x->d_err;
    H.xw_n = x->world;
    H.xw_epoch = x->epoch;
    for (int p = 0; p < x->world; p++) H.xw_ack[p] = (unsigned *)(x->peer_base[p] + x->flags_off) + ORBFE_MAX_RANKS + x->rank;
    return orbfe_search_for_initialization_hooked(m, npairs, (const OrbfeKeyPoint *)(hb + x->kps_off), hb + x->desc_off, (const int *)(hb + x->cnt_off),
                                                  x->cap, d_f1_idx, d_f2_idx, d_prev_matched, min_x, min_y, max_x, max_y, window, nnratio,
                                                  check_orientation, d_match12, d_nmatches, s, &H);
}

extern "C" int orbfe_rig_exchange_wait(OrbfeRigExchange *x, void *stream) {
    if (!x) return set_error(ORBFE_ERR_ARG, "x is NULL");
    ORBFE_CUDA_TRY(cudaSetDevice(x->c->device));
    cudaStream_t s = stream ? (cudaStream_t)stream : x->c->stream;
    wait_flags_kernel<<<1, 32, 0, s>>>((unsigned *)(x->base + x->flags_off), x->world, x->epoch, x->d_err, 1);
    ORBFE_CUDA_TRY(cudaGetLastError());
    x->waited = x->epoch;
    return ORBFE_OK;
}

extern "C" int orbfe_rig_exchange_release(OrbfeRigExchange *x, void *stream) {
    if (!x) return set_error(ORBFE_ERR_ARG, "x is NULL");
    ORBFE_CUDA_TRY(cudaSetDevice(x->c->device));
    cudaStream_t s = stream ? (cudaStream_t)stream : x->c->stream;
    AckTargets t;
    t.n = x->world;
    for (int p = 0; p < x->world; p++) t.p[p] = (unsigned *)(x->peer_base[p] + x->flags_off) + ORBFE_MAX_RANKS + x->rank;
    publish_kernel<<<1, 32, 0, s>>>(t, x->waited);
    ORBFE_CUDA_TRY(cudaGetLastError());
    return ORBFE_OK;
}

extern "C" int orbfe_rig_exchange_buffers(OrbfeRigExchange *x, OrbfeKeyPoint **d_all_kps, uint8_t **d_all_desc, int **d_all_counts) {
    if (!x) return set_error(ORBFE_ERR_ARG, "x is NULL");
    uint8_t *hb = x->base + (size_t)(x->waited & 1u) * x->half_bytes;
    if (d_all_kps) *d_all_kps = (OrbfeKeyPoint *)(hb + x->kps_off);
    if (d_all_desc) *d_all_desc = hb + x->desc_off;
    if (d_all_counts) *d_all_counts = (int *)(hb + x->cnt_off);
    return ORBFE_OK;
}

extern "C" int orbfe_rig_exchange_buffers_produced(OrbfeRigExchange *x, OrbfeKeyPoint **d_all_kps, uint8_t **d_all_desc, int **d_all_counts) {
    if (!x) return set_error(ORBFE_ERR_ARG, "x is NULL");
    uint8_t *hb = x->base + (size_t)(x->epoch & 1u) * x->half_bytes;
    if (d_all_kps) *d_all_kps = (OrbfeKeyPoint *)(hb + x->kps_off);
    if (d_all_desc) *d_all_desc = hb + x->desc_off;
    if (d_all_counts) *d_all_counts = (int *)(hb + x->cnt_off);
    return ORBFE_OK;
}

extern "C" int orbfe_rig_exchange_check(OrbfeRigExchange *x, void *stream) {
    if (!x) return set_error(ORBFE_ERR_ARG, "x is NULL");
    ORBFE_CUDA_TRY(cudaSetDevice(x->c->device));
    cudaStream_t s = stream ? (cudaStream_t)stream : x->c->stream;
    ORBFE_CUDA_TRY(cudaMemcpyAsync(x->h_err, x->d_err, sizeof(int), cudaMemcpyDeviceToHost, s));
    ORBFE_CUDA_TRY(cudaStreamSynchronize(s));
    if (*x->h_err) {
        const int code = *x->h_err;
        cudaMemsetAsync(x->d_err, 0, sizeof(int), s);
        return set_error(ORBFE_ERR_INTERNAL, "rig exchange: wait for %s timed out (a peer rank is not taking part)", code == 1 ? "data" : "buffer release");
    }
    return ORBFE_OK;
}

extern "C" size_t orbfe_rig_exchange_bytes(const OrbfeRigExchange *x) { return x ? x->last_bytes : 0; }
