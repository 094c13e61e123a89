// Multi-GPU exchange of the training path (C ABI: include/sd_b200.h, "multi-GPU" section).
//
// The reference trains on one host; its exchange point is the single call `regressors[level].learn(features, b)`
// (superviseddescent.hpp:207): with the samples sharded over ranks, [A^T A | A^T b] is a SUM over the shards.
// One process per GPU; the collectives are NCCL over NVLink / NVSwitch.  libnccl is bound at run time with dlopen
// (the soname a torch process has already loaded is reused; a C++ host gets the system library), so the shared
// object has no link-time dependency on it and single-GPU users never touch it.
//
//   sd_allreduce_gram       every rank gets the summed upper row bands (replicated solve follows)
//   sd_reduce_scatter_gram  the owner of each band (sd_panel_owner) gets its sum (distributed factorisation follows)
// Both move only what the solve reads: each band of SD_PANEL_ROWS rows from its first diagonal column to the end of the row,
// packed into one contiguous buffer by an HBM-speed kernel (about half of the D x (D+M) buffer).
#include "sd_internal.cuh"

#include <dlfcn.h>
#include <nccl.h>

#include <cstdlib>
#include <cstring>

namespace {

struct NcclApi {
    void* handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Reduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    ncclResult_t (*GetVersion)(int*) = nullptr;
    std::string error;
};

NcclApi& nccl()
{
    static NcclApi api;
    static bool tried = false;
    if (tried) return api;
    tried = true;
    const char* names[] = {getenv("SD_B200_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
        if (!n || !*n) continue;
        api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (api.handle) break;
    }
    if (!api.handle) { api.error = std::string("libnccl.so.2 could not be loaded: ") + (dlerror() ? dlerror() : "?"); return api; }
#define SD_BIND(field, sym)                                                              \
    api.field = reinterpret_cast<decltype(api.field)>(dlsym(api.handle, sym));           \
    if (!api.field) { api.error = std::string("symbol missing in libnccl: ") + sym; api.handle = nullptr; return api; }
    SD_BIND(GetUniqueId, "ncclGetUniqueId")
    SD_BIND(CommInitRank, "ncclCommInitRank")
    SD_BIND(CommDestroy, "ncclCommDestroy")
    SD_BIND(AllReduce, "ncclAllReduce")
    SD_BIND(Reduce, "ncclReduce")
    SD_BIND(Broadcast, "ncclBroadcast")
    SD_BIND(AllGather, "ncclAllGather")
    SD_BIND(GroupStart, "ncclGroupStart")
    SD_BIND(GroupEnd, "ncclGroupEnd")
    SD_BIND(GetErrorString, "ncclGetErrorString")
    SD_BIND(GetVersion, "ncclGetVersion")
#undef SD_BIND
    return api;
}

// pack / unpack of the row bands the solve reads: band p = rows [p*SD_PANEL_ROWS, ...), columns [p*SD_PANEL_ROWS, W)
__global__ void band_copy_kernel(float* __restrict__ G, long long ldg, int D, int W, float* __restrict__ flat,
                                 const long long* __restrict__ offsets, int nranks, int rank, int unpack)
{
    const int r0 = blockIdx.y * SD_PANEL_ROWS;
    if (nranks > 1 && sd_panel_owner(r0, nranks) != rank) return;
    const int nrows = (D - r0 < SD_PANEL_ROWS) ? D - r0 : SD_PANEL_ROWS;
    const int w = W - r0;                           // multiple of 4 when W is
    const long long total4 = (long long)nrows * (w >> 2);
    float* dst = flat + offsets[blockIdx.y];
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total4; idx += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(idx / (w >> 2));
        const int c = (int)(idx - (long long)r * (w >> 2)) << 2;
        float4* g = reinterpret_cast<float4*>(G + (long long)(r0 + r) * ldg + r0 + c);
        float4* f = reinterpret_cast<float4*>(dst + (long long)r * w + c);
        if (unpack) *g = *f; else *f = *g;
    }
}

}  // namespace

struct sd_comm {
    ncclComm_t comm = nullptr;
    bool owned = true;
    int rank = 0, nranks = 1;
    long long* d_offsets = nullptr;     // band offsets of the last packed layout
    std::vector<long long> h_offsets;
    int off_D = -1, off_W = -1;
};

int sd_comm_nccl_check(sd_ctx* ctx, int r, const char* what)
{
    if (r == (int)ncclSuccess) return SD_OK;
    NcclApi& n = nccl();
    return sd_fail(ctx, SD_ERR_CUDA, "NCCL error %d (%s) at %s", r, n.GetErrorString ? n.GetErrorString((ncclResult_t)r) : "?", what);
}

#define SD_NCCL(ctx, call)                                                       \
    do {                                                                         \
        int _r = (int)(call);                                                    \
        if (_r != (int)ncclSuccess) return sd_comm_nccl_check((ctx), _r, #call); \
    } while (0)

bool sd_gram_is_scattered(int D, int64_t ldg, const float* d_G)
{
    return (ldg % 4) == 0 && (reinterpret_cast<uintptr_t>(d_G) & 15) == 0 && D > 2 * SD_PANEL_ROWS;
}

int sd_comm_rank_of(const sd_comm* c) { return c ? c->rank : 0; }
int sd_comm_size_of(const sd_comm* c) { return c ? c->nranks : 1; }

int sd_comm_bcast(sd_ctx* ctx, sd_comm* c, float* d_buf, size_t count, int root, cudaStream_t stream)
{
    if (!c || c->nranks == 1 || count == 0) return SD_OK;
    SD_NCCL(ctx, nccl().Broadcast(d_buf, d_buf, count, ncclFloat32, root, c->comm, stream));
    return SD_OK;
}
int sd_comm_group_start(sd_ctx* ctx) { SD_NCCL(ctx, nccl().GroupStart()); return SD_OK; }
int sd_comm_group_end(sd_ctx* ctx) { SD_NCCL(ctx, nccl().GroupEnd()); return SD_OK; }
int sd_comm_allreduce_f64(sd_ctx* ctx, sd_comm* c, double* d_buf, size_t count, cudaStream_t stream)
{
    if (!c || c->nranks == 1 || count == 0) return SD_OK;
    SD_NCCL(ctx, nccl().AllReduce(d_buf, d_buf, count, ncclFloat64, ncclSum, c->comm, stream));
    return SD_OK;
}

int sd_comm_allreduce_f32(sd_ctx* ctx, sd_comm* c, float* d_buf, size_t count, cudaStream_t stream)
{
    if (!c || c->nranks == 1 || count == 0) return SD_OK;
    SD_NCCL(ctx, nccl().AllReduce(d_buf, d_buf, count, ncclFloat32, ncclSum, c->comm, stream));
    return SD_OK;
}

namespace {

// offsets of the packed bands; returns the total float count
long long band_layout(sd_ctx* ctx, sd_comm* c, int D, int W, int* nbands_out)
{
    const int nb = sd_div_up(D, SD_PANEL_ROWS);
    *nbands_out = nb;
    if (c->off_D == D && c->off_W == W && c->d_offsets) return c->h_offsets[nb];
    c->h_offsets.assign(nb + 1, 0);
    for (int p = 0; p < nb; ++p) {
        const int r0 = p * SD_PANEL_ROWS;
        const int nrows = (D - r0 < SD_PANEL_ROWS) ? D - r0 : SD_PANEL_ROWS;
        c->h_offsets[p + 1] = c->h_offsets[p] + (long long)nrows * (W - r0);
    }
    if (c->d_offsets) { cudaStreamSynchronize(ctx->stream); cudaFree(c->d_offsets); c->d_offsets = nullptr; }
    if (cudaMalloc(&c->d_offsets, (nb + 1) * sizeof(long long)) != cudaSuccess) return -1;
    if (cudaMemcpyAsync(c->d_offsets, c->h_offsets.data(), (nb + 1) * sizeof(long long), cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) return -1;
    cudaStreamSynchronize(ctx->stream);          // h_offsets is pageable
    c->off_D = D; c->off_W = W;
    return c->h_offsets[nb];
}

int gram_exchange(sd_ctx* ctx, sd_comm* c, float* d_G, int64_t ldg, int D, int M, bool scatter)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, c && d_G && D >= 1 && M >= 0 && ldg >= D + M, "bad argument");
    if (c->nranks == 1) return SD_OK;
    NcclApi& n = nccl();
    const int W = (int)ldg;                          // the padding columns travel too (keeps every row a multiple of 4 floats)
    if (!sd_gram_is_scattered(D, ldg, d_G)) {
        // small or unaligned: the whole buffer in one all-reduce (a superset of what the owners need)
        SD_NCCL(ctx, n.AllReduce(d_G, d_G, (size_t)D * ldg, ncclFloat32, ncclSum, c->comm, ctx->stream));
        return SD_OK;
    }
    int nb = 0;
    const long long total = band_layout(ctx, c, D, W, &nb);
    if (total < 0) return sd_fail(ctx, SD_ERR_CUDA, "band layout allocation failed");
    float* flat = (float*)sd_workspace(ctx, SD_WS_GRAM_EXT, (size_t)total * sizeof(float));
    if (!flat) return SD_ERR_CUDA;
    const dim3 grid(64, nb);
    band_copy_kernel<<<grid, 256, 0, ctx->stream>>>(d_G, ldg, D, W, flat, c->d_offsets, 1, 0, 0);
    SD_LAUNCH_CHECK(ctx, "band_copy_kernel(pack)");
    if (!scatter) {
        SD_NCCL(ctx, n.AllReduce(flat, flat, (size_t)total, ncclFloat32, ncclSum, c->comm, ctx->stream));
        band_copy_kernel<<<grid, 256, 0, ctx->stream>>>(d_G, ldg, D, W, flat, c->d_offsets, 1, 0, 1);
        SD_LAUNCH_CHECK(ctx, "band_copy_kernel(unpack)");
    } else {
        // one rooted reduce per band, root = its owner, all in one group (one launch per rank)
        SD_NCCL(ctx, n.GroupStart());
        for (int p = 0; p < nb; ++p) {
            float* b = flat + c->h_offsets[p];
            const size_t cnt = (size_t)(c->h_offsets[p + 1] - c->h_offsets[p]);
            const int root = sd_panel_owner((int64_t)p * SD_PANEL_ROWS, c->nranks);
            int r = (int)n.Reduce(b, b, cnt, ncclFloat32, ncclSum, root, c->comm, ctx->stream);
            if (r != (int)ncclSuccess) { n.GroupEnd(); return sd_comm_nccl_check(ctx, r, "ncclReduce(band)"); }
        }
        SD_NCCL(ctx, n.GroupEnd());
        band_copy_kernel<<<grid, 256, 0, ctx->stream>>>(d_G, ldg, D, W, flat, c->d_offsets, c->nranks, c->rank, 1);
        SD_LAUNCH_CHECK(ctx, "band_copy_kernel(unpack own)");
    }
    return SD_OK;
}

}  // namespace

extern "C" {

int sd_comm_get_unique_id(uint8_t* id_out)
{
    if (!id_out) return SD_ERR_INVALID;
    NcclApi& n = nccl();
    if (!n.handle) return SD_ERR_UNSUPPORTED;
    static_assert(sizeof(ncclUniqueId) == SD_COMM_ID_BYTES, "ncclUniqueId size");
    ncclUniqueId id;
    if (n.GetUniqueId(&id) != ncclSuccess) return SD_ERR_CUDA;
    memcpy(id_out, &id, sizeof(id));
    return SD_OK;
}

int sd_comm_create(sd_ctx* ctx, const uint8_t* id, int rank, int nranks, sd_comm** out)
{
    if (!ctx || !out) return SD_ERR_INVALID;
    *out = nullptr;
    SD_REQUIRE(ctx, nranks >= 1 && rank >= 0 && rank < nranks, "bad rank / nranks");
    sd_comm* c = new sd_comm();
    c->rank = rank;
    c->nranks = nranks;
    if (nranks > 1) {
        SD_REQUIRE(ctx, id != nullptr, "a unique id is needed for more than one rank");
        NcclApi& n = nccl();
        if (!n.handle) { delete c; return sd_fail(ctx, SD_ERR_UNSUPPORTED, "%s", n.error.c_str()); }
        ncclUniqueId uid;
        memcpy(&uid, id, sizeof(uid));
        cudaSetDevice(ctx->device);
        int r = (int)n.CommInitRank(&c->comm, nranks, uid, rank);
        if (r != (int)ncclSuccess) { delete c; return sd_comm_nccl_check(ctx, r, "ncclCommInitRank"); }
    }
    *out = c;
    return SD_OK;
}

int sd_comm_adopt(sd_ctx* ctx, void* nccl_comm, int rank, int nranks, sd_comm** out)
{
    if (!ctx || !out) return SD_ERR_INVALID;
    *out = nullptr;
    SD_REQUIRE(ctx, nranks >= 1 && rank >= 0 && rank < nranks && (nranks == 1 || nccl_comm), "bad argument");
    NcclApi& n = nccl();
    if (nranks > 1 && !n.handle) return sd_fail(ctx, SD_ERR_UNSUPPORTED, "%s", n.error.c_str());
    sd_comm* c = new sd_comm();
    c->comm = (ncclComm_t)nccl_comm;
    c->owned = false;
    c->rank = rank;
    c->nranks = nranks;
    *out = c;
    return SD_OK;
}

void sd_comm_destroy(sd_comm* c)
{
    if (!c) return;
    if (c->d_offsets) cudaFree(c->d_offsets);
    if (c->comm && c->owned) nccl().CommDestroy(c->comm);
    delete c;
}

int sd_comm_rank(const sd_comm* c) { return c ? c->rank : 0; }
int sd_comm_size(const sd_comm* c) { return c ? c->nranks : 1; }

int sd_allreduce_gram(sd_ctx* ctx, sd_comm* comm, float* d_G, int64_t ldg, int D, int M)
{
    return gram_exchange(ctx, comm, d_G, ldg, D, M, false);
}

int sd_reduce_scatter_gram(sd_ctx* ctx, sd_comm* comm, float* d_G, int64_t ldg, int D, int M)
{
    return gram_exchange(ctx, comm, d_G, ldg, D, M, true);
}

int sd_comm_sum_int64(sd_ctx* ctx, sd_comm* c, int64_t* h_value)
{
    if (!ctx || !c || !h_value) return SD_ERR_INVALID;
    if (c->nranks == 1) return SD_OK;
    int64_t* d = reinterpret_cast<int64_t*>(reinterpret_cast<char*>(ctx->d_scratch) + 256);
    int64_t* h = reinterpret_cast<int64_t*>(reinterpret_cast<char*>(ctx->h_scratch) + 256);
    *h = *h_value;
    SD_CUDA(ctx, cudaMemcpyAsync(d, h, sizeof(int64_t), cudaMemcpyHostToDevice, ctx->stream));
    SD_NCCL(ctx, nccl().AllReduce(d, d, 1, ncclInt64, ncclSum, c->comm, ctx->stream));
    SD_CUDA(ctx, cudaMemcpyAsync(h, d, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *h_value = *h;
    return SD_OK;
}

int sd_comm_allgather(sd_ctx* ctx, sd_comm* c, const void* d_send, size_t bytes_per_rank, void* d_recv)
{
    if (!ctx || !c || !d_send || !d_recv) return SD_ERR_INVALID;
    if (c->nranks == 1) {
        if (d_send != d_recv) SD_CUDA(ctx, cudaMemcpyAsync(d_recv, d_send, bytes_per_rank, cudaMemcpyDeviceToDevice, ctx->stream));
        return SD_OK;
    }
    SD_NCCL(ctx, nccl().AllGather(d_send, d_recv, bytes_per_rank, ncclInt8, c->comm, ctx->stream));
    return SD_OK;
}

}  // extern "C"
