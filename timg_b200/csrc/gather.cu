// K7: gather the encoded frames of all ranks onto one rank over NCCL (one process per GPU).
//
// The reference is a single process; this is the one exchange of the sharded path (SURVEY 8e): frames are
// independent units, every rank encodes its own batch, and only the encoded bytes (<< the pixels) travel.
// Fixed-slot protocol, no host synchronisation anywhere:
//   * every rank sends `slot_bytes` of its output buffer (a bound all ranks agree on once, e.g. the largest
//     batch seen during warm-up plus a margin) and its n+1 frame offsets, as grouped ncclSend/ncclRecv;
//   * on the root, rank r's bytes land at dst + r * slot_bytes and a small kernel turns the received
//     relative offsets into absolute ones: frame i of rank r is
//       [dst_offsets[r * (n + 1) + i], dst_offsets[r * (n + 1) + i + 1])  inside dst.
//     A rank whose batch did not fit its slot is flagged in status (bit r), never read past.
// Everything runs on the context's gather stream behind an event on the compute stream, so the kernels of
// the next batch overlap the transfer; b200timg_gather_wait orders later work (or the host) after it.
// NCCL is loaded lazily (dlopen) so that single-GPU users of the library do not need it.
#include <dlfcn.h>
#include <nccl.h>

#include "common.cuh"

namespace b200timg {

struct NcclApi {
    void *lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
};

static NcclApi *nccl_api(b200timg_ctx *ctx) {
    static NcclApi api;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);      // the copy already in the process (e.g. torch's) wins by soname
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (h) {
            api.lib = h;
            api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(h, "ncclGetUniqueId"));
            api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(h, "ncclCommInitRank"));
            api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
            api.GroupStart = reinterpret_cast<decltype(api.GroupStart)>(dlsym(h, "ncclGroupStart"));
            api.GroupEnd = reinterpret_cast<decltype(api.GroupEnd)>(dlsym(h, "ncclGroupEnd"));
            api.Send = reinterpret_cast<decltype(api.Send)>(dlsym(h, "ncclSend"));
            api.Recv = reinterpret_cast<decltype(api.Recv)>(dlsym(h, "ncclRecv"));
            api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(h, "ncclGetErrorString"));
        }
    }
    if (!api.lib || !api.GetUniqueId || !api.CommInitRank || !api.GroupStart || !api.GroupEnd || !api.Send || !api.Recv) {
        if (ctx) ctx->fail(B200TIMG_ENODEV, "gather: libnccl.so.2 could not be loaded");
        return nullptr;
    }
    return &api;
}

#define B2_NCCL(ctx, api, call)                                                              \
    do {                                                                                     \
        ncclResult_t r__ = (call);                                                           \
        if (r__ != ncclSuccess)                                                              \
            return (ctx)->fail(B200TIMG_ECUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call,  \
                               (api)->GetErrorString ? (api)->GetErrorString(r__) : "nccl error"); \
    } while (0)

// root: relative offsets of every rank -> absolute positions in dst; status bit r = rank r overflowed its slot
__global__ void __launch_bounds__(256)
gather_offsets_kernel(unsigned long long *__restrict__ offs, int nranks, int n1, unsigned long long slot, unsigned int *__restrict__ status) {
    const int r = blockIdx.x;
    unsigned long long *o = offs + (long long)r * n1;
    const unsigned long long total = o[n1 - 1];
    __syncthreads();                                             // everyone has read the total before it is rewritten
    if (threadIdx.x == 0 && total > slot) atomicOr(status, 1u << (r & 31));
    for (int i = threadIdx.x; i < n1; i += blockDim.x) o[i] = (unsigned long long)r * slot + min(o[i], slot);
}

static int gather_streams(b200timg_ctx *ctx) {
    if (ctx->gather_stream) return B200TIMG_OK;
    // highest priority: the NCCL send/recv kernels must get SM slots WHILE the next batch's kernels run -- at equal priority the
    // block scheduler keeps feeding the running compute grid and the transfer only advances in the gaps between kernels;
    // fewer NCCL channels make that worse
    int prio_least = 0, prio_greatest = 0;
    B2_CUDA(ctx, cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest));
    B2_CUDA(ctx, cudaStreamCreateWithPriority(&ctx->gather_stream, cudaStreamNonBlocking, prio_greatest));
    B2_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_gather_ready, cudaEventDisableTiming));
    for (auto &e : ctx->ev_gather_done) B2_CUDA(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    return B200TIMG_OK;
}

}  // namespace b200timg

using namespace b200timg;

extern "C" {

int b200timg_gather_unique_id(char *id128) {
    if (!id128) return B200TIMG_EINVAL;
    NcclApi *api = nccl_api(nullptr);
    if (!api) return B200TIMG_ENODEV;
    static_assert(sizeof(ncclUniqueId) == B200TIMG_NCCL_ID_BYTES, "ncclUniqueId size");
    ncclUniqueId id;
    if (api->GetUniqueId(&id) != ncclSuccess) return B200TIMG_ECUDA;
    memcpy(id128, &id, sizeof id);
    return B200TIMG_OK;
}

int b200timg_gather_init(b200timg_ctx *ctx, const char *id128, int rank, int nranks) {
    if (!ctx || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    NcclApi *api = nccl_api(ctx);
    if (!api) return B200TIMG_ENODEV;
    ncclUniqueId id;
    memcpy(&id, id128, sizeof id);
    ncclComm_t comm;
    B2_NCCL(ctx, api, api->CommInitRank(&comm, nranks, id, rank));
    ctx->nccl_comm = comm; ctx->nccl_owned = true; ctx->nccl_rank = rank; ctx->nccl_nranks = nranks;
    return gather_streams(ctx);
}

int b200timg_gather_attach(b200timg_ctx *ctx, void *nccl_comm, int rank, int nranks) {
    if (!ctx || !nccl_comm || nranks < 1 || rank < 0 || rank >= nranks) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!nccl_api(ctx)) return B200TIMG_ENODEV;
    ctx->nccl_comm = nccl_comm; ctx->nccl_owned = false; ctx->nccl_rank = rank; ctx->nccl_nranks = nranks;
    return gather_streams(ctx);
}

void b200timg_gather_shutdown(b200timg_ctx *ctx) {
    if (!ctx) return;
    if (ctx->gather_stream) {
        cudaStreamSynchronize(ctx->gather_stream);
        cudaEventDestroy(ctx->ev_gather_ready);
        for (auto &e : ctx->ev_gather_done) cudaEventDestroy(e);
        cudaStreamDestroy(ctx->gather_stream);
        ctx->gather_stream = nullptr;
    }
    if (ctx->nccl_comm && ctx->nccl_owned) {
        NcclApi *api = nccl_api(nullptr);
        if (api && api->CommDestroy) api->CommDestroy(static_cast<ncclComm_t>(ctx->nccl_comm));
    }
    ctx->nccl_comm = nullptr;
}

int b200timg_gather(b200timg_ctx *ctx, const char *d_payload, const uint64_t *d_offsets, int n_frames, size_t slot_bytes,
                    char *d_dst, uint64_t *d_dst_offsets, uint32_t *d_status, int root) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->nccl_comm) return ctx->fail(B200TIMG_EINVAL, "gather: call b200timg_gather_init or _attach first");
    const int nranks = ctx->nccl_nranks, rank = ctx->nccl_rank;
    if (!d_payload || !d_offsets || n_frames <= 0 || root < 0 || root >= nranks || (rank == root && (!d_dst || !d_dst_offsets)))
        return ctx->fail(B200TIMG_EINVAL, "gather: bad args");
    NcclApi *api = nccl_api(ctx);
    if (!api) return B200TIMG_ENODEV;
    ncclComm_t comm = static_cast<ncclComm_t>(ctx->nccl_comm);
    cudaStream_t gs = ctx->gather_stream;
    const size_t n1 = (size_t)n_frames + 1;
    // the payload is ready once the compute stream gets here
    B2_CUDA(ctx, cudaEventRecord(ctx->ev_gather_ready, ctx->stream));
    B2_CUDA(ctx, cudaStreamWaitEvent(gs, ctx->ev_gather_ready, 0));
    if (rank == root) {
        if (!d_status) { B2_CUDA(ctx, ctx->gather_status.reserve(64)); d_status = ctx->gather_status.as<uint32_t>(); }
        B2_CUDA(ctx, cudaMemsetAsync(d_status, 0, sizeof(uint32_t), gs));
        B2_CUDA(ctx, cudaMemcpyAsync(d_dst + (size_t)root * slot_bytes, d_payload, slot_bytes, cudaMemcpyDeviceToDevice, gs));
        B2_CUDA(ctx, cudaMemcpyAsync(d_dst_offsets + (size_t)root * n1, d_offsets, n1 * sizeof(uint64_t), cudaMemcpyDeviceToDevice, gs));
        B2_NCCL(ctx, api, api->GroupStart());
        for (int r = 0; r < nranks; ++r) {
            if (r == root) continue;
            B2_NCCL(ctx, api, api->Recv(d_dst_offsets + (size_t)r * n1, n1, ncclUint64, r, comm, gs));
            B2_NCCL(ctx, api, api->Recv(d_dst + (size_t)r * slot_bytes, slot_bytes, ncclUint8, r, comm, gs));
        }
        B2_NCCL(ctx, api, api->GroupEnd());
        ctx->pending_kernel = "gather_offsets_kernel";
        gather_offsets_kernel<<<nranks, 256, 0, gs>>>(reinterpret_cast<unsigned long long *>(d_dst_offsets), nranks, (int)n1,
                                                       (unsigned long long)slot_bytes, d_status);
        ctx->launches++;
        B2_CUDA(ctx, cudaGetLastError());
    } else {
        B2_NCCL(ctx, api, api->GroupStart());
        B2_NCCL(ctx, api, api->Send(d_offsets, n1, ncclUint64, root, comm, gs));
        B2_NCCL(ctx, api, api->Send(d_payload, slot_bytes, ncclUint8, root, comm, gs));
        B2_NCCL(ctx, api, api->GroupEnd());
    }
    const int ticket = (int)(ctx->gather_seq++ & 0x3fffffff);
    B2_CUDA(ctx, cudaEventRecord(ctx->ev_gather_done[ticket & 3], gs));
    return ticket;
}

// ticket: what b200timg_gather returned.  block_host != 0: return when that gather has completed; else only
// order the compute stream after it.  The last four gathers can be waited for individually.
int b200timg_gather_wait(b200timg_ctx *ctx, int ticket, int block_host) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->gather_stream || ticket < 0) return B200TIMG_OK;
    const long long seq = (long long)(ctx->gather_seq & 0x3fffffff);
    if (seq - ticket > 4 || ticket >= seq) return ctx->fail(B200TIMG_EINVAL, "gather_wait: ticket %d is not one of the last four gathers", ticket);
    if (block_host) B2_CUDA(ctx, cudaEventSynchronize(ctx->ev_gather_done[ticket & 3]));
    else B2_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_gather_done[ticket & 3], 0));
    return B200TIMG_OK;
}

}  // extern "C"
