// The decoders' shared host plumbing and their gather kernel (decode.cuh).
#include "decode.cuh"

namespace b200timg {

namespace {

// item g of the stream: byte g - run_start[r] of run r (0 past the end of the files)
__global__ void __launch_bounds__(256)
decode_gather_kernel(const uint8_t *__restrict__ files, unsigned long long size, const unsigned long long *__restrict__ run_off,
                     const unsigned long long *__restrict__ run_start, int n_runs, uint8_t *__restrict__ stream) {
    const unsigned long long total = n_runs > 0 ? run_start[n_runs] : 0;
    for (unsigned long long g = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; g < total;
         g += (unsigned long long)gridDim.x * blockDim.x) {
        const int r = mixed_owner(run_start, n_runs, g);
        const unsigned long long o = run_off[r] + (g - run_start[r]);
        stream[g] = o < size ? files[o] : 0;
    }
}

}  // namespace

int staged_upload(b200timg_ctx *ctx, Upload &up, std::vector<char> &host, int n, const uint8_t *const *files,
                  const size_t *sizes, size_t *o_files) {
    if (files) *o_files = mixed_put(host, nullptr, 0);
    size_t bytes = host.size();
    for (int f = 0; f < n; ++f) bytes += sizes[f];
    if (up.ev) B2_CUDA(ctx, cudaEventSynchronize(up.ev));
    else B2_CUDA(ctx, cudaEventCreateWithFlags(&up.ev, cudaEventDisableTiming));
    B2_CUDA(ctx, up.stage.reserve(bytes));
    B2_CUDA(ctx, up.arena.reserve(bytes));
    memcpy(up.stage.p, host.data(), host.size());
    char *dst = up.stage.as<char>() + host.size();
    for (int f = 0; f < n; ++f) { memcpy(dst, files[f], sizes[f]); dst += sizes[f]; }
    B2_CUDA(ctx, cudaMemcpyAsync(up.arena.p, up.stage.p, bytes, cudaMemcpyHostToDevice, ctx->stream));
    B2_CUDA(ctx, cudaEventRecord(up.ev, ctx->stream));
    return B200TIMG_OK;
}

int launch_gather(b200timg_ctx *ctx, const Runs &runs, const char *d_arena, size_t o_files, unsigned long long files_len,
                  uint8_t *d_stream) {
    B2_KERNEL(ctx, "decode_gather_kernel");
    decode_gather_kernel<<<grid_for(ctx, (long long)runs.total()), 256, 0, ctx->stream>>>(
        reinterpret_cast<const uint8_t *>(d_arena + o_files), files_len,
        reinterpret_cast<const unsigned long long *>(d_arena + runs.o_off),
        reinterpret_cast<const unsigned long long *>(d_arena + runs.o_start), (int)runs.off.size(), d_stream);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

int check_dev_outputs(b200timg_ctx *ctx, const char *tag, const void *d_frames, const void *d_status, const char *status_name) {
    if (!d_frames || !d_status) return ctx->fail(B200TIMG_EINVAL, "%s: null output", tag);
    if (reinterpret_cast<uintptr_t>(d_frames) % 4 || reinterpret_cast<uintptr_t>(d_status) % 4)
        return ctx->fail(B200TIMG_EINVAL, "%s: d_frames and %s must be 4-byte aligned (whole RGBA pixels, int32)", tag,
                         status_name);
    return B200TIMG_OK;
}

}  // namespace b200timg
