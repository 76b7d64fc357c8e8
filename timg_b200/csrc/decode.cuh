// What the GIF, JPEG and PNG decoders (gif.cu, jpeg.cu, png_decode.cu) share: the staged upload of a call's
// descriptors and files, the gather of byte runs of those files into one stream, the per-file argument checks and the
// host form of a device decode.  Each decoder keeps its own walk, descriptors, scratch layout and kernels.
#pragma once
#include "common.cuh"

namespace b200timg {

// The call's one host -> device copy through `up`: `host` (laid out with mixed_put), then, when `files` is given, the
// n files back to back from the next 16-byte boundary of `host`, which is returned in *o_files.  The pinned stage is
// rewritten only once the previous copy through `up` has run: the host waits for that copy, not for the kernels after it.
int staged_upload(b200timg_ctx *ctx, Upload &up, std::vector<char> &host, int n = 0, const uint8_t *const *files = nullptr,
                  const size_t *sizes = nullptr, size_t *o_files = nullptr);

// Byte runs of the uploaded files, gathered into one stream by launch_gather: run r is the start[r + 1] - start[r]
// bytes at offset off[r] of the files, and lands at start[r] of the stream.
struct Runs {
    std::vector<unsigned long long> off, start{0};
    size_t o_off = 0, o_start = 0;                 // where put placed off and start in the call's arena
    void add(unsigned long long o, unsigned long long len) { off.push_back(o); start.push_back(start.back() + len); }
    unsigned long long total() const { return start.back(); }
    void put(std::vector<char> &arena) {
        o_off = mixed_put(arena, off.data(), sizeof(unsigned long long) * off.size());
        o_start = mixed_put(arena, start.data(), sizeof(unsigned long long) * start.size());
    }
};

// decode_gather_kernel over the runs: the files are the files_len bytes at d_arena + o_files (bytes past them read as
// 0), the stream is written to d_stream.
int launch_gather(b200timg_ctx *ctx, const Runs &runs, const char *d_arena, size_t o_files, unsigned long long files_len,
                  uint8_t *d_stream);

// The outputs of a *_dev call: canvases of whole RGBA pixels and int32 statuses, neither null, both 4-byte aligned.
int check_dev_outputs(b200timg_ctx *ctx, const char *tag, const void *d_frames, const void *d_status, const char *status_name);

// The n files of a multi-file decode through the format's host walk (`what` names it in errors); every one must be
// taken by the device.
template <class Parse, class Walk>
int parse_files(b200timg_ctx *ctx, const char *tag, const char *what, Walk walk, int n, const uint8_t *const *files,
                const size_t *sizes, std::vector<Parse> &ps) {
    if (n <= 0) return ctx->fail(B200TIMG_EINVAL, "%s: n_files %d <= 0", tag, n);
    if (!files || !sizes) return ctx->fail(B200TIMG_EINVAL, "%s: null files or sizes", tag);
    ps.resize((size_t)n);
    for (int f = 0; f < n; ++f) {
        if (!files[f] || sizes[f] == 0) return ctx->fail(B200TIMG_EINVAL, "%s: file %d has no data", tag, f);
        if (walk(files[f], sizes[f], ps[(size_t)f]) != 0)
            return ctx->fail(B200TIMG_EINVAL, "%s: file %d: stb's %s fails", tag, f, what);
        if (!ps[(size_t)f].supported)
            return ctx->fail(B200TIMG_EINVAL, "%s: file %d is not taken by the device: %s", tag, f, ps[(size_t)f].why);
    }
    return B200TIMG_OK;
}

// The host form of a device decode: launch(d_frames, d_status) decodes into ctx->in_stage, with the n_status int32
// statuses after the canvas_bytes of canvases; both are copied down and the call waits for them.
template <class Launch>
int decode_to_host(b200timg_ctx *ctx, size_t canvas_bytes, int n_status, uint8_t *frames, int32_t *status, Launch launch) {
    B2_CUDA(ctx, ctx->in_stage.reserve(canvas_bytes + 4 * (size_t)n_status + 16));
    B2_CUDA(ctx, ctx->pinned.reserve(4 * (size_t)n_status + 64));
    int32_t *d_status = reinterpret_cast<int32_t *>(ctx->in_stage.as<char>() + (canvas_bytes + 15) / 16 * 16);
    B2_TRY(launch(ctx->in_stage.as<uint8_t>(), d_status));
    B2_CUDA(ctx, cudaMemcpyAsync(frames, ctx->in_stage.p, canvas_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    B2_CUDA(ctx, cudaMemcpyAsync(ctx->pinned.p, d_status, 4 * (size_t)n_status, cudaMemcpyDeviceToHost, ctx->stream));
    B2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(status, ctx->pinned.p, 4 * (size_t)n_status);
    return B200TIMG_OK;
}

}  // namespace b200timg
