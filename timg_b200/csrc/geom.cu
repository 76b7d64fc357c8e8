// Geometry passes around the hot path (SURVEY 8f rank 3 / row a15): byte moves and one reduction, HBM-bound.
//   exif_kernel    ApplyExifOp: mirror, 180 degrees, +-90 degrees               src/jpeg-source.cc:84-119
//   window_kernel  crop (--crop-border: src/graphics-magick-source.cc:232-237) and the wrap-around scroll
//                  window, many positions per launch (Scroll(), :383-389: display(x, y) =
//                  img((x_init + dx*pos + x) % W, (y_init + dy*pos + y) % H))
//   bbox_kernel    --auto-crop: Magick::Image::trim() (:238-240).  GraphicsMagick is not part of the reference
//                  tree; what is implemented is its documented rule with fuzz 0 -- the bounding box of the pixels
//                  that differ from the corner colours (left/top edges against the top-left pixel, right edge
//                  against the top-right, bottom edge against the bottom-left).  PARITY UNPINNED for that rule;
//                  the byte moves are exact by construction and are checked against numpy restatements.
// Algorithmic bytes: 4 B read + 4 B written per output pixel (bbox: 4 B read per pixel).
#include "common.cuh"

namespace b200timg {

__global__ void __launch_bounds__(256)
exif_kernel(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, int w, int h, int mirror, int angle, int n_frames) {
    // output pixel -> source pixel.  The reference applies mirror first, then the rotation.
    const int ow = (angle == 90 || angle == -90) ? h : w, oh = (angle == 90 || angle == -90) ? w : h;
    const long long npx = (long long)ow * oh, total = npx * n_frames;
    for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long long)gridDim.x * blockDim.x) {
        const long long f = g / npx, i = g - f * npx;
        const int oy = (int)(i / ow), ox = (int)(i - (long long)oy * ow);
        int x, y;                                    // position in the mirrored image
        if (angle == 180) { x = w - 1 - ox; y = h - 1 - oy; }              // swap first <-> last pixel (:98-104)
        else if (angle == 90) { x = oy; y = ox; }                           // result(new_x = y, x) = orig(x, y)  (:112-114)
        else if (angle == -90) { x = oy; y = h - 1 - ox; }                  // new_x = h - y - 1
        else { x = ox; y = oy; }
        if (mirror) x = w - 1 - x;                   // row reversed in place before anything else (:88-96)
        out[g] = in[f * (long long)w * h + (long long)y * w + x];
    }
}

// n_pos windows of dw x dh pixels, window k at (x0 + dx * (pos0 + k), y0 + dy * (pos0 + k)), wrapping around
__global__ void __launch_bounds__(256)
window_kernel(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, int w, int h, int dw, int dh, long long x0, long long y0,
              int dx, int dy, long long pos0, int n_pos) {
    const long long npx = (long long)dw * dh, total = npx * n_pos;
    for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long long)gridDim.x * blockDim.x) {
        const long long k = g / npx, i = g - k * npx;
        const int y = (int)(i / dw), x = (int)(i - (long long)y * dw);
        const long long xs = (x0 + (long long)dx * (pos0 + k) + x) % w, ys = (y0 + (long long)dy * (pos0 + k) + y) % h;
        out[g] = in[ys * w + xs];
    }
}

// rect[f] = {min x, min y, max x, max y} of the pixels of frame f that differ from the corner colours; starts as
// {w, h, -1, -1} (an image of one colour has no such pixel)
__global__ void __launch_bounds__(256)
bbox_kernel(const uint32_t *__restrict__ in, int w, int h, int *__restrict__ rect) {
    __shared__ int s[4];
    const int f = blockIdx.y;
    const uint32_t *img = in + (long long)f * w * h;
    const uint32_t tl = img[0], tr = img[w - 1], bl = img[(long long)(h - 1) * w];
    if (threadIdx.x == 0) { s[0] = w; s[1] = h; s[2] = -1; s[3] = -1; }
    __syncthreads();
    int x0 = w, y0 = h, x1 = -1, y1 = -1;
    const long long npx = (long long)w * h;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npx; i += (long long)gridDim.x * blockDim.x) {
        const uint32_t p = img[i];
        const int y = (int)(i / w), x = (int)(i - (long long)y * w);
        if (p != tl) { x0 = min(x0, x); y0 = min(y0, y); }
        if (p != tr) x1 = max(x1, x);
        if (p != bl) y1 = max(y1, y);
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) {
        x0 = min(x0, __shfl_xor_sync(0xffffffffu, x0, d)); y0 = min(y0, __shfl_xor_sync(0xffffffffu, y0, d));
        x1 = max(x1, __shfl_xor_sync(0xffffffffu, x1, d)); y1 = max(y1, __shfl_xor_sync(0xffffffffu, y1, d));
    }
    if ((threadIdx.x & 31) == 0) { atomicMin(&s[0], x0); atomicMin(&s[1], y0); atomicMax(&s[2], x1); atomicMax(&s[3], y1); }
    __syncthreads();
    if (threadIdx.x == 0) {
        int *r = rect + 4 * f;
        atomicMin(&r[0], s[0]); atomicMin(&r[1], s[1]); atomicMax(&r[2], s[2]); atomicMax(&r[3], s[3]);
    }
}

int launch_exif(b200timg_ctx *ctx, const uint8_t *d_in, uint8_t *d_out, int w, int h, int mirror, int angle, int n_frames) {
    if (angle != 0 && angle != 180 && angle != 90 && angle != -90) return ctx->fail(B200TIMG_EINVAL, "exif: angle %d", angle);
    B2_KERNEL(ctx, "exif_kernel");
    exif_kernel<<<grid_for(ctx, (long long)w * h * n_frames), 256, 0, ctx->stream>>>(
        reinterpret_cast<const uint32_t *>(d_in), reinterpret_cast<uint32_t *>(d_out), w, h, mirror ? 1 : 0, angle, n_frames);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

int launch_windows(b200timg_ctx *ctx, const uint8_t *d_in, uint8_t *d_out, int w, int h, int dw, int dh, long long x0, long long y0,
                   int dx, int dy, long long pos0, int n_pos) {
    if (dw <= 0 || dh <= 0 || n_pos <= 0 || x0 < 0 || y0 < 0 || x0 + (long long)dx * pos0 < 0 || y0 + (long long)dy * pos0 < 0 ||
        x0 + (long long)dx * (pos0 + n_pos - 1) < 0 || y0 + (long long)dy * (pos0 + n_pos - 1) < 0)
        return ctx->fail(B200TIMG_EINVAL, "window: negative source position (the reference guarantees none, :372-375)");
    B2_KERNEL(ctx, "window_kernel");
    window_kernel<<<grid_for(ctx, (long long)dw * dh * n_pos), 256, 0, ctx->stream>>>(
        reinterpret_cast<const uint32_t *>(d_in), reinterpret_cast<uint32_t *>(d_out), w, h, dw, dh, x0, y0, dx, dy, pos0, n_pos);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

int launch_bbox(b200timg_ctx *ctx, const uint8_t *d_in, int w, int h, int n_frames, int *d_rect) {
    std::vector<int> init((size_t)4 * n_frames);
    for (int f = 0; f < n_frames; ++f) { init[4 * f] = w; init[4 * f + 1] = h; init[4 * f + 2] = -1; init[4 * f + 3] = -1; }
    B2_CUDA(ctx, cudaMemcpyAsync(d_rect, init.data(), sizeof(int) * init.size(), cudaMemcpyHostToDevice, ctx->stream));
    B2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));            // `init` is a local
    B2_KERNEL(ctx, "bbox_kernel");
    const long long npx = (long long)w * h;
    unsigned bx = (unsigned)std::min<long long>((npx + 255) / 256, (long long)ctx->sm_count * 4);
    bbox_kernel<<<dim3(bx < 1 ? 1 : bx, n_frames), 256, 0, ctx->stream>>>(reinterpret_cast<const uint32_t *>(d_in), w, h, d_rect);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

}  // namespace b200timg

using namespace b200timg;

extern "C" {

// host-buffer forms of the three passes (upload -> kernel -> download)
int b200timg_exif_op(b200timg_ctx *ctx, const uint8_t *fb, int w, int h, int mirror, int angle, uint8_t *out) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!fb || !out || w <= 0 || h <= 0) return ctx->fail(B200TIMG_EINVAL, "exif: bad args");
    const size_t bytes = (size_t)w * h * 4;
    ctx->resident_fb = nullptr;
    B2_CUDA(ctx, ctx->in_stage.reserve(bytes));
    B2_CUDA(ctx, ctx->fb_scaled.reserve(bytes));
    B2_CUDA(ctx, cudaMemcpyAsync(ctx->in_stage.p, fb, bytes, cudaMemcpyHostToDevice, ctx->stream));
    B2_TRY(launch_exif(ctx, ctx->in_stage.as<uint8_t>(), ctx->fb_scaled.as<uint8_t>(), w, h, mirror, angle, 1));
    B2_CUDA(ctx, cudaMemcpyAsync(out, ctx->fb_scaled.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    B2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return B200TIMG_OK;
}

int b200timg_trim_bbox(b200timg_ctx *ctx, const uint8_t *fb, int w, int h, int rect_xywh[4]) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!fb || !rect_xywh || w <= 0 || h <= 0) return ctx->fail(B200TIMG_EINVAL, "trim: bad args");
    const size_t bytes = (size_t)w * h * 4;
    B2_CUDA(ctx, ctx->in_stage.reserve(bytes));
    B2_CUDA(ctx, ctx->misc.reserve(4096));
    B2_CUDA(ctx, ctx->pinned.reserve(64));
    B2_CUDA(ctx, cudaMemcpyAsync(ctx->in_stage.p, fb, bytes, cudaMemcpyHostToDevice, ctx->stream));
    int *d_rect = reinterpret_cast<int *>(ctx->misc.as<char>() + 1024);
    B2_TRY(launch_bbox(ctx, ctx->in_stage.as<uint8_t>(), w, h, 1, d_rect));
    B2_CUDA(ctx, cudaMemcpyAsync(ctx->pinned.p, d_rect, 4 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    B2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const int *r = ctx->pinned.as<int>();
    if (r[2] < r[0] || r[3] < r[1]) { rect_xywh[0] = 0; rect_xywh[1] = 0; rect_xywh[2] = w; rect_xywh[3] = h; }   // nothing to trim against: keep the image
    else { rect_xywh[0] = r[0]; rect_xywh[1] = r[1]; rect_xywh[2] = r[2] - r[0] + 1; rect_xywh[3] = r[3] - r[1] + 1; }
    return B200TIMG_OK;
}

// n_pos windows of dw x dh from one w x h image (crop: n_pos = 1, dx = dy = 0); out: n_pos * dw * dh * 4 bytes
int b200timg_windows(b200timg_ctx *ctx, const uint8_t *img, int w, int h, int dw, int dh, long long x0, long long y0, int dx, int dy,
                     long long first_pos, int n_pos, uint8_t *out) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!img || !out || w <= 0 || h <= 0) return ctx->fail(B200TIMG_EINVAL, "windows: bad args");
    const size_t ib = (size_t)w * h * 4, ob = (size_t)dw * dh * 4 * (size_t)(n_pos > 0 ? n_pos : 0);
    ctx->resident_fb = nullptr;
    B2_CUDA(ctx, ctx->in_stage.reserve(ib));
    B2_CUDA(ctx, ctx->fb_scaled.reserve(ob));
    B2_CUDA(ctx, cudaMemcpyAsync(ctx->in_stage.p, img, ib, cudaMemcpyHostToDevice, ctx->stream));
    B2_TRY(launch_windows(ctx, ctx->in_stage.as<uint8_t>(), ctx->fb_scaled.as<uint8_t>(), w, h, dw, dh, x0, y0, dx, dy, first_pos, n_pos));
    B2_CUDA(ctx, cudaMemcpyAsync(out, ctx->fb_scaled.p, ob, cudaMemcpyDeviceToHost, ctx->stream));
    B2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return B200TIMG_OK;
}

// device-resident forms for pipelines that keep the frames on the GPU
int b200timg_exif_op_dev(b200timg_ctx *ctx, const uint8_t *d_in, uint8_t *d_out, int w, int h, int mirror, int angle, int n_frames) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    return launch_exif(ctx, d_in, d_out, w, h, mirror, angle, n_frames);
}
int b200timg_windows_dev(b200timg_ctx *ctx, const uint8_t *d_img, int w, int h, int dw, int dh, long long x0, long long y0, int dx, int dy,
                         long long first_pos, int n_pos, uint8_t *d_out) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    return launch_windows(ctx, d_img, d_out, w, h, dw, dh, x0, y0, dx, dy, first_pos, n_pos);
}

}  // extern "C"
