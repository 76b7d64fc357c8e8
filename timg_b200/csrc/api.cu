// The extern "C" surface declared in include/b200timg.h: context management, host-buffer
// entry points (upload -> kernels -> download) and the batched pipelines.
#include <algorithm>
#include <cmath>
#include <cstdlib>

#include "decode.cuh"

using namespace b200timg;

namespace {

// Every entry point starts here: a context belongs to one device, whatever the caller's current one is.
int check_ctx(b200timg_ctx *ctx) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    return B200TIMG_OK;
}

// Upload helper: pageable or pinned host memory -> device, async on the ctx stream.
int upload(b200timg_ctx *ctx, void *dst, const void *src, size_t bytes) {
    B2_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return B200TIMG_OK;
}
int download(b200timg_ctx *ctx, void *dst, const void *src, size_t bytes) {
    B2_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    return B200TIMG_OK;
}
int sync(b200timg_ctx *ctx) {
    B2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return B200TIMG_OK;
}

inline int round_to_sixel(int px) { px += 5; return px - px % 6; }   // src/sixel-canvas.cc:91-94

}  // namespace

extern "C" {

int b200timg_version(void) { return 100; }

int b200timg_ctx_create(int device, void *stream, b200timg_ctx **out) {
    if (!out) return B200TIMG_EINVAL;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) {
        cudaGetLastError();
        return B200TIMG_ENODEV;   // no CPU fallback by design
    }
    if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return B200TIMG_ENODEV; }
    b200timg_ctx *ctx = new b200timg_ctx();
    ctx->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) ctx->sm_count = prop.multiProcessorCount;
    if (stream) { ctx->stream = (cudaStream_t)stream; ctx->own_stream = false; }
    else {
        if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {
            delete ctx; return B200TIMG_ECUDA;
        }
        ctx->own_stream = true;
    }
    *out = ctx;
    return B200TIMG_OK;
}

void b200timg_ctx_destroy(b200timg_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (auto &r : ctx->prof) { cudaEventDestroy(r.begin); cudaEventDestroy(r.end); }
    ctx->prof.clear();
    b200timg_gather_shutdown(ctx);
    ctx->gather_status.release();
    ctx->in_stage.release(); ctx->fb_scaled.release(); ctx->prev_stage.release();
    ctx->out_stage.release(); ctx->offsets.release(); ctx->cells.release(); ctx->rows.release();
    ctx->tables.release(); ctx->sixel_work.release(); ctx->misc.release(); ctx->scale_list.release(); ctx->scale_tmp.release(); ctx->tri_tables.release();
    ctx->mixed_up.release(); ctx->gif_up.release(); ctx->jpeg_up.release(); ctx->png_up.release(); ctx->qoi_up.release();
    ctx->raster_up.release();
    ctx->gif_scratch.release(); ctx->jpeg_scratch.release(); ctx->png_scratch.release(); ctx->qoi_scratch.release();
    ctx->raster_scratch.release();
    ctx->pinned.release(); ctx->pinned_io.release();
    ctx->png_sums.release(); ctx->gfx_ids.release();
    ctx->dfl_raw.release(); ctx->dfl_scratch.release(); ctx->dfl_meta.release(); ctx->dfl_tokens.release(); ctx->dfl_png.release();
    for (int i = 0; i < 4; ++i) { ctx->gfx_stage[i].release(); if (ctx->ev_gfx[i]) cudaEventDestroy(ctx->ev_gfx[i]); }
    for (int i = 0; i < 2; ++i) { ctx->pipe_in[i].release(); ctx->pipe_out[i].release(); }
    if (ctx->parts_ready) {
        for (int i = 0; i < 4; ++i) { cudaStreamSynchronize(ctx->part_stream[i]); cudaStreamDestroy(ctx->part_stream[i]); cudaEventDestroy(ctx->ev_part[i]); }
        cudaEventDestroy(ctx->ev_fork);
    }
    if (ctx->pipe_ready) {
        for (int i = 0; i < 2; ++i) { cudaEventDestroy(ctx->ev_up[i]); cudaEventDestroy(ctx->ev_write[i]); cudaEventDestroy(ctx->ev_d2h[i]); cudaEventDestroy(ctx->ev_scaled[i]); }
        cudaEventDestroy(ctx->ev_prep);
        cudaStreamDestroy(ctx->copy_stream); cudaStreamDestroy(ctx->d2h_stream);
    }
    if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
    if (ctx->plan) free_plan(ctx->plan);
    delete ctx;
}

const char *b200timg_last_error(const b200timg_ctx *ctx) { return ctx ? ctx->err : "null ctx"; }
uint64_t b200timg_kernel_launches(const b200timg_ctx *ctx) { return ctx ? ctx->launches : 0; }

// ---- per-kernel timing --------------------------------------------------------------------
int b200timg_profile(b200timg_ctx *ctx, int enable) {
    if (const int rc = check_ctx(ctx)) return rc;
    cudaStreamSynchronize(ctx->stream);
    for (auto &r : ctx->prof) { cudaEventDestroy(r.begin); cudaEventDestroy(r.end); }
    ctx->prof.clear();
    ctx->profiling = enable != 0;
    return B200TIMG_OK;
}

int b200timg_profile_report(b200timg_ctx *ctx, char *buf, size_t cap) {
    if (!ctx || !buf || cap < 2) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    struct Agg { const char *name; int n; double ms; };
    std::vector<Agg> agg;
    for (auto &r : ctx->prof) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, r.begin, r.end) != cudaSuccess) { cudaGetLastError(); continue; }
        bool found = false;
        for (auto &a : agg) if (strcmp(a.name, r.name) == 0) { a.n++; a.ms += ms; found = true; break; }
        if (!found) agg.push_back({r.name, 1, (double)ms});
    }
    size_t pos = 0;
    for (auto &a : agg) {
        const int n = snprintf(buf + pos, cap - pos, "%s %d %.6f\n", a.name, a.n, a.ms);
        if (n < 0 || (size_t)n >= cap - pos) return ctx->fail(B200TIMG_ENOSPC, "profile report truncated");
        pos += (size_t)n;
    }
    buf[pos] = 0;
    return B200TIMG_OK;
}

// Encode n device-resident, already scaled + padded + composed frames (w x h, h % 6 == 0).
int b200timg_sixel_dev(b200timg_ctx *ctx, const uint8_t *d_fb, int w, int h, int n_frames, char *d_out,
                       size_t out_cap, uint64_t *d_offsets) {
    B2_TRY(check_ctx(ctx));
    if (!d_fb || !d_out || !d_offsets || w <= 0 || h <= 0 || n_frames <= 0) return ctx->fail(B200TIMG_EINVAL, "sixel_dev: bad args");
    return launch_sixel(ctx, d_fb, w, h, n_frames, d_out, out_cap, d_offsets, 3);
}

// ---- geometry: ImageSource::CalcScaleToFitDisplay, src/image-source.cc:47-153 ------------
int b200timg_calc_fit(const b200timg_fit_opts *o, int img_w, int img_h, int rotated,
                      int *target_w, int *target_h) {
    if (!o || !target_w || !target_h || img_w <= 0 || img_h <= 0) return B200TIMG_EINVAL;
    int width = o->width, height = o->height;
    bool fill_w = o->fill_width != 0, fill_h = o->fill_height != 0;
    float stretch = o->width_stretch;
    if (rotated) {                                   // :52-56
        std::swap(width, height);
        std::swap(fill_w, fill_h);
        stretch = 1.0f / o->width_stretch;
    }
    const float kMaxAccept = 5.0f;                   // :59-63
    if (stretch > kMaxAccept) stretch = kMaxAccept;
    if (stretch < 1 / kMaxAccept) stretch = 1 / kMaxAccept;
    if (stretch > 1.0f) width = (int)((float)width / stretch);      // :65-70
    else height = (int)((float)height * stretch);
    const float wfrac = (float)width / (float)img_w;
    const float hfrac = (float)height / (float)img_h;
    if (!o->upscale && (fill_h || wfrac > 1.0f) && (fill_w || hfrac > 1.0f)) {   // :75-86
        *target_w = img_w; *target_h = img_h;
        if (o->cell_x_px == 2) { *target_w *= 2; return 1; }
        return 0;
    }
    int tw = width, th = height;
    if (fill_w && fill_h) {
        const float f = wfrac > hfrac ? wfrac : hfrac;
        tw = (int)roundf(f * (float)img_w); th = (int)roundf(f * (float)img_h);
    } else if (fill_h) {
        tw = (int)roundf(hfrac * (float)img_w);
    } else if (fill_w) {
        th = (int)roundf(wfrac * (float)img_h);
    } else {
        const float f = wfrac < hfrac ? wfrac : hfrac;
        tw = (int)roundf(f * (float)img_w); th = (int)roundf(f * (float)img_h);
    }
    if (stretch > 1.0f) tw = (int)((float)tw * stretch);            // :120-125
    else th = (int)((float)th / stretch);
    if (o->cell_x_px > 0 && o->cell_x_px <= 2 && o->cell_y_px > 0 && o->cell_y_px <= 2) {
        tw = tw / o->cell_x_px * o->cell_x_px;                      // :129-133
        th = th / o->cell_y_px * o->cell_y_px;
    }
    if (tw <= 0) tw = 1;
    if (th <= 0) th = 1;
    if (o->upscale_integer && tw > img_w && th > img_h) {           // :139-150
        const float aspect = o->cell_x_px == 2 ? 2.0f : 1.0f;
        const float wf = 1.0f * (float)tw / aspect / (float)img_w;
        const float hf = 1.0f * (float)th / (float)img_h;
        const float smaller = wf < hf ? wf : hf;
        if (smaller > 1.0f) {
            const double fl = std::floor((double)smaller);
            tw = (int)((double)aspect * fl * (double)img_w);
            th = (int)(fl * (double)img_h);
        }
    }
    *target_w = tw; *target_h = th;
    return (tw != img_w || th != img_h) ? 1 : 0;
}

int b200timg_as256(uint32_t p) {   // src/framebuffer.h:37-52
    const uint32_t r = p & 0xff, g = (p >> 8) & 0xff, b = (p >> 16) & 0xff;
    if (r == g && g == b) return (int)((232 + (r * 23 / 255)) & 0xff);
    auto cube = [](uint32_t v) -> uint32_t {
        return v < 47 ? 0 : v < 115 ? 1 : v < 155 ? 2 : v < 195 ? 3 : v < 235 ? 4 : 5;
    };
    return (int)(16 + 36 * cube(r) + 6 * cube(g) + cube(b));
}

// ---- compose ---------------------------------------------------------------------------
int b200timg_compose_dev(b200timg_ctx *ctx, uint8_t *d_fb, int w, int h, int n_frames, int has_bg,
                         uint32_t bg, uint32_t pattern, int pw, int ph, int start_row) {
    B2_TRY(check_ctx(ctx));
    if (!d_fb || w <= 0 || h <= 0 || n_frames <= 0) return ctx->fail(B200TIMG_EINVAL, "compose: bad args");
    return launch_compose(ctx, d_fb, w, h, n_frames, has_bg, bg, pattern, pw, ph, start_row);
}

int b200timg_compose_bg(b200timg_ctx *ctx, uint8_t *fb, int w, int h, int has_bg, uint32_t bg,
                        uint32_t pattern, int pw, int ph, int start_row) {
    B2_TRY(check_ctx(ctx));
    if (!fb || w <= 0 || h <= 0) return ctx->fail(B200TIMG_EINVAL, "compose: bad args");
    const size_t bytes = (size_t)w * h * 4;
    ctx->resident_fb = nullptr;
    B2_CUDA(ctx, ctx->fb_scaled.reserve(bytes));
    B2_TRY(upload(ctx, ctx->fb_scaled.p, fb, bytes));
    B2_TRY(launch_compose(ctx, ctx->fb_scaled.as<uint8_t>(), w, h, 1, has_bg, bg, pattern, pw, ph, start_row));
    B2_TRY(download(ctx, fb, ctx->fb_scaled.p, bytes));
    return sync(ctx);
}

// Compose the frame b200timg_has_transparency uploaded last (same fb, w, h) and download the result: the adapter's
// "scan, ask for the background colour only if needed, compose" costs one upload instead of two.
int b200timg_compose_bg_resident(b200timg_ctx *ctx, uint8_t *fb, int w, int h, int has_bg, uint32_t bg,
                                 uint32_t pattern, int pw, int ph, int start_row) {
    B2_TRY(check_ctx(ctx));
    if (!fb || w <= 0 || h <= 0) return ctx->fail(B200TIMG_EINVAL, "compose: bad args");
    if (ctx->resident_fb != fb || ctx->resident_w != w || ctx->resident_h != h)
        return b200timg_compose_bg(ctx, fb, w, h, has_bg, bg, pattern, pw, ph, start_row);     // nothing resident: plain path
    const size_t bytes = (size_t)w * h * 4;
    B2_TRY(launch_compose(ctx, ctx->fb_scaled.as<uint8_t>(), w, h, 1, has_bg, bg, pattern, pw, ph, start_row));
    B2_TRY(download(ctx, fb, ctx->fb_scaled.p, bytes));
    ctx->resident_fb = nullptr;
    return sync(ctx);
}

int b200timg_has_transparency(b200timg_ctx *ctx, const uint8_t *fb, int w, int h, int start_row,
                              int *result) {
    B2_TRY(check_ctx(ctx));
    if (!fb || !result || w <= 0 || h <= 0) return ctx->fail(B200TIMG_EINVAL, "has_transparency: bad args");
    const size_t bytes = (size_t)w * h * 4;
    B2_CUDA(ctx, ctx->fb_scaled.reserve(bytes));
    B2_CUDA(ctx, ctx->misc.reserve(64));
    B2_CUDA(ctx, ctx->pinned.reserve(64));
    B2_TRY(upload(ctx, ctx->fb_scaled.p, fb, bytes));
    B2_TRY(launch_has_transparency(ctx, ctx->fb_scaled.as<uint8_t>(), w, h, start_row < 0 ? 0 : start_row,
                                   ctx->misc.as<int>()));
    B2_TRY(download(ctx, ctx->pinned.p, ctx->misc.p, sizeof(int)));
    B2_TRY(sync(ctx));
    *result = *ctx->pinned.as<int>() ? 1 : 0;
    ctx->resident_fb = fb; ctx->resident_w = w; ctx->resident_h = h;      // still in ctx->fb_scaled for b200timg_compose_bg_resident
    return B200TIMG_OK;
}

// ---- blocks ----------------------------------------------------------------------------
size_t b200timg_blocks_bound(int w, int h) {   // src/unicode-block-canvas.cc:405-424
    const size_t max_cell = 2 + 5 + 11 + 1 + 5 + 11 + 1 + 3;
    const size_t rows = (size_t)(h + 1) / 2;
    return 9 + rows * (9 + (size_t)w * max_cell + 5);
}

int b200timg_blocks_encode(b200timg_ctx *ctx, const uint8_t *fb, int w, int h, const uint8_t *prev_fb,
                           int flags, int x_indent_cells, char *out, size_t cap, size_t *size) {
    B2_TRY(check_ctx(ctx));
    if (!fb || !size || w <= 0 || h <= 0 || (!out && cap)) return ctx->fail(B200TIMG_EINVAL, "blocks: bad args");
    const size_t bytes = (size_t)w * h * 4;
    const size_t bound = b200timg_blocks_bound(w, h) + 32;
    ctx->resident_fb = nullptr;
    B2_CUDA(ctx, ctx->fb_scaled.reserve(bytes));
    B2_CUDA(ctx, ctx->out_stage.reserve(bound));
    B2_CUDA(ctx, ctx->offsets.reserve(2 * sizeof(uint64_t)));
    B2_CUDA(ctx, ctx->pinned.reserve(64));
    B2_TRY(upload(ctx, ctx->fb_scaled.p, fb, bytes));
    if (prev_fb) {
        B2_CUDA(ctx, ctx->prev_stage.reserve(bytes));
        B2_TRY(upload(ctx, ctx->prev_stage.p, prev_fb, bytes));
    }
    B2_TRY(launch_blocks(ctx, ctx->fb_scaled.as<uint8_t>(), prev_fb ? ctx->prev_stage.as<uint8_t>() : nullptr,
                         prev_fb ? 1 : 0, w, h, 1, flags, x_indent_cells, ctx->out_stage.as<char>(), bound,
                         ctx->offsets.as<uint64_t>()));
    B2_TRY(download(ctx, ctx->pinned.p, ctx->offsets.p, 2 * sizeof(uint64_t)));
    B2_TRY(sync(ctx));
    const size_t n = (size_t)ctx->pinned.as<uint64_t>()[1];
    *size = n;
    if (n > cap) return ctx->fail(B200TIMG_ENOSPC, "blocks: need %zu bytes, have %zu", n, cap);
    if (n) { B2_TRY(download(ctx, out, ctx->out_stage.p, n)); B2_TRY(sync(ctx)); }
    return B200TIMG_OK;
}

// ---- scale -----------------------------------------------------------------------------
int b200timg_scale_dev(b200timg_ctx *ctx, const uint8_t *d_in, int iw, int ih, int fmt, uint8_t *d_out,
                       int ow, int oh, int n_frames) {
    B2_TRY(check_ctx(ctx));
    if (!d_in || !d_out || iw <= 0 || ih <= 0 || ow <= 0 || oh <= 0 || n_frames <= 0)
        return ctx->fail(B200TIMG_EINVAL, "scale: bad args");
    return launch_scale(ctx, d_in, iw, ih, fmt, d_out, ow, oh, oh, n_frames);
}

int b200timg_scale_rgba(b200timg_ctx *ctx, const uint8_t *in, int iw, int ih, int fmt, uint8_t *out,
                        int ow, int oh) {
    return b200timg_scale_rgba_mode(ctx, in, iw, ih, fmt, out, ow, oh, 0);
}

int b200timg_scale_rgba_mode(b200timg_ctx *ctx, const uint8_t *in, int iw, int ih, int fmt, uint8_t *out,
                             int ow, int oh, int fast) {
    B2_TRY(check_ctx(ctx));
    if (!in || !out || iw <= 0 || ih <= 0 || ow <= 0 || oh <= 0) return ctx->fail(B200TIMG_EINVAL, "scale: bad args");
    const size_t ib = (size_t)iw * ih * 4, ob = (size_t)ow * oh * 4;
    B2_CUDA(ctx, ctx->in_stage.reserve(ib));
    ctx->resident_fb = nullptr;
    B2_CUDA(ctx, ctx->fb_scaled.reserve(ob));
    B2_TRY(upload(ctx, ctx->in_stage.p, in, ib));
    if (fast == 2) B2_TRY(launch_scale_bilinear(ctx, ctx->in_stage.as<uint8_t>(), iw, ih, fmt, ctx->fb_scaled.as<uint8_t>(), ow, oh, oh, 1, nullptr));
    else B2_TRY(launch_scale(ctx, ctx->in_stage.as<uint8_t>(), iw, ih, fmt, ctx->fb_scaled.as<uint8_t>(), ow, oh, oh, 1, nullptr, fast));
    B2_TRY(download(ctx, out, ctx->fb_scaled.p, ob));
    return sync(ctx);
}

int b200timg_yuv_scale(b200timg_ctx *ctx, const uint8_t *in, int iw, int ih, int fmt, uint8_t *out, int ow, int oh) {
    B2_TRY(check_ctx(ctx));
    if (!in || !out || iw <= 0 || ih <= 0 || ow <= 0 || oh <= 0)
        return ctx->fail(B200TIMG_EINVAL, "yuv_scale: bad args");
    B2_TRY(yuv_check_format(ctx, fmt, iw, ih));
    const size_t ib = (size_t)yuv_frame_bytes(fmt, iw, ih), ob = (size_t)ow * oh * 4;
    B2_CUDA(ctx, ctx->in_stage.reserve(ib));
    ctx->resident_fb = nullptr;
    B2_CUDA(ctx, ctx->fb_scaled.reserve(ob));
    B2_TRY(upload(ctx, ctx->in_stage.p, in, ib));
    B2_TRY(launch_yuv_scale(ctx, ctx->in_stage.as<uint8_t>(), iw, ih, fmt, ctx->fb_scaled.as<uint8_t>(), ow, oh, oh, 1));
    B2_TRY(download(ctx, out, ctx->fb_scaled.p, ob));
    return sync(ctx);
}

// ---- sixel -----------------------------------------------------------------------------
size_t b200timg_sixel_bound(int w, int h) {
    // our stream: header + <=256 palette definitions; per 6-row band every column has <= 6
    // (colour, bits) entries of <= 8 bytes ("!nnnnn?" gap + char), plus "#ccc" and "$" per colour and
    // column tile (tiles of <= 4096 columns), plus "-"
    const size_t bands = (size_t)(h + 5) / 6, tiles = (size_t)(w + 4095) / 4096;
    return 32 + 256 * 18 + bands * ((size_t)w * 48 + tiles * 256 * 5 + 1) + 2;
}

int b200timg_sixel_encode(b200timg_ctx *ctx, const uint8_t *fb, int w, int h, char *out, size_t cap,
                          size_t *size) {
    B2_TRY(check_ctx(ctx));
    if (!fb || !size || w <= 0 || h <= 0 || (h % 6) != 0 || (!out && cap))
        return ctx->fail(B200TIMG_EINVAL, "sixel: bad args (height must be a multiple of 6)");
    // one pass: the frame is encoded into a device staging buffer of worst-case size, and exactly the
    // encoded bytes come back (or ENOSPC with the size needed, nothing copied)
    const size_t bytes = (size_t)w * h * 4, bound = b200timg_sixel_bound(w, h);
    ctx->resident_fb = nullptr;
    B2_CUDA(ctx, ctx->fb_scaled.reserve(bytes));
    B2_CUDA(ctx, ctx->out_stage.reserve(bound));
    B2_CUDA(ctx, ctx->offsets.reserve(2 * sizeof(uint64_t)));
    B2_CUDA(ctx, ctx->pinned.reserve(64));
    B2_TRY(upload(ctx, ctx->fb_scaled.p, fb, bytes));
    B2_TRY(launch_sixel(ctx, ctx->fb_scaled.as<uint8_t>(), w, h, 1, ctx->out_stage.as<char>(), bound,
                        ctx->offsets.as<uint64_t>(), 3));
    B2_TRY(download(ctx, ctx->pinned.p, ctx->offsets.p, 2 * sizeof(uint64_t)));
    B2_TRY(sync(ctx));
    const size_t n = (size_t)ctx->pinned.as<uint64_t>()[1];
    *size = n;
    if (n > bound) return ctx->fail(B200TIMG_ECUDA, "sixel: encoded size %zu exceeds the bound %zu", n, bound);
    if (n > cap) return ctx->fail(B200TIMG_ENOSPC, "sixel: need %zu bytes, have %zu", n, cap);
    B2_TRY(download(ctx, out, ctx->out_stage.p, n));
    return sync(ctx);
}

int b200timg_sixel_debug(b200timg_ctx *ctx, uint32_t *palette, uint32_t *counts, uint8_t *index, size_t index_bytes) {
    B2_TRY(check_ctx(ctx));
    return sixel_debug_fetch(ctx, palette, counts, index, index_bytes);
}

// ---- batches -----------------------------------------------------------------------------
static int validate_batch(b200timg_ctx *ctx, const b200timg_batch *b) {
    if (!b || b->n_frames <= 0 || b->src_w <= 0 || b->src_h <= 0 || b->out_w <= 0 || b->out_h <= 0)
        return ctx->fail(B200TIMG_EINVAL, "batch: bad geometry");
    return B200TIMG_OK;
}

static size_t src_frame_bytes(const b200timg_batch *b) {
    if (const long long yuv = yuv_frame_bytes(b->src_fmt, b->src_w, b->src_h)) return (size_t)yuv;
    return (size_t)b->src_w * b->src_h * 4;
}

// scale stage of a batch: the STB-semantics scaler (exact or B200TIMG_FAST_SCALE), the libswscale-style bilinear
// one (B200TIMG_BILINEAR_SCALE), or colour conversion + bilinear scaling of decoder YUV in one pass
static int batch_scale(b200timg_ctx *ctx, const b200timg_batch *b, const uint8_t *d_src, uint8_t *d_fb, int frame_rows,
                       const ComposeSpec *cs) {
    const int f = b->src_fmt & 0xf;
    if (yuv_frame_bytes(b->src_fmt, 2, 2))
        return launch_yuv_scale(ctx, d_src, b->src_w, b->src_h, b->src_fmt, d_fb, b->out_w, b->out_h, frame_rows, b->n_frames);
    if (f != B200TIMG_FMT_RGBA && f != B200TIMG_FMT_RGB32) return ctx->fail(B200TIMG_EINVAL, "batch: unknown source format %d", b->src_fmt);
    if (b->flags & B200TIMG_BILINEAR_SCALE)
        return launch_scale_bilinear(ctx, d_src, b->src_w, b->src_h, f, d_fb, b->out_w, b->out_h, frame_rows, b->n_frames, cs);
    return launch_scale(ctx, d_src, b->src_w, b->src_h, f, d_fb, b->out_w, b->out_h, frame_rows, b->n_frames, cs,
                        (b->flags & B200TIMG_FAST_SCALE) != 0);
}

int b200timg_blocks_batch_dev(b200timg_ctx *ctx, const b200timg_batch *b, const uint8_t *d_src,
                              char *d_out, size_t out_cap, uint64_t *d_offsets) {
    B2_TRY(check_ctx(ctx));
    B2_TRY(validate_batch(ctx, b));
    if (!d_src || !d_out || !d_offsets) return ctx->fail(B200TIMG_EINVAL, "batch: null pointer");
    const size_t fb_bytes = (size_t)b->out_w * b->out_h * 4 * b->n_frames;
    ctx->resident_fb = nullptr;
    B2_CUDA(ctx, ctx->fb_scaled.reserve(fb_bytes));
    uint8_t *d_fb = ctx->fb_scaled.as<uint8_t>();
    const ComposeSpec cs = make_compose_spec(b->has_bg, b->bg, b->pattern, b->pattern_w, b->pattern_h);
    B2_TRY(batch_scale(ctx, b, d_src, d_fb, b->out_h, &cs));
    if (ctx->ev_after_scale) B2_CUDA(ctx, cudaEventRecord(ctx->ev_after_scale, ctx->stream));
    return launch_blocks(ctx, d_fb, nullptr, b->animation == 2 ? 3 : b->animation ? 2 : 0, b->out_w, b->out_h, b->n_frames, b->flags,
                         b->x_indent_cells, d_out, out_cap, d_offsets);
}

// One slice of a sixel batch: scale (+ fused compose), pad strip, then the per-frame front kernels.
static int sixel_slice_front(b200timg_ctx *ctx, const b200timg_batch *b, const uint8_t *d_src, int f0, int n, bool reserve) {
    const int hp = round_to_sixel(b->out_h);
    const size_t frame_bytes = (size_t)b->out_w * hp * 4;
    uint8_t *d_fb_all = ctx->fb_scaled.as<uint8_t>(), *d_fb = d_fb_all + (size_t)f0 * frame_bytes;
    // scale with AlphaComposeBackground fused into the epilogue (what the sources do, e.g.
    // src/stb-image-source.cc:56-60); then only the pad strip is cleared and composed, exactly the
    // canvas' own start_row = height call (src/sixel-canvas.cc:115-118).
    const ComposeSpec cs = make_compose_spec(b->has_bg, b->bg, b->pattern, b->pattern_w, b->pattern_h);
    b200timg_batch sub = *b;
    sub.n_frames = n;
    B2_TRY(batch_scale(ctx, &sub, d_src + (size_t)f0 * src_frame_bytes(b), d_fb, hp, &cs));
    if (ctx->ev_after_scale) B2_CUDA(ctx, cudaEventRecord(ctx->ev_after_scale, ctx->stream));
    if (hp != b->out_h) {
        B2_CUDA(ctx, cudaMemset2DAsync(d_fb + (size_t)b->out_h * b->out_w * 4, frame_bytes, 0,
                                       (size_t)(hp - b->out_h) * b->out_w * 4, n, ctx->stream));
        B2_TRY(launch_compose(ctx, d_fb, b->out_w, hp, n, b->has_bg, b->bg, b->pattern, b->pattern_w, b->pattern_h, b->out_h));
    }
    return launch_sixel_front(ctx, d_fb_all, b->out_w, hp, b->n_frames, f0, n, reserve);
}

static int parts_init(b200timg_ctx *ctx) {
    if (ctx->parts_ready) return B200TIMG_OK;
    for (int i = 0; i < 4; ++i) {
        B2_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->part_stream[i], cudaStreamNonBlocking));
        B2_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_part[i], cudaEventDisableTiming));
    }
    B2_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
    ctx->parts_ready = true;
    return B200TIMG_OK;
}

static int sixel_batch_phases(b200timg_ctx *ctx, const b200timg_batch *b, const uint8_t *d_src,
                              char *d_out, size_t out_cap, uint64_t *d_offsets, int phases) {
    const int hp = round_to_sixel(b->out_h);
    if (phases == 2)     // scaled frames are still in ctx->fb_scaled from the prepare phase
        return launch_sixel_back(ctx, b->out_w, hp, b->n_frames, d_out, out_cap, d_offsets, 2);
    // SixelCanvas::Send (src/sixel-canvas.cc:109-120): pad to a multiple of 6 rows with
    // transparent pixels, compose the background into the pad strip only, keep the rest.
    const size_t frame_bytes = (size_t)b->out_w * hp * 4;
    ctx->resident_fb = nullptr;
    B2_CUDA(ctx, ctx->fb_scaled.reserve(frame_bytes * b->n_frames));
    // Large device-resident batches run as slices on separate streams: the palette and dither kernels of a slice are
    // latency-bound (one CTA per frame), so the scaler and the emitter of the other slices fill the machine meanwhile.
    // Timing runs (b200timg_profile) keep the plain in-order chain so that per-kernel durations stay meaningful.
    int parts = 1;
    // slices pay for thousands of small frames (C5); for a batch of some hundred 4K frames a second launch sequence
    // gains nothing, so batches below 512 frames stay one in-order chain
    if (phases == 3 && !ctx->profiling && !ctx->ev_after_scale && b->n_frames >= 512) parts = 4;
    if (const char *e = getenv("B200TIMG_PARTS")) parts = std::max(1, std::min(4, std::min(atoi(e), b->n_frames)));
    if (parts == 1) {
        B2_TRY(sixel_slice_front(ctx, b, d_src, 0, b->n_frames, true));
        return launch_sixel_back(ctx, b->out_w, hp, b->n_frames, d_out, out_cap, d_offsets, phases);
    }
    B2_TRY(parts_init(ctx));
    cudaStream_t main_stream = ctx->stream;
    const int per = (b->n_frames + parts - 1) / parts;
    // everything a slice would allocate is sized for the whole batch first: nothing may be re-allocated while slices run
    ctx->part_slots = parts; ctx->part_max_frames = per;
    B2_CUDA(ctx, cudaEventRecord(ctx->ev_fork, main_stream));
    int rc = B200TIMG_OK;
    for (int k = 0; k < parts && rc == B200TIMG_OK; ++k) {
        const int f0 = k * per, n = std::min(per, b->n_frames - f0);
        if (n <= 0) break;
        ctx->stream = ctx->part_stream[k];
        ctx->part_slot = k;
        if (cudaStreamWaitEvent(ctx->stream, ctx->ev_fork, 0) != cudaSuccess) rc = ctx->fail(B200TIMG_ECUDA, "batch: stream wait failed");
        if (rc == B200TIMG_OK) rc = sixel_slice_front(ctx, b, d_src, f0, n, k == 0);
        if (rc == B200TIMG_OK && cudaEventRecord(ctx->ev_part[k], ctx->stream) != cudaSuccess) rc = ctx->fail(B200TIMG_ECUDA, "batch: event record failed");
        if (rc == B200TIMG_OK && cudaStreamWaitEvent(main_stream, ctx->ev_part[k], 0) != cudaSuccess) rc = ctx->fail(B200TIMG_ECUDA, "batch: stream wait failed");
    }
    ctx->stream = main_stream;
    ctx->part_slot = 0; ctx->part_slots = 1; ctx->part_max_frames = 0;
    if (rc != B200TIMG_OK) {                       // leave no slice running behind the caller's back
        for (int k = 0; k < parts; ++k) cudaStreamSynchronize(ctx->part_stream[k]);
        return rc;
    }
    return launch_sixel_back(ctx, b->out_w, hp, b->n_frames, d_out, out_cap, d_offsets, phases);
}

int b200timg_sixel_batch_dev(b200timg_ctx *ctx, const b200timg_batch *b, const uint8_t *d_src,
                             char *d_out, size_t out_cap, uint64_t *d_offsets) {
    B2_TRY(check_ctx(ctx));
    B2_TRY(validate_batch(ctx, b));
    if (!d_src || !d_out || !d_offsets) return ctx->fail(B200TIMG_EINVAL, "batch: null pointer");
    return sixel_batch_phases(ctx, b, d_src, d_out, out_cap, d_offsets, 3);
}

// ---- kitty / iTerm2 batches ------------------------------------------------------------------
// the protocol description; mixed batches take the tmux indent per frame, so g->indent_cells is read for uniform ones only
static int validate_protocol(b200timg_ctx *ctx, const b200timg_graphics *g, bool uses_indent) {
    if (!g) return ctx->fail(B200TIMG_EINVAL, "graphics: null protocol description");
    const int protocol = g->protocol & ~B200TIMG_DEFLATE;
    if (protocol != B200TIMG_KITTY && protocol != B200TIMG_ITERM2 && protocol != B200TIMG_KITTY_TMUX)
        return ctx->fail(B200TIMG_EINVAL, "graphics: unknown protocol %d", g->protocol);
    if (protocol != B200TIMG_ITERM2 && !g->ids) return ctx->fail(B200TIMG_EINVAL, "graphics: kitty needs one image id per frame (ids is NULL)");
    if (protocol == B200TIMG_KITTY_TMUX && (g->cell_x_px <= 0 || g->cell_y_px <= 0 || (uses_indent && g->indent_cells < 0)))
        return ctx->fail(B200TIMG_EINVAL, "graphics: tmux placeholders need a positive cell size and indent >= 0 (cell %dx%d, indent %d)",
                         g->cell_x_px, g->cell_y_px, uses_indent ? g->indent_cells : 0);
    return B200TIMG_OK;
}

static int validate_graphics(b200timg_ctx *ctx, const b200timg_batch *b, const b200timg_graphics *g) {
    B2_TRY(validate_protocol(ctx, g, true));
    if (b->animation != 0) return ctx->fail(B200TIMG_EINVAL, "graphics: kitty / iTerm2 frames have no delta encoding (animation must be 0)");
    if (b200timg_png_size(b->out_w, b->out_h, g->rgb24) > 0x7fffffffu)
        return ctx->fail(B200TIMG_EINVAL, "graphics: the PNG of a %dx%d frame does not fit one IDAT chunk", b->out_w, b->out_h);
    return B200TIMG_OK;
}

// offsets[0..n]: the running sum of the frame sizes
static void graphics_offsets(const b200timg_batch *b, const b200timg_graphics *g, uint64_t *offsets) {
    offsets[0] = 0;
    const bool kitty = (g->protocol & ~B200TIMG_DEFLATE) != B200TIMG_ITERM2;
    for (int f = 0; f < b->n_frames; ++f) offsets[f + 1] = offsets[f] + b200timg_graphics_size(g, b->out_w, b->out_h, kitty ? g->ids[f] : 0);
}

int b200timg_graphics_batch_dev(b200timg_ctx *ctx, const b200timg_batch *b, const b200timg_graphics *g,
                                const uint8_t *d_src, char *d_out, size_t out_cap, uint64_t *d_offsets) {
    B2_TRY(check_ctx(ctx));
    B2_TRY(validate_batch(ctx, b));
    if (!d_src || !d_out || !d_offsets) return ctx->fail(B200TIMG_EINVAL, "batch: null pointer");
    B2_TRY(validate_graphics(ctx, b, g));
    const int n = b->n_frames;
    const bool kitty = (g->protocol & ~B200TIMG_DEFLATE) != B200TIMG_ITERM2;   // either kitty form: image ids go up too
    const bool deflate = (g->protocol & B200TIMG_DEFLATE) != 0;              // sizes known only on the device
    // offsets (and kitty's ids) are computed here and go up from a pinned slot; the slot is only rewritten once the
    // copy that last read it has run, which never waits unless four batches are queued behind each other
    const int slot = ctx->gfx_slot;
    ctx->gfx_slot = (slot + 1) % 4;
    if (ctx->ev_gfx[slot]) B2_CUDA(ctx, cudaEventSynchronize(ctx->ev_gfx[slot]));
    else B2_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_gfx[slot], cudaEventDisableTiming));
    const size_t off_bytes = (size_t)(n + 1) * sizeof(uint64_t), id_bytes = kitty ? (size_t)n * sizeof(uint32_t) : 0;
    B2_CUDA(ctx, ctx->gfx_stage[slot].reserve(off_bytes + id_bytes));
    uint64_t *h_offs = ctx->gfx_stage[slot].as<uint64_t>();
    if (!deflate) {
        graphics_offsets(b, g, h_offs);
        B2_CUDA(ctx, cudaMemcpyAsync(d_offsets, h_offs, off_bytes, cudaMemcpyHostToDevice, ctx->stream));
    }
    if (kitty) {
        B2_CUDA(ctx, ctx->gfx_ids.reserve(id_bytes));
        memcpy(h_offs + n + 1, g->ids, id_bytes);
        B2_CUDA(ctx, cudaMemcpyAsync(ctx->gfx_ids.p, h_offs + n + 1, id_bytes, cudaMemcpyHostToDevice, ctx->stream));
    }
    B2_CUDA(ctx, cudaEventRecord(ctx->ev_gfx[slot], ctx->stream));
    const size_t fb_bytes = (size_t)b->out_w * b->out_h * 4 * n;
    ctx->resident_fb = nullptr;
    B2_CUDA(ctx, ctx->fb_scaled.reserve(fb_bytes));
    uint8_t *d_fb = ctx->fb_scaled.as<uint8_t>();
    const ComposeSpec cs = make_compose_spec(b->has_bg, b->bg, b->pattern, b->pattern_w, b->pattern_h);
    B2_TRY(batch_scale(ctx, b, d_src, d_fb, b->out_h, &cs));
    if (ctx->ev_after_scale) B2_CUDA(ctx, cudaEventRecord(ctx->ev_after_scale, ctx->stream));
    return launch_graphics(ctx, d_fb, b->out_w, b->out_h, n, *g, ctx->gfx_ids.as<uint32_t>(), d_offsets, d_out, out_cap);
}

static int pipe_init(b200timg_ctx *ctx) {
    if (ctx->pipe_ready) return B200TIMG_OK;
    B2_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
    B2_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->d2h_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
        B2_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_up[i], cudaEventDisableTiming));
        B2_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_write[i], cudaEventDisableTiming));
        B2_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_d2h[i], cudaEventDisableTiming));
        B2_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_scaled[i], cudaEventDisableTiming));
    }
    B2_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_prep, cudaEventDisableTiming));
    ctx->pipe_ready = true;
    return B200TIMG_OK;
}

// Host-buffer batch: the batch is cut into chunks; while chunk k runs its kernels, chunk k+1 is
// uploading and chunk k-1's encoded bytes are downloading (three streams, double-buffered staging).
// Per chunk the encoded size is known before anything is written (sixel), bounded (blocks) or a closed
// formula known before the call (graphics), so the caller's buffer is never overrun and *exactly* the
// encoded bytes cross PCIe on the way back.
enum class Encoder { blocks, sixel, graphics };
static int batch_host_impl(b200timg_ctx *ctx, const b200timg_batch *b, const uint8_t *src, char *out,
                           size_t out_cap, uint64_t *offsets, Encoder enc, const b200timg_graphics *gfx);
static int batch_host(b200timg_ctx *ctx, const b200timg_batch *b, const uint8_t *src, char *out,
                      size_t out_cap, uint64_t *offsets, Encoder enc, const b200timg_graphics *gfx = nullptr) {
    const int rc = batch_host_impl(ctx, b, src, out, out_cap, offsets, enc, gfx);
    if (rc != B200TIMG_OK && ctx && ctx->pipe_ready) {      // nothing may still be reading or writing the caller's buffers
        cudaStreamSynchronize(ctx->copy_stream); cudaStreamSynchronize(ctx->stream); cudaStreamSynchronize(ctx->d2h_stream);
        cudaGetLastError();
    }
    return rc;
}
static int batch_host_impl(b200timg_ctx *ctx, const b200timg_batch *b, const uint8_t *src, char *out,
                           size_t out_cap, uint64_t *offsets, Encoder enc, const b200timg_graphics *gfx) {
    B2_TRY(check_ctx(ctx));
    B2_TRY(validate_batch(ctx, b));
    if (!src || !out || !offsets) return ctx->fail(B200TIMG_EINVAL, "batch: null pointer");
    const bool sixel = enc == Encoder::sixel, graphics = enc == Encoder::graphics;
    // stored-block graphics: every size is known before the call; with B200TIMG_DEFLATE they are read back per chunk,
    // and running short of out_cap still completes offsets[] (nothing more is downloaded)
    const bool deflate = graphics && gfx && (gfx->protocol & B200TIMG_DEFLATE), sized = graphics && !deflate;
    bool short_of_space = false;
    if (graphics) B2_TRY(validate_graphics(ctx, b, gfx));
    if (sized) {                                               // every size is known now: nothing runs if they do not fit
        graphics_offsets(b, gfx, offsets);
        if (offsets[b->n_frames] > out_cap)
            return ctx->fail(B200TIMG_ENOSPC, "batch: need %llu bytes (have %zu)", (unsigned long long)offsets[b->n_frames], out_cap);
    }
    B2_TRY(pipe_init(ctx));
    const size_t frame_bytes = src_frame_bytes(b);
    int chunk = (int)std::max<size_t>(1, ((size_t)672 << 20) / frame_bytes);
    if (const char *e = getenv("B200TIMG_CHUNK_FRAMES")) chunk = std::max(1, atoi(e));      // test knob
    // delta-encoded animations chain frame to frame: every chunk after the first re-uploads its predecessor's last
    // frame as a halo (animation = 2: scaled, used as the reference of the chunk's first frame, not emitted)
    const bool anim = enc == Encoder::blocks && b->animation != 0;
    chunk = std::min(chunk, b->n_frames);
    const int n_chunks = (b->n_frames + chunk - 1) / chunk;
    const size_t blocks_bound = sixel      ? b200timg_sixel_bound(b->out_w, round_to_sixel(b->out_h)) * (size_t)chunk
                                : graphics ? b200timg_graphics_size(gfx, b->out_w, b->out_h, 0xffffffffu) * (size_t)chunk
                                           : b200timg_blocks_bound(b->out_w, b->out_h) * (size_t)chunk + 64;
    for (int i = 0; i < 2 && i < n_chunks; ++i) B2_CUDA(ctx, ctx->pipe_in[i].reserve(frame_bytes * (chunk + 1)));
    B2_CUDA(ctx, ctx->offsets.reserve((size_t)(chunk + 2) * sizeof(uint64_t)));
    B2_CUDA(ctx, ctx->pinned.reserve((size_t)(chunk + 2) * sizeof(uint64_t)));
    uint64_t *h_offs = ctx->pinned.as<uint64_t>();

    auto upload_chunk = [&](int k) -> int {
        const int i = k & 1, halo = (anim && k > 0) ? 1 : 0;
        const int f0 = k * chunk - halo, nf = std::min(chunk, b->n_frames - k * chunk) + halo;
        B2_CUDA(ctx, cudaMemcpyAsync(ctx->pipe_in[i].p, src + (size_t)f0 * frame_bytes, frame_bytes * nf,
                                     cudaMemcpyHostToDevice, ctx->copy_stream));
        B2_CUDA(ctx, cudaEventRecord(ctx->ev_up[i], ctx->copy_stream));
        return B200TIMG_OK;
    };
    B2_TRY(upload_chunk(0));
    if (n_chunks > 1) B2_TRY(upload_chunk(1));
    size_t base_bytes = 0;
    if (!sized) offsets[0] = 0;
    for (int k = 0; k < n_chunks; ++k) {
        const int i = k & 1, f0 = k * chunk, nf = std::min(chunk, b->n_frames - f0);
        const int halo = (anim && k > 0) ? 1 : 0;             // the sub-batch then starts one frame early
        b200timg_batch sub = *b;
        sub.n_frames = nf + halo;
        if (halo) sub.animation = 2;
        const uint8_t *d_in = ctx->pipe_in[i].as<uint8_t>();
        B2_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_up[i], 0));
        if (k >= 2) B2_CUDA(ctx, cudaEventSynchronize(ctx->ev_d2h[i]));            // pipe_out[i] is free again
        B2_CUDA(ctx, ctx->pipe_out[i].reserve(blocks_bound));
        ctx->ev_after_scale = ctx->ev_scaled[i];                                   // recorded once pipe_in[i] has been consumed
        b200timg_graphics sub_gfx = {};
        if (graphics) {                                        // field by field: the tmux fields exist only where they are read
            sub_gfx.protocol = gfx->protocol;
            sub_gfx.rgb24 = gfx->rgb24;
            sub_gfx.ids = gfx->ids ? gfx->ids + f0 : nullptr;
            if ((gfx->protocol & ~B200TIMG_DEFLATE) == B200TIMG_KITTY_TMUX) {
                sub_gfx.cell_x_px = gfx->cell_x_px;
                sub_gfx.cell_y_px = gfx->cell_y_px;
                sub_gfx.indent_cells = gfx->indent_cells;
            }
        }
        const int rc_k = sixel ? sixel_batch_phases(ctx, &sub, d_in, ctx->pipe_out[i].as<char>(), blocks_bound, ctx->offsets.as<uint64_t>(), 3)
                       : graphics ? b200timg_graphics_batch_dev(ctx, &sub, &sub_gfx, d_in, ctx->pipe_out[i].as<char>(), blocks_bound,
                                                                ctx->offsets.as<uint64_t>())
                                  : b200timg_blocks_batch_dev(ctx, &sub, d_in, ctx->pipe_out[i].as<char>(), blocks_bound,
                                                              ctx->offsets.as<uint64_t>());
        ctx->ev_after_scale = nullptr;
        B2_TRY(rc_k);
        if (k + 2 < n_chunks) {                                                    // refill pipe_in[i] as soon as this chunk's scaler is done
            B2_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_scaled[i], 0));
            B2_TRY(upload_chunk(k + 2));
        }
        size_t total = 0;
        if (sized) total = (size_t)(offsets[f0 + nf] - offsets[f0]);              // known before the call
        else {
            B2_CUDA(ctx, cudaMemcpyAsync(h_offs, ctx->offsets.p, (size_t)(nf + halo + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
            B2_CUDA(ctx, cudaEventRecord(ctx->ev_prep, ctx->stream));
            B2_CUDA(ctx, cudaEventSynchronize(ctx->ev_prep));                      // sizes of this chunk are on the host
            total = (size_t)h_offs[nf + halo];                                     // a halo frame contributes no bytes
            for (int j = 1; j <= nf; ++j) offsets[f0 + j] = base_bytes + h_offs[j + halo];
        }
        if (deflate && (short_of_space || base_bytes + total > out_cap)) {
            short_of_space = true;
            base_bytes += total;
            continue;
        }
        if (base_bytes + total > out_cap) {
            return ctx->fail(B200TIMG_ENOSPC, "batch: need more than %zu bytes (have %zu)", base_bytes + total, out_cap);
        }
        if (total > blocks_bound) return ctx->fail(B200TIMG_ECUDA, "batch: encoded size %zu exceeds the staging bound %zu", total, blocks_bound);
        B2_CUDA(ctx, cudaEventRecord(ctx->ev_write[i], ctx->stream));
        B2_CUDA(ctx, cudaStreamWaitEvent(ctx->d2h_stream, ctx->ev_write[i], 0));
        if (total) B2_CUDA(ctx, cudaMemcpyAsync(out + base_bytes, ctx->pipe_out[i].p, total, cudaMemcpyDeviceToHost, ctx->d2h_stream));
        B2_CUDA(ctx, cudaEventRecord(ctx->ev_d2h[i], ctx->d2h_stream));
        base_bytes += total;
    }
    B2_CUDA(ctx, cudaStreamSynchronize(ctx->d2h_stream));
    if (short_of_space) {
        B2_TRY(sync(ctx));
        return ctx->fail(B200TIMG_ENOSPC, "batch: need %zu bytes (have %zu)", base_bytes, out_cap);
    }
    return sync(ctx);
}

// ---- mixed batches ------------------------------------------------------------------------------------------------
static int validate_mixed(b200timg_ctx *ctx, const b200timg_mixed_batch *b, bool blocks) {
    if (!b || b->n_frames <= 0 || !b->frames)
        return ctx->fail(B200TIMG_EINVAL, "mixed batch: needs n_frames > 0 and a frames array (n_frames %d, frames %s)",
                         b ? b->n_frames : 0, b && b->frames ? "set" : "NULL");
    if (b->n_frames > 65535) return ctx->fail(B200TIMG_EINVAL, "mixed batch: %d frames, at most 65535 per call", b->n_frames);
    if (b->src_fmt != B200TIMG_FMT_RGBA && b->src_fmt != B200TIMG_FMT_RGB32)
        return ctx->fail(B200TIMG_EINVAL, "mixed batch: source format %d is not RGBA or RGB32 (YUV sources are not supported)", b->src_fmt);
    if (b->flags & B200TIMG_BILINEAR_SCALE)
        return ctx->fail(B200TIMG_EINVAL, "mixed batch: B200TIMG_BILINEAR_SCALE is not supported (the STB scaler only)");
    for (int f = 0; f < b->n_frames; ++f) {
        const b200timg_frame &F = b->frames[f];
        if (F.src_w <= 0 || F.src_h <= 0 || F.out_w <= 0 || F.out_h <= 0)
            return ctx->fail(B200TIMG_EINVAL, "mixed batch: frame %d: non-positive size %dx%d -> %dx%d", f, F.src_w, F.src_h, F.out_w, F.out_h);
        if (F.src_offset & 3)
            return ctx->fail(B200TIMG_EINVAL, "mixed batch: frame %d: src_offset %llu is not a multiple of 4", f,
                             (unsigned long long)F.src_offset);
        if (F.x_indent_cells < 0) return ctx->fail(B200TIMG_EINVAL, "mixed batch: frame %d: negative indent %d", f, F.x_indent_cells);
        if (blocks && (b->flags & B200TIMG_QUARTER) && (F.out_w & 1))
            return ctx->fail(B200TIMG_EINVAL, "mixed batch: frame %d: quarter blocks need an even width (got %d); the "
                             "reference reads past the row end there", f, F.out_w);
    }
    return B200TIMG_OK;
}

int b200timg_scale_mixed_dev(b200timg_ctx *ctx, const b200timg_mixed_batch *b, const uint8_t *d_src, uint8_t *d_out) {
    B2_TRY(check_ctx(ctx));
    B2_TRY(validate_mixed(ctx, b, false));
    if (!d_src || !d_out) return ctx->fail(B200TIMG_EINVAL, "mixed batch: null pointer");
    if ((reinterpret_cast<uintptr_t>(d_src) | reinterpret_cast<uintptr_t>(d_out)) & 3)
        return ctx->fail(B200TIMG_EINVAL, "mixed batch: pixel buffers must be 4-byte aligned");
    MixedPlan mp;
    B2_TRY(plan_scale_mixed(ctx, b, mp));
    B2_TRY(staged_upload(ctx, ctx->mixed_up, mp.arena));
    const ComposeSpec cs = make_compose_spec(b->has_bg, b->bg, b->pattern, b->pattern_w, b->pattern_h);
    return launch_scale_mixed(ctx, mp, ctx->mixed_up.arena.as<char>(), d_src, d_out, b->n_frames, b->src_fmt == B200TIMG_FMT_RGB32, cs);
}

int b200timg_blocks_mixed_dev(b200timg_ctx *ctx, const b200timg_mixed_batch *b, const uint8_t *d_src,
                              char *d_out, size_t out_cap, uint64_t *d_offsets) {
    B2_TRY(check_ctx(ctx));
    B2_TRY(validate_mixed(ctx, b, true));
    if (!d_src || !d_out || !d_offsets) return ctx->fail(B200TIMG_EINVAL, "mixed batch: null pointer");
    if (reinterpret_cast<uintptr_t>(d_src) & 3) return ctx->fail(B200TIMG_EINVAL, "mixed batch: pixel buffers must be 4-byte aligned");
    MixedPlan mp;
    B2_TRY(plan_scale_mixed(ctx, b, mp));
    B2_TRY(plan_blocks_mixed(ctx, b, mp));
    ctx->resident_fb = nullptr;
    B2_CUDA(ctx, ctx->fb_scaled.reserve((size_t)mp.out_px * 4));
    B2_TRY(staged_upload(ctx, ctx->mixed_up, mp.arena));
    const ComposeSpec cs = make_compose_spec(b->has_bg, b->bg, b->pattern, b->pattern_w, b->pattern_h);
    uint8_t *d_fb = ctx->fb_scaled.as<uint8_t>();
    B2_TRY(launch_scale_mixed(ctx, mp, ctx->mixed_up.arena.as<char>(), d_src, d_fb, b->n_frames, b->src_fmt == B200TIMG_FMT_RGB32, cs));
    return launch_blocks_mixed(ctx, mp, ctx->mixed_up.arena.as<char>(), d_fb, b->n_frames, b->flags, d_out, out_cap, d_offsets);
}

// Host buffers: upload the sources, run the device variant into staging bounded by the sum of the frames' block bounds,
// read the offsets, then download exactly the encoded bytes (or nothing, with ENOSPC).
int b200timg_blocks_mixed(b200timg_ctx *ctx, const b200timg_mixed_batch *b, const uint8_t *src,
                          char *out, size_t out_cap, uint64_t *offsets) {
    B2_TRY(check_ctx(ctx));
    B2_TRY(validate_mixed(ctx, b, true));
    if (!src || !out || !offsets) return ctx->fail(B200TIMG_EINVAL, "mixed batch: null pointer");
    const int n = b->n_frames;
    size_t src_bytes = 0, bound = 64;
    for (int f = 0; f < n; ++f) {
        const b200timg_frame &F = b->frames[f];
        src_bytes = std::max(src_bytes, (size_t)F.src_offset + (size_t)F.src_w * F.src_h * 4);
        bound += b200timg_blocks_bound(F.out_w, F.out_h);
    }
    B2_CUDA(ctx, ctx->in_stage.reserve(src_bytes));
    B2_CUDA(ctx, ctx->out_stage.reserve(bound));
    B2_CUDA(ctx, ctx->offsets.reserve((size_t)(n + 1) * sizeof(uint64_t)));
    B2_CUDA(ctx, ctx->pinned.reserve((size_t)(n + 1) * sizeof(uint64_t)));
    B2_TRY(upload(ctx, ctx->in_stage.p, src, src_bytes));
    B2_TRY(b200timg_blocks_mixed_dev(ctx, b, ctx->in_stage.as<uint8_t>(), ctx->out_stage.as<char>(), bound, ctx->offsets.as<uint64_t>()));
    B2_TRY(download(ctx, ctx->pinned.p, ctx->offsets.p, (size_t)(n + 1) * sizeof(uint64_t)));
    B2_TRY(sync(ctx));
    memcpy(offsets, ctx->pinned.p, (size_t)(n + 1) * sizeof(uint64_t));
    const size_t total = (size_t)offsets[n];
    if (total > bound) return ctx->fail(B200TIMG_ECUDA, "mixed batch: encoded size %zu exceeds the bound %zu", total, bound);
    if (total > out_cap) return ctx->fail(B200TIMG_ENOSPC, "mixed batch: need %zu bytes (have %zu)", total, out_cap);
    if (total) B2_TRY(download(ctx, out, ctx->out_stage.p, total));
    return sync(ctx);
}

// What the sixel encoder cannot take beyond validate_mixed: emit5's entry word holds x in 12 bits (wider frames take the
// look-back emitter of the uniform batch), and the ditherer's per-band progress table holds 2048 bands of 32 rows.
static int validate_sixel_mixed(b200timg_ctx *ctx, const b200timg_mixed_batch *b) {
    B2_TRY(validate_mixed(ctx, b, false));
    for (int f = 0; f < b->n_frames; ++f) {
        const b200timg_frame &F = b->frames[f];
        if (F.out_w > 4095)
            return ctx->fail(B200TIMG_EINVAL, "sixel mixed batch: frame %d: width %d, at most 4095 (use the uniform batch)", f, F.out_w);
        if ((round_to_sixel(F.out_h) + 31) / 32 > 2048)
            return ctx->fail(B200TIMG_EINVAL, "sixel mixed batch: frame %d: height %d, the sixel path takes at most 65536 rows", f, F.out_h);
    }
    return B200TIMG_OK;
}

int b200timg_sixel_mixed_dev(b200timg_ctx *ctx, const b200timg_mixed_batch *b, const uint8_t *d_src,
                             char *d_out, size_t out_cap, uint64_t *d_offsets) {
    B2_TRY(check_ctx(ctx));
    B2_TRY(validate_sixel_mixed(ctx, b));
    if (!d_src || !d_out || !d_offsets) return ctx->fail(B200TIMG_EINVAL, "mixed batch: null pointer");
    if (reinterpret_cast<uintptr_t>(d_src) & 3) return ctx->fail(B200TIMG_EINVAL, "mixed batch: pixel buffers must be 4-byte aligned");
    MixedPlan mp;
    B2_TRY(plan_scale_mixed(ctx, b, mp, true));
    B2_TRY(plan_sixel_mixed(ctx, b, mp));
    ctx->resident_fb = nullptr;
    B2_CUDA(ctx, ctx->fb_scaled.reserve((size_t)mp.out_px * 4));
    B2_TRY(staged_upload(ctx, ctx->mixed_up, mp.arena));
    const ComposeSpec cs = make_compose_spec(b->has_bg, b->bg, b->pattern, b->pattern_w, b->pattern_h);
    uint8_t *d_fb = ctx->fb_scaled.as<uint8_t>();
    const char *d_arena = ctx->mixed_up.arena.as<char>();
    B2_TRY(launch_scale_mixed(ctx, mp, d_arena, d_src, d_fb, b->n_frames, b->src_fmt == B200TIMG_FMT_RGB32, cs));
    B2_TRY(launch_pad_mixed(ctx, mp, d_arena, d_fb, b->n_frames, cs));
    return launch_sixel_mixed(ctx, mp, d_arena, d_fb, b->n_frames, d_out, out_cap, d_offsets);
}

// As b200timg_blocks_mixed: staging bounded by the sum of the frames' sixel bounds, offsets read back, then exactly the
// encoded bytes (or nothing, with ENOSPC).
int b200timg_sixel_mixed(b200timg_ctx *ctx, const b200timg_mixed_batch *b, const uint8_t *src,
                         char *out, size_t out_cap, uint64_t *offsets) {
    B2_TRY(check_ctx(ctx));
    B2_TRY(validate_sixel_mixed(ctx, b));
    if (!src || !out || !offsets) return ctx->fail(B200TIMG_EINVAL, "mixed batch: null pointer");
    const int n = b->n_frames;
    size_t src_bytes = 0, bound = 0;
    for (int f = 0; f < n; ++f) {
        const b200timg_frame &F = b->frames[f];
        src_bytes = std::max(src_bytes, (size_t)F.src_offset + (size_t)F.src_w * F.src_h * 4);
        bound += b200timg_sixel_bound(F.out_w, round_to_sixel(F.out_h));
    }
    B2_CUDA(ctx, ctx->in_stage.reserve(src_bytes));
    B2_CUDA(ctx, ctx->out_stage.reserve(bound));
    B2_CUDA(ctx, ctx->offsets.reserve((size_t)(n + 1) * sizeof(uint64_t)));
    B2_CUDA(ctx, ctx->pinned.reserve((size_t)(n + 1) * sizeof(uint64_t)));
    B2_TRY(upload(ctx, ctx->in_stage.p, src, src_bytes));
    B2_TRY(b200timg_sixel_mixed_dev(ctx, b, ctx->in_stage.as<uint8_t>(), ctx->out_stage.as<char>(), bound, ctx->offsets.as<uint64_t>()));
    B2_TRY(download(ctx, ctx->pinned.p, ctx->offsets.p, (size_t)(n + 1) * sizeof(uint64_t)));
    B2_TRY(sync(ctx));
    memcpy(offsets, ctx->pinned.p, (size_t)(n + 1) * sizeof(uint64_t));
    const size_t total = (size_t)offsets[n];
    if (total > bound) return ctx->fail(B200TIMG_ECUDA, "sixel mixed batch: encoded size %zu exceeds the bound %zu", total, bound);
    if (total > out_cap) return ctx->fail(B200TIMG_ENOSPC, "sixel mixed batch: need %zu bytes (have %zu)", total, out_cap);
    if (total) B2_TRY(download(ctx, out, ctx->out_stage.p, total));
    return sync(ctx);
}

// Only the fields a mixed page reads, so that nothing else of the caller's description reaches the kernels.
static b200timg_graphics graphics_mixed_desc(const b200timg_graphics *g) {
    b200timg_graphics r = {};
    r.protocol = g->protocol;
    r.rgb24 = g->rgb24;
    r.ids = (g->protocol & ~B200TIMG_DEFLATE) != B200TIMG_ITERM2 ? g->ids : nullptr;
    if ((g->protocol & ~B200TIMG_DEFLATE) == B200TIMG_KITTY_TMUX) { r.cell_x_px = g->cell_x_px; r.cell_y_px = g->cell_y_px; }
    return r;
}

int b200timg_graphics_mixed_dev(b200timg_ctx *ctx, const b200timg_mixed_batch *b, const b200timg_graphics *g,
                                const uint8_t *d_src, char *d_out, size_t out_cap, uint64_t *d_offsets) {
    B2_TRY(check_ctx(ctx));
    B2_TRY(validate_mixed(ctx, b, false));
    B2_TRY(validate_protocol(ctx, g, false));
    if (!d_src || !d_out || !d_offsets) return ctx->fail(B200TIMG_EINVAL, "mixed batch: null pointer");
    if (reinterpret_cast<uintptr_t>(d_src) & 3) return ctx->fail(B200TIMG_EINVAL, "mixed batch: pixel buffers must be 4-byte aligned");
    const b200timg_graphics gr = graphics_mixed_desc(g);
    MixedPlan mp;
    B2_TRY(plan_scale_mixed(ctx, b, mp));
    B2_TRY(plan_graphics_mixed(ctx, b, gr, mp));
    ctx->resident_fb = nullptr;
    B2_CUDA(ctx, ctx->fb_scaled.reserve((size_t)mp.out_px * 4));
    B2_TRY(staged_upload(ctx, ctx->mixed_up, mp.arena));
    const ComposeSpec cs = make_compose_spec(b->has_bg, b->bg, b->pattern, b->pattern_w, b->pattern_h);
    uint8_t *d_fb = ctx->fb_scaled.as<uint8_t>();
    const char *d_arena = ctx->mixed_up.arena.as<char>();
    B2_TRY(launch_scale_mixed(ctx, mp, d_arena, d_src, d_fb, b->n_frames, b->src_fmt == B200TIMG_FMT_RGB32, cs));
    return launch_graphics_mixed(ctx, mp, d_arena, d_fb, b->n_frames, gr, d_offsets, d_out, out_cap);
}

// Host buffers.  Stored blocks: every size is known before the call, so ENOSPC comes before anything runs.
// B200TIMG_DEFLATE: staging bounded by the stored sizes, offsets read back, then exactly the encoded bytes (or nothing,
// with ENOSPC and the offsets complete).
int b200timg_graphics_mixed(b200timg_ctx *ctx, const b200timg_mixed_batch *b, const b200timg_graphics *g,
                            const uint8_t *src, char *out, size_t out_cap, uint64_t *offsets) {
    B2_TRY(check_ctx(ctx));
    B2_TRY(validate_mixed(ctx, b, false));
    B2_TRY(validate_protocol(ctx, g, false));
    if (!src || !out || !offsets) return ctx->fail(B200TIMG_EINVAL, "mixed batch: null pointer");
    const int n = b->n_frames;
    const bool deflate = (g->protocol & B200TIMG_DEFLATE) != 0, kitty = (g->protocol & ~B200TIMG_DEFLATE) != B200TIMG_ITERM2;
    size_t src_bytes = 0, bound = 0;
    std::vector<uint64_t> sized(n + 1, 0);
    for (int f = 0; f < n; ++f) {
        const b200timg_frame &F = b->frames[f];
        src_bytes = std::max(src_bytes, (size_t)F.src_offset + (size_t)F.src_w * F.src_h * 4);
        b200timg_graphics gf = graphics_mixed_desc(g);
        gf.indent_cells = F.x_indent_cells;
        if (b200timg_png_size(F.out_w, F.out_h, g->rgb24) > 0x7fffffffu)
            return ctx->fail(B200TIMG_EINVAL, "graphics mixed batch: frame %d: the PNG of a %dx%d frame does not fit one IDAT chunk", f,
                             F.out_w, F.out_h);
        sized[f + 1] = sized[f] + b200timg_graphics_size(&gf, F.out_w, F.out_h, kitty ? g->ids[f] : 0);
    }
    bound = (size_t)sized[n];
    if (!deflate) {
        memcpy(offsets, sized.data(), sizeof(uint64_t) * (n + 1));
        if (bound > out_cap) return ctx->fail(B200TIMG_ENOSPC, "graphics mixed batch: need %zu bytes (have %zu)", bound, out_cap);
    }
    B2_CUDA(ctx, ctx->in_stage.reserve(src_bytes));
    B2_CUDA(ctx, ctx->out_stage.reserve(std::max<size_t>(bound, 1)));
    B2_CUDA(ctx, ctx->offsets.reserve((size_t)(n + 1) * sizeof(uint64_t)));
    B2_CUDA(ctx, ctx->pinned.reserve((size_t)(n + 1) * sizeof(uint64_t)));
    B2_TRY(upload(ctx, ctx->in_stage.p, src, src_bytes));
    B2_TRY(b200timg_graphics_mixed_dev(ctx, b, g, ctx->in_stage.as<uint8_t>(), ctx->out_stage.as<char>(), bound, ctx->offsets.as<uint64_t>()));
    B2_TRY(download(ctx, ctx->pinned.p, ctx->offsets.p, (size_t)(n + 1) * sizeof(uint64_t)));
    B2_TRY(sync(ctx));
    memcpy(offsets, ctx->pinned.p, (size_t)(n + 1) * sizeof(uint64_t));
    const size_t total = (size_t)offsets[n];
    if (total > bound) return ctx->fail(B200TIMG_ECUDA, "graphics mixed batch: encoded size %zu exceeds the bound %zu", total, bound);
    if (total > out_cap) return ctx->fail(B200TIMG_ENOSPC, "graphics mixed batch: need %zu bytes (have %zu)", total, out_cap);
    if (total) B2_TRY(download(ctx, out, ctx->out_stage.p, total));
    return sync(ctx);
}

int b200timg_blocks_batch(b200timg_ctx *ctx, const b200timg_batch *b, const uint8_t *src, char *out,
                          size_t out_cap, uint64_t *offsets) {
    return batch_host(ctx, b, src, out, out_cap, offsets, Encoder::blocks);
}
int b200timg_sixel_batch(b200timg_ctx *ctx, const b200timg_batch *b, const uint8_t *src, char *out,
                         size_t out_cap, uint64_t *offsets) {
    return batch_host(ctx, b, src, out, out_cap, offsets, Encoder::sixel);
}
int b200timg_graphics_batch(b200timg_ctx *ctx, const b200timg_batch *b, const b200timg_graphics *g, const uint8_t *src,
                            char *out, size_t out_cap, uint64_t *offsets) {
    return batch_host(ctx, b, src, out, out_cap, offsets, Encoder::graphics, g);
}

}  // extern "C"
