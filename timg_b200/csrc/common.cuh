// Shared internals of libb200timg: context, scratch arena, error plumbing and the
// strict-IEEE float helpers every bit-exact kernel uses.
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/b200timg.h"

namespace b200timg {

// A grow-only device buffer (never shrinks; freed with the ctx).
struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = bytes + (bytes >> 3) + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <typename T> T *as() const { return reinterpret_cast<T *>(p); }
};

struct HostBuf {   // pinned staging
    void *p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr; cap = 0;
        size_t want = bytes + (bytes >> 3) + 256;
        cudaError_t e = cudaMallocHost(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
    template <typename T> T *as() const { return reinterpret_cast<T *>(p); }
};

// One caller's host -> device upload (staged_upload, decode.cu): the pinned stage, the device arena it is copied to,
// and the event that says the last copy out of the stage has run.
struct Upload {
    HostBuf stage;
    DevBuf arena;
    cudaEvent_t ev = nullptr;
    void release() { stage.release(); arena.release(); if (ev) cudaEventDestroy(ev); ev = nullptr; }
};

}  // namespace b200timg

namespace b200timg { struct ResamplePlan; void free_plan(ResamplePlan *); }

struct b200timg_ctx {
    int device = 0;
    b200timg::ResamplePlan *plan = nullptr;   // cached resampling tables (host copy) ...
    int plan_key[4] = {0, 0, 0, 0};           // ... for this iw, ih, ow, oh (device copy in `tables`)
    long long fixed_geom_key = -1;            // which tile-origin arrays are uploaded behind ctx->misc + 4096
    size_t sixel_idx_off = 0;                 // where the last sixel encode put its index planes
    const void *resident_fb = nullptr;        // host frame whose copy b200timg_has_transparency left in fb_scaled ...
    int resident_w = 0, resident_h = 0;       // ... (cleared by anything else that writes fb_scaled)
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int sm_count = 132;                       // H100 SXM; replaced by the device's count at ctx creation
    uint64_t launches = 0;
    char err[512] = {0};
    // optional per-kernel timing (b200timg_profile): CUDA events on the launching stream
    bool profiling = false;
    const char *pending_kernel = "?";
    struct ProfRec { const char *name; cudaEvent_t begin, end; };
    std::vector<ProfRec> prof;

    // scratch, grown on demand
    b200timg::DevBuf in_stage;     // uploaded source frames (host entry points)
    b200timg::DevBuf fb_scaled;    // scaled (+padded) RGBA framebuffers of a batch
    b200timg::DevBuf prev_stage;   // previous frame for single-frame delta encode
    b200timg::DevBuf out_stage;    // encoded bytes (host entry points)
    b200timg::DevBuf offsets;      // uint64 [n+1]
    b200timg::DevBuf cells;        // per-cell records of the block encoder
    b200timg::DevBuf rows;         // per-rowpair records
    b200timg::DevBuf tables;       // resampler coefficient tables
    b200timg::DevBuf sixel_work;   // palettes, LUTs, index planes, band tables
    b200timg::DevBuf misc;         // small flags / sizes
    b200timg::DevBuf tri_tables;   // bilinear / YUV scaler tap tables ...
    int tri_key[5] = {0, 0, 0, 0, 0};          // ... for this (kind, iw, ih, ow, oh), device pointers cached in tri_params;
    std::vector<char> tri_params;              // kind names the scaler and, for YUV, the chroma layout
    int yuv_geom[4] = {0, 0, 0, 0};            // window extents of the tiled YUV kernel for the cached key
    bool yuv_geom_valid = false;
    b200timg::DevBuf scale_tmp;    // float4 intermediate + flags of the two-pass scaler (long filters)
    b200timg::DevBuf scale_list;   // work list of tiles the opaque-only scaler hands to the general one
    b200timg::HostBuf pinned;      // staging for sizes / offsets
    b200timg::DevBuf png_sums;     // per frame: Adler-32 and IDAT CRC-32 of the PNG (png.cu)
    b200timg::DevBuf gfx_ids;      // kitty image ids of a graphics batch
    // B200TIMG_DEFLATE (deflate.cu, png.cu): scanline streams, per-segment blocks and their records, the parse's
    // tokens, the PNG files
    b200timg::DevBuf dfl_raw, dfl_scratch, dfl_meta, dfl_tokens, dfl_png;
    // offsets + ids of a graphics batch go up from here; a slot is reused once its copy has run (ev_gfx)
    b200timg::HostBuf gfx_stage[4];
    cudaEvent_t ev_gfx[4] = {nullptr, nullptr, nullptr, nullptr};
    int gfx_slot = 0;
    b200timg::HostBuf pinned_io;   // staging for pageable payloads
    // host-batch pipeline: upload of chunk k+1 / download of chunk k-1 overlap the kernels of chunk k
    cudaStream_t copy_stream = nullptr, d2h_stream = nullptr;
    cudaEvent_t ev_up[2] = {nullptr, nullptr}, ev_write[2] = {nullptr, nullptr}, ev_d2h[2] = {nullptr, nullptr}, ev_scaled[2] = {nullptr, nullptr}, ev_prep = nullptr;
    cudaEvent_t ev_after_scale = nullptr;      // set by the host pipeline: recorded right after the scaler of a batch call
    b200timg::DevBuf pipe_in[2], pipe_out[2];
    bool pipe_ready = false;
    // slices of a large device-resident batch on their own streams (api.cu: sixel_batch_phases)
    cudaStream_t part_stream[4] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t ev_part[4] = {nullptr, nullptr, nullptr, nullptr}, ev_fork = nullptr;
    bool parts_ready = false;
    int part_slot = 0, part_slots = 1, part_max_frames = 0;   // which slice is being launched / how many / frames per slice
    bool sixel_attrs_set = false;            // cudaFuncSetAttribute done for this context's device
    // K7 gather (gather.cu): NCCL communicator (owned or attached), its stream and ordering events
    void *nccl_comm = nullptr;
    bool nccl_owned = false;
    int nccl_rank = 0, nccl_nranks = 1;
    cudaStream_t gather_stream = nullptr;
    cudaEvent_t ev_gather_ready = nullptr, ev_gather_done[4] = {nullptr, nullptr, nullptr, nullptr};
    uint64_t gather_seq = 0;
    b200timg::DevBuf gather_status;
    // One upload per caller, so that a call waits only for the previous copy of its own kind:
    //   mixed batches (b200timg_mixed_batch): the call's tables and descriptors;
    //   GIF decode (gif.cu): file + frame descriptors;
    //   JPEG decode (jpeg.cu): files + descriptors + Huffman tables;
    //   PNG decode (png_decode.cu): files + descriptors;
    //   QOI decode (qoi.cu): files + descriptors;
    //   BMP / TGA / PNM decode (raster.cu): files + descriptors.
    b200timg::Upload mixed_up, gif_up, jpeg_up, png_up, qoi_up, raster_up;
    // the decoders' per-call scratch: GIF code streams, index planes and per-frame reach; JPEG streams, decoder
    // states, coefficients and planes; PNG zlib streams, raw planes, source indices and copy records; QOI tile maps,
    // op records and segment states; RLE TGA tile maps and packet records
    b200timg::DevBuf gif_scratch, jpeg_scratch, png_scratch, qoi_scratch, raster_scratch;

    int fail(int code, const char *fmt, ...) {
        va_list ap; va_start(ap, fmt);
        vsnprintf(err, sizeof err, fmt, ap);
        va_end(ap);
        return code;
    }
};

#define B2_CUDA(ctx, call)                                                         \
    do {                                                                           \
        cudaError_t e__ = (call);                                                  \
        if (e__ != cudaSuccess)                                                    \
            return (ctx)->fail(e__ == cudaErrorMemoryAllocation ? B200TIMG_ENOMEM  \
                                                                : B200TIMG_ECUDA,  \
                               "%s:%d %s -> %s", __FILE__, __LINE__, #call,        \
                               cudaGetErrorString(e__));                           \
    } while (0)

#define B2_KERNEL(ctx, kname)                                                      \
    do {                                                                           \
        (ctx)->pending_kernel = (kname);                                           \
        if ((ctx)->profiling) {                                                    \
            b200timg_ctx::ProfRec r__;                                             \
            r__.name = (kname);                                                    \
            cudaEventCreate(&r__.begin); cudaEventCreate(&r__.end);                \
            cudaEventRecord(r__.begin, (ctx)->stream);                             \
            (ctx)->prof.push_back(r__);                                            \
        }                                                                          \
    } while (0)

#define B2_LAUNCH_CHECK(ctx)                                                       \
    do {                                                                           \
        (ctx)->launches++;                                                         \
        if ((ctx)->profiling && !(ctx)->prof.empty())                              \
            cudaEventRecord((ctx)->prof.back().end, (ctx)->stream);                \
        cudaError_t e__ = cudaGetLastError();                                      \
        if (e__ != cudaSuccess)                                                    \
            return (ctx)->fail(B200TIMG_ECUDA, "%s:%d kernel %s launch -> %s",     \
                               __FILE__, __LINE__, (ctx)->pending_kernel,          \
                               cudaGetErrorString(e__));                           \
    } while (0)

#define B2_TRY(expr)                          \
    do {                                      \
        int rc__ = (expr);                    \
        if (rc__ != B200TIMG_OK) return rc__; \
    } while (0)

namespace b200timg {

// CTAs of `threads` threads for a grid-stride loop over `items`: one item per thread, at most 16 CTAs per SM, at least 1
inline unsigned grid_for(b200timg_ctx *ctx, long long items, int threads = 256) {
    long long b = (items + threads - 1) / threads;
    const long long cap = (long long)ctx->sm_count * 16;
    if (b > cap) b = cap;
    return (unsigned)(b < 1 ? 1 : b);
}

// ---- strict IEEE-754 single precision, never contracted into FMA ------------------
// The reference is compiled for baseline x86-64 (SSE2, no FMA): every * and + rounds
// separately.  These intrinsics map to single SASS FMUL/FADD/MUFU+fixup and are never
// fused by ptxas, independent of -fmad.
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float fsqrt(float a) { return __fsqrt_rn(a); }

// LinearColor::gamma (src/framebuffer.h:169-172): sqrt, saturate at 255, truncate.
__device__ __forceinline__ uint32_t ungamma(float v) {
    const float s = fsqrt(v);
    return (s > 255.0f) ? 255u : __float2uint_rz(s);
}

struct __align__(4) px4 { uint8_t r, g, b, a; };

__device__ __forceinline__ uint32_t pack_rgba(uint32_t r, uint32_t g, uint32_t b, uint32_t a) {
    return r | (g << 8) | (b << 16) | (a << 24);
}

// LinearColor::AlphaBlend + repack (src/framebuffer.h:142-161,169-172) of one RGBA8 pixel onto a
// linearised background colour; opaque pixels pass through.
__device__ __forceinline__ uint32_t blend_px(uint32_t p, float bgr, float bgg, float bgb) {
    const uint32_t a8 = p >> 24;
    if (a8 == 0xffu) return p;
    const uint32_t r8 = p & 0xff, g8 = (p >> 8) & 0xff, b8 = (p >> 16) & 0xff;
    const float a = (float)a8, ia = (float)(0xff - a8);
    const float r = fdiv(fadd(fmul((float)(r8 * r8), a), fmul(bgr, ia)), 255.0f);
    const float g = fdiv(fadd(fmul((float)(g8 * g8), a), fmul(bgg, ia)), 255.0f);
    const float b = fdiv(fadd(fmul((float)(b8 * b8), a), fmul(bgb, ia)), 255.0f);
    return pack_rgba(ungamma(r), ungamma(g), ungamma(b), 0xffu);
}

// What AlphaComposeBackground would do to a pixel at (x, y): resolved once on the host.
struct ComposeSpec {
    int active;                  // 0: leave pixels alone (no getter, transparent bg)
    int use_pattern, pw, ph;
    float bg[2][3];              // linearised background and pattern colours
};
inline ComposeSpec make_compose_spec(int has_bg, uint32_t bg, uint32_t pattern, int pw, int ph) {
    ComposeSpec c;
    c.active = (has_bg && (bg >> 24) != 0) ? 1 : 0;                       // src/framebuffer.cc:111,121
    c.use_pattern = !((pattern >> 24) == 0 || pattern == bg || pw <= 0 || ph <= 0);   // :124-125
    c.pw = pw > 0 ? pw : 1; c.ph = ph > 0 ? ph : 1;
    const uint32_t cols[2] = {bg, pattern};
    for (int k = 0; k < 2; ++k)
        for (int ch = 0; ch < 3; ++ch) { const uint32_t v = (cols[k] >> (8 * ch)) & 0xff; c.bg[k][ch] = (float)(v * v); }
    return c;
}
__device__ __forceinline__ uint32_t compose_at(const ComposeSpec &c, uint32_t p, int x, int y) {
    if (!c.active || (p >> 24) == 0xffu) return p;
    const int sel = c.use_pattern ? (((x / c.pw) + (y / c.ph)) & 1) : 0;
    return blend_px(p, c.bg[sel][0], c.bg[sel][1], c.bg[sel][2]);
}

// per-stage launchers (defined in the .cu files); all device pointers
int launch_compose(b200timg_ctx *ctx, uint8_t *d_fb, int w, int h, int n_frames, int has_bg,
                   uint32_t bg, uint32_t pattern, int pw, int ph, int start_row);
int launch_has_transparency(b200timg_ctx *ctx, const uint8_t *d_fb, int w, int h,
                            int start_row, int *d_flag);
// Block encode of n frames of w x h at d_fb (frame stride w*h*4).  prev_mode: 0 none,
// 1 = explicit d_prev (single frame), 2 = animation (frame f vs f-1, frame 0 full).
int launch_blocks(b200timg_ctx *ctx, const uint8_t *d_fb, const uint8_t *d_prev, int prev_mode,
                  int w, int h, int n_frames, int flags, int x_indent, char *d_out,
                  size_t out_cap, uint64_t *d_offsets);
// cs != nullptr fuses AlphaComposeBackground (start_row 0) into the scaler's epilogue.
// fast != 0: the <= 1 LSB arithmetic (FMA, no 1/255 round trip) where a kernel offers it; 0: bit-exact.
int launch_scale(b200timg_ctx *ctx, const uint8_t *d_in, int iw, int ih, int fmt, uint8_t *d_out,
                 int ow, int oh, int out_frame_rows, int n_frames, const ComposeSpec *cs = nullptr, int fast = 0);
// libswscale-style bilinear (triangle) scalers, bilinear.cu: RGBA -> RGBA and decoder YUV -> RGBA
int launch_scale_bilinear(b200timg_ctx *ctx, const uint8_t *d_in, int iw, int ih, int fmt, uint8_t *d_out, int ow, int oh,
                          int out_frame_rows, int n_frames, const ComposeSpec *cs);
// bytes of one tightly packed frame of a YUV B200TIMG_FMT_* code (0 if fmt is not one), and its argument check
long long yuv_frame_bytes(int fmt, int iw, int ih);
int yuv_check_format(b200timg_ctx *ctx, int fmt, int iw, int ih);
int launch_yuv_scale(b200timg_ctx *ctx, const uint8_t *d_in, int iw, int ih, int fmt, uint8_t *d_out, int ow, int oh,
                     int out_frame_rows, int n_frames);
int launch_sixel(b200timg_ctx *ctx, const uint8_t *d_fb, int w, int h, int n_frames, char *d_out,
                 size_t out_cap, uint64_t *d_offsets, int phases);
int launch_sixel_front(b200timg_ctx *ctx, const uint8_t *d_fb, int w, int h, int n_total, int f0, int n, bool reserve);
int launch_sixel_back(b200timg_ctx *ctx, int w, int h, int n_frames, char *d_out, size_t out_cap, uint64_t *d_offsets, int phases);
// kitty / iTerm2 text of n composed frames at d_out + d_offsets[f] (png.cu); d_ids: kitty image ids.  With
// B200TIMG_DEFLATE the offsets are computed on the device and written to d_offsets.
int launch_graphics(b200timg_ctx *ctx, const uint8_t *d_frames, int w, int h, int n_frames, const b200timg_graphics &gr,
                    const uint32_t *d_ids, uint64_t *d_offsets, char *d_out, size_t out_cap);
// deflate.cu: the dynamic-Huffman blocks of every 65535-byte segment of n scanline streams (frame f at
// d_raw + f * raw_stride) into DFL_SLOT-byte scratch slots, then every block at its bit offset in its frame's PNG slot
struct DeflateSeg { uint32_t bits, stored; };     // the block's size in bits (dynamic) or stored = 1
constexpr long long DFL_SLOT = 65552;             // >= the largest dynamic block kept (65538 bytes) + one zero word
int launch_deflate(b200timg_ctx *ctx, const uint8_t *d_raw, long long raw_stride, int raw_len, int n_frames, int nseg,
                   uint8_t *d_scratch, DeflateSeg *d_info);
int launch_deflate_pack(b200timg_ctx *ctx, const uint8_t *d_raw, long long raw_stride, int raw_len, int n_frames, int nseg,
                        const uint8_t *d_scratch, const DeflateSeg *d_info, const unsigned long long *d_start, uint8_t *d_png,
                        long long png_stride, int zoff);
int sixel_debug_fetch(b200timg_ctx *ctx, uint32_t *h_palette, uint32_t *h_counts, uint8_t *h_index, size_t index_bytes);

// ---- mixed batches (b200timg_mixed_batch) ----------------------------------------------------------------------
// One frame of a mixed batch as the block encoder sees it (blocks.cu).
struct __align__(16) MixedBlocksFrame {
    unsigned long long fb_px;    // first pixel of the scaled frame, in pixels from the batch's framebuffer
    unsigned long long cell0;    // first cell record
    int w, h, cols, rows, row_offset, indent;
};
// Everything the kernels of one mixed call read that the host computes, built once per call and uploaded in one copy
// to ctx->mixed_up.arena: the scaler's tables and frame descriptors (plan_scale_mixed, resample.cu) and the block
// encoder's (plan_blocks_mixed, blocks.cu).
struct MixedPlan {
    std::vector<char> arena;                       // host image of the upload
    size_t o_scale = 0, o_p1 = 0, o_p2 = 0, o_tab = 0, o_blocks = 0, o_rows = 0;   // byte offsets of its parts
    std::vector<unsigned> p1, p2;                  // [n+1] first CTA of each frame in the scaler's two passes
    std::vector<int> group_end;                    // scaler frame groups: frames [previous end, end)
    size_t tmp_elems = 0;                          // float4 intermediate of the largest group
    unsigned long long out_px = 0;                 // scaled pixels of the whole batch
    unsigned rowpairs = 0;                         // block encoder: (frame, row pair) items ...
    unsigned long long cells = 0;                  // ... and cell records
    // sixel encoder (plan_sixel_mixed): arena offsets of its descriptors and item lists, the sizes of its workspace parts
    size_t o_sixel = 0, o_sband = 0, o_scta = 0, o_slist[2] = {0, 0};
    int sixel_list[2] = {0, 0};                    // frames whose median-cut tables fit shared memory / need global memory
    unsigned sixel_bands = 0, sixel_ctas = 0;      // flat (frame, band) and (frame, dither CTA) items
    int sixel_nwarps = 0, sixel_wmax = 0, sixel_split = 0;
    size_t sixel_pal_smem = 0, sixel_ent = 0, sixel_idx = 0, sixel_bnd = 0, sixel_scr = 0, sixel_prog = 0;
    // kitty / iTerm2 encoder (plan_graphics_mixed): arena offsets of its descriptors, item starts, ids and offsets, the
    // lengths of its flat item lists and the sizes of its scratch
    size_t o_gfx = 0, o_gchk = 0, o_gtile = 0, o_ggrid = 0, o_gseg = 0, o_graw = 0, o_gpiece = 0, o_gids = 0, o_goffs = 0;
    unsigned gfx_chk = 0, gfx_tiles = 0, gfx_grid = 0, gfx_segs = 0, gfx_pieces = 0;
    unsigned long long gfx_raw = 0, gfx_raw_slots = 0, gfx_png_slots = 0;
    std::vector<uint64_t> gfx_offsets;             // stored blocks: [n+1] running sum of the frame sizes
};

// The frame that owns flat item `item` of a mixed call's list: the last f with start[f] <= item (frames without items
// share their start).
template <class T>
__device__ __forceinline__ int mixed_owner(const T *__restrict__ start, int n, T item) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (start[mid] <= item) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// ---- kitty / iTerm2 (png.cu, deflate.cu) -----------------------------------------------------------------------
struct PngGeom {
    int w, h, bpp;                 // bpp 4 (RGBA, colour type 6) or 3 (RGB, colour type 2)
    long long row_bytes;           // 1 + w*bpp
    long long raw_len;             // h * row_bytes : the filtered scanline stream
    long long nblocks;             // stored deflate blocks of <= 65535 bytes
    long long zlib_len;            // 2 + 5*nblocks + raw_len + 4
    long long png_len;             // 8 + 25 + 12 + zlib_len + 12
    long long idat_data_off;       // offset of the first zlib byte inside the PNG
};
struct GfxSpec {
    int protocol;                           // B200TIMG_KITTY, B200TIMG_ITERM2 or B200TIMG_KITTY_TMUX
    int w, h;
    long long png_len, tiles;
    int cols, rows, indent;                 // tmux form: the placeholder grid (kitty-canvas.cc:174-176), else 0
};
// One frame of a mixed kitty / iTerm2 batch (plan_graphics_mixed, png.cu).  The tile count and the placeholder grid's
// cols, rows and indent are in s; with B200TIMG_DEFLATE, s describes the stored-size bound.
struct __align__(16) MixedGfxFrame {
    PngGeom g;
    GfxSpec s;
    unsigned long long fb;         // first byte of the scaled frame in launch_scale_mixed's output
    long long raw_off, png_off;    // B200TIMG_DEFLATE: the frame's scanline slot in ctx->dfl_raw, PNG slot in ctx->dfl_png
    unsigned seg0;                 // B200TIMG_DEFLATE: its first 65535-byte segment in the call's flat segment list
    uint32_t ihdr;                 // CRC-32 of its IHDR chunk
};
// appends bytes at a 16-byte boundary of the arena and returns their offset
inline size_t mixed_put(std::vector<char> &a, const void *p, size_t bytes) {
    const size_t o = (a.size() + 15) / 16 * 16;
    a.resize(o + bytes);
    if (bytes) memcpy(a.data() + o, p, bytes);
    return o;
}
// sixel_rows: every frame's output takes round_to_sixel(out_h) rows (the sixel encoder's padded frames)
int plan_scale_mixed(b200timg_ctx *ctx, const b200timg_mixed_batch *b, MixedPlan &mp, bool sixel_rows = false);
int plan_blocks_mixed(b200timg_ctx *ctx, const b200timg_mixed_batch *b, MixedPlan &mp);
// scale + fused compose of every frame into d_out (frames back to back)
int launch_scale_mixed(b200timg_ctx *ctx, const MixedPlan &mp, const char *d_arena, const uint8_t *d_src, uint8_t *d_out,
                       int n_frames, int bgra, const ComposeSpec &cs);
int launch_blocks_mixed(b200timg_ctx *ctx, const MixedPlan &mp, const char *d_arena, const uint8_t *d_fb, int n_frames,
                        int flags, char *d_out, size_t out_cap, uint64_t *d_offsets);
// the sixel encoder's pad strips (rows out_h .. round_to_sixel(out_h) - 1: transparent, then composed) of a plan made
// with sixel_rows
int launch_pad_mixed(b200timg_ctx *ctx, const MixedPlan &mp, const char *d_arena, uint8_t *d_out, int n_frames, const ComposeSpec &cs);
// palette -> table -> map / dither -> emit5 -> layout -> offsets -> compaction of the padded frames of a plan made with
// sixel_rows; plan_sixel_mixed adds the encoder's descriptors to the arena and reserves ctx->sixel_work
int plan_sixel_mixed(b200timg_ctx *ctx, const b200timg_mixed_batch *b, MixedPlan &mp);
int launch_sixel_mixed(b200timg_ctx *ctx, const MixedPlan &mp, const char *d_arena, const uint8_t *d_fb, int n_frames,
                       char *d_out, size_t out_cap, uint64_t *d_offsets);
// kitty / iTerm2 text of the composed frames of a plan made without sixel_rows; plan_graphics_mixed adds the encoder's
// descriptors, item lists, ids and (stored blocks) offsets to the arena
int plan_graphics_mixed(b200timg_ctx *ctx, const b200timg_mixed_batch *b, const b200timg_graphics &gr, MixedPlan &mp);
int launch_graphics_mixed(b200timg_ctx *ctx, const MixedPlan &mp, const char *d_arena, const uint8_t *d_fb, int n_frames,
                          const b200timg_graphics &gr, uint64_t *d_offsets, char *d_out, size_t out_cap);
// deflate.cu over the flat segment list of a mixed batch (seg_start[n_frames + 1], frames' slots in desc)
int launch_deflate_mixed(b200timg_ctx *ctx, const uint8_t *d_raw, const MixedGfxFrame *d_desc, const unsigned *d_seg_start,
                         int n_frames, unsigned n_segs, uint8_t *d_scratch, DeflateSeg *d_info);
int launch_deflate_pack_mixed(b200timg_ctx *ctx, const uint8_t *d_raw, const MixedGfxFrame *d_desc, const unsigned *d_seg_start,
                              int n_frames, unsigned n_segs, const uint8_t *d_scratch, const DeflateSeg *d_info,
                              const unsigned long long *d_start, uint8_t *d_png, int zoff);

}  // namespace b200timg
