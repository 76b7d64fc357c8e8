/* b200timg.h -- C ABI of the H100-native timg hot path.
 *
 * Drop-in boundary for hzeller/timg's per-pixel hot path (paths below are relative to
 * the reference tree):
 *   scale      ImageScaler::Create/Scale                 src/image-scaler.h:33-39, .cc:75-97
 *   compose    Framebuffer::AlphaComposeBackground       src/framebuffer.h:103-106, .cc:108-150
 *   blocks     UnicodeBlockCanvas::Send (+FindBestGlyph, AppendDoubleRow)
 *                                                         src/unicode-block-canvas.cc:162-403
 *   sixel      the libsixel calls inside SixelCanvas::Send's encode lambda
 *                                                         src/sixel-canvas.cc:134-148
 *   geometry   ImageSource::CalcScaleToFitDisplay        src/image-source.cc:47-153
 *
 * Plain pointers and sizes only; no C++/torch types.  All pixel buffers are RGBA8,
 * row-major, tightly packed (src/framebuffer.h:26-61).  Colours passed as uint32_t are
 * the four rgba_t bytes in memory order: r | g<<8 | b<<16 | a<<24.
 *
 * Every entry point runs hand-written sm_90a CUDA kernels.  There is NO CPU fallback:
 * if no CUDA device is usable, b200timg_ctx_create fails with B200TIMG_ENODEV and nothing
 * else can be called.
 *
 * Return value: 0 (B200TIMG_OK) or a negative B200TIMG_E* code; b200timg_last_error()
 * gives a human-readable reason.  The reference's methods return void and cannot fail
 * (src/terminal-canvas.h:39, src/image-scaler.h:38); the adapters in INTEGRATION.md abort
 * on a negative code, which is the reference's behaviour on allocation failure too.
 *
 * Threading: a ctx is thread-compatible (one caller at a time per ctx), like the
 * reference's canvases (src/unicode-block-canvas.h:70-79 are plain members).
 * Current device: every entry point that takes a ctx makes the ctx's device the calling thread's current CUDA
 * device (cudaSetDevice) and leaves it so; hosts that juggle several devices in one thread re-select theirs.
 */
#ifndef B200TIMG_H
#define B200TIMG_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200TIMG_OK        0
#define B200TIMG_EINVAL   (-1)  /* bad argument (null pointer, non-positive size, odd width in quarter mode) */
#define B200TIMG_ENOMEM   (-2)  /* device or pinned-host allocation failed */
#define B200TIMG_ECUDA    (-3)  /* a CUDA call or kernel failed; see b200timg_last_error */
#define B200TIMG_ENOSPC   (-4)  /* caller's output buffer too small; *size holds the needed size */
#define B200TIMG_ENODEV   (-5)  /* no usable CUDA device (this library has no CPU path) */

/* flags for the block encoders: UnicodeBlockCanvas ctor args, src/unicode-block-canvas.h:38-39 */
#define B200TIMG_QUARTER   1    /* use_quarter: 2x2 px per cell instead of 1x2 */
#define B200TIMG_UPPER     2    /* use_upper_half_block (TIMG_USE_UPPER_BLOCK) */
#define B200TIMG_COLOR8    4    /* use_256_color (--color8) */
/* batch flag (not a reference option): let the scaler use fused multiply-adds and skip the
 * byte*(1/255) .. *255 round trip where a kernel offers it.  Result within 1 LSB per channel of
 * ImageScaler::Scale's instead of bit-identical.  Meant for -p sixel, whose quantiser is compared
 * by a colour-difference tolerance anyway; never set it for the block modes' byte parity. */
#define B200TIMG_FAST_SCALE 8
/* batch flag: scale RGBA with the libswscale-style bilinear (triangle) filter of the reference's default
 * build (src/image-scaler.cc:45-72) instead of the STB build's Mitchell/box.  libswscale is not part of
 * the reference tree and its result is version/SIMD dependent: parity unpinned, distance measured in tests. */
#define B200TIMG_BILINEAR_SCALE 16

/* input colour formats: ImageScaler::ColorFmt, src/image-scaler.h:26-29 */
#define B200TIMG_FMT_RGBA  0
#define B200TIMG_FMT_RGB32 1    /* BGRA in memory */
/* decoder output of the video source (src/video-source.cc:59-89): planar / semi-planar YUV, converted
 * and scaled to RGBA in one pass (batch entry points and b200timg_yuv_scale only).  A frame is w*h luma bytes
 * followed by the chroma planes (I420: U then V, each (w/2)*(h/2); NV12: interleaved UV); w and h even.
 * Limited ("TV") range BT.601 unless B200TIMG_FMT_FULL_RANGE is or'ed in (the reference's YUVJ formats).
 * Every frame is tightly packed, planes back to back, no row padding; the low nibble of fmt is the format:
 *   code  format   libav                   one frame                                            needs
 *   2     I420     yuv420p  / yuvj420p     Y w*h, U (w/2)*(h/2), V (w/2)*(h/2) bytes              w, h even
 *   3     NV12     nv12                    Y w*h, then (w/2)*(h/2) interleaved U,V byte pairs     w, h even
 *   4     I422     yuv422p  / yuvj422p     Y w*h, U (w/2)*h, V (w/2)*h bytes                      w even
 *   5     I444     yuv444p  / yuvj444p     Y, U, V each w*h bytes
 *   6     I440     yuv440p  / yuvj440p     Y w*h, U w*(h/2), V w*(h/2) bytes                      h even
 *   7     I420_10  yuv420p10le             as I420, 16-bit little-endian samples, value in bits 0-9   w, h even
 *   8     I422_10  yuv422p10le             as I422, 16-bit samples, value in bits 0-9                 w even
 *   9     I444_10  yuv444p10le             as I444, 16-bit samples, value in bits 0-9
 *   10    P010     p010le                  as NV12, 16-bit samples, value in bits 6-15                w, h even
 * Only the 10 value bits of a 16-bit sample are read.  10-bit samples are divided by 4 into the 8-bit domain and
 * converted with the same BT.601 coefficients.  Chroma is filtered at half the output width (two output pixels
 * share a sample) except for 4:4:4, which libswscale interpolates at the full output width.  A frame whose size is
 * not a multiple of its chroma subsampling, and any other code, is B200TIMG_EINVAL. */
#define B200TIMG_FMT_I420  2
#define B200TIMG_FMT_NV12  3
#define B200TIMG_FMT_I422  4
#define B200TIMG_FMT_I444  5
#define B200TIMG_FMT_I440  6
#define B200TIMG_FMT_I420_10 7
#define B200TIMG_FMT_I422_10 8
#define B200TIMG_FMT_I444_10 9
#define B200TIMG_FMT_P010  10
#define B200TIMG_FMT_FULL_RANGE 0x10

typedef struct b200timg_ctx b200timg_ctx;

/* device: CUDA ordinal.  stream: a cudaStream_t (as void*) to launch on, or NULL for a
 * stream owned by the ctx. */
int  b200timg_ctx_create(int device, void *stream, b200timg_ctx **out);
void b200timg_ctx_destroy(b200timg_ctx *ctx);
const char *b200timg_last_error(const b200timg_ctx *ctx);
int  b200timg_version(void);
/* Number of this library's kernels launched through ctx since creation. */
uint64_t b200timg_kernel_launches(const b200timg_ctx *ctx);

/* ---- geometry (host only) : ImageSource::CalcScaleToFitDisplay, src/image-source.cc:47-153.
 * Fields mirror DisplayOptions (src/display-options.h:33-55). Returns 1 if the image needs
 * scaling, 0 if not, negative on error. */
typedef struct {
    int width, height;          /* available pixels */
    int cell_x_px, cell_y_px;   /* 1x2 half, 2x2 quarter, font cell size for sixel */
    float width_stretch;
    int upscale, upscale_integer, fill_width, fill_height;
} b200timg_fit_opts;
int b200timg_calc_fit(const b200timg_fit_opts *opts, int img_w, int img_h,
                      int fit_in_rotated, int *target_w, int *target_h);

/* rgba_t::As256TermColor, src/framebuffer.h:37-52 (host helper, used by tests). */
int b200timg_as256(uint32_t rgba);

/* ======================= single frame, HOST buffers ==============================
 * These are the bodies of the reference's methods: they upload, run the kernels,
 * and download inside the call. */

/* ImageScaler::Scale with the STB scaler's semantics (src/image-scaler.cc:75-97):
 * Mitchell when shrinking, BOX when enlarging, point-sample copy at scale 1, edge clamp,
 * alpha-weighted, per axis.  in: iw*ih*4 bytes, out: ow*oh*4 bytes. */
int b200timg_scale_rgba(b200timg_ctx *ctx, const uint8_t *in, int iw, int ih, int fmt,
                        uint8_t *out, int ow, int oh);
/* mode 0: as above; 1: the <= 1 LSB arithmetic described at B200TIMG_FAST_SCALE; 2: the libswscale-style
 * bilinear filter described at B200TIMG_BILINEAR_SCALE. */
int b200timg_scale_rgba_mode(b200timg_ctx *ctx, const uint8_t *in, int iw, int ih, int fmt,
                             uint8_t *out, int ow, int oh, int fast);

/* The video source's sws_scale(decoder YUV -> RGBA at the target size), src/video-source.cc:59-89,352-354:
 * fmt = any YUV code above (| B200TIMG_FMT_FULL_RANGE); in: one frame of that layout (I420 / NV12: iw*ih*3/2
 * bytes); out: ow*oh*4 bytes. */
int b200timg_yuv_scale(b200timg_ctx *ctx, const uint8_t *in, int iw, int ih, int fmt,
                       uint8_t *out, int ow, int oh);

/* Framebuffer::AlphaComposeBackground (src/framebuffer.cc:108-150), in place on fb.
 * has_bg==0 models a null bgcolor_getter ("-b none"); the lazy getter itself stays on
 * the C++ side: the adapter resolves it only if this frame has a pixel with a<255
 * (b200timg_has_transparency). */
int b200timg_compose_bg(b200timg_ctx *ctx, uint8_t *fb, int w, int h, int has_bg,
                        uint32_t bg, uint32_t pattern, int pattern_w, int pattern_h,
                        int start_row);
/* b200timg_compose_bg on the copy b200timg_has_transparency(fb, w, h) just uploaded (one upload for "scan, fetch the
 * background colour lazily, compose"); falls back to b200timg_compose_bg if that copy is gone. */
int b200timg_compose_bg_resident(b200timg_ctx *ctx, uint8_t *fb, int w, int h, int has_bg,
                                 uint32_t bg, uint32_t pattern, int pattern_w, int pattern_h,
                                 int start_row);
/* *result = 1 if any pixel at or after start_row has alpha < 255 (the reference's
 * early-out scan, src/framebuffer.cc:113-117). */
int b200timg_has_transparency(b200timg_ctx *ctx, const uint8_t *fb, int w, int h,
                              int start_row, int *result);

/* Worst-case encoded size of one block frame: UnicodeBlockCanvas::RequestBuffers,
 * src/unicode-block-canvas.cc:405-424. */
size_t b200timg_blocks_bound(int w, int h);

/* UnicodeBlockCanvas::Send's image bytes (everything after the prefix):
 * row pairs -> glyph pick -> ANSI bytes, src/unicode-block-canvas.cc:361-399.
 * prev_fb: NULL for a full frame, else the previous frame (same w,h) for
 * emit_difference (:344-346; the backing store equals the previous frame).
 * x_indent_cells: the reference's x after "x /= 2" (:334).
 * *size == 0 means "nothing changed" (:390-395). */
int b200timg_blocks_encode(b200timg_ctx *ctx, const uint8_t *fb, int w, int h,
                           const uint8_t *prev_fb, int flags, int x_indent_cells,
                           char *out, size_t cap, size_t *size);

/* Worst-case encoded size of one sixel frame of w x h (h a multiple of 6).
 * Size limits of the sixel path (the reference has none; both are far beyond any terminal): w <= 99999 and
 * h <= 65536 (with h a multiple of 6: 65532).  Every sixel entry point rejects a larger frame with B200TIMG_EINVAL and
 * a message naming the limit before it launches anything.  Frames up to 4095 px wide take the fast emit kernel, wider
 * ones a column-tiled one ((w + 4095) / 4096 tiles); b200timg_sixel_shape_of reports which. */
size_t b200timg_sixel_bound(int w, int h);

/* What libsixel does inside SixelCanvas::Send (src/sixel-canvas.cc:134-148):
 * sixel_dither_new(256) + sixel_dither_initialize(RGBA8888, LARGE_LUM,
 * REP_AVERAGE_COLORS, QUALITY_AUTO) + sixel_encode: 15-bit histogram -> median cut
 * (<=256) -> Floyd-Steinberg -> DCS q ... ST stream.  fb must already be padded to a
 * multiple of 6 rows (round_to_sixel, :91-94) and composed; alpha is ignored. */
int b200timg_sixel_encode(b200timg_ctx *ctx, const uint8_t *fb, int w, int h,
                          char *out, size_t cap, size_t *size);

/* ======================= batches, many frames per call ===========================
 * A batch is n_frames independent source frames of identical geometry, contiguous in
 * memory (frame f at src + f*src_w*src_h*4, or f times the frame size of a YUV src_fmt).  Each runs
 *     scale (src -> out_w x out_h) -> compose -> encode
 * entirely on the device; the scaled framebuffer never leaves it.  Encoded frames are
 * written back to back into `out`; offsets[f]..offsets[f+1] delimit frame f
 * (offsets has n_frames+1 entries).  This is the unit the renderer's grid
 * (src/renderer.cc:103-148) and the animation loops (src/video-source.cc:298-366)
 * produce one Send() at a time in the reference. */
typedef struct {
    int n_frames;
    int src_w, src_h, src_fmt;
    int out_w, out_h;           /* from b200timg_calc_fit */
    /* compose (DisplayOptions: bgcolor_getter result, bg_pattern_color, pattern_size) */
    int has_bg;
    uint32_t bg, pattern;
    int pattern_w, pattern_h;
    /* block modes */
    int flags;                  /* B200TIMG_QUARTER | _UPPER | _COLOR8 */
    int x_indent_cells;
    int animation;              /* 1: frame f>0 is delta-encoded against frame f-1
                                   (Send with dy == -height, :344-346); frame 0 is full.
                                   2: the same, but frame 0 is a HALO -- scaled and used as frame 1's
                                   predecessor, never emitted (offsets[0] == offsets[1]).  A rank that owns
                                   frames [lo, hi) of a sharded animation passes frames [lo-1, hi) this way
                                   and produces exactly the bytes an unsharded run produces for lo..hi-1. */
} b200timg_batch;

/* Device-resident variants: d_src, d_out, d_offsets are DEVICE pointers; nothing crosses
 * PCIe.  The call is asynchronous on the ctx stream (no size is read back).
 * OUTPUT CAPACITY CONTRACT: the call cannot fail with B200TIMG_ENOSPC because it never learns the sizes on the
 * host.  d_offsets is always complete and exact (d_offsets[n_frames] = the bytes the batch needs); a frame whose
 * end would lie beyond out_cap is NOT written (nothing is ever written out of bounds, earlier frames are intact).
 * One exception in degree: sixel frames wider than 4095 px go through a single-pass emitter that places every band and
 * column tile on its own, so of the FIRST frame that does not fit, the pieces that end before out_cap may be written
 * (with the bytes a large enough buffer gets); still nothing at or beyond out_cap, and the offsets are exact.
 * The caller therefore either passes out_cap >= n_frames * b200timg_{blocks,sixel}_bound(out_w, padded out_h)
 * (cannot overflow) or compares d_offsets[n_frames] with out_cap when it reads the offsets, and repeats the call
 * with a larger buffer if it is greater -- exactly what the host variants do internally. */
int b200timg_blocks_batch_dev(b200timg_ctx *ctx, const b200timg_batch *b,
                              const uint8_t *d_src, char *d_out, size_t out_cap,
                              uint64_t *d_offsets);
int b200timg_sixel_batch_dev(b200timg_ctx *ctx, const b200timg_batch *b,
                             const uint8_t *d_src, char *d_out, size_t out_cap,
                             uint64_t *d_offsets);

/* Host variants (the plugin-level call): src/out/offsets are HOST pointers (pinned or
 * pageable); upload, kernels, and download of exactly the encoded bytes happen inside. */
int b200timg_blocks_batch(b200timg_ctx *ctx, const b200timg_batch *b, const uint8_t *src,
                          char *out, size_t out_cap, uint64_t *offsets);
int b200timg_sixel_batch(b200timg_ctx *ctx, const b200timg_batch *b, const uint8_t *src,
                         char *out, size_t out_cap, uint64_t *offsets);

/* ======================= mixed batches: one grid page of differently sized images ====================
 * The batches above share one geometry.  A page of `timg --grid=CxR a.jpg b.png ...` does not: every image has its own
 * source size, its own b200timg_calc_fit result for the grid's per-image box (src/timg.cc:938-939) and its own x
 * position (src/renderer.cc:103-148: column offset plus centering).  A mixed batch describes such a page: frame f has
 * its own source and output geometry and indent, the page shares the colour format, the block flags and the
 * compose options (one DisplayOptions).  Frame f's bytes are exactly those of the single-frame path on that image
 * (ImageScaler::Scale -> AlphaComposeBackground -> UnicodeBlockCanvas::Send of a full frame, as the uniform batch
 * composes them), whatever the frame's place in the batch, the batch size or the variant called.  A call runs a fixed
 * number of kernels and uploads its tables and descriptors in one copy, however many geometries the page has; frames
 * of equal geometry share one resampling plan.  The scaler's float intermediate is bounded: a page whose
 * intermediate exceeds 2 GiB runs as several frame groups (the count depends on bytes, never on geometries).
 * Source frames: RGBA or RGB32, tightly packed, frame f at src + frames[f].src_offset.
 * Rejected with B200TIMG_EINVAL: n_frames <= 0 or > 65535, frames == NULL, a non-positive size, a negative indent, a
 * src_offset that is not a multiple of 4, an odd out_w in quarter mode (the message names the frame), a YUV or
 * unknown src_fmt, B200TIMG_BILINEAR_SCALE, more than 2^31 - 1 row pairs or scaler work items in one call.
 * B200TIMG_FAST_SCALE is accepted and ignored: mixed batches always scale bit-exactly.
 * Out of scope: delta frames (a grid page has none, so there is no animation field), YUV sources, the bilinear
 * scaler, and the kitty / iTerm2 encoders (they build on b200timg_scale_mixed_dev's output).  The sixel encoder takes
 * mixed batches: b200timg_sixel_mixed_dev below. */
typedef struct {
    uint64_t src_offset;        /* bytes from the batch's source pointer to this frame's first pixel; multiple of 4 */
    int src_w, src_h;           /* source geometry of this image */
    int out_w, out_h;           /* its b200timg_calc_fit result */
    int x_indent_cells;         /* UnicodeBlockCanvas::Send's x after "x /= 2" for this image (column offset + centering) */
} b200timg_frame;

typedef struct {
    int n_frames;
    int src_fmt;                /* B200TIMG_FMT_RGBA or B200TIMG_FMT_RGB32 */
    int flags;                  /* B200TIMG_QUARTER | _UPPER | _COLOR8 (| _FAST_SCALE: accepted, computed exactly) */
    int has_bg;                 /* compose, shared by the page: as b200timg_batch */
    uint32_t bg, pattern;
    int pattern_w, pattern_h;
    const b200timg_frame *frames;   /* HOST pointer, n_frames entries */
} b200timg_mixed_batch;

/* Scale + fused compose of every frame (DEVICE pointers, asynchronous): frame f's out_w*out_h*4 bytes land at d_out
 * plus the sum of the earlier frames' out_w*out_h*4; d_src and d_out 4-byte aligned. */
int b200timg_scale_mixed_dev(b200timg_ctx *ctx, const b200timg_mixed_batch *b, const uint8_t *d_src, uint8_t *d_out);
/* scale -> compose -> half/quarter blocks; frames back to back, offsets[n_frames + 1] as in the uniform batches.
 * The _dev variant follows the OUTPUT CAPACITY CONTRACT above; the sum of b200timg_blocks_bound(out_w, out_h) over the
 * frames cannot overflow.  The host variant returns B200TIMG_ENOSPC with offsets[] complete (offsets[n_frames] = the
 * bytes needed) and writes nothing at or beyond out_cap. */
int b200timg_blocks_mixed_dev(b200timg_ctx *ctx, const b200timg_mixed_batch *b, const uint8_t *d_src,
                              char *d_out, size_t out_cap, uint64_t *d_offsets);
int b200timg_blocks_mixed(b200timg_ctx *ctx, const b200timg_mixed_batch *b, const uint8_t *src,
                          char *out, size_t out_cap, uint64_t *offsets);
/* scale -> compose -> pad -> sixel (a `-p sixel` grid page): frame f's bytes are exactly those of b200timg_sixel_batch_dev
 * on a one-frame batch of that image with flags = 0 -- exact scale with the compose fused, padded to a multiple of 6
 * rows, the background composed into the pad strip only (SixelCanvas::Send), palette, Floyd-Steinberg dither, DCS
 * stream -- whatever the frame's place in the batch, the batch size or the variant called.  x_indent_cells and the
 * block flags are ignored (the cursor move is the caller's prefix, as for the uniform sixel batch);
 * B200TIMG_FAST_SCALE is accepted and ignored.  The default kernels always run (B200TIMG_EMIT and B200TIMG_PARTS do
 * not apply).  Rejected with B200TIMG_EINVAL besides the cases above: out_w > 4095 and a padded
 * height over 65536 rows (the message names the frame; wider images go through the uniform batch).
 * The _dev variant follows the OUTPUT CAPACITY CONTRACT above.  The host variant stages into the sum of
 * b200timg_sixel_bound(out_w, round_to_sixel(out_h)) over the frames and returns B200TIMG_ENOSPC with offsets[]
 * complete and nothing written at or beyond out_cap.  b200timg_sixel_debug then reports frame 0. */
int b200timg_sixel_mixed_dev(b200timg_ctx *ctx, const b200timg_mixed_batch *b, const uint8_t *d_src,
                             char *d_out, size_t out_cap, uint64_t *d_offsets);
int b200timg_sixel_mixed(b200timg_ctx *ctx, const b200timg_mixed_batch *b, const uint8_t *src,
                         char *out, size_t out_cap, uint64_t *offsets);

/* Device-resident single stages, for tests and for callers that keep frames on the GPU
 * (e.g. an NVDEC front end).  All pointers are DEVICE pointers. */
int b200timg_scale_dev(b200timg_ctx *ctx, const uint8_t *d_in, int iw, int ih, int fmt,
                       uint8_t *d_out, int ow, int oh, int n_frames);
int b200timg_compose_dev(b200timg_ctx *ctx, uint8_t *d_fb, int w, int h, int n_frames,
                         int has_bg, uint32_t bg, uint32_t pattern, int pattern_w,
                         int pattern_h, int start_row);

/* The sixel stage alone on n device-resident frames that are already scaled, padded to a
 * multiple of 6 rows and composed (e.g. BASELINE config 5: 1280x720 frames shown unscaled). */
int b200timg_sixel_dev(b200timg_ctx *ctx, const uint8_t *d_fb, int w, int h, int n_frames,
                       char *d_out, size_t out_cap, uint64_t *d_offsets);

/* Per-kernel timing with CUDA events recorded on the ctx stream around every launch.
 * profile(ctx,1) clears and starts, profile(ctx,0) stops and clears.  The report is text, one
 * line per kernel: "<name> <launches> <total_ms>".  Timing adds two event records per launch,
 * so throughput numbers are taken with profiling off. */
int b200timg_profile(b200timg_ctx *ctx, int enable);
int b200timg_profile_report(b200timg_ctx *ctx, char *buf, size_t cap);

/* Introspection for tests: after b200timg_sixel_encode, the palette (256 words r|g<<8|b<<16),
 * counts[0] = palette entries in use, counts[1] = occupied 15-bit histogram cells, and the
 * palette-index plane (w*h bytes) of that frame.  Any pointer may be NULL. */
int b200timg_sixel_debug(b200timg_ctx *ctx, uint32_t *palette, uint32_t *counts, uint8_t *index,
                         size_t index_bytes);

/* Host-only introspection of the resampling plan behind b200timg_scale_* (no GPU needed):
 * the per-axis contributor tables and the pass order that reproduce the reference scaler's
 * arithmetic (third_party/stb/stb_image_resize2.h:3267-3635, 6859-6905).  axis 0 = horizontal,
 * 1 = vertical.  first/count/lead have out_w (or out_h) entries, coeff has entries*widest.
 * flags: bit0 vertical pass first, bit1 plain copy (both axes at scale 1), bit2 horizontal taps
 * use a single accumulator.  Any output pointer may be NULL. */
int b200timg_resample_plan(int in_w, int in_h, int out_w, int out_h, int axis, int *widest,
                           int *flags, int32_t *first, int32_t *count, int32_t *lead,
                           float *coeff, size_t coeff_cap);

/* Host-only introspection of the launch shapes behind the sixel entry points (no GPU needed): what the library would
 * launch for n_frames frames of w x h that are a slice of a batch of n_total frames (n_total == n_frames for a whole
 * batch; b200timg_sixel_encode is a batch of one) on a device with sm_count multiprocessors.  Computed by the functions
 * the launches call, the environment switches they honour included (B200TIMG_DITHER_SPLIT, B200TIMG_DITHER_WARPS,
 * B200TIMG_EMIT).  Returns B200TIMG_EINVAL for a geometry the launch rejects (h not a multiple of 6, w > 99999,
 * h > 65536, more than 65535 frames) and for out == NULL, sm_count <= 0, n_frames <= 0 or n_total < n_frames. */
typedef struct {
    int step_px, ent_cap, palette_global;      /* palette: sampling step, entries per median-cut table (<= 32768),
                                                  1 = tables in global memory (more than 25600 entries), 0 = shared */
    int nb32, dither_ctas, bands_per_cta, dither_warps, dither_rounds;
                                               /* dither: bands of 32 rows, CTAs per frame (> 1 only for batches of fewer
                                                  frames than SMs: min(sm_count / n_total, (nb32 + 7) / 8)), bands per
                                                  CTA, warps per CTA (<= 24), rounds of a warp over its CTA's bands */
    int emit_mode, emit_tiles, tile_w;         /* emit: 1/4/5 band scratch + compaction (5 up to 4095 px), 2/3 single
                                                  pass; their column tiles ((w + 4095) / 4096) and a tile's width */
} b200timg_sixel_shape;
int b200timg_sixel_shape_of(int w, int h, int n_frames, int n_total, int sm_count, b200timg_sixel_shape *out);

/* ======================= geometry passes around the path (SURVEY 8f rank 3, row a15) ===============
 * ApplyExifOp (src/jpeg-source.cc:84-119): mirror each row, then rotate by 0, 180, 90 or -90 degrees exactly as
 * the reference's loops do (90 / -90: out is h x w).  in and out: w*h*4 bytes. */
int b200timg_exif_op(b200timg_ctx *ctx, const uint8_t *fb, int w, int h, int mirror, int angle, uint8_t *out);
int b200timg_exif_op_dev(b200timg_ctx *ctx, const uint8_t *d_in, uint8_t *d_out, int w, int h, int mirror, int angle,
                         int n_frames);
/* --auto-crop = Magick::Image::trim() (src/graphics-magick-source.cc:238-240; GraphicsMagick is not in the tree:
 * its documented rule with fuzz 0 is restated, parity unpinned): rect = {x, y, w, h} of the bounding box of the
 * pixels differing from the corner colours (left and top edges against the top-left pixel, right edge against the
 * top-right, bottom edge against the bottom-left).  A single-colour image keeps its full size. */
int b200timg_trim_bbox(b200timg_ctx *ctx, const uint8_t *fb, int w, int h, int rect_xywh[4]);
/* n_pos windows of dw x dh pixels cut from one w x h image, window k at
 *     ((x0 + dx*(first_pos + k)) mod w, (y0 + dy*(first_pos + k)) mod h), wrapping around
 * -- the scroll animation of src/graphics-magick-source.cc:383-389 (one launch for many positions) and, with
 * n_pos = 1 and dx = dy = 0, a plain crop (--crop-border, :232-237).  out: n_pos * dw*dh*4 bytes. */
int b200timg_windows(b200timg_ctx *ctx, const uint8_t *img, int w, int h, int dw, int dh, long long x0, long long y0,
                     int dx, int dy, long long first_pos, int n_pos, uint8_t *out);
int b200timg_windows_dev(b200timg_ctx *ctx, const uint8_t *d_img, int w, int h, int dw, int dh, long long x0,
                         long long y0, int dx, int dy, long long first_pos, int n_pos, uint8_t *d_out);

/* ======================= Kitty / iTerm2 canvases: PNG + base64 (SURVEY 8f rank 2) ===================
 * png::Encode (src/timg-png.cc:90-152): signature, IHDR, one IDAT holding the zlib stream of the scanlines (each
 * row filtered with "Sub"), IEND.  rgb24 != 0: colour type 2 (png::ColorEncoding::kRGB_24), else RGBA.  The
 * reference deflates with libdeflate (third party, not in its tree); this stream uses stored deflate blocks, so it
 * decodes to the same pixels but is not the same bytes, and its size is exactly b200timg_png_size().
 * EncodeBase64 (src/timg-base64.h:28-53) of the file goes to b64 when given.  The framed batches below add the
 * protocol framing (src/kitty-canvas.cc:196-226, src/iterm2-canvas.cc:66-72) on the device. */
size_t b200timg_png_size(int w, int h, int rgb24);
size_t b200timg_base64_size(size_t n_bytes);
int b200timg_png_encode(b200timg_ctx *ctx, const uint8_t *fb, int w, int h, int rgb24, uint8_t *out, size_t cap,
                        char *b64, size_t b64_cap);
/* n device-resident frames -> n files at d_png + f*png_size (and their base64 at d_b64 + f*base64_size, or NULL) */
int b200timg_png_batch_dev(b200timg_ctx *ctx, const uint8_t *d_frames, int w, int h, int n_frames, int rgb24,
                           uint8_t *d_png, char *d_b64);

/* Kitty / iTerm2 batches: scale -> compose -> PNG -> base64 -> protocol framing for many frames per call.
 * The bytes of frame f are exactly what KittyGraphicsCanvas::Send (src/kitty-canvas.cc:190-229, plain or in its
 * tmux form) or ITerm2GraphicsCanvas::Send (src/iterm2-canvas.cc:66-73) append after the queued prefix:
 *     kitty   "\e_Ga=T,i=<id>,q=2,f=100,m=<0|1>;" base64 in chunks of 4096 characters, each but the last followed
 *             by "\e\\\e_Gq=2,m=<0|1>;", then "\e\\" "\n"
 *     kitty in tmux (B200TIMG_KITTY_TMUX, what timg sends when the terminal runs inside tmux): every kitty command
 *             wrapped in tmux's passthrough, escapes doubled, the image placed by Unicode placeholders:
 *             "\ePtmux;" "\e\e_Ga=T,i=<id>,q=2,f=100,m=<0|1>,U=1,c=<cols>,r=<rows>;" base64 chunk 0, per further
 *             chunk "\e\e\\" "\e\\" "\ePtmux;" "\e\e_Gq=2,m=<0|1>;" chunk k, then "\e\e\\" "\e\\" "\r" and per
 *             placeholder row r < rows:  ["\e[<indent>C"] "\e[38:2:<id>>16&255>:<id>>8&255>:<id&255>m",
 *             cols x (U+10EEEE, diacritic(r), diacritic(c), [diacritic(id >> 24) if nonzero]), "\e[39m\n\r"
 *             with cols = w / cell_x_px, rows = ceil(h / cell_y_px), indent = indent_cells and kitty's row / column
 *             diacritics (src/kitty-canvas.cc:255-344; none for values >= 297, and the reference's bytes for the
 *             14 values from 283 on, see png.cu)
 *     iTerm2  "\e]1337;File=size=<n>;width=<w>px;height=<h>px;inline=1:" base64 "\a\n"
 * with this library's stored-block PNG (the bytes b200timg_png_encode produces).  Cursor moves and the prefix stay
 * with the caller, as do kitty's image ids (CreateId and the animation flip-buffer, src/kitty-canvas.cc:142-172)
 * and, for the tmux form, enabling tmux's passthrough (the adapter does it as the reference does).
 * Scale and compose are those of the blocks batch (FAST / BILINEAR scale, YUV sources); rgb24 is
 * independent of has_bg.  Rejected with B200TIMG_EINVAL: animation != 0 (no delta frames), an unknown protocol,
 * ids == NULL for either kitty form, cell_x_px <= 0, cell_y_px <= 0 or indent_cells < 0 for the tmux form, a PNG
 * larger than one IDAT chunk (2^31 - 1 bytes).
 * Frame sizes are a closed formula (b200timg_graphics_size: the PNG size is fixed, the id only changes digit counts
 * and, in tmux, the placeholders' id diacritic), so offsets[f] is the running sum of the sizes.  Every part that
 * depends on the id is largest at id = 0xffffffff, so b200timg_graphics_size(g, w, h, 0xffffffff) bounds the size of
 * a frame of any id.  The _dev variant follows the OUTPUT CAPACITY CONTRACT
 * above and does not synchronise the host (offsets and ids are uploaded from context-owned pinned staging); the
 * host variant returns B200TIMG_ENOSPC before launching anything when out_cap is too small (offsets complete,
 * offsets[n_frames] = the bytes needed) and downloads exactly the encoded bytes. */
#define B200TIMG_KITTY      1
#define B200TIMG_ITERM2     2
#define B200TIMG_KITTY_TMUX 4   /* KittyGraphicsCanvas with tmux_passthrough_needed (3 is not a protocol) */
/* B200TIMG_DEFLATE, OR'ed into protocol (any of the three): the PNG's zlib stream is compressed, as timg does for
 * --compress levels 1-9 (DisplayOptions::compress_pixel_level > 0); level 0 is the stored path above.  All levels
 * 1-9 map to this library's one compressor (libdeflate's per-level trade-offs are not reproduced): per 65535-byte
 * segment of the scanline stream, a greedy LZ77 parse (matches of 4 to 258 bytes, up to 32768 bytes back, into the
 * previous segment too) and one dynamic-Huffman block, or the stored block where that is not at least 2 bytes
 * smaller.  A frame's PNG is therefore never longer than b200timg_png_size().  The output is deterministic: a frame's
 * bytes depend on that frame only (not on its place in the batch, the batch size or the variant called).  libdeflate
 * is not in the reference's tree, so the deflate bytes are not the reference's: they decode to the same pixels, and
 * every byte around them (PNG chunks and CRCs, base64, chunking, headers, placeholders) is what the reference's own
 * code writes around this stream.
 * Sizes depend on the data: b200timg_graphics_size with the bit set returns the stored size, an UPPER BOUND.  The _dev
 * variant computes d_offsets on the device (exact) and follows the OUTPUT CAPACITY CONTRACT.  The host variant reads
 * the offsets back chunk by chunk; on B200TIMG_ENOSPC offsets[] is complete (offsets[n_frames] = the bytes needed) and
 * nothing is written at or beyond out_cap.  Any other bit, and 3 | B200TIMG_DEFLATE, is B200TIMG_EINVAL.
 * b200timg_png_encode and b200timg_png_batch_dev keep stored blocks. */
#define B200TIMG_DEFLATE    8
typedef struct {
    int protocol;               /* B200TIMG_KITTY, B200TIMG_ITERM2 or B200TIMG_KITTY_TMUX, optionally | B200TIMG_DEFLATE */
    int rgb24;                  /* DisplayOptions::local_alpha_handling: PNG colour type 2, else RGBA (type 6) */
    const uint32_t *ids;        /* kitty (either form): n_frames image ids (HOST pointer), the i= of each frame;
                                   ignored for iTerm2 */
    /* read for B200TIMG_KITTY_TMUX only, so callers built before these fields existed keep working: */
    int cell_x_px, cell_y_px;   /* DisplayOptions::cell_x_px / cell_y_px: the placeholder grid's cell size */
    int indent_cells;           /* x / cell_x_px of KittyGraphicsCanvas::Send: cells each placeholder row moves right */
} b200timg_graphics;
/* exact bytes of one frame (host only); 0 for an invalid protocol, size, cell size or indent.  The id is the
 * argument: g->ids is not read. */
size_t b200timg_graphics_size(const b200timg_graphics *g, int w, int h, uint32_t id);
int b200timg_graphics_batch_dev(b200timg_ctx *ctx, const b200timg_batch *b, const b200timg_graphics *g,
                                const uint8_t *d_src, char *d_out, size_t out_cap, uint64_t *d_offsets);
int b200timg_graphics_batch(b200timg_ctx *ctx, const b200timg_batch *b, const b200timg_graphics *g,
                            const uint8_t *src, char *out, size_t out_cap, uint64_t *offsets);

/* ======================= K7: gather of the encoded frames over NCCL ==============================
 * One process per GPU (SURVEY 8e).  The reference is a single process and has no counterpart; frames are
 * independent units, every rank encodes its own batch (b200timg_*_batch_dev) and this call moves the
 * encoded bytes to `root`.  Fixed-slot protocol without any host synchronisation: every rank passes the same
 * slot_bytes (>= the size of any rank's batch, <= the capacity of d_payload); on root, rank r's bytes land at
 * d_dst + r*slot_bytes and frame i of rank r is
 *     [d_dst_offsets[r*(n_frames+1) + i], d_dst_offsets[r*(n_frames+1) + i + 1])   (absolute, inside d_dst).
 * d_dst: nranks*slot_bytes bytes, d_dst_offsets: nranks*(n_frames+1) entries, both only read on root.
 * *d_status (optional, root): bit r set if rank r's batch did not fit its slot (its frames are then truncated
 * at the slot end, nothing is read or written out of bounds).  The transfer runs on the context's gather
 * stream behind the compute stream, so the next batch's kernels overlap it.  b200timg_gather returns a ticket
 * (>= 0) or a negative error; b200timg_gather_wait(ctx, ticket, block_host) orders the compute stream (or the
 * host) after that gather -- call it before consuming d_dst or overwriting d_payload.  The last four gathers
 * can be waited for individually (double-buffered callers wait for the one that used the buffer they reuse). */
#define B200TIMG_NCCL_ID_BYTES 128
int  b200timg_gather_unique_id(char id[B200TIMG_NCCL_ID_BYTES]);            /* ncclGetUniqueId; share it with all ranks */
int  b200timg_gather_init(b200timg_ctx *ctx, const char id[B200TIMG_NCCL_ID_BYTES], int rank, int nranks);   /* ncclCommInitRank */
int  b200timg_gather_attach(b200timg_ctx *ctx, void *nccl_comm, int rank, int nranks);  /* use the caller's ncclComm_t */
void b200timg_gather_shutdown(b200timg_ctx *ctx);
int  b200timg_gather(b200timg_ctx *ctx, const char *d_payload, const uint64_t *d_offsets, int n_frames,
                     size_t slot_bytes, char *d_dst, uint64_t *d_dst_offsets, uint32_t *d_status, int root);
int  b200timg_gather_wait(b200timg_ctx *ctx, int ticket, int block_host);

#ifdef __cplusplus
}
#endif
#endif /* B200TIMG_H */
