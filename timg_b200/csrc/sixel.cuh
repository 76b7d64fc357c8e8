// Shared declarations of the sixel kernels (sixel.cu: palette / LUT / dither, sixel_emit.cu: byte emit).
#pragma once
#include "common.cuh"

namespace b200timg {

constexpr int SIXEL_HDR_CAP = 4672;    // DCS q + raster attributes (<= 29 bytes) + 256 palette definitions of <= 18 bytes

struct SixelFrameHdr {
    uint32_t ncolors, origcolors, diffuse, header_len;
    uint32_t frame_size, pad0, pad1, pad2;
    uint32_t palette[256];             // r | g << 8 | b << 16
};

struct SixelWork {                     // device pointers into ctx->sixel_work
    SixelFrameHdr *hdr;                // [n_frames]
    uint32_t *ent_a, *ent_b;           // [n_frames][ent_cap] median-cut tables (bucket << 16 | count)
    uint8_t *lut;                      // [n_frames][32768]
    uint8_t *index;                    // [n_frames][w*h]
    uint32_t *boundary;                // [n_frames][nb32][w] packed errors of each 32-row band's last row
    uint32_t *band_bytes;              // [n_frames][nbands]  sizes
    uint32_t *band_off;                // [n_frames][nbands]  offset of each band's first byte inside its frame
    char *scratch;                     // [n_frames][nbands][band_cap] band bytes before compaction
    size_t band_cap;
    int ent_cap, nb32, nbands;
    // single-pass emit (sixel_emit.cu)
    char *hdr_bytes;                   // [n_frames][SIXEL_HDR_CAP] header + palette definitions of each frame
    unsigned long long *desc;          // [n_frames * nbands * ntiles] look-back descriptors: flag << 62 | bytes
    uint32_t *ctl;                     // [0] CTA ticket, [1] status (bit 0: output buffer too small)
};

// One frame of a mixed-geometry sixel batch (b200timg_sixel_mixed_dev): its padded geometry and where its parts live.
// Offsets count elements from the bases in SixelWork (ent_a / ent_b, index, scratch) and from the dither's boundary and
// progress arrays; headers and nearest-colour tables stay dense per frame (W.hdr + f, W.lut + f * 32768).
struct __align__(16) MixedSixelFrame {
    unsigned long long fb_px;          // first pixel of the padded frame in the scaled framebuffer
    unsigned long long idx;            // first index byte
    unsigned long long ent;            // first median-cut table entry
    unsigned long long bnd;            // first boundary element of the dither (uint4)
    unsigned long long scr;            // first scratch byte of band 0
    unsigned long long band_cap;       // scratch bytes per band
    int w, h, nb32, nbands, ent_cap;   // h: padded rows (a multiple of 6)
    int band0, prog0;                  // first flat band (band_bytes / band_off) and first progress flag
    int cols_per_warp, bands_per_cta;  // emit5's column split; the dither's bands per CTA
};
// What the mixed kernels read besides SixelWork: the descriptors and the flat item lists (all in ctx->mixed_up.arena).
struct MixedSixelParams {
    const MixedSixelFrame *desc;
    const unsigned *band_start;        // [n + 1] first flat band of each frame (emit, compaction)
    const unsigned *cta_start;         // [n + 1] first dither CTA of each frame
    const int *list;                   // palette launch: the frames it covers
    int n_frames, n_list, nwarps;      // nwarps: the dither launch's warps per CTA
};

// mixed batches: the frame that owns flat item `item`: the last f with start[f] <= item
__device__ __forceinline__ int sixel_owner(const unsigned *__restrict__ start, int n, unsigned item) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (start[mid] <= item) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__device__ __forceinline__ uint32_t hash15(uint32_t px) {   // (r>>3)<<10 | (g>>3)<<5 | (b>>3)
    return ((px & 0xf8) << 7) | ((px >> 6) & 0x3e0) | ((px >> 19) & 0x1f);
}
__device__ __forceinline__ uint32_t key5(uint32_t entry, int plane) { return (entry >> (26 - 5 * plane)) & 31; }

// ------------------------------------------------------------------ block helpers (1024 thr)
template <int NT>
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t *s_w /*[NT/32]*/, uint32_t &total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += o; }
    if (lane == 31) s_w[wid] = inc;
    __syncthreads();
    uint32_t pre = 0, tot = 0;
    for (int k = 0; k < NT / 32; ++k) { if (k < wid) pre += s_w[k]; tot += s_w[k]; }
    total = tot;
    __syncthreads();
    return pre + inc - v;
}


// ---- number formatting shared by the emitters
__device__ __forceinline__ uint32_t ndig_u(uint32_t v) { uint32_t n = 1; while (v >= 10) { v /= 10; ++n; } return n; }
__device__ __forceinline__ char *put_num_u(char *o, uint32_t v) {
    char tmp[10]; int n = 0;
    do { tmp[n++] = (char)('0' + v % 10); v /= 10; } while (v);
    while (n) *o++ = tmp[--n];
    return o;
}

// The <=6 distinct (colour, bits) pairs of column x of a 6-row band: slot i is valid iff row i is the
// first row showing its colour (fixed slots, so everything stays in registers).  Returns the valid mask.
__device__ __forceinline__ uint32_t column_entries(const uint8_t *__restrict__ idx, int w, int x, uint32_t *c, uint32_t *bits) {
#pragma unroll
    for (int i = 0; i < 6; ++i) c[i] = idx[(long long)i * w + x];
    uint32_t valid = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        bool seen = false;
        uint32_t b = 0;
#pragma unroll
        for (int j = 0; j < 6; ++j) {
            if (j < i && c[j] == c[i]) seen = true;
            if (j >= i && c[j] == c[i]) b |= 1u << j;
        }
        bits[i] = b;
        if (!seen) valid |= 1u << i;
    }
    return valid;
}

int launch_sixel_emit(b200timg_ctx *ctx, int w, int h, int n_frames, const SixelWork &W, char *d_out, size_t out_cap,
                      uint64_t *d_offsets);
size_t sixel_dither_workspace(int w, int h, int n_frames, size_t *o_bnd, size_t *o_prog);
int launch_sixel_dither(b200timg_ctx *ctx, const uint32_t *fb, int w, int h, int n_frames, int n_total, const SixelWork &W, void *d_bnd, void *d_prog);

// ---- launch shapes (host).  The launchers and b200timg_sixel_shape_of both call these, so what the introspection reports
// is what a launch does.
// What the sixel path takes: h a multiple of 6, w <= 99999, h <= 65536 (2048 bands of 32 rows), n_frames <= 65535 and at
// most 2^31 - 1 emit CTAs.  B200TIMG_OK, or B200TIMG_EINVAL with the reason in msg.
int sixel_check_geometry(int w, int h, int n_frames, char *msg, size_t msg_cap);
// K4 of a frame of npix pixels: sampling step, entries of each median-cut table, and whether the two tables fit the
// palette kernel's shared memory (tables_smem bytes) or live in global memory.
struct SixelPaletteShape { long long step_px; int ent_cap; bool smem_tables; size_t tables_smem; };
SixelPaletteShape sixel_palette_shape(long long npix);
// K5 of a launch over n_frames frames of nb32 bands, a slice of a batch of n_total: CTAs per frame, bands per CTA, warps
// per CTA and rounds of a warp over its CTA's bands.  A frame is split only when the batch has fewer frames than SMs, and
// then into at most sm_count / n_frames CTAs, so that every CTA of the launch is resident at once (bands wait for the
// band above).  env: honour B200TIMG_DITHER_SPLIT / B200TIMG_DITHER_WARPS (the uniform launches do, mixed batches do not).
struct SixelDitherShape { int per_frame, bands_per_cta, nwarps, rounds; };
SixelDitherShape sixel_dither_shape(int nb32, int n_frames, int n_total, int sm_count, bool env);
// K6: the emitter a frame w wide takes (5 emit5: band scratch + compaction; 2 emit2: single pass; B200TIMG_EMIT honoured)
// and emit2's column tiles.
int sixel_emit_mode(int w);
void sixel_emit_tiling(int w, int *ntiles, int *tw, int *cpw);

int launch_sixel_dither_mixed(b200timg_ctx *ctx, const uint32_t *fb, unsigned n_ctas, const MixedSixelParams &M, const SixelWork &W,
                              void *d_bnd, void *d_prog, size_t n_prog, bool split);
size_t sixel_emit_workspace(int w, int h, int n_frames, size_t *o_hdr_bytes, size_t *o_desc, size_t *o_ctl);

}  // namespace b200timg
