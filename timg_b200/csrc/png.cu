// Kitty / iTerm2 canvases' per-frame encode (SURVEY 8f rank 2): PNG container + base64 + protocol framing.
//   png::Encode            src/timg-png.cc:90-152   signature, IHDR, one IDAT (zlib stream of the scanlines, every
//                                                   row filtered with the "Sub" filter, type 1), IEND, CRC per chunk
//   EncodeBase64           src/timg-base64.h:28-53
//   framing                src/kitty-canvas.cc:190-229, src/iterm2-canvas.cc:66-73
//   tmux placeholders      src/kitty-canvas.cc:55-74,255-344 (the Unicode placeholder grid after the tmux form)
// The reference compresses the filtered scanlines with libdeflate, a third-party library that is not part of its
// tree.  Here the zlib stream uses stored (uncompressed) deflate blocks -- a valid stream any PNG decoder accepts,
// whose size is a closed formula, so every frame of a batch lands at a fixed offset and all stages are
// embarrassingly parallel.  Every byte of the file is a closed function of the frame (png_byte) except the three
// checksums, which one pass computes from the frame:
//   png_check_kernel      CRC-32 (IDAT) and Adler-32 (zlib) of 4 KB segments, one thread per segment
//   png_seal_kernel       combine the segment checksums (GF(2) polynomial arithmetic for CRC, modular for Adler)
//                         into two words per frame (and write them into the files of png_fill_kernel)
//   png_fill_kernel       the PNG files (b200timg_png_*), checksum fields zero until png_seal_kernel
//   base64_kernel         3 bytes -> 4 characters of those files
//   graphics_emit_kernel  the framed kitty / iTerm2 text of a batch straight from the frames (b200timg_graphics_*):
//                         no PNG file is written in between
//   graphics_grid_kernel  kitty's tmux form: the rows of Unicode placeholders that follow the image data
// Parity: the framed text equals, byte for byte, what the reference's canvases produce with a stored-block
// compressor in place of libdeflate (tests/golden/graphics.npz); the files parse with Python's zlib / struct.
#include <algorithm>

#include "common.cuh"

namespace b200timg {

// PngGeom (common.cuh): the layout of one frame's stored-block PNG
static PngGeom png_geom(int w, int h, int rgb24) {
    PngGeom g;
    g.w = w; g.h = h; g.bpp = rgb24 ? 3 : 4;
    g.row_bytes = 1 + (long long)w * g.bpp;
    g.raw_len = g.row_bytes * h;
    g.nblocks = (g.raw_len + 65534) / 65535;
    if (g.nblocks == 0) g.nblocks = 1;
    g.zlib_len = 2 + 5 * g.nblocks + g.raw_len + 4;
    g.idat_data_off = 8 + 25 + 8;
    g.png_len = g.idat_data_off + g.zlib_len + 4 + 12;
    return g;
}

// byte i of the filtered scanline stream of one frame
__device__ __forceinline__ uint8_t raw_byte(const uint8_t *__restrict__ fb, const PngGeom &g, long long i) {
    const long long y = i / g.row_bytes, c = i - y * g.row_bytes;
    if (c == 0) return 1;                                               // filter type: Sub
    const long long x = (c - 1) / g.bpp, ch = (c - 1) - x * g.bpp;
    const uint8_t *px = fb + ((long long)y * g.w + x) * 4;
    const uint8_t cur = px[ch];
    return x == 0 ? cur : (uint8_t)(cur - px[ch - 4]);                  // src/timg-png.cc:119-126
}

__device__ __forceinline__ void put_be32(uint8_t *p, uint32_t v) { p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; }

// byte o (0 <= o < png_len) of one frame's PNG file: the file layout, written down once.  The three checksum
// fields are closed functions of the frame too, but not per byte; they are passed in (zero while they are computed).
__device__ __forceinline__ uint8_t png_byte(const uint8_t *__restrict__ fb, const PngGeom &g, long long o, uint32_t ihdr_crc,
                                            uint32_t idat_crc, uint32_t adler) {
    if (o < 8) { const uint8_t sig[8] = {0x89, 0x50, 0x4E, 0x47, '\r', '\n', 0x1A, '\n'}; return sig[o]; }
    if (o < 29) {                                                       // IHDR chunk: length, type, 13 data bytes
        const long long k = o - 8;
        const uint8_t hdr[21] = {0, 0, 0, 13, 'I', 'H', 'D', 'R', (uint8_t)(g.w >> 24), (uint8_t)(g.w >> 16), (uint8_t)(g.w >> 8), (uint8_t)g.w,
                                 (uint8_t)(g.h >> 24), (uint8_t)(g.h >> 16), (uint8_t)(g.h >> 8), (uint8_t)g.h, 8, (uint8_t)(g.bpp == 4 ? 6 : 2), 0, 0, 0};
        return hdr[k];
    }
    if (o < 33) return (uint8_t)(ihdr_crc >> (8 * (32 - o)));          // IHDR CRC, big-endian
    if (o < g.idat_data_off) {                                          // IDAT length + type
        const long long k = o - 33;
        const uint8_t hd[8] = {(uint8_t)(g.zlib_len >> 24), (uint8_t)(g.zlib_len >> 16), (uint8_t)(g.zlib_len >> 8), (uint8_t)g.zlib_len, 'I', 'D', 'A', 'T'};
        return hd[k];
    }
    const long long z = o - g.idat_data_off;
    if (z < g.zlib_len) {
        if (z < 2) return z == 0 ? 0x78 : 0x01;                         // zlib header: deflate, 32K window, no preset dictionary, level 0
        if (z >= g.zlib_len - 4) return (uint8_t)(adler >> (8 * (g.zlib_len - 1 - z)));   // Adler-32, big-endian
        const long long d = z - 2, blk = d / 65540, in = d - blk * 65540;         // 5-byte header + up to 65535 bytes
        const long long start = blk * 65535;
        const long long len = min((long long)65535, g.raw_len - start);
        if (in == 0) return blk == g.nblocks - 1 ? 1 : 0;              // BFINAL, BTYPE = 00 (stored)
        if (in == 1) return (uint8_t)len;
        if (in == 2) return (uint8_t)(len >> 8);
        if (in == 3) return (uint8_t)~len;
        if (in == 4) return (uint8_t)(~len >> 8);
        return raw_byte(fb, g, start + in - 5);
    }
    if (z < g.zlib_len + 4) return (uint8_t)(idat_crc >> (8 * (g.zlib_len + 3 - z)));  // IDAT CRC, big-endian
    const uint8_t iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82};
    return iend[z - (g.zlib_len + 4)];
}

// the files with zero checksum fields; png_seal_kernel writes them
__global__ void __launch_bounds__(256)
png_fill_kernel(const uint8_t *__restrict__ frames, uint8_t *__restrict__ out, PngGeom g, int n_frames) {
    const long long per = g.png_len, total = per * n_frames;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long f = t / per, o = t - f * per;
        out[t] = png_byte(frames + f * (long long)g.w * g.h * 4, g, o, 0, 0, 0);
    }
}

// ---- checksums ---------------------------------------------------------------------------------------
constexpr uint32_t CRC_POLY = 0xedb88320u;
__host__ __device__ __forceinline__ uint32_t crc_byte(uint32_t c, uint8_t b) {
    c ^= b;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (CRC_POLY & (0u - (c & 1u)));
    return c;
}
// a(x) * b(x) mod p(x), reflected representation (the arithmetic of zlib's crc32_combine)
__host__ __device__ inline uint32_t multmodp(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ 0xedb88320u : b >> 1;
    }
    return p;
}
// x^(8*n) mod p(x)
__host__ __device__ inline uint32_t x8nmodp(unsigned long long n) {
    uint32_t sq = multmodp(multmodp(multmodp(1u << 30, 1u << 30), multmodp(1u << 30, 1u << 30)),
                           multmodp(multmodp(1u << 30, 1u << 30), multmodp(1u << 30, 1u << 30)));     // x^8 = (x^1)^8
    uint32_t p = 1u << 31;                                               // x^0
    while (n) { if (n & 1) p = multmodp(sq, p); sq = multmodp(sq, sq); n >>= 1; }
    return p;
}

// CRC-32 of the IHDR chunk (type + 13 data bytes): a function of (w, h, colour type) only, computed on the host
static uint32_t ihdr_crc(const PngGeom &g) {
    const uint8_t b[17] = {'I', 'H', 'D', 'R', (uint8_t)(g.w >> 24), (uint8_t)(g.w >> 16), (uint8_t)(g.w >> 8), (uint8_t)g.w,
                           (uint8_t)(g.h >> 24), (uint8_t)(g.h >> 16), (uint8_t)(g.h >> 8), (uint8_t)g.h, 8, (uint8_t)(g.bpp == 4 ? 6 : 2), 0, 0, 0};
    uint32_t c = 0xffffffffu;
    for (int k = 0; k < 17; ++k) c = crc_byte(c, b[k]);
    return c ^ 0xffffffffu;
}

constexpr int PNG_SEG = 4096;
struct SegSum { uint32_t crc, a, b; };     // finalized CRC-32 of the segment; Adler-32 partial sums of its raw bytes (a without the initial 1)

// Where a flat work item of the kernels below lives and what its frame looks like.  Every kernel body reads per-frame
// quantities through one of two accessors:
//   *Uniform  a b200timg_batch: every frame has one PngGeom / GfxSpec, items frame-major at a fixed count per frame,
//             frame f's pixels at frames + f * w * h * 4, its slots at f * stride
//   *Mixed    a mixed batch: frame f's geometry, pixels and slots in desc[f] (MixedGfxFrame), its items
//             start[f] .. start[f + 1] - 1 of a flat list, found by binary search (mixed_owner)
// The bodies are __forceinline__ templates called from the unchanged uniform kernels, so those compile as before.
__host__ __device__ inline int png_crc_segs(const PngGeom &g) { return (int)((4 + g.zlib_len + PNG_SEG - 1) / PNG_SEG); }
__host__ __device__ inline int png_raw_segs(const PngGeom &g) { return (int)((g.raw_len + PNG_SEG - 1) / PNG_SEG); }

struct CheckItem { const uint8_t *fb; PngGeom g; long long s; int nseg_crc; };
struct CheckUniform {
    const uint8_t *frames; const PngGeom &g; int n_frames, nseg_crc, nseg_raw;
    __device__ __forceinline__ long long total() const { return ((long long)nseg_crc + nseg_raw) * n_frames; }
    __device__ __forceinline__ CheckItem at(long long t) const {
        const long long per = (long long)nseg_crc + nseg_raw, f = t / per, s = t - f * per;
        return CheckItem{frames + f * (long long)g.w * g.h * 4, g, s, nseg_crc};
    }
};
struct CheckMixed {
    const uint8_t *frames; const MixedGfxFrame *desc; const unsigned *start; int n_frames, with_crc;
    __device__ __forceinline__ long long total() const { return start[n_frames]; }
    __device__ __forceinline__ CheckItem at(long long t) const {
        const int f = mixed_owner(start, n_frames, (unsigned)t);
        const MixedGfxFrame &D = desc[f];
        return CheckItem{frames + D.fb, D.g, t - start[f], with_crc ? png_crc_segs(D.g) : 0};
    }
};

// One thread per PNG_SEG-byte segment of the region [type "IDAT" .. end of zlib stream] (CRC, over the bytes
// png_byte gives with the Adler field zero) and of the raw scanline stream (Adler).  Reads the frames only.
template <class A>
__device__ __forceinline__ void png_check_body(const A &a, SegSum *__restrict__ seg) {
    const long long total = a.total();
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const CheckItem it = a.at(t);
        const PngGeom &g = it.g;
        const uint8_t *fb = it.fb;
        const long long s = it.s;
        const int nseg_crc = it.nseg_crc;
        SegSum r = {0, 0, 0};
        if (s < nseg_crc) {
            const long long lo = s * PNG_SEG, hi = min(lo + PNG_SEG, 4 + g.zlib_len);
            const long long o0 = g.idat_data_off - 4;                                  // the chunk type
            uint32_t c = 0xffffffffu;
            for (long long i = lo; i < hi; ++i) c = crc_byte(c, png_byte(fb, g, o0 + i, 0, 0, 0));
            r.crc = c ^ 0xffffffffu;
        } else {
            const long long lo = (s - nseg_crc) * PNG_SEG, hi = min(lo + PNG_SEG, g.raw_len);
            uint32_t a = 0, b = 0;
            for (long long i = lo; i < hi; ++i) { a += raw_byte(fb, g, i); b += a; }   // <= 4096 * 255 and its triangle sum: no overflow
            r.a = a % 65521u; r.b = b % 65521u;
        }
        seg[t] = r;
    }
}
__global__ void __launch_bounds__(128)
png_check_kernel(const uint8_t *__restrict__ frames, PngGeom g, int n_frames, int nseg_crc, int nseg_raw, SegSum *__restrict__ seg) {
    png_check_body(CheckUniform{frames, g, n_frames, nseg_crc, nseg_raw}, seg);
}
__global__ void __launch_bounds__(128)
png_check_mixed_kernel(const uint8_t *__restrict__ frames, const MixedGfxFrame *__restrict__ desc, const unsigned *__restrict__ start,
                       int n_frames, int with_crc, SegSum *__restrict__ seg) {
    png_check_body(CheckMixed{frames, desc, start, n_frames, with_crc}, seg);
}

// Combines the segment sums s of frame f into two words: sums[2f] = Adler-32, sums[2f+1] = IDAT CRC-32.
// png != nullptr: also writes the three checksum fields into the file at png + f * png_len.
__device__ __forceinline__ void png_seal_body(const PngGeom &g, int f, int nseg_crc, int nseg_raw, const SegSum *__restrict__ s,
                                              uint32_t xn_full, uint32_t *__restrict__ sums, uint8_t *__restrict__ png, uint32_t ihdr) {
    // Adler-32 of the raw stream: A = 1 + sum a_i, B = sum over segments (b_i + len_i * A_before_i)
    unsigned long long A = 1, B = 0;
    for (int i = 0; i < nseg_raw; ++i) {
        const long long len = min((long long)PNG_SEG, g.raw_len - (long long)i * PNG_SEG);
        B = (B + s[nseg_crc + i].b + (unsigned long long)(len % 65521) * A) % 65521ull;
        A = (A + s[nseg_crc + i].a) % 65521ull;
    }
    const uint32_t adler = (uint32_t)((B << 16) | A);
    // CRC-32 of "IDAT" + zlib stream: segment CRCs were computed with the Adler field still zero.  CRC is linear over
    // GF(2): crc(m ^ d) = crc(m) ^ crc0(d) for equal lengths (crc0 = without init / final xor), and the 4 Adler bytes
    // are the last 4 bytes of the region, so their contribution is the plain register update over those bytes.
    uint32_t crc = 0;
    const long long region = 4 + g.zlib_len;
    for (int i = 0; i < nseg_crc; ++i) {
        const long long len = min((long long)PNG_SEG, region - (long long)i * PNG_SEG);
        const uint32_t xn = len == PNG_SEG ? xn_full : x8nmodp((unsigned long long)len);
        crc = i == 0 ? s[i].crc : (multmodp(xn, crc) ^ s[i].crc);     // crc32_combine(crc, s[i].crc, len)
    }
    uint32_t d = 0;                                                    // zero-init, no final xor: pure linear part
    for (int k = 3; k >= 0; --k) d = crc_byte(d, (uint8_t)(adler >> (8 * k)));
    crc ^= d;
    sums[2 * f] = adler;
    sums[2 * f + 1] = crc;
    if (png) {
        uint8_t *p = png + (long long)f * g.png_len;
        put_be32(p + 29, ihdr);
        put_be32(p + g.idat_data_off + g.zlib_len - 4, adler);
        put_be32(p + g.idat_data_off + g.zlib_len, crc);
    }
}
// one CTA per frame, its segments frame-major
__global__ void __launch_bounds__(32)
png_seal_kernel(PngGeom g, int nseg_crc, int nseg_raw, const SegSum *__restrict__ seg, uint32_t xn_full, uint32_t *__restrict__ sums,
                uint8_t *__restrict__ png, uint32_t ihdr) {
    const int f = blockIdx.x;
    if (threadIdx.x != 0) return;
    png_seal_body(g, f, nseg_crc, nseg_raw, seg + (long long)f * (nseg_crc + nseg_raw), xn_full, sums, png, ihdr);
}
// one CTA per frame of a mixed batch, its segments from start[f]
__global__ void __launch_bounds__(32)
png_seal_mixed_kernel(const MixedGfxFrame *__restrict__ desc, const unsigned *__restrict__ start, int with_crc,
                      const SegSum *__restrict__ seg, uint32_t xn_full, uint32_t *__restrict__ sums) {
    const int f = blockIdx.x;
    if (threadIdx.x != 0) return;
    const PngGeom g = desc[f].g;
    png_seal_body(g, f, with_crc ? png_crc_segs(g) : 0, png_raw_segs(g), seg + start[f], xn_full, sums, nullptr, 0);
}

// The checksum pass shared by the PNG files and the framed batches: segment sums from the frames, then two words per
// frame in ctx->png_sums (and, when png is given, the checksum fields of those files).
static int launch_png_sums(b200timg_ctx *ctx, const uint8_t *d_frames, const PngGeom &g, int n_frames, uint8_t *d_png,
                           bool with_crc = true);

// ---- base64 (src/timg-base64.h:28-53): n bytes -> 4*ceil(n/3) characters, per frame ---------------------
__global__ void __launch_bounds__(256)
base64_kernel(const uint8_t *__restrict__ in, long long in_stride, long long n, char *__restrict__ out, long long out_stride, int n_frames) {
    const long long groups = (n + 2) / 3, total = groups * n_frames;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long f = t / groups, gi = t - f * groups;
        const uint8_t *p = in + f * in_stride + gi * 3;
        const long long left = n - gi * 3;
        const uint32_t b0 = p[0], b1 = left > 1 ? p[1] : 0, b2 = left > 2 ? p[2] : 0;
        const char *tab = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
        char *o = out + f * out_stride + gi * 4;
        o[0] = tab[b0 >> 2];
        o[1] = tab[((b0 & 3) << 4) | (b1 >> 4)];
        o[2] = left > 1 ? tab[((b1 & 15) << 2) | (b2 >> 6)] : '=';
        o[3] = left > 2 ? tab[b2 & 63] : '=';
    }
}

static unsigned png_grid(b200timg_ctx *ctx, long long items, int threads) {
    long long b = (items + threads - 1) / threads;
    const long long cap = (long long)ctx->sm_count * 32;
    if (b > cap) b = cap;
    return (unsigned)(b < 1 ? 1 : b);
}

static int launch_png_sums(b200timg_ctx *ctx, const uint8_t *d_frames, const PngGeom &g, int n_frames, uint8_t *d_png,
                           bool with_crc) {
    const int nseg_crc = with_crc ? (int)((4 + g.zlib_len + PNG_SEG - 1) / PNG_SEG) : 0, nseg_raw = (int)((g.raw_len + PNG_SEG - 1) / PNG_SEG);
    B2_CUDA(ctx, ctx->cells.reserve(sizeof(SegSum) * (size_t)(nseg_crc + nseg_raw) * n_frames));
    B2_CUDA(ctx, ctx->png_sums.reserve(2 * sizeof(uint32_t) * (size_t)n_frames));
    SegSum *seg = ctx->cells.as<SegSum>();
    B2_KERNEL(ctx, "png_check_kernel");
    png_check_kernel<<<png_grid(ctx, (long long)(nseg_crc + nseg_raw) * n_frames, 128), 128, 0, ctx->stream>>>(d_frames, g, n_frames, nseg_crc, nseg_raw, seg);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "png_seal_kernel");
    png_seal_kernel<<<n_frames, 32, 0, ctx->stream>>>(g, nseg_crc, nseg_raw, seg, x8nmodp(PNG_SEG), ctx->png_sums.as<uint32_t>(), d_png, ihdr_crc(g));
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

// n frames (RGBA8, device) -> n PNG files at d_png + f * png_len; optionally their base64 text at d_b64 + f * b64_len
int launch_png(b200timg_ctx *ctx, const uint8_t *d_frames, int w, int h, int n_frames, int rgb24, uint8_t *d_png, char *d_b64) {
    const PngGeom g = png_geom(w, h, rgb24);
    if (g.zlib_len > 0x7fffffffll) return ctx->fail(B200TIMG_EINVAL, "png: frame too large for one IDAT chunk");
    B2_KERNEL(ctx, "png_fill_kernel");
    png_fill_kernel<<<png_grid(ctx, g.png_len * n_frames, 256), 256, 0, ctx->stream>>>(d_frames, d_png, g, n_frames);
    B2_LAUNCH_CHECK(ctx);
    B2_TRY(launch_png_sums(ctx, d_frames, g, n_frames, d_png));
    if (d_b64) {
        const long long b64_len = (g.png_len + 2) / 3 * 4;
        B2_KERNEL(ctx, "base64_kernel");
        base64_kernel<<<png_grid(ctx, (g.png_len + 2) / 3 * n_frames, 256), 256, 0, ctx->stream>>>(d_png, g.png_len, g.png_len, d_b64, b64_len, n_frames);
        B2_LAUNCH_CHECK(ctx);
    }
    return B200TIMG_OK;
}

// ---- kitty / iTerm2 framing (src/kitty-canvas.cc:190-229, src/iterm2-canvas.cc:66-73) ------------------------------
// The framed text of a frame is cut into tiles of GFX_BYTES PNG bytes: kitty's chunk, 4096 base64 characters
// (kitty-canvas.cc:43-44).  Tile c starts at header + c * (4096 + separator) in the frame's text; tile 0 carries
// the header, every tile but the last the separator (kitty) and the last one the trailer.  kitty's tmux form wraps
// every command in tmux's passthrough and follows the trailer with a grid of Unicode placeholders (below).
constexpr int GFX_BYTES = 3072;
constexpr int GFX_SEP = 13;                 // "\e\\\e_Gq=2,m=<0|1>;"
constexpr int GFX_SEP_TMUX = 24;            // "\e\e\\" "\e\\" "\ePtmux;" "\e\e_G" "q=2,m=<0|1>;"

// GfxSpec (common.cuh): one frame's framing; the placeholder fields are read for the tmux form only
static GfxSpec gfx_spec(const b200timg_graphics &gr, const PngGeom &g) {
    GfxSpec s{gr.protocol & ~B200TIMG_DEFLATE, g.w, g.h, g.png_len, (g.png_len + GFX_BYTES - 1) / GFX_BYTES, 0, 0, 0};
    if (s.protocol == B200TIMG_KITTY_TMUX) {
        s.cols = g.w / gr.cell_x_px;
        s.rows = (g.h + gr.cell_y_px - 1) / gr.cell_y_px;
        s.indent = gr.indent_cells;
    }
    return s;
}

// ---- kitty's row / column diacritics (Unicode placeholders, src/kitty-canvas.cc:255-344) ----------------------------
// Value v (a placeholder's row, its column, the top byte of the image id) is written as the v-th combining mark of the
// kitty graphics protocol's list (rowcolumn-diacritics.txt), nothing for v >= DIAC_N.  The list, as runs of consecutive
// code points:
struct CodeRun { uint32_t first; int count; };
constexpr CodeRun kDiacRuns[] = {
    {0x0305, 1}, {0x030D, 2}, {0x0310, 1}, {0x0312, 1}, {0x033D, 3}, {0x0346, 1}, {0x034A, 3}, {0x0350, 3},
    {0x0357, 1}, {0x035B, 1}, {0x0363, 13}, {0x0483, 5}, {0x0592, 4}, {0x0597, 3}, {0x059C, 6}, {0x05A8, 2},
    {0x05AB, 2}, {0x05AF, 1}, {0x05C4, 1}, {0x0610, 8}, {0x0657, 5}, {0x065D, 2}, {0x06D6, 7}, {0x06DF, 4},
    {0x06E4, 1}, {0x06E7, 2}, {0x06EB, 2}, {0x0730, 1}, {0x0732, 2}, {0x0735, 2}, {0x073A, 1}, {0x073D, 1},
    {0x073F, 3}, {0x0743, 1}, {0x0745, 1}, {0x0747, 1}, {0x0749, 2}, {0x07EB, 7}, {0x07F3, 1}, {0x0816, 4},
    {0x081B, 9}, {0x0825, 3}, {0x0829, 5}, {0x0951, 1}, {0x0953, 2}, {0x0F82, 2}, {0x0F86, 2}, {0x135D, 3},
    {0x17DD, 1}, {0x193A, 1}, {0x1A17, 1}, {0x1A75, 8}, {0x1B6B, 1}, {0x1B6D, 7}, {0x1CD0, 3}, {0x1CDA, 2},
    {0x1CE0, 1}, {0x1DC0, 2}, {0x1DC3, 7}, {0x1DCB, 2}, {0x1DD1, 22}, {0x1DFE, 1}, {0x20D0, 2}, {0x20D4, 4},
    {0x20DB, 2}, {0x20E1, 1}, {0x20E7, 1}, {0x20E9, 1}, {0x20F0, 1}, {0x2CEF, 3}, {0x2DE0, 32}, {0xA66F, 1},
    {0xA67C, 2}, {0xA6F0, 2}, {0xA8E0, 18}, {0xAAB0, 1}, {0xAAB2, 2}, {0xAAB7, 2}, {0xAABE, 2}, {0xAAC1, 1},
    {0xFE20, 7}, {0x10A0F, 1}, {0x10A38, 1}, {0x1D185, 5}, {0x1D1AA, 4}, {0x1D242, 3},
};
constexpr int DIAC_N = 297;
// Byte parity with the reference: its table spells the 14 code points above U+FFFF (values 283..296) as the string
// literals "\u10A0F" and so on, and a C++ \u escape takes exactly four hex digits, so the compiled reference writes
// U+10A0 followed by the letter 'F' instead of U+10A0F.  The table below reproduces those bytes (still 4 per value):
// UTF-8 of cp >> 4, then the last hex digit as an upper-case ASCII letter or digit.
struct DiacTable {
    uint32_t utf8[DIAC_N];                  // bytes of value v, first byte in the low 8 bits
    uint8_t len[DIAC_N];                    // 2, 3, or 4 (the values above U+FFFF)
    uint32_t prefix[DIAC_N + 1];            // prefix[v] = len[0] + ... + len[v - 1]
};
constexpr uint32_t utf8_bmp(uint32_t cp, int &n) {        // cp in [0x80, 0xFFFF]
    if (cp < 0x800) { n = 2; return (0xC0u | cp >> 6) | (0x80u | (cp & 63)) << 8; }
    n = 3;
    return (0xE0u | cp >> 12) | (0x80u | (cp >> 6 & 63)) << 8 | (0x80u | (cp & 63)) << 16;
}
constexpr DiacTable make_diac_table() {
    DiacTable t{};
    int v = 0;
    for (const CodeRun &r : kDiacRuns)
        for (int k = 0; k < r.count; ++k, ++v) {
            const uint32_t cp = r.first + k;
            int n = 0;
            uint32_t b = utf8_bmp(cp > 0xffff ? cp >> 4 : cp, n);
            if (cp > 0xffff) b |= (uint32_t)"0123456789ABCDEF"[cp & 15] << (8 * n++);
            t.utf8[v] = b;
            t.len[v] = (uint8_t)n;
            t.prefix[v + 1] = t.prefix[v] + n;
        }
    return t;
}
constexpr int diac_count() { int n = 0; for (const CodeRun &r : kDiacRuns) n += r.count; return n; }
static_assert(diac_count() == DIAC_N, "kitty's list has 297 diacritics");
static constexpr DiacTable kDiac = make_diac_table();           // the host's copy (frame sizes)
__constant__ DiacTable c_diac = make_diac_table();              // the device's copy

__host__ __device__ inline const DiacTable &diac() {
#ifdef __CUDA_ARCH__
    return c_diac;
#else
    return kDiac;
#endif
}
__host__ __device__ inline int diac_len(long long v) { return v < DIAC_N ? diac().len[v] : 0; }
__host__ __device__ inline long long diac_prefix(long long v) { return diac().prefix[v < DIAC_N ? v : DIAC_N]; }   // sum of diac_len(u), u < v
__device__ __forceinline__ int put_diac(char *p, long long v) {
    if (v >= DIAC_N) return 0;
    const uint32_t b = c_diac.utf8[v];
    const int n = c_diac.len[v];
    for (int k = 0; k < n; ++k) p[k] = (char)(b >> (8 * k));
    return n;
}

// p == nullptr: count only
__host__ __device__ inline int put_str(char *p, const char *s) {
    int n = 0;
    for (; s[n]; ++n) if (p) p[n] = s[n];
    return n;
}
__host__ __device__ inline int put_dec(char *p, unsigned long long v) {
    char t[20];
    int n = 0;
    do { t[n++] = (char)('0' + v % 10); v /= 10; } while (v);
    if (p) for (int i = 0; i < n; ++i) p[i] = t[n - 1 - i];
    return n;
}
__host__ __device__ inline char *at(char *p, int n) { return p ? p + n : nullptr; }

// "\e_Ga=T,i=<id>,q=2,f=100,m=<0|1>;" (kitty-canvas.cc:197-203),
// "\ePtmux;\e\e_Ga=T,i=<id>,q=2,f=100,m=<0|1>,U=1,c=<cols>,r=<rows>;" (the tmux form: passthrough, escape doubled) or
// "\e]1337;File=size=<n>;width=<w>px;height=<h>px;inline=1:" (iterm2-canvas.cc:67-69)
__host__ __device__ inline int gfx_header(char *p, const GfxSpec &s, uint32_t id) {
    int n = 0;
    if (s.protocol != B200TIMG_ITERM2) {
        const bool tmux = s.protocol == B200TIMG_KITTY_TMUX;
        if (tmux) n += put_str(at(p, n), "\033Ptmux;\033");
        n += put_str(at(p, n), "\033_Ga=T,i=");
        n += put_dec(at(p, n), id);
        n += put_str(at(p, n), ",q=2,f=100,m=");
        n += put_dec(at(p, n), s.png_len > GFX_BYTES);
        if (tmux) {
            n += put_str(at(p, n), ",U=1,c=");
            n += put_dec(at(p, n), (unsigned)s.cols);
            n += put_str(at(p, n), ",r=");
            n += put_dec(at(p, n), (unsigned)s.rows);
        }
        n += put_str(at(p, n), ";");
    } else {
        n += put_str(at(p, n), "\033]1337;File=size=");
        n += put_dec(at(p, n), (unsigned long long)s.png_len);
        n += put_str(at(p, n), ";width=");
        n += put_dec(at(p, n), (unsigned)s.w);
        n += put_str(at(p, n), "px;height=");
        n += put_dec(at(p, n), (unsigned)s.h);
        n += put_str(at(p, n), "px;inline=1:");
    }
    return n;
}
// what follows tile c: kitty's chunk separator (kitty-canvas.cc:212-220) or the trailer (:222-229 / iterm2-canvas.cc:72-73).
// The tmux form's trailer ends the passthrough and carries the "\r" that starts the placeholder grid (kitty-canvas.cc:60).
__host__ __device__ inline int gfx_suffix(char *p, const GfxSpec &s, long long c) {
    const bool tmux = s.protocol == B200TIMG_KITTY_TMUX;
    if (c + 1 < s.tiles) {
        if (s.protocol == B200TIMG_ITERM2) return 0;
        const int n = put_str(p, tmux ? "\033\033\\\033\\\033Ptmux;\033\033_Gq=2,m=" : "\033\\\033_Gq=2,m=");
        return n + put_dec(at(p, n), s.png_len - (c + 1) * GFX_BYTES > GFX_BYTES) + put_str(at(p, n + 1), ";");
    }
    return put_str(p, s.protocol == B200TIMG_KITTY ? "\033\\\n" : tmux ? "\033\033\\\033\\\r" : "\a\n");
}
__host__ __device__ inline int gfx_sep(const GfxSpec &s) {
    return s.protocol == B200TIMG_KITTY ? GFX_SEP : s.protocol == B200TIMG_KITTY_TMUX ? GFX_SEP_TMUX : 0;
}
// header, base64 of the PNG with its separators and the trailer: where the tmux form's placeholder grid starts
__host__ __device__ inline long long gfx_text_len(const GfxSpec &s, uint32_t id) {
    return gfx_header(nullptr, s, id) + (s.png_len + 2) / 3 * 4 + (long long)gfx_sep(s) * (s.tiles - 1) + gfx_suffix(nullptr, s, s.tiles - 1);
}

// ---- the tmux form's placeholder grid (AppendUnicodePicureTiles, src/kitty-canvas.cc:58-74) ---------------------------
// rows lines of
//     ["\e[<indent>C" if indent > 0] "\e[38:2:<id>>16&255>:<id>>8&255>:<id&255>m"
//     cols x ( U+10EEEE  D(r) D(c) [D(id >> 24) if id >> 24 != 0] )   "\e[39m\n\r"
// with D(v) the diacritic of value v.  Only D(r) differs between rows, so row r starts at
// r * grid_row_base + cols * diac_prefix(r) within the grid, and the grid has rows * grid_row_base + cols * diac_prefix(rows) bytes.
constexpr int GRID_ROW_TAIL = 7;            // "\e[39m\n\r"
__host__ __device__ inline int grid_row_head(char *p, const GfxSpec &s, uint32_t id) {
    int n = 0;
    if (s.indent > 0) {
        n += put_str(at(p, n), "\033[");
        n += put_dec(at(p, n), (unsigned)s.indent);
        n += put_str(at(p, n), "C");
    }
    n += put_str(at(p, n), "\033[38:2:");
    n += put_dec(at(p, n), (id >> 16) & 255);
    n += put_str(at(p, n), ":");
    n += put_dec(at(p, n), (id >> 8) & 255);
    n += put_str(at(p, n), ":");
    n += put_dec(at(p, n), id & 255);
    n += put_str(at(p, n), "m");
    return n;
}
// bytes of a row without its row diacritics
__host__ __device__ inline long long grid_row_base(const GfxSpec &s, uint32_t id) {
    const uint32_t msb = id >> 24;
    return grid_row_head(nullptr, s, id) + (long long)s.cols * (4 + (msb ? diac_len(msb) : 0)) + diac_prefix(s.cols) + GRID_ROW_TAIL;
}

// A closed formula: every part that depends on the id (its digits, the colour's digits, the msb diacritic) is largest
// at id = 0xffffffff, so the size at that id bounds the size at any id of the same geometry.
__host__ __device__ inline size_t gfx_frame_size(const GfxSpec &s, uint32_t id) {
    long long n = gfx_text_len(s, id);
    if (s.protocol == B200TIMG_KITTY_TMUX) n += (long long)s.rows * grid_row_base(s, id) + (long long)s.cols * diac_prefix(s.rows);
    return (size_t)n;
}

__device__ __forceinline__ char b64_char(uint32_t v) {
    return (char)(v < 26 ? 'A' + v : v < 52 ? 'a' + (v - 26) : v < 62 ? '0' + (v - 52) : v == 62 ? '+' : '/');
}

// B200TIMG_DEFLATE: a frame's PNG length (and so its kitty chunks and iTerm2's size=) comes from png_lens on the
// device; s then describes the stored-size bound
__host__ __device__ inline GfxSpec frame_spec(const GfxSpec &s, const uint32_t *png_lens, int f) {
    GfxSpec r = s;
    if (png_lens) { r.png_len = png_lens[f]; r.tiles = (r.png_len + GFX_BYTES - 1) / GFX_BYTES; }
    return r;
}

constexpr int GFX_THREADS = 256;
// s_txt[shift .. end) -> base[shift .. end), base 16-byte aligned: 16-byte stores, bytes at the two ends
__device__ __forceinline__ void copy_out16(char *base, const char *s_txt, int shift, int end) {
    const int nvec = (end + 15) / 16;
    for (int v = threadIdx.x; v < nvec; v += GFX_THREADS) {
        const int a = 16 * v, b = a + 16;
        if (a >= shift && b <= end) *reinterpret_cast<uint4 *>(base + a) = *reinterpret_cast<const uint4 *>(s_txt + a);
        else for (int k = max(a, shift); k < min(b, end); ++k) base[k] = s_txt[k];
    }
}

// tile c of frame f: its frame's framing (frame_spec applied), PNG geometry, pixels, IHDR CRC and PNG slot
struct TileItem { int f; long long c; GfxSpec s; PngGeom g; const uint8_t *fb; uint32_t ihdr; long long png0; };
struct TileUniform {
    const uint8_t *frames; const PngGeom &g; const GfxSpec &s_max; int n_frames; uint32_t ihdr; long long png_stride;
    __device__ __forceinline__ long long total() const { return (long long)n_frames * s_max.tiles; }
    __device__ __forceinline__ TileItem at(long long t, const uint32_t *png_lens) const {
        const int f = (int)(t / s_max.tiles);
        return TileItem{f, t - (long long)f * s_max.tiles, frame_spec(s_max, png_lens, f), g, frames + (long long)f * g.w * g.h * 4,
                        ihdr, f * png_stride};
    }
};
struct TileMixed {
    const uint8_t *frames; const MixedGfxFrame *desc; const unsigned *start; int n_frames;
    __device__ __forceinline__ long long total() const { return start[n_frames]; }
    __device__ __forceinline__ TileItem at(long long t, const uint32_t *png_lens) const {
        const int f = mixed_owner(start, n_frames, (unsigned)t);
        const MixedGfxFrame &D = desc[f];
        return TileItem{f, t - start[f], frame_spec(D.s, png_lens, f), D.g, frames + D.fb, D.ihdr, D.png_off};
    }
};

// One CTA per tile (grid-stride): stage the tile's PNG bytes from the frame, build its text in shared memory at the
// destination's alignment mod 16, copy it out with 16-byte stores.  A frame that would end beyond out_cap is skipped.
template <class A>
__device__ __forceinline__ void graphics_emit_body(const A &a, const uint32_t *__restrict__ ids, const uint32_t *__restrict__ sums,
                                                   const uint64_t *__restrict__ offsets, char *__restrict__ out, unsigned long long out_cap,
                                                   const uint8_t *__restrict__ pngs, const uint32_t *__restrict__ png_lens) {
    __shared__ uint8_t s_png[GFX_BYTES];
    __shared__ __align__(16) char s_txt[4352];          // 15 (alignment) + header (<= 72) + 4096 + separator (<= 24)
    const long long total = a.total();
    for (long long t = blockIdx.x; t < total; t += gridDim.x) {
        const TileItem it = a.at(t, png_lens);
        const int f = it.f;
        const long long c = it.c;
        const GfxSpec &s = it.s;
        if (c >= s.tiles || offsets[f + 1] > out_cap) continue;          // the same for every thread of the CTA
        const uint32_t id = ids ? ids[f] : 0u;
        const uint8_t *fb = it.fb;
        const uint32_t adler = sums[2 * f], crc = sums[2 * f + 1];
        const long long lo = c * GFX_BYTES;
        const int nb = (int)min((long long)GFX_BYTES, s.png_len - lo);
        for (int k = threadIdx.x; k < nb; k += GFX_THREADS)
            s_png[k] = pngs ? pngs[it.png0 + lo + k] : png_byte(fb, it.g, lo + k, it.ihdr, crc, adler);
        const int hl = gfx_header(nullptr, s, id), pre = c == 0 ? hl : 0;
        const unsigned long long pos = c == 0 ? 0ull : (unsigned long long)hl + c * (4096ull + gfx_sep(s));
        char *dst = out + offsets[f] + pos;
        const int shift = (int)((uintptr_t)dst & 15);
        char *txt = s_txt + shift;
        const int groups = (nb + 2) / 3, body = pre + 4 * groups;
        const int len = body + gfx_suffix(nullptr, s, c);
        if (threadIdx.x == 0) {
            if (c == 0) gfx_header(txt, s, id);
            gfx_suffix(txt + body, s, c);
        }
        __syncthreads();
        for (int k = threadIdx.x; k < groups; k += GFX_THREADS) {      // EncodeBase64, src/timg-base64.h:28-53
            const int left = nb - 3 * k;
            const uint32_t b0 = s_png[3 * k], b1 = left > 1 ? s_png[3 * k + 1] : 0, b2 = left > 2 ? s_png[3 * k + 2] : 0;
            char *o = txt + pre + 4 * k;
            o[0] = b64_char(b0 >> 2);
            o[1] = b64_char(((b0 & 3) << 4) | (b1 >> 4));
            o[2] = left > 1 ? b64_char(((b1 & 15) << 2) | (b2 >> 6)) : '=';
            o[3] = left > 2 ? b64_char(b2 & 63) : '=';
        }
        __syncthreads();
        copy_out16(dst - shift, s_txt, shift, shift + len);             // dst - shift is 16-byte aligned
        __syncthreads();                                                // staging is reused by the next tile
    }
}
__global__ void __launch_bounds__(GFX_THREADS)
graphics_emit_kernel(const uint8_t *__restrict__ frames, PngGeom g, GfxSpec s_max, int n_frames, const uint32_t *__restrict__ ids,
                     const uint32_t *__restrict__ sums, uint32_t ihdr, const uint64_t *__restrict__ offsets, char *__restrict__ out,
                     unsigned long long out_cap, const uint8_t *__restrict__ pngs, long long png_stride,
                     const uint32_t *__restrict__ png_lens) {
    graphics_emit_body(TileUniform{frames, g, s_max, n_frames, ihdr, png_stride}, ids, sums, offsets, out, out_cap, pngs, png_lens);
}
__global__ void __launch_bounds__(GFX_THREADS)
graphics_emit_mixed_kernel(const uint8_t *__restrict__ frames, const MixedGfxFrame *__restrict__ desc, const unsigned *__restrict__ start,
                           int n_frames, const uint32_t *__restrict__ ids, const uint32_t *__restrict__ sums,
                           const uint64_t *__restrict__ offsets, char *__restrict__ out, unsigned long long out_cap,
                           const uint8_t *__restrict__ pngs, const uint32_t *__restrict__ png_lens) {
    graphics_emit_body(TileMixed{frames, desc, start, n_frames}, ids, sums, offsets, out, out_cap, pngs, png_lens);
}

// The tmux form's placeholder grid.  One CTA per item of up to GRID_CELLS placeholders of one row (grid-stride; a row
// of more cells is several items, so shared memory stays bounded however narrow the cells): each thread writes one
// placeholder at its closed-form position in shared memory, at the destination's alignment mod 16; the first item of
// a row adds the row's head, the last its tail; the text goes out with 16-byte stores.  Frames that would end beyond
// out_cap are skipped, as in graphics_emit_kernel.
constexpr int GRID_CELLS = 256;
__host__ __device__ inline int grid_segs(int cols) { return cols > GRID_CELLS ? (cols + GRID_CELLS - 1) / GRID_CELLS : 1; }
// piece sg of placeholder row r of frame f, that frame's framing (frame_spec applied) and its pieces per row
struct GridItem { int f, r, sg, segs; GfxSpec s; };
struct GridUniform {
    const GfxSpec &s_all; int n_frames;
    __device__ __forceinline__ int segs() const { return grid_segs(s_all.cols); }
    __device__ __forceinline__ long long total() const { return (long long)s_all.rows * segs() * n_frames; }
    __device__ __forceinline__ GridItem at(long long t, const uint32_t *png_lens) const {
        const int segs_ = segs();
        const long long per_frame = (long long)s_all.rows * segs_;
        const int f = (int)(t / per_frame);
        const long long q = t - (long long)f * per_frame;
        const int r = (int)(q / segs_);
        return GridItem{f, r, (int)(q - (long long)r * segs_), segs_, frame_spec(s_all, png_lens, f)};
    }
};
struct GridMixed {
    const MixedGfxFrame *desc; const unsigned *start; int n_frames;
    __device__ __forceinline__ long long total() const { return start[n_frames]; }
    __device__ __forceinline__ GridItem at(long long t, const uint32_t *png_lens) const {
        const int f = mixed_owner(start, n_frames, (unsigned)t);
        const GfxSpec s = frame_spec(desc[f].s, png_lens, f);
        const int segs_ = grid_segs(s.cols), q = (int)(t - start[f]), r = q / segs_;
        return GridItem{f, r, q - r * segs_, segs_, s};
    }
};
template <class A>
__device__ __forceinline__ void graphics_grid_body(const A &a, const uint32_t *__restrict__ ids, const uint64_t *__restrict__ offsets,
                                                   char *__restrict__ out, unsigned long long out_cap, const uint32_t *__restrict__ png_lens) {
    __shared__ __align__(16) char s_txt[4096];          // 15 (alignment) + head (<= 32) + 256 placeholders (<= 15 each) + tail (7)
    const long long total = a.total();
    for (long long t = blockIdx.x; t < total; t += gridDim.x) {
        const GridItem it = a.at(t, png_lens);
        const int f = it.f, r = it.r, sg = it.sg, segs = it.segs;
        const GfxSpec &s = it.s;
        if (offsets[f + 1] > out_cap) continue;          // the same for every thread of the CTA
        const uint32_t id = ids[f], msb = id >> 24;
        const int head = grid_row_head(nullptr, s, id);
        const int cell = 4 + diac_len(r) + (msb ? diac_len(msb) : 0);        // a placeholder without its column diacritic
        const long long row = gfx_text_len(s, id) + (long long)r * grid_row_base(s, id) + (long long)s.cols * diac_prefix(r);
        const int c0 = sg * GRID_CELLS, c1 = min(s.cols, c0 + GRID_CELLS);
        const bool last = sg == segs - 1;
        // this item's part of the row: bytes [lo, hi) counted from the row's start
        const long long lo = sg == 0 ? 0 : head + (long long)c0 * cell + diac_prefix(c0);
        const long long hi = head + (long long)c1 * cell + diac_prefix(c1) + (last ? GRID_ROW_TAIL : 0);
        char *dst = out + offsets[f] + row + lo;
        const int shift = (int)((uintptr_t)dst & 15), len = (int)(hi - lo);
        if (threadIdx.x == 0) {
            if (sg == 0) grid_row_head(s_txt + shift, s, id);
            if (last) put_str(s_txt + shift + len - GRID_ROW_TAIL, "\033[39m\n\r");
        }
        for (int c = c0 + threadIdx.x; c < c1; c += GFX_THREADS) {
            char *o = s_txt + shift + (int)(head + (long long)c * cell + diac_prefix(c) - lo);
            o[0] = '\xf4'; o[1] = '\x8e'; o[2] = '\xbb'; o[3] = '\xae';   // U+10EEEE, kitty's placeholder
            o += 4;
            o += put_diac(o, r);
            o += put_diac(o, c);
            if (msb) put_diac(o, msb);
        }
        __syncthreads();
        copy_out16(dst - shift, s_txt, shift, shift + len);
        __syncthreads();
    }
}
__global__ void __launch_bounds__(GFX_THREADS)
graphics_grid_kernel(GfxSpec s_all, int n_frames, const uint32_t *__restrict__ ids, const uint64_t *__restrict__ offsets,
                     char *__restrict__ out, unsigned long long out_cap, const uint32_t *__restrict__ png_lens) {
    graphics_grid_body(GridUniform{s_all, n_frames}, ids, offsets, out, out_cap, png_lens);
}
__global__ void __launch_bounds__(GFX_THREADS)
graphics_grid_mixed_kernel(const MixedGfxFrame *__restrict__ desc, const unsigned *__restrict__ start, int n_frames,
                           const uint32_t *__restrict__ ids, const uint64_t *__restrict__ offsets, char *__restrict__ out,
                           unsigned long long out_cap, const uint32_t *__restrict__ png_lens) {
    graphics_grid_body(GridMixed{desc, start, n_frames}, ids, offsets, out, out_cap, png_lens);
}

// ---- B200TIMG_DEFLATE: the PNG of every frame, with a compressed zlib body, in a slot of the stored size ----------------
// raw_fill_kernel writes the scanline streams, deflate.cu compresses them segment by segment, deflate_layout_kernel
// places the blocks and sizes the frames, deflate_pack_kernel writes the blocks, png_wrap_kernel everything around them
// but the IDAT CRC, which png_crc_kernel / png_crc_seal_kernel compute from the file's bytes.
// byte i of frame f's scanline stream and where it goes in the raw slots
struct RawItem { const uint8_t *fb; PngGeom g; long long i, dst; };
struct RawUniform {
    const uint8_t *frames; const PngGeom &g; int n_frames; long long raw_stride;
    __device__ __forceinline__ long long total() const { return g.raw_len * n_frames; }
    __device__ __forceinline__ RawItem at(long long t) const {
        const long long f = t / g.raw_len, i = t - f * g.raw_len;
        return RawItem{frames + f * (long long)g.w * g.h * 4, g, i, f * raw_stride + i};
    }
};
struct RawMixed {
    const uint8_t *frames; const MixedGfxFrame *desc; const unsigned long long *start; int n_frames;
    __device__ __forceinline__ long long total() const { return (long long)start[n_frames]; }
    __device__ __forceinline__ RawItem at(long long t) const {
        const int f = mixed_owner(start, n_frames, (unsigned long long)t);
        const MixedGfxFrame &D = desc[f];
        const long long i = t - (long long)start[f];
        return RawItem{frames + D.fb, D.g, i, D.raw_off + i};
    }
};
template <class A>
__device__ __forceinline__ void raw_fill_body(const A &a, uint8_t *__restrict__ raw) {
    const long long total = a.total();
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const RawItem it = a.at(t);
        raw[it.dst] = raw_byte(it.fb, it.g, it.i);
    }
}
__global__ void __launch_bounds__(256)
raw_fill_kernel(const uint8_t *__restrict__ frames, PngGeom g, int n_frames, uint8_t *__restrict__ raw, long long raw_stride) {
    raw_fill_body(RawUniform{frames, g, n_frames, raw_stride}, raw);
}
__global__ void __launch_bounds__(256)
raw_fill_mixed_kernel(const uint8_t *__restrict__ frames, const MixedGfxFrame *__restrict__ desc, const unsigned long long *__restrict__ start,
                      int n_frames, uint8_t *__restrict__ raw) {
    raw_fill_body(RawMixed{frames, desc, start, n_frames}, raw);
}

// frame f's PNG geometry, framing (stored-size bound), segment count and where its segments start in the flat lists
struct LayoutUniform {
    const PngGeom &g; const GfxSpec &s; int nseg;
    __device__ __forceinline__ const PngGeom &geom(int) const { return g; }
    __device__ __forceinline__ const GfxSpec &spec(int) const { return s; }
    __device__ __forceinline__ int segs(int) const { return nseg; }
    __device__ __forceinline__ long long seg(int f, int k) const { return (long long)f * nseg + k; }
};
struct LayoutMixed {
    const MixedGfxFrame *desc;
    __device__ __forceinline__ const PngGeom &geom(int f) const { return desc[f].g; }
    __device__ __forceinline__ const GfxSpec &spec(int f) const { return desc[f].s; }
    __device__ __forceinline__ int segs(int f) const { return (int)desc[f].g.nblocks; }
    __device__ __forceinline__ long long seg(int f, int k) const { return (long long)desc[f].seg0 + k; }
};

// One CTA: per frame, the bit offset of every block (in order; a stored block's size depends on where it lands), the
// PNG length and the frame's framed size; then offsets[] as their running sum.
template <class A>
__device__ __forceinline__ void deflate_layout_body(const A &a, int n_frames, const DeflateSeg *__restrict__ info,
                                                    unsigned long long *__restrict__ start, uint32_t *__restrict__ png_lens,
                                                    const uint32_t *__restrict__ ids, uint64_t *__restrict__ offsets) {
    __shared__ unsigned long long part[1024];
    for (int f = threadIdx.x; f < n_frames; f += blockDim.x) {
        unsigned long long e = 0;
        const PngGeom &g = a.geom(f);
        const GfxSpec &s = a.spec(f);
        const int nseg = a.segs(f);
        for (int k = 0; k < nseg; ++k) {
            const long long t = a.seg(f, k);
            start[t] = e;
            const DeflateSeg sg = info[t];
            const long long n = min((long long)65535, g.raw_len - (long long)k * 65535);
            e = sg.stored ? ((e + 10) & ~7ull) + 32 + 8ull * n : e + sg.bits;
        }
        png_lens[f] = (uint32_t)(g.idat_data_off + 2 + (e + 7) / 8 + 4 + 4 + 12);
        offsets[f + 1] = gfx_frame_size(frame_spec(s, png_lens, f), ids ? ids[f] : 0u);
    }
    __syncthreads();
    const int per = (n_frames + 1023) / 1024, a0 = min(n_frames, (int)threadIdx.x * per), b0 = min(n_frames, a0 + per);
    unsigned long long sum = 0;
    for (int f = a0; f < b0; ++f) sum += offsets[f + 1];
    part[threadIdx.x] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long r = 0;
        for (int i = 0; i < 1024; ++i) { const unsigned long long v = part[i]; part[i] = r; r += v; }
        offsets[0] = 0;
    }
    __syncthreads();
    unsigned long long r = part[threadIdx.x];
    for (int f = a0; f < b0; ++f) { r += offsets[f + 1]; offsets[f + 1] = r; }
}
__global__ void __launch_bounds__(1024)
deflate_layout_kernel(PngGeom g, GfxSpec s, int n_frames, int nseg, const DeflateSeg *__restrict__ info,
                      unsigned long long *__restrict__ start, uint32_t *__restrict__ png_lens, const uint32_t *__restrict__ ids,
                      uint64_t *__restrict__ offsets) {
    deflate_layout_body(LayoutUniform{g, s, nseg}, n_frames, info, start, png_lens, ids, offsets);
}
__global__ void __launch_bounds__(1024)
deflate_layout_mixed_kernel(const MixedGfxFrame *__restrict__ desc, int n_frames, const DeflateSeg *__restrict__ info,
                            unsigned long long *__restrict__ start, uint32_t *__restrict__ png_lens, const uint32_t *__restrict__ ids,
                            uint64_t *__restrict__ offsets) {
    deflate_layout_body(LayoutMixed{desc}, n_frames, info, start, png_lens, ids, offsets);
}

// one thread per frame: signature, IHDR, IDAT length and type, zlib header, Adler-32, IEND of the file at p
__device__ __forceinline__ void png_wrap_body(const PngGeom &g, int f, const uint32_t *__restrict__ png_lens, const uint32_t *__restrict__ sums,
                                              uint32_t ihdr, uint8_t *__restrict__ png, long long png0) {
    uint8_t *p = png + png0;
    PngGeom gf = g;
    gf.png_len = png_lens[f];
    gf.zlib_len = gf.png_len - gf.idat_data_off - 16;
    for (long long o = 0; o < gf.idat_data_off + 2; ++o) p[o] = png_byte(nullptr, gf, o, ihdr, 0, 0);
    put_be32(p + gf.idat_data_off + gf.zlib_len - 4, sums[2 * f]);
    for (long long o = gf.png_len - 12; o < gf.png_len; ++o) p[o] = png_byte(nullptr, gf, o, ihdr, 0, 0);
}
__global__ void png_wrap_kernel(PngGeom g, int n_frames, const uint32_t *__restrict__ png_lens, const uint32_t *__restrict__ sums,
                                uint32_t ihdr, uint8_t *__restrict__ png, long long png_stride) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames) return;
    png_wrap_body(g, f, png_lens, sums, ihdr, png, f * png_stride);
}
__global__ void png_wrap_mixed_kernel(const MixedGfxFrame *__restrict__ desc, int n_frames, const uint32_t *__restrict__ png_lens,
                                      const uint32_t *__restrict__ sums, uint8_t *__restrict__ png) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames) return;
    const MixedGfxFrame &D = desc[f];
    png_wrap_body(D.g, f, png_lens, sums, D.ihdr, png, D.png_off);
}

// piece s of frame f and its frame's PNG slot
struct PieceUniform {
    int n_frames, npiece; long long png_stride;
    __device__ __forceinline__ long long total() const { return (long long)npiece * n_frames; }
    __device__ __forceinline__ void at(long long t, long long &f, long long &s, long long &png0) const {
        f = t / npiece; s = t - f * npiece; png0 = f * png_stride;
    }
};
struct PieceMixed {
    const MixedGfxFrame *desc; const unsigned *start; int n_frames;
    __device__ __forceinline__ long long total() const { return start[n_frames]; }
    __device__ __forceinline__ void at(long long t, long long &f, long long &s, long long &png0) const {
        f = mixed_owner(start, n_frames, (unsigned)t); s = t - start[f]; png0 = desc[f].png_off;
    }
};
// CRC-32 of PNG_SEG-byte pieces of each file's [type "IDAT" .. end of zlib stream]; pieces past the end are empty
template <class A>
__device__ __forceinline__ void png_crc_body(const A &a, const uint8_t *__restrict__ png, const uint32_t *__restrict__ png_lens,
                                             SegSum *__restrict__ seg) {
    const long long total = a.total();
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        long long f, s, png0;
        a.at(t, f, s, png0);
        const long long region = (long long)png_lens[f] - 53;                 // "IDAT" + zlib stream
        const long long lo = s * PNG_SEG, hi = min(lo + PNG_SEG, region);
        const uint8_t *p = png + png0 + 37;
        uint32_t c = 0xffffffffu;
        for (long long i = lo; i < hi; ++i) c = crc_byte(c, p[i]);
        seg[t] = SegSum{c ^ 0xffffffffu, 0, 0};
    }
}
__global__ void __launch_bounds__(128)
png_crc_kernel(const uint8_t *__restrict__ png, long long png_stride, const uint32_t *__restrict__ png_lens, int n_frames,
               int npiece, SegSum *__restrict__ seg) {
    png_crc_body(PieceUniform{n_frames, npiece, png_stride}, png, png_lens, seg);
}
__global__ void __launch_bounds__(128)
png_crc_mixed_kernel(const MixedGfxFrame *__restrict__ desc, const unsigned *__restrict__ start, int n_frames,
                     const uint8_t *__restrict__ png, const uint32_t *__restrict__ png_lens, SegSum *__restrict__ seg) {
    png_crc_body(PieceMixed{desc, start, n_frames}, png, png_lens, seg);
}

// frame f's IDAT CRC from its npiece piece CRCs at seg + s0, into its file at png + png0
__device__ __forceinline__ void png_crc_seal_body(const SegSum *__restrict__ seg, long long s0, int f, int npiece,
                                                  const uint32_t *__restrict__ png_lens, uint32_t xn_full, uint8_t *__restrict__ png,
                                                  long long png0) {
    const long long region = (long long)png_lens[f] - 53;
    uint32_t crc = 0;
    for (int i = 0; i < npiece && (long long)i * PNG_SEG < region; ++i) {
        const long long len = min((long long)PNG_SEG, region - (long long)i * PNG_SEG);
        const uint32_t xn = len == PNG_SEG ? xn_full : x8nmodp((unsigned long long)len);
        crc = i == 0 ? seg[s0].crc : (multmodp(xn, crc) ^ seg[s0 + i].crc);
    }
    put_be32(png + png0 + 37 + region, crc);
}
__global__ void png_crc_seal_kernel(const SegSum *__restrict__ seg, int n_frames, int npiece, const uint32_t *__restrict__ png_lens,
                                    uint32_t xn_full, uint8_t *__restrict__ png, long long png_stride) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames) return;
    png_crc_seal_body(seg, (long long)f * npiece, f, npiece, png_lens, xn_full, png, f * png_stride);
}
__global__ void png_crc_seal_mixed_kernel(const MixedGfxFrame *__restrict__ desc, const unsigned *__restrict__ start, int n_frames,
                                          const SegSum *__restrict__ seg, const uint32_t *__restrict__ png_lens, uint32_t xn_full,
                                          uint8_t *__restrict__ png) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames) return;
    png_crc_seal_body(seg, start[f], f, (int)(start[f + 1] - start[f]), png_lens, xn_full, png, desc[f].png_off);
}

// The PNG files of a B200TIMG_DEFLATE batch at ctx->dfl_png (stride png_stride), their lengths at *png_lens and the
// frames' offsets at d_offsets.
static int launch_png_deflate(b200timg_ctx *ctx, const uint8_t *d_frames, const PngGeom &g, int n_frames, const GfxSpec &s,
                              const uint32_t *d_ids, uint64_t *d_offsets, long long png_stride, uint32_t **png_lens) {
    const int nseg = (int)g.nblocks, npiece = (int)((4 + g.zlib_len + PNG_SEG - 1) / PNG_SEG);
    const long long raw_stride = (g.raw_len + 15) / 16 * 16, segs = (long long)nseg * n_frames;
    B2_CUDA(ctx, ctx->dfl_raw.reserve((size_t)(raw_stride * n_frames)));
    B2_CUDA(ctx, ctx->dfl_scratch.reserve((size_t)(segs * DFL_SLOT)));
    B2_CUDA(ctx, ctx->dfl_png.reserve((size_t)(png_stride * n_frames)));
    const size_t info_b = sizeof(DeflateSeg) * segs, start_b = sizeof(unsigned long long) * segs, lens_b = (sizeof(uint32_t) * n_frames + 7) / 8 * 8;
    B2_CUDA(ctx, ctx->dfl_meta.reserve(info_b + start_b + lens_b + sizeof(SegSum) * (size_t)npiece * n_frames));
    DeflateSeg *info = ctx->dfl_meta.as<DeflateSeg>();
    unsigned long long *start = reinterpret_cast<unsigned long long *>(ctx->dfl_meta.as<uint8_t>() + info_b);
    uint32_t *lens = reinterpret_cast<uint32_t *>(ctx->dfl_meta.as<uint8_t>() + info_b + start_b);
    SegSum *pieces = reinterpret_cast<SegSum *>(ctx->dfl_meta.as<uint8_t>() + info_b + start_b + lens_b);
    uint8_t *raw = ctx->dfl_raw.as<uint8_t>(), *png = ctx->dfl_png.as<uint8_t>();
    B2_KERNEL(ctx, "raw_fill_kernel");
    raw_fill_kernel<<<png_grid(ctx, g.raw_len * n_frames, 256), 256, 0, ctx->stream>>>(d_frames, g, n_frames, raw, raw_stride);
    B2_LAUNCH_CHECK(ctx);
    B2_TRY(launch_png_sums(ctx, d_frames, g, n_frames, nullptr, false));          // Adler-32 only
    B2_TRY(launch_deflate(ctx, raw, raw_stride, (int)g.raw_len, n_frames, nseg, ctx->dfl_scratch.as<uint8_t>(), info));
    B2_KERNEL(ctx, "deflate_layout_kernel");
    deflate_layout_kernel<<<1, 1024, 0, ctx->stream>>>(g, s, n_frames, nseg, info, start, lens, d_ids, d_offsets);
    B2_LAUNCH_CHECK(ctx);
    B2_CUDA(ctx, cudaMemsetAsync(png, 0, (size_t)(png_stride * n_frames), ctx->stream));
    B2_TRY(launch_deflate_pack(ctx, raw, raw_stride, (int)g.raw_len, n_frames, nseg, ctx->dfl_scratch.as<uint8_t>(), info, start, png,
                               png_stride, (int)g.idat_data_off + 2));
    B2_KERNEL(ctx, "png_wrap_kernel");
    png_wrap_kernel<<<(n_frames + 127) / 128, 128, 0, ctx->stream>>>(g, n_frames, lens, ctx->png_sums.as<uint32_t>(), ihdr_crc(g), png,
                                                                     png_stride);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "png_crc_kernel");
    png_crc_kernel<<<png_grid(ctx, (long long)npiece * n_frames, 128), 128, 0, ctx->stream>>>(png, png_stride, lens, n_frames, npiece, pieces);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "png_crc_seal_kernel");
    png_crc_seal_kernel<<<(n_frames + 127) / 128, 128, 0, ctx->stream>>>(pieces, n_frames, npiece, lens, x8nmodp(PNG_SEG), png, png_stride);
    B2_LAUNCH_CHECK(ctx);
    *png_lens = lens;
    return B200TIMG_OK;
}

// n composed frames (RGBA8, device) -> their framed kitty / iTerm2 text at d_out + d_offsets[f].  Stored blocks:
// the offsets are already on the device, computed by the caller from b200timg_graphics_size.  B200TIMG_DEFLATE:
// the offsets are computed here, on the device.
int launch_graphics(b200timg_ctx *ctx, const uint8_t *d_frames, int w, int h, int n_frames, const b200timg_graphics &gr,
                    const uint32_t *d_ids, uint64_t *d_offsets, char *d_out, size_t out_cap) {
    const PngGeom g = png_geom(w, h, gr.rgb24);
    if (g.png_len > 0x7fffffffll) return ctx->fail(B200TIMG_EINVAL, "graphics: frame too large for one IDAT chunk");
    const GfxSpec s = gfx_spec(gr, g);
    const uint32_t *ids = s.protocol == B200TIMG_ITERM2 ? nullptr : d_ids;
    const long long png_stride = (g.png_len + 15) / 16 * 16;
    uint32_t *png_lens = nullptr;
    if (gr.protocol & B200TIMG_DEFLATE) B2_TRY(launch_png_deflate(ctx, d_frames, g, n_frames, s, ids, d_offsets, png_stride, &png_lens));
    else B2_TRY(launch_png_sums(ctx, d_frames, g, n_frames, nullptr));
    const long long tiles = s.tiles * n_frames, cap = (long long)ctx->sm_count * 16;
    B2_KERNEL(ctx, "graphics_emit_kernel");
    graphics_emit_kernel<<<(unsigned)std::min(tiles, cap), GFX_THREADS, 0, ctx->stream>>>(
        d_frames, g, s, n_frames, ids, ctx->png_sums.as<uint32_t>(), ihdr_crc(g), d_offsets, d_out, (unsigned long long)out_cap,
        png_lens ? ctx->dfl_png.as<uint8_t>() : nullptr, png_stride, png_lens);
    B2_LAUNCH_CHECK(ctx);
    if (s.protocol == B200TIMG_KITTY_TMUX) {
        const long long items = (long long)n_frames * s.rows * (s.cols > GRID_CELLS ? (s.cols + GRID_CELLS - 1) / GRID_CELLS : 1);
        B2_KERNEL(ctx, "graphics_grid_kernel");
        graphics_grid_kernel<<<(unsigned)std::min(items, cap), GFX_THREADS, 0, ctx->stream>>>(s, n_frames, ids, d_offsets, d_out,
                                                                                              (unsigned long long)out_cap, png_lens);
        B2_LAUNCH_CHECK(ctx);
    }
    return B200TIMG_OK;
}

// ---- mixed batches (b200timg_graphics_mixed_dev) ----------------------------------------------------------------------
// Frame f's descriptor and the starts of its items in every flat list of the call.  Its scaled pixels follow the
// earlier frames' back to back (as launch_scale_mixed writes them), its scanline and PNG slots likewise (16-byte
// aligned).  Stored blocks: the frame sizes are a closed formula, so the offsets are computed here and go up with the
// arena.
int plan_graphics_mixed(b200timg_ctx *ctx, const b200timg_mixed_batch *b, const b200timg_graphics &gr, MixedPlan &mp) {
    const int n = b->n_frames;
    const bool deflate = (gr.protocol & B200TIMG_DEFLATE) != 0, kitty = (gr.protocol & ~B200TIMG_DEFLATE) != B200TIMG_ITERM2;
    std::vector<MixedGfxFrame> desc(n);
    std::vector<unsigned> chk(n + 1), tile(n + 1), grid(n + 1), seg(n + 1), piece(n + 1);
    std::vector<unsigned long long> raw(n + 1);
    mp.gfx_offsets.assign(n + 1, 0);
    unsigned long long fb = 0, n_chk = 0, n_tile = 0, n_grid = 0, n_seg = 0, n_piece = 0, n_raw = 0, raw_off = 0, png_off = 0;
    for (int f = 0; f < n; ++f) {
        const b200timg_frame &F = b->frames[f];
        MixedGfxFrame &D = desc[f];
        D.g = png_geom(F.out_w, F.out_h, gr.rgb24);
        if (D.g.png_len > 0x7fffffffll)
            return ctx->fail(B200TIMG_EINVAL, "graphics mixed batch: frame %d: the PNG of a %dx%d frame does not fit one IDAT chunk", f,
                             F.out_w, F.out_h);
        b200timg_graphics gf = gr;
        gf.indent_cells = F.x_indent_cells;
        D.s = gfx_spec(gf, D.g);
        D.fb = fb;
        D.raw_off = (long long)raw_off;
        D.png_off = (long long)png_off;
        D.seg0 = (unsigned)n_seg;
        D.ihdr = ihdr_crc(D.g);
        chk[f] = (unsigned)n_chk; tile[f] = (unsigned)n_tile; grid[f] = (unsigned)n_grid; seg[f] = (unsigned)n_seg;
        piece[f] = (unsigned)n_piece; raw[f] = n_raw;
        fb += (unsigned long long)F.out_w * F.out_h * 4;
        n_chk += (unsigned long long)(deflate ? 0 : png_crc_segs(D.g)) + png_raw_segs(D.g);
        n_tile += (unsigned long long)D.s.tiles;
        if (D.s.protocol == B200TIMG_KITTY_TMUX) n_grid += (unsigned long long)D.s.rows * grid_segs(D.s.cols);
        n_seg += (unsigned long long)D.g.nblocks;
        n_piece += (unsigned long long)png_crc_segs(D.g);
        n_raw += (unsigned long long)D.g.raw_len;
        raw_off += (unsigned long long)(D.g.raw_len + 15) / 16 * 16;
        png_off += (unsigned long long)(D.g.png_len + 15) / 16 * 16;
        if (std::max({n_chk, n_tile, n_grid, n_seg, n_piece}) > 0x7fffffffull)
            return ctx->fail(B200TIMG_EINVAL, "graphics mixed batch: more than 2^31 - 1 work items in one call (at frame %d)", f);
        mp.gfx_offsets[f + 1] = mp.gfx_offsets[f] + gfx_frame_size(D.s, kitty ? gr.ids[f] : 0u);
    }
    chk[n] = (unsigned)n_chk; tile[n] = (unsigned)n_tile; grid[n] = (unsigned)n_grid; seg[n] = (unsigned)n_seg;
    piece[n] = (unsigned)n_piece; raw[n] = n_raw;
    mp.o_gfx = mixed_put(mp.arena, desc.data(), sizeof(MixedGfxFrame) * n);
    mp.o_gchk = mixed_put(mp.arena, chk.data(), sizeof(unsigned) * (n + 1));
    mp.o_gtile = mixed_put(mp.arena, tile.data(), sizeof(unsigned) * (n + 1));
    mp.o_ggrid = mixed_put(mp.arena, grid.data(), sizeof(unsigned) * (n + 1));
    mp.o_gseg = mixed_put(mp.arena, seg.data(), sizeof(unsigned) * (n + 1));
    mp.o_gpiece = mixed_put(mp.arena, piece.data(), sizeof(unsigned) * (n + 1));
    mp.o_graw = mixed_put(mp.arena, raw.data(), sizeof(unsigned long long) * (n + 1));
    mp.o_gids = kitty ? mixed_put(mp.arena, gr.ids, sizeof(uint32_t) * n) : 0;
    mp.o_goffs = mixed_put(mp.arena, mp.gfx_offsets.data(), sizeof(uint64_t) * (n + 1));
    mp.gfx_chk = (unsigned)n_chk; mp.gfx_tiles = (unsigned)n_tile; mp.gfx_grid = (unsigned)n_grid;
    mp.gfx_segs = (unsigned)n_seg; mp.gfx_pieces = (unsigned)n_piece;
    mp.gfx_raw = n_raw; mp.gfx_raw_slots = raw_off; mp.gfx_png_slots = png_off;
    return B200TIMG_OK;
}

// The uniform chain over the plan's flat lists: checksums, (deflate: scanlines, segments, layout, pack, wrap, IDAT CRC),
// framing, placeholders -- a fixed number of launches whatever the page's geometries.
int launch_graphics_mixed(b200timg_ctx *ctx, const MixedPlan &mp, const char *d_arena, const uint8_t *d_fb, int n_frames,
                          const b200timg_graphics &gr, uint64_t *d_offsets, char *d_out, size_t out_cap) {
    const int protocol = gr.protocol & ~B200TIMG_DEFLATE;
    const bool deflate = (gr.protocol & B200TIMG_DEFLATE) != 0;
    const MixedGfxFrame *desc = reinterpret_cast<const MixedGfxFrame *>(d_arena + mp.o_gfx);
    auto list = [&](size_t o) { return reinterpret_cast<const unsigned *>(d_arena + o); };
    const uint32_t *ids = protocol == B200TIMG_ITERM2 ? nullptr : reinterpret_cast<const uint32_t *>(d_arena + mp.o_gids);
    B2_CUDA(ctx, ctx->cells.reserve(sizeof(SegSum) * (size_t)mp.gfx_chk));
    B2_CUDA(ctx, ctx->png_sums.reserve(2 * sizeof(uint32_t) * (size_t)n_frames));
    uint32_t *sums = ctx->png_sums.as<uint32_t>();
    uint32_t *png_lens = nullptr;
    uint8_t *png = nullptr;
    if (deflate) {
        const size_t info_b = sizeof(DeflateSeg) * mp.gfx_segs, start_b = sizeof(unsigned long long) * mp.gfx_segs,
                     lens_b = (sizeof(uint32_t) * n_frames + 7) / 8 * 8;
        B2_CUDA(ctx, ctx->dfl_raw.reserve((size_t)mp.gfx_raw_slots));
        B2_CUDA(ctx, ctx->dfl_scratch.reserve((size_t)mp.gfx_segs * DFL_SLOT));
        B2_CUDA(ctx, ctx->dfl_png.reserve((size_t)mp.gfx_png_slots));
        B2_CUDA(ctx, ctx->dfl_meta.reserve(info_b + start_b + lens_b + sizeof(SegSum) * (size_t)mp.gfx_pieces));
        DeflateSeg *info = ctx->dfl_meta.as<DeflateSeg>();
        unsigned long long *start = reinterpret_cast<unsigned long long *>(ctx->dfl_meta.as<uint8_t>() + info_b);
        png_lens = reinterpret_cast<uint32_t *>(ctx->dfl_meta.as<uint8_t>() + info_b + start_b);
        SegSum *pieces = reinterpret_cast<SegSum *>(ctx->dfl_meta.as<uint8_t>() + info_b + start_b + lens_b);
        uint8_t *raw = ctx->dfl_raw.as<uint8_t>();
        png = ctx->dfl_png.as<uint8_t>();
        B2_KERNEL(ctx, "raw_fill_mixed_kernel");
        raw_fill_mixed_kernel<<<png_grid(ctx, (long long)mp.gfx_raw, 256), 256, 0, ctx->stream>>>(
            d_fb, desc, reinterpret_cast<const unsigned long long *>(d_arena + mp.o_graw), n_frames, raw);
        B2_LAUNCH_CHECK(ctx);
        B2_KERNEL(ctx, "png_check_mixed_kernel");
        png_check_mixed_kernel<<<png_grid(ctx, mp.gfx_chk, 128), 128, 0, ctx->stream>>>(d_fb, desc, list(mp.o_gchk), n_frames, 0,
                                                                                        ctx->cells.as<SegSum>());
        B2_LAUNCH_CHECK(ctx);
        B2_KERNEL(ctx, "png_seal_mixed_kernel");
        png_seal_mixed_kernel<<<n_frames, 32, 0, ctx->stream>>>(desc, list(mp.o_gchk), 0, ctx->cells.as<SegSum>(), x8nmodp(PNG_SEG), sums);
        B2_LAUNCH_CHECK(ctx);
        B2_TRY(launch_deflate_mixed(ctx, raw, desc, list(mp.o_gseg), n_frames, mp.gfx_segs, ctx->dfl_scratch.as<uint8_t>(), info));
        B2_KERNEL(ctx, "deflate_layout_mixed_kernel");
        deflate_layout_mixed_kernel<<<1, 1024, 0, ctx->stream>>>(desc, n_frames, info, start, png_lens, ids, d_offsets);
        B2_LAUNCH_CHECK(ctx);
        B2_CUDA(ctx, cudaMemsetAsync(png, 0, (size_t)mp.gfx_png_slots, ctx->stream));
        B2_TRY(launch_deflate_pack_mixed(ctx, raw, desc, list(mp.o_gseg), n_frames, mp.gfx_segs, ctx->dfl_scratch.as<uint8_t>(), info,
                                         start, png, (int)(8 + 25 + 8) + 2));
        B2_KERNEL(ctx, "png_wrap_mixed_kernel");
        png_wrap_mixed_kernel<<<(n_frames + 127) / 128, 128, 0, ctx->stream>>>(desc, n_frames, png_lens, sums, png);
        B2_LAUNCH_CHECK(ctx);
        B2_KERNEL(ctx, "png_crc_mixed_kernel");
        png_crc_mixed_kernel<<<png_grid(ctx, mp.gfx_pieces, 128), 128, 0, ctx->stream>>>(desc, list(mp.o_gpiece), n_frames, png, png_lens,
                                                                                         pieces);
        B2_LAUNCH_CHECK(ctx);
        B2_KERNEL(ctx, "png_crc_seal_mixed_kernel");
        png_crc_seal_mixed_kernel<<<(n_frames + 127) / 128, 128, 0, ctx->stream>>>(desc, list(mp.o_gpiece), n_frames, pieces, png_lens,
                                                                                   x8nmodp(PNG_SEG), png);
        B2_LAUNCH_CHECK(ctx);
    } else {
        B2_CUDA(ctx, cudaMemcpyAsync(d_offsets, d_arena + mp.o_goffs, sizeof(uint64_t) * (n_frames + 1), cudaMemcpyDeviceToDevice,
                                     ctx->stream));
        B2_KERNEL(ctx, "png_check_mixed_kernel");
        png_check_mixed_kernel<<<png_grid(ctx, mp.gfx_chk, 128), 128, 0, ctx->stream>>>(d_fb, desc, list(mp.o_gchk), n_frames, 1,
                                                                                        ctx->cells.as<SegSum>());
        B2_LAUNCH_CHECK(ctx);
        B2_KERNEL(ctx, "png_seal_mixed_kernel");
        png_seal_mixed_kernel<<<n_frames, 32, 0, ctx->stream>>>(desc, list(mp.o_gchk), 1, ctx->cells.as<SegSum>(), x8nmodp(PNG_SEG), sums);
        B2_LAUNCH_CHECK(ctx);
    }
    const long long cap = (long long)ctx->sm_count * 16;
    B2_KERNEL(ctx, "graphics_emit_mixed_kernel");
    graphics_emit_mixed_kernel<<<(unsigned)std::min<long long>(mp.gfx_tiles, cap), GFX_THREADS, 0, ctx->stream>>>(
        d_fb, desc, list(mp.o_gtile), n_frames, ids, sums, d_offsets, d_out, (unsigned long long)out_cap, png, png_lens);
    B2_LAUNCH_CHECK(ctx);
    if (protocol == B200TIMG_KITTY_TMUX) {
        B2_KERNEL(ctx, "graphics_grid_mixed_kernel");
        graphics_grid_mixed_kernel<<<(unsigned)std::min<long long>(mp.gfx_grid, cap), GFX_THREADS, 0, ctx->stream>>>(
            desc, list(mp.o_ggrid), n_frames, ids, d_offsets, d_out, (unsigned long long)out_cap, png_lens);
        B2_LAUNCH_CHECK(ctx);
    }
    return B200TIMG_OK;
}

}  // namespace b200timg

using namespace b200timg;

extern "C" {

size_t b200timg_png_size(int w, int h, int rgb24) { return (size_t)png_geom(w, h, rgb24).png_len; }
size_t b200timg_base64_size(size_t n) { return (n + 2) / 3 * 4; }

size_t b200timg_graphics_size(const b200timg_graphics *g, int w, int h, uint32_t id) {
    if (!g || w <= 0 || h <= 0) return 0;
    const int protocol = g->protocol & ~B200TIMG_DEFLATE;
    if (protocol == B200TIMG_KITTY_TMUX) {
        if (g->cell_x_px <= 0 || g->cell_y_px <= 0 || g->indent_cells < 0) return 0;
    } else if (protocol != B200TIMG_KITTY && protocol != B200TIMG_ITERM2) {
        return 0;
    }
    return gfx_frame_size(gfx_spec(*g, png_geom(w, h, g->rgb24)), id);
}

int b200timg_png_batch_dev(b200timg_ctx *ctx, const uint8_t *d_frames, int w, int h, int n_frames, int rgb24, uint8_t *d_png, char *d_b64) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!d_frames || !d_png || w <= 0 || h <= 0 || n_frames <= 0) return ctx->fail(B200TIMG_EINVAL, "png: bad args");
    return launch_png(ctx, d_frames, w, h, n_frames, rgb24, d_png, d_b64);
}

// one frame, host buffers: out gets the PNG (b200timg_png_size bytes), b64 (optional) its base64 text
int b200timg_png_encode(b200timg_ctx *ctx, const uint8_t *fb, int w, int h, int rgb24, uint8_t *out, size_t cap, char *b64, size_t b64_cap) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!fb || !out || w <= 0 || h <= 0) return ctx->fail(B200TIMG_EINVAL, "png: bad args");
    const size_t n = b200timg_png_size(w, h, rgb24), nb = b200timg_base64_size(n);
    if (cap < n || (b64 && b64_cap < nb)) return ctx->fail(B200TIMG_ENOSPC, "png: need %zu (+%zu base64) bytes", n, nb);
    const size_t bytes = (size_t)w * h * 4;
    ctx->resident_fb = nullptr;
    B2_CUDA(ctx, ctx->in_stage.reserve(bytes));
    B2_CUDA(ctx, ctx->out_stage.reserve((n + 15) / 16 * 16 + nb + 16));
    B2_CUDA(ctx, cudaMemcpyAsync(ctx->in_stage.p, fb, bytes, cudaMemcpyHostToDevice, ctx->stream));
    uint8_t *d_png = ctx->out_stage.as<uint8_t>();
    char *d_b64 = b64 ? ctx->out_stage.as<char>() + (n + 15) / 16 * 16 : nullptr;
    B2_TRY(launch_png(ctx, ctx->in_stage.as<uint8_t>(), w, h, 1, rgb24, d_png, d_b64));
    B2_CUDA(ctx, cudaMemcpyAsync(out, d_png, n, cudaMemcpyDeviceToHost, ctx->stream));
    if (b64) B2_CUDA(ctx, cudaMemcpyAsync(b64, d_b64, nb, cudaMemcpyDeviceToHost, ctx->stream));
    B2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return B200TIMG_OK;
}

}  // extern "C"
