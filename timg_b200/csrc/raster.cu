// BMP, TGA and binary PNM (P5 / P6) files on the device: the RGBA buffer stbi__load_and_postprocess_8bit(.., 4) gives
// timg's STB source for them (src/stb-image-source.cc:140-157; third_party/stb/stb_image.h stbi__bmp_load,
// stbi__tga_load and stbi__pnm_load of stb v2.30), read from a file as the source reads it: bytes past the end read as
// 0 and every quirk of the three loaders is kept (see include/b200timg.h).
//   host walk            stb's tests and header walks: the data start, row stride, palette and pixel layout of a file
//   tga_tile_kernel      one thread per TILE bytes of an RLE TGA's packet stream: for each of the P bytes a tile can be
//                        entered at (bytes of a packet begun before it), the exit byte in the next tile and the pixels
//                        of the packets begun in the tile, from one backward pass over the tile
//   tga_chunk_kernel     one thread per (chunk of CHUNK tiles, entry byte): the composition of the chunk's tile maps
//   tga_super_kernel     one thread per (super-chunk of CHUNK chunks, entry byte): the composition of its chunk maps
//   tga_top_kernel       one thread: the entry of every super-chunk, in order (a map that starts a file resets)
//   tga_packet_kernel    one thread per tile: its true entry (super-chunk entry, then the chunk and tile maps before
//                        it) and the byte offset and first pixel of every packet begun in it
//   raster_canvas_kernel one thread per canvas pixel of every file: its bytes read in place from the upload (an RLE
//                        pixel finds its packet by two binary searches: tile, then packet)
//   raster_alpha_kernel  one thread per canvas pixel: BMP's all-zero-alpha rule, once every alpha of the file is known
// A call launches 7 kernels whatever its files hold.
#include <climits>
#include <cstdlib>

#include "decode.cuh"

namespace b200timg {

namespace {

constexpr int TILE = 1024;           // RLE stream bytes per tile
constexpr int P = 513;               // entry bytes of a tile: a packet is at most 1 + 128 * 4 bytes
constexpr int CHUNK = 32;            // tiles per chunk, and chunks per super-chunk
constexpr int RCAP = TILE / 2;       // packets begun in a tile: each takes at least 2 bytes
constexpr int TILE_T = 8;            // threads of tga_tile_kernel (each has a TILE-word column of shared memory)
constexpr unsigned MAX_DIM = 1u << 24;   // STBI_MAX_DIMENSIONS

enum { F_BMP = 0, F_TGA = 1, F_PNM = 2 };
// pixel layouts
enum { L_PAL1, L_PAL4, L_PAL8, L_BGR24, L_BGRA32, L_MASK16, L_MASK32, L_TGA_RAW, L_TGA_RLE, L_PNM8, L_PNM16 };

struct __align__(16) RasterFile {
    unsigned long long off;          // the file's first byte in the uploaded files
    unsigned long long size;         // its bytes: reads at or past size give 0
    unsigned long long px0;          // its first canvas pixel
    unsigned long long data;         // where stb's reader starts the pixels (may be at or past size)
    unsigned long long stride;       // BMP: bytes from one file row to the next
    unsigned long long pal;          // the palette's first byte
    unsigned w, h;
    int layout, flip;                // flip: canvas row y is file row h - 1 - y
    int B;                           // TGA / PNM: bytes of one pixel value (TGA: index bytes when indexed)
    int comp;                        // TGA: stb's channels of a value; PNM: 1 or 3
    int indexed, rgb16;              // TGA
    int npal;                        // BMP: psize (may be <= 0: every index reads stb's uninitialised pal[]);
                                     // TGA: palette entries
    int pal_bytes;                   // BMP: 3 or 4 bytes per entry
    int alpha_rule;                  // BMP: all alpha 0 becomes 255
    unsigned mask[4];                // BMP: r, g, b, a
    int shift[4], count[4];
    unsigned tile0;                  // RLE TGA: its first tile
    unsigned pad_;
};

__device__ __forceinline__ unsigned rd(const uint8_t *b, unsigned long long size, unsigned long long pos) {
    return pos < size ? b[pos] : 0u;
}

// ---- RLE TGA packet boundaries -------------------------------------------------------------------------------------
// A map entry: pixels (bits 0-47), exit byte (48-57); bit 63 of entry 0: the map starts a file.
constexpr unsigned long long HEAD = 1ull << 63;
constexpr unsigned long long PX_MASK = (1ull << 48) - 1;
__device__ __forceinline__ unsigned long long ment(unsigned x, unsigned long long p) { return p | (unsigned long long)x << 48; }
struct Cur { unsigned x; unsigned long long p; };  // entry byte and first pixel inside the file

__device__ __forceinline__ Cur apply(const unsigned long long *m, Cur c) {
    const unsigned long long e0 = m[0];
    const unsigned long long e = (e0 & HEAD) ? e0 : m[c.x];
    Cur r;
    r.x = (unsigned)(e >> 48) & 1023;
    r.p = (e & PX_MASK) + ((e0 & HEAD) ? 0ull : c.p);
    return r;
}

__device__ __forceinline__ unsigned pkt_len(unsigned cmd, int B) { return cmd & 128 ? 1 + B : 1 + ((cmd & 127) + 1) * B; }

__global__ void __launch_bounds__(TILE_T)
tga_tile_kernel(const uint8_t *__restrict__ files, const RasterFile *__restrict__ fd, const unsigned *__restrict__ tile0,
                int n, unsigned n_tiles, unsigned long long *__restrict__ maps, int32_t *__restrict__ status,
                unsigned *__restrict__ aor, unsigned long long *__restrict__ pend) {
    __shared__ uint32_t dp[TILE * TILE_T];          // (pixels | exit << 18) of a packet chain begun at byte p
    uint32_t *D = dp + threadIdx.x;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    const unsigned long long g0 = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (unsigned long long i = g0; i < (unsigned long long)n; i += stride) { status[i] = 1; aor[i] = 0; pend[i] = 0; }
    for (unsigned long long t = g0; t < n_tiles; t += stride) {
        const int f = mixed_owner(tile0, n, (unsigned)t);
        const RasterFile &F = fd[f];
        const uint8_t *b = files + F.off;
        const unsigned k = (unsigned)t - F.tile0;
        const unsigned long long a = F.data + (unsigned long long)k * TILE;
        for (int p = TILE - 1; p >= 0; --p) {
            uint32_t v = 0;
            if (a + p < F.size) {
                const unsigned cmd = b[a + p], nx = p + pkt_len(cmd, F.B), np = (cmd & 127) + 1;
                v = nx >= (unsigned)TILE ? (np | (nx - TILE) << 18) : D[nx * TILE_T] + np;
            }
            D[p * TILE_T] = v;
        }
        for (int e = 0; e < P; ++e) {
            const uint32_t v = D[(k == 0 ? 0 : e) * TILE_T];
            maps[t * P + e] = ment(v >> 18, v & 0x3ffff) | (k == 0 ? HEAD : 0);
        }
    }
}

// one thread per (span, entry byte): the composition of `per` consecutive maps of `src` (n_src maps)
__device__ __forceinline__ void compose(const unsigned long long *__restrict__ src, unsigned n_src, unsigned n_dst,
                                        unsigned long long *__restrict__ dst) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < (unsigned long long)n_dst * P;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned c = (unsigned)(i / P), e = (unsigned)(i % P);
        const unsigned t0 = c * CHUNK, t1 = min(t0 + CHUNK, n_src);
        unsigned long long head = 0;
        Cur s{e, 0};
        for (unsigned t = t0; t < t1; ++t) {
            head |= src[t * (unsigned long long)P] & HEAD;
            s = apply(src + t * (unsigned long long)P, s);
        }
        dst[i] = ment(s.x, s.p) | (e == 0 ? head : 0);
    }
}

__global__ void __launch_bounds__(256)
tga_chunk_kernel(const unsigned long long *__restrict__ maps, unsigned n_tiles, unsigned n_chunks,
                 unsigned long long *__restrict__ cmaps) {
    compose(maps, n_tiles, n_chunks, cmaps);
}

__global__ void __launch_bounds__(256)
tga_super_kernel(const unsigned long long *__restrict__ cmaps, unsigned n_chunks, unsigned n_supers,
                 unsigned long long *__restrict__ smaps) {
    compose(cmaps, n_chunks, n_supers, smaps);
}

__global__ void __launch_bounds__(32)
tga_top_kernel(const unsigned long long *__restrict__ smaps, unsigned n_supers, Cur *__restrict__ sentry) {
    if (threadIdx.x != 0) return;
    Cur s{0, 0};
    for (unsigned u = 0; u < n_supers; ++u) { sentry[u] = s; s = apply(smaps + u * (unsigned long long)P, s); }
}

__global__ void __launch_bounds__(256)
tga_packet_kernel(const uint8_t *__restrict__ files, const RasterFile *__restrict__ fd, const unsigned *__restrict__ tile0,
                  int n, unsigned n_tiles, const unsigned long long *__restrict__ maps,
                  const unsigned long long *__restrict__ cmaps, const Cur *__restrict__ sentry,
                  uint32_t *__restrict__ tpx, uint32_t *__restrict__ nrec, uint32_t *__restrict__ rpx,
                  uint16_t *__restrict__ rpos, unsigned long long *__restrict__ pend) {
    for (unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; t < n_tiles;
         t += (unsigned long long)gridDim.x * blockDim.x) {
        const int f = mixed_owner(tile0, n, (unsigned)t);
        const RasterFile &F = fd[f];
        const unsigned k = (unsigned)t - F.tile0;
        Cur s{0, 0};
        if (k != 0) {
            const unsigned c = (unsigned)t / CHUNK;
            s = sentry[c / CHUNK];
            for (unsigned u = c / CHUNK * CHUNK; u < c; ++u) s = apply(cmaps + u * (unsigned long long)P, s);
            for (unsigned u = c * CHUNK; u < t; ++u) s = apply(maps + u * (unsigned long long)P, s);
        }
        const uint8_t *b = files + F.off;
        const unsigned long long a = F.data + (unsigned long long)k * TILE, e = min(a + TILE, F.size);
        unsigned long long pos = a + s.x, p = s.p;
        tpx[t] = (uint32_t)min(p, 0xffffffffull);
        unsigned j = 0;
        for (; pos < e; ++j) {
            const unsigned cmd = b[pos];
            rpx[t * RCAP + j] = (uint32_t)min(p, 0xffffffffull);
            rpos[t * RCAP + j] = (uint16_t)(pos - a);
            p += (cmd & 127) + 1;
            pos += pkt_len(cmd, F.B);
        }
        nrec[t] = j;
        if (e == F.size) pend[f] = p;               // the file's last tile: pixels before the first packet past the end
    }
}

// ---- canvases ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t rgba(unsigned r, unsigned g, unsigned b, unsigned a) {
    return r | g << 8 | b << 16 | a << 24;
}

__device__ __forceinline__ unsigned rgb16_chan(unsigned v) { return v * 255 / 31; }

// stbi__shiftsigned of v & mask
__device__ __forceinline__ unsigned shiftsigned(unsigned v, int shift, int bits) {
    const unsigned mul[9] = {0, 0xff, 0x55, 0x49, 0x11, 0x21, 0x41, 0x81, 0x01};
    const unsigned sh[9] = {0, 0, 0, 1, 0, 2, 4, 6, 0};
    v = shift < 0 ? v << -shift : v >> shift;
    v >>= (8 - bits);
    return (v * mul[bits]) >> sh[bits];
}

// A TGA value of B bytes at pos: the palette lookup, RGB16 expansion or raw channels, stb's BGR swap and the
// conversion to 4 channels
__device__ __forceinline__ uint32_t tga_value(const RasterFile &F, const uint8_t *b, unsigned long long pos) {
    unsigned c[4] = {0, 0, 0, 0};
    if (F.indexed) {
        unsigned idx = rd(b, F.size, pos) | (F.B == 2 ? rd(b, F.size, pos + 1) << 8 : 0u);
        if (idx >= (unsigned)F.npal) idx = 0;
        if (F.rgb16) {
            pos = F.pal + 2ull * idx;
        } else {
            for (int j = 0; j < F.comp; ++j) c[j] = rd(b, F.size, F.pal + (unsigned long long)idx * F.comp + j);
        }
    } else if (!F.rgb16) {
        for (int j = 0; j < F.comp; ++j) c[j] = rd(b, F.size, pos + j);
    }
    if (F.rgb16) {
        const unsigned v = rd(b, F.size, pos) | rd(b, F.size, pos + 1) << 8;
        return rgba(rgb16_chan((v >> 10) & 31), rgb16_chan((v >> 5) & 31), rgb16_chan(v & 31), 255);
    }
    switch (F.comp) {
        case 1: return rgba(c[0], c[0], c[0], 255);
        case 2: return rgba(c[0], c[0], c[0], c[1]);
        case 3: return rgba(c[2], c[1], c[0], 255);
        default: return rgba(c[2], c[1], c[0], c[3]);
    }
}

__global__ void __launch_bounds__(256)
raster_canvas_kernel(const uint8_t *__restrict__ files, const RasterFile *__restrict__ fd,
                     const unsigned long long *__restrict__ px0, int n, unsigned long long total,
                     const uint32_t *__restrict__ tpx, const uint32_t *__restrict__ nrec,
                     const uint32_t *__restrict__ rpx, const uint16_t *__restrict__ rpos,
                     const unsigned long long *__restrict__ pend, const unsigned *__restrict__ tile0,
                     uint32_t *__restrict__ out, int32_t *__restrict__ status, unsigned *__restrict__ aor) {
    for (unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; k < total;
         k += (unsigned long long)gridDim.x * blockDim.x) {
        const int f = mixed_owner(px0, n, k);
        const RasterFile &F = fd[f];
        const uint8_t *b = files + F.off;
        const unsigned q = (unsigned)(k - F.px0), x = q % F.w, y = q / F.w;
        const unsigned long long row = F.flip ? F.h - 1 - y : y;
        uint32_t v = 0;
        if (F.layout <= L_MASK32) {                  // BMP
            const unsigned long long r0 = F.data + row * F.stride;
            int idx = -1;
            if (F.layout == L_PAL1) idx = (rd(b, F.size, r0 + (x >> 3)) >> (7 - (x & 7))) & 1;
            else if (F.layout == L_PAL4) idx = (rd(b, F.size, r0 + (x >> 1)) >> (x & 1 ? 0 : 4)) & 15;
            else if (F.layout == L_PAL8) idx = rd(b, F.size, r0 + x);
            if (idx >= 0) {
                if (idx >= F.npal) {
                    status[f] = -1;                  // stb reads its uninitialised pal[idx]
                } else {
                    const unsigned long long e = F.pal + (unsigned long long)idx * F.pal_bytes;
                    v = rgba(rd(b, F.size, e + 2), rd(b, F.size, e + 1), rd(b, F.size, e), 255);
                }
            } else if (F.layout == L_BGR24) {
                const unsigned long long e = r0 + 3ull * x;
                v = rgba(rd(b, F.size, e + 2), rd(b, F.size, e + 1), rd(b, F.size, e), 255);
            } else if (F.layout == L_BGRA32) {
                const unsigned long long e = r0 + 4ull * x;
                v = rgba(rd(b, F.size, e + 2), rd(b, F.size, e + 1), rd(b, F.size, e), rd(b, F.size, e + 3));
            } else {
                const unsigned long long e = r0 + (F.layout == L_MASK16 ? 2ull : 4ull) * x;
                unsigned w = rd(b, F.size, e) | rd(b, F.size, e + 1) << 8;
                if (F.layout == L_MASK32) w |= rd(b, F.size, e + 2) << 16 | rd(b, F.size, e + 3) << 24;
                unsigned ch[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) ch[i] = shiftsigned(w & F.mask[i], F.shift[i], F.count[i]) & 255;
                if (!F.mask[3]) ch[3] = 255;
                v = rgba(ch[0], ch[1], ch[2], ch[3]);
            }
            if (F.alpha_rule && (v >> 24) && !aor[f]) atomicOr(aor + f, 1u);
        } else if (F.layout == L_TGA_RAW) {
            v = tga_value(F, b, F.data + (row * F.w + x) * (unsigned long long)F.B);
        } else if (F.layout == L_TGA_RLE) {
            const unsigned qf = (unsigned)(row * F.w + x);
            unsigned long long pos = F.size;         // past the stream's last packet: a value of zero bytes
            if (qf < pend[f]) {
                unsigned lo = F.tile0, hi = tile0[f + 1] - 1;
                while (lo < hi) {
                    const unsigned mid = (lo + hi + 1) >> 1;
                    if (tpx[mid] <= qf) lo = mid; else hi = mid - 1;
                }
                const unsigned long long r0 = (unsigned long long)lo * RCAP;
                unsigned a = 0, z = nrec[lo] - 1;
                while (a < z) {
                    const unsigned mid = (a + z + 1) >> 1;
                    if (rpx[r0 + mid] <= qf) a = mid; else z = mid - 1;
                }
                const unsigned long long h = F.data + (unsigned long long)(lo - F.tile0) * TILE + rpos[r0 + a];
                pos = h + 1 + (b[h] & 128 ? 0ull : (unsigned long long)(qf - rpx[r0 + a]) * F.B);
            }
            v = tga_value(F, b, pos);
        } else {                                     // PNM: the raster lies inside the file
            const unsigned long long e = F.data + (row * F.w + x) * (unsigned long long)F.B;
            const int s = F.layout == L_PNM16 ? 2 : 1;   // 16 bits: the second byte of each big-endian sample
            if (F.comp == 1) { const unsigned g = b[e + s - 1]; v = rgba(g, g, g, 255); }
            else v = rgba(b[e + s - 1], b[e + 2 * s - 1], b[e + 3 * s - 1], 255);
        }
        out[k] = v;
    }
}

__global__ void __launch_bounds__(256)
raster_alpha_kernel(const RasterFile *__restrict__ fd, const unsigned long long *__restrict__ px0, int n,
                    unsigned long long total, const unsigned *__restrict__ aor, uint32_t *__restrict__ out) {
    for (unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; k < total;
         k += (unsigned long long)gridDim.x * blockDim.x) {
        const int f = mixed_owner(px0, n, k);
        if (fd[f].alpha_rule && !aor[f]) out[k] |= 0xff000000u;
    }
}

// ---- host walk -----------------------------------------------------------------------------------------------------
struct Parse {
    int format = 0;
    unsigned w = 0, h = 0;
    int channels = 0, bpp = 0, palette = 0, top_down = 0, rle = 0;
    bool supported = false;
    char why[96] = {0};
    RasterFile F;                    // the descriptor, but for off, px0 and tile0
};

// stb's reader over a file: bytes at or past the end read as 0.  A negative stbi__skip before the end moves stb to
// the end of its 128-byte buffer, which is not a function of the file: neg records it.  At or past the end it
// changes nothing.
struct Rd {
    const uint8_t *d;
    unsigned long long S, pos = 0;
    bool neg = false;
    unsigned get8() { const unsigned v = pos < S ? d[pos] : 0u; ++pos; return v; }
    unsigned le16() { const unsigned a = get8(); return a | get8() << 8; }
    unsigned le32() { const unsigned a = le16(); return a | le16() << 16; }
    void skip(long long k) {
        if (k < 0) { if (pos < S) neg = true; return; }
        pos += (unsigned long long)k;
    }
    unsigned long long bytes_read() const { return pos > S ? S + 1 : pos; }   // stb's count, frozen one past the end
};

bool unsupported(Parse &P, const char *why) {
    P.supported = false;
    snprintf(P.why, sizeof P.why, "%s", why);
    return true;
}

bool mad3_ok(long long a, long long b, long long c) {   // stbi__mad3sizes_valid(a, b, c, 0)
    if (a < 0 || b < 0 || c < 0) return false;
    if (b && a > INT_MAX / b) return false;
    if (c && a * b > INT_MAX / c) return false;
    return true;
}

int high_bit(unsigned z) { return z ? 31 - __builtin_clz(z) : -1; }

int bmp_walk(Rd &r, Parse &P) {
    RasterFile &F = P.F;
    if (r.S < 18) return -1;         // stb's test reads 18 bytes; past the end it zeroes its first byte
    if (r.get8() != 'B' || r.get8() != 'M') return -1;
    r.le32(); r.le16(); r.le16();
    const int offset = (int)r.le32();
    const unsigned hsz = r.le32();
    if (hsz != 12 && hsz != 40 && hsz != 56 && hsz != 108 && hsz != 124) return -1;
    int extra_read = 14;
    if (offset < 0) return -1;
    unsigned x, y;
    if (hsz == 12) { x = r.le16(); y = r.le16(); } else { x = r.le32(); y = r.le32(); }
    if (r.le16() != 1) return -1;
    const int bpp = (int)r.le16();
    unsigned mr = 0, mg = 0, mb = 0, ma = 0, all_a = 255;
    auto defaults = [&](int compress) {   // stbi__bmp_set_mask_defaults
        if (compress != 0) return;
        if (bpp == 16) { mr = 31u << 10; mg = 31u << 5; mb = 31u; }
        else if (bpp == 32) { mr = 0xffu << 16; mg = 0xffu << 8; mb = 0xffu; ma = 0xffu << 24; all_a = 0; }
        else mr = mg = mb = ma = 0;
    };
    if (hsz != 12) {
        const int compress = (int)r.le32();
        if (compress == 1 || compress == 2 || compress >= 4) return -1;
        if (compress == 3 && bpp != 16 && bpp != 32) return -1;
        for (int i = 0; i < 5; ++i) r.le32();
        if (hsz == 40 || hsz == 56) {
            if (hsz == 56) for (int i = 0; i < 4; ++i) r.le32();
            if (bpp == 16 || bpp == 32) {
                if (compress == 0) defaults(0);
                else if (compress == 3) {
                    mr = r.le32(); mg = r.le32(); mb = r.le32();
                    extra_read += 12;
                    if (mr == mg && mg == mb) return -1;
                } else return -1;
            }
        } else {
            mr = r.le32(); mg = r.le32(); mb = r.le32(); ma = r.le32();
            if (compress != 3) defaults(compress);
            for (int i = 0; i < 13; ++i) r.le32();
            if (hsz == 124) for (int i = 0; i < 4; ++i) r.le32();
        }
    }
    const int yi = (int)y;
    F.flip = yi > 0;
    const unsigned long long ya = yi < 0 ? (unsigned long long)(-(long long)yi) : (unsigned long long)yi;
    if (ya > MAX_DIM || x > MAX_DIM) return -1;
    y = (unsigned)ya;
    int psize = 0;
    if (hsz == 12) { if (bpp < 24) psize = (offset - extra_read - 24) / 3; }
    else if (bpp < 16) psize = (offset - extra_read - (int)hsz) >> 2;
    if (psize == 0) {
        const unsigned long long done = r.bytes_read();
        if (done == 0 || done > 1024) return -1;
        if ((unsigned long long)offset < done || (unsigned long long)offset - done > 1024) return -1;
        r.skip((long long)offset - (long long)done);
    }
    P.channels = (bpp == 24 && ma == 0xff000000u) ? 3 : ma ? 4 : 3;
    if (!mad3_ok(4, x, y)) return -1;
    P.format = F_BMP; P.w = x; P.h = y; P.bpp = bpp; P.top_down = !F.flip;
    if (bpp < 16) {
        if (psize == 0 || psize > 256) return -1;
        F.pal = r.pos; F.pal_bytes = hsz == 12 ? 3 : 4;
        if (psize > 0) r.pos += (unsigned long long)psize * F.pal_bytes;
        r.skip((long long)offset - extra_read - (long long)hsz - (long long)psize * F.pal_bytes);
        unsigned long long width;
        if (bpp == 1) { width = (x + 7ull) >> 3; F.layout = L_PAL1; }
        else if (bpp == 4) { width = (x + 1ull) >> 1; F.layout = L_PAL4; }
        else if (bpp == 8) { width = x; F.layout = L_PAL8; }
        else return -1;
        F.stride = width + ((0 - width) & 3);
        F.npal = psize;
        P.palette = psize;
    } else {
        r.skip((long long)offset - extra_read - (long long)hsz);
        const int easy = bpp == 24 ? 1 : (bpp == 32 && mb == 0xff && mg == 0xff00 && mr == 0xff0000 && ma == 0xff000000u) ? 2 : 0;
        if (!easy) {
            if (!mr || !mg || !mb) return -1;
            const unsigned m[4] = {mr, mg, mb, ma};
            for (int i = 0; i < 4; ++i) {
                F.mask[i] = m[i];
                F.shift[i] = high_bit(m[i]) - 7;
                F.count[i] = __builtin_popcount(m[i]);
                if (F.count[i] > 8) return -1;
            }
            F.layout = bpp == 16 ? L_MASK16 : L_MASK32;
        } else {
            F.layout = easy == 1 ? L_BGR24 : L_BGRA32;
        }
        const unsigned long long width = bpp == 24 ? 3ull * x : bpp == 16 ? 2ull * x : 0;
        F.stride = (bpp == 24 || bpp == 16 ? width : 4ull * x) + ((0 - width) & 3);
        F.alpha_rule = all_a == 0 && ma != 0;
    }
    F.data = r.pos;
    if (r.neg) return unsupported(P, "a negative stbi__skip: stb's position depends on its read buffer"), 0;
    if (x == 0 || y == 0) return unsupported(P, "zero-area BMP"), 0;
    P.supported = true;
    return 0;
}

int tga_comp(int bits, bool grey, int *rgb16) {   // stbi__tga_get_comp
    *rgb16 = 0;
    switch (bits) {
        case 8: return 1;
        case 16: if (grey) return 2; *rgb16 = 1; return 3;
        case 15: *rgb16 = 1; return 3;
        case 24: case 32: return bits / 8;
        default: return 0;
    }
}

int tga_walk(Rd &r, Parse &P) {
    RasterFile &F = P.F;
    {   // stbi__tga_test
        r.get8();
        const unsigned ct = r.get8();
        if (ct > 1) return -1;
        const unsigned ty = r.get8();
        if (ct == 1) {
            if (ty != 1 && ty != 9) return -1;
            r.skip(4);
            const unsigned sz = r.get8();
            if (sz != 8 && sz != 15 && sz != 16 && sz != 24 && sz != 32) return -1;
            r.skip(4);
        } else {
            if (ty != 2 && ty != 3 && ty != 10 && ty != 11) return -1;
            r.skip(9);
        }
        if (r.le16() < 1 || r.le16() < 1) return -1;
        const unsigned sz = r.get8();
        if (ct == 1 && sz != 8 && sz != 16) return -1;
        if (sz != 8 && sz != 15 && sz != 16 && sz != 24 && sz != 32) return -1;
    }
    r.pos = 0;
    const unsigned id_len = r.get8(), indexed = r.get8();
    int type = (int)r.get8();
    const unsigned pal_start = r.le16(), pal_len = r.le16(), pal_bits = r.get8();
    r.le16(); r.le16();
    const unsigned w = r.le16(), h = r.le16(), bpp = r.get8(), desc = r.get8();
    int rle = 0;
    if (type >= 8) { type -= 8; rle = 1; }
    int rgb16 = 0;
    const int comp = indexed ? tga_comp((int)pal_bits, false, &rgb16) : tga_comp((int)bpp, type == 3, &rgb16);
    if (!comp) return -1;
    if (!mad3_ok(w, h, comp) || !mad3_ok(4, w, h)) return -1;   // the load, then stbi__convert_format to 4 channels
    P.format = F_TGA; P.w = w; P.h = h; P.channels = comp; P.bpp = (int)bpp; P.rle = rle;
    F.flip = 1 - ((desc >> 5) & 1);
    P.top_down = !F.flip;
    F.comp = comp; F.rgb16 = rgb16; F.indexed = indexed != 0;
    F.B = indexed ? (int)bpp / 8 : rgb16 ? 2 : comp;
    r.skip(id_len);
    if (!indexed && !rle && !rgb16) {
        F.layout = L_TGA_RAW; F.data = r.pos;
        if (r.pos + (unsigned long long)w * h * comp > r.S)
            return unsupported(P, "a raw TGA cut short: stbi__getn leaves the rest uninitialised"), 0;
        P.supported = true;
        return 0;
    }
    if (indexed) {
        if (pal_len == 0) return -1;
        r.skip(pal_start);
        F.pal = r.pos; F.npal = (int)pal_len; P.palette = (int)pal_len;
        const unsigned long long bytes = (unsigned long long)pal_len * (rgb16 ? 2 : comp);
        if (!rgb16 && r.pos + bytes > r.S) return -1;           // stbi__getn of the palette fails
        r.pos += bytes;
    }
    F.layout = rle ? L_TGA_RLE : L_TGA_RAW;
    F.data = r.pos;
    P.supported = true;
    return 0;
}

bool pnm_space(unsigned c) { return c == ' ' || c == '\t' || c == '\n' || c == '\v' || c == '\f' || c == '\r'; }

int pnm_walk(Rd &r, Parse &P) {
    RasterFile &F = P.F;
    if (r.get8() != 'P') return -1;
    const unsigned t = r.get8();
    if (t != '5' && t != '6') return -1;
    const int n = t == '6' ? 3 : 1;
    // Any read at the end stops the header with the raster (at least one byte) cut short: stbi__getn fails.
    auto eof = [&] { return r.pos >= r.S; };
    int c = (signed char)r.get8();
    auto skip_ws = [&] {
        for (;;) {
            while (!eof() && pnm_space((unsigned)c)) c = (signed char)r.get8();
            if (eof() || c != '#') break;
            while (!eof() && c != '\n' && c != '\r') c = (signed char)r.get8();
        }
    };
    auto integer = [&] {
        int v = 0;
        while (!eof() && c >= '0' && c <= '9') {
            v = v * 10 + (c - '0');
            c = (signed char)r.get8();
            if (v > 214748364 || (v == 214748364 && c > '7')) return 0;   // overflow: stb's error value
        }
        return v;
    };
    skip_ws();
    const int x = integer();
    if (x == 0) return -1;
    skip_ws();
    const int y = integer();
    if (y == 0) return -1;
    skip_ws();
    const int maxv = integer();
    if (maxv > 65535) return -1;
    const int bpc = maxv > 255 ? 16 : 8;
    if ((unsigned)x > MAX_DIM || (unsigned)y > MAX_DIM) return -1;
    const long long bytes = (long long)n * x * y * (bpc / 8);
    if (bytes > INT_MAX) return -1;                                  // stbi__mad4sizes_valid
    if (r.pos > r.S || r.pos + (unsigned long long)bytes > r.S) return -1;   // "PNM file truncated"
    P.format = F_PNM; P.w = (unsigned)x; P.h = (unsigned)y; P.channels = n; P.bpp = n * bpc; P.top_down = 1;
    F.layout = bpc == 16 ? L_PNM16 : L_PNM8; F.comp = n; F.B = n * bpc / 8; F.data = r.pos;
    if (bpc == 8 && !mad3_ok(4, x, y)) return -1;                    // stbi__convert_format to 4 channels
    if (bpc == 16 && 8ll * x * y >= (1ll << 31))
        return unsupported(P, "16-bit PNM of 2^28 pixels or more: stbi__convert_format16's size overflows"), 0;
    P.supported = true;
    return 0;
}

// stb's order: BMP, then PNM, then TGA (the three magics exclude each other)
int raster_walk(const uint8_t *d, size_t size, Parse &P) {
    P = Parse();
    memset(&P.F, 0, sizeof P.F);
    Rd r{d, size};
    if (size >= 2 && d[0] == 'B' && d[1] == 'M') return bmp_walk(r, P);
    if (size >= 2 && d[0] == 'P' && (d[1] == '5' || d[1] == '6')) return pnm_walk(r, P);
    return tga_walk(r, P);
}

void fill_info(const Parse &P, b200timg_raster_info *info) {
    memset(info, 0, sizeof *info);
    info->format = P.format; info->w = (int)P.w; info->h = (int)P.h; info->channels = P.channels;
    info->bpp = P.bpp; info->palette = P.palette; info->top_down = P.top_down; info->rle = P.rle;
    info->supported = P.supported ? 1 : 0;
    snprintf(info->reason, sizeof info->reason, "%s", P.supported ? "" : P.why);
}

// Device scratch of one call (ctx->raster_up.arena + ctx->raster_scratch): the files + 184 bytes per file; per RLE
// stream byte about 4 bytes of tile maps (P * 8 / TILE), 3 bytes of packet records (RCAP * 6 / TILE) and 1/8 byte of
// chunk maps.
int launch_raster(b200timg_ctx *ctx, int n, const uint8_t *const *files, const size_t *sizes,
                  const std::vector<Parse> &ps, uint8_t *d_frames, int32_t *d_status) {
    std::vector<RasterFile> fdesc((size_t)n);
    std::vector<unsigned> tile0(1, 0);
    std::vector<unsigned long long> px0(1, 0);
    unsigned long long off = 0, tiles = 0;
    for (int f = 0; f < n; ++f) {
        RasterFile &F = fdesc[(size_t)f];
        F = ps[(size_t)f].F;
        F.off = off; F.size = sizes[f]; F.px0 = px0.back();
        F.w = ps[(size_t)f].w; F.h = ps[(size_t)f].h;
        F.tile0 = (unsigned)tiles;
        if (F.layout == L_TGA_RLE && F.data < F.size) tiles += (F.size - F.data + TILE - 1) / TILE;
        if (tiles >= (1ull << 31) / RCAP) return ctx->fail(B200TIMG_EINVAL, "raster: 2^31 RLE packet slots or more in one call");
        off += sizes[f];
        tile0.push_back((unsigned)tiles);
        px0.push_back(px0.back() + (unsigned long long)F.w * F.h);
    }
    const unsigned n_tiles = (unsigned)tiles, n_chunks = (n_tiles + CHUNK - 1) / CHUNK,
                   n_supers = (n_chunks + CHUNK - 1) / CHUNK;

    std::vector<char> arena;
    const size_t o_fd = mixed_put(arena, fdesc.data(), sizeof(RasterFile) * fdesc.size());
    const size_t o_t0 = mixed_put(arena, tile0.data(), sizeof(unsigned) * tile0.size());
    const size_t o_p0 = mixed_put(arena, px0.data(), sizeof(unsigned long long) * px0.size());
    size_t o_file;
    B2_TRY(staged_upload(ctx, ctx->raster_up, arena, n, files, sizes, &o_file));
    auto al = [](unsigned long long v) { return (v + 255) / 256 * 256; };
    const size_t s_maps = 0, s_cm = s_maps + al(8ull * P * n_tiles), s_sm = s_cm + al(8ull * P * n_chunks),
                 s_se = s_sm + al(8ull * P * n_supers), s_tpx = s_se + al(sizeof(Cur) * n_supers),
                 s_nr = s_tpx + al(4ull * n_tiles), s_rpx = s_nr + al(4ull * n_tiles),
                 s_rpos = s_rpx + al(4ull * RCAP * n_tiles), s_pend = s_rpos + al(2ull * RCAP * n_tiles),
                 s_aor = s_pend + al(8ull * n), s_end = s_aor + al(4ull * n);
    B2_CUDA(ctx, ctx->raster_scratch.reserve(s_end));
    const char *A = ctx->raster_up.arena.as<char>();
    char *S = ctx->raster_scratch.as<char>();
    const uint8_t *d_files = reinterpret_cast<const uint8_t *>(A + o_file);
    const RasterFile *d_fd = reinterpret_cast<const RasterFile *>(A + o_fd);
    const unsigned *d_t0 = reinterpret_cast<const unsigned *>(A + o_t0);
    const unsigned long long *d_p0 = reinterpret_cast<const unsigned long long *>(A + o_p0);
    unsigned long long *d_maps = reinterpret_cast<unsigned long long *>(S + s_maps);
    unsigned long long *d_cm = reinterpret_cast<unsigned long long *>(S + s_cm);
    unsigned long long *d_sm = reinterpret_cast<unsigned long long *>(S + s_sm);
    Cur *d_se = reinterpret_cast<Cur *>(S + s_se);
    uint32_t *d_tpx = reinterpret_cast<uint32_t *>(S + s_tpx), *d_nr = reinterpret_cast<uint32_t *>(S + s_nr),
             *d_rpx = reinterpret_cast<uint32_t *>(S + s_rpx);
    uint16_t *d_rpos = reinterpret_cast<uint16_t *>(S + s_rpos);
    unsigned long long *d_pend = reinterpret_cast<unsigned long long *>(S + s_pend);
    unsigned *d_aor = reinterpret_cast<unsigned *>(S + s_aor);
    const unsigned long long total = px0.back();

    B2_KERNEL(ctx, "tga_tile_kernel");
    tga_tile_kernel<<<grid_for(ctx, std::max((long long)n_tiles, (long long)n), TILE_T), TILE_T, 0, ctx->stream>>>(
        d_files, d_fd, d_t0, n, n_tiles, d_maps, d_status, d_aor, d_pend);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "tga_chunk_kernel");
    tga_chunk_kernel<<<grid_for(ctx, (long long)n_chunks * P), 256, 0, ctx->stream>>>(d_maps, n_tiles, n_chunks, d_cm);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "tga_super_kernel");
    tga_super_kernel<<<grid_for(ctx, (long long)n_supers * P), 256, 0, ctx->stream>>>(d_cm, n_chunks, n_supers, d_sm);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "tga_top_kernel");
    tga_top_kernel<<<1, 32, 0, ctx->stream>>>(d_sm, n_supers, d_se);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "tga_packet_kernel");
    tga_packet_kernel<<<grid_for(ctx, n_tiles), 256, 0, ctx->stream>>>(d_files, d_fd, d_t0, n, n_tiles, d_maps, d_cm,
                                                                        d_se, d_tpx, d_nr, d_rpx, d_rpos, d_pend);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "raster_canvas_kernel");
    raster_canvas_kernel<<<grid_for(ctx, (long long)total), 256, 0, ctx->stream>>>(
        d_files, d_fd, d_p0, n, total, d_tpx, d_nr, d_rpx, d_rpos, d_pend, d_t0, reinterpret_cast<uint32_t *>(d_frames),
        d_status, d_aor);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "raster_alpha_kernel");
    raster_alpha_kernel<<<grid_for(ctx, (long long)total), 256, 0, ctx->stream>>>(d_fd, d_p0, n, total, d_aor,
                                                                                  reinterpret_cast<uint32_t *>(d_frames));
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

}  // namespace
}  // namespace b200timg

using namespace b200timg;

extern "C" {

int b200timg_raster_parse(const uint8_t *data, size_t size, b200timg_raster_info *info) {
    if (!data || size == 0 || !info) return B200TIMG_EINVAL;
    Parse P;
    if (raster_walk(data, size, P) != 0) return B200TIMG_EINVAL;
    fill_info(P, info);
    return B200TIMG_OK;
}

int b200timg_raster_frames_dev(b200timg_ctx *ctx, int n_files, const uint8_t *const *files, const size_t *sizes,
                               uint8_t *d_frames, int32_t *d_status) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    B2_TRY(check_dev_outputs(ctx, "raster", d_frames, d_status, "d_status"));
    std::vector<Parse> ps;
    B2_TRY(parse_files(ctx, "raster", "header walk", raster_walk, n_files, files, sizes, ps));
    return launch_raster(ctx, n_files, files, sizes, ps, d_frames, d_status);
}

int b200timg_raster_frames(b200timg_ctx *ctx, int n_files, const uint8_t *const *files, const size_t *sizes,
                           uint8_t *frames, int32_t *status) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!frames || !status) return ctx->fail(B200TIMG_EINVAL, "raster: null output");
    std::vector<Parse> ps;
    B2_TRY(parse_files(ctx, "raster", "header walk", raster_walk, n_files, files, sizes, ps));
    size_t bytes = 0;
    for (const Parse &P : ps) bytes += (size_t)P.w * P.h * 4;
    return decode_to_host(ctx, bytes, n_files, frames, status, [&](uint8_t *d_frames, int32_t *d_status) {
        return launch_raster(ctx, n_files, files, sizes, ps, d_frames, d_status);
    });
}

}  // extern "C"
