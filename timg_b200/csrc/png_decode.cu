// PNG files on the device: the RGBA buffer stbi__load_and_postprocess_8bit(.., 4) returns for the STB source's PNG
// branch (src/stb-image-source.cc:141-157), with every quirk of stb's chunk walk, zlib reader and unfiltering.
// png.cu is the encoder; this file only decodes.
//   host walk              stbi__parse_png_file's chunk walk (third_party/stb/stb_image.h:5079-5262) without
//                          inflating: IHDR, PLTE / tRNS as stb's palette array sees them, the IDAT payloads as runs
//   decode_gather_kernel   (decode.cu) the IDAT payloads of every file into one zlib stream per file
//   png_inflate_kernel     one CTA per file: stb's zlib reader (:4125-4509), restated bit for bit.  Thread 0 reads the
//                          block headers; the symbols of a Huffman block are decoded by every thread of the CTA
//                          (self-synchronising subsequences, as jpeg_sync_kernel), thread 0 alone only in the last
//                          bits of the stream; literals go to the raw plane, every back-reference inside the image
//                          becomes one (position, length, distance) record, and no copied byte is written.  Stored
//                          blocks are copied by the whole CTA.  Output past the image is counted, never stored.
//   png_expand_kernel      one thread per raw byte: its source index (itself for a literal, i - dist inside a copy)
//   png_jump_kernel        pointer jumping over the source indices, launched JUMP_ROUNDS times; a round that finds
//                          every index resolved makes the later rounds return at once
//   png_resolve_kernel     one thread per raw byte: the filtered byte, read through its resolved source
//   png_unfilter_kernel    one CTA per image (an Adam7 pass is an image): a wavefront in which row r trails row r-1
//                          by one pixel, so Up, Avg and Paeth read finished bytes; palette indices are range-checked
//   png_color_kernel       one thread per canvas pixel: sample extraction, depth scaling, tRNS key, palette, 16->8,
//                          stbi__convert_format to RGBA and the Adam7 scatter
// A call launches 6 + JUMP_ROUNDS kernels whatever its file count.
#include <algorithm>
#include <climits>

#include "decode.cuh"

namespace b200timg {

namespace {

constexpr int JUMP_ROUNDS = 32;                    // > log2 of the longest raw plane a call takes (2^32 bytes)
constexpr int INF_T = 512;
constexpr int UNF_T = 512;
constexpr int K_FAIL = 0, K_UNDEFINED = 1, K_OK = 2;   // per-file key, lowered with atomicMin
constexpr unsigned long long RAW_CAP = 1ull << 31;     // raw bytes one file may need on the device
constexpr unsigned long long CANVAS_CAP = 1ull << 31;  // canvas bytes of one file

__constant__ int c_xorig[7] = {0, 4, 0, 2, 0, 1, 0}, c_yorig[7] = {0, 0, 4, 0, 2, 0, 1};
__constant__ int c_xspc[7] = {8, 8, 4, 4, 2, 2, 1}, c_yspc[7] = {8, 8, 8, 4, 4, 2, 2};
const int XORIG[7] = {0, 4, 0, 2, 0, 1, 0}, YORIG[7] = {0, 0, 4, 0, 2, 0, 1};
const int XSPC[7] = {8, 8, 4, 4, 2, 2, 1}, YSPC[7] = {8, 8, 8, 4, 4, 2, 2};
const uint8_t DEPTH_SCALE[9] = {0, 0xff, 0x55, 0, 0x11, 0, 0, 0, 0x01};

// ---- descriptors -------------------------------------------------------------------------------------------------
struct __align__(16) PngFile {
    unsigned long long px0;                        // first pixel of the canvas in d_frames
    unsigned long long stream0, L;                 // the file's zlib stream in the stream scratch, and its length
    unsigned long long raw0, need;                 // its raw plane (global byte index) and the bytes the image reads
    unsigned long long rec0;                       // its first copy record
    unsigned long long limit;                      // stbi__zexpand's largest buffer: more output fails
    int w, h, depth, color, img_n, interlace, zlib_header, has_trans;
    int pal_count;                                 // palette entries stb has written (an index past them is undefined)
    int img0;                                      // its first image (pass) in the image list
    unsigned long long pass_off[7];                // raw offset of each pass inside the file (0 for an empty pass)
    int pass_w[7], pass_h[7], pass_wb[7];          // pass geometry; pass_wb: filtered bytes per row
    uint16_t tc16[3];
    uint8_t tc[3], pad_[5];
    uint32_t pal[256];                             // stb's palette[] as RGBA (alpha from tRNS), zero past pal_count
};

struct __align__(16) PngImage {                    // one unfilter wavefront: a file, or one Adam7 pass of it
    unsigned long long off;                        // global raw index of its first filter byte
    int file, w, h, wb, fb;                        // fb: filter_bytes
    int pal_depth;                                 // palette images: the bit depth (index range check), else 0
};

// ---- host walk ---------------------------------------------------------------------------------------------------
struct Run { unsigned long long off, len; };

struct Parse {
    unsigned w = 0, h = 0;
    int depth = 0, color = 0, interlace = 0, img_n = 0, pal_img_n = 0, iphone = 0, has_trans = 0, trns = 0, apng = 0;
    unsigned pal_len = 0, pal_count = 0;
    uint8_t palette[1024] = {};
    uint8_t tc[3] = {0, 0, 0};
    uint16_t tc16[3] = {0, 0, 0};
    std::vector<Run> idat;
    unsigned long long idat_bytes = 0, need = 0, limit = 0;
    bool supported = false;
    char why[96] = {0};
};

struct Rd {                                        // stbi__get8 / get32be / skip: bytes past the end read as 0
    const uint8_t *p;
    size_t n, pos = 0;
    unsigned get8() { const unsigned v = pos < n ? p[pos] : 0; ++pos; return v; }
    unsigned get16() { const unsigned a = get8(); return (a << 8) | get8(); }
    unsigned get32() { const unsigned a = get16(); return (a << 16) | get16(); }
};

constexpr unsigned T4(char a, char b, char c, char d) {
    return ((unsigned)(uint8_t)a << 24) | ((unsigned)(uint8_t)b << 16) | ((unsigned)(uint8_t)c << 8) | (uint8_t)d;
}

// HasAPNGHeader (src/image-source.cc:297-326): an acTL among the chunk headers in the first 1024 bytes
int apng_header(const uint8_t *d, size_t size) {
    size_t pos = 8;
    while (pos < 1024) {
        if (pos + 8 > size) break;
        if (!memcmp(d + pos + 4, "acTL", 4)) return 1;
        pos += ((size_t)d[pos] << 24 | (size_t)d[pos + 1] << 16 | (size_t)d[pos + 2] << 8 | d[pos + 3]) + 12;
    }
    return 0;
}

// Raw bytes one image of x*y pixels takes: (filtered row bytes + 1) * y
unsigned long long image_bytes(const Parse &P, unsigned long long x, unsigned long long y) {
    return (((unsigned long long)P.img_n * x * P.depth + 7) / 8 + 1) * y;
}

// 0: the walk reaches IEND (P.supported says whether the device takes the file); -1: stb's walk fails
int png_walk(const uint8_t *d, size_t size, Parse &P) {
    static const uint8_t sig[8] = {137, 80, 78, 71, 13, 10, 26, 10};
    Rd s{d, size};
    for (int i = 0; i < 8; ++i)
        if (s.get8() != sig[i]) return -1;
    P.apng = apng_header(d, size);
    auto unsup = [&](const char *why) { P.supported = false; snprintf(P.why, sizeof P.why, "%s", why); };
    P.supported = true;
    bool first = true, idata = false;
    unsigned long long ioff = 0;
    for (;;) {
        const unsigned len = s.get32(), type = s.get32();
        auto skip = [&]() { s.pos += len; };
        // stbi__skip takes an int: a negative length moves stb to the end of its read buffer, not of the file
        const bool skipped = type == T4('C', 'g', 'B', 'I') ||
                             (type != T4('I', 'H', 'D', 'R') && type != T4('P', 'L', 'T', 'E') &&
                              type != T4('t', 'R', 'N', 'S') && type != T4('I', 'D', 'A', 'T') &&
                              type != T4('I', 'E', 'N', 'D') && !first && (type & (1u << 29)));
        if (skipped && len >= 0x80000000u) {
            unsup("a skipped chunk of 2^31 bytes or more");
            return 0;
        }
        switch (type) {
        case T4('C', 'g', 'B', 'I'):
            P.iphone = 1;
            skip();
            break;
        case T4('I', 'H', 'D', 'R'): {
            if (!first) return -1;
            first = false;
            if (len != 13) return -1;
            P.w = s.get32(); P.h = s.get32();
            if (P.h > (1u << 24) || P.w > (1u << 24)) return -1;
            P.depth = (int)s.get8();
            if (P.depth != 1 && P.depth != 2 && P.depth != 4 && P.depth != 8 && P.depth != 16) return -1;
            P.color = (int)s.get8();
            if (P.color > 6) return -1;
            if (P.color == 3 && P.depth == 16) return -1;
            if (P.color == 3) P.pal_img_n = 3; else if (P.color & 1) return -1;
            if (s.get8()) return -1;                                    // compression
            if (s.get8()) return -1;                                    // filter method
            P.interlace = (int)s.get8();
            if (P.interlace > 1) return -1;
            if (!P.w || !P.h) return -1;
            if (!P.pal_img_n) {
                P.img_n = (P.color & 2 ? 3 : 1) + (P.color & 4 ? 1 : 0);
                if ((1u << 30) / P.w / (unsigned)P.img_n < P.h) return -1;
            } else {
                P.img_n = 1;
                if ((1u << 30) / P.w / 4 < P.h) return -1;
            }
            break;
        }
        case T4('P', 'L', 'T', 'E'): {
            if (first) return -1;
            if (len > 256 * 3) return -1;
            P.pal_len = len / 3;
            if (P.pal_len * 3 != len) return -1;
            for (unsigned i = 0; i < P.pal_len; ++i) {
                P.palette[i * 4 + 0] = (uint8_t)s.get8();
                P.palette[i * 4 + 1] = (uint8_t)s.get8();
                P.palette[i * 4 + 2] = (uint8_t)s.get8();
                P.palette[i * 4 + 3] = 255;
            }
            P.pal_count = std::max(P.pal_count, P.pal_len);
            break;
        }
        case T4('t', 'R', 'N', 'S'): {
            if (first) return -1;
            if (idata) return -1;
            if (P.pal_img_n) {
                if (P.pal_len == 0) return -1;
                if (len > P.pal_len) return -1;
                P.pal_img_n = 4;
                P.trns = 1;
                for (unsigned i = 0; i < len; ++i) P.palette[i * 4 + 3] = (uint8_t)s.get8();
            } else {
                if (!(P.img_n & 1)) return -1;
                if (len != (unsigned)P.img_n * 2) return -1;
                P.has_trans = 1;
                P.trns = 2;
                for (int k = 0; k < P.img_n && k < 3; ++k) {
                    const unsigned v = s.get16();
                    if (P.depth == 16) P.tc16[k] = (uint16_t)v;
                    else P.tc[k] = (uint8_t)((v & 255) * DEPTH_SCALE[P.depth]);
                }
            }
            break;
        }
        case T4('I', 'D', 'A', 'T'): {
            if (first) return -1;
            if (P.pal_img_n && !P.pal_len) return -1;
            if (len > (1u << 30)) return -1;
            if ((int)(uint32_t)(ioff + len) < (int)(uint32_t)ioff) return -1;
            if (s.pos + len > s.n) return -1;                           // stbi__getn: outofdata
            if (len) {                                                  // a zero-length IDAT allocates nothing
                idata = true;
                P.idat.push_back({s.pos, len});
            }
            s.pos += len;
            ioff += len;
            break;
        }
        case T4('I', 'E', 'N', 'D'): {
            if (first) return -1;
            if (!idata) return -1;
            P.idat_bytes = ioff;
            // the raw bytes the image reads, pass by pass
            P.need = 0;
            if (!P.interlace) P.need = image_bytes(P, P.w, P.h);
            else
                for (int p = 0; p < 7; ++p) {
                    const unsigned long long x = (P.w - XORIG[p] + XSPC[p] - 1) / XSPC[p];
                    const unsigned long long y = (P.h - YORIG[p] + YSPC[p] - 1) / YSPC[p];
                    if (x && y) P.need += image_bytes(P, x, y);
                }
            // stbi_zlib_decode_malloc_guesssize_headerflag's initial size and the largest buffer stbi__zexpand reaches
            const uint32_t bpl = (P.w * (uint32_t)P.depth + 7) / 8;
            const int guess = (int)(bpl * P.h * (uint32_t)P.img_n + P.h);
            if (guess <= 0) unsup("stb's initial inflate buffer size is not a positive int");
            else {
                unsigned long long lim = (unsigned long long)guess;
                while (lim <= 0x7fffffffull) lim *= 2;
                P.limit = lim;
            }
            if (P.need > RAW_CAP) unsup("more than 2^31 raw bytes");
            if ((unsigned long long)P.w * P.h * 4 > CANVAS_CAP) unsup("a canvas of more than 2^31 bytes");
            if (P.idat_bytes >= (1ull << 31)) unsup("2^31 IDAT bytes or more");
            return 0;
        }
        default:
            if (first) return -1;
            if ((type & (1u << 29)) == 0) return -1;                    // unknown critical chunk
            skip();
            break;
        }
        s.get32();                                                      // CRC, never checked
    }
}

}  // namespace
}  // namespace b200timg

namespace b200timg {
namespace {

// ---- the device inflater: stb's zbuf, restated -------------------------------------------------------------------
struct ZHuff {                                     // stbi__zhuffman
    uint16_t fast[512];
    uint16_t firstcode[16];
    int maxcode[17];
    uint16_t firstsymbol[16];
    uint8_t size[288];
    uint16_t value[288];
};

__device__ __constant__ int c_len_base[31] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31,
                                              35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258, 0, 0};
__device__ __constant__ int c_len_extra[31] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2,
                                               3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0, 0, 0};
__device__ __constant__ int c_dist_base[32] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193,
                                               257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289,
                                               16385, 24577, 0, 0};
__device__ __constant__ int c_dist_extra[32] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6,
                                                7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13, 0, 0};
__device__ __constant__ uint8_t c_clen_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

__device__ __forceinline__ int bitrev16(unsigned v) { return (int)(__brev(v) >> 16); }

// stbi__zbuild_huffman (:4125-4170): false where stb fails
__device__ bool zbuild(ZHuff &z, const uint8_t *sizelist, int num) {
    int sizes[17], next_code[16];
    for (int i = 0; i < 17; ++i) sizes[i] = 0;
    for (int i = 0; i < 512; ++i) z.fast[i] = 0;
    for (int i = 0; i < 288; ++i) z.size[i] = 0;
    for (int i = 0; i < num; ++i) ++sizes[sizelist[i]];
    sizes[0] = 0;
    for (int i = 1; i < 16; ++i)
        if (sizes[i] > (1 << i)) return false;
    int code = 0, k = 0;
    for (int i = 1; i < 16; ++i) {
        next_code[i] = code;
        z.firstcode[i] = (uint16_t)code;
        z.firstsymbol[i] = (uint16_t)k;
        code = code + sizes[i];
        if (sizes[i] && code - 1 >= (1 << i)) return false;
        z.maxcode[i] = code << (16 - i);
        code <<= 1;
        k += sizes[i];
    }
    z.maxcode[16] = 0x10000;
    for (int i = 0; i < num; ++i) {
        const int s = sizelist[i];
        if (s) {
            const int c = next_code[s] - z.firstcode[s] + z.firstsymbol[s];
            const uint16_t fastv = (uint16_t)((s << 9) | i);
            z.size[c] = (uint8_t)s;
            z.value[c] = (uint16_t)i;
            if (s <= 9) {
                int j = (int)(__brev((unsigned)next_code[s]) >> (32 - s));
                while (j < 512) { z.fast[j] = fastv; j += 1 << s; }
            }
            ++next_code[s];
        }
    }
    return true;
}

struct ZBuf {
    const uint8_t *d;
    unsigned long long L, F;                       // stream length, next byte stbi__zget8 reads
    uint32_t cb;                                   // code_buffer
    int nb, hit;                                   // num_bits, hit_zeof_once
    __device__ bool eof() const { return F >= L; }
    __device__ unsigned get8() { return eof() ? 0u : d[F++]; }
    __device__ void fill() {                       // stbi__fill_bits
        do {
            if (cb >= (1u << nb)) { F = L; return; }
            cb |= get8() << nb;
            nb += 8;
        } while (nb <= 24);
    }
    __device__ unsigned receive(int n) {           // stbi__zreceive
        if (nb < n) fill();
        const unsigned k = cb & ((1u << n) - 1);
        cb >>= n;
        nb -= n;
        return k;
    }
    __device__ int decode(const ZHuff &z) {        // stbi__zhuffman_decode and its slow path
        if (nb < 16) {
            if (eof()) {
                if (!hit) { hit = 1; nb += 16; }
                else return -1;
            } else fill();
        }
        const int b = z.fast[cb & 511];
        if (b) {
            const int s = b >> 9;
            cb >>= s;
            nb -= s;
            return b & 511;
        }
        const int k = bitrev16(cb);
        int s;
        for (s = 10;; ++s)
            if (k < z.maxcode[s]) break;
        if (s >= 16) return -1;
        const int c = (k >> (16 - s)) - z.firstcode[s] + z.firstsymbol[s];
        if (c >= 288) return -1;
        if (z.size[c] != s) return -1;
        cb >>= s;
        nb -= s;
        return z.value[c];
    }
};

// stbi__compute_huffman_codes (:4360-4408): false where stb fails
__device__ bool dynamic_tables(ZBuf &a, ZHuff &len, ZHuff &dist, ZHuff &clen, uint8_t *lencodes) {
    const int hlit = (int)a.receive(5) + 257, hdist = (int)a.receive(5) + 1, hclen = (int)a.receive(4) + 4;
    const int ntot = hlit + hdist;
    uint8_t cls[19];
    for (int i = 0; i < 19; ++i) cls[i] = 0;
    for (int i = 0; i < hclen; ++i) cls[c_clen_order[i]] = (uint8_t)a.receive(3);
    if (!zbuild(clen, cls, 19)) return false;
    int n = 0;
    while (n < ntot) {
        int c = a.decode(clen);
        if (c < 0 || c >= 19) return false;
        if (c < 16) lencodes[n++] = (uint8_t)c;
        else {
            uint8_t fill = 0;
            if (c == 16) {
                c = (int)a.receive(2) + 3;
                if (n == 0) return false;
                fill = lencodes[n - 1];
            } else if (c == 17) c = (int)a.receive(3) + 3;
            else c = (int)a.receive(7) + 11;
            if (ntot - n < c) return false;
            for (int i = 0; i < c; ++i) lencodes[n + i] = fill;
            n += c;
        }
    }
    if (n != ntot) return false;
    if (!zbuild(len, lencodes, hlit)) return false;
    return zbuild(dist, lencodes + hlit, hdist);
}

// ---- the parallel symbol decode -----------------------------------------------------------------------------------
// Inside a Huffman block, a unit (a literal, an end-of-block, or a length with its extra bits, distance code and extra
// bits) starts where the previous one ends, and stb's reader decodes it the same way whatever it has buffered, as long
// as it never reaches the end of the stream.  So a unit boundary is a bit position P, and a window of INF_T
// subsequences of SUB_BITS bits is decoded speculatively (Weissenberger & Schmidt, as jpeg_sync_kernel does): every
// thread walks from a guessed start to the first boundary past its end, and the CTA iterates until each start equals
// its predecessor's exit up to the first thread that meets the block's end (or an error).  Round r makes thread r's
// start exact, so the result never depends on how fast that converges.  stb's buffered-byte frontier F (num_bits is
// 8F - P) only matters near the stream's end: a window stays END_GUARD bits clear of it, each thread maps the five
// frontiers its start can have to the one at its exit, and thread 0 chains those maps to resume stb's exact reader.
constexpr int SUB_BITS = 256;
constexpr unsigned long long END_GUARD = 256;

struct PBits {                                     // the stream as bits, zeros past its end
    const uint8_t *d;
    unsigned long long L;
    __device__ __forceinline__ uint32_t peek(unsigned long long P) const {   // the 32 bits from P, LSB first
        const unsigned long long b = P >> 3;
        unsigned long long w = 0;
        for (int i = 0; i < 5; ++i) w |= (unsigned long long)(b + i < L ? d[b + i] : 0) << (8 * i);
        return (uint32_t)(w >> (P & 7));
    }
};

// stbi__zhuffman_decode on a full buffer: the symbol (or -1) and its length s
__device__ __forceinline__ int pdecode(const ZHuff &z, uint32_t cb, int &s) {
    const int b = z.fast[cb & 511];
    if (b) { s = b >> 9; return b & 511; }
    const int k = bitrev16(cb);
    for (s = 10;; ++s)
        if (k < z.maxcode[s]) break;
    if (s >= 16) return -1;
    const int c = (k >> (16 - s)) - z.firstcode[s] + z.firstsymbol[s];
    if (c >= 288 || z.size[c] != s) return -1;
    return z.value[c];
}

// stbi__fill_bits' effect on the frontier of each candidate: a read needing thr bits with fewer buffered refills
// to the first byte boundary more than 24 bits past P
template <bool FMAP>
__device__ __forceinline__ void fill_op(unsigned long long *F, unsigned long long P, int thr) {
    if (FMAP)
#pragma unroll
        for (int k = 0; k < 5; ++k)
            if ((long long)(F[k] * 8) - (long long)P < thr) F[k] = (P >> 3) + 4;
}

// Units from P until P >= end: 0 (end passed), 1 (end-of-block; P after it), 2 (an error stb reports; P at it).
// MODE 0 counts output bytes; 1 also counts the copy records inside the image, maps frontiers and flags "bad dist";
// 2 writes the literals and the records.
template <int MODE>
__device__ int walk(const PBits &r, const ZHuff &Lt, const ZHuff &Dt, unsigned long long &P, unsigned long long end,
                    unsigned long long pos, unsigned long long need, unsigned long long &outc, unsigned &nrc,
                    unsigned long long *F, bool &bad, uint8_t *out, uint2 *rec) {
    while (P < end) {
        fill_op<MODE == 1>(F, P, 16);
        int s;
        int z = pdecode(Lt, r.peek(P), s);
        if (z < 0) return 2;
        P += (unsigned)s;
        if (z < 256) {
            if (MODE == 2 && pos < need) out[pos] = (uint8_t)z;
            ++pos; ++outc;
            continue;
        }
        if (z == 256) return 1;
        if (z >= 286) return 2;
        z -= 257;
        unsigned ln = (unsigned)c_len_base[z];
        int e = c_len_extra[z];
        if (e) { fill_op<MODE == 1>(F, P, e); ln += r.peek(P) & ((1u << e) - 1); P += (unsigned)e; }
        fill_op<MODE == 1>(F, P, 16);
        const int zd = pdecode(Dt, r.peek(P), s);
        if (zd < 0 || zd >= 30) return 2;
        P += (unsigned)s;
        unsigned dist = (unsigned)c_dist_base[zd];
        e = c_dist_extra[zd];
        if (e) { fill_op<MODE == 1>(F, P, e); dist += r.peek(P) & ((1u << e) - 1); P += (unsigned)e; }
        if (pos < dist) bad = true;
        else if (pos < need) {
            if (MODE == 2) rec[nrc] = make_uint2((unsigned)pos, ln | (dist << 16));
            ++nrc;
        }
        pos += ln; outc += ln;
    }
    return 0;
}

// stbi__parse_huffman_block from a's state, serially, to the block's end or the first error
__device__ void serial_symbols(ZBuf &a, const ZHuff &Lt, const ZHuff &Dt, const PngFile &f, uint8_t *out, uint2 *rec,
                               unsigned long long &pos, unsigned &nr, bool &ok) {
    while (ok) {
        int z = a.decode(Lt);
        if (z < 256) {
            if (z < 0) { ok = false; break; }
            if (pos + 1 > f.limit) { ok = false; break; }
            if (pos < f.need) out[pos] = (uint8_t)z;
            ++pos;
        } else {
            if (z == 256) {
                if (a.hit && a.nb < 16) ok = false;
                break;
            }
            if (z >= 286) { ok = false; break; }
            z -= 257;
            int ln = c_len_base[z];
            if (c_len_extra[z]) ln += (int)a.receive(c_len_extra[z]);
            z = a.decode(Dt);
            if (z < 0 || z >= 30) { ok = false; break; }
            int dist = c_dist_base[z];
            if (c_dist_extra[z]) dist += (int)a.receive(c_dist_extra[z]);
            if (pos < (unsigned long long)dist) { ok = false; break; }   // bad dist
            if (pos + (unsigned)ln > f.limit) { ok = false; break; }
            if (pos < f.need) rec[f.rec0 + nr++] = make_uint2((unsigned)pos, (unsigned)ln | ((unsigned)dist << 16));
            pos += (unsigned)ln;
        }
    }
}

// Exclusive sum over the CTA through s[INF_T]; *total gets the sum.  Ends with a barrier.
__device__ __forceinline__ unsigned long long cta_excl_scan(unsigned long long v, unsigned long long *s,
                                                            unsigned long long *total) {
    const int t = threadIdx.x;
    s[t] = v;
    __syncthreads();
    for (int d = 1; d < INF_T; d <<= 1) {
        const unsigned long long x = t >= d ? s[t - d] : 0ull;
        __syncthreads();
        s[t] += x;
        __syncthreads();
    }
    const unsigned long long incl = s[t];
    *total = s[INF_T - 1];
    __syncthreads();
    return incl - v;
}

// One CTA per file.  Thread 0 runs stb's reader through the block headers, stored blocks (copied by every thread) and
// the last END_GUARD bits of the stream; the symbols of Huffman blocks are decoded by the whole CTA, a window at a
// time.  The raw plane gets the literals of positions < need; copies inside the image become records
// (pos, len | dist << 16), in output order.
__global__ void __launch_bounds__(INF_T, 1)
png_inflate_kernel(const PngFile *__restrict__ fd, const uint8_t *__restrict__ stream, uint8_t *__restrict__ raw,
                   uint2 *__restrict__ rec, unsigned *__restrict__ nrec, int *__restrict__ key) {
    __shared__ ZHuff s_len, s_dist, s_clen;
    __shared__ uint8_t s_codes[286 + 32 + 137];
    __shared__ unsigned long long s_src, s_dst, s_n;
    __shared__ unsigned long long s_start[INF_T], s_ex[INF_T], s_scan[INF_T], s_fmap[INF_T][5];
    __shared__ int s_kind[INF_T];
    __shared__ unsigned long long s_P0, s_pos;
    __shared__ unsigned s_nr;
    __shared__ int s_state;                        // 0 continue, 1 stored copy pending, 2 stop, 3 Huffman symbols
    __shared__ int s_stop_after, s_mode, s_nact, s_tend, s_bad, s_bdone;
    const int t = threadIdx.x;
    const PngFile &f = fd[blockIdx.x];
    uint8_t *out = raw + f.raw0;
    const PBits rd{stream + f.stream0, f.L};
    ZBuf a;
    unsigned long long pos = 0;
    unsigned nr = 0;
    bool ok = true, fixed_built = false;
    if (t == 0) {
        a.d = stream + f.stream0; a.L = f.L; a.F = 0; a.cb = 0; a.nb = 0; a.hit = 0;
        if (f.zlib_header) {                       // stbi__parse_zlib_header
            const unsigned cmf = a.get8(), flg = a.get8();
            if (a.eof() || (cmf * 256 + flg) % 31 != 0 || (flg & 32) || (cmf & 15) != 8) ok = false;
        }
        a.cb = 0; a.nb = 0; a.hit = 0;
    }
    for (;;) {
        if (t == 0) {
            s_state = 2;
            s_stop_after = 1;
            if (ok) {
                const unsigned final_ = a.receive(1), type = a.receive(2);
                s_stop_after = (int)final_;
                if (type == 0) {                   // stbi__parse_uncompressed_block
                    uint8_t hd[4];
                    int k = 0;
                    if (a.nb & 7) a.receive(a.nb & 7);
                    while (a.nb > 0) { hd[k++] = (uint8_t)(a.cb & 255); a.cb >>= 8; a.nb -= 8; }
                    if (a.nb < 0) ok = false;
                    while (ok && k < 4) hd[k++] = (uint8_t)a.get8();
                    if (ok) {
                        const unsigned ln = hd[1] * 256u + hd[0], nln = hd[3] * 256u + hd[2];
                        if (nln != (ln ^ 0xffffu)) ok = false;
                        else if (a.F + ln > a.L) ok = false;                    // read past buffer
                        else if (pos + ln > f.limit) ok = false;                // outofmem
                        else {
                            s_src = a.F; s_dst = pos;
                            s_n = pos >= f.need ? 0ull : (f.need - pos < ln ? f.need - pos : (unsigned long long)ln);
                            a.F += ln;
                            pos += ln;
                            s_state = 1;
                        }
                    }
                } else if (type == 3) ok = false;
                else {
                    if (type == 1) {
                        if (!fixed_built) {
                            uint8_t *l = s_codes;
                            for (int i = 0; i < 288; ++i) l[i] = i <= 143 ? 8 : i <= 255 ? 9 : i <= 279 ? 7 : 8;
                            zbuild(s_len, l, 288);
                            for (int i = 0; i < 32; ++i) l[i] = 5;
                            zbuild(s_dist, l, 32);
                            fixed_built = true;
                        }
                    } else {
                        fixed_built = false;
                        if (!dynamic_tables(a, s_len, s_dist, s_clen, s_codes)) ok = false;
                    }
                    if (ok) s_state = 3;
                }
            }
            if (!ok) s_state = 2;
            s_bdone = 0;
        }
        __syncthreads();
        const int st = s_state;
        if (st == 1) {
            const uint8_t *src = stream + f.stream0 + s_src;
            uint8_t *dst = out + s_dst;
            for (unsigned long long i = t; i < s_n; i += INF_T) dst[i] = src[i];
        }
        while (st == 3) {                          // the block's symbols, a window at a time
            if (t == 0) {
                s_mode = 0;
                if (ok && !s_bdone) {
                    const unsigned long long P0 = 8 * a.F - (unsigned long long)a.nb, bits = 8 * a.L;
                    const unsigned long long room = bits > END_GUARD + P0 ? bits - END_GUARD - P0 : 0ull;
                    const int nact = (int)(room / SUB_BITS < (unsigned long long)INF_T ? room / SUB_BITS : INF_T);
                    if (!a.hit && nact >= 4) {
                        s_mode = 1; s_P0 = P0; s_nact = nact; s_pos = pos; s_nr = nr; s_bad = 0;
                    } else serial_symbols(a, s_len, s_dist, f, out, rec, pos, nr, ok);
                }
            }
            __syncthreads();
            if (s_mode == 0) break;
            const int nact = s_nact;
            const bool act = t < nact;
            unsigned long long start = s_P0 + (unsigned long long)t * SUB_BITS, ex = start, outc = 0;
            const unsigned long long end = start + SUB_BITS;
            int kind = 0, tend;
            bool dirty = true, bad = false;
            unsigned nrc = 0;
            for (;;) {                             // synchronise the subsequences
                if (act && dirty) {
                    unsigned long long P = start;
                    outc = 0;
                    kind = walk<0>(rd, s_len, s_dist, P, end, 0, 0, outc, nrc, nullptr, bad, nullptr, nullptr);
                    ex = P;
                    dirty = false;
                }
                s_ex[t] = ex;
                s_kind[t] = act ? kind : 0;
                if (t == 0) s_tend = nact - 1;
                __syncthreads();
                if (act && kind) atomicMin(&s_tend, t);
                __syncthreads();
                tend = s_tend;
                bool ch = false;
                if (act && t > 0 && s_ex[t - 1] != start) {
                    start = s_ex[t - 1];
                    dirty = true;
                    ch = t <= tend;
                }
                if (!__syncthreads_or(ch)) break;
            }
            const bool mine = act && t <= tend;
            unsigned long long tot_out, tot_rec;
            const unsigned long long base = s_pos + cta_excl_scan(mine ? outc : 0ull, s_scan, &tot_out);
            nrc = 0;
            bad = false;
            if (mine) {                            // copy records, frontier map, "bad dist"
                unsigned long long F[5], P = start, oc = 0;
                for (int k = 0; k < 5; ++k) F[k] = (start >> 3) + k;
                walk<1>(rd, s_len, s_dist, P, end, base, f.need, oc, nrc, F, bad, nullptr, nullptr);
                for (int k = 0; k < 5; ++k) s_fmap[t][k] = F[k];
                s_start[t] = start;
                if (bad) atomicOr(&s_bad, 1);
            }
            const unsigned long long rbase = s_nr + cta_excl_scan(mine ? (unsigned long long)nrc : 0ull, s_scan, &tot_rec);
            if (mine) {
                unsigned long long P = start, oc = 0;
                unsigned idx = 0;
                walk<2>(rd, s_len, s_dist, P, end, base, f.need, oc, idx, nullptr, bad, out, rec + f.rec0 + rbase);
            }
            __syncthreads();
            if (t == 0) {
                if (s_kind[tend] == 2 || s_bad) ok = false;
                pos = s_pos + tot_out;
                nr = s_nr + (unsigned)tot_rec;
                if (pos > f.limit) ok = false;
                unsigned long long F = a.F;        // chain the frontier maps from the exact reader
                for (int k = 0; k <= tend; ++k) {
                    const long long rel = (long long)(F - (s_start[k] >> 3));
                    F = s_fmap[k][rel < 0 ? 0 : rel > 4 ? 4 : rel];
                }
                const unsigned long long Pe = s_ex[tend];
                a.F = F;
                a.nb = (int)(8 * F - Pe);
                a.cb = a.nb == 0 ? 0u : rd.peek(Pe) & (a.nb >= 32 ? ~0u : (1u << a.nb) - 1);
                if (s_kind[tend] == 1) s_bdone = 1;   // end-of-block, with hit_zeof_once still 0
            }
            __syncthreads();
        }
        if (t == 0 && st == 3 && !ok) s_state = 2;
        __syncthreads();
        const bool stop = s_state == 2 || s_stop_after;
        __syncthreads();
        if (stop) break;
    }
    if (t == 0) {
        if (ok && pos < f.need) ok = false;        // not enough pixels (pass by pass, the same total)
        nrec[blockIdx.x] = nr;
        key[blockIdx.x] = ok ? K_OK : K_FAIL;
    }
}

// Source index of every raw byte: itself for a literal, i - dist for a byte inside a copy record.
__global__ void __launch_bounds__(256)
png_expand_kernel(const PngFile *__restrict__ fd, const unsigned long long *__restrict__ file_raw0, int n_files,
                  const uint2 *__restrict__ rec, const unsigned *__restrict__ nrec, unsigned *__restrict__ src) {
    const unsigned long long total = file_raw0[n_files];
    for (unsigned long long g = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; g < total;
         g += (unsigned long long)gridDim.x * blockDim.x) {
        const int fi = mixed_owner(file_raw0, n_files, g);
        const PngFile &f = fd[fi];
        const unsigned i = (unsigned)(g - f.raw0);
        const uint2 *r = rec + f.rec0;
        int lo = 0, hi = (int)nrec[fi] - 1, k = -1;        // the last record starting at or before i
        while (lo <= hi) {
            const int mid = (lo + hi) >> 1;
            if (r[mid].x <= i) { k = mid; lo = mid + 1; } else hi = mid - 1;
        }
        unsigned s = i;
        if (k >= 0 && i < r[k].x + (r[k].y & 0xffffu)) s = i - (r[k].y >> 16);
        src[g] = (unsigned)(f.raw0 + s);
    }
}

// One pointer-jumping round: src[i] = src[src[i]].  Round r returns at once if round r - 1 changed nothing.
__global__ void __launch_bounds__(256)
png_jump_kernel(unsigned *src, unsigned long long total, unsigned *changed, int round) {
    if (round > 0 && !*(volatile unsigned *)&changed[round - 1]) return;
    bool ch = false;
    for (unsigned long long g = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; g < total;
         g += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned s = src[g], t = src[s];
        if (t != s) { src[g] = t; ch = true; }
    }
    if (__syncthreads_or(ch) && threadIdx.x == 0) atomicOr(&changed[round], 1u);
}

__global__ void __launch_bounds__(256)
png_resolve_kernel(const uint8_t *__restrict__ raw, const unsigned *__restrict__ src, unsigned long long total,
                   uint8_t *__restrict__ flt) {
    for (unsigned long long g = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; g < total;
         g += (unsigned long long)gridDim.x * blockDim.x)
        flt[g] = raw[src[g]];
}

__device__ __forceinline__ int paeth(int a, int b, int c) {   // stbi__paeth
    const int thresh = c * 3 - (a + b);
    const int lo = a < b ? a : b, hi = a < b ? b : a;
    const int t0 = (hi <= thresh) ? lo : c;
    return (thresh <= lo) ? hi : t0;
}

// One CTA per image.  Thread t takes channel t % fb of row r0 + t / fb; at step s it unfilters pixel s - t / fb of its
// row, so the row above finished that pixel (and the one left of it) in earlier steps.  The filter bytes stay.
__global__ void __launch_bounds__(UNF_T)
png_unfilter_kernel(const PngImage *__restrict__ imgs, const PngFile *__restrict__ fd, uint8_t *flt,
                    int *__restrict__ key) {
    const PngImage im = imgs[blockIdx.x];
    const int fb = im.fb, rows = UNF_T / fb, t = threadIdx.x;
    const int lr = t / fb, c = t % fb;
    const bool lane = lr < rows;
    const int cols = (im.wb + fb - 1) / fb;
    const unsigned long long stride = (unsigned long long)im.wb + 1;
    const int pal_n = im.pal_depth ? fd[im.file].pal_count : 0;
    bool bad_filter = false, bad_index = false;
    for (int r0 = 0; r0 < im.h; r0 += rows) {
        const int row = r0 + lr;
        const bool live = lane && row < im.h;
        uint8_t *cur = flt + im.off + (unsigned long long)row * stride;
        const uint8_t *prior = cur - stride;
        int ft = 0, a = 0, cu = 0;                 // filter, left byte, upper-left byte (same channel)
        if (live) {
            ft = cur[0];
            if (ft > 4) { bad_filter = true; ft = 0; }
        }
        const bool top = row == 0;
        for (int s = 0; s < cols + rows - 1; ++s) {
            const int k = s - lr;
            if (live && k >= 0 && k < cols) {
                const int b = k * fb + c;
                if (b < im.wb) {
                    const int x = cur[1 + b];
                    const int up = top ? 0 : prior[1 + b];
                    int v;
                    switch (ft) {
                    case 1: v = x + a; break;
                    case 2: v = x + up; break;
                    case 3: v = x + ((up + a) >> 1); break;
                    case 4: v = x + paeth(a, up, cu); break;
                    default: v = x; break;
                    }
                    v &= 255;
                    cur[1 + b] = (uint8_t)v;
                    a = v; cu = up;
                    if (pal_n) {
                        const int d = im.pal_depth, per = 8 / d;
                        for (int q = 0; q < per; ++q) {
                            const long long si = (long long)b * per + q;
                            if (si < im.w && ((v >> (8 - d * (q + 1))) & ((1 << d) - 1)) >= pal_n) bad_index = true;
                        }
                    }
                }
            }
            __syncthreads();
        }
    }
    if (bad_filter) atomicMin(key + im.file, K_FAIL);
    if (bad_index) atomicMin(key + im.file, K_UNDEFINED);
}

__device__ __forceinline__ unsigned sample(const uint8_t *row, int depth, unsigned long long s) {
    if (depth == 8) return row[s];
    if (depth == 16) return ((unsigned)row[2 * s] << 8) | row[2 * s + 1];
    const unsigned long long bit = s * (unsigned)depth;
    return (row[bit >> 3] >> (8 - depth - (int)(bit & 7))) & ((1u << depth) - 1);
}

__device__ __forceinline__ int adam7_pass(int x, int y) {
    const int xm = x & 7, ym = y & 7;
    if (ym & 1) return 6;
    if (xm & 1) return 5;
    if (ym & 2) return 4;
    if (xm & 2) return 3;
    if (ym & 4) return 2;
    if (xm & 4) return 1;
    return 0;
}

__global__ void __launch_bounds__(256)
png_color_kernel(const PngFile *__restrict__ fd, const unsigned long long *__restrict__ file_px0, int n_files,
                 const uint8_t *__restrict__ flt, const int *__restrict__ key, uint32_t *__restrict__ out,
                 int32_t *__restrict__ status) {
    const unsigned long long total = file_px0[n_files];
    for (unsigned long long p = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; p < total;
         p += (unsigned long long)gridDim.x * blockDim.x) {
        const int fi = mixed_owner(file_px0, n_files, p);
        const PngFile &f = fd[fi];
        const unsigned long long o = p - f.px0;
        const int y = (int)(o / (unsigned)f.w), x = (int)(o - (unsigned long long)y * (unsigned)f.w);
        if (o == 0) {
            const int k = key[fi];
            status[fi] = k == K_OK ? 1 : k == K_UNDEFINED ? -1 : 0;
        }
        int pass = 0, i = x, j = y;
        if (f.interlace) {
            pass = adam7_pass(x, y);
            i = (x - c_xorig[pass]) / c_xspc[pass];
            j = (y - c_yorig[pass]) / c_yspc[pass];
        }
        const uint8_t *row = flt + f.raw0 + f.pass_off[pass] + (unsigned long long)j * (f.pass_wb[pass] + 1) + 1;
        const unsigned long long s0 = (unsigned long long)i * f.img_n;
        const int d = f.depth;
        const unsigned scale = (f.color == 0 && d < 8) ? (unsigned)(d == 1 ? 0xff : d == 2 ? 0x55 : 0x11) : 1u;
        uint32_t px;
        if (f.color == 3) {
            px = f.pal[sample(row, d, s0) & 255];
        } else if (f.img_n <= 2) {
            const unsigned g = sample(row, d, s0);
            unsigned g8 = d == 16 ? g >> 8 : (g * scale) & 255, a8 = 255;
            if (f.img_n == 2) { const unsigned av = sample(row, d, s0 + 1); a8 = d == 16 ? av >> 8 : av; }
            else if (f.has_trans) a8 = (d == 16 ? g == f.tc16[0] : g8 == f.tc[0]) ? 0 : 255;
            px = pack_rgba(g8, g8, g8, a8);
        } else {
            unsigned v[4];
            for (int q = 0; q < f.img_n; ++q) v[q] = sample(row, d, s0 + q);
            unsigned a8 = 255;
            if (f.img_n == 4) a8 = d == 16 ? v[3] >> 8 : v[3];
            else if (f.has_trans) {
                const bool m = d == 16 ? (v[0] == f.tc16[0] && v[1] == f.tc16[1] && v[2] == f.tc16[2])
                                       : (v[0] == f.tc[0] && v[1] == f.tc[1] && v[2] == f.tc[2]);
                if (m) a8 = 0;
            }
            if (d == 16) { v[0] >>= 8; v[1] >>= 8; v[2] >>= 8; }
            px = pack_rgba(v[0] & 255, v[1] & 255, v[2] & 255, a8);
        }
        out[p] = px;
    }
}

}  // namespace
}  // namespace b200timg

namespace b200timg {
namespace {

void fill_info(const Parse &P, b200timg_png_info *info) {
    memset(info, 0, sizeof *info);
    info->w = (int)P.w; info->h = (int)P.h;
    info->bit_depth = P.depth; info->color_type = P.color; info->interlace = P.interlace;
    info->palette_len = (int)P.pal_len;
    info->trns = P.trns;
    info->cgbi = P.iphone;
    info->apng = P.apng;
    info->idat_bytes = P.idat_bytes;
    info->supported = P.supported ? 1 : 0;
    snprintf(info->reason, sizeof info->reason, "%s", P.supported ? "" : P.why);
}

// Device scratch of one call (ctx->png_up.arena + ctx->png_scratch): the files + 1.2 KB per file + 32 bytes per image +
// 16 bytes per IDAT; the zlib streams, 6 bytes per raw byte the images read (literal plane, source index, filtered
// plane), 8 bytes per copy record (at most need / 3 + 1 per file), 8 bytes per file.
int launch_png(b200timg_ctx *ctx, int n, const uint8_t *const *files, const size_t *sizes, const std::vector<Parse> &ps,
               uint8_t *d_frames, int32_t *d_status) {
    std::vector<PngFile> fdesc((size_t)n);
    std::vector<PngImage> imgs;
    Runs runs;
    std::vector<unsigned long long> file_raw0(1, 0), file_px0(1, 0);
    unsigned long long file_off = 0, stream = 0, recs = 0;
    for (int fi = 0; fi < n; ++fi) {
        const Parse &P = ps[(size_t)fi];
        PngFile &F = fdesc[(size_t)fi];
        memset(&F, 0, sizeof F);
        F.px0 = file_px0.back();
        file_px0.push_back(F.px0 + (unsigned long long)P.w * P.h);
        F.stream0 = stream; F.L = P.idat_bytes;
        for (const Run &r : P.idat) runs.add(file_off + r.off, r.len);
        stream += P.idat_bytes;
        F.raw0 = file_raw0.back(); F.need = P.need;
        file_raw0.push_back(F.raw0 + P.need);
        F.rec0 = recs; recs += P.need / 3 + 1;
        F.limit = P.limit;
        F.w = (int)P.w; F.h = (int)P.h; F.depth = P.depth; F.color = P.color; F.img_n = P.img_n;
        F.interlace = P.interlace; F.zlib_header = !P.iphone; F.has_trans = P.has_trans;
        F.pal_count = P.color == 3 ? (int)P.pal_count : 0;
        for (int k = 0; k < 3; ++k) { F.tc[k] = P.tc[k]; F.tc16[k] = P.tc16[k]; }
        for (unsigned i = 0; i < 256; ++i)
            F.pal[i] = i < P.pal_count ? (uint32_t)P.palette[i * 4] | (uint32_t)P.palette[i * 4 + 1] << 8 |
                                             (uint32_t)P.palette[i * 4 + 2] << 16 | (uint32_t)P.palette[i * 4 + 3] << 24
                                       : 0u;
        F.img0 = (int)imgs.size();
        const int fb = P.depth < 8 ? 1 : P.img_n * (P.depth / 8);
        unsigned long long off = 0;
        for (int p = 0; p < (P.interlace ? 7 : 1); ++p) {
            const unsigned long long x = P.interlace ? (P.w - XORIG[p] + XSPC[p] - 1) / XSPC[p] : P.w;
            const unsigned long long y = P.interlace ? (P.h - YORIG[p] + YSPC[p] - 1) / YSPC[p] : P.h;
            F.pass_w[p] = (int)x; F.pass_h[p] = (int)y;
            F.pass_wb[p] = (int)((P.img_n * x * P.depth + 7) / 8);
            F.pass_off[p] = off;
            if (!x || !y) continue;
            PngImage im;
            memset(&im, 0, sizeof im);
            im.off = F.raw0 + off; im.file = fi; im.w = (int)x; im.h = (int)y; im.wb = F.pass_wb[p]; im.fb = fb;
            im.pal_depth = P.color == 3 ? P.depth : 0;
            imgs.push_back(im);
            off += image_bytes(P, x, y);
        }
        file_off += sizes[fi];
    }
    const unsigned long long raw_total = file_raw0.back();
    if (raw_total >= (1ull << 32))
        return ctx->fail(B200TIMG_EINVAL, "png: %llu raw bytes in one call (less than 2^32)", raw_total);
    const int n_img = (int)imgs.size();

    std::vector<char> arena;
    const size_t o_fd = mixed_put(arena, fdesc.data(), sizeof(PngFile) * fdesc.size());
    const size_t o_im = mixed_put(arena, imgs.data(), sizeof(PngImage) * imgs.size());
    runs.put(arena);
    const size_t o_fr = mixed_put(arena, file_raw0.data(), sizeof(unsigned long long) * file_raw0.size());
    const size_t o_fp = mixed_put(arena, file_px0.data(), sizeof(unsigned long long) * file_px0.size());
    size_t o_file;
    B2_TRY(staged_upload(ctx, ctx->png_up, arena, n, files, sizes, &o_file));
    auto al = [](unsigned long long v) { return (v + 255) / 256 * 256; };
    const size_t s_stream = 0, s_raw = al(stream), s_src = s_raw + al(raw_total), s_flt = s_src + al(4 * raw_total),
                 s_rec = s_flt + al(raw_total), s_nrec = s_rec + al(8 * recs), s_key = s_nrec + al(4ull * n),
                 s_ch = s_key + al(4ull * n), s_end = s_ch + al(4ull * JUMP_ROUNDS);
    B2_CUDA(ctx, ctx->png_scratch.reserve(s_end));
    const char *A = ctx->png_up.arena.as<char>();
    char *S = ctx->png_scratch.as<char>();
    const PngFile *d_fd = reinterpret_cast<const PngFile *>(A + o_fd);
    const unsigned long long *d_fr = reinterpret_cast<const unsigned long long *>(A + o_fr);
    uint8_t *d_stream = reinterpret_cast<uint8_t *>(S + s_stream);
    uint8_t *d_raw = reinterpret_cast<uint8_t *>(S + s_raw);
    unsigned *d_src = reinterpret_cast<unsigned *>(S + s_src);
    uint8_t *d_flt = reinterpret_cast<uint8_t *>(S + s_flt);
    uint2 *d_rec = reinterpret_cast<uint2 *>(S + s_rec);
    unsigned *d_nrec = reinterpret_cast<unsigned *>(S + s_nrec);
    int *d_key = reinterpret_cast<int *>(S + s_key);
    unsigned *d_ch = reinterpret_cast<unsigned *>(S + s_ch);
    B2_CUDA(ctx, cudaMemsetAsync(d_ch, 0, 4ull * JUMP_ROUNDS, ctx->stream));

    B2_TRY(launch_gather(ctx, runs, A, o_file, file_off, d_stream));
    B2_KERNEL(ctx, "png_inflate_kernel");
    png_inflate_kernel<<<n, INF_T, 0, ctx->stream>>>(d_fd, d_stream, d_raw, d_rec, d_nrec, d_key);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "png_expand_kernel");
    png_expand_kernel<<<grid_for(ctx, (long long)raw_total), 256, 0, ctx->stream>>>(d_fd, d_fr, n, d_rec, d_nrec, d_src);
    B2_LAUNCH_CHECK(ctx);
    for (int r = 0; r < JUMP_ROUNDS; ++r) {
        B2_KERNEL(ctx, "png_jump_kernel");
        png_jump_kernel<<<grid_for(ctx, (long long)raw_total), 256, 0, ctx->stream>>>(d_src, raw_total, d_ch, r);
        B2_LAUNCH_CHECK(ctx);
    }
    B2_KERNEL(ctx, "png_resolve_kernel");
    png_resolve_kernel<<<grid_for(ctx, (long long)raw_total), 256, 0, ctx->stream>>>(d_raw, d_src, raw_total, d_flt);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "png_unfilter_kernel");
    png_unfilter_kernel<<<n_img, UNF_T, 0, ctx->stream>>>(reinterpret_cast<const PngImage *>(A + o_im), d_fd, d_flt, d_key);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "png_color_kernel");
    png_color_kernel<<<grid_for(ctx, (long long)file_px0.back()), 256, 0, ctx->stream>>>(
        d_fd, reinterpret_cast<const unsigned long long *>(A + o_fp), n, d_flt, d_key,
        reinterpret_cast<uint32_t *>(d_frames), d_status);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

}  // namespace
}  // namespace b200timg

using namespace b200timg;

extern "C" {

int b200timg_png_parse(const uint8_t *png, size_t size, b200timg_png_info *info) {
    if (!png || size == 0 || !info) return B200TIMG_EINVAL;
    Parse P;
    if (png_walk(png, size, P) != 0) return B200TIMG_EINVAL;
    fill_info(P, info);
    return B200TIMG_OK;
}

int b200timg_png_frames_dev(b200timg_ctx *ctx, int n_files, const uint8_t *const *files, const size_t *sizes,
                            uint8_t *d_frames, int32_t *d_status) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    B2_TRY(check_dev_outputs(ctx, "png", d_frames, d_status, "d_status"));
    std::vector<Parse> ps;
    B2_TRY(parse_files(ctx, "png", "chunk walk", png_walk, n_files, files, sizes, ps));
    return launch_png(ctx, n_files, files, sizes, ps, d_frames, d_status);
}

int b200timg_png_frames(b200timg_ctx *ctx, int n_files, const uint8_t *const *files, const size_t *sizes,
                        uint8_t *frames, int32_t *status) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!frames || !status) return ctx->fail(B200TIMG_EINVAL, "png: null output");
    std::vector<Parse> ps;
    B2_TRY(parse_files(ctx, "png", "chunk walk", png_walk, n_files, files, sizes, ps));
    size_t bytes = 0;
    for (const Parse &P : ps) bytes += (size_t)P.w * P.h * 4;
    return decode_to_host(ctx, bytes, n_files, frames, status, [&](uint8_t *d_frames, int32_t *d_status) {
        return launch_png(ctx, n_files, files, sizes, ps, d_frames, d_status);
    });
}

}  // extern "C"
