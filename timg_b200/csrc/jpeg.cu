// Baseline JPEGs on the device (SURVEY 8f rank 4): the RGBA buffer stbi__load_and_postprocess_8bit(.., 4) returns for
// the STB source's JPEG branch (src/stb-image-source.cc:141-157) on x86-64, where stbi__setup_jpeg picks the SSE2
// IDCT, colour conversion and hv_2 resampler (third_party/stb/stb_image.h:3822-3841).
//   host walk              stbi__decode_jpeg_header / stbi__decode_jpeg_image's marker walk, Huffman and quantisation
//                          tables as the scan sees them, and the scan's segments (restart intervals) as byte runs
//   decode_gather_kernel   (decode.cu) the runs of every segment into one destuffed byte stream per segment (FF 00
//                          and fill bytes dropped)
//   jpeg_sync_kernel       self-synchronising Huffman decode (Weissenberger & Schmidt): each thread decodes its
//                          64-byte subsequence from a guessed state until it passes the subsequence's end; a CTA
//                          iterates until every start state equals its predecessor's exit
//   jpeg_fixup_kernel      one CTA per segment walks the subsequences in order, re-decodes any whose start differs from
//                          its predecessor's exit (so correctness never depends on convergence) and scans the blocks
//                          each subsequence starts into its first block index
//   jpeg_decode_kernel     the final decode from the synchronised states: dequantised AC coefficients, DC differences,
//                          Huffman errors and the restart rule (:2970-2976, :3002-3006)
//   jpeg_dc_kernel         per segment and component: DC prediction, stbi__addints_valid / stbi__mul2shorts_valid,
//                          (short)(dc * dequant[0])
//   jpeg_idct_kernel       stbi__idct_simd's arithmetic (16-bit wrapping adds, saturating packs) into the component
//                          planes (stride w2)
//   jpeg_color_kernel      one thread per output pixel: load_jpeg_image's resampler state machine in closed form, then
//                          YCbCr (SSE2 for i < img_x & ~7, scalar for the tail), RGB, CMYK, YCCK or grey
// A call launches these seven kernels whatever its file count.
#include <algorithm>
#include <climits>

#include "decode.cuh"

namespace b200timg {

namespace {

constexpr int SUB_BYTES = 64;                      // subsequence length of the synchronising decoder
constexpr int SYNC_T = 128;                        // subsequences per sync CTA (one of them overlaps the previous CTA)
constexpr int FIX_T = 512;
constexpr int DC_T = 512;
constexpr unsigned long long NO_EVENT = ~0ull;

// ---- tables ------------------------------------------------------------------------------------------------------
struct Huff {                                      // stbi__huffman + its fast_ac table (AC tables)
    uint32_t maxcode[18];
    int delta[17];
    int16_t fast_ac[512];
    uint8_t fast[512];
    uint8_t size[257];
    uint8_t values[256];
    uint8_t pad_[7];
};

const uint8_t DEZIGZAG[79] = {0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48,
                              41, 34, 27, 20, 13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                              30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63,
                              63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63};
__constant__ uint8_t c_dezigzag[80] = {0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48,
                                      41, 34, 27, 20, 13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                      30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63,
                                      63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63};

// Inclusive sum over the N threads of a CTA through s[N]; s[N - 1] holds the total until the next call.
template <class T, int N>
__device__ __forceinline__ T block_incl_scan(T v, T *s) {
    const int t = threadIdx.x;
    s[t] = v;
    __syncthreads();
    for (int d = 1; d < N; d <<= 1) {
        const T a = t >= d ? s[t - d] : T(0);
        __syncthreads();
        s[t] += a;
        __syncthreads();
    }
    return s[t];
}

// stbi__build_huffman (:2004-2047) and stbi__build_fast_ac (:2051-2074); false where stb fails
bool build_huff(Huff &h, const int count[16], const uint8_t *vals, int n, bool ac) {
    memset(&h, 0, sizeof h);
    int k = 0;
    for (int i = 0; i < 16; ++i)
        for (int j = 0; j < count[i]; ++j) {
            h.size[k++] = (uint8_t)(i + 1);
            if (k >= 257) return false;
        }
    h.size[k] = 0;
    uint16_t code[257] = {};
    unsigned c = 0;
    k = 0;
    int j;
    for (j = 1; j <= 16; ++j) {
        h.delta[j] = k - (int)c;
        if (h.size[k] == j) {
            while (h.size[k] == j) code[k++] = (uint16_t)(c++);
            if (c - 1 >= (1u << j)) return false;
        }
        h.maxcode[j] = c << (16 - j);
        c <<= 1;
    }
    h.maxcode[j] = 0xffffffffu;
    memset(h.fast, 255, sizeof h.fast);
    for (int i = 0; i < k; ++i) {
        const int s = h.size[i];
        if (s <= 9) {
            const int cc = code[i] << (9 - s), m = 1 << (9 - s);
            for (int q = 0; q < m; ++q) h.fast[cc + q] = (uint8_t)i;
        }
    }
    for (int i = 0; i < n; ++i) h.values[i] = vals[i];
    if (ac)
        for (int i = 0; i < 512; ++i) {
            const uint8_t fast = h.fast[i];
            h.fast_ac[i] = 0;
            if (fast < 255) {
                const int rs = h.values[fast], run = (rs >> 4) & 15, magbits = rs & 15, len = h.size[fast];
                if (magbits && len + magbits <= 9) {
                    int kk = ((i << len) & 511) >> (9 - magbits);
                    const int m = 1 << (magbits - 1);
                    if (kk < m) kk += (int)(~0u << magbits) + 1;
                    if (kk >= -128 && kk <= 127) h.fast_ac[i] = (int16_t)((kk * 256) + (run * 16) + (len + magbits));
                }
            }
        }
    return true;
}

// ---- descriptors -------------------------------------------------------------------------------------------------
struct __align__(16) JpegFile {
    unsigned long long px0;                        // first pixel of the canvas in d_frames
    unsigned long long plane0[4];                  // component planes in the plane scratch
    unsigned long long unit0;                      // first block of the file in the coefficient scratch
    int w, h, ncomp, mode;                         // mode: 0 grey, 1 YCbCr, 2 RGB, 3 CMYK, 4 YCCK
    int cw2[4], cy[4], hs[4], vs[4];               // plane stride, component rows (img_comp.y), expansion factors
    int ch[4], cv[4];                              // sampling factors
    int upm, mcu_x, interleaved, bw;               // blocks per MCU, MCUs per row; non-interleaved: blocks per row
    int u_comp[64], u_dx[64], u_dy[64];            // block u of an MCU: component, block column / row inside the MCU
    int dc_tab[4], ac_tab[4];                      // per component: index into the call's Huffman tables
    uint16_t dq[4][64];                            // per component: its dequantisation table (row-major)
};

struct __align__(16) JpegSeg {
    unsigned long long data;                       // destuffed bytes in the stream scratch
    unsigned long long unit0;                      // first block of the segment inside its file
    unsigned L;                                    // destuffed length
    int marker;                                    // the marker that ends it (-1: end of file)
    int file, units, check;                        // check: stb's restart test runs after its last MCU
    unsigned sub0, nsub;                           // its subsequences in the flat list
};

// ---- host walk ---------------------------------------------------------------------------------------------------
struct Comp { int id, h, v, tq, hd, ha, x, y, w2, h2; };
struct Run { unsigned long long off, len; };
struct HostSeg { std::vector<Run> runs; unsigned long long L = 0; int marker = -1; };

struct Parse {
    int w = 0, h = 0, n = 0, hmax = 1, vmax = 1, mcu_x = 0, mcu_y = 0, progressive = 0, ri = 0;
    int jfif = 0, app14 = -1, rgb = 0, scan_n = 0, order[4] = {0, 0, 0, 0};
    Comp c[4] = {};
    uint16_t dq[4][64] = {};
    Huff dc[4], ac[4];
    bool dc_def[4] = {false, false, false, false}, ac_def[4] = {false, false, false, false};
    std::vector<HostSeg> segs;
    bool supported = false;
    char why[96] = {0};
};

struct Rd {                                        // stbi__get8 / get16be / skip: bytes past the end read as 0
    const uint8_t *p;
    size_t n, pos = 0;
    int get8() { const int v = pos < n ? p[pos] : 0; ++pos; return v; }
    int get16() { const int a = get8(); return (a << 8) | get8(); }
    bool eof() const { return pos >= n; }
    int marker() {                                 // stbi__get_marker without the cached marker
        int x = get8();
        if (x != 0xff) return 0xff;                // STBI__MARKER_none
        while (x == 0xff) { if (eof()) return 0; x = get8(); }
        return x;
    }
};
constexpr int M_NONE = 0xff;

// stbi__process_marker (:3100-3201): 0 fails
int process_marker(Rd &s, Parse &P, int m) {
    if (m == M_NONE) return 0;
    if (m == 0xDD) {
        if (s.get16() != 4) return 0;
        P.ri = s.get16();
        return 1;
    }
    if (m == 0xDB) {
        int L = s.get16() - 2;
        while (L > 0) {
            const int q = s.get8(), p = q >> 4, t = q & 15;
            if (p != 0 && p != 1) return 0;
            if (t > 3) return 0;
            for (int i = 0; i < 64; ++i) P.dq[t][DEZIGZAG[i]] = (uint16_t)(p ? s.get16() : s.get8());
            L -= p ? 129 : 65;
        }
        return L == 0;
    }
    if (m == 0xC4) {
        int L = s.get16() - 2;
        while (L > 0) {
            const int q = s.get8(), tc = q >> 4, th = q & 15;
            if (tc > 1 || th > 3) return 0;
            int sizes[16], n = 0;
            for (int i = 0; i < 16; ++i) { sizes[i] = s.get8(); n += sizes[i]; }
            if (n > 256) return 0;
            L -= 17;
            uint8_t v[256];
            Huff &hf = tc == 0 ? P.dc[th] : P.ac[th];
            // stb builds before reading the values; a failed build leaves the table half built, but the call fails
            for (int i = 0; i < n; ++i) v[i] = (uint8_t)s.get8();
            if (!build_huff(hf, sizes, v, n, tc != 0)) return 0;
            (tc == 0 ? P.dc_def : P.ac_def)[th] = true;
            L -= n;
        }
        return L == 0;
    }
    if ((m >= 0xE0 && m <= 0xEF) || m == 0xFE) {
        int L = s.get16();
        if (L < 2) return 0;
        L -= 2;
        if (m == 0xE0 && L >= 5) {
            const char tag[5] = {'J', 'F', 'I', 'F', 0};
            int ok = 1;
            for (int i = 0; i < 5; ++i) if (s.get8() != tag[i]) ok = 0;
            L -= 5;
            if (ok) P.jfif = 1;
        } else if (m == 0xEE && L >= 12) {
            const char tag[6] = {'A', 'd', 'o', 'b', 'e', 0};
            int ok = 1;
            for (int i = 0; i < 6; ++i) if (s.get8() != tag[i]) ok = 0;
            L -= 6;
            if (ok) { s.get8(); s.get16(); s.get16(); P.app14 = s.get8(); L -= 6; }
        }
        s.pos += (size_t)L;                        // stbi__skip with a negative L cannot happen: L >= 0 here
        return 1;
    }
    return 0;
}

// The entropy-coded bytes from s.pos to the first marker, as stb's grow reads them: runs of data bytes (FF 00 is a
// data FF, FF fill bytes are dropped, an FF run at the end of the file is a data FF), the marker, and s.pos after it.
void scan_segment(Rd &s, HostSeg &g) {
    size_t p = s.pos;
    auto add = [&](size_t a, size_t b) {
        if (b <= a) return;
        if (!g.runs.empty() && g.runs.back().off + g.runs.back().len == a) g.runs.back().len += b - a;
        else g.runs.push_back({a, b - a});
        g.L += b - a;
    };
    for (;;) {
        const uint8_t *q = p < s.n ? (const uint8_t *)memchr(s.p + p, 0xff, s.n - p) : nullptr;
        if (!q) { add(p, s.n); g.marker = -1; s.pos = s.n; return; }
        const size_t f = (size_t)(q - s.p);
        add(p, f);
        size_t i = f + 1;
        while (i < s.n && s.p[i] == 0xff) ++i;
        if (i >= s.n) { add(f, f + 1); g.marker = -1; s.pos = s.n; return; }
        if (s.p[i] == 0) { add(f, f + 1); p = i + 1; continue; }
        g.marker = s.p[i];
        s.pos = i + 1;
        return;
    }
}

// 0: parsed (P.supported says whether the device takes it); -1: stb's walk fails, so the source fails
int jpeg_walk(const uint8_t *d, size_t size, Parse &P) {
    Rd s{d, size};
    auto unsup = [&](const char *why) { P.supported = false; snprintf(P.why, sizeof P.why, "%s", why); return 0; };
    if (s.marker() != 0xD8) return -1;                                          // no SOI
    int m = s.marker();
    while (!(m == 0xC0 || m == 0xC1 || m == 0xC2)) {
        if (!process_marker(s, P, m)) return -1;
        m = s.marker();
        while (m == M_NONE) {
            if (s.eof()) return -1;                                             // no SOF
            m = s.marker();
        }
    }
    P.progressive = m == 0xC2;
    // stbi__process_frame_header (:3265-3355)
    const int Lf = s.get16();
    if (Lf < 11) return -1;
    if (s.get8() != 8) return -1;
    P.h = s.get16(); if (P.h == 0) return -1;
    P.w = s.get16(); if (P.w == 0) return -1;
    if (P.h > (1 << 24) || P.w > (1 << 24)) return -1;
    P.n = s.get8();
    if (P.n != 1 && P.n != 3 && P.n != 4) return -1;
    if (Lf != 8 + 3 * P.n) return -1;
    for (int i = 0; i < P.n; ++i) {
        Comp &c = P.c[i];
        c.id = s.get8();
        if (P.n == 3 && c.id == "RGB"[i]) ++P.rgb;
        const int q = s.get8();
        c.h = q >> 4; if (!c.h || c.h > 4) return -1;
        c.v = q & 15; if (!c.v || c.v > 4) return -1;
        c.tq = s.get8(); if (c.tq > 3) return -1;
    }
    if ((long long)P.w * P.h * P.n > INT_MAX) return -1;                        // stbi__mad3sizes_valid
    for (int i = 0; i < P.n; ++i) { P.hmax = std::max(P.hmax, P.c[i].h); P.vmax = std::max(P.vmax, P.c[i].v); }
    for (int i = 0; i < P.n; ++i)
        if (P.hmax % P.c[i].h || P.vmax % P.c[i].v) return -1;
    P.mcu_x = (P.w + P.hmax * 8 - 1) / (P.hmax * 8);
    P.mcu_y = (P.h + P.vmax * 8 - 1) / (P.vmax * 8);
    for (int i = 0; i < P.n; ++i) {
        Comp &c = P.c[i];
        c.x = (P.w * c.h + P.hmax - 1) / P.hmax;
        c.y = (P.h * c.v + P.vmax - 1) / P.vmax;
        c.w2 = P.mcu_x * c.h * 8;
        c.h2 = P.mcu_y * c.v * 8;
    }
    if (P.progressive) return unsup("progressive (SOF2)");
    // stbi__decode_jpeg_image (:3413-3448)
    bool scanned = false;
    m = s.marker();
    while (m != 0xD9) {
        if (m == 0xDA) {
            if (scanned) return unsup("more than one scan");
            const int Ls = s.get16();
            P.scan_n = s.get8();
            if (P.scan_n < 1 || P.scan_n > 4 || P.scan_n > P.n) return -1;
            if (Ls != 6 + 2 * P.scan_n) return -1;
            for (int i = 0; i < P.scan_n; ++i) {
                const int id = s.get8(), q = s.get8();
                int which = 0;
                while (which < P.n && P.c[which].id != id) ++which;
                if (which == P.n) return -1;
                P.c[which].hd = q >> 4; if (P.c[which].hd > 3) return -1;
                P.c[which].ha = q & 15; if (P.c[which].ha > 3) return -1;
                P.order[i] = which;
            }
            if (s.get8() != 0) return -1;                                       // spec_start
            s.get8();
            if (s.get8() != 0) return -1;                                       // succ_high / succ_low
            if (P.scan_n != P.n) return unsup("a scan without every component");
            for (int i = 0; i < P.scan_n; ++i) {
                for (int j = 0; j < i; ++j)
                    if (P.order[j] == P.order[i]) return unsup("a component twice in the scan");
                const Comp &c = P.c[P.order[i]];
                if (!P.dc_def[c.hd] || !P.ac_def[c.ha]) return unsup("a Huffman table the scan uses is not defined");
            }
            scanned = true;
            // the segments: one per restart interval, up to the first that does not end in RSTn
            const long long mcus = P.n == 1 ? (long long)((P.c[0].x + 7) >> 3) * ((P.c[0].y + 7) >> 3)
                                            : (long long)P.mcu_x * P.mcu_y;
            const long long nint = P.ri ? (mcus + P.ri - 1) / P.ri : 1;
            const bool full_last = P.ri && mcus % P.ri == 0;
            for (long long k = 0; k < nint; ++k) {
                P.segs.emplace_back();
                scan_segment(s, P.segs.back());
                const int mk = P.segs.back().marker;
                if (k + 1 < nint && !(mk >= 0xD0 && mk <= 0xD7)) { P.supported = true; return 0; }   // bails (-1) or fails first
            }
            // after the scan: the marker that ended it; an RSTn there is skipped as :3427-3433 and :3002-3006 do
            const int mk = P.segs.back().marker;
            if (mk < 0) m = M_NONE;
            else if (mk >= 0xD0 && mk <= 0xD7) {
                if (full_last) {                                                // reset, then stbi__skip_jpeg_junk_at_end
                    m = M_NONE;
                    while (!s.eof()) {
                        int x = s.get8();
                        bool found = false;
                        while (x == 0xff) {
                            if (s.eof()) break;
                            x = s.get8();
                            if (x != 0 && x != 0xff) { found = true; break; }
                        }
                        if (found) { m = x; break; }
                    }
                } else m = s.marker();
            } else m = mk;
            continue;
        } else if (m == 0xDC) {
            const int Ld = s.get16(), NL = s.get16();
            if (Ld != 4 || NL != P.h) return -1;
        } else if (!process_marker(s, P, m)) {
            break;                                                              // stb returns 1 here
        }
        m = s.marker();
    }
    if (!scanned) return unsup("no scan is decoded before the walk stops (uninitialised planes)");
    P.supported = true;
    return 0;
}

}  // namespace
}  // namespace b200timg

namespace b200timg {
namespace {

// ---- the device decoder: stb's bit reader and block decoder, restated ---------------------------------------------
// A state is (P, nomore, code_bits, u, z): P bits consumed, stb's nomore flag, code_bits bits buffered (stb's
// code_buffer holds stream bits P .. P + code_bits - 1, left aligned, where bytes from the segment's end on read as 0),
// block u of the MCU, next coefficient z (0: the block's DC).  The bytes fetched follow: F = L once nomore is set
// (the zero bytes grow appends after the marker move no stream position), else (P + code_bits) / 8.  So a state
// rebuilds stb's reader exactly, also past the marker.
__device__ __forceinline__ unsigned long long st_pack(unsigned long long P, bool nomore, int cb, int u, int z) {
    return (P << 20) | ((unsigned long long)nomore << 19) | ((unsigned)cb << 13) | ((unsigned)u << 7) | (unsigned)z;
}
__device__ __forceinline__ int st_u(unsigned long long s) { return (int)((s >> 7) & 63); }
__device__ __forceinline__ int st_z(unsigned long long s) { return (int)(s & 127); }

struct Dec {
    const uint8_t *d;
    unsigned L, F;
    int cb, marker_end;
    uint32_t buf;
    bool nomore;
    unsigned long long P;                           // bits consumed since the segment's start
    __device__ void init(const uint8_t *data, unsigned len, int mend, unsigned long long s) {
        d = data; L = len; marker_end = mend; nomore = false;
        P = s >> 20; nomore = (s >> 19) & 1; cb = (int)((s >> 13) & 63);
        F = nomore ? L : (unsigned)((P + (unsigned)cb) >> 3);
        const unsigned long long b0 = P >> 3;
        unsigned long long w = 0;                   // stream bytes b0 .. b0 + 4, big-endian
        for (int i = 0; i < 5; ++i) w = (w << 8) | (unsigned)(b0 + i < L ? d[b0 + i] : 0);
        const uint32_t top = (uint32_t)((w << (24 + (P & 7))) >> 32);
        buf = cb ? (top >> (32 - cb)) << (32 - cb) : 0u;
    }
    __device__ void grow() {                        // stbi__grow_buffer_unsafe
        do {
            unsigned b = 0;
            if (!nomore) {
                if (F >= L) {
                    if (marker_end) { nomore = true; return; }
                } else b = d[F];
                ++F;
            }
            buf |= b << (24 - cb);
            cb += 8;
        } while (cb <= 24);
    }
    __device__ void consume(int s) { buf <<= s; cb -= s; P += (unsigned)s; }
    __device__ int huff(const Huff &h) {            // stbi__jpeg_huff_decode
        if (cb < 16) grow();
        int k = h.fast[buf >> 23];
        if (k < 255) {
            const int s = h.size[k];
            if (s > cb) return -1;
            consume(s);
            return h.values[k];
        }
        const uint32_t temp = buf >> 16;
        for (k = 10;; ++k)
            if (temp < h.maxcode[k]) break;
        if (k == 17) return -1;
        if (k > cb) return -1;
        const int c = (int)((buf >> (32 - k)) & ((1u << k) - 1)) + h.delta[k];
        if (c < 0 || c >= 256) return -1;
        consume(k);
        return h.values[c];
    }
    __device__ int extend(int n) {                  // stbi__extend_receive, n in 1..15
        if (cb < n) grow();
        if (cb < n) return 0;
        const int sgn = (int)(buf >> 31);
        uint32_t k = (buf << n) | (buf >> (32 - n));
        const uint32_t m = (1u << n) - 1;
        buf = k & ~m;
        k &= m;
        cb -= n; P += (unsigned)n;
        return (int)k + ((int)((~0u << n) + 1) & (sgn - 1));
    }
};

// One step of stbi__jpeg_decode_block from (u, z): the DC (z == 0) or one AC symbol.  Returns 0, 1 at the block's end,
// -1 for a DC Huffman error, -2 for an AC one.  Writes only when blk is not null.
template <bool WRITE>
__device__ __forceinline__ int dec_step(Dec &D, const JpegFile &f, const Huff *__restrict__ tabs, int &u, int &z,
                                        int16_t *blk, int *dcdiff) {
    const int c = f.u_comp[u];
    if (z == 0) {
        if (D.cb < 16) D.grow();
        const int t = D.huff(tabs[f.dc_tab[c]]);
        if (t < 0 || t > 15) return -1;
        const int diff = t ? D.extend(t) : 0;
        if (WRITE) *dcdiff = diff;
        z = 1;
        return 0;
    }
    const Huff &h = tabs[f.ac_tab[c]];
    int k = z;
    if (D.cb < 16) D.grow();
    const int r = h.fast_ac[D.buf >> 23];
    if (r) {
        k += (r >> 4) & 15;
        const int s = r & 15;
        if (s > D.cb) return -2;
        D.consume(s);
        const int zig = c_dezigzag[k++];
        if (WRITE) blk[zig] = (int16_t)((r >> 8) * f.dq[c][zig]);
    } else {
        const int rs = D.huff(h);
        if (rs < 0) return -2;
        const int s = rs & 15, rr = rs >> 4;
        if (s == 0) {
            if (rs != 0xf0) { z = 0; return 1; }
            k += 16;
        } else {
            k += rr;
            const int zig = c_dezigzag[k++];
            const int v = D.extend(s);
            if (WRITE) blk[zig] = (int16_t)(v * f.dq[c][zig]);
        }
    }
    if (k >= 64) { z = 0; return 1; }
    z = k;
    return 0;
}

// Off the true path an invalid code is not an error: end the block and move one bit on, so every walk makes progress.
__device__ __forceinline__ void dec_recover(Dec &D, int &z) {
    z = 0;
    if (D.cb < 1) D.grow();
    if (D.cb < 1) D.grow();
    if (D.cb >= 1) D.consume(1);
}

__device__ __forceinline__ void next_block(const JpegFile &f, int &u) { if (++u == f.upm) u = 0; }

// Walk from s until the first symbol boundary at or past bit `end`: the exit state and the blocks whose DC was read.
__device__ unsigned long long dec_walk(const JpegFile &f, const JpegSeg &g, const uint8_t *stream, const Huff *tabs,
                                       unsigned long long s, unsigned long long end, unsigned &count) {
    Dec D;
    D.init(stream + g.data, g.L, g.marker >= 0, s);
    int u = st_u(s), z = st_z(s);
    unsigned n = 0;
    while (D.P < end) {
        if (z == 0) ++n;
        const int r = dec_step<false>(D, f, tabs, u, z, nullptr, nullptr);
        if (r == 1) next_block(f, u);
        else if (r < 0) { dec_recover(D, z); next_block(f, u); }
    }
    count = n;
    return st_pack(D.P, D.nomore, D.cb, u, z);
}

__device__ __forceinline__ unsigned long long sub_end(const JpegSeg &g, unsigned k) {
    return 8ull * SUB_BYTES * (k - g.sub0 + 1);
}

// ---- kernels -----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SYNC_T)
jpeg_sync_kernel(const JpegFile *__restrict__ fd, const JpegSeg *__restrict__ sd, const unsigned *__restrict__ seg_sub,
                 int n_seg, const Huff *__restrict__ tabs, const uint8_t *__restrict__ stream, unsigned n_sub,
                 unsigned long long *__restrict__ st, unsigned long long *__restrict__ ex, unsigned *__restrict__ cnt) {
    __shared__ unsigned long long s_ex[SYNC_T];
    const int t = threadIdx.x;
    const long long k = (long long)blockIdx.x * (SYNC_T - 1) + t - 1;
    const bool valid = k >= 0 && k < (long long)n_sub;
    int si = 0;
    bool first = true, last = true;
    unsigned long long start = 0, exit_ = 0, end = 0;
    unsigned count = 0;
    if (valid) {
        si = mixed_owner(seg_sub, n_seg, (unsigned)k);
        const JpegSeg &g = sd[si];
        first = (unsigned)k == g.sub0;
        last = (unsigned)k == g.sub0 + g.nsub - 1;
        start = first ? 0ull : st_pack(8ull * SUB_BYTES * (unsigned long long)(k - g.sub0), false, 0, 0, 0);
        end = sub_end(g, (unsigned)k);
    }
    bool dirty = true;
    for (int round = 0; round <= SYNC_T; ++round) {
        if (valid && !last && dirty) {
            const JpegSeg &g = sd[si];
            exit_ = dec_walk(fd[g.file], g, stream, tabs, start, end, count);
        }
        dirty = false;
        s_ex[t] = exit_;
        __syncthreads();
        if (t > 0 && valid && !first) {
            const unsigned long long prev = s_ex[t - 1];
            if (prev != start) { start = prev; dirty = true; }
        }
        if (!__syncthreads_or(dirty)) break;
    }
    if (valid && (t > 0 || k == 0)) { st[k] = start; ex[k] = exit_; cnt[k] = last ? 0u : count; }
}

// One CTA per segment: make every start state its predecessor's exit, in order, then scan the block counts.
__global__ void __launch_bounds__(FIX_T)
jpeg_fixup_kernel(const JpegFile *__restrict__ fd, const JpegSeg *__restrict__ sd, const Huff *__restrict__ tabs,
                  const uint8_t *__restrict__ stream, unsigned long long *__restrict__ st, unsigned long long *__restrict__ ex,
                  unsigned *__restrict__ cnt, unsigned *__restrict__ ustart) {
    __shared__ unsigned s_scan[FIX_T];
    __shared__ unsigned s_first;
    const JpegSeg g = sd[blockIdx.x];
    const JpegFile &f = fd[g.file];
    const unsigned e = g.sub0 + g.nsub;
    unsigned carry = 0;
    for (unsigned b = g.sub0; b < e; b += FIX_T) {
        const unsigned k = b + threadIdx.x;
        for (;;) {
            if (threadIdx.x == 0) s_first = UINT_MAX;
            __syncthreads();
            if (k < e && k > g.sub0 && st[k] != ex[k - 1]) atomicMin(&s_first, k);
            __syncthreads();
            const unsigned m = s_first;
            if (m == UINT_MAX) break;
            if (threadIdx.x == 0) {
                for (unsigned j = m; j < e; ++j) {
                    if (j > m && st[j] == ex[j - 1]) break;
                    st[j] = ex[j - 1];
                    if (j == e - 1) break;
                    unsigned c;
                    ex[j] = dec_walk(f, g, stream, tabs, st[j], sub_end(g, j), c);
                    cnt[j] = c;
                }
            }
            __syncthreads();
        }
        const unsigned v = k < e ? cnt[k] : 0u;
        const unsigned incl = block_incl_scan<unsigned, FIX_T>(v, s_scan);
        if (k < e) ustart[k] = carry + incl - v;
        carry += s_scan[FIX_T - 1];
        __syncthreads();
    }
}

// The final decode: each subsequence writes the blocks whose DC it reads (a block begun before its start belongs to
// the previous one).  Errors and the restart rule lower the file's event key: block * 4 + {0 DC code, 2 AC code,
// 3 restart bail}; jpeg_dc_kernel adds 1 (DC overflow).
__global__ void __launch_bounds__(128)
jpeg_decode_kernel(const JpegFile *__restrict__ fd, const JpegSeg *__restrict__ sd, const unsigned *__restrict__ seg_sub,
                   int n_seg, const Huff *__restrict__ tabs, const uint8_t *__restrict__ stream, unsigned n_sub,
                   const unsigned long long *__restrict__ st, const unsigned *__restrict__ ustart,
                   int16_t *__restrict__ coef, int *__restrict__ dcdiff, unsigned long long *__restrict__ key) {
    const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_sub) return;
    const int si = mixed_owner(seg_sub, n_seg, k);
    const JpegSeg &g = sd[si];
    const JpegFile &f = fd[g.file];
    const bool last = k == g.sub0 + g.nsub - 1;
    const unsigned long long end = sub_end(g, k), s = st[k];
    Dec D;
    D.init(stream + g.data, g.L, g.marker >= 0, s);
    int u = st_u(s), z = st_z(s);
    while (z != 0) {                                // the tail of a block the previous subsequence owns
        const int r = dec_step<false>(D, f, tabs, u, z, nullptr, nullptr);
        if (r < 0) return;
        if (r == 1) next_block(f, u);
    }
    for (unsigned unit = ustart[k]; (int)unit < g.units && (last || D.P < end); ++unit) {
        const unsigned long long gb = g.unit0 + unit;        // block index inside the file
        int16_t *blk = coef + (f.unit0 + gb) * 64;
        int4 *b4 = reinterpret_cast<int4 *>(blk);
        for (int i = 0; i < 8; ++i) b4[i] = make_int4(0, 0, 0, 0);
        int *dd = dcdiff + f.unit0 + gb;
        int r;
        do r = dec_step<true>(D, f, tabs, u, z, blk, dd); while (r == 0);
        if (r < 0) { atomicMin(key + g.file, gb * 4 + (r == -1 ? 0 : 2)); return; }
        next_block(f, u);
        if (g.check && (int)unit == g.units - 1) {  // todo reached 0: the restart test
            if (D.cb < 24) D.grow();
            if (!(D.nomore && g.marker >= 0xD0 && g.marker <= 0xD7)) atomicMin(key + g.file, gb * 4 + 3);
        }
    }
}

__device__ __forceinline__ bool mul2shorts_valid(int a, int b) {
    if (b == 0 || b == -1) return true;
    if ((a >= 0) == (b >= 0)) return a <= SHRT_MAX / b;
    if (b < 0) return a <= SHRT_MIN / b;
    return a >= SHRT_MIN / b;
}

// One CTA per segment: DC prediction per component (reset at every restart), stb's two checks, data[0].
__global__ void __launch_bounds__(DC_T)
jpeg_dc_kernel(const JpegFile *__restrict__ fd, const JpegSeg *__restrict__ sd, const int *__restrict__ dcdiff,
               int16_t *__restrict__ coef, unsigned long long *__restrict__ key) {
    __shared__ long long s_scan[DC_T];
    const JpegSeg g = sd[blockIdx.x];
    const JpegFile &f = fd[g.file];
    long long carry[4] = {0, 0, 0, 0};
    for (int b = 0; b < g.units; b += DC_T) {
        const int unit = b + threadIdx.x;
        const bool in = unit < g.units;
        const unsigned long long gb = g.unit0 + (unsigned)unit;
        const int c = in ? f.u_comp[gb % (unsigned)f.upm] : -1;
        const long long diff = in ? dcdiff[f.unit0 + gb] : 0;
        long long mine = 0;
        for (int q = 0; q < f.ncomp; ++q) {
            const long long incl = block_incl_scan<long long, DC_T>(c == q ? diff : 0ll, s_scan);
            if (c == q) mine = carry[q] + incl;
            carry[q] += s_scan[DC_T - 1];
            __syncthreads();
        }
        if (in) {
            const int dq0 = f.dq[c][0];
            if (mine < INT_MIN || mine > INT_MAX || !mul2shorts_valid((int)mine, dq0))
                atomicMin(key + g.file, gb * 4 + 1);
            else
                coef[(f.unit0 + gb) * 64] = (int16_t)((int)mine * dq0);
        }
    }
}

// stbi__idct_simd (:2533-2700): 16-bit wrapping adds of the inputs, 32-bit products and sums, saturating packs.
__device__ __forceinline__ void idct_pass(int r[8], int bias, int shift) {
    auto w16 = [](int v) { return (int)(int16_t)v; };
    auto sat = [](int v) { return v < -32768 ? -32768 : v > 32767 ? 32767 : v; };
    const int A = (int)(0.5411961f * 4096 + 0.5), B = (int)(-1.847759065f * 4096 + 0.5), Cc = (int)(0.765366865f * 4096 + 0.5);
    const int Dd = (int)(-1.961570560f * 4096 + 0.5), E = (int)(0.298631336f * 4096 + 0.5), Ff = (int)(3.072711026f * 4096 + 0.5);
    const int G = (int)(-0.390180644f * 4096 + 0.5), H = (int)(2.053119869f * 4096 + 0.5), I = (int)(1.501321110f * 4096 + 0.5);
    const int J = (int)(1.175875602f * 4096 + 0.5), K = (int)(-0.899976223f * 4096 + 0.5), Lc = (int)(-2.562915447f * 4096 + 0.5);
    const int t2e = r[2] * A + r[6] * (A + B), t3e = r[2] * (A + Cc) + r[6] * A;
    const int t0e = w16(r[0] + r[4]) * 4096, t1e = w16(r[0] - r[4]) * 4096;
    const int x0 = t0e + t3e, x3 = t0e - t3e, x1 = t1e + t2e, x2 = t1e - t2e;
    const int y0o = r[7] * (Dd + E) + r[3] * Dd, y2o = r[7] * Dd + r[3] * (Dd + Ff);
    const int y1o = r[5] * (G + H) + r[1] * G, y3o = r[5] * G + r[1] * (G + I);
    const int s17 = w16(r[1] + r[7]), s35 = w16(r[3] + r[5]);
    const int y4o = s17 * (J + K) + s35 * J, y5o = s17 * J + s35 * (J + Lc);
    const int x4 = y0o + y4o, x5 = y1o + y5o, x6 = y2o + y5o, x7 = y3o + y4o;
    r[0] = sat((x0 + bias + x7) >> shift); r[7] = sat((x0 + bias - x7) >> shift);
    r[1] = sat((x1 + bias + x6) >> shift); r[6] = sat((x1 + bias - x6) >> shift);
    r[2] = sat((x2 + bias + x5) >> shift); r[5] = sat((x2 + bias - x5) >> shift);
    r[3] = sat((x3 + bias + x4) >> shift); r[4] = sat((x3 + bias - x4) >> shift);
}

__global__ void __launch_bounds__(128)
jpeg_idct_kernel(const JpegFile *__restrict__ fd, const unsigned long long *__restrict__ file_unit0, int n_files,
                 const int16_t *__restrict__ coef, uint8_t *__restrict__ planes) {
    const unsigned long long total = file_unit0[n_files];
    for (unsigned long long gu = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; gu < total;
         gu += (unsigned long long)gridDim.x * blockDim.x) {
        const int fi = mixed_owner(file_unit0, n_files, gu);
        const JpegFile &f = fd[fi];
        const unsigned long long b = gu - f.unit0;
        int c, x2, y2;
        if (f.interleaved) {
            const unsigned long long mcu = b / (unsigned)f.upm;
            const int u = (int)(b - mcu * (unsigned)f.upm);
            c = f.u_comp[u];
            const int mx = (int)(mcu % (unsigned)f.mcu_x), my = (int)(mcu / (unsigned)f.mcu_x);
            x2 = (mx * f.ch[c] + f.u_dx[u]) * 8;
            y2 = (my * f.cv[c] + f.u_dy[u]) * 8;
        } else {
            c = f.u_comp[0];
            x2 = (int)(b % (unsigned)f.bw) * 8;
            y2 = (int)(b / (unsigned)f.bw) * 8;
        }
        const int4 *src = reinterpret_cast<const int4 *>(coef + gu * 64);
        int v[64];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int4 q = src[i];
            const int w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) { v[i * 8 + j * 2] = (int16_t)(w[j] & 0xffff); v[i * 8 + j * 2 + 1] = (int16_t)((unsigned)w[j] >> 16); }
        }
#pragma unroll
        for (int col = 0; col < 8; ++col) {                        // column pass
            int r[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) r[i] = v[i * 8 + col];
            idct_pass(r, 512, 10);
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i * 8 + col] = r[i];
        }
        uint8_t *o = planes + f.plane0[c] + (size_t)y2 * f.cw2[c] + x2;
#pragma unroll
        for (int row = 0; row < 8; ++row) {                        // row pass, packus
            int r[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) r[i] = v[row * 8 + i];
            idct_pass(r, 65536 + (128 << 17), 17);
            uint32_t lo = 0, hi = 0;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                lo |= (uint32_t)min(max(r[i], 0), 255) << (8 * i);
                hi |= (uint32_t)min(max(r[i + 4], 0), 255) << (8 * i);
            }
            *reinterpret_cast<uint2 *>(o + (size_t)row * f.cw2[c]) = make_uint2(lo, hi);
        }
    }
}

// One component sample at output (x, y): load_jpeg_image's resampler (:3900-3942) in closed form.
__device__ __forceinline__ int sample(const JpegFile &f, const uint8_t *__restrict__ planes, int k, int x, int y) {
    const int hs = f.hs[k], vs = f.vs[k], cy = f.cy[k], stride = f.cw2[k];
    const int t = y + (vs >> 1), q = t / vs, ystep = t - q * vs;
    const int line1 = min(q, cy - 1), line0 = min(max(q - 1, 0), cy - 1);
    const bool bot = ystep >= (vs >> 1);
    const uint8_t *N = planes + f.plane0[k] + (size_t)(bot ? line1 : line0) * stride;
    const uint8_t *Fr = planes + f.plane0[k] + (size_t)(bot ? line0 : line1) * stride;
    const int wl = (f.w + hs - 1) / hs;
    if (hs == 1 && vs == 1) return N[x];
    if (hs == 1 && vs == 2) return (3 * N[x] + Fr[x] + 2) >> 2;
    if (hs == 2 && vs == 1) {                       // stbi__resample_row_h_2
        if (wl == 1) return N[0];
        if (x == 0) return N[0];
        if (x == 1) return (3 * N[0] + N[1] + 2) >> 2;
        const int i = x >> 1;
        if (i == wl - 1) return (x & 1) ? N[wl - 1] : (3 * N[wl - 2] + N[wl - 1] + 2) >> 2;
        return (x & 1) ? (3 * N[i] + N[i + 1] + 2) >> 2 : (3 * N[i] + N[i - 1] + 2) >> 2;
    }
    if (hs == 2 && vs == 2) {                       // stbi__resample_row_hv_2_simd: its vector part and tail agree
        auto T = [&](int i) { return 3 * N[i] + Fr[i]; };
        if (wl == 1 || x == 0) return (T(0) + 2) >> 2;
        if (x == 2 * wl - 1) return (T(wl - 1) + 2) >> 2;
        const int i = x >> 1;
        return (x & 1) ? (3 * T(i) + T(i + 1) + 8) >> 4 : (3 * T(i) + T(i - 1) + 8) >> 4;
    }
    return N[x / hs];                               // stbi__resample_row_generic
}

__device__ __forceinline__ int blinn(int x, int y) { const unsigned t = (unsigned)(x * y + 128); return (int)((t + (t >> 8)) >> 8); }
__device__ __forceinline__ int clamp255(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }

// stbi__YCbCr_to_RGB_simd: SSE2 arithmetic for x < (img_x & ~7), the scalar fixed-point formula after
__device__ __forceinline__ void ycc(int x, int w, int Y, int Cb, int Cr, int &r, int &g, int &b) {
    if (x < (w & ~7)) {
        const int cr0c = (short)(1.40200f * 4096.0f + 0.5f), cr1c = -(short)(0.71414f * 4096.0f + 0.5f);
        const int cb0c = -(short)(0.34414f * 4096.0f + 0.5f), cb1c = (short)(1.77200f * 4096.0f + 0.5f);
        auto w16 = [](int v) { return (int)(int16_t)v; };
        const int yws = Y * 16 + 8, crw = w16((Cr - 128) * 256), cbw = w16((Cb - 128) * 256);
        const int cr0 = (cr0c * crw) >> 16, cb0 = (cb0c * cbw) >> 16, cb1 = (cbw * cb1c) >> 16, cr1 = (crw * cr1c) >> 16;
        const int rws = w16(cr0 + yws), gws = w16(w16(cb0 + yws) + cr1), bws = w16(yws + cb1);
        r = clamp255(rws >> 4); g = clamp255(gws >> 4); b = clamp255(bws >> 4);
    } else {
        const int yf = (Y << 20) + (1 << 19), cr = Cr - 128, cb = Cb - 128;
        const int k0 = ((int)(1.40200f * 4096.0f + 0.5f)) << 8, k1 = ((int)(0.71414f * 4096.0f + 0.5f)) << 8;
        const int k2 = ((int)(0.34414f * 4096.0f + 0.5f)) << 8, k3 = ((int)(1.77200f * 4096.0f + 0.5f)) << 8;
        r = clamp255((yf + cr * k0) >> 20);
        g = clamp255((int)(yf + cr * -k1 + (int)((unsigned)(cb * -k2) & 0xffff0000u)) >> 20);
        b = clamp255((yf + cb * k3) >> 20);
    }
}

__global__ void __launch_bounds__(256)
jpeg_color_kernel(const JpegFile *__restrict__ fd, const unsigned long long *__restrict__ file_px0, int n_files,
                  const uint8_t *__restrict__ planes, const unsigned long long *__restrict__ key, uint32_t *__restrict__ out,
                  int32_t *__restrict__ status) {
    const unsigned long long total = file_px0[n_files];
    for (unsigned long long p = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; p < total;
         p += (unsigned long long)gridDim.x * blockDim.x) {
        const int fi = mixed_owner(file_px0, n_files, p);
        const JpegFile &f = fd[fi];
        const unsigned long long o = p - f.px0;
        const int y = (int)(o / (unsigned)f.w), x = (int)(o - (unsigned long long)y * (unsigned)f.w);
        if (o == 0) {
            const unsigned long long e = key[fi];
            status[fi] = e == NO_EVENT ? 1 : (e & 3) == 3 ? -1 : 0;
        }
        const int s0 = sample(f, planes, 0, x, y);
        int r, g, b;
        if (f.mode == 0) { r = g = b = s0; }
        else {
            const int s1 = sample(f, planes, 1, x, y), s2 = sample(f, planes, 2, x, y);
            if (f.mode == 2) { r = s0; g = s1; b = s2; }
            else if (f.mode == 3) {
                const int m = sample(f, planes, 3, x, y);
                r = blinn(s0, m); g = blinn(s1, m); b = blinn(s2, m);
            } else {
                ycc(x, f.w, s0, s1, s2, r, g, b);
                if (f.mode == 4) {
                    const int m = sample(f, planes, 3, x, y);
                    r = blinn(255 - r, m); g = blinn(255 - g, m); b = blinn(255 - b, m);
                }
            }
        }
        out[p] = pack_rgba((uint32_t)r, (uint32_t)g, (uint32_t)b, 255u);
    }
}

}  // namespace
}  // namespace b200timg

namespace b200timg {
namespace {

void fill_info(const Parse &P, b200timg_jpeg_info *info) {
    memset(info, 0, sizeof *info);
    info->w = P.w; info->h = P.h; info->n_comp = P.n;
    for (int i = 0; i < P.n; ++i) { info->h_samp[i] = P.c[i].h; info->v_samp[i] = P.c[i].v; }
    info->restart_interval = P.ri;
    info->progressive = P.progressive;
    info->supported = P.supported ? 1 : 0;
    snprintf(info->reason, sizeof info->reason, "%s", P.supported ? "" : P.why);
}

// Device scratch of one call (ctx->jpeg_up.arena + ctx->jpeg_scratch): the files + descriptors + deduplicated Huffman
// tables (2.4 KB each) + 16 bytes per byte run; destuffed streams, 20 bytes per 64-byte subsequence, 132 bytes per
// 8x8 block (coefficients and DC difference), the component planes (sum of w2 * h2), 8 bytes per file.
int launch_jpeg(b200timg_ctx *ctx, int n, const uint8_t *const *files, const size_t *sizes, const std::vector<Parse> &ps,
                uint8_t *d_frames, int32_t *d_status) {
    std::vector<JpegFile> fdesc((size_t)n);
    std::vector<JpegSeg> sdesc;
    std::vector<Huff> tabs;
    Runs runs;
    std::vector<unsigned long long> file_unit0(1, 0), file_px0(1, 0);
    std::vector<unsigned> seg_sub(1, 0);
    unsigned long long plane = 0, file_off = 0, stream = 0;
    unsigned nsub = 0;
    auto tab_index = [&](const Huff &h) {
        for (size_t i = 0; i < tabs.size(); ++i)
            if (!memcmp(&tabs[i], &h, sizeof h)) return (int)i;
        tabs.push_back(h);
        return (int)tabs.size() - 1;
    };
    for (int fi = 0; fi < n; ++fi) {
        const Parse &P = ps[(size_t)fi];
        JpegFile &F = fdesc[(size_t)fi];
        memset(&F, 0, sizeof F);
        F.px0 = file_px0.back();
        file_px0.push_back(F.px0 + (unsigned long long)P.w * P.h);
        F.w = P.w; F.h = P.h; F.ncomp = P.n;
        const bool is_rgb = P.n == 3 && (P.rgb == 3 || (P.app14 == 0 && !P.jfif));
        F.mode = P.n == 1 ? 0 : P.n == 3 ? (is_rgb ? 2 : 1) : P.app14 == 0 ? 3 : P.app14 == 2 ? 4 : 1;
        for (int c = 0; c < P.n; ++c) {
            const Comp &C = P.c[c];
            F.plane0[c] = plane; plane += ((unsigned long long)C.w2 * C.h2 + 15) / 16 * 16;
            F.cw2[c] = C.w2; F.cy[c] = C.y; F.hs[c] = P.hmax / C.h; F.vs[c] = P.vmax / C.v;
            F.ch[c] = C.h; F.cv[c] = C.v;
            F.dc_tab[c] = tab_index(P.dc[C.hd]);
            F.ac_tab[c] = tab_index(P.ac[C.ha]);
            memcpy(F.dq[c], P.dq[C.tq], sizeof F.dq[c]);
        }
        long long mcus;
        if (P.n == 1) {
            F.interleaved = 0; F.upm = 1; F.u_comp[0] = 0;
            F.bw = (P.c[0].x + 7) >> 3;
            mcus = (long long)F.bw * ((P.c[0].y + 7) >> 3);
        } else {
            F.interleaved = 1; F.mcu_x = P.mcu_x;
            int u = 0;
            for (int k = 0; k < P.scan_n; ++k) {
                const int c = P.order[k];
                for (int y = 0; y < P.c[c].v; ++y)
                    for (int x = 0; x < P.c[c].h; ++x) { F.u_comp[u] = c; F.u_dx[u] = x; F.u_dy[u] = y; ++u; }
            }
            F.upm = u;
            mcus = (long long)P.mcu_x * P.mcu_y;
        }
        F.unit0 = file_unit0.back();
        file_unit0.push_back(F.unit0 + (unsigned long long)mcus * F.upm);
        const long long ri = P.ri ? P.ri : mcus;
        const long long nint = P.ri ? (mcus + P.ri - 1) / P.ri : 1;
        for (size_t s = 0; s < P.segs.size(); ++s) {
            const HostSeg &hs = P.segs[s];
            JpegSeg g;
            memset(&g, 0, sizeof g);
            g.data = stream; g.L = (unsigned)hs.L; g.marker = hs.marker; g.file = fi;
            const long long m0 = (long long)s * ri, m1 = std::min(mcus, m0 + ri);
            g.unit0 = (unsigned long long)m0 * F.upm;
            g.units = (int)((m1 - m0) * F.upm);
            g.check = P.ri && (long long)s + 1 < nint;
            g.sub0 = nsub;
            g.nsub = (unsigned)std::max<unsigned long long>(1, (hs.L + SUB_BYTES - 1) / SUB_BYTES);
            nsub += g.nsub;
            seg_sub.push_back(nsub);
            for (const Run &r : hs.runs) runs.add(file_off + r.off, r.len);
            stream += hs.L;
            sdesc.push_back(g);
        }
        file_off += sizes[fi];
    }
    seg_sub.pop_back();
    const int n_seg = (int)sdesc.size();
    const unsigned long long units = file_unit0.back();
    if (units > (1ull << 31)) return ctx->fail(B200TIMG_EINVAL, "jpeg: %llu blocks in one call (at most 2^31)", units);

    std::vector<char> arena;
    const size_t o_fd = mixed_put(arena, fdesc.data(), sizeof(JpegFile) * fdesc.size());
    const size_t o_sd = mixed_put(arena, sdesc.data(), sizeof(JpegSeg) * sdesc.size());
    const size_t o_tab = mixed_put(arena, tabs.data(), sizeof(Huff) * tabs.size());
    const size_t o_ss = mixed_put(arena, seg_sub.data(), sizeof(unsigned) * seg_sub.size());
    runs.put(arena);
    const size_t o_fu = mixed_put(arena, file_unit0.data(), sizeof(unsigned long long) * file_unit0.size());
    const size_t o_fp = mixed_put(arena, file_px0.data(), sizeof(unsigned long long) * file_px0.size());
    size_t o_file;
    B2_TRY(staged_upload(ctx, ctx->jpeg_up, arena, n, files, sizes, &o_file));
    auto al = [](unsigned long long v) { return (v + 255) / 256 * 256; };
    const size_t s_stream = 0, s_st = al(stream), s_ex = s_st + al(8ull * nsub), s_cnt = s_ex + al(8ull * nsub),
                 s_us = s_cnt + al(4ull * nsub), s_coef = s_us + al(4ull * nsub), s_dc = s_coef + al(128ull * units),
                 s_plane = s_dc + al(4ull * units), s_key = s_plane + al(plane), s_end = s_key + al(8ull * n);
    B2_CUDA(ctx, ctx->jpeg_scratch.reserve(s_end));
    const char *A = ctx->jpeg_up.arena.as<char>();
    char *S = ctx->jpeg_scratch.as<char>();
    const JpegFile *d_fd = reinterpret_cast<const JpegFile *>(A + o_fd);
    const JpegSeg *d_sd = reinterpret_cast<const JpegSeg *>(A + o_sd);
    const Huff *d_tab = reinterpret_cast<const Huff *>(A + o_tab);
    const unsigned *d_ss = reinterpret_cast<const unsigned *>(A + o_ss);
    const uint8_t *d_stream = reinterpret_cast<const uint8_t *>(S + s_stream);
    unsigned long long *d_st = reinterpret_cast<unsigned long long *>(S + s_st);
    unsigned long long *d_ex = reinterpret_cast<unsigned long long *>(S + s_ex);
    unsigned *d_cnt = reinterpret_cast<unsigned *>(S + s_cnt);
    unsigned *d_us = reinterpret_cast<unsigned *>(S + s_us);
    int16_t *d_coef = reinterpret_cast<int16_t *>(S + s_coef);
    int *d_dc = reinterpret_cast<int *>(S + s_dc);
    uint8_t *d_plane = reinterpret_cast<uint8_t *>(S + s_plane);
    unsigned long long *d_key = reinterpret_cast<unsigned long long *>(S + s_key);
    B2_CUDA(ctx, cudaMemsetAsync(d_key, 0xff, 8ull * n, ctx->stream));

    B2_TRY(launch_gather(ctx, runs, A, o_file, file_off, reinterpret_cast<uint8_t *>(S + s_stream)));
    B2_KERNEL(ctx, "jpeg_sync_kernel");
    jpeg_sync_kernel<<<(nsub + SYNC_T - 2) / (SYNC_T - 1), SYNC_T, 0, ctx->stream>>>(d_fd, d_sd, d_ss, n_seg, d_tab, d_stream,
                                                                                   nsub, d_st, d_ex, d_cnt);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "jpeg_fixup_kernel");
    jpeg_fixup_kernel<<<n_seg, FIX_T, 0, ctx->stream>>>(d_fd, d_sd, d_tab, d_stream, d_st, d_ex, d_cnt, d_us);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "jpeg_decode_kernel");
    jpeg_decode_kernel<<<(nsub + 127) / 128, 128, 0, ctx->stream>>>(d_fd, d_sd, d_ss, n_seg, d_tab, d_stream, nsub, d_st,
                                                                    d_us, d_coef, d_dc, d_key);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "jpeg_dc_kernel");
    jpeg_dc_kernel<<<n_seg, DC_T, 0, ctx->stream>>>(d_fd, d_sd, d_dc, d_coef, d_key);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "jpeg_idct_kernel");
    jpeg_idct_kernel<<<grid_for(ctx, (long long)units, 128), 128, 0, ctx->stream>>>(
        d_fd, reinterpret_cast<const unsigned long long *>(A + o_fu), n, d_coef, d_plane);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "jpeg_color_kernel");
    jpeg_color_kernel<<<grid_for(ctx, (long long)file_px0.back()), 256, 0, ctx->stream>>>(
        d_fd, reinterpret_cast<const unsigned long long *>(A + o_fp), n, d_plane, d_key,
        reinterpret_cast<uint32_t *>(d_frames), d_status);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

}  // namespace
}  // namespace b200timg

using namespace b200timg;

extern "C" {

int b200timg_jpeg_parse(const uint8_t *jpg, size_t size, b200timg_jpeg_info *info) {
    if (!jpg || size == 0 || !info) return B200TIMG_EINVAL;
    Parse P;
    if (jpeg_walk(jpg, size, P) != 0) return B200TIMG_EINVAL;
    fill_info(P, info);
    return B200TIMG_OK;
}

int b200timg_jpeg_frames_dev(b200timg_ctx *ctx, int n_files, const uint8_t *const *files, const size_t *sizes,
                             uint8_t *d_frames, int32_t *d_status) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    B2_TRY(check_dev_outputs(ctx, "jpeg", d_frames, d_status, "d_status"));
    std::vector<Parse> ps;
    B2_TRY(parse_files(ctx, "jpeg", "header walk", jpeg_walk, n_files, files, sizes, ps));
    return launch_jpeg(ctx, n_files, files, sizes, ps, d_frames, d_status);
}

int b200timg_jpeg_frames(b200timg_ctx *ctx, int n_files, const uint8_t *const *files, const size_t *sizes,
                         uint8_t *frames, int32_t *status) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!frames || !status) return ctx->fail(B200TIMG_EINVAL, "jpeg: null output");
    std::vector<Parse> ps;
    B2_TRY(parse_files(ctx, "jpeg", "header walk", jpeg_walk, n_files, files, sizes, ps));
    size_t bytes = 0;
    for (const Parse &P : ps) bytes += (size_t)P.w * P.h * 4;
    return decode_to_host(ctx, bytes, n_files, frames, status, [&](uint8_t *d_frames, int32_t *d_status) {
        return launch_jpeg(ctx, n_files, files, sizes, ps, d_frames, d_status);
    });
}

}  // extern "C"
