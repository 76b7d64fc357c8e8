// The reference's OTHER scaler: libswscale with SWS_BILINEAR, used
//   * by ImageScaler in the default (video-enabled) build, RGBA -> RGBA      src/image-scaler.cc:45-72
//   * by the video source, decoder YUV -> RGBA at the target size in one go  src/video-source.cc:59-89,352-354
// libswscale is a third-party library that is not part of the reference tree (any version the distro ships,
// CMakeLists.txt:72-74), its result depends on version and SIMD path, and for RGBA input it round-trips through
// chroma-subsampled YUV: there is no arithmetic to pin.  PARITY UNPINNED -- this file implements what
// "bilinear" means there (a triangle filter whose support grows with the downscale ratio, centre-aligned
// sampling, edge clamp, BT.601 limited-range or full-range conversion) in float, and the tests measure the
// distance to the libswscale 9.1 that happens to be bundled with the image's OpenCV wheel (tolerance stated
// there), plus bit-level agreement with a float64 numpy statement of the same filter to within 1 LSB.
//
//   yuv_rgba_kernel<F>   decoder YUV frame (8-bit 4:2:0 I420 / NV12, 4:2:2, 4:4:4, 4:4:0, 10-bit 4:2:0 / 4:2:2 /
//                        4:4:4 planar and P010) -> RGBA at ow x oh: colour conversion fused into the resampler, the
//                        RGBA source-size intermediate never exists (SURVEY 8f rank 1).  1.5-6 B/px cross PCIe
//                        instead of 4 plus a host conversion pass.  One instantiation per format (YuvFmt).
//   bilinear_rgba_kernel RGBA -> RGBA triangle filter (the a3 row).
// One thread per output pixel; taps come from per-axis tables built on the host.  Algorithmic bytes:
// source bytes read once + 4*ow*oh written.
#include <algorithm>
#include <cmath>
#include <type_traits>
#include <vector>

#include "common.cuh"

namespace b200timg {

struct TriAxis { std::vector<int32_t> first, count; std::vector<float> coeff; int widest = 1; };

// dst index i samples the source at (i + 0.5) * src/dst - 0.5; upscaling: 2 taps; downscaling by r: triangle of half-width r
static void build_tri_axis(int src, int dst, TriAxis *t) {
    const double r = (double)src / (double)dst;
    const double half = r > 1.0 ? r : 1.0;
    t->widest = (int)std::ceil(2.0 * half) + 1;
    t->first.assign(dst, 0); t->count.assign(dst, 0); t->coeff.assign((size_t)dst * t->widest, 0.0f);
    for (int i = 0; i < dst; ++i) {
        const double c = (i + 0.5) * r - 0.5;
        int lo = (int)std::ceil(c - half), hi = (int)std::floor(c + half);
        if (lo == hi && half == 1.0) hi = lo + 1;
        std::vector<double> w;
        double sum = 0.0;
        for (int j = lo; j <= hi; ++j) { const double v = std::max(0.0, 1.0 - std::fabs(j - c) / half); w.push_back(v); sum += v; }
        // edge clamp: fold the weights of out-of-range taps onto the border sample
        const int clo = std::max(lo, 0), chi = std::min(hi, src - 1);
        std::vector<double> f((size_t)(chi - clo + 1), 0.0);
        for (int j = lo; j <= hi; ++j) f[(size_t)(std::min(std::max(j, 0), src - 1) - clo)] += w[(size_t)(j - lo)];
        t->first[i] = clo; t->count[i] = chi - clo + 1;
        for (int k = 0; k <= chi - clo; ++k) t->coeff[(size_t)i * t->widest + k] = (float)(f[(size_t)k] / sum);
    }
}

struct TriDev { const int32_t *first, *count; const float *coeff; int widest; };

struct YuvParams {
    int iw, ih, ow, oh, out_frame_rows, full_range;
    long long frame_bytes;
    TriDev yh, yv, ch, cv;
};

// Compile-time description of a decoder format (the low nibble of B200TIMG_FMT_*): chroma subsampling shifts,
// 8- or 16-bit samples (10 value bits, low or high), planar or interleaved chroma, and whether chroma is filtered at
// half the output width (libswscale's packed-RGB writers) or at the full width (its full chroma interpolation, which
// it switches on for sources without chroma subsampling).
template <int F> struct YuvFmt {
    static constexpr int sx = (F == B200TIMG_FMT_I444 || F == B200TIMG_FMT_I440 || F == B200TIMG_FMT_I444_10) ? 0 : 1;
    static constexpr int sy = (F == B200TIMG_FMT_I422 || F == B200TIMG_FMT_I444 || F == B200TIMG_FMT_I422_10 ||
                               F == B200TIMG_FMT_I444_10) ? 0 : 1;
    static constexpr bool wide = F >= B200TIMG_FMT_I420_10;        // 16-bit little-endian samples
    static constexpr bool high10 = F == B200TIMG_FMT_P010;         // value in bits 6..15, else bits 0..9
    static constexpr bool semi = F == B200TIMG_FMT_NV12 || F == B200TIMG_FMT_P010;
    static constexpr bool full = sx == 0 && sy == 0;               // chroma at the full output width
    using S = typename std::conditional<wide, uint16_t, uint8_t>::type;     // one sample
    using Q = typename std::conditional<wide, uint2, uint32_t>::type;       // four samples (one staging load)
    __device__ static __forceinline__ float val(S s) { return (float)(high10 ? (s >> 6) : wide ? (s & 0x3ff) : s); }
    // two 16-bit samples of a word -> their 10 value bits (identity for bytes)
    __device__ static __forceinline__ uint32_t bits2(uint32_t w) { return high10 ? (w >> 6) & 0x03ff03ffu : wide ? w & 0x03ff03ffu : w; }
    __device__ static __forceinline__ uint32_t bits(uint32_t w) { return bits2(w); }
    __device__ static __forceinline__ uint2 bits(uint2 w) { return make_uint2(bits2(w.x), bits2(w.y)); }
};

__device__ __forceinline__ uint32_t sat8(float v) { return __float2uint_rn(fminf(fmaxf(v, 0.0f), 255.0f)); }

// filtered Y, Cb, Cr (8-bit domain) -> packed RGBA
__device__ __forceinline__ uint32_t yuv_to_rgba(float y, float u, float v, int full_range) {
    float r, g, b;
    u -= 128.0f; v -= 128.0f;
    if (full_range) {                         // JPEG / "yuvj": Y, Cb, Cr over 0..255
        r = y + 1.402f * v; g = y - 0.344136f * u - 0.714136f * v; b = y + 1.772f * u;
    } else {                                  // ITU-R BT.601, Y 16..235, Cb/Cr 16..240 (SWS_CS_DEFAULT)
        const float yl = 1.164383f * (y - 16.0f);
        r = yl + 1.596027f * v; g = yl - 0.391762f * u - 0.812968f * v; b = yl + 2.017232f * u;
    }
    return pack_rgba(sat8(r), sat8(g), sat8(b), 0xffu);
}

template <int F>
__global__ void __launch_bounds__(256)
yuv_rgba_kernel(const uint8_t *__restrict__ in, uint32_t *__restrict__ out, YuvParams P) {
    using T = YuvFmt<F>;
    using S = typename T::S;
    const int ox = blockIdx.x * 32 + (threadIdx.x & 31), oy = blockIdx.y * 8 + (threadIdx.x >> 5), f = blockIdx.z;
    if (ox >= P.ow || oy >= P.oh) return;
    const S *Y = reinterpret_cast<const S *>(in + (long long)f * P.frame_bytes);
    const int cw = P.iw >> T::sx, chh = P.ih >> T::sy;
    const S *U = Y + (long long)P.iw * P.ih, *V = U + (long long)cw * chh;
    float y = 0.0f, u = 0.0f, v = 0.0f;
    {
        const int x0 = P.yh.first[ox], nx = P.yh.count[ox], y0 = P.yv.first[oy], ny = P.yv.count[oy];
        const float *hx = P.yh.coeff + (long long)ox * P.yh.widest, *hy = P.yv.coeff + (long long)oy * P.yv.widest;
        for (int j = 0; j < ny; ++j) {
            const S *row = Y + (long long)(y0 + j) * P.iw + x0;
            float a = 0.0f;
            for (int i = 0; i < nx; ++i) a = fmaf(T::val(row[i]), hx[i], a);
            y = fmaf(a, hy[j], y);
        }
    }
    {
        // libswscale's packed-RGB writers (without SWS_FULL_CHR_H_INT, which the reference does not set) carry chroma at
        // half the OUTPUT width: the two pixels of an output pair share one chroma sample.  4:4:4 sources make it
        // switch to full chroma interpolation: one chroma sample per output pixel.
        const int cx = T::full ? ox : ox >> 1;
        const int x0 = P.ch.first[cx], nx = P.ch.count[cx], y0 = P.cv.first[oy], ny = P.cv.count[oy];
        const float *hx = P.ch.coeff + (long long)cx * P.ch.widest, *hy = P.cv.coeff + (long long)oy * P.cv.widest;
        for (int j = 0; j < ny; ++j) {
            float au = 0.0f, av = 0.0f;
            if (T::semi) {
                const S *row = U + ((long long)(y0 + j) * cw + x0) * 2;
                for (int i = 0; i < nx; ++i) { au = fmaf(T::val(row[2 * i]), hx[i], au); av = fmaf(T::val(row[2 * i + 1]), hx[i], av); }
            } else {
                const S *ru = U + (long long)(y0 + j) * cw + x0, *rv = V + (long long)(y0 + j) * cw + x0;
                for (int i = 0; i < nx; ++i) { au = fmaf(T::val(ru[i]), hx[i], au); av = fmaf(T::val(rv[i]), hx[i], av); }
            }
            u = fmaf(au, hy[j], u); v = fmaf(av, hy[j], v);
        }
    }
    if (T::wide) { y *= 0.25f; u *= 0.25f; v *= 0.25f; }      // 10-bit -> 8-bit domain (exact: a power of two)
    out[((long long)f * P.out_frame_rows + oy) * P.ow + ox] = yuv_to_rgba(y, u, v, P.full_range);
}


// ---- tiled variant: the same filter, separable inside a 64 x 32 output tile -------------------------
// The per-pixel kernel above redoes the horizontal taps of every source row for every output row that uses
// it.  Here a tile stages its luma / chroma sample windows in shared memory once (8- or 16-bit samples, the
// 10 value bits already extracted), runs the vertical taps into float rows (luma at source width, chroma at the
// chroma plane's width), then the horizontal taps, converts and stores.  Needs iw % 8 == 0 and a source
// pointer aligned to 8 bytes (8-bit formats) or 16 bytes (16-bit formats): every staging load is then one
// aligned word of four samples (two words for interleaved chroma).
constexpr int YT_W = 64, YT_H = 32, YT_NT = 256;
struct YuvTileGeom { int nix, niy, ncx, ncy; };        // window extents (luma cols/rows, chroma cols/rows), maxima over tiles

template <int F>
__global__ void __launch_bounds__(YT_NT)
yuv_rgba_tiled_kernel(const uint8_t *__restrict__ in, uint32_t *__restrict__ out, YuvParams P, YuvTileGeom G) {
    using T = YuvFmt<F>;
    using S = typename T::S;
    using Q = typename T::Q;
    extern __shared__ __align__(16) uint8_t s_yuv[];
    const int tid = threadIdx.x, f = blockIdx.z;
    const int ox0 = blockIdx.x * YT_W, oy0 = blockIdx.y * YT_H;
    const int tw = min(YT_W, P.ow - ox0), th = min(YT_H, P.oh - oy0);
    const int cxa = T::full ? ox0 : ox0 >> 1;                     // first output chroma column of this tile
    const int cw = P.iw >> T::sx, chh = P.ih >> T::sy;
    // window origins (tables are monotone), x origins aligned down to 4 samples
    const int ix0 = P.yh.first[ox0] & ~3, iy0 = P.yv.first[oy0];
    const int cx0 = P.ch.first[cxa] & ~3, cy0 = P.cv.first[oy0];
    const int nixw = (G.nix + 7) >> 2, ncxw = (G.ncx + 7) >> 2;   // 4-sample words per staged row (origin alignment slack included)
    const int ypitch = nixw * 4, cpitch = ncxw * 4;               // samples
    S *Yw = reinterpret_cast<S *>(s_yuv);                         // [niy][ypitch]
    S *Uw = Yw + G.niy * ypitch, *Vw = Uw + G.ncy * cpitch;       // [ncy][cpitch] each
    const int staged = (G.niy * ypitch + 2 * G.ncy * cpitch) * (int)sizeof(S);
    float *TY = reinterpret_cast<float *>(s_yuv + staged + ((16 - (staged & 15)) & 15));   // [YT_H][ypitch]
    float *TU = TY + YT_H * ypitch, *TV = TU + YT_H * cpitch;    // [YT_H][cpitch]
    const S *Y = reinterpret_cast<const S *>(in + (long long)f * P.frame_bytes);
    const S *C = Y + (long long)P.iw * P.ih;
    for (int u = tid; u < G.niy * nixw; u += YT_NT) {
        const int ly = u / nixw, g = u - ly * nixw, y = iy0 + ly, x = ix0 + 4 * g;
        Q v{};
        if (y < P.ih && x < P.iw) v = T::bits(__ldg(reinterpret_cast<const Q *>(Y + (long long)y * P.iw + x)));
        reinterpret_cast<Q *>(Yw + ly * ypitch)[g] = v;
    }
    for (int u = tid; u < G.ncy * ncxw; u += YT_NT) {
        const int ly = u / ncxw, g = u - ly * ncxw, y = cy0 + ly, x = cx0 + 4 * g;
        Q pu{}, pv{};
        if (y < chh && x < cw) {
            if constexpr (T::semi && !T::wide) {
                const uint2 q = __ldg(reinterpret_cast<const uint2 *>(C + ((long long)y * cw + x) * 2));      // U0 V0 U1 V1 | U2 V2 U3 V3
                pu = __byte_perm(q.x, q.y, 0x6420); pv = __byte_perm(q.x, q.y, 0x7531);
            } else if constexpr (T::semi) {
                const uint4 q = __ldg(reinterpret_cast<const uint4 *>(C + ((long long)y * cw + x) * 2));      // U0 V0 | U1 V1 | U2 V2 | U3 V3
                pu = T::bits(make_uint2(__byte_perm(q.x, q.y, 0x5410), __byte_perm(q.z, q.w, 0x5410)));
                pv = T::bits(make_uint2(__byte_perm(q.x, q.y, 0x7632), __byte_perm(q.z, q.w, 0x7632)));
            } else {
                pu = T::bits(__ldg(reinterpret_cast<const Q *>(C + (long long)y * cw + x)));
                pv = T::bits(__ldg(reinterpret_cast<const Q *>(C + (long long)cw * chh + (long long)y * cw + x)));
            }
        }
        reinterpret_cast<Q *>(Uw + ly * cpitch)[g] = pu;
        reinterpret_cast<Q *>(Vw + ly * cpitch)[g] = pv;
    }
    __syncthreads();
    // vertical taps: luma rows -> TY, chroma rows -> TU / TV
    for (int u = tid; u < th * ypitch; u += YT_NT) {
        const int ty = u / ypitch, x = u - ty * ypitch, oy = oy0 + ty;
        const int y0 = P.yv.first[oy] - iy0, ny = P.yv.count[oy];
        const float *hy = P.yv.coeff + (long long)oy * P.yv.widest;
        float a = 0.0f;
        for (int j = 0; j < ny; ++j) a = fmaf((float)Yw[(y0 + j) * ypitch + x], hy[j], a);
        TY[ty * ypitch + x] = a;
    }
    for (int u = tid; u < th * cpitch; u += YT_NT) {
        const int ty = u / cpitch, x = u - ty * cpitch, oy = oy0 + ty;
        const int y0 = P.cv.first[oy] - cy0, ny = P.cv.count[oy];
        const float *hy = P.cv.coeff + (long long)oy * P.cv.widest;
        float au = 0.0f, av = 0.0f;
        for (int j = 0; j < ny; ++j) { au = fmaf((float)Uw[(y0 + j) * cpitch + x], hy[j], au); av = fmaf((float)Vw[(y0 + j) * cpitch + x], hy[j], av); }
        TU[ty * cpitch + x] = au; TV[ty * cpitch + x] = av;
    }
    __syncthreads();
    // horizontal taps + colour conversion: thread -> (row, column), consecutive lanes on consecutive columns
    for (int u = tid; u < th * YT_W; u += YT_NT) {
        const int ty = u >> 6, tx = u & 63, ox = ox0 + tx, oy = oy0 + ty;
        if (tx >= tw) continue;
        float y = 0.0f, uu = 0.0f, vv = 0.0f;
        {
            const int x0 = P.yh.first[ox] - ix0, nx = P.yh.count[ox];
            const float *hx = P.yh.coeff + (long long)ox * P.yh.widest, *row = TY + ty * ypitch + x0;
            for (int i = 0; i < nx; ++i) y = fmaf(row[i], hx[i], y);
        }
        {
            const int cx = T::full ? ox : ox >> 1, x0 = P.ch.first[cx] - cx0, nx = P.ch.count[cx];
            const float *hx = P.ch.coeff + (long long)cx * P.ch.widest, *ru = TU + ty * cpitch + x0, *rv = TV + ty * cpitch + x0;
            for (int i = 0; i < nx; ++i) { uu = fmaf(ru[i], hx[i], uu); vv = fmaf(rv[i], hx[i], vv); }
        }
        if (T::wide) { y *= 0.25f; uu *= 0.25f; vv *= 0.25f; }
        out[((long long)f * P.out_frame_rows + oy) * P.ow + ox] = yuv_to_rgba(y, uu, vv, P.full_range);
    }
}

struct BilinearParams { int iw, ih, ow, oh, out_frame_rows, bgra; TriDev h, v; ComposeSpec cs; };

__global__ void __launch_bounds__(256)
bilinear_rgba_kernel(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, BilinearParams P) {
    const int ox = blockIdx.x * 32 + (threadIdx.x & 31), oy = blockIdx.y * 8 + (threadIdx.x >> 5), f = blockIdx.z;
    if (ox >= P.ow || oy >= P.oh) return;
    const uint32_t *src = in + (long long)f * P.iw * P.ih;
    const int x0 = P.h.first[ox], nx = P.h.count[ox], y0 = P.v.first[oy], ny = P.v.count[oy];
    const float *hx = P.h.coeff + (long long)ox * P.h.widest, *hy = P.v.coeff + (long long)oy * P.v.widest;
    float c[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    for (int j = 0; j < ny; ++j) {
        const uint32_t *row = src + (long long)(y0 + j) * P.iw + x0;
        float a[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        for (int i = 0; i < nx; ++i) {
            const uint32_t p = row[i];
            const float w = hx[i];
            a[0] = fmaf((float)(p & 0xff), w, a[0]); a[1] = fmaf((float)((p >> 8) & 0xff), w, a[1]);
            a[2] = fmaf((float)((p >> 16) & 0xff), w, a[2]); a[3] = fmaf((float)(p >> 24), w, a[3]);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) c[k] = fmaf(a[k], hy[j], c[k]);
    }
    const uint32_t r = sat8(P.bgra ? c[2] : c[0]), g = sat8(c[1]), b = sat8(P.bgra ? c[0] : c[2]), al = sat8(c[3]);
    out[((long long)f * P.out_frame_rows + oy) * P.ow + ox] = compose_at(P.cs, pack_rgba(r, g, b, al), ox, oy);
}

// ---- host side: tables cached per geometry in ctx->tri_tables -------------------------------------
static size_t al16(size_t v) { return (v + 15) / 16 * 16; }

struct TriUpload {
    std::vector<char> host;
    size_t add(const TriAxis &t, int n, TriDev *d_rel) {           // returns nothing useful; fills offsets in d_rel as integers
        const size_t o_f = host.size(); host.resize(o_f + al16(sizeof(int32_t) * n));
        memcpy(host.data() + o_f, t.first.data(), sizeof(int32_t) * n);
        const size_t o_c = host.size(); host.resize(o_c + al16(sizeof(int32_t) * n));
        memcpy(host.data() + o_c, t.count.data(), sizeof(int32_t) * n);
        const size_t o_k = host.size(); host.resize(o_k + al16(sizeof(float) * t.coeff.size()));
        memcpy(host.data() + o_k, t.coeff.data(), sizeof(float) * t.coeff.size());
        d_rel->first = reinterpret_cast<const int32_t *>(o_f);
        d_rel->count = reinterpret_cast<const int32_t *>(o_c);
        d_rel->coeff = reinterpret_cast<const float *>(o_k);
        d_rel->widest = t.widest;
        return o_f;
    }
};
static void rebase(TriDev *d, const char *base) {
    d->first = reinterpret_cast<const int32_t *>(base + reinterpret_cast<size_t>(d->first));
    d->count = reinterpret_cast<const int32_t *>(base + reinterpret_cast<size_t>(d->count));
    d->coeff = reinterpret_cast<const float *>(base + reinterpret_cast<size_t>(d->coeff));
}

// tables are rebuilt only when the geometry changes (a batch pipeline calls the scaler once per chunk)
static bool tri_cached(b200timg_ctx *ctx, int kind, int iw, int ih, int ow, int oh, void *params, size_t bytes) {
    const int key[5] = {kind, iw, ih, ow, oh};
    if (memcmp(key, ctx->tri_key, sizeof key) == 0 && ctx->tri_params.size() == bytes) { memcpy(params, ctx->tri_params.data(), bytes); return true; }
    return false;
}
static void tri_remember(b200timg_ctx *ctx, int kind, int iw, int ih, int ow, int oh, const void *params, size_t bytes) {
    const int key[5] = {kind, iw, ih, ow, oh};
    memcpy(ctx->tri_key, key, sizeof key);
    ctx->tri_params.assign(static_cast<const char *>(params), static_cast<const char *>(params) + bytes);
}

static int upload_tri(b200timg_ctx *ctx, TriUpload &up) {
    B2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));                 // earlier launches may still read the old tables
    B2_CUDA(ctx, ctx->tri_tables.reserve(up.host.size()));
    B2_CUDA(ctx, cudaMemcpyAsync(ctx->tri_tables.p, up.host.data(), up.host.size(), cudaMemcpyHostToDevice, ctx->stream));
    B2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));                 // up.host is a local
    return B200TIMG_OK;
}

// Bytes of one tightly packed frame of a YUV format (any FULL_RANGE bit ignored); 0 for a code that is not one.
long long yuv_frame_bytes(int fmt, int iw, int ih) {
    const int f = fmt & 0xf;
    if (f < B200TIMG_FMT_I420 || f > B200TIMG_FMT_P010) return 0;
    const bool wide = f >= B200TIMG_FMT_I420_10;
    const int sx = (f == B200TIMG_FMT_I444 || f == B200TIMG_FMT_I440 || f == B200TIMG_FMT_I444_10) ? 0 : 1;
    const int sy = (f == B200TIMG_FMT_I422 || f == B200TIMG_FMT_I444 || f == B200TIMG_FMT_I422_10 || f == B200TIMG_FMT_I444_10) ? 0 : 1;
    return (wide ? 2 : 1) * ((long long)iw * ih + 2ll * (iw >> sx) * (ih >> sy));
}

static const char *yuv_fmt_name(int f) {
    static const char *const names[] = {"I420", "NV12", "I422", "I444", "I440", "I420_10", "I422_10", "I444_10", "P010"};
    return f >= B200TIMG_FMT_I420 && f <= B200TIMG_FMT_P010 ? names[f - B200TIMG_FMT_I420] : "?";
}

// EINVAL unless fmt is a YUV code and iw x ih is a multiple of its chroma subsampling
int yuv_check_format(b200timg_ctx *ctx, int fmt, int iw, int ih) {
    const int f = fmt & 0xf;
    if (!yuv_frame_bytes(fmt, 2, 2)) return ctx->fail(B200TIMG_EINVAL, "yuv: unknown source format %d", fmt);
    const bool hsub = f != B200TIMG_FMT_I444 && f != B200TIMG_FMT_I440 && f != B200TIMG_FMT_I444_10;
    const bool vsub = f != B200TIMG_FMT_I422 && f != B200TIMG_FMT_I444 && f != B200TIMG_FMT_I422_10 && f != B200TIMG_FMT_I444_10;
    if ((hsub && (iw & 1)) || (vsub && (ih & 1)))
        return ctx->fail(B200TIMG_EINVAL, "yuv: %s frames need an even %s (got %dx%d)", yuv_fmt_name(f),
                         hsub && vsub ? "width and height" : hsub ? "width" : "height", iw, ih);
    return B200TIMG_OK;
}

template <int F> struct YuvKernelName;
#define B2_YUV_NAMES(F, sfx) template <> struct YuvKernelName<F> { \
    static constexpr const char *tiled = "yuv_rgba_tiled_kernel_" sfx, *simple = "yuv_rgba_kernel_" sfx; };
B2_YUV_NAMES(B200TIMG_FMT_I420, "i420") B2_YUV_NAMES(B200TIMG_FMT_NV12, "nv12") B2_YUV_NAMES(B200TIMG_FMT_I422, "i422")
B2_YUV_NAMES(B200TIMG_FMT_I444, "i444") B2_YUV_NAMES(B200TIMG_FMT_I440, "i440") B2_YUV_NAMES(B200TIMG_FMT_I420_10, "i420_10")
B2_YUV_NAMES(B200TIMG_FMT_I422_10, "i422_10") B2_YUV_NAMES(B200TIMG_FMT_I444_10, "i444_10") B2_YUV_NAMES(B200TIMG_FMT_P010, "p010")
#undef B2_YUV_NAMES

template <int F>
static int launch_yuv_fmt(b200timg_ctx *ctx, const uint8_t *d_in, int iw, int ih, int fmt, uint8_t *d_out, int ow, int oh,
                          int out_frame_rows, int n_frames) {
    using T = YuvFmt<F>;
    const int cw = iw >> T::sx, ch = ih >> T::sy, cow = T::full ? ow : (ow + 1) / 2;
    // libswscale's unscaled yuv2rgb converters exist for 8-bit 4:2:0 only: they replicate chroma rows (2x2 blocks
    // share a sample); every other format goes through the scaler's triangle filter even at scale 1
    const bool replicate = (F == B200TIMG_FMT_I420 || F == B200TIMG_FMT_NV12) && ow == iw && oh == ih;
    YuvParams P;
    P.iw = iw; P.ih = ih; P.ow = ow; P.oh = oh; P.out_frame_rows = out_frame_rows;
    P.full_range = (fmt & B200TIMG_FMT_FULL_RANGE) != 0;
    P.frame_bytes = yuv_frame_bytes(F, iw, ih);
    // the tables (and the tile extents beside them) depend on the chroma layout, not only on the geometry: it is part
    // of the cache key.  I420 / NV12 and the other layouts that share tables share an entry.
    const int kind = 1 | T::sx << 4 | T::sy << 5 | (int)T::full << 6 | (int)(F == B200TIMG_FMT_I420 || F == B200TIMG_FMT_NV12) << 7;
    TriDev td[4];
    if (!tri_cached(ctx, kind, iw, ih, ow, oh, td, sizeof td)) {
        TriAxis yh, yv, chx, cvy;
        build_tri_axis(iw, ow, &yh); build_tri_axis(ih, oh, &yv); build_tri_axis(cw, cow, &chx); build_tri_axis(ch, oh, &cvy);
        if (replicate) {
            cvy.widest = 1; cvy.coeff.assign((size_t)oh, 1.0f);
            for (int y = 0; y < oh; ++y) { cvy.first[y] = y >> 1; cvy.count[y] = 1; }
        }
        TriUpload up;
        up.add(yh, ow, &td[0]); up.add(yv, oh, &td[1]); up.add(chx, cow, &td[2]); up.add(cvy, oh, &td[3]);
        {   // tile window extents for the tiled kernel
            auto extent = [](const TriAxis &t, int n, int tile, int align) {
                int best = 1;
                for (int a = 0; a < n; a += tile) {
                    const int b = std::min(n, a + tile) - 1;
                    const int lo = t.first[a] & ~(align - 1), hi = t.first[b] + t.count[b];
                    best = std::max(best, hi - lo);
                }
                return best;
            };
            ctx->yuv_geom[0] = extent(yh, ow, YT_W, 4); ctx->yuv_geom[1] = extent(yv, oh, YT_H, 1);
            ctx->yuv_geom[2] = extent(chx, cow, T::full ? YT_W : YT_W / 2, 4); ctx->yuv_geom[3] = extent(cvy, oh, YT_H, 1);
            ctx->yuv_geom_valid = true;
        }
        ctx->tri_key[0] = 0;
        B2_TRY(upload_tri(ctx, up));
        const char *base = ctx->tri_tables.as<char>();
        for (auto &t : td) rebase(&t, base);
        tri_remember(ctx, kind, iw, ih, ow, oh, td, sizeof td);
    }
    P.yh = td[0]; P.yv = td[1]; P.ch = td[2]; P.cv = td[3];
    const uintptr_t align = T::wide ? 15 : 7;
    if ((iw & 7) == 0 && (reinterpret_cast<uintptr_t>(d_in) & align) == 0 && !getenv("B200TIMG_YUV_SIMPLE") && ctx->yuv_geom_valid) {
        // window extents of a 64 x 32 tile (maxima over tiles), from the host copies of the tables
        const YuvTileGeom G{ctx->yuv_geom[0], ctx->yuv_geom[1], ctx->yuv_geom[2], ctx->yuv_geom[3]};
        const int nixw = (G.nix + 7) >> 2, ncxw = (G.ncx + 7) >> 2;
        const size_t bytes = ((size_t)G.niy * nixw * 4 + 2 * (size_t)G.ncy * ncxw * 4) * sizeof(typename T::S) + 16 +
                             sizeof(float) * ((size_t)YT_H * nixw * 4 + 2 * (size_t)YT_H * ncxw * 4);
        if (bytes <= 200 * 1024) {
            B2_CUDA(ctx, cudaFuncSetAttribute(yuv_rgba_tiled_kernel<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
            B2_KERNEL(ctx, YuvKernelName<F>::tiled);
            yuv_rgba_tiled_kernel<F><<<dim3((ow + YT_W - 1) / YT_W, (oh + YT_H - 1) / YT_H, n_frames), YT_NT, bytes, ctx->stream>>>(
                d_in, reinterpret_cast<uint32_t *>(d_out), P, G);
            B2_LAUNCH_CHECK(ctx);
            return B200TIMG_OK;
        }
    }
    B2_KERNEL(ctx, YuvKernelName<F>::simple);
    yuv_rgba_kernel<F><<<dim3((ow + 31) / 32, (oh + 7) / 8, n_frames), 256, 0, ctx->stream>>>(d_in, reinterpret_cast<uint32_t *>(d_out), P);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

// fmt: any B200TIMG_FMT_* YUV code, optionally | B200TIMG_FMT_FULL_RANGE
int launch_yuv_scale(b200timg_ctx *ctx, const uint8_t *d_in, int iw, int ih, int fmt, uint8_t *d_out, int ow, int oh,
                     int out_frame_rows, int n_frames) {
    if (out_frame_rows < oh) return ctx->fail(B200TIMG_EINVAL, "yuv: frame rows < out height");
    B2_TRY(yuv_check_format(ctx, fmt, iw, ih));
    if (n_frames > 65535) return ctx->fail(B200TIMG_EINVAL, "yuv: too many frames for one launch");
    switch (fmt & 0xf) {
    case B200TIMG_FMT_I420: return launch_yuv_fmt<B200TIMG_FMT_I420>(ctx, d_in, iw, ih, fmt, d_out, ow, oh, out_frame_rows, n_frames);
    case B200TIMG_FMT_NV12: return launch_yuv_fmt<B200TIMG_FMT_NV12>(ctx, d_in, iw, ih, fmt, d_out, ow, oh, out_frame_rows, n_frames);
    case B200TIMG_FMT_I422: return launch_yuv_fmt<B200TIMG_FMT_I422>(ctx, d_in, iw, ih, fmt, d_out, ow, oh, out_frame_rows, n_frames);
    case B200TIMG_FMT_I444: return launch_yuv_fmt<B200TIMG_FMT_I444>(ctx, d_in, iw, ih, fmt, d_out, ow, oh, out_frame_rows, n_frames);
    case B200TIMG_FMT_I440: return launch_yuv_fmt<B200TIMG_FMT_I440>(ctx, d_in, iw, ih, fmt, d_out, ow, oh, out_frame_rows, n_frames);
    case B200TIMG_FMT_I420_10: return launch_yuv_fmt<B200TIMG_FMT_I420_10>(ctx, d_in, iw, ih, fmt, d_out, ow, oh, out_frame_rows, n_frames);
    case B200TIMG_FMT_I422_10: return launch_yuv_fmt<B200TIMG_FMT_I422_10>(ctx, d_in, iw, ih, fmt, d_out, ow, oh, out_frame_rows, n_frames);
    case B200TIMG_FMT_I444_10: return launch_yuv_fmt<B200TIMG_FMT_I444_10>(ctx, d_in, iw, ih, fmt, d_out, ow, oh, out_frame_rows, n_frames);
    default: return launch_yuv_fmt<B200TIMG_FMT_P010>(ctx, d_in, iw, ih, fmt, d_out, ow, oh, out_frame_rows, n_frames);
    }
}

int launch_scale_bilinear(b200timg_ctx *ctx, const uint8_t *d_in, int iw, int ih, int fmt, uint8_t *d_out, int ow, int oh,
                          int out_frame_rows, int n_frames, const ComposeSpec *cs) {
    if (out_frame_rows < oh) return ctx->fail(B200TIMG_EINVAL, "scale: frame rows < out height");
    if (n_frames > 65535) return ctx->fail(B200TIMG_EINVAL, "scale: too many frames for one launch");
    BilinearParams P;
    P.iw = iw; P.ih = ih; P.ow = ow; P.oh = oh; P.out_frame_rows = out_frame_rows; P.bgra = fmt == B200TIMG_FMT_RGB32;
    if (cs) P.cs = *cs; else { memset(&P.cs, 0, sizeof P.cs); P.cs.pw = P.cs.ph = 1; }
    TriDev td[2];
    if (!tri_cached(ctx, 2, iw, ih, ow, oh, td, sizeof td)) {
        TriAxis h, v;
        build_tri_axis(iw, ow, &h); build_tri_axis(ih, oh, &v);
        TriUpload up;
        up.add(h, ow, &td[0]); up.add(v, oh, &td[1]);
        ctx->tri_key[0] = 0;
        B2_TRY(upload_tri(ctx, up));
        const char *base = ctx->tri_tables.as<char>();
        for (auto &t : td) rebase(&t, base);
        tri_remember(ctx, 2, iw, ih, ow, oh, td, sizeof td);
    }
    P.h = td[0]; P.v = td[1];
    B2_KERNEL(ctx, "bilinear_rgba_kernel");
    bilinear_rgba_kernel<<<dim3((ow + 31) / 32, (oh + 7) / 8, n_frames), 256, 0, ctx->stream>>>(
        reinterpret_cast<const uint32_t *>(d_in), reinterpret_cast<uint32_t *>(d_out), P);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

}  // namespace b200timg
