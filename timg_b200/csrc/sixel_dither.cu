// K5: libsixel's sixel_quant_apply_palette with Floyd-Steinberg diffusion (quant.c diffuse_fs /
// error_diffuse, reached from sixel_encode, call site src/sixel-canvas.cc:144-145) as a wavefront.
//
// Semantics kept bit for bit (oracle/sixel_oracle.c mode 1): the error of a pixel is added tap by tap
// into 8-bit clamped pixels -- 1/16 from (x-1,y-1), 5/16 from (x,y-1), 3/16 from (x+1,y-1), 7/16 from
// (x-1,y), each e*k/16 with C truncation and a clamp to [0,255] after every add; no diffusion from the
// last row / last column; x = 0's below-left tap lands on the same row's last pixel; the palette index
// is the nearest-colour table entry of the pixel's 15-bit cell.
//
// Shape: a warp owns a band of 32 rows, lane l runs row l two columns behind lane l-1.  What changed
// against round 1 is the instruction diet:
//   * a pixel is two packed s16x2 registers (R|G, B|0); a clamped tap add is ONE DPX instruction
//     (VIADDMNMX.S16x2.RELU: max(min(a+b, 255), 0) per half) instead of IMAD+SHF+add+min+max per channel;
//   * the four truncated taps of an error value come from a 511-entry table (one 32-bit word: t7|t3|t5|t1
//     as signed bytes), fetched once per channel by the pixel's own lane; a tap is moved into s16x2 form
//     with one PRMT (sign replication);
//   * the lane below receives the three table words by shuffle; lane 0 reads the band above's last row
//     from a staged copy of the boundary row, lane 31 appends to this band's boundary row;
//   * palette entries are pre-packed as (256 - P) per half, so error + 256 (the table index) is one add.
// Bands are pipelined warp to warp through the boundary rows (global memory, L2) and per-band progress
// counters: in shared memory inside a CTA, in global memory between the CTAs of one frame when a frame
// is split over several CTAs (small batches: single-frame latency).
#include <algorithm>
#include <cstdlib>

#include "sixel.cuh"

namespace b200timg {

#ifdef CUSIM
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t s) { return __byte_perm(a, b, s); }
#else
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t s) {
    uint32_t d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(s));
    return d;
}
#endif

constexpr int D2_WMAX = 24;                       // warps per CTA (upper bound)
constexpr int D2_CH = 16;                         // columns per staged chunk
constexpr int D2_IN_STRIDE = D2_CH + 1;           // odd: lanes hit distinct banks
constexpr int D2_OUT_STRIDE = 20;
constexpr int D2_WARP_SMEM = 2 * 32 * D2_IN_STRIDE * 4 + 32 * D2_OUT_STRIDE + D2_CH * 16;   // in tiles | out tile | boundary chunk

struct TapW { uint32_t r, g, b; };                // table words of one pixel's error, per channel

// tap k of (R,G) as s16x2 / of B as (s16, 0): byte k of the table word, sign-extended
template <int K> __device__ __forceinline__ uint32_t tap_rg(const TapW &t) {
    constexpr uint32_t sel = (uint32_t)K | ((8u | K) << 4) | ((4u + K) << 8) | ((8u | (4u + K)) << 12);
    return prmt(t.r, t.g, sel);
}
template <int K> __device__ __forceinline__ uint32_t tap_b(const TapW &t) {
    constexpr uint32_t sel = (uint32_t)K | ((8u | K) << 4) | (4u << 8) | (4u << 12);
    return prmt(t.b, 0u, sel);
}
__device__ __forceinline__ uint32_t add_clamp(uint32_t v, uint32_t t) { return __viaddmin_s16x2_relu(v, t, 0x00ff00ffu); }

struct Dither2Geom { int w, h, nb32, bands_per_cta, nwarps; unsigned spin_ns; };   // spin_ns: pause between two polls of the band above

// The CTA's frame and its part of the frame's bands (see sixel.cu's accessors):
//   DitherUniform  CTA blockIdx.x of frame blockIdx.y, Dither2Geom's geometry for every frame
//   DitherMixed    flat CTA blockIdx.x of a mixed batch; the block size (nwarps) is the launch's, a frame with fewer
//                  bands than warps leaves the spare warps idle after the setup barrier
struct DitherUniform {
    typedef Dither2Geom Params;
    const Dither2Geom &G; int f, g;
    __device__ __forceinline__ explicit DitherUniform(const Dither2Geom &p) : G(p), f(blockIdx.y), g(blockIdx.x) {}
    __device__ __forceinline__ int w() const { return G.w; }
    __device__ __forceinline__ int h() const { return G.h; }
    __device__ __forceinline__ int nb32() const { return G.nb32; }
    __device__ __forceinline__ int bands_per_cta() const { return G.bands_per_cta; }
    __device__ __forceinline__ int nwarps() const { return G.nwarps; }
    __device__ __forceinline__ unsigned spin_ns() const { return G.spin_ns; }
    __device__ __forceinline__ long long px0() const { return (long long)f * G.w * G.h; }
    __device__ __forceinline__ long long idx0() const { return (long long)f * G.w * G.h; }
    __device__ __forceinline__ long long bnd0() const { return (long long)f * G.nb32 * G.w; }
    __device__ __forceinline__ long long prog0() const { return (long long)f * G.nb32; }
};
struct DitherMixed {
    typedef MixedSixelParams Params;
    MixedSixelFrame D; int f, g, nw;
    __device__ __forceinline__ explicit DitherMixed(const MixedSixelParams &P) : nw(P.nwarps) {
        f = sixel_owner(P.cta_start, P.n_frames, blockIdx.x);
        g = (int)(blockIdx.x - P.cta_start[f]);
        D = P.desc[f];
    }
    __device__ __forceinline__ int w() const { return D.w; }
    __device__ __forceinline__ int h() const { return D.h; }
    __device__ __forceinline__ int nb32() const { return D.nb32; }
    __device__ __forceinline__ int bands_per_cta() const { return D.bands_per_cta; }
    __device__ __forceinline__ int nwarps() const { return nw; }
    __device__ __forceinline__ unsigned spin_ns() const { return 256; }     // the uniform default
    __device__ __forceinline__ long long px0() const { return (long long)D.fb_px; }
    __device__ __forceinline__ long long idx0() const { return (long long)D.idx; }
    __device__ __forceinline__ long long bnd0() const { return (long long)D.bnd; }
    __device__ __forceinline__ long long prog0() const { return (long long)D.prog0; }
};

template <class A>
__global__ void __launch_bounds__(D2_WMAX * 32)
sixel_dither2_kernel(const uint32_t *__restrict__ fb, typename A::Params G, SixelWork W, uint4 *__restrict__ bnd_all, int *__restrict__ gprog_all) {
    extern __shared__ __align__(16) uint8_t s_dyn2[];            // lut[32768] | per-warp tiles
    __shared__ uint2 s_pal2[256];                                // (256 - P) per half: .x = R | G << 16, .y = B | 256 << 16
    __shared__ uint32_t s_tap[512];                              // [e + 256] -> t7 | t3 << 8 | t5 << 16 | t1 << 24 (signed bytes)
    __shared__ volatile int s_progress[2048];             // columns completed by the last row of each band of this CTA
    const A a(G);
    const int f = a.f, g = a.g;
    const SixelFrameHdr *hdr = W.hdr + f;
    if (!hdr->diffuse) return;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int nthreads = a.nwarps() * 32, w = a.w(), h = a.h();
    uint8_t *s_lut = s_dyn2;
    for (int i = tid; i < 32768 / 16; i += nthreads)
        reinterpret_cast<uint4 *>(s_lut)[i] = reinterpret_cast<const uint4 *>(W.lut + (long long)f * 32768)[i];
    for (int i = tid; i < 256; i += nthreads) {
        const uint32_t p = hdr->palette[i];
        s_pal2[i] = make_uint2((256u - (p & 0xff)) | ((256u - ((p >> 8) & 0xff)) << 16), (256u - ((p >> 16) & 0xff)) | (256u << 16));
    }
    for (int i = tid; i < 512; i += nthreads) {
        const int e = i - 256;
        const int t7 = e * 7 / 16, t3 = e * 3 / 16, t5 = e * 5 / 16, t1 = e / 16;          // C truncation (error_diffuse)
        s_tap[i] = (uint32_t)(t7 & 0xff) | ((uint32_t)(t3 & 0xff) << 8) | ((uint32_t)(t5 & 0xff) << 16) | ((uint32_t)(t1 & 0xff) << 24);
    }
    const int band_lo = g * a.bands_per_cta(), band_hi = min(a.nb32(), band_lo + a.bands_per_cta());
    const int nlocal = band_hi - band_lo;
    for (int i = tid; i < nlocal; i += nthreads) s_progress[i] = 0;
    __syncthreads();
    uint32_t *s_in = reinterpret_cast<uint32_t *>(s_dyn2 + 32768 + (size_t)wid * D2_WARP_SMEM);   // [2][32][D2_IN_STRIDE]
    uint8_t *s_out = reinterpret_cast<uint8_t *>(s_in + 2 * 32 * D2_IN_STRIDE);                    // [32][D2_OUT_STRIDE]
    uint4 *s_bnd = reinterpret_cast<uint4 *>(s_out + 32 * D2_OUT_STRIDE);                          // [D2_CH]
    const uint32_t *frame = fb + a.px0();
    uint8_t *index = W.index + a.idx0();
    uint4 *bnd = bnd_all + a.bnd0();
    volatile int *gprog = gprog_all + a.prog0();
    const int hrow = lane >> 4, hcol = lane & 15;                // half-warp staging coordinates (odd widths)
    const int qrow = lane >> 3, qcol = lane & 7;                 // quarter-warp staging coordinates (even widths: pixel pairs)
    const bool even_w = (w & 1) == 0;
    const TapW Z = {0u, 0u, 0u};

    for (int band = band_lo + wid; band < band_hi; band += a.nwarps()) {
        const int lb = band - band_lo;
        const int y = band * 32 + lane;
        const bool row_ok = y < h, last_row = (y == h - 1);
        const bool prev_remote = band > 0 && lb == 0;            // the band above belongs to another CTA
        const bool publish_remote = band + 1 < a.nb32() && band + 1 == band_hi;
        const uint4 *bin = band > 0 ? bnd + (long long)(band - 1) * w : nullptr;
        uint4 *bout = bnd + (long long)band * w;
        TapW own = Z, a0 = Z, a1 = Z, a2 = Z, e_first = Z;
        const int steps = w + 62, nchunks = (steps + D2_CH - 1) / D2_CH;
        // staging of a chunk (16 skewed columns x 32 rows).  Even widths: 8 lanes per row, a pixel PAIR per lane (8-byte loads,
        // half the load instructions: the frame loads were 11 % of the kernel's instructions); odd widths: 16 lanes per row.
        uint32_t pre[16];
        auto load_chunk = [&](int c) {
            if (even_w) {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int r = 4 * i + qrow, yy = band * 32 + r, x = c * D2_CH - 2 * r + 2 * qcol;
                    uint2 v = make_uint2(0u, 0u);
                    if (yy < h && x >= 0 && x < w) v = *reinterpret_cast<const uint2 *>(frame + (long long)yy * w + x);
                    pre[2 * i] = v.x; pre[2 * i + 1] = v.y;
                }
            } else {
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const int r = 2 * i + hrow, yy = band * 32 + r, x = c * D2_CH - 2 * r + hcol;
                    pre[i] = (yy < h && x >= 0 && x < w) ? frame[(long long)yy * w + x] : 0u;
                }
            }
        };
        auto store_chunk = [&](int c) {
            uint32_t *t = s_in + (c & 1) * 32 * D2_IN_STRIDE;
            if (even_w) {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    uint32_t *q = t + (4 * i + qrow) * D2_IN_STRIDE + 2 * qcol;
                    q[0] = pre[2 * i]; q[1] = pre[2 * i + 1];
                }
            } else {
#pragma unroll
                for (int i = 0; i < 16; ++i) t[(2 * i + hrow) * D2_IN_STRIDE + hcol] = pre[i];
            }
        };
        load_chunk(0); store_chunk(0);
        __syncwarp();
        for (int c = 0; c < nchunks; ++c) {
            const int t0 = c * D2_CH;
            if (c + 1 < nchunks) load_chunk(c + 1);              // in flight while this chunk computes
            if (band > 0) {                                      // stay behind the band above's last row
                const int need = min(w, t0 + D2_CH + 1);
                if (lane == 0) {
                    if (prev_remote) { while (gprog[band - 1] < need) __nanosleep(a.spin_ns()); __threadfence(); }
                    else { while (s_progress[lb - 1] < need) __nanosleep(a.spin_ns()); __threadfence_block(); }
                }
                __syncwarp();
                const int bx = t0 + 1 + lane;                    // lane 0 consumes column t+1 at step t
                if (lane < D2_CH) s_bnd[lane] = bx < w ? __ldcg(bin + bx) : make_uint4(0u, 0u, 0u, 0u);
                if (c == 0 && lane == 0) { const uint4 q = __ldcg(bin); a0.r = q.x; a0.g = q.y; a0.b = q.z; }   // (0, y-1): lane 0 has no warm-up step
                __syncwarp();
            }
            const uint32_t *tin = s_in + (c & 1) * 32 * D2_IN_STRIDE + lane * D2_IN_STRIDE;
            const bool interior = (t0 - 62 >= 1) && (t0 + D2_CH - 1 <= w - 2) && (band * 32 + 31 < h - 1);
            if (interior) {
#pragma unroll 4
                for (int j = 0; j < D2_CH; ++j) {
                    TapW n;
                    n.r = __shfl_up_sync(0xffffffffu, own.r, 1); n.g = __shfl_up_sync(0xffffffffu, own.g, 1); n.b = __shfl_up_sync(0xffffffffu, own.b, 1);
                    if (lane == 0) { if (band > 0) { const uint4 q = s_bnd[j]; n.r = q.x; n.g = q.y; n.b = q.z; } else n = Z; }
                    a2 = a1; a1 = a0; a0 = n;
                    const uint32_t px = tin[j];
                    uint32_t vrg = prmt(px, 0u, 0x4140u), vb = prmt(px, 0u, 0x4442u);
                    vrg = add_clamp(vrg, tap_rg<3>(a2)); vb = add_clamp(vb, tap_b<3>(a2));        // 1/16 from (x-1, y-1)
                    vrg = add_clamp(vrg, tap_rg<2>(a1)); vb = add_clamp(vb, tap_b<2>(a1));        // 5/16 from (x,   y-1)
                    vrg = add_clamp(vrg, tap_rg<1>(a0)); vb = add_clamp(vb, tap_b<1>(a0));        // 3/16 from (x+1, y-1)
                    vrg = add_clamp(vrg, tap_rg<0>(own)); vb = add_clamp(vb, tap_b<0>(own));      // 7/16 from (x-1, y)
                    const uint32_t cell = ((vrg & 0xf8u) << 7) | ((vrg >> 14) & 0x3e0u) | (vb >> 3);
                    const uint32_t ci = s_lut[cell];
                    const uint2 np = s_pal2[ci];
                    const uint32_t erg = vrg + np.x, eb = vb + np.y;                                // error + 256 per half
                    own.r = s_tap[erg & 0x1ffu]; own.g = s_tap[erg >> 16]; own.b = s_tap[eb & 0x1ffu];
                    s_out[lane * D2_OUT_STRIDE + j] = (uint8_t)ci;
                    if (lane == 31) __stcg(bout + (t0 + j - 62), make_uint4(own.r, own.g, own.b, 0u));
                }
            } else {
#pragma unroll 2
                for (int j = 0; j < D2_CH; ++j) {
                    const int t = t0 + j, x = t - 2 * lane;
                    TapW n;
                    n.r = __shfl_up_sync(0xffffffffu, own.r, 1); n.g = __shfl_up_sync(0xffffffffu, own.g, 1); n.b = __shfl_up_sync(0xffffffffu, own.b, 1);
                    if (lane == 0) { if (band > 0) { const uint4 q = s_bnd[j]; n.r = q.x; n.g = q.y; n.b = q.z; } else n = Z; }
                    a2 = a1; a1 = a0; a0 = n;
                    uint32_t ci = 0;
                    if (x >= 0 && x < w && row_ok) {
                        const uint32_t px = tin[j];
                        uint32_t vrg = prmt(px, 0u, 0x4140u), vb = prmt(px, 0u, 0x4442u);
                        vrg = add_clamp(vrg, tap_rg<3>(a2)); vb = add_clamp(vb, tap_b<3>(a2));
                        vrg = add_clamp(vrg, tap_rg<2>(a1)); vb = add_clamp(vb, tap_b<2>(a1));
                        vrg = add_clamp(vrg, tap_rg<1>(a0)); vb = add_clamp(vb, tap_b<1>(a0));
                        if (x == w - 1) { vrg = add_clamp(vrg, tap_rg<1>(e_first)); vb = add_clamp(vb, tap_b<1>(e_first)); }   // libsixel: (0,y)'s below-left tap
                        vrg = add_clamp(vrg, tap_rg<0>(own)); vb = add_clamp(vb, tap_b<0>(own));
                        const uint32_t cell = ((vrg & 0xf8u) << 7) | ((vrg >> 14) & 0x3e0u) | (vb >> 3);
                        ci = s_lut[cell];
                        if (x < w - 1 && !last_row) {
                            const uint2 np = s_pal2[ci];
                            const uint32_t erg = vrg + np.x, eb = vb + np.y;
                            own.r = s_tap[erg & 0x1ffu]; own.g = s_tap[erg >> 16]; own.b = s_tap[eb & 0x1ffu];
                        } else {
                            own = Z;
                        }
                        if (x == 0) e_first = own;
                        if (lane == 31) __stcg(bout + x, make_uint4(own.r, own.g, own.b, 0u));
                    } else if (x >= w) {
                        own = Z;
                    }
                    s_out[lane * D2_OUT_STRIDE + j] = (uint8_t)ci;
                }
            }
            __syncwarp();
            // write this chunk's indices: 16 contiguous bytes per row -- as 8 two-byte stores (even widths) or 16 single bytes
            if (even_w) {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int r = 4 * i + qrow, yy = band * 32 + r, x = t0 - 2 * r + 2 * qcol;
                    if (yy < h && x >= 0 && x < w)
                        *reinterpret_cast<unsigned short *>(index + (long long)yy * w + x) =
                            *reinterpret_cast<const unsigned short *>(s_out + r * D2_OUT_STRIDE + 2 * qcol);
                }
            } else {
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const int r = 2 * i + hrow, yy = band * 32 + r, x = t0 - 2 * r + hcol;
                    if (yy < h && x >= 0 && x < w) index[(long long)yy * w + x] = s_out[r * D2_OUT_STRIDE + hcol];
                }
            }
            {   // publish progress: lane 31's boundary stores of this chunk are ordered before the flag
                const int done = min(w, t0 + D2_CH - 62);
                if (lane == 31 && done > 0) {
                    if (publish_remote) { __threadfence(); gprog[band] = done; }
                    __threadfence_block();
                    s_progress[lb] = done;
                }
            }
            if (c + 1 < nchunks) store_chunk(c + 1);
            __syncwarp();
        }
    }
}

size_t sixel_dither_workspace(int w, int h, int n_frames, size_t *o_bnd, size_t *o_prog) {
    const size_t nb32 = (size_t)(h + 31) / 32;
    size_t off = 0;
    *o_bnd = off; off += (sizeof(uint4) * nb32 * (size_t)w * n_frames + 255) / 256 * 256;
    *o_prog = off; off += (sizeof(int) * nb32 * n_frames + 255) / 256 * 256;
    return off;
}

SixelDitherShape sixel_dither_shape(int nb32, int n_frames, int n_total, int sm_count, bool env) {
    SixelDitherShape S;
    // CTAs per frame: 1 when the batch fills the GPU, more (up to one round of bands per CTA) for small batches.
    // All CTAs of a launch must be resident together when a frame is split (bands wait for the band above).
    int per_frame = 1;
    if (n_total < sm_count) {
        per_frame = std::max(1, std::min(sm_count / n_total, (nb32 + 7) / 8));
        if (const char *e = env ? getenv("B200TIMG_DITHER_SPLIT") : nullptr) per_frame = std::max(1, std::min(atoi(e), nb32));
        if ((long long)per_frame * n_frames > sm_count) per_frame = std::max(1, sm_count / n_frames);
    }
    S.bands_per_cta = (nb32 + per_frame - 1) / per_frame;
    S.per_frame = (nb32 + S.bands_per_cta - 1) / S.bands_per_cta;
    // warps per CTA: full rounds over the CTA's bands.  Fewer warps = more rounds but a smaller share of the time spent
    // filling and draining the band pipeline (each band starts ~80 columns behind the one above).
    int wmax = D2_WMAX;
    if (const char *e = env ? getenv("B200TIMG_DITHER_WARPS") : nullptr) wmax = std::max(1, std::min(atoi(e), D2_WMAX));
    S.rounds = (S.bands_per_cta + wmax - 1) / wmax;
    S.nwarps = (S.bands_per_cta + S.rounds - 1) / S.rounds;
    return S;
}

// n_frames: frames of this launch (fb, W, d_bnd and d_prog already point at its first frame); n_total: frames of the
// whole batch this launch is a slice of -- the "split a frame over several CTAs" decision looks at the batch, so a
// slice that shares the GPU with another slice does not spread itself over every SM.
int launch_sixel_dither(b200timg_ctx *ctx, const uint32_t *fb, int w, int h, int n_frames, int n_total, const SixelWork &W, void *d_bnd, void *d_prog) {
    Dither2Geom G;
    G.w = w; G.h = h; G.nb32 = (h + 31) / 32;
    // A chunk of 16 columns x 32 rows takes a warp several microseconds; polling the band above every 32 ns spends a
    // noticeable share of the kernel's issue slots in the wait loop, slots the producing warps need.
    G.spin_ns = 256;
    if (const char *e = getenv("B200TIMG_DITHER_SPIN")) G.spin_ns = (unsigned)std::max(0, std::min(atoi(e), 100000));
    const SixelDitherShape S = sixel_dither_shape(G.nb32, n_frames, n_total, ctx->sm_count, true);
    const int per_frame = S.per_frame;
    G.bands_per_cta = S.bands_per_cta;
    G.nwarps = S.nwarps;
    const size_t smem = 32768 + (size_t)G.nwarps * D2_WARP_SMEM;
    B2_CUDA(ctx, cudaFuncSetAttribute(sixel_dither2_kernel<DitherUniform>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32768 + D2_WMAX * D2_WARP_SMEM));
    if (per_frame > 1) B2_CUDA(ctx, cudaMemsetAsync(d_prog, 0, sizeof(int) * (size_t)G.nb32 * n_frames, ctx->stream));
    B2_KERNEL(ctx, "sixel_dither2_kernel");
    sixel_dither2_kernel<DitherUniform><<<dim3(per_frame, n_frames), G.nwarps * 32, smem, ctx->stream>>>(fb, G, W, static_cast<uint4 *>(d_bnd), static_cast<int *>(d_prog));
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

// One launch over every frame's dither CTAs (M.cta_start); the block size is the largest any frame asks for.
int launch_sixel_dither_mixed(b200timg_ctx *ctx, const uint32_t *fb, unsigned n_ctas, const MixedSixelParams &M, const SixelWork &W,
                              void *d_bnd, void *d_prog, size_t n_prog, bool split) {
    const size_t smem = 32768 + (size_t)M.nwarps * D2_WARP_SMEM;
    B2_CUDA(ctx, cudaFuncSetAttribute(sixel_dither2_kernel<DitherMixed>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32768 + D2_WMAX * D2_WARP_SMEM));
    if (split) B2_CUDA(ctx, cudaMemsetAsync(d_prog, 0, sizeof(int) * n_prog, ctx->stream));
    B2_KERNEL(ctx, "sixel_dither2_mixed_kernel");
    sixel_dither2_kernel<DitherMixed><<<n_ctas, M.nwarps * 32, smem, ctx->stream>>>(fb, M, W, static_cast<uint4 *>(d_bnd), static_cast<int *>(d_prog));
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

}  // namespace b200timg
