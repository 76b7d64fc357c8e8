// K1: ImageScaler::Scale on the device -- separable polyphase resampling of RGBA8 frames
// with the reference's (STB build) exact arithmetic: decode byte*(1/255), alpha-weighted
// 7-channel float pixels [R G B A R*A G*A B*A], horizontal taps alternating between two
// accumulators (or one when <=3 taps), vertical taps summed in input-row order, un-weight by
// 1/A unless A < 2^-120, encode trunc(clamp(v*255+0.5)).  Which axis runs first follows the
// reference's cost model (resample_tables.cu).  Every * and + is a separate IEEE rounding
// (__fmul_rn/__fadd_rn), like the reference's SSE2 code.
//
// Kernels: copies for unscaled frames; <= 8 taps per axis: the v3 kernel (FAST arithmetic, opaque tiles), the
// planar kernel (vertical first, rows of 16 bytes) and the fixed-tap kernel (either order); longer filters: the two
// 1-D passes of the twopass_* kernels.  Algorithmic bytes: 4*iw*ih read + 4*ow*oh written.
#include <algorithm>
#include <cstdlib>
#include <map>
#include <tuple>
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "resample_tables.h"

#ifndef CUSIM
#include <cuda.h>            // CUtensorMap: types only -- the encoder comes from the runtime's driver entry point, nothing links libcuda
#else
struct alignas(64) CUtensorMap { unsigned long long opaque[16]; };
#define __grid_constant__
#endif

namespace b200timg {

// ---- TMA (cp.async.bulk.tensor) staging of a source window: one thread issues the copy of a [rows][cols] box of the
// [frames][ih][iw] u32 tensor into shared memory, the hardware fills cells outside the image with zeros and signals an
// mbarrier with the byte count.  SASS: UTMALDG + SYNCS.
#ifndef CUSIM
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void *dst, const CUtensorMap *map, unsigned long long *bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(reinterpret_cast<unsigned long long>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
#endif

struct ResampleParams {
    int iw, ih, ow, oh, out_frame_rows, n_frames;
    int bgra;
    int h_widest, v_widest, h_sequential;
    const int32_t *h_first, *h_count, *h_lead, *v_first, *v_count;
    const float *h_coeff, *v_coeff;
    ComposeSpec cs;              // fused AlphaComposeBackground (cs.active == 0: none)
};

__device__ __forceinline__ uint32_t encode_px(const float *e) {
    float r = e[0], g = e[1], b = e[2];
    const float a = e[3];
    const float tiny = 7.5231638452626401e-37f;          // 2^-120
    if (!(a < tiny)) {
        const float ia = fdiv(1.0f, a);
        r = fmul(e[4], ia); g = fmul(e[5], ia); b = fmul(e[6], ia);
    }
    auto enc = [](float v) -> uint32_t {
        const float f = fadd(fmul(v, 255.0f), 0.5f);
        return __float2uint_rz(fminf(fmaxf(f, 0.0f), 255.0f));     // NaN -> 0 either way (cvt.rzi of NaN is 0)
    };
    return pack_rgba(enc(r), enc(g), enc(b), enc(a));
}

// byte k of p as a float without the (quarter-rate) I2F unit: 0x4B0000bb is 2^23 + bb exactly.
__device__ __forceinline__ float byte_f(uint32_t p, int k) {
    return fsub(__uint_as_float(__byte_perm(p, 0x4B000000u, 0x7540u | (uint32_t)k)), 8388608.0f);
}
__device__ __forceinline__ float4 decode_pm(uint32_t p, int bgra) {       // (R*A, G*A, B*A, A)
    const float k = 1.0f / 255.0f;
    const float c0 = fmul(byte_f(p, 0), k), c1 = fmul(byte_f(p, 1), k), c2 = fmul(byte_f(p, 2), k), a = fmul(byte_f(p, 3), k);
    const float r = bgra ? c2 : c0, b = bgra ? c0 : c2;
    return make_float4(fmul(r, a), fmul(c1, a), fmul(b, a), a);
}
__device__ __forceinline__ float4 decode_plain(uint32_t p, int bgra) {    // (R, G, B, -)
    const float k = 1.0f / 255.0f;
    const float c0 = fmul(byte_f(p, 0), k), c1 = fmul(byte_f(p, 1), k), c2 = fmul(byte_f(p, 2), k);
    return make_float4(bgra ? c2 : c0, c1, bgra ? c0 : c2, 0.0f);
}
// pass 0: (R*A, G*A, B*A, A); pass 1: (R, G, B, 0) -- one code path: the weight is A or 1.0 (x*1.0f is exact)
__device__ __forceinline__ float4 decode_sel(uint32_t p, int bgra, bool plain) {
    const float k = 1.0f / 255.0f;
    const float c0 = fmul(byte_f(p, 0), k), c1 = fmul(byte_f(p, 1), k), c2 = fmul(byte_f(p, 2), k), a = fmul(byte_f(p, 3), k);
    const float r = bgra ? c2 : c0, b = bgra ? c0 : c2, m = plain ? 1.0f : a;
    return make_float4(fmul(r, m), fmul(c1, m), fmul(b, m), plain ? 0.0f : a);
}
__device__ __forceinline__ float4 mul4(float4 v, float w) { return make_float4(fmul(v.x, w), fmul(v.y, w), fmul(v.z, w), fmul(v.w, w)); }
__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(fadd(a.x, b.x), fadd(a.y, b.y), fadd(a.z, b.z), fadd(a.w, b.w)); }

// ---- fixed-tap fast path ------------------------------------------------------------------
// One CTA produces a tile of output pixels.  The input window the tile needs is decoded ONCE into shared memory as
// float4 pixels, the first pass (vertical or horizontal, whichever the reference's cost model picks) writes a float4
// intermediate tile to shared memory, the second pass reads it.  Only 4 of the 7 channels are carried (A, R*A, G*A,
// B*A): the un-weighted R,G,B are needed only where the filtered alpha is < 2^-120 (fully transparent output), and
// tiles that contain such a pixel run a second pass for them.  The kernel is specialised so the inner loops carry no
// predicates and no run-time trip counts: every output uses exactly HC horizontal and VC vertical taps (the
// per-axis widest count rounded up to 2/4/6/8); taps an output does not have are zero coefficients
// reading staged (finite) pixels, which adds +0 and changes nothing.  The staged window is padded
// accordingly (zeros outside the image), its origin per tile column/row comes from the host.
struct FixedGeom { int nix, niy; const int32_t *tile_ix0, *tile_iy0; };
constexpr int FTW = 64;

template <bool VFIRST, int HC, int VC, int TH, int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB)
resample_fixed_kernel(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, ResampleParams P, FixedGeom G) {
    extern __shared__ float4 s_px[];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, f = blockIdx.z;
    const int ox0 = blockIdx.x * FTW, oy0 = blockIdx.y * TH;
    const int ix0 = G.tile_ix0[blockIdx.x], iy0 = G.tile_iy0[blockIdx.y];
    const int nix = G.nix, niy = G.niy;
    float4 *Din = s_px;
    float4 *T = s_px + (size_t)niy * nix;
    int *s_hfirst = reinterpret_cast<int *>(T + (VFIRST ? TH * nix : niy * FTW));   // [FTW]
    int *s_vfirst = s_hfirst + FTW;                                                   // [TH]
    float *s_hc = reinterpret_cast<float *>(s_vfirst + TH);                          // [FTW][HC+1]
    float *s_vc = s_hc + FTW * (HC + 1);                                              // [TH][VC+1]
    if (tid < FTW) {
        const int ox = ox0 + tid;
        const bool ok = ox < P.ow;
        s_hfirst[tid] = ok ? P.h_first[ox] - ix0 : 0;
#pragma unroll
        for (int i = 0; i < HC; ++i) s_hc[tid * (HC + 1) + i] = (ok && i < P.h_widest) ? P.h_coeff[(long long)ox * P.h_widest + i] : 0.0f;
    } else if (tid < FTW + TH) {
        const int t = tid - FTW, oy = oy0 + t;
        const bool ok = oy < P.oh;
        s_vfirst[t] = ok ? P.v_first[oy] - iy0 : 0;
#pragma unroll
        for (int i = 0; i < VC; ++i) s_vc[t * (VC + 1) + i] = (ok && i < P.v_widest) ? P.v_coeff[(long long)oy * P.v_widest + i] : 0.0f;
    }
    const uint32_t *src = in + (long long)f * P.iw * P.ih;
    const bool hseq = P.h_sequential != 0;
    const float tiny = 7.5231638452626401e-37f;       // 2^-120
    constexpr int NW = NT / 32, RSTEP = NT / FTW, RPT = TH / RSTEP;   // warps, row stride, rows per thread
    const int tx = tid & (FTW - 1), tyb = tid >> 6;   // this thread's pixels: column tx, rows tyb + RSTEP*q

    float4 res[RPT], plain[RPT];
    bool need_plain = false;
    for (int pass = 0; pass < 2; ++pass) {
        // stage + decode the window once.  All of a thread's global loads (up to 4 rows x 4 column
        // groups) are issued before the first one is consumed, so their latencies overlap.
        for (int ly0 = 0; ly0 < niy; ly0 += 4 * NW)
            for (int lx0 = 0; lx0 < nix; lx0 += 128) {
                uint32_t pv[4][4];
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const int ly = ly0 + wid + r * NW, y = iy0 + ly;
                    const uint32_t *row = src + (long long)y * P.iw + ix0;
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const int lx = lx0 + lane + 32 * c;
                        pv[r][c] = (ly < niy && lx < nix && y < P.ih && ix0 + lx < P.iw) ? row[lx] : 0u;
                    }
                }
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const int ly = ly0 + wid + r * NW;
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const int lx = lx0 + lane + 32 * c;
                        if (ly < niy && lx < nix) Din[ly * nix + lx] = decode_sel(pv[r][c], P.bgra, pass != 0);
                    }
                }
            }
        __syncthreads();
        float4 acc[RPT];
        if (VFIRST) {
#pragma unroll
            for (int r = 0; r < TH / NW; ++r) {
                const int ty = wid + r * NW;
                float vc[VC];
#pragma unroll
                for (int k = 0; k < VC; ++k) vc[k] = s_vc[ty * (VC + 1) + k];
                const float4 *rp[VC];
#pragma unroll
                for (int k = 0; k < VC; ++k) rp[k] = Din + (s_vfirst[ty] + k) * nix + lane;
                float4 *trow = T + ty * nix + lane;
                for (int lx0 = 0; lx0 < nix; lx0 += 128) {
#pragma unroll
                    for (int it = 0; it < 4; ++it) {
                        const int o = lx0 + 32 * it;
                        if (o + lane < nix) {
                            float4 a = mul4(rp[0][o], vc[0]);
#pragma unroll
                            for (int k = 1; k < VC; ++k) a = add4(a, mul4(rp[k][o], vc[k]));
                            trow[o] = a;
                        }
                    }
                }
            }
            __syncthreads();
            float hc[HC];
#pragma unroll
            for (int i = 0; i < HC; ++i) hc[i] = s_hc[tx * (HC + 1) + i];
            const float4 *tbase = T + s_hfirst[tx];
#pragma unroll
            for (int q = 0; q < RPT; ++q) {
                const float4 *row = tbase + (tyb + RSTEP * q) * nix;
                if (hseq) {
                    float4 a = mul4(row[0], hc[0]);
#pragma unroll
                    for (int i = 1; i < (HC < 3 ? HC : 3); ++i) a = add4(a, mul4(row[i], hc[i]));
                    acc[q] = a;
                } else {
                    float4 a0 = mul4(row[0], hc[0]), a1 = mul4(row[1], hc[1]);
#pragma unroll
                    for (int i = 2; i < HC; ++i) { if (i & 1) a1 = add4(a1, mul4(row[i], hc[i])); else a0 = add4(a0, mul4(row[i], hc[i])); }
                    acc[q] = add4(a0, a1);
                }
            }
        } else {
            float hc[HC];
#pragma unroll
            for (int i = 0; i < HC; ++i) hc[i] = s_hc[tx * (HC + 1) + i];
            const int hn0 = s_hfirst[tx];
            for (int ly = tyb; ly < niy; ly += RSTEP) {
                const float4 *row = Din + ly * nix + hn0;
                float4 r;
                if (hseq) {
                    r = mul4(row[0], hc[0]);
#pragma unroll
                    for (int i = 1; i < (HC < 3 ? HC : 3); ++i) r = add4(r, mul4(row[i], hc[i]));
                } else {
                    float4 a0 = mul4(row[0], hc[0]), a1 = mul4(row[1], hc[1]);
#pragma unroll
                    for (int i = 2; i < HC; ++i) { if (i & 1) a1 = add4(a1, mul4(row[i], hc[i])); else a0 = add4(a0, mul4(row[i], hc[i])); }
                    r = add4(a0, a1);
                }
                T[ly * FTW + tx] = r;
            }
            __syncthreads();
#pragma unroll
            for (int q = 0; q < RPT; ++q) {
                const int ty = tyb + RSTEP * q;
                const float4 *col = T + s_vfirst[ty] * FTW + tx;
                const float *vc = s_vc + ty * (VC + 1);
                float4 a = mul4(col[0], vc[0]);
#pragma unroll
                for (int k = 1; k < VC; ++k) a = add4(a, mul4(col[k * FTW], vc[k]));
                acc[q] = a;
            }
        }
#pragma unroll
        for (int q = 0; q < RPT; ++q) { if (pass == 0) res[q] = acc[q]; else plain[q] = acc[q]; }
        if (pass == 0) {
#pragma unroll
            for (int q = 0; q < RPT; ++q) if (ox0 + tx < P.ow && oy0 + tyb + RSTEP * q < P.oh && res[q].w < tiny) need_plain = true;
            if (!__syncthreads_or(need_plain)) break;
        }
    }
    if (ox0 + tx < P.ow) {
#pragma unroll
        for (int q = 0; q < RPT; ++q) {
            const int oy = oy0 + tyb + RSTEP * q;
            if (oy < P.oh) {
                float v[7];
                v[3] = res[q].w; v[4] = res[q].x; v[5] = res[q].y; v[6] = res[q].z;
                const bool transparent = res[q].w < tiny;
                v[0] = transparent ? plain[q].x : 0.f; v[1] = transparent ? plain[q].y : 0.f; v[2] = transparent ? plain[q].z : 0.f;
                out[((long long)f * P.out_frame_rows + oy) * P.ow + ox0 + tx] = compose_at(P.cs, encode_px(v), ox0 + tx, oy);
            }
        }
    }
}

// ---- planar fast path (vertical pass first, <= 8 taps per axis) ---------------------------
// Same arithmetic again, reorganised around what limits resample_fixed_kernel (shared-memory
// wavefronts and issue slots): every filtered channel is an independent plane, so the
// window is staged as separate float planes and
//   * the vertical pass produces 4 neighbouring columns per thread (one LDS.128 per tap and plane),
//   * the horizontal pass maps lanes to output ROWS: a warp works on one output column at a time, its
//     taps and start index are warp-uniform and every tap is one conflict-free wavefront (odd pitch),
//   * the encoded pixels go through a small transpose buffer so global stores stay coalesced.
// Channel passes: a tile whose window is fully opaque (the common case: photos, video) needs only the
// three colour planes -- decoded alpha is exactly 1.0f (255 * fl(1/255) rounds to 1), so R*A == R, and
// the filtered alpha is the same tap sum over the constant 1.0, computed from the coefficients alone in
// the same order.  Other tiles run (R*A, G*A, B*A), then A, and -- only if some output alpha is
// < 2^-120 -- the un-weighted (R, G, B) planes, exactly like the float4 kernels above.
struct PlanarGeom { int nix, niy, sp, tp; unsigned grp_magic; const int32_t *tile_ix0, *tile_iy0; };   // grp_magic: floor(2^32/(sp/4))+1
constexpr int PTH = 32;          // output rows per tile (= lanes of the horizontal pass)
constexpr int PNT = 256;

template <int HC, int VC, int PTW>
__device__ __forceinline__ void resample_planar_body(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, const ResampleParams &P,
                                                     const PlanarGeom &G, int bx, int by, int f) {
    extern __shared__ float4 s_px[];
    float *S = reinterpret_cast<float *>(s_px);                   // [3][niy][sp]
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int ox0 = bx * PTW, oy0 = by * PTH;
    const int ix0 = G.tile_ix0[bx], iy0 = G.tile_iy0[by];
    const int niy = G.niy, sp = G.sp, tp = G.tp;
    const int splane = niy * sp, tplane = PTH * tp;
    float *T = S + 3 * splane;                                    // [3][PTH][tp]
    float *s_hc = T + 3 * tplane + ((4 - ((3 * tplane) & 3)) & 3); // [PTW][8], 16-byte aligned
    float *s_vc = s_hc + PTW * 8;                                 // [PTH][8]
    int *s_hfirst = reinterpret_cast<int *>(s_vc + PTH * 8);      // [PTW]
    int *s_vfirst = s_hfirst + PTW;                               // [PTH]
    uint32_t *O = reinterpret_cast<uint32_t *>(S);                // [PTH][PTW+1], reuses S after the last pass
    if (tid < PTW) {
        const int ox = ox0 + tid;
        const bool ok = ox < P.ow;
        s_hfirst[tid] = ok ? P.h_first[ox] - ix0 : 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) s_hc[tid * 8 + i] = (ok && i < P.h_widest) ? P.h_coeff[(long long)ox * P.h_widest + i] : 0.0f;
    } else if (tid < PTW + PTH) {
        const int t = tid - PTW, oy = oy0 + t;
        const bool ok = oy < P.oh;
        s_vfirst[t] = ok ? P.v_first[oy] - iy0 : 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) s_vc[t * 8 + i] = (ok && i < P.v_widest) ? P.v_coeff[(long long)oy * P.v_widest + i] : 0.0f;
    }
    const uint32_t *src = in + (long long)f * P.iw * P.ih;
    const bool hseq = P.h_sequential != 0;
    const int kr = P.bgra ? 2 : 0, kb = P.bgra ? 0 : 2;          // byte index of R and B in the source pixel
    const float tiny = 7.5231638452626401e-37f;       // 2^-120
    const float k255 = 1.0f / 255.0f;
    constexpr int NJ = PTW / 8;                       // output columns per warp: wid + 8*j, row = lane
    const int ngrp = sp >> 2;                         // 4-column groups per window row
    const int n_stage = niy * ngrp;

    // ---- staging: a unit is 4 neighbouring source pixels (one 16-byte load) -> one float4 per plane
    uint4 raw[4];
    int soff[4];                                      // S offset of the unit, -1: none
    auto load_chunk = [&](int u0) -> bool {           // all loads of a thread are issued before the first use
        bool ok255 = true;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int u = u0 + tid + r * PNT;
            const int ly = (int)__umulhi((unsigned)u, G.grp_magic), g = u - ly * ngrp;
            const int y = iy0 + ly, x = ix0 + 4 * g;
            raw[r] = make_uint4(0u, 0u, 0u, 0u);
            soff[r] = u < n_stage ? ly * sp + 4 * g : -1;
            if (u < n_stage && y < P.ih && x < P.iw) {
                raw[r] = __ldg(reinterpret_cast<const uint4 *>(src + (long long)y * P.iw + x));
                ok255 = ok255 && ((raw[r].x & raw[r].y & raw[r].z & raw[r].w) >= 0xff000000u);
            }
        }
        return ok255;
    };
    // mode 0: R*A,G*A,B*A   1: A   2: R,G,B
    auto decode_chunk = [&](int mode) {
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            if (soff[r] < 0) continue;
            const uint32_t pv[4] = {raw[r].x, raw[r].y, raw[r].z, raw[r].w};
            float *d = S + soff[r];
            if (mode == 1) {
                *reinterpret_cast<float4 *>(d) = make_float4(fmul(byte_f(pv[0], 3), k255), fmul(byte_f(pv[1], 3), k255),
                                                             fmul(byte_f(pv[2], 3), k255), fmul(byte_f(pv[3], 3), k255));
                continue;
            }
            float c[3][4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                c[0][e] = fmul(byte_f(pv[e], kr), k255); c[1][e] = fmul(byte_f(pv[e], 1), k255); c[2][e] = fmul(byte_f(pv[e], kb), k255);
                if (mode == 0) {
                    const float a = fmul(byte_f(pv[e], 3), k255);
                    c[0][e] = fmul(c[0][e], a); c[1][e] = fmul(c[1][e], a); c[2][e] = fmul(c[2][e], a);
                }
            }
            *reinterpret_cast<float4 *>(d) = make_float4(c[0][0], c[0][1], c[0][2], c[0][3]);
            *reinterpret_cast<float4 *>(d + splane) = make_float4(c[1][0], c[1][1], c[1][2], c[1][3]);
            *reinterpret_cast<float4 *>(d + 2 * splane) = make_float4(c[2][0], c[2][1], c[2][2], c[2][3]);
        }
    };
    auto stage = [&](int mode, bool have_first_chunk) {
        for (int u0 = 0; u0 < n_stage; u0 += 4 * PNT) {
            if (!(have_first_chunk && u0 == 0)) load_chunk(u0);
            if (mode == 0) decode_chunk(0); else if (mode == 1) decode_chunk(1); else decode_chunk(2);
        }
    };
    // ---- vertical: T[c][ty][4g..4g+3] = sum_k S[c][vfirst[ty]+k][4g..] * vc[ty][k], rows in order.
    // A warp covers 4 output rows x 8 column groups: with an odd T pitch its scalar stores hit 32
    // different banks, and each LDS.128 touches four 128-byte row segments (the minimum).
    auto vertical = [&](auto np_tag) {
        constexpr int NP = decltype(np_tag)::value;
        const int ty = 4 * wid + (lane >> 3);
        const float4 v0 = *reinterpret_cast<const float4 *>(s_vc + ty * 8), v1 = *reinterpret_cast<const float4 *>(s_vc + ty * 8 + 4);
        const float vc[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
        const float *sb = S + s_vfirst[ty] * sp + 4 * (lane & 7);
        float *t = T + ty * tp + 4 * (lane & 7);
        for (int g = lane & 7; g < ngrp; g += 8, sb += 32, t += 32) {
#pragma unroll
            for (int c = 0; c < NP; ++c) {
                float4 a = mul4(*reinterpret_cast<const float4 *>(sb + c * splane), vc[0]);
#pragma unroll
                for (int k = 1; k < VC; ++k) a = add4(a, mul4(*reinterpret_cast<const float4 *>(sb + c * splane + k * sp), vc[k]));
                float *tc = t + c * tplane;
                tc[0] = a.x; tc[1] = a.y; tc[2] = a.z; tc[3] = a.w;
            }
        }
    };
    // tap sum of one output: HC taps alternating between two accumulators (or sequential when <= 3 taps)
    auto hsum1 = [&](auto tap, const float *hc) -> float {
        if (hseq) {
            float a = fmul(tap(0), hc[0]);
#pragma unroll
            for (int i = 1; i < (HC < 3 ? HC : 3); ++i) a = fadd(a, fmul(tap(i), hc[i]));
            return a;
        }
        float a0 = fmul(tap(0), hc[0]), a1 = fmul(tap(1), hc[1]);
#pragma unroll
        for (int i = 2; i < HC; ++i) { if (i & 1) a1 = fadd(a1, fmul(tap(i), hc[i])); else a0 = fadd(a0, fmul(tap(i), hc[i])); }
        return fadd(a0, a1);
    };
    // ---- horizontal: lane = output row, the warp's column changes with j
    auto horizontal = [&](auto np_tag, float (*r)[3]) {
        constexpr int NP = decltype(np_tag)::value;
        const float *trow = T + lane * tp;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const int tx = wid + 8 * j;
            const float4 h0 = *reinterpret_cast<const float4 *>(s_hc + tx * 8), h1 = *reinterpret_cast<const float4 *>(s_hc + tx * 8 + 4);
            const float hc[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
            const float *row = trow + s_hfirst[tx];
#pragma unroll
            for (int c = 0; c < NP; ++c) {
                const float *rc = row + c * tplane;
                r[j][c] = hsum1([&](int i) { return rc[i]; }, hc);
            }
        }
    };
    using I1 = std::integral_constant<int, 1>;
    using I3 = std::integral_constant<int, 3>;

    float pm[NJ][3], al[NJ], pl[NJ][3];
    bool have_pl = false;
    // is every pixel of the window opaque?  (decoded alpha is then exactly 1.0f)
    bool ok255 = load_chunk(0);
    for (int u0 = 4 * PNT; u0 < n_stage; u0 += 4 * PNT) ok255 = load_chunk(u0) && ok255;
    const bool opaque = __syncthreads_and(ok255) != 0;           // also orders the table writes above
    const bool one_chunk = n_stage <= 4 * PNT;                   // then raw[] still holds the window
#pragma unroll 1
    for (int rep = 0; rep < 2; ++rep) {
        // rep 0: weighted colour planes (un-weighted == weighted when opaque); rep 1: un-weighted colour planes
        if (rep == 0 && !opaque) stage(0, one_chunk); else stage(2, rep == 0 && one_chunk);
        __syncthreads();
        vertical(I3());
        __syncthreads();
        if (rep == 1) { horizontal(I3(), pl); have_pl = true; break; }
        horizontal(I3(), pm);
        if (opaque) {
            // filtered alpha of an all-ones window: the same two tap sums over the constant 1.0f
            const float4 v0 = *reinterpret_cast<const float4 *>(s_vc + lane * 8), v1 = *reinterpret_cast<const float4 *>(s_vc + lane * 8 + 4);
            const float vc[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
            float av = vc[0];
#pragma unroll
            for (int k = 1; k < VC; ++k) av = fadd(av, vc[k]);
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
                const int tx = wid + 8 * j;
                const float4 h0 = *reinterpret_cast<const float4 *>(s_hc + tx * 8), h1 = *reinterpret_cast<const float4 *>(s_hc + tx * 8 + 4);
                const float hc[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
                al[j] = hsum1([&](int) { return av; }, hc);
            }
            break;
        }
        // alpha plane
        __syncthreads();                               // T of the colour pass has been consumed
        stage(1, false);
        __syncthreads();
        vertical(I1());
        __syncthreads();
        float a1[NJ][3];
        horizontal(I1(), a1);
        bool need_plain = false;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            al[j] = a1[j][0];
            if (ox0 + wid + 8 * j < P.ow && oy0 + lane < P.oh && al[j] < tiny) need_plain = true;
        }
        if (!__syncthreads_or(need_plain)) break;
    }
    __syncthreads();                                   // every warp is done with S and T
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
        const int tx = wid + 8 * j;
        float v[7];
        v[3] = al[j]; v[4] = pm[j][0]; v[5] = pm[j][1]; v[6] = pm[j][2];
        if (have_pl) { v[0] = pl[j][0]; v[1] = pl[j][1]; v[2] = pl[j][2]; }      // only read when al < 2^-120
        else { v[0] = pm[j][0]; v[1] = pm[j][1]; v[2] = pm[j][2]; }
        O[lane * (PTW + 1) + tx] = compose_at(P.cs, encode_px(v), ox0 + tx, oy0 + lane);
    }
    __syncthreads();
    {
        static_assert(PTW == 32, "store loop maps a lane to a column");
        uint32_t *orow = out + ((long long)f * P.out_frame_rows + oy0 + wid) * P.ow + ox0 + lane;
        const bool col_ok = ox0 + lane < P.ow;
#pragma unroll
        for (int i = 0; i < PTH / 8; ++i)
            if (col_ok && oy0 + wid + 8 * i < P.oh) orow[(long long)(8 * i) * P.ow] = O[(wid + 8 * i) * (PTW + 1) + lane];
    }
}

template <int HC, int VC, int PTW, int MINB>
__global__ void __launch_bounds__(PNT, MINB)
resample_planar_kernel(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, ResampleParams P, PlanarGeom G) {
    resample_planar_body<HC, VC, PTW>(in, out, P, G, blockIdx.x, blockIdx.y, blockIdx.z);
}

// The same tiles driven by a work list (tiles the opaque-only v3 kernel handed back): list[0] = number of
// 64x32 v3 tiles, list[1 + 3k ..] = (v3 tile x, tile y, frame); each is two 32x32 planar tiles.
template <int HC, int VC, int MINB>
__global__ void __launch_bounds__(PNT, MINB)
resample_planar_list_kernel(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, ResampleParams P, PlanarGeom G,
                            const uint32_t *__restrict__ list) {
    const uint32_t n = list[0] * 2u;
    for (uint32_t e = blockIdx.x; e < n; e += gridDim.x) {
        const uint32_t *t = list + 1 + 3 * (e >> 1);
        const int bx = (int)t[0] * 2 + (int)(e & 1u);
        if (bx * 32 < P.ow) resample_planar_body<HC, VC, 32>(in, out, P, G, bx, (int)t[1], (int)t[2]);
        __syncthreads();
    }
}

typedef void (*PlanarFn)(const uint32_t *, uint32_t *, ResampleParams, PlanarGeom);
template <int HC, int PTW, int MINB>
static PlanarFn planar_v(int vc) {
    switch (vc) {
    case 2: return resample_planar_kernel<HC, 2, PTW, MINB>;
    case 4: return resample_planar_kernel<HC, 4, PTW, MINB>;
    case 6: return resample_planar_kernel<HC, 6, PTW, MINB>;
    default: return resample_planar_kernel<HC, 8, PTW, MINB>;
    }
}
template <int PTW, int MINB>
static PlanarFn planar_h(int hc, int vc) {
    switch (hc) {
    case 2: return planar_v<2, PTW, MINB>(vc);
    case 4: return planar_v<4, PTW, MINB>(vc);
    case 6: return planar_v<6, PTW, MINB>(vc);
    default: return planar_v<8, PTW, MINB>(vc);
    }
}

typedef void (*FixedFn)(const uint32_t *, uint32_t *, ResampleParams, FixedGeom);
struct FixedVariant { FixedFn fn; int th, nt; };
// Tile 64x16, 256 threads, 3 CTAs/SM (80 registers of the SM's 64 K), chosen among {16x256x3, 16x256x4,
// 8x128x8, 8x256x4, 16x512x2, 32x512x2} for C2 frames.
template <bool VF, int HC>
static FixedVariant fixed_v(int vc) {
    switch (vc) {
    case 2: return {resample_fixed_kernel<VF, HC, 2, 16, 256, 3>, 16, 256};
    case 4: return {resample_fixed_kernel<VF, HC, 4, 16, 256, 3>, 16, 256};
    case 6: return {resample_fixed_kernel<VF, HC, 6, 16, 256, 3>, 16, 256};
    default: return {resample_fixed_kernel<VF, HC, 8, 16, 256, 3>, 16, 256};
    }
}
template <bool VF>
static FixedVariant fixed_h(int hc, int vc) {
    switch (hc) {
    case 2: return fixed_v<VF, 2>(vc);
    case 4: return fixed_v<VF, 4>(vc);
    case 6: return fixed_v<VF, 6>(vc);
    default: return fixed_v<VF, 8>(vc);
    }
}
static int fixed_class(int widest) { return widest <= 2 ? 2 : widest <= 4 ? 4 : widest <= 6 ? 6 : 8; }


// ---- two-pass kernels for long filters (> 8 taps on an axis: strong downscales such as 4K -> a grid cell,
// 1080p -> 160 columns) -----------------------------------------------------------------------------
// The fixed-tap kernels above stage a whole 2-D window per tile; with 24..48 taps per axis the window no longer
// fits and its halo dwarfs the tile.  Here each pass is a plain 1-D filter over a float4 intermediate image
// (R*A, G*A, B*A, A) kept in global memory (a few MB per frame, written and read once):
//   pass 1 (the axis the reference's cost model runs first) decodes the source bytes on the fly,
//   pass 2 filters the intermediate, un-weights, encodes, composes.
// The reference's arithmetic and summation order (vertical taps in row order; horizontal taps alternating between two
// accumulators, or sequential when <= 3).  Output pixels whose filtered alpha is below
// 2^-120 need the un-weighted colour planes: pass 2 raises a per-frame flag for them and a second pair of
// passes (which return at once when the flag is down -- always, for opaque sources) fills them in.
struct TwoPassParams {
    ResampleParams P;
    float4 *tmp;                 // [n_frames][first-pass rows][first-pass cols]
    int *need_plain;             // [n_frames] raised by the weighted second pass
    unsigned char *mask;         // [n_frames][oh][ow] 1 = this pixel's filtered alpha is < 2^-120
};

template <bool PLAIN> __device__ __forceinline__ float4 decode_tp(uint32_t p, int bgra) { return PLAIN ? decode_plain(p, bgra) : decode_pm(p, bgra); }

// pass 1, vertical first: tmp[oy][x] = sum_k decode(src[vfirst[oy] + k][x]) * vc[oy][k]
template <bool PLAIN>
__global__ void __launch_bounds__(256)
twopass_v1_kernel(const uint32_t *__restrict__ in, TwoPassParams T) {
    const ResampleParams &P = T.P;
    const int x = blockIdx.x * 256 + threadIdx.x, oy = blockIdx.y, f = blockIdx.z;
    if (PLAIN && !T.need_plain[f]) return;
    if (x >= P.iw) return;
    const uint32_t *src = in + (long long)f * P.iw * P.ih + (long long)P.v_first[oy] * P.iw + x;
    const float *vc = P.v_coeff + (long long)oy * P.v_widest;
    const int cnt = P.v_count[oy];
    float4 a = mul4(decode_tp<PLAIN>(src[0], P.bgra), vc[0]);
    for (int k = 1; k < cnt; ++k) a = add4(a, mul4(decode_tp<PLAIN>(src[(long long)k * P.iw], P.bgra), vc[k]));
    T.tmp[((long long)f * P.oh + oy) * P.iw + x] = a;
}
// pass 1, horizontal first: tmp[y][ox] = sum_i decode(src[y][hfirst[ox] + i]) * hc[ox][i]
template <bool PLAIN>
__global__ void __launch_bounds__(256)
twopass_h1_kernel(const uint32_t *__restrict__ in, TwoPassParams T) {
    const ResampleParams &P = T.P;
    const int ox = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5), f = blockIdx.z;
    if (PLAIN && !T.need_plain[f]) return;
    if (ox >= P.ow || y >= P.ih) return;
    const uint32_t *row = in + (long long)f * P.iw * P.ih + (long long)y * P.iw + P.h_first[ox];
    const float *hc = P.h_coeff + (long long)ox * P.h_widest;
    const int cnt = P.h_count[ox];
    float4 r;
    if (P.h_sequential) {
        r = mul4(decode_tp<PLAIN>(row[0], P.bgra), hc[0]);
        for (int i = 1; i < cnt; ++i) r = add4(r, mul4(decode_tp<PLAIN>(row[i], P.bgra), hc[i]));
    } else {
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        float4 a0 = z, a1 = z;
        for (int i = 0; i < cnt; ++i) { const float4 t = mul4(decode_tp<PLAIN>(row[i], P.bgra), hc[i]); if (i & 1) a1 = add4(a1, t); else a0 = add4(a0, t); }
        r = add4(a0, a1);
    }
    T.tmp[((long long)f * P.ih + y) * P.ow + ox] = r;
}
// pass 1, horizontal first, FLAT: the same sums as twopass_h1_kernel with the (row, output column) pairs of `rows` source rows
// laid out flat over the CTA's threads -- with few output columns (C1: 67 = two full 32-column tiles and one of 3) the tiled
// mapping leaves 30 % of the lanes idle; here a CTA's rows x ow outputs fill its 256 threads to within a few per cent.
template <bool PLAIN>
__global__ void __launch_bounds__(256)
twopass_h1f_kernel(const uint32_t *__restrict__ in, TwoPassParams T, int rows) {
    const ResampleParams &P = T.P;
    const int f = blockIdx.y, y0 = blockIdx.x * rows;
    if (PLAIN && !T.need_plain[f]) return;
    const int n = min(rows, P.ih - y0) * P.ow;
    for (int idx = threadIdx.x; idx < n; idx += 256) {
        const int ry = idx / P.ow, ox = idx - ry * P.ow, y = y0 + ry;
        const uint32_t *row = in + (long long)f * P.iw * P.ih + (long long)y * P.iw + P.h_first[ox];
        const float *hc = P.h_coeff + (long long)ox * P.h_widest;
        const int cnt = P.h_count[ox];
        float4 r;
        if (P.h_sequential) {
            r = mul4(decode_tp<PLAIN>(row[0], P.bgra), hc[0]);
            for (int i = 1; i < cnt; ++i) r = add4(r, mul4(decode_tp<PLAIN>(row[i], P.bgra), hc[i]));
        } else {
            const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            float4 a0 = z, a1 = z;
            for (int i = 0; i < cnt; ++i) { const float4 t = mul4(decode_tp<PLAIN>(row[i], P.bgra), hc[i]); if (i & 1) a1 = add4(a1, t); else a0 = add4(a0, t); }
            r = add4(a0, a1);
        }
        T.tmp[((long long)f * P.ih + y) * P.ow + ox] = r;
    }
}
// pass 1, horizontal first, STAGED: the same sums as twopass_h1_kernel, but a warp decodes the stretch of its source row
// that the CTA's 32 output columns need ONCE into shared memory (coalesced 128-byte loads) and the taps then read
// float4s from there -- the plain kernel decodes every source pixel once per output that uses it (~4x for the long
// filters this path serves) through uncoalesced 4-byte loads.  warp = source row, lane = output column.
struct H1sGeom { int nwin, cpitch; };            // window columns per tile (max over tiles), coefficient pitch (odd)
template <bool PLAIN>
__global__ void __launch_bounds__(256)
twopass_h1s_kernel(const uint32_t *__restrict__ in, TwoPassParams T, H1sGeom G) {
    extern __shared__ float4 s_h1[];                                     // [8][nwin] decoded pixels | [32][cpitch] coefficients
    const ResampleParams &P = T.P;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, f = blockIdx.z;
    if (PLAIN && !T.need_plain[f]) return;
    const int ox0 = blockIdx.x * 32, ox = ox0 + lane, y = blockIdx.y * 8 + wid;
    float *s_c = reinterpret_cast<float *>(s_h1 + 8 * G.nwin);
    for (int i = threadIdx.x; i < 32 * P.h_widest; i += 256) {
        const int o = i / P.h_widest, k = i - o * P.h_widest;
        s_c[o * G.cpitch + k] = ox0 + o < P.ow ? P.h_coeff[(long long)(ox0 + o) * P.h_widest + k] : 0.0f;
    }
    const int c0 = P.h_first[ox0];
    if (y < P.ih) {
        const uint32_t *row = in + (long long)f * P.iw * P.ih + (long long)y * P.iw;
        float4 *srow = s_h1 + wid * G.nwin;
        const int c1 = min(P.iw, c0 + G.nwin);
        for (int c = c0 + lane; c < c1; c += 32) srow[c - c0] = decode_tp<PLAIN>(row[c], P.bgra);
    }
    __syncthreads();
    if (ox >= P.ow || y >= P.ih) return;
    const float4 *v = s_h1 + wid * G.nwin + (P.h_first[ox] - c0);
    const float *hc = s_c + lane * G.cpitch;
    const int cnt = P.h_count[ox];
    float4 r;
    if (P.h_sequential) {
        r = mul4(v[0], hc[0]);
        for (int i = 1; i < cnt; ++i) r = add4(r, mul4(v[i], hc[i]));
    } else {
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        float4 a0 = z, a1 = z;
        for (int i = 0; i < cnt; ++i) { const float4 t = mul4(v[i], hc[i]); if (i & 1) a1 = add4(a1, t); else a0 = add4(a0, t); }
        r = add4(a0, a1);
    }
    T.tmp[((long long)f * P.ih + y) * P.ow + ox] = r;
}
// pass 2: filter the intermediate along the other axis, then un-weight / encode / compose (weighted pass) or
// fill in the pixels whose alpha came out as zero (plain pass)
template <bool VFIRST, bool PLAIN>
__global__ void __launch_bounds__(256)
twopass_2_kernel(uint32_t *__restrict__ out, TwoPassParams T) {
    const ResampleParams &P = T.P;
    const int ox = blockIdx.x * 32 + (threadIdx.x & 31), oy = blockIdx.y * 8 + (threadIdx.x >> 5), f = blockIdx.z;
    if (PLAIN && !T.need_plain[f]) return;
    if (ox >= P.ow || oy >= P.oh) return;
    const float tiny = 7.5231638452626401e-37f;       // 2^-120
    uint32_t *dst = out + ((long long)f * P.out_frame_rows + oy) * P.ow + ox;
    float4 r;
    if (VFIRST) {                                     // second pass is horizontal, over tmp[oy][0..iw)
        const float4 *row = T.tmp + ((long long)f * P.oh + oy) * P.iw + P.h_first[ox];
        const float *hc = P.h_coeff + (long long)ox * P.h_widest;
        const int cnt = P.h_count[ox];
        if (P.h_sequential) {
            r = mul4(row[0], hc[0]);
            for (int i = 1; i < cnt; ++i) r = add4(r, mul4(row[i], hc[i]));
        } else {
            const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            float4 a0 = z, a1 = z;
            for (int i = 0; i < cnt; ++i) { const float4 t = mul4(row[i], hc[i]); if (i & 1) a1 = add4(a1, t); else a0 = add4(a0, t); }
            r = add4(a0, a1);
        }
    } else {                                          // second pass is vertical, over tmp[0..ih)[ox]
        const float4 *col = T.tmp + ((long long)f * P.ih + P.v_first[oy]) * P.ow + ox;
        const float *vc = P.v_coeff + (long long)oy * P.v_widest;
        const int cnt = P.v_count[oy];
        r = mul4(col[0], vc[0]);
        for (int k = 1; k < cnt; ++k) r = add4(r, mul4(col[(long long)k * P.ow], vc[k]));
    }
    float v[7];
    unsigned char *m = T.mask + ((long long)f * P.oh + oy) * P.ow + ox;
    if (!PLAIN) {
        const bool hole = r.w < tiny;                 // un-weighted colour needed: left to the plain passes
        *m = hole ? 1 : 0;
        if (hole) { T.need_plain[f] = 1; return; }    // (every writer stores 1: benign)
        v[0] = v[1] = v[2] = 0.f; v[3] = r.w; v[4] = r.x; v[5] = r.y; v[6] = r.z;
        *dst = compose_at(P.cs, encode_px(v), ox, oy);
    } else if (*m) {
        v[0] = r.x; v[1] = r.y; v[2] = r.z; v[3] = 0.f; v[4] = v[5] = v[6] = 0.f;   // alpha < 2^-120 encodes to 0 either way
        *dst = compose_at(P.cs, encode_px(v), ox, oy);
    }
}

// both axes point-sampled (scale 1): plain copy, with the BGRA swizzle if asked (:6938-6940).
__global__ void __launch_bounds__(256)
resample_copy_kernel(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, ResampleParams P) {
    const long long frame_px = (long long)P.ow * P.oh;
    const long long total = frame_px * P.n_frames;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += stride) {
        const long long f = g / frame_px, i = g - f * frame_px;
        const int oy = (int)(i / P.ow), ox = (int)(i - (long long)oy * P.ow);
        uint32_t p = in[(long long)f * P.iw * P.ih + (long long)P.v_first[oy] * P.iw + P.h_first[ox]];
        if (P.bgra) p = (p & 0xff00ff00u) | ((p & 0xff) << 16) | ((p >> 16) & 0xff);
        out[((long long)f * P.out_frame_rows + oy) * P.ow + ox] = compose_at(P.cs, p, ox, oy);
    }
}

// scale 1 in both axes and identity tap tables (the C5 shape: frames shown unscaled): 16-byte copies, 4 pixels per thread,
// compose fused.  grid = (quads of a frame, frames).
__global__ void __launch_bounds__(256)
resample_copy4_kernel(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, ResampleParams P) {
    const int qpr = P.ow >> 2, nq = qpr * P.oh, f = blockIdx.y;
    const uint4 *src = reinterpret_cast<const uint4 *>(in + (long long)f * P.iw * P.ih);
    uint4 *dst = reinterpret_cast<uint4 *>(out + (long long)f * P.out_frame_rows * P.ow);
    for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += gridDim.x * blockDim.x) {
        uint4 v = __ldcs(src + q);                                       // read once
        if (P.bgra) {
            v.x = (v.x & 0xff00ff00u) | ((v.x & 0xff) << 16) | ((v.x >> 16) & 0xff);
            v.y = (v.y & 0xff00ff00u) | ((v.y & 0xff) << 16) | ((v.y >> 16) & 0xff);
            v.z = (v.z & 0xff00ff00u) | ((v.z & 0xff) << 16) | ((v.z >> 16) & 0xff);
            v.w = (v.w & 0xff00ff00u) | ((v.w & 0xff) << 16) | ((v.w >> 16) & 0xff);
        }
        if (P.cs.active && (v.x & v.y & v.z & v.w) < 0xff000000u) {      // some pixel of the group is not opaque
            const int oy = q / qpr, ox = (q - oy * qpr) << 2;
            v.x = compose_at(P.cs, v.x, ox, oy); v.y = compose_at(P.cs, v.y, ox + 1, oy);
            v.z = compose_at(P.cs, v.z, ox + 2, oy); v.w = compose_at(P.cs, v.w, ox + 3, oy);
        }
        dst[q] = v;
    }
}

// ---- v3: opaque tiles, vertical pass first, <= 8 taps per axis ------------------------------
// What limits the planar kernel above is shared-memory bandwidth and issue slots spent outside the tap
// sums: it stages three float planes (12 B/px) and every tap of the vertical pass is a 16-byte load.
// v3 keeps the window as the RAW pixels (4 B/px: a plain 16-byte copy, no decode at staging) and turns
// bytes into floats at the point of use (PRMT into the mantissa of 2^23, one FSUB), two neighbouring
// columns per thread; the tap sums work on register PAIRS -- (R,G) of a pixel, (B,B) of two pixels.
// The arithmetic is the FAST mode: the reference's filter with FFMA and the 1/255 .. *255 round trip dropped,
// within 1 LSB of the reference (BASELINE.md's stated gate for the Mitchell path); used where the result feeds the
// sixel quantiser, whose own parity is a delta-E tolerance.  (Bit-exact scaling takes the planar kernel.)
// Tiles whose window is not fully opaque are handed to the planar kernel through a work list.
struct F2 { float x, y; };
#ifdef CUSIM
__device__ __forceinline__ F2 f2_add(F2 a, F2 b) { return F2{a.x + b.x, a.y + b.y}; }
__device__ __forceinline__ F2 f2_fma(F2 a, F2 b, F2 c) { return F2{fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)}; }
#else
// sm_90 has no packed FP32 arithmetic: each lane is one round-to-nearest FADD / FFMA.
__device__ __forceinline__ F2 f2_add(F2 a, F2 b) { return F2{__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)}; }
__device__ __forceinline__ F2 f2_fma(F2 a, F2 b, F2 c) { return F2{__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)}; }
#endif
// acc = v * c   /   acc += v * c
__device__ __forceinline__ F2 f2_mul(F2 v, float c) { return f2_fma(v, F2{c, c}, F2{0.0f, 0.0f}); }
__device__ __forceinline__ F2 f2_mac(F2 a, F2 v, float c) { return f2_fma(v, F2{c, c}, a); }
__device__ __forceinline__ float f1_mac(float a, float v, float c) { return fmaf(v, c, a); }

// two bytes -> a float pair (exact integers): two PRMTs into the mantissa of 2^23 and ONE packed subtraction.
__device__ __forceinline__ F2 byte_pair(uint32_t pa, uint32_t sa, uint32_t pb, uint32_t sb) {
    return f2_add(F2{__uint_as_float(__byte_perm(pa, 0x4B000000u, sa)), __uint_as_float(__byte_perm(pb, 0x4B000000u, sb))},
                  F2{-8388608.0f, -8388608.0f});
}
// trunc(clamp(v + 0.5, 0, 255)): the float -> u8 conversion saturates by itself
__device__ __forceinline__ uint32_t sat_u8(float v) {
#ifdef CUSIM
    return __float2uint_rz(fminf(fmaxf(v + 0.5f, 0.0f), 255.0f));
#else
    uint32_t r;
    asm("cvt.rzi.u8.f32 %0, %1;" : "=r"(r) : "f"(v + 0.5f));
    return r;
#endif
}

struct V3Geom { int nix, niy, sp, tp; unsigned grp_magic; const int32_t *tile_ix0, *tile_iy0; uint32_t *fallback; int use_tma; };   // grp_magic: floor(2^32/(sp/4))+1
// Tuning switch (tools/build_variant.sh builds variant libraries to compare on C2 frames): CTAs/SM asked of the
// compiler.  2 (the default) leaves 3 resident when the kernel fits 80 registers; 3 forces 80 registers and spills.
#ifndef V3_MINB_VALUE
#define V3_MINB_VALUE 2
#endif
constexpr int V3_TW = 64, V3_TH = 32, V3_NT = 256, V3_MINB = V3_MINB_VALUE;   // 3 CTAs/SM: <= 80 registers (84 cost a third of the occupancy)

template <int HC, int VC>
__global__ void __launch_bounds__(V3_NT, (VC >= 8 ? 2 : V3_MINB))      // the 8-row register windows do not fit 80 registers
resample_v3_kernel(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, ResampleParams P, V3Geom G,
                   const __grid_constant__ CUtensorMap tmap) {
    extern __shared__ __align__(128) float4 s_px[];
    __shared__ __align__(8) unsigned long long s_mbar;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, f = blockIdx.z;
    const int ox0 = blockIdx.x * V3_TW, oy0 = blockIdx.y * V3_TH;
    const int ix0 = G.tile_ix0[blockIdx.x], iy0 = G.tile_iy0[blockIdx.y];
    const int niy = G.niy, sp = G.sp, tp = G.tp;
    uint32_t *S = reinterpret_cast<uint32_t *>(s_px);                        // [niy][sp] raw pixels
    float2 *TRG = reinterpret_cast<float2 *>(S + niy * sp);                  // [V3_TH][tp]  (R, G) after the vertical pass
    float *TB = reinterpret_cast<float *>(TRG + V3_TH * tp);                 // [V3_TH][tp]
    float *s_hc = TB + V3_TH * tp + ((4 - ((V3_TH * tp) & 3)) & 3);         // [V3_TW][8], 16-byte aligned (tp odd, V3_TH * tp * 12 % 16 handled here)
    float *s_vc = s_hc + V3_TW * 8;                                          // [V3_TH][8]
    // completion index of every output column / row of the tile: the window column / row at which its LAST tap arrives
    // (first + taps - 1), and a -1 behind the last entry so the walks below stop without a bound check
    int *s_hlast = reinterpret_cast<int *>(s_vc + V3_TH * 8);                // [V3_TW + 1]
    int *s_vlast = s_hlast + V3_TW + 1;                                      // [V3_TH + 1]
    uint32_t *O = S;                                                         // [V3_TH][V3_TW + 1] once S is dead
#ifndef CUSIM
    if (G.use_tma) {                                                         // the window is on its way while the tap tables are set up
        if (tid == 0) mbar_init(&s_mbar, 1);
        __syncthreads();
        if (tid == 0) {
            mbar_expect_tx(&s_mbar, (uint32_t)(niy * sp) * 4u);
            tma_load_3d(S, &tmap, &s_mbar, ix0, iy0, f);
        }
    }
#endif
    if (tid < V3_TW) {
        const int ox = ox0 + tid;
        const bool ok = ox < P.ow;
        s_hlast[tid] = P.h_first[min(ox, P.ow - 1)] - ix0 + HC - 1;   // columns past the image edge repeat the last one (zero weights): the walk stays monotone
        if (tid == 0) { s_hlast[V3_TW] = -1; s_vlast[V3_TH] = -1; }
#pragma unroll
        for (int i = 0; i < 8; ++i) s_hc[tid * 8 + i] = (ok && i < P.h_widest) ? P.h_coeff[(long long)ox * P.h_widest + i] : 0.0f;
    } else if (tid < V3_TW + V3_TH) {
        const int t = tid - V3_TW, oy = oy0 + t;
        const bool ok = oy < P.oh;
        s_vlast[t] = P.v_first[min(oy, P.oh - 1)] - iy0 + VC - 1;
#pragma unroll
        for (int i = 0; i < 8; ++i) s_vc[t * 8 + i] = (ok && i < P.v_widest) ? P.v_coeff[(long long)oy * P.v_widest + i] : 0.0f;
    }
    // ---- stage the window: plain 16-byte copies; cells outside the image are zero (their taps have zero weight)
    const uint32_t *src = in + (long long)f * P.iw * P.ih;
    const int ngrp = sp >> 2, n_stage = niy * ngrp;
    bool ok255 = true;
    bool fold = false;                 // interior TMA tile: every cell is a pixel, the opacity test rides on the vertical pass's loads
#ifndef CUSIM
    if (G.use_tma) {
        mbar_wait(&s_mbar, 0);                                               // the window has landed (zero-filled outside the image)
        if (iy0 + niy <= P.ih && ix0 + sp <= P.iw) {
            fold = true;
        } else {
            for (int u = tid; u < n_stage; u += V3_NT) {
                const int ly = (int)__umulhi((unsigned)u, G.grp_magic), g = u - ly * ngrp;
                if (iy0 + ly < P.ih && ix0 + 4 * g < P.iw) {                 // iw % 4 == 0 on this path: a group is inside or outside as a whole
                    const uint4 raw = *reinterpret_cast<const uint4 *>(S + ly * sp + 4 * g);
                    ok255 = ok255 && ((raw.x & raw.y & raw.z & raw.w) >= 0xff000000u);
                }
            }
        }
    } else
#endif
    for (int u = tid; u < n_stage; u += V3_NT) {
        const int ly = (int)__umulhi((unsigned)u, G.grp_magic), g = u - ly * ngrp;
        const int y = iy0 + ly, x = ix0 + 4 * g;
        uint4 raw = make_uint4(0u, 0u, 0u, 0u);
        if (y < P.ih && x < P.iw) {
            raw = __ldg(reinterpret_cast<const uint4 *>(src + (long long)y * P.iw + x));
            ok255 = ok255 && ((raw.x & raw.y & raw.z & raw.w) >= 0xff000000u);
        }
        *reinterpret_cast<uint4 *>(S + ly * sp + 4 * g) = raw;
    }
    if (!__syncthreads_and(ok255)) {                              // some pixel of the window has alpha < 255: planar kernel's job
        if (tid == 0) {
            const uint32_t k = atomicAdd(G.fallback, 1u);
            uint32_t *e = G.fallback + 1 + 3 * k;
            e[0] = blockIdx.x; e[1] = blockIdx.y; e[2] = blockIdx.z;
        }
        return;
    }
    const uint32_t sel_r = 0x7540u | (P.bgra ? 2u : 0u), sel_g = 0x7541u, sel_b = 0x7540u | (P.bgra ? 0u : 2u);
    // ---- vertical, streaming: a thread owns two neighbouring columns and 8 consecutive output rows.  It walks down
    // the input rows those outputs need ONCE: each row is loaded and converted once into a VC-deep register window
    // (slot = row mod VC, static because the walk is unrolled by VC), and an output row is produced the moment its
    // last tap arrives -- its taps are then exactly the window, oldest first.  Loads and byte->float conversions per
    // intermediate pixel drop from VC to ~1.4 (input rows per output row, plus the window warm-up of each group).
    const int ncp = sp >> 1;
    uint32_t amask = 0xffffffffu;                                            // AND of every pixel this thread reads
    {
        const int j0 = (wid >> 1) * 8, j1 = j0 + 8;
        const int f0 = s_vlast[j0] - (VC - 1), rend = s_vlast[j1 - 1] + 1;    // input rows [f0, rend) of the window
        for (int cp = (wid & 1) * 32 + lane; cp < ncp; cp += 64) {
            F2 w0[VC], w1[VC], wb[VC];
            int j = j0, ej = f0 + VC - 1;                                      // next output row and its last input row
            const uint32_t *scol = S + 2 * cp;
#pragma unroll 1
            for (int r0 = f0; r0 < rend; r0 += VC) {
#pragma unroll
                for (int sl = 0; sl < VC; ++sl) {
                    const int r = r0 + sl;
                    if (r < rend) {
                        const uint2 pp = *reinterpret_cast<const uint2 *>(scol + r * sp);
                        amask &= pp.x & pp.y;
                        w0[sl] = byte_pair(pp.x, sel_r, pp.x, sel_g);
                        w1[sl] = byte_pair(pp.y, sel_r, pp.y, sel_g);
                        wb[sl] = byte_pair(pp.x, sel_b, pp.y, sel_b);
                        // uniform: every thread walks the same rows.  No j < j1 test: a row of the NEXT group completing at this
                        // very input row (only when enlarging) has exactly this window as its taps -- the duplicate write
                        // stores the same values the owner stores; the sentinel ends the walk at the tile's last row.
                        while (j < j1 && ej == r) {
                            const float4 v0 = *reinterpret_cast<const float4 *>(s_vc + j * 8), v1 = *reinterpret_cast<const float4 *>(s_vc + j * 8 + 4);
                            const float vc[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
                            F2 a0 = f2_mul(w0[(sl + 1) % VC], vc[0]), a1 = f2_mul(w1[(sl + 1) % VC], vc[0]);
                            F2 ab = f2_mul(wb[(sl + 1) % VC], vc[0]);
#pragma unroll
                            for (int k = 1; k < VC; ++k) {
                                a0 = f2_mac(a0, w0[(sl + 1 + k) % VC], vc[k]);
                                a1 = f2_mac(a1, w1[(sl + 1 + k) % VC], vc[k]);
                                ab = f2_mac(ab, wb[(sl + 1 + k) % VC], vc[k]);
                            }
                            float2 *t = TRG + j * tp + 2 * cp;
                            t[0] = make_float2(a0.x, a0.y); t[1] = make_float2(a1.x, a1.y);
                            float *tb = TB + j * tp + 2 * cp;
                            tb[0] = ab.x; tb[1] = ab.y;
                            ++j;
                            ej = j < j1 ? s_vlast[j] : -1;
                        }
                    }
                }
            }
        }
    }
    if (!__syncthreads_and(!fold || amask >= 0xff000000u)) {      // (interior TMA tiles) a pixel that was read is not opaque
        if (tid == 0) {
            const uint32_t k = atomicAdd(G.fallback, 1u);
            uint32_t *e = G.fallback + 1 + 3 * k;
            e[0] = blockIdx.x; e[1] = blockIdx.y; e[2] = blockIdx.z;
        }
        return;
    }
    // ---- horizontal, streaming the same way along x: lane = output row, a warp owns 8 consecutive output columns
    // and walks the intermediate columns they need once (window of HC columns in registers).  Pixels go straight
    // into the transpose buffer O (it aliases S, which is dead now).
    const bool hseq = P.h_sequential != 0;
    {
        const int tx0 = wid * 8, tx1 = tx0 + 8;
        const int f0 = s_hlast[tx0] - (HC - 1), cend = s_hlast[tx1 - 1] + 1;
        const float2 *trow = TRG + lane * tp;
        const float *brow = TB + lane * tp;
        F2 wrg[HC]; float wbb[HC];
        int tx = tx0, etx = f0 + HC - 1;
#pragma unroll 1
        for (int c0 = f0; c0 < cend; c0 += HC) {
#pragma unroll
            for (int sl = 0; sl < HC; ++sl) {
                const int c = c0 + sl;
                if (c < cend) {
                    const float2 q = trow[c];
                    wrg[sl] = F2{q.x, q.y}; wbb[sl] = brow[c];
                    while (tx < tx1 && etx == c) {                // same argument as in the vertical walk
                        const float4 h0 = *reinterpret_cast<const float4 *>(s_hc + tx * 8), h1 = *reinterpret_cast<const float4 *>(s_hc + tx * 8 + 4);
                        const float hc[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
                        F2 c2; float cb;
                        if (hseq) {
                            F2 a = f2_mul(wrg[(sl + 1) % HC], hc[0]);
                            float b = wbb[(sl + 1) % HC] * hc[0];
#pragma unroll
                            for (int i = 1; i < (HC < 3 ? HC : 3); ++i) {
                                a = f2_mac(a, wrg[(sl + 1 + i) % HC], hc[i]); b = f1_mac(b, wbb[(sl + 1 + i) % HC], hc[i]);
                            }
                            c2 = a; cb = b;
                        } else {
                            F2 a0 = f2_mul(wrg[(sl + 1) % HC], hc[0]), a1 = f2_mul(wrg[(sl + 2) % HC], hc[1]);
                            float b0 = wbb[(sl + 1) % HC] * hc[0];
                            float b1 = wbb[(sl + 2) % HC] * hc[1];
#pragma unroll
                            for (int i = 2; i < HC; ++i) {
                                if (i & 1) { a1 = f2_mac(a1, wrg[(sl + 1 + i) % HC], hc[i]); b1 = f1_mac(b1, wbb[(sl + 1 + i) % HC], hc[i]); }
                                else { a0 = f2_mac(a0, wrg[(sl + 1 + i) % HC], hc[i]); b0 = f1_mac(b0, wbb[(sl + 1 + i) % HC], hc[i]); }
                            }
                            c2 = F2{a0.x + a1.x, a0.y + a1.y};
                            cb = b0 + b1;
                        }
                        const uint32_t r8 = sat_u8(c2.x), g8 = sat_u8(c2.y), b8 = sat_u8(cb);
                        O[lane * (V3_TW + 1) + tx] = pack_rgba(r8, g8, b8, 0xffu);    // opaque in, opaque out: nothing to compose
                        ++tx;
                        etx = tx < tx1 ? s_hlast[tx] : -1;
                    }
                }
            }
        }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < V3_TH / 8; ++i) {
        const int ty = wid + 8 * i, oy = oy0 + ty;
        if (oy < P.oh) {
            uint32_t *orow = out + ((long long)f * P.out_frame_rows + oy) * P.ow + ox0;
            if (ox0 + lane < P.ow) orow[lane] = O[ty * (V3_TW + 1) + lane];
            if (ox0 + lane + 32 < P.ow) orow[lane + 32] = O[ty * (V3_TW + 1) + lane + 32];
        }
    }
}

// Tensor map of a batch of source frames for the v3 kernel's window: u32 elements, dims (iw, ih, frames), box (cols, rows, 1),
// no swizzle, zero fill outside.  False when the geometry does not meet TMA's alignment rules (the kernel then stages
// with plain 16-byte loads) or when B200TIMG_TMA=0.
static bool v3_tensor_map(CUtensorMap *map, const uint32_t *src, int iw, int ih, int n_frames, int box_cols, int box_rows) {
#ifdef CUSIM
    return false;
#else
    if (const char *e = getenv("B200TIMG_TMA")) if (atoi(e) == 0) return false;
    if ((iw & 3) || (reinterpret_cast<uintptr_t>(src) & 15) || box_cols > 256 || box_rows > 256 || (box_cols & 3)) return false;
    typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                 const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeFn encode = [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) p = nullptr;
        return reinterpret_cast<EncodeFn>(p);
    }();
    if (!encode) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)iw, (cuuint64_t)ih, (cuuint64_t)n_frames};
    const cuuint64_t strides[2] = {(cuuint64_t)iw * 4, (cuuint64_t)iw * ih * 4};
    const cuuint32_t box[3] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    return encode(map, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, const_cast<uint32_t *>(src), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
#endif
}

typedef void (*V3Fn)(const uint32_t *, uint32_t *, ResampleParams, V3Geom, const CUtensorMap);
template <int HC>
static V3Fn v3_v(int vc) {
    switch (vc) {
    case 2: return resample_v3_kernel<HC, 2>;
    case 4: return resample_v3_kernel<HC, 4>;
    case 6: return resample_v3_kernel<HC, 6>;
    default: return resample_v3_kernel<HC, 8>;
    }
}
static V3Fn v3_h(int hc, int vc) {
    switch (hc) {
    case 2: return v3_v<2>(vc);
    case 4: return v3_v<4>(vc);
    case 6: return v3_v<6>(vc);
    default: return v3_v<8>(vc);
    }
}
typedef void (*PlanarListFn)(const uint32_t *, uint32_t *, ResampleParams, PlanarGeom, const uint32_t *);
template <int HC>
static PlanarListFn planar_list_v(int vc) {
    switch (vc) {
    case 2: return resample_planar_list_kernel<HC, 2, 3>;
    case 4: return resample_planar_list_kernel<HC, 4, 3>;
    case 6: return resample_planar_list_kernel<HC, 6, 3>;
    default: return resample_planar_list_kernel<HC, 8, 3>;
    }
}
static PlanarListFn planar_list_h(int hc, int vc) {
    switch (hc) {
    case 2: return planar_list_v<2>(vc);
    case 4: return planar_list_v<4>(vc);
    case 6: return planar_list_v<6>(vc);
    default: return planar_list_v<8>(vc);
    }
}

// ---- plan cache + upload ----------------------------------------------------------------
static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

int launch_scale(b200timg_ctx *ctx, const uint8_t *d_in, int iw, int ih, int fmt, uint8_t *d_out,
                 int ow, int oh, int out_frame_rows, int n_frames, const ComposeSpec *cs, int fast) {
    if (out_frame_rows < oh) return ctx->fail(B200TIMG_EINVAL, "scale: frame rows < out height");
    if ((reinterpret_cast<uintptr_t>(d_in) & 3) || (reinterpret_cast<uintptr_t>(d_out) & 3))
        return ctx->fail(B200TIMG_EINVAL, "scale: pixel buffers must be 4-byte aligned");
    if (!ctx->plan) ctx->plan = new ResamplePlan();
    int *key = ctx->plan_key;
    const bool hit = key[0] == iw && key[1] == ih && key[2] == ow && key[3] == oh;
    ResamplePlan *pl = ctx->plan;
    if (!hit) {
        key[0] = 0;
        if (!build_resample_plan(iw, ih, ow, oh, pl)) return ctx->fail(B200TIMG_EINVAL, "scale: degenerate geometry");
    }
    // table layout in ctx->tables: [h_first|h_count|h_lead|v_first|v_count|h_coeff|v_coeff]
    const size_t o_hf = 0, o_hc = o_hf + align_up(sizeof(int32_t) * ow, 16), o_hl = o_hc + align_up(sizeof(int32_t) * ow, 16);
    const size_t o_vf = o_hl + align_up(sizeof(int32_t) * ow, 16), o_vc = o_vf + align_up(sizeof(int32_t) * oh, 16);
    const size_t o_hk = o_vc + align_up(sizeof(int32_t) * oh, 16);
    const size_t o_vk = o_hk + align_up(sizeof(float) * pl->h.coeff.size(), 16);
    const size_t total = o_vk + align_up(sizeof(float) * pl->v.coeff.size(), 16);
    if (!hit) {
        B2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));          // tables may be in use by earlier launches
        B2_CUDA(ctx, ctx->tables.reserve(total));
        B2_CUDA(ctx, ctx->pinned_io.reserve(total));
        char *h = ctx->pinned_io.as<char>();
        memcpy(h + o_hf, pl->h.first.data(), sizeof(int32_t) * ow);
        memcpy(h + o_hc, pl->h.count.data(), sizeof(int32_t) * ow);
        memcpy(h + o_hl, pl->h.lead.data(), sizeof(int32_t) * ow);
        memcpy(h + o_vf, pl->v.first.data(), sizeof(int32_t) * oh);
        memcpy(h + o_vc, pl->v.count.data(), sizeof(int32_t) * oh);
        memcpy(h + o_hk, pl->h.coeff.data(), sizeof(float) * pl->h.coeff.size());
        memcpy(h + o_vk, pl->v.coeff.data(), sizeof(float) * pl->v.coeff.size());
        B2_CUDA(ctx, cudaMemcpyAsync(ctx->tables.p, h, total, cudaMemcpyHostToDevice, ctx->stream));
        B2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));          // pinned_io is reused by callers
        key[0] = iw; key[1] = ih; key[2] = ow; key[3] = oh;
    }
    const char *t = ctx->tables.as<char>();
    ResampleParams P;
    P.iw = iw; P.ih = ih; P.ow = ow; P.oh = oh; P.out_frame_rows = out_frame_rows; P.n_frames = n_frames;
    P.bgra = fmt == B200TIMG_FMT_RGB32;
    if (cs) P.cs = *cs; else { memset(&P.cs, 0, sizeof P.cs); P.cs.pw = P.cs.ph = 1; }
    P.h_widest = pl->h.widest; P.v_widest = pl->v.widest; P.h_sequential = pl->h_sequential ? 1 : 0;
    P.h_first = reinterpret_cast<const int32_t *>(t + o_hf);
    P.h_count = reinterpret_cast<const int32_t *>(t + o_hc);
    P.h_lead = reinterpret_cast<const int32_t *>(t + o_hl);
    P.v_first = reinterpret_cast<const int32_t *>(t + o_vf);
    P.v_count = reinterpret_cast<const int32_t *>(t + o_vc);
    P.h_coeff = reinterpret_cast<const float *>(t + o_hk);
    P.v_coeff = reinterpret_cast<const float *>(t + o_vk);
    const uint32_t *in = reinterpret_cast<const uint32_t *>(d_in);
    uint32_t *out = reinterpret_cast<uint32_t *>(d_out);
    bool identity = pl->copy_only && iw == ow && ih == oh && (ow & 3) == 0 && n_frames <= 65535 && (long long)ow * oh < (1ll << 31) &&
                    ((reinterpret_cast<uintptr_t>(d_in) | reinterpret_cast<uintptr_t>(d_out)) & 15) == 0;
    for (int x = 0; identity && x < ow; ++x) identity = pl->h.first[x] == x;
    for (int y = 0; identity && y < oh; ++y) identity = pl->v.first[y] == y;
    if (identity) {
        const int nq = (ow >> 2) * oh;
        const int bx = std::max(1, std::min((nq + 255) / 256, std::max(1, ctx->sm_count * 8 / std::max(1, std::min(n_frames, ctx->sm_count * 8)))));
        B2_KERNEL(ctx, "resample_copy_kernel");
        resample_copy4_kernel<<<dim3((unsigned)bx, (unsigned)n_frames), 256, 0, ctx->stream>>>(in, out, P);
    } else if (pl->copy_only) {
        long long blocks = ((long long)ow * oh * n_frames + 255) / 256;
        if (blocks > (long long)ctx->sm_count * 16) blocks = (long long)ctx->sm_count * 16;
        B2_KERNEL(ctx, "resample_copy_kernel");
        resample_copy_kernel<<<(unsigned)blocks, 256, 0, ctx->stream>>>(in, out, P);
    } else {
        if (n_frames > 65535) return ctx->fail(B200TIMG_EINVAL, "scale: too many frames for one launch");
        // fastest path: vertical pass first, <= 8 taps per axis, 16-byte aligned rows -> v3 kernel (opaque tiles)
        // with the planar kernel taking the tiles that contain transparency
        if (pl->vertical_first && pl->h.widest <= 8 && pl->v.widest <= 8 && (iw & 3) == 0 &&
            (reinterpret_cast<uintptr_t>(d_in) & 15) == 0 && !getenv("B200TIMG_NO_PLANAR")) {
            const int hc = fixed_class(pl->h.widest), vc = fixed_class(pl->v.widest);
            auto tile_origins = [&](const AxisTable &T, int n_out, int tile, int taps, bool align4, std::vector<int32_t> &orig) -> int {
                const int nt = (n_out + tile - 1) / tile;
                orig.resize(nt);
                int span = 1;
                for (int j = 0; j < nt; ++j) {
                    int lo = 0x7fffffff, hi = -1;
                    for (int x = j * tile; x < std::min(n_out, (j + 1) * tile); ++x) { lo = std::min(lo, T.first[x]); hi = std::max(hi, T.first[x] + taps - 1); }
                    if (align4) lo &= ~3;                            // aligned 16-byte loads
                    orig[j] = lo; span = std::max(span, hi - lo + 1);
                }
                return span;
            };
            std::vector<int32_t> tix, tiy, tix3;
            const int ptw = 32;
            const int nix = tile_origins(pl->h, ow, ptw, hc, true, tix), niy = tile_origins(pl->v, oh, PTH, vc, false, tiy);
            const int ntx = (int)tix.size(), nty = (int)tiy.size();
            const int sp = (nix + 3) & ~3, tp = sp | 1;   // odd T pitch >= the 4-column groups written per row
            const size_t psmem = sizeof(float) * (3 * ((size_t)niy * sp + (size_t)PTH * tp) + 4 + (size_t)ptw * 8 + PTH * 8) + sizeof(int) * (ptw + PTH);
            const size_t smem_cap = 75 * 1024;           // 3 CTAs/SM (80 registers) rather than 2
            const bool planar_ok = psmem <= smem_cap && (size_t)PTH * (ptw + 1) <= 3 * (size_t)niy * sp;
            // v3 geometry: 64 x 32 output tiles
            const int nix3 = tile_origins(pl->h, ow, V3_TW, hc, true, tix3);
            const int ntx3 = (int)tix3.size();
            const int sp3 = (nix3 + 3) & ~3, tp3 = sp3 | 1;
            const size_t v3smem = sizeof(uint32_t) * (size_t)niy * sp3 + (sizeof(float2) + sizeof(float)) * (size_t)V3_TH * tp3 + 16 +
                                  sizeof(float) * ((size_t)V3_TW * 8 + V3_TH * 8) + sizeof(int) * (V3_TW + V3_TH + 2);
            // v3 pays off in the FAST arithmetic only; bit-exact scaling takes the planar kernel
            const bool v3_ok = planar_ok && fast && v3smem <= 100 * 1024 &&
                               (size_t)V3_TH * (V3_TW + 1) <= (size_t)niy * sp3;
            if (planar_ok) {
                B2_CUDA(ctx, ctx->misc.reserve(4096 + sizeof(int32_t) * (size_t)(ntx + nty + ntx3)));
                int32_t *d_t = reinterpret_cast<int32_t *>(ctx->misc.as<char>() + 4096);
                B2_CUDA(ctx, cudaMemcpyAsync(d_t, tix.data(), sizeof(int32_t) * ntx, cudaMemcpyHostToDevice, ctx->stream));
                B2_CUDA(ctx, cudaMemcpyAsync(d_t + ntx, tiy.data(), sizeof(int32_t) * nty, cudaMemcpyHostToDevice, ctx->stream));
                B2_CUDA(ctx, cudaMemcpyAsync(d_t + ntx + nty, tix3.data(), sizeof(int32_t) * ntx3, cudaMemcpyHostToDevice, ctx->stream));
                PlanarGeom PG{nix, niy, sp, tp, (unsigned)(0x100000000ull / (unsigned)(sp / 4)) + 1u, d_t, d_t + ntx};
                if (v3_ok) {
                    // one work list per concurrently running slice of a batch (api.cu), sized before any slice starts
                    const size_t list_words = 1 + 3 * (size_t)ntx3 * nty * (size_t)std::max(n_frames, ctx->part_max_frames);
                    B2_CUDA(ctx, ctx->scale_list.reserve(sizeof(uint32_t) * list_words * (size_t)ctx->part_slots));
                    uint32_t *d_list = ctx->scale_list.as<uint32_t>() + list_words * (size_t)ctx->part_slot;
                    B2_CUDA(ctx, cudaMemsetAsync(d_list, 0, sizeof(uint32_t), ctx->stream));
                    V3Geom VG{nix3, niy, sp3, tp3, (unsigned)(0x100000000ull / (unsigned)(sp3 / 4)) + 1u, d_t + ntx + nty, d_t + ntx, d_list, 0};
                    CUtensorMap tmap;
                    memset(&tmap, 0, sizeof tmap);
                    VG.use_tma = v3_tensor_map(&tmap, in, iw, ih, n_frames, sp3, niy) ? 1 : 0;
                    V3Fn fn = v3_h(hc, vc);
                    B2_CUDA(ctx, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
                    B2_KERNEL(ctx, "resample_v3_fast_kernel");
                    fn<<<dim3(ntx3, nty, n_frames), V3_NT, v3smem, ctx->stream>>>(in, out, P, VG, tmap);
                    B2_LAUNCH_CHECK(ctx);
                    PlanarListFn lf = planar_list_h(hc, vc);              // tiles with transparency (none for photos / video)
                    B2_CUDA(ctx, cudaFuncSetAttribute(lf, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap));
                    B2_KERNEL(ctx, "resample_planar_list_kernel");
                    lf<<<ctx->sm_count * 3, PNT, psmem, ctx->stream>>>(in, out, P, PG, d_list);
                    B2_LAUNCH_CHECK(ctx);
                    return B200TIMG_OK;
                }
                PlanarFn fn = planar_h<32, 3>(hc, vc);
                B2_CUDA(ctx, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap));
                const dim3 grid(ntx, nty, n_frames);
                B2_KERNEL(ctx, "resample_planar_kernel");
                fn<<<grid, PNT, psmem, ctx->stream>>>(in, out, P, PG);
                B2_LAUNCH_CHECK(ctx);
                return B200TIMG_OK;
            }
        }
        if (pl->h.widest <= 8 && pl->v.widest <= 8) {
            const int hc = fixed_class(pl->h.widest), vc = fixed_class(pl->v.widest);
            const FixedVariant fv = pl->vertical_first ? fixed_h<true>(hc, vc) : fixed_h<false>(hc, vc);
            const int FTHv = fv.th;
            const int ntx = (ow + FTW - 1) / FTW, nty = (oh + FTHv - 1) / FTHv;
            std::vector<int32_t> tix(ntx), tiy(nty);
            int nix = 1, niy = 1;
            for (int j = 0; j < ntx; ++j) {
                int lo = 0x7fffffff, hi = -1;
                for (int x = j * FTW; x < std::min(ow, (j + 1) * FTW); ++x) { lo = std::min(lo, pl->h.first[x]); hi = std::max(hi, pl->h.first[x] + hc - 1); }
                tix[j] = lo; nix = std::max(nix, hi - lo + 1);
            }
            for (int j = 0; j < nty; ++j) {
                int lo = 0x7fffffff, hi = -1;
                for (int y = j * FTHv; y < std::min(oh, (j + 1) * FTHv); ++y) { lo = std::min(lo, pl->v.first[y]); hi = std::max(hi, pl->v.first[y] + vc - 1); }
                tiy[j] = lo; niy = std::max(niy, hi - lo + 1);
            }
            const size_t fsmem = sizeof(float4) * ((size_t)nix * niy + (pl->vertical_first ? (size_t)FTHv * nix : (size_t)niy * FTW))
                               + sizeof(int) * (FTW + FTHv) + sizeof(float) * ((size_t)FTW * (hc + 1) + (size_t)FTHv * (vc + 1));
            if (fsmem <= 100 * 1024) {
                // tile origins live behind the flag word in ctx->misc (re-uploaded per call: a few hundred bytes)
                B2_CUDA(ctx, ctx->misc.reserve(4096 + sizeof(int32_t) * (size_t)(ntx + nty)));
                int32_t *d_t = reinterpret_cast<int32_t *>(ctx->misc.as<char>() + 4096);
                B2_CUDA(ctx, cudaMemcpyAsync(d_t, tix.data(), sizeof(int32_t) * ntx, cudaMemcpyHostToDevice, ctx->stream));
                B2_CUDA(ctx, cudaMemcpyAsync(d_t + ntx, tiy.data(), sizeof(int32_t) * nty, cudaMemcpyHostToDevice, ctx->stream));
                FixedGeom FG{nix, niy, d_t, d_t + ntx};
                B2_CUDA(ctx, cudaFuncSetAttribute(fv.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
                const dim3 grid(ntx, nty, n_frames);
                B2_KERNEL(ctx, "resample_fixed_kernel");
                fv.fn<<<grid, fv.nt, fsmem, ctx->stream>>>(in, out, P, FG);
                B2_LAUNCH_CHECK(ctx);
                return B200TIMG_OK;
            }
        }
        // long filters: two 1-D passes over a float4 intermediate in global memory
        const size_t t_elems = pl->vertical_first ? (size_t)oh * iw : (size_t)ih * ow;
        const size_t o_tmp = 0, o_flag = (sizeof(float4) * t_elems * n_frames + 255) / 256 * 256;
        const size_t o_mask = o_flag + (sizeof(int) * (size_t)n_frames + 255) / 256 * 256;
        B2_CUDA(ctx, ctx->scale_tmp.reserve(o_mask + (size_t)ow * oh * n_frames));
        char *tb = ctx->scale_tmp.as<char>();
        TwoPassParams T;
        T.P = P; T.tmp = reinterpret_cast<float4 *>(tb + o_tmp); T.need_plain = reinterpret_cast<int *>(tb + o_flag);
        T.mask = reinterpret_cast<unsigned char *>(tb + o_mask);
        B2_CUDA(ctx, cudaMemsetAsync(T.need_plain, 0, sizeof(int) * (size_t)n_frames, ctx->stream));
        const dim3 g2((ow + 31) / 32, (oh + 7) / 8, n_frames);
        for (int plain = 0; plain < 2; ++plain) {
            if (pl->vertical_first) {
                const dim3 g1((iw + 255) / 256, oh, n_frames);
                B2_KERNEL(ctx, plain ? "twopass_plain_kernels" : "twopass_v1_kernel");
                if (plain) twopass_v1_kernel<true><<<g1, 256, 0, ctx->stream>>>(in, T); else twopass_v1_kernel<false><<<g1, 256, 0, ctx->stream>>>(in, T);
                B2_LAUNCH_CHECK(ctx);
                B2_KERNEL(ctx, plain ? "twopass_plain_kernels" : "twopass_2_kernel");
                if (plain) twopass_2_kernel<true, true><<<g2, 256, 0, ctx->stream>>>(out, T); else twopass_2_kernel<true, false><<<g2, 256, 0, ctx->stream>>>(out, T);
                B2_LAUNCH_CHECK(ctx);
            } else {
                const dim3 g1((ow + 31) / 32, (ih + 7) / 8, n_frames);
                // staged variant: window of a 32-column tile = first[tile start] .. max(first + count) over the tile
                H1sGeom HG{1, pl->h.widest | 1};
                for (int x0 = 0; x0 < ow; x0 += 32) {
                    int hi = 0;
                    for (int x = x0; x < std::min(ow, x0 + 32); ++x) hi = std::max(hi, pl->h.first[x] + pl->h.count[x]);
                    HG.nwin = std::max(HG.nwin, hi - pl->h.first[x0]);
                }
                const size_t h1smem = sizeof(float4) * 8 * (size_t)HG.nwin + sizeof(float) * 32 * (size_t)HG.cpitch;
                B2_KERNEL(ctx, plain ? "twopass_plain_kernels" : "twopass_h1_kernel");
                // staging pays when the 32-column tiles are mostly full (4K -> 337 columns); with 67 columns the third
                // tile stages a whole window for 3 outputs: plain kernel
                const bool tiles_full = (long long)((ow + 31) / 32) * 32 * 100 <= (long long)ow * 115;
                if (h1smem <= 72 * 1024 && tiles_full && !getenv("B200TIMG_NO_H1S")) {
                    if (plain) {
                        B2_CUDA(ctx, cudaFuncSetAttribute(twopass_h1s_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 72 * 1024));
                        twopass_h1s_kernel<true><<<g1, 256, h1smem, ctx->stream>>>(in, T, HG);
                    } else {
                        B2_CUDA(ctx, cudaFuncSetAttribute(twopass_h1s_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 72 * 1024));
                        twopass_h1s_kernel<false><<<g1, 256, h1smem, ctx->stream>>>(in, T, HG);
                    }
                } else if (!tiles_full && ow <= 4096 && n_frames <= 65535 && !getenv("B200TIMG_NO_H1F")) {
                    // few output columns: flat (row, column) mapping; rows per CTA chosen so that rows x ow fills whole 256-thread rounds
                    int rows = 8; double best = 0.0;
                    for (int r = 4; r <= 64; ++r) {
                        const long long items = (long long)r * ow, slots = (items + 255) / 256 * 256;
                        const double fill = (double)items / (double)slots;
                        if (fill > best + 1e-9) { best = fill; rows = r; }
                    }
                    const dim3 gf((ih + rows - 1) / rows, n_frames);
                    if (plain) twopass_h1f_kernel<true><<<gf, 256, 0, ctx->stream>>>(in, T, rows); else twopass_h1f_kernel<false><<<gf, 256, 0, ctx->stream>>>(in, T, rows);
                } else if (plain) twopass_h1_kernel<true><<<g1, 256, 0, ctx->stream>>>(in, T); else twopass_h1_kernel<false><<<g1, 256, 0, ctx->stream>>>(in, T);
                B2_LAUNCH_CHECK(ctx);
                B2_KERNEL(ctx, plain ? "twopass_plain_kernels" : "twopass_2_kernel");
                if (plain) twopass_2_kernel<false, true><<<g2, 256, 0, ctx->stream>>>(out, T); else twopass_2_kernel<false, false><<<g2, 256, 0, ctx->stream>>>(out, T);
                B2_LAUNCH_CHECK(ctx);
            }
        }
        return B200TIMG_OK;
    }
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

// ---- mixed-geometry batches (b200timg_mixed_batch) ---------------------------------------------------------------
// Frames of different geometry in a fixed number of launches: the two 1-D passes of the twopass_* kernels (same
// decode, tap order, accumulators, un-weighting and encode), each over a flat list of (frame, CTA) items so that one
// launch covers every frame whatever its geometry and tap count.  Frame f's pass-p CTAs are p_start[f] ..
// p_start[f + 1] - 1 and each covers 256 consecutive elements of the frame's pass output, row-major:
//   pass 1  the first axis of the frame's plan, into a float4 intermediate (vertical first: oh x iw; else ih x ow);
//   pass 2  the other axis, un-weight, encode, compose (or the plain copy of a copy_only frame).
// Transparency follows the twopass scheme: pixels whose filtered alpha is below 2^-120 raise their frame's flag and are
// filled in by a second pair of passes on the un-weighted colour planes (which returns at once for opaque frames).
struct __align__(16) MixedScaleFrame {
    unsigned long long src_off;    // bytes from the batch's source
    unsigned long long out_px;     // first output pixel (and mask byte), in pixels from the batch's output
    unsigned long long tmp_off;    // first intermediate element, in float4 from the group's intermediate
    unsigned long long tab;        // this geometry's tables, in 4-byte words from the table arena:
                                   // h_first[ow] h_count[ow] v_first[oh] v_count[oh] h_coeff[ow][hw] v_coeff[oh][vw]
    int iw, ih, ow, oh, h_widest, v_widest, vertical_first, h_sequential, copy_only;
    int out_rows;                  // rows the frame takes in the output: oh, or the sixel encoder's multiple of 6
};

// frame that owns flat item b: the last f with start[f] <= b (frames without items share their start)
__device__ __forceinline__ int mixed_frame_of(const unsigned *__restrict__ start, int n, unsigned b) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (start[mid] <= b) lo = mid; else hi = mid - 1;
    }
    return lo;
}
// horizontal taps as twopass_h1_kernel / twopass_2_kernel sum them; ld(i) is tap i's float4
template <class Load>
__device__ __forceinline__ float4 mixed_hsum(Load ld, const float *hc, int cnt, bool sequential) {
    if (sequential) {
        float4 r = mul4(ld(0), hc[0]);
        for (int i = 1; i < cnt; ++i) r = add4(r, mul4(ld(i), hc[i]));
        return r;
    }
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 a0 = z, a1 = z;
    for (int i = 0; i < cnt; ++i) { const float4 t = mul4(ld(i), hc[i]); if (i & 1) a1 = add4(a1, t); else a0 = add4(a0, t); }
    return add4(a0, a1);
}
// vertical taps in input-row order, as twopass_v1_kernel / twopass_2_kernel
template <class Load>
__device__ __forceinline__ float4 mixed_vsum(Load ld, const float *vc, int cnt) {
    float4 a = mul4(ld(0), vc[0]);
    for (int k = 1; k < cnt; ++k) a = add4(a, mul4(ld(k), vc[k]));
    return a;
}

struct MixedScaleArgs {
    const uint8_t *src;
    const MixedScaleFrame *frames;
    const unsigned *start;         // p1 or p2 of the plan
    const int32_t *tab;
    float4 *tmp;
    int *need_plain;               // [n_frames]
    unsigned char *mask;           // [output pixels] 1 = filtered alpha < 2^-120
    uint32_t *out;
    int n_frames, bgra;
    unsigned b0, b1;               // this launch covers items b0 .. b1 - 1
    ComposeSpec cs;
};

template <bool PLAIN>
__global__ void __launch_bounds__(256)
mixed_pass1_kernel(MixedScaleArgs A) {
    const unsigned b = A.b0 + blockIdx.x;
    if (b >= A.b1) return;
    const int f = mixed_frame_of(A.start, A.n_frames, b);
    if (PLAIN && !A.need_plain[f]) return;
    const MixedScaleFrame F = A.frames[f];
    const long long e = (long long)(b - A.start[f]) * 256 + threadIdx.x;
    const uint32_t *in = reinterpret_cast<const uint32_t *>(A.src + F.src_off);
    const int32_t *h_first = A.tab + F.tab, *h_count = h_first + F.ow, *v_first = h_count + F.ow, *v_count = v_first + F.oh;
    const float *h_coeff = reinterpret_cast<const float *>(v_count + F.oh), *v_coeff = h_coeff + (long long)F.ow * F.h_widest;
    const int bgra = A.bgra;
    float4 r;
    if (F.vertical_first) {                       // tmp[oy][x] = sum_k decode(src[v_first[oy] + k][x]) * vc[oy][k]
        if (e >= (long long)F.oh * F.iw) return;
        const int oy = (int)(e / F.iw), x = (int)(e - (long long)oy * F.iw);
        const uint32_t *col = in + (long long)v_first[oy] * F.iw + x;
        const int iw = F.iw;
        r = mixed_vsum([&](int k) { return decode_tp<PLAIN>(col[(long long)k * iw], bgra); },
                       v_coeff + (long long)oy * F.v_widest, v_count[oy]);
    } else {                                      // tmp[y][ox] = sum_i decode(src[y][h_first[ox] + i]) * hc[ox][i]
        if (e >= (long long)F.ih * F.ow) return;
        const int y = (int)(e / F.ow), ox = (int)(e - (long long)y * F.ow);
        const uint32_t *row = in + (long long)y * F.iw + h_first[ox];
        r = mixed_hsum([&](int i) { return decode_tp<PLAIN>(row[i], bgra); }, h_coeff + (long long)ox * F.h_widest,
                       h_count[ox], F.h_sequential != 0);
    }
    A.tmp[F.tmp_off + e] = r;
}

template <bool PLAIN>
__global__ void __launch_bounds__(256)
mixed_pass2_kernel(MixedScaleArgs A) {
    const unsigned b = A.b0 + blockIdx.x;
    if (b >= A.b1) return;
    const int f = mixed_frame_of(A.start, A.n_frames, b);
    if (PLAIN && !A.need_plain[f]) return;
    const MixedScaleFrame F = A.frames[f];
    const long long e = (long long)(b - A.start[f]) * 256 + threadIdx.x;
    if (e >= (long long)F.ow * F.oh) return;
    const int oy = (int)(e / F.ow), ox = (int)(e - (long long)oy * F.ow);
    const int32_t *h_first = A.tab + F.tab, *h_count = h_first + F.ow, *v_first = h_count + F.ow, *v_count = v_first + F.oh;
    const float *h_coeff = reinterpret_cast<const float *>(v_count + F.oh), *v_coeff = h_coeff + (long long)F.ow * F.h_widest;
    uint32_t *dst = A.out + F.out_px + e;
    if (F.copy_only) {                            // both axes point-sampled, as resample_copy_kernel
        if (PLAIN) return;
        uint32_t p = reinterpret_cast<const uint32_t *>(A.src + F.src_off)[(long long)v_first[oy] * F.iw + h_first[ox]];
        if (A.bgra) p = (p & 0xff00ff00u) | ((p & 0xff) << 16) | ((p >> 16) & 0xff);
        *dst = compose_at(A.cs, p, ox, oy);
        return;
    }
    const float4 *tmp = A.tmp + F.tmp_off;
    float4 r;
    if (F.vertical_first) {                       // second pass is horizontal, over tmp[oy][0..iw)
        const float4 *row = tmp + (long long)oy * F.iw + h_first[ox];
        r = mixed_hsum([&](int i) { return row[i]; }, h_coeff + (long long)ox * F.h_widest, h_count[ox], F.h_sequential != 0);
    } else {                                      // second pass is vertical, over tmp[0..ih)[ox]
        const float4 *col = tmp + (long long)v_first[oy] * F.ow + ox;
        const int ow = F.ow;
        r = mixed_vsum([&](int k) { return col[(long long)k * ow]; }, v_coeff + (long long)oy * F.v_widest, v_count[oy]);
    }
    const float tiny = 7.5231638452626401e-37f;   // 2^-120
    float v[7];
    unsigned char *m = A.mask + F.out_px + e;
    if (!PLAIN) {
        const bool hole = r.w < tiny;             // un-weighted colour needed: left to the plain passes
        *m = hole ? 1 : 0;
        if (hole) { A.need_plain[f] = 1; return; }
        v[0] = v[1] = v[2] = 0.f; v[3] = r.w; v[4] = r.x; v[5] = r.y; v[6] = r.z;
        *dst = compose_at(A.cs, encode_px(v), ox, oy);
    } else if (*m) {
        v[0] = r.x; v[1] = r.y; v[2] = r.z; v[3] = 0.f; v[4] = v[5] = v[6] = 0.f;
        *dst = compose_at(A.cs, encode_px(v), ox, oy);
    }
}

// Tables and descriptors of every frame; frames of equal geometry share one plan.  Frame groups bound the float
// intermediate: a group closes before the frame that would take it past the budget (a frame alone may exceed it).
int plan_scale_mixed(b200timg_ctx *ctx, const b200timg_mixed_batch *mb, MixedPlan &mp, bool sixel_rows) {
    const int n = mb->n_frames;
    unsigned long long budget = 2ull << 30;
    if (const char *e = getenv("B200TIMG_MIXED_GROUP_BYTES")) budget = std::max(1ull, strtoull(e, nullptr, 10));   // test knob
    std::vector<MixedScaleFrame> desc(n);
    std::vector<int32_t> tab;
    struct Geom { int iw, ih, ow, oh; unsigned long long tab; int hw, vw, vertical_first, h_sequential, copy_only; };
    std::vector<Geom> geoms;
    std::map<std::tuple<int, int, int, int>, size_t> index;     // geometry -> its entry in geoms
    mp.p1.assign(n + 1, 0); mp.p2.assign(n + 1, 0);
    mp.group_end.clear();
    unsigned long long p1 = 0, p2 = 0, out_px = 0, group_tmp = 0;
    ResamplePlan pl;
    for (int f = 0; f < n; ++f) {
        const b200timg_frame &F = mb->frames[f];
        MixedScaleFrame &D = desc[f];
        const auto key = std::make_tuple(F.src_w, F.src_h, F.out_w, F.out_h);
        const auto hit = index.find(key);
        const size_t g = hit != index.end() ? hit->second : geoms.size();
        if (g == geoms.size()) {
            index.emplace(key, g);
            if (!build_resample_plan(F.src_w, F.src_h, F.out_w, F.out_h, &pl))
                return ctx->fail(B200TIMG_EINVAL, "mixed batch: frame %d: degenerate geometry %dx%d -> %dx%d", f, F.src_w, F.src_h,
                                 F.out_w, F.out_h);
            geoms.push_back({F.src_w, F.src_h, F.out_w, F.out_h, tab.size(), pl.h.widest, pl.v.widest, pl.vertical_first ? 1 : 0,
                             pl.h_sequential ? 1 : 0, pl.copy_only ? 1 : 0});
            auto put = [&](const void *p, size_t words) { const int32_t *w = static_cast<const int32_t *>(p); tab.insert(tab.end(), w, w + words); };
            put(pl.h.first.data(), F.out_w); put(pl.h.count.data(), F.out_w);
            put(pl.v.first.data(), F.out_h); put(pl.v.count.data(), F.out_h);
            put(pl.h.coeff.data(), pl.h.coeff.size()); put(pl.v.coeff.data(), pl.v.coeff.size());
        }
        const Geom &G = geoms[g];
        D.src_off = F.src_offset;
        D.out_px = out_px;
        D.tab = G.tab;
        D.iw = F.src_w; D.ih = F.src_h; D.ow = F.out_w; D.oh = F.out_h;
        D.h_widest = G.hw; D.v_widest = G.vw;
        D.vertical_first = G.vertical_first; D.h_sequential = G.h_sequential; D.copy_only = G.copy_only;
        D.out_rows = sixel_rows ? (F.out_h + 5) / 6 * 6 : F.out_h;
        const unsigned long long elems = D.copy_only ? 0ull
                                       : D.vertical_first ? (unsigned long long)F.out_h * F.src_w : (unsigned long long)F.src_h * F.out_w;
        if (group_tmp && (group_tmp + elems) * sizeof(float4) > budget) { mp.group_end.push_back(f); group_tmp = 0; }
        D.tmp_off = group_tmp;
        group_tmp += elems;
        mp.tmp_elems = std::max<size_t>(mp.tmp_elems, (size_t)group_tmp);
        mp.p1[f] = (unsigned)p1; mp.p2[f] = (unsigned)p2;
        p1 += (elems + 255) / 256;
        p2 += ((unsigned long long)F.out_w * F.out_h + 255) / 256;
        out_px += (unsigned long long)F.out_w * D.out_rows;
        if (p1 > 0x7fffffffull || p2 > 0x7fffffffull)
            return ctx->fail(B200TIMG_EINVAL, "mixed batch: more than 2^31 - 1 scaler work items in one call (at frame %d)", f);
    }
    mp.group_end.push_back(n);
    mp.p1[n] = (unsigned)p1; mp.p2[n] = (unsigned)p2;
    mp.out_px = out_px;
    mp.o_scale = mixed_put(mp.arena, desc.data(), sizeof(MixedScaleFrame) * n);
    mp.o_p1 = mixed_put(mp.arena, mp.p1.data(), sizeof(unsigned) * (n + 1));
    mp.o_p2 = mixed_put(mp.arena, mp.p2.data(), sizeof(unsigned) * (n + 1));
    mp.o_tab = mixed_put(mp.arena, tab.data(), sizeof(int32_t) * tab.size());
    return B200TIMG_OK;
}

// The sixel encoder's pad strip of every frame (rows oh .. out_rows - 1), one CTA per frame: what the uniform batch does
// with a memset and a compose from start_row = oh (SixelCanvas::Send, src/sixel-canvas.cc:109-120).
__global__ void __launch_bounds__(256)
mixed_pad_kernel(const MixedScaleFrame *__restrict__ frames, uint32_t *__restrict__ out, ComposeSpec cs) {
    const MixedScaleFrame F = frames[blockIdx.x];
    const int n = (F.out_rows - F.oh) * F.ow;
    uint32_t *strip = out + F.out_px + (long long)F.oh * F.ow;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int y = i / F.ow, x = i - y * F.ow;
        strip[i] = compose_at(cs, 0u, x, F.oh + y);
    }
}

int launch_pad_mixed(b200timg_ctx *ctx, const MixedPlan &mp, const char *d_arena, uint8_t *d_out, int n_frames, const ComposeSpec &cs) {
    B2_KERNEL(ctx, "mixed_pad_kernel");
    mixed_pad_kernel<<<n_frames, 256, 0, ctx->stream>>>(reinterpret_cast<const MixedScaleFrame *>(d_arena + mp.o_scale),
                                                        reinterpret_cast<uint32_t *>(d_out), cs);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

int launch_scale_mixed(b200timg_ctx *ctx, const MixedPlan &mp, const char *d_arena, const uint8_t *d_src, uint8_t *d_out,
                       int n_frames, int bgra, const ComposeSpec &cs) {
    // scratch: [intermediate of the largest group | need_plain per frame | mask per output pixel]
    const size_t o_flag = (sizeof(float4) * std::max<size_t>(1, mp.tmp_elems) + 255) / 256 * 256;
    const size_t o_mask = o_flag + (sizeof(int) * (size_t)n_frames + 255) / 256 * 256;
    B2_CUDA(ctx, ctx->scale_tmp.reserve(o_mask + (size_t)mp.out_px));
    char *tb = ctx->scale_tmp.as<char>();
    MixedScaleArgs A;
    A.src = d_src;
    A.frames = reinterpret_cast<const MixedScaleFrame *>(d_arena + mp.o_scale);
    A.tab = reinterpret_cast<const int32_t *>(d_arena + mp.o_tab);
    A.tmp = reinterpret_cast<float4 *>(tb);
    A.need_plain = reinterpret_cast<int *>(tb + o_flag);
    A.mask = reinterpret_cast<unsigned char *>(tb + o_mask);
    A.out = reinterpret_cast<uint32_t *>(d_out);
    A.n_frames = n_frames; A.bgra = bgra; A.cs = cs;
    B2_CUDA(ctx, cudaMemsetAsync(A.need_plain, 0, sizeof(int) * (size_t)n_frames, ctx->stream));
    int f0 = 0;
    for (const int f1 : mp.group_end) {
        for (int plain = 0; plain < 2; ++plain) {
            // a group without pass-1 work (copy_only frames only) still launches one CTA, so that the number of
            // launches depends on the group count alone
            A.start = reinterpret_cast<const unsigned *>(d_arena + mp.o_p1);
            A.b0 = mp.p1[f0]; A.b1 = mp.p1[f1];
            B2_KERNEL(ctx, plain ? "mixed_plain_kernels" : "mixed_pass1_kernel");
            if (plain) mixed_pass1_kernel<true><<<std::max(1u, A.b1 - A.b0), 256, 0, ctx->stream>>>(A);
            else mixed_pass1_kernel<false><<<std::max(1u, A.b1 - A.b0), 256, 0, ctx->stream>>>(A);
            B2_LAUNCH_CHECK(ctx);
            A.start = reinterpret_cast<const unsigned *>(d_arena + mp.o_p2);
            A.b0 = mp.p2[f0]; A.b1 = mp.p2[f1];
            B2_KERNEL(ctx, plain ? "mixed_plain_kernels" : "mixed_pass2_kernel");
            if (plain) mixed_pass2_kernel<true><<<std::max(1u, A.b1 - A.b0), 256, 0, ctx->stream>>>(A);
            else mixed_pass2_kernel<false><<<std::max(1u, A.b1 - A.b0), 256, 0, ctx->stream>>>(A);
            B2_LAUNCH_CHECK(ctx);
        }
        f0 = f1;
    }
    return B200TIMG_OK;
}

}  // namespace b200timg

// Host-only introspection of the resampling plan (tests pin it against the oracle on CPU).
extern "C" int b200timg_resample_plan(int in_w, int in_h, int out_w, int out_h, int axis, int *widest,
                                      int *flags, int32_t *first, int32_t *count, int32_t *lead,
                                      float *coeff, size_t coeff_cap) {
    b200timg::ResamplePlan plan;
    if (!b200timg::build_resample_plan(in_w, in_h, out_w, out_h, &plan)) return B200TIMG_EINVAL;
    const b200timg::AxisTable &T = axis == 0 ? plan.h : plan.v;
    if (widest) *widest = T.widest;
    if (flags) *flags = (plan.vertical_first ? 1 : 0) | (plan.copy_only ? 2 : 0) | (plan.h_sequential ? 4 : 0);
    if (coeff_cap < T.coeff.size()) return B200TIMG_ENOSPC;
    if (first) memcpy(first, T.first.data(), sizeof(int32_t) * T.out_size);
    if (count) memcpy(count, T.count.data(), sizeof(int32_t) * T.out_size);
    if (lead) memcpy(lead, T.lead.data(), sizeof(int32_t) * T.out_size);
    if (coeff) memcpy(coeff, T.coeff.data(), sizeof(float) * T.coeff.size());
    return B200TIMG_OK;
}
