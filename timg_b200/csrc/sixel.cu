// K4-K6: what libsixel computes inside SixelCanvas::Send (src/sixel-canvas.cc:134-148) --
//   sixel_dither_new(256); sixel_dither_initialize(RGBA8888, LARGE_LUM, REP_AVERAGE_COLORS,
//   QUALITY_AUTO); sixel_encode(...)
// restated for the device.  libsixel is not part of the reference tree; the algorithm below is
// the published one (quant.c: computeHistogram / mediancut / lookup_fast / diffuse_fs; tosixel.c)
// with the two raster-order dependencies replaced by order-free rules so it can run in parallel
// (oracle/sixel_oracle.c "mode 1" is the CPU statement of exactly these semantics, and the tests
// require bit-identical palettes / index planes / decoded images against it):
//   * the colour table handed to median cut starts in bucket order (libsixel: first-seen order;
//     only the treatment of equal sort keys differs);
//   * the nearest-palette memo of a 15-bit colour cell is the nearest entry to the cell CENTRE
//     (libsixel: to the first pixel that happened to hit the cell in raster order).
// Everything else -- sampling stride, 15-bit histogram, luminance-weighted split axis, median by
// pixel count, box order by population, plain-mean representative, Floyd-Steinberg with the error
// added into 8-bit clamped pixels tap by tap (7/16 right, 3/16 below-left, 5/16 below, 1/16
// below-right, C truncation, no diffusion from the last row/column, x=0's below-left tap landing
// on the same row's last pixel) -- is libsixel's.
//
// Kernels (per frame unless noted):
//   sixel_palette_kernel   1 CTA : sampled histogram (packed u16 smem atomics) -> compaction ->
//                                  median cut (stable counting sort by 5-bit key, block scans)
//   sixel_lut_kernel       32 CTAs: 32768-entry nearest-colour table
//   sixel_dither_kernel    1 CTA : FS wavefront; a warp owns a band of 32 rows with a 2-column
//                                  skew between lanes (errors handed down by shuffle), bands are
//                                  pipelined warp to warp through a boundary row + progress flag
//   sixel_emit_kernel<0/1> 1 CTA per 6-row band: sizes, then bytes (per-colour RLE rows)
// Algorithmic bytes per frame: 4*W*H read + encoded bytes written; index plane (1 B/px), boundary
// rows, LUT and tables are intermediates.
#include <cstdlib>

#include "sixel.cuh"

namespace b200timg {

constexpr int PT = 1024;   // palette kernel threads

// quant.c largestByLuminosity: spreads are in 5-bit key units, colour values are key << 3
__device__ __forceinline__ int pick_plane(int d0, int d1, int d2) {
    const double lum[3] = {0.2989, 0.5866, 0.1145};
    const int spreads[3] = {d0 << 3, d1 << 3, d2 << 3};
    int plane = 0; double best = 0.0;
#pragma unroll
    for (int p = 0; p < 3; ++p) { const double sp = lum[p] * (double)spreads[p]; if (sp > best) { plane = p; best = sp; } }
    return plane;
}

// ---- per-frame geometry of the front and back kernels ------------------------------------------------------------
// Each kernel below reads the quantities that differ between frames through an accessor:
//   *Uniform  a b200timg_batch: every frame has the launch's geometry, frame f at f times the frame size, the CTA's frame
//             and item from blockIdx as before (these instantiations compile to the same SASS as the plain kernels did)
//   *Mixed    a mixed batch: a MixedSixelFrame per frame and flat item lists (MixedSixelParams)
struct NoMixed {};                        // the uniform kernels' (unused) last parameter

struct PaletteUniform {                   // one CTA per frame
    typedef NoMixed Params;
    int w, h; const SixelWork &W; int f;
    __device__ __forceinline__ PaletteUniform(int w_, int h_, const SixelWork &W_, const NoMixed &) : w(w_), h(h_), W(W_), f(blockIdx.x) {}
    __device__ __forceinline__ bool skip() const { return false; }
    __device__ __forceinline__ long long npix() const { return (long long)w * h; }
    __device__ __forceinline__ long long px0(long long n) const { return (long long)f * n; }
    __device__ __forceinline__ int ent_cap() const { return W.ent_cap; }
    __device__ __forceinline__ long long ent0() const { return (long long)f * W.ent_cap; }
};
struct PaletteMixed {                     // one CTA per listed frame (a launch may list none: one idle CTA)
    typedef MixedSixelParams Params;
    MixedSixelFrame D; int f; bool out;
    __device__ __forceinline__ PaletteMixed(int, int, const SixelWork &, const MixedSixelParams &P) {
        out = (int)blockIdx.x >= P.n_list;
        f = out ? 0 : P.list[blockIdx.x];
        D = P.desc[f];
    }
    __device__ __forceinline__ bool skip() const { return out; }
    __device__ __forceinline__ long long npix() const { return (long long)D.w * D.h; }
    __device__ __forceinline__ long long px0(long long) const { return (long long)D.fb_px; }
    __device__ __forceinline__ int ent_cap() const { return D.ent_cap; }
    __device__ __forceinline__ long long ent0() const { return (long long)D.ent; }
};

// SMEM_TABLES: the two median-cut tables live in shared memory (the histogram aliases the second
// one: it is dead once the first is compacted); otherwise they are in global memory (L2).
template <bool SMEM_TABLES, class G>
__global__ void __launch_bounds__(PT)
sixel_palette_kernel(const uint32_t *__restrict__ fb, int w, int h, SixelWork W, typename G::Params M) {
    extern __shared__ uint32_t s_hist[];               // 16384 words: two u16 counters per word (then table T)
    __shared__ uint32_t s_w[PT / 32];
    __shared__ int b_ind[256], b_col[256], b_med[256], t_ind[256], t_col[256], t_med[256];   // b_med: cached split (-1: none)
    __shared__ uint32_t b_sum[256], b_low[256], t_sum[256], t_low[256];
    __shared__ int s_mn[3], s_mx[3];
    __shared__ uint32_t s_cnt[32], s_base[32], s_run[32];
    __shared__ unsigned short s_wh[32][32];
    __shared__ uint32_t w_cnt[32][32], w_base[32][32], w_run[32][32];      // per-warp counting-sort scratch
    __shared__ int s_todo[32], s_ntodo, s_boxes, s_done;
    __shared__ unsigned long long s_med;

    const G g(w, h, W, M);
    if (g.skip()) return;
    const int f = g.f, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const long long npix = g.npix();
    const uint32_t *frame = fb + g.px0(npix);
    SixelFrameHdr *hdr = W.hdr + f;
    const int t_words = g.ent_cap() > 16384 ? g.ent_cap() : 16384;
    uint32_t *E = SMEM_TABLES ? s_hist + t_words : W.ent_a + g.ent0();
    uint32_t *T = SMEM_TABLES ? s_hist : W.ent_b + g.ent0();

    // quant.c computeHistogram, QUALITY_LOW: step = length/depth/max_sample*depth (bytes)
    unsigned long long step_px = (unsigned long long)npix / 18383ull;
    if ((unsigned long long)npix < 18383ull) step_px = 6;
    if (step_px == 0) step_px = 1;
    const long long ns = (npix + (long long)step_px - 1) / (long long)step_px;

    for (int i = tid; i < 16384; i += PT) s_hist[i] = 0;
    __syncthreads();
    for (long long k = tid; k < ns; k += PT) {
        const uint32_t b = hash15(frame[k * (long long)step_px]);
        atomicAdd(&s_hist[b >> 1], 1u << (16 * (b & 1)));    // counts <= ns <= 36766 < 65536: no carry
    }
    __syncthreads();
    // compaction in bucket order: thread t owns buckets [32t, 32t+32)
    uint32_t mine = 0;
    for (int k = 0; k < 16; ++k) { const uint32_t v = s_hist[tid * 16 + k]; mine += ((v & 0xffff) != 0) + ((v >> 16) != 0); }
    uint32_t n_ent;
    uint32_t pos = block_excl_scan<PT>(mine, s_w, n_ent);
    for (int k = 0; k < 16; ++k) {
        const uint32_t v = s_hist[tid * 16 + k];
        const uint32_t b0 = (uint32_t)(tid * 32 + 2 * k);
        if (v & 0xffff) E[pos++] = (b0 << 16) | (v & 0xffff);
        if (v >> 16) E[pos++] = ((b0 + 1) << 16) | (v >> 16);
    }
    __syncthreads();
    if (tid == 0) { hdr->origcolors = n_ent; hdr->diffuse = n_ent > 256 ? 1 : 0; }
    if (n_ent <= 256) {                                 // "Image already has few enough colors"
        if (tid < 256) {
            uint32_t pal = 0;
            if ((uint32_t)tid < n_ent) { const uint32_t e = E[tid]; pal = (key5(e, 0) << 3) | (key5(e, 1) << 11) | (key5(e, 2) << 19); }
            hdr->palette[tid] = pal;
        }
        if (tid == 0) hdr->ncolors = n_ent;
        return;
    }
    // ---- mediancut().  The reference algorithm is sequential: always split the first box (in
    // population order) that still holds >= 2 colours, 255 times.  A split only reorders the entries
    // inside its own box and its outcome (median index, lower population) does not depend on any other
    // box, so splits are computed speculatively, up to 32 boxes per round with one warp each (block-wide
    // for boxes > 1024 entries), cached per box, and then consumed by one warp in exactly the
    // sequential order.  Unused speculative results are harmless (the box is merely left sorted).
    {
        uint32_t sacc = 0;
        for (uint32_t i = tid; i < n_ent; i += PT) sacc += E[i] & 0xffff;
        uint32_t total; const uint32_t dummy = block_excl_scan<PT>(sacc, s_w, total); (void)dummy;
        if (tid == 0) { b_ind[0] = 0; b_col[0] = (int)n_ent; b_sum[0] = total; b_med[0] = -1; s_boxes = 1; s_done = 0; }
    }
    for (;;) {
        __syncthreads();
        if (wid == 0) {                                  // up to 32 uncached splittable boxes, in order
            const int nb = s_boxes;
            int count = 0;
            for (int c0 = 0; c0 < nb; c0 += 32) {
                const int j = c0 + lane;
                const bool flag = j < nb && b_col[j] >= 2 && b_med[j] < 0;
                const uint32_t m = __ballot_sync(0xffffffffu, flag);
                const int pos = count + __popc(m & ((1u << lane) - 1));
                if (flag && pos < 32) s_todo[pos] = j;
                count += __popc(m);
            }
            if (lane == 0) s_ntodo = min(count, 32);
        }
        __syncthreads();
        const int ntodo = s_ntodo;
        // (a) big boxes of this round: block-wide, one after the other
        for (int t = 0; t < ntodo; ++t) {
            const int bi = s_todo[t];
            const int start = b_ind[bi], size = b_col[bi];
            if (size <= 1024) continue;
            const uint32_t sm = b_sum[bi];
            uint32_t *B = E + start, *TB = T + start;
            if (tid == 0) { s_mn[0] = s_mn[1] = s_mn[2] = 31; s_mx[0] = s_mx[1] = s_mx[2] = 0; s_med = ~0ull; }
            if (tid < 32) { s_cnt[tid] = 0; s_run[tid] = 0; }
            __syncthreads();
            int mn0 = 31, mn1 = 31, mn2 = 31, mx0 = 0, mx1 = 0, mx2 = 0;         // findBoxBoundaries
            for (int i = tid; i < size; i += PT) {
                const uint32_t e = B[i];
                const int k0 = key5(e, 0), k1 = key5(e, 1), k2 = key5(e, 2);
                mn0 = min(mn0, k0); mx0 = max(mx0, k0); mn1 = min(mn1, k1); mx1 = max(mx1, k1); mn2 = min(mn2, k2); mx2 = max(mx2, k2);
            }
#pragma unroll
            for (int d = 16; d; d >>= 1) {
                mn0 = min(mn0, __shfl_xor_sync(0xffffffffu, mn0, d)); mx0 = max(mx0, __shfl_xor_sync(0xffffffffu, mx0, d));
                mn1 = min(mn1, __shfl_xor_sync(0xffffffffu, mn1, d)); mx1 = max(mx1, __shfl_xor_sync(0xffffffffu, mx1, d));
                mn2 = min(mn2, __shfl_xor_sync(0xffffffffu, mn2, d)); mx2 = max(mx2, __shfl_xor_sync(0xffffffffu, mx2, d));
            }
            if (lane == 0) {
                atomicMin(&s_mn[0], mn0); atomicMax(&s_mx[0], mx0); atomicMin(&s_mn[1], mn1); atomicMax(&s_mx[1], mx1);
                atomicMin(&s_mn[2], mn2); atomicMax(&s_mx[2], mx2);
            }
            __syncthreads();
            const int plane = pick_plane(s_mx[0] - s_mn[0], s_mx[1] - s_mn[1], s_mx[2] - s_mn[2]);
            for (int i = tid; i < size; i += PT) atomicAdd(&s_cnt[key5(B[i], plane)], 1u);   // stable counting sort
            __syncthreads();
            if (tid < 32) {
                const uint32_t c = s_cnt[tid]; uint32_t inc = c;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += o; }
                s_base[tid] = inc - c;
            }
            for (int t0 = 0; t0 < size; t0 += PT) {
                s_wh[wid][lane] = 0;
                __syncthreads();
                const int i = t0 + tid;
                const bool valid = i < size;
                uint32_t e = 0, k = 0, rank = 0;
                const uint32_t vmask = __ballot_sync(0xffffffffu, valid);
                if (valid) {
                    e = B[i]; k = key5(e, plane);
                    const uint32_t m = __match_any_sync(vmask, k);
                    rank = __popc(m & ((1u << lane) - 1));
                    if (rank == 0) s_wh[wid][k] = (unsigned short)__popc(m);
                }
                __syncthreads();
                if (valid) {
                    uint32_t pp = s_base[k] + s_run[k] + rank;
                    for (int w2 = 0; w2 < wid; ++w2) pp += s_wh[w2][k];
                    TB[pp] = e;
                }
                __syncthreads();
                if (tid < 32) { uint32_t acc = 0; for (int w2 = 0; w2 < 32; ++w2) acc += s_wh[w2][tid]; s_run[tid] += acc; }
                __syncthreads();
            }
            for (int i = tid; i < size; i += PT) B[i] = TB[i];
            __syncthreads();
            {   // median by pixel count: smallest i in [1, size-2] with sum(count[0..i)) >= sm/2, else size-1
                const uint32_t half = sm / 2;
                uint32_t carry = 0;
                for (int t0 = 0; t0 < size; t0 += PT) {
                    const int i = t0 + tid;
                    const uint32_t c = i < size ? (B[i] & 0xffff) : 0;
                    uint32_t tot; const uint32_t before = carry + block_excl_scan<PT>(c, s_w, tot);
                    if (i >= 1 && i <= size - 2 && before >= half) atomicMin(&s_med, ((unsigned long long)i << 32) | before);
                    carry += tot;
                    __syncthreads();
                    if (s_med != ~0ull) break;
                }
            }
            __syncthreads();
            if (tid == 0) {
                if (s_med != ~0ull) { b_med[bi] = (int)(s_med >> 32); b_low[bi] = (uint32_t)s_med; }
                else { b_med[bi] = size - 1; b_low[bi] = sm - (B[size - 1] & 0xffff); }
            }
            __syncthreads();
        }
        // (b) small boxes of this round: one warp each, all at once
        if (wid < ntodo) {
            const int bi = s_todo[wid];
            const int start = b_ind[bi], size = b_col[bi];
            if (size <= 1024) {
                const uint32_t sm = b_sum[bi];
                uint32_t *B = E + start, *TB = T + start;
                uint32_t *cnt = w_cnt[wid], *base = w_base[wid], *run = w_run[wid];
                cnt[lane] = 0; run[lane] = 0;
                int mn0 = 31, mn1 = 31, mn2 = 31, mx0 = 0, mx1 = 0, mx2 = 0;
                for (int i = lane; i < size; i += 32) {
                    const uint32_t e = B[i];
                    const int k0 = key5(e, 0), k1 = key5(e, 1), k2 = key5(e, 2);
                    mn0 = min(mn0, k0); mx0 = max(mx0, k0); mn1 = min(mn1, k1); mx1 = max(mx1, k1); mn2 = min(mn2, k2); mx2 = max(mx2, k2);
                }
#pragma unroll
                for (int d = 16; d; d >>= 1) {
                    mn0 = min(mn0, __shfl_xor_sync(0xffffffffu, mn0, d)); mx0 = max(mx0, __shfl_xor_sync(0xffffffffu, mx0, d));
                    mn1 = min(mn1, __shfl_xor_sync(0xffffffffu, mn1, d)); mx1 = max(mx1, __shfl_xor_sync(0xffffffffu, mx1, d));
                    mn2 = min(mn2, __shfl_xor_sync(0xffffffffu, mn2, d)); mx2 = max(mx2, __shfl_xor_sync(0xffffffffu, mx2, d));
                }
                const int plane = pick_plane(mx0 - mn0, mx1 - mn1, mx2 - mn2);
                __syncwarp();
                for (int t0 = 0; t0 < size; t0 += 32) {            // stable counting sort by the 5-bit key
                    const int i = t0 + lane;
                    const bool valid = i < size;
                    const uint32_t vm = __ballot_sync(0xffffffffu, valid);
                    if (valid) {
                        const uint32_t k = key5(B[i], plane);
                        const uint32_t m = __match_any_sync(vm, k);
                        if ((m & ((1u << lane) - 1)) == 0) cnt[k] += __popc(m);
                    }
                    __syncwarp();
                }
                {
                    const uint32_t c = cnt[lane]; uint32_t inc = c;
#pragma unroll
                    for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += o; }
                    base[lane] = inc - c;
                }
                __syncwarp();
                for (int t0 = 0; t0 < size; t0 += 32) {
                    const int i = t0 + lane;
                    const bool valid = i < size;
                    const uint32_t vm = __ballot_sync(0xffffffffu, valid);
                    uint32_t k = 0, m = 0;
                    if (valid) {
                        const uint32_t e = B[i];
                        k = key5(e, plane);
                        m = __match_any_sync(vm, k);
                        TB[base[k] + run[k] + __popc(m & ((1u << lane) - 1))] = e;
                    }
                    __syncwarp();
                    if (valid && (m & ((1u << lane) - 1)) == 0) run[k] += __popc(m);
                    __syncwarp();
                }
                for (int i = lane; i < size; i += 32) B[i] = TB[i];
                __syncwarp();
                const uint32_t half = sm / 2;
                uint32_t carry = 0; int median = size - 1; uint32_t lower = 0; bool found = false;
                for (int t0 = 0; t0 < size && !found; t0 += 32) {
                    const int i = t0 + lane;
                    const uint32_t c = i < size ? (B[i] & 0xffff) : 0;
                    uint32_t inc = c;
#pragma unroll
                    for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += o; }
                    const uint32_t before = carry + inc - c;
                    const uint32_t hit = __ballot_sync(0xffffffffu, i >= 1 && i <= size - 2 && before >= half);
                    if (hit) {
                        const int src = __ffs(hit) - 1;
                        median = t0 + src; lower = __shfl_sync(0xffffffffu, before, src); found = true;
                    }
                    carry += __shfl_sync(0xffffffffu, inc, 31);
                }
                if (!found) lower = sm - (B[size - 1] & 0xffff);
                if (lane == 0) { b_med[bi] = median; b_low[bi] = lower; }
            }
        }
        __syncthreads();
        // (c) consume cached splits in the sequential order (one warp)
        if (wid == 0) {
            int done = 0;
            for (;;) {
                const int nb = s_boxes;
                if (nb >= 256) { done = 1; break; }
                int first = 1 << 30;
                for (int j = lane; j < nb; j += 32) if (b_col[j] >= 2) { first = j; break; }
#pragma unroll
                for (int d = 16; d; d >>= 1) first = min(first, __shfl_xor_sync(0xffffffffu, first, d));
                if (first >= nb) { done = 1; break; }
                if (b_med[first] < 0) break;                      // not computed yet: next round
                const int ia = first, in_ = nb, nb1 = nb + 1;
                const int start = b_ind[ia], size = b_col[ia], median = b_med[ia];
                const uint32_t sm = b_sum[ia], lower = b_low[ia];
                __syncwarp();
                if (lane == 0) {
                    b_col[ia] = median; b_sum[ia] = lower; b_med[ia] = -1;
                    b_ind[in_] = start + median; b_col[in_] = size - median; b_sum[in_] = sm - lower; b_med[in_] = -1;
                    s_boxes = nb1;
                }
                __syncwarp();
                // stable re-sort by population: only box ia (shrunk) and the new last box moved
                const uint32_t sA = lower, sN = sm - lower;
                int cntA = 0, cntN = 0;
                int my_pos[8];
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const int j = c * 32 + lane;
                    bool pa = false, pn = false;
                    my_pos[c] = -1;
                    if (j < nb1 && j != ia && j != in_) {
                        const uint32_t me = b_sum[j];
                        my_pos[c] = j - (j > ia ? 1 : 0) + (((sA > me) || (sA == me && ia < j)) ? 1 : 0) + ((sN > me) ? 1 : 0);
                        pa = (me > sA) || (me == sA && j < ia);
                        pn = me >= sN;
                    }
                    cntA += __popc(__ballot_sync(0xffffffffu, pa));
                    cntN += __popc(__ballot_sync(0xffffffffu, pn));
                }
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const int j = c * 32 + lane;
                    if (j < nb1) {
                        int pos = my_pos[c];
                        if (j == ia) pos = cntA + (sN > sA ? 1 : 0);
                        if (j == in_) pos = cntN + (sA >= sN ? 1 : 0);
                        t_ind[pos] = b_ind[j]; t_col[pos] = b_col[j]; t_sum[pos] = b_sum[j]; t_med[pos] = b_med[j]; t_low[pos] = b_low[j];
                    }
                }
                __syncwarp();
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const int j = c * 32 + lane;
                    if (j < nb1) { b_ind[j] = t_ind[j]; b_col[j] = t_col[j]; b_sum[j] = t_sum[j]; b_med[j] = t_med[j]; b_low[j] = t_low[j]; }
                }
                __syncwarp();
            }
            if (lane == 0) s_done = done;
        }
        __syncthreads();
        if (s_done) break;
    }
    // colormapFromBv, SIXEL_REP_AVERAGE_COLORS: plain mean of the box's colour values
    if (tid < 256) {
        uint32_t pal = 0;
        if (tid < s_boxes) {
            uint32_t s0 = 0, s1 = 0, s2 = 0; const int st = b_ind[tid], n = b_col[tid];
            for (int i = 0; i < n; ++i) { const uint32_t e = E[st + i]; s0 += key5(e, 0) << 3; s1 += key5(e, 1) << 3; s2 += key5(e, 2) << 3; }
            pal = (s0 / (uint32_t)n) | ((s1 / (uint32_t)n) << 8) | ((s2 / (uint32_t)n) << 16);
        }
        hdr->palette[tid] = pal;
    }
    if (tid == 0) hdr->ncolors = 256;
}

// nearest palette entry (first minimum, complexion 1) for the centre of every 15-bit cell
__global__ void __launch_bounds__(256)
sixel_lut_kernel(SixelWork W) {
    __shared__ uint32_t s_pal[256];
    const int f = blockIdx.y;
    const SixelFrameHdr *hdr = W.hdr + f;
    s_pal[threadIdx.x] = hdr->palette[threadIdx.x];
    __syncthreads();
    const int n = (int)hdr->ncolors;
    const uint32_t cell = blockIdx.x * 256 + threadIdx.x;
    // centre of the cell as packed bytes; squared distance = dot(|d|, |d|) with d the per-byte absolute difference
    // (VABSDIFF4 + IDP.4A); "first minimum" = minimum of (distance << 8 | index)
    const uint32_t c = (((cell >> 10) & 31) << 3 | 4) | ((((cell >> 5) & 31) << 3 | 4) << 8) | (((cell & 31) << 3 | 4) << 16);
    uint32_t best = 0xffffffffu;
    for (int i = 0; i < n; ++i) {
        const uint32_t d = __vabsdiffu4(c, s_pal[i]);
        best = min(best, (__dp4a(d, d, 0u) << 8) | (uint32_t)i);
    }
    const uint32_t bi = n > 0 ? (best & 255u) : 0u;
    W.lut[(long long)f * 32768 + cell] = (uint8_t)bi;
}

struct MapUniform {                       // frame blockIdx.y
    typedef NoMixed Params;
    long long n; int f;
    __device__ __forceinline__ MapUniform(long long npix, const NoMixed &, int f_) : n(npix), f(f_) {}
    __device__ __forceinline__ long long npix() const { return n; }
    __device__ __forceinline__ long long px0() const { return (long long)f * n; }
    __device__ __forceinline__ long long idx0() const { return (long long)f * n; }
};
struct MapMixed {
    typedef MixedSixelParams Params;
    MixedSixelFrame D;
    __device__ __forceinline__ MapMixed(long long, const MixedSixelParams &P, int f) : D(P.desc[f]) {}
    __device__ __forceinline__ long long npix() const { return (long long)D.w * D.h; }
    __device__ __forceinline__ long long px0() const { return (long long)D.fb_px; }
    __device__ __forceinline__ long long idx0() const { return (long long)D.idx; }
};

// no diffusion (<= 256 distinct sampled colours): plain table lookup per pixel
template <class G>
__global__ void __launch_bounds__(256)
sixel_map_kernel(const uint32_t *__restrict__ fb, long long npix, SixelWork W, typename G::Params M) {
    const int f = blockIdx.y;
    if (W.hdr[f].diffuse) return;
    const uint8_t *lut = W.lut + (long long)f * 32768;
    const G g(npix, M, f);
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < g.npix(); i += stride)
        W.index[g.idx0() + i] = lut[hash15(fb[g.px0() + i])];
}

// ---- Floyd-Steinberg wavefront --------------------------------------------------------------
constexpr uint32_t EZ = 256u | (256u << 9) | (256u << 18);     // packed zero error (each channel biased by 256)
__device__ __forceinline__ int fs_tap(int v, int e, int k) {      // error_diffuse(): c = v + e*k/16, clamp
    const int t = e * k;
    const int q = (t + ((t >> 31) & 15)) >> 4;                  // C division truncates toward zero
    return min(255, max(0, v + q));
}
// One pixel's quantisation error, unpacked: e[c] in [-255,255] and bias[c] = (e<0 ? 15 : 0), so that
// error_diffuse()'s  e*k/16 (C truncation)  is  (e*k + bias) >> 4  -- one IMAD and one shift per tap.
struct FsErr {
    int e[3], b[3];
    __device__ __forceinline__ void zero() { e[0] = e[1] = e[2] = 0; b[0] = b[1] = b[2] = 0; }
    __device__ __forceinline__ void set(int r, int g, int bl) {
        e[0] = r; e[1] = g; e[2] = bl;
        b[0] = (r >> 31) & 15; b[1] = (g >> 31) & 15; b[2] = (bl >> 31) & 15;
    }
    __device__ __forceinline__ void unpack(uint32_t p) { set((int)(p & 511) - 256, (int)((p >> 9) & 511) - 256, (int)((p >> 18) & 511) - 256); }
    __device__ __forceinline__ uint32_t pack() const { return (uint32_t)(e[0] + 256) | ((uint32_t)(e[1] + 256) << 9) | ((uint32_t)(e[2] + 256) << 18); }
};
__device__ __forceinline__ int fs_add(int v, const FsErr &er, int c, int k) {
    return min(255, max(0, v + ((er.e[c] * k + er.b[c]) >> 4)));
}
constexpr int DW_MAX = 24;     // warps per frame CTA (upper bound; the launch picks how many)
constexpr int DCH = 16;        // columns per staged chunk
constexpr int DIN_STRIDE = DCH + 1;              // u32 words per staged row (odd: lanes hit distinct banks)
constexpr int DOUT_STRIDE = 20;                  // bytes per staged output row (5 words: conflict-free)
constexpr int DWARP_SMEM = 2 * 32 * DIN_STRIDE * 4 + 32 * DOUT_STRIDE;   // per warp

// A warp owns a band of 32 rows; lane l runs row band*32+l two columns behind lane l-1, so the three
// errors it needs from the row above arrive by one shuffle per step.  Pixels are staged through
// shared memory in chunks of DCH steps, pre-skewed (row r of the tile starts at column base-2r) and
// loaded/stored by half-warps so global traffic is 64-byte segments instead of 32 scattered lines.
// Consecutive bands are pipelined through a boundary row of packed errors in global memory (L2)
// plus a per-band progress counter in shared memory.
__global__ void __launch_bounds__(DW_MAX * 32)
sixel_dither_kernel(const uint32_t *__restrict__ fb, int w, int h, int nwarps, SixelWork W) {
    extern __shared__ __align__(16) uint8_t s_dyn[];              // lut[32768] | per-warp tiles
    __shared__ uint32_t s_pal[256];
    __shared__ volatile int s_progress[2048];                     // columns completed by each band's last row
    const int f = blockIdx.x;
    const SixelFrameHdr *hdr = W.hdr + f;
    if (!hdr->diffuse) return;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int nthreads = nwarps * 32;
    uint8_t *s_lut = s_dyn;
    for (int i = tid; i < 32768 / 4; i += nthreads)
        reinterpret_cast<uint32_t *>(s_lut)[i] = reinterpret_cast<const uint32_t *>(W.lut + (long long)f * 32768)[i];
    for (int i = tid; i < 256; i += nthreads) s_pal[i] = hdr->palette[i];     // nthreads may be < 256
    for (int i = tid; i < W.nb32; i += nthreads) s_progress[i] = 0;
    __syncthreads();
    uint32_t *s_in = reinterpret_cast<uint32_t *>(s_dyn + 32768 + (size_t)wid * DWARP_SMEM);   // [2][32][DIN_STRIDE]
    uint8_t *s_out = reinterpret_cast<uint8_t *>(s_in + 2 * 32 * DIN_STRIDE);                    // [32][DOUT_STRIDE]
    const uint32_t *frame = fb + (long long)f * w * h;
    uint8_t *index = W.index + (long long)f * w * h;
    uint32_t *bnd = W.boundary + (long long)f * W.nb32 * w;
    const int hrow = lane >> 4, hcol = lane & 15;                 // half-warp staging coordinates

    for (int band = wid; band < W.nb32; band += nwarps) {
        const int y = band * 32 + lane;
        const bool row_ok = y < h;
        const bool last_row = (y == h - 1);
        const uint32_t *bin = band > 0 ? bnd + (long long)(band - 1) * w : nullptr;
        uint32_t *bout = bnd + (long long)band * w;
        uint32_t last_e = EZ;
        FsErr up_m1, up_0, up_p1, own, e_first;
        up_m1.zero(); up_0.zero(); up_p1.zero(); own.zero(); e_first.zero();
        const int steps = w + 62, nchunks = (steps + DCH - 1) / DCH;
        // pre-skewed load of chunk c into registers: element i covers tile row 2i+hrow, column hcol
        uint32_t pre[16];
        auto load_chunk = [&](int c) {
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const int r = 2 * i + hrow, yy = band * 32 + r, x = c * DCH - 2 * r + hcol;
                pre[i] = (yy < h && x >= 0 && x < w) ? frame[(long long)yy * w + x] : 0u;
            }
        };
        auto store_chunk = [&](int c) {
            uint32_t *t = s_in + (c & 1) * 32 * DIN_STRIDE;
#pragma unroll
            for (int i = 0; i < 16; ++i) t[(2 * i + hrow) * DIN_STRIDE + hcol] = pre[i];
        };
        load_chunk(0); store_chunk(0);
        __syncwarp();
        for (int c = 0; c < nchunks; ++c) {
            const int t0 = c * DCH;
            if (c + 1 < nchunks) load_chunk(c + 1);                // in flight while this chunk computes
            uint32_t binreg = EZ;
            if (band > 0) {                                       // stay behind the previous band's last row
                const int need = min(w, t0 + DCH + 1);
                if (lane == 0) { while (s_progress[band - 1] < need) __nanosleep(32); __threadfence_block(); }
                __syncwarp();
                const int bx = t0 + 1 + lane;                     // lane 0 consumes bin[t+1] at step t
                if (lane < DCH && bx < w) binreg = __ldcg(bin + bx);
                if (c == 0 && lane == 0) up_p1.unpack(__ldcg(bin));   // e(0, y-1): lane 0 has no warm-up step
            }
            const uint32_t *tin = s_in + (c & 1) * 32 * DIN_STRIDE + lane * DIN_STRIDE;
            uint32_t bkeep = EZ;
            // interior chunk: every lane is strictly inside its row for all DCH steps and no lane runs the
            // frame's last row -> the step needs no range checks and always diffuses
            const bool interior = (t0 - 62 >= 1) && (t0 + DCH - 1 <= w - 2) && (band * 32 + 31 < h - 1);
            if (interior) {
#pragma unroll 4
                for (int j = 0; j < DCH; ++j) {
                    uint32_t recv = __shfl_up_sync(0xffffffffu, last_e, 1);
                    const uint32_t b0 = __shfl_sync(0xffffffffu, binreg, j);
                    if (lane == 0) recv = b0;
                    up_m1 = up_0; up_0 = up_p1; up_p1.unpack(recv);
                    const uint32_t px = tin[j];
                    int v[3] = {(int)(px & 0xff), (int)((px >> 8) & 0xff), (int)((px >> 16) & 0xff)};
#pragma unroll
                    for (int ch = 0; ch < 3; ++ch) {
                        v[ch] = fs_add(v[ch], up_m1, ch, 1);
                        v[ch] = fs_add(v[ch], up_0, ch, 5);
                        v[ch] = fs_add(v[ch], up_p1, ch, 3);
                        v[ch] = fs_add(v[ch], own, ch, 7);
                    }
                    const uint32_t cell = ((uint32_t)(v[0] >> 3) << 10) | ((uint32_t)(v[1] >> 3) << 5) | (uint32_t)(v[2] >> 3);
                    const uint32_t ci = s_lut[cell];
                    const uint32_t pal = s_pal[ci];
                    own.set(v[0] - (int)(pal & 0xff), v[1] - (int)((pal >> 8) & 0xff), v[2] - (int)((pal >> 16) & 0xff));
                    last_e = own.pack();
                    s_out[lane * DOUT_STRIDE + j] = (uint8_t)ci;
                    const uint32_t e31 = __shfl_sync(0xffffffffu, last_e, 31);
                    if (lane == j) bkeep = e31;
                }
            } else {
#pragma unroll 2
                for (int j = 0; j < DCH; ++j) {
                    const int t = t0 + j, x = t - 2 * lane;
                    uint32_t recv = __shfl_up_sync(0xffffffffu, last_e, 1);
                    const uint32_t b0 = __shfl_sync(0xffffffffu, binreg, j);
                    if (lane == 0) recv = b0;
                    up_m1 = up_0; up_0 = up_p1; up_p1.unpack(recv);
                    uint32_t ci = 0;
                    if (x >= 0 && x < w && row_ok) {
                        const uint32_t px = tin[j];
                        int v[3] = {(int)(px & 0xff), (int)((px >> 8) & 0xff), (int)((px >> 16) & 0xff)};
#pragma unroll
                        for (int ch = 0; ch < 3; ++ch) {
                            v[ch] = fs_add(v[ch], up_m1, ch, 1);                       // from (x-1, y-1)
                            v[ch] = fs_add(v[ch], up_0, ch, 5);                        // from (x,   y-1)
                            v[ch] = fs_add(v[ch], up_p1, ch, 3);                       // from (x+1, y-1)
                            if (x == w - 1) v[ch] = fs_add(v[ch], e_first, ch, 3);     // libsixel: (0,y)'s below-left tap
                            v[ch] = fs_add(v[ch], own, ch, 7);                         // from (x-1, y)
                        }
                        const uint32_t cell = ((uint32_t)(v[0] >> 3) << 10) | ((uint32_t)(v[1] >> 3) << 5) | (uint32_t)(v[2] >> 3);
                        ci = s_lut[cell];
                        const uint32_t pal = s_pal[ci];
                        if (x < w - 1 && !last_row) own.set(v[0] - (int)(pal & 0xff), v[1] - (int)((pal >> 8) & 0xff), v[2] - (int)((pal >> 16) & 0xff));
                        else own.zero();
                        if (x == 0) e_first = own;
                        last_e = own.pack();
                    } else if (x >= w) {
                        last_e = EZ;
                    }
                    s_out[lane * DOUT_STRIDE + j] = (uint8_t)ci;
                    const uint32_t e31 = __shfl_sync(0xffffffffu, last_e, 31);      // the band's last row, column t-62
                    if (lane == j) bkeep = e31;
                }
            }
            __syncwarp();
            // write this chunk's indices: half-warp per row, 16 contiguous bytes
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const int r = 2 * i + hrow, yy = band * 32 + r, x = t0 - 2 * r + hcol;
                if (yy < h && x >= 0 && x < w) index[(long long)yy * w + x] = s_out[r * DOUT_STRIDE + hcol];
            }
            {   // boundary row for the next band, then publish progress
                const int x = t0 + lane - 62;
                if (lane < DCH && x >= 0 && x < w) __stcg(bout + x, bkeep);
                __threadfence_block();                            // every storing lane orders its own store ...
                __syncwarp();                                     // ... before lane 0 raises the flag
                const int done = min(w, t0 + DCH - 62);
                if (lane == 0 && done > 0) s_progress[band] = done;
            }
            if (c + 1 < nchunks) store_chunk(c + 1);
            __syncwarp();
        }
    }
}

// ---- emit ------------------------------------------------------------------------------------
// Branch-light formatting for values < 10000 (run lengths, gaps and colour numbers are bounded by
// the frame width <= 4095 and 255): no loops, so lanes of a warp do not serialise on digit counts.
__device__ __forceinline__ uint32_t ndig4(uint32_t v) { return 1u + (v >= 10u) + (v >= 100u) + (v >= 1000u); }
__device__ __forceinline__ char *put_num4(char *o, uint32_t v) {
    const uint32_t d3 = v / 1000u, r3 = v - d3 * 1000u, d2 = r3 / 100u, r2 = r3 - d2 * 100u, d1 = r2 / 10u, d0 = r2 - d1 * 10u;
    if (v >= 1000u) *o++ = (char)('0' + d3);
    if (v >= 100u) *o++ = (char)('0' + d2);
    if (v >= 10u) *o++ = (char)('0' + d1);
    *o++ = (char)('0' + d0);
    return o;
}
__device__ __forceinline__ uint32_t rle_len(uint32_t n) { return n > 3u ? 2u + ndig4(n) : n; }   // tosixel.c sixel_put_flash
__device__ __forceinline__ char *put_rle(char *o, uint32_t n, char ch) {
    if (n > 3u) { *o++ = '!'; o = put_num4(o, n); *o++ = ch; }
    else { if (n > 0u) *o++ = ch; if (n > 1u) *o++ = ch; if (n > 2u) *o++ = ch; }
    return o;
}

constexpr int ET = 512, EW = ET / 32;
// sorted entry word: colour [18:26) | x [6:18) | bits [0:6)  -> ascending order == (colour, x)
__device__ __forceinline__ uint32_t ent_pack(uint32_t c, uint32_t x, uint32_t bits) { return (c << 18) | (x << 6) | bits; }

struct EmitGeom { int w, h, cols_per_warp; };

// Walk the sorted entries [lo, hi) once and call `emit(c, bits, gap, len, first_of_colour)` for every run
// that STARTS in the range (a run = same colour, consecutive x, same bits; it may extend past hi, and
// entries at lo that continue a run started before lo belong to their head's owner and are skipped).
// gap = blank columns between this run and the colour's previous entry (or x for its first entry).
template <typename F>
__device__ __forceinline__ void walk_runs(const uint32_t *sorted, int lo, int hi, int n, F emit) {
    int i = lo;
    uint32_t prev = 0; bool have_prev = false;          // the entry just before i, in sorted order
    if (i > 0 && i < hi) { prev = sorted[i - 1]; have_prev = true; }
    while (i < hi) {
        const uint32_t e = sorted[i];
        if (have_prev && e == prev + 64u) { prev = e; ++i; continue; }        // continues a run: x+1, same colour and bits
        uint32_t cur = e, L = 1;
        while (i + (int)L < n && sorted[i + L] == cur + 64u) { cur += 64u; ++L; }
        const uint32_t c = e >> 18, x = (e >> 6) & 4095u;
        const bool same_colour = have_prev && (prev >> 18) == c;
        emit(c, e & 63u, same_colour ? x - ((prev >> 6) & 4095u) - 1u : x, L, !same_colour);
        prev = cur; have_prev = true;
        i += (int)L;
    }
}

// One CTA per 6-row band.  (1) per-warp counting sort of the band's (colour, x, bits) entries by
// colour -- warps own contiguous column ranges, so warp-major order is x order and the sort is
// stable; (2) every run head sizes its "gap + run" bytes, block scan -> offsets; (3) WRITE: bytes.
__global__ void __launch_bounds__(ET)
sixel_emit_kernel(EmitGeom G, SixelWork W) {
    extern __shared__ uint32_t s_sorted[];                   // [6*w]
    __shared__ uint32_t s_cnt[EW][256];
    __shared__ uint32_t s_mask[EW * 256];
    __shared__ uint32_t s_w[ET / 32];
    const int band = blockIdx.x, f = blockIdx.y, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int w = G.w;
    const SixelFrameHdr *hdr = W.hdr + f;
    const uint8_t *idx = W.index + ((long long)f * G.h + (long long)band * 6) * w;

    for (int i = tid; i < EW * 256; i += ET) { (&s_cnt[0][0])[i] = 0; s_mask[i] = 0; }
    __syncthreads();

    // (1a) count entries per (warp, colour): shared-memory atomics, a few per column
    const int x_lo = wid * G.cols_per_warp, x_hi = min(w, x_lo + G.cols_per_warp);
    uint32_t *cnt = s_cnt[wid];
    for (int x = x_lo + lane; x < x_hi; x += 32) {
        uint32_t col[6], bits[6];
        const uint32_t valid = column_entries(idx, w, x, col, bits);
#pragma unroll
        for (int s = 0; s < 6; ++s) if (valid & (1u << s)) atomicAdd(&cnt[col[s]], 1u);
    }
    __syncthreads();
    // per-colour totals -> colour bases -> per (warp, colour) start offsets (in place)
    uint32_t tot_c = 0;
    if (tid < 256) for (int k = 0; k < EW; ++k) tot_c += s_cnt[k][tid];
    uint32_t n_ent; const uint32_t cb = block_excl_scan<ET>(tid < 256 ? tot_c : 0, s_w, n_ent);
    if (tid < 256) {
        uint32_t run = cb;
        for (int k = 0; k < EW; ++k) { const uint32_t v = s_cnt[k][tid]; s_cnt[k][tid] = run; run += v; }
    }
    __syncthreads();
    // (1b) scatter.  Ranks must follow x: per 32-column step the lanes holding each colour are
    // collected in a per-warp mask table (one atomicOr per entry); an entry's rank is the number of
    // lower lanes in its colour's mask, and the lowest lane advances the (warp, colour) cursor.
    uint32_t *M = s_mask + wid * 256;
    const uint32_t lt = (1u << lane) - 1;
    for (int x0 = x_lo; x0 < x_hi; x0 += 32) {
        const int x = x0 + lane;
        uint32_t col[6], bits[6];
        const uint32_t valid = x < x_hi ? column_entries(idx, w, x, col, bits) : 0u;
#pragma unroll
        for (int s = 0; s < 6; ++s) if (valid & (1u << s)) atomicOr(&M[col[s]], 1u << lane);
        __syncwarp();
        uint32_t mk[6];
#pragma unroll
        for (int s = 0; s < 6; ++s)
            if (valid & (1u << s)) {
                mk[s] = M[col[s]];
                s_sorted[cnt[col[s]] + __popc(mk[s] & lt)] = ent_pack(col[s], (uint32_t)x, bits[s]);
            }
        __syncwarp();
#pragma unroll
        for (int s = 0; s < 6; ++s)
            if ((valid & (1u << s)) && (mk[s] & lt) == 0) { cnt[col[s]] += (uint32_t)__popc(mk[s]); M[col[s]] = 0; }
        __syncwarp();
    }
    __syncthreads();
    // (2) sizes
    const int n = (int)n_ent;
    const uint32_t minc = s_sorted[0] >> 18;
    const int per = (n + ET - 1) / ET, lo = min(n, tid * per), hi = min(n, lo + per);
    uint32_t local = 0;
    walk_runs(s_sorted, lo, hi, n, [&](uint32_t c, uint32_t, uint32_t gap, uint32_t len, bool first) {
        local += rle_len(gap) + rle_len(len) + (first ? 1u + ndig4(c) + (c != minc ? 1u : 0u) : 0u);
    });
    uint32_t band_total; uint32_t at = block_excl_scan<ET>(local, s_w, band_total);
    if (tid == 0) W.band_bytes[(long long)f * W.nbands + band] = band_total;
    // (3) bytes, into this band's scratch slot (compacted into the final stream later)
    char *o = W.scratch + ((size_t)f * W.nbands + band) * W.band_cap + at;
    walk_runs(s_sorted, lo, hi, n, [&](uint32_t c, uint32_t bits, uint32_t gap, uint32_t len, bool first) {
        if (first) { if (c != minc) *o++ = '$'; *o++ = '#'; o = put_num4(o, c); }
        o = put_rle(o, gap, '?');
        o = put_rle(o, len, (char)('?' + bits));
    });
}

// ---- emit v1b: one walk instead of two -------------------------------------------------------------------------------
// Per-line instruction counts show v1 spending a large share of its instructions in the sizes walk and in the byte-wise,
// heavily divergent formatting of the write walk (every lane of a warp sits in another branch of put_rle / put_num4 and
// stores single bytes to global memory).  v1b walks the sorted entries ONCE: every run head builds its <= 3 pieces
// (colour introducer, gap, run) as 64-bit values with branch-light arithmetic and appends them to a thread-private slot
// in shared memory (word-interleaved over the threads, so the stores are conflict-free; the <= 3 words a piece touches
// are all stored, no branches); the slot's fill IS the thread's size, and after the block scan the slot is copied out with
// aligned 4-byte stores.  The slots take over the sort's count/mask tables.  A thread whose bytes do not fit its slot
// (noise frames) falls back to v1's write walk for its own range.
constexpr int SLOT_WORDS = 22;                   // words of a slot
constexpr int STASH_STEPS = 6;                   // 32-column steps of a warp whose column entries stay in registers (w <= 3072)
constexpr uint32_t SLOT_MAX = 4 * (SLOT_WORDS - 3);   // an append may START at byte <= SLOT_MAX (it touches <= 3 words)
static_assert(SLOT_WORDS * ET >= 2 * EW * 256, "the slots alias the sort's tables");

// decimal strings of 0..4095 (run lengths, gaps and colour numbers of a <= 4095 px wide band): the digits, most significant
// first, as a little-endian byte string, zero above them.  Built at compile time, read through the L1.
struct DecTable { uint32_t v[4096]; };
constexpr DecTable make_dec_table() {
    DecTable t{};
    for (uint32_t n = 0; n < 4096; ++n) {
        uint32_t s = 0, m = n, nd = 0;
        do { s = (s << 8) | (0x30u + m % 10u); m /= 10u; ++nd; } while (m);          // last digit ends up in the top byte of the nd used
        t.v[n] = s;
    }
    return t;
}
__device__ const DecTable k_dec = make_dec_table();
__device__ __forceinline__ uint32_t dec4(uint32_t v, uint32_t &nd) {     // v < 4096
    const uint32_t s = __ldg(&k_dec.v[v]);
    nd = 4u - ((uint32_t)__clz((int)s) >> 3);
    return s;
}
__device__ __forceinline__ unsigned long long rle_piece4(uint32_t n, uint32_t ch, uint32_t &len) {   // tosixel.c sixel_put_flash
    if (n > 3u) {
        uint32_t nd;
        const uint32_t d = dec4(n, nd);
        len = 2u + nd;
        return 0x21ull | ((unsigned long long)d << 8) | ((unsigned long long)ch << (8u * (1u + nd)));
    }
    len = n;
    return (unsigned long long)((ch * 0x010101u) & ((1u << (8u * n)) - 1u));
}
// append the first len (<= 8) bytes of v (zero above them) at byte `pos` of the slot; `cur` = the partial word at pos
__device__ __forceinline__ void slot_append(uint32_t *slot, uint32_t &pos, uint32_t &cur, unsigned long long v, uint32_t len) {
    const uint32_t sh = 8u * (pos & 3u);
    const uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
    const uint32_t w0 = cur | (lo << sh);
    const uint32_t w1 = __funnelshift_l(lo, hi, sh);
    const uint32_t w2 = sh ? (hi >> (32u - sh)) : 0u;
    uint32_t *p = slot + min(pos >> 2, (uint32_t)(SLOT_WORDS - 3)) * ET;   // clamped: an overflowing thread only needs its byte count
    p[0] = w0; p[ET] = w1; p[2 * ET] = w2;
    const uint32_t np = pos + len, adv = (np >> 2) - (pos >> 2);
    cur = adv == 0u ? w0 : (adv == 1u ? w1 : w2);            // v is zero above len: the word at np holds nothing beyond np
    pos = np;
}

// Phase clocks of the emit kernels (tools/bench_sixel_emit.py --clocks): built only with -DB200TIMG_EMIT_CLOCKS.  Thread 0
// stamps clock64() after a CTA barrier at every phase boundary (the instrumented build adds barriers where a phase has
// none) and adds the CTA's phase durations to g_emit_clocks[kernel][phase]; b200timg_emit_clocks() reads and clears them.
#ifdef B200TIMG_EMIT_CLOCKS
constexpr int EMIT_CLK_PHASES = 8;
__device__ unsigned long long g_emit_clocks[2][EMIT_CLK_PHASES];     // [0: emit1b, 1: emit5][phase], SM cycles summed over CTAs
#define EMIT_CLK_BEGIN long long clk_[EMIT_CLK_PHASES + 1]; int clk_n_ = 0; if (threadIdx.x == 0) clk_[clk_n_] = clock64(); ++clk_n_
#define EMIT_CLK() do { __syncthreads(); if (threadIdx.x == 0) clk_[clk_n_] = clock64(); ++clk_n_; } while (0)
#define EMIT_CLK_END(kern) do { if (threadIdx.x == 0) for (int k_ = 0; k_ + 1 < clk_n_; ++k_) \
        atomicAdd(&g_emit_clocks[kern][k_], (unsigned long long)(clk_[k_ + 1] - clk_[k_])); } while (0)
#else
#define EMIT_CLK_BEGIN do {} while (0)
#define EMIT_CLK() do {} while (0)
#define EMIT_CLK_END(kern) do {} while (0)
#endif

// emit5 (V5) is v1b with two changes, both chosen from v1b's phase clocks (DESIGN.md §5):
//   * the band's six index rows (one contiguous block of 6*w bytes) come in with coalesced word loads, all in flight at
//     once and issued before the table zeroing, into the entry array (dead until the scatter); the count pass reads its
//     columns from there.  v1b's count pass waited for one global round trip per 32-column step.  (w <= 3072 only: wider
//     bands re-read their columns in the scatter pass, so they keep v1b's loads.)
//   * the copy-out: when no slot overflowed, every thread moves its slot's bytes to their place in one contiguous byte
//     image of the band in shared memory (the entry array again), and the CTA writes that image to the 256-byte aligned
//     scratch slot with 16-byte stores.  v1b's threads each stored their ~32 bytes as 4-byte words, a warp store touching
//     32 sectors.
constexpr int ROW_WORDS = (6 * 32 * STASH_STEPS * EW + 3) / 4 / ET + 1;   // words of the staged rows per thread (+1: misalignment)

// Band accessors (emit, compaction): the CTA's frame and 6-row band, where the band's index rows, size, offset and
// scratch slot live.
template <class Dims>                     // EmitGeom (emit) or NoMixed (compaction): the kernels' parameters as before
struct BandUniform {                      // band blockIdx.x of frame blockIdx.y
    typedef Dims Params;
    const Dims &G; int band, f;
    __device__ __forceinline__ explicit BandUniform(const Dims &g) : G(g), band(blockIdx.x), f(blockIdx.y) {}
    __device__ __forceinline__ int w() const { return G.w; }
    __device__ __forceinline__ int cols_per_warp() const { return G.cols_per_warp; }
    __device__ __forceinline__ int width(int w_) const { return w_; }      // compaction: its own w / h parameters
    __device__ __forceinline__ int height(int h_) const { return h_; }
    __device__ __forceinline__ int nbands(const SixelWork &W) const { return W.nbands; }
    __device__ __forceinline__ long long idx0(int w_) const { return ((long long)f * G.h + (long long)band * 6) * w_; }
    __device__ __forceinline__ long long slot(const SixelWork &W) const { return (long long)f * W.nbands + band; }
    __device__ __forceinline__ size_t scr(const SixelWork &W) const { return ((size_t)f * W.nbands + band) * W.band_cap; }
};
typedef BandUniform<EmitGeom> EmitBands;
typedef BandUniform<NoMixed> CompactBands;
struct BandMixed {                        // flat band blockIdx.x
    typedef MixedSixelParams Params;
    MixedSixelFrame D; int band, f;
    __device__ __forceinline__ explicit BandMixed(const MixedSixelParams &P) {
        f = sixel_owner(P.band_start, P.n_frames, blockIdx.x);
        band = (int)(blockIdx.x - P.band_start[f]);
        D = P.desc[f];
    }
    __device__ __forceinline__ int w() const { return D.w; }
    __device__ __forceinline__ int cols_per_warp() const { return D.cols_per_warp; }
    __device__ __forceinline__ int width(int) const { return D.w; }
    __device__ __forceinline__ int height(int) const { return D.h; }
    __device__ __forceinline__ int nbands(const SixelWork &) const { return D.nbands; }
    __device__ __forceinline__ long long idx0(int w_) const { return (long long)D.idx + (long long)band * 6 * w_; }
    __device__ __forceinline__ long long slot(const SixelWork &) const { return (long long)D.band0 + band; }
    __device__ __forceinline__ size_t scr(const SixelWork &) const { return (size_t)D.scr + (size_t)band * D.band_cap; }
};

template <bool V5, class A>
__global__ void __launch_bounds__(ET, 2)
sixel_emit1b_kernel(typename A::Params G, SixelWork W) {
    extern __shared__ uint32_t s_sorted[];                   // [6*w]
    __shared__ uint32_t s_tab[SLOT_WORDS * ET];              // sort: cnt[EW][256] | mask[EW][256]; afterwards: slots
    __shared__ uint32_t s_w[ET / 32];
    const A a(G);
    const int band = a.band, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int w = a.w();
    const uint8_t *idx = W.index + a.idx0(w);
    EMIT_CLK_BEGIN;
    const bool stash = a.cols_per_warp() <= 32 * STASH_STEPS;
    const uint8_t *cols = idx;                               // where the count pass reads the band's rows
    if (V5 && stash) {
        // aligned words covering [idx, idx + 6w).  The <= 3 bytes outside the band stay inside the index region: sixel_plan
        // starts it on a 256-byte boundary and pads its end to one (o_idx, align_up(npix * n_frames, 256)), so rounding
        // the first band's start down or the last band's end up to a word never leaves it.
        const uint32_t a = (uint32_t)(reinterpret_cast<uintptr_t>(idx) & 3u);
        const uint32_t *gw = reinterpret_cast<const uint32_t *>(idx - a);
        const int nw = (int)((a + 6u * (uint32_t)w + 3u) >> 2);
        uint32_t rw[ROW_WORDS];
#pragma unroll
        for (int k = 0; k < ROW_WORDS; ++k) { const int j = tid + k * ET; rw[k] = j < nw ? gw[j] : 0u; }
        for (int i = tid; i < 2 * EW * 256; i += ET) s_tab[i] = 0;
#pragma unroll
        for (int k = 0; k < ROW_WORDS; ++k) { const int j = tid + k * ET; if (j < nw) s_sorted[j] = rw[k]; }
        cols = reinterpret_cast<const uint8_t *>(s_sorted) + a;
    } else {
        for (int i = tid; i < 2 * EW * 256; i += ET) s_tab[i] = 0;
    }
    __syncthreads();
    if (!V5) EMIT_CLK();                                     // zero
    // (1) the sort: as in v1, but the column entries (<= 6 distinct colours of a column with their row bits) are computed
    // once: the count pass parks them in registers (3 words per 32-column step, steps unrolled) for the scatter pass
    const int x_lo = wid * a.cols_per_warp(), x_hi = min(w, x_lo + a.cols_per_warp());
    uint32_t *cnt = s_tab + wid * 256, *M = s_tab + EW * 256 + wid * 256;
    uint32_t k0[STASH_STEPS], k1[STASH_STEPS], k2[STASH_STEPS];     // colours 0-3 | colours 4-5, valid, bits 5 | bits 0-4
    if (stash) {
#pragma unroll
        for (int t = 0; t < STASH_STEPS; ++t) {
            const int x = x_lo + 32 * t + lane;
            k0[t] = k1[t] = k2[t] = 0;
            if (x < x_hi) {
                uint32_t col[6], bits[6];
                const uint32_t valid = column_entries(cols, w, x, col, bits);
#pragma unroll
                for (int s = 0; s < 6; ++s) if (valid & (1u << s)) atomicAdd(&cnt[col[s]], 1u);
                k0[t] = col[0] | (col[1] << 8) | (col[2] << 16) | (col[3] << 24);
                k1[t] = col[4] | (col[5] << 8) | (valid << 16) | (bits[5] << 22);
                k2[t] = bits[0] | (bits[1] << 6) | (bits[2] << 12) | (bits[3] << 18) | (bits[4] << 24);
            }
        }
    } else {
        for (int x = x_lo + lane; x < x_hi; x += 32) {
            uint32_t col[6], bits[6];
            const uint32_t valid = column_entries(idx, w, x, col, bits);
#pragma unroll
            for (int s = 0; s < 6; ++s) if (valid & (1u << s)) atomicAdd(&cnt[col[s]], 1u);
        }
    }
    __syncthreads();
    EMIT_CLK();                                              // count
    uint32_t tot_c = 0;
    if (tid < 256) for (int k = 0; k < EW; ++k) tot_c += s_tab[k * 256 + tid];
    uint32_t n_ent; const uint32_t cb = block_excl_scan<ET>(tid < 256 ? tot_c : 0, s_w, n_ent);
    if (tid < 256) {
        uint32_t run = cb;
        for (int k = 0; k < EW; ++k) { const uint32_t v = s_tab[k * 256 + tid]; s_tab[k * 256 + tid] = run; run += v; }
    }
    __syncthreads();
    EMIT_CLK();                                              // offsets
    const uint32_t lt = (1u << lane) - 1;
    auto scatter_step = [&](int x, uint32_t valid, const uint32_t *col, const uint32_t *bits) {
#pragma unroll
        for (int s = 0; s < 6; ++s) if (valid & (1u << s)) atomicOr(&M[col[s]], 1u << lane);
        __syncwarp();
        uint32_t mk[6];
#pragma unroll
        for (int s = 0; s < 6; ++s)
            if (valid & (1u << s)) {
                mk[s] = M[col[s]];
                s_sorted[cnt[col[s]] + __popc(mk[s] & lt)] = ent_pack(col[s], (uint32_t)x, bits[s]);
            }
        __syncwarp();
#pragma unroll
        for (int s = 0; s < 6; ++s)
            if ((valid & (1u << s)) && (mk[s] & lt) == 0) { cnt[col[s]] += (uint32_t)__popc(mk[s]); M[col[s]] = 0; }
        __syncwarp();
    };
    if (stash) {
#pragma unroll
        for (int t = 0; t < STASH_STEPS; ++t) {
            if (x_lo + 32 * t < x_hi) {                      // warp-uniform
                const uint32_t col[6] = {k0[t] & 255u, (k0[t] >> 8) & 255u, (k0[t] >> 16) & 255u, k0[t] >> 24, k1[t] & 255u, (k1[t] >> 8) & 255u};
                const uint32_t bits[6] = {k2[t] & 63u, (k2[t] >> 6) & 63u, (k2[t] >> 12) & 63u, (k2[t] >> 18) & 63u, (k2[t] >> 24) & 63u, (k1[t] >> 22) & 63u};
                scatter_step(x_lo + 32 * t + lane, (k1[t] >> 16) & 63u, col, bits);
            }
        }
    } else {
        for (int x0 = x_lo; x0 < x_hi; x0 += 32) {
            const int x = x0 + lane;
            uint32_t col[6], bits[6];
            const uint32_t valid = x < x_hi ? column_entries(idx, w, x, col, bits) : 0u;
            scatter_step(x, valid, col, bits);
        }
    }
    __syncthreads();                                         // the tables are dead: s_tab is the slot array from here on
    EMIT_CLK();                                              // scatter
    // (2) one walk: bytes into the slot, size = the slot's fill
    const int n = (int)n_ent;
    const uint32_t minc = s_sorted[0] >> 18;
    const int per = (n + ET - 1) / ET, lo = min(n, tid * per), hi = min(n, lo + per);
    uint32_t *slot = s_tab + tid;
    uint32_t pos = 0, cur = 0;
    bool ovf = false;
    walk_runs(s_sorted, lo, hi, n, [&](uint32_t c, uint32_t bits, uint32_t gap, uint32_t len, bool first) {
        uint32_t pl;
        if (first) {
            uint32_t nd;
            unsigned long long v = 0x23ull | ((unsigned long long)dec4(c, nd) << 8);
            pl = 1u + nd;
            if (c != minc) { v = 0x24ull | (v << 8); ++pl; }
            ovf |= pos > SLOT_MAX;
            slot_append(slot, pos, cur, v, pl);
        }
        uint32_t rl;
        const unsigned long long gv = rle_piece4(gap, 0x3fu, pl), rv = rle_piece4(len, 0x3fu + bits, rl);
        ovf |= pos > SLOT_MAX;
        if (pl + rl <= 8u) {                                 // nearly always: blank columns + run in one append
            slot_append(slot, pos, cur, gv | (rv << (8u * pl)), pl + rl);
        } else {
            slot_append(slot, pos, cur, gv, pl);
            ovf |= pos > SLOT_MAX;
            slot_append(slot, pos, cur, rv, rl);
        }
    });
    const uint32_t local = pos;
    EMIT_CLK();                                              // walk
    uint32_t band_total; const uint32_t at = block_excl_scan<ET>(local, s_w, band_total);
    if (tid == 0) W.band_bytes[a.slot(W)] = band_total;
    EMIT_CLK();                                              // scan
    // (3) the slot's bytes to `at` of this band's 16-byte aligned scratch place (v1b), or of its image in shared memory
    // (emit5): head bytes up to a word boundary, whole words realigned with a funnel shift, tail bytes
    char *const band_out = W.scratch + a.scr(W);
    char *o = band_out + at;
    auto slot_out = [&](char *d) {
        const uint32_t head = min(local, (4u - (at & 3u)) & 3u);
        const uint32_t w0 = slot[0];
        for (uint32_t k = 0; k < head; ++k) d[k] = (char)(w0 >> (8u * k));
        const uint32_t nw = (local - head) >> 2;
        uint32_t *dw = reinterpret_cast<uint32_t *>(d + head);
        uint32_t a = w0;
        for (uint32_t j = 0; j < nw; ++j) {
            const uint32_t b = slot[(j + 1) * ET];
            dw[j] = __funnelshift_r(a, b, 8u * head);
            a = b;
        }
        const uint32_t done = head + 4u * nw;
        for (uint32_t k = done; k < local; ++k) d[k] = (char)(slot[(k >> 2) * ET] >> (8u * (k & 3u)));
    };
    // emit5: the entry array is dead (every walk ended before the scan's barriers) and holds the band's image when no
    // slot overflowed (<= 84 bytes a thread) and the image fits its 24*w bytes (narrow bands)
    if (V5 && !__syncthreads_or(ovf) && band_total <= 24u * (uint32_t)w) {
        char *img = reinterpret_cast<char *>(s_sorted);
        slot_out(img + at);
        __syncthreads();
        const uint32_t n16 = band_total >> 4;
        const uint4 *s16 = reinterpret_cast<const uint4 *>(img);
        uint4 *d16 = reinterpret_cast<uint4 *>(band_out);
        for (uint32_t j = tid; j < n16; j += ET) d16[j] = s16[j];
        const uint32_t t = (n16 << 4) + (uint32_t)tid;
        if (t < band_total) band_out[t] = img[t];
    } else if (!ovf) {
        slot_out(o);
    } else {                                                 // v1's write walk for this thread's range
        walk_runs(s_sorted, lo, hi, n, [&](uint32_t c, uint32_t bits, uint32_t gap, uint32_t len, bool first) {
            if (first) { if (c != minc) *o++ = '$'; *o++ = '#'; o = put_num4(o, c); }
            o = put_rle(o, gap, '?');
            o = put_rle(o, len, (char)('?' + bits));
        });
    }
    EMIT_CLK();                                              // copy-out
    EMIT_CLK_END(V5 ? 1 : 0);
}

// per frame: header length, band offsets (exclusive, in place), frame size
struct LayoutUniform {                    // frame blockIdx.x
    typedef NoMixed Params;
    const SixelWork &W; int f;
    __device__ __forceinline__ LayoutUniform(const SixelWork &W_, const NoMixed &, int f_) : W(W_), f(f_) {}
    __device__ __forceinline__ int w(int w_) const { return w_; }
    __device__ __forceinline__ int h(int h_) const { return h_; }
    __device__ __forceinline__ int nbands() const { return W.nbands; }
    __device__ __forceinline__ long long band0() const { return (long long)f * W.nbands; }
};
struct LayoutMixed {
    typedef MixedSixelParams Params;
    MixedSixelFrame D;
    __device__ __forceinline__ LayoutMixed(const SixelWork &, const MixedSixelParams &P, int f) : D(P.desc[f]) {}
    __device__ __forceinline__ int w(int) const { return D.w; }
    __device__ __forceinline__ int h(int) const { return D.h; }
    __device__ __forceinline__ int nbands() const { return D.nbands; }
    __device__ __forceinline__ long long band0() const { return (long long)D.band0; }
};

template <class G>
__global__ void __launch_bounds__(256)
sixel_layout_kernel(int w, int h, SixelWork W, typename G::Params M) {
    __shared__ uint32_t s_w[8];
    __shared__ uint32_t s_carry;
    const int f = blockIdx.x, tid = threadIdx.x;
    const G lay(W, M, f);
    SixelFrameHdr *hdr = W.hdr + f;
    uint32_t len = 0;
    if ((uint32_t)tid < hdr->ncolors) {
        const uint32_t p = hdr->palette[tid];
        const uint32_t r = ((p & 0xff) * 100 + 127) / 255, g = (((p >> 8) & 0xff) * 100 + 127) / 255, b = (((p >> 16) & 0xff) * 100 + 127) / 255;
        len = 1 + ndig_u((uint32_t)tid) + 3 + ndig_u(r) + 1 + ndig_u(g) + 1 + ndig_u(b);
    }
    uint32_t pal_total; (void)block_excl_scan<256>(len, s_w, pal_total);
    const uint32_t header = 8 + ndig_u((uint32_t)lay.w(w)) + 1 + ndig_u((uint32_t)lay.h(h)) + pal_total;
    if (tid == 0) s_carry = header;
    __syncthreads();
    uint32_t *bb = W.band_bytes + lay.band0();
    for (int b0 = 0; b0 < lay.nbands(); b0 += 256) {
        const int b = b0 + tid;
        const uint32_t v = b < lay.nbands() ? bb[b] + (b > 0 ? 1u : 0u) : 0;       // '-' before every band but the first
        uint32_t tot; const uint32_t at = block_excl_scan<256>(v, s_w, tot);
        if (b < lay.nbands()) W.band_off[lay.band0() + b] = s_carry + at + (b > 0 ? 1u : 0u);   // band's first data byte
        __syncthreads();
        if (tid == 0) s_carry += tot;
        __syncthreads();
    }
    if (tid == 0) { hdr->header_len = header; hdr->frame_size = s_carry + 2; }   // + ESC backslash
}

__global__ void __launch_bounds__(1024)
sixel_sizes_to_offsets_kernel(const SixelFrameHdr *__restrict__ hdr, int n, uint64_t *__restrict__ offsets) {
    __shared__ unsigned long long s_wv[32];
    __shared__ unsigned long long c_run;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) c_run = 0;
    __syncthreads();
    for (int i0 = 0; i0 < n; i0 += 1024) {
        const int i = i0 + tid;
        unsigned long long v = i < n ? hdr[i].frame_size : 0ull;
        const unsigned long long mine = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const unsigned long long o = __shfl_up_sync(0xffffffffu, v, d); if (lane >= d) v += o; }
        if (lane == 31) s_wv[wid] = v;
        __syncthreads();
        unsigned long long pre = 0, tot = 0;
        for (int k = 0; k < 32; ++k) { if (k < wid) pre += s_wv[k]; tot += s_wv[k]; }
        if (i < n) offsets[i] = c_run + pre + v - mine;
        __syncthreads();
        if (tid == 0) c_run += tot;
        __syncthreads();
    }
    if (tid == 0) offsets[n] = c_run;
}

// Final assembly: header + palette (band 0's CTA), every band's bytes copied from its scratch slot
// to its place in the compacted stream, '-' between bands, ST at the end.  Pure byte traffic.
template <class A>
__global__ void __launch_bounds__(256)
sixel_compact_kernel(int w, int h, SixelWork W, const uint64_t *__restrict__ offsets, char *__restrict__ out,
                     unsigned long long out_cap, typename A::Params M) {
    __shared__ uint32_t s_w[8];
    const A a(M);
    const int band = a.band, f = a.f, tid = threadIdx.x;
    const SixelFrameHdr *hdr = W.hdr + f;
    const unsigned long long fbase = offsets[f];
    if (fbase + hdr->frame_size > out_cap) return;           // never write out of bounds
    const uint32_t boff = W.band_off[a.slot(W)];
    const uint32_t n = W.band_bytes[a.slot(W)];
    const char *src = W.scratch + a.scr(W);
    char *dst = out + fbase + boff;
    {   // word copy: 4-byte aligned stores, source words realigned with a funnel shift
        const uint32_t head = min(n, (uint32_t)((4 - (reinterpret_cast<uintptr_t>(dst) & 3)) & 3));
        if ((uint32_t)tid < head) dst[tid] = src[tid];
        const uint32_t nw = (n - head) >> 2, m = head & 3;                 // src slot is 16-byte aligned
        const uint32_t *sw = reinterpret_cast<const uint32_t *>(src + head - m);
        uint32_t *dw = reinterpret_cast<uint32_t *>(dst + head);
        for (uint32_t j = tid; j < nw; j += 256) dw[j] = m ? __funnelshift_r(sw[j], sw[j + 1], 8 * m) : sw[j];
        const uint32_t done = head + (nw << 2);
        if (done + tid < n) dst[done + tid] = src[done + tid];           // < 4 tail bytes
    }
    if (tid == 0) {
        if (band > 0) dst[-1] = '-';                         // DECGNL between bands
        if (band == a.nbands(W) - 1) { out[fbase + hdr->frame_size - 2] = '\033'; out[fbase + hdr->frame_size - 1] = '\\'; }
    }
    if (band == 0) {                                         // DCS q, raster attributes, palette definitions
        if (tid == 0) {
            char *o = out + fbase;
            *o++ = '\033'; *o++ = 'P'; *o++ = 'q'; *o++ = '"'; *o++ = '1'; *o++ = ';'; *o++ = '1'; *o++ = ';';
            o = put_num_u(o, (uint32_t)a.width(w)); *o++ = ';'; o = put_num_u(o, (uint32_t)a.height(h));
        }
        const uint32_t fixed = 8 + ndig_u((uint32_t)a.width(w)) + 1 + ndig_u((uint32_t)a.height(h));
        uint32_t len = 0, r = 0, g = 0, b = 0;
        if ((uint32_t)tid < hdr->ncolors) {                  // output_rgb_palette_definition: (v*100+127)/255 percent
            const uint32_t p = hdr->palette[tid];
            r = ((p & 0xff) * 100 + 127) / 255; g = (((p >> 8) & 0xff) * 100 + 127) / 255; b = (((p >> 16) & 0xff) * 100 + 127) / 255;
            len = 1 + ndig_u((uint32_t)tid) + 3 + ndig_u(r) + 1 + ndig_u(g) + 1 + ndig_u(b);
        }
        uint32_t tot; const uint32_t at = block_excl_scan<256>(len, s_w, tot);
        if (len) {
            char *q = out + fbase + fixed + at;
            *q++ = '#'; q = put_num_u(q, (uint32_t)tid); *q++ = ';'; *q++ = '2'; *q++ = ';';
            q = put_num_u(q, r); *q++ = ';'; q = put_num_u(q, g); *q++ = ';'; q = put_num_u(q, b);
        }
    }
}

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ---- host side ------------------------------------------------------------------------------------
// The chain of a batch is  front (per frame: palette, table, dither, band sizes)  ->  back (sizes -> offsets ->
// bytes in their final place).  The front part can be run for SLICES of the batch on different streams
// (launch_sixel_front with f0 / n): a batch pipeline overlaps the latency-bound per-frame kernels of one
// slice with the scaler of the next.
struct SixelPlan {
    SixelWork W;
    bool emit_v1, dither_v1;
    int emit_mode;                            // 1: v1, 4: v1b, 5: emit5 (scratch arena + compaction), 2: emit2, 3: emit3
    EmitGeom G;
    SixelPaletteShape pal;
    size_t emit_smem, o_d2_bnd, o_d2_prog;
    long long npix;
};

int sixel_check_geometry(int w, int h, int n_frames, char *msg, size_t msg_cap) {
    msg[0] = 0;
    if (w <= 0 || h <= 0 || n_frames <= 0) snprintf(msg, msg_cap, "sixel: bad geometry %d x %d, %d frames", w, h, n_frames);
    else if (h % 6) snprintf(msg, msg_cap, "sixel: height %d is not a multiple of 6", h);
    else if (n_frames > 65535) snprintf(msg, msg_cap, "sixel: %d frames, at most 65535 in one launch", n_frames);
    else if (w > 99999) snprintf(msg, msg_cap, "sixel: width %d, at most 99999 px", w);
    else if ((h + 31) / 32 > 2048) snprintf(msg, msg_cap, "sixel: height %d, at most 65536 rows", h);
    else if ((unsigned long long)n_frames * (h / 6) * ((w + 4095) / 4096) > 0x7fffffffull)
        snprintf(msg, msg_cap, "sixel: more than 2^31 - 1 bands x column tiles in one launch");
    return msg[0] ? B200TIMG_EINVAL : B200TIMG_OK;
}

SixelPaletteShape sixel_palette_shape(long long npix) {
    SixelPaletteShape P;
    // quant.c computeHistogram, QUALITY_LOW (the palette kernel computes the same step)
    P.step_px = npix / 18383; if (npix < 18383) P.step_px = 6; if (P.step_px == 0) P.step_px = 1;
    const long long ns = (npix + P.step_px - 1) / P.step_px;
    P.ent_cap = (int)std::min<long long>(32768, ns);
    const size_t t_words = P.ent_cap > 16384 ? (size_t)P.ent_cap : 16384;      // the histogram aliases the second table
    P.tables_smem = sizeof(uint32_t) * (t_words + (size_t)P.ent_cap);
    P.smem_tables = P.tables_smem <= 200 * 1024;
    return P;
}

// The emitters (B200TIMG_EMIT=1..5): v1, v1b (4) and emit5 (5, the default up to 4095 px) write per-band bytes into a
// scratch arena for the compaction kernel; emit2 (sixel_emit.cu: single pass, any width -- what wider frames get) and
// emit3 (v1's sort + entry-parallel formatting + look-back placement; slower than v1 on C2 frames) place their own.
// Every mode but the default is kept for A/B runs.
int sixel_emit_mode(int w) {
    const bool v1_fits = w <= 4095 && sizeof(uint32_t) * (size_t)6 * w <= (size_t)(227 - 36) * 1024;
    const bool v1b_fits = w <= 4095 && sizeof(uint32_t) * (size_t)6 * w <= (size_t)(227 - 47) * 1024;
    int mode = v1b_fits ? 5 : v1_fits ? 1 : 2;           // 5 = emit5 (v1b with staged rows and a coalesced copy-out)
    if (getenv("B200TIMG_EMIT_V2")) mode = 2;
    if (const char *e = getenv("B200TIMG_EMIT")) mode = atoi(e);
    if (mode < 1 || mode > 5 || (mode == 1 && !v1_fits) || (mode >= 4 && !v1b_fits)) mode = 2;
    return mode;
}

static int sixel_plan(b200timg_ctx *ctx, int w, int h, int n_frames, bool reserve, SixelPlan *S) {
    char why[96];
    if (sixel_check_geometry(w, h, n_frames, why, sizeof why) != B200TIMG_OK) return ctx->fail(B200TIMG_EINVAL, "%s", why);
    SixelWork &W = S->W;
    const long long npix = (long long)w * h;
    S->npix = npix;
    S->pal = sixel_palette_shape(npix);
    W.ent_cap = S->pal.ent_cap;
    W.nb32 = (h + 31) / 32; W.nbands = h / 6;
    // workspace carve-up
    size_t off = 0;
    const size_t o_hdr = off; off += align_up(sizeof(SixelFrameHdr) * n_frames, 256);
    const size_t o_ea = off; off += align_up(sizeof(uint32_t) * (size_t)W.ent_cap * n_frames, 256);
    const size_t o_eb = off; off += align_up(sizeof(uint32_t) * (size_t)W.ent_cap * n_frames, 256);
    const size_t o_lut = off; off += align_up((size_t)32768 * n_frames, 256);
    const size_t o_idx = off; off += align_up((size_t)npix * n_frames, 256);
    const size_t o_bnd = off; off += align_up(sizeof(uint32_t) * (size_t)W.nb32 * w * n_frames, 256);
    const size_t o_bb = off; off += align_up(sizeof(uint32_t) * (size_t)W.nbands * n_frames, 256);
    const size_t o_bo = off; off += align_up(sizeof(uint32_t) * (size_t)W.nbands * n_frames, 256);
    // worst case of one band: <= 6 entries per column, <= 7 bytes each ("!nnnn?" + char), "$#ccc" per colour
    W.band_cap = align_up((size_t)w * 42 + 256 * 5 + 16, 256);
    const size_t o_scr = off;
    S->emit_mode = sixel_emit_mode(w);
    S->emit_v1 = S->emit_mode == 1 || S->emit_mode >= 4;
    if (S->emit_v1) off += W.band_cap * W.nbands * n_frames;
    S->dither_v1 = getenv("B200TIMG_DITHER_V1") != nullptr;      // round-1 ditherer, kept for A/B runs
    size_t d_bnd, d_prog;
    const size_t o_d2 = off; off += sixel_dither_workspace(w, h, n_frames, &d_bnd, &d_prog);
    size_t e_hdr, e_desc, e_ctl;
    const size_t o_e2 = off; off += sixel_emit_workspace(w, h, n_frames, &e_hdr, &e_desc, &e_ctl);
    if (reserve) B2_CUDA(ctx, ctx->sixel_work.reserve(off));
    if (!ctx->sixel_work.p || ctx->sixel_work.cap < off) return ctx->fail(B200TIMG_EINVAL, "sixel: write phase without prepare");
    ctx->sixel_idx_off = o_idx;
    char *base = ctx->sixel_work.as<char>();
    W.hdr = reinterpret_cast<SixelFrameHdr *>(base + o_hdr);
    W.ent_a = reinterpret_cast<uint32_t *>(base + o_ea); W.ent_b = reinterpret_cast<uint32_t *>(base + o_eb);
    W.lut = reinterpret_cast<uint8_t *>(base + o_lut); W.index = reinterpret_cast<uint8_t *>(base + o_idx);
    W.boundary = reinterpret_cast<uint32_t *>(base + o_bnd); W.band_bytes = reinterpret_cast<uint32_t *>(base + o_bb);
    W.band_off = reinterpret_cast<uint32_t *>(base + o_bo); W.scratch = base + o_scr;
    W.hdr_bytes = base + o_e2 + e_hdr;
    W.desc = reinterpret_cast<unsigned long long *>(base + o_e2 + e_desc);
    W.ctl = reinterpret_cast<uint32_t *>(base + o_e2 + e_ctl);
    S->o_d2_bnd = o_d2 + d_bnd; S->o_d2_prog = o_d2 + d_prog;
    S->G.w = w; S->G.h = h; S->G.cols_per_warp = ((w + EW - 1) / EW + 31) / 32 * 32;
    const size_t smem_limit = 227 * 1024 - 36 * 1024;   // the emit kernel also has ~33 KB of static shared memory
    S->emit_smem = sizeof(uint32_t) * (size_t)6 * w;
    if (!ctx->sixel_attrs_set) {                         // function attributes are per device, i.e. per context
        B2_CUDA(ctx, cudaFuncSetAttribute(sixel_palette_kernel<false, PaletteUniform>, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536));
        B2_CUDA(ctx, cudaFuncSetAttribute(sixel_emit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_limit));
        B2_CUDA(ctx, cudaFuncSetAttribute(sixel_emit1b_kernel<false, EmitBands>, cudaFuncAttributeMaxDynamicSharedMemorySize, (227 - 47) * 1024));
        B2_CUDA(ctx, cudaFuncSetAttribute(sixel_emit1b_kernel<true, EmitBands>, cudaFuncAttributeMaxDynamicSharedMemorySize, (227 - 47) * 1024));
        B2_CUDA(ctx, cudaFuncSetAttribute(sixel_dither_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 32768 + DW_MAX * DWARP_SMEM));
        // unconditionally: which variant a frame takes depends on ITS size, not on the first frame this context saw
        B2_CUDA(ctx, cudaFuncSetAttribute(sixel_palette_kernel<true, PaletteUniform>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        ctx->sixel_attrs_set = true;
    }
    return B200TIMG_OK;
}

// frames [f0, f0 + n) of a batch of n_total: palette -> table -> (map | dither) -> band sizes (v1 emitter), on ctx->stream
int launch_sixel_front(b200timg_ctx *ctx, const uint8_t *d_fb, int w, int h, int n_total, int f0, int n, bool reserve) {
    if ((reinterpret_cast<uintptr_t>(d_fb) & 3)) return ctx->fail(B200TIMG_EINVAL, "sixel: framebuffer must be 4-byte aligned");
    SixelPlan S;
    B2_TRY(sixel_plan(ctx, w, h, n_total, reserve, &S));
    SixelWork W = S.W;                                    // the slice's view of the per-frame arrays
    const long long npix = S.npix;
    W.hdr += f0; W.ent_a += (long long)f0 * W.ent_cap; W.ent_b += (long long)f0 * W.ent_cap; W.lut += (long long)f0 * 32768;
    W.index += (long long)f0 * npix; W.boundary += (long long)f0 * W.nb32 * w;
    W.band_bytes += (long long)f0 * W.nbands; W.band_off += (long long)f0 * W.nbands;
    W.scratch += (size_t)f0 * W.nbands * W.band_cap;
    const uint32_t *fb = reinterpret_cast<const uint32_t *>(d_fb) + (long long)f0 * npix;
    char *base = ctx->sixel_work.as<char>();
    B2_KERNEL(ctx, "sixel_palette_kernel");
    if (S.pal.smem_tables) sixel_palette_kernel<true, PaletteUniform><<<n, PT, S.pal.tables_smem, ctx->stream>>>(fb, w, h, W, NoMixed());
    else sixel_palette_kernel<false, PaletteUniform><<<n, PT, 65536, ctx->stream>>>(fb, w, h, W, NoMixed());
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "sixel_lut_kernel");
    sixel_lut_kernel<<<dim3(128, n), 256, 0, ctx->stream>>>(W);
    B2_LAUNCH_CHECK(ctx);
    {
        long long blocks = (npix + 255) / 256; if (blocks > 64) blocks = 64;
        B2_KERNEL(ctx, "sixel_map_kernel");
        sixel_map_kernel<MapUniform><<<dim3((unsigned)blocks, n), 256, 0, ctx->stream>>>(fb, npix, W, NoMixed());
        B2_LAUNCH_CHECK(ctx);
    }
    if (!S.dither_v1) {
        B2_TRY(launch_sixel_dither(ctx, fb, w, h, n, n_total, W, base + S.o_d2_bnd + sizeof(uint4) * (size_t)f0 * W.nb32 * w,
                                   base + S.o_d2_prog + sizeof(int) * (size_t)f0 * W.nb32));
    } else {
        B2_KERNEL(ctx, "sixel_dither_kernel");
        // warps per frame: as many as fit, but in full rounds over the 32-row bands
        const int rounds = (W.nb32 + DW_MAX - 1) / DW_MAX;
        const int nwarps = (W.nb32 + rounds - 1) / rounds;
        const size_t dsmem = 32768 + (size_t)nwarps * DWARP_SMEM;
        sixel_dither_kernel<<<n, nwarps * 32, dsmem, ctx->stream>>>(fb, w, h, nwarps, W);
        B2_LAUNCH_CHECK(ctx);
    }
    if (S.emit_v1) {
        B2_KERNEL(ctx, S.emit_mode == 5 ? "sixel_emit5_kernel" : "sixel_emit_kernel");
        if (S.emit_mode == 5) sixel_emit1b_kernel<true, EmitBands><<<dim3(W.nbands, n), ET, S.emit_smem, ctx->stream>>>(S.G, W);
        else if (S.emit_mode == 4) sixel_emit1b_kernel<false, EmitBands><<<dim3(W.nbands, n), ET, S.emit_smem, ctx->stream>>>(S.G, W);
        else sixel_emit_kernel<<<dim3(W.nbands, n), ET, S.emit_smem, ctx->stream>>>(S.G, W);
        B2_LAUNCH_CHECK(ctx);
    }
    return B200TIMG_OK;
}

// the whole batch: sizes -> offsets (phase 1), bytes into d_out (phase 2)
int launch_sixel_back(b200timg_ctx *ctx, int w, int h, int n_frames, char *d_out, size_t out_cap, uint64_t *d_offsets, int phases) {
    SixelPlan S;
    B2_TRY(sixel_plan(ctx, w, h, n_frames, false, &S));
    const SixelWork &W = S.W;
    if (!S.emit_v1) {
        if (!(phases & 2)) return B200TIMG_OK;
        if (S.emit_mode == 2) return launch_sixel_emit(ctx, w, h, n_frames, W, d_out, out_cap, d_offsets);
        return launch_sixel_emit3(ctx, w, h, n_frames, W, d_out, out_cap, d_offsets);
    }
    if (phases & 1) {
        B2_KERNEL(ctx, "sixel_layout_kernel");
        sixel_layout_kernel<LayoutUniform><<<n_frames, 256, 0, ctx->stream>>>(w, h, W, NoMixed());
        B2_LAUNCH_CHECK(ctx);
        B2_KERNEL(ctx, "sixel_sizes_to_offsets_kernel");
        sixel_sizes_to_offsets_kernel<<<1, 1024, 0, ctx->stream>>>(W.hdr, n_frames, d_offsets);
        B2_LAUNCH_CHECK(ctx);
    }
    if (!(phases & 2)) return B200TIMG_OK;
    B2_KERNEL(ctx, "sixel_compact_kernel");
    sixel_compact_kernel<CompactBands><<<dim3(W.nbands, n_frames), 256, 0, ctx->stream>>>(w, h, W, d_offsets, d_out, (unsigned long long)out_cap, NoMixed());
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

// phases: 1 = everything up to and including the frame offsets (sizes known, nothing written),
//         2 = write the bytes.  3 = both, back to back without a host round trip.
int launch_sixel(b200timg_ctx *ctx, const uint8_t *d_fb, int w, int h, int n_frames, char *d_out,
                 size_t out_cap, uint64_t *d_offsets, int phases) {
    if (phases & 1) B2_TRY(launch_sixel_front(ctx, d_fb, w, h, n_frames, 0, n_frames, true));
    return launch_sixel_back(ctx, w, h, n_frames, d_out, out_cap, d_offsets, phases);
}

// ---- mixed-geometry batches (b200timg_sixel_mixed_dev) -----------------------------------------------------------
// The same kernels over frames of different geometry, in a fixed number of launches: the palette kernel twice (frames
// whose median-cut tables fit shared memory, frames that need the global tables), then the table, map, dither, emit5,
// layout, offsets and compaction kernels once each.  Each frame gets exactly what sixel_plan gives a one-frame batch of
// its geometry (table size, band scratch, emit5's column split), so its bytes are that batch's.  Headers and tables stay
// dense per frame; everything else is packed frame after frame and found through the frame's MixedSixelFrame.

// ctx->sixel_work of a mixed plan: [hdr | ent_a | ent_b | lut | index | band sizes | band offsets | scratch | dither
// boundary rows | dither progress]
static size_t mixed_sixel_work(const MixedPlan &mp, int n, char *base, SixelWork *W, size_t *o_bnd, size_t *o_prog) {
    size_t off = 0;
    const size_t o_hdr = off; off += align_up(sizeof(SixelFrameHdr) * n, 256);
    const size_t o_ea = off; off += align_up(sizeof(uint32_t) * mp.sixel_ent, 256);
    const size_t o_eb = off; off += align_up(sizeof(uint32_t) * mp.sixel_ent, 256);
    const size_t o_lut = off; off += align_up((size_t)32768 * n, 256);
    const size_t o_idx = off; off += align_up(mp.sixel_idx, 256);
    const size_t o_bb = off; off += align_up(sizeof(uint32_t) * mp.sixel_bands, 256);
    const size_t o_bo = off; off += align_up(sizeof(uint32_t) * mp.sixel_bands, 256);
    const size_t o_scr = off; off += align_up(mp.sixel_scr, 256);
    *o_bnd = off; off += align_up(sizeof(uint4) * mp.sixel_bnd, 256);
    *o_prog = off; off += align_up(sizeof(int) * mp.sixel_prog, 256);
    if (W) {
        *W = SixelWork{};
        W->hdr = reinterpret_cast<SixelFrameHdr *>(base + o_hdr);
        W->ent_a = reinterpret_cast<uint32_t *>(base + o_ea); W->ent_b = reinterpret_cast<uint32_t *>(base + o_eb);
        W->lut = reinterpret_cast<uint8_t *>(base + o_lut); W->index = reinterpret_cast<uint8_t *>(base + o_idx);
        W->band_bytes = reinterpret_cast<uint32_t *>(base + o_bb); W->band_off = reinterpret_cast<uint32_t *>(base + o_bo);
        W->scratch = base + o_scr;
    }
    return off;
}

int plan_sixel_mixed(b200timg_ctx *ctx, const b200timg_mixed_batch *mb, MixedPlan &mp) {
    const int n = mb->n_frames;
    std::vector<MixedSixelFrame> desc(n);
    std::vector<unsigned> band_start(n + 1), cta_start(n + 1);
    std::vector<int> list[2];
    unsigned long long px = 0;
    size_t ent = 0, idx = 0, bnd = 0, scr = 0, prog = 0;
    unsigned bands = 0, ctas = 0;
    int nwarps = 1, wmax = 1, split = 0;
    size_t pal_smem = 0;
    for (int f = 0; f < n; ++f) {
        const b200timg_frame &F = mb->frames[f];
        MixedSixelFrame &D = desc[f];
        const int w = F.out_w, h = (F.out_h + 5) / 6 * 6;
        const long long npix = (long long)w * h;
        const SixelPaletteShape P = sixel_palette_shape(npix);
        D.w = w; D.h = h;
        D.ent_cap = P.ent_cap;
        D.nb32 = (h + 31) / 32; D.nbands = h / 6;
        D.fb_px = px; px += (unsigned long long)npix;
        D.idx = idx; idx += align_up((size_t)npix, 16);
        D.ent = ent; ent += (size_t)D.ent_cap;
        D.bnd = bnd; bnd += (size_t)D.nb32 * w;
        D.prog0 = (int)prog; prog += (size_t)D.nb32;
        D.band_cap = align_up((size_t)w * 42 + 256 * 5 + 16, 256);
        D.scr = scr; scr += D.band_cap * D.nbands;
        D.band0 = (int)bands; band_start[f] = bands; bands += (unsigned)D.nbands;
        D.cols_per_warp = ((w + EW - 1) / EW + 31) / 32 * 32;
        const SixelDitherShape DS = sixel_dither_shape(D.nb32, n, n, ctx->sm_count, false);
        D.bands_per_cta = DS.bands_per_cta;
        nwarps = std::max(nwarps, DS.nwarps);
        split |= DS.per_frame > 1;
        cta_start[f] = ctas; ctas += (unsigned)DS.per_frame;
        if (P.smem_tables) { list[0].push_back(f); pal_smem = std::max(pal_smem, P.tables_smem); }
        else list[1].push_back(f);
        wmax = std::max(wmax, w);
    }
    band_start[n] = bands; cta_start[n] = ctas;
    mp.sixel_list[0] = (int)list[0].size(); mp.sixel_list[1] = (int)list[1].size();
    for (auto &l : list) if (l.empty()) l.push_back(0);               // a launch without frames still reads list[0]
    mp.o_sixel = mixed_put(mp.arena, desc.data(), sizeof(MixedSixelFrame) * n);
    mp.o_sband = mixed_put(mp.arena, band_start.data(), sizeof(unsigned) * (n + 1));
    mp.o_scta = mixed_put(mp.arena, cta_start.data(), sizeof(unsigned) * (n + 1));
    mp.o_slist[0] = mixed_put(mp.arena, list[0].data(), sizeof(int) * list[0].size());
    mp.o_slist[1] = mixed_put(mp.arena, list[1].data(), sizeof(int) * list[1].size());
    mp.sixel_bands = bands; mp.sixel_ctas = ctas;
    mp.sixel_nwarps = nwarps; mp.sixel_wmax = wmax; mp.sixel_split = split;
    mp.sixel_pal_smem = pal_smem;
    mp.sixel_ent = ent; mp.sixel_idx = idx; mp.sixel_bnd = bnd; mp.sixel_scr = scr; mp.sixel_prog = prog;
    size_t o_bnd, o_prog;
    B2_CUDA(ctx, ctx->sixel_work.reserve(mixed_sixel_work(mp, n, nullptr, nullptr, &o_bnd, &o_prog)));
    return B200TIMG_OK;
}

int launch_sixel_mixed(b200timg_ctx *ctx, const MixedPlan &mp, const char *d_arena, const uint8_t *d_fb, int n,
                       char *d_out, size_t out_cap, uint64_t *d_offsets) {
    char *base = ctx->sixel_work.as<char>();
    SixelWork W;
    size_t o_bnd, o_prog;
    mixed_sixel_work(mp, n, base, &W, &o_bnd, &o_prog);
    ctx->sixel_idx_off = (size_t)(reinterpret_cast<char *>(W.index) - base);      // b200timg_sixel_debug: frame 0
    const uint32_t *fb = reinterpret_cast<const uint32_t *>(d_fb);
    MixedSixelParams M;
    M.desc = reinterpret_cast<const MixedSixelFrame *>(d_arena + mp.o_sixel);
    M.band_start = reinterpret_cast<const unsigned *>(d_arena + mp.o_sband);
    M.cta_start = reinterpret_cast<const unsigned *>(d_arena + mp.o_scta);
    M.n_frames = n; M.nwarps = mp.sixel_nwarps;
    B2_CUDA(ctx, cudaFuncSetAttribute(sixel_palette_kernel<true, PaletteMixed>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    B2_CUDA(ctx, cudaFuncSetAttribute(sixel_palette_kernel<false, PaletteMixed>, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536));
    B2_CUDA(ctx, cudaFuncSetAttribute(sixel_emit1b_kernel<true, BandMixed>, cudaFuncAttributeMaxDynamicSharedMemorySize, (227 - 47) * 1024));
    for (int k = 0; k < 2; ++k) {                 // every launch runs even without frames: the launch count stays fixed
        M.list = reinterpret_cast<const int *>(d_arena + mp.o_slist[k]);
        M.n_list = mp.sixel_list[k];
        const unsigned grid = (unsigned)std::max(1, M.n_list);
        B2_KERNEL(ctx, "sixel_palette_mixed_kernel");
        if (k == 0) sixel_palette_kernel<true, PaletteMixed><<<grid, PT, std::max<size_t>(mp.sixel_pal_smem, 4), ctx->stream>>>(fb, 0, 0, W, M);
        else sixel_palette_kernel<false, PaletteMixed><<<grid, PT, 65536, ctx->stream>>>(fb, 0, 0, W, M);
        B2_LAUNCH_CHECK(ctx);
    }
    M.list = nullptr; M.n_list = 0;
    B2_KERNEL(ctx, "sixel_lut_kernel");
    sixel_lut_kernel<<<dim3(128, n), 256, 0, ctx->stream>>>(W);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "sixel_map_mixed_kernel");
    sixel_map_kernel<MapMixed><<<dim3(64, n), 256, 0, ctx->stream>>>(fb, 0, W, M);
    B2_LAUNCH_CHECK(ctx);
    B2_TRY(launch_sixel_dither_mixed(ctx, fb, mp.sixel_ctas, M, W, base + o_bnd, base + o_prog, mp.sixel_prog, mp.sixel_split != 0));
    B2_KERNEL(ctx, "sixel_emit5_mixed_kernel");
    sixel_emit1b_kernel<true, BandMixed><<<mp.sixel_bands, ET, sizeof(uint32_t) * (size_t)6 * mp.sixel_wmax, ctx->stream>>>(M, W);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "sixel_layout_mixed_kernel");
    sixel_layout_kernel<LayoutMixed><<<n, 256, 0, ctx->stream>>>(0, 0, W, M);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "sixel_sizes_to_offsets_kernel");
    sixel_sizes_to_offsets_kernel<<<1, 1024, 0, ctx->stream>>>(W.hdr, n, d_offsets);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "sixel_compact_mixed_kernel");
    sixel_compact_kernel<BandMixed><<<mp.sixel_bands, 256, 0, ctx->stream>>>(0, 0, W, d_offsets, d_out, (unsigned long long)out_cap, M);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

// Introspection for tests: palette, colour counts and index plane of frame 0 of the last encode.
int sixel_debug_fetch(b200timg_ctx *ctx, uint32_t *h_palette, uint32_t *h_counts, uint8_t *h_index, size_t index_bytes) {
    if (!ctx->sixel_work.p) return ctx->fail(B200TIMG_EINVAL, "sixel: nothing encoded yet");
    SixelFrameHdr host;
    B2_CUDA(ctx, cudaMemcpyAsync(&host, ctx->sixel_work.p, sizeof host, cudaMemcpyDeviceToHost, ctx->stream));
    if (h_index && index_bytes)
        B2_CUDA(ctx, cudaMemcpyAsync(h_index, ctx->sixel_work.as<char>() + ctx->sixel_idx_off, index_bytes,
                                     cudaMemcpyDeviceToHost, ctx->stream));
    B2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (h_palette) memcpy(h_palette, host.palette, sizeof host.palette);
    if (h_counts) { h_counts[0] = host.ncolors; h_counts[1] = host.origcolors; }
    return B200TIMG_OK;
}

}  // namespace b200timg

extern "C" int b200timg_sixel_shape_of(int w, int h, int n_frames, int n_total, int sm_count, b200timg_sixel_shape *out) {
    using namespace b200timg;
    char why[96];
    if (!out || sm_count <= 0 || n_frames <= 0 || n_total < n_frames) return B200TIMG_EINVAL;
    if (sixel_check_geometry(w, h, n_total, why, sizeof why) != B200TIMG_OK) return B200TIMG_EINVAL;      // as sixel_plan
    const SixelPaletteShape P = sixel_palette_shape((long long)w * h);
    out->step_px = (int)P.step_px; out->ent_cap = P.ent_cap; out->palette_global = P.smem_tables ? 0 : 1;
    out->nb32 = (h + 31) / 32;
    const SixelDitherShape D = sixel_dither_shape(out->nb32, n_frames, n_total, sm_count, true);
    out->dither_ctas = D.per_frame; out->bands_per_cta = D.bands_per_cta; out->dither_warps = D.nwarps; out->dither_rounds = D.rounds;
    out->emit_mode = sixel_emit_mode(w);
    int cpw;
    sixel_emit_tiling(w, &out->emit_tiles, &out->tile_w, &cpw);
    return B200TIMG_OK;
}

#ifdef B200TIMG_EMIT_CLOCKS
// instrumented builds only: the summed phase clocks [2][8] since the last call (then cleared); 0 or -3 (CUDA error)
extern "C" int b200timg_emit_clocks(unsigned long long *out) {
    using b200timg::g_emit_clocks;
    static const unsigned long long zero[2][b200timg::EMIT_CLK_PHASES] = {};
    if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(out, g_emit_clocks, sizeof zero) != cudaSuccess ||
        cudaMemcpyToSymbol(g_emit_clocks, zero, sizeof zero) != cudaSuccess)
        return -3;
    return 0;
}
#endif
