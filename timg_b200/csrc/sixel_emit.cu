// K6: the sixel byte stream of libsixel's sixel_encode (call site src/sixel-canvas.cc:144-145; grammar
// of tosixel.c: "#c" colour select, sixel characters 0x3F + 6 row bits, "!n c" run-length form for runs
// longer than 3, "$" carriage return after a colour's pass, "-" between bands) -- single pass.
//
// One CTA per (frame, 6-row band, column tile).  It
//   A  turns each column of the band into its <= 6 distinct (colour, row bits) entries and compacts
//      them per warp in column order,
//   B  ranks the entries with a one-pass 8-bit radix sort on the colour (warp-private histograms,
//      match-based ranking, so equal colours keep their x order -- no shared-memory atomics),
//   C  scatters them into (colour, x) order,
//   D  sizes every run head ("gap + run", colour intro, "$"), scans the sizes, formats the bytes into a
//      shared-memory window and copies the window to its final place with aligned word stores.
// The final place of a CTA's bytes in the frame-after-frame output is the sum of the sizes of all the
// CTAs before it: a decoupled look-back over per-CTA descriptors (size published as soon as it is known,
// inclusive prefix once resolved; CTAs take their place from an atomic ticket, so every predecessor of a
// waiting CTA is running or done).  The look-back of one warp overlaps the formatting of the others.
// Frame f's first CTA also copies the header + palette definitions (sixel_header_kernel), its last CTA
// appends ST.  Nothing is written, and status bit 0 is raised, if the caller's buffer is too small;
// offsets[] is complete either way, so offsets[n_frames] is the size needed.
//
// Algorithmic bytes: 1 B/px index plane read + encoded bytes written.
#include "sixel.cuh"

namespace b200timg {

constexpr int E2T = 1024, E2W = E2T / 32;
constexpr uint32_t M26 = (1u << 26) - 1;      // sorted entry: colour [18:26) | x [6:18) | bits [0:6); [26:31) = encoded length
constexpr int E2_MAX_CHUNKS = 768;            // ent_cap / 32 with ent_cap = 192 * cpw, cpw <= 128

struct Emit2Geom {
    int w, h, nbands, ntiles, tw;             // tw: columns per tile (<= 4096)
    int cpw;                                  // columns per warp, multiple of 32, <= 128
    int ent_cap;                              // 192 * cpw entries
    unsigned n_cta;
};

// lanes of the warp holding the same 8-bit key (valid lanes only)
__device__ __forceinline__ uint32_t match_key8(uint32_t key, bool valid) {
    const uint32_t vm = __ballot_sync(0xffffffffu, valid);
    uint32_t m = 0;
    if (valid) m = __match_any_sync(vm, key);
    return m;
}

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xffffffffu, v, d); if (lane >= d) v += o; }
    return v;
}

// decimal digits of v (< 100000), most significant first, as a little-endian byte string
__device__ __forceinline__ uint32_t ndig5(uint32_t v) { return 1u + (v >= 10u) + (v >= 100u) + (v >= 1000u) + (v >= 10000u); }
__device__ __forceinline__ unsigned long long digits5(uint32_t v, uint32_t nd) {
    const uint32_t q1 = v / 10u, q2 = q1 / 10u, q3 = q2 / 10u, q4 = q3 / 10u;
    const unsigned long long full = (unsigned long long)(0x30u + q4) | ((unsigned long long)(0x30u + q3 - q4 * 10u) << 8) |
                                    ((unsigned long long)(0x30u + q2 - q3 * 10u) << 16) | ((unsigned long long)(0x30u + q1 - q2 * 10u) << 24) |
                                    ((unsigned long long)(0x30u + v - q1 * 10u) << 32);
    return full >> (8u * (5u - nd));
}
// tosixel.c sixel_put_flash: runs of up to 3 are written out, longer ones as "!<n><c>"
__device__ __forceinline__ uint32_t rle_len5(uint32_t n) { return n > 3u ? 2u + ndig5(n) : n; }
__device__ __forceinline__ unsigned long long rle_bytes(uint32_t n, uint32_t ch, uint32_t &nb) {
    if (n > 3u) {
        const uint32_t nd = ndig5(n);
        nb = 2u + nd;
        return 0x21ull | (digits5(n, nd) << 8) | ((unsigned long long)ch << (8u * (1u + nd)));
    }
    nb = n;
    return (unsigned long long)ch * (0x010101ull & ((1ull << (8u * n)) - 1ull));
}

// What sorted entry i contributes to the stream.  Entries are in (colour, x) order; a run is a maximal
// sequence of entries of one colour at consecutive x with the same row bits, written by its first entry.
struct RunInfo { uint32_t c, bits, gap, len, first, last, bytes; };
__device__ __forceinline__ bool run_info(const uint32_t *s, int i, int n, int x0, RunInfo &r) {
    const uint32_t e = s[i] & M26;
    const uint32_t p = i > 0 ? (s[i - 1] & M26) : 0xffffffffu;
    const uint32_t c = e >> 18, x = (e >> 6) & 4095u;
    const bool same = i > 0 && (p >> 18) == c;
    if (same && e == p + 64u) return false;                              // continues the previous entry's run
    uint32_t L = 1;
    while (i + (int)L < n && (s[i + L] & M26) == e + 64u * L) ++L;
    const int j = i + (int)L;
    r.c = c; r.bits = e & 63u; r.len = L;
    r.first = same ? 0u : 1u;
    r.last = (j == n || ((s[j] & M26) >> 18) != c) ? 1u : 0u;
    r.gap = same ? x - ((p >> 6) & 4095u) - 1u : (uint32_t)x0 + x;       // blank columns before the run
    r.bytes = rle_len5(r.gap) + rle_len5(L) + (r.first ? 1u + ndig5(c) : 0u) + r.last;
    return true;
}

// bytes [0, n) of shared memory (4-byte aligned) -> dst (any alignment): aligned 4-byte global stores,
// source words realigned with a funnel shift
__device__ __forceinline__ void copy_window(char *dst, const uint32_t *s32, uint32_t n, int tid) {
    const uint8_t *s8 = reinterpret_cast<const uint8_t *>(s32);
    const uint32_t head = min(n, (uint32_t)((4 - (reinterpret_cast<uintptr_t>(dst) & 3)) & 3));
    if ((uint32_t)tid < head) dst[tid] = (char)s8[tid];
    const uint32_t nw = (n - head) >> 2;
    uint32_t *dw = reinterpret_cast<uint32_t *>(dst + head);
    for (uint32_t j = tid; j < nw; j += E2T) dw[j] = head ? __funnelshift_r(s32[j], s32[j + 1], 8 * head) : s32[j];
    const uint32_t done = head + (nw << 2);
    if (done + tid < n) dst[done + tid] = (char)s8[done + tid];
}

__global__ void __launch_bounds__(E2T, 1)
sixel_emit2_kernel(Emit2Geom G, SixelWork W, uint64_t *__restrict__ offsets, char *__restrict__ out, unsigned long long out_cap) {
    extern __shared__ __align__(16) uint32_t s_e2[];      // ent[ent_cap] (later: byte window) | sorted[ent_cap] | hist[32][256] u16
    __shared__ uint32_t s_cbase[256], s_w[E2W], s_wcnt[E2W], s_chunk[E2_MAX_CHUNKS];
    __shared__ uint32_t s_vid;
    __shared__ unsigned long long s_excl;
    uint32_t *s_ent = s_e2, *s_sorted = s_e2 + G.ent_cap;
    unsigned short *s_hist = reinterpret_cast<unsigned short *>(s_sorted + G.ent_cap);
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint32_t lt = (1u << lane) - 1u;

    if (tid == 0) s_vid = atomicAdd(&W.ctl[0], 1u);
    for (int i = tid; i < E2W * 256 / 2; i += E2T) reinterpret_cast<uint32_t *>(s_hist)[i] = 0;
    __syncthreads();
    const uint32_t vid = s_vid;
    const int per_frame = G.nbands * G.ntiles;
    const int f = (int)(vid / (uint32_t)per_frame), rem = (int)(vid - (uint32_t)f * per_frame);
    const int band = rem / G.ntiles, tile = rem - band * G.ntiles;
    const int x0 = tile * G.tw, tw = min(G.tw, G.w - x0);
    const SixelFrameHdr *hdr = W.hdr + f;
    const uint8_t *idx = W.index + ((long long)f * G.h + (long long)band * 6) * G.w + x0;

    // ---- A: column entries, compacted per warp in column order.  word: bits | x_in_warp << 6 | colour << 13
    const int xl = wid * G.cpw, xh = min(tw, xl + G.cpw), wbase = wid * 6 * G.cpw;
    int n_w = 0;
    for (int xb = xl; xb < xh; xb += 32) {
        const int x = xb + lane;
        uint32_t col[6], bits[6];
        const uint32_t valid = x < xh ? column_entries(idx, G.w, x, col, bits) : 0u;
        const uint32_t k = (uint32_t)__popc(valid);
        const uint32_t incl = warp_incl_scan(k, lane);
        int p = wbase + n_w + (int)(incl - k);
#pragma unroll
        for (int s = 0; s < 6; ++s)
            if (valid & (1u << s)) s_ent[p++] = bits[s] | ((uint32_t)(x - xl) << 6) | (col[s] << 13);
        n_w += (int)__shfl_sync(0xffffffffu, incl, 31);
    }
    __syncwarp();
    // ---- B: rank inside (warp, colour): entries of one warp are in x order, a batch of 32 is ranked by
    // matching colours; the first lane of each group advances the warp's private counter of that colour
    {
        unsigned short *h = s_hist + wid * 256;
        for (int i0 = 0; i0 < n_w; i0 += 32) {
            const int i = i0 + lane;
            const bool v = i < n_w;
            const uint32_t e = v ? s_ent[wbase + i] : 0u;
            const uint32_t c = (e >> 13) & 255u;
            const uint32_t m = match_key8(c, v);
            const uint32_t r = (uint32_t)__popc(m & lt);
            uint32_t old = 0;
            if (v && r == 0) { old = h[c]; h[c] = (unsigned short)(old + (uint32_t)__popc(m)); }
            old = __shfl_sync(0xffffffffu, old, (__ffs((int)m) - 1) & 31);
            if (v) s_ent[wbase + i] = e | ((old + r) << 21);
            __syncwarp();
        }
    }
    __syncthreads();
    // ---- colour totals -> colour bases; hist[w][c] becomes the number of entries of c in earlier warps
    uint32_t tot_c = 0;
    if (tid < 256) {
        for (int k = 0; k < E2W; ++k) { const uint32_t v = s_hist[k * 256 + tid]; s_hist[k * 256 + tid] = (unsigned short)tot_c; tot_c += v; }
    }
    uint32_t n_ent;
    const uint32_t cb = block_excl_scan<E2T>(tid < 256 ? tot_c : 0u, s_w, n_ent);
    if (tid < 256) s_cbase[tid] = cb;
    __syncthreads();
    // ---- C: scatter into (colour, x) order
    {
        const unsigned short *h = s_hist + wid * 256;
        for (int i = lane; i < n_w; i += 32) {
            const uint32_t e = s_ent[wbase + i];
            const uint32_t c = (e >> 13) & 255u;
            const uint32_t pos = s_cbase[c] + h[c] + (e >> 21);
            s_sorted[pos] = (c << 18) | ((uint32_t)(xl + (int)((e >> 6) & 127u)) << 6) | (e & 63u);
        }
    }
    __syncthreads();
    // ---- D: sizes.  A warp takes 32 consecutive entries at a time; the size is parked in the entry word.
    const int n = (int)n_ent, nchunks = (n + 31) >> 5;
    for (int i0 = wid * 32; i0 < n; i0 += E2T) {
        const int i = i0 + lane;
        uint32_t len = 0;
        RunInfo r;
        if (i < n && run_info(s_sorted, i, n, x0, r)) len = r.bytes;
        if (i < n) s_sorted[i] = (s_sorted[i] & M26) | (len << 26);
        const uint32_t incl = warp_incl_scan(len, lane);
        if (lane == 31) s_chunk[i0 >> 5] = incl;
    }
    __syncthreads();
    uint32_t band_total;
    {
        const uint32_t v = tid < nchunks ? s_chunk[tid] : 0u;
        const uint32_t base = block_excl_scan<E2T>(v, s_w, band_total);
        if (tid < nchunks) s_chunk[tid] = base;
    }
    const bool first_cta = band == 0 && tile == 0, last_cta = band == G.nbands - 1 && tile == G.ntiles - 1;
    const uint32_t hdr_len = first_cta ? hdr->header_len : 0u;
    const uint32_t pre = (tile == 0 && band > 0) ? 1u : 0u;                   // '-' : next band
    const unsigned long long agg = (unsigned long long)hdr_len + pre + band_total + (last_cta ? 2u : 0u);
    // ---- look-back (warp 0) while the other warps already format
    if (wid == 0) {
        const unsigned long long VMASK = (1ull << 62) - 1ull;
        volatile unsigned long long *desc = W.desc;
        if (lane == 0) desc[vid] = (1ull << 62) | agg;
        unsigned long long excl = 0;
        long long look = (long long)vid - 1;
        while (look >= 0) {
            const long long j = look - lane;
            unsigned long long d = 2ull << 62;                                // before the first CTA: inclusive prefix 0
            if (j >= 0) { while (((d = desc[j]) >> 62) == 0ull) __nanosleep(64); }
            const uint32_t have = __ballot_sync(0xffffffffu, (d >> 62) == 2ull);
            const int stop = have ? __ffs((int)have) - 1 : 31;                // nearest predecessor with a resolved prefix
            unsigned long long v = lane <= stop ? (d & VMASK) : 0ull;
#pragma unroll
            for (int k = 16; k; k >>= 1) v += __shfl_xor_sync(0xffffffffu, v, k);
            excl += v;
            if (have) break;
            look -= 32;
        }
        if (lane == 0) { desc[vid] = (2ull << 62) | (excl + agg); s_excl = excl; }
    }
    // ---- D: bytes, one shared-memory window at a time (the entry list is dead: reuse it)
    uint8_t *s_out8 = reinterpret_cast<uint8_t *>(s_ent);
    const uint32_t S = (uint32_t)G.ent_cap * 4u;
    bool ovf = false;
    for (uint32_t win0 = 0; win0 == 0 || win0 < band_total; win0 += S) {
        for (int i0 = wid * 32; i0 < n; i0 += E2T) {
            const int i = i0 + lane;
            const uint32_t len = i < n ? (s_sorted[i] >> 26) : 0u;
            const uint32_t incl = warp_incl_scan(len, lane);
            const uint32_t off = s_chunk[i0 >> 5] + incl - len;
            RunInfo r;
            if (len && off + len > win0 && off < win0 + S && run_info(s_sorted, i, n, x0, r)) {
                uint32_t at = off - win0;                                    // may wrap below 0: the window test catches it
                auto put = [&](unsigned long long v, uint32_t nb) {
                    for (uint32_t k = 0; k < nb; ++k, v >>= 8) { const uint32_t q = at + k; if (q < S) s_out8[q] = (uint8_t)v; }
                    at += nb;
                };
                if (r.first) { const uint32_t nd = ndig5(r.c); put(0x23ull | (digits5(r.c, nd) << 8), 1u + nd); }
                uint32_t nb;
                unsigned long long v = rle_bytes(r.gap, 0x3fu, nb); put(v, nb);
                v = rle_bytes(r.len, 0x3fu + r.bits, nb); put(v, nb);
                if (r.last) put(0x24ull, 1u);
            }
        }
        __syncthreads();                                                     // window complete; s_excl visible
        const unsigned long long excl = s_excl;
        ovf = excl + agg > out_cap;
        if (!ovf) {
            const uint32_t nbytes = min(S, band_total - win0);
            copy_window(out + excl + hdr_len + pre + win0, s_ent, nbytes, tid);
        }
        __syncthreads();
    }
    const unsigned long long excl = s_excl;
    if (!ovf) {
        if (first_cta) {
            const char *hb = W.hdr_bytes + (size_t)f * SIXEL_HDR_CAP;
            for (uint32_t i = tid; i < hdr_len; i += E2T) out[excl + i] = hb[i];
        }
        if (tid == 0 && pre) out[excl + hdr_len] = '-';
        if (tid == 0 && last_cta) { out[excl + agg - 2] = '\033'; out[excl + agg - 1] = '\\'; }
    } else if (tid == 0) {
        atomicOr(&W.ctl[1], 1u);
    }
    if (tid == 0) {
        if (first_cta) offsets[f] = excl;
        if (vid == G.n_cta - 1) offsets[f + 1] = excl + agg;
    }
}

// per frame: "ESC P q" + raster attributes + palette definitions (output_rgb_palette_definition:
// percentages (v*100+127)/255) into W.hdr_bytes, its length into hdr->header_len
__global__ void __launch_bounds__(256)
sixel_header_kernel(int w, int h, SixelWork W) {
    __shared__ uint32_t s_w[8];
    const int f = blockIdx.x, tid = threadIdx.x;
    SixelFrameHdr *hdr = W.hdr + f;
    char *hb = W.hdr_bytes + (size_t)f * SIXEL_HDR_CAP;
    const uint32_t fixed = 8 + ndig_u((uint32_t)w) + 1 + ndig_u((uint32_t)h);
    if (tid == 0) {
        char *o = hb;
        *o++ = '\033'; *o++ = 'P'; *o++ = 'q'; *o++ = '"'; *o++ = '1'; *o++ = ';'; *o++ = '1'; *o++ = ';';
        o = put_num_u(o, (uint32_t)w); *o++ = ';'; o = put_num_u(o, (uint32_t)h);
    }
    uint32_t len = 0, r = 0, g = 0, b = 0;
    if ((uint32_t)tid < hdr->ncolors) {
        const uint32_t p = hdr->palette[tid];
        r = ((p & 0xff) * 100 + 127) / 255; g = (((p >> 8) & 0xff) * 100 + 127) / 255; b = (((p >> 16) & 0xff) * 100 + 127) / 255;
        len = 1 + ndig_u((uint32_t)tid) + 3 + ndig_u(r) + 1 + ndig_u(g) + 1 + ndig_u(b);
    }
    uint32_t tot; const uint32_t at = block_excl_scan<256>(len, s_w, tot);
    if (len) {
        char *q = hb + fixed + at;
        *q++ = '#'; q = put_num_u(q, (uint32_t)tid); *q++ = ';'; *q++ = '2'; *q++ = ';';
        q = put_num_u(q, r); *q++ = ';'; q = put_num_u(q, g); *q++ = ';'; q = put_num_u(q, b);
    }
    if (tid == 0) { hdr->header_len = fixed + tot; hdr->frame_size = 0; }
}

static size_t align_up_e(size_t v, size_t a) { return (v + a - 1) / a * a; }

void sixel_emit_tiling(int w, int *ntiles, int *tw, int *cpw) {
    *ntiles = (w + 4095) / 4096;
    int t = (w + *ntiles - 1) / *ntiles;
    t = (t + 31) / 32 * 32;
    *tw = t;
    int c = ((t + E2W - 1) / E2W + 31) / 32 * 32;
    *cpw = c;
}

size_t sixel_emit_workspace(int w, int h, int n_frames, size_t *o_hdr_bytes, size_t *o_desc, size_t *o_ctl) {
    int ntiles, tw, cpw;
    sixel_emit_tiling(w, &ntiles, &tw, &cpw);
    size_t off = 0;
    *o_hdr_bytes = off; off += align_up_e((size_t)SIXEL_HDR_CAP * n_frames, 256);
    *o_desc = off; off += align_up_e(sizeof(unsigned long long) * (size_t)n_frames * (h / 6) * ntiles, 256);
    *o_ctl = off; off += 256;
    return off;
}

int launch_sixel_emit(b200timg_ctx *ctx, int w, int h, int n_frames, const SixelWork &W, char *d_out, size_t out_cap,
                      uint64_t *d_offsets) {
    Emit2Geom G;
    G.w = w; G.h = h; G.nbands = h / 6;
    sixel_emit_tiling(w, &G.ntiles, &G.tw, &G.cpw);
    G.ent_cap = 192 * G.cpw;
    const unsigned long long n_cta = (unsigned long long)n_frames * G.nbands * G.ntiles;    // < 2^31: sixel_check_geometry
    G.n_cta = (unsigned)n_cta;
    const size_t smem = sizeof(uint32_t) * 2 * (size_t)G.ent_cap + sizeof(unsigned short) * E2W * 256;
    B2_CUDA(ctx, cudaFuncSetAttribute(sixel_emit2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // descriptors + ticket + status are contiguous: one memset
    B2_CUDA(ctx, cudaMemsetAsync(W.desc, 0, reinterpret_cast<char *>(W.ctl) + 256 - reinterpret_cast<char *>(W.desc), ctx->stream));
    B2_KERNEL(ctx, "sixel_header_kernel");
    sixel_header_kernel<<<n_frames, 256, 0, ctx->stream>>>(w, h, W);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "sixel_emit2_kernel");
    sixel_emit2_kernel<<<G.n_cta, E2T, smem, ctx->stream>>>(G, W, d_offsets, d_out, (unsigned long long)out_cap);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

}  // namespace b200timg
