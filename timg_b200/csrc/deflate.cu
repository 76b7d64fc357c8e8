// The compressor behind B200TIMG_DEFLATE: the zlib body of each frame's PNG as dynamic-Huffman deflate blocks.
//
// A segment is one 65535-byte block of the stored layout (png.cu): segment k of a frame covers bytes
// [65535k, 65535(k+1)) of its filtered scanline stream.  Every segment of every frame of a batch is an independent
// work item of one warp (deflate_segment_kernel):
//   parse    greedy LZ77.  At each position the candidate is the most recent earlier position with the same hash
//            of the next 4 bytes (a 2^13-entry table that keeps the low 16 bits of the position), taken if at least
//            4 bytes match and it lies at most 32768 bytes back; it may lie in the previous segment's bytes (input
//            only).  The warp looks at 32 positions at once: lane i's candidate is the table's entry or, if newer,
//            the highest earlier lane with the same hash, so the first lane with a match sees exactly what a
//            sequential parse would, and the parse does not depend on scheduling.
//   codes    canonical Huffman codes from the segment's symbol counts (in-place minimum-redundancy lengths, then
//            limited to 15 bits, 7 for the code-length code, by the Kraft-sum adjustment), code lengths run-length
//            coded with 16 / 17 / 18.  Fewer than two used symbols are padded to two so that every code is complete.
//   block    one BTYPE 10 block into the segment's scratch slot, starting at bit 0, BFINAL clear -- unless it is not
//            smaller than the stored block (5 + len bytes) by at least 2 bytes; then the segment stays stored.
// deflate_pack_kernel then writes every block at its bit offset in its frame's zlib stream (offsets from a per-frame
// scan, png.cu) and sets BFINAL on the frame's last block.  A stored block that lands at bit offset o takes
// 3 bits, padding to a byte, LEN, NLEN and the bytes: it ends no later than in the stored layout if o does, and a
// dynamic block ends 16 bits earlier, so no frame's stream is longer than its stored form.
#include <algorithm>

#include "common.cuh"

namespace b200timg {

constexpr int DFL_SEG = 65535, DFL_WIN = 32768, DFL_MIN = 4, DFL_MAX = 258;
constexpr int DFL_HBITS = 13, DFL_WARPS = 4;
constexpr int DFL_NLIT = 286, DFL_NDIST = 30, DFL_NCL = 19, DFL_NSYM = DFL_NLIT + DFL_NDIST + DFL_NCL;
constexpr int DFL_CL = DFL_NLIT + DFL_NDIST;      // where the code-length code's symbols start

struct DflWarp {                                  // one warp's shared state
    uint16_t head[1 << DFL_HBITS];                // hash -> low 16 bits of the latest position with that hash
    uint32_t freq[DFL_NSYM];                      // lit/len, distance, code-length symbol counts
    uint8_t len[DFL_NSYM];
    uint16_t code[DFL_NSYM];                      // bit-reversed canonical codes
    uint16_t rle[DFL_NLIT + DFL_NDIST];           // code-length symbols: symbol | extra value << 5
    uint32_t key[DFL_NLIT];                       // Huffman build: counts sorted ascending, then depths
    uint16_t sym[DFL_NLIT];
    int nrle;
    uint32_t hdr_bits;
};
constexpr size_t DFL_SMEM = sizeof(DflWarp) * DFL_WARPS;

__constant__ uint8_t c_cl_order[DFL_NCL] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

__device__ __forceinline__ uint32_t load4(const uint8_t *p) { return p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
__device__ __forceinline__ uint32_t dfl_hash(uint32_t v) { return (v * 2654435761u) >> (32 - DFL_HBITS); }

// length 3..258 -> symbol 257..285, extra bits and their value (RFC 1951 3.2.5)
__device__ __forceinline__ void len_sym(int len, int &sym, int &nx, int &xv) {
    if (len == 258) { sym = 285; nx = 0; xv = 0; return; }
    const int l = len - 3;
    if (l < 8) { sym = 257 + l; nx = 0; xv = 0; return; }
    const int nb = 31 - __clz(l);
    nx = nb - 2;
    const int hi = (l >> nx) & 3;
    sym = 257 + 4 * (nb - 1) + hi;
    xv = l - ((4 | hi) << nx);
}
// distance 1..32768 -> symbol 0..29, extra bits and their value
__device__ __forceinline__ void dist_sym(int dist, int &sym, int &nx, int &xv) {
    const int d = dist - 1;
    if (d < 4) { sym = d; nx = 0; xv = 0; return; }
    const int nb = 31 - __clz(d);
    nx = nb - 1;
    const int hi = (d >> nx) & 1;
    sym = 2 * nb + hi;
    xv = d - ((2 | hi) << nx);
}

// bits [pos, pos + n) of a zeroed word stream get v (LSB first, n <= 32)
__device__ __forceinline__ void put_bits(uint32_t *w, unsigned long long pos, uint32_t v, int n) {
    if (!n) return;
    const unsigned long long k = pos >> 5;
    const int sh = (int)(pos & 31);
    atomicOr(w + k, v << sh);
    if (sh + n > 32) atomicOr(w + k + 1, v >> (32 - sh));
}

// Warp-collective: positions q of the lanes with ok set go into the hash table; of several lanes with the same hash
// the highest (latest) position wins.
__device__ __forceinline__ void dfl_insert(DflWarp &w, const uint8_t *R, int q, bool ok) {
    const uint32_t h = ok ? dfl_hash(load4(R + q)) : 0xffffffffu;
    const unsigned grp = __match_any_sync(0xffffffffu, h);
    if (ok && (grp >> (threadIdx.x & 31)) == 1u) w.head[h] = (uint16_t)q;
    __syncwarp();
}

// Warp-collective: code lengths (<= limit) of a Huffman code for freq[0..n), in len[0..n).
__device__ void huff_lengths(DflWarp &w, const uint32_t *freq, int n, int limit, uint8_t *len) {
    const int lane = threadIdx.x & 31;
    int used = 0;
    for (int i = lane; i < n; i += 32) used += freq[i] != 0;
    used = __reduce_add_sync(0xffffffffu, used);
    auto f = [&](int i) -> uint32_t { return freq[i] ? freq[i] : (used < 2 && i < 2) ? 1u : 0u; };
    int m = 0;
    for (int i = lane; i < n; i += 32) {
        const uint32_t fi = f(i);
        len[i] = 0;
        if (!fi) continue;
        ++m;
        int r = 0;                                                  // rank by (count, symbol)
        for (int j = 0; j < n; ++j) { const uint32_t fj = f(j); r += fj && (fj < fi || (fj == fi && j < i)); }
        w.key[r] = fi;
        w.sym[r] = (uint16_t)i;
    }
    m = __reduce_add_sync(0xffffffffu, m);
    __syncwarp();
    if (lane == 0) {
        uint32_t *A = w.key;                                        // m >= 2: minimum-redundancy lengths in place
        A[0] += A[1];
        int root = 0, leaf = 2;
        for (int next = 1; next < m - 1; ++next) {
            if (leaf >= m || A[root] < A[leaf]) { A[next] = A[root]; A[root++] = next; } else A[next] = A[leaf++];
            if (leaf >= m || (root < next && A[root] < A[leaf])) { A[next] += A[root]; A[root++] = next; } else A[next] += A[leaf++];
        }
        A[m - 2] = 0;
        for (int next = m - 3; next >= 0; --next) A[next] = A[A[next]] + 1;
        int avbl = 1, cnt_used = 0, depth = 0, root2 = m - 2, next2 = m - 1;
        while (avbl > 0) {
            while (root2 >= 0 && (int)A[root2] == depth) { ++cnt_used; --root2; }
            while (avbl > cnt_used) { A[next2--] = depth; --avbl; }
            avbl = 2 * cnt_used; ++depth; cnt_used = 0;
        }
        uint32_t cnt[33] = {0};
        for (int i = 0; i < m; ++i) ++cnt[min(A[i], 32u)];
        for (int i = limit + 1; i <= 32; ++i) cnt[limit] += cnt[i];
        uint32_t total = 0;
        for (int i = limit; i > 0; --i) total += cnt[i] << (limit - i);
        while (total != (1u << limit)) {                            // over-subscribed after the cut: lengthen codes
            --cnt[limit];
            for (int i = limit - 1; i > 0; --i)
                if (cnt[i]) { --cnt[i]; cnt[i + 1] += 2; break; }
            --total;
        }
        int j = m;                                                  // the most frequent symbols get the shortest codes
        for (int i = 1; i <= limit; ++i)
            for (uint32_t c = cnt[i]; c > 0; --c) len[w.sym[--j]] = (uint8_t)i;
    }
    __syncwarp();
}

__device__ void huff_codes(const uint8_t *len, int n, uint16_t *code) {
    uint32_t cnt[16] = {0}, next[16] = {0};
    for (int i = 0; i < n; ++i) ++cnt[len[i]];
    cnt[0] = 0;
    uint32_t c = 0;
    for (int b = 1; b < 16; ++b) { c = (c + cnt[b - 1]) << 1; next[b] = c; }
    for (int i = 0; i < n; ++i)
        if (len[i]) code[i] = (uint16_t)(__brev(next[len[i]]++) >> (32 - len[i]));
}

// Where segment t of the flat segment list lives: its frame's scanline stream R (raw_len bytes), its index k in that
// frame, the frame's segment count and PNG slot.
//   DflUniform  a b200timg_batch: nseg segments per frame, frame f's stream at raw + f * raw_stride, PNG at f * png_stride
//   DflMixed    a mixed batch: frame f's segments seg_start[f] .. seg_start[f + 1] - 1, its slots in desc[f]
struct DflItem { const uint8_t *R; int raw_len, k, nseg; long long png0; };
struct DflUniform {
    const uint8_t *raw; long long raw_stride; int raw_len, n_frames, nseg; long long png_stride;
    __device__ __forceinline__ long long total() const { return (long long)n_frames * nseg; }
    __device__ __forceinline__ DflItem at(long long t) const {
        const int f = (int)(t / nseg), k = (int)(t - (long long)f * nseg);
        return DflItem{raw + f * raw_stride, raw_len, k, nseg, f * png_stride};
    }
};
struct DflMixed {
    const uint8_t *raw; const MixedGfxFrame *desc; const unsigned *seg_start; int n_frames;
    __device__ __forceinline__ long long total() const { return seg_start[n_frames]; }
    __device__ __forceinline__ DflItem at(long long t) const {
        const int f = mixed_owner(seg_start, n_frames, (unsigned)t);
        const MixedGfxFrame &D = desc[f];
        return DflItem{raw + D.raw_off, (int)D.g.raw_len, (int)(t - seg_start[f]), (int)D.g.nblocks, D.png_off};
    }
};

template <class A>
__device__ __forceinline__ void deflate_segment_body(const A &a, uint32_t *__restrict__ tokens, uint8_t *__restrict__ scratch,
                                                     DeflateSeg *__restrict__ info) {
    extern __shared__ __align__(16) uint8_t dfl_smem[];
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    DflWarp &w = reinterpret_cast<DflWarp *>(dfl_smem)[threadIdx.x >> 5];
    const long long gw = (long long)blockIdx.x * DFL_WARPS + (threadIdx.x >> 5), nw = (long long)gridDim.x * DFL_WARPS;
    uint32_t *tok = tokens + gw * DFL_SEG;
    const long long total = a.total();
    for (long long t = gw; t < total; t += nw) {
        const DflItem it = a.at(t);
        const uint8_t *R = it.R;
        const int raw_len = it.raw_len, k = it.k;
        const int s0 = k * DFL_SEG, n = min(DFL_SEG, raw_len - s0), end = s0 + n;
        for (int i = lane; i < (1 << DFL_HBITS); i += 32) w.head[i] = 0;
        for (int i = lane; i < DFL_NSYM; i += 32) w.freq[i] = 0;
        __syncwarp();
        for (int q0 = max(0, s0 - DFL_WIN); q0 < s0; q0 += 32)
            dfl_insert(w, R, q0 + lane, q0 + lane < s0 && q0 + lane + 4 <= raw_len);

        int p = s0, ntok = 0;
        uint32_t xbits = 0;                                          // extra bits of lengths and distances
        while (p < end) {
            const int q = p + lane;
            const bool hq = q + 4 <= end;
            const uint32_t v = hq ? load4(R + q) : 0u;
            const uint32_t h = hq ? dfl_hash(v) : 0xffffffffu;
            int c = -1;
            if (hq) {
                const int cand = q - ((q - (int)w.head[h]) & 0xffff);
                if (cand < q && q - cand <= DFL_WIN) c = cand;
            }
            const unsigned lower = __match_any_sync(FULL, h) & ((1u << lane) - 1u);
            if (hq && lower) c = p + 31 - __clz(lower);
            const unsigned hits = __ballot_sync(FULL, c >= 0 && load4(R + c) == v);
            const int nlit = hits ? __ffs(hits) - 1 : min(32, end - p);
            if (lane < nlit) { tok[ntok + lane] = R[q]; atomicAdd(&w.freq[R[q]], 1u); }
            dfl_insert(w, R, q, lane < nlit && q + 4 <= raw_len);
            ntok += nlit;
            p += nlit;
            if (!hits) continue;
            const int c0 = __shfl_sync(FULL, c, nlit), maxlen = min(DFL_MAX, end - p);
            int len = DFL_MIN;
            for (;;) {
                const int i = len + lane;
                const unsigned stop = __ballot_sync(FULL, i >= maxlen || R[p + i] != R[c0 + i]);
                if (stop) { len += __ffs(stop) - 1; break; }
                len += 32;
            }
            int s, nx, xv;
            len_sym(len, s, nx, xv);
            xbits += nx;
            if (lane == 0) atomicAdd(&w.freq[s], 1u);
            dist_sym(p - c0, s, nx, xv);
            xbits += nx;
            if (lane == 0) { atomicAdd(&w.freq[DFL_NLIT + s], 1u); tok[ntok] = 0x80000000u | (uint32_t)len << 16 | (uint32_t)(p - c0 - 1); }
            for (int i0 = 0; i0 < len; i0 += 32) dfl_insert(w, R, p + i0 + lane, i0 + lane < len && p + i0 + lane + 4 <= raw_len);
            ++ntok;
            p += len;
        }
        if (lane == 0) w.freq[256] = 1;                              // end of block
        __syncwarp();

        huff_lengths(w, w.freq, DFL_NLIT, 15, w.len);
        huff_lengths(w, w.freq + DFL_NLIT, DFL_NDIST, 15, w.len + DFL_NLIT);
        int hlit = DFL_NLIT, hdist = DFL_NDIST;
        while (hlit > 257 && !w.len[hlit - 1]) --hlit;
        while (hdist > 1 && !w.len[DFL_NLIT + hdist - 1]) --hdist;
        if (lane == 0) {                                             // run-length code the lit/len + distance lengths
            const int total = hlit + hdist;
            auto seq = [&](int i) { return (int)(i < hlit ? w.len[i] : w.len[DFL_NLIT + i - hlit]); };
            int nr = 0;
            for (int i = 0; i < total;) {
                const int v = seq(i);
                int r = 1;
                while (i + r < total && seq(i + r) == v) ++r;
                i += r;
                if (v == 0) {
                    while (r >= 11) { const int e = min(r, 138); w.rle[nr++] = (uint16_t)(18 | (e - 11) << 5); r -= e; }
                    if (r >= 3) { w.rle[nr++] = (uint16_t)(17 | (r - 3) << 5); r = 0; }
                } else {
                    w.rle[nr++] = (uint16_t)v;
                    --r;
                    while (r >= 3) { const int e = min(r, 6); w.rle[nr++] = (uint16_t)(16 | (e - 3) << 5); r -= e; }
                }
                while (r-- > 0) w.rle[nr++] = (uint16_t)v;
            }
            for (int j = 0; j < nr; ++j) ++w.freq[DFL_CL + (w.rle[j] & 31)];
            w.nrle = nr;
        }
        __syncwarp();
        huff_lengths(w, w.freq + DFL_CL, DFL_NCL, 7, w.len + DFL_CL);
        int hclen = DFL_NCL;
        while (hclen > 4 && !w.len[DFL_CL + c_cl_order[hclen - 1]]) --hclen;

        uint32_t bits = 0;                                           // the dynamic block's exact size
        for (int i = lane; i < DFL_NSYM; i += 32) bits += w.freq[i] * w.len[i];
        bits = __reduce_add_sync(FULL, bits) + 3 + 14 + 3 * hclen + xbits + 2 * w.freq[DFL_CL + 16] + 3 * w.freq[DFL_CL + 17] +
               7 * w.freq[DFL_CL + 18];
        const bool dynamic = bits + 16 <= 40 + 8u * (uint32_t)n;
        if (lane == 0) info[t] = DeflateSeg{dynamic ? bits : 0u, dynamic ? 0u : 1u};
        if (dynamic) {
            uint32_t *W = reinterpret_cast<uint32_t *>(scratch + t * DFL_SLOT);
            for (int i = lane; i <= (int)(bits + 31) / 32; i += 32) W[i] = 0;
            __syncwarp();
            if (lane == 0) {
                huff_codes(w.len, DFL_NLIT, w.code);
                huff_codes(w.len + DFL_NLIT, DFL_NDIST, w.code + DFL_NLIT);
                huff_codes(w.len + DFL_CL, DFL_NCL, w.code + DFL_CL);
                unsigned long long pos = 0;
                put_bits(W, pos, 2u << 1, 3); pos += 3;              // BFINAL 0 (set when packed), BTYPE 10
                put_bits(W, pos, hlit - 257, 5); pos += 5;
                put_bits(W, pos, hdist - 1, 5); pos += 5;
                put_bits(W, pos, hclen - 4, 4); pos += 4;
                for (int i = 0; i < hclen; ++i) { put_bits(W, pos, w.len[DFL_CL + c_cl_order[i]], 3); pos += 3; }
                for (int j = 0; j < w.nrle; ++j) {
                    const int s = w.rle[j] & 31, e = w.rle[j] >> 5, ne = s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0;
                    put_bits(W, pos, w.code[DFL_CL + s] | (uint32_t)e << w.len[DFL_CL + s], w.len[DFL_CL + s] + ne);
                    pos += w.len[DFL_CL + s] + ne;
                }
                w.hdr_bits = (uint32_t)pos;
            }
            __syncwarp();
            unsigned long long pos = w.hdr_bits;
            for (int i0 = 0; i0 < ntok; i0 += 32) {                  // 32 tokens at a time, placed by a warp scan
                const int i = i0 + lane;
                uint32_t v1 = 0, v2 = 0;
                int n1 = 0, n2 = 0;
                if (i < ntok) {
                    const uint32_t tk = tok[i];
                    if (!(tk >> 31)) { v1 = w.code[tk]; n1 = w.len[tk]; }
                    else {
                        int s, nx, xv;
                        len_sym((int)(tk >> 16 & 0x1ff), s, nx, xv);
                        v1 = w.code[s] | (uint32_t)xv << w.len[s]; n1 = w.len[s] + nx;
                        dist_sym((int)(tk & 0xffff) + 1, s, nx, xv);
                        v2 = w.code[DFL_NLIT + s] | (uint32_t)xv << w.len[DFL_NLIT + s]; n2 = w.len[DFL_NLIT + s] + nx;
                    }
                }
                const uint32_t nb = n1 + n2;
                uint32_t incl = nb;
                for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(FULL, incl, d); if (lane >= d) incl += o; }
                const unsigned long long at = pos + incl - nb;
                put_bits(W, at, v1, n1);
                put_bits(W, at + n1, v2, n2);
                pos += __shfl_sync(FULL, incl, 31);
            }
            if (lane == 0) put_bits(W, pos, w.code[256], w.len[256]);
        }
        __syncwarp();
    }
}
__global__ void __launch_bounds__(32 * DFL_WARPS)
deflate_segment_kernel(const uint8_t *__restrict__ raw, long long raw_stride, int raw_len, int n_frames, int nseg,
                       uint32_t *__restrict__ tokens, uint8_t *__restrict__ scratch, DeflateSeg *__restrict__ info) {
    deflate_segment_body(DflUniform{raw, raw_stride, raw_len, n_frames, nseg, 0}, tokens, scratch, info);
}
__global__ void __launch_bounds__(32 * DFL_WARPS)
deflate_segment_mixed_kernel(const uint8_t *__restrict__ raw, const MixedGfxFrame *__restrict__ desc, const unsigned *__restrict__ seg_start,
                             int n_frames, uint32_t *__restrict__ tokens, uint8_t *__restrict__ scratch, DeflateSeg *__restrict__ info) {
    deflate_segment_body(DflMixed{raw, desc, seg_start, n_frames}, tokens, scratch, info);
}

// One CTA per segment (grid-stride): the segment's block at bit 8 * zoff + start[t] of its frame's PNG slot (slot
// zeroed beforehand).  Words the block covers entirely are stored, the two it shares with its neighbours are OR'ed.
template <class A_>
__device__ __forceinline__ void deflate_pack_body(const A_ &a, const uint8_t *__restrict__ scratch, const DeflateSeg *__restrict__ info,
                                                  const unsigned long long *__restrict__ start, uint8_t *__restrict__ png, int zoff) {
    for (long long t = blockIdx.x; t < a.total(); t += gridDim.x) {
        const DflItem it = a.at(t);
        const int raw_len = it.raw_len, k = it.k, nseg = it.nseg;
        const DeflateSeg sg = info[t];
        const uint32_t n = (uint32_t)min(DFL_SEG, raw_len - k * DFL_SEG);
        const unsigned long long A = 8ull * zoff + start[t];
        const unsigned long long P = (A + 10) & ~7ull;               // a stored block's LEN, after 3 bits and padding
        const unsigned long long B = sg.stored ? P + 32 + 8ull * n : A + sg.bits;
        uint32_t *D = reinterpret_cast<uint32_t *>(png + it.png0);
        const uint32_t *S = reinterpret_cast<const uint32_t *>(scratch + t * DFL_SLOT);
        const uint8_t *Rs = it.R + (long long)k * DFL_SEG;
        for (unsigned long long wd = (A >> 5) + threadIdx.x; wd <= (B - 1) >> 5; wd += blockDim.x) {
            const unsigned long long lo = wd * 32;
            uint32_t v = 0;
            if (!sg.stored) {
                const long long o = (long long)lo - (long long)A;
                if (o < 0) v = S[0] << (int)-o;
                else {
                    const int sh = (int)(o & 31);
                    const uint32_t a = S[o >> 5];
                    v = sh ? (a >> sh) | (S[(o >> 5) + 1] << (32 - sh)) : a;
                }
            } else {
                for (int b = 0; b < 4; ++b) {
                    const unsigned long long q = lo + 8 * b;
                    if (q < P || q >= B) continue;
                    const long long i = (long long)(q - P) >> 3;
                    const uint32_t byte = i == 0 ? n & 255 : i == 1 ? n >> 8 : i == 2 ? ~n & 255 : i == 3 ? (~n >> 8) & 255 : Rs[i - 4];
                    v |= byte << (8 * b);
                }
            }
            if (k == nseg - 1 && wd == A >> 5) v |= 1u << (A & 31);   // BFINAL
            if (lo >= A && lo + 32 <= B) D[wd] = v;
            else atomicOr(D + wd, v);
        }
    }
}
__global__ void __launch_bounds__(256)
deflate_pack_kernel(const uint8_t *__restrict__ raw, long long raw_stride, int raw_len, int n_frames, int nseg,
                    const uint8_t *__restrict__ scratch, const DeflateSeg *__restrict__ info,
                    const unsigned long long *__restrict__ start, uint8_t *__restrict__ png, long long png_stride, int zoff) {
    deflate_pack_body(DflUniform{raw, raw_stride, raw_len, n_frames, nseg, png_stride}, scratch, info, start, png, zoff);
}
__global__ void __launch_bounds__(256)
deflate_pack_mixed_kernel(const uint8_t *__restrict__ raw, const MixedGfxFrame *__restrict__ desc, const unsigned *__restrict__ seg_start,
                          int n_frames, const uint8_t *__restrict__ scratch, const DeflateSeg *__restrict__ info,
                          const unsigned long long *__restrict__ start, uint8_t *__restrict__ png, int zoff) {
    deflate_pack_body(DflMixed{raw, desc, seg_start, n_frames}, scratch, info, start, png, zoff);
}

int launch_deflate(b200timg_ctx *ctx, const uint8_t *d_raw, long long raw_stride, int raw_len, int n_frames, int nseg,
                   uint8_t *d_scratch, DeflateSeg *d_info) {
    const long long items = (long long)n_frames * nseg;
    const long long ctas = std::min<long long>((items + DFL_WARPS - 1) / DFL_WARPS, (long long)ctx->sm_count * 2);
    B2_CUDA(ctx, ctx->dfl_tokens.reserve((size_t)ctas * DFL_WARPS * DFL_SEG * sizeof(uint32_t)));
    B2_CUDA(ctx, cudaFuncSetAttribute(deflate_segment_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DFL_SMEM));
    B2_KERNEL(ctx, "deflate_segment_kernel");
    deflate_segment_kernel<<<(unsigned)ctas, 32 * DFL_WARPS, DFL_SMEM, ctx->stream>>>(d_raw, raw_stride, raw_len, n_frames, nseg,
                                                                                    ctx->dfl_tokens.as<uint32_t>(), d_scratch, d_info);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

int launch_deflate_pack(b200timg_ctx *ctx, const uint8_t *d_raw, long long raw_stride, int raw_len, int n_frames, int nseg,
                        const uint8_t *d_scratch, const DeflateSeg *d_info, const unsigned long long *d_start, uint8_t *d_png,
                        long long png_stride, int zoff) {
    const long long items = (long long)n_frames * nseg;
    B2_KERNEL(ctx, "deflate_pack_kernel");
    deflate_pack_kernel<<<(unsigned)std::min<long long>(items, (long long)ctx->sm_count * 16), 256, 0, ctx->stream>>>(
        d_raw, raw_stride, raw_len, n_frames, nseg, d_scratch, d_info, d_start, d_png, png_stride, zoff);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

// The same two passes over a mixed batch's flat segment list: the launch shapes follow the list's length as above.
int launch_deflate_mixed(b200timg_ctx *ctx, const uint8_t *d_raw, const MixedGfxFrame *d_desc, const unsigned *d_seg_start,
                         int n_frames, unsigned n_segs, uint8_t *d_scratch, DeflateSeg *d_info) {
    const long long ctas = std::min<long long>((n_segs + DFL_WARPS - 1) / DFL_WARPS, (long long)ctx->sm_count * 2);
    B2_CUDA(ctx, ctx->dfl_tokens.reserve((size_t)ctas * DFL_WARPS * DFL_SEG * sizeof(uint32_t)));
    B2_CUDA(ctx, cudaFuncSetAttribute(deflate_segment_mixed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DFL_SMEM));
    B2_KERNEL(ctx, "deflate_segment_mixed_kernel");
    deflate_segment_mixed_kernel<<<(unsigned)ctas, 32 * DFL_WARPS, DFL_SMEM, ctx->stream>>>(d_raw, d_desc, d_seg_start, n_frames,
                                                                                          ctx->dfl_tokens.as<uint32_t>(), d_scratch, d_info);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

int launch_deflate_pack_mixed(b200timg_ctx *ctx, const uint8_t *d_raw, const MixedGfxFrame *d_desc, const unsigned *d_seg_start,
                              int n_frames, unsigned n_segs, const uint8_t *d_scratch, const DeflateSeg *d_info,
                              const unsigned long long *d_start, uint8_t *d_png, int zoff) {
    B2_KERNEL(ctx, "deflate_pack_mixed_kernel");
    deflate_pack_mixed_kernel<<<(unsigned)std::min<long long>(n_segs, (long long)ctx->sm_count * 16), 256, 0, ctx->stream>>>(
        d_raw, d_desc, d_seg_start, n_frames, d_scratch, d_info, d_start, d_png, zoff);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

}  // namespace b200timg
