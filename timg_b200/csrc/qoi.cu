// QOI files on the device: the RGBA buffer qoi_read(filename, &desc, 4) returns for timg's QOI source
// (src/qoi-image-source.cc:42-77, third_party/qoi/qoi.h:488-590), with every quirk of qoi_decode: the op stream is the
// bytes [14, size - 8) whatever the last 8 bytes hold, an op that starts there may read into them, the last value
// repeats to the end of the image once the ops run out, ops past the last pixel are ignored, and the header's channel
// count never reaches the ops.
//   host walk            qoi_decode's header checks; the files' op regions cut into tiles, chunks and segment slots
//   qoi_tile_kernel      one thread per TILE bytes of op region: for each of the 5 phases a tile can be entered at
//                        (bytes of an op begun in the tile before), its exit phase, op count and pixel count
//   qoi_chunk_kernel     one thread per CHUNK tiles: the composition of their maps (a map that starts a file resets)
//   qoi_top_kernel       one CTA: the chunks' entry states (phase, op index and first pixel inside their file)
//   qoi_ops_kernel       one thread per tile: each live op's first pixel and the byte offset of each segment's first op
//   qoi_spec_kernel      one thread per segment (SEG consecutive live ops of a file): decodes it from the initial state
//                        (px {0,0,0,255}, an all-zero index), storing its state at the checkpoints every CK ops
//   qoi_sync_kernel      ROUNDS launches: each segment re-decodes from its predecessor's exit of the previous round and
//                        stops where its state can be adopted (below); a round that changes no exit makes the later
//                        rounds return at once
//   qoi_fixup_kernel     one CTA per file: segments whose entry still differs from their predecessor's exit, in order,
//                        by one thread, so the result never depends on how far the rounds got
//   qoi_canvas_kernel    one thread per pixel: the value of the op that owns it (binary search on first pixels)
// A decoder state is (px, index[64]): 260 bytes, compared word for word.  A state S reached at a checkpoint can be
// adopted in place of the stored state T there when px is equal and no slot where they differ is read by an INDEX op
// after the checkpoint before an op writes it: every later op then computes the same px, so the stored values and
// states stay, and only the differing slots not written since are patched into the later states.  With equal states
// this is the usual self-synchronisation stop.
// A call launches 7 + ROUNDS kernels whatever its files hold.
#include <algorithm>
#include <climits>

#include "decode.cuh"

namespace b200timg {

namespace {

constexpr int TILE = 64;             // op-region bytes per tile
constexpr int CHUNK = 64;            // tiles per chunk
constexpr int TOP_T = 1024;          // threads of qoi_top_kernel
constexpr int SEG = 256;             // live ops per segment
constexpr int CK = 64;               // ops between checkpoints
constexpr int NI = SEG / CK;         // intervals per segment; a segment stores NI - 1 inner checkpoints
constexpr int ROUNDS = 8;            // qoi_sync_kernel launches
constexpr int DEC_T = 128;           // threads of the spec and sync kernels (each has a 64-word index column)
constexpr int FIX_T = 128;
constexpr unsigned HEADER = 14, PADDING = 8;
constexpr unsigned long long SIZE_CAP = 1ull << 31;   // qoi_read holds the file size in an int
constexpr uint32_t PX0 = 0xff000000u;                 // {0, 0, 0, 255}

struct __align__(16) QoiFile {
    unsigned long long off;          // the file's first byte in the uploaded files
    unsigned long long op0;          // its first op slot in the first-pixel and value arrays
    unsigned long long px0;          // its first canvas pixel
    unsigned end;                    // size - 8: ops start before it
    unsigned npx;                    // w * h
    unsigned tile0, seg0;            // its first tile and segment slot
    int channels, pad_;
};

struct St { uint32_t px, idx[64]; };  // a decoder state, as qoi_decode holds it

// A map entry: pixels (bits 0-31), ops (32-59), exit phase (60-62); bit 63 of entry 0: the map starts a file.  A call
// has less than OPS_CAP op bytes, so a run of chunks that one thread of qoi_top_kernel composes fits both fields.
constexpr unsigned long long HEAD = 1ull << 63;
constexpr unsigned long long OPS_CAP = 1ull << 36;
__device__ __forceinline__ unsigned long long ment(unsigned x, unsigned long long o, unsigned long long p) {
    return p | o << 32 | (unsigned long long)x << 60;
}
struct Cur { unsigned x, o; unsigned long long p; };  // phase, op index and first pixel inside the file

__device__ __forceinline__ Cur apply(const unsigned long long *m, Cur c) {
    const unsigned long long e0 = m[0];
    const unsigned long long e = (e0 & HEAD) ? e0 : m[c.x];
    Cur r;
    r.x = (unsigned)(e >> 60) & 7;
    r.o = (unsigned)((e >> 32) & 0xfffffff) + ((e0 & HEAD) ? 0u : c.o);
    r.p = (e & 0xffffffffull) + ((e0 & HEAD) ? 0ull : c.p);
    return r;
}

__device__ __forceinline__ unsigned op_len(unsigned b) { return b == 0xfe ? 4 : b == 0xff ? 5 : (b >> 6) == 2 ? 2 : 1; }
__device__ __forceinline__ unsigned op_px(unsigned b) { return (b >> 6) == 3 && b < 0xfe ? (b & 63) + 1 : 1; }
__device__ __forceinline__ unsigned qhash(uint32_t v) {
    return ((v & 255) * 3 + ((v >> 8) & 255) * 5 + ((v >> 16) & 255) * 7 + (v >> 24) * 11) & 63;
}

// ---- op boundaries -----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
qoi_tile_kernel(const uint8_t *__restrict__ files, const QoiFile *__restrict__ fd, const unsigned *__restrict__ tile0,
                int n, unsigned n_tiles, unsigned long long *__restrict__ maps, unsigned *__restrict__ nlive,
                int32_t *__restrict__ status, unsigned *__restrict__ round_changed) {
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    const unsigned long long g0 = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (unsigned long long i = g0; i < (unsigned long long)n; i += stride) { nlive[i] = 0; status[i] = 1; }
    for (unsigned long long i = g0; i <= (unsigned long long)ROUNDS; i += stride) round_changed[i] = 0;
    for (unsigned long long t = g0; t < n_tiles; t += stride) {
        const int f = mixed_owner(tile0, n, (unsigned)t);
        const QoiFile F = fd[f];
        const uint8_t *b = files + F.off;
        const unsigned k = (unsigned)t - F.tile0, a = HEADER + k * TILE;
        const unsigned e = min(a + TILE, F.end);
        for (unsigned ph = 0; ph < 5; ++ph) {
            if (k == 0 && ph > 0) { maps[t * 5 + ph] = maps[t * 5]; continue; }
            unsigned pos = a + ph, o = 0, p = 0;
            while (pos < e) { const unsigned c = b[pos]; ++o; p += op_px(c); pos += op_len(c); }
            maps[t * 5 + ph] = ment(pos < e ? 0 : pos - e, o, p) | (k == 0 && ph == 0 ? HEAD : 0);
        }
    }
}

__global__ void __launch_bounds__(256)
qoi_chunk_kernel(const unsigned long long *__restrict__ maps, unsigned n_tiles, unsigned n_chunks,
                 unsigned long long *__restrict__ cmaps) {
    for (unsigned long long c = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks;
         c += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned t0 = (unsigned)c * CHUNK, t1 = min(t0 + CHUNK, n_tiles);
        unsigned long long head = 0;
        Cur s[5];
#pragma unroll
        for (unsigned ph = 0; ph < 5; ++ph) s[ph] = Cur{ph, 0, 0};
        for (unsigned t = t0; t < t1; ++t) {
            head |= maps[t * 5ull] & HEAD;
#pragma unroll
            for (int ph = 0; ph < 5; ++ph) s[ph] = apply(maps + t * 5ull, s[ph]);
        }
#pragma unroll
        for (int ph = 0; ph < 5; ++ph) cmaps[c * 5 + ph] = ment(s[ph].x, s[ph].o, s[ph].p) | (ph == 0 ? head : 0);
    }
}

// The entry state of every chunk: each thread composes a run of chunks, thread 0 walks the runs, each thread its own.
__global__ void __launch_bounds__(TOP_T)
qoi_top_kernel(const unsigned long long *__restrict__ cmaps, unsigned n_chunks, Cur *__restrict__ centry) {
    __shared__ unsigned long long agg[TOP_T * 5];
    const unsigned q = (n_chunks + TOP_T - 1) / TOP_T, c0 = threadIdx.x * q, c1 = min(c0 + q, n_chunks);
    unsigned long long head = 0;
    for (unsigned c = c0; c < c1; ++c) head |= cmaps[c * 5ull] & HEAD;
    for (unsigned ph = 0; ph < 5; ++ph) {
        Cur s{ph, 0, 0};
        for (unsigned c = c0; c < c1; ++c) s = apply(cmaps + c * 5ull, s);
        agg[threadIdx.x * 5 + ph] = ment(s.x, s.o, s.p) | (ph == 0 ? head : 0);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        Cur s{0, 0, 0};
        for (int i = 0; i < TOP_T; ++i) {                 // agg[i] becomes thread i's entry state, in place
            const Cur nx = apply(agg + i * 5, s);      // an empty run composed to the identity
            agg[i * 5] = s.x; agg[i * 5 + 1] = s.o; agg[i * 5 + 2] = s.p;
            s = nx;
        }
    }
    __syncthreads();
    Cur s{(unsigned)agg[threadIdx.x * 5], (unsigned)agg[threadIdx.x * 5 + 1], agg[threadIdx.x * 5 + 2]};
    for (unsigned c = c0; c < c1; ++c) { centry[c] = s; s = apply(cmaps + c * 5ull, s); }
}

// Every live op (first pixel < w*h) gets its first pixel; every SEG-th its byte offset; the last one sets nlive.
__global__ void __launch_bounds__(256)
qoi_ops_kernel(const uint8_t *__restrict__ files, const QoiFile *__restrict__ fd, const unsigned *__restrict__ tile0,
               int n, unsigned n_tiles, const unsigned long long *__restrict__ maps, const Cur *__restrict__ centry,
               uint32_t *__restrict__ fpx, uint32_t *__restrict__ segoff, unsigned *__restrict__ nlive) {
    for (unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; t < n_tiles;
         t += (unsigned long long)gridDim.x * blockDim.x) {
        const int f = mixed_owner(tile0, n, (unsigned)t);
        const QoiFile F = fd[f];
        const unsigned k = (unsigned)t - F.tile0;
        Cur s{0, 0, 0};
        if (k != 0) {
            s = centry[t / CHUNK];
            for (unsigned u = (unsigned)t / CHUNK * CHUNK; u < t; ++u) s = apply(maps + u * 5ull, s);
        }
        const uint8_t *b = files + F.off;
        const unsigned a = HEADER + k * TILE, e = min(a + TILE, F.end);
        unsigned long long p = s.p;
        unsigned o = s.o;
        for (unsigned pos = a + s.x; pos < e && p < F.npx;) {
            const unsigned c = b[pos], len = op_len(c), np = op_px(c);
            fpx[F.op0 + o] = (uint32_t)p;
            if (o % SEG == 0) segoff[F.seg0 + o / SEG] = pos;
            if (p + np >= F.npx || pos + len >= F.end) nlive[f] = o + 1;
            ++o; p += np; pos += len;
        }
    }
}

// ---- values ------------------------------------------------------------------------------------------------------
struct Seg {                         // where a segment's ops and stored states are
    const uint8_t *b;                // its file
    unsigned pos;                    // byte offset of its first op
    unsigned long long op;           // its first op slot
    unsigned nops;
};

struct Scratch {
    const uint8_t *files;
    const QoiFile *fd;
    const unsigned *seg0;
    int n;
    const uint32_t *segoff;
    const unsigned *nlive;
    uint32_t *val;
    St *entry, *ck, *xs[2];          // ck: NI - 1 per segment slot; xs: the exits, by round parity
    unsigned long long *iw, *ib;     // per interval: slots written, slots read by INDEX before any write in it
    unsigned *chg;                   // the segment's exit changed in the last round that ran
    unsigned *round_changed;         // [r]: round r changed an exit
};

__device__ __forceinline__ Seg seg_of(const Scratch &S, const QoiFile &F, unsigned s, unsigned nl) {
    Seg g;
    g.b = S.files + F.off;
    g.pos = S.segoff[F.seg0 + s];
    g.op = F.op0 + (unsigned long long)s * SEG;
    g.nops = min((unsigned)SEG, nl - s * SEG);
    return g;
}

// ops [i0, i1) of segment g from px / T (column of stride `ts`): the values, and the interval's slot masks
__device__ __forceinline__ void run_ops(const Seg &g, unsigned &pos, uint32_t &px, uint32_t *T, int ts, uint32_t *val,
                                        unsigned i0, unsigned i1, unsigned long long &w, unsigned long long &rb) {
    w = 0; rb = 0;
    for (unsigned i = i0; i < i1; ++i) {
        const unsigned c = g.b[pos];
        if (c == 0xfe) {
            px = (px & 0xff000000u) | g.b[pos + 1] | (uint32_t)g.b[pos + 2] << 8 | (uint32_t)g.b[pos + 3] << 16;
            pos += 4;
        } else if (c == 0xff) {
            px = g.b[pos + 1] | (uint32_t)g.b[pos + 2] << 8 | (uint32_t)g.b[pos + 3] << 16 | (uint32_t)g.b[pos + 4] << 24;
            pos += 5;
        } else if ((c >> 6) == 0) {
            if (!((w >> c) & 1)) rb |= 1ull << c;
            px = T[c * ts];
            pos += 1;
        } else if ((c >> 6) == 1) {
            const uint32_t r = (px + ((c >> 4) & 3) - 2) & 255, gg = ((px >> 8) + ((c >> 2) & 3) - 2) & 255,
                           bb = ((px >> 16) + (c & 3) - 2) & 255;
            px = (px & 0xff000000u) | r | gg << 8 | bb << 16;
            pos += 1;
        } else if ((c >> 6) == 2) {
            const unsigned d = g.b[pos + 1];
            const uint32_t vg = (c & 63) - 32;
            const uint32_t r = (px + vg - 8 + ((d >> 4) & 15)) & 255, gg = ((px >> 8) + vg) & 255,
                           bb = ((px >> 16) + vg - 8 + (d & 15)) & 255;
            px = (px & 0xff000000u) | r | gg << 8 | bb << 16;
            pos += 2;
        } else {
            pos += 1;                                       // RUN: px stays, the index is still written
        }
        const unsigned h = qhash(px);
        T[h * ts] = px;
        w |= 1ull << h;
        val[g.op + i] = px;
    }
}

__device__ __forceinline__ void put_state(St *d, uint32_t px, const uint32_t *T, int ts) {
    d->px = px;
    for (int i = 0; i < 64; ++i) d->idx[i] = T[i * ts];
}

// Segment slot q (segment g) from the entry state in px / T.  fresh: nothing is stored yet (the speculative pass).
// Else the stored states are consistent with the stored entry, and the decode stops at the first position (entry,
// checkpoint or exit) whose state can be adopted.  The exit goes to *xn (the old one is *xo; they may be the same).
// Returns whether the exit differs from *xo.
__device__ __forceinline__ bool resync(const Scratch &S, const Seg &g, unsigned q, uint32_t px, uint32_t *T, int ts, bool fresh,
                       const St *xo, St *xn) {
    const unsigned ni = (g.nops + CK - 1) / CK;
    unsigned pos = g.pos;
    for (unsigned c = 0;; ++c) {
        St *stored = c == 0 ? S.entry + q : c < ni ? S.ck + (size_t)q * (NI - 1) + (c - 1) : nullptr;
        if (c == ni) {                                      // the exit
            bool ch = fresh;
            if (!fresh) {
                ch = xo->px != px;
                for (int i = 0; i < 64; ++i) ch |= xo->idx[i] != T[i * ts];
            }
            put_state(xn, px, T, ts);
            return ch;
        }
        if (!fresh && stored->px == px) {
            unsigned long long d = 0;
            for (int i = 0; i < 64; ++i) d |= (unsigned long long)(stored->idx[i] != T[i * ts]) << i;
            unsigned long long rb = 0, wacc = 0;
            for (unsigned k = c; k < ni; ++k) { rb |= S.ib[(size_t)q * NI + k] & ~wacc; wacc |= S.iw[(size_t)q * NI + k]; }
            if (!(d & rb)) {                                // adopt: patch the differing slots forward
                unsigned long long m = d;
                for (unsigned k = c; k <= ni; ++k) {
                    if (k > c) m &= ~S.iw[(size_t)q * NI + k - 1];
                    if (k < ni) {
                        St *t = k == 0 ? S.entry + q : S.ck + (size_t)q * (NI - 1) + (k - 1);
                        for (unsigned long long r = m; r; r &= r - 1) t->idx[__ffsll((long long)r) - 1] = T[(__ffsll((long long)r) - 1) * ts];
                    } else {
                        if (xn != xo) { xn->px = xo->px; for (int i = 0; i < 64; ++i) xn->idx[i] = xo->idx[i]; }
                        for (unsigned long long r = m; r; r &= r - 1) xn->idx[__ffsll((long long)r) - 1] = T[(__ffsll((long long)r) - 1) * ts];
                    }
                }
                return m != 0;
            }
        }
        put_state(stored, px, T, ts);
        unsigned long long w, rb;
        run_ops(g, pos, px, T, ts, S.val, c * CK, min((c + 1) * CK, g.nops), w, rb);
        S.iw[(size_t)q * NI + c] = w;
        S.ib[(size_t)q * NI + c] = rb;
    }
}

__device__ __forceinline__ void load_state(const St *s, uint32_t &px, uint32_t *T, int ts) {
    px = s->px;
    for (int i = 0; i < 64; ++i) T[i * ts] = s->idx[i];
}

__global__ void __launch_bounds__(DEC_T)
qoi_spec_kernel(Scratch S, unsigned n_slots) {
    __shared__ uint32_t tab[64 * DEC_T];
    uint32_t *T = tab + threadIdx.x;
    for (unsigned long long q = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; q < n_slots;
         q += (unsigned long long)gridDim.x * blockDim.x) {
        const int f = mixed_owner(S.seg0, S.n, (unsigned)q);
        const QoiFile F = S.fd[f];
        const unsigned s = (unsigned)q - F.seg0, nl = S.nlive[f];
        if (s * (unsigned long long)SEG >= nl) continue;
        for (int i = 0; i < 64; ++i) T[i * DEC_T] = 0;
        resync(S, seg_of(S, F, s, nl), (unsigned)q, PX0, T, DEC_T, true, nullptr, S.xs[0] + q);
    }
}

__global__ void __launch_bounds__(DEC_T)
qoi_sync_kernel(Scratch S, unsigned n_slots, int round) {
    if (round > 1 && !*(volatile unsigned *)&S.round_changed[round - 1]) return;
    __shared__ uint32_t tab[64 * DEC_T];
    uint32_t *T = tab + threadIdx.x;
    const St *xprev = (round & 1) ? S.xs[0] : S.xs[1];   // selected, not indexed: S stays in the parameter space
    St *xcur = (round & 1) ? S.xs[1] : S.xs[0];
    bool any = false;
    for (unsigned long long q = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; q < n_slots;
         q += (unsigned long long)gridDim.x * blockDim.x) {
        const int f = mixed_owner(S.seg0, S.n, (unsigned)q);
        const QoiFile F = S.fd[f];
        const unsigned s = (unsigned)q - F.seg0, nl = S.nlive[f];
        if (s * (unsigned long long)SEG >= nl) continue;
        bool ch = false;
        if (s == 0) {
            xcur[q] = xprev[q];
        } else {
            uint32_t px;
            load_state(xprev + q - 1, px, T, DEC_T);
            ch = resync(S, seg_of(S, F, s, nl), (unsigned)q, px, T, DEC_T, false, xprev + q, xcur + q);
        }
        S.chg[q] = ch;
        any |= ch;
    }
    if (__syncthreads_or(any) && threadIdx.x == 0) atomicOr(&S.round_changed[round], 1u);
}

// One CTA per file: finds the segments whose predecessor's exit changed in the last round, and re-syncs them and
// every segment after them whose predecessor's exit changes here, in order, on thread 0.
__global__ void __launch_bounds__(FIX_T)
qoi_fixup_kernel(Scratch S) {
    int last = 1;                                           // the last round that ran
    while (last < ROUNDS && S.round_changed[last]) ++last;
    if (!S.round_changed[last]) return;                     // it changed nothing: every entry is its predecessor's exit
    __shared__ uint32_t T[64];
    __shared__ unsigned found, next;
    const QoiFile F = S.fd[blockIdx.x];
    const unsigned nl = S.nlive[blockIdx.x], nseg = (nl + SEG - 1) / SEG;
    St *x = (last & 1) ? S.xs[1] : S.xs[0];
    unsigned s = 1;
    while (s < nseg) {
        if (threadIdx.x == 0) found = UINT_MAX;
        __syncthreads();
        unsigned first = UINT_MAX;                          // the first segment from s whose predecessor changed
        for (unsigned base = s; base < nseg; base += FIX_T) {
            const unsigned t = base + threadIdx.x;
            if (t < nseg && S.chg[F.seg0 + t - 1]) atomicMin(&found, t);
            __syncthreads();
            first = found;
            __syncthreads();                                // every thread has read found before the next atomicMin
            if (first != UINT_MAX) break;
        }
        if (first == UINT_MAX) break;
        if (threadIdx.x == 0) {
            unsigned u = first;
            for (; u < nseg; ++u) {
                const unsigned q = F.seg0 + u;
                uint32_t px;
                load_state(x + q - 1, px, T, 1);
                if (!resync(S, seg_of(S, F, u, nl), q, px, T, 1, false, x + q, x + q)) break;
            }
            next = u + 1;
        }
        __syncthreads();
        s = next;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256)
qoi_canvas_kernel(const QoiFile *__restrict__ fd, const unsigned long long *__restrict__ px0, int n,
                  const unsigned *__restrict__ nlive, const uint32_t *__restrict__ fpx, const uint32_t *__restrict__ val,
                  unsigned long long total, uint32_t *__restrict__ out, int32_t *__restrict__ status) {
    for (unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; k < total;
         k += (unsigned long long)gridDim.x * blockDim.x) {
        const int f = mixed_owner(px0, n, k);
        const QoiFile &F = fd[f];
        const uint32_t q = (uint32_t)(k - F.px0);
        const unsigned nl = nlive[f];
        uint32_t v = PX0;
        if (nl) {
            const uint32_t *fp = fpx + F.op0;
            unsigned lo = q / 62 < nl ? q / 62 : nl - 1, hi = min(q, nl - 1);   // an op covers 1..62 pixels
            while (lo < hi) {
                const unsigned mid = (lo + hi + 1) >> 1;
                if (fp[mid] <= q) lo = mid; else hi = mid - 1;
            }
            v = val[F.op0 + lo];
        }
        out[k] = v;
        if (F.channels == 3 && (v >> 24) != 255) status[f] = 2;
    }
}

// ---- host walk ---------------------------------------------------------------------------------------------------
struct Parse {
    unsigned w = 0, h = 0;
    int channels = 0, colorspace = 0;
    bool supported = false;
    char why[96] = {0};
};

unsigned be32(const uint8_t *d) { return (unsigned)d[0] << 24 | (unsigned)d[1] << 16 | (unsigned)d[2] << 8 | d[3]; }

// 0: qoi_decode takes the header (P.supported says whether the device takes the file); -1: it returns NULL
int qoi_walk(const uint8_t *d, size_t size, Parse &P) {
    if (size < HEADER + PADDING) return -1;
    P.w = be32(d + 4); P.h = be32(d + 8); P.channels = d[12]; P.colorspace = d[13];
    if (P.w == 0 || P.h == 0 || P.channels < 3 || P.channels > 4 || P.colorspace > 1 || be32(d) != 0x716f6966u ||
        P.h >= 400000000u / P.w)
        return -1;
    P.supported = size < SIZE_CAP;
    if (!P.supported) snprintf(P.why, sizeof P.why, "%zu bytes: qoi_read holds the size in an int", size);
    return 0;
}

void fill_info(const Parse &P, b200timg_qoi_info *info) {
    memset(info, 0, sizeof *info);
    info->w = (int)P.w; info->h = (int)P.h; info->channels = P.channels; info->colorspace = P.colorspace;
    info->supported = P.supported ? 1 : 0;
    snprintf(info->reason, sizeof info->reason, "%s", P.supported ? "" : P.why);
}

// Device scratch of one call (ctx->qoi_up.arena + ctx->qoi_scratch): the files + 48 bytes per file; per op-region
// byte 8 bytes (first pixel and value of an op, which takes at least one byte) and 40 / TILE bytes of tile maps; per
// segment slot (one per SEG op-region bytes) 6 * 260 bytes of states (the entry, NI - 1 checkpoints and the two exits),
// NI * 16 bytes of slot masks and 8 bytes of offset and change flag.
int launch_qoi(b200timg_ctx *ctx, int n, const uint8_t *const *files, const size_t *sizes, const std::vector<Parse> &ps,
               uint8_t *d_frames, int32_t *d_status) {
    std::vector<QoiFile> fdesc((size_t)n);
    std::vector<unsigned> tile0(1, 0), seg0(1, 0);
    std::vector<unsigned long long> px0(1, 0);
    unsigned long long off = 0, ops = 0, tiles = 0, segs = 0;
    for (int f = 0; f < n; ++f) {
        const Parse &P = ps[(size_t)f];
        QoiFile &F = fdesc[(size_t)f];
        memset(&F, 0, sizeof F);
        const unsigned long long region = sizes[f] - PADDING > HEADER ? sizes[f] - PADDING - HEADER : 0;
        F.off = off; F.op0 = ops; F.px0 = px0.back();
        F.end = (unsigned)(sizes[f] - PADDING);
        F.npx = P.w * P.h;
        F.tile0 = (unsigned)tiles; F.seg0 = (unsigned)segs;
        F.channels = P.channels;
        off += sizes[f]; ops += region;
        tiles += (region + TILE - 1) / TILE;
        segs += (region + SEG - 1) / SEG;
        if (ops >= OPS_CAP) return ctx->fail(B200TIMG_EINVAL, "qoi: 2^36 op bytes or more in one call");
        tile0.push_back((unsigned)tiles); seg0.push_back((unsigned)segs);
        px0.push_back(px0.back() + F.npx);
    }
    const unsigned n_tiles = (unsigned)tiles, n_chunks = (n_tiles + CHUNK - 1) / CHUNK, n_slots = (unsigned)segs;

    std::vector<char> arena;
    const size_t o_fd = mixed_put(arena, fdesc.data(), sizeof(QoiFile) * fdesc.size());
    const size_t o_t0 = mixed_put(arena, tile0.data(), sizeof(unsigned) * tile0.size());
    const size_t o_s0 = mixed_put(arena, seg0.data(), sizeof(unsigned) * seg0.size());
    const size_t o_p0 = mixed_put(arena, px0.data(), sizeof(unsigned long long) * px0.size());
    size_t o_file;
    B2_TRY(staged_upload(ctx, ctx->qoi_up, arena, n, files, sizes, &o_file));
    auto al = [](unsigned long long v) { return (v + 255) / 256 * 256; };
    const size_t s_maps = 0, s_cm = s_maps + al(40ull * n_tiles), s_ce = s_cm + al(40ull * n_chunks),
                 s_fpx = s_ce + al(sizeof(Cur) * n_chunks), s_val = s_fpx + al(4 * ops), s_so = s_val + al(4 * ops),
                 s_nl = s_so + al(4ull * n_slots), s_ent = s_nl + al(4ull * n), s_ck = s_ent + al(sizeof(St) * n_slots),
                 s_x0 = s_ck + al(sizeof(St) * (NI - 1) * (size_t)n_slots), s_x1 = s_x0 + al(sizeof(St) * n_slots),
                 s_iw = s_x1 + al(sizeof(St) * n_slots), s_ib = s_iw + al(8ull * NI * n_slots),
                 s_chg = s_ib + al(8ull * NI * n_slots), s_rc = s_chg + al(4ull * n_slots), s_end = s_rc + al(4 * (ROUNDS + 1));
    B2_CUDA(ctx, ctx->qoi_scratch.reserve(s_end));
    const char *A = ctx->qoi_up.arena.as<char>();
    char *B = ctx->qoi_scratch.as<char>();
    const uint8_t *d_files = reinterpret_cast<const uint8_t *>(A + o_file);
    const QoiFile *d_fd = reinterpret_cast<const QoiFile *>(A + o_fd);
    const unsigned *d_t0 = reinterpret_cast<const unsigned *>(A + o_t0);
    unsigned long long *d_maps = reinterpret_cast<unsigned long long *>(B + s_maps);
    unsigned long long *d_cm = reinterpret_cast<unsigned long long *>(B + s_cm);
    Cur *d_ce = reinterpret_cast<Cur *>(B + s_ce);
    uint32_t *d_fpx = reinterpret_cast<uint32_t *>(B + s_fpx);
    unsigned *d_nl = reinterpret_cast<unsigned *>(B + s_nl);
    Scratch S;
    S.files = d_files; S.fd = d_fd; S.seg0 = reinterpret_cast<const unsigned *>(A + o_s0); S.n = n;
    uint32_t *d_so = reinterpret_cast<uint32_t *>(B + s_so);
    S.segoff = d_so; S.nlive = d_nl;
    S.val = reinterpret_cast<uint32_t *>(B + s_val);
    S.entry = reinterpret_cast<St *>(B + s_ent); S.ck = reinterpret_cast<St *>(B + s_ck);
    S.xs[0] = reinterpret_cast<St *>(B + s_x0); S.xs[1] = reinterpret_cast<St *>(B + s_x1);
    S.iw = reinterpret_cast<unsigned long long *>(B + s_iw); S.ib = reinterpret_cast<unsigned long long *>(B + s_ib);
    S.chg = reinterpret_cast<unsigned *>(B + s_chg); S.round_changed = reinterpret_cast<unsigned *>(B + s_rc);

    const long long init = std::max(std::max((long long)n_tiles, (long long)n), (long long)ROUNDS + 1);
    B2_KERNEL(ctx, "qoi_tile_kernel");
    qoi_tile_kernel<<<grid_for(ctx, init), 256, 0, ctx->stream>>>(d_files, d_fd, d_t0, n, n_tiles, d_maps, d_nl,
                                                                   d_status, S.round_changed);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "qoi_chunk_kernel");
    qoi_chunk_kernel<<<grid_for(ctx, n_chunks), 256, 0, ctx->stream>>>(d_maps, n_tiles, n_chunks, d_cm);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "qoi_top_kernel");
    qoi_top_kernel<<<1, TOP_T, 0, ctx->stream>>>(d_cm, n_chunks, d_ce);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "qoi_ops_kernel");
    qoi_ops_kernel<<<grid_for(ctx, n_tiles), 256, 0, ctx->stream>>>(d_files, d_fd, d_t0, n, n_tiles, d_maps, d_ce,
                                                                     d_fpx, d_so, d_nl);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "qoi_spec_kernel");
    qoi_spec_kernel<<<grid_for(ctx, n_slots, DEC_T), DEC_T, 0, ctx->stream>>>(S, n_slots);
    B2_LAUNCH_CHECK(ctx);
    for (int r = 1; r <= ROUNDS; ++r) {
        B2_KERNEL(ctx, "qoi_sync_kernel");
        qoi_sync_kernel<<<grid_for(ctx, n_slots, DEC_T), DEC_T, 0, ctx->stream>>>(S, n_slots, r);
        B2_LAUNCH_CHECK(ctx);
    }
    B2_KERNEL(ctx, "qoi_fixup_kernel");
    qoi_fixup_kernel<<<n, FIX_T, 0, ctx->stream>>>(S);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "qoi_canvas_kernel");
    qoi_canvas_kernel<<<grid_for(ctx, (long long)px0.back()), 256, 0, ctx->stream>>>(
        d_fd, reinterpret_cast<const unsigned long long *>(A + o_p0), n, d_nl, d_fpx, S.val, px0.back(),
        reinterpret_cast<uint32_t *>(d_frames), d_status);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

}  // namespace
}  // namespace b200timg

using namespace b200timg;

extern "C" {

int b200timg_qoi_parse(const uint8_t *qoi, size_t size, b200timg_qoi_info *info) {
    if (!qoi || size == 0 || !info) return B200TIMG_EINVAL;
    Parse P;
    if (qoi_walk(qoi, size, P) != 0) return B200TIMG_EINVAL;
    fill_info(P, info);
    return B200TIMG_OK;
}

int b200timg_qoi_frames_dev(b200timg_ctx *ctx, int n_files, const uint8_t *const *files, const size_t *sizes,
                            uint8_t *d_frames, int32_t *d_status) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    B2_TRY(check_dev_outputs(ctx, "qoi", d_frames, d_status, "d_status"));
    std::vector<Parse> ps;
    B2_TRY(parse_files(ctx, "qoi", "header check", qoi_walk, n_files, files, sizes, ps));
    return launch_qoi(ctx, n_files, files, sizes, ps, d_frames, d_status);
}

int b200timg_qoi_frames(b200timg_ctx *ctx, int n_files, const uint8_t *const *files, const size_t *sizes,
                        uint8_t *frames, int32_t *status) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!frames || !status) return ctx->fail(B200TIMG_EINVAL, "qoi: null output");
    std::vector<Parse> ps;
    B2_TRY(parse_files(ctx, "qoi", "header check", qoi_walk, n_files, files, sizes, ps));
    size_t bytes = 0;
    for (const Parse &P : ps) bytes += (size_t)P.w * P.h * 4;
    return decode_to_host(ctx, bytes, n_files, frames, status, [&](uint8_t *d_frames, int32_t *d_status) {
        return launch_qoi(ctx, n_files, files, sizes, ps, d_frames, d_status);
    });
}

}  // extern "C"
