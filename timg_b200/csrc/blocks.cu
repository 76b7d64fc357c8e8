// K3: UnicodeBlockCanvas::Send image bytes on the device -- half/quarter block glyph pick
// (FindBestGlyph, src/unicode-block-canvas.cc:162-227) and the ANSI byte stream of
// AppendDoubleRow/Send (:230-321, :361-399), byte-identical to the reference.
//
// The reference walks cells left to right carrying serial state (last emitted fg, last
// emitted cell's bg, pending x_skip / y_skip).  Restated as data-parallel passes:
//   pass A  (grid = row pairs x frames): per cell glyph pick; "previous emitted cell" and
//           "previous fg-carrying cell" found with block-wide max-scans; per-cell byte
//           length; exclusive add-scan -> offset inside the row.  One 16-byte record/cell.
//   pass B  (one block per frame): empty-row runs (y_skip) + exclusive scan over rows.
//   pass C  (one block): exclusive scan over frame sizes -> compact batch offsets.
//   pass D  (grid = row pairs x frames): every cell writes its bytes at its final offset.
// All comparisons are on the full 32-bit rgba like rgba_t::operator== (framebuffer.h:30-33).
//
// Algorithmic bytes per frame: 4*W*H read (+4*W*H for the previous frame in delta mode)
// + encoded bytes written.  Cell records (16 B/cell, written once, read once) are
// intermediates.
#include "common.cuh"

namespace b200timg {

enum : uint32_t { kBackground = 0, kTopLeft, kTopRight, kBotLeft, kBotRight, kLeftBar,
                  kTopLeftBotRight, kLowerBlock, kUpperBlock };

// meta word layout
constexpr uint32_t M_BLOCK_MASK = 0xf, M_EMIT_FG = 1u << 4, M_EMIT_BG = 1u << 5,
                   M_BG_TRANSP = 1u << 6, M_SKIPPED = 1u << 7, M_FIRST = 1u << 8;
constexpr int M_XSKIP_SHIFT = 9;

struct __align__(16) CellRec { uint32_t fg, bg, meta, off; };
struct __align__(16) RowRec { uint32_t len, nonempty, off, yskip; };
struct __align__(16) FrameRec { uint32_t size, trailing, pad0, pad1; };

struct Lin { float r, g, b, a; };

__device__ __forceinline__ Lin lin_of(uint32_t p) {   // LinearColor(rgba_t), framebuffer.h:143
    const uint32_t r = p & 0xff, g = (p >> 8) & 0xff, b = (p >> 16) & 0xff;
    Lin l; l.r = (float)(r * r); l.g = (float)(g * g); l.b = (float)(b * b); l.a = (float)(p >> 24);
    return l;
}
__device__ __forceinline__ uint32_t repack(const Lin &l) {   // framebuffer.h:150-152
    return pack_rgba(ungamma(l.r), ungamma(l.g), ungamma(l.b), __float2uint_rz(l.a) & 0xff);
}
__device__ __forceinline__ float dist(const Lin &t, const Lin &o) {   // t.dist(o), :145-148
    const float dr = fsub(o.r, t.r), dg = fsub(o.g, t.g), db = fsub(o.b, t.b);
    return fadd(fadd(fmul(dr, dr), fmul(dg, dg)), fmul(db, db));
}
// avd() over 2, 3 or 4 values in list order (framebuffer.h:177-194)
__device__ __forceinline__ float avd2(Lin &m, const Lin &a, const Lin &b) {
    m.r = fdiv(fadd(a.r, b.r), 2.f); m.g = fdiv(fadd(a.g, b.g), 2.f);
    m.b = fdiv(fadd(a.b, b.b), 2.f); m.a = fdiv(fadd(a.a, b.a), 2.f);
    return fadd(dist(m, a), dist(m, b));          // 0 + d(a) is exact
}
__device__ __forceinline__ float avd3(Lin &m, const Lin &a, const Lin &b, const Lin &c) {
    m.r = fdiv(fadd(fadd(a.r, b.r), c.r), 3.f); m.g = fdiv(fadd(fadd(a.g, b.g), c.g), 3.f);
    m.b = fdiv(fadd(fadd(a.b, b.b), c.b), 3.f); m.a = fdiv(fadd(fadd(a.a, b.a), c.a), 3.f);
    return fadd(fadd(dist(m, a), dist(m, b)), dist(m, c));
}
__device__ __forceinline__ float avd4(Lin &m, const Lin &a, const Lin &b, const Lin &c, const Lin &d) {
    m.r = fdiv(fadd(fadd(fadd(a.r, b.r), c.r), d.r), 4.f);
    m.g = fdiv(fadd(fadd(fadd(a.g, b.g), c.g), d.g), 4.f);
    m.b = fdiv(fadd(fadd(fadd(a.b, b.b), c.b), d.b), 4.f);
    m.a = fdiv(fadd(fadd(fadd(a.a, b.a), c.a), d.a), 4.f);
    return fadd(fadd(fadd(dist(m, a), dist(m, b)), dist(m, c)), dist(m, d));
}

__device__ __forceinline__ bool transparent(uint32_t p) { return (p >> 24) < 0x60u; }   // :154

struct Pick { uint32_t fg, bg, block; };

__device__ __forceinline__ Pick pick_half(uint32_t top, uint32_t bot, bool upper) {   // :164-172
    Pick p;
    if (top == bot || (transparent(top) && transparent(bot))) { p.fg = top; p.bg = bot; p.block = kBackground; }
    else if (upper) { p.fg = top; p.bg = bot; p.block = kUpperBlock; }
    else { p.fg = bot; p.bg = top; p.block = kLowerBlock; }
    return p;
}

__device__ Pick pick_quarter(uint32_t t0, uint32_t t1, uint32_t b0, uint32_t b1, bool upper) {  // :174-227
    Pick p;
    const bool tt = transparent(t0) && transparent(t1);
    const bool bt = transparent(b0) && transparent(b1);
    const Lin tl = lin_of(t0), tr = lin_of(t1), bl = lin_of(b0), br = lin_of(b1);
    if (tt && bt) { p.fg = b0; p.bg = t0; p.block = kBackground; return p; }
    if (tt) { Lin m; avd2(m, bl, br); p.fg = repack(m); p.bg = t0; p.block = kLowerBlock; return p; }
    if (bt) { Lin m; avd2(m, tl, tr); p.fg = repack(m); p.bg = b0; p.block = kUpperBlock; return p; }

    Lin best_fg = {0, 0, 0, 0}, best_bg = {0, 0, 0, 0};
    uint32_t best_block = kBackground;
    float best_d = 1e12f;
    bool done = false;
    // The 8 candidates in the reference's order; first strict minimum wins, stop at d<1.
#define B2_TRY_PICK(BLOCK, D, FG, BG)                                    \
    if (!done) {                                                         \
        const float d__ = (D);                                           \
        if (d__ < best_d) {                                              \
            best_fg = (FG); best_bg = (BG); best_block = (BLOCK);        \
            if (d__ < 1.0f) done = true; else best_d = d__;              \
        }                                                                \
    }
    { Lin bg; const float d = avd4(bg, tl, tr, bl, br); B2_TRY_PICK(kBackground, d, bg, bg) }
    if (!done) { Lin bg; const float d = avd3(bg, tr, bl, br); B2_TRY_PICK(kTopLeft, d, tl, bg) }
    if (!done) { Lin bg; const float d = avd3(bg, tl, bl, br); B2_TRY_PICK(kTopRight, d, tr, bg) }
    if (!done) { Lin bg; const float d = avd3(bg, tl, tr, br); B2_TRY_PICK(kBotLeft, d, bl, bg) }
    if (!done) { Lin bg; const float d = avd3(bg, tl, tr, bl); B2_TRY_PICK(kBotRight, d, br, bg) }
    if (!done) { Lin bg, fg; float d = avd2(bg, tr, br); d = fadd(d, avd2(fg, tl, bl)); B2_TRY_PICK(kLeftBar, d, fg, bg) }
    if (!done) { Lin bg, fg; float d = avd2(bg, tr, bl); d = fadd(d, avd2(fg, tl, br)); B2_TRY_PICK(kTopLeftBotRight, d, fg, bg) }
    if (!done) {
        Lin bg, fg; float d;
        if (upper) { d = avd2(bg, bl, br); d = fadd(d, avd2(fg, tl, tr)); B2_TRY_PICK(kUpperBlock, d, fg, bg) }
        else       { d = avd2(bg, tl, tr); d = fadd(d, avd2(fg, bl, br)); B2_TRY_PICK(kLowerBlock, d, fg, bg) }
    }
#undef B2_TRY_PICK
    p.fg = repack(best_fg); p.bg = repack(best_bg); p.block = best_block;
    return p;
}

// rgba_t::As256TermColor, src/framebuffer.h:37-52
__host__ __device__ __forceinline__ uint32_t as256(uint32_t p) {
    const uint32_t r = p & 0xff, g = (p >> 8) & 0xff, b = (p >> 16) & 0xff;
    if (r == g && g == b) return (232 + (r * 23 / 255)) & 0xff;
    auto cube = [](uint32_t v) -> uint32_t {
        return v < 47 ? 0 : v < 115 ? 1 : v < 155 ? 2 : v < 195 ? 3 : v < 235 ? 4 : 5;
    };
    return 16 + 36 * cube(r) + 6 * cube(g) + cube(b);
}

__device__ __forceinline__ uint32_t ndig8(uint32_t v) { return v >= 100 ? 3 : v >= 10 ? 2 : 1; }
__device__ __forceinline__ uint32_t ndig(uint32_t v) {
    uint32_t n = 1;
    while (v >= 10) { v /= 10; ++n; }
    return n;
}
__device__ __forceinline__ uint32_t color_len(uint32_t p, bool color8) {   // digits + ';' each
    if (color8) return ndig8(as256(p)) + 1;
    return ndig8(p & 0xff) + ndig8((p >> 8) & 0xff) + ndig8((p >> 16) & 0xff) + 3;
}
__device__ __forceinline__ uint32_t yskip_len(uint32_t ys) {   // :249-258
    return ys == 0 ? 0 : (ys <= 4 ? ys : 3 + ndig(ys));
}

// ---------------------------------------------------------------- block-wide scans
// Inclusive scans over 256 threads; result for thread i covers threads 0..i.
__device__ __forceinline__ void block_scan_max2(int &a, int &b, int *smem /*[16]*/) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int oa = __shfl_up_sync(0xffffffffu, a, d), ob = __shfl_up_sync(0xffffffffu, b, d);
        if (lane >= d) { a = max(a, oa); b = max(b, ob); }
    }
    if (lane == 31) { smem[wid] = a; smem[8 + wid] = b; }
    __syncthreads();
    int pa = -1, pb = -1;
    for (int k = 0; k < wid; ++k) { pa = max(pa, smem[k]); pb = max(pb, smem[8 + k]); }
    a = max(a, pa); b = max(b, pb);
    __syncthreads();
}
__device__ __forceinline__ uint32_t block_scan_add(uint32_t v, uint32_t *smem /*[8]*/, uint32_t &total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += o;
    }
    if (lane == 31) smem[wid] = v;
    __syncthreads();
    uint32_t pre = 0, tot = 0;
    for (int k = 0; k < 8; ++k) { if (k < wid) pre += smem[k]; tot += smem[k]; }
    total = tot;
    __syncthreads();
    return v + pre;   // inclusive
}

struct BlocksParams {
    int w, h, n_frames, cols, rows;       // cols = cells per row, rows = row pairs
    int quarter, upper, color8, indent;
    int row_offset;                       // -1 when odd height and lower block (:356-358)
    int prev_mode;                        // 0 none, 1 explicit prev, 2 animation, 3 animation whose frame 0 is a halo (not emitted)
    long long frame_px;
};

constexpr int BT = 256;

// Where a CTA's row pair and its frame live.  The pass bodies below read every per-frame quantity through one of
// these accessors:
//   UniformGeom  a b200timg_batch: every frame has P's geometry, frame f at fb + f * P.frame_px, records frame-major
//   MixedGeom    a mixed batch: each frame has its own geometry and record offsets (MixedBlocksFrame), no delta frames
struct UniformGeom {
    typedef BlocksParams Params;
    const BlocksParams &P;
    int f, r;                             // frame, row pair
    __device__ __forceinline__ UniformGeom(const BlocksParams &p, int f_, int r_) : P(p), f(f_), r(r_) {}
    __device__ __forceinline__ explicit UniformGeom(const BlocksParams &p) : P(p), f(blockIdx.y), r(blockIdx.x) {}
    __device__ __forceinline__ int quarter() const { return P.quarter; }
    __device__ __forceinline__ int upper() const { return P.upper; }
    __device__ __forceinline__ int color8() const { return P.color8; }
    __device__ __forceinline__ int w() const { return P.w; }
    __device__ __forceinline__ int h() const { return P.h; }
    __device__ __forceinline__ int cols() const { return P.cols; }
    __device__ __forceinline__ int rows() const { return P.rows; }
    __device__ __forceinline__ int row_offset() const { return P.row_offset; }
    __device__ __forceinline__ int indent() const { return P.indent; }
    __device__ __forceinline__ int prev_mode() const { return P.prev_mode; }
    __device__ __forceinline__ long long frame_px0() const { return (long long)f * P.frame_px; }        // first pixel
    __device__ __forceinline__ long long prev_px0() const { return (long long)(f - 1) * P.frame_px; }
    __device__ __forceinline__ long long first_row_rec() const { return (long long)f * P.rows; }
    __device__ __forceinline__ long long first_cell_rec() const { return ((long long)f * P.rows + r) * P.cols; }
};

struct MixedBlocksParams {
    const MixedBlocksFrame *desc;
    const unsigned *row_start;            // [n_frames + 1] first (frame, row pair) item of each frame
    int n_frames, flags;
};
struct MixedGeom {
    typedef MixedBlocksParams Params;
    MixedBlocksFrame D;
    unsigned row0;                        // the frame's first row record (its first flat item)
    int f, r, flags;
    __device__ __forceinline__ MixedGeom(const MixedBlocksFrame *frames, const unsigned *row_start, int f_, int r_)
        : D(frames[f_]), row0(row_start[f_]), f(f_), r(r_), flags(0) {}
    // one CTA per flat item blockIdx.x
    __device__ __forceinline__ explicit MixedGeom(const MixedBlocksParams &Q) : flags(Q.flags) {
        f = mixed_owner(Q.row_start, Q.n_frames, blockIdx.x);
        row0 = Q.row_start[f];
        r = (int)(blockIdx.x - row0);
        D = Q.desc[f];
    }
    __device__ __forceinline__ int quarter() const { return flags & B200TIMG_QUARTER; }
    __device__ __forceinline__ int upper() const { return flags & B200TIMG_UPPER; }
    __device__ __forceinline__ int color8() const { return flags & B200TIMG_COLOR8; }
    __device__ __forceinline__ int w() const { return D.w; }
    __device__ __forceinline__ int h() const { return D.h; }
    __device__ __forceinline__ int cols() const { return D.cols; }
    __device__ __forceinline__ int rows() const { return D.rows; }
    __device__ __forceinline__ int row_offset() const { return D.row_offset; }
    __device__ __forceinline__ int indent() const { return D.indent; }
    __device__ __forceinline__ int prev_mode() const { return 0; }
    __device__ __forceinline__ long long frame_px0() const { return (long long)D.fb_px; }
    __device__ __forceinline__ long long prev_px0() const { return 0; }                                  // never read: no delta
    __device__ __forceinline__ long long first_row_rec() const { return row0; }
    __device__ __forceinline__ long long first_cell_rec() const { return (long long)D.cell0 + (long long)r * D.cols; }
};

// pass A.  A kernel template rather than a body shared by two kernels (as rowscan and emit are): this way the uniform
// instantiation is optimised as one function, exactly as before the mixed form existed, and compiles to the same SASS.
template <class G>
__global__ void __launch_bounds__(BT)
blocks_pick_kernel(const uint32_t *__restrict__ fb, const uint32_t *__restrict__ prev_single,
                   typename G::Params P, CellRec *__restrict__ cells, RowRec *__restrict__ rows) {
    __shared__ int s_i[16];
    __shared__ uint32_t s_u[8];
    __shared__ uint32_t s_fg[BT], s_bg[BT];
    __shared__ int c_last_emit, c_last_fgidx;
    __shared__ uint32_t c_last_bg, c_last_fg, c_run;

    const G g(P);
    const int r = g.r, f = g.f, tid = threadIdx.x;
    const uint32_t *frame = fb + g.frame_px0();
    const uint32_t *prev = nullptr;
    if (g.prev_mode() == 1) prev = prev_single;
    else if (g.prev_mode() >= 2 && f > 0) prev = fb + g.prev_px0();

    const int top_row = 2 * r + g.row_offset(), bot_row = top_row + 1;
    const bool top_ok = top_row >= 0, bot_ok = bot_row < g.h();
    const uint32_t *trow = frame + (long long)top_row * g.w(), *brow = frame + (long long)bot_row * g.w();
    const uint32_t *ptrow = prev ? prev + (long long)top_row * g.w() : nullptr;
    const uint32_t *pbrow = prev ? prev + (long long)bot_row * g.w() : nullptr;

    if (tid == 0) { c_last_emit = -1; c_last_fgidx = -1; c_last_bg = 0; c_last_fg = 0; c_run = 0; }
    __syncthreads();

    CellRec *crow = cells + g.first_cell_rec();
    const bool upper = g.upper() != 0, color8 = g.color8() != 0;

    for (int c0 = 0; c0 < g.cols(); c0 += BT) {
        const int c = c0 + tid;
        const bool valid = c < g.cols();
        bool skipped = true;
        Pick pk; pk.fg = 0; pk.bg = 0; pk.block = kBackground;
        if (valid) {
            uint32_t t0 = 0, t1 = 0, b0 = 0, b1 = 0;
            bool same = prev != nullptr;
            if (g.quarter()) {
                if (top_ok) { const uint2 v = *reinterpret_cast<const uint2 *>(trow + 2 * c); t0 = v.x; t1 = v.y; }
                if (bot_ok) { const uint2 v = *reinterpret_cast<const uint2 *>(brow + 2 * c); b0 = v.x; b1 = v.y; }
                if (prev) {
                    uint32_t q0 = 0, q1 = 0, q2 = 0, q3 = 0;
                    if (top_ok) { const uint2 v = *reinterpret_cast<const uint2 *>(ptrow + 2 * c); q0 = v.x; q1 = v.y; }
                    if (bot_ok) { const uint2 v = *reinterpret_cast<const uint2 *>(pbrow + 2 * c); q2 = v.x; q3 = v.y; }
                    same = (t0 == q0) && (t1 == q1) && (b0 == q2) && (b1 == q3);
                }
                if (!same) pk = pick_quarter(t0, t1, b0, b1, upper);
            } else {
                if (top_ok) t0 = trow[c];
                if (bot_ok) b0 = brow[c];
                if (prev) {
                    const uint32_t q0 = top_ok ? ptrow[c] : 0u, q2 = bot_ok ? pbrow[c] : 0u;
                    same = (t0 == q0) && (b0 == q2);
                }
                if (!same) pk = pick_half(t0, b0, upper);
            }
            skipped = same;
        }
        s_fg[tid] = pk.fg; s_bg[tid] = pk.bg;
        int ka = skipped ? -1 : tid;
        int kb = (!skipped && pk.block != kBackground) ? tid : -1;
        const int my_a = ka, my_b = kb;
        block_scan_max2(ka, kb, s_i);            // inclusive; syncs make s_fg/s_bg visible
        // exclusive = value at tid-1
        int pa = __shfl_up_sync(0xffffffffu, ka, 1), pb = __shfl_up_sync(0xffffffffu, kb, 1);
        if ((tid & 31) == 0) {
            // need the inclusive value of the previous warp's last lane: recompute from smem-free
            // path: inclusive(tid) with own key removed equals max over < tid
            pa = -1; pb = -1;
        }
        // For lane 0 of warps > 0 recover via a second tiny exchange through shared memory.
        __shared__ int s_la[8], s_lb[8];
        if ((tid & 31) == 31) { s_la[tid >> 5] = ka; s_lb[tid >> 5] = kb; }
        __syncthreads();
        if ((tid & 31) == 0 && tid > 0) { pa = s_la[(tid >> 5) - 1]; pb = s_lb[(tid >> 5) - 1]; }
        (void)my_a; (void)my_b;

        uint32_t len = 0, meta = M_SKIPPED;
        if (!skipped) {
            const bool have_emit = (pa >= 0) || (c_last_emit >= 0);
            const int prev_idx = (pa >= 0) ? (c0 + pa) : c_last_emit;
            const uint32_t prev_bg = (pa >= 0) ? s_bg[pa] : c_last_bg;
            const bool have_fg = (pb >= 0) || (c_last_fgidx >= 0);
            const uint32_t prev_fg = (pb >= 0) ? s_fg[pb] : c_last_fg;
            const bool emit_fg = (pk.block != kBackground) && (!have_fg || pk.fg != prev_fg);   // :270-279
            const bool emit_bg = !have_emit || pk.bg != prev_bg;                                // :282-297
            const bool bgt = transparent(pk.bg);
            const uint32_t xskip = have_emit ? (uint32_t)(c - prev_idx - 1) : (uint32_t)(c + g.indent());
            len = (xskip > 0 ? 3 + ndig(xskip) : 0)
                + ((emit_fg || emit_bg) ? 2 : 0)
                + (emit_fg ? 5 + color_len(pk.fg, color8) : 0)
                + (emit_bg ? (bgt ? 3 : 5 + color_len(pk.bg, color8)) : 0)
                + (pk.block == kBackground ? 1 : 3);
            meta = pk.block | (emit_fg ? M_EMIT_FG : 0) | (emit_bg ? M_EMIT_BG : 0)
                 | (bgt ? M_BG_TRANSP : 0) | (have_emit ? 0 : M_FIRST) | (xskip << M_XSKIP_SHIFT);
        }
        uint32_t total;
        const uint32_t incl = block_scan_add(len, s_u, total);
        if (valid) {
            CellRec rec; rec.fg = pk.fg; rec.bg = pk.bg; rec.meta = meta; rec.off = c_run + incl - len;
            crow[c] = rec;
        }
        __syncthreads();                          // everyone has read the carries
        if (tid == BT - 1) {                      // ka/kb of the last thread = chunk maxima
            if (ka >= 0) { c_last_emit = c0 + ka; c_last_bg = s_bg[ka]; }
            if (kb >= 0) { c_last_fgidx = c0 + kb; c_last_fg = s_fg[kb]; }
            c_run += total;
        }
        __syncthreads();
    }
    if (tid == 0) {
        RowRec rr; rr.nonempty = c_last_emit >= 0 ? 1u : 0u;
        rr.len = rr.nonempty ? c_run + 5 : 0;     // + "\033[0m\n" (:313-318)
        rr.off = 0; rr.yskip = 0;
        rows[g.first_row_rec() + r] = rr;
    }
}


template <class G>
__device__ __forceinline__ void blocks_rowscan(const G &g, RowRec *__restrict__ rows, FrameRec *__restrict__ frames) {
    __shared__ int s_i[16];
    __shared__ uint32_t s_u[8];
    __shared__ int s_l[8];
    __shared__ int c_last; __shared__ uint32_t c_run;
    const int f = g.f, tid = threadIdx.x;
    RowRec *rr = rows + g.first_row_rec();
    if (tid == 0) { c_last = -1; c_run = 0; }
    __syncthreads();
    for (int r0 = 0; r0 < g.rows(); r0 += BT) {
        const int r = r0 + tid;
        const bool valid = r < g.rows();
        RowRec me; me.len = 0; me.nonempty = 0; me.off = 0; me.yskip = 0;
        if (valid) me = rr[r];
        int k = me.nonempty ? tid : -1, dummy = -1;
        block_scan_max2(k, dummy, s_i);
        int pk = __shfl_up_sync(0xffffffffu, k, 1);
        if ((tid & 31) == 31) s_l[tid >> 5] = k;
        __syncthreads();
        if ((tid & 31) == 0) pk = tid > 0 ? s_l[(tid >> 5) - 1] : -1;
        uint32_t tot = 0, ys = 0;
        if (me.nonempty) {
            const int prev_row = pk >= 0 ? r0 + pk : c_last;
            ys = (uint32_t)(r - prev_row - 1);
            tot = yskip_len(ys) + me.len;
        }
        uint32_t total;
        const uint32_t incl = block_scan_add(tot, s_u, total);
        if (valid) { me.off = c_run + incl - tot; me.yskip = ys; rr[r] = me; }
        __syncthreads();
        if (tid == BT - 1) { if (k >= 0) c_last = r0 + k; c_run += total; }
        __syncthreads();
    }
    if (tid == 0) {
        FrameRec fr; fr.pad0 = fr.pad1 = 0;
        if (c_last < 0) { fr.size = 0; fr.trailing = 0; }                 // :390-395
        else {
            fr.trailing = (uint32_t)(g.rows() - 1 - c_last);
            fr.size = c_run + (fr.trailing ? 3 + ndig(fr.trailing) : 0);  // :397-399
        }
        if (g.prev_mode() == 3 && f == 0) { fr.size = 0; fr.trailing = 0; }   // halo frame of a sharded animation: reference only
        frames[f] = fr;
    }
}

__global__ void __launch_bounds__(BT)
blocks_rowscan_kernel(BlocksParams P, RowRec *__restrict__ rows, FrameRec *__restrict__ frames) {
    blocks_rowscan(UniformGeom(P, blockIdx.x, 0), rows, frames);
}

// Exclusive scan of a strided uint32 "size" field into uint64 offsets[n+1]; one block.
__global__ void __launch_bounds__(1024)
sizes_to_offsets_kernel(const uint32_t *__restrict__ sizes, int stride_words, int n,
                        uint64_t *__restrict__ offsets) {
    __shared__ unsigned long long s_w[32];
    __shared__ unsigned long long c_run;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) c_run = 0;
    __syncthreads();
    for (int i0 = 0; i0 < n; i0 += 1024) {
        const int i = i0 + tid;
        unsigned long long v = i < n ? sizes[(long long)i * stride_words] : 0ull;
        const unsigned long long mine = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long o = __shfl_up_sync(0xffffffffu, v, d);
            if (lane >= d) v += o;
        }
        if (lane == 31) s_w[wid] = v;
        __syncthreads();
        unsigned long long pre = 0, tot = 0;
        for (int k = 0; k < 32; ++k) { if (k < wid) pre += s_w[k]; tot += s_w[k]; }
        if (i < n) offsets[i] = c_run + pre + v - mine;
        __syncthreads();
        if (tid == 0) c_run += tot;
        __syncthreads();
    }
    if (tid == 0) offsets[n] = c_run;
}

// ---- byte emission helpers
__device__ __forceinline__ char *put_num(char *o, uint32_t v) {
    char tmp[10]; int n = 0;
    do { tmp[n++] = (char)('0' + v % 10); v /= 10; } while (v);
    while (n) *o++ = tmp[--n];
    return o;
}
__device__ __forceinline__ char *put_u8s(char *o, uint32_t v) {   // "ddd;" (:474-491)
    if (v >= 100) { *o++ = (char)('0' + v / 100); v %= 100; *o++ = (char)('0' + v / 10); *o++ = (char)('0' + v % 10); }
    else if (v >= 10) { *o++ = (char)('0' + v / 10); *o++ = (char)('0' + v % 10); }
    else *o++ = (char)('0' + v);
    *o++ = ';';
    return o;
}
__device__ __forceinline__ char *put_color(char *o, uint32_t p, bool color8) {   // :113-122
    if (color8) return put_u8s(o, as256(p));
    o = put_u8s(o, p & 0xff); o = put_u8s(o, (p >> 8) & 0xff); return put_u8s(o, (p >> 16) & 0xff);
}

template <class G>
__device__ __forceinline__ void blocks_emit(const G &g, bool color8, const CellRec *__restrict__ cells,
                                            const RowRec *__restrict__ rows, const FrameRec *__restrict__ frames,
                                            const uint64_t *__restrict__ offsets, char *__restrict__ out,
                                            unsigned long long out_cap) {
    const int r = g.r, f = g.f, tid = threadIdx.x;
    const RowRec rr = rows[g.first_row_rec() + r];
    const FrameRec fr = frames[f];
    const unsigned long long fbase = offsets[f];
    if (fr.size == 0 || fbase + fr.size > out_cap) return; // nothing to write / never write out of bounds
    if (r == 0 && tid == 0 && fr.size && fr.trailing) {    // trailing cursor-down, :397-399
        char *o = out + fbase + fr.size - (3 + ndig(fr.trailing));
        *o++ = '\033'; *o++ = '['; o = put_num(o, fr.trailing); *o++ = 'B';
    }
    if (!rr.nonempty) return;
    char *rbase = out + fbase + rr.off;
    const uint32_t yb = yskip_len(rr.yskip);
    if (tid == 0) {                                        // end of line, :317
        char *o = rbase + yb + rr.len - 5;
        o[0] = '\033'; o[1] = '['; o[2] = '0'; o[3] = 'm'; o[4] = '\n';
    }
    const CellRec *crow = cells + g.first_cell_rec();
    for (int c = tid; c < g.cols(); c += BT) {
        const CellRec rec = crow[c];
        if (rec.meta & M_SKIPPED) continue;
        if (rec.meta & M_FIRST) {                          // pending y_skip, :249-258
            char *o = rbase;
            if (rr.yskip && rr.yskip <= 4) { for (uint32_t k = 0; k < rr.yskip; ++k) *o++ = '\n'; }
            else if (rr.yskip) { *o++ = '\033'; *o++ = '['; o = put_num(o, rr.yskip); *o++ = 'B'; }
        }
        char *o = rbase + yb + rec.off;
        const uint32_t xskip = rec.meta >> M_XSKIP_SHIFT;
        if (xskip) { *o++ = '\033'; *o++ = '['; o = put_num(o, xskip); *o++ = 'C'; }   // :260-263
        const bool efg = rec.meta & M_EMIT_FG, ebg = rec.meta & M_EMIT_BG;
        if (efg || ebg) { *o++ = '\033'; *o++ = '['; }
        if (efg) {
            *o++ = '3'; *o++ = '8'; *o++ = ';'; *o++ = color8 ? '5' : '2'; *o++ = ';';
            o = put_color(o, rec.fg, color8);
        }
        if (ebg) {
            if (rec.meta & M_BG_TRANSP) { *o++ = '4'; *o++ = '9'; *o++ = ';'; }
            else {
                *o++ = '4'; *o++ = '8'; *o++ = ';'; *o++ = color8 ? '5' : '2'; *o++ = ';';
                o = put_color(o, rec.bg, color8);
            }
        }
        if (efg || ebg) o[-1] = 'm';                       // :299-301
        const uint32_t blk = rec.meta & M_BLOCK_MASK;
        if (blk == kBackground) *o++ = ' ';
        else {
            // U+2598,259D,2596,2597,258C,259A,2584,2580 -> E2 96 xx (:78-88)
            const uint32_t last = (0x80849A8C97969D98ull >> (8 * (blk - 1))) & 0xff;
            *o++ = (char)0xE2; *o++ = (char)0x96; *o++ = (char)last;
        }
    }
}

__global__ void __launch_bounds__(BT)
blocks_emit_kernel(BlocksParams P, const CellRec *__restrict__ cells, const RowRec *__restrict__ rows,
                   const FrameRec *__restrict__ frames, const uint64_t *__restrict__ offsets,
                   char *__restrict__ out, unsigned long long out_cap) {
    blocks_emit(UniformGeom(P, blockIdx.y, blockIdx.x), P.color8 != 0, cells, rows, frames, offsets, out, out_cap);
}

// ---- mixed batches: one CTA per (frame, row pair) item of the flat list row_start describes (pick, emit), one per
// frame (rowscan); frame f's items are row_start[f] .. row_start[f + 1] - 1
__global__ void __launch_bounds__(BT)
blocks_rowscan_mixed_kernel(const MixedBlocksFrame *__restrict__ desc, const unsigned *__restrict__ row_start,
                            RowRec *__restrict__ rows, FrameRec *__restrict__ frames) {
    blocks_rowscan(MixedGeom(desc, row_start, blockIdx.x, 0), rows, frames);
}
__global__ void __launch_bounds__(BT)
blocks_emit_mixed_kernel(const MixedBlocksFrame *__restrict__ desc, const unsigned *__restrict__ row_start, int n_frames,
                         int flags, const CellRec *__restrict__ cells, const RowRec *__restrict__ rows,
                         const FrameRec *__restrict__ frames, const uint64_t *__restrict__ offsets,
                         char *__restrict__ out, unsigned long long out_cap) {
    const int f = mixed_owner(row_start, n_frames, blockIdx.x);
    blocks_emit(MixedGeom(desc, row_start, f, (int)(blockIdx.x - row_start[f])), (flags & B200TIMG_COLOR8) != 0, cells, rows,
                frames, offsets, out, out_cap);
}

int launch_blocks(b200timg_ctx *ctx, const uint8_t *d_fb, const uint8_t *d_prev, int prev_mode,
                  int w, int h, int n_frames, int flags, int x_indent, char *d_out,
                  size_t out_cap, uint64_t *d_offsets) {
    BlocksParams P;
    P.w = w; P.h = h; P.n_frames = n_frames;
    P.quarter = (flags & B200TIMG_QUARTER) ? 1 : 0;
    P.upper = (flags & B200TIMG_UPPER) ? 1 : 0;
    P.color8 = (flags & B200TIMG_COLOR8) ? 1 : 0;
    if (P.quarter && (w & 1))
        return ctx->fail(B200TIMG_EINVAL, "quarter blocks need an even width (got %d); the "
                         "reference reads past the row end there", w);
    P.cols = P.quarter ? w / 2 : w;
    P.rows = (h + 1) / 2;
    P.indent = x_indent;
    P.row_offset = ((h & 1) && !P.upper) ? -1 : 0;
    P.prev_mode = prev_mode;
    P.frame_px = (long long)w * h;
    if (P.rows > 65535 || n_frames > 65535)
        return ctx->fail(B200TIMG_EINVAL, "too many rows/frames for one launch");

    const size_t n_cells = (size_t)n_frames * P.rows * P.cols;
    const size_t n_rows = (size_t)n_frames * P.rows;
    B2_CUDA(ctx, ctx->cells.reserve(n_cells * sizeof(CellRec)));
    B2_CUDA(ctx, ctx->rows.reserve(n_rows * sizeof(RowRec) + (size_t)n_frames * sizeof(FrameRec) + 64));
    CellRec *cells = ctx->cells.as<CellRec>();
    RowRec *rows = ctx->rows.as<RowRec>();
    FrameRec *frames = reinterpret_cast<FrameRec *>(rows + n_rows);

    const dim3 grid(P.rows, n_frames);
    B2_KERNEL(ctx, "blocks_pick_kernel");
    blocks_pick_kernel<UniformGeom><<<grid, BT, 0, ctx->stream>>>(reinterpret_cast<const uint32_t *>(d_fb),
                                                     reinterpret_cast<const uint32_t *>(d_prev), P, cells, rows);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "blocks_rowscan_kernel");
    blocks_rowscan_kernel<<<n_frames, BT, 0, ctx->stream>>>(P, rows, frames);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "sizes_to_offsets_kernel");
    sizes_to_offsets_kernel<<<1, 1024, 0, ctx->stream>>>(reinterpret_cast<const uint32_t *>(frames),
                                                         sizeof(FrameRec) / 4, n_frames, d_offsets);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "blocks_emit_kernel");
    blocks_emit_kernel<<<grid, BT, 0, ctx->stream>>>(P, cells, rows, frames, d_offsets, d_out,
                                                     (unsigned long long)out_cap);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

// Block records of a mixed batch: frame f's scaled pixels follow the earlier frames' back to back (as
// launch_scale_mixed writes them), its row and cell records follow the earlier frames' likewise.
int plan_blocks_mixed(b200timg_ctx *ctx, const b200timg_mixed_batch *mb, MixedPlan &mp) {
    const int n = mb->n_frames;
    const bool quarter = (mb->flags & B200TIMG_QUARTER) != 0, upper = (mb->flags & B200TIMG_UPPER) != 0;
    std::vector<MixedBlocksFrame> desc(n);
    std::vector<unsigned> row_start(n + 1);
    unsigned long long px = 0, cells = 0, rows = 0;
    for (int f = 0; f < n; ++f) {
        const b200timg_frame &F = mb->frames[f];
        MixedBlocksFrame &D = desc[f];
        D.fb_px = px; D.cell0 = cells;
        D.w = F.out_w; D.h = F.out_h;
        D.cols = quarter ? F.out_w / 2 : F.out_w;
        D.rows = (F.out_h + 1) / 2;
        D.row_offset = ((F.out_h & 1) && !upper) ? -1 : 0;
        D.indent = F.x_indent_cells;
        row_start[f] = (unsigned)rows;
        px += (unsigned long long)F.out_w * F.out_h;
        cells += (unsigned long long)D.rows * D.cols;
        rows += (unsigned long long)D.rows;
        if (rows > 0x7fffffffull)
            return ctx->fail(B200TIMG_EINVAL, "mixed batch: more than 2^31 - 1 row pairs in one call (at frame %d)", f);
    }
    row_start[n] = (unsigned)rows;
    mp.o_blocks = mixed_put(mp.arena, desc.data(), sizeof(MixedBlocksFrame) * n);
    mp.o_rows = mixed_put(mp.arena, row_start.data(), sizeof(unsigned) * (n + 1));
    mp.rowpairs = (unsigned)rows; mp.cells = cells;
    return B200TIMG_OK;
}

int launch_blocks_mixed(b200timg_ctx *ctx, const MixedPlan &mp, const char *d_arena, const uint8_t *d_fb, int n_frames,
                        int flags, char *d_out, size_t out_cap, uint64_t *d_offsets) {
    B2_CUDA(ctx, ctx->cells.reserve((size_t)mp.cells * sizeof(CellRec)));
    B2_CUDA(ctx, ctx->rows.reserve((size_t)mp.rowpairs * sizeof(RowRec) + (size_t)n_frames * sizeof(FrameRec) + 64));
    CellRec *cells = ctx->cells.as<CellRec>();
    RowRec *rows = ctx->rows.as<RowRec>();
    FrameRec *frames = reinterpret_cast<FrameRec *>(rows + mp.rowpairs);
    const MixedBlocksFrame *desc = reinterpret_cast<const MixedBlocksFrame *>(d_arena + mp.o_blocks);
    const unsigned *row_start = reinterpret_cast<const unsigned *>(d_arena + mp.o_rows);
    const uint32_t *fb = reinterpret_cast<const uint32_t *>(d_fb);
    B2_KERNEL(ctx, "blocks_pick_mixed_kernel");
    blocks_pick_kernel<MixedGeom><<<mp.rowpairs, BT, 0, ctx->stream>>>(fb, nullptr, MixedBlocksParams{desc, row_start, n_frames, flags},
                                                                       cells, rows);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "blocks_rowscan_mixed_kernel");
    blocks_rowscan_mixed_kernel<<<n_frames, BT, 0, ctx->stream>>>(desc, row_start, rows, frames);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "sizes_to_offsets_kernel");
    sizes_to_offsets_kernel<<<1, 1024, 0, ctx->stream>>>(reinterpret_cast<const uint32_t *>(frames),
                                                         sizeof(FrameRec) / 4, n_frames, d_offsets);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "blocks_emit_mixed_kernel");
    blocks_emit_mixed_kernel<<<mp.rowpairs, BT, 0, ctx->stream>>>(desc, row_start, n_frames, flags, cells, rows, frames,
                                                                  d_offsets, d_out, (unsigned long long)out_cap);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

}  // namespace b200timg
