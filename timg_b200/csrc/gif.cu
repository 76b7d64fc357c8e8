// Animated GIFs on the device (SURVEY 8f rank 4): the canvases the STB source's GIF branch collects
// (src/stb-image-source.cc:120-140), frame k = the k-th return of stbi__gif_load_next(.., two_back = NULL)
// (third_party/stb/stb_image.h:6779-6951).
//   host walk           the block structure, palette state, delays and every error visible without decoding a raster
//                       (the walk ends each raster just after its terminator, as both of stb's raster exits do)
//   decode_gather_kernel (decode.cu) drops the sub-block length bytes: every frame's payload as one contiguous code
//                       stream
//   gif_lzw_kernel      one warp per frame: lane 0 walks the codes, the warp copies long strings; writes the frame's
//                       index plane in stream order up to the rectangle's area, then only validates (:6694-6776)
//   gif_compose_kernel  one thread per canvas pixel over the frames in order: dispose, overlay, first-frame background
//                       (:6808-6838, :6896-6904), interlaced rows through a rank table (:6680-6689)
// A call launches these three kernels whatever its frame count.
#include <algorithm>

#include "decode.cuh"

namespace b200timg {

namespace {

constexpr int GIF_DICT = 8192;                     // stb's codes[8192]: lzw_cs 12 gives 13-bit codes

struct __align__(16) GifFrame {
    unsigned long long plane;                      // first byte of the frame's index plane
    unsigned long long code0, code_len;            // its code stream in the gathered payload
    int rx, ry, rw, rh;                            // the rectangle
    int lzw_cs;
    int dispose2;                                  // before this frame: restore last frame's marked pixels (dispose 2, 3)
    int interlaced;
    unsigned rank0;                                // first entry of its row -> stream rank table (interlaced frames)
    int bg_alt;                                    // entry bgindex's alpha if frame 0 left a pixel unmarked, else -1
    int pad_[3];
};

// ---- host: stbi__gif_load_next's walk ------------------------------------------------------------------------
struct Reader {                                    // stbi__get8 / get16le / skip: bytes past the end read as 0
    const uint8_t *p;
    size_t n, pos = 0;
    int get8() { const int v = pos < n ? p[pos] : 0; ++pos; return v; }
    int get16() { const int a = get8(); return a | (get8() << 8); }
    void skip(size_t k) { pos += k; }
};

struct WalkFrame {
    int rx, ry, rw, rh, lzw_cs, dispose2, interlaced, bg_alt;
    uint32_t pal[256];                             // the colour table at raster time, RGBA (out's byte order)
    size_t sb0, sb1;                               // its sub-blocks [sb0, sb1) in Walk::sb_off / sb_len
    int delay;
};

struct Walk {
    int w = 0, h = 0, bgindex = 0;
    uint32_t bgpix = 0;                            // what the first-frame rule writes: pal[bgindex] bytes, alpha 255
    std::vector<WalkFrame> frames;
    std::vector<unsigned long long> sb_off;        // file offset of each sub-block's data
    std::vector<int> sb_len;
};

inline uint32_t pal_rgba(const uint8_t e[4]) {     // stb keeps {b, g, r, a}; out_gif_code writes r, g, b, a
    return (uint32_t)e[2] | ((uint32_t)e[1] << 8) | ((uint32_t)e[0] << 16) | ((uint32_t)e[3] << 24);
}

// false: not GIF87a / GIF89a.  Stops at the terminator or at the first error the walk can see.
bool gif_walk(const uint8_t *gif, size_t size, Walk &wk) {
    Reader s{gif, size};
    if (s.get8() != 'G' || s.get8() != 'I' || s.get8() != 'F' || s.get8() != '8') return false;
    const int version = s.get8();
    if (version != '7' && version != '9') return false;
    if (s.get8() != 'a') return false;
    uint8_t pal[256][4] = {}, lpal[256][4] = {};   // g is memset to 0 by the caller (stb-image-source.cc:122)
    wk.w = s.get16(); wk.h = s.get16();
    const int flags = s.get8();
    wk.bgindex = s.get8();
    s.get8();                                      // ratio
    int transparent = -1, eflags = 0, delay = 0;
    auto parse_table = [&](uint8_t (*t)[4], int num, int transp) {
        for (int i = 0; i < num; ++i) {
            t[i][2] = (uint8_t)s.get8(); t[i][1] = (uint8_t)s.get8(); t[i][0] = (uint8_t)s.get8();
            t[i][3] = transp == i ? 0 : 255;
        }
    };
    if (flags & 0x80) parse_table(pal, 2 << (flags & 7), -1);
    // Alpha of pal[bgindex] had frame 0 left a pixel unmarked (the first-frame rule sets it to 255, :6900); only the
    // device knows whether it did, so both versions are carried.
    int alt_a = -1;
    for (;;) {
        const int dispose = (eflags & 0x1C) >> 2;  // the previous frame's disposal, applied before this one
        WalkFrame fr{};
        fr.dispose2 = wk.frames.empty() ? 0 : (dispose == 2 || dispose == 3);
        bool got = false;
        while (!got) {
            const int tag = s.get8();
            if (tag == 0x2C) {
                const int x = s.get16(), y = s.get16(), w = s.get16(), h = s.get16();
                if (x + w > wk.w || y + h > wk.h) return true;                 // bad Image Descriptor
                const int lflags = s.get8();
                fr.rx = x; fr.ry = y; fr.rw = w; fr.rh = h;
                fr.interlaced = (lflags & 0x40) ? 1 : 0;
                const uint8_t (*table)[4];
                bool global = false;
                if (lflags & 0x80) {
                    parse_table(lpal, 2 << (lflags & 7), (eflags & 1) ? transparent : -1);
                    table = lpal;
                } else if (flags & 0x80) {
                    table = pal; global = true;
                } else return true;                                           // missing color table
                const int lzw_cs = s.get8();
                if (lzw_cs > 12) return true;
                fr.lzw_cs = lzw_cs;
                for (int i = 0; i < 256; ++i) fr.pal[i] = pal_rgba(table[i]);
                fr.bg_alt = (global && alt_a >= 0 && wk.bgindex > 0) ? alt_a : -1;
                fr.sb0 = wk.sb_off.size();
                for (int len; (len = s.get8()) != 0;) { wk.sb_off.push_back(s.pos); wk.sb_len.push_back(len); s.skip(len); }
                fr.sb1 = wk.sb_off.size();
                got = true;
            } else if (tag == 0x21) {
                const int ext = s.get8();
                if (ext == 0xF9) {                                             // Graphic Control Extension
                    const int len = s.get8();
                    if (len == 4) {
                        eflags = s.get8();
                        delay = 10 * s.get16();
                        if (transparent >= 0) { pal[transparent][3] = 255; if (transparent == wk.bgindex && alt_a >= 0) alt_a = 255; }
                        if (eflags & 1) {
                            transparent = s.get8();
                            pal[transparent][3] = 0;
                            if (transparent == wk.bgindex && alt_a >= 0) alt_a = 0;
                        } else { s.skip(1); transparent = -1; }
                    } else { s.skip(len); continue; }                          // its terminator is read as the next tag
                }
                for (int len; (len = s.get8()) != 0;) s.skip(len);
            } else if (tag == 0x3B) {
                return true;
            } else return true;                                               // unknown code
        }
        fr.delay = delay;
        if (wk.frames.empty()) {
            wk.bgpix = (uint32_t)pal[wk.bgindex][0] | ((uint32_t)pal[wk.bgindex][1] << 8) |
                       ((uint32_t)pal[wk.bgindex][2] << 16) | 0xff000000u;   // memcpy of {b, g, r, a}: stored as is
            alt_a = 255;
        }
        wk.frames.push_back(fr);
    }
}

int walk_or_fail(b200timg_ctx *ctx, const uint8_t *gif, size_t size, Walk &wk) {
    if (!gif || size == 0) return ctx ? ctx->fail(B200TIMG_EINVAL, "gif: no data") : B200TIMG_EINVAL;
    if (!gif_walk(gif, size, wk)) return ctx ? ctx->fail(B200TIMG_EINVAL, "gif: not a GIF") : B200TIMG_EINVAL;
    if (wk.w <= 0 || wk.h <= 0) return ctx ? ctx->fail(B200TIMG_EINVAL, "gif: zero-sized screen %dx%d", wk.w, wk.h) : B200TIMG_EINVAL;
    if (wk.frames.empty()) return ctx ? ctx->fail(B200TIMG_EINVAL, "gif: no frame") : B200TIMG_EINVAL;
    return B200TIMG_OK;
}

// ---- kernels ---------------------------------------------------------------------------------------------------
// stbi__process_gif_raster with the dictionary as (start, len) into the frame's own index stream: an entry is always
// the previous code's output plus the first byte of the current one, so no prefix chain is ever followed.
constexpr int GIF_SHORT = 16;                      // strings up to this long are written by lane 0 alone
__global__ void __launch_bounds__(32)
gif_lzw_kernel(const GifFrame *__restrict__ desc, const uint8_t *__restrict__ payload, uint8_t *__restrict__ planes,
               unsigned long long *__restrict__ reach, int32_t *__restrict__ valid) {
    __shared__ uint32_t e_start[GIF_DICT];
    __shared__ uint16_t e_len[GIF_DICT];
    const int f = blockIdx.x, lane = threadIdx.x;
    const GifFrame d = desc[f];
    const uint8_t *in = payload + d.code0;
    uint8_t *out = planes + d.plane;
    const unsigned long long area = (unsigned long long)d.rw * d.rh;
    const int lzw_cs = d.lzw_cs, clear = 1 << lzw_cs;
    // lane 0's walk
    unsigned long long pos = 0, byte = 0, buf = 0;
    int nb = 0, codesize = lzw_cs + 1, codemask = (1 << codesize) - 1, avail = clear + 2, oldcode = -1, first = 1, err = 0;
    unsigned long long old_start = 0;
    int old_len = 0;
    bool done = false;
    for (;;) {
        unsigned long long c_src = 0, c_dst = 0;
        int c_len = 0;
        if (lane == 0) {
            while (!done) {
                if (nb < codesize) {
                    if (byte >= d.code_len) { done = true; break; }           // the zero-length sub-block
                    buf |= (unsigned long long)in[byte++] << nb;
                    nb += 8;
                    continue;
                }
                const int code = (int)(buf & (unsigned)codemask);
                buf >>= codesize; nb -= codesize;
                if (code == clear) {
                    codesize = lzw_cs + 1; codemask = (1 << codesize) - 1; avail = clear + 2; oldcode = -1; first = 0;
                    continue;
                }
                if (code == clear + 1) { done = true; break; }                 // end of information
                if (code > avail || first) { err = 1; done = true; break; }   // illegal code / no clear code
                if (oldcode >= 0) {
                    if (avail + 1 > GIF_DICT) { err = 1; done = true; break; } // too many codes
                    e_start[avail] = (uint32_t)min(old_start, 0xffffffffull);
                    e_len[avail] = (uint16_t)(old_len + 1);
                    ++avail;
                } else if (code == avail) { err = 1; done = true; break; }
                int len;
                unsigned long long src = 0;
                if (code < clear) {
                    len = 1;
                    if (pos < area) out[pos] = (uint8_t)code;
                } else {
                    src = e_start[code]; len = e_len[code];
                    if (pos < area) {
                        if (len > GIF_SHORT) { c_src = src; c_dst = pos; c_len = len; }
                        else {
                            // src + (i mod (pos - src)): a string that runs into its own output (code == avail)
                            // repeats with the previous string's period
                            const unsigned long long per = pos - src;
                            for (int i = 0; i < len && pos + i < area; ++i) out[pos + i] = out[src + (i % per)];
                        }
                    }
                }
                if ((avail & codemask) == 0 && avail <= 0x0FFF) { ++codesize; codemask = (1 << codesize) - 1; }
                oldcode = code; old_start = pos; old_len = len;
                pos += len;
                if (c_len) break;
            }
        }
        c_len = __shfl_sync(0xffffffffu, c_len, 0);
        const int stop = __shfl_sync(0xffffffffu, done ? 1 : 0, 0);
        if (c_len) {
            c_src = __shfl_sync(0xffffffffu, c_src, 0);
            c_dst = __shfl_sync(0xffffffffu, c_dst, 0);
            __syncwarp();                           // lane 0's writes are visible to the warp
            const unsigned long long per = c_dst - c_src;
            for (int i = lane; i < c_len && c_dst + i < area; i += 32) out[c_dst + i] = out[c_src + (i % per)];
            __syncwarp();
        }
        if (stop) break;
    }
    if (lane == 0) {
        reach[f] = min(pos, area);
        if (err) atomicMin(valid, f);
    }
}

// Every canvas pixel through all frames: out, background and history stay in registers.
__global__ void __launch_bounds__(256)
gif_compose_kernel(const GifFrame *__restrict__ desc, const uint32_t *__restrict__ pal, const uint32_t *__restrict__ rank,
                   const uint8_t *__restrict__ planes, const unsigned long long *__restrict__ reach, uint32_t *__restrict__ out,
                   int w, int h, int n_frames, int bgindex, uint32_t bgpix) {
    const long long npx = (long long)w * h;
    const bool unmarked0 = reach[0] < (unsigned long long)npx;   // frame 0 left a pixel unmarked (:6896-6904)
    for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < npx; g += (long long)gridDim.x * blockDim.x) {
        const int y = (int)(g / w), x = (int)(g - (long long)y * w);
        uint32_t o = 0, bk = 0;
        bool hist = false;
        for (int f = 0; f < n_frames; ++f) {
            const GifFrame &d = desc[f];
            if (f > 0) {
                if (d.dispose2 && hist) o = bk;
                bk = o;
            }
            hist = false;
            const int xr = x - d.rx, yr = y - d.ry;
            if (xr >= 0 && xr < d.rw && yr >= 0 && yr < d.rh) {
                const unsigned long long r = d.interlaced ? rank[d.rank0 + yr] : (unsigned)yr;
                const unsigned long long p = r * (unsigned)d.rw + xr;
                if (p < reach[f]) {
                    hist = true;
                    const int idx = planes[d.plane + p];
                    uint32_t c = pal[(size_t)f * 256 + idx];
                    if (d.bg_alt >= 0 && unmarked0 && idx == bgindex) c = (c & 0xffffffu) | ((uint32_t)d.bg_alt << 24);
                    if ((c >> 24) > 128) o = c;
                }
            }
            if (f == 0 && bgindex > 0 && !hist) o = bgpix;
            out[(size_t)f * npx + g] = o;
        }
    }
}

// Device scratch of one call (ctx->gif_up.arena + ctx->gif_scratch):
//   file + 80 n (descriptors) + 1024 n (palettes) + 4 sum(interlaced rh) + 16 S (S sub-blocks) + P (code streams)
//   + sum(rw * rh) (index planes) + 8 n (reach), each part 16-byte aligned.
int launch_gif(b200timg_ctx *ctx, const uint8_t *gif, size_t size, const Walk &wk, int n, uint8_t *d_frames, int32_t *d_valid) {
    std::vector<GifFrame> desc((size_t)n);
    std::vector<uint32_t> pal((size_t)n * 256), rank;
    Runs runs;                                     // the sub-blocks of frames 0..n-1
    unsigned long long plane = 0;
    for (int f = 0; f < n; ++f) {
        const WalkFrame &w = wk.frames[(size_t)f];
        GifFrame &d = desc[(size_t)f];
        memset(&d, 0, sizeof d);
        d.rx = w.rx; d.ry = w.ry; d.rw = w.rw; d.rh = w.rh; d.lzw_cs = w.lzw_cs; d.dispose2 = w.dispose2;
        d.interlaced = w.interlaced; d.bg_alt = w.bg_alt;
        d.plane = plane; plane += (unsigned long long)w.rw * w.rh;
        d.code0 = runs.total();
        for (size_t s = w.sb0; s < w.sb1; ++s) runs.add(wk.sb_off[s], (unsigned)wk.sb_len[s]);
        d.code_len = runs.total() - d.code0;
        memcpy(&pal[(size_t)f * 256], w.pal, sizeof w.pal);
        d.rank0 = (unsigned)rank.size();
        if (w.interlaced) {                        // stb's pass loop (:6680-6689) at row granularity
            const size_t r0 = rank.size();
            rank.resize(r0 + (size_t)w.rh);
            int cur = 0, step = 8, parse = 3;
            for (int k = 0; k < w.rh; ++k) {
                rank[r0 + (size_t)cur] = (uint32_t)k;
                cur += step;
                while (cur >= w.rh && parse > 0) { step = 1 << parse; cur = step >> 1; --parse; }
            }
        }
    }
    const unsigned long long paylen = runs.total();
    std::vector<char> arena;
    const int32_t n32 = n;
    const size_t o_n = mixed_put(arena, &n32, sizeof n32);
    const size_t o_desc = mixed_put(arena, desc.data(), sizeof(GifFrame) * desc.size());
    const size_t o_pal = mixed_put(arena, pal.data(), sizeof(uint32_t) * pal.size());
    const size_t o_rank = mixed_put(arena, rank.data(), sizeof(uint32_t) * rank.size());
    runs.put(arena);
    size_t o_file;
    B2_TRY(staged_upload(ctx, ctx->gif_up, arena, 1, &gif, &size, &o_file));
    const size_t s_pay = 0, s_plane = (paylen + 15) / 16 * 16, s_reach = s_plane + (plane + 15) / 16 * 16;
    B2_CUDA(ctx, ctx->gif_scratch.reserve(s_reach + sizeof(unsigned long long) * (size_t)n));
    const char *A = ctx->gif_up.arena.as<char>();
    char *S = ctx->gif_scratch.as<char>();
    const GifFrame *d_desc = reinterpret_cast<const GifFrame *>(A + o_desc);
    unsigned long long *d_reach = reinterpret_cast<unsigned long long *>(S + s_reach);
    B2_CUDA(ctx, cudaMemcpyAsync(d_valid, A + o_n, sizeof(int32_t), cudaMemcpyDeviceToDevice, ctx->stream));

    B2_TRY(launch_gather(ctx, runs, A, o_file, size, reinterpret_cast<uint8_t *>(S + s_pay)));
    B2_KERNEL(ctx, "gif_lzw_kernel");
    gif_lzw_kernel<<<n, 32, 0, ctx->stream>>>(d_desc, reinterpret_cast<const uint8_t *>(S + s_pay),
                                              reinterpret_cast<uint8_t *>(S + s_plane), d_reach, d_valid);
    B2_LAUNCH_CHECK(ctx);
    B2_KERNEL(ctx, "gif_compose_kernel");
    gif_compose_kernel<<<grid_for(ctx, (long long)wk.w * wk.h), 256, 0, ctx->stream>>>(
        d_desc, reinterpret_cast<const uint32_t *>(A + o_pal), reinterpret_cast<const uint32_t *>(A + o_rank),
        reinterpret_cast<const uint8_t *>(S + s_plane), d_reach, reinterpret_cast<uint32_t *>(d_frames), wk.w, wk.h, n,
        wk.bgindex, wk.bgpix);
    B2_LAUNCH_CHECK(ctx);
    return B200TIMG_OK;
}

int gif_frames_args(b200timg_ctx *ctx, const uint8_t *gif, size_t size, int n_frames, const void *a, const void *b, Walk &wk) {
    if (!a || !b) return ctx->fail(B200TIMG_EINVAL, "gif: null output");
    B2_TRY(walk_or_fail(ctx, gif, size, wk));
    if (n_frames < 1 || n_frames > (int)wk.frames.size())
        return ctx->fail(B200TIMG_EINVAL, "gif: n_frames %d outside 1..%d", n_frames, (int)wk.frames.size());
    return B200TIMG_OK;
}

}  // namespace

}  // namespace b200timg

using namespace b200timg;

extern "C" {

int b200timg_gif_parse(const uint8_t *gif, size_t size, int *w, int *h, int *n_frames, int32_t *delays_ms, int delays_cap) {
    if (!w || !h || !n_frames) return B200TIMG_EINVAL;
    Walk wk;
    B2_TRY(walk_or_fail(nullptr, gif, size, wk));
    *w = wk.w; *h = wk.h; *n_frames = (int)wk.frames.size();
    if (delays_ms)
        for (int k = 0; k < delays_cap && k < (int)wk.frames.size(); ++k) delays_ms[k] = wk.frames[(size_t)k].delay;
    return B200TIMG_OK;
}

int b200timg_gif_frames_dev(b200timg_ctx *ctx, const uint8_t *gif, size_t size, int n_frames, uint8_t *d_frames, int32_t *d_valid) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    Walk wk;
    B2_TRY(gif_frames_args(ctx, gif, size, n_frames, d_frames, d_valid, wk));
    B2_TRY(check_dev_outputs(ctx, "gif", d_frames, d_valid, "d_valid"));
    return launch_gif(ctx, gif, size, wk, n_frames, d_frames, d_valid);
}

int b200timg_gif_frames(b200timg_ctx *ctx, const uint8_t *gif, size_t size, int n_frames, uint8_t *frames, int *n_valid) {
    if (!ctx) return B200TIMG_EINVAL;
    B2_CUDA(ctx, cudaSetDevice(ctx->device));
    Walk wk;
    B2_TRY(gif_frames_args(ctx, gif, size, n_frames, frames, n_valid, wk));
    return decode_to_host(ctx, (size_t)wk.w * wk.h * 4 * (size_t)n_frames, 1, frames, n_valid,
                          [&](uint8_t *d_frames, int32_t *d_valid) { return launch_gif(ctx, gif, size, wk, n_frames, d_frames, d_valid); });
}

}  // extern "C"
