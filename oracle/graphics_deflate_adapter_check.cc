// TEST INFRASTRUCTURE.  The kitty / iTerm2 adapters with deflate = true (B200TIMG_DEFLATE, timg's --compress > 0)
// through the C++ drop-in: links the reference's own KittyGraphicsCanvas / ITerm2GraphicsCanvas, compiled by
// oracle/graphics_deflate.mk with oracle/deflate_replay/libdeflate.h in place of libdeflate, B200KittyCanvas /
// B200ITerm2Canvas (timg_b200/csrc/adapters.h) and libb200timg.so into one binary.  Each adapter runs first; the zlib
// stream of every PNG it wrote is taken from its output and handed to the reference canvas' png::Encode, which then
// runs over the same frames and, as it may encode on its pool's threads in any order, gets each frame's stream by
// that frame's filtered scanlines.  The bytes that reach the two file descriptors must be identical: PNG chunks
// and CRCs, base64, chunking, headers, cursor moves and (tmux form) the passthrough wrappers and placeholder grid.
//
// This binary defines time() (pinned, so both sides' CreateId give the same image ids), system() (returns 0, runs no
// shell: the tmux form's constructor calls it) and oracle_replay_stream() (the stream of the frame whose scanlines
// are being encoded).
// Needs a GPU.
#include <fcntl.h>
#include <sys/mman.h>
#include <unistd.h>

#include <csignal>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <atomic>
#include <string>
#include <vector>

#include "adapters.h"
#include "iterm2-canvas.h"
#include "kitty-canvas.h"
#include "thread-pool.h"

using namespace timg;

static constexpr time_t kPinnedTime = (200 << 17) | 0x123;      // ids 0xC8009180 + k: msb 200, 10 digits
struct Replay { std::string raw, stream; };                   // a frame's filtered scanlines and our zlib stream of them
static std::vector<Replay> g_replay;
static std::atomic<int> g_served{0};

extern "C" time_t time(time_t *t) {
    if (t) *t = kPinnedTime;
    return kPinnedTime;
}
extern "C" int system(const char *command) { return command ? 0 : 1; }
extern "C" const uint8_t *oracle_replay_stream(const void *in, size_t in_nbytes, size_t *n) {
    for (const Replay &r : g_replay)
        if (r.raw.size() == in_nbytes && memcmp(r.raw.data(), in, in_nbytes) == 0) {
            ++g_served;
            *n = r.stream.size();
            return (const uint8_t *)r.stream.data();
        }
    fprintf(stderr, "no stream for these scanlines\n");
    abort();
}

static volatile sig_atomic_t g_no_interrupt = 0;

static uint32_t mix(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
    return x;
}
// smooth gradients with a little noise and a few flat bars: compressible, so the PNGs carry dynamic-Huffman blocks
static void fill(Framebuffer *fb, uint32_t seed) {
    const int w = fb->width();
    int i = 0;
    for (rgba_t *p = fb->begin(); p != fb->end(); ++p, ++i) {
        const int x = i % w, y = i / w;
        const uint32_t v = mix(seed * 0x9e3779b1U + (uint32_t)i);
        const bool bar = (x / 16 + y / 16 + (int)seed) % 5 == 0;
        p->r = bar ? 200 : (uint8_t)(x + (v & 3));
        p->g = bar ? 40 : (uint8_t)(y * 2 + (v >> 8 & 3));
        p->b = bar ? 90 : (uint8_t)(x + y + seed);
        p->a = bar ? 255 : (uint8_t)(160 + (v >> 16 & 63));
    }
}
static std::string slurp(int fd) {
    const off_t n = lseek(fd, 0, SEEK_END);
    std::string s((size_t)n, '\0');
    if (n && pread(fd, &s[0], n, 0) != n) abort();
    return s;
}

// cursor off, an animation (StartOfAnimation, then AnimationFrame with dy = -previous height), cursor on
template <class Canvas, class... Args>
static std::string run_canvas(const std::vector<Framebuffer *> &frames, int x, Args... args) {
    const int fd = memfd_create("canvas_out", 0);
    {
        BufferedWriteSequencer seq(fd, false, 4, true, g_no_interrupt);
        {
            Canvas canvas(&seq, args...);
            canvas.CursorOff();
            int last_h = 0;
            for (size_t i = 0; i < frames.size(); ++i) {
                canvas.Send(x, i == 0 ? 0 : -last_h, *frames[i], i == 0 ? SeqType::StartOfAnimation : SeqType::AnimationFrame,
                            Duration::Millis(10));
                last_h = frames[i]->height();
            }
            canvas.CursorOn();
        }
        seq.Flush();
    }
    std::string s = slurp(fd);
    close(fd);
    return s;
}

static std::string unbase64(const std::string &s) {
    std::string out;
    uint32_t acc = 0;
    int bits = 0;
    for (char c : s) {
        int v = c >= 'A' && c <= 'Z' ? c - 'A' : c >= 'a' && c <= 'z' ? c - 'a' + 26 : c >= '0' && c <= '9' ? c - '0' + 52
              : c == '+' ? 62 : c == '/' ? 63 : -1;
        if (v < 0) continue;                                        // '=' padding
        acc = acc << 6 | (uint32_t)v;
        bits += 6;
        if (bits >= 8) { bits -= 8; out += (char)(acc >> bits & 255); }
    }
    return out;
}

// The PNGs of a canvas' output, in order: kitty's "_G...m=<0|1>;<base64>" commands (either form; m=0 ends a PNG),
// iTerm2's "File=...:<base64>\a".
static std::vector<std::string> pngs_of(const std::string &text) {
    std::vector<std::string> out;
    std::string b64;
    for (size_t pos = 0; pos < text.size(); ++pos) {
        if (text.compare(pos, 2, "_G") == 0) {
            const size_t semi = text.find(';', pos), m = text.find("m=", pos);
            const size_t end = text.find('\033', semi);
            b64 += text.substr(semi + 1, end - semi - 1);
            if (text[m + 2] == '0') { out.push_back(unbase64(b64)); b64.clear(); }
            pos = end;
        } else if (text.compare(pos, 5, "File=") == 0) {
            const size_t colon = text.find(':', pos), end = text.find('\a', colon);
            out.push_back(unbase64(text.substr(colon + 1, end - colon - 1)));
            pos = end;
        }
    }
    return out;
}

// the Sub-filtered scanlines png::Encode compresses (src/timg-png.cc:119-134)
static std::string scanlines(const Framebuffer &fb, bool rgb24) {
    const int bpp = rgb24 ? 3 : 4;
    std::string out;
    for (int y = 0; y < fb.height(); ++y) {
        const rgba_t *row = fb.begin() + (size_t)y * fb.width();
        out += (char)1;
        for (int x = 0; x < fb.width(); ++x) {
            const uint8_t c[4] = {row[x].r, row[x].g, row[x].b, row[x].a};
            const uint8_t p[4] = {x ? row[x - 1].r : (uint8_t)0, x ? row[x - 1].g : (uint8_t)0, x ? row[x - 1].b : (uint8_t)0,
                                  x ? row[x - 1].a : (uint8_t)0};
            for (int k = 0; k < bpp; ++k) out += (char)(uint8_t)(c[k] - p[k]);
        }
    }
    return out;
}

// the IDAT data (the zlib stream) of a PNG of this library: one IDAT right after IHDR
static std::string zlib_of(const std::string &png) {
    const uint8_t *p = (const uint8_t *)png.data();
    const size_t n = (size_t)p[33] << 24 | (size_t)p[34] << 16 | (size_t)p[35] << 8 | p[36];
    return png.substr(41, n);
}

int main() {
    int failures = 0;
    ThreadPool pool(2);
    for (int rgb24 = 0; rgb24 < 2; ++rgb24) {
        DisplayOptions opts;
        opts.cell_x_px = 9; opts.cell_y_px = 18;
        opts.local_alpha_handling = rgb24 != 0;
        opts.compress_pixel_level = 1;
        std::vector<Framebuffer *> frames;                     // three frames of changing width, 2 deflate segments each
        for (int k = 0; k < 3; ++k) {
            Framebuffer *f = new Framebuffer(200 + 7 * k, 100 + k);
            fill(f, 300 + k);
            frames.push_back(f);
        }
        for (int form = 0; form < 3; ++form) {                 // kitty, kitty in tmux, iTerm2
            std::string ours;
            if (form == 2) ours = run_canvas<B200ITerm2Canvas>(frames, 18, opts, true);
            else ours = run_canvas<B200KittyCanvas>(frames, 18, form == 1, opts, true);
            const std::vector<std::string> pngs = pngs_of(ours);
            g_replay.clear();
            g_served = 0;
            size_t png_bytes = 0, stored_bytes = 0;
            for (size_t i = 0; i < pngs.size() && i < frames.size(); ++i) {
                g_replay.push_back(Replay{scanlines(*frames[i], rgb24 != 0), zlib_of(pngs[i])});
                png_bytes += pngs[i].size();
                stored_bytes += b200timg_png_size(frames[i]->width(), frames[i]->height(), rgb24);
            }
            std::string ref;
            if (pngs.size() == frames.size()) {
                if (form == 2) ref = run_canvas<ITerm2GraphicsCanvas>(frames, 18, &pool, opts);
                else ref = run_canvas<KittyGraphicsCanvas>(frames, 18, &pool, form == 1, opts);
            }
            const bool same = !ref.empty() && ref == ours && g_served == (int)frames.size();
            const bool compressed = png_bytes < stored_bytes;
            const char *name = form == 0 ? "kitty" : form == 1 ? "kitty-tmux" : "iterm2";
            printf("%s rgb24=%d : %zu bytes %s, PNGs %zu of %zu stored bytes %s\n", name, rgb24, ours.size(),
                   same ? "identical" : "DIFFERENT", png_bytes, stored_bytes, compressed ? "compressed" : "NOT COMPRESSED");
            failures += !same + !compressed;
        }
        for (Framebuffer *f : frames) delete f;
    }
    printf(failures ? "GRAPHICS DEFLATE ADAPTER CHECK FAILED (%d)\n" : "GRAPHICS DEFLATE ADAPTER CHECK OK (%d failures)\n", failures);
    return failures ? 1 : 0;
}
