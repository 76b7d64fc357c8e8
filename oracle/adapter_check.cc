// TEST INFRASTRUCTURE.  Links the reference's own objects (oracle/_ref/*.o), the C++ adapters
// (timg_b200/csrc/adapters.h) and libb200timg.so into one binary and drives BOTH canvases/scalers
// through the reference's own plugin surface (ImageScaler, TerminalCanvas, BufferedWriteSequencer),
// comparing the bytes that reach the file descriptor.  This is the drop-in proof at the C++ level:
// same calls a timg maintainer's build would make (INTEGRATION.md).  Needs a GPU.
#include <fcntl.h>
#include <sys/mman.h>
#include <unistd.h>

#include <csignal>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <string>
#include <vector>

#include "adapters.h"
#include "unicode-block-canvas.h"

using namespace timg;

static volatile sig_atomic_t g_no_interrupt = 0;

static uint32_t mix(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
    return x;
}
static void fill(Framebuffer *fb, uint32_t seed, bool alpha) {
    int i = 0;
    for (rgba_t *p = fb->begin(); p != fb->end(); ++p, ++i) {
        const uint32_t v = mix(seed * 0x9e3779b1U + (uint32_t)i);
        p->r = v; p->g = v >> 8; p->b = v >> 16; p->a = alpha ? (v >> 24) : 255;
    }
}
static std::string slurp(int fd) {
    const off_t n = lseek(fd, 0, SEEK_END);
    std::string s((size_t)n, '\0');
    if (n && pread(fd, &s[0], n, 0) != n) abort();
    return s;
}

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

int main() {
    int failures = 0;
    // ---- ImageScaler: reference STB scaler vs B200ImageScaler
    for (int t = 0; t < 6; ++t) {
        const int iw = 320 + 37 * t, ih = 200 + 11 * t, ow = 45 + 60 * t, oh = 30 + 41 * t;
        Framebuffer in(iw, ih), a(ow, oh), b(ow, oh);
        fill(&in, 100 + t, t & 1);
        ImageScaler::Create(iw, ih, ImageScaler::ColorFmt::kRGBA, ow, oh)->Scale(in, &a);
        B200CreateImageScaler(iw, ih, ImageScaler::ColorFmt::kRGBA, ow, oh)->Scale(in, &b);
        const bool same = memcmp((const void *)a.begin(), (const void *)b.begin(), (size_t)ow * oh * 4) == 0;
        printf("scale %dx%d -> %dx%d : %s\n", iw, ih, ow, oh, same ? "identical" : "DIFFERENT");
        failures += !same;
        // ---- AlphaComposeBackground
        Framebuffer c(a), d(b);
        const rgba_t bg = {20, 40, 160, 255}, pat = {200, 190, 10, 255};
        c.AlphaComposeBackground([bg]() { return bg; }, pat, 3, 2, t);
        B200AlphaComposeBackground(&d, [bg]() { return bg; }, pat, 3, 2, t);
        const bool same2 = memcmp((const void *)c.begin(), (const void *)d.begin(), (size_t)ow * oh * 4) == 0;
        printf("compose %dx%d start_row %d : %s\n", ow, oh, t, same2 ? "identical" : "DIFFERENT");
        failures += !same2;
    }
    // ---- UnicodeBlockCanvas vs B200BlockCanvas: an animation with sparse changes, all flag combinations
    for (int flags = 0; flags < 8; ++flags) {
        const bool quarter = flags & 1, upper = flags & 2, color8 = flags & 4;
        const int w = quarter ? 96 : 77, h = 45;
        std::vector<Framebuffer *> frames;
        for (int k = 0; k < 5; ++k) {
            Framebuffer *f = new Framebuffer(w, h);
            fill(f, 7, k == 0);                                   // same base content ...
            for (int j = 0; j < 6 * k; ++j) f->SetPixel((13 * j + 5 * k) % w, (7 * j + 3 * k) % h, rgba_t{(uint8_t)(40 * k), 9, (uint8_t)j, 255});
            frames.push_back(f);
        }
        const std::string ref = run_canvas<UnicodeBlockCanvas>(frames, 4, quarter, upper, color8);
        const std::string got = run_canvas<B200BlockCanvas>(frames, 4, quarter, upper, color8);
        const bool same = ref == got;
        printf("blocks quarter=%d upper=%d color8=%d : %zu bytes %s\n", quarter, upper, color8, ref.size(), same ? "identical" : "DIFFERENT");
        failures += !same;
        for (Framebuffer *f : frames) delete f;
    }
    // ---- B200SixelCanvas: the in-tree part of SixelCanvas::Send (src/sixel-canvas.cc:100-155) around the
    // library's DCS stream.  The reference's own SixelCanvas cannot be linked (libsixel is not in the tree),
    // so the expected bytes are assembled from what that function writes: queued prefix (cursor off, cursor
    // right by x / cell_x_px), the cursor-placement mode string (:66-79), the stream of the frame padded to a
    // multiple of 6 rows with the pad strip composed by the REFERENCE's AlphaComposeBackground (:109-120),
    // then "\r" or "\n" (:150).
    for (int broken = 0; broken < 2; ++broken) {
        DisplayOptions opts;
        opts.cell_x_px = 9; opts.cell_y_px = 18;
        const rgba_t bg = {10, 20, 30, 255};
        opts.bgcolor_getter = [bg]() { return bg; };
        opts.bg_pattern_color = rgba_t{70, 80, 90, 255};
        opts.pattern_size = 1;
        SixelOptions so;
        so.known_broken_cursor_placement = broken != 0;
        const int w = 100, h = 45, hp = 48, x_px = 18;
        Framebuffer fb(w, h);
        fill(&fb, 55 + broken, false);
        std::vector<Framebuffer *> one{&fb};
        const std::string got = run_canvas<B200SixelCanvas>(one, x_px, so, opts);
        Framebuffer padded(w, hp);                                    // zero-initialised == transparent
        padded.AlphaComposeBackground(opts.bgcolor_getter, opts.bg_pattern_color, opts.pattern_size * opts.cell_x_px,
                                      opts.pattern_size * opts.cell_y_px / 2, h);
        std::copy(fb.begin(), fb.end(), padded.begin());
        std::string dcs(b200timg_sixel_bound(w, hp), '\0');
        size_t n = 0;
        B200Context::Check(b200timg_sixel_encode(B200Context::Get(), (const uint8_t *)padded.begin(), w, hp, &dcs[0], dcs.size(), &n),
                           "sixel_encode");
        dcs.resize(n);
        const std::string want = std::string("\033[?25l") + "\033[2C" +
                                 (broken ? "\033[80l\033[?7730l\033[?8452h" : "\033[80h\033[?7730h\033[?8452l") + dcs +
                                 (broken ? "\n" : "\r") + "\033[?25h";
        const bool same = got == want;
        printf("sixel canvas framing broken_cursor=%d : %zu bytes %s\n", broken, got.size(), same ? "identical" : "DIFFERENT");
        failures += !same;
        const bool dcs_ok = dcs.size() > 8 && dcs.compare(0, 3, "\033Pq") == 0 && dcs.compare(dcs.size() - 2, 2, "\033\\") == 0;
        failures += !dcs_ok;
    }
    printf(failures ? "ADAPTER CHECK FAILED (%d)\n" : "ADAPTER CHECK OK (%d failures)\n", failures);
    return failures ? 1 : 0;
}
