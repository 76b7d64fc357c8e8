// TEST INFRASTRUCTURE.  The kitty / iTerm2 half of the C++ drop-in check (oracle/adapter_check.cc does the block,
// sixel, scaler and compose half): links the reference's own KittyGraphicsCanvas / ITerm2GraphicsCanvas objects,
// compiled by oracle/graphics.mk with oracle/deflate_stored/libdeflate.h (stored deflate blocks) in place of
// libdeflate, the adapters (timg_b200/csrc/adapters.h) and libb200timg.so into one binary, drives both canvases
// through the reference's own TerminalCanvas + BufferedWriteSequencer and compares the bytes that reach the file
// descriptor: PNG, base64, chunking and headers must all be identical.  Kitty's image ids come from a time() seed on
// either side, so "i=<digits>" is normalised.  Needs a GPU.
#include <fcntl.h>
#include <sys/mman.h>
#include <unistd.h>

#include <csignal>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "adapters.h"
#include "iterm2-canvas.h"
#include "kitty-canvas.h"
#include "thread-pool.h"

using namespace timg;

static volatile sig_atomic_t g_no_interrupt = 0;

static uint32_t mix(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
    return x;
}
static void fill(Framebuffer *fb, uint32_t seed) {
    int i = 0;
    for (rgba_t *p = fb->begin(); p != fb->end(); ++p, ++i) {
        const uint32_t v = mix(seed * 0x9e3779b1U + (uint32_t)i);
        p->r = v; p->g = v >> 8; p->b = v >> 16; p->a = v >> 24;
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

// ",i=<digits>" -> ",i=#"
static std::string strip_ids(const std::string &s) {
    std::string r;
    for (size_t i = 0; i < s.size(); ++i) {
        r += s[i];
        if (s[i] == ',' && s.compare(i + 1, 2, "i=") == 0) {
            r += "i=#";
            i += 3;
            while (i < s.size() && s[i] >= '0' && s[i] <= '9') ++i;
            --i;
        }
    }
    return r;
}

int main() {
    int failures = 0;
    ThreadPool pool(2);
    for (int rgb24 = 0; rgb24 < 2; ++rgb24) {
        DisplayOptions opts;
        opts.cell_x_px = 9; opts.cell_y_px = 18;
        opts.local_alpha_handling = rgb24 != 0;
        std::vector<Framebuffer *> frames;                     // three frames of changing width, 4 to 6 kitty chunks
        for (int k = 0; k < 3; ++k) {
            Framebuffer *f = new Framebuffer(100 + 7 * k, 45);
            fill(f, 300 + k);
            frames.push_back(f);
        }
        const std::string rk = strip_ids(run_canvas<KittyGraphicsCanvas>(frames, 18, &pool, false, opts));
        const std::string gk = strip_ids(run_canvas<B200KittyCanvas>(frames, 18, opts));
        printf("kitty rgb24=%d : %zu bytes %s\n", rgb24, rk.size(), rk == gk ? "identical" : "DIFFERENT");
        failures += rk != gk;
        const std::string ri = run_canvas<ITerm2GraphicsCanvas>(frames, 18, &pool, opts);
        const std::string gi = run_canvas<B200ITerm2Canvas>(frames, 18, opts);
        printf("iterm2 rgb24=%d : %zu bytes %s\n", rgb24, ri.size(), ri == gi ? "identical" : "DIFFERENT");
        failures += ri != gi;
        for (Framebuffer *f : frames) delete f;
    }
    printf(failures ? "GRAPHICS ADAPTER CHECK FAILED (%d)\n" : "GRAPHICS ADAPTER CHECK OK (%d failures)\n", failures);
    return failures ? 1 : 0;
}
