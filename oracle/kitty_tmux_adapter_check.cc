// TEST INFRASTRUCTURE.  kitty's tmux form through the C++ drop-in: links the reference's own KittyGraphicsCanvas
// (compiled by oracle/graphics_tmux.mk with oracle/deflate_stored/libdeflate.h, stored deflate blocks, in place of
// libdeflate), B200KittyCanvas (timg_b200/csrc/adapters.h) and libb200timg.so into one binary, drives both with
// tmux_passthrough_needed = true through the reference's own TerminalCanvas + BufferedWriteSequencer and compares the
// bytes that reach the file descriptor: passthrough framing, chunking and the Unicode placeholder grid.
//
// This binary defines time() and system(), which take the calls of everything linked into it:
//   time()   returns a pinned value, so both sides' CreateId start from the same seed and produce the same image ids
//            (no normalisation; the seed gives 10-digit ids with a nonzero top byte, i.e. an id diacritic);
//   system() records the command and returns 0, so no shell runs.  Each canvas must make exactly one call, the
//            reference's "tmux set -p allow-passthrough on" command.
// Needs a GPU.
#include <fcntl.h>
#include <sys/mman.h>
#include <unistd.h>

#include <csignal>
#include <cstdio>
#include <cstdlib>
#include <ctime>
#include <string>
#include <vector>

#include "adapters.h"
#include "kitty-canvas.h"
#include "thread-pool.h"

using namespace timg;

static constexpr time_t kPinnedTime = (200 << 17) | 0x123;      // ids 0xC8009180 + k: msb 200, 10 digits
static const char kPassthroughCommand[] = "tmux set -p allow-passthrough on > /dev/null 2>&1";
static std::vector<std::string> g_system_calls;

extern "C" time_t time(time_t *t) {
    if (t) *t = kPinnedTime;
    return kPinnedTime;
}
extern "C" int system(const char *command) {
    if (!command) return 1;
    g_system_calls.push_back(command);
    return 0;
}

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

// the canvas just run made exactly one system() call, with the reference's command
static bool one_passthrough_call() {
    const bool ok = g_system_calls.size() == 1 && g_system_calls[0] == kPassthroughCommand;
    g_system_calls.clear();
    return ok;
}

int main() {
    int failures = 0;
    ThreadPool pool(2);
    struct Geometry { int cell_x, cell_y, x, w0, h; };
    // 9x18 cells indented by 2; 1x2 cells on frames 300 px wide, whose columns reach the last diacritics and beyond
    const Geometry geos[] = {{9, 18, 18, 100, 45}, {1, 2, 5, 300, 21}};
    for (const Geometry &geo : geos) {
        for (int rgb24 = 0; rgb24 < 2; ++rgb24) {
            DisplayOptions opts;
            opts.cell_x_px = geo.cell_x; opts.cell_y_px = geo.cell_y;
            opts.local_alpha_handling = rgb24 != 0;
            std::vector<Framebuffer *> frames;                 // three frames of changing width
            for (int k = 0; k < 3; ++k) {
                Framebuffer *f = new Framebuffer(geo.w0 + 7 * k, geo.h + k);
                fill(f, 500 + k);
                frames.push_back(f);
            }
            g_system_calls.clear();
            const std::string rk = run_canvas<KittyGraphicsCanvas>(frames, geo.x, &pool, true, opts);
            const bool ref_call = one_passthrough_call();
            const std::string gk = run_canvas<B200KittyCanvas>(frames, geo.x, true, opts);
            const bool our_call = one_passthrough_call();
            const bool same = rk == gk && rk.find("\033Ptmux;") != std::string::npos;
            printf("kitty-tmux cells=%dx%d x=%d rgb24=%d : %zu bytes %s, passthrough command %s\n", geo.cell_x, geo.cell_y, geo.x,
                   rgb24, rk.size(), same ? "identical" : "DIFFERENT", ref_call && our_call ? "once on each side" : "WRONG");
            failures += !same + !(ref_call && our_call);
            for (Framebuffer *f : frames) delete f;
        }
    }
    printf(failures ? "KITTY TMUX ADAPTER CHECK FAILED (%d)\n" : "KITTY TMUX ADAPTER CHECK OK (%d failures)\n", failures);
    return failures ? 1 : 0;
}
