// TEST INFRASTRUCTURE ONLY -- never linked into or called from the product.
//
// extern "C" door onto the UNMODIFIED reference KittyGraphicsCanvas in its tmux form (tmux_passthrough_needed =
// true), compiled by oracle/graphics_tmux.mk with oracle/deflate_stored/libdeflate.h in place of libdeflate (stored
// deflate blocks).  As ref_graphics.cc does for the plain canvases, the bytes a Send produces are captured through the
// reference's own BufferedWriteSequencer into a memfd.
//
// The tmux form's constructor runs system("tmux set -p allow-passthrough on ...") and kitty's image ids are seeded
// from time().  This library defines both (graphics_tmux.mk links it with -Bsymbolic-functions, so the reference's
// objects inside it call these, while other code in the process keeps libc's): system() only records the command
// and returns 0, so no shell ever runs; time() returns $REF_GRAPHICS_TIME when set, which makes the ids, and the
// goldens, reproducible.
#include <fcntl.h>
#include <sys/mman.h>
#include <unistd.h>

#include <csignal>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <string>

#include "buffered-write-sequencer.h"
#include "display-options.h"
#include "framebuffer.h"
#include "kitty-canvas.h"
#include "thread-pool.h"

namespace {
static volatile sig_atomic_t g_never_interrupted = 0;
static std::string g_system_calls;            // every command passed to system(), one per line

struct TmuxCanvasDoor {
    int fd;
    off_t consumed = 0;
    timg::DisplayOptions opts;                 // the canvas keeps a reference to it
    timg::ThreadPool *pool;
    timg::BufferedWriteSequencer *seq;
    timg::KittyGraphicsCanvas *canvas;
};
}  // namespace

extern "C" {

int system(const char *command) {
    if (!command) return 1;                    // "a shell is available"
    g_system_calls += command;
    g_system_calls += '\n';
    return 0;
}

time_t time(time_t *t) {
    const char *pinned = getenv("REF_GRAPHICS_TIME");
    timespec ts{};
    if (!pinned) clock_gettime(CLOCK_REALTIME, &ts);
    const time_t now = pinned ? (time_t)strtoll(pinned, nullptr, 10) : ts.tv_sec;
    if (t) *t = now;
    return now;
}

// The commands system() was given so far (newline-terminated, concatenated) into out; their length, or -1 if they
// do not fit.
long ref_graphics_tmux_system_calls(char *out, long cap) {
    const long n = (long)g_system_calls.size();
    if (n > cap) return -1;
    memcpy(out, g_system_calls.data(), (size_t)n);
    return n;
}

// rgb24 = DisplayOptions::local_alpha_handling
void *ref_graphics_tmux_new(int rgb24, int cell_x_px, int cell_y_px) {
    TmuxCanvasDoor *d = new TmuxCanvasDoor;
    d->fd = memfd_create("timg_ref_graphics_tmux", 0);
    d->opts.local_alpha_handling = rgb24 != 0;
    d->opts.cell_x_px = cell_x_px;
    d->opts.cell_y_px = cell_y_px;
    d->pool = new timg::ThreadPool(1);
    d->seq = new timg::BufferedWriteSequencer(d->fd, false, 4, true, g_never_interrupted);
    d->canvas = new timg::KittyGraphicsCanvas(d->seq, d->pool, true, d->opts);
    return d;
}

// Bytes of one Send(x, dy, fb, seq_type) (timg::SeqType's value), copied to out; -1 if they do not fit.
long ref_graphics_tmux_send(void *h, int x, int dy, const uint8_t *fb, int w, int hgt, int seq_type, char *out, long cap) {
    TmuxCanvasDoor *d = (TmuxCanvasDoor *)h;
    timg::Framebuffer f(w, hgt);
    memcpy((void *)f.begin(), fb, (size_t)w * hgt * 4);
    d->canvas->Send(x, dy, f, (timg::SeqType)seq_type, timg::Duration());
    d->seq->Flush();
    const off_t end = lseek(d->fd, 0, SEEK_END);
    const long n = (long)(end - d->consumed);
    if (n > cap) return -1;
    if (n > 0 && pread(d->fd, out, n, d->consumed) != n) return -2;
    d->consumed = end;
    return n;
}

void ref_graphics_tmux_free(void *h) {
    TmuxCanvasDoor *d = (TmuxCanvasDoor *)h;
    delete d->canvas;
    delete d->seq;
    delete d->pool;
    close(d->fd);
    delete d;
}

}  // extern "C"
