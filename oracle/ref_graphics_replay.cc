// TEST INFRASTRUCTURE ONLY -- never linked into or called from the product.
//
// extern "C" door onto the UNMODIFIED reference canvases KittyGraphicsCanvas (plain and tmux form) and
// ITerm2GraphicsCanvas, compiled by oracle/graphics_deflate.mk with oracle/deflate_replay/libdeflate.h in place of
// libdeflate: each Send writes, around the zlib stream given with it, exactly what the reference writes around
// libdeflate's.  As ref_graphics.cc does, the bytes are captured through the reference's own BufferedWriteSequencer
// into a memfd.  As ref_graphics_tmux.cc does, this library defines system() (records nothing, runs no shell: the
// tmux form's constructor calls it) for the reference's objects, linked with -Bsymbolic-functions.
#include <fcntl.h>
#include <sys/mman.h>
#include <unistd.h>

#include <csignal>
#include <cstdint>
#include <cstring>
#include <vector>

#include "buffered-write-sequencer.h"
#include "display-options.h"
#include "framebuffer.h"
#include "iterm2-canvas.h"
#include "kitty-canvas.h"
#include "terminal-canvas.h"
#include "thread-pool.h"

namespace {
static volatile sig_atomic_t g_never_interrupted = 0;
static std::vector<uint8_t> g_stream;

struct ReplayDoor {
    int fd;
    off_t consumed = 0;
    timg::DisplayOptions opts;                 // the canvases keep a reference to it
    timg::ThreadPool *pool;
    timg::BufferedWriteSequencer *seq;
    timg::TerminalCanvas *canvas;
};
}  // namespace

extern "C" {

// the stream given with the current Send (one Send at a time: the canvas' pool has one thread and Send flushes)
const uint8_t *oracle_replay_stream(const void *, size_t, size_t *n) {
    *n = g_stream.size();
    return g_stream.data();
}

int system(const char *command) { return command ? 0 : 1; }

// protocol 1 = kitty, 2 = iTerm2, 4 = kitty in tmux; rgb24 = DisplayOptions::local_alpha_handling
void *ref_replay_new(int protocol, int rgb24, int cell_x_px, int cell_y_px) {
    ReplayDoor *d = new ReplayDoor;
    d->fd = memfd_create("timg_ref_graphics_replay", 0);
    d->opts.local_alpha_handling = rgb24 != 0;
    d->opts.cell_x_px = cell_x_px;
    d->opts.cell_y_px = cell_y_px;
    d->opts.compress_pixel_level = 1;
    d->pool = new timg::ThreadPool(1);
    d->seq = new timg::BufferedWriteSequencer(d->fd, false, 4, true, g_never_interrupted);
    if (protocol == 2) d->canvas = new timg::ITerm2GraphicsCanvas(d->seq, d->pool, d->opts);
    else d->canvas = new timg::KittyGraphicsCanvas(d->seq, d->pool, protocol == 4, d->opts);
    return d;
}

// Bytes of one Send(x, 0, fb, FrameImmediate) whose PNG carries the zlib stream z, copied to out; -1 if they do not fit.
long ref_replay_send(void *h, const uint8_t *z, long z_len, int x, const uint8_t *fb, int w, int hgt, char *out, long cap) {
    ReplayDoor *d = (ReplayDoor *)h;
    g_stream.assign(z, z + z_len);
    timg::Framebuffer f(w, hgt);
    memcpy((void *)f.begin(), fb, (size_t)w * hgt * 4);
    d->canvas->Send(x, 0, f, timg::SeqType::FrameImmediate, timg::Duration());
    d->seq->Flush();
    const off_t end = lseek(d->fd, 0, SEEK_END);
    const long n = (long)(end - d->consumed);
    if (n > cap) return -1;
    if (n > 0 && pread(d->fd, out, n, d->consumed) != n) return -2;
    d->consumed = end;
    return n;
}

void ref_replay_free(void *h) {
    ReplayDoor *d = (ReplayDoor *)h;
    delete d->canvas;
    delete d->seq;
    delete d->pool;
    close(d->fd);
    delete d;
}

}  // extern "C"
