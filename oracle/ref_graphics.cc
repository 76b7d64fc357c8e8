// TEST INFRASTRUCTURE ONLY -- never linked into or called from the product.
//
// extern "C" doors onto the UNMODIFIED reference canvases KittyGraphicsCanvas (tmux_passthrough_needed = false)
// and ITerm2GraphicsCanvas, compiled by oracle/Makefile with oracle/deflate_stored/libdeflate.h in place of
// libdeflate (stored deflate blocks).  As ref_shim.cc's block-canvas door does, the bytes a Send produces are
// captured through the reference's own BufferedWriteSequencer into a memfd.
#include <fcntl.h>
#include <sys/mman.h>
#include <unistd.h>

#include <csignal>
#include <cstdint>
#include <cstring>

#include "buffered-write-sequencer.h"
#include "display-options.h"
#include "framebuffer.h"
#include "iterm2-canvas.h"
#include "kitty-canvas.h"
#include "terminal-canvas.h"
#include "thread-pool.h"

namespace {
static volatile sig_atomic_t g_never_interrupted = 0;

struct GraphicsCanvasDoor {
    int fd;
    off_t consumed = 0;
    timg::DisplayOptions opts;                 // the canvases keep a reference to it
    timg::ThreadPool *pool;
    timg::BufferedWriteSequencer *seq;
    timg::TerminalCanvas *canvas;
};
}  // namespace

extern "C" {

// protocol 1 = kitty, 2 = iTerm2; rgb24 = DisplayOptions::local_alpha_handling
void *ref_graphics_new(int protocol, int rgb24, int cell_x_px, int cell_y_px) {
    GraphicsCanvasDoor *d = new GraphicsCanvasDoor;
    d->fd = memfd_create("timg_ref_graphics", 0);
    d->opts.local_alpha_handling = rgb24 != 0;
    d->opts.cell_x_px = cell_x_px;
    d->opts.cell_y_px = cell_y_px;
    d->pool = new timg::ThreadPool(1);
    d->seq = new timg::BufferedWriteSequencer(d->fd, false, 4, true, g_never_interrupted);
    if (protocol == 1) d->canvas = new timg::KittyGraphicsCanvas(d->seq, d->pool, false, d->opts);
    else d->canvas = new timg::ITerm2GraphicsCanvas(d->seq, d->pool, d->opts);
    return d;
}

// Bytes of one Send(x, dy, fb, seq_type) (timg::SeqType's value), copied to out; -1 if they do not fit.
long ref_graphics_send(void *h, int x, int dy, const uint8_t *fb, int w, int hgt, int seq_type, char *out, long cap) {
    GraphicsCanvasDoor *d = (GraphicsCanvasDoor *)h;
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

void ref_graphics_free(void *h) {
    GraphicsCanvasDoor *d = (GraphicsCanvasDoor *)h;
    delete d->canvas;
    delete d->seq;
    delete d->pool;
    close(d->fd);
    delete d;
}

}  // extern "C"
