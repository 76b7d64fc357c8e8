// TEST INFRASTRUCTURE ONLY -- never linked into or called from the product.
//
// An extern "C" door onto the UNMODIFIED reference QOIImageSource (src/qoi-image-source.cc), linked against
// oracle/_ref/libtimg_ref.so (oracle/Makefile) by oracle/qoi.mk.  ref_qoi_run runs LoadAndScale and then SendFrames
// once; with capture != 0 its sink keeps the framebuffer it is handed, with its dx, for ref_qoi_fetch; with capture == 0
// the sink drops it (a timing run: one decode and nothing else).
//   - A box larger than the image, cell 1x1 and has_bg = 0 (a null bgcolor_getter): the scaler keeps the size and
//     the compose step leaves pixels alone, so the frame is qoi_read's raw canvas.
//   - Real options: the reference's scaled frame, composed only for a 4-channel header, exactly as its canvases
//     receive it.
#include <csignal>
#include <cstdint>
#include <cstring>
#include <vector>

#include "display-options.h"
#include "framebuffer.h"
#include "qoi-image-source.h"
#include "timg-time.h"

namespace {
volatile sig_atomic_t g_never_interrupted = 0;

struct QoiRun {
    std::vector<uint8_t> bytes;
    int w = 0, h = 0, dx = 0, n = 0;
};
}  // namespace

extern "C" {

// nullptr if the source fails to load; else a handle holding the frame sent (*w x *h, sent at column *dx).
void *ref_qoi_run(const char *path, int width, int height, int cell_x_px, int cell_y_px, int has_bg, uint32_t bg,
                  uint32_t pattern, int pattern_size, int capture, int *w, int *h, int *dx) {
    timg::DisplayOptions o;
    o.width = width;
    o.height = height;
    o.cell_x_px = cell_x_px;
    o.cell_y_px = cell_y_px;
    timg::rgba_t bgc, pat;
    memcpy(&bgc, &bg, 4);
    memcpy(&pat, &pattern, 4);
    if (has_bg) o.bgcolor_getter = [bgc]() { return bgc; };
    o.bg_pattern_color = pat;
    o.pattern_size = pattern_size;
    timg::QOIImageSource src(path);
    if (!src.LoadAndScale(o, 0, -1)) return nullptr;
    QoiRun *r = new QoiRun;
    src.SendFrames(timg::Duration::Millis(0), 1, g_never_interrupted,
                   [&](int x, int, const timg::Framebuffer &fb, timg::SeqType, timg::Duration) {
                       if (capture) {
                           const uint8_t *p = (const uint8_t *)fb.begin();
                           r->bytes.assign(p, p + (size_t)fb.width() * fb.height() * 4);
                       }
                       r->w = fb.width();
                       r->h = fb.height();
                       r->dx = x;
                       ++r->n;
                   });
    *w = r->w;
    *h = r->h;
    *dx = r->dx;
    return r;
}

// Copies a captured run's frame (*w * *h * 4 bytes of ref_qoi_run).
void ref_qoi_fetch(void *h, uint8_t *out) {
    const QoiRun *r = (const QoiRun *)h;
    if (!r->bytes.empty()) memcpy(out, r->bytes.data(), r->bytes.size());
}

void ref_qoi_free(void *h) { delete (QoiRun *)h; }

}  // extern "C"
