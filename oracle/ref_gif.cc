// TEST INFRASTRUCTURE ONLY -- never linked into or called from the product.
//
// An extern "C" door onto the UNMODIFIED reference STBImageSource (src/stb-image-source.cc), linked against
// oracle/_ref/libtimg_ref.so (oracle/Makefile) by oracle/gif.mk.  ref_stb_gif_run runs LoadAndScale and then
// SendFrames once; with capture != 0 its sink keeps every framebuffer it is handed, with its dx, dy and the frame's
// delay, for ref_stb_gif_fetch; with capture == 0 the sink drops them (a timing run: one decode and nothing else).
//   - A box larger than the image and has_bg = 0 (a null bgcolor_getter): the scaler keeps the size and the compose
//     step leaves pixels alone, so the frames are stb's raw canvases (stbi__gif_load_next with two_back = NULL).
//   - Real options: the reference's scaled and composed frames, exactly as its canvases receive them.
#include <csignal>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "display-options.h"
#include "framebuffer.h"
#include "stb-image-source.h"
#include "timg-time.h"

namespace {
volatile sig_atomic_t g_never_interrupted = 0;

struct GifRun {
    std::vector<uint8_t> bytes;     // the frames back to back
    std::vector<int> meta;          // {w, h, dx, dy, delay_ms} per frame
    int n = 0;
};
}  // namespace

extern "C" {

// nullptr if the source fails to load; else a handle holding the frames sent (*n_frames) and their bytes (*bytes).
void *ref_stb_gif_run(const char *path, int width, int height, int cell_x_px, int cell_y_px, int has_bg, uint32_t bg,
                      uint32_t pattern, int pattern_size, int capture, int *n_frames, long long *bytes) {
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
    timg::STBImageSource src(path);
    if (!src.LoadAndScale(o, 0, -1)) return nullptr;
    GifRun *r = new GifRun;
    int64_t last_ns = 0;                            // the sink gets the time since the first frame: delays are steps
    src.SendFrames(timg::Duration::Millis(1LL << 40), 1, g_never_interrupted,
                   [&](int x, int dy, const timg::Framebuffer &fb, timg::SeqType, timg::Duration end) {
                       if (capture) {
                           const size_t len = (size_t)fb.width() * fb.height() * 4;
                           const uint8_t *p = (const uint8_t *)fb.begin();
                           r->bytes.insert(r->bytes.end(), p, p + len);
                           r->meta.insert(r->meta.end(), {fb.width(), fb.height(), x, dy,
                                                          (int)((end.nanoseconds() - last_ns) / 1000000)});
                       }
                       last_ns = end.nanoseconds();
                       ++r->n;
                   });
    *n_frames = r->n;
    *bytes = (long long)r->bytes.size();
    return r;
}

// Copies a captured run's frames (the *bytes of ref_stb_gif_run) and meta (5 ints per frame).
void ref_stb_gif_fetch(void *h, uint8_t *out, int *meta) {
    const GifRun *r = (const GifRun *)h;
    if (!r->bytes.empty()) memcpy(out, r->bytes.data(), r->bytes.size());
    if (!r->meta.empty()) memcpy(meta, r->meta.data(), r->meta.size() * sizeof(int));
}

void ref_stb_gif_free(void *h) { delete (GifRun *)h; }

}  // extern "C"
