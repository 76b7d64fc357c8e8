/* TEST INFRASTRUCTURE ONLY: a QOI encoder written from the published format description (qoiformat.org,
 * "The Quite OK Image Format, Specification Version 1.0").  Each pixel, compared with the previous one (initially
 * {0,0,0,255}), becomes the first op that can express it, in the order the specification's encoder tries them: extend
 * a run (flushed at 62 pixels and at the end), an index hit, a small difference, a luma difference, an RGB op when
 * alpha is unchanged, else an RGBA op.  The 64-entry table is updated with every pixel that is not a run repeat or an
 * index hit.  Input is always RGBA; `channels` is only the header field. */
#include <stdint.h>

static void put32(uint8_t *o, long *n, uint32_t v) {
    o[(*n)++] = (uint8_t)(v >> 24); o[(*n)++] = (uint8_t)(v >> 16); o[(*n)++] = (uint8_t)(v >> 8); o[(*n)++] = (uint8_t)v;
}

/* bytes written, or -1 if cap is too small (the worst case is 14 + 5 * w * h + 8) */
long orc_qoi_encode(const uint8_t *rgba, int w, int h, int channels, int colorspace, uint8_t *out, long cap) {
    const long npx = (long)w * h;
    if (cap < 22 + 5 * npx) return -1;
    long n = 0;
    put32(out, &n, 0x716f6966u);                            /* "qoif" */
    put32(out, &n, (uint32_t)w);
    put32(out, &n, (uint32_t)h);
    out[n++] = (uint8_t)channels;
    out[n++] = (uint8_t)colorspace;
    uint32_t seen[64] = {0};
    uint8_t pr = 0, pg = 0, pb = 0, pa = 255;
    int run = 0;
    for (long i = 0; i < npx; ++i) {
        const uint8_t r = rgba[4 * i], g = rgba[4 * i + 1], b = rgba[4 * i + 2], a = rgba[4 * i + 3];
        if (r == pr && g == pg && b == pb && a == pa) {
            if (++run == 62 || i == npx - 1) { out[n++] = (uint8_t)(0xc0 | (run - 1)); run = 0; }
            continue;
        }
        if (run) { out[n++] = (uint8_t)(0xc0 | (run - 1)); run = 0; }
        const uint32_t v = (uint32_t)r | (uint32_t)g << 8 | (uint32_t)b << 16 | (uint32_t)a << 24;
        const int slot = (r * 3 + g * 5 + b * 7 + a * 11) % 64;
        if (seen[slot] == v) {
            out[n++] = (uint8_t)slot;
        } else {
            seen[slot] = v;
            if (a == pa) {
                const int dr = (int8_t)(r - pr), dg = (int8_t)(g - pg), db = (int8_t)(b - pb);
                const int rg = dr - dg, bg = db - dg;
                if (dr >= -2 && dr <= 1 && dg >= -2 && dg <= 1 && db >= -2 && db <= 1) {
                    out[n++] = (uint8_t)(0x40 | (dr + 2) << 4 | (dg + 2) << 2 | (db + 2));
                } else if (dg >= -32 && dg <= 31 && rg >= -8 && rg <= 7 && bg >= -8 && bg <= 7) {
                    out[n++] = (uint8_t)(0x80 | (dg + 32));
                    out[n++] = (uint8_t)((rg + 8) << 4 | (bg + 8));
                } else {
                    out[n++] = 0xfe; out[n++] = r; out[n++] = g; out[n++] = b;
                }
            } else {
                out[n++] = 0xff; out[n++] = r; out[n++] = g; out[n++] = b; out[n++] = a;
            }
        }
        pr = r; pg = g; pb = b; pa = a;
    }
    for (int k = 0; k < 7; ++k) out[n++] = 0;
    out[n++] = 1;
    return n;
}
