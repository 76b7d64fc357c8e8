/* TEST INFRASTRUCTURE ONLY: our own LZW encoder for GIF rasters, the part of a GIF writer that is not byte framing
 * (oracle/gif.py frames the file around it).  Code widths follow the decoder the tests pin against
 * (stbi__process_gif_raster, third_party/stb/stb_image.h:6694-6776): after every code but a clear, the decoder's next
 * free entry grows unless the code follows a clear, and the width grows when that entry reaches a power of two below
 * 4096.  The encoder restates that walk so every code it writes is read at the width it was written with.
 *
 * orc_gif_lzw(idx, n, lzw_cs, policy, subblock, out, cap): the raster's bytes -- lzw_cs, sub-blocks of at most
 * `subblock` (1..255) data bytes, the zero-length terminator.  policy:
 *   0  clear first, and again whenever the table fills (4096 entries; 8192 for lzw_cs 12)
 *   1  no clear first (a decoder that requires one fails at the first code), then as 0
 *   2  clear first, then never again: once full the table stops growing on this side while the decoder keeps
 *      adding entries past 4096 (a "deferred clear" stream; stb fails with "too many codes" after 8192)
 * Indices must be below 1 << lzw_cs (lzw_cs 0 and 1 allow 0 and 0..1).  End of information is written when it fits
 * the current width.  Returns the bytes written, -1 on a bad argument, -2 if cap is too small. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    uint8_t *out;
    long cap, len;          /* bytes of out used, the current sub-block's length byte at blk */
    long blk;
    int subblock;
    uint32_t acc;
    int nacc;
    int dec_cs, dec_avail, dec_old, lzw_cs;
    int overflow;
} Enc;

static void put_byte(Enc *e, uint8_t b) {
    if (e->blk < 0 || e->out[e->blk] == e->subblock) {
        if (e->len >= e->cap) { e->overflow = 1; return; }
        e->blk = e->len;
        e->out[e->len++] = 0;
    }
    if (e->len >= e->cap) { e->overflow = 1; return; }
    e->out[e->len++] = b;
    e->out[e->blk]++;
}

static void emit(Enc *e, int code) {
    const int clear = 1 << e->lzw_cs;
    e->acc |= (uint32_t)code << e->nacc;
    e->nacc += e->dec_cs;
    while (e->nacc >= 8) { put_byte(e, (uint8_t)e->acc); e->acc >>= 8; e->nacc -= 8; }
    if (code == clear) {
        e->dec_cs = e->lzw_cs + 1; e->dec_avail = clear + 2; e->dec_old = 0;
    } else if (code != clear + 1) {
        if (e->dec_old) e->dec_avail++;
        if ((e->dec_avail & ((1 << e->dec_cs) - 1)) == 0 && e->dec_avail <= 0x0FFF) e->dec_cs++;
        e->dec_old = 1;
    }
}

long orc_gif_lzw(const uint8_t *idx, long n, int lzw_cs, int policy, int subblock, uint8_t *out, long cap) {
    if (lzw_cs < 0 || lzw_cs > 12 || policy < 0 || policy > 2 || subblock < 1 || subblock > 255 || cap < 2 || n < 0)
        return -1;
    const int clear = 1 << lzw_cs, limit = lzw_cs < 12 ? 4096 : 8192;
    for (long i = 0; i < n; ++i)
        if (idx[i] >= clear) return -1;
    /* trie: child[w * 256 + c] is valid when stamp[...] == gen */
    uint16_t *child = (uint16_t *)malloc(sizeof(uint16_t) * 8192 * 256);
    uint32_t *stamp = (uint32_t *)calloc(8192 * 256, sizeof(uint32_t));
    if (!child || !stamp) { free(child); free(stamp); return -1; }
    uint32_t gen = 1;
    Enc e = {out, cap, 0, -1, subblock, 0, 0, lzw_cs + 1, clear + 2, 0, lzw_cs, 0};
    out[e.len++] = (uint8_t)lzw_cs;
    int next = clear + 2;
    if (policy != 1) emit(&e, clear);
    if (n > 0) {
        int w = idx[0];
        for (long i = 1; i < n; ++i) {
            const int c = idx[i];
            const long k = (long)w * 256 + c;
            /* a longer match is taken only if its code fits the width the decoder reads the next code with (stb's
             * width lags the table by one code, which matters for lzw_cs 0 and 1) */
            if (stamp[k] == gen && child[k] < (1 << e.dec_cs)) { w = child[k]; continue; }
            emit(&e, w);
            if (next < limit) { stamp[k] = gen; child[k] = (uint16_t)next++; }
            if (next == limit && policy != 2) {
                emit(&e, clear);
                ++gen; next = clear + 2;
            }
            w = c;
        }
        emit(&e, w);
    }
    if (clear + 1 < (1 << e.dec_cs)) emit(&e, clear + 1);
    if (e.nacc > 0) put_byte(&e, (uint8_t)e.acc);
    if (e.len >= e.cap) e.overflow = 1;
    else out[e.len++] = 0;
    free(child); free(stamp);
    return e.overflow ? -2 : e.len;
}
