/* TEST INFRASTRUCTURE ONLY -- never linked into or called from the product path.
 *
 * PARITY UNPINNED.  The reference's sixel path is 30 lines of glue (src/sixel-canvas.cc:100-155)
 * around libsixel, a third-party dependency that is NOT vendored under /root/reference and not
 * installed in this image (CMakeLists.txt:44-46: pkg_check_modules(LIBSIXEL ... libsixel), no
 * version pin; Ubuntu 24.04 ships 1.10.3).  The reference holds no test, golden vector or
 * fixture for this path.  What follows restates libsixel's published algorithm (saitoha/libsixel
 * 1.8-1.10: src/quant.c computeHistogram / mediancut / lookup_fast / diffuse_fs,
 * src/tosixel.c sixel_encode_header / sixel_encode_body / sixel_put_node / sixel_put_flash)
 * for exactly the call sequence the reference makes (src/sixel-canvas.cc:134-148):
 *     sixel_dither_new(256)                       -> reqcolors 256, FS diffusion, complexion 1
 *     sixel_dither_initialize(RGBA8888, SIXEL_LARGE_LUM, SIXEL_REP_AVERAGE_COLORS, QUALITY_AUTO)
 *     sixel_encode(pixels, w, h, 0, dither, output)
 * It cannot be checked against libsixel here, so parity for sixel is judged by decoding
 * (orc_sixel_decode) and comparing images within a stated tolerance, not by bytes.
 * Where libsixel's result depends on qsort's treatment of equal keys (implementation
 * defined), this restatement uses a stable sort.
 */
#include <limits.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

typedef struct { uint8_t c[3]; uint32_t count; } hcolor_t;   /* one occupied 15-bit bucket */
typedef struct { int ind, colors; uint32_t sum; } box_t;

static unsigned hash15(const uint8_t *p) {          /* quant.c computeHash(pixel, 3) */
    return ((unsigned)(p[0] >> 3) << 10) | ((unsigned)(p[1] >> 3) << 5) | (unsigned)(p[2] >> 3);
}

/* stable merge sort of hcolor_t by one channel ascending (compareplane) */
static void sort_plane(hcolor_t *a, int n, int plane, hcolor_t *tmp) {
    if (n < 2) return;
    const int m = n / 2;
    sort_plane(a, m, plane, tmp); sort_plane(a + m, n - m, plane, tmp);
    int i = 0, j = m, k = 0;
    while (i < m && j < n) tmp[k++] = (a[j].c[plane] < a[i].c[plane]) ? a[j++] : a[i++];
    while (i < m) tmp[k++] = a[i++];
    while (j < n) tmp[k++] = a[j++];
    memcpy(a, tmp, (size_t)n * sizeof *a);
}
static void sort_boxes(box_t *b, int n) {           /* sumcompare: descending by sum, stable */
    for (int i = 1; i < n; i++) {
        box_t v = b[i]; int j = i - 1;
        while (j >= 0 && b[j].sum < v.sum) { b[j + 1] = b[j]; j--; }
        b[j + 1] = v;
    }
}

/* quant.c sixel_quant_make_palette -> computeColorMapFromInput.  rgb: w*h*3 bytes.
 * Returns number of palette entries (<=256); *origcolors = occupied buckets. */
/* mode 0: libsixel-faithful.  mode 1: "device semantics" -- the two places where libsixel's result
 * depends on raster order are replaced by order-free rules so that a parallel implementation can
 * be compared bit for bit: (a) the histogram table starts in bucket-index order instead of
 * first-seen order (only changes how ties sort), (b) the nearest-colour memo of a 15-bit cell is
 * the nearest palette entry to the cell CENTRE instead of to whichever pixel hit the cell first. */
static int make_palette(const uint8_t *rgb, long npix, uint8_t *palette, int *origcolors, int mode) {
    const unsigned depth = 3, reqcolors = 256, max_sample = 18383;      /* QUALITY_AUTO -> LOW */
    const unsigned long length = (unsigned long)npix * depth;
    unsigned long step = length / depth / max_sample * depth;
    if (length < (unsigned long)max_sample * depth) step = 6 * depth;
    if (step <= 0) step = depth;
    uint16_t *hist = (uint16_t *)calloc(1 << 15, sizeof(uint16_t));
    uint16_t *refmap = (uint16_t *)malloc((1 << 15) * sizeof(uint16_t));
    int nref = 0;
    for (unsigned long i = 0; i < length; i += step) {
        const unsigned b = hash15(rgb + i);
        if (hist[b] == 0) refmap[nref++] = (uint16_t)b;
        if (hist[b] < 65535) hist[b]++;
    }
    hcolor_t *tab = (hcolor_t *)malloc((size_t)(nref ? nref : 1) * sizeof *tab);
    if (mode == 1) { nref = 0; for (unsigned b = 0; b < (1u << 15); b++) if (hist[b]) refmap[nref++] = (uint16_t)b; }
    for (int i = 0; i < nref; i++) {                 /* first-seen order; colour = 5-bit value << 3 */
        const unsigned b = refmap[i];
        tab[i].c[0] = (uint8_t)(((b >> 10) & 31) << 3);
        tab[i].c[1] = (uint8_t)(((b >> 5) & 31) << 3);
        tab[i].c[2] = (uint8_t)((b & 31) << 3);
        tab[i].count = hist[b];
    }
    free(hist); free(refmap);
    *origcolors = nref;
    int ncolors;
    if ((unsigned)nref <= reqcolors) {               /* "Image already has few enough colors" */
        for (int i = 0; i < nref; i++) memcpy(palette + 3 * i, tab[i].c, 3);
        ncolors = nref;
    } else {                                         /* mediancut() */
        box_t bv[256];
        hcolor_t *tmp = (hcolor_t *)malloc((size_t)nref * sizeof *tmp);
        uint32_t sum = 0;
        for (int i = 0; i < nref; i++) sum += tab[i].count;
        bv[0].ind = 0; bv[0].colors = nref; bv[0].sum = sum;
        int boxes = 1, multi = nref > 1;
        while (boxes < (int)reqcolors && multi) {
            int bi;
            for (bi = 0; bi < boxes && bv[bi].colors < 2; ++bi) ;
            if (bi >= boxes) { multi = 0; break; }
            /* splitBox */
            const int start = bv[bi].ind, size = bv[bi].colors; const uint32_t sm = bv[bi].sum;
            int mn[3] = {255, 255, 255}, mx[3] = {0, 0, 0};
            for (int i = 0; i < size; i++)
                for (int p = 0; p < 3; p++) {
                    const int v = tab[start + i].c[p];
                    if (v < mn[p]) mn[p] = v;
                    if (v > mx[p]) mx[p] = v;
                }
            static const double lum[3] = {0.2989, 0.5866, 0.1145};       /* largestByLuminosity */
            int plane = 0; double best = 0.0;
            for (int p = 0; p < 3; p++) {
                const double spread = lum[p] * (mx[p] - mn[p]);
                if (spread > best) { plane = p; best = spread; }
            }
            sort_plane(tab + start, size, plane, tmp);
            uint32_t lower = tab[start].count; int i;
            for (i = 1; i < size - 1 && lower < sm / 2; ++i) lower += tab[start + i].count;
            const int median = i;
            bv[bi].colors = median; bv[bi].sum = lower;
            bv[boxes].ind = start + median; bv[boxes].colors = size - median; bv[boxes].sum = sm - lower;
            ++boxes;
            sort_boxes(bv, boxes);
        }
        memset(palette, 0, 768);                     /* newColorMap(newcolors): unused entries stay 0 */
        for (int b = 0; b < boxes; b++)              /* colormapFromBv, REP_AVERAGE_COLORS: plain mean */
            for (int p = 0; p < 3; p++) {
                unsigned long s = 0;
                for (int i = 0; i < bv[b].colors; i++) s += tab[bv[b].ind + i].c[p];
                palette[3 * b + p] = (uint8_t)(s / (unsigned long)bv[b].colors);
            }
        free(tmp);
        ncolors = (int)reqcolors;
    }
    free(tab);
    return ncolors;
}

static void fs_add(uint8_t *data, long pos, int error, int num) {       /* quant.c error_diffuse */
    int c = data[pos * 3] + error * num / 16;
    if (c < 0) c = 0;
    if (c >= 1 << 8) c = (1 << 8) - 1;
    data[pos * 3] = (uint8_t)c;
}

/* quant.c sixel_quant_apply_palette (foptimize=1, foptimize_palette=0, complexion=1) */
static void apply_palette(uint8_t *rgb, int w, int h, const uint8_t *palette, int ncolors, int diffuse,
                          uint8_t *index, int mode) {
    uint16_t *cache = (uint16_t *)calloc(1 << 15, sizeof(uint16_t));
    if (mode == 1)
        for (unsigned b = 0; b < (1u << 15); b++) {
            const int c[3] = {(int)(((b >> 10) & 31) << 3 | 4), (int)(((b >> 5) & 31) << 3 | 4), (int)((b & 31) << 3 | 4)};
            int diff = INT_MAX, ci = -1;
            for (int i = 0; i < ncolors; i++) {
                int d = 0, r;
                r = c[0] - palette[i * 3 + 0]; d += r * r;
                r = c[1] - palette[i * 3 + 1]; d += r * r;
                r = c[2] - palette[i * 3 + 2]; d += r * r;
                if (d < diff) { diff = d; ci = i; }
            }
            cache[b] = (uint16_t)(ci + 1);
        }
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const long pos = (long)y * w + x;
            const uint8_t *px = rgb + pos * 3;
            const unsigned hsh = hash15(px);               /* lookup_fast */
            int ci;
            if (cache[hsh]) ci = cache[hsh] - 1;
            else {
                int diff = INT_MAX; ci = -1;
                for (int i = 0; i < ncolors; i++) {
                    int d = 0, r;
                    r = px[0] - palette[i * 3 + 0]; d += r * r;
                    r = px[1] - palette[i * 3 + 1]; d += r * r;
                    r = px[2] - palette[i * 3 + 2]; d += r * r;
                    if (d < diff) { diff = d; ci = i; }
                }
                cache[hsh] = (uint16_t)(ci + 1);
            }
            index[pos] = (uint8_t)ci;
            if (diffuse && x < w - 1 && y < h - 1)         /* diffuse_fs: 7/16 r, 3/16 bl, 5/16 b, 1/16 br */
                for (int n = 0; n < 3; n++) {
                    const int off = rgb[pos * 3 + n] - palette[ci * 3 + n];
                    fs_add(rgb + n, pos + 1, off, 7);
                    fs_add(rgb + n, pos + w - 1, off, 3);
                    fs_add(rgb + n, pos + w, off, 5);
                    fs_add(rgb + n, pos + w + 1, off, 1);
                }
        }
    free(cache);
}

/* ---- tosixel.c emitter ---- */
typedef struct { char *p, *end; int save_pixel, save_count, active_palette, overflow; } emit_t;
static void e_putc(emit_t *e, int c) { if (e->p < e->end) *e->p++ = (char)c; else e->overflow = 1; }
static void e_putnum(emit_t *e, int v) { char b[16]; int n = sprintf(b, "%d", v); for (int i = 0; i < n; i++) e_putc(e, b[i]); }
static void e_flash(emit_t *e) {                           /* sixel_put_flash */
    if (e->save_count > 3) { e_putc(e, '!'); e_putnum(e, e->save_count); e_putc(e, e->save_pixel); }
    else for (int n = 0; n < e->save_count; n++) e_putc(e, e->save_pixel);
    e->save_pixel = 0; e->save_count = 0;
}
static void e_pixel(emit_t *e, int pix) {                  /* sixel_put_pixel */
    if (pix < 0 || pix > '?') pix = 0;
    pix += '?';
    if (pix == e->save_pixel) e->save_count++;
    else { e_flash(e); e->save_pixel = pix; e->save_count = 1; }
}
typedef struct node_s { struct node_s *next; int pal, sx, mx; const uint8_t *map; } node_t;
static int put_node(emit_t *e, int x, const node_t *np) {  /* sixel_put_node */
    if (e->active_palette != np->pal) { e_putc(e, '#'); e_putnum(e, np->pal); e->active_palette = np->pal; }
    for (; x < np->sx; ++x) e_pixel(e, 0);
    for (; x < np->mx; ++x) e_pixel(e, np->map[x]);
    e_flash(e);
    return x;
}

static void put_header(emit_t *e, int w, int h, const uint8_t *palette, int ncolors) {
    e_putc(e, 033); e_putc(e, 'P'); e_putc(e, 'q');                        /* sixel_encode_header */
    e_putc(e, '"'); e_putnum(e, 1); e_putc(e, ';'); e_putnum(e, 1); e_putc(e, ';'); e_putnum(e, w); e_putc(e, ';'); e_putnum(e, h);
    for (int n = 0; n < ncolors; n++) {                                    /* output_rgb_palette_definition */
        e_putc(e, '#'); e_putnum(e, n); e_putc(e, ';'); e_putc(e, '2'); e_putc(e, ';');
        e_putnum(e, (palette[n * 3 + 0] * 100 + 127) / 255); e_putc(e, ';');
        e_putnum(e, (palette[n * 3 + 1] * 100 + 127) / 255); e_putc(e, ';');
        e_putnum(e, (palette[n * 3 + 2] * 100 + 127) / 255);
    }
}

static long encode_body(const uint8_t *index, int w, int h, const uint8_t *palette, int ncolors, char *out, long cap) {
    emit_t E = { out, out + cap, 0, 0, -1, 0 };
    emit_t *e = &E;
    put_header(e, w, h, palette, ncolors);
    uint8_t *map = (uint8_t *)calloc((size_t)ncolors * w, 1);
    node_t *pool = (node_t *)malloc((size_t)(ncolors * (w / 2 + 2)) * sizeof(node_t));
    int i = 0;
    for (int y = 0; y < h; y++) {
        for (int x = 0; x < w; x++) {
            const int pix = index[(long)y * w + x];
            if (pix < ncolors) map[(long)pix * w + x] |= (uint8_t)(1 << i);
        }
        if (++i < 6 && (y + 1) < h) continue;
        node_t *top = NULL; int npool = 0;
        for (int c = 0; c < ncolors; c++) {
            const uint8_t *m = map + (long)c * w;
            for (int sx = 0; sx < w; sx++) {
                if (m[sx] == 0) continue;
                int mx;
                for (mx = sx + 1; mx < w; mx++) {
                    if (m[mx] != 0) continue;
                    int n;
                    for (n = 1; (mx + n) < w; n++) if (m[mx + n] != 0) break;
                    if (n >= 10 || (mx + n) >= w) break;
                    mx = mx + n - 1;
                }
                node_t *np = &pool[npool++];
                np->pal = c; np->sx = sx; np->mx = mx; np->map = m;
                node_t head; head.next = top; node_t *tp = &head;
                while (tp->next != NULL) {
                    if (np->sx < tp->next->sx) break;
                    else if (np->sx == tp->next->sx && np->mx > tp->next->mx) break;
                    tp = tp->next;
                }
                np->next = tp->next; tp->next = np; top = head.next;
                sx = mx - 1;
            }
        }
        if (y != 5) e_putc(e, '-');                                        /* DECGNL before every band but the first */
        for (int x = 0; top != NULL;) {
            node_t *np = top;
            if (x > np->sx) { e_putc(e, '$'); x = 0; }                      /* DECGCR */
            x = put_node(e, x, np);
            top = np->next;                                                /* np was the head */
            node_t **link = &top;
            while (*link != NULL) {
                if ((*link)->sx < x) { link = &(*link)->next; continue; }
                node_t *q = *link;
                x = put_node(e, x, q);
                *link = q->next;                                           /* delete q */
                link = &top;                                               /* rescan from the top */
            }
        }
        i = 0;
        memset(map, 0, (size_t)ncolors * w);
    }
    e_putc(e, 033); e_putc(e, '\\');                                       /* sixel_encode_footer */
    free(map); free(pool);
    return E.overflow ? -1 : (long)(E.p - out);
}

/* ---- the device's byte stream (timg_b200/csrc/sixel.cu, sixel_emit.cu) ----
 * The same header, palette definitions and ST as encode_body; a band, though, is written colour by colour instead of
 * in libsixel's node order.  Within each 6-row band, for every colour present, in ascending order: '$' (except before
 * the band's first colour), "#c", then every run of that colour (consecutive columns with the same row bits) as its
 * gap of blank columns since the colour's previous run (or since x = 0) followed by the run itself, each written as
 * "!n" + character when longer than 3 and as repeated characters otherwise.  '-' goes between bands.
 * index: w*h palette indices; palette: ncolors RGB triples.  Returns bytes written, or -1 if cap was too small. */
static void put_rep(emit_t *e, int n, int ch) {
    if (n > 3) { e_putc(e, '!'); e_putnum(e, n); e_putc(e, ch); }
    else for (int k = 0; k < n; k++) e_putc(e, ch);
}

long orc_sixel_stream(const uint8_t *index, int w, int h, const uint8_t *palette, int ncolors, char *out, long cap) {
    emit_t E = { out, out + cap, 0, 0, -1, 0 };
    emit_t *e = &E;
    put_header(e, w, h, palette, ncolors);
    uint8_t *bits = (uint8_t *)malloc((size_t)256 * w);       /* [colour][x]: the band's rows of that colour */
    for (int y0 = 0; y0 < h; y0 += 6) {
        memset(bits, 0, (size_t)256 * w);
        for (int r = 0; r < 6 && y0 + r < h; r++)
            for (int x = 0; x < w; x++) bits[(size_t)index[(long)(y0 + r) * w + x] * w + x] |= (uint8_t)(1 << r);
        if (y0 > 0) e_putc(e, '-');
        int first = 1;
        for (int c = 0; c < 256; c++) {
            const uint8_t *m = bits + (size_t)c * w;
            int end = 0;                                       /* one past the colour's previous run */
            for (int x = 0; x < w;) {
                if (!m[x]) { x++; continue; }
                if (end == 0) {                                /* the colour's first run in this band */
                    if (!first) e_putc(e, '$');
                    e_putc(e, '#'); e_putnum(e, c);
                    first = 0;
                }
                int x1 = x + 1;
                while (x1 < w && m[x1] == m[x]) x1++;
                put_rep(e, x - end, '?');
                put_rep(e, x1 - x, '?' + m[x]);
                end = x = x1;
            }
        }
    }
    free(bits);
    e_putc(e, 033); e_putc(e, '\\');
    return E.overflow ? -1 : (long)(E.p - out);
}

/* RGBA8 in (alpha dropped: sixel_helper_normalize_pixelformat RGBA8888 -> RGB888).
 * palette_out: 768 bytes or NULL; index_out: w*h bytes or NULL.
 * Returns bytes written, or -1 if cap was too small. */
long orc_sixel_encode(const uint8_t *rgba, int w, int h, int mode, char *out, long cap, uint8_t *palette_out,
                      int *ncolors_out, int *origcolors_out, uint8_t *index_out) {
    const long npix = (long)w * h;
    uint8_t *rgb = (uint8_t *)malloc((size_t)npix * 3);
    for (long i = 0; i < npix; i++) { rgb[3 * i] = rgba[4 * i]; rgb[3 * i + 1] = rgba[4 * i + 1]; rgb[3 * i + 2] = rgba[4 * i + 2]; }
    uint8_t palette[768]; int orig = 0;
    const int ncolors = make_palette(rgb, npix, palette, &orig, mode);
    /* sixel_dither_initialize: origcolors <= reqcolors switches diffusion off */
    const int diffuse = orig > 256;
    uint8_t *index = (uint8_t *)malloc((size_t)npix);
    apply_palette(rgb, w, h, palette, ncolors, diffuse, index, mode);
    const long n = encode_body(index, w, h, palette, ncolors, out, cap);
    if (palette_out) memcpy(palette_out, palette, 768);
    if (ncolors_out) *ncolors_out = ncolors;
    if (origcolors_out) *origcolors_out = orig;
    if (index_out) memcpy(index_out, index, (size_t)npix);
    free(rgb); free(index);
    return n;
}

/* Palette only (for comparing the device median cut with the restatement). */
int orc_sixel_palette(const uint8_t *rgba, int w, int h, int mode, uint8_t *palette_out, int *origcolors_out) {
    const long npix = (long)w * h;
    uint8_t *rgb = (uint8_t *)malloc((size_t)npix * 3);
    for (long i = 0; i < npix; i++) { rgb[3 * i] = rgba[4 * i]; rgb[3 * i + 1] = rgba[4 * i + 1]; rgb[3 * i + 2] = rgba[4 * i + 2]; }
    int orig = 0;
    const int n = make_palette(rgb, npix, palette_out, &orig, mode);
    if (origcolors_out) *origcolors_out = orig;
    free(rgb);
    return n;
}

/* ---- a small DEC sixel decoder (VT340 semantics for the subset any encoder here emits):
 * DCS P1;P2;P3 q  "Pan;Pad;Ph;Pv  #n;2;r;g;b  #n  ?..~  !n c  $  -  ST.
 * rgb_out: w*h*3 (w,h from the raster attributes, which must be present); unpainted pixels are
 * 0,0,0.  Returns 0, or negative on malformed input. */
int orc_sixel_decode(const char *s, long len, uint8_t *rgb_out, long cap_px, int *w_out, int *h_out,
                     int *colors_used) {
    long i = 0;
    if (len < 4 || s[0] != 033 || s[1] != 'P') return -1;
    i = 2;
    while (i < len && s[i] != 'q') i++;
    if (i >= len) return -2;
    i++;
    int pal[256][3]; memset(pal, 0, sizeof pal);
    uint8_t used[256]; memset(used, 0, sizeof used);
    int w = 0, h = 0, x = 0, band = 0, cur = 0, rep = 1;
    while (i < len) {
        const unsigned char ch = (unsigned char)s[i];
        if (ch == 033) break;
        if (ch == '"') {
            int v[4] = {0, 0, 0, 0}, k = 0; i++;
            while (i < len && ((s[i] >= '0' && s[i] <= '9') || s[i] == ';')) {
                if (s[i] == ';') k++; else if (k < 4) v[k] = v[k] * 10 + (s[i] - '0');
                i++;
            }
            w = v[2]; h = v[3];
            if ((long)w * h > cap_px) return -3;
            memset(rgb_out, 0, (size_t)w * h * 3);
            continue;
        }
        if (ch == '#') {
            int v[5] = {0, 0, 0, 0, 0}, k = 0; i++;
            while (i < len && ((s[i] >= '0' && s[i] <= '9') || s[i] == ';')) {
                if (s[i] == ';') k++; else if (k < 5) v[k] = v[k] * 10 + (s[i] - '0');
                i++;
            }
            if (v[0] > 255) return -4;
            cur = v[0];
            if (k >= 4 && v[1] == 2) { pal[cur][0] = v[2] * 255 / 100; pal[cur][1] = v[3] * 255 / 100; pal[cur][2] = v[4] * 255 / 100; }
            continue;
        }
        if (ch == '!') {
            rep = 0; i++;
            while (i < len && s[i] >= '0' && s[i] <= '9') { rep = rep * 10 + (s[i] - '0'); i++; }
            continue;
        }
        if (ch == '$') { x = 0; i++; continue; }
        if (ch == '-') { x = 0; band++; i++; continue; }
        if (ch >= '?' && ch <= '~') {
            const int bits = ch - '?';
            if (!w || !h) return -5;
            for (int r = 0; r < rep; r++, x++) {
                if (x >= w) continue;
                for (int b = 0; b < 6; b++)
                    if (bits & (1 << b)) {
                        const int y = band * 6 + b;
                        if (y < h) { uint8_t *p = rgb_out + ((long)y * w + x) * 3; p[0] = (uint8_t)pal[cur][0]; p[1] = (uint8_t)pal[cur][1]; p[2] = (uint8_t)pal[cur][2]; used[cur] = 1; }
                    }
            }
            rep = 1; i++;
            continue;
        }
        i++;   /* ignore anything else (newlines etc) */
    }
    if (i + 1 >= len || s[i] != 033 || s[i + 1] != '\\') return -6;
    int nu = 0; for (int k = 0; k < 256; k++) nu += used[k];
    *w_out = w; *h_out = h; if (colors_used) *colors_used = nu;
    return 0;
}
