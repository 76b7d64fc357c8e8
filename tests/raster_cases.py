"""BMP, TGA and binary PNM files for the raster decoder's tests, built deterministically, and a plan model of how
raster.cu cuts an RLE TGA's packet stream.

corpus(): (name, bytes) of ordinary files of every layout and of each stb quirk the device reproduces.
rejections(): (name, bytes, outcome) of damaged headers: 'einval' (stb's source fails), 'unsupported' (the parse
takes the file but the device does not) or 'ok'.
tile_cases(): (name, bytes, where) of RLE streams aimed at the tile, chunk and super-chunk edges; `where` names the
stream offsets the model says a packet header must sit on, and test_raster_parse.py checks it.

The model: the packet stream is the bytes [data, size) of the file; tiles of TILE bytes, CHUNK tiles to a chunk and
CHUNK chunks to a super-chunk; a tile map has P entry bytes.  These mirror the constexprs of raster.cu.
"""
import numpy as np

from oracle import raster as R
import png_cases as pc

TILE, P, CHUNK = 1024, 513, 32
LAUNCHES = 7
TGA_HEADER = 18


def photo(w, h, seed, ch=3):
    return pc.photo(w, h, seed, ch=ch) if ch != 3 else pc.photo(w, h, seed)


def indices(w, h, n, seed):
    return np.random.default_rng(seed).integers(0, n, (h, w)).astype(np.uint8)


def palette(n, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, 3)).astype(np.uint8)


def rgba(a):
    a = np.asarray(a, np.uint8)
    return a if a.shape[-1] == 4 else np.concatenate([a, np.full(a.shape[:2] + (1,), 255, np.uint8)], -1)


# ---- BMP ---------------------------------------------------------------------------------------------------------
def bmps():
    img = photo(37, 23, 1)
    yield "bmp24_h40", R.bmp(img, 24)
    yield "bmp24_top_down", R.bmp(img, 24, top_down=True)
    yield "bmp24_h12_os2", R.bmp(img, 24, hsz=12)
    yield "bmp24_h56", R.bmp(img, 24, hsz=56)
    yield "bmp24_h108", R.bmp(img, 24, hsz=108)
    yield "bmp24_h124", R.bmp(img, 24, hsz=124)
    yield "bmp24_gap_twice", R.bmp(img, 24, gap=20)                       # the gap is skipped twice
    yield "bmp24_h12_gap_twice", R.bmp(img, 24, hsz=12, gap=7)
    yield "bmp24_ma_ff000000", R.bmp(img, 24, hsz=108, masks=(0, 0, 0, 0xFF000000), fields=dict(compress=-1))
    a = photo(29, 17, 2, ch=4)
    yield "bmp32_alpha", R.bmp(a, 32)
    zero = a.copy(); zero[..., 3] = 0
    yield "bmp32_alpha_all_zero", R.bmp(zero, 32)                          # all_a: alpha becomes 255
    yield "bmp32_h108_alpha_all_zero", R.bmp(zero, 32, hsz=108)            # defaults ran: 255
    yield "bmp32_h108_bitfields_alpha_zero", R.bmp(zero, 32, hsz=108, compress=3,
                                                   masks=(0xFF0000, 0xFF00, 0xFF, 0xFF000000))   # stays 0
    yield "bmp32_h40_bitfields_rgb", R.bmp(a, 32, masks=(0xFF0000, 0xFF00, 0xFF, 0))
    yield "bmp32_h124_masks_abgr", R.bmp(a, 32, hsz=124, compress=3, masks=(0xFF, 0xFF00, 0xFF0000, 0xFF000000))
    yield "bmp32_h108_4bit_masks", R.bmp(a, 32, hsz=108, compress=3, masks=(0xF000, 0x0F00, 0x00F0, 0x000F))
    yield "bmp16_555", R.bmp(img, 16)
    yield "bmp16_565_bitfields", R.bmp(img, 16, masks=(0xF800, 0x07E0, 0x001F, 0))
    yield "bmp16_h108_4444", R.bmp(a, 16, hsz=108, compress=3, masks=(0x0F00, 0x00F0, 0x000F, 0xF000))
    yield "bmp16_noncontiguous", R.bmp(img, 16, masks=(0x5400, 0x02A0, 0x0015, 0))
    yield "bmp32_noncontiguous_alpha", R.bmp(a, 32, hsz=108, compress=3,
                                             masks=(0x00AA0000, 0x0000CC00, 0x000000F0, 0x55000000))
    for bpp, n in ((1, 2), (4, 16), (8, 256)):
        for w in (1, 7, 13, 33):
            yield f"bmp{bpp}_w{w}", R.bmp(indices(w, 9, n, w + bpp), bpp, palette=palette(n, bpp))
    yield "bmp8_small_palette", R.bmp(indices(21, 6, 12, 3), 8, palette=palette(12, 5))
    # a 12-byte header's psize is (offset - 38) / 3: 4 entries short of the palette written, so indices 36-39 of 40
    # read stb's uninitialised pal[] (status -1) and indices below 36 decode
    yield "bmp8_h12_os2", R.bmp(indices(15, 8, 36, 4), 8, hsz=12, palette=palette(40, 6))
    yield "bmp8_h12_os2_last_entries", R.bmp(indices(15, 8, 40, 4), 8, hsz=12, palette=palette(40, 6))
    yield "bmp4_h124_gap", R.bmp(indices(15, 8, 16, 4), 4, hsz=124, palette=palette(16, 7), gap=9)
    yield "bmp8_top_down", R.bmp(indices(17, 5, 256, 8), 8, palette=palette(256, 9), top_down=True)
    full = R.bmp(photo(40, 30, 3), 24)
    yield "bmp24_truncated", full[:len(full) // 2 + 3]                     # the rest reads as 0
    yield "bmp24_header_only", full[:54]
    p8 = R.bmp(indices(30, 10, 256, 10), 8, palette=palette(256, 11))
    yield "bmp8_truncated_palette", p8[:54 + 300]
    # palette index at or past psize: stb reads its uninitialised pal[] (status -1)
    yield "bmp8_index_past_psize", R.bmp(np.array([[0, 1, 2, 3, 9, 1]], np.uint8), 8, palette=palette(4, 12))
    yield "bmp1_psize_1", R.bmp(np.array([[0, 1, 0]], np.uint8), 1, palette=palette(1, 13))
    yield "bmp1_psize_1_all_0", R.bmp(np.zeros((3, 5), np.uint8), 1, palette=palette(1, 13))
    yield "bmp8_psize_negative", R.bmp(np.zeros((2, 4), np.uint8), 8, palette=palette(4, 14), offset=50)
    yield "bmp8_h12_psize_negative", R.bmp(np.zeros((2, 4), np.uint8), 8, hsz=12, offset=30)


# ---- TGA ---------------------------------------------------------------------------------------------------------
def _bgr(img):
    img = np.asarray(img, np.uint8)
    return img[..., [2, 1, 0] + ([3] if img.shape[-1] == 4 else [])]


def _rgb16(img):
    img = np.asarray(img, np.uint16)
    v = (img[..., 0] >> 3) << 10 | (img[..., 1] >> 3) << 5 | img[..., 2] >> 3 | 0x8000
    return v.astype("<u2")


def _file_order(img, top):
    return img if top else img[::-1]


def tga_file(img, rle):
    """A bottom-up 24-bit TGA of an RGB image, raw (type 2) or RLE (type 10)."""
    h, w = img.shape[:2]
    raw = _bgr(_file_order(img, False)).tobytes()
    return R.tga(w, h, R.rle_encode(raw, 3) if rle else raw, 10 if rle else 2, 24)


def tgas():
    img = photo(31, 19, 21)
    a = photo(23, 15, 22, ch=4)
    g = indices(27, 11, 256, 23)
    yield "tga2_24_bottom_up", R.tga(31, 19, _bgr(_file_order(img, False)).tobytes(), 2, 24)
    yield "tga2_24_top_down", R.tga(31, 19, _bgr(img).tobytes(), 2, 24, desc=0x20)
    yield "tga2_24_right_to_left", R.tga(31, 19, _bgr(img).tobytes(), 2, 24, desc=0x30)
    yield "tga2_32", R.tga(23, 15, _bgr(_file_order(a, False)).tobytes(), 2, 32, desc=8)
    yield "tga2_16", R.tga(31, 19, _rgb16(img).tobytes(), 2, 16)
    yield "tga2_15", R.tga(31, 19, _rgb16(img).tobytes(), 2, 15, desc=0x20)
    yield "tga2_8_grey", R.tga(27, 11, g.tobytes(), 2, 8)
    yield "tga3_8", R.tga(27, 11, g.tobytes(), 3, 8, desc=0x20)
    yield "tga3_16_grey_alpha", R.tga(27, 11, np.stack([g, 255 - g], -1).tobytes(), 3, 16)
    yield "tga3_15_as_rgb16", R.tga(31, 19, _rgb16(img).tobytes(), 3, 15)
    yield "tga3_24_bgr", R.tga(31, 19, img.tobytes(), 3, 24)
    yield "tga2_24_id_field", R.tga(31, 19, _bgr(img).tobytes(), 2, 24, ident=b"oracle id field")
    yield "tga2_24_cmap_fields_ignored", R.tga(31, 19, _bgr(img).tobytes(), 2, 24, cmap=0, pal_len=7, pal_bits=24)
    pal = palette(200, 24)
    idx = indices(27, 11, 230, 25)                                         # indices >= 200 read entry 0
    yield "tga1_8_pal24", R.tga(27, 11, idx.tobytes(), 1, 8, palette=_bgr(pal).tobytes(), pal_len=200, pal_bits=24)
    yield "tga1_8_pal24_start5", R.tga(27, 11, idx.tobytes(), 1, 8, palette=bytes(5) + _bgr(pal).tobytes(),
                                       pal_len=200, pal_bits=24, pal_start=5)
    pal4 = np.concatenate([pal, np.arange(200, dtype=np.uint8)[:, None]], -1)
    yield "tga1_8_pal32", R.tga(27, 11, idx.tobytes(), 1, 8, palette=_bgr(pal4).tobytes(), pal_len=200, pal_bits=32)
    yield "tga1_8_pal8", R.tga(27, 11, idx.tobytes(), 1, 8, palette=pal[:, 0].tobytes(), pal_len=200, pal_bits=8)
    idx16 = np.random.default_rng(26).integers(0, 320, (11, 27)).astype("<u2")
    pal16 = _rgb16(palette(300, 27)).tobytes()
    yield "tga1_16_pal16", R.tga(27, 11, idx16.tobytes(), 1, 16, palette=pal16, pal_len=300, pal_bits=16)
    yield "tga1_16_pal15_cut", R.tga(27, 11, idx16.tobytes(), 1, 16, palette=pal16, pal_len=300, pal_bits=15)[:400]
    yield "tga1_8_cut_raster", R.tga(27, 11, idx.tobytes(), 1, 8, palette=_bgr(pal).tobytes(), pal_len=200,
                                     pal_bits=24)[:18 + 600 + 100]
    yield "tga2_16_cut", R.tga(31, 19, _rgb16(img).tobytes(), 2, 16)[:500]
    # RLE
    for bpp, B, vals in ((24, 3, _bgr(_file_order(img, False))), (32, 4, _bgr(_file_order(a, False)))):
        hh, ww = vals.shape[:2]
        yield f"tga10_{bpp}", R.tga(ww, hh, R.rle_encode(vals.tobytes(), B), 10, bpp)
    flat = np.repeat(np.repeat(photo(8, 6, 28), 5, 0), 7, 1)               # long runs across rows
    yield "tga10_24_runs", R.tga(56, 30, R.rle_encode(_bgr(flat).tobytes(), 3), 10, 24, desc=0x20)
    yield "tga10_16", R.tga(31, 19, R.rle_encode(_rgb16(img).tobytes(), 2), 10, 16)
    yield "tga11_8", R.tga(27, 11, R.rle_encode(np.repeat(g, 3, 1)[:, :27].tobytes(), 1), 11, 8)
    yield "tga11_16_grey_alpha", R.tga(27, 11, R.rle_encode(np.stack([g, g], -1).tobytes(), 2), 11, 16)
    yield "tga9_8_pal24", R.tga(27, 11, R.rle_encode(np.repeat(idx, 2, 1)[:, :27].tobytes(), 1), 9, 8,
                                palette=_bgr(pal).tobytes(), pal_len=200, pal_bits=24)
    yield "tga9_16_pal16", R.tga(27, 11, R.rle_encode(idx16.tobytes(), 2), 9, 16, palette=pal16, pal_len=300, pal_bits=16)
    o = R.Rle(3).run(128, b"\x01\x02\x03").raw(bytes(range(30))).run(100, b"\x09\x08\x07").run(128, b"\xff\x00\x80")
    yield "tga10_past_image_end", R.tga(10, 20, o.bytes(), 10, 24)       # 268 pixels of packets for 200
    stream = R.rle_encode(_bgr(img).tobytes(), 3)
    yield "tga10_cut_stream", R.tga(31, 19, stream[:len(stream) // 2], 10, 24)   # then 1-pixel raw packets of zeros
    yield "tga10_cut_mid_packet", R.tga(4, 4, R.Rle(3).raw(bytes(range(24))).bytes()[:10], 10, 24)
    yield "tga10_empty_stream", R.tga(5, 3, b"", 10, 24)
    yield "tga10_id_field", R.tga(31, 19, stream, 10, 24, ident=bytes(range(255)))


# ---- PNM ---------------------------------------------------------------------------------------------------------
def pnms():
    g = indices(33, 21, 256, 31)
    c = photo(29, 13, 32)
    yield "p5_8", R.pnm(g)
    yield "p6_8", R.pnm(c)
    g16 = np.random.default_rng(33).integers(0, 65536, (21, 33))
    yield "p5_16", R.pnm(g16, 65535)
    yield "p6_16", R.pnm(np.random.default_rng(34).integers(0, 1000, (13, 29, 3)), 1000)
    yield "p5_16_example", b"P5 2 1 65535\n\x12\x34\x56\x78"
    yield "p5_maxval_1", R.pnm(g & 1, 1)
    yield "p6_comments", R.pnm(c, header=b"P6#a\n# comment one\n 29 #two\r13\n#three\n255\n")
    yield "p5_tab_ws", R.pnm(g, header=b"P5\t33\v21\f255\r")
    yield "p5_raster_after_one_char", R.pnm(g, header=b"P5 33 21 255 ")            # the raster starts at the next byte
    yield "p5_raster_after_hash", R.pnm(g, header=b"P5 33 21 255#")
    yield "p5_maxval_0", R.pnm(g, header=b"P5 33 21 0\n")
    yield "p5_maxval_overflow", R.pnm(g, header=b"P5 33 21 9999999999")    # stb's error value 0: 8 bits, mid-number
    yield "p6_trailing_bytes", R.pnm(c) + b"trailing"
    yield "p5_1x1", b"P5 1 1 255 \x7f"


def corpus():
    yield from bmps()
    yield from tgas()
    yield from pnms()


# ---- damaged headers -----------------------------------------------------------------------------------------------
def rejections():
    img = photo(6, 4, 41)
    p8 = indices(6, 4, 4, 42)
    pal = palette(4, 43)
    yield "bmp_size_17", R.bmp(img, 24)[:17], "einval"
    yield "bmp_hsz_64", R.bmp(img, 24, fields=dict(hsz=64)), "einval"
    yield "bmp_planes_2", R.bmp(img, 24, planes=2), "einval"
    yield "bmp_rle8", R.bmp(p8, 8, palette=pal, fields=dict(compress=1)), "einval"
    yield "bmp_rle4", R.bmp(p8, 4, palette=pal, fields=dict(compress=2)), "einval"
    yield "bmp_jpeg", R.bmp(img, 24, fields=dict(compress=4)), "einval"
    yield "bmp_bitfields_24", R.bmp(img, 24, fields=dict(compress=3)), "einval"
    yield "bmp_masks_equal", R.bmp(img, 16, masks=(0x7C00, 0x7C00, 0x7C00, 0)), "einval"
    yield "bmp_mask_zero", R.bmp(img, 16, masks=(0x7C00, 0, 0x1F, 0)), "einval"
    yield "bmp_mask_9_bits", R.bmp(img, 32, masks=(0x1FF0000, 0xFF00, 0xFF, 0)), "einval"
    yield "bmp_alpha_mask_9_bits", R.bmp(img, 32, hsz=108, compress=3, masks=(0xFF0000, 0xFF00, 0xFF, 0xFF800000)), "einval"
    yield "bmp_h12_16bpp", R.bmp(img, 16, hsz=12), "einval"
    yield "bmp_h40_compress_neg", R.bmp(img, 16, fields=dict(compress=-1)), "einval"
    yield "bmp_psize_0", R.bmp(p8, 8, palette=None), "einval"
    yield "bmp_psize_257", R.bmp(p8, 8, palette=palette(257, 44)), "einval"
    yield "bmp_psize_256", R.bmp(p8, 8, palette=palette(256, 44)), "ok"
    yield "bmp_bpp_2", R.bmp(p8, 8, palette=pal, fields=dict(bpp=2)), "einval"
    yield "bmp_offset_negative", R.bmp(img, 24, offset=-1), "einval"
    yield "bmp_offset_before_header", R.bmp(img, 24, offset=53), "einval"
    yield "bmp_offset_gap_1024", R.bmp(img, 24, offset=54 + 1024), "ok"
    yield "bmp_offset_gap_1025", R.bmp(img, 24, offset=54 + 1025), "einval"
    yield "bmp_w_2_24", R.bmp(img, 24, size=(1 << 24, 1)), "ok"
    yield "bmp_w_2_24_plus_1", R.bmp(img, 24, size=((1 << 24) + 1, 1)), "einval"
    yield "bmp_h_neg_2_24_plus_1", R.bmp(img, 24, size=(1, (1 << 24) + 1), top_down=True), "einval"
    yield "bmp_area_2_29", R.bmp(img, 24, size=(1 << 15, 1 << 14)), "einval"        # 4*w*h > INT_MAX
    yield "bmp_area_below", R.bmp(img, 24, size=(1 << 15, (1 << 14) - 1)), "ok"
    yield "bmp_w_0", R.bmp(img, 24, size=(0, 4)), "unsupported"
    yield "bmp_h_0", R.bmp(img, 24, size=(6, 0)), "unsupported"
    raw = _bgr(img).tobytes()
    yield "tga_cmap_type_2", R.tga(6, 4, raw, 2, 24, cmap=2), "einval"
    yield "tga_type_4", R.tga(6, 4, raw, 4, 24), "einval"
    yield "tga_type_1_no_cmap", R.tga(6, 4, raw, 1, 8, cmap=0), "einval"
    yield "tga_type_2_with_cmap", R.tga(6, 4, raw, 2, 24, cmap=1, pal_bits=24), "einval"
    yield "tga_bpp_12", R.tga(6, 4, raw, 2, 12), "einval"
    yield "tga_pal_bits_12", R.tga(6, 4, p8.tobytes(), 1, 8, palette=bytes(12), pal_len=4, pal_bits=12), "einval"
    yield "tga_indexed_bpp_24", R.tga(6, 4, raw, 1, 24, palette=bytes(12), pal_len=4, pal_bits=24), "einval"
    yield "tga_w_0", R.tga(0, 4, raw, 2, 24), "einval"
    yield "tga_h_0", R.tga(6, 0, raw, 2, 24), "einval"
    yield "tga_pal_len_0", R.tga(6, 4, p8.tobytes(), 1, 8, palette=b"", pal_len=0, pal_bits=24), "einval"
    yield "tga_pal_truncated", R.tga(6, 4, b"", 1, 8, palette=bytes(11), pal_len=4, pal_bits=24), "einval"
    yield "tga_pal_exact", R.tga(6, 4, b"", 1, 8, palette=bytes(12), pal_len=4, pal_bits=24), "ok"
    yield "tga_raw_cut", R.tga(6, 4, raw[:-1], 2, 24), "unsupported"
    yield "tga_raw_exact", R.tga(6, 4, raw, 2, 24), "ok"
    yield "tga_area_2_29", R.tga(32768, 16384, b"", 10, 24), "einval"
    yield "tga_area_below", R.tga(32768, 16383, b"", 10, 24), "ok"
    g = indices(6, 4, 256, 45)
    yield "pnm_p3", R.pnm(g, header=b"P3 6 4 255\n"), "einval"
    yield "pnm_w_0", R.pnm(g, header=b"P5 0 4 255\n"), "einval"
    yield "pnm_h_0", R.pnm(g, header=b"P5 6 0 255\n"), "einval"
    yield "pnm_w_overflow", R.pnm(g, header=b"P5 2147483648 4 255\n"), "einval"
    yield "pnm_w_2147483647", R.pnm(g, header=b"P5 2147483647 4 255\n"), "einval"      # past STBI_MAX_DIMENSIONS
    yield "pnm_maxval_65536", R.pnm(g, header=b"P5 6 4 65536\n"), "einval"
    yield "pnm_maxval_65535_cut", R.pnm(g, header=b"P5 6 4 65535\n"), "einval"          # 48 bytes of 24 * 2
    yield "pnm_truncated", R.pnm(g, header=b"P5 6 4 255\n")[:-1], "einval"
    yield "pnm_no_raster", b"P5 6 4 255", "einval"
    yield "pnm_16bit_2_28_px", R.pnm(np.zeros((1, 1), np.uint8), header=b"P5 16384 16384 65535\n"), "einval"
    yield "pnm_8bit_area_2_29", R.pnm(np.zeros((1, 1), np.uint8), header=b"P5 32768 16384 255\n"), "einval"


def unsupported_big():
    """(name, header bytes, file size, outcome) for parse-only checks of files too large to build: the walk reads only
    the header, so the file is the header padded by b200timg_raster_parse's size argument."""
    yield "pnm_16bit_2_28_px", b"P5 16384 16384 65535\n", 21 + 16384 * 16384 * 2, "unsupported"
    yield "pnm_16bit_below", b"P5 16383 16384 65535\n", 21 + 16383 * 16384 * 2, "ok"
    yield "pnm_8bit_area_2_29", b"P5 32768 16384 255\n", 19 + 32768 * 16384, "einval"


# ---- RLE tile model ------------------------------------------------------------------------------------------------
def packet_starts(data, B):
    """Stream offsets (from the packet stream's first byte, 18 + id length) of every packet header before the end."""
    s = data[TGA_HEADER + data[0]:]
    out, pos = [], 0
    while pos < len(s):
        out.append(pos)
        c = s[pos]
        pos += 1 + (B if c & 128 else ((c & 127) + 1) * B)
    return out


def _rle_file(o, w):
    npx = sum(((o.b[s] & 127) + 1) for s in o.starts)
    h = max(1, npx // w)
    return R.tga(w, h, o.bytes(), 10, 8 * o.B)


def tile_cases():
    """(name, bytes, where): where = dict(header_at=[stream offsets that must start a packet], B=bytes per value)."""
    out = []
    for B in (1, 3, 4):
        v = bytes(range(1, B + 1))
        # a header on the first and on the last byte of a tile, and at a chunk and a super-chunk edge: 1-pixel raw
        # packets (1 + B bytes) up to the edge - k, then one filler packet of the length that lands there
        for edge, tag in ((TILE, "tile"), (CHUNK * TILE, "chunk")):
            for k in (0, 1):
                # one raw packet of n pixels, then runs of 1 + B bytes, land a header exactly on the edge - k
                o, target = R.Rle(B), edge - k
                n = (1 - target) % (1 + B) or 1 + B
                o.raw(bytes(range(n * B)))
                while len(o.b) < target:
                    o.run(1 + len(o.starts) % 128, v)
                for i in range(40):
                    o.run(1 + i % 128, v) if i % 2 else o.raw(bytes([i & 0x7F]) * (B * (1 + i % 5)))
                out.append((f"rle_B{B}_{tag}_edge_minus{k}", _rle_file(o, 97), dict(header_at=[target], B=B)))
        # the densest chain: runs of B + 1 bytes, across three chunks
        o = R.Rle(B)
        for i in range(3 * CHUNK * TILE // (B + 1)):
            o.run(1 + i % 128, bytes([(i * 7 + j) & 255 for j in range(B)]))
        out.append((f"rle_B{B}_densest", _rle_file(o, 1000), dict(header_at=[0], B=B)))
        # the sparsest: 128-pixel raw packets (1 + 128 B bytes) whose bytes look like headers, across two chunks
        o = R.Rle(B)
        rng = np.random.default_rng(50 + B)
        while len(o.b) < 2 * CHUNK * TILE + 3 * TILE:
            o.raw(rng.integers(0, 256, 128 * B, dtype=np.uint8).tobytes())
        out.append((f"rle_B{B}_sparsest", _rle_file(o, 512), dict(header_at=[0], B=B)))
    # packets across the first super-chunk edge
    o = R.Rle(3)
    rng = np.random.default_rng(60)
    while len(o.b) < CHUNK * CHUNK * TILE + 5 * TILE:
        n = int(rng.integers(1, 129))
        o.run(n, rng.integers(0, 256, 3, dtype=np.uint8).tobytes()) if rng.integers(0, 2) else \
            o.raw(rng.integers(0, 256, 3 * n, dtype=np.uint8).tobytes())
    out.append(("rle_B3_super_edge", _rle_file(o, 2048), dict(header_at=[0], B=3, spans_super=True)))
    return out


def front_files(k):
    """k ordinary files of the three formats to put in front of a case in one call."""
    kinds = [lambda i: R.bmp(photo(20 + i, 11 + i, 70 + i), 24),
             lambda i: R.tga(17 + i, 9, R.rle_encode(_bgr(photo(17 + i, 9, 80 + i)).tobytes(), 3), 10, 24),
             lambda i: R.pnm(photo(13 + i, 7 + i, 90 + i))]
    return [kinds[i % 3](i) for i in range(k)]


def golden():
    """(name, bytes, parse, sha, status, frame_sha, (frame_w, frame_h)) per pinned case from tests/golden/raster.npz.
    parse: 1 decoded, 0 parsed only, -1 rejected."""
    import os
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "raster.npz"))
    files = dict(all_files())
    return [(str(n), files[str(n)], int(p), str(s), int(st), str(fs), (int(fw), int(fh)))
            for n, p, s, st, fs, fw, fh in zip(z["name"], z["parse"], z["sha"], z["status"], z["frame_sha"],
                                               z["frame_w"], z["frame_h"])]


def all_files():
    yield from corpus()
    for name, data, _ in rejections():
        yield name, data
    for name, data, _ in tile_cases():
        yield name, data


DECODED_MAX_PX = 1 << 22          # files past this are pinned by their parse only
FRAME_OPTS = dict(width=40 * 9, height=20 * 18, cell=(9, 18), has_bg=True, bg=0xFF302010, pattern=0xFF808080,
                  pattern_size=2)
FRAME_CASES = ("bmp32_alpha", "bmp24_h40", "tga2_32", "tga10_24", "tga3_16_grey_alpha", "p6_8", "p5_16")
