"""PNG files for the device decoder's tests: Pillow-written files, oracle/png.py files covering every colour type x bit
depth, filters, Adam7, tRNS, chunk placement, zlib settings, hand-made deflate streams, and damaged copies."""
import functools
import io
import zlib

import numpy as np
from PIL import Image

from oracle import png as W

DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}


def photo(w, h, seed=0, ch=3):
    """Smooth gradients plus noise: what a photo looks like to the filters and the entropy coder."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    a = np.stack([x * 255 // max(1, w - 1), y * 255 // max(1, h - 1), ((x + 2 * y) * 3) % 256, (x * y) % 256][:ch], -1)
    return (a + rng.integers(-24, 25, a.shape)).clip(0, 255).astype(np.uint8)


def screenshot(w, h, seed=0):
    """Flat panels with glyph-like edges: what a terminal screenshot or a plot looks like."""
    rng = np.random.default_rng(seed)
    img = np.full((h, w, 3), 30, np.uint8)
    img[: h // 12] = (60, 60, 70)
    img[:, : w // 6] = (45, 45, 50)
    glyphs = rng.integers(0, 2, (h // 16, w // 8, 16, 8)).astype(bool) & (rng.random((h // 16, w // 8, 1, 1)) < 0.4)
    g = glyphs.transpose(0, 2, 1, 3).reshape(h // 16 * 16, w // 8 * 8)
    img[: g.shape[0], : g.shape[1]][g] = (220, 220, 210)
    return img


def pillow(img, mode="RGB", **kw):
    b = io.BytesIO()
    Image.fromarray(img).convert(mode).save(b, "PNG", **kw)
    return b.getvalue()


def _palette(n, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (n, 3))


def _px(color, depth, w, h, seed, pal_n=None):
    s = W.samples(w, h, color, depth, seed)
    if color == 3 and pal_n:
        s %= pal_n
    return s


def writer_cases():
    """(name, bytes) from oracle/png.py that the reference decodes (or fails) deterministically."""
    out = []
    for color, depths in DEPTHS.items():
        for depth in depths:
            for w, h, filters, il in ((1, 1, (0,), 0), (13, 7, (4, 3, 2, 1, 0), 0), (9, 11, (3, 4, 1, 2, 0), 1)):
                pal = _palette(1 << min(depth, 8), color * 16 + depth) if color == 3 else None
                s = _px(color, depth, w, h, depth + w, None if pal is None else len(pal))
                out.append((f"c{color}d{depth}_{w}x{h}_il{il}", W.png(s, depth, color, il, filters, plte=pal)))
    # filters on row 0 (Up, Avg, Paeth read a zero row) and filter type 5
    s = W.samples(17, 5, 2, 8, 1)
    for ft in range(5):
        out.append((f"row0_filter{ft}", W.png(s, 8, 2, 0, (ft, 4, 3))))
    out.append(("filter5", W.png(s, 8, 2, 0, (1, 5))))
    # stb takes depths the PNG spec does not allow for colour types 2, 4 and 6
    for color, depth in ((2, 4), (4, 2), (6, 1), (2, 1)):
        out.append((f"odd_c{color}d{depth}", W.png(W.samples(11, 6, color, depth, 3), depth, color, 0, (4, 1, 2))))
    # tRNS
    g8, g1, g16 = W.samples(12, 6, 0, 8, 4), W.samples(12, 6, 0, 1, 5), W.samples(12, 6, 0, 16, 6)
    out.append(("trns_grey8", W.png(g8, 8, 0, trns=int(g8[2, 3, 0]).to_bytes(2, "big"))))
    out.append(("trns_grey1_key1", W.png(g1, 1, 0, trns=b"\x00\x01")))
    out.append(("trns_grey2_key_high_byte", W.png(W.samples(12, 6, 0, 2, 7), 2, 0, trns=b"\x01\x02")))
    out.append(("trns_grey16", W.png(g16, 16, 0, trns=int(g16[1, 1, 0]).to_bytes(2, "big"))))
    rgb, rgb16 = W.samples(12, 6, 2, 8, 8), W.samples(12, 6, 2, 16, 9)
    out.append(("trns_rgb8", W.png(rgb, 8, 2, trns=b"".join(int(v).to_bytes(2, "big") for v in rgb[0, 0]))))
    out.append(("trns_rgb16", W.png(rgb16, 16, 2, trns=b"".join(int(v).to_bytes(2, "big") for v in rgb16[3, 4]))))
    out.append(("trns_rgb16_il", W.png(rgb16, 16, 2, 1, (4,), trns=b"".join(int(v).to_bytes(2, "big") for v in rgb16[0, 0]))))
    pal = _palette(16, 1)
    p4 = W.samples(12, 6, 3, 4, 10) % 16
    out.append(("trns_pal_partial", W.png(p4, 4, 3, plte=pal, trns=bytes([0, 64, 128]))))
    out.append(("trns_pal_full_il", W.png(p4, 4, 3, 1, (2, 4), plte=pal, trns=bytes(range(0, 256, 16)))))
    out.append(("trns_after_idat", W.png(g8, 8, 0, after_idat=[(b"tRNS", b"\x00\x01")])))
    out.append(("trns_before_plte", W.png(p4, 4, 3, plte=pal, before_idat=[(b"tRNS", b"\x00")])))
    out.append(("trns_too_long", W.png(p4, 4, 3, plte=pal, trns=bytes(17))))
    out.append(("trns_with_alpha", W.png(W.samples(5, 5, 4, 8, 1), 8, 4, trns=b"\x00\x01")))
    out.append(("trns_bad_len", W.png(g8, 8, 0, trns=b"\x00\x01\x02")))
    # a second PLTE after tRNS resets its entries' alpha; entries past it keep the first PLTE's values
    pal2 = _palette(8, 2)
    twice = W.png(p4, 4, 3, plte=pal, trns=bytes([10] * 16))
    i = twice.index(b"IDAT") - 4
    out.append(("plte_second_shorter", twice[:i] + W.chunk(b"PLTE", np.asarray(pal2, np.uint8).tobytes()) + twice[i:]))
    out.append(("plte_bad_len", W.png(p4, 4, 3, before_idat=[(b"PLTE", bytes(10))])))
    out.append(("pal_index_oob", W.png(p4, 4, 3, plte=pal[:5])))
    out.append(("pal_index_oob_filter5", W.png(p4, 4, 3, 0, (0, 5), plte=pal[:5])))
    out.append(("no_plte", W.png(p4, 4, 3)))
    # IDAT splits, CgBI, chunk placement, APNG
    for name, sizes in (("idat1", [1]), ("idat0_1_5", [0, 1, 5]), ("idat7", [7])):
        out.append((name, W.png(rgb, 8, 2, 0, (4, 1), idat_sizes=sizes)))
    zero_first = W.png(rgb, 8, 2, 0, (4,))
    i = zero_first.index(b"IDAT") - 4
    out.append(("idat_zero_then_trns", zero_first[:i] + W.chunk(b"IDAT") + W.chunk(b"tRNS", bytes(6)) + zero_first[i:]))
    out.append(("cgbi", W.png(rgb, 8, 2, 0, (1,), cgbi=True)))
    out.append(("cgbi_rgba", W.png(W.samples(12, 6, 6, 8, 3), 8, 6, 0, (4,), cgbi=True)))
    anc = [(b"tEXt", b"k\x00v"), (b"zzZz", b"\x01\x02")]
    out.append(("ancillary", W.png(rgb, 8, 2, before_idat=anc, after_idat=anc)))
    out.append(("unknown_critical", W.png(rgb, 8, 2, before_idat=[(b"ZZZZ", b"x")])))
    out.append(("apng", W.png(rgb, 8, 2, before_idat=[(b"acTL", bytes(8)), (b"fcTL", bytes(26))],
                              after_idat=[(b"fcTL", bytes(26)), (b"fdAT", bytes(4) + zlib.compress(b"\x00" * 40))])))
    out.append(("data_after_iend", W.png(rgb, 8, 2) + b"junk" * 5))
    out.append(("no_iend", W.png(rgb, 8, 2, iend=False)))
    out.append(("ihdr_twice", W.png(rgb, 8, 2, before_idat=[(b"IHDR", bytes(13))])))
    out.append(("no_idat", W.png(rgb, 8, 2, zdata=b"")))
    # zlib levels, strategies, window bits, data after the final block
    big = W.samples(40, 30, 2, 8, 11)
    for lv in range(10):
        out.append((f"level{lv}", W.png(big, 8, 2, 0, (lv % 5,), level=lv)))
    for nm, st in (("filtered", zlib.Z_FILTERED), ("huffman", zlib.Z_HUFFMAN_ONLY), ("rle", zlib.Z_RLE),
                   ("fixed", zlib.Z_FIXED)):
        out.append((f"strategy_{nm}", W.png(big, 8, 2, 0, (1, 2), strategy=st)))
    for wb in range(9, 16):
        out.append((f"wbits{wb}", W.png(big, 8, 2, 0, (4,), wbits=wb)))
    out.append(("tail_junk", W.png(big, 8, 2, tail=b"\xff\x13\x37junk")))
    out.append(("short_raw", W.png(big, 8, 2, zdata=zlib.compress(W.raw_stream(big, 8, 2)[:-3]))))
    out.append(("extra_raw", W.png(big, 8, 2, zdata=zlib.compress(W.raw_stream(big, 8, 2) + bytes(999)))))
    out.append(("bad_zlib_header", W.png(big, 8, 2, zdata=b"\x78\x02" + zlib.compress(W.raw_stream(big, 8, 2))[2:])))
    out.append(("fdict", W.png(big, 8, 2, zdata=b"\x78\x20" + zlib.compress(W.raw_stream(big, 8, 2))[2:])))
    return out + stream_cases()


def _raw_png(raw_body, w, h, depth=8, color=0, cgbi=False, adler=True):
    s = np.zeros((h, w, W.CHANNELS[color]), np.int64)
    z = raw_body if cgbi else W.zlib_wrap(raw_body) if adler else b"\x78\x01" + raw_body
    return W.png(s, depth, color, zdata=z, cgbi=cgbi)


def stream_cases():
    """Hand-made deflate streams around a 6x4 grey image (28 raw bytes with the filter bytes)."""
    raw = bytes([0, 1, 2, 3, 4, 5, 6] * 4)
    lit = list(raw)
    out = []

    def bw_png(build, **kw):
        bw = W.BitWriter()
        build(bw)
        return _raw_png(bw.bytes(), 6, 4, **kw)

    out.append(("s_stored", bw_png(lambda b: W.stored(b, raw, 1))))
    out.append(("s_stored_empty_blocks", bw_png(lambda b: [W.stored(b, b"", 0), W.stored(b, raw[:9], 0),
                                                           W.stored(b, b"", 0), W.stored(b, raw[9:], 1)])))
    out.append(("s_stored_nlen", bw_png(lambda b: W.stored(b, raw, 1, nlen=0x1234))))
    out.append(("s_stored_past_buffer", _raw_png(b"\x01\xff\x00\x00\xff" + raw, 6, 4, cgbi=True)))
    out.append(("s_fixed", bw_png(lambda b: W.fixed(b, lit[:7] + [("copy", 21, 7)], 1))))
    out.append(("s_fixed_tiny_blocks", bw_png(lambda b: [W.fixed(b, [v], 0) for v in lit[:-1]] + [W.fixed(b, [lit[-1]], 1)])))
    out.append(("s_type3", bw_png(lambda b: [b.put(1, 1), b.put(3, 2), b.put(0, 20)])))
    out.append(("s_len286", bw_png(lambda b: W.fixed(b, lit[:7] + [("dsym", 286, 0)], 1))))
    out.append(("s_len287", bw_png(lambda b: W.fixed(b, lit[:7] + [("dsym", 287, 0)], 1))))
    out.append(("s_dist30", bw_png(lambda b: W.fixed(b, lit[:7] + [("dsym", 257, 30)], 1))))
    out.append(("s_dist31", bw_png(lambda b: W.fixed(b, lit[:7] + [("dsym", 257, 31)], 1))))
    out.append(("s_dist_before_start", bw_png(lambda b: W.fixed(b, lit[:3] + [("copy", 25, 4)], 1))))
    out.append(("s_dist_at_start", bw_png(lambda b: W.fixed(b, lit[:3] + [("copy", 25, 3)], 1))))
    # dynamic blocks: a complete code, incomplete codes, a single-code distance tree
    L = [0] * 286
    for v in set(lit):
        L[v] = 4
    L[256], L[269] = 4, 4                            # EOB, length 21 (code 269: 19..22, 2 extra bits); 9 of 16 codes
    D = [0] * 3
    D[2] = 1                                         # one distance code: dist 3 only -- the distance tree has one code
    D2 = [0] * 5
    D2[4] = 1                                        # distance code 4: 5..6 (1 extra bit)
    copy21 = ("copy", 21, 7)

    def dyn(ops, lit_l, dist_l, **kw):
        return lambda b: W.dynamic(b, ops, 1, lit_l, dist_l, **kw)
    out.append(("s_dyn_incomplete", bw_png(dyn(lit[:7] + [("copy", 21, 5)], L, D2))))
    D7 = [0] * 6
    D7[5] = 1                                        # distance code 5: 7..8
    out.append(("s_dyn_incomplete_dist7", bw_png(dyn(lit[:7] + [copy21], L, D7))))
    out.append(("s_dyn_single_dist_3", bw_png(dyn(lit[:7] + [("copy", 21, 3)], L, D))))
    Lbad = list(L)
    out.append(("s_dyn_unused_code", bw_png(dyn(lit[:7] + [("bits", 15, 4)], Lbad, D7))))
    over = [1] * 3 + [0] * 283                       # three codes of length 1: over-subscribed
    out.append(("s_dyn_oversubscribed", bw_png(dyn([], over, [1], end=False))))
    out.append(("s_dyn_16_first", bw_png(dyn([], L, D7, clen_seq=[(16, 0)] + [(0, 0)] * 291, end=False))))
    out.append(("s_dyn_overrun", bw_png(dyn([], L, D7, clen_seq=[(18, 127)] * 3, end=False))))
    out.append(("s_dyn_hlit288", bw_png(lambda b: W.dynamic(b, lit[:7] + [copy21], 1, L + [4, 4], D7))))
    # a stream cut at every bit of its last 4 bytes, with and without the Adler-32 after it
    full = W.BitWriter()
    W.fixed(full, lit[:7] + [copy21], 1)
    nbits = len(full.bits)
    for cut in range(max(0, nbits - 32), nbits + 1):
        bw = W.BitWriter()
        bw.bits = full.bits[:cut]
        body = bw.bytes()
        out.append((f"s_cut{nbits - cut}_raw", _raw_png(body, 6, 4, cgbi=True)))
        out.append((f"s_cut{nbits - cut}_zlib", _raw_png(body, 6, 4)))
    return out


def pillow_cases():
    out = []
    img = photo(37, 23, 1, 4)
    for mode in ("RGB", "RGBA", "L", "LA", "P", "1", "I;16"):
        out.append((f"pil_{mode}", pillow(img, mode)))
    return out


def golden_cases():
    return pillow_cases() + writer_cases()


@functools.lru_cache(maxsize=1)
def sized_cases():
    """(name, bytes) at the sizes a user opens."""
    return [
        ("4k_rgb_photo", pillow(photo(3840, 2160, 10), "RGB")),
        ("4k_rgba_photo", pillow(photo(3840, 2160, 11, 4), "RGBA")),
        ("4k_screenshot_l9", pillow(screenshot(3840, 2160, 12), "RGB", compress_level=9)),
        ("4k_interlaced", W.png(photo(3840, 2160, 13).astype(np.int64), 8, 2, 1, (4, 1, 2, 3, 0), level=6)),
        ("solid_8192", pillow(np.full((8192, 8192, 3), (12, 200, 77), np.uint8), "RGB")),
        ("1x1", pillow(photo(1, 1, 14), "RGB")),
        ("1x16384", pillow(photo(1, 16384, 15), "RGB")),
        ("16384x1", pillow(photo(16384, 1, 16), "RGB")),
    ]


def bomb_case(extra=300 << 20):
    """A 64x64 RGB image whose stream inflates `extra` bytes past it (runs of zeros, then the final block)."""
    img = photo(64, 64, 17)
    raw = W.raw_stream(img.astype(np.int64), 8, 2)
    co = zlib.compressobj(9)
    z = co.compress(raw)
    chunk = bytes(1 << 20)
    for _ in range(extra >> 20):
        z += co.compress(chunk)
    z += co.flush()
    return W.png(img.astype(np.int64), 8, 2, zdata=z)


def golden():
    """The pinned corpus of tests/golden/png.npz: list of (name, bytes, canvas sha256 or '', status, supported)."""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "png.npz"))
    d, o = z["data"].tobytes(), z["offsets"]
    return [(str(z["names"][i]), d[o[i]:o[i + 1]], str(z["sha"][i]), int(z["status"][i]), bool(z["supported"][i]))
            for i in range(len(z["names"]))]
