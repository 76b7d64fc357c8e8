"""TEST INFRASTRUCTURE ONLY: BMP, TGA and binary PNM files for the raster decoder's tests, and the reference's decode.

Writers from the published format descriptions (Microsoft's BITMAPFILEHEADER / BITMAPINFOHEADER / BITMAPV4/V5HEADER and
OS/2 BITMAPCOREHEADER, Truevision's TGA 2.0 specification, Netpbm's PGM / PPM pages):
- bmp(): any header size (12, 40, 56, 108, 124), 1/4/8-bit palettes, 16/24/32 bits, BI_BITFIELDS masks, a gap before
  bfOffBits, bottom-up or top-down rows.  Damaged files are made by overriding header fields.
- tga(): image types 1-3 and 9-11, palettes of 15/16/24/32 bits at any first-entry offset, an id field, the two
  origin bits; Rle() writes packets one by one, so a test chooses where every header falls.
- pnm(): P5 / P6 at any maxval, with the header text given or built.
ref_stb(): the UNMODIFIED reference STBImageSource through oracle/gif.py's door (oracle/_ref/libtimg_gif_ref.so), which
reads a real file as timg does: the raw canvas, or None if the source fails.
"""
import struct

import numpy as np

from oracle import gif as G


# ---- BMP ---------------------------------------------------------------------------------------------------------
def _rows(img, bpp, masks=None):
    """The file rows of img (indices [h, w] for bpp < 16, else [h, w, 4] RGBA), top row first, padded to 4 bytes."""
    h, w = img.shape[:2]
    out = []
    for y in range(h):
        r = img[y]
        if bpp == 1:
            bits = np.zeros((w + 7) // 8 * 8, np.uint8)
            bits[:w] = r & 1
            row = np.packbits(bits).tobytes()
        elif bpp == 4:
            v = np.zeros((w + 1) // 2 * 2, np.uint8)
            v[:w] = r & 15
            row = (v[0::2] << 4 | v[1::2]).astype(np.uint8).tobytes()
        elif bpp == 8:
            row = r.astype(np.uint8).tobytes()
        elif bpp == 24:
            row = r[:, [2, 1, 0]].astype(np.uint8).tobytes()
        else:
            mr, mg, mb, ma = masks
            vals = np.zeros(w, np.uint64)
            for c, m in enumerate((mr, mg, mb, ma)):
                if not m:
                    continue
                lo = (m & -m).bit_length() - 1
                n = bin(m).count("1")
                contiguous = m >> lo == (1 << n) - 1
                v = (r[:, c].astype(np.uint64) << max(0, n - 8)) >> max(0, 8 - n)
                if contiguous:
                    vals |= (v << lo) & m
                else:                            # spread the value's bits over the mask's bits, low to high
                    k = 0
                    for bit in range(32):
                        if m >> bit & 1:
                            vals |= ((v >> k) & 1) << bit
                            k += 1
            row = vals.astype("<u2" if bpp == 16 else "<u4").tobytes()
        row += bytes((-len(row)) & 3)
        out.append(row)
    return out


def bmp(img, bpp=24, hsz=40, compress=None, masks=None, palette=None, top_down=False, gap=0, offset=None,
        planes=1, size=None, fields=None, tail=b""):
    """A BMP file.  img: [h, w] palette indices for bpp < 16, else [h, w, 3 or 4] RGB(A).  masks (r, g, b, a): written
    as BI_BITFIELDS (compress 3) in a 40/56-byte header, or into the mask fields of a 108/124-byte one.  palette: [n, 3]
    RGB.  gap: bytes between the header (+ palette) and the pixels.  offset, size (w, h), fields (a dict of
    header field -> value: 'compress', 'bpp', 'hsz', 'offset') override what would be written."""
    img = np.asarray(img)
    h, w = img.shape[:2]
    if img.ndim == 3 and img.shape[2] == 3:
        img = np.concatenate([img, np.full((h, w, 1), 255, np.uint8)], -1)
    if compress is None:
        compress = 3 if masks is not None and hsz in (40, 56) else 0
    if masks is None and bpp in (16, 32):
        masks = (31 << 10, 31 << 5, 31, 0) if bpp == 16 else (0xFF0000, 0xFF00, 0xFF, 0xFF000000)
    f = dict(compress=compress, bpp=bpp, hsz=hsz)
    f.update(fields or {})
    pal = b""
    if palette is not None:
        pal = b"".join(bytes([b, g, r]) + (b"" if hsz == 12 else b"\0") for r, g, b in np.asarray(palette, np.uint8))
    extra = 12 if f["compress"] == 3 and hsz in (40, 56) else 0
    sw, sh = size if size is not None else (w, h)
    if hsz == 12:
        info = struct.pack("<IHHHH", 12, sw & 0xFFFF, sh & 0xFFFF, planes, f["bpp"])
    else:
        info = struct.pack("<IiiHHIIiiII", f["hsz"], sw, -sh if top_down else sh, planes, f["bpp"], f["compress"] & 0xFFFFFFFF,
                           0, 2835, 2835, 0, 0)
        if hsz == 56:
            info += bytes(16)
        if extra:
            info += struct.pack("<III", *(masks or (0, 0, 0))[:3])
        if hsz in (108, 124):
            mr, mg, mb, ma = masks if masks is not None else (0, 0, 0, 0)
            info += struct.pack("<IIII", mr, mg, mb, ma) + b"BGRs" + bytes(48)
            if hsz == 124:
                info += bytes(16)
    rows = _rows(img, bpp, masks) if bpp in (1, 4, 8, 16, 24, 32) else []
    if not top_down:
        rows = rows[::-1]
    pix = b"".join(rows)
    off = 14 + len(info) + len(pal) + gap if offset is None else offset
    off = f.get("offset", off)
    head = b"BM" + struct.pack("<IHHI", 14 + len(info) + len(pal) + gap + len(pix), 0, 0, off & 0xFFFFFFFF)
    return head + info + pal + bytes(gap) + pix + tail


# ---- TGA ---------------------------------------------------------------------------------------------------------
class Rle:
    """A TGA RLE stream written packet by packet: run(n, value) or raw(values), each value of B bytes."""

    def __init__(self, B):
        self.B, self.b, self.starts = B, bytearray(), []

    def run(self, n, value):
        assert 1 <= n <= 128 and len(value) == self.B
        self.starts.append(len(self.b))
        self.b += bytes([0x80 | (n - 1)]) + bytes(value)
        return self

    def raw(self, values):
        values = bytes(values)
        n = len(values) // self.B
        assert 1 <= n <= 128 and len(values) == n * self.B
        self.starts.append(len(self.b))
        self.b += bytes([n - 1]) + values
        return self

    def bytes(self):
        return bytes(self.b)


def rle_encode(values, B):
    """values (bytes, a multiple of B): runs of 2+ equal values as run packets, the rest as raw packets of <= 128."""
    vals = [values[i:i + B] for i in range(0, len(values), B)]
    o, i, lit = Rle(B), 0, []
    while i < len(vals):
        j = i
        while j + 1 < len(vals) and vals[j + 1] == vals[i] and j + 1 - i < 128:
            j += 1
        if j > i:
            if lit:
                o.raw(b"".join(lit)); lit = []
            o.run(j - i + 1, vals[i])
            i = j + 1
        else:
            lit.append(vals[i]); i += 1
            if len(lit) == 128:
                o.raw(b"".join(lit)); lit = []
    if lit:
        o.raw(b"".join(lit))
    return o.bytes()


def tga(w, h, data, itype=2, bpp=24, palette=b"", pal_len=None, pal_bits=0, pal_start=0, ident=b"", desc=0,
        cmap=None, x0=0, y0=0):
    """A TGA file: header, id field, palette bytes (as given: pal_len entries of pal_bits; pal_start is the
    first-entry index field, which stb skips as bytes, so the caller puts that many bytes in front), data as given (a
    raw raster in file order, or an RLE stream).  desc: the descriptor byte (0x20: top-down, 0x10: right-to-left)."""
    if cmap is None:
        cmap = 1 if itype in (1, 9) else 0
    if pal_len is None:
        pal_len = len(palette) * 8 // max(1, pal_bits) if pal_bits else 0
    head = struct.pack("<BBBHHBHHHHBB", len(ident), cmap, itype, pal_start, pal_len, pal_bits, x0, y0, w, h, bpp, desc)
    return head + ident + bytes(palette) + bytes(data)


# ---- PNM ---------------------------------------------------------------------------------------------------------
def pnm(img, maxv=255, header=None):
    """P5 ([h, w] grey) or P6 ([h, w, 3]); samples above 255 are written big-endian in 2 bytes as Netpbm says."""
    img = np.asarray(img)
    h, w = img.shape[:2]
    magic = b"P6" if img.ndim == 3 else b"P5"
    if header is None:
        header = magic + b"\n%d %d\n%d\n" % (w, h, maxv)
    return header + img.astype(">u2" if maxv > 255 else np.uint8).tobytes()


# ---- the reference -----------------------------------------------------------------------------------------------
def have_ref():
    return G.have_ref()


def ref_stb(data, **opts):
    """The reference STB source's canvas for a file: [h, w, 4] uint8, or None if the source fails to load.  opts: the
    box, cell and compose options of oracle.gif.ref_stb_gif, for the frame timg sends at real options."""
    r = G.ref_stb_gif(data, **opts)
    if r is None:
        return None
    frames, _ = r
    return frames[0]
