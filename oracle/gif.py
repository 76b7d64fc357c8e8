"""TEST INFRASTRUCTURE ONLY: GIF files for the decoder's tests, and the reference's decode of them.

- lzw(): our LZW raster encoder (oracle/gif_writer.c in liboracle.so).
- gif(): a GIF87a / GIF89a file around such rasters -- global and / or local palettes of 2..256 entries, any lzw_cs
  0..12, three clear policies, the sub-block length, interlace, a rectangle per frame, a Graphic Control Extension
  (dispose 0-3, transparency, delay) or none, comment and NETSCAPE extensions.  Malformed files are made by byte
  surgery on its output.
- ref_stb_gif(): the UNMODIFIED reference STBImageSource (LoadAndScale + SendFrames) through oracle/ref_gif.cc, built
  by oracle/gif.mk into oracle/_ref/libtimg_gif_ref.so.
"""
import ctypes as C
import os
import struct
import tempfile

import numpy as np

from oracle import lib as _orc_lib

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_GIF_SO = os.path.join(_HERE, "_ref", "libtimg_gif_ref.so")
_REF = None

CLEAR_START, NO_START_CLEAR, DEFERRED_CLEAR = 0, 1, 2


def lzw(idx, lzw_cs=8, policy=CLEAR_START, subblock=255):
    """The raster of a frame's index stream (in the order the decoder reads it): lzw_cs, sub-blocks, terminator."""
    L = _orc_lib()
    f = L.orc_gif_lzw
    f.restype = C.c_long
    f.argtypes = [C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_long]
    idx = np.ascontiguousarray(idx, dtype=np.uint8).reshape(-1)
    cap = 64 + idx.size * 3 + idx.size // 8
    out = np.empty(cap, np.uint8)
    n = f(idx.ctypes.data, idx.size, lzw_cs, policy, subblock, out.ctypes.data, cap)
    if n < 0:
        raise ValueError(f"orc_gif_lzw failed ({n}): lzw_cs {lzw_cs}, max index {int(idx.max()) if idx.size else 0}")
    return out[:n].tobytes()


def _table(pal):
    pal = np.asarray(pal, dtype=np.uint8).reshape(-1, 3)
    n = pal.shape[0]
    bits = max(0, int(n).bit_length() - 2)
    assert 2 <= n <= 256 and n == 2 << bits, f"palette of {n} entries: 2..256, a power of two"
    return bits, pal.tobytes()


def interlace_order(h):
    """Rows in the order an interlaced raster stores them (passes 0::8, 4::8, 2::4, 1::2)."""
    return [r for start, step in ((0, 8), (4, 8), (2, 4), (1, 2)) for r in range(start, h, step)]


def gce(dispose=0, transparent=None, delay=0):
    flags = (dispose & 7) << 2 | (1 if transparent is not None else 0)
    return b"\x21\xf9\x04" + struct.pack("<BHB", flags, delay, transparent or 0) + b"\x00"


def netscape(loops=0):
    return b"\x21\xff\x0bNETSCAPE2.0\x03\x01" + struct.pack("<H", loops) + b"\x00"


def comment(text=b"oracle"):
    out = b"\x21\xfe"
    for i in range(0, len(text), 255):
        out += bytes([len(text[i:i + 255])]) + text[i:i + 255]
    return out + b"\x00"


def image(idx, x=0, y=0, lpal=None, interlace=False, lzw_cs=8, policy=CLEAR_START, subblock=255, raster=None, size=None):
    """Image descriptor, optional local table and raster of one frame; idx: [rh, rw] palette indices.  raster: the
    raster's bytes as given (lzw_cs, sub-blocks, terminator) in place of the encoding of idx (a stream shorter or
    longer than the rectangle, or a malformed one); size: the descriptor's (rw, rh) if not idx's shape."""
    idx = np.asarray(idx, dtype=np.uint8)
    rh, rw = idx.shape if size is None else size[::-1]
    flags = 0x40 if interlace else 0
    tab = b""
    if lpal is not None:
        bits, tab = _table(lpal)
        flags |= 0x80 | bits
    rows = idx[interlace_order(rh)] if interlace else idx
    data = lzw(rows, lzw_cs, policy, subblock) if raster is None else raster
    return b"\x2c" + struct.pack("<HHHHB", x, y, rw, rh, flags) + tab + data


def codes(values, lzw_cs, widths):
    """A raster of explicit codes: values[i] written LSB first with widths[i] bits, in one sub-block per 255 bytes."""
    acc, n, out = 0, 0, bytearray()
    for v, wd in zip(values, widths):
        acc |= v << n
        n += wd
        while n >= 8:
            out.append(acc & 255); acc >>= 8; n -= 8
    if n:
        out.append(acc & 255)
    blocks = b"".join(bytes([len(out[i:i + 255])]) + bytes(out[i:i + 255]) for i in range(0, len(out), 255))
    return bytes([lzw_cs]) + blocks + b"\x00"


def gif(w, h, frames, gpal=None, bgindex=0, version=b"89a", head=b"", trailer=True):
    """frames: list of dicts with the keys of image() plus 'gce' (a dict for gce(), or None for no extension) and
    'pre' (bytes placed before the frame's extensions).  head: bytes after the screen descriptor (NETSCAPE, comments)."""
    flags, tab = 0, b""
    if gpal is not None:
        bits, tab = _table(gpal)
        flags = 0x80 | 0x70 | bits
    out = b"GIF" + version + struct.pack("<HHBBB", w, h, flags, bgindex, 0) + tab + head
    for fr in frames:
        fr = dict(fr)
        out += fr.pop("pre", b"")
        g = fr.pop("gce", None)
        if g is not None:
            out += gce(**g)
        out += image(**fr)
    return out + (b"\x3b" if trailer else b"")


def have_ref():
    return os.path.exists(REF_GIF_SO)


def _ref():
    global _REF
    if _REF is None:
        L = C.CDLL(REF_GIF_SO)
        L.ref_stb_gif_run.restype = C.c_void_p
        L.ref_stb_gif_run.argtypes = [C.c_char_p] + [C.c_int] * 5 + [C.c_uint32, C.c_uint32, C.c_int, C.c_int,
                                                                     C.POINTER(C.c_int), C.POINTER(C.c_longlong)]
        L.ref_stb_gif_fetch.restype = None
        L.ref_stb_gif_fetch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.ref_stb_gif_free.restype = None
        L.ref_stb_gif_free.argtypes = [C.c_void_p]
        _REF = L
    return _REF


RAW_BOX = 1 << 20


def ref_stb_gif_path(path, width=RAW_BOX, height=RAW_BOX, cell=(1, 1), has_bg=False, bg=0, pattern=0, pattern_size=1,
                     capture=True, out=None):
    """One run of the reference's STB source (LoadAndScale + SendFrames) on a file: None if the source fails to load;
    else (n_frames, meta [n, 5] int32 of {w, h, dx, dy, delay_ms}, the frames' bytes back to back).  out: a uint8
    array to receive the bytes (allocated if None).  capture=False: the sink drops the frames, and only n_frames is
    returned (meta and bytes are None) -- one decode and nothing else, for timing."""
    L = _ref()
    n, nbytes = C.c_int(0), C.c_longlong(0)
    h = L.ref_stb_gif_run(os.fsencode(path), width, height, cell[0], cell[1], int(has_bg), bg, pattern, pattern_size,
                          int(capture), C.byref(n), C.byref(nbytes))
    if not h:
        return None
    try:
        if not capture:
            return n.value, None, None
        meta = np.zeros((max(1, n.value), 5), np.int32)
        if out is None:
            out = np.empty(max(1, nbytes.value), np.uint8)
        assert out.dtype == np.uint8 and out.flags.c_contiguous and out.size >= nbytes.value
        L.ref_stb_gif_fetch(h, out.ctypes.data, meta.ctypes.data)
        return n.value, meta[:n.value], out
    finally:
        L.ref_stb_gif_free(h)


def ref_stb_gif(data, width=RAW_BOX, height=RAW_BOX, cell=(1, 1), has_bg=False, bg=0, pattern=0, pattern_size=1):
    """What the reference's STB source sends for a GIF: (list of [h, w, 4] uint8 frames, meta [n, 5] int32 of
    {w, h, dx, dy, delay_ms}), or None if the source fails to load.  The default box and has_bg=False give stb's raw
    canvases; width / height (pixels), cell, and the compose options give the frames a canvas receives."""
    with tempfile.NamedTemporaryFile(suffix=".gif") as f:
        f.write(data)
        f.flush()
        r = ref_stb_gif_path(f.name, width, height, cell, has_bg, bg, pattern, pattern_size)
    if r is None:
        return None
    n, meta, out = r
    frames, o = [], 0
    for k in range(n):
        fw, fh = int(meta[k, 0]), int(meta[k, 1])
        frames.append(out[o:o + fw * fh * 4].reshape(fh, fw, 4))
        o += fw * fh * 4
    return frames, meta
