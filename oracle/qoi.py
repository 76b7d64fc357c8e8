"""TEST INFRASTRUCTURE ONLY: QOI files for the decoder's tests, and the reference's decode of them.

- encode(): our encoder, written from the published format description (oracle/qoi_writer.c in liboracle.so).
- Ops / stream(): hand-made op streams -- any op with any argument, free header fields, chosen or missing padding,
  trailing bytes.
- ref_qoi(): the UNMODIFIED reference QOIImageSource (LoadAndScale + SendFrames) through oracle/ref_qoi.cc, built by
  oracle/qoi.mk into oracle/_ref/libtimg_qoi_ref.so.
"""
import ctypes as C
import os
import struct
import tempfile

import numpy as np

from oracle import lib as _orc_lib

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_QOI_SO = os.path.join(_HERE, "_ref", "libtimg_qoi_ref.so")
_REF = None
MAGIC = b"qoif"
PADDING = bytes(7) + b"\x01"


def header(w, h, channels=4, colorspace=0, magic=MAGIC):
    return magic + struct.pack(">IIBB", w, h, channels, colorspace)


def encode(rgba, channels=4, colorspace=0):
    """A QOI file of an [h, w, 4] uint8 image; channels and colorspace are only written to the header."""
    rgba = np.ascontiguousarray(rgba, dtype=np.uint8)
    h, w = rgba.shape[:2]
    f = _orc_lib().orc_qoi_encode
    f.restype = C.c_long
    f.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_long]
    cap = 22 + 5 * w * h
    out = np.empty(cap, np.uint8)
    n = f(rgba.ctypes.data, w, h, channels, colorspace, out.ctypes.data, cap)
    assert n > 0
    return out[:n].tobytes()


class Ops:
    """An op-level writer: each method appends one op with any argument; bytes() is the op stream."""

    def __init__(self):
        self.b = bytearray()
        self.starts = []                          # byte offset (in the op stream) of each op

    def _op(self, *bs):
        self.starts.append(len(self.b))
        self.b += bytes(bs)
        return self

    def rgb(self, r, g, b):
        return self._op(0xFE, r & 255, g & 255, b & 255)

    def rgba(self, r, g, b, a):
        return self._op(0xFF, r & 255, g & 255, b & 255, a & 255)

    def index(self, i):
        assert 0 <= i < 64
        return self._op(i)

    def diff(self, dr, dg, db):
        assert all(-2 <= d <= 1 for d in (dr, dg, db))
        return self._op(0x40 | (dr + 2) << 4 | (dg + 2) << 2 | (db + 2))

    def luma(self, dg, dr_dg, db_dg):
        assert -32 <= dg <= 31 and -8 <= dr_dg <= 7 and -8 <= db_dg <= 7
        return self._op(0x80 | (dg + 32), (dr_dg + 8) << 4 | (db_dg + 8))

    def run(self, n):
        assert 1 <= n <= 62
        return self._op(0xC0 | (n - 1))

    def raw(self, data):
        """Bytes as they are (one op start recorded at their first byte)."""
        self.starts.append(len(self.b))
        self.b += bytes(data)
        return self

    def bytes(self):
        return bytes(self.b)


def stream(w, h, ops, channels=4, colorspace=0, padding=PADDING, trailing=b"", magic=MAGIC):
    """A file of a header, the op stream (an Ops or bytes), the padding as given (b"" for none) and trailing bytes."""
    body = ops.bytes() if isinstance(ops, Ops) else bytes(ops)
    return header(w, h, channels, colorspace, magic) + body + padding + trailing


def hash_slot(r, g, b, a):
    return (r * 3 + g * 5 + b * 7 + a * 11) % 64


def have_ref():
    return os.path.exists(REF_QOI_SO)


def _ref():
    global _REF
    if _REF is None:
        L = C.CDLL(REF_QOI_SO)
        L.ref_qoi_run.restype = C.c_void_p
        L.ref_qoi_run.argtypes = [C.c_char_p] + [C.c_int] * 5 + [C.c_uint32, C.c_uint32, C.c_int, C.c_int] + \
            [C.POINTER(C.c_int)] * 3
        L.ref_qoi_fetch.restype = None
        L.ref_qoi_fetch.argtypes = [C.c_void_p, C.c_void_p]
        L.ref_qoi_free.restype = None
        L.ref_qoi_free.argtypes = [C.c_void_p]
        _REF = L
    return _REF


RAW_BOX = 1 << 20


def ref_qoi_path(path, width=RAW_BOX, height=RAW_BOX, cell=(1, 1), has_bg=False, bg=0, pattern=0, pattern_size=1,
                 capture=True):
    """One run of the reference's QOI source on a file: None if it fails to load; else the [h, w, 4] uint8 frame it
    sends (capture=False: True, after one decode and nothing else, for timing)."""
    L = _ref()
    w, h, dx = C.c_int(0), C.c_int(0), C.c_int(0)
    hd = L.ref_qoi_run(os.fsencode(path), width, height, cell[0], cell[1], int(has_bg), bg, pattern, pattern_size,
                       int(capture), C.byref(w), C.byref(h), C.byref(dx))
    if not hd:
        return None
    try:
        if not capture:
            return True
        out = np.empty((h.value, w.value, 4), np.uint8)
        L.ref_qoi_fetch(hd, out.ctypes.data)
        return out
    finally:
        L.ref_qoi_free(hd)


def ref_qoi(data, width=RAW_BOX, height=RAW_BOX, cell=(1, 1), has_bg=False, bg=0, pattern=0, pattern_size=1):
    """What the reference's QOI source sends for a file ([h, w, 4] uint8), or None if it fails to load.  The default
    box and has_bg=False give qoi_read's raw canvas; width / height (pixels), cell and the compose options give the
    frame a canvas receives (composed only for a 4-channel header)."""
    with tempfile.NamedTemporaryFile(suffix=".qoi") as f:
        f.write(data)
        f.flush()
        return ref_qoi_path(f.name, width, height, cell, has_bg, bg, pattern, pattern_size)
