"""The replay oracle of B200TIMG_DEFLATE (oracle/_ref/libtimg_graphics_replay.so, built by oracle/graphics_deflate.mk):
the reference's own PNG writer and kitty / iTerm2 canvases around a zlib stream handed to them.  Fed the stored-block
stream of this library's stored path, it must write exactly the goldens of tests/golden/graphics.npz (which the
reference's canvases wrote with a stored-block compressor), so what it writes around a compressed stream is the
reference's framing of that stream.  No GPU; skips where the replay library was not built."""
import ctypes as C
import os
import re
import struct
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import graphics_cases as gcases  # noqa: E402
from test_graphics_oracle import GOLD, full_goldens  # noqa: E402

REPLAY_LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref",
                          "libtimg_graphics_replay.so")
_lib = None


def replay_lib():
    global _lib
    if _lib is None:
        if not os.path.exists(REPLAY_LIB):
            pytest.skip("oracle/_ref/libtimg_graphics_replay.so was not built (reference sources absent)")
        L = C.CDLL(REPLAY_LIB)
        L.ref_replay_new.restype = C.c_void_p
        L.ref_replay_new.argtypes = [C.c_int] * 4
        L.ref_replay_send.restype = C.c_long
        L.ref_replay_send.argtypes = [C.c_void_p, C.c_char_p, C.c_long, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_char_p, C.c_long]
        L.ref_replay_free.argtypes = [C.c_void_p]
        _lib = L
    return _lib


class ReplayCanvas:
    """One reference canvas (protocol 1 kitty, 2 iTerm2, 4 kitty in tmux); send() -> the bytes of one Send."""

    def __init__(self, protocol, rgb24, cell=(9, 18)):
        self.h = replay_lib().ref_replay_new(protocol, int(rgb24), cell[0], cell[1])

    def send(self, zlib_stream, fb, x=0):
        fb = np.ascontiguousarray(fb, dtype=np.uint8)
        h, w = fb.shape[:2]
        cap = 64 * len(zlib_stream) + (1 << 20)
        out = C.create_string_buffer(cap)
        n = replay_lib().ref_replay_send(self.h, zlib_stream, len(zlib_stream), x, fb.ctypes.data, w, h, out, cap)
        assert n >= 0, n
        return out.raw[:n]

    def __del__(self):
        if _lib is not None and getattr(self, "h", None):
            _lib.ref_replay_free(self.h)


def scanlines(fb, rgb24):
    """The Sub-filtered scanline stream of a frame (src/timg-png.cc:119-134)."""
    px = np.ascontiguousarray(fb[..., :3] if rgb24 else fb).astype(np.uint8)
    d = px.copy()
    d[:, 1:] = px[:, 1:] - px[:, :-1]
    h = px.shape[0]
    return np.concatenate([np.ones((h, 1), np.uint8), d.reshape(h, -1)], axis=1).tobytes()


def stored_zlib(raw):
    """The stored-block zlib stream of the library's stored path (png.cu)."""
    out = bytearray(b"\x78\x01")
    blocks = [raw[i:i + 65535] for i in range(0, len(raw), 65535)] or [b""]
    for k, b in enumerate(blocks):
        out += bytes([k == len(blocks) - 1]) + struct.pack("<HH", len(b), len(b) ^ 0xFFFF) + b
    return bytes(out + struct.pack(">I", zlib.adler32(raw)))


def with_id(text, id_):
    """Kitty's i= (the reference seeds it from time()) replaced by id_."""
    return re.sub(rb"i=\d+,", b"i=%d," % id_, text, count=1)


@pytest.mark.parametrize("pname,name,fb,rgb24", full_goldens(), ids=lambda v: v if isinstance(v, str) else "")
def test_replay_of_the_stored_stream_writes_the_golden(pname, name, fb, rgb24):
    canvas = ReplayCanvas(gcases.KITTY if pname == "kitty" else gcases.ITERM2, rgb24)
    got = canvas.send(stored_zlib(scanlines(fb, rgb24)), fb)
    want = GOLD[f"{pname}/{name}"].tobytes()
    if pname == "kitty":
        got = with_id(got, int(GOLD[f"{pname}/{name}/id"][0]))
    assert got == want
