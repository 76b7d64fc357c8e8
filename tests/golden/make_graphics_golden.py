"""Regenerates tests/golden/graphics.npz from the reference's own kitty / iTerm2 canvases:
    make -C oracle all && make -C oracle -f graphics.mk && python tests/golden/make_graphics_golden.py

oracle/graphics.mk compiles the UNMODIFIED KittyGraphicsCanvas (no tmux passthrough), ITerm2GraphicsCanvas and
PNG writer with oracle/deflate_stored/libdeflate.h (stored deflate blocks) in place of libdeflate, so the reference's
own code writes the whole framed stream -- Sub filter, chunk CRCs, base64, chunking, headers -- around the PNG bytes
this library produces.  Scaled and composed cases go through the reference's scaler and AlphaComposeBackground
(oracle/_ref/libtimg_ref.so, oracle/Makefile) first.

Inputs are not stored: tests/graphics_cases.py regenerates them.  "<protocol>/<case>" holds the bytes after the
cursor prefix (or, above graphics_cases.FULL_GOLDEN_BYTES, "<...>/sha" and "<...>/len"); "<...>/id" the kitty
image id the canvas picked.  CreateId seeds from time(), so only the ids differ between two runs; the tests pass
them back.
"""
import ctypes as C
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import oracle  # noqa: E402
import graphics_cases as gcases  # noqa: E402

_GFX = None


def gfx_ref():
    global _GFX
    if _GFX is None:
        p = os.path.join(ROOT, "oracle", "_ref", "libtimg_graphics_ref.so")
        if not os.path.exists(p):
            raise RuntimeError(f"{p} not built: make -C oracle -f graphics.mk (needs the reference's sources)")
        L = C.CDLL(p)
        oracle._sig(L, "ref_graphics_new", C.c_void_p, [C.c_int] * 4)
        oracle._sig(L, "ref_graphics_send", C.c_long, [C.c_void_p, C.c_int, C.c_int, oracle.u8p, C.c_int, C.c_int,
                                                       C.c_int, C.c_char_p, C.c_long])
        oracle._sig(L, "ref_graphics_free", None, [C.c_void_p])
        _GFX = L
    return _GFX


class RefGraphicsCanvas:
    """The reference's KittyGraphicsCanvas (no tmux) or ITerm2GraphicsCanvas behind its own BufferedWriteSequencer
    (oracle/ref_graphics.cc)."""
    CELL_X, CELL_Y, X = 9, 18, 18          # Send(x = 18) queues "\e[2C" before the image bytes

    def __init__(self, protocol, rgb24):
        self._h = gfx_ref().ref_graphics_new(protocol, int(rgb24), self.CELL_X, self.CELL_Y)

    def send(self, fb):
        """(image bytes after the cursor prefix, kitty's i= or 0) of Send(x, 0, fb, FrameImmediate)."""
        fb = np.ascontiguousarray(fb, dtype=np.uint8)
        h, w = fb.shape[:2]
        cap = 4096 + w * h * 8
        buf = C.create_string_buffer(cap)
        n = gfx_ref().ref_graphics_send(self._h, self.X, 0, oracle._ptr(fb), w, h, 1, buf, cap)
        assert n > 0, n
        out = buf.raw[:n]
        prefix = b"\033[%dC" % (self.X // self.CELL_X)          # the prefix asked for, stripped
        assert out.startswith(prefix), out[:16]
        out = out[len(prefix):]
        m = re.match(rb"\033_Ga=T,i=(\d+),", out)
        return out, int(m.group(1)) if m else 0

    def __del__(self):
        if getattr(self, "_h", None):
            gfx_ref().ref_graphics_free(self._h)
            self._h = None


def main(path=os.path.join(HERE, "graphics.npz")):
    g = {}

    def put(key, out, id_, digest=False):
        if digest:
            g[key + "/sha"] = np.frombuffer(gcases.sha(out), np.uint8)
            g[key + "/len"] = np.array([len(out)], np.int64)
        else:
            g[key] = np.frombuffer(out, np.uint8)
        g[key + "/id"] = np.array([id_], np.uint32)

    for proto, pname in ((gcases.KITTY, "kitty"), (gcases.ITERM2, "iterm2")):
        for name, fb, rgb24 in gcases.graphics_frame_cases():
            out, id_ = RefGraphicsCanvas(proto, rgb24).send(fb)
            put(f"{pname}/{name}", out, id_, digest=len(out) > gcases.FULL_GOLDEN_BYTES and not name.startswith("blocks"))
    src, ow, oh, kw = gcases.graphics_checker_case()
    fb = oracle.ref_compose_bg(oracle.ref_scale(src, ow, oh), **kw)
    put("kitty/checker_rgb1", *RefGraphicsCanvas(gcases.KITTY, 1).send(fb))
    put("iterm2/checker_rgb0", *RefGraphicsCanvas(gcases.ITERM2, 0).send(fb))
    cv = RefGraphicsCanvas(gcases.KITTY, 1)
    for f, fr in enumerate(gcases.c4_graphics_frames()):
        fb = oracle.ref_compose_bg(oracle.ref_scale(fr, 337, 190), oracle.rgba_u32(0, 0, 0))
        put(f"kitty/c4_rgb1/{f}", *cv.send(fb), digest=True)
    np.savez_compressed(path, **g)
    print(f"wrote {len(g)} graphics outputs; {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main(*sys.argv[1:])
