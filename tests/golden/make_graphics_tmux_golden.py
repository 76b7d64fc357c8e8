"""Regenerates tests/golden/graphics_tmux.npz from the reference's own KittyGraphicsCanvas in its tmux form
(tmux_passthrough_needed = true):
    make -C oracle all && make -C oracle -f graphics_tmux.mk && python tests/golden/make_graphics_tmux_golden.py

The canvas is compiled by oracle/graphics_tmux.mk with a stored-block compressor in place of libdeflate (see
make_graphics_golden.py), so its own code writes the passthrough framing, the chunking and the Unicode placeholder
grid around the PNG bytes this library produces.  Its door (oracle/ref_graphics_tmux.cc) records the constructor's
system() call instead of running a shell, and returns $REF_GRAPHICS_TIME from time(): the reference seeds its image
ids from time() once per process, so every seed of graphics_tmux_cases.SEEDS runs in a subprocess of its own.

Inputs are not stored: tests/graphics_tmux_cases.py regenerates them.  "<seed>/<case>" holds the bytes after the
cursor prefix (or, above graphics_cases.FULL_GOLDEN_BYTES, "<...>/sha" and "<...>/len"), "<...>/id" the image id,
"<...>/geo" (w, h, rgb24, cell_x_px, cell_y_px, indent).
"""
import ctypes as C
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import oracle  # noqa: E402
import graphics_cases as gcases  # noqa: E402
import graphics_tmux_cases as tcases  # noqa: E402

PASSTHROUGH_COMMAND = b"tmux set -p allow-passthrough on > /dev/null 2>&1\n"
_TMUX = None


def tmux_ref():
    global _TMUX
    if _TMUX is None:
        p = os.path.join(ROOT, "oracle", "_ref", "libtimg_graphics_tmux_ref.so")
        if not os.path.exists(p):
            raise RuntimeError(f"{p} not built: make -C oracle -f graphics_tmux.mk (needs the reference's sources)")
        L = C.CDLL(p)
        oracle._sig(L, "ref_graphics_tmux_new", C.c_void_p, [C.c_int] * 3)
        oracle._sig(L, "ref_graphics_tmux_send", C.c_long, [C.c_void_p, C.c_int, C.c_int, oracle.u8p, C.c_int, C.c_int,
                                                            C.c_int, C.c_char_p, C.c_long])
        oracle._sig(L, "ref_graphics_tmux_free", None, [C.c_void_p])
        oracle._sig(L, "ref_graphics_tmux_system_calls", C.c_long, [C.c_char_p, C.c_long])
        _TMUX = L
    return _TMUX


def _system_calls():
    buf = C.create_string_buffer(1 << 12)
    n = tmux_ref().ref_graphics_tmux_system_calls(buf, len(buf))
    assert n >= 0
    return buf.raw[:n]


class RefTmuxCanvas:
    """The reference's KittyGraphicsCanvas(..., tmux_passthrough_needed = true, ...) behind its own
    BufferedWriteSequencer."""

    def __init__(self, rgb24, cell):
        before = _system_calls()
        self.cell = cell
        self._h = tmux_ref().ref_graphics_tmux_new(int(rgb24), cell[0], cell[1])
        assert _system_calls() == before + PASSTHROUGH_COMMAND      # the constructor enabled tmux's passthrough once

    def send(self, fb, x):
        """(image bytes after the cursor prefix, i=) of Send(x, 0, fb, FrameImmediate)."""
        fb = np.ascontiguousarray(fb, dtype=np.uint8)
        h, w = fb.shape[:2]
        rows, cols = -(-h // self.cell[1]), w // self.cell[0]
        cap = 4096 + w * h * 8 + rows * cols * 16 + rows * 64
        buf = C.create_string_buffer(cap)
        n = tmux_ref().ref_graphics_tmux_send(self._h, x, 0, oracle._ptr(fb), w, h, 1, buf, cap)
        assert n > 0, n
        out = buf.raw[:n]
        indent = x // self.cell[0]
        prefix = b"\033[%dC" % indent if indent else b""
        assert out.startswith(prefix + b"\033Ptmux;"), out[:16]
        out = out[len(prefix):]
        return out, int(re.match(rb"\033Ptmux;\033\033_Ga=T,i=(\d+),", out).group(1))

    def __del__(self):
        if getattr(self, "_h", None):
            tmux_ref().ref_graphics_tmux_free(self._h)
            self._h = None


def seed_outputs(seed):
    """Every golden of one id seed (this process's time() is pinned to it)."""
    g = {}

    def put(key, out, id_, geo, digest=False):
        key = f"{seed}/{key}"
        assert key + "/id" not in g, key
        if digest:
            g[key + "/sha"] = np.frombuffer(gcases.sha(out), np.uint8)
            g[key + "/len"] = np.array([len(out)], np.int64)
        else:
            g[key] = np.frombuffer(out, np.uint8)
        g[key + "/id"] = np.array([id_], np.uint32)
        g[key + "/geo"] = np.array(geo, np.int32)

    def send(name, fb, rgb24, cell, x, digest=None):
        out, id_ = RefTmuxCanvas(rgb24, cell).send(fb, x)
        if digest is None:
            digest = len(out) > gcases.FULL_GOLDEN_BYTES and not name.startswith("blocks")
        put(name, out, id_, (fb.shape[1], fb.shape[0], rgb24, cell[0], cell[1], x // cell[0]), digest)

    for case in tcases.seed_cases():
        send(*case)
    if seed != "t0":
        return g
    for case in tcases.frame_cases() + tcases.geometry_cases():
        send(*case)
    cv = RefTmuxCanvas(1, tcases.CELL)
    for f, fr in enumerate(tcases.c4_graphics_frames()):
        fb = oracle.ref_compose_bg(oracle.ref_scale(fr, 337, 190), oracle.rgba_u32(0, 0, 0))
        out, id_ = cv.send(fb, tcases.X)
        put(f"c4_rgb1/{f}", out, id_, (337, 190, 1, tcases.CELL[0], tcases.CELL[1], tcases.X // tcases.CELL[0]), True)
    send("c2_rgb1", tcases.c2_frame(), 1, tcases.CELL, tcases.X, digest=True)
    return g


def main(path=os.path.join(HERE, "graphics_tmux.npz")):
    g = {}
    with tempfile.TemporaryDirectory() as d:
        for seed, t in tcases.SEEDS.items():
            part = os.path.join(d, seed + ".npz")
            env = dict(os.environ, REF_GRAPHICS_TIME=str(t))
            subprocess.run([sys.executable, os.path.abspath(__file__), "--seed", seed, part], env=env, check=True)
            with np.load(part) as z:
                g.update({k: z[k] for k in z.files})
    np.savez_compressed(path, **g)
    print(f"wrote {sum(1 for k in g if k.endswith('/id'))} tmux outputs; {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    if len(sys.argv) == 4 and sys.argv[1] == "--seed":
        np.savez(sys.argv[3], **seed_outputs(sys.argv[2]))
    else:
        main(*sys.argv[1:])
