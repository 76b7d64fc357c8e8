"""Deterministic inputs of the kitty tmux-form goldens (tests/golden/graphics_tmux.npz, written by
tests/golden/make_graphics_tmux_golden.py).

The reference seeds kitty's image ids from time(): id = (time << 7) + k for its k-th image.  Each seed below is one
pinned time, so the ids, and with them the colour escape and the id diacritic of every placeholder, are reproducible:
  t0     time 0: ids 1, 2, ... -- no id diacritic, colour 0:0:<k>
  msb2   id >> 24 = 3 (a 2-byte diacritic)
  msb3   id >> 24 = 200 (a 3-byte diacritic), 10-digit ids
  msb255 id >> 24 = 255 (the id 0xffffffff would have), 10-digit ids
"""
from timg_b200 import synth

import graphics_cases as gcases
from cases import c4_frames, sha  # noqa: F401  (re-exported for the golden writer and the tests)

SEEDS = {"t0": 0, "msb2": (3 << 17) | 0x5, "msb3": (200 << 17) | 0x123, "msb255": 0x1FF3579}
CELL = (9, 18)                          # cell size of the frame cases; Send(x = 18) indents the grid by 2 cells
X = 18
C4_FRAMES = 3                           # 4K -> 337x190 (C4), composed onto black
C2_W, C2_H = 2700, 1519                 # C2's output geometry: 300 columns at 9-px cells, 85 rows at 18 px


def geometry_cases():
    """(name, frame, rgb24, cell, x) reaching the grid's edges: 1-px cells whose columns (300x4) or rows (4x300) reach
    diacritic values 283..296 and >= 297, no column at all (w < cell_x_px), heights of exactly two cells and one pixel
    more, indents of 0, 1 and 12 cells."""
    f = synth.frame_np
    return [("cells1_300x4_rgb0", f(31, 300, 4, "noisea"), 0, (1, 1), 0),
            ("cells1_4x300_rgb1", f(32, 4, 300, "noisea"), 1, (1, 1), 0),
            ("cols0_5x20_rgb0", f(33, 5, 20, "noisea"), 0, (9, 18), 0),
            ("hexact_27x36_rgb1", f(34, 27, 36, "noisea"), 1, (9, 18), 9),
            ("hexact1_27x37_rgb0", f(35, 27, 37, "alpha"), 0, (9, 18), 108),
            ("indent12_40x19_rgb1", f(36, 40, 19, "noisea"), 1, (4, 19), 48)]


def seed_cases():
    """(name, frame, rgb24, cell, x) sent under every id seed."""
    f = synth.frame_np
    return [("s_2x3_rgb1", f(41, 2, 3, "noisea"), 1, CELL, X),
            ("s_70x40_rgb0", f(42, 70, 40, "noisea"), 0, CELL, X),
            ("s_cells1_300x4_rgb1", f(43, 300, 4, "noisea"), 1, (1, 1), 0)]


def frame_cases():
    """graphics_cases' single frames (both colour types, 3072*k-byte PNGs and one byte either side, several stored
    blocks, alpha) at 9x18 cells, indent 2."""
    return [(name, fb, rgb24, CELL, X) for name, fb, rgb24 in gcases.graphics_frame_cases()]


def c2_frame():
    return synth.frame_np(77, C2_W, C2_H, "photo")


def c4_graphics_frames():
    return c4_frames(C4_FRAMES)
