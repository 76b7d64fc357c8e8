"""The kitty tmux-form goldens (tests/golden/graphics_tmux.npz) are what the reference's own KittyGraphicsCanvas writes
with tmux_passthrough_needed = true, around a stored-block PNG.  Every golden stored in full must unwrap (tmux
passthrough stripped, escapes un-doubled) to kitty commands whose payload decodes to the input frame, followed by a
rows x cols grid of Unicode placeholders carrying each cell's row and column and the image id; and
b200timg_graphics_size must give every golden's length and be largest at id 0xffffffff.  No GPU.

The row / column diacritics are not restated here: the map from a diacritic's bytes to its value is read off the
golden of a 300x4 frame at 1-px cells, whose first row carries values 0..299 as its columns."""
import base64
import os
import re
import sys

import numpy as np
import pytest

import timg_b200

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import graphics_tmux_cases as tcases  # noqa: E402
from test_graphics_oracle import png_pixels  # noqa: E402

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "graphics_tmux.npz"))
PLACEHOLDER = "\U0010EEEE".encode()
DIAC_N = 297


def all_cases():
    """name -> (frame, rgb24, cell, x) of every case that has a single-frame golden."""
    return {name: (fb, rgb24, cell, x) for name, fb, rgb24, cell, x in
            tcases.frame_cases() + tcases.geometry_cases() + tcases.seed_cases() + [("c2_rgb1", None, 1, tcases.CELL, tcases.X)]}


def golden_keys():
    """every "<seed>/<case>" (c4 frames included)"""
    return sorted(k[:-len("/id")] for k in GOLD.files if k.endswith("/id"))


def unwrap_tmux(text):
    """(kitty commands inside tmux's passthrough wrappers, the rest): "\\ePtmux;" + content with every escape doubled
    + "\\e\\\\", back to back."""
    cmds, pos = [], 0
    while text.startswith(b"\033Ptmux;", pos):
        pos += 7
        out = bytearray()
        while True:
            b = text[pos]
            if b == 0x1B:
                nxt = text[pos + 1]
                if nxt == 0x1B:
                    out.append(0x1B)
                    pos += 2
                    continue
                assert nxt == ord("\\"), text[pos:pos + 8]
                pos += 2
                break
            out.append(b)
            pos += 1
        cmds.append(bytes(out))
    return cmds, text[pos:]


def kitty_tmux_payload(text):
    """(base64 payload, i=, c=, r=, the placeholder grid) of a tmux-form frame, checking every command's framing."""
    cmds, rest = unwrap_tmux(text)
    assert cmds
    m = re.fullmatch(rb"\033_Ga=T,i=(\d+),q=2,f=100,m=([01]),U=1,c=(\d+),r=(\d+);([A-Za-z0-9+/=]+)\033\\", cmds[0])
    assert m, cmds[0][:80]
    id_, more, cols, rows = int(m.group(1)), int(m.group(2)), int(m.group(3)), int(m.group(4))
    parts = [m.group(5)]
    for c in cmds[1:]:
        assert more and len(parts[-1]) == 4096
        m = re.fullmatch(rb"\033_Gq=2,m=([01]);([A-Za-z0-9+/=]+)\033\\", c)
        assert m, c[:40]
        more = int(m.group(1))
        parts.append(m.group(2))
    assert not more and 0 < len(parts[-1]) <= 4096
    assert rest.startswith(b"\r")
    return b"".join(parts), id_, cols, rows, rest[1:]


def diacritic_tokens(b):
    """a run of diacritics -> its tokens: one UTF-8 code point, plus the ASCII hex digit that follows it in the
    reference's entries above U+FFFF"""
    toks, s = [], b.decode("utf-8")
    for ch in s:
        if ch in "0123456789ABCDEF":
            assert toks
            toks[-1] += ch
        else:
            toks.append(ch)
    return toks


def diacritic_values():
    """token -> value, from row 0 of the 1-px-cell 300x4 golden: cell c of row 0 is D(0) D(c)."""
    text = GOLD["t0/cells1_300x4_rgb0"].tobytes()
    grid = kitty_tmux_payload(text)[4]
    row0 = grid[:grid.index(b"\033[39m")]
    cells = row0.split(PLACEHOLDER)[1:]
    toks = [diacritic_tokens(c) for c in cells]
    assert len(toks) == 300 and all(t[0] == toks[0][0] for t in toks)
    assert all(len(t) == 2 for t in toks[:DIAC_N]) and all(len(t) == 1 for t in toks[DIAC_N:])
    values = {t[1]: c for c, t in enumerate(toks[:DIAC_N])}
    assert len(values) == DIAC_N and values[toks[0][0]] == 0
    return values


def check_grid(grid, id_, cols, rows, indent, values):
    """rows lines of [indent] colour(id), cols placeholders (row, column, [id >> 24]), reset + "\\n\\r"."""
    msb = id_ >> 24
    head = (b"\033[%dC" % indent if indent > 0 else b"") + b"\033[38:2:%d:%d:%dm" % ((id_ >> 16) & 255, (id_ >> 8) & 255, id_ & 255)
    lines = grid.split(b"\033[39m\n\r")
    assert len(lines) == rows + 1 and lines[-1] == b""
    inverse = {v: t for t, v in values.items()}
    for r, line in enumerate(lines[:-1]):
        assert line.startswith(head), (r, line[:30])
        cells = line[len(head):].split(PLACEHOLDER)
        assert cells[0] == b"" and len(cells) == cols + 1, (r, len(cells))
        for c, cell in enumerate(cells[1:]):
            want = [inverse[v] for v in (r, c) if v < DIAC_N] + ([inverse[msb]] if msb else [])
            assert diacritic_tokens(cell) == want, (r, c)


def frame_of(name):
    fb, rgb24, _, _ = all_cases()[name]
    return fb, rgb24


@pytest.mark.parametrize("key", [k for k in golden_keys() if k in GOLD.files])
def test_golden_unwraps_decodes_and_places_the_frame(key):
    text = GOLD[key].tobytes()
    w, h, rgb24, cx, cy, indent = (int(v) for v in GOLD[key + "/geo"])
    fb, rgb24_case = frame_of(key.split("/", 1)[1])
    assert rgb24 == rgb24_case and fb.shape[:2] == (h, w)
    b64, id_, cols, rows, grid = kitty_tmux_payload(text)
    assert id_ == int(GOLD[key + "/id"][0])
    assert (cols, rows) == (w // cx, -(-h // cy))
    px, ctype = png_pixels(base64.b64decode(b64, validate=True))
    assert ctype == (2 if rgb24 else 6)
    assert (px == (fb[..., :3] if rgb24 else fb)).all()
    check_grid(grid, id_, cols, rows, indent, diacritic_values())


def test_goldens_cover_the_grid_edges_and_the_id_seeds():
    full = [k for k in golden_keys() if k in GOLD.files]
    geos = {k: [int(v) for v in GOLD[k + "/geo"]] for k in full}
    assert any(w // cx > DIAC_N for w, h, _, cx, cy, _ in geos.values())              # columns past the list
    assert any(-(-h // cy) > DIAC_N for w, h, _, cx, cy, _ in geos.values())          # rows past the list
    assert any(w // cx == 0 for w, h, _, cx, cy, _ in geos.values())
    assert {0, 1, 2, 12} <= {g[5] for g in geos.values()}
    assert any(h % cy == 0 for w, h, _, cx, cy, _ in geos.values()) and any(h % cy == 1 for w, h, _, cx, cy, _ in geos.values())
    msbs = {int(GOLD[k + "/id"][0]) >> 24 for k in full}
    assert {0, 3, 200, 255} <= msbs
    assert max(int(GOLD[k + "/id"][0]) for k in full) >= 10 ** 9


def test_graphics_size_equals_every_golden_length():
    checked = 0
    for key in golden_keys():
        w, h, rgb24, cx, cy, indent = (int(v) for v in GOLD[key + "/geo"])
        n = GOLD[key].size if key in GOLD.files else int(GOLD[key + "/len"][0])
        id_ = int(GOLD[key + "/id"][0])
        assert timg_b200.graphics_size(timg_b200.KITTY_TMUX, w, h, rgb24, id_, cell=(cx, cy), indent=indent) == n, key
        checked += 1
    assert checked >= 40


def test_graphics_size_is_largest_at_the_largest_id():
    """b200timg_graphics_batch sizes its chunk buffers with the size at id 0xffffffff."""
    rng = np.random.default_rng(5)
    ids = [0, 1, 9, 10, 255, 256, 65535, 1 << 24, (3 << 24) + 77, 200 << 24, 0xFEFFFFFF, 0xFF000000, 0xFFFFFFFE,
           *rng.integers(0, 1 << 32, 40, dtype=np.uint64).tolist()]
    for w, h, cx, cy, indent in ((1, 1, 1, 1, 0), (300, 4, 1, 1, 0), (4, 300, 1, 1, 3), (2700, 1519, 9, 18, 2),
                                 (5, 20, 9, 18, 0), (640, 480, 7, 15, 120), (3840, 2, 1, 1, 0)):
        for rgb24 in (0, 1):
            top = timg_b200.graphics_size(timg_b200.KITTY_TMUX, w, h, rgb24, 0xFFFFFFFF, cell=(cx, cy), indent=indent)
            for id_ in ids:
                n = timg_b200.graphics_size(timg_b200.KITTY_TMUX, w, h, rgb24, int(id_), cell=(cx, cy), indent=indent)
                assert 0 < n <= top, (w, h, cx, cy, indent, id_)


def test_graphics_size_rejects_bad_cells_and_indents():
    T = timg_b200.KITTY_TMUX
    assert timg_b200.graphics_size(T, 10, 10, cell=(9, 18)) > 0
    for cell, indent in (((0, 18), 0), ((9, 0), 0), ((-1, 18), 0), ((9, -3), 0), ((9, 18), -1), (None, 0)):
        assert timg_b200.graphics_size(T, 10, 10, cell=cell, indent=indent) == 0, (cell, indent)
    assert timg_b200.graphics_size(3, 10, 10, cell=(9, 18)) == 0
