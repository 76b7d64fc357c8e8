"""The kitty / iTerm2 goldens (tests/golden/graphics.npz) are what the reference's own canvases write with a
stored-block compressor in place of libdeflate.  Every golden stored in full must parse as its protocol says and
decode to the input frame's pixels -- this pins the stand-in compressor, so the byte identity tests on the GPU
(test_graphics_gpu.py) are not circular -- and b200timg_graphics_size must give every golden's length.  No GPU."""
import base64
import os
import re
import struct
import sys
import zlib

import numpy as np
import pytest

import timg_b200

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import graphics_cases as gcases  # noqa: E402

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "graphics.npz"))
PROTOCOLS = {"kitty": gcases.KITTY, "iterm2": gcases.ITERM2}


def kitty_payload(text):
    """base64 payload of a kitty stream (src/kitty-canvas.cc:190-229, no tmux), checking every chunk's framing."""
    m = re.match(rb"\033_Ga=T,i=(\d+),q=2,f=100,m=([01]);", text)
    assert m, text[:40]
    pos, more, parts = m.end(), int(m.group(2)), []
    while True:
        end = text.index(b"\033\\", pos)
        chunk = text[pos:end]
        assert 0 < len(chunk) <= 4096 and (len(chunk) == 4096 or not more), len(chunk)
        parts.append(chunk)
        pos = end + 2
        if not more:
            break
        m = re.compile(rb"\033_Gq=2,m=([01]);").match(text, pos)
        assert m, text[pos:pos + 20]
        pos, more = m.end(), int(m.group(1))
    assert text[pos:] == b"\n"
    return b"".join(parts)


def iterm2_payload(text, w, h):
    m = re.match(rb"\033\]1337;File=size=(\d+);width=(\d+)px;height=(\d+)px;inline=1:", text)
    assert m and (int(m.group(2)), int(m.group(3))) == (w, h)
    assert text.endswith(b"\a\n")
    data = text[m.end():-2]
    assert len(base64.b64decode(data)) == int(m.group(1))
    return data


def png_pixels(data):
    """Parse a PNG: chunk CRCs, IHDR, zlib stream (Adler-32 checked by zlib), Sub filter undone."""
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, chunks = 8, []
    while pos < len(data):
        n, typ = struct.unpack(">I4s", data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + n]
        assert zlib.crc32(typ + body) == struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0], typ
        chunks.append((typ, body))
        pos += 12 + n
    assert [c[0] for c in chunks] == [b"IHDR", b"IDAT", b"IEND"]
    w, h, depth, ctype = struct.unpack(">IIBB", chunks[0][1][:10])
    bpp = 4 if ctype == 6 else 3
    raw = np.frombuffer(zlib.decompress(chunks[1][1]), np.uint8).reshape(h, 1 + w * bpp)
    assert (raw[:, 0] == 1).all()
    return np.cumsum(raw[:, 1:].reshape(h, w, bpp).astype(np.uint32), axis=1).astype(np.uint8), ctype


def full_goldens():
    """(protocol name, case name, frame, rgb24) of every golden stored in full."""
    out = []
    for pname in PROTOCOLS:
        for name, fb, rgb24 in gcases.graphics_frame_cases():
            if f"{pname}/{name}" in GOLD:
                out.append((pname, name, fb, rgb24))
    return out


@pytest.mark.parametrize("pname,name,fb,rgb24", full_goldens(), ids=lambda v: v if isinstance(v, str) else "")
def test_golden_parses_and_decodes_to_the_frame(pname, name, fb, rgb24):
    text = GOLD[f"{pname}/{name}"].tobytes()
    h, w = fb.shape[:2]
    b64 = kitty_payload(text) if pname == "kitty" else iterm2_payload(text, w, h)
    if pname == "kitty":
        assert int(re.match(rb"\033_Ga=T,i=(\d+),", text).group(1)) == int(GOLD[f"{pname}/{name}/id"][0])
    px, ctype = png_pixels(base64.b64decode(b64, validate=True))
    assert ctype == (2 if rgb24 else 6)
    assert (px == (fb[..., :3] if rgb24 else fb)).all()


def test_several_stored_blocks_and_chunk_boundaries_are_covered():
    names = [n for _, n, _, _ in full_goldens()]
    assert any(n.startswith("blocks") for n in names)
    for rgb24 in (0, 1):
        sizes = {gcases.png_size(fb.shape[1], fb.shape[0], r) for _, fb, r in gcases.graphics_frame_cases() if r == rgb24}
        for k in range(1, 20):
            if 3072 * k in sizes:
                assert {3072 * k - 1, 3072 * k + 1} <= sizes
                break
        else:
            pytest.fail("no PNG of exactly 3072*k bytes")


def test_graphics_size_equals_every_golden_length():
    geo = {name: (fb.shape[1], fb.shape[0], rgb24) for name, fb, rgb24 in gcases.graphics_frame_cases()}
    _, ow, oh, _ = gcases.graphics_checker_case()
    geo["checker_rgb0"], geo["checker_rgb1"] = (ow, oh, 0), (ow, oh, 1)
    checked = 0
    for key in GOLD.files:
        parts = key.split("/")
        if parts[-1] == "id" or parts[-1] == "sha":
            continue
        pname, name = parts[0], parts[1]
        w, h, rgb24 = geo[name] if name in geo else (337, 190, 1)          # c4_rgb1/<f>/len
        n = int(GOLD[key][0]) if parts[-1] == "len" else GOLD[key].size
        idkey = key[:-len("/len")] if parts[-1] == "len" else key
        id_ = int(GOLD[idkey + "/id"][0])
        assert timg_b200.graphics_size(PROTOCOLS[pname], w, h, rgb24, id_) == n, key
        assert gcases.png_size(w, h, rgb24) == timg_b200.lib().b200timg_png_size(w, h, rgb24)
        checked += 1
    assert checked >= 40


def test_graphics_size_rejects_unknown_protocol():
    assert timg_b200.graphics_size(3, 10, 10) == 0
    assert timg_b200.graphics_size(gcases.KITTY, 0, 10) == 0
