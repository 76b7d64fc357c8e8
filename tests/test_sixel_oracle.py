"""CPU checks of the sixel restatement (PARITY UNPINNED: libsixel is not in the reference tree):
stream grammar, decoder round trip, and how far the order-free "device semantics" (mode 1) are
from the libsixel-faithful raster-order semantics (mode 0)."""
import re

import numpy as np

import oracle
from timg_b200 import synth


def pct(pal):
    return ((pal.astype(int) * 100 + 127) // 255) * 255 // 100


def test_stream_grammar_and_roundtrip():
    fb = synth.frame_np(7, 97, 36, "photo")
    data, det = oracle.sixel_encode(fb, True)
    assert data.startswith(b'\x1bPq"1;1;97;36#0;2;') and data.endswith(b"\x1b\\")
    assert re.fullmatch(rb'\x1bPq"1;1;97;36(#\d+;2;\d+;\d+;\d+){%d}[#!$\-0-9?-~]+\x1b\\' % det["ncolors"], data)
    img, used = oracle.sixel_decode(data)
    assert img.shape == (36, 97, 3) and used <= 256
    assert (img == pct(det["palette"])[det["index"]]).all()
    assert data.count(b"-") == 36 // 6 - 1


def test_device_stream_by_hand():
    """oracle.sixel_stream, the statement of the device emitters' bytes, on a 5x12 frame written out by hand."""
    pal = np.array([[0, 0, 0], [255, 0, 0], [0, 0, 255]], np.uint8)
    idx = np.zeros((12, 5), np.uint8)
    idx[:6, 1:3] = 1
    idx[0, 4] = 2
    idx[6:] = 2
    want = (b'\x1bPq"1;1;5;12#0;2;0;0;0#1;2;100;0;0#2;2;0;0;100'
            b"#0~??~}$#1?~~$#2!4?@"      # band 0: colour 0's runs (a bits change at x=4 starts one), gaps as '?'
            b"-#2!5~\x1b\\")             # band 1: one run of the whole width
    assert oracle.sixel_stream(pal, idx) == want


def test_device_stream_decodes_to_the_index_plane():
    rng = np.random.default_rng(5)
    for w, h, n, runs in [(1, 6, 1, 1), (97, 36, 256, 1), (300, 18, 5, 9), (4095, 12, 40, 60), (23, 24, 2, 3)]:
        pal = rng.integers(0, 256, (n, 3), dtype=np.uint8)
        idx = rng.integers(0, n, (h, (w + runs - 1) // runs), dtype=np.uint8).repeat(runs, 1)[:, :w].copy()
        data = oracle.sixel_stream(pal, idx)
        img, _ = oracle.sixel_decode(data)
        assert (img == pct(pal)[idx]).all(), (w, h, n)
        assert data.count(b"-") == h // 6 - 1


def test_few_colours_means_no_dither():
    fb = np.zeros((12, 40, 4), np.uint8)
    fb[..., 3] = 255
    fb[:, :20, 0] = 200
    fb[6:, :, 1] = 96
    data, det = oracle.sixel_encode(fb, True)
    assert det["origcolors"] == 4 and det["ncolors"] == 4
    img, used = oracle.sixel_decode(data)
    assert used == 4
    want = fb[..., :3] & 0xF8                         # palette entries are the 5-bit cell bases
    assert (img == pct(want)).all()


def test_device_semantics_stay_close_to_libsixel_semantics():
    """mode 1 (order-free) vs mode 0 (raster order, first-come memo): same quality, different pattern."""
    for kind, w, h in [("photo", 337, 192), ("noise", 200, 96), ("alpha", 160, 120)]:
        fb = synth.frame_np(1234, w, h, kind)
        a, _ = oracle.sixel_decode(oracle.sixel_encode(fb, mode=0))
        b, _ = oracle.sixel_decode(oracle.sixel_encode(fb, mode=1))
        src = fb[..., :3]
        ea, eb = oracle.mean_delta_e(a, src, 2), oracle.mean_delta_e(b, src, 2)
        assert abs(ea - eb) < 0.5, (kind, ea, eb)
        assert oracle.mean_delta_e(a, b, 2) < 3.0, kind


def test_fs_quirks_are_restated():
    """Last row / last column do not diffuse; error is clamped into 8-bit pixels."""
    fb = synth.frame_np(3, 64, 12, "photo")
    _, d = oracle.sixel_encode(fb, True)
    assert d["origcolors"] > 256 or d["ncolors"] <= 256
