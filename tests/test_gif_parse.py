"""b200timg_gif_parse (host only) against the reference's STB source: the screen, the frames its loop collects and
their delays, for every file of the GIF corpus (tests/gif_cases.py) and the Pillow-written files pinned in
tests/golden/gif.npz.  Files whose animation an LZW error ends (found only by decoding, on the device) parse to more
frames than the reference collects; the walk must then stop exactly where the reference's would without the error."""
import os

import numpy as np
import pytest

import gif_cases
import timg_b200
from oracle import gif as G

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "gif.npz"))
NAMES = [str(n) for n in GOLD["names"]]
KEYS = [f"c/{n}" for n in NAMES] + [f"pil/{k}" for k in range(int(GOLD["pil_count"]))]

# corpus files an LZW error ends: the frame whose raster fails, and the frames the walk sees
LZW_ERRORS = {"no-clear-frame0": (0, 4), "no-clear-frame1": (1, 4), "no-clear-last": (3, 4),
              "illegal-code-gt-avail-frame2": (2, 3), "illegal-code-eq-avail-frame2": (2, 3),
              "stream-longer-then-illegal": (2, 3), "too-many-codes-frame1": (1, 2)}


def _file(key):
    return GOLD[f"{key}/file"].tobytes()


@pytest.mark.parametrize("key", KEYS)
def test_parse_matches_the_reference(key):
    data, n_valid = _file(key), int(GOLD[f"{key}/n_valid"])
    delays = list(GOLD[f"{key}/delays"])
    name = key[2:]
    if n_valid == 0 and name not in LZW_ERRORS:
        with pytest.raises(timg_b200.B200Error) as e:            # the reference's source fails: so does the parse
            timg_b200.gif_parse(data)
        assert e.value.code == timg_b200.EINVAL
        return
    w, h, got = timg_b200.gif_parse(data)
    if n_valid:
        assert [w, h] == list(GOLD[f"{key}/wh"])
    if name in LZW_ERRORS:
        bad, walked = LZW_ERRORS[name]
        assert n_valid == bad and len(got) == walked
    else:
        assert len(got) == n_valid
    assert got[:n_valid] == delays


def test_corpus_writer_reproduces_the_pinned_files():
    """tests/gif_cases.py (through oracle/gif.py and oracle/gif_writer.c) still writes the files the pins are of."""
    for name, data in gif_cases.corpus().items():
        assert data == _file(f"c/{name}"), name


@pytest.mark.skipif(not G.have_ref(), reason="oracle/_ref/libtimg_gif_ref.so not built (needs the reference's sources)")
@pytest.mark.parametrize("key", KEYS)
def test_pins_match_the_live_reference(key):
    import hashlib
    data = _file(key)
    ref = G.ref_stb_gif(data)
    frames = ref[0] if ref is not None else []
    assert len(frames) == int(GOLD[f"{key}/n_valid"])
    assert hashlib.sha256(b"".join(f.tobytes() for f in frames)).hexdigest() == str(GOLD[f"{key}/sha"])
    if ref is not None:
        w, h, delays = timg_b200.gif_parse(data)
        assert delays[:len(frames)] == list(ref[1][:, 4])
        assert (ref[1][:, 0] == w).all() and (ref[1][:, 1] == h).all()


def test_delays_are_ten_times_the_last_gce():
    pal = np.arange(12, dtype=np.uint8).reshape(4, 3)
    idx = np.zeros((2, 2), np.uint8)
    data = G.gif(2, 2, [dict(idx=idx, gce=dict(delay=7)), dict(idx=idx, gce=None), dict(idx=idx, gce=dict(delay=65535))],
                 gpal=pal)
    assert timg_b200.gif_parse(data) == (2, 2, [70, 70, 655350])


@pytest.mark.parametrize("data", [b"", b"GIF8", b"GIF88a" + bytes(20), b"\x89PNG\r\n\x1a\n" + bytes(40),
                                  b"GIF89a" + bytes(7) + b"\x3b",                                 # no frame
                                  G.gif(0, 5, [dict(idx=np.zeros((0, 0), np.uint8))], gpal=np.zeros((2, 3))),
                                  G.gif(5, 0, [dict(idx=np.zeros((0, 0), np.uint8))], gpal=np.zeros((2, 3)))])
def test_parse_rejects(data):
    with pytest.raises(timg_b200.B200Error) as e:
        timg_b200.gif_parse(data)
    assert e.value.code == timg_b200.EINVAL


def test_parse_null_pointers():
    import ctypes as C
    L = timg_b200.lib()
    data = _file(KEYS[0])
    w = C.c_int()
    assert L.b200timg_gif_parse(None, 10, C.byref(w), C.byref(w), C.byref(w), None, 0) == timg_b200.EINVAL
    assert L.b200timg_gif_parse(data, len(data), None, C.byref(w), C.byref(w), None, 0) == timg_b200.EINVAL
