"""The decoder edge cases (tests/decode_edge_cases.py) on the GPU: every case against its pin in
tests/golden/decode_edges.npz and, where oracle/gif.mk's door onto the reference's STB source is built, against the
reference itself by test_decode_gpu.check's rules.  PNG and JPEG cases are decoded alone and behind 1, 2 and 5 clean
files (for JPEG, with odd subsequence counts, so every call-global sync CTA boundary moves); the statuses and
canvases must not change.  A JPEG case aimed behind n front files has its event at the sync-CTA edge it names in
the call with those n files in front."""
import collections
import functools
import hashlib

import numpy as np
import pytest

import decode_edge_cases as E
import timg_b200
from oracle import gif as G
from test_decode_gpu import check

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=1)
def _by_class():
    out = collections.defaultdict(list)
    for c in E.all_cases():
        out[(c.fmt, c.cls)].append(c)
    return out


FILE_CLASSES = sorted(k for k in _by_class() if k[0] != "gif")
GIF_CASES = [c.name for c in E.gif_cases()]


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _placement(c, front):
    """Where the plan model puts a JPEG case's event behind `front` (for the failure message)."""
    if c.cls not in ("jpeg_flip", "jpeg_cut", "jpeg_huffman_error"):
        return ""
    lengths = [len(s) for s in E.destuffed_map(E.golden_bases()[c.name.split("_")[1]])]
    fl = [[len(s) for s in E.destuffed_map(f)] for f in front]
    return str(E.jpeg_place(fl, lengths, c.where["seg"], c.where["off"]))


@pytest.mark.parametrize("key", FILE_CLASSES, ids=[k[1] for k in FILE_CLASSES])
def test_file_cases(ctx, key):
    fmt, _ = key
    pins = E.golden()
    fronts = E.front_files() if fmt == "jpeg" else E.png_front_files()
    decode = ctx.jpeg_frames if fmt == "jpeg" else ctx.png_frames
    for c in _by_class()[key]:
        if c.cls.startswith("png_window_") and "bit" in c.where:
            assert E.png_locate(c.where["plan"]["windows"], c.where["bit"]) == \
                (c.where["window"], c.where["sub"], c.where["delta"]), c.name
        if "front" in c.where:                     # the plan model puts the event at call-global subsequence k
            lengths = [len(s) for s in E.destuffed_map(E.golden_bases()[c.name.split("_")[1]])]
            fl = [[len(s) for s in E.destuffed_map(f)] for f in fronts[:c.where["front"]]]
            assert E.jpeg_place(fl, lengths, c.where["seg"], c.where["off"])["sub"] == c.where["k"] - (c.where["d"] < 0)
        want, sha = pins[c.name]
        canv, status = decode([c.data])
        got = int(status[0])
        assert got == want, f"{c.name}: status {got}, pinned {want} {_placement(c, [])}"
        if want == 1:
            assert _sha(canv[0]) == sha, f"{c.name}: canvas differs from the pin {_placement(c, [])}"
        if G.have_ref():
            check(c.name, c.data, canv[0], got)
        for n in (1, 2, 5):
            bc, bs = decode(fronts[:n] + [c.data])
            assert (bs[:n] == 1).all(), f"{c.name}: a front file failed"
            assert int(bs[n]) == got, f"{c.name} behind {n}: status {int(bs[n])}, alone {got} {_placement(c, fronts[:n])}"
            if got == 1:
                assert (bc[n] == canv[0]).all(), f"{c.name} behind {n}: canvas differs {_placement(c, fronts[:n])}"


@pytest.mark.parametrize("name", GIF_CASES)
def test_gif_cases(ctx, name):
    c = next(c for c in E.gif_cases() if c.name == name)
    want_n, sha = E.golden()[name]
    try:
        timg_b200.gif_parse(c.data)
    except timg_b200.B200Error:
        assert want_n == 0, f"{name}: the host parse refuses a file the reference decodes"
        return
    frames, n_valid = ctx.gif_frames(c.data)
    assert n_valid == want_n, f"{name}: {n_valid} frames, pinned {want_n}"
    assert hashlib.sha256(b"".join(np.ascontiguousarray(f).tobytes() for f in frames[:n_valid])).hexdigest() == sha
    if G.have_ref():
        ref = G.ref_stb_gif(c.data)
        want = ref[0] if ref is not None else []
        assert n_valid == len(want)
        for k in range(n_valid):
            assert (frames[k] == want[k]).all(), f"{name}: frame {k}"
