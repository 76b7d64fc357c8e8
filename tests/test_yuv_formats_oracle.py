"""CPU checks of the restatement behind the 4:2:2 / 4:4:4 / 4:4:0 / 10-bit video front (tests/yuv_cases.py): its
distance to the libswscale 9.1 bundled with the image's OpenCV wheel, called as the reference calls it
(sws_getContext(fmt -> RGBA, SWS_BILINEAR) + sws_scale), and its agreement with the 4:2:0 statement the I420 / NV12
kernels are held to.  No GPU needed.

Stated tolerances (max / mean absolute error over R, G, B against libswscale), per format.  Measured with this file's
inputs over GEOMS, limited and (where libav has a yuvj twin) full range:
    I422    max 9, mean 3.09      I420_10 max 10, mean 2.51
    I444    max 1, mean 0.01      I422_10 max 9,  mean 3.09
    I440    max 8, mean 2.50      I444_10 max 1,  mean 0.01
                                  P010    max 10, mean 2.51
4:4:4 matches because libswscale interpolates its chroma at the full output width and so does the restatement; the
subsampled formats keep libswscale's half-width chroma and its fixed-point arithmetic accounts for the rest (the same
distance as I420 in test_yuv_gpu.py).
"""
import os
import sys

import numpy as np
import pytest

import oracle
import timg_b200
from timg_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import yuv_cases as Y  # noqa: E402

GEOMS = [(640, 480, 450, 337, "photo"), (1920, 1080, 320, 90, "photo"), (256, 128, 300, 200, "noise"),
         (3840, 216, 2700, 152, "photo"), (64, 48, 64, 48, "noise"), (130, 98, 67, 50, "alpha")]

SWS_TOL = {Y.I422: (12, 3.5), Y.I444: (2, 0.05), Y.I440: (12, 3.0), Y.I420_10: (12, 3.0), Y.I422_10: (12, 3.5),
           Y.I444_10: (2, 0.05), Y.P010: (12, 3.0)}
YUVJ = (Y.I422, Y.I444, Y.I440)          # the new formats whose full-range variant is a libav yuvj format


def _frame(fmt, iw, ih, kind):
    return Y.rgba_to_yuv_np(synth.frame_np(3 + iw, iw, ih, kind), fmt)


@pytest.mark.parametrize("fmt", Y.NEW_FORMATS, ids=lambda f: Y.NAMES[f])
@pytest.mark.parametrize("iw,ih,ow,oh,kind", GEOMS)
def test_restatement_matches_libswscale(fmt, iw, ih, ow, oh, kind):
    if not oracle.swscale():
        pytest.skip("no libswscale in this environment")
    buf = _frame(fmt, iw, ih, kind)
    planes = Y.planes_np(buf, fmt, iw, ih)
    tmax, tmean = SWS_TOL[fmt]
    for fr in ((0, Y.FULL_RANGE) if fmt in YUVJ else (0,)):
        want = Y.yuv_to_rgba_np(planes, fmt, ow, oh, full_range=bool(fr))
        ref = Y.sws_yuv_to_rgba(buf, fmt | fr, iw, ih, ow, oh)
        e = np.abs(want[..., :3].astype(int) - ref[..., :3])
        assert e.max() <= tmax and e.mean() <= tmean, (Y.NAMES[fmt], fr, int(e.max()), float(e.mean()))
        assert (want[..., 3] == 255).all()


@pytest.mark.parametrize("iw,ih,ow,oh,kind", GEOMS)
def test_420_restatement_equals_yuv420_statement(iw, ih, ow, oh, kind):
    """The general statement on I420 / NV12 is the one the existing 4:2:0 kernels are held to, bit for bit."""
    i420 = oracle.rgba_to_i420_np(synth.frame_np(5 + iw, iw, ih, kind))
    assert (Y.rgba_to_yuv_np(synth.frame_np(5 + iw, iw, ih, kind), Y.I420) == i420).all()
    Yp, U, V = Y.planes_np(i420, Y.I420, iw, ih)
    nv12 = np.concatenate([Yp.reshape(-1), np.stack([U, V], -1).reshape(-1)])
    assert (Y.rgba_to_yuv_np(synth.frame_np(5 + iw, iw, ih, kind), Y.NV12) == nv12).all()
    for fr in (False, True):
        want = oracle.yuv420_to_rgba_np(i420, iw, ih, ow, oh, full_range=fr)
        assert (Y.yuv_to_rgba_np(Y.planes_np(i420, Y.I420, iw, ih), Y.I420, ow, oh, fr) == want).all()
        want = oracle.yuv420_to_rgba_np(nv12, iw, ih, ow, oh, nv12=True, full_range=fr)
        assert (Y.yuv_to_rgba_np(Y.planes_np(nv12, Y.NV12, iw, ih), Y.NV12, ow, oh, fr) == want).all()


def test_10bit_statement_reads_only_the_value_bits():
    iw, ih = 64, 48
    img = synth.frame_np(11, iw, ih, "photo")
    rng = np.random.default_rng(5)
    for fmt in (Y.I420_10, Y.I422_10, Y.I444_10, Y.P010):
        buf = Y.rgba_to_yuv_np(img, fmt)
        stray = rng.integers(0, 64, buf.size).astype(np.uint16)
        noisy = buf | (stray if fmt == Y.P010 else stray << 10)
        for a, b in zip(Y.planes_np(buf, fmt, iw, ih), Y.planes_np(noisy, fmt, iw, ih)):
            assert (a == b).all()


def test_layouts_and_libav_names():
    for fmt in Y.LAYOUT:
        buf = Y.rgba_to_yuv_np(synth.frame_np(1, 32, 16, "photo"), fmt)
        assert buf.nbytes == timg_b200.yuv_frame_bytes(fmt, 32, 16) == buf.itemsize * Y.frame_samples(fmt, 32, 16)
        assert timg_b200.yuv_frame_bytes(fmt | timg_b200.FMT_FULL_RANGE, 32, 16) == buf.nbytes
        if fmt >= Y.I420_10:
            assert buf.dtype == np.uint16 and int(buf.max()) < (1 << 16) and (fmt == Y.P010 or int(buf.max()) < 1024)
    assert [getattr(timg_b200, "FMT_" + Y.NAMES[f]) for f in sorted(Y.LAYOUT)] == sorted(Y.LAYOUT)
    if not oracle.swscale():
        pytest.skip("no libswscale in this environment")
    ids = {Y.LAYOUT[f][0]: Y.av_pix_fmt(Y.LAYOUT[f][0]) for f in Y.LAYOUT}
    assert all(v is not None for v in ids.values()) and len(set(ids.values())) == len(ids), ids
    assert ids["yuv420p"] == 0 and ids["nv12"] == 23          # the ids oracle.sws_scale_np documents
    assert Y.av_pix_fmt("no-such-format") is None
