"""GPU parity: the resampling kernel through the C ABI vs the CPU oracle (bit-identical to the
reference's STB scaler) and the golden fixtures.  Bit-exact, every geometry."""
import os

import numpy as np
import pytest

import cases
import oracle
from timg_b200 import synth

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")


def test_scale_cuda_matches_golden_and_oracle(ctx):
    g = np.load(os.path.join(G, "scale.npz"))
    for name, img, ow, oh, fmt in cases.scale_cases():
        got = ctx.scale(img, ow, oh, fmt)
        assert (got == g[name]).all(), f"{name}: vs golden, max diff {np.abs(got.astype(int) - g[name]).max()}"
        assert (got == oracle.stb_resize(img, ow, oh, fmt)).all(), name


def test_scale_cuda_random_geometries(ctx):
    rng = np.random.default_rng(12)
    for it in range(60):
        iw, ih = int(rng.integers(1, 500)), int(rng.integers(1, 400))
        mode = it % 5
        if mode == 0:
            ow, oh = int(rng.integers(1, 500)), int(rng.integers(1, 400))
        elif mode == 1:
            ow, oh = max(1, iw // int(rng.integers(1, 12))), max(1, ih // int(rng.integers(1, 12)))
        elif mode == 2:
            ow, oh = iw * int(rng.integers(1, 4)), ih * int(rng.integers(1, 4))
        elif mode == 3:
            ow, oh = iw, int(rng.integers(1, 400))
        else:
            ow, oh = int(rng.integers(1, 500)), ih
        img = synth.frame_np(900 + it, iw, ih, ["noisea", "photo", "alpha", "noise"][it % 4])
        fmt = it % 2
        want = oracle.stb_resize(img, ow, oh, fmt)
        got = ctx.scale(img, ow, oh, fmt)
        assert (got == want).all(), (iw, ih, ow, oh, fmt, int(np.abs(got.astype(int) - want).max()))


def test_scale_cuda_config_geometries_full_size(ctx):
    """BASELINE configs at full size against the oracle: C3 1080p->320x90 and C2 4K->2700x1519."""
    for iw, ih, ow, oh, kind in [(1920, 1080, 320, 90, "photo"), (3840, 2160, 2700, 1519, "photo"),
                                 (3840, 2160, 337, 190, "noise")]:
        img = synth.frame_np(1234, iw, ih, kind)
        want = oracle.stb_resize(img, ow, oh)
        got = ctx.scale(img, ow, oh)
        assert (got == want).all(), (iw, ih, ow, oh)


def test_identity_scale_is_copy(ctx):
    img = synth.frame_np(5, 333, 77, "noisea")
    assert (ctx.scale(img, 333, 77) == img).all()


def _vfirst_small_taps(iw, ih, ow, oh):
    import timg_b200
    h, v = timg_b200.resample_plan(iw, ih, ow, oh, 0), timg_b200.resample_plan(iw, ih, ow, oh, 1)
    return bool(h["flags"] & 1) and not (h["flags"] & 2) and h["widest"] <= 8 and v["widest"] <= 8


def test_scale_cuda_planar_path(ctx):
    """The v3 kernel (opaque tiles) + planar kernel (vertical pass first, <= 8 taps, width % 4 == 0): opaque windows (3 colour
    planes + analytic alpha), windows with partial alpha (weighted planes + alpha plane), windows with
    fully transparent output pixels (un-weighted planes too), tiles mixing all three; both byte orders."""
    rng = np.random.default_rng(77)
    geoms = [(640, 360, 450, 253), (256, 200, 300, 260), (512, 300, 333, 299), (400, 240, 399, 200),
             (1024, 64, 720, 45), (64, 1000, 45, 703), (344, 331, 282, 274), (160, 496, 141, 266),
             (648, 257, 357, 132), (416, 451, 416, 280), (412, 190, 775, 190), (232, 399, 456, 515),
             (308, 379, 618, 335), (260, 137, 804, 73), (32, 222, 608, 513)]
    ran_planar = 0
    for it, (iw, ih, ow, oh) in enumerate(geoms):
        for kind in ("photo", "noise", "noisea", "alpha", "holes"):
            if kind == "holes":                       # opaque photo with fully transparent and faint patches
                img = synth.frame_np(40 + it, iw, ih, "photo")
                for _ in range(6):
                    x0, y0 = int(rng.integers(0, iw)), int(rng.integers(0, ih))
                    img[y0:y0 + int(rng.integers(1, 60)), x0:x0 + int(rng.integers(1, 60)), 3] = int(rng.choice([0, 0, 1, 200]))
            else:
                img = synth.frame_np(40 + it, iw, ih, kind)
            fmt = it % 2
            ctx.profile(True)
            got = ctx.scale(img, ow, oh, fmt)
            rep = ctx.profile_report()
            ctx.profile(False)
            want = oracle.stb_resize(img, ow, oh, fmt)
            assert (got == want).all(), (iw, ih, ow, oh, kind, fmt, int(np.abs(got.astype(int) - want).max()))
            if "resample_planar_kernel" in rep:     # v3 = opaque tiles, planar = the rest
                assert _vfirst_small_taps(iw, ih, ow, oh)
                ran_planar += 1
    assert ran_planar >= 50 or os.environ.get("B200TIMG_NO_PLANAR"), ran_planar


def test_scale_cuda_planar_off_matches(ctx, monkeypatch):
    """Same frame through the planar kernel and through the float4 kernels it replaces."""
    img = synth.frame_np(9, 640, 360, "alpha")
    a = ctx.scale(img, 450, 253)
    monkeypatch.setenv("B200TIMG_NO_PLANAR", "1")
    b = ctx.scale(img, 450, 253)
    assert (a == b).all()


# B200TIMG_FAST_SCALE: fused multiply-adds, no byte*(1/255) .. *255 round trip.  Stated tolerance (BASELINE.md:
# "<= 1 LSB for Mitchell vs STB"): every channel within 1 of the reference, and fewer than 0.5 % of the pixels
# differing at all (measured: <= 0.05 %).
FAST_MAX_LSB = 1
FAST_MAX_FRACTION = 0.005


@pytest.mark.parametrize("iw,ih,ow,oh,kind", [(128, 96, 90, 67, "photo"), (256, 128, 200, 100, "noise"),
                                               (3840, 128, 2700, 90, "photo"), (640, 480, 450, 337, "noise"),
                                               (1024, 64, 720, 45, "photo"), (512, 300, 333, 299, "noisea"),
                                               (640, 360, 450, 253, "alpha")])
def test_scale_cuda_fast_mode_within_one_lsb(ctx, iw, ih, ow, oh, kind):
    img = synth.frame_np(5 + iw, iw, ih, kind)
    for fmt in (0, 1):
        want = oracle.stb_resize(img, ow, oh, fmt)
        got = ctx.scale(img, ow, oh, fmt, fast=True)
        d = np.abs(got.astype(int) - want)
        assert d.max() <= FAST_MAX_LSB, (iw, ih, ow, oh, kind, fmt, int(d.max()))
        assert (d.max(-1) > 0).mean() < FAST_MAX_FRACTION
