"""Every launch shape of the scaler (copy, v3, planar, fixed in both pass orders, the two-pass kernels with each first pass)
against the CPU restatement of the reference's STB scaler (bit for bit) and a plain float64 statement of the same filter
(within 1 LSB).  The cases and the classes they stand for are in scale_shape_cases.py; every case first asks the library
whether it really is in its class."""
import numpy as np
import pytest

import oracle
import scale_shape_cases as sc
import timg_b200
from timg_b200 import synth

pytestmark = pytest.mark.gpu

# the profile name each route's first kernel launches under
KERNEL = {"copy4": "resample_copy_kernel", "copy": "resample_copy_kernel", "v3": "resample_v3_fast_kernel",
          "planar": "resample_planar_kernel", "fixed": "resample_fixed_kernel", "tp_v": "twopass_v1_kernel",
          "tp_h1s": "twopass_h1s_kernel", "tp_h1f": "twopass_h1f_kernel", "tp_h1": "twopass_h1_kernel"}
FAST_MAX_FRACTION = 0.005


def setup(monkeypatch, group, name):
    case = sc.by_name(group)[name]
    sc.apply_env(monkeypatch)
    sc.check_class(case)
    return case


def first_diff(a, b):
    bad = np.argwhere(a != b)
    return f"{len(bad)} differ, first at (y, x, c) = {tuple(bad[0])}: {a[tuple(bad[0])]} != {b[tuple(bad[0])]}" if len(bad) else "equal"


def scale_profiled(ctx, img, case, fast):
    ctx.profile(True)
    got = ctx.scale(img, case.ow, case.oh, case.fmt, fast=fast)
    rep = ctx.profile_report()
    ctx.profile(False)
    return got, rep


def check_case(ctx, case):
    img = sc.frame(case)
    want = oracle.stb_resize(img, case.ow, case.oh, case.fmt)
    exact_route = timg_b200.scale_shape(case.iw, case.ih, case.ow, case.oh)["route"]
    got, rep = scale_profiled(ctx, img, case, False)
    assert (got == want).all(), f"{case.name}: exact ({exact_route}) vs oracle: {first_diff(got, want)}"
    assert KERNEL[exact_route] in rep, (case.name, exact_route, rep)
    ref = sc.ref_f64(img, case.ow, case.oh, case.fmt)
    d = np.abs(got.astype(int) - ref)
    print(f"{case.name}: {exact_route}, {100 * (d.max(-1) > 0).mean():.3f} % of pixels 1 LSB from float64")
    assert d.max() <= 1, f"{case.name}: exact vs float64 statement: {int(d.max())} LSB"
    fast_route = timg_b200.scale_shape(case.iw, case.ih, case.ow, case.oh, fast=True)["route"]
    fast, rep = scale_profiled(ctx, img, case, True)
    assert KERNEL[fast_route] in rep, (case.name, fast_route, rep)
    if fast_route != "v3" or case.kind == "faint":
        # FAST only changes whether v3 runs; a frame without opaque tiles leaves every v3 tile to the planar list kernel
        assert (fast == got).all(), f"{case.name}: FAST ({fast_route}) vs exact: {first_diff(fast, got)}"
        return
    # the float64 statement sits up to 1 LSB from the bit-exact result too (on > 1 % of the pixels of some box
    # enlargements): FAST may add FAST_MAX_FRACTION to the fraction the exact result already has
    exact_frac = (np.abs(got.astype(int) - ref).max(-1) > 0).mean()
    for other, what, base in ((want, "oracle", 0.0), (ref, "float64", exact_frac)):
        d = np.abs(fast.astype(int) - other)
        frac = (d.max(-1) > 0).mean()
        print(f"{case.name}: FAST v3, {100 * frac:.3f} % of pixels 1 LSB from the {what}")
        assert d.max() <= 1, f"{case.name}: FAST vs {what}: {int(d.max())} LSB"
        assert frac < base + FAST_MAX_FRACTION, f"{case.name}: FAST vs {what}: {frac:.4f} (exact: {base:.4f})"


@pytest.mark.parametrize("group", ["class", "threshold", "filter", "edge", "content"])
def test_case_table(ctx, monkeypatch, group):
    for name in sc.names(group):
        check_case(ctx, setup(monkeypatch, group, name))


def _dev(torch, a):
    return timg_b200._device_tensor(torch, a)


@pytest.mark.parametrize("src_off", [0, 16, 4])
@pytest.mark.parametrize("iw,ih,ow,oh", [(640, 360, 450, 253), (200, 200, 114, 114), (3840, 200, 337, 18), (100, 900, 50, 100),
                                         (128, 64, 128, 64)])
def test_scale_dev_batches(ctx, monkeypatch, src_off, iw, ih, ow, oh):
    """b200timg_scale_dev on 3 distinct frames (grid.z) with the source at a 16-byte aligned and at a 4-byte offset: each
    frame equals the oracle, and the call takes the class scale_shape reports for that alignment (an unaligned source
    leaves planar for fixed, the 16-byte copy for the plain one)."""
    import torch
    sc.apply_env(monkeypatch)
    frames = np.stack([synth.frame_np(300 + i, iw, ih, ("photo", "noisea", "alpha")[i]) for i in range(3)])
    frames[1, ::7, ::5, 3] = 0
    frames[1, ih // 4:ih // 2, iw // 4:iw // 2, 3] = 0       # outputs of frame 1 only whose filtered alpha is 0
    flat = np.zeros(frames.nbytes + 64, np.uint8)
    flat[src_off:src_off + frames.nbytes] = frames.reshape(-1)
    d_src = _dev(torch, flat)
    assert d_src.data_ptr() % 16 == 0
    d_out = torch.zeros(3 * ow * oh * 4, dtype=torch.uint8, device=d_src.device)
    s = timg_b200.scale_shape(iw, ih, ow, oh, 3, False, src_off % 16 == 0, True)
    if src_off % 16:
        assert s["route"] not in ("planar", "v3", "copy4"), s
    ctx.profile(True)
    rc = timg_b200.lib().b200timg_scale_dev(ctx.h, d_src.data_ptr() + src_off, iw, ih, timg_b200.FMT_RGBA, d_out.data_ptr(), ow, oh, 3)
    assert rc == 0, timg_b200.lib().b200timg_last_error(ctx.h)
    timg_b200.device_sync(torch)
    rep = ctx.profile_report()
    ctx.profile(False)
    assert KERNEL[s["route"]] in rep, (s["route"], rep)
    out = d_out.cpu().numpy().reshape(3, oh, ow, 4)
    for f in range(3):
        want = oracle.stb_resize(frames[f], ow, oh)
        assert (out[f] == want).all(), f"frame {f}: {first_diff(out[f], want)}"


@pytest.mark.parametrize("start_row", [0, 1, 17, 52])
def test_scale_dev_then_compose_dev(ctx, monkeypatch, start_row):
    """b200timg_scale_dev followed by b200timg_compose_dev with a checkerboard: AlphaComposeBackground from start_row on."""
    import torch
    sc.apply_env(monkeypatch)
    iw, ih, ow, oh, n = 300, 200, 163, 53, 2
    frames = np.stack([synth.frame_np(60 + i, iw, ih, "noisea") for i in range(n)])
    frames[0, 40:90, 30:120, 3] = 0
    d_src = _dev(torch, frames)
    d_out = torch.zeros(n * ow * oh * 4, dtype=torch.uint8, device=d_src.device)
    L = timg_b200.lib()
    assert L.b200timg_scale_dev(ctx.h, d_src.data_ptr(), iw, ih, 0, d_out.data_ptr(), ow, oh, n) == 0
    bg, pat = timg_b200.rgba_u32(20, 40, 60), timg_b200.rgba_u32(200, 180, 160)
    assert L.b200timg_compose_dev(ctx.h, d_out.data_ptr(), ow, oh, n, 1, bg, pat, 5, 3, start_row) == 0, L.b200timg_last_error(ctx.h)
    timg_b200.device_sync(torch)
    out = d_out.cpu().numpy().reshape(n, oh, ow, 4)
    for f in range(n):
        want = oracle.compose_bg(oracle.stb_resize(frames[f], ow, oh), bg, pat, 5, 3, start_row)
        assert (out[f] == want).all(), f"frame {f}: {first_diff(out[f], want)}"


@pytest.mark.parametrize("iw,ih,ow,oh", [(640, 360, 450, 253), (200, 200, 113, 114), (3840, 200, 337, 18), (100, 900, 50, 100),
                                         (2000, 100, 27, 50), (64, 64, 65, 65), (128, 64, 128, 64)])
def test_kitty_batch_composes_in_every_route(ctx, monkeypatch, iw, ih, ow, oh):
    """A kitty batch (stored PNGs) with a checkerboard background: the compose fused into each route's epilogue.  The PNG's
    pixels equal oracle.compose_bg(oracle.stb_resize(...))."""
    import base64
    from test_graphics_oracle import kitty_payload, png_pixels
    sc.apply_env(monkeypatch)
    n = 2
    frames = np.stack([synth.frame_np(80 + i, iw, ih, ("noisea", "alpha")[i]) for i in range(n)])
    frames[0, ::9, ::4, 3] = 0
    frames[1, ih // 3:ih // 2, iw // 3:iw // 2, 3] = 0       # outputs of frame 1 only whose filtered alpha is 0
    bg, pat = timg_b200.rgba_u32(10, 20, 30), timg_b200.rgba_u32(220, 210, 200)
    b = timg_b200.Batch(n_frames=n, src_w=iw, src_h=ih, src_fmt=0, out_w=ow, out_h=oh, has_bg=1, bg=bg, pattern=pat,
                        pattern_w=4, pattern_h=6, flags=0, x_indent_cells=0, animation=0)
    outs = ctx.graphics_batch(frames, b, timg_b200.KITTY, False, [1, 2])
    for f in range(n):
        got = png_pixels(base64.b64decode(kitty_payload(outs[f])))[0]
        want = oracle.compose_bg(oracle.stb_resize(frames[f], ow, oh), bg, pat, 4, 6)
        assert got.shape == want.shape and (got == want).all(), f"frame {f}: {first_diff(got, want)}"
