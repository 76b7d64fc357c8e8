"""Every launch shape of the sixel chain (palette variant, dither CTAs / warps / rounds / hand-overs, emitter and column
tiles) against the CPU statement of the same semantics (oracle mode 1): colour count, palette, the whole index plane, and the
stream decoding to palette[index].  The cases and the classes they stand for are in sixel_shape_cases.py; every case first asks
the library, for the device it runs on, whether it really is in its class."""
import ctypes as C
import re

import numpy as np
import pytest

import oracle
import sixel_shape_cases as sc
import timg_b200

pytestmark = pytest.mark.gpu

FRAMING = rb'\x1bPq"1;1;\d+;\d+(#\d+;2;\d+;\d+;\d+)+[#!$\-0-9?-~]+\x1b\\'


def pct(pal):
    return ((pal.astype(int) * 100 + 127) // 255) * 255 // 100


def sm_count():
    import torch
    if torch.cuda.is_available():
        return torch.cuda.get_device_properties(0).multi_processor_count
    return 132                                      # the CPU kernel simulator's device


def setup(monkeypatch, group, name):
    case = sc.by_name(sm_count(), group)[name]
    sc.apply_env(monkeypatch, case)
    sc.check_class(case, sm_count())
    return case


def first_diff(a, b):
    bad = np.argwhere(a != b)
    return f"{len(bad)} differ, first at (y, x) = {tuple(bad[0][:2])}: {a[tuple(bad[0])]} != {b[tuple(bad[0])]}" if len(bad) else "equal"


def check_stream(case, fb, data, det):
    """The stream's framing, its size against the bound, and that it decodes to the oracle's palette[index]."""
    h, w = fb.shape[:2]
    assert len(data) <= timg_b200.lib().b200timg_sixel_bound(w, h), "b200timg_sixel_bound"
    assert data.startswith(b'\x1bPq"1;1;%d;%d#0;2;' % (w, h)) and data.endswith(b"\x1b\\")
    assert re.fullmatch(FRAMING, data)
    img, used = oracle.sixel_decode(data)
    assert img.shape == (h, w, 3)
    want = pct(det["palette"])[det["index"]]
    assert (img == want).all(), f"{case.name}: decoded stream vs oracle palette[index]: {first_diff(img, want)}"


def check_frame(ctx, case, fb):
    """One frame through b200timg_sixel_encode against the oracle: colour count, palette, index plane, stream."""
    h, w = fb.shape[:2]
    data = ctx.sixel_encode(fb)
    pal, orig, idx = ctx.sixel_debug(w, h)
    _, det = oracle.sixel_encode(fb, True, mode=1)
    assert orig == det["origcolors"], f"{case.name}: occupied cells {orig} != {det['origcolors']}"
    if case.diffuse is not None:
        assert (orig > 256) == case.diffuse, f"{case.name}: {orig} cells, the case is there for diffuse = {case.diffuse}"
    if case.kind == "allcells":
        assert orig == 32768
    assert pal.shape == det["palette"].shape and (pal == det["palette"]).all(), f"{case.name}: palette: {first_diff(pal, det['palette'])}"
    assert (idx == det["index"]).all(), f"{case.name}: index plane: {first_diff(idx, det['index'])}"
    check_stream(case, fb, data, det)
    return data


@pytest.mark.parametrize("name", sc.names("palette"))
def test_palette_classes(ctx, monkeypatch, name):
    case = setup(monkeypatch, "palette", name)
    check_frame(ctx, case, sc.frame(case))


@pytest.mark.parametrize("name", sc.names("dither"))
def test_dither_classes(ctx, monkeypatch, name):
    case = setup(monkeypatch, "dither", name)
    fb = sc.frame(case)
    data = check_frame(ctx, case, fb)
    if case.env:                                    # the knobs change the launch, never the bytes
        sc.apply_env(monkeypatch, case._replace(env={}))
        assert ctx.sixel_encode(fb) == data


def _sixel_dev(ctx, frames, out_cap=None, fill=0, guard=0):
    """b200timg_sixel_dev on [n, h, w, 4] frames: (output bytes incl. guard, offsets[n + 1])."""
    import torch
    n, h, w = frames.shape[:3]
    d = timg_b200._device_tensor(torch, frames)
    cap = n * timg_b200.lib().b200timg_sixel_bound(w, h) if out_cap is None else out_cap
    out = torch.full((cap + guard,), fill, dtype=torch.uint8, device=d.device)
    offs = torch.zeros(n + 1, dtype=torch.int64, device=d.device)
    rc = timg_b200.lib().b200timg_sixel_dev(ctx.h, d.data_ptr(), w, h, n, out.data_ptr(), cap, offs.data_ptr())
    assert rc == 0, timg_b200.lib().b200timg_last_error(ctx.h)
    timg_b200.device_sync(torch)
    return out.cpu().numpy(), offs.cpu().numpy()


def _batch(n, w, h):
    return timg_b200.Batch(n_frames=n, src_w=w, src_h=h, src_fmt=0, out_w=w, out_h=h, has_bg=1, bg=timg_b200.rgba_u32(0, 0, 0),
                           pattern=0, pattern_w=0, pattern_h=0, flags=0, x_indent_cells=0, animation=0)


def _sixel_batch_dev(ctx, frames, out_cap=None, fill=0, guard=0):
    """b200timg_sixel_batch_dev at scale 1 (opaque frames of a multiple of 6 rows pass through the scaler unchanged)."""
    import torch
    n, h, w = frames.shape[:3]
    b = _batch(n, w, h)
    d = timg_b200._device_tensor(torch, frames)
    cap = n * timg_b200.lib().b200timg_sixel_bound(w, h) if out_cap is None else out_cap
    out = torch.full((cap + guard,), fill, dtype=torch.uint8, device=d.device)
    offs = torch.zeros(n + 1, dtype=torch.int64, device=d.device)
    rc = timg_b200.lib().b200timg_sixel_batch_dev(ctx.h, C.byref(b), d.data_ptr(), out.data_ptr(), cap, offs.data_ptr())
    assert rc == 0, timg_b200.lib().b200timg_last_error(ctx.h)
    timg_b200.device_sync(torch)
    return out.cpu().numpy(), offs.cpu().numpy()


def _check_batch(ctx, monkeypatch, case, run, checked):
    """Frames `checked` of the batch: each against its own oracle run and against the single-frame entry point."""
    frames = np.stack([sc.frame(case, i) for i in range(case.n_total)])
    out, offs = run(ctx, frames)
    assert offs[0] == 0 and (np.diff(offs) > 0).all()
    sc.apply_env(monkeypatch, case._replace(env={}))
    for f in checked:
        data = out[int(offs[f]):int(offs[f + 1])].tobytes()
        _, det = oracle.sixel_encode(frames[f], True, mode=1)
        assert (det["origcolors"] > 256) == case.diffuse
        check_stream(case._replace(name=f"{case.name} frame {f}"), frames[f], data, det)
        assert data == ctx.sixel_encode(frames[f]), f"{case.name}: frame {f} differs from its single-frame encode"


@pytest.mark.parametrize("name", ["half-sm-split2", "sm-minus-1", "sm-plus-5"])
def test_batches_of_distinct_frames(ctx, monkeypatch, name):
    case = setup(monkeypatch, "batch", name)
    _check_batch(ctx, monkeypatch, case, _sixel_dev, range(case.n))


def test_batch_with_natural_rounds(ctx, monkeypatch):
    """26 bands on one CTA of 13 warps: the shape every frame of a full batch of tall frames takes."""
    case = setup(monkeypatch, "batch", "natural-rounds2")
    _check_batch(ctx, monkeypatch, case, _sixel_dev, (0, case.n // 2, case.n - 1))


@pytest.mark.parametrize("name", ["parts2", "parts4"])
def test_batch_slices(ctx, monkeypatch, name):
    case = setup(monkeypatch, "batch", name)
    _check_batch(ctx, monkeypatch, case, _sixel_batch_dev, range(case.n_total))


@pytest.mark.parametrize("name", sc.names("wide"))
def test_wide_and_tall_frames(ctx, monkeypatch, name):
    case = setup(monkeypatch, "wide", name)
    fb = sc.frame(case)
    if case.w > 20000:      # the CPU encoder takes minutes at this width: few colours, so the picture is known without it
        data = ctx.sixel_encode(fb)
        assert len(data) <= timg_b200.lib().b200timg_sixel_bound(case.w, case.h) and re.fullmatch(FRAMING, data)
        img, used = oracle.sixel_decode(data)
        assert used == 5 and (img == pct(fb[..., :3] & 0xF8)).all()
        return
    data = check_frame(ctx, case, fb)
    if case.kind == "solid" and case.expect["emit_tiles"] == 1:
        assert b"!%d~" % case.w in data             # one run per band


@pytest.mark.parametrize("w,h,limit", [(100000, 6, b"99999"), (4, 65538, b"65536")])
def test_frames_beyond_the_limits_are_rejected_before_any_launch(ctx, w, h, limit):
    fb = np.zeros((h, w, 4), np.uint8)
    before = ctx.launches
    buf, n = C.create_string_buffer(64), C.c_size_t()
    rc = timg_b200.lib().b200timg_sixel_encode(ctx.h, fb.ctypes.data_as(timg_b200.u8p), w, h, buf, 64, C.byref(n))
    assert rc == timg_b200.EINVAL
    assert limit in timg_b200.lib().b200timg_last_error(ctx.h)
    assert ctx.launches == before


@pytest.mark.parametrize("name", sc.names("capacity"))
@pytest.mark.parametrize("entry", ["sixel_dev", "sixel_batch_dev"])
def test_capacity_contract_device(ctx, monkeypatch, name, entry):
    """out_cap ending inside frame 2 of 4: offsets complete and exact, frames 0 and 1 intact, nothing written from frame 2 on.
    The single-pass emitter of frames wider than 4095 px places every band x tile on its own: of frame 2 it may write the
    pieces that end before out_cap (with the bytes an uncapped run puts there), and nothing at or beyond out_cap."""
    case = setup(monkeypatch, "capacity", name)
    single_pass = case.expect["emit_mode"] == 2
    run = _sixel_dev if entry == "sixel_dev" else _sixel_batch_dev
    frames = np.stack([sc.frame(case, i) for i in range(case.n)])
    full, offs = run(ctx, frames)
    k = 2
    cap = int(offs[k]) + (int(offs[k + 1]) - int(offs[k])) // 2
    out, offs2 = run(ctx, frames, out_cap=cap, fill=0xA5, guard=4096)
    assert (offs2 == offs).all()
    assert (out[:int(offs[k])] == full[:int(offs[k])]).all()
    assert (out[cap:] == 0xA5).all()
    mid, ref = out[int(offs[k]):cap], full[int(offs[k]):cap]
    if single_pass:
        assert ((mid == 0xA5) | (mid == ref)).all() and (mid[-64:] == 0xA5).any()
    else:
        assert (mid == 0xA5).all()                                   # frame 2 is not written at all
    for f in range(k):
        assert out[int(offs[f]):int(offs[f + 1])].tobytes() == ctx.sixel_encode(frames[f])


@pytest.mark.parametrize("name", sc.names("capacity"))
def test_capacity_contract_host(ctx, monkeypatch, name):
    """b200timg_sixel_batch: ENOSPC, offsets complete, nothing at or past out_cap."""
    case = setup(monkeypatch, "capacity", name)
    frames = np.stack([sc.frame(case, i) for i in range(case.n)])
    want = ctx.sixel_batch(frames, _batch(case.n, case.w, case.h))
    offs = np.cumsum([0] + [len(x) for x in want]).astype(np.uint64)
    cap = int(offs[2]) + len(want[2]) // 2
    out = np.full(cap + 4096, 0xA5, np.uint8)
    hoffs = np.zeros(case.n + 1, np.uint64)
    b = _batch(case.n, case.w, case.h)
    rc = timg_b200.lib().b200timg_sixel_batch(ctx.h, C.byref(b), frames.ctypes.data, out.ctypes.data, cap, hoffs.ctypes.data)
    assert rc == timg_b200.ENOSPC
    assert (hoffs == offs).all()
    assert (out[cap:] == 0xA5).all()
