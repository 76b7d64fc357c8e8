"""Sixel mixed batches (b200timg_sixel_mixed): a `-p sixel` grid page of differently sized images scaled, composed,
padded, quantised, dithered and sixel-encoded in one call, against the one-frame uniform batch and the oracle,
independent of the batch's composition, the capacity contract, the rejected arguments and the launch count."""
import ctypes as C

import numpy as np
import pytest

import oracle
import timg_b200
from timg_b200 import synth

pytestmark = pytest.mark.gpu

BG = timg_b200.rgba_u32(10, 20, 30)
PATTERN = timg_b200.rgba_u32(200, 190, 180)
COMPOSE = dict(has_bg=True, bg=BG, pattern=PATTERN, pattern_w=8, pattern_h=4)


def pct(pal):
    return ((pal.astype(int) * 100 + 127) // 255) * 255 // 100


def _few_colours(w, h):
    """Four flat colours in blocks: <= 256 sampled colours, so the map kernel runs instead of the ditherer."""
    im = np.zeros((h, w, 4), np.uint8)
    cols = [(250, 10, 10), (10, 250, 10), (10, 10, 250), (240, 240, 20)]
    for y in range(h):
        for x in range(w):
            im[y, x, :3] = cols[(x // 8 + y // 5) % 4]
    im[..., 3] = 255
    return im


def _page():
    """(images, outs): about 20 images of the geometries a sixel grid page meets.  Padded frames with 25600 < w * h <
    36766 take the palette kernel's global-table variant, every other frame the shared-memory one."""
    spec = [
        (synth.frame_np(1, 1280, 720, "photo"), (337, 190)),         # height 190: a 2-row pad strip
        (synth.frame_np(2, 640, 480, "noise"), (161, 121)),          # odd width and height
        (synth.frame_np(3, 640, 480, "alpha"), (160, 119)),          # transparency, 5-row pad strip
        (_few_colours(64, 40), (64, 40)),                            # <= 256 colours: map, no dither
        (synth.frame_np(5, 400, 300, "photo"), (180, 178)),          # 180 x 180 padded: global median-cut tables
        (synth.frame_np(6, 400, 300, "noisea"), (200, 161)),         # 200 x 162: global tables, random alpha
        (synth.frame_np(7, 50, 40, "photo"), (1, 1)),
        (synth.frame_np(8, 50, 400, "photo"), (1, 100)),
        (synth.frame_np(9, 400, 50, "noise"), (100, 1)),
        (synth.frame_np(10, 300, 1200, "photo"), (60, 400)),         # 13 bands of 32 rows
        (synth.frame_np(11, 8190, 12, "photo"), (4095, 6)),          # the widest frame the mixed path takes
        (synth.frame_np(12, 120, 80, "photo"), (240, 160)),          # upscale
        (synth.frame_np(13, 96, 64, "noise"), (96, 64)),             # identity
        (synth.frame_np(14, 300, 200, "alpha"), (100, 67)),
        (synth.frame_np(15, 1920, 1080, "photo"), (320, 180)),
        (synth.frame_np(16, 33, 17, "noise"), (66, 34)),
        (synth.frame_np(17, 480, 640, "photo"), (60, 80)),
        (synth.frame_np(18, 256, 256, "noisea"), (128, 128)),
        (synth.frame_np(19, 800, 600, "photo"), (400, 300)),         # 400 x 300: shared-memory tables again
        (synth.frame_np(1, 1280, 720, "photo"), (337, 190)),         # a repeated geometry
    ]
    return [s[0] for s in spec], [s[1] for s in spec]


PAGE = None


def page():
    global PAGE
    if PAGE is None:
        PAGE = _page()
    return PAGE


def _hp(h):
    return (h + 5) // 6 * 6


def _uniform(ctx, frames, ow, oh):
    """b200timg_sixel_batch_dev with flags = 0 on frames of one geometry ([n, h, w, 4]): each frame's bytes."""
    import torch
    frames = np.ascontiguousarray(frames)
    n, ih, iw = frames.shape[:3]
    ub = timg_b200.Batch(n_frames=n, src_w=iw, src_h=ih, src_fmt=0, out_w=ow, out_h=oh, has_bg=1, bg=BG, pattern=PATTERN,
                         pattern_w=8, pattern_h=4, flags=0, x_indent_cells=0, animation=0)
    d_src = timg_b200._device_tensor(torch, frames)
    cap = timg_b200.lib().b200timg_sixel_bound(ow, _hp(oh)) * n
    d_out = torch.zeros(cap, dtype=torch.uint8, device=d_src.device)
    d_offs = torch.zeros(n + 1, dtype=torch.int64, device=d_src.device)
    timg_b200.device_sync(torch)
    ctx._chk(timg_b200.lib().b200timg_sixel_batch_dev(ctx.h, C.byref(ub), d_src.data_ptr(), d_out.data_ptr(), cap,
                                                      d_offs.data_ptr()))
    timg_b200.device_sync(torch)
    o, data = d_offs.cpu().numpy(), d_out.cpu().numpy()
    return [data[o[f]:o[f + 1]].tobytes() for f in range(n)]


def _oracle_fb(img, ow, oh):
    """What SixelCanvas::Send encodes: scale, compose, pad to a multiple of 6 rows, compose the pad strip only."""
    fb = oracle.compose_bg(oracle.stb_resize(img, ow, oh), BG, PATTERN, 8, 4)
    padded = np.zeros((_hp(oh), ow, 4), np.uint8)
    padded[:oh] = fb
    return oracle.compose_bg(padded, BG, PATTERN, 8, 4, start_row=oh)


def _dev(ctx, imgs, outs, flags=0, **kw):
    import torch
    flat, offs = timg_b200.pack_mixed(imgs)
    b, keep = timg_b200.mixed_batch([im.shape for im in imgs], outs, offs, None, flags, **COMPOSE)
    d_src = timg_b200._device_tensor(torch, flat)
    d_out, d_offs = ctx.sixel_mixed_dev(d_src, b, **kw)
    timg_b200.device_sync(torch)
    o, data = d_offs.cpu().numpy(), d_out.cpu().numpy()
    return [data[o[f]:o[f + 1]].tobytes() for f in range(len(imgs))]


def test_sixel_mixed_page_matches_uniform_batch_and_oracle(ctx):
    imgs, outs = page()
    assert sum(25600 < w * _hp(h) < 36766 for w, h in outs) >= 2          # both palette variants run
    got = ctx.sixel_mixed(imgs, outs, **COMPOSE)
    # b200timg_sixel_debug after a mixed call: frame 0's palette, counts and index plane
    w0, h0 = outs[0][0], _hp(outs[0][1])
    pal0, orig0, idx0 = ctx.sixel_debug(w0, h0)
    _, det0 = oracle.sixel_encode(_oracle_fb(imgs[0], *outs[0]), True, mode=1)
    assert orig0 == det0["origcolors"] and (pal0 == det0["palette"]).all() and (idx0 == det0["index"]).all()
    for f, (img, (ow, oh)) in enumerate(zip(imgs, outs)):
        assert got[f] == _uniform(ctx, img[None], ow, oh)[0], (f, ow, oh)
        fb = _oracle_fb(img, ow, oh)
        _, det = oracle.sixel_encode(fb, True, mode=1)
        dec, _ = oracle.sixel_decode(got[f])
        assert dec.shape == (_hp(oh), ow, 3), f
        assert (dec == pct(det["palette"])[det["index"]]).all(), (f, ow, oh)
        assert got[f].startswith(b'\x1bPq"1;1;%d;%d#0;2;' % (ow, _hp(oh))) and got[f].endswith(b"\x1b\\"), f
    assert got[0] == got[-1]
    few = oracle.sixel_encode(_oracle_fb(imgs[3], *outs[3]), True, mode=1)[1]
    assert few["origcolors"] <= 256


def test_sixel_mixed_ignores_block_fields(ctx):
    """x_indent_cells, QUARTER / UPPER / COLOR8 (odd widths too) and FAST_SCALE leave the bytes alone."""
    imgs, outs = page()
    keep = [1, 2, 3, 13]
    imgs, outs = [imgs[f] for f in keep], [outs[f] for f in keep]
    want = _dev(ctx, imgs, outs)
    flat, offs = timg_b200.pack_mixed(imgs)
    flags = timg_b200.QUARTER | timg_b200.UPPER | timg_b200.COLOR8 | timg_b200.FAST_SCALE
    b, _ = timg_b200.mixed_batch([im.shape for im in imgs], outs, offs, [3, 0, 7, 250], flags, **COMPOSE)
    cap = ctx.sixel_mixed_bound(outs)
    out = np.zeros(cap, np.uint8)
    o = np.zeros(len(imgs) + 1, np.uint64)
    ctx._chk(timg_b200.lib().b200timg_sixel_mixed(ctx.h, C.byref(b), flat.ctypes.data, out.ctypes.data, cap, o.ctypes.data))
    assert [out[int(o[i]):int(o[i + 1])].tobytes() for i in range(len(imgs))] == want


def test_sixel_mixed_independent_of_order_variant_grouping_and_split(ctx, monkeypatch):
    imgs, outs = page()
    whole = ctx.sixel_mixed(imgs, outs, **COMPOSE)
    perm = np.random.default_rng(7).permutation(len(imgs))
    got = ctx.sixel_mixed([imgs[p] for p in perm], [outs[p] for p in perm], **COMPOSE)
    assert got == [whole[p] for p in perm]
    assert _dev(ctx, imgs, outs) == whole
    monkeypatch.setenv("B200TIMG_MIXED_GROUP_BYTES", "1")                 # every frame its own scaler group
    assert _dev(ctx, imgs, outs) == whole
    assert ctx.sixel_mixed(imgs, outs, **COMPOSE) == whole
    monkeypatch.delenv("B200TIMG_MIXED_GROUP_BYTES")
    # the tall frame alone (its bands split over several dither CTAs) and among more frames than the GPU has SMs
    # (one CTA per frame)
    import torch
    props = torch.cuda.get_device_properties(0) if torch.cuda.is_available() else None
    n_sm = props.multi_processor_count if props is not None else 132
    f0 = 9
    assert ctx.sixel_mixed([imgs[f0]], [outs[f0]], **COMPOSE) == [whole[f0]]
    small = [synth.frame_np(40 + k, 24 + k % 7, 18 + k % 5, "photo") for k in range(n_sm + 8)]
    small_outs = [(8 + k % 9, 5 + k % 4) for k in range(n_sm + 8)]
    mid = len(small) // 2
    res = ctx.sixel_mixed(small[:mid] + [imgs[f0]] + small[mid:], small_outs[:mid] + [outs[f0]] + small_outs[mid:], **COMPOSE)
    assert res[mid] == whole[f0]
    for k in (0, mid + 1, len(res) - 1):
        j = k if k < mid else k - 1
        assert res[k] == _uniform(ctx, small[j][None], *small_outs[j])[0], k


def test_sixel_mixed_uniform_geometry_equals_uniform_batch(ctx):
    """A mixed batch whose frames share C4's output geometry equals b200timg_sixel_batch_dev byte for byte."""
    n, iw, ih, ow, oh = 4, 1280, 720, 675, 380
    frames = np.stack([synth.frame_np(60 + i, iw, ih, "alpha" if i % 2 else "photo") for i in range(n)])
    assert ctx.sixel_mixed(list(frames), [(ow, oh)] * n, **COMPOSE) == _uniform(ctx, frames, ow, oh)


def test_sixel_mixed_capacity_contract(ctx):
    import torch
    imgs, outs = page()
    keep = [1, 2, 3, 6, 12, 13, 16]
    imgs, outs = [imgs[f] for f in keep], [outs[f] for f in keep]
    want = ctx.sixel_mixed(imgs, outs, **COMPOSE)
    sizes = np.array([len(w) for w in want], np.int64)
    ends = np.cumsum(sizes)
    total = int(ends[-1])
    # device variant: a cap that ends inside frame 3
    cap = int(ends[2]) + int(sizes[3]) // 2
    flat, offs = timg_b200.pack_mixed(imgs)
    b, _ = timg_b200.mixed_batch([im.shape for im in imgs], outs, offs, None, 0, **COMPOSE)
    d_src = timg_b200._device_tensor(torch, flat)
    d_out = torch.full((total + 64,), 0xA5, dtype=torch.uint8, device=d_src.device)
    timg_b200.device_sync(torch)
    _, d_offs = ctx.sixel_mixed_dev(d_src, b, d_out=d_out, out_cap=cap)
    timg_b200.device_sync(torch)
    o, data = d_offs.cpu().numpy(), d_out.cpu().numpy()
    assert list(o) == [0] + list(ends)
    assert b"".join(want[:3]) == data[:int(ends[2])].tobytes()
    assert (data[int(ends[2]):] == 0xA5).all()                  # frames past the cap are not written
    # host variant: ENOSPC, offsets complete, nothing written past out_cap (here: nothing at all)
    out = np.full(total + 64, 0x5A, np.uint8)
    offsets = np.zeros(len(imgs) + 1, np.uint64)
    rc = timg_b200.lib().b200timg_sixel_mixed(ctx.h, C.byref(b), flat.ctypes.data, out.ctypes.data, total - 1,
                                               offsets.ctypes.data)
    assert rc == timg_b200.ENOSPC
    assert list(offsets) == [0] + list(ends)
    assert (out == 0x5A).all()
    rc = timg_b200.lib().b200timg_sixel_mixed(ctx.h, C.byref(b), flat.ctypes.data, out.ctypes.data, total,
                                               offsets.ctypes.data)
    assert rc == timg_b200.OK and out[:total].tobytes() == b"".join(want) and (out[total:] == 0x5A).all()


def _call(ctx, frame_list, null_frames=False, **kw):
    d = dict(n_frames=len(frame_list), src_fmt=0, flags=0, has_bg=1, bg=BG, pattern=0, pattern_w=0, pattern_h=0)
    d.update(kw)
    arr = (timg_b200.Frame * len(frame_list))(*frame_list)
    b = timg_b200.MixedBatch(frames=None if null_frames else arr, **d)
    src = np.zeros(1 << 16, np.uint8)
    out = np.zeros(1 << 16, np.uint8)
    offs = np.zeros(len(frame_list) + 2, np.uint64)
    rc = timg_b200.lib().b200timg_sixel_mixed(ctx.h, C.byref(b), src.ctypes.data, out.ctypes.data, out.size, offs.ctypes.data)
    return rc, timg_b200.lib().b200timg_last_error(ctx.h).decode()


@pytest.mark.parametrize("case,kw,needle", [
    ("no frames", dict(n_frames=0), "n_frames > 0"),
    ("null frames", dict(null_frames=True), "frames array"),
    ("zero src", dict(fr=(0, 0, 8, 8, 4, 0)), "non-positive size"),
    ("negative out", dict(fr=(0, 8, 8, 4, -1, 0)), "non-positive size"),
    ("unaligned offset", dict(fr=(2, 8, 8, 4, 4, 0)), "not a multiple of 4"),
    ("yuv", dict(src_fmt=timg_b200.FMT_I420), "source format"),
    ("bilinear", dict(flags=timg_b200.BILINEAR_SCALE), "BILINEAR"),
    ("negative indent", dict(fr=(0, 8, 8, 4, 4, -1)), "negative indent"),
    ("too wide", dict(fr=(0, 8, 8, 4096, 4, 0)), "frame 1: width 4096"),
    ("too tall", dict(fr=(0, 8, 8, 4, 65533, 0)), "frame 1: height 65533"),
])
def test_sixel_mixed_rejected_arguments(ctx, case, kw, needle):
    kw = dict(kw)
    good = timg_b200.Frame(0, 8, 8, 4, 4, 0)
    frames = [good, good]
    if "fr" in kw:
        frames[1] = timg_b200.Frame(*kw.pop("fr"))
    rc, msg = _call(ctx, frames, **kw)
    assert rc == timg_b200.EINVAL, case
    assert needle in msg, (case, msg)


def test_sixel_mixed_launches_do_not_grow_with_geometries(ctx):
    import torch
    n = 64
    distinct = [synth.frame_np(500 + k, 64 + 5 * k, 48 + 3 * k, "photo") for k in range(n)]
    distinct_outs = [(16 + 2 * (k % 20), 9 + k % 13) for k in range(n)]
    same = [synth.frame_np(600 + k, 200, 120, "photo") for k in range(n)]
    counts = []
    for imgs, outs in ((distinct, distinct_outs), (same, [(40, 24)] * n)):
        assert len(set(zip([im.shape for im in imgs], outs))) in (1, n)
        flat, offs = timg_b200.pack_mixed(imgs)
        b, keep = timg_b200.mixed_batch([im.shape for im in imgs], outs, offs)
        d_src = timg_b200._device_tensor(torch, flat)
        before = ctx.launches
        ctx.sixel_mixed_dev(d_src, b)
        timg_b200.device_sync(torch)
        counts.append(ctx.launches - before)
    assert counts[0] == counts[1], counts
