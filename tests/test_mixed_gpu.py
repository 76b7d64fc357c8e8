"""Mixed batches (b200timg_mixed_batch): a grid page of differently sized images scaled, composed and block-encoded in
one call, against the single-frame path and the oracle, independent of the batch's composition, the capacity contract,
the rejected arguments and the launch count."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle
import timg_b200
from timg_b200 import synth

pytestmark = pytest.mark.gpu

BG = timg_b200.rgba_u32(10, 20, 30)
PATTERN = timg_b200.rgba_u32(200, 190, 180)
COMPOSE = dict(has_bg=True, bg=BG, pattern=PATTERN, pattern_w=8, pattern_h=4)


def _half_transparent(seed, w, h):
    """Photo colours, alpha 0 on the left half and a column band: the scaler's un-weighted (plain) passes run."""
    im = synth.frame_np(seed, w, h, "photo")
    im[:, : w // 2, 3] = 0
    im[:, w // 2 + 7: w // 2 + 11, 3] = 0
    return im


def _fit(iw, ih, w, h, **kw):
    return timg_b200.calc_fit(iw, ih, w, h, 1, 2, **kw)[1:]


def _page():
    """(images, outs, indents): about 20 images of the geometries a grid page meets."""
    spec = [
        (synth.frame_np(1, 3840, 2160, "photo"), (336, 190)),        # 4K, > 8 taps per axis
        (synth.frame_np(2, 3840, 2160, "noise"), (337, 190)),        # odd width: half blocks only
        (synth.frame_np(3, 800, 600, "photo"), (600, 450)),          # mild downscale, <= 8 taps
        (synth.frame_np(4, 640, 480, "alpha"), (68, 50)),            # C1-like, transparency
        (synth.frame_np(5, 120, 80, "photo"), _fit(120, 80, 240, 200, upscale=True)),   # BOX upscale
        (synth.frame_np(6, 64, 48, "alpha"), (64, 48)),              # identity
        (synth.frame_np(7, 96, 64, "noise"), (96, 64)),              # identity
        (synth.frame_np(8, 50, 40, "photo"), (1, 1)),
        (synth.frame_np(9, 50, 40, "alpha"), (2, 2)),
        (synth.frame_np(10, 300, 200, "photo"), (150, 101)),         # odd height
        (synth.frame_np(11, 300, 200, "alpha"), (100, 67)),          # odd height, transparency
        (synth.frame_np(12, 480, 640, "photo"), (60, 80)),           # portrait
        (synth.frame_np(13, 1080, 1920, "alpha"), (90, 160)),        # tall portrait, long filters
        (synth.frame_np(14, 256, 256, "noisea"), (128, 128)),        # random alpha
        (synth.frame_np(15, 200, 100, "alpha"), (100, 50)),
        (synth.frame_np(16, 1920, 1080, "photo"), (320, 90)),        # C3 geometry
        (synth.frame_np(17, 33, 17, "noise"), (66, 34)),             # upscale of an odd source
        (synth.frame_np(18, 1000, 10, "photo"), (100, 1)),
        (synth.frame_np(19, 10, 1000, "photo"), (2, 100)),
        (_half_transparent(20, 160, 96), (80, 48)),                  # fully transparent regions
        (synth.frame_np(1, 3840, 2160, "photo"), (336, 190)),        # a repeated geometry shares its plan
    ]
    assert spec[4][1] == (240, 160)
    indents = [(0, 1, 250)[i % 3] for i in range(len(spec))]
    return [s[0] for s in spec], [s[1] for s in spec], indents


PAGE = None


def page():
    global PAGE
    if PAGE is None:
        PAGE = _page()
    return PAGE


def _quarter_ok(outs):
    return [f for f, (ow, _) in enumerate(outs) if ow % 2 == 0]


def _select(page_, keep):
    imgs, outs, ind = page_
    return [imgs[f] for f in keep], [outs[f] for f in keep], [ind[f] for f in keep]


def _single(ctx, img, ow, oh, flags, indent, fmt=timg_b200.FMT_RGBA):
    fb = ctx.compose_bg(ctx.scale(img, ow, oh, fmt), BG, PATTERN, 8, 4)
    return ctx.blocks_encode(fb, flags=flags, x_indent_cells=indent)


def _oracle(img, ow, oh, flags, indent, fmt=timg_b200.FMT_RGBA):
    fb = oracle.compose_bg(oracle.stb_resize(img, ow, oh, fmt), BG, PATTERN, 8, 4)
    quarter = bool(flags & timg_b200.QUARTER)
    cv = oracle.BlockCanvas(quarter, bool(flags & timg_b200.UPPER), bool(flags & timg_b200.COLOR8))
    return cv.send(fb, x=2 * indent if quarter else indent)


@pytest.mark.parametrize("flags", range(8))
def test_mixed_page_matches_single_frames_and_oracle(ctx, flags):
    imgs, outs, ind = page()
    if flags & timg_b200.QUARTER:
        imgs, outs, ind = _select(page(), _quarter_ok(outs))
    got = ctx.blocks_mixed(imgs, outs, ind, flags, **COMPOSE)
    for f, (img, (ow, oh), x) in enumerate(zip(imgs, outs, ind)):
        assert got[f] == _single(ctx, img, ow, oh, flags, x), (f, ow, oh)
        assert got[f] == _oracle(img, ow, oh, flags, x), (f, ow, oh)


def test_mixed_page_rgb32_sources(ctx):
    imgs, outs, ind = _select(page(), [2, 3, 5, 9, 10, 13, 16])
    bgra = [np.ascontiguousarray(im[..., [2, 1, 0, 3]]) for im in imgs]
    got = ctx.blocks_mixed(bgra, outs, ind, timg_b200.UPPER, src_fmt=timg_b200.FMT_RGB32, **COMPOSE)
    for f, (img, (ow, oh), x) in enumerate(zip(bgra, outs, ind)):
        assert got[f] == _single(ctx, img, ow, oh, timg_b200.UPPER, x, timg_b200.FMT_RGB32), f
        assert got[f] == _oracle(img, ow, oh, timg_b200.UPPER, x, timg_b200.FMT_RGB32), f


def test_scale_mixed_equals_scale_then_compose(ctx):
    imgs, outs, _ = page()
    got = ctx.scale_mixed(imgs, outs, **COMPOSE)
    for f, (img, (ow, oh)) in enumerate(zip(imgs, outs)):
        want = ctx.compose_bg(ctx.scale(img, ow, oh), BG, PATTERN, 8, 4)
        assert (got[f] == want).all(), f
        assert (got[f] == oracle.compose_bg(oracle.stb_resize(img, ow, oh), BG, PATTERN, 8, 4)).all(), f
        if oracle.have_ref():
            assert (got[f] == oracle.ref_compose_bg(oracle.ref_scale(img, ow, oh), BG, PATTERN, 8, 4)).all(), f
    plain = ctx.scale_mixed(imgs, outs, has_bg=False)       # without a background the scaler's own pixels come out
    for f, (img, (ow, oh)) in enumerate(zip(imgs, outs)):
        assert (plain[f] == ctx.scale(img, ow, oh)).all(), f


def test_mixed_independent_of_order_size_and_variant(ctx, monkeypatch):
    import torch
    imgs, outs, ind = page()
    flags = timg_b200.COLOR8
    whole = ctx.blocks_mixed(imgs, outs, ind, flags, **COMPOSE)
    perm = np.random.default_rng(5).permutation(len(imgs))
    got = ctx.blocks_mixed([imgs[p] for p in perm], [outs[p] for p in perm], [ind[p] for p in perm], flags, **COMPOSE)
    assert got == [whole[p] for p in perm]
    # one image alone, among 7 and among 64
    f0 = 3
    alone = ctx.blocks_mixed([imgs[f0]], [outs[f0]], [ind[f0]], flags, **COMPOSE)
    assert alone == [whole[f0]]
    small = [synth.frame_np(40 + k, 40 + 3 * k, 30 + 2 * k, "photo") for k in range(63)]
    small_outs = [(10 + k, 7 + k % 5) for k in range(63)]
    for n_others in (6, 63):
        im = small[:n_others // 2] + [imgs[f0]] + small[n_others // 2:n_others]
        oo = small_outs[:n_others // 2] + [outs[f0]] + small_outs[n_others // 2:n_others]
        xi = [0] * (n_others // 2) + [ind[f0]] + [0] * (n_others - n_others // 2)
        res = ctx.blocks_mixed(im, oo, xi, flags, **COMPOSE)
        assert res[n_others // 2] == whole[f0], n_others
    # device variant, in one group and with every frame its own group
    flat, offs = timg_b200.pack_mixed(imgs)
    b, keep = timg_b200.mixed_batch([im.shape for im in imgs], outs, offs, ind, flags, **COMPOSE)
    d_src = timg_b200._device_tensor(torch, flat)
    for group_bytes in (None, "1", str(40 << 20)):
        if group_bytes:
            monkeypatch.setenv("B200TIMG_MIXED_GROUP_BYTES", group_bytes)
        d_out, d_offs = ctx.blocks_mixed_dev(d_src, b)
        timg_b200.device_sync(torch)
        o, data = d_offs.cpu().numpy(), d_out.cpu().numpy()
        assert [data[o[f]:o[f + 1]].tobytes() for f in range(len(imgs))] == whole, group_bytes
        assert ctx.blocks_mixed(imgs, outs, ind, flags, **COMPOSE) == whole, group_bytes


def test_mixed_uniform_geometry_equals_uniform_batch(ctx):
    """A mixed batch whose frames share C3's geometry equals b200timg_blocks_batch_dev byte for byte."""
    import torch
    n, iw, ih, ow, oh = 4, 1920, 1080, 320, 90
    frames = np.stack([synth.frame_np(60 + i, iw, ih, "alpha" if i % 2 else "photo") for i in range(n)])
    flags, indent = timg_b200.QUARTER, 3
    ub = timg_b200.Batch(n_frames=n, src_w=iw, src_h=ih, src_fmt=0, out_w=ow, out_h=oh, has_bg=1, bg=BG, pattern=PATTERN,
                         pattern_w=8, pattern_h=4, flags=flags, x_indent_cells=indent, animation=0)
    d_src = timg_b200._device_tensor(torch, frames)
    cap = timg_b200.lib().b200timg_blocks_bound(ow, oh) * n
    d_out = torch.zeros(cap, dtype=torch.uint8, device=d_src.device)
    d_offs = torch.zeros(n + 1, dtype=torch.int64, device=d_src.device)
    timg_b200.device_sync(torch)                                # torch's fills run on torch's stream
    ctx._chk(timg_b200.lib().b200timg_blocks_batch_dev(ctx.h, C.byref(ub), d_src.data_ptr(), d_out.data_ptr(), cap,
                                                       d_offs.data_ptr()))
    timg_b200.device_sync(torch)
    o, data = d_offs.cpu().numpy(), d_out.cpu().numpy()
    uniform = [data[o[f]:o[f + 1]].tobytes() for f in range(n)]
    mixed = ctx.blocks_mixed(list(frames), [(ow, oh)] * n, [indent] * n, flags, **COMPOSE)
    assert mixed == uniform


def test_mixed_capacity_contract(ctx):
    import torch
    imgs, outs, ind = _select(page(), [3, 5, 6, 9, 10, 11, 14])
    want = ctx.blocks_mixed(imgs, outs, ind, 0, **COMPOSE)
    sizes = np.array([len(w) for w in want], np.int64)
    ends = np.cumsum(sizes)
    total = int(ends[-1])
    flat, offs = timg_b200.pack_mixed(imgs)
    b, keep = timg_b200.mixed_batch([im.shape for im in imgs], outs, offs, ind, 0, **COMPOSE)
    d_src = timg_b200._device_tensor(torch, flat)
    # device variant: a cap that ends inside frame 3
    cap = int(ends[2]) + int(sizes[3]) // 2
    d_out = torch.full((total + 64,), 0xA5, dtype=torch.uint8, device=d_src.device)
    timg_b200.device_sync(torch)
    _, d_offs = ctx.blocks_mixed_dev(d_src, b, d_out=d_out, out_cap=cap)
    timg_b200.device_sync(torch)
    o, data = d_offs.cpu().numpy(), d_out.cpu().numpy()
    assert list(o) == [0] + list(ends)
    assert b"".join(want[:3]) == data[:int(ends[2])].tobytes()
    assert (data[int(ends[2]):] == 0xA5).all()                  # frames past the cap are not written
    # host variant: ENOSPC, offsets complete, nothing written
    out = np.full(total + 64, 0x5A, np.uint8)
    offsets = np.zeros(len(imgs) + 1, np.uint64)
    rc = timg_b200.lib().b200timg_blocks_mixed(ctx.h, C.byref(b), flat.ctypes.data, out.ctypes.data, total - 1,
                                                offsets.ctypes.data)
    assert rc == timg_b200.ENOSPC
    assert int(offsets[-1]) == total and list(offsets) == [0] + list(ends)
    assert (out == 0x5A).all()
    rc = timg_b200.lib().b200timg_blocks_mixed(ctx.h, C.byref(b), flat.ctypes.data, out.ctypes.data, total,
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
    rc = timg_b200.lib().b200timg_blocks_mixed(ctx.h, C.byref(b), src.ctypes.data, out.ctypes.data, out.size, offs.ctypes.data)
    return rc, timg_b200.lib().b200timg_last_error(ctx.h).decode()


@pytest.mark.parametrize("case,kw,needle", [
    ("no frames", dict(n_frames=0), "n_frames > 0"),
    ("null frames", dict(null_frames=True), "frames array"),
    ("zero src", dict(fr=(0, 0, 8, 8, 4, 0)), "non-positive size"),
    ("negative out", dict(fr=(0, 8, 8, 4, -1, 0)), "non-positive size"),
    ("unaligned offset", dict(fr=(2, 8, 8, 4, 4, 0)), "not a multiple of 4"),
    ("odd quarter width", dict(fr=(0, 8, 8, 5, 4, 0), flags=timg_b200.QUARTER), "frame 1: quarter blocks need an even width"),
    ("yuv", dict(src_fmt=timg_b200.FMT_I420), "source format"),
    ("bilinear", dict(flags=timg_b200.BILINEAR_SCALE), "BILINEAR"),
    ("negative indent", dict(fr=(0, 8, 8, 4, 4, -1)), "negative indent"),
])
def test_mixed_rejected_arguments(ctx, case, kw, needle):
    kw = dict(kw)
    good = timg_b200.Frame(0, 8, 8, 4, 4, 0)
    frames = [good, good]
    if "fr" in kw:
        frames[1] = timg_b200.Frame(*kw.pop("fr"))
    rc, msg = _call(ctx, frames, **kw)
    assert rc == timg_b200.EINVAL, case
    assert needle in msg, (case, msg)


def test_mixed_launches_do_not_grow_with_geometries(ctx):
    import torch
    n = 64
    distinct = [synth.frame_np(500 + k, 64 + 5 * k, 48 + 3 * k, "photo") for k in range(n)]
    distinct_outs = [(16 + 2 * (k % 20), 9 + k % 13) for k in range(n)]
    same = [synth.frame_np(600 + k, 200, 120, "photo") for k in range(n)]
    counts = []
    for imgs, outs in ((distinct, distinct_outs), (same, [(40, 24)] * n)):
        assert len(set(zip([im.shape for im in imgs], outs))) in (1, n)
        flat, offs = timg_b200.pack_mixed(imgs)
        b, keep = timg_b200.mixed_batch([im.shape for im in imgs], outs, offs, flags=timg_b200.QUARTER)
        d_src = timg_b200._device_tensor(torch, flat)
        before = ctx.launches
        ctx.blocks_mixed_dev(d_src, b)
        counts.append(ctx.launches - before)
    assert counts[0] == counts[1], counts
