"""Kitty / iTerm2 mixed batches (b200timg_graphics_mixed): a `-pk` / `-pi` grid page of differently sized images
scaled, composed, PNG-encoded and framed in one call, against the one-frame uniform batch, the oracle and the
reference's bytes, independent of the batch's composition, the capacity contract, the rejected arguments and the
launch count -- for kitty, iTerm2 and kitty's tmux form, with stored blocks and B200TIMG_DEFLATE."""
import base64
import ctypes as C
import os
import sys

import numpy as np
import pytest

import oracle
import timg_b200
from timg_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import graphics_cases as gcases  # noqa: E402
import graphics_tmux_cases as tcases  # noqa: E402
from test_graphics_oracle import GOLD as PLAIN_GOLD, iterm2_payload, kitty_payload, png_pixels  # noqa: E402
from test_graphics_tmux_oracle import GOLD as TMUX_GOLD, all_cases, golden_keys, kitty_tmux_payload  # noqa: E402

pytestmark = pytest.mark.gpu

K, I, T, D = timg_b200.KITTY, timg_b200.ITERM2, timg_b200.KITTY_TMUX, timg_b200.DEFLATE
BG = timg_b200.rgba_u32(30, 60, 200)
PATTERN = timg_b200.rgba_u32(200, 180, 20)
COMPOSE = dict(has_bg=True, bg=BG, pattern=PATTERN, pattern_w=4, pattern_h=3)
CELL = (9, 18)
PROTOS = {"kitty": K, "iterm2": I, "tmux": T}


def _page(rgb24):
    """(images, outs, indents): about 20 images of the geometries a grid page meets, for one colour type."""
    for k in range(2, 40):                                              # PNGs of 3072*k bytes and one byte either side
        chunk = [gcases._png_geometry(3072 * k + d, rgb24) for d in (-1, 0, 1)]
        if None not in chunk:
            break
    spec = [
        (synth.frame_np(1, 1280, 720, "photo"), (337, 190)),
        (synth.frame_np(2, 640, 480, "alpha"), (160, 119)),            # transparency onto the checkerboard
        (synth.frame_np(3, 640, 480, "noise"), (161, 121)),            # odd sizes
        (synth.frame_np(4, 50, 40, "photo"), (1, 1)),
        (synth.frame_np(5, 50, 400, "alpha"), (1, 100)),
        (synth.frame_np(6, 400, 50, "noise"), (100, 1)),
        (synth.frame_np(7, 120, 80, "photo"), (240, 160)),             # upscale
        (synth.frame_np(8, 96, 64, "noisea"), (96, 64)),               # identity
        (synth.frame_np(9, 440, 800, "photo"), (110, 200)),            # scanlines above 65535 bytes: several blocks / segments
        (synth.frame_np(10, 4800, 40, "photo"), (2400, 20)),           # 266 placeholders per tmux row: two grid items
        (synth.frame_np(11, 300, 200, "alpha"), (100, 67)),
        (synth.frame_np(12, 33, 17, "noise"), (66, 34)),
        (synth.frame_np(13, 480, 640, "photo"), (60, 80)),
        (synth.frame_np(14, 256, 256, "noisea"), (128, 128)),
        (synth.frame_np(15, 1920, 1080, "photo"), (320, 180)),
        (synth.frame_np(1, 1280, 720, "photo"), (337, 190)),           # a repeated geometry
    ]
    for k, (w, h) in enumerate(chunk):
        spec.append((synth.frame_np(20 + k, w, h, "noisea"), (w, h)))
    imgs, outs = [s[0] for s in spec], [s[1] for s in spec]
    return imgs, outs, [(3 * f) % 14 for f in range(len(outs))]


def _ids(n, seed=0):
    return [(0x01020304 * (f + 1) + 977 * seed) & 0xFFFFFFFF for f in range(n)]


def _uniform(ctx, img, ow, oh, proto, rgb24, id_, indent, compose=COMPOSE):
    """b200timg_graphics_batch_dev with flags = 0 on this image alone."""
    import torch
    ih, iw = img.shape[:2]
    b = timg_b200.Batch(n_frames=1, src_w=iw, src_h=ih, src_fmt=0, out_w=ow, out_h=oh, has_bg=int(compose["has_bg"]),
                        bg=compose.get("bg", 0), pattern=compose.get("pattern", 0), pattern_w=compose.get("pattern_w", 0),
                        pattern_h=compose.get("pattern_h", 0), flags=0, x_indent_cells=0, animation=0)
    d_src = timg_b200._device_tensor(torch, img[None])
    cell = CELL if (proto & ~D) == T else None
    d_out, d_offs = ctx.graphics_batch_dev(d_src, b, proto, rgb24, [id_], cell=cell, indent=indent)
    timg_b200.device_sync(torch)
    o = d_offs.cpu().numpy()
    return d_out.cpu().numpy()[o[0]:o[1]].tobytes()


def _mixed_dev(ctx, imgs, outs, proto, rgb24, ids, indents, compose=COMPOSE, cell=CELL, **kw):
    import torch
    flat, offs = timg_b200.pack_mixed(imgs)
    b, keep = timg_b200.mixed_batch([im.shape for im in imgs], outs, offs, indents, **compose)
    g, keep_ids = timg_b200.graphics(proto, rgb24, ids, cell)
    d_src = timg_b200._device_tensor(torch, flat)
    d_out, d_offs = ctx.graphics_mixed_dev(d_src, b, g, **kw)
    timg_b200.device_sync(torch)
    o, data = d_offs.cpu().numpy(), d_out.cpu().numpy()
    return [data[o[f]:o[f + 1]].tobytes() for f in range(len(imgs))], o


def _decode(text, proto, w, h):
    p = proto & ~D
    b64 = kitty_payload(text) if p == K else iterm2_payload(text, w, h) if p == I else kitty_tmux_payload(text)[0]
    return png_pixels(base64.b64decode(b64))[0]


@pytest.mark.parametrize("deflate", [False, True], ids=["stored", "deflate"])
@pytest.mark.parametrize("rgb24", [0, 1])
@pytest.mark.parametrize("pname", list(PROTOS))
def test_page_matches_uniform_batch_and_oracle(ctx, pname, rgb24, deflate):
    imgs, outs, indents = _page(rgb24)
    proto = PROTOS[pname] | (D if deflate else 0)
    ids = _ids(len(imgs))
    ids[15], indents[15] = ids[0], indents[0]                            # the repeated image: the same bytes
    got = ctx.graphics_mixed(imgs, outs, PROTOS[pname], rgb24, ids, indents, CELL, deflate, **COMPOSE)
    for f, (img, (ow, oh)) in enumerate(zip(imgs, outs)):
        assert got[f] == _uniform(ctx, img, ow, oh, proto, rgb24, ids[f], indents[f]), (pname, f, ow, oh)
        want = oracle.compose_bg(oracle.stb_resize(img, ow, oh), BG, PATTERN, 4, 3)
        dec = _decode(got[f], proto, ow, oh)
        assert (dec == want[..., :dec.shape[2]]).all(), (pname, f)
    assert got[0] == got[15]


@pytest.mark.parametrize("pname", ["kitty", "iterm2"])
def test_identity_page_equals_the_reference_bytes(ctx, pname):
    """graphics_cases' frames, one page per colour type, unscaled and without compose: graphics.npz byte for byte."""
    for rgb24 in (0, 1):
        cases = [(n, fb) for n, fb, r in gcases.graphics_frame_cases() if r == rgb24]
        ids = [int(PLAIN_GOLD[f"{pname}/{n}/id"][0]) for n, _ in cases]
        imgs = [fb for _, fb in cases]
        outs = [(fb.shape[1], fb.shape[0]) for fb in imgs]
        got = ctx.graphics_mixed(imgs, outs, PROTOS[pname], rgb24, ids, has_bg=False)
        for (n, _), text in zip(cases, got):
            key = f"{pname}/{n}"
            if key in PLAIN_GOLD:
                assert text == PLAIN_GOLD[key].tobytes(), key
            else:
                assert gcases.sha(text) == PLAIN_GOLD[key + "/sha"].tobytes(), key


def test_tmux_page_equals_the_reference_bytes(ctx):
    """graphics_tmux.npz's t0 cases at 9x18 cells (indents 2, and 0, 1, 12 for the geometry cases) in one page per
    colour type, each frame with its own indent."""
    cases = all_cases()
    keys = [k for k in golden_keys() if k.startswith("t0/") and k.split("/", 1)[1] in cases and k != "t0/c2_rgb1"]
    keys = [k for k in keys if tuple(int(v) for v in TMUX_GOLD[k + "/geo"][3:5]) == CELL]
    assert {int(TMUX_GOLD[k + "/geo"][5]) for k in keys} >= {0, 1, 2, 12}
    for rgb24 in (0, 1):
        page = [k for k in keys if int(TMUX_GOLD[k + "/geo"][2]) == rgb24]
        imgs = [cases[k.split("/", 1)[1]][0] for k in page]
        outs = [(int(TMUX_GOLD[k + "/geo"][0]), int(TMUX_GOLD[k + "/geo"][1])) for k in page]
        assert all((im.shape[1], im.shape[0]) == o for im, o in zip(imgs, outs))
        ids = [int(TMUX_GOLD[k + "/id"][0]) for k in page]
        indents = [int(TMUX_GOLD[k + "/geo"][5]) for k in page]
        got = ctx.graphics_mixed(imgs, outs, T, rgb24, ids, indents, CELL, has_bg=False)
        for k, text in zip(page, got):
            if k in TMUX_GOLD.files:
                assert text == TMUX_GOLD[k].tobytes(), k
            else:
                assert len(text) == int(TMUX_GOLD[k + "/len"][0]) and gcases.sha(text) == TMUX_GOLD[k + "/sha"].tobytes(), k


@pytest.mark.parametrize("deflate", [False, True], ids=["stored", "deflate"])
def test_independent_of_order_grouping_variant_and_company(ctx, monkeypatch, deflate):
    imgs, outs, indents = _page(1)
    ids = _ids(len(imgs))
    proto = T | (D if deflate else 0)
    whole = ctx.graphics_mixed(imgs, outs, T, 1, ids, indents, CELL, deflate, **COMPOSE)
    perm = np.random.default_rng(3).permutation(len(imgs))
    got = ctx.graphics_mixed([imgs[p] for p in perm], [outs[p] for p in perm], T, 1, [ids[p] for p in perm],
                             [indents[p] for p in perm], CELL, deflate, **COMPOSE)
    assert got == [whole[p] for p in perm]
    assert _mixed_dev(ctx, imgs, outs, proto, 1, ids, indents)[0] == whole
    monkeypatch.setenv("B200TIMG_MIXED_GROUP_BYTES", "1")                 # every frame its own scaler group
    assert _mixed_dev(ctx, imgs, outs, proto, 1, ids, indents)[0] == whole
    assert ctx.graphics_mixed(imgs, outs, T, 1, ids, indents, CELL, deflate, **COMPOSE) == whole
    monkeypatch.delenv("B200TIMG_MIXED_GROUP_BYTES")
    # one frame alone, and the same frame among more small frames than the GPU has SMs
    import torch
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    f0 = 8
    assert ctx.graphics_mixed([imgs[f0]], [outs[f0]], T, 1, [ids[f0]], [indents[f0]], CELL, deflate, **COMPOSE) == [whole[f0]]
    small = [synth.frame_np(40 + k, 24 + k % 7, 18 + k % 5, "photo") for k in range(n_sm + 8)]
    small_outs = [(8 + k % 9, 5 + k % 4) for k in range(n_sm + 8)]
    mid = len(small) // 2
    page_ids = _ids(len(small) + 1, 1)
    page_ids[mid] = ids[f0]
    page_ind = [k % 5 for k in range(len(small) + 1)]
    page_ind[mid] = indents[f0]
    res = ctx.graphics_mixed(small[:mid] + [imgs[f0]] + small[mid:], small_outs[:mid] + [outs[f0]] + small_outs[mid:], T, 1,
                             page_ids, page_ind, CELL, deflate, **COMPOSE)
    assert res[mid] == whole[f0]
    for k in (0, mid + 1, len(res) - 1):
        j = k if k < mid else k - 1
        assert res[k] == _uniform(ctx, small[j], *small_outs[j], proto, 1, page_ids[k], page_ind[k]), k


@pytest.mark.parametrize("deflate", [False, True], ids=["stored", "deflate"])
def test_ids_of_every_length_and_msb_diacritic(ctx, deflate):
    """ids of 1 to 10 digits; msb values with a 2-, 3- and 4-byte diacritic (and none past the list)."""
    ids = [7, 42, 999, 1234, 56789, 123456, 1234567, 12345678, (1 << 24) + 5, (40 << 24) + 77, (290 & 255) << 24 | 3,
           0xFFFFFFFF, 2_000_000_000]
    assert {len(str(i)) for i in ids} == set(range(1, 11))
    imgs = [synth.frame_np(300 + k, 40 + 3 * k, 30 + k, "alpha") for k in range(len(ids))]
    outs = [(20 + 5 * k, 19 + 2 * k) for k in range(len(ids))]
    indents = [k % 4 for k in range(len(ids))]
    for pname in ("kitty", "tmux"):
        proto = PROTOS[pname] | (D if deflate else 0)
        got = ctx.graphics_mixed(imgs, outs, PROTOS[pname], 0, ids, indents, CELL, deflate, **COMPOSE)
        for f in range(len(ids)):
            assert got[f] == _uniform(ctx, imgs[f], *outs[f], proto, 0, ids[f], indents[f]), (pname, f)


@pytest.mark.parametrize("deflate", [False, True], ids=["stored", "deflate"])
def test_uniform_geometry_equals_uniform_batch(ctx, deflate):
    """A mixed page whose frames share C4's geometry (4K -> 337x190) equals b200timg_graphics_batch_dev byte for byte."""
    import torch
    frames = gcases.c4_graphics_frames()
    n = frames.shape[0]
    ih, iw = frames.shape[1:3]
    ids = _ids(n, 5)
    b = timg_b200.Batch(n_frames=n, src_w=iw, src_h=ih, src_fmt=0, out_w=337, out_h=190, has_bg=1, bg=BG, pattern=PATTERN,
                        pattern_w=4, pattern_h=3, flags=0, x_indent_cells=0, animation=0)
    proto = K | (D if deflate else 0)
    d_out, d_offs = ctx.graphics_batch_dev(timg_b200._device_tensor(torch, frames), b, proto, 1, ids)
    timg_b200.device_sync(torch)
    o = d_offs.cpu().numpy()
    want = [d_out.cpu().numpy()[o[f]:o[f + 1]].tobytes() for f in range(n)]
    assert ctx.graphics_mixed(list(frames), [(337, 190)] * n, K, 1, ids, deflate=deflate, **COMPOSE) == want


@pytest.mark.parametrize("deflate", [False, True], ids=["stored", "deflate"])
def test_capacity_contract(ctx, deflate):
    import torch
    imgs, outs, indents = _page(0)
    keep = [1, 2, 3, 6, 8, 11, 12]
    imgs, outs, indents = [imgs[f] for f in keep], [outs[f] for f in keep], [indents[f] for f in keep]
    ids = _ids(len(imgs))
    proto = T | (D if deflate else 0)
    want = ctx.graphics_mixed(imgs, outs, T, 0, ids, indents, CELL, deflate, **COMPOSE)
    sizes = np.array([len(w) for w in want], np.int64)
    ends = np.cumsum(sizes)
    total = int(ends[-1])
    cap = int(ends[3]) + int(sizes[4]) // 2                                # ends inside frame 4
    flat, offs = timg_b200.pack_mixed(imgs)
    b, _ = timg_b200.mixed_batch([im.shape for im in imgs], outs, offs, indents, **COMPOSE)
    g, keep_ids = timg_b200.graphics(proto, 0, ids, CELL)
    d_src = timg_b200._device_tensor(torch, flat)
    d_out = torch.full((total + 64,), 0xA5, dtype=torch.uint8, device=d_src.device)
    timg_b200.device_sync(torch)
    _, d_offs = ctx.graphics_mixed_dev(d_src, b, g, d_out=d_out, out_cap=cap)
    timg_b200.device_sync(torch)
    o, data = d_offs.cpu().numpy(), d_out.cpu().numpy()
    assert list(o) == [0] + list(ends)
    assert b"".join(want[:4]) == data[:int(ends[3])].tobytes()
    assert (data[int(ends[3]):] == 0xA5).all()                  # frame 4 and later are not written at all
    out = np.full(total + 64, 0x5A, np.uint8)
    offsets = np.zeros(len(imgs) + 1, np.uint64)
    rc = timg_b200.lib().b200timg_graphics_mixed(ctx.h, C.byref(b), C.byref(g), flat.ctypes.data, out.ctypes.data, total - 1,
                                                  offsets.ctypes.data)
    assert rc == timg_b200.ENOSPC
    assert list(offsets) == [0] + list(ends)
    assert (out == 0x5A).all()
    rc = timg_b200.lib().b200timg_graphics_mixed(ctx.h, C.byref(b), C.byref(g), flat.ctypes.data, out.ctypes.data, total,
                                                  offsets.ctypes.data)
    assert rc == timg_b200.OK and out[:total].tobytes() == b"".join(want) and (out[total:] == 0x5A).all()


_IDS = (C.c_uint32 * 4)(1, 2, 3, 4)


@pytest.mark.parametrize("case,kw,needle", [
    ("no frames", dict(n_frames=0), "n_frames > 0"),
    ("null frames", dict(null_frames=True), "frames array"),
    ("too many frames", dict(n_frames=65536), "at most 65535"),
    ("zero src", dict(fr=(0, 0, 8, 8, 4, 0)), "non-positive size"),
    ("unaligned offset", dict(fr=(2, 8, 8, 4, 4, 0)), "not a multiple of 4"),
    ("yuv", dict(src_fmt=timg_b200.FMT_I420), "source format"),
    ("bilinear", dict(flags=timg_b200.BILINEAR_SCALE), "BILINEAR"),
    ("negative indent", dict(fr=(0, 8, 8, 4, 4, -1)), "negative indent"),
    ("unknown protocol", dict(g=(5, 0, True, 9, 18)), "unknown protocol"),
    ("3 | deflate", dict(g=(3 | D, 0, True, 9, 18)), "unknown protocol"),
    ("null ids", dict(g=(K, 0, False, 0, 0)), "ids is NULL"),
    ("tmux cell x", dict(g=(T, 0, True, 0, 18)), "cell size"),
    ("tmux cell y", dict(g=(T | D, 0, True, 9, -1)), "cell size"),
    ("huge png", dict(fr=(0, 8, 8, 30000, 30000, 0)), "frame 1: the PNG"),
])
def test_rejected_arguments(ctx, case, kw, needle):
    kw = dict(kw)
    good = timg_b200.Frame(0, 8, 8, 4, 4, 0)
    frames = [good, good]
    if "fr" in kw:
        frames[1] = timg_b200.Frame(*kw.pop("fr"))
    proto, rgb24, with_ids, cx, cy = kw.pop("g", (K, 0, True, 0, 0))
    g = timg_b200.Graphics(proto, rgb24, C.cast(_IDS, C.POINTER(C.c_uint32)) if with_ids else None, cx, cy, -7)
    null_frames = kw.pop("null_frames", False)
    d = dict(n_frames=len(frames), src_fmt=0, flags=0, has_bg=1, bg=0, pattern=0, pattern_w=0, pattern_h=0)
    d.update(kw)
    arr = (timg_b200.Frame * len(frames))(*frames)
    b = timg_b200.MixedBatch(frames=None if null_frames else arr, **d)
    src = np.zeros(1 << 16, np.uint8)
    out = np.zeros(1 << 16, np.uint8)
    offs = np.zeros(len(frames) + 2, np.uint64)
    rc = timg_b200.lib().b200timg_graphics_mixed(ctx.h, C.byref(b), C.byref(g), src.ctypes.data, out.ctypes.data, out.size,
                                                  offs.ctypes.data)
    msg = timg_b200.lib().b200timg_last_error(ctx.h).decode()
    assert rc == timg_b200.EINVAL, (case, msg)
    assert needle in msg, (case, msg)


@pytest.mark.parametrize("deflate", [False, True], ids=["stored", "deflate"])
def test_launches_do_not_grow_with_geometries(ctx, deflate):
    import torch
    n = 64
    distinct = [synth.frame_np(500 + k, 64 + 5 * k, 48 + 3 * k, "photo") for k in range(n)]
    distinct_outs = [(16 + 2 * (k % 20), 9 + k % 13) for k in range(n)]
    same = [synth.frame_np(600 + k, 200, 120, "photo") for k in range(n)]
    counts = []
    for imgs, outs in ((distinct, distinct_outs), (same, [(40, 24)] * n)):
        assert len(set(zip([im.shape for im in imgs], outs))) in (1, n)
        before = ctx.launches
        _mixed_dev(ctx, imgs, outs, T | (D if deflate else 0), 0, _ids(n), [k % 3 for k in range(n)])
        counts.append(ctx.launches - before)
    assert counts[0] == counts[1], counts
