"""The GIF corpus of the decoder's tests: every quirk of stbi__gif_load_next as the STB source calls it
(third_party/stb/stb_image.h:6779-6951, two_back = NULL), written by oracle/gif.py from fixed seeds.  Malformed files are
byte surgery on well-formed ones.  tests/golden/make_gif_golden.py pins the reference's canvases of every file here."""
import numpy as np

from oracle import gif as G


def _rng(seed):
    return np.random.default_rng(seed)


def _pal(rng, n):
    return rng.integers(0, 256, (n, 3), dtype=np.uint8)


def _blobs(rng, h, w, n_colors, n_blobs=6):
    """Flat regions with some noise: strings of every length, like drawn content."""
    idx = np.zeros((h, w), np.uint8)
    for _ in range(n_blobs):
        y0, x0 = rng.integers(0, h), rng.integers(0, w)
        idx[y0:y0 + rng.integers(1, h + 1), x0:x0 + rng.integers(1, w + 1)] = rng.integers(0, n_colors)
    noise = rng.random((h, w)) < 0.05
    idx[noise] = rng.integers(0, n_colors, int(noise.sum()))
    return idx


def animation(seed, w, h, n, n_colors=64, rect_frac=0.5, transparent=True, interlace=False, lzw_cs=8):
    """n frames over a w x h screen: frame 0 full, later frames sub-rectangles of up to rect_frac of each side with
    dispose 0..3 in turn and (transparent) a transparency index."""
    rng = _rng(seed)
    pal = _pal(rng, 256)
    frames = [dict(idx=_blobs(rng, h, w, n_colors), lzw_cs=lzw_cs, interlace=interlace,
                   gce=dict(dispose=1, delay=int(rng.integers(0, 20))))]
    for k in range(1, n):
        rw = int(rng.integers(1, max(2, int(w * rect_frac)) + 1))
        rh = int(rng.integers(1, max(2, int(h * rect_frac)) + 1))
        x, y = int(rng.integers(0, w - rw + 1)), int(rng.integers(0, h - rh + 1))
        t = int(rng.integers(0, n_colors)) if transparent else None
        frames.append(dict(idx=_blobs(rng, rh, rw, n_colors, 3), x=x, y=y, lzw_cs=lzw_cs, interlace=interlace,
                           gce=dict(dispose=k % 4, transparent=t, delay=int(rng.integers(0, 20)))))
    return G.gif(w, h, frames, gpal=pal, head=G.netscape())


def _replace_gce_len(data, new_len):
    i = data.index(b"\x21\xf9\x04")
    return data[:i + 2] + bytes([new_len]) + data[i + 3:]


def _nth(data, pat, k):
    i = -1
    for _ in range(k + 1):
        i = data.index(pat, i + 1)
    return i


def corpus():
    """name -> GIF bytes."""
    C = {}
    rng = _rng(20261017)
    pal = _pal(rng, 256)

    # plain animations: disposals 0-3, transparency, sub-rectangles, delays, interlace
    C["anim-64x48x12"] = animation(1, 64, 48, 12)
    C["anim-interlaced-40x30x6"] = animation(2, 40, 30, 6, interlace=True)
    C["anim-opaque-33x17x5"] = animation(3, 33, 17, 5, transparent=False, rect_frac=1.0)
    C["anim-cs4-50x20x7"] = animation(4, 50, 20, 7, n_colors=16, lzw_cs=4)
    # interlaced heights 1..8 (the passes collapse) and odd widths
    for hh in range(1, 9):
        idx = _rng(100 + hh).integers(0, 256, (hh, 7), dtype=np.uint8)
        C[f"interlace-h{hh}"] = G.gif(7, hh, [dict(idx=idx, interlace=True)], gpal=pal)
    # lzw_cs 0, 1, 2, 12 (0 and 1 are outside the GIF specification; stb takes them)
    for cs in (0, 1, 2, 12):
        n = min(256, 1 << cs)
        frames = [dict(idx=_rng(200 + cs).integers(0, n, (21, 19), dtype=np.uint8), lzw_cs=cs,
                       gce=dict(dispose=1, delay=3)),
                  dict(idx=_rng(300 + cs).integers(0, n, (9, 11), dtype=np.uint8), x=3, y=5, lzw_cs=cs,
                       gce=dict(dispose=2, transparent=0, delay=4))]
        C[f"lzw-cs{cs}"] = G.gif(19, 21, frames, gpal=pal[:max(2, n)] if cs <= 8 else pal)
    # sub-block lengths 1 and 7, a frame of width 0
    C["subblock-1"] = G.gif(16, 16, [dict(idx=_blobs(rng, 16, 16, 8), subblock=1)], gpal=pal)
    C["subblock-7-two"] = G.gif(16, 16, [dict(idx=_blobs(rng, 16, 16, 8), subblock=7),
                                          dict(idx=_blobs(rng, 5, 9, 8), x=2, y=1, subblock=7)], gpal=pal)
    zero_w = G.gif(12, 10, [dict(idx=_blobs(rng, 10, 12, 8), gce=dict(dispose=2)),
                            dict(idx=np.zeros((4, 0), np.uint8), x=3, y=3, gce=dict(dispose=1)),
                            dict(idx=_blobs(rng, 4, 4, 8), x=1, y=1)], gpal=pal)
    C["rect-w0"] = zero_w
    # the first-frame background rule: bgindex > 0 with a partial first frame, bgindex == transparent, bgindex past
    # the global table (zeros, made opaque by the rule), and 0 (no rule)
    f0 = dict(idx=_blobs(rng, 6, 8, 4), x=2, y=3, gce=dict(dispose=1, transparent=5))
    f1 = dict(idx=np.full((10, 12), 5, np.uint8), gce=None)
    f2 = dict(idx=np.full((10, 12), 5, np.uint8), gce=dict(dispose=0, transparent=1))
    for bg in (0, 3, 5):
        C[f"bg{bg}-transparent5"] = G.gif(12, 10, [f0, f1, f2], gpal=pal[:8], bgindex=bg)
    C["bg-past-table"] = G.gif(12, 10, [dict(idx=_blobs(rng, 6, 8, 4), x=1, y=1),
                                        dict(idx=np.full((10, 12), 3, np.uint8), gce=dict(dispose=2)),
                                        dict(idx=np.full((3, 3), 3, np.uint8), x=2, y=2, gce=None)],
                               gpal=pal[:4], bgindex=200)
    full0 = dict(idx=_blobs(rng, 10, 12, 4), gce=dict(transparent=3))
    C["bg-full-first-frame"] = G.gif(12, 10, [full0, dict(idx=np.full((10, 12), 3, np.uint8), gce=None)],
                                     gpal=pal[:8], bgindex=3)
    C["bg-past-table-index-drawn"] = G.gif(8, 8, [dict(idx=np.full((4, 4), 2, np.uint8), x=0, y=0, lzw_cs=8),
                                                  dict(idx=np.full((8, 8), 250, np.uint8))],
                                           gpal=pal[:4], bgindex=250)
    # indices past a table's size, local tables with and without transparency, lpal carry-over (a smaller local
    # table leaves the entries of a larger one), frames with no GCE (eflags, transparent, delay persist)
    big_l, small_l = _pal(rng, 64), _pal(rng, 4)
    C["lpal-carry"] = G.gif(10, 9, [
        dict(idx=rng.integers(0, 64, (9, 10), dtype=np.uint8), lpal=big_l, gce=dict(dispose=1, transparent=7, delay=9)),
        dict(idx=rng.integers(0, 64, (5, 6), dtype=np.uint8), x=2, y=2, lpal=small_l, gce=None),
        dict(idx=rng.integers(0, 64, (4, 4), dtype=np.uint8), x=0, y=5, lpal=small_l, gce=dict(dispose=3, delay=2)),
        dict(idx=rng.integers(0, 255, (9, 10), dtype=np.uint8), gce=None)], gpal=pal[:16], bgindex=2)
    C["no-global-local-only"] = G.gif(6, 5, [dict(idx=rng.integers(0, 8, (5, 6), dtype=np.uint8), lpal=pal[:8]),
                                             dict(idx=rng.integers(0, 8, (2, 2), dtype=np.uint8), x=4, y=3,
                                                  lpal=pal[8:16], gce=dict(dispose=2, transparent=1))])
    C["gif87a"] = G.gif(9, 7, [dict(idx=_blobs(rng, 7, 9, 16))], gpal=pal[:16], version=b"87a")
    C["comment-netscape"] = G.gif(9, 7, [dict(idx=_blobs(rng, 7, 9, 16), pre=G.comment(b"x" * 300)),
                                         dict(idx=_blobs(rng, 3, 3, 16), pre=G.comment(), gce=dict(delay=7))],
                                  gpal=pal[:16], head=G.netscape(3) + G.comment(b"head"))
    C["no-trailer"] = G.gif(9, 7, [dict(idx=_blobs(rng, 7, 9, 16)), dict(idx=_blobs(rng, 3, 3, 16))], gpal=pal[:16],
                            trailer=False)

    # errors the walk sees
    base = animation(5, 24, 20, 5)
    C["bad-tag"] = base[:_nth(base, b"\x21\xf9\x04", 3)] + b"\x99" + base[_nth(base, b"\x21\xf9\x04", 3):]
    C["gce-len-5"] = _replace_gce_len(base, 5)          # its terminator is read as a tag (0: unknown code)
    g3 = _nth(base, b"\x21\xf9\x04", 2)
    C["gce-len-3-later"] = base[:g3 + 2] + b"\x03" + base[g3 + 3:]
    bad_rect = bytearray(G.gif(10, 10, [dict(idx=_blobs(rng, 10, 10, 8)), dict(idx=_blobs(rng, 4, 4, 8), x=6, y=6)],
                               gpal=pal))
    d = _nth(bytes(bad_rect), b"\x2c\x06\x00\x06\x00", 0)
    bad_rect[d + 1] = 7                                    # x + w = 11 > 10
    C["rect-outside"] = bytes(bad_rect)
    C["no-color-table"] = G.gif(6, 6, [dict(idx=_blobs(rng, 6, 6, 4), lpal=pal[:4]), dict(idx=_blobs(rng, 2, 2, 4))])
    cs13 = bytearray(G.gif(6, 6, [dict(idx=_blobs(rng, 6, 6, 4)), dict(idx=_blobs(rng, 3, 3, 4), x=1, y=1)], gpal=pal))
    d = _nth(bytes(cs13), b"\x2c\x01\x00\x01\x00", 0)
    cs13[d + 10] = 13                                      # lzw_cs 13 (the byte after the descriptor's flags)
    C["lzw-cs13"] = bytes(cs13)
    d1, d3 = _nth(base, b"\x2c", 0), _nth(base, b"\x2c", 2)    # frame 0's and frame 2's image descriptors
    for name, cut in (("in-frame0-raster", d1 + 40), ("in-frame0-descriptor", d1 + 4), ("in-frame2-raster", d3 + 30),
                      ("before-trailer", len(base) - 1), ("in-last-terminator", len(base) - 2)):
        C[f"truncated-{name}"] = base[:cut]

    # errors only decoding finds: no clear code at frame 0, 1 and the last frame; an illegal code; too many codes
    def anim_with(policy_at, n=4):
        r = _rng(77)
        frames = [dict(idx=_blobs(r, 16, 20, 32), policy=G.NO_START_CLEAR if k == policy_at else G.CLEAR_START,
                       gce=dict(dispose=k % 4, transparent=1, delay=5))
                  if k == 0 else
                  dict(idx=_blobs(r, 8, 9, 32), x=k, y=k, policy=G.NO_START_CLEAR if k == policy_at else G.CLEAR_START,
                       gce=dict(dispose=k % 4, transparent=1, delay=5)) for k in range(n)]
        return G.gif(20, 16, frames, gpal=pal)
    C["no-clear-frame0"] = anim_with(0)
    C["no-clear-frame1"] = anim_with(1)
    C["no-clear-last"] = anim_with(3)
    r = _rng(78)
    ok = [dict(idx=_blobs(r, 16, 20, 32), gce=dict(dispose=1, delay=5)),
          dict(idx=_blobs(r, 8, 9, 32), x=1, y=1, gce=dict(dispose=2, transparent=1, delay=6))]
    # after a clear (avail 258): 300 > avail; 258 == avail with no previous code; a clear and then only an EOI
    C["illegal-code-gt-avail-frame2"] = G.gif(20, 16, ok + [
        dict(idx=np.zeros((8, 9), np.uint8), x=2, y=2, raster=G.codes([256, 7, 300, 257], 8, [9] * 4))], gpal=pal)
    C["illegal-code-eq-avail-frame2"] = G.gif(20, 16, ok + [
        dict(idx=np.zeros((8, 9), np.uint8), x=2, y=2, raster=G.codes([256, 258, 257], 8, [9] * 3))], gpal=pal)
    C["eoi-only-frame2"] = G.gif(20, 16, ok + [
        dict(idx=np.zeros((8, 9), np.uint8), x=2, y=2, raster=G.codes([256, 257], 8, [9] * 2)),
        dict(idx=_blobs(r, 3, 3, 32), x=5, y=5)], gpal=pal)
    # frame 0 covers the screen but its stream stops short: whether the first-frame rule runs (and makes pal[bgindex]
    # opaque for later frames) is known only after decoding
    short = _blobs(r, 16, 20, 4)
    for name, n_idx in (("short", 150), ("exact", 320)):
        C[f"bg-rule-{name}-stream"] = G.gif(20, 16, [
            dict(idx=short, raster=G.lzw(short.reshape(-1)[:n_idx]), gce=dict(dispose=1, transparent=6)),
            dict(idx=np.full((16, 20), 6, np.uint8), gce=None),
            dict(idx=np.full((16, 20), 6, np.uint8), gce=dict(transparent=2))], gpal=pal[:8], bgindex=6)
    # a stream longer than its rectangle: the codes past the area are still checked
    C["stream-longer-than-rect"] = G.gif(20, 16, ok + [
        dict(idx=np.zeros((2, 2), np.uint8), x=3, y=3, raster=G.lzw(_blobs(r, 8, 9, 32)))], gpal=pal)
    C["stream-longer-then-illegal"] = G.gif(20, 16, ok + [
        dict(idx=np.zeros((1, 2), np.uint8), x=3, y=3, raster=G.codes([256, 7, 8, 9, 10, 11, 400], 8, [9] * 7))],
        gpal=pal)
    noise = _rng(9).integers(0, 256, (120, 100), dtype=np.uint8)
    C["too-many-codes-frame1"] = G.gif(100, 120, [dict(idx=_blobs(rng, 120, 100, 8)),
                                                  dict(idx=noise, policy=G.DEFERRED_CLEAR, gce=dict(delay=1))],
                                       gpal=pal)
    C["deferred-clear-fits"] = G.gif(60, 50, [dict(idx=_rng(10).integers(0, 256, (50, 60), dtype=np.uint8),
                                                   policy=G.DEFERRED_CLEAR)], gpal=pal)
    C["long-table-clears"] = G.gif(100, 120, [dict(idx=noise), dict(idx=noise[:60, :50] // 64, x=5, y=7, lzw_cs=2)],
                                   gpal=pal)
    return C


def sized(name):
    """The animations of the size tests, written from fixed seeds: 480x270 x 120 frames with small sub-rectangles
    and transparency, 1920x1080 x 64 frames, one 4096x2160 frame."""
    if name == "480x270x120":
        return animation(11, 480, 270, 120, rect_frac=0.25)
    if name == "1920x1080x64":
        return animation(12, 1920, 1080, 64, rect_frac=0.6)
    if name == "4096x2160x1":
        return animation(13, 4096, 2160, 1)
    raise KeyError(name)


SIZED = ("480x270x120", "1920x1080x64", "4096x2160x1")
