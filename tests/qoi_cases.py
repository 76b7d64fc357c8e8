"""QOI files for the decoder's tests, built deterministically, and a small plan model of how qoi.cu splits a file.

corpus(): (name, bytes) of ordinary images (oracle/qoi.py's encoder) and hand-made op streams (its op writer): the
quirks of qoi_decode, truncations, padding and trailing bytes, and every header rejection on both sides of its bound.
split_cases(): (name, bytes, where) aimed at the decoder's split points: ops straddling tile and chunk boundaries,
ops at segment and checkpoint edges, a slot that only the sync rounds or the fix-up carry to where it is read, and a
stream that never synchronises.  `where` says where the case lands in the model's terms; test_qoi_parse.py checks it.

The model: an op's length follows from its first byte; op starts are tiled by TILE bytes of the op region (which
starts at byte 14), CHUNK tiles to a chunk; live ops (first pixel < w*h) are cut into segments of SEG ops, each with a
checkpoint every CK ops; ROUNDS sync rounds run before the fix-up.  These mirror the constexprs of qoi.cu.
"""
import numpy as np

from oracle import qoi as Q
import png_cases as pc
from timg_b200 import synth

TILE, CHUNK, SEG, CK, ROUNDS = 64, 64, 256, 64, 8
LAUNCHES = 7 + ROUNDS
HEADER = 14


def op_len(b):
    return 4 if b == 0xFE else 5 if b == 0xFF else 2 if b >> 6 == 2 else 1


def op_pixels(b):
    return (b & 63) + 1 if b >> 6 == 3 and b < 0xFE else 1


def live_ops(data):
    """(byte offset in the file, first pixel) of every op qoi_decode reads: it starts before size - 8, and pixels
    remain."""
    w, h = int.from_bytes(data[4:8], "big"), int.from_bytes(data[8:12], "big")
    end, pos, px, out = len(data) - 8, HEADER, 0, []
    while pos < end and px < w * h:
        out.append((pos, px))
        px += op_pixels(data[pos])
        pos += op_len(data[pos])
    return out


def tile_of(offset):
    return (offset - HEADER) // TILE


def rgb_for_slot(slot, k):
    """An opaque colour whose index slot is `slot`, varied by k."""
    g, b = (k * 37) & 255, (k * 91 + 11) & 255
    r = (43 * (slot - 5 * g - 7 * b - 11 * 255)) % 64 + 64 * (k % 4)   # 43 = 3^-1 mod 64
    assert Q.hash_slot(r, g, b, 255) == slot
    return r, g, b


# ---- ordinary images ---------------------------------------------------------------------------------------------
def gradient(w, h):
    """A horizontal ramp that only DIFF ops encode: px never resets, so no segment synchronises by itself."""
    img = np.zeros((h, w, 4), np.uint8)
    x = np.arange(w * h).reshape(h, w)
    img[..., 0] = x % 256
    img[..., 1] = (x // 2) % 256
    img[..., 3] = 255
    return img


def photo_smooth(w, h, seed=0):
    """A camera-like photo: smooth shading, 40 discs of their own colour, luminance noise (sigma 2.5) and a little
    chroma noise.  Our encoder gives about 45 % of the RGBA size, mostly LUMA and DIFF ops with about 1 % RGB ops --
    the mix QOI gives real photos, unlike png_cases.photo, whose +-24 noise makes nearly every op RGB."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([128 + 90 * np.sin(x / 370 + c) * np.cos(y / 290 - c) + 30 * np.sin((x + y) / 97 + 2 * c)
                     for c in (0.0, 0.8, 1.9)], -1)
    for _ in range(40):
        cx, cy, r = rng.integers(0, w), rng.integers(0, h), rng.integers(20, max(21, w // 8))
        m = (x - cx) ** 2 + (y - cy) ** 2 < r * r
        base[m] = base[m] * 0.4 + rng.integers(0, 256, 3) * 0.6
    img = base + rng.normal(0, 2.5, (h, w, 1)) + rng.normal(0, 1.0, (h, w, 3))
    return rgba(np.clip(img, 0, 255).astype(np.uint8))


def rgba(a):
    a = np.asarray(a, np.uint8)
    return a if a.shape[-1] == 4 else np.concatenate([a, np.full(a.shape[:2] + (1,), 255, np.uint8)], -1)


def images():
    yield "photo_rgb_cs0", Q.encode(rgba(pc.photo(160, 90, 1)), 3, 0)
    yield "photo_rgba_cs1", Q.encode(pc.photo(150, 100, 2, ch=4), 4, 1)
    yield "photo_smooth_rgb", Q.encode(photo_smooth(640, 360, 12), 3, 0)
    yield "photo_alpha_in_rgb3", Q.encode(pc.photo(600, 300, 11, ch=4), 3, 0)      # status 2, scaled at FRAME_OPTS
    yield "screenshot_rgb", Q.encode(rgba(pc.screenshot(256, 144, 3)), 3, 0)
    yield "screenshot_rgba_cs1", Q.encode(rgba(pc.screenshot(200, 120, 4)), 4, 1)
    yield "alpha_rgba", Q.encode(synth.frame_np(5, 120, 80, "alpha"), 4, 0)
    yield "noise_rgba", Q.encode(synth.frame_np(6, 70, 90, "noise"), 4, 0)
    yield "noise_rgb", Q.encode(rgba(synth.frame_np(7, 90, 70, "noise")[..., :3]), 3, 1)
    yield "gradient_rgb", Q.encode(gradient(300, 40), 3, 0)
    yield "solid_rgba", Q.encode(np.full((64, 96, 4), (10, 20, 30, 255), np.uint8), 4, 0)
    yield "px_1x1", Q.encode(np.array([[[9, 8, 7, 200]]], np.uint8), 4, 0)
    yield "row_16384x1", Q.encode(rgba(pc.photo(16384, 1, 8)), 3, 0)
    yield "col_1x16384", Q.encode(rgba(pc.photo(1, 16384, 9)), 4, 0)


# ---- hand-made streams -------------------------------------------------------------------------------------------
def _tail_base():
    o = Q.Ops()
    for k in range(40):
        o.rgb(*rgb_for_slot(k % 64, k))
    o.luma(5, -3, 2).diff(1, -2, 0).rgba(1, 2, 3, 4).index(7).run(3).rgb(9, 9, 9).luma(-32, 7, -8).rgba(200, 100, 50, 25)
    return o


def streams():
    for n in (1, 2, 17, 61, 62):
        yield f"run_{n}", Q.stream(8, 8, Q.Ops().rgb(1, 2, 3).run(n).diff(1, 1, 1))
    yield "run_across_end", Q.stream(5, 3, Q.Ops().rgb(1, 2, 3).run(13).rgb(4, 5, 6).run(62).rgb(7, 7, 7))
    yield "leading_run_index53", Q.stream(6, 2, Q.Ops().run(3).index(53).diff(1, 0, -1).index(53))
    for ch in (3, 4):
        yield f"index_unwritten_ch{ch}", Q.stream(4, 2, Q.Ops().index(0).index(12).rgb(5, 6, 7).index(40), channels=ch)
    yield "rgb3_with_rgba_ops", Q.stream(4, 4, Q.Ops().rgb(10, 20, 30).rgba(1, 2, 3, 128).run(4), channels=3)
    yield "rgb3_alpha_255", Q.stream(4, 4, Q.Ops().rgba(1, 2, 3, 255).rgb(10, 20, 30).run(6), channels=3)
    yield "rgb3_index_zero_slot", Q.stream(3, 1, Q.Ops().rgb(1, 1, 1).index(33), channels=3)
    base = _tail_base()
    body = base.bytes()
    npx = len(base.starts) + 2
    for cut in range(len(body) - 24, len(body) + 1):
        yield f"truncated_at_{cut}", Q.stream(npx, 1, body[:cut])
    yield "zero_ops", Q.stream(7, 5, b"")
    yield "missing_padding", Q.stream(npx, 1, base, padding=b"")
    yield "padding_0_only", Q.stream(npx, 1, base, padding=bytes(8))
    yield "trailing_bytes", Q.stream(npx, 1, base, trailing=bytes([0xFE, 1, 2, 3, 0x41, 0x7F, 0xC5]))
    yield "runs_past_last_pixel", Q.stream(12, 1, base)
    yield "op_reads_into_padding", Q.stream(50, 1, Q.Ops().rgb(1, 2, 3).raw(b"\xff\x10"), padding=bytes(6) + b"\x20\x01")


def rejections():
    """(name, bytes, accepted by qoi_decode).  Parse only where accepted files would be too large to decode."""
    ok = Q.Ops().rgb(1, 2, 3).bytes()
    yield "size_21", Q.header(1, 1) + bytes(7), False
    yield "size_22", Q.header(1, 1) + bytes(8), True
    yield "bad_magic", Q.stream(1, 1, ok, magic=b"qoiF"), False
    yield "w_0", Q.stream(0, 4, ok), False
    yield "h_0", Q.stream(4, 0, ok), False
    yield "w_1_h_1", Q.stream(1, 1, ok), True
    for ch in (2, 3, 4, 5):
        yield f"channels_{ch}", Q.stream(2, 2, ok, channels=ch), ch in (3, 4)
    for cs in (1, 2, 255):
        yield f"colorspace_{cs}", Q.stream(2, 2, ok, colorspace=cs), cs <= 1
    # h >= 400000000 / w (unsigned): both sides, parse only
    yield "pixels_max_20000x19999", Q.stream(20000, 19999, ok), True
    yield "pixels_max_20000x20000", Q.stream(20000, 20000, ok), False
    yield "pixels_max_3x133333332", Q.stream(3, 133333332, ok), True
    yield "pixels_max_3x133333333", Q.stream(3, 133333333, ok), False
    yield "pixels_max_w_400000001", Q.stream(400000001, 1, ok), False


def corpus():
    """(name, bytes) of every file the golden pins (rejections included)."""
    yield from images()
    yield from streams()
    for name, data, _ in rejections():
        yield name, data


DECODED_MAX_PX = 1 << 20          # rejection-side files past this are pinned by their parse only


# ---- split points ------------------------------------------------------------------------------------------------
def _filler(o, n, k0=0):
    """n RGB ops cycling through every slot."""
    for k in range(n):
        o.rgb(*rgb_for_slot((k0 + k) % 64, k0 + k))
    return o


def split_cases():
    """(name, bytes, where): where is a dict the model checks -- 'straddle' (the op's offset, the tile boundary it
    crosses), 'op_at' (op index, the op's first byte), 'rounds' (segments - 1, the stale slot's reader segment)."""
    out = []
    # 4- and 5-byte ops straddling tile and chunk boundaries at every offset: DIFF ops (1 byte) up to the boundary - j
    for boundary in (TILE, 2 * TILE, CHUNK * TILE):
        for j in range(1, 5):
            for kind in ("rgb", "rgba", "luma"):
                if kind == "luma" and j > 1:
                    continue
                if kind == "rgb" and j > 3:
                    continue
                o = Q.Ops()
                for k in range(boundary - j):
                    o.diff((k % 4) - 2, 1, -1)
                at = len(o.b)
                {"rgb": lambda: o.rgb(200, 10, 20), "rgba": lambda: o.rgba(1, 2, 3, 9),
                 "luma": lambda: o.luma(7, -2, 3)}[kind]()
                _filler(o, 20)
                out.append((f"straddle_{kind}_tile{boundary // TILE}_minus{j}", Q.stream(len(o.starts), 1, o),
                            dict(straddle=(HEADER + at, HEADER + boundary))))
    # ops at checkpoint and segment edges: an INDEX of an early slot, a RUN and an RGBA there
    for at in (CK - 1, CK, CK + 1, SEG - 1, SEG, SEG + 1, 2 * SEG):
        for kind in ("index", "run", "rgba"):
            o = Q.Ops().rgb(77, 88, 99)                        # slot of (77, 88, 99) is read later
            slot = Q.hash_slot(77, 88, 99, 255)
            k = 1
            while len(o.starts) < at:
                r = rgb_for_slot((slot + 1 + k) % 64, k)
                if Q.hash_slot(*r, 255) != slot:
                    o.rgb(*r)
                k += 1
            {"index": lambda: o.index(slot), "run": lambda: o.run(9), "rgba": lambda: o.rgba(5, 6, 7, 130)}[kind]()
            _filler(o, 70, 3)
            npx = len(o.starts) + 8
            out.append((f"edge_{kind}_op{at}", Q.stream(npx, 1, o), dict(op_at=(at, o.b[o.starts[at]]))))
    # a slot written only in segment 0 and read in segment m: the rounds carry it one segment per round, so the file
    # needs m rounds (ROUNDS - 1: the rounds suffice; ROUNDS: the last round still changes an exit; ROUNDS + 1: only
    # the fix-up reaches the reader)
    for m in (ROUNDS - 1, ROUNDS, ROUNDS + 1):
        h = 17
        o = Q.Ops().rgb(*rgb_for_slot(h, 1000))
        seq = [s for s in range(64) if s != h]
        k = 0
        while len(o.starts) < m * SEG:
            o.rgb(*rgb_for_slot(seq[k % 63], k))
            k += 1
        o.index(h)
        while len(o.starts) < (m + 1) * SEG:
            o.rgb(*rgb_for_slot(seq[k % 63], k))
            k += 1
        out.append((f"stale_slot_rounds_{m}", Q.stream(len(o.starts), 1, o), dict(rounds=(m, h))))
    out.append(("syncs_nowhere", Q.encode(gradient(SEG * 3, 12), 3, 0), dict(diff_only=True)))
    return out


def front_files(k):
    """k ordinary files to put in front of a split case in one call."""
    return [Q.encode(rgba(pc.photo(40 + 7 * i, 30 + 5 * i, 50 + i)), 4, 0) for i in range(k)]


def golden():
    """(name, bytes, parse, sha, status, frame_sha, (frame_w, frame_h)) per pinned case from tests/golden/qoi.npz.
    parse: 1 decoded, 0 parsed only, -1 rejected."""
    import os
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "qoi.npz"))
    files = dict(corpus())
    return [(str(n), files[str(n)], int(p), str(s), int(st), str(fs), (int(fw), int(fh)))
            for n, p, s, st, fs, fw, fh in zip(z["name"], z["parse"], z["sha"], z["status"], z["frame_sha"],
                                               z["frame_w"], z["frame_h"])]


# real options for the scaled-frame pins: a 40x20-cell box of 9x18-pixel cells, a background and a 2-cell pattern
FRAME_OPTS = dict(width=40 * 9, height=20 * 18, cell=(9, 18), has_bg=True, bg=0xFF302010, pattern=0xFF808080,
                  pattern_size=2)
FRAME_CASES = ("photo_rgba_cs1", "alpha_rgba", "noise_rgba", "rgb3_with_rgba_ops", "rgb3_alpha_255", "photo_alpha_in_rgb3",
               "index_unwritten_ch3", "index_unwritten_ch4", "screenshot_rgb")
