"""Deterministic inputs of the kitty / iTerm2 framing goldens (tests/golden/graphics.npz, written by
tests/golden/make_graphics_golden.py): single frames shown unscaled, and small batches with scale + compose."""
from timg_b200 import synth

from cases import c4_frames, sha  # noqa: F401  (re-exported for the golden writer and the tests)

KITTY, ITERM2 = 1, 2
FULL_GOLDEN_BYTES = 24 << 10            # text up to this size (and the several-block frames) is stored in full
C4_GRAPHICS_FRAMES = 3                  # 4K -> 337x190 (C4), composed onto black


def png_size(w, h, rgb24):
    """Bytes of this library's stored-block PNG: signature + IHDR + IDAT(zlib: 2 + 5 per block + scanlines + 4) + IEND."""
    raw = h * (1 + w * (3 if rgb24 else 4))
    return 63 + 5 * max(1, -(-raw // 65535)) + raw


def _png_geometry(target, rgb24):
    """The first (w, h), h <= 64, whose PNG is exactly `target` bytes, or None."""
    for h in range(1, 65):
        for w in range(1, 4096):
            n = png_size(w, h, rgb24)
            if n == target:
                return w, h
            if n > target:
                break
    return None


def graphics_frame_cases():
    """(name, frame, rgb24): frames whose framed text is pinned byte for byte, for both protocols.  Covers 1x1, 2x3,
    PNGs of exactly 3072*k bytes (kitty's chunk) and one byte either side, scanlines above 65535 bytes (several
    stored blocks) and an RGBA frame with alpha."""
    out = []
    for rgb24 in (0, 1):
        sizes = [("1x1", 1, 1), ("2x3", 2, 3), ("blocks", 110 if rgb24 else 82, 200)]      # 66200 / 65800 scanline bytes
        found = 0
        for k in range(1, 40):                     # the first two k for which all three sizes exist
            geos = [_png_geometry(3072 * k + d, rgb24) for d in (-1, 0, 1)]
            if None in geos:
                continue
            sizes += [(f"chunk{k}{tag}", w, h) for tag, (w, h) in zip(("m1", "eq", "p1"), geos)]
            found += 1
            if found == 2:
                break
        for tag, w, h in sizes:
            kind = "photo" if tag == "blocks" else "noisea"
            out.append((f"{tag}_rgb{rgb24}", synth.frame_np(w * 7 + h + rgb24, w, h, kind), rgb24))
        out.append((f"alpha300x200_rgb{rgb24}", synth.frame_np(4242, 300, 200, "alpha"), rgb24))
    return out


def graphics_checker_case():
    """A transparent frame scaled and composed onto a checkerboard: (src, ow, oh, compose kwargs)."""
    from timg_b200 import rgba_u32
    return (synth.frame_np(515, 160, 100, "alpha"), 97, 61,
            dict(bg=rgba_u32(30, 60, 200), pattern=rgba_u32(200, 180, 20), pw=4, ph=3))


def c4_graphics_frames():
    return c4_frames(C4_GRAPHICS_FRAMES)

