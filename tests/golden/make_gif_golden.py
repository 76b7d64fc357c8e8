"""Regenerates tests/golden/gif.npz from the reference's own GIF decode:
    make -C oracle all && make -C oracle -f gif.mk && python tests/golden/make_gif_golden.py

oracle/gif.mk links oracle/ref_gif.cc against the UNMODIFIED STBImageSource, so every canvas pinned here is what
stbi__gif_load_next returned to the reference's own loop (LoadAndScale with a box larger than the image and no
background: stb's raw canvases).

Stored per corpus file ("c/<name>/..."): the file itself (tests/gif_cases.py writes it from fixed seeds; the stored
bytes are what the tests decode), the screen, the frames the reference collects, their delays and the SHA-256 of
those canvases back to back.  "pil/<k>/..." holds the same for four small GIFs written by a third-party encoder
(Pillow), committed as data.  "sized/<name>/..." pins the canvases of the large animations, which are not stored:
gif_cases.sized() rewrites them.
"""
import hashlib
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from oracle import gif as G  # noqa: E402
import gif_cases  # noqa: E402


def pil_gifs():
    from PIL import Image
    rng = np.random.default_rng(4242)
    out = []
    # an RGB animation quantised by Pillow, with a disposal and per-frame durations
    frames = []
    for k in range(5):
        a = np.zeros((37, 53, 3), np.uint8)
        a[..., 0] = np.linspace(0, 255, 53)[None, :]
        a[..., 1] = (np.arange(37)[:, None] * 7 + 40 * k) % 256
        a[5 + 3 * k:15 + 3 * k, 10:30] = rng.integers(0, 256, 3)
        frames.append(Image.fromarray(a))
    b = io.BytesIO()
    frames[0].save(b, "GIF", save_all=True, append_images=frames[1:], duration=[30, 40, 50, 60, 70], loop=0, disposal=2)
    out.append(b.getvalue())
    # palette frames with transparency and optimised sub-rectangles
    pal = rng.integers(0, 256, 48).tolist()
    ims = []
    for k in range(4):
        p = np.zeros((24, 32), np.uint8)
        p[4 + k:12 + k, 3 * k:3 * k + 10] = 1 + k
        im = Image.fromarray(p, "P")
        im.putpalette(pal)
        ims.append(im)
    b = io.BytesIO()
    ims[0].save(b, "GIF", save_all=True, append_images=ims[1:], transparency=0, duration=100, loop=0, disposal=1)
    out.append(b.getvalue())
    # one interlaced still
    b = io.BytesIO()
    Image.fromarray(rng.integers(0, 256, (19, 23, 3), dtype=np.uint8)).save(b, "GIF", interlace=True)
    out.append(b.getvalue())
    # a greyscale animation written without optimisation
    g = [Image.fromarray(((np.arange(16 * 16).reshape(16, 16) + 9 * k) % 256).astype(np.uint8), "L") for k in range(3)]
    b = io.BytesIO()
    g[0].save(b, "GIF", save_all=True, append_images=g[1:], optimize=False, duration=20)
    out.append(b.getvalue())
    return out


def pin(d, key, data, store_file=True):
    ref = G.ref_stb_gif(data)
    frames = ref[0] if ref is not None else []
    if store_file:
        d[f"{key}/file"] = np.frombuffer(data, np.uint8)
    d[f"{key}/n_valid"] = np.int32(len(frames))
    d[f"{key}/delays"] = np.array(ref[1][:, 4] if ref is not None else [], np.int32)
    d[f"{key}/sha"] = np.array(hashlib.sha256(b"".join(f.tobytes() for f in frames)).hexdigest())
    if frames:
        d[f"{key}/wh"] = np.array([frames[0].shape[1], frames[0].shape[0]], np.int32)


def main():
    if not G.have_ref():
        raise SystemExit(f"{G.REF_GIF_SO} not built: make -C oracle -f gif.mk (needs the reference's sources)")
    d = {}
    names = []
    for name, data in gif_cases.corpus().items():
        pin(d, f"c/{name}", data)
        names.append(name)
    d["names"] = np.array(names)
    for k, data in enumerate(pil_gifs()):
        pin(d, f"pil/{k}", data)
    d["pil_count"] = np.int32(len(pil_gifs()))
    for name in gif_cases.SIZED:
        pin(d, f"sized/{name}", gif_cases.sized(name), store_file=False)
    np.savez_compressed(os.path.join(HERE, "gif.npz"), **d)


if __name__ == "__main__":
    main()
