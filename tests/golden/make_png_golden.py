"""Writes tests/golden/png.npz: the PNG corpus (Pillow-written files, oracle/png.py files, hand-made deflate streams,
damaged copies) with the SHA-256 of the reference STB source's canvas, the status the device must report and the host
parse's supported flag.  Needs oracle/_ref/libtimg_gif_ref.so (oracle/gif.mk).

    python tests/golden/make_png_golden.py"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

import png_cases as pc  # noqa: E402
import timg_b200  # noqa: E402
from oracle import gif as G  # noqa: E402


def palette_index_unwritten(data):
    """A palette image (colour type 3) with an index at or past every entry its PLTE chunks wrote."""
    import io
    import struct
    from PIL import Image
    pos, written, color = 8, 0, None
    while pos + 8 <= len(data):
        n, typ = struct.unpack(">I4s", data[pos:pos + 8])
        if typ == b"IHDR":
            color = data[pos + 17]
        elif typ == b"PLTE":
            written = max(written, n // 3)
        elif typ == b"IEND":
            break
        pos += 12 + n
    if color != 3:
        return False
    idx = np.asarray(Image.open(io.BytesIO(data)))  # mode P: the indices, whatever the palette holds
    return int(idx.max()) >= written


def main():
    assert G.have_ref(), "build oracle/_ref/libtimg_gif_ref.so first (make -C oracle -f gif.mk)"
    names, blobs, shas, status, supported = [], [], [], [], []
    for name, data in pc.golden_cases():
        try:
            sup = timg_b200.png_parse(data)["supported"]
        except timg_b200.B200Error:
            sup = False
        r = G.ref_stb_gif(data)
        if r is None:
            st, sha = 0, ""
        elif palette_index_unwritten(data):       # stb reads palette entries it never wrote: undefined canvas
            st, sha = -1, ""
        else:
            st, sha = 1, hashlib.sha256(np.ascontiguousarray(r[0][0]).tobytes()).hexdigest()
        names.append(name); blobs.append(data); shas.append(sha); status.append(st); supported.append(sup)
    offs = np.cumsum([0] + [len(b) for b in blobs]).astype(np.int64)
    np.savez_compressed(os.path.join(HERE, "png.npz"), names=np.array(names), data=np.frombuffer(b"".join(blobs), np.uint8),
                        offsets=offs, sha=np.array(shas), status=np.array(status, np.int32),
                        supported=np.array(supported))
    print(f"{len(names)} files, {offs[-1]} bytes, status counts {np.unique(status, return_counts=True)}")


if __name__ == "__main__":
    main()
