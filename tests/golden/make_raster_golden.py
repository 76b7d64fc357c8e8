"""Writes tests/golden/raster.npz: for every file of tests/raster_cases.py (the corpus, the damaged headers and the RLE
tile cases), the parse outcome (1 decoded, 0 parsed only -- not taken by the device, or too large to decode here --,
-1 rejected: the reference's STB source fails), the SHA-256 of the reference's raw canvas, the status the device must
report (-1 where the canvas reads stb's uninitialised BMP palette, which is then not pinned, else 1) and, for
raster_cases.FRAME_CASES, the SHA-256 and size of the frame the reference sends at FRAME_OPTS.  Every file is rebuilt
by the code, so only these results are stored.  Needs oracle/_ref/libtimg_gif_ref.so (oracle/gif.mk).

    python tests/golden/make_raster_golden.py"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE), HERE]

import raster_cases as rc  # noqa: E402
from oracle import raster as R  # noqa: E402

# files whose canvas reads a BMP palette index at or past psize
UNINITIALISED = ("bmp8_index_past_psize", "bmp1_psize_1", "bmp8_psize_negative", "bmp8_h12_psize_negative",
                 "bmp8_h12_os2_last_entries")


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def pin(name, data, outcome):
    if outcome in ("unsupported", "big"):
        return 0, "", 0, "", 0, 0
    c = R.ref_stb(data)
    if c is None:
        return -1, "", 0, "", 0, 0
    if name in UNINITIALISED:
        return 1, "", -1, "", 0, 0
    if name not in rc.FRAME_CASES:
        return 1, sha(c), 1, "", 0, 0
    fr = R.ref_stb(data, **rc.FRAME_OPTS)
    return 1, sha(c), 1, sha(fr), fr.shape[1], fr.shape[0]


def outcome_of(name, data):
    import timg_b200
    try:
        info = timg_b200.raster_parse(data)
    except timg_b200.B200Error:
        return "einval"
    if not info["supported"]:
        return "unsupported"
    return "big" if info["w"] * info["h"] > rc.DECODED_MAX_PX else "ok"


def main():
    assert R.have_ref(), "build oracle/_ref/libtimg_gif_ref.so first (make -C oracle -f gif.mk)"
    cols = {k: [] for k in ("name", "parse", "sha", "status", "frame_sha", "frame_w", "frame_h")}
    for name, data in rc.all_files():
        for k, v in zip(cols, (name,) + pin(name, data, outcome_of(name, data))):
            cols[k].append(v)
    out = os.path.join(HERE, "raster.npz")
    np.savez_compressed(out, **{k: np.array(v) for k, v in cols.items()})
    print(f"{len(cols['name'])} cases (parse {np.unique(cols['parse'], return_counts=True)}, status "
          f"{np.unique(cols['status'], return_counts=True)}), {os.path.getsize(out)} bytes")


if __name__ == "__main__":
    main()
