"""Writes tests/golden/decode_edges.npz: for every case of tests/decode_edge_cases.py, the status the device must
report and the SHA-256 of the reference STB source's canvas (of every frame, for a GIF), plus the Pillow-written JPEG
bases the JPEG cases are cut from and the JPEG files placed in front of them (Pillow's bytes vary by version; every
other case is rebuilt by the code).  Needs
oracle/_ref/libtimg_gif_ref.so (oracle/gif.mk).

    python tests/golden/make_decode_edges_golden.py"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE), HERE]

import decode_edge_cases as E  # noqa: E402
import timg_b200  # noqa: E402
from make_jpeg_golden import bails  # noqa: E402
from make_png_golden import palette_index_unwritten  # noqa: E402
from oracle import gif as G  # noqa: E402


def reference(case):
    """(status, sha256): what the device must report for a case, from the reference's decode."""
    r = G.ref_stb_gif(case.data)
    if case.fmt == "gif":                          # the frames the reference's loop collects: their count and bytes
        frames = [] if r is None else r[0]
        return len(frames), hashlib.sha256(b"".join(np.ascontiguousarray(f).tobytes() for f in frames)).hexdigest()
    if r is None:
        return 0, ""
    if case.fmt == "png" and palette_index_unwritten(case.data):
        return -1, ""
    if case.fmt == "jpeg" and timg_b200.jpeg_parse(case.data)["supported"] and bails(case.data):
        return -1, ""
    return 1, hashlib.sha256(np.ascontiguousarray(r[0][0]).tobytes()).hexdigest()


def main():
    assert G.have_ref(), "build oracle/_ref/libtimg_gif_ref.so first (make -C oracle -f gif.mk)"
    bases, fronts = E.jpeg_base_files(), E.make_front_files()
    names, status, shas = [], [], []
    for c in E.all_cases(bases, fronts):
        st, sha = reference(c)
        names.append(c.name); status.append(st); shas.append(sha)
    np.savez_compressed(E.golden_path(), names=np.array(names), status=np.array(status, np.int32), sha=np.array(shas),
                        **{f"base/{k}": np.frombuffer(v, np.uint8) for k, v in bases.items()},
                        **{f"front/{i}": np.frombuffer(v, np.uint8) for i, v in enumerate(fronts)})
    print(f"{len(names)} cases, status counts {np.unique(status, return_counts=True)}, "
          f"{os.path.getsize(E.golden_path())} bytes")


if __name__ == "__main__":
    main()
