"""Writes tests/golden/jpeg.npz: the JPEG corpus (Pillow-written files, oracle/jpeg.py files, damaged copies, the
restart-boundary sweep) with the SHA-256 of the reference STB source's canvas, the status the device must report and
the host parse's supported flag.  Needs oracle/_ref/libtimg_gif_ref.so (oracle/gif.mk).

    python tests/golden/make_jpeg_golden.py"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

import jpeg_cases as jc  # noqa: E402
import timg_b200  # noqa: E402
from oracle import gif as G  # noqa: E402



def bails(data):
    """A restart interval other than the last ends without an RSTn after it (truncated, or a marker missing): stb
    returns success there with the rest of its planes uninitialised, unless a decode error comes first."""
    info = timg_b200.jpeg_parse(data)
    ri = info["restart_interval"]
    if not ri:
        return False
    hmax, vmax = max(info["h_samp"]), max(info["v_samp"])
    if info["n_comp"] == 1:
        cx = -(-info["w"] * info["h_samp"][0] // hmax)
        cy = -(-info["h"] * info["v_samp"][0] // vmax)
        mcus = -(-cx // 8) * -(-cy // 8)
    else:
        mcus = -(-info["w"] // (8 * hmax)) * -(-info["h"] // (8 * vmax))
    n_rst, i = 0, jc.scan_start(data)
    while i < len(data) - 1:                       # RSTn markers up to the first other marker
        if data[i] == 0xFF:
            j = i + 1
            while j < len(data) and data[j] == 0xFF:
                j += 1
            if j < len(data) and 0xD0 <= data[j] <= 0xD7:
                n_rst += 1
            elif j < len(data) and data[j] != 0:
                break
            i = j + 1
            continue
        i += 1
    return n_rst < -(-mcus // ri) - 1


def main():
    assert G.have_ref(), "build oracle/_ref/libtimg_gif_ref.so first (make -C oracle -f gif.mk)"
    cases = jc.small_cases() + jc.surgery_cases() + jc.review_case() + jc.segment_sweep() + jc.writer_cases()
    names, blobs, shas, status, supported = [], [], [], [], []
    for name, data in cases:
        try:
            sup = timg_b200.jpeg_parse(data)["supported"]
        except timg_b200.B200Error:
            sup = False
        r = G.ref_stb_gif(data)
        if r is None:
            st, sha = 0, ""
        elif sup and bails(data):
            st, sha = -1, ""
        else:
            st, sha = 1, hashlib.sha256(np.ascontiguousarray(r[0][0]).tobytes()).hexdigest()
        names.append(name); blobs.append(data); shas.append(sha); status.append(st); supported.append(sup)
    offs = np.cumsum([0] + [len(b) for b in blobs]).astype(np.int64)
    np.savez_compressed(os.path.join(HERE, "jpeg.npz"), names=np.array(names), data=np.frombuffer(b"".join(blobs), np.uint8),
                        offsets=offs, sha=np.array(shas), status=np.array(status, np.int32),
                        supported=np.array(supported))
    print(f"{len(names)} files, {offs[-1]} bytes")


if __name__ == "__main__":
    main()
