"""Writes tests/golden/qoi.npz: for every case of tests/qoi_cases.py (the corpus and the split-point cases), the parse
outcome (1 decoded, 0 accepted but pinned by its parse only, -1 rejected: the reference's QOI source fails), the
SHA-256 of the reference's raw canvas, the status the device must report (2 for a 3-channel header with some alpha
below 255, else 1) and, for qoi_cases.FRAME_CASES, the SHA-256 and size of the frame the reference sends at FRAME_OPTS.  Every
file is rebuilt by the code, so only these results are stored.  Needs oracle/_ref/libtimg_qoi_ref.so (oracle/qoi.mk).

    python tests/golden/make_qoi_golden.py"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE), HERE]

import qoi_cases as qc  # noqa: E402
from oracle import qoi as Q  # noqa: E402


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def status_of(data, canvas):
    return 2 if data[12] == 3 and (canvas[..., 3] != 255).any() else 1


def pin(name, data, parse_only):
    if parse_only:
        return 0, "", 0, "", 0, 0
    c = Q.ref_qoi(data)
    if c is None:
        return -1, "", 0, "", 0, 0
    if name not in qc.FRAME_CASES:
        return 1, sha(c), status_of(data, c), "", 0, 0
    fr = Q.ref_qoi(data, **qc.FRAME_OPTS)
    return 1, sha(c), status_of(data, c), sha(fr), fr.shape[1], fr.shape[0]


def main():
    assert Q.have_ref(), "build oracle/_ref/libtimg_qoi_ref.so first (make -C oracle -f qoi.mk)"
    parse_only = {n for n, d, ok in qc.rejections()
                  if ok and int.from_bytes(d[4:8], "big") * int.from_bytes(d[8:12], "big") > qc.DECODED_MAX_PX}
    cols = {k: [] for k in ("name", "parse", "sha", "status", "frame_sha", "frame_w", "frame_h")}
    for name, data in qc.corpus():
        for k, v in zip(cols, (name,) + pin(name, data, name in parse_only)):
            cols[k].append(v)
    split = {k: [] for k in ("split_name", "split_sha", "split_status")}
    for name, data, _ in qc.split_cases():
        p, s, st = pin(name, data, False)[:3]
        assert p == 1, name
        split["split_name"].append(name); split["split_sha"].append(s); split["split_status"].append(st)
    out = os.path.join(HERE, "qoi.npz")
    np.savez_compressed(out, **{k: np.array(v) for k, v in cols.items()}, **{k: np.array(v) for k, v in split.items()})
    print(f"{len(cols['name'])} corpus cases (parse {np.unique(cols['parse'], return_counts=True)}, status "
          f"{np.unique(cols['status'], return_counts=True)}), {len(split['split_name'])} split cases, "
          f"{os.path.getsize(out)} bytes")


if __name__ == "__main__":
    main()
