"""Regenerates tests/golden/*.npz from the reference itself (oracle/_ref/libtimg_ref.so, i.e. the
UNMODIFIED timg translation units compiled by oracle/Makefile, which needs the reference's sources):
    python tests/golden/make_golden.py

Inputs are not stored: tests/cases.py regenerates them deterministically.  Outputs are stored
in full (zip-compressed), keyed by case name, except the large ones of reference.npz (digests).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import oracle  # noqa: E402
import cases  # noqa: E402


def main():
    blocks = {}
    for name, case in cases.block_cases():
        outs = cases.run_block_case(lambda q, u, c: oracle.RefBlockCanvas(q, u, c), case)
        for i, o in enumerate(outs):
            blocks[f"{name}/{i}"] = np.frombuffer(o, np.uint8)
    np.savez_compressed(os.path.join(HERE, "blocks.npz"), **blocks)
    comp = {}
    for name, fb, kw in cases.compose_cases():
        comp[name] = oracle.ref_compose_bg(fb, **kw)
    np.savez_compressed(os.path.join(HERE, "compose.npz"), **comp)
    sc = {}
    for name, img, ow, oh, fmt in cases.scale_cases():
        sc[name] = oracle.ref_scale(img, ow, oh, fmt)
    np.savez_compressed(os.path.join(HERE, "scale.npz"), **sc)
    fit = []
    rng = np.random.default_rng(5)
    for _ in range(400):
        iw, ih = int(rng.integers(1, 5000)), int(rng.integers(1, 5000))
        width, height = int(rng.integers(1, 3000)), int(rng.integers(1, 3000))
        cx, cy = [(1, 2), (2, 2), (9, 18), (1, 1)][int(rng.integers(0, 4))]
        st = float(np.float32([1.0, 0.5, 2.0, 0.1, 7.0, 1.0, 0.8889][int(rng.integers(0, 7))]))
        fl = [int(v) for v in rng.integers(0, 2, 5)]
        args = (iw, ih, width, height, cx, cy, st, *fl)
        r = oracle.calc_fit(iw, ih, width, height, cx, cy, st, *map(bool, fl), impl=oracle.ref().ref_calc_fit)
        fit.append(list(args) + [int(r[0]), r[1], r[2]])
    np.savez_compressed(os.path.join(HERE, "fit.npz"), rows=np.array(fit, np.float64))
    total = sum(os.path.getsize(os.path.join(HERE, f)) for f in os.listdir(HERE) if f.endswith(".npz"))
    print(f"wrote {len(blocks)} block outputs, {len(comp)} compose outputs, {len(fit)} fit rows; {total} bytes")
    reference()


def reference():
    """reference.npz: what the tests that once called the reference directly compare against.  Small outputs
    are stored in full; frames and canvases of the config geometries as SHA-256 digests (cases.sha)."""
    bg = oracle.rgba_u32(0, 0, 0)
    g = {"as256": np.array([oracle.ref().ref_as256(v) for v in cases.as256_values()], np.uint8)}
    for seed in range(6):
        outs = cases.run_block_case(lambda *f: oracle.RefBlockCanvas(*f), cases.random_block_case(seed))
        for i, o in enumerate(outs):
            g[f"blocks_random/{seed}/{i}"] = np.frombuffer(o, np.uint8)
    for i, (fb, kw) in enumerate(cases.random_compose_cases()):
        g[f"compose_random/{i}"] = oracle.ref_compose_bg(fb, **kw)
    for i, (img, ow, oh, fmt) in enumerate(cases.random_scale_cases()):
        g[f"scale_random/{i}"] = cases.sha(oracle.ref_scale(img, ow, oh, fmt))
    for iw, ih, fit, kind in cases.CONFIG_GEOMETRIES:
        _, ow, oh = oracle.calc_fit(iw, ih, *fit)
        s = oracle.ref_scale(cases.config_frame(iw, ih, kind), ow, oh)
        g[f"config_scale/{iw}x{ih}-{ow}x{oh}"] = cases.sha(s)
        g[f"config_compose/{iw}x{ih}-{ow}x{oh}"] = cases.sha(oracle.ref_compose_bg(s, bg))
    for f, fr in enumerate(cases.c1_frames()):
        fb = oracle.ref_compose_bg(oracle.ref_scale(fr, 67, 50), bg)
        g[f"c1_blocks/{f}"] = cases.sha(oracle.RefBlockCanvas(False).send(fb))
    cv = oracle.RefBlockCanvas(True)
    for f, fr in enumerate(cases.c3_frames()):
        fb = oracle.ref_compose_bg(oracle.ref_scale(fr, 320, 90), bg)
        g[f"c3_blocks/{f}"] = cases.sha(cv.send(fb, 0, 0 if f == 0 else -90))
    for f, fr in enumerate(cases.c4_frames()):
        fb = np.zeros((192, 337, 4), np.uint8)                            # 337x190, padded to a multiple of 6 rows
        fb[:190] = oracle.ref_compose_bg(oracle.ref_scale(fr, 337, 190), bg)
        g[f"c4_padded/{f}"] = cases.sha(oracle.ref_compose_bg(fb, bg, start_row=190))
    g = {k: np.frombuffer(v, np.uint8) if isinstance(v, bytes) else v for k, v in g.items()}
    np.savez_compressed(os.path.join(HERE, "reference.npz"), **g)
    print(f"wrote {len(g)} reference outputs; {os.path.getsize(os.path.join(HERE, 'reference.npz'))} bytes")


if __name__ == "__main__":
    main()
