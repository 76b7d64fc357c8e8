"""JPEG files for the device decoder's tests, written by Pillow from seeded content: baseline at 4:4:4, 4:2:2 and 4:2:0,
greyscale, CMYK (Adobe), restart markers, progressive, and byte surgery on them (truncation, flipped scan bits, a
second scan)."""
import io

import numpy as np
from PIL import Image

SUBSAMPLING = {"444": 0, "422": 1, "420": 2}


def photo(w, h, seed=0):
    """Smooth gradients plus noise: what a photo looks like to the entropy coder."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    a = np.stack([x * 255 // max(1, w - 1), y * 255 // max(1, h - 1), ((x + 2 * y) * 3) % 256], -1)
    return (a + rng.integers(-24, 25, a.shape)).clip(0, 255).astype(np.uint8)


def jpeg(img, mode="RGB", **kw):
    b = io.BytesIO()
    Image.fromarray(img).convert(mode).save(b, "JPEG", **kw)
    return b.getvalue()


def scan_start(data):
    """Offset of the first entropy-coded byte (after the SOS header)."""
    i = data.index(b"\xff\xda")
    return i + 2 + int.from_bytes(data[i + 2:i + 4], "big")


def small_cases():
    """(name, bytes): every file the device takes, at the widths that split the SSE2 / scalar colour paths."""
    out = []
    for w in (1, 7, 8, 9, 15, 16, 17, 33):
        for name, sub in SUBSAMPLING.items():
            out.append((f"w{w}_{name}", jpeg(photo(w, 11, w), quality=85, subsampling=sub)))
    out.append(("grey", jpeg(photo(37, 21, 1), "L", quality=90)))
    out.append(("cmyk", jpeg(photo(29, 19, 2), "CMYK", quality=90)))
    out.append(("q100_444", jpeg(photo(40, 24, 3), quality=100, subsampling=0)))
    out.append(("q10_420", jpeg(photo(40, 24, 4), quality=10, subsampling=2)))
    for rows in (1, 2):
        out.append((f"dri_rows{rows}_420", jpeg(photo(70, 50, 5), quality=85, subsampling=2, restart_marker_rows=rows)))
    out.append(("dri_blocks1_444", jpeg(photo(45, 20, 6), quality=85, subsampling=0, restart_marker_blocks=1)))
    out.append(("dri_blocks3_grey", jpeg(photo(45, 20, 7), "L", quality=85, restart_marker_blocks=3)))
    return out


def surgery_cases():
    """(name, bytes): damaged files; the reference decides each one's fate."""
    base = jpeg(photo(64, 48, 8), quality=85, subsampling=2)
    dri = jpeg(photo(64, 48, 9), quality=85, subsampling=2, restart_marker_rows=1)
    s0, s1 = scan_start(base), scan_start(dri)
    out = []
    for frac in (0.1, 0.5, 0.9):
        out.append((f"trunc{frac}", base[:s0 + int((len(base) - s0) * frac)]))
        out.append((f"trunc_dri{frac}", dri[:s1 + int((len(dri) - s1) * frac)]))
    out.append(("trunc_eoi", base[:-2]))
    for k, pos in enumerate((0.05, 0.3, 0.7)):
        b = bytearray(base)
        i = s0 + int((len(base) - 2 - s0) * pos)
        if b[i] != 0xff and b[i - 1] != 0xff:
            b[i] ^= 0x5a
        out.append((f"flip{k}", bytes(b)))
    out.append(("junk_after_eoi", base + b"\x00\x13\x37junk\xff"))
    return out


def sized_cases():
    """(name, bytes) at the sizes a user opens."""
    return [
        ("4k_420", jpeg(photo(3840, 2160, 10), quality=85, subsampling=2)),
        ("4096x2160_444_dri", jpeg(photo(4096, 2160, 11), quality=85, subsampling=0, restart_marker_rows=1)),
        ("1x1", jpeg(photo(1, 1, 12), quality=85)),
        ("1x8192", jpeg(photo(1, 8192, 13), quality=85, subsampling=2)),
        ("8192x1", jpeg(photo(8192, 1, 14), quality=85, subsampling=2)),
    ]


# the file of a review: 34x27 4:4:4, restart every 11 MCUs, its last segment 65 bytes long (1 mod 64)
SEG_1MOD64 = ("eNr7f+P/AwYBLzdPNwZGRgYGRiBk+H+bwZlBWkhEXERQWlxMXE5GWkHDSVtDVVUj0MrWwCkhNDUlPjQ2OqtiZmNW4YTi6NjWrW0T5i1evXZ1es"
              "Oek7uWHZ+5YvUSkCGMMnJyGsoaftrafkvyYvOWkAz+H2AQ5GCQZlBiZhRkYBJkZBZk/H+EQR7oTlZGMGCAAkYmZhZWNnYOTi5uoIKtAgxMjMzM"
              "TCzMrKwsLEDZWqA8A4sgq5CioSObcGAiu1KhiFHjxIUcyk4bD4oGXfygYpxU1MTJJSYuISmlqqauoallYmpmbmFp5ezi6ubu4ekVHBIaFh4RGZ"
              "WckpqWnpGZVVxSWlZeUVnV3NLa1t7R2TVp8pSp06bPmDlr0eIlS5ctX7Fy1abNW7Zu275j565Dh48cPXb8xMlTly5fuXrt+o2btx4+evzk6bPn"
              "L16++vjp85ev377/+PkL5C9GBmZGGMDqL2AgMDKxsDCzsIP8xchUDlIgyMKqaMgm5BjInlgorGTUyCHiNHHhxoOcysZBH0STii5yiamYPFT9CP"
              "Ia2GfEeayJLJ/BPYbw110GFgbu/7cYeJgZgVHILMhgz1AQpVd1csr76d8P/711b/KFTxvPf+++/OfUg7DplsIyYlNP+cRuiVk962B23/NNM71+"
              "1tfY3/3PIIVQeILpGlChiK72lBm7M3aGmzZdlz2favz/Qu6nfz/qd/8zLZnXFvH899GX/1IYs73ndHZBTFwXejYwpn1LV/j91+2/91+59mWbzZ"
              "ryj+LLf07guvDEuVVpQoDx/5sAyCtPsg==")


def review_case():
    import base64
    import zlib
    return [("seg_1mod64_review", zlib.decompress(base64.b64decode(SEG_1MOD64)))]


def segment_sweep():
    """Scans and restart intervals whose destuffed length is 1, 2 or 3 mod 64 (a block's DC in the last bytes)."""
    out, want = [], {1: 0, 2: 0, 3: 0}
    for seed in range(400):
        if all(v >= 3 for v in want.values()):
            break
        w, h = 20 + seed % 29, 9 + seed % 23
        kw = dict(quality=25 + seed % 60, subsampling=seed % 3)
        if seed % 2:
            kw["restart_marker_blocks"] = 3 + seed % 9
        data = jpeg(photo(w, h, seed), **kw)
        lens = _segment_lengths(data)
        hits = [m for m in (1, 2, 3) if any(L > 64 and L % 64 == m for L in lens) and want[m] < 3]
        if hits:
            want[hits[0]] += 1
            out.append((f"sweep{seed}_mod{hits[0]}", data))
    return out


def _segment_lengths(data):
    """Destuffed lengths of the scan's segments (between markers)."""
    s = scan_start(data)
    lens, cur, i = [], 0, s
    while i < len(data):
        if data[i] == 0xFF:
            j = i + 1
            while j < len(data) and data[j] == 0xFF:
                j += 1
            if j < len(data) and data[j] == 0:
                cur += 1
                i = j + 1
                continue
            lens.append(cur)
            cur = 0
            if j >= len(data) or not 0xD0 <= data[j] <= 0xD7:
                break
            i = j + 1
            continue
        cur += 1
        i += 1
    return lens


def writer_cases():
    """Files from oracle/jpeg.py: sampling factors Pillow cannot write, ids, Adobe transforms, 16-bit DQT, SOF1, DNL,
    fill bytes, junk, a DC that overflows a short, a missing RST and a second scan."""
    from oracle import jpeg as W
    img = W.photo(41, 29, 3)
    p3, p1, p4 = W.planes_from(img, 3), W.planes_from(img, 1), W.planes_from(img, 4)
    out = []
    for name, samp in {"440": [(1, 2), (1, 1), (1, 1)], "h3": [(3, 1), (1, 1), (1, 1)], "v3h3": [(3, 3), (1, 1), (1, 1)],
                       "h4v4": [(4, 4), (2, 2), (1, 1)], "chroma_above": [(1, 1), (2, 2), (2, 1)],
                       "h4v1": [(4, 1), (2, 1), (1, 1)], "v4": [(1, 4), (1, 2), (1, 1)]}.items():
        out.append((f"w_{name}", W.write(p3, samp, 41, 29)))
    out.append(("w_grey_h2v2", W.write(p1, [(2, 2)], 41, 29)))
    out.append(("w_ids_rgb", W.write([img[..., c] for c in range(3)], [(1, 1)] * 3, 41, 29, ids=[ord("R"), ord("G"), ord("B")], jfif=False)))
    for t in (0, 1, 2):
        out.append((f"w_adobe{t}_3", W.write(p3 if t else [img[..., c] for c in range(3)], [(1, 1)] * 3, 41, 29, jfif=False, adobe=t)))
        out.append((f"w_adobe{t}_4", W.write(p4, [(2, 2), (1, 1), (1, 1), (2, 2)], 41, 29, jfif=False, adobe=t)))
    out.append(("w_4comp_noadobe", W.write(p4, [(1, 1)] * 4, 41, 29)))
    out.append(("w_dqt16_sof1", W.write(p3, [(2, 2), (1, 1), (1, 1)], 41, 29, dqt16=True, sof1=True)))
    for ri in (1, 5, 7):
        out.append((f"w_dri{ri}_fill", W.write(p3, [(2, 1), (1, 1), (1, 1)], 41, 29, restart=ri, fill=ri % 3)))
    out.append(("w_dnl_junk", W.write(p3, [(2, 2), (1, 1), (1, 1)], 41, 29, dnl=True, junk=b"\x00junk\xff\xd8")))
    q1 = [np.ones(64, np.int64)] * 3
    big = [np.full(64, 200, np.int64)] * 3
    out.append(("w_dc_overflow", W.write(p3, [(1, 1)] * 3, 41, 29, quant=q1, declared_quant=big, dqt16=True)))
    rst = W.write(p3, [(1, 1)] * 3, 41, 29, restart=4)
    out.append(("w_missing_rst", W.drop_rst(rst, 1)))
    out.append(("w_second_scan", W.second_scan(W.write(p3, [(1, 1)] * 3, 41, 29))))
    out.append(("w_trunc", W.truncate(W.write(p3, [(2, 2), (1, 1), (1, 1)], 41, 29), 0.6)))
    out.append(("w_4097", W.write(W.planes_from(W.photo(4097, 9, 4), 3), [(2, 2), (1, 1), (1, 1)], 4097, 9)))
    return out


def golden():
    """The pinned corpus of tests/golden/jpeg.npz: list of (name, bytes, canvas sha256 or '', status, supported)."""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg.npz"))
    d, o = z["data"].tobytes(), z["offsets"]
    return [(str(z["names"][i]), d[o[i]:o[i + 1]], str(z["sha"][i]), int(z["status"][i]), bool(z["supported"][i]))
            for i in range(len(z["names"]))]
