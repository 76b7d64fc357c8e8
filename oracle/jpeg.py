"""A numpy baseline JPEG writer for the files Pillow cannot produce.

write() encodes 1, 3 or 4 component planes with any sampling factors 1..4 (chroma above luma, 4:4:0, 3 and 4 included),
any component ids, JFIF and / or Adobe APP14 (transform 0, 1, 2), 8- or 16-bit DQT, SOF0 or SOF1, a restart interval
(RSTn markers, optional fill bytes before each), DNL and junk after EOI.  Huffman tables are built from the image's
own symbol counts (length-limited to 16 bits), so short codes take stb's fast paths and long ones its slow path.
Byte surgery helpers damage a file: drop_rst() removes one restart marker, second_scan() repeats the scan, truncate()
cuts the scan.  Everything is deterministic, so a seed pins a file."""
import struct

import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45,
                   38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])


def _dct_matrix():
    m = np.zeros((8, 8))
    for k in range(8):
        for n in range(8):
            m[k, n] = (np.sqrt(1 / 8) if k == 0 else np.sqrt(2 / 8)) * np.cos(np.pi * (2 * n + 1) * k / 16)
    return m


_D = _dct_matrix()


def planes_from(img, n):
    """Component planes (uint8 [h, w] each) of an RGB image: YCbCr (n = 3), grey (n = 1), CMYK-like (n = 4)."""
    f = img.astype(np.float64)
    r, g, b = f[..., 0], f[..., 1], f[..., 2]
    y = 0.299 * r + 0.587 * g + 0.114 * b
    if n == 1:
        return [y.round().clip(0, 255).astype(np.uint8)]
    cb = 128 - 0.168736 * r - 0.331264 * g + 0.5 * b
    cr = 128 + 0.5 * r - 0.418688 * g - 0.081312 * b
    ps = [y, cb, cr]
    if n == 4:
        ps.append(255 - np.maximum(np.maximum(r, g), b) * 0.5)
    return [p.round().clip(0, 255).astype(np.uint8) for p in ps]


def _bits(v):
    return 0 if v == 0 else int(abs(int(v))).bit_length()


def _code_lengths(freq):
    """Huffman code lengths (<= 16) for the symbols with nonzero counts."""
    syms = [s for s in range(256) if freq[s]]
    if len(syms) == 1:
        return {syms[0]: 1}
    import heapq
    heap = [(int(freq[s]), i, [s]) for i, s in enumerate(syms)]
    heapq.heapify(heap)
    depth = {s: 0 for s in syms}
    k = len(heap)
    while len(heap) > 1:
        a, b = heapq.heappop(heap), heapq.heappop(heap)
        for s in a[2] + b[2]:
            depth[s] += 1
        heapq.heappush(heap, (a[0] + b[0], k, a[2] + b[2]))
        k += 1
    if max(depth.values()) > 16:                   # flatten: every symbol gets 8 or 9 bits
        ln = 8 if len(syms) < 256 else 9
        depth = {s: ln for s in syms}
    return depth


def _table(freq):
    """(counts[16], values, {symbol: (code, length)}) canonical from the code lengths."""
    depth = _code_lengths(freq)
    order = sorted(depth, key=lambda s: (depth[s], s))
    counts = [0] * 16
    for s in order:
        counts[depth[s] - 1] += 1
    codes, code, prev = {}, 0, depth[order[0]]
    for i, s in enumerate(order):
        if i:
            code += 1
            code <<= depth[s] - prev
        elif depth[s] > 1:
            pass
        prev = depth[s]
        codes[s] = (code, depth[s])
    return counts, order, codes


class _Bits:
    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0

    def put(self, v, n):
        for i in range(n - 1, -1, -1):
            self.acc = (self.acc << 1) | ((v >> i) & 1)
            self.n += 1
            if self.n == 8:
                self.out.append(self.acc)
                if self.acc == 0xFF:
                    self.out.append(0)
                self.acc = self.n = 0

    def flush(self):
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)


def _seg(marker, payload):
    return bytes([0xFF, marker]) + struct.pack(">H", len(payload) + 2) + payload


def write(planes, samp, w, h, quant=None, ids=None, jfif=True, adobe=None, dqt16=False, sof1=False, restart=0,
          fill=0, dnl=False, junk=b"", qscale=1.0, declared_quant=None):
    """A baseline JPEG of w x h.  planes: full-resolution uint8 [h, w] per component (downsampled here by box
    averaging); samp: (h, v) per component.  quant: one 64-entry row-major table per component (default: flat tables
    scaled by qscale); declared_quant: tables written to the DQT instead (the coefficients stay quantised by quant),
    e.g. to make a DC overflow a short.  restart: MCUs per interval; fill: FF fill bytes before each RSTn and EOI."""
    n = len(planes)
    hmax, vmax = max(s[0] for s in samp), max(s[1] for s in samp)
    mcux, mcuy = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    if quant is None:
        base = 1 + (np.add.outer(np.arange(8), np.arange(8)) * 2 * qscale).round().astype(int)
        quant = [np.clip(base, 1, 65535 if dqt16 else 255)] * n
    quant = [np.asarray(q, dtype=np.int64).reshape(64) for q in quant]
    coefs = []
    for c in range(n):
        hc, vc = samp[c]
        fx, fy = hmax // hc, vmax // vc
        cw, ch = -(-w * hc // hmax), -(-h * vc // vmax)
        full = np.pad(planes[c].astype(np.float64), ((0, vmax * 8 * mcuy - h), (0, hmax * 8 * mcux - w)), mode="edge")
        sub = full.reshape(full.shape[0] // fy, fy, full.shape[1] // fx, fx).mean(axis=(1, 3))
        bh, bw = mcuy * vc, mcux * hc
        blocks = sub[:bh * 8, :bw * 8].reshape(bh, 8, bw, 8).transpose(0, 2, 1, 3) - 128
        d = np.einsum("ij,abjk,lk->abil", _D, blocks, _D)
        q = np.round(d.reshape(bh, bw, 64) / quant[c]).astype(np.int64)
        q = np.clip(q, -1023, 1023)
        q[..., 0] = np.clip(q[..., 0], -2047, 2047)
        coefs.append((q, (cw + 7) // 8, (ch + 7) // 8))
    # block order of the scan
    order = []
    if n == 1:
        q, bw1, bh1 = coefs[0]
        order = [(0, y, x) for y in range(bh1) for x in range(bw1)]
        per_mcu = 1
    else:
        for my in range(mcuy):
            for mx in range(mcux):
                for c in range(n):
                    for y in range(samp[c][1]):
                        for x in range(samp[c][0]):
                            order.append((c, my * samp[c][1] + y, mx * samp[c][0] + x))
        per_mcu = sum(s[0] * s[1] for s in samp)
    tabs = [min(c, 1) for c in range(n)]             # luma tables 0, chroma tables 1
    # symbols with DC prediction reset at every restart
    syms = []
    pred = [0] * n
    for i, (c, y, x) in enumerate(order):
        if restart and i and i % (restart * per_mcu) == 0:
            pred = [0] * n
            syms.append(("rst", i // (restart * per_mcu) - 1))
        zz = coefs[c][0][y, x][ZIGZAG]
        diff = int(zz[0]) - pred[c]
        pred[c] = int(zz[0])
        syms.append(("dc", c, diff))
        run = 0
        last = max([k for k in range(1, 64) if zz[k]] or [0])
        for k in range(1, last + 1):
            v = int(zz[k])
            if v == 0:
                run += 1
                continue
            while run > 15:
                syms.append(("ac", c, 0xF0, 0))
                run -= 16
            syms.append(("ac", c, (run << 4) | _bits(v), v))
            run = 0
        if last < 63:
            syms.append(("ac", c, 0x00, 0))
    nt = 2 if n > 1 else 1
    fdc, fac = np.zeros((nt, 256), np.int64), np.zeros((nt, 256), np.int64)
    for s in syms:
        if s[0] == "dc":
            fdc[tabs[s[1]], _bits(s[2])] += 1
        elif s[0] == "ac":
            fac[tabs[s[1]], s[2]] += 1
    dcs = [_table(fdc[t]) for t in range(nt)]
    acs = [_table(fac[t] if fac[t].any() else np.eye(256, dtype=np.int64)[0]) for t in range(nt)]
    bits = _Bits()
    data = bytearray()
    for s in syms:
        if s[0] == "rst":
            bits.flush()
            data += bits.out + b"\xff" * fill + bytes([0xFF, 0xD0 + s[1] % 8])
            bits.out = bytearray()
        elif s[0] == "dc":
            t = tabs[s[1]]
            nb = _bits(s[2])
            code, ln = dcs[t][2][nb]
            bits.put(code, ln)
            if nb:
                bits.put(s[2] if s[2] > 0 else s[2] + (1 << nb) - 1, nb)
        else:
            t = tabs[s[1]]
            code, ln = acs[t][2][s[2]]
            bits.put(code, ln)
            nb = s[2] & 15
            if nb:
                bits.put(s[3] if s[3] > 0 else s[3] + (1 << nb) - 1, nb)
    bits.flush()
    data += bits.out
    # headers
    ids = ids if ids is not None else list(range(1, n + 1))
    out = b"\xff\xd8"
    if jfif:
        out += _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    if adobe is not None:
        out += _seg(0xEE, b"Adobe\x00" + struct.pack(">BHHB", 100, 0, 0, adobe))
    dq = declared_quant if declared_quant is not None else quant
    for c in range(n):
        q = np.asarray(dq[c], dtype=np.int64).reshape(64)[ZIGZAG]
        if dqt16:
            out += _seg(0xDB, bytes([0x10 | c]) + b"".join(struct.pack(">H", int(v)) for v in q))
        else:
            out += _seg(0xDB, bytes([c]) + bytes(int(v) for v in q))
    out += _seg(0xC1 if sof1 else 0xC0, struct.pack(">BHHB", 8, h, w, n) +
                b"".join(bytes([ids[c], (samp[c][0] << 4) | samp[c][1], c]) for c in range(n)))
    for t in range(nt):
        for tc, tab in ((0, dcs[t]), (1, acs[t])):
            out += _seg(0xC4, bytes([(tc << 4) | t]) + bytes(tab[0]) + bytes(tab[1]))
    if restart:
        out += _seg(0xDD, struct.pack(">H", restart))
    out += _seg(0xDA, bytes([n]) + b"".join(bytes([ids[c], (tabs[c] << 4) | tabs[c]]) for c in range(n)) + b"\x00\x3f\x00")
    out += bytes(data)
    if dnl:
        out += _seg(0xDC, struct.pack(">H", h))
    return out + b"\xff" * fill + b"\xff\xd9" + junk


def scan_start(data):
    i = data.index(b"\xff\xda")
    return i + 2 + int.from_bytes(data[i + 2:i + 4], "big")


def drop_rst(data, k=0):
    """The file without its k-th restart marker."""
    s = scan_start(data)
    pos = [i for i in range(s, len(data) - 1) if data[i] == 0xFF and 0xD0 <= data[i + 1] <= 0xD7]
    i = pos[k]
    return data[:i] + data[i + 2:]


def second_scan(data):
    """The scan repeated after itself (a baseline file with two scans)."""
    i = data.index(b"\xff\xda")
    return data[:-2] + data[i:]


def truncate(data, frac):
    s = scan_start(data)
    return data[:s + int((len(data) - s) * frac)]


def photo(w, h, seed=0):
    """Smooth gradients plus noise."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    a = np.stack([x * 255 // max(1, w - 1), y * 255 // max(1, h - 1), ((x + 2 * y) * 3) % 256], -1)
    return (a + rng.integers(-24, 25, a.shape)).clip(0, 255).astype(np.uint8)
