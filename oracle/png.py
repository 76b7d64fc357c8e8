"""PNG writer for the device decoder's tests (numpy + stdlib zlib): what Pillow does not write.

- png(): any colour type x bit depth, a filter per row (Avg and Paeth on row 0 included), Adam7, tRNS, extra chunks
  anywhere (a second PLTE, CgBI, unknown critical / ancillary chunks, APNG's acTL / fcTL / fdAT), IDATs split at any
  lengths (zero-length and one-byte IDATs included), any zlib level / strategy / window bits, data after the stream.
- Deflate bit writer (BitWriter, stored(), fixed(), dynamic()) for hand-made streams: incomplete codes, codes
  286/287 and 30/31, distances before the start, bad code-length sequences, LEN/NLEN mismatches, block type 3.
"""
import struct
import zlib

import numpy as np

SIG = b"\x89PNG\r\n\x1a\n"
ADAM7 = [(0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2)]
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}


def chunk(tag, data=b""):
    return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xffffffff)


def ihdr(w, h, depth, color, interlace=0):
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, color, 0, 0, interlace))


def pack_rows(samples, depth):
    """[h, w*channels] integer samples -> list of packed row bytes (big-endian 16-bit, MSB-first sub-byte)."""
    rows = []
    for r in samples:
        r = np.asarray(r, np.int64)
        if depth == 16:
            rows.append(r.astype(">u2").tobytes())
        elif depth == 8:
            rows.append(r.astype(np.uint8).tobytes())
        else:
            per = 8 // depth
            n = -(-len(r) // per) * per
            p = np.zeros(n, np.int64)
            p[:len(r)] = r
            p = p.reshape(-1, per)
            b = np.zeros(len(p), np.int64)
            for q in range(per):
                b |= p[:, q] << (8 - depth * (q + 1))
            rows.append(b.astype(np.uint8).tobytes())
    return rows


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(rows, bpp, filters):
    """Filter each row with filters[r % len(filters)] (0-4; other values are written as the type byte, unfiltered).
    Row 0's Up/Avg/Paeth see a zero row above, as the PNG spec and stb's first_row_filter both do."""
    out, prev = [], bytes(len(rows[0]) if rows else 0)
    for r, row in enumerate(rows):
        ft = filters[r % len(filters)]
        cur = np.frombuffer(row, np.uint8).astype(np.int64)
        up = np.frombuffer(prev, np.uint8).astype(np.int64)
        a = np.concatenate([np.zeros(min(bpp, len(cur)), np.int64), cur[:-bpp] if len(cur) > bpp else cur[:0]])
        c = np.concatenate([np.zeros(min(bpp, len(up)), np.int64), up[:-bpp] if len(up) > bpp else up[:0]])
        pred = {1: a, 2: up, 3: (a + up) >> 1, 4: _paeth(a, up, c) if len(cur) else a}.get(ft, 0)
        out.append(bytes([ft & 255]) + ((cur - pred) & 255).astype(np.uint8).tobytes())
        prev = row
    return b"".join(out)


def raw_stream(samples, depth, color, interlace=0, filters=(0,)):
    """The filtered scanlines of [h, w, channels] samples, Adam7 passes in order when interlace."""
    h, w, ch = samples.shape
    bpp = max(1, ch * depth // 8)
    if not interlace:
        return filter_rows(pack_rows(samples.reshape(h, w * ch), depth), bpp, filters)
    out = b""
    for x0, y0, dx, dy in ADAM7:
        sub = samples[y0::dy, x0::dx]
        if sub.size:
            out += filter_rows(pack_rows(sub.reshape(sub.shape[0], -1), depth), bpp, filters)
    return out


def split(data, sizes):
    """data cut into pieces of the given sizes (cycled); the last piece takes the rest."""
    out, i, k = [], 0, 0
    while i < len(data):
        n = sizes[k % len(sizes)]
        out.append(data[i:i + n])
        i += n
        k += 1
    return out or [b""]


def png(samples, depth, color, interlace=0, filters=(0,), level=6, strategy=zlib.Z_DEFAULT_STRATEGY, wbits=15,
        plte=None, trns=None, before_idat=(), after_idat=(), idat_sizes=None, zdata=None, tail=b"", cgbi=False,
        iend=True, size=None):
    """A PNG of [h, w, channels] samples.  plte: [n, 3] entries; trns: bytes of the tRNS chunk; before_idat /
    after_idat: extra (tag, data) chunks; zdata: the IDAT payload as given (else zlib of the scanlines at level,
    strategy, wbits); idat_sizes: IDAT payload sizes (cycled); tail: bytes after the zlib stream inside the IDATs;
    cgbi: a CgBI chunk first and a raw deflate stream; size: (w, h) written in IHDR instead of the samples' shape."""
    h, w = samples.shape[:2]
    if size:
        w, h = size
    if zdata is None:
        raw = raw_stream(samples, depth, color, interlace, filters)
        co = zlib.compressobj(level, zlib.DEFLATED, -wbits if cgbi else wbits, 9, strategy)
        zdata = co.compress(raw) + co.flush()
    zdata += tail
    out = SIG + (chunk(b"CgBI", b"\x50\x00\x20\x06") if cgbi else b"") + ihdr(w, h, depth, color, interlace)
    for tag, data in before_idat:
        out += chunk(tag, data)
    if plte is not None:
        out += chunk(b"PLTE", np.asarray(plte, np.uint8).tobytes())
    if trns is not None:
        out += chunk(b"tRNS", trns)
    for piece in (split(zdata, idat_sizes) if idat_sizes else [zdata]):
        out += chunk(b"IDAT", piece)
    for tag, data in after_idat:
        out += chunk(tag, data)
    return out + (chunk(b"IEND") if iend else b"")


def samples(w, h, color, depth, seed=0):
    """Seeded [h, w, channels] samples in range for the depth: gradients, flat areas and noise."""
    rng = np.random.default_rng(seed)
    ch = CHANNELS[color]
    top = (1 << depth) - 1
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([(x * 7 + y * 3 + 40 * c) for c in range(ch)], -1) % (top + 1)
    noise = rng.integers(0, top + 1, base.shape)
    flat = ((x // 5 + y // 3) % 3 == 0)[..., None]
    return np.where(flat, base, noise).astype(np.int64)


# ---- deflate bit writer ---------------------------------------------------------------------------------------------
class BitWriter:
    """Bits LSB first.  marks: the bit at which each symbol op of fixed() / dynamic() starts (the end-of-block
    included); blocks: (header bit, first symbol or stored-data bit) of each block -- so a test can place an event to
    the bit (a 7- or 9-bit fixed literal moves every later mark by one)."""
    def __init__(self):
        self.bits = []
        self.marks = []
        self.blocks = []

    def put(self, v, n):                           # n bits of v, LSB first (header fields, extra bits)
        self.bits += [(v >> i) & 1 for i in range(n)]

    def code(self, c, n):                          # a Huffman code, MSB first
        self.bits += [(c >> (n - 1 - i)) & 1 for i in range(n)]

    def align(self):
        while len(self.bits) % 8:
            self.bits.append(0)

    def bytes(self):
        return np.packbits(np.asarray(self.bits, np.uint8), bitorder="little").tobytes()


def canonical(lengths):
    """Canonical codes (code, length) for a length list (0: absent), as DEFLATE assigns them."""
    mx = max(lengths) if any(lengths) else 0
    bl = [0] * (mx + 1)
    for L in lengths:
        if L:
            bl[L] += 1
    nxt, code = [0] * (mx + 2), 0
    for b in range(1, mx + 1):
        code = (code + (bl[b - 1] if b > 1 else 0)) << 1 if b > 1 else 0
        nxt[b] = code
    out = {}
    for s, L in enumerate(lengths):
        if L:
            out[s] = (nxt[L], L)
            nxt[L] += 1
    return out


FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32
LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
             4097, 6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]


def _symbols(bw, ops, lit, dist):
    """ops: ints (literal / symbol), ('copy', length, distance) or ('sym', lit_symbol) / ('dsym', lit, dist_sym)."""
    for op in ops:
        bw.marks.append(len(bw.bits))
        if isinstance(op, int):
            bw.code(*lit[op])
        elif op[0] == "copy":
            _, ln, d = op
            k = max(i for i in range(29) if LEN_BASE[i] <= ln and (i < 28 or ln == 258))
            bw.code(*lit[257 + k])
            bw.put(ln - LEN_BASE[k], LEN_EXTRA[k])
            j = max(i for i in range(30) if DIST_BASE[i] <= d)
            bw.code(*dist[j])
            bw.put(d - DIST_BASE[j], DIST_EXTRA[j])
        elif op[0] == "dsym":                      # a length symbol followed by a raw distance symbol
            bw.code(*lit[op[1]])
            bw.code(*dist[op[2]])
        elif op[0] == "bits":
            bw.put(op[1], op[2])


def stored(bw, data, final, nlen=None, n=None):
    """A stored block; n: the LEN field if not len(data)."""
    start = len(bw.bits)
    bw.put(final, 1)
    bw.put(0, 2)
    bw.align()
    n = len(data) if n is None else n
    bw.put(n, 16)
    bw.put((n ^ 0xffff) if nlen is None else nlen, 16)
    bw.blocks.append((start, len(bw.bits)))
    for b in data:
        bw.put(b, 8)


def fixed(bw, ops, final):
    start = len(bw.bits)
    bw.put(final, 1)
    bw.put(1, 2)
    bw.blocks.append((start, len(bw.bits)))
    _symbols(bw, list(ops) + [256], canonical(FIXED_LIT), canonical(FIXED_DIST))


def dynamic(bw, ops, final, lit_lengths, dist_lengths, clen_seq=None, end=True):
    """A dynamic block whose code lengths are sent one literal code-length symbol each (a 5-bit code for all 19
    code-length symbols), unless clen_seq gives the raw code-length symbol sequence as (symbol, extra value) pairs."""
    start = len(bw.bits)
    bw.put(final, 1)
    bw.put(2, 2)
    hlit, hdist = len(lit_lengths), len(dist_lengths)
    bw.put(hlit - 257, 5)
    bw.put(hdist - 1, 5)
    bw.put(19 - 4, 4)
    for _ in range(19):
        bw.put(5, 3)
    cl = canonical([5] * 19)
    seq = clen_seq if clen_seq is not None else [(L, 0) for L in list(lit_lengths) + list(dist_lengths)]
    for sym, extra in seq:
        bw.code(*cl[sym])
        if sym == 16:
            bw.put(extra, 2)
        elif sym == 17:
            bw.put(extra, 3)
        elif sym == 18:
            bw.put(extra, 7)
    bw.blocks.append((start, len(bw.bits)))
    _symbols(bw, list(ops) + ([256] if end else []), canonical(lit_lengths), canonical(dist_lengths))


def zlib_wrap(body, adler=b"\x00\x00\x00\x01"):
    return b"\x78\x01" + body + adler
