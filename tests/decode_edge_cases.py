"""Files aimed at the places where the device decoders split their work, and a plan model that says where that is.

The PNG inflate, PNG unfilter, JPEG sync / fix-up and GIF LZW kernels decode in parallel pieces: windows of 256-bit
subsequences, row groups, 64-byte subsequences in CTAs of 128 and fix-up batches of 512, strings that lane 0 or the
warp writes.  The corpus files are small enough that their errors and stream ends only ever reach the serial paths.
Each case here names the piece it aims at; the plan model below is a small restatement of how the kernels split a
file, so a test can check that the case lands there (the kernels report no launch shape), and the constants it uses
are compared with the kernels' own constexprs.

A failure case has a clean twin the reference decodes, and the event is the only difference between them.
Case: name, fmt ("png", "jpeg", "gif"), cls (the planned class), data, twin (name of the clean twin or None),
where (the planned location: what the plan model must find), diff (what the twin check compares)."""
import collections
import functools
import os
import re

import numpy as np

import jpeg_cases as jc
import png_cases as pc
from oracle import gif as G
from oracle import png as W

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "timg_b200", "csrc")

# the kernels' split, as the plan model restates it (test_decode_edges.py compares them with the sources)
INF_T, SUB_BITS, END_GUARD, UNF_T = 512, 256, 256, 512          # png_decode.cu
SUB_BYTES, SYNC_T, FIX_T = 64, 128, 512                          # jpeg.cu
GIF_SHORT = 16                                                   # gif.cu
MODEL_CONSTANTS = {"png_decode.cu": dict(INF_T=INF_T, SUB_BITS=SUB_BITS, END_GUARD=END_GUARD, UNF_T=UNF_T),
                   "jpeg.cu": dict(SUB_BYTES=SUB_BYTES, SYNC_T=SYNC_T, FIX_T=FIX_T),
                   "gif.cu": dict(GIF_SHORT=GIF_SHORT)}

Case = collections.namedtuple("Case", "name fmt cls data twin where diff")


def kernel_constants(src):
    """name -> value of every integer constexpr in timg_b200/csrc/<src>."""
    text = open(os.path.join(CSRC, src)).read()
    return {m.group(1): int(m.group(2)) for m in re.finditer(
        r"constexpr\s+(?:unsigned\s+long\s+long|unsigned|int)\s+(\w+)\s*=\s*(\d+)(?:u?ll|u)?\s*;", text)}


# ---- PNG inflate: plan model ----------------------------------------------------------------------------------------
def png_windows(L, P0, units, stop):
    """The windows png_inflate_kernel decodes a Huffman block in: [(start bit, nact)].  L: stream bytes; P0: the bit
    after the block's header; units: the block's unit starts (absolute bits, ascending); stop: the start of the unit
    that ends the block (end-of-block or an error).  A window takes min(INF_T, room / SUB_BITS) subsequences when that
    is at least 4, room being what lies between its start and END_GUARD bits before the stream's end; the next one
    starts at the first unit boundary at or after its end; a block's rest after the last window is serial."""
    out, P = [], P0
    while True:
        room = 8 * L - END_GUARD - P if 8 * L > END_GUARD + P else 0
        nact = min(room // SUB_BITS, INF_T)
        if nact < 4:
            return out
        out.append((P, nact))
        end = P + nact * SUB_BITS
        if stop < end:
            return out
        P = next(u for u in units if u >= end)


def png_locate(windows, bit):
    """(window, subsequence, offset) of a bit, or None where the serial reader decodes it."""
    for w, (P, nact) in enumerate(windows):
        if P <= bit < P + nact * SUB_BITS:
            return w, (bit - P) // SUB_BITS, (bit - P) % SUB_BITS
    return None


class Stream:
    """A hand-made deflate stream of blocks; bits and marks are the BitWriter's, `off` the zlib header's 16 bits."""

    def __init__(self, blocks, zlib=True, pad=0):
        bw = W.BitWriter()
        for b in blocks:
            kind = b[0]
            if kind == "fixed":
                W.fixed(bw, b[1], b[2])
            elif kind == "dyn":
                W.dynamic(bw, b[1], b[2], DYN_LIT, DYN_DIST)
            else:
                W.stored(bw, b[1], b[2], n=b[3] if len(b) > 3 else None)
        self.bw, self.zlib, self.off = bw, zlib, 16 if zlib else 0
        body = bw.bytes()
        self.data = (W.zlib_wrap(body) if zlib else body) + bytes(pad)
        self.L = len(self.data)

    def block_plan(self, k, stop=None):
        """Windows of block k (stop: the unit that ends it, default its end-of-block)."""
        start, p0 = self.bw.blocks[k]
        nxt = self.bw.blocks[k + 1][0] if k + 1 < len(self.bw.blocks) else len(self.bw.bits)
        units = [m + self.off for m in self.bw.marks if p0 <= m < nxt] + [nxt + self.off]
        return png_windows(self.L, p0 + self.off, units, units[-2] if stop is None else stop)


# the dynamic block: 8-bit codes for 0..143, the end-of-block and the 29 length symbols, 9-bit codes for 144..159 --
# an incomplete code whose all-ones byte is unused; 30 distance codes of 5 bits
DYN_LIT = [8] * 144 + [9] * 16 + [0] * 96 + [8] * 30
DYN_DIST = [5] * 30


def _grey(w, h, seed):
    """Filter-0 rows of 8-bit grey samples below 144: each a fixed (and dynamic) 8-bit literal; the raw bytes."""
    img = np.random.default_rng(seed).integers(0, 144, (h, w))
    return np.concatenate([np.zeros((h, 1), np.int64), img], 1).ravel().tolist()


def _widen(ops, i, k, w):
    """ops with k literals just before index i made 9 bits long (values 144..159), filter bytes skipped: every later
    unit starts k bits later."""
    ops = list(ops)
    j = i - 1
    while k:
        if j % (w + 1):                            # a sample, not a filter byte
            ops[j] = 144 + j % 16
            k -= 1
        j -= 1
    return ops


def _png(stream, w, h, idat_sizes=None):
    s = np.zeros((h, w, 1), np.int64)
    return W.png(s, 8, 0, zdata=stream.data, cgbi=not stream.zlib, idat_sizes=idat_sizes)


INF_W, INF_H = 200, 100                            # one full window, a second of ~112 subsequences, the serial tail
PNG_EVENTS = {                                     # name -> (ops replacing the literals from the unit on, output length)
    "len286": lambda pos: ([("dsym", 286, 0)], None),
    "len287": lambda pos: ([("dsym", 287, 0)], None),
    "dist30": lambda pos: ([("dsym", 257, 30)], None),
    "dist31": lambda pos: ([("dsym", 257, 31)], None),
    "dist_far": lambda pos: ([("copy", 3, pos + 1)], 3),
    "unused_code": lambda pos: ([("bits", 0xff, 8)], None),
}


def _inflate_at(kind, event, w, t, delta, zlib=True):
    """(case, twin) with `event` at unit start P0 + SUB_BITS t + delta of window w of a 200x100 stream; t < 0 counts
    from the window's end."""
    base = _grey(INF_W, INF_H, 1)
    blk = "dyn" if event == "unused_code" else "fixed"
    twin_s = Stream([(blk, base, 1)], zlib)
    wins = twin_s.block_plan(0)
    j = twin_s.bw.marks.index(wins[w][0] - twin_s.off)      # the unit the window starts at
    rel = SUB_BITS * (t % wins[w][1]) + delta
    for _ in range(4):
        q, k = divmod(rel, 8)                      # q units from the window's start, k of them 9-bit literals
        i = j + q
        ops = _widen(base, i, k, INF_W)
        ev, n_out = PNG_EVENTS[event](i)
        ev_ops = ops[:i] + ev + ops[i + (n_out or 1):]
        s = Stream([(blk, ev_ops, 1)], zlib)
        twin = Stream([(blk, ops, 1)], zlib)
        bit = s.bw.marks[i] + s.off
        wins = s.block_plan(0, stop=bit)
        want = SUB_BITS * (t % wins[w][1]) + delta
        assert bit == wins[w][0] + rel
        if want == rel:
            break
        rel = want
    tn = f"{kind}_twin_i{i}_k{k}_{blk}{'' if zlib else '_raw'}"
    where = dict(window=w, sub=t % wins[w][1], delta=delta, bit=bit, nact=wins[w][1])
    diff = dict(bits=(s.bw.bits, twin.bw.bits), at=bit - s.off,
                same_size=n_out is not None, end=s.bw.marks[i + len(ev)] if n_out else None,
                twin_end=twin.bw.marks[i + n_out] if n_out else None)
    return (Case(f"{kind}_{event}_w{w}t{t}d{delta}{'' if zlib else '_raw'}", "png", f"png_window_{event}",
                 _png(s, INF_W, INF_H), tn, dict(where, plan=_plan_of(s, 0, bit)), diff),
            Case(tn, "png", "png_twin", _png(twin, INF_W, INF_H), None, {}, None))


def _plan_of(stream, k, stop):
    return dict(L=stream.L, blocks=stream.bw.blocks, off=stream.off, stop=stop,
                windows=stream.block_plan(k, stop))


def png_window_events():
    """Events inside a window: codes 286 / 287 and 30 / 31, a distance past the output so far, an unused code of an
    incomplete dynamic code, at subsequences 0, 1, 3, 4, 255, 510, 511 of window 0 and the first and last of window 1,
    at offsets 0, 1, 8 and 255 into them (255: the unit crosses the subsequence's end)."""
    out, twins = [], {}
    for event in PNG_EVENTS:
        for w, ts in ((0, (0, 1, 3, 4, 255, 510, 511)), (1, (0, -1))):
            for t in ts:
                for delta in (0, 1, 8, 255):
                    if t == 0 and delta == 1:
                        continue                   # no unit starts 1 bit after the one a window starts at
                    c, tw = _inflate_at("inf", event, w, t, delta)
                    out.append(c)
                    twins[tw.name] = tw
    return out + list(twins.values())


def png_threshold_cases():
    """A window needs 4 subsequences: room after the second block's header of 1023, 1024 and 1025 bits (3, 4, 4)."""
    out = []
    w, h = 16, 9
    base = _grey(w, h, 2)
    for room in (1023, 1024, 1025):
        for zlib in (True, False):
            off = 16 if zlib else 0
            # block 1: the first row; widen it so block 2's P0 = -room mod 8
            first = base[:w + 1]
            for k in range(8):
                s = Stream([("fixed", _widen(first, w + 1, k, w), 0), ("fixed", base[w + 1:], 1)], zlib)
                p0 = s.bw.blocks[1][1] + off
                if (8 * s.L - END_GUARD - p0 - room) % 8 == 0:
                    break
            pad = (room + END_GUARD + p0) // 8 - s.L
            assert pad >= 0
            s = Stream([("fixed", _widen(first, w + 1, k, w), 0), ("fixed", base[w + 1:], 1)], zlib, pad=pad)
            plan = s.block_plan(1)
            assert 8 * s.L - END_GUARD - (s.bw.blocks[1][1] + off) == room
            out.append(Case(f"inf_room{room}{'' if zlib else '_raw'}", "png", "png_window_threshold", _png(s, w, h), None,
                            dict(room=room, nact=(plan[0][1] if plan else room // SUB_BITS), windowed=bool(plan),
                                 plan=_plan_of(s, 1, None)), None))
    return out


def png_block_end_cases():
    """End-of-block at a subsequence boundary and one bit before it; blocks shorter than a subsequence inside a long
    stream; 40 one-symbol fixed blocks then a long dynamic block."""
    out = []
    base = _grey(INF_W, INF_H, 3)
    p0 = 19
    for t in (1, 300, 511):
        for delta in (0, 255):
            target = p0 + SUB_BITS * t + delta
            # block 1 holds the literals before index i (k widened), so its end-of-block starts at the target
            i, k = divmod(target - p0, 8)
            ops = _widen(base, i, k, INF_W)
            s = Stream([("fixed", ops[:i], 0), ("fixed", ops[i:], 1)])
            eob = s.bw.marks[i] + s.off
            assert eob == target
            out.append(Case(f"inf_eob_t{t}d{delta}", "png", "png_block_end", _png(s, INF_W, INF_H), None,
                            dict(window=0, sub=t, delta=delta, bit=eob, plan=_plan_of(s, 0, eob)), None))
    n = len(base)
    cuts = list(range(0, n, 20)) + [n]
    s = Stream([("fixed", base[a:b], int(b == n)) for a, b in zip(cuts, cuts[1:])])
    out.append(Case("inf_short_blocks", "png", "png_block_end", _png(s, INF_W, INF_H), None,
                    dict(blocks=len(cuts) - 1, plan=_plan_of(s, 0, None)), None))
    s = Stream([("fixed", [v], 0) for v in base[:40]] + [("dyn", base[40:], 1)])
    out.append(Case("inf_40_tiny_then_dynamic", "png", "png_block_end", _png(s, INF_W, INF_H), None,
                    dict(blocks=41, plan=_plan_of(s, 40, None)), None))
    return out


def png_stored_cases():
    """Huffman -> stored -> Huffman with the first block ending at each bit mod 8, after a window; a final stored
    block whose LEN reaches the stream's end exactly (CgBI: nothing follows) and one byte past it (stb: "read past
    buffer")."""
    out = []
    base = _grey(INF_W, INF_H, 4)
    n1, n2 = 16000, 3000
    for m in range(8):
        for k in range(8):
            ops = _widen(base, n1, k, INF_W)
            s = Stream([("fixed", ops[:n1], 0), ("stored", bytes(ops[n1:n1 + n2]), 0), ("fixed", ops[n1 + n2:], 1)])
            if (s.bw.blocks[1][0] + s.off) % 8 == m:
                break
        out.append(Case(f"inf_huff_stored_huff_end{m}", "png", "png_stored", _png(s, INF_W, INF_H), None,
                        dict(end_mod8=m, plan=_plan_of(s, 0, None)), None))
    streams = [Stream([("fixed", base[:n1], 0), ("stored", bytes(base[n1:]), 1, len(base) - n1 + extra)], zlib=False)
               for extra in (0, 1)]
    at = streams[0].bw.blocks[1][1] - 32           # the LEN and NLEN fields
    for extra, s in enumerate(streams):
        out.append(Case(f"inf_stored_{'past' if extra else 'to'}_end_raw", "png", "png_stored", _png(s, INF_W, INF_H),
                        "inf_stored_to_end_raw" if extra else None, dict(len_past_end=extra, plan=_plan_of(s, 0, None)),
                        dict(bits=(s.bw.bits, streams[0].bw.bits), at=at, same_size=True, end=at + 32, twin_end=at + 32)
                        if extra else None))
    return out


def png_end_cases():
    """The long stream cut at every bit of its last 6 bytes, raw (CgBI) and zlib-wrapped (the cut body, then the
    Adler-32): the windows hand over to the serial reader on a truncated stream."""
    out = []
    base = _grey(INF_W, INF_H, 5)
    for zlib in (True, False):
        full = Stream([("fixed", base, 1)], zlib)
        twin = f"inf_cut0{'' if zlib else '_raw'}"
        nb = len(full.bw.bits)
        for cut in range(nb - 48, nb + 1):
            s = Stream([], zlib)
            s.bw.bits = full.bw.bits[:cut]
            body = s.bw.bytes()
            s.data = (W.zlib_wrap(body) if zlib else body)
            s.L = len(s.data)
            name = f"inf_cut{nb - cut}{'' if zlib else '_raw'}"
            out.append(Case(name, "png", "png_end", _png(s, INF_W, INF_H), None if cut == nb else twin,
                            dict(cut_bits=nb - cut, windows=png_windows(s.L, 3 + full.off,
                                                                        [m + full.off for m in full.bw.marks if m < cut],
                                                                        full.bw.marks[-1] + full.off)),
                            None if cut == nb else dict(bits=(s.bw.bits, full.bw.bits), at=cut, prefix=True)))
    return out


def png_copy_cases():
    """Copy records through expand, pointer jumping and resolve: distances 1, 2, 3, 258, 32767, 32768; a copy whose
    source lies inside copies, chained across three windows; a copy crossing the image's last raw byte in a window;
    the stream in 1- and 7-byte IDATs."""
    out = []
    w, h = 256, 200                                # 51400 raw bytes: four windows
    base = _grey(w, h, 6)
    n = len(base)
    dist_rows = dict(zip((1, 2, 3, 258, 32767, 32768), range(180, 186)))
    chain = {46 * 257 + 20: 11000, 108 * 257 + 20: 62 * 257, 170 * 257 + 20: 62 * 257}   # each copies the one before
    at = {r * 257 + 30: (100, d) for d, r in dist_rows.items()}
    at.update({p: (150, d) for p, d in chain.items()})
    at[n - 10] = (258, 500)                        # runs 248 bytes past the image, then 600 more literals
    ops, p, plan_at = [], 0, {}
    while p < n:                                   # copies only inside rows: every filter byte stays a literal 0
        if p in at:
            ln, d = at[p]
            plan_at[d] = len(ops)
            ops.append(("copy", ln, d))
            p += ln
        else:
            ops.append(base[p])
            p += 1
    last = len(ops) - 1
    ops += base[1:601]
    s = Stream([("fixed", ops, 1)])
    plan = _plan_of(s, 0, None)
    out.append(Case("inf_copies", "png", "png_copy", _png(s, w, h), None,
                    dict(distances=sorted(d for d in plan_at if d in dist_rows),
                         chain_windows=[png_locate(plan["windows"], s.bw.marks[i] + s.off)[0]
                                        for i, op in enumerate(ops) if isinstance(op, tuple) and op[1] == 150],
                         last_copy=png_locate(plan["windows"], s.bw.marks[last] + s.off), plan=plan), None))
    for sizes in ((1,), (7,)):
        out.append(Case(f"inf_copies_idat{sizes[0]}", "png", "png_copy", _png(s, w, h, idat_sizes=list(sizes)), None,
                        dict(idat=sizes[0], plan=plan), None))
    return out


# ---- PNG unfilter ---------------------------------------------------------------------------------------------------
UNF_FORMATS = {                                    # name -> (colour type, depth, filter bytes)
    "grey1": (0, 1, 1), "grey8": (0, 8, 1), "pal4": (3, 4, 1), "greyalpha8": (4, 8, 2), "rgb8": (2, 8, 3),
    "rgba8": (6, 8, 4), "rgb16": (2, 16, 6), "rgba16": (6, 16, 8)}


def unfilter_rows(fb):
    """Rows per step of png_unfilter_kernel's wavefront."""
    return UNF_T // fb


def png_unfilter_cases():
    """Filter widths 1..8 at heights rows - 1, rows, rows + 1 and 2 rows + 1; all five filter types on the first and
    last row of a row group; Adam7 with passes that cross a row group; a palette index past the entries and filter
    type 5, each only in the second row group."""
    out = []
    pal = np.random.default_rng(9).integers(0, 256, (16, 3))
    for fmt, (color, depth, fb) in UNF_FORMATS.items():
        rows = unfilter_rows(fb)
        wd = 5 if depth < 8 else 3
        for h in (rows - 1, rows, rows + 1, 2 * rows + 1):
            s = W.samples(wd, h, color, depth, h + fb)
            filt = [(r * 3 + 1) % 5 for r in range(h)]
            out.append(Case(f"unf_{fmt}_h{h}", "png", "png_unfilter_height",
                            W.png(s, depth, color, 0, filt, plte=pal if color == 3 else None), None,
                            dict(fb=fb, rows=rows, groups=-(-h // rows)), None))
        h = 2 * rows + 1
        s = W.samples(wd, h, color, depth, 77 + fb)
        for ft in range(5):
            filt = [(r + ft) % 5 for r in range(h)]
            for r in (rows - 1, rows, 2 * rows - 1, 2 * rows):
                filt[r] = ft
            out.append(Case(f"unf_{fmt}_edge_filter{ft}", "png", "png_unfilter_edge_rows",
                            W.png(s, depth, color, 0, filt, plte=pal if color == 3 else None), None,
                            dict(fb=fb, rows=rows, filter=ft, at=[rows - 1, rows, 2 * rows - 1, 2 * rows]), None))
    for fmt, h in (("grey8", 1100), ("rgba16", 600), ("rgb8", 1400)):
        color, depth, fb = UNF_FORMATS[fmt]
        s = W.samples(4, h, color, depth, 5 + h)
        out.append(Case(f"unf_adam7_{fmt}_h{h}", "png", "png_unfilter_adam7", W.png(s, depth, color, 1, (4, 1, 3, 2, 0)),
                        None, dict(fb=fb, rows=unfilter_rows(fb), pass_rows=[len(range(y0, h, dy)) for _, y0, _, dy in W.ADAM7]),
                        None))
    # palette index past the entries / filter 5, only in the second row group
    rows = unfilter_rows(1)
    h = 2 * rows + 3
    p4 = W.samples(9, h, 3, 4, 31) % 8
    ok = W.png(p4, 4, 3, 0, (1, 2, 3, 4, 0), plte=pal[:8])
    out.append(Case("unf_pal_clean", "png", "png_twin", ok, None, {}, None))
    oob = p4.copy()
    oob[rows + 2, 4] = 12
    out.append(Case("unf_pal_oob_group1", "png", "png_unfilter_late_event", W.png(oob, 4, 3, 0, (1, 2, 3, 4, 0), plte=pal[:8]),
                    "unf_pal_clean", dict(fb=1, rows=rows, row=rows + 2, group=1), dict(samples=(oob, p4))))
    filt = [(1, 2, 3, 4, 0)[r % 5] for r in range(h)]
    f5 = list(filt)
    f5[rows + 5] = 5
    out.append(Case("unf_filter5_group1", "png", "png_unfilter_late_event", W.png(p4, 4, 3, 0, f5, plte=pal[:8]),
                    "unf_pal_clean", dict(fb=1, rows=rows, row=rows + 5, group=1), dict(filters=(f5, filt))))
    return out


# ---- GIF LZW --------------------------------------------------------------------------------------------------------
def gif_strings(codes, lzw_cs):
    """The plan of a raster's codes as stbi__process_gif_raster reads them: per code, (code, width, string length,
    period, kind), kind being 'clear', 'eoi', 'lit', 'entry', 'kwkwk' or 'illegal'.  The period is the distance back
    to the string's source (what the warp copy repeats): a KwKwK string runs into its own output."""
    clear = 1 << lzw_cs
    out, avail, size, old, pos, starts, lens = [], clear + 2, lzw_cs + 1, None, 0, {}, {}
    for c in codes:
        width = size
        if c == clear:
            out.append((c, width, 0, 0, "clear"))
            avail, size, old = clear + 2, lzw_cs + 1, None
            continue
        if c == clear + 1:
            out.append((c, width, 0, 0, "eoi"))
            break
        if c > avail or (old is None and c == avail):
            out.append((c, width, 0, 0, "illegal"))
            break
        if old is not None:
            if avail + 1 > 8192:
                out.append((c, width, 0, 0, "illegal"))
                break
            starts[avail], lens[avail] = old[0], old[1] + 1
            avail += 1
        if c < clear:
            n, per, kind = 1, 0, "lit"
        else:
            n, per = lens[c], pos - starts[c]
            kind = "kwkwk" if per < n else "entry"
        out.append((c, width, n, per, kind))
        if (avail & ((1 << size) - 1)) == 0 and avail <= 0x0FFF:
            size += 1
        old = (pos, n)
        pos += n
    return out


def _widths(codes, lzw_cs):
    return [p[1] for p in gif_strings(codes, lzw_cs)] + [lzw_cs + 1] * (len(codes) - len(gif_strings(codes, lzw_cs)))


def flat_run(n, value, lzw_cs=8):
    """Codes of a flat run of one index: a literal, then codes clear + 2, clear + 3, ... each a KwKwK code one
    longer than the last (string k: length k + 1, period k)."""
    clear = 1 << lzw_cs
    return [clear, value] + [clear + 2 + k for k in range(n)]


def _gif(w, h, rasters, interlace=False):
    pal = np.random.default_rng(3).integers(0, 256, (256, 3))
    return G.gif(w, h, [dict(idx=np.zeros((h, w), np.uint8), raster=r, interlace=interlace, gce=dict(delay=2))
                        for r in rasters], gpal=pal)


def _raster(codes, lzw_cs=8, end=True):
    codes = list(codes) + ([(1 << lzw_cs) + 1] if end else [])
    return G.codes(codes, lzw_cs, _widths(codes, lzw_cs))


def read_codes(raster, lzw_cs):
    """The codes of a raster (lzw_cs byte, sub-blocks, terminator), read at the widths stb reads them, up to the end
    of information."""
    i, data = 1, b""
    while raster[i]:
        data += raster[i + 1:i + 1 + raster[i]]
        i += 1 + raster[i]
    acc, nb, pos, codes = int.from_bytes(data, "little"), 8 * len(data), 0, []
    while True:
        plan = gif_strings(codes + [0], lzw_cs)
        wd = plan[-1][1]
        if pos + wd > nb:
            return codes
        c = (acc >> pos) & ((1 << wd) - 1)
        pos += wd
        if c == (1 << lzw_cs) + 1:
            return codes
        codes.append(c)


def periodic_codes(p, n, policy=G.CLEAR_START):
    """The encoder's codes for n pixels cycling through the indices 1..p: long strings whose bytes are not all equal,
    so a copy from the wrong source changes the canvas; KwKwK periods are multiples of p."""
    return read_codes(G.lzw((np.arange(n) % p + 1).astype(np.uint8), 8, policy), 8)


def _upto(codes, lzw_cs, hit):
    """codes up to and including the first whose plan entry (code, width, length, period, kind) satisfies hit."""
    plan = gif_strings(codes, lzw_cs)
    return codes[:next(i for i, e in enumerate(plan) if hit(e)) + 1]


def _area(codes, lzw_cs=8):
    return sum(e[2] for e in gif_strings(codes, lzw_cs))


@functools.lru_cache(maxsize=1)
def gif_cases():
    """Strings of 15, 16, 17, 31, 32, 33, 64 and ~3800 bytes; KwKwK periods 1..33; long strings across the end of the
    rectangle's area followed by a legal stream and by an illegal code; a full dictionary (4095, and 8191 at lzw_cs
    12); interlaced frames of height 1..17 with long strings across pass boundaries; 600 frames whose only error is in
    the last.  Long strings come from content cycling through 3 or more indices, or follow distinct literals, so the
    source of every copy matters."""
    out = []
    per3 = periodic_codes(3, 20000)
    for n in (15, 16, 17, 31, 32, 33, 64):         # ends with the first string of n bytes, then another literal
        codes = _upto(per3, 8, lambda e: e[2] == n) + [7]
        out.append(Case(f"gif_string{n}", "gif", "gif_string_length", _gif(_area(codes), 1, [_raster(codes)]), None,
                        dict(longest=n, plan=gif_strings(codes + [257], 8)), None))
    for per in (1, 2, 16, 17, 31, 33):             # ends with the first KwKwK code of period per
        if per == 1:                               # distinct literals, then a run of one index
            codes = [256, 1, 2, 3, 4, 5] + [262 + k for k in range(40)]
        else:
            codes = _upto(periodic_codes(per, 40 * per * per), 8, lambda e: e[4] == "kwkwk" and e[3] == per)
        out.append(Case(f"gif_kwkwk_period{per}", "gif", "gif_kwkwk", _gif(_area(codes), 1, [_raster(codes)]), None,
                        dict(period=per, plan=gif_strings(codes + [257], 8)), None))
    # ~3800 bytes: distinct literals, then a run through the whole 12-bit dictionary (lengths 1..3834)
    codes = [256, 1, 2, 3, 4, 5] + list(range(262, 4096))
    area = _area(codes)
    out.append(Case("gif_dict4095_long_last", "gif", "gif_full_dictionary", _gif(2048, -(-area // 2048), [_raster(codes)]),
                    None, dict(longest=4096 - 262 + 1, plan=gif_strings(codes + [257], 8)), None))
    # the encoder filling the table with period-3 strings, clearing and going on
    full = periodic_codes(3, 3 << 20)
    area = _area(full)
    out.append(Case("gif_dict4095_periodic", "gif", "gif_full_dictionary", _gif(2048, -(-area // 2048), [_raster(full)]),
                    None, dict(clears=full.count(256), plan=gif_strings(full + [257], 8)), None))
    head12 = [4096, 1, 2, 3, 4, 5]
    codes12 = head12 + [4102 + k for k in range(300)]
    codes12 = codes12 + [4102 + 299] * (8192 - 4102 - 300)        # entries to 8191, the longest strings last
    area12 = _area(codes12, 12)
    out.append(Case("gif_cs12_dict8191", "gif", "gif_full_dictionary",
                    _gif(1024, -(-area12 // 1024), [_raster(codes12, 12)]), None,
                    dict(plan=gif_strings(codes12 + [4097], 12)), None))
    over = codes12 + [4102 + 299]
    out.append(Case("gif_cs12_dict_overflow", "gif", "gif_full_dictionary",
                    _gif(1024, -(-area12 // 1024), [_raster(over, 12)]), "gif_cs12_dict8191",
                    dict(plan=gif_strings(over, 12)), dict(codes=(over, codes12 + [4097]))))
    # long strings across the end of the area: the first of >= 63 bytes has all but 44 inside; then the end, more
    # legal codes, or an illegal code
    codes = _upto(per3, 8, lambda e: e[2] >= 63)
    area = _area(codes)
    avail = 258 + len(codes) - 2
    for tail, name in (([], "eoi"), ([1, 2, 258], "legal"), ([avail + 5], "illegal")):
        cs = codes + tail
        out.append(Case(f"gif_straddle_{name}", "gif", "gif_area_end", _gif(area - 44, 1, [_raster(cs, 8, name != "illegal")]),
                        "gif_straddle_eoi" if name == "illegal" else None,
                        dict(area=area - 44, last=gif_strings(cs, 8)[-1], plan=gif_strings(cs, 8)),
                        dict(codes=(cs, codes + [257])) if name == "illegal" else None))
    # interlaced frames: a period-3 pattern whose long strings cross rows and passes
    for h in range(1, 18):
        idx = (np.arange(40 * h) % 3).reshape(h, 40).astype(np.uint8)
        f = G.gif(40, h, [dict(idx=idx, interlace=True, gce=dict(delay=2))],
                  gpal=np.random.default_rng(h).integers(0, 256, (4, 3)))
        out.append(Case(f"gif_interlaced_h{h}", "gif", "gif_interlaced", f, None, dict(h=h), None))
    # 600 frames of 8x8; the last one's raster holds an illegal code
    good = G.lzw((np.arange(64) * 5 % 7).astype(np.uint8), 8)
    bad = _raster([256, 1, 300], end=False)                                          # 300 > avail
    base, broken = _gif(8, 8, [good] * 600), _gif(8, 8, [good] * 599 + [bad])
    out.append(Case("gif_600_frames_clean", "gif", "gif_many_frames", base, None, dict(frames=600), None))
    out.append(Case("gif_600_frames_error_in_599", "gif", "gif_many_frames", broken, "gif_600_frames_clean",
                    dict(frames=600, error_frame=599), dict(bytes=(broken, base))))
    return out


# ---- JPEG -----------------------------------------------------------------------------------------------------------
def destuffed_map(data):
    """Per segment of the scan: (destuffed length, file offset of each destuffed byte)."""
    s = jc.scan_start(data)
    segs, cur, i = [], [], s
    while i < len(data):
        if data[i] == 0xFF:
            j = i + 1
            while j < len(data) and data[j] == 0xFF:
                j += 1
            if j < len(data) and data[j] == 0:
                cur.append(i)
                i = j + 1
                continue
            segs.append(cur)
            cur = []
            if j >= len(data) or not 0xD0 <= data[j] <= 0xD7:
                return segs
            i = j + 1
            continue
        cur.append(i)
        i += 1
    segs.append(cur)
    return segs


def jpeg_subsequences(lengths):
    """Subsequences of a file's segments, as jpeg.cu counts them: ceil(L / SUB_BYTES), at least 1."""
    return [max(1, -(-L // SUB_BYTES)) for L in lengths]


def jpeg_place(front, lengths, seg, off):
    """Where destuffed byte `off` of segment `seg` lands when the file follows files whose segment lengths are
    `front` (a list of lists) in one call: global subsequence, its sync CTA(s) (CTA c owns 127c - 1 .. 127c + 126),
    and the fix-up batch inside its segment."""
    g0 = sum(sum(jpeg_subsequences(f)) for f in front)
    k = g0 + sum(jpeg_subsequences(lengths)[:seg]) + off // SUB_BYTES
    ctas = [c for c in (k // (SYNC_T - 1), (k + 1) // (SYNC_T - 1)) if (SYNC_T - 1) * c - 1 <= k <= (SYNC_T - 1) * c + SYNC_T - 2]
    return dict(sub=k, local_sub=off // SUB_BYTES, cta=sorted(set(ctas)), batch=(off // SUB_BYTES) // FIX_T,
                sub_off=off % SUB_BYTES)


JPEG_BASES = {                                     # name -> Pillow arguments; a segment of more than 514 subsequences
    "b420": dict(size=(352, 272), quality=92, subsampling=2),
    "b444": dict(size=(256, 200), quality=90, subsampling=0),
    "bgrey": dict(size=(400, 320), quality=95, mode="L"),
    "b420dri": dict(size=(352, 400), quality=92, subsampling=2, restart_marker_rows=10),
}


def jpeg_base_files():
    """name -> bytes of the Pillow-written bases (stored in tests/golden/decode_edges.npz; Pillow's bytes vary)."""
    out = {}
    for name, a in JPEG_BASES.items():
        a = dict(a)
        w, h = a.pop("size")
        mode = a.pop("mode", "RGB")
        for seed in range(20, 60):                 # the first whose flip targets hold no 0xFF
            d = jc.jpeg(jc.photo(w, h, seed), mode, **a)
            segs = destuffed_map(d)
            seg = _flip_segment(name, segs)
            if all(d[segs[seg][SUB_BYTES * k + e]] != 0xFF for k in FLIP_KS for e in (-1, 0, 1)
                   if SUB_BYTES * k + 1 < len(segs[seg])):
                out[name] = d
                break
    return out


def _flip_segment(name, segs):
    """The longest segment; the first of a DRI file (its subsequences are then numbered from 0 in a call of its own)."""
    return 0 if "dri" in name else max(range(len(segs)), key=lambda i: len(segs[i]))


FLIP_KS = (126, 127, 128, 253, 254, 511, 512, 513)


CTA_KS, FIX_KS = (126, 127, 128, 253, 254), (511, 512, 513)
FRONT_AIMS = (0, 1, 2, 5)                          # front files a case is aimed behind


def _aims(fronts, length):
    """(k, n, local k): k counted globally behind the first n front files, for the sync-CTA edges (every n) and the
    fix-up-batch edges (which do not move: n = 0), wherever the segment holds it."""
    g0 = [sum(sum(jpeg_subsequences([len(s) for s in destuffed_map(f)])) for f in fronts[:n]) for n in FRONT_AIMS]
    out = [(k, n, k - g) for k in CTA_KS for n, g in zip(FRONT_AIMS, g0)] + [(k, 0, k) for k in FIX_KS]
    return [(k, n, lk) for k, n, lk in out if 1 <= lk and SUB_BYTES * lk + 8 < length]


def ff_run(data, segs, seg, off, n=6):
    """The file with destuffed bytes off .. off + n of a segment replaced by 0xFF (written FF 00): 48 one bits, which
    no code of a JPEG Huffman table may be, in place of the same number of scan bytes."""
    last = segs[seg][off + n - 1]
    end = last + (2 if data[last] == 0xFF else 1)
    return data[:segs[seg][off]] + b"\xff\x00" * n + data[end:]


def jpeg_cases(bases, fronts):
    """On 4:2:0, 4:4:4, grey and DRI bases, at destuffed offsets 64k - 1, 64k and 64k + 1 of the first (or longest)
    segment, with k at the sync CTAs' edges counted globally behind 0, 1, 2 and 5 front files, and at the fix-up
    batches' edges: bit flips that make or remove no 0xFF, 48-bit runs of ones (a Huffman error: status 0), and cuts
    so the segment ends at 64k + 0..3.  In the DRI base, a restart bail (a dropped RST) before and after a Huffman
    error in another segment; in a file written with a DC quantiser that overflows a short, a DC overflow before and
    after a Huffman error in another sync CTA."""
    out = []
    for bname, data in bases.items():
        segs = destuffed_map(data)
        lengths = [len(s) for s in segs]
        seg = _flip_segment(bname, segs)
        out.append(Case(f"j_{bname}", "jpeg", "jpeg_twin", data, None, dict(lengths=lengths), None))
        for k, n, lk in _aims(fronts, lengths[seg]):
            tag = f"k{k}" + (f"_f{n}" if n else "")
            for d in (-1, 0, 1):
                off = SUB_BYTES * lk + d
                where = dict(seg=seg, off=off, k=k, front=n, d=d, **jpeg_place([], lengths, seg, off))
                e = ff_run(data, segs, seg, off)
                out.append(Case(f"j_{bname}_ones_{tag}{d:+d}", "jpeg", "jpeg_huffman_error", e, f"j_{bname}", where,
                                dict(bytes=(e, data), at=segs[seg][off], destuffed=(seg, off, 6))))
                # no flips in the DRI base: a flip there can end an interval's decode short of its RST, where stb
                # returns success with the rest of the canvas unset, and no file-level rule tells that apart
                fo = segs[seg][off]
                if "dri" in bname or data[fo] == 0xFF:
                    continue
                b = bytearray(data)
                b[fo] ^= next(m for m in (0x10, 0x04, 0x40, 0x01) if (b[fo] ^ m) != 0xFF)
                out.append(Case(f"j_{bname}_flip_{tag}{d:+d}", "jpeg", "jpeg_flip", bytes(b), f"j_{bname}", where,
                                dict(bytes=(bytes(b), data), at=fo, same_size=True)))
            if n in (0, 5):
                for j in range(4):
                    off = SUB_BYTES * lk + j
                    fo = segs[seg][off]
                    out.append(Case(f"j_{bname}_cut_{tag}+{j}", "jpeg", "jpeg_cut", data[:fo], f"j_{bname}",
                                    dict(seg=seg, end=off, off=off, k=k, front=n, d=j,
                                         **jpeg_place([], lengths, seg, off)),
                                    dict(bytes=(data[:fo], data), at=fo, prefix=True)))
    out += _restart_order_cases(bases["b420dri"])
    out += _dc_order_cases()
    return out


def _restart_order_cases(data):
    """A restart bail (RST 0 dropped: stb returns success, status -1) before a Huffman error in segment 2, and a
    Huffman error in segment 0 before a bail at RST 1 (status 0)."""
    from oracle import jpeg as JW
    segs = destuffed_map(data)
    lengths = [len(s) for s in segs]
    out = []
    off0, off2 = SUB_BYTES * 127, SUB_BYTES * 127
    err0, err2 = ff_run(data, segs, 0, off0), ff_run(data, segs, 2, off2)
    out.append(Case("j_dri_drop_rst0", "jpeg", "jpeg_restart_order", JW.drop_rst(data, 0), "j_b420dri",
                    dict(events=["bail0"]), dict(rst=(JW.drop_rst(data, 0), data))))
    out.append(Case("j_dri_bail0_then_error_seg2", "jpeg", "jpeg_restart_order", JW.drop_rst(err2, 0), None,
                    dict(events=["bail0", "error2"], error=jpeg_place([], lengths, 2, off2)), None))
    out.append(Case("j_dri_error_seg0_then_bail1", "jpeg", "jpeg_restart_order", JW.drop_rst(err0, 1), None,
                    dict(events=["error0", "bail1"], error=jpeg_place([], lengths, 0, off0)), None))
    dup = _dup_rst(data, 1)
    out.append(Case("j_dri_dup_rst1", "jpeg", "jpeg_restart_order", dup, "j_b420dri", dict(events=["dup1"]),
                    dict(rst=(dup, data))))
    return out


def _dup_rst(data, k):
    """The file with its k-th restart marker written twice."""
    i, seen = jc.scan_start(data), 0
    while True:
        i = data.index(b"\xff", i)
        if 0xD0 <= data[i + 1] <= 0xD7:
            if seen == k:
                return data[:i + 2] + data[i:]
            seen += 1
        i += 2


DC_W, DC_H = 512, 256


def _dc_planes(bright=None):
    """Mid-grey plus noise (every block's DC small) and, if given, one white 8x8 block whose DC overflows a short
    once multiplied by the declared quantiser."""
    img = (128 + np.random.default_rng(41).integers(-24, 25, (DC_H, DC_W))).astype(np.uint8)
    if bright is not None:
        by, bx = divmod(bright, DC_W // 8)
        img[8 * by:8 * by + 8, 8 * bx:8 * bx + 8] = 255
    return img


def _dc_file(bright=None):
    from oracle import jpeg as JW
    return JW.write([_dc_planes(bright)], [(1, 1)], DC_W, DC_H, quant=[np.ones(64, np.int64)],
                    declared_quant=[np.full(64, 200, np.int64)], dqt16=True)


def _dc_order_cases():
    """A DC overflow (quantised with 1, declared 200) in an early sync CTA before a Huffman error in a later one, and
    the reverse; with each event alone against the clean file."""
    clean = _dc_file()
    segs = destuffed_map(clean)
    n_blocks = (DC_W // 8) * (DC_H // 8)
    out = [Case("j_dc_clean", "jpeg", "jpeg_twin", clean, None, dict(lengths=[len(segs[0])]), None)]
    for bname, bright, err_k in (("early", n_blocks // 12, 254), ("late", n_blocks - 40, 127)):
        f = _dc_file(bright)
        fs = destuffed_map(f)
        # the writer's tables follow the file's statistics, so the scans differ from the start; the blocks are alike,
        # so the white block's bytes lie near its share of the scan
        dc_off = len(fs[0]) * bright // n_blocks
        dc_at = jpeg_place([], [len(fs[0])], 0, dc_off)
        err_off = SUB_BYTES * err_k
        both = ff_run(f, fs, 0, err_off)
        err_at = jpeg_place([], [len(fs[0])], 0, err_off)
        out.append(Case(f"j_dc_overflow_{bname}", "jpeg", "jpeg_dc_order", f, "j_dc_clean",
                        dict(events=["dc"], dc=dc_at), dict(samples=(_dc_planes(bright), _dc_planes()))))
        order = ["dc", "error"] if dc_off < err_off else ["error", "dc"]
        out.append(Case(f"j_dc_overflow_{bname}_error_k{err_k}", "jpeg", "jpeg_dc_order", both, None,
                        dict(events=order, dc=dc_at, error=err_at), None))
    return out


def front_files():
    """Clean files placed in front of a case, with odd subsequence counts (the stored ones; Pillow's bytes vary):
    they move JPEG's call-global subsequence index, so every CTA boundary moves; PNG and GIF files are independent."""
    return golden_fronts()


def make_front_files():
    out = []
    for seed in range(40):
        d = jc.jpeg(jc.photo(48 + seed * 7, 40 + seed * 3, 100 + seed), quality=80, subsampling=2)
        if sum(jpeg_subsequences([len(s) for s in destuffed_map(d)])) % 2:
            out.append(d)
        if len(out) == 5:
            return out
    raise AssertionError("no five front files with odd subsequence counts")


@functools.lru_cache(maxsize=1)
def png_cases():
    return (png_window_events() + png_threshold_cases() + png_block_end_cases() + png_stored_cases() + png_end_cases()
            + png_copy_cases() + png_unfilter_cases())


@functools.lru_cache(maxsize=1)
def png_front_files():
    return [pc.pillow(pc.photo(23 + 4 * k, 17 + 2 * k, 50 + k), "RGB") for k in range(5)]


def all_cases(bases=None, fronts=None):
    """Every case; bases, fronts: the JPEG base and front files (default: the stored ones)."""
    return (png_cases() + jpeg_cases(bases if bases is not None else golden_bases(),
                                     fronts if fronts is not None else golden_fronts()) + gif_cases())


def golden_path():
    return os.path.join(HERE, "golden", "decode_edges.npz")


@functools.lru_cache(maxsize=1)
def golden():
    z = np.load(golden_path())
    return {str(n): (int(s), str(h)) for n, s, h in zip(z["names"], z["status"], z["sha"])}


@functools.lru_cache(maxsize=1)
def golden_bases():
    z = np.load(golden_path())
    return {k[5:]: z[k].tobytes() for k in z.files if k.startswith("base/")}


@functools.lru_cache(maxsize=1)
def golden_fronts():
    z = np.load(golden_path())
    return [z[f"front/{i}"].tobytes() for i in range(5)]
