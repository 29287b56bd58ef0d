"""A baseline / extended-sequential JPEG writer that works from quantised coefficients, written from ITU-T T.81 (B.2 syntax, F.1.2
Huffman encoding, C canonical codes) and not from the decoder or its oracle, so that the coefficients it is given are ground truth
for the decoder's tests.

It needs no DCT: the caller hands it per component int64 [blocks_y, blocks_x, 64] coefficients in natural order, DC absolute (the
value after DC prediction).  Everything a decoder's table and marker handling can be asked to do is a parameter: any Huffman tables
(counts, values) in any slot, any DC / AC / quantisation slot per component, 8- or 16-bit DQT, component ids, SOF0 / SOF1,
JFIF / Adobe / APPn / COM segments, DRI, fill bytes before markers, garbage before RSTn and the RSTn numbering.  `edit` rewrites a
block's symbols before they are coded, for streams no encoder writes (runs past coefficient 63, invalid codes).

write_jpeg returns (file bytes, Log).  The log holds what a decoder must produce and where every field of the stream lies:
  coefs        per component int16 [blocks_y, blocks_x, 64]: the DC running sum of each interval wrapped to int16, as libjpeg stores
               it in a JCOEF, and the AC values (valid only where `edit` left the block alone)
  intervals    unstuffed bytes per restart interval (padding included, garbage excluded)
  code_pos     bit offset of every Huffman code within its unstuffed interval; code_len, val_len its code and value lengths;
               interval its interval; is_dc whether it is a DC code
  scan_begin   file offset of the first entropy-coded byte
  stuffed      file offsets of every 0xFF that a stuffed 0x00 follows; rst: file offsets of every RSTn marker's 0xFF
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

# ZIGZAG[k] = natural (row-major) index of the k-th coefficient of the zigzag sequence (T.81 figure A.6)
ZIGZAG = []
for _s in range(15):
    _cells = [(i, _s - i) for i in range(8) if 0 <= _s - i < 8]
    ZIGZAG += [r * 8 + c for r, c in (_cells if _s % 2 else _cells[::-1])]
ZIGZAG = np.array(ZIGZAG, np.int64)

ALL_AC = [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 16)]     # EOB, ZRL and every run / size pair


@dataclass
class Comp:
    cid: int
    hs: int = 1
    vs: int = 1
    tq: int = 0
    td: int = 0
    ta: int = 0


@dataclass
class Log:
    coefs: list
    intervals: list
    code_pos: np.ndarray
    code_len: np.ndarray
    val_len: np.ndarray
    interval: np.ndarray
    is_dc: np.ndarray
    scan_begin: int = 0
    stuffed: list = field(default_factory=list)
    rst: list = field(default_factory=list)


def table(lengths: dict):
    """(counts, values) of the canonical table with the given code length per symbol, symbols of one length in ascending order."""
    counts = [0] * 16
    values = []
    for ln in range(1, 17):
        syms = sorted(s for s, l in lengths.items() if l == ln)
        counts[ln - 1] = len(syms)
        values += syms
    return counts, values


def uniform(symbols, length: int):
    """Every symbol at one code length."""
    return table({s: length for s in symbols})


def codes(counts, values):
    """{symbol: (code, length)} by T.81 C.2 (generate_code_table); a symbol listed twice keeps its first code."""
    out, code, k = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(counts[ln - 1]):
            out.setdefault(values[k], (code, ln))
            code += 1
            k += 1
        code <<= 1
    return out


def category(v: int) -> int:
    return abs(int(v)).bit_length()


def value_bits(v: int, s: int) -> int:
    """F.1.2.1: the s low-order bits of v, or of v - 1 when v is negative."""
    return (v if v >= 0 else v - 1) & ((1 << s) - 1)


def block_symbols(dc_diff: int, zz):
    """F.1.2: [('dc', s, bits), ('ac', rs, s, bits) ...] for one block, zz the 64 coefficients in zigzag order."""
    s = category(dc_diff)
    if s > 15:
        raise ValueError(f"DC difference {dc_diff} needs category {s}")
    out = [("dc", s, value_bits(dc_diff, s))]
    last = 0
    for k in np.flatnonzero(zz[1:]) + 1:
        v, run = int(zz[k]), int(k) - last - 1
        last = int(k)
        while run > 15:
            out.append(("ac", 0xF0, 0, 0))
            run -= 16
        s = category(v)
        if s > 15:
            raise ValueError(f"AC value {v} needs category {s}")
        out.append(("ac", (run << 4) | s, s, value_bits(v, s)))
    if last < 63:
        out.append(("ac", 0x00, 0, 0))
    return out


class _Bits:
    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0
        self.pos = 0

    def put(self, v: int, n: int):
        if n == 0:
            return
        self.acc = (self.acc << n) | (v & ((1 << n) - 1))
        self.n += n
        self.pos += n
        while self.n >= 8:
            self.n -= 8
            self.out.append((self.acc >> self.n) & 255)
        self.acc &= (1 << self.n) - 1

    def flush(self):
        """Pads with 1-bits to a byte boundary (F.1.2.3)."""
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)
        return bytes(self.out)


def _seg(marker: int, payload: bytes) -> bytes:
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


JFIF = (0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")


def adobe(transform: int):
    return (0xEE, b"Adobe\x00\x64\x00\x00\x00\x00" + bytes([transform]))


def _per(x, k, default):
    if x is None:
        return default
    return x(k) if callable(x) else x


def write_jpeg(h, w, comps, coefs, *, dc_tables, ac_tables, qtables, q16=(), sof=0xC0, restart=0, segments=(JFIF,),
               rst_number=None, fill_before_rst=None, garbage_before_rst=None, fill_before_eoi=0, edit=None, dht_order=None):
    """The file and its Log.

    comps: [Comp]; one component is a non-interleaved scan (one block per MCU), three an interleaved one.
    coefs: per component int64 [mcus_y * vs, mcus_x * hs, 64] in natural order (for one component [ceil(h / 8), ceil(w / 8), 64]).
    dc_tables / ac_tables: {slot: (counts, values)}, written in that order (dht_order: a list of ('dc' | 'ac', slot) instead).
    qtables: {slot: 64 values in natural order}; slots in q16 (or with a value above 255) are written with Pq = 1.
    restart: DRI in MCUs (0: none).  rst_number(k): the n of the RSTn that ends interval k (default k % 8).
    fill_before_rst / garbage_before_rst: per marker k, the number of 0xFF fill bytes / the bytes put in front of it (an int or bytes,
    or a function of k).  edit(c, by, bx, symbols) -> symbols rewrites one block's symbols; ('raw', n, bits) emits n bits as they are.
    """
    nc = len(comps)
    if nc == 1:
        mx, my, blocks = -(-w // 8), -(-h // 8), [(0, 0, 0)]
    else:
        hmax, vmax = max(c.hs for c in comps), max(c.vs for c in comps)
        mx, my = -(-w // (8 * hmax)), -(-h // (8 * vmax))
        blocks = [(ci, v, u) for ci, c in enumerate(comps) for v in range(c.vs) for u in range(c.hs)]
    for ci, c in enumerate(comps):
        want = (my, mx) if nc == 1 else (my * c.vs, mx * c.hs)
        if tuple(coefs[ci].shape[:2]) != want:
            raise ValueError(f"component {ci}: coefficients {coefs[ci].shape[:2]}, expected {want}")
    dc_codes = {k: codes(*t) for k, t in dc_tables.items()}
    ac_codes = {k: codes(*t) for k, t in ac_tables.items()}

    f = bytearray(b"\xff\xd8")
    for m, payload in segments:
        f += _seg(m, payload)
    for slot, q in qtables.items():
        q = np.asarray(q, np.int64)[ZIGZAG]
        wide = slot in q16 or int(q.max()) > 255
        f += _seg(0xDB, bytes([(16 if wide else 0) | slot]) + b"".join(int(v).to_bytes(2 if wide else 1, "big") for v in q))
    f += _seg(sof, bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([nc]) +
              b"".join(bytes([c.cid, (c.hs << 4) | c.vs, c.tq]) for c in comps))
    order = dht_order or [("dc", s) for s in dc_tables] + [("ac", s) for s in ac_tables]
    for kind, slot in order:
        counts, values = (dc_tables if kind == "dc" else ac_tables)[slot]
        f += _seg(0xC4, bytes([(16 if kind == "ac" else 0) | slot] + list(counts) + list(values)))
    if restart:
        f += _seg(0xDD, restart.to_bytes(2, "big"))
    f += _seg(0xDA, bytes([nc]) + b"".join(bytes([c.cid, (c.td << 4) | c.ta]) for c in comps) + b"\x00\x3f\x00")

    # the truth: the running sum of the DC differences within an interval is the absolute DC, which a JCOEF holds wrapped to int16
    log = Log([np.asarray(cf, np.int64).astype(np.int16) for cf in coefs], [], *[None] * 5, scan_begin=len(f))
    pos, clen, vlen, ivl, isdc = [], [], [], [], []
    n_mcu = mx * my
    ri = restart or n_mcu
    n_int = -(-n_mcu // ri)
    for k in range(n_int):
        bw = _Bits()
        pred = [0] * nc
        for mcu in range(k * ri, min(n_mcu, (k + 1) * ri)):
            my_, mx_ = divmod(mcu, mx)
            for ci, v, u in blocks:
                c = comps[ci]
                by, bx = (my_, mx_) if nc == 1 else (my_ * c.vs + v, mx_ * c.hs + u)
                cf = coefs[ci][by, bx]
                dc = int(cf[0])
                syms = block_symbols(dc - pred[ci], np.asarray(cf)[ZIGZAG])
                pred[ci] = dc
                if edit is not None:
                    syms = edit(ci, by, bx, syms)
                for sym in syms:
                    if sym[0] == "raw":
                        bw.put(sym[2], sym[1])
                        continue
                    is_dc = sym[0] == "dc"
                    code, ln = (dc_codes[c.td] if is_dc else ac_codes[c.ta])[sym[1]]
                    s, bits = (sym[1], sym[2]) if is_dc else (sym[2], sym[3])
                    pos.append(bw.pos)
                    clen.append(ln)
                    vlen.append(s)
                    ivl.append(k)
                    isdc.append(is_dc)
                    bw.put(code, ln)
                    bw.put(bits, s)
        data = bw.flush()
        log.intervals.append(len(data))
        base = len(f)
        stuffed = data.replace(b"\xff", b"\xff\x00")
        log.stuffed += [base + i for i in range(len(stuffed) - 1) if stuffed[i] == 0xFF and stuffed[i + 1] == 0]
        f += stuffed
        if k + 1 < n_int:
            g = _per(garbage_before_rst, k, b"")
            f += g if isinstance(g, (bytes, bytearray)) else bytes(g)
            f += b"\xff" * _per(fill_before_rst, k, 0)
            log.rst.append(len(f))
            f += bytes([0xFF, 0xD0 + _per(rst_number, k, k % 8)])
    f += b"\xff" * fill_before_eoi + b"\xff\xd9"
    log.code_pos, log.code_len, log.val_len = np.array(pos, np.int64), np.array(clen, np.int64), np.array(vlen, np.int64)
    log.interval, log.is_dc = np.array(ivl, np.int64), np.array(isdc, bool)
    return bytes(f), log


def grid(h, w, comps):
    """Shapes [blocks_y, blocks_x] per component that write_jpeg expects."""
    if len(comps) == 1:
        return [(-(-h // 8), -(-w // 8))]
    hmax, vmax = max(c.hs for c in comps), max(c.vs for c in comps)
    mx, my = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    return [(my * c.vs, mx * c.hs) for c in comps]
