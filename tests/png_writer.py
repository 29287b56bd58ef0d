"""Deflate and PNG written from the specifications (RFC 1950, 1951, PNG), for streams Pillow never writes: stored, fixed and dynamic
blocks with chosen code lengths, empty stored blocks, matches at the limits of length and distance across block, row and IDAT
boundaries, streams of fixed blocks only, and a dynamic header hidden inside a block's data."""
from __future__ import annotations

import heapq
import struct
import zlib

LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289,
         16385, 24577]
DEXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


class BitWriter:
    def __init__(self):
        self.bits = []

    def put(self, v, n):
        self.bits += [(v >> i) & 1 for i in range(n)]

    def code(self, c, n):                      # Huffman codes go most significant bit first
        self.bits += [(c >> (n - 1 - i)) & 1 for i in range(n)]

    def align(self):
        self.bits += [0] * (-len(self.bits) % 8)

    def tobytes(self):
        b = self.bits + [0] * (-len(self.bits) % 8)
        return bytes(sum(b[i + k] << k for k in range(8)) for i in range(0, len(b), 8))


def canonical(lengths):
    count = [0] * 16
    for n in lengths:
        count[n] += 1
    count[0] = 0
    code, nxt = 0, [0] * 16
    for n in range(1, 16):
        code = (code + count[n - 1]) << 1
        nxt[n] = code
    codes = []
    for n in lengths:
        codes.append((nxt[n], n) if n else None)
        if n:
            nxt[n] += 1
    return codes


def huffman_lengths(freq, limit=15):
    """Code lengths of a complete code over the symbols with freq > 0 (at least two get a code), at most limit bits."""
    syms = [s for s, f in enumerate(freq) if f > 0]
    if len(syms) < 2:
        syms = (syms + [s for s in range(len(freq)) if s not in syms])[:2]
    while True:
        heap = [(max(freq[s], 1), i, [s]) for i, s in enumerate(syms)]
        heapq.heapify(heap)
        depth = [0] * len(freq)
        k = len(heap)
        while len(heap) > 1:
            f1, _, a = heapq.heappop(heap)
            f2, _, b = heapq.heappop(heap)
            for s in a + b:
                depth[s] += 1
            heapq.heappush(heap, (f1 + f2, k, a + b))
            k += 1
        if max(depth) <= limit:
            return depth
        freq = [(f + 1) // 2 if f else 0 for f in freq]     # flatten and retry


def tokens_of(data: bytes, max_dist=32768, min_len=3):
    """Greedy LZ77: a list of literal ints and (length, distance) pairs."""
    out, i, last = [], 0, {}
    while i < len(data):
        best = (0, 0)
        key = data[i:i + 3]
        if len(key) == 3 and key in last:
            for j in reversed(last[key][-8:]):
                if i - j > max_dist:
                    continue
                n = 0
                while n < 258 and i + n < len(data) and data[j + n] == data[i + n]:
                    n += 1
                if n > best[0]:
                    best = (n, i - j)
        for k in range(i, i + max(best[0], 1)):
            if k + 3 <= len(data):
                last.setdefault(data[k:k + 3], []).append(k)
        if best[0] >= min_len:
            out.append(best)
            i += best[0]
        else:
            out.append(data[i])
            i += 1
    return out


def _sym(t):
    if isinstance(t, int):
        return t, None
    length, dist = t
    ls = max(i for i in range(29) if LBASE[i] <= length)
    if length == 258:
        ls = 28
    ds = max(i for i in range(30) if DBASE[i] <= dist)
    return 257 + ls, ds


def _emit_tokens(w, tokens, lcodes, dcodes):
    for t in tokens:
        s, ds = _sym(t)
        w.code(*lcodes[s])
        if ds is not None:
            length, dist = t
            ls = s - 257
            w.put(length - LBASE[ls], LEXTRA[ls])
            w.code(*dcodes[ds])
            w.put(dist - DBASE[ds], DEXTRA[ds])
    w.code(*lcodes[256])


def stored(w, data: bytes, final: int):
    w.put(final, 1)
    w.put(0, 2)
    w.align()
    w.put(len(data), 16)
    w.put(~len(data) & 0xFFFF, 16)
    for b in data:
        w.put(b, 8)


FIXED_LENGTHS = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8


def fixed(w, tokens, final: int):
    w.put(final, 1)
    w.put(1, 2)
    _emit_tokens(w, tokens, canonical(FIXED_LENGTHS), canonical([5] * 30))


def dynamic(w, tokens, final: int, lit_lengths=None, dist_lengths=None):
    lf, df = [0] * 286, [0] * 30
    for t in tokens:
        s, ds = _sym(t)
        lf[s] += 1
        if ds is not None:
            df[ds] += 1
    lf[256] += 1
    ll = lit_lengths or huffman_lengths(lf)
    dl = dist_lengths or huffman_lengths(df)
    nlen = max(257, max(i for i, n in enumerate(ll) if n) + 1)
    ndist = max(1, max([i for i, n in enumerate(dl) if n] or [0]) + 1)
    lens = list(ll[:nlen]) + list(dl[:ndist])
    # run-length code the lengths: 16 repeats, 17 / 18 zero runs
    rl, i = [], 0
    while i < len(lens):
        n = 1
        while i + n < len(lens) and lens[i + n] == lens[i]:
            n += 1
        if lens[i] == 0 and n >= 3:
            n = min(n, 138)
            rl.append((18, n - 11, 7) if n >= 11 else (17, n - 3, 3))
        elif i > 0 and lens[i] == lens[i - 1] and n >= 3:
            n = min(n, 6)
            rl.append((16, n - 3, 2))
        else:
            n = 1
            rl.append((lens[i], 0, 0))
        i += n
    cf = [0] * 19
    for s, _, _ in rl:
        cf[s] += 1
    cl = huffman_lengths(cf, 7)
    ncode = max(4, max(k for k in range(19) if cl[CL_ORDER[k]]) + 1)
    w.put(final, 1)
    w.put(2, 2)
    w.put(nlen - 257, 5)
    w.put(ndist - 1, 5)
    w.put(ncode - 4, 4)
    for k in range(ncode):
        w.put(cl[CL_ORDER[k]], 3)
    cc = canonical(cl)
    for s, extra, nb in rl:
        w.code(*cc[s])
        w.put(extra, nb)
    _emit_tokens(w, tokens, canonical(ll[:nlen] + [0] * (286 - nlen)), canonical(list(dl[:ndist]) + [0] * (30 - ndist)))


def zlib_stream(blocks, raw: bytes, cinfo: int = 7) -> bytes:
    """blocks: a list of (kind, payload, extra kwargs) with kind 'stored' (bytes), 'fixed' or 'dynamic' (tokens); raw: the bytes they
    inflate to, for the Adler-32."""
    w = BitWriter()
    for k, (kind, payload, kw) in enumerate(blocks):
        final = int(k == len(blocks) - 1)
        {"stored": stored, "fixed": fixed, "dynamic": dynamic}[kind](w, payload, final, **kw)
    cmf = (cinfo << 4) | 8
    flg = (31 - (cmf << 8) % 31) % 31
    return bytes([cmf, flg]) + w.tobytes() + struct.pack(">I", zlib.adler32(raw))


def chunk(t: bytes, d: bytes) -> bytes:
    return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xFFFFFFFF)


def png(w, h, depth, color_type, zdata: bytes, palette: bytes = b"", extra: bytes = b"", idat_sizes=None, interlace=0) -> bytes:
    """A PNG around the zlib stream zdata, split into IDAT chunks of idat_sizes bytes (one chunk by default)."""
    out = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, color_type, 0, 0, interlace)) + extra
    if palette:
        out += chunk(b"PLTE", palette)
    i, k = 0, 0
    while i < len(zdata) or k == 0:
        n = len(zdata) - i if not idat_sizes else idat_sizes[k % len(idat_sizes)]
        out += chunk(b"IDAT", zdata[i:i + n])
        i += n
        k += 1
    return out + chunk(b"IEND", b"")
