"""PNG decode restated in pure Python and numpy, for the tests of the GPU decoder (tokenpacker_b200/png.py).

inflate() is RFC 1951 written out: it returns the inflated bytes and, per block, where it starts and ends in the stream, its type,
its output and, for every byte, the position it copies (itself for a literal), which is what the decoder's chain and second decode
produce.  unfilter() and convert() are the PNG filters and PIL's convert('RGB') of each supported mode.  Checked against zlib and
PIL by tests/test_png_host.py.  The rules PIL follows (Pillow 12):
  - 2- and 4-bit gray is scaled by 85 and 17; 1-bit gray opens as mode '1' and converts to 0 / 255;
  - a palette index past the end of PLTE gives (0, 0, 0);
  - tRNS and the alpha channel are dropped by convert('RGB'); gAMA, iCCP and sRGB are not applied;
  - IDAT CRCs are not checked; a bad Adler-32 and a filter type above 4 raise;
  - data past the last row is ignored, and missing rows are zeros (the GPU decoder reports both as a status instead).
"""
from __future__ import annotations

import struct
import zlib

import numpy as np

SIGNATURE = b"\x89PNG\r\n\x1a\n"
LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289,
         16385, 24577]
DEXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}


class Corrupt(Exception):
    """The stream is one zlib reports an error on (or one the decoder reports, such as a short stream)."""


class Unsupported(Exception):
    """A file the decoder refuses."""


class _Bits:
    def __init__(self, data: bytes, pos: int):
        self.data, self.pos, self.nbits = data, pos, 8 * len(data)

    def get(self, n: int) -> int:
        if self.pos + n > self.nbits:
            raise Corrupt("stream ends early")
        v = 0
        for i in range(n):
            q = self.pos + i
            v |= ((self.data[q >> 3] >> (q & 7)) & 1) << i
        self.pos += n
        return v


def _code(lengths):
    """{(length, code): symbol} of a canonical code, and whether it is complete / over-subscribed."""
    count = [0] * 16
    for n in lengths:
        count[n] += 1
    left = 1
    for n in range(1, 16):
        left = 2 * left - count[n]
        if left < 0:
            return None, left
    code, nxt = 0, [0] * 16
    for n in range(1, 16):
        code = (code + count[n - 1]) << 1 if n > 1 else 0
        nxt[n] = code
    table = {}
    for s, n in enumerate(lengths):
        if n:
            table[(n, nxt[n])] = s
            nxt[n] += 1
    return table, (0 if count[0] == len(lengths) else left)


def _decode(b: _Bits, table) -> int:
    code = 0
    for n in range(1, 16):
        code = (code << 1) | b.get(1)
        if (n, code) in table:
            return table[(n, code)]
    raise Corrupt("invalid code")


def _acceptable(lengths, left):
    nonzero = [n for n in lengths if n]
    return left == 0 or (left > 0 and len(nonzero) == 1 and nonzero[0] == 1)


def read_dynamic(b: _Bits):
    nlen, ndist, ncode = b.get(5) + 257, b.get(5) + 1, b.get(4) + 4
    if nlen > 286 or ndist > 30:
        raise Corrupt("too many length or distance symbols")
    cl = [0] * 19
    for i in range(ncode):
        cl[CL_ORDER[i]] = b.get(3)
    table, left = _code(cl)
    if table is None or left != 0 or not any(cl):
        raise Corrupt("invalid code lengths set")
    lens = []
    while len(lens) < nlen + ndist:
        sym = _decode(b, table)
        if sym < 16:
            lens.append(sym)
            continue
        if sym == 16:
            if not lens:
                raise Corrupt("invalid bit length repeat")
            val, rep = lens[-1], 3 + b.get(2)
        elif sym == 17:
            val, rep = 0, 3 + b.get(3)
        else:
            val, rep = 0, 11 + b.get(7)
        if len(lens) + rep > nlen + ndist:
            raise Corrupt("invalid bit length repeat")
        lens += [val] * rep
    lit, dist = lens[:nlen], lens[nlen:]
    if lit[256] == 0:
        raise Corrupt("invalid code -- missing end-of-block")
    lt, ll = _code(lit)
    dt, dl = _code(dist)
    if lt is None or not _acceptable(lit, ll):
        raise Corrupt("invalid literal/lengths set")
    if dt is None or not _acceptable(dist, dl):
        raise Corrupt("invalid distances set")
    return lt, dt


def is_dynamic_header(stream: bytes, bit: int) -> bool:
    """Does a dynamic block header zlib accepts start at bit of stream?"""
    b = _Bits(stream, bit)
    try:
        b.get(1)
        if b.get(2) != 2:
            return False
        read_dynamic(b)
        return True
    except Corrupt:
        return False


_FIXED = None


def _fixed():
    global _FIXED
    if _FIXED is None:
        lit = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
        _FIXED = (_code(lit)[0], _code([5] * 30)[0])
    return _FIXED


def inflate(zdata: bytes, window: int = 32768):
    """The zlib stream zdata inflated: (bytes, blocks, sources).  blocks: dicts of start_bit, end_bit, type, final, out_offset,
    out_bytes and matches (a list of (position, length, distance)); sources: int64 array, the position each byte copies (its own
    for a literal).  Raises Corrupt where zlib raises."""
    if len(zdata) < 2 or (zdata[0] & 15) != 8 or (zdata[0] >> 4) > 7 or ((zdata[0] << 8) | zdata[1]) % 31 or zdata[1] & 32:
        raise Unsupported("zlib header")
    b = _Bits(zdata, 16)
    out, src, blocks = bytearray(), [], []
    final = 0
    while not final:
        start = b.pos
        final, btype = b.get(1), b.get(2)
        o0 = len(out)
        matches = []
        if btype == 0:
            b.pos = (b.pos + 7) & ~7
            n, nn = b.get(16), b.get(16)
            if n != (~nn & 0xFFFF):
                raise Corrupt("invalid stored block lengths")
            if b.pos + 8 * n > b.nbits:
                raise Corrupt("stream ends early")
            p = b.pos >> 3
            for k in range(n):
                src.append(len(out))
                out.append(zdata[p + k])
            b.pos += 8 * n
        elif btype in (1, 2):
            lt, dt = _fixed() if btype == 1 else read_dynamic(b)
            while True:
                sym = _decode(b, lt)
                if sym < 256:
                    src.append(len(out))
                    out.append(sym)
                    continue
                if sym == 256:
                    break
                sym -= 257
                if sym >= 29:
                    raise Corrupt("invalid literal/length code")
                length = LBASE[sym] + b.get(LEXTRA[sym])
                ds = _decode(b, dt)
                if ds >= 30:
                    raise Corrupt("invalid distance code")
                d = DBASE[ds] + b.get(DEXTRA[ds])
                if d > len(out) or d > window:
                    raise Corrupt("invalid distance too far back")
                matches.append((len(out), length, d))
                for _ in range(length):
                    src.append(len(out) - d)
                    out.append(out[-d])
        else:
            raise Corrupt("invalid block type")
        blocks.append(dict(start_bit=start, end_bit=b.pos, type=btype, final=final, out_offset=o0, out_bytes=len(out) - o0,
                           matches=matches))
    end = (b.pos + 7) >> 3
    if end + 4 > len(zdata):
        raise Corrupt("stream ends early")
    if struct.unpack(">I", zdata[end:end + 4])[0] != zlib.adler32(bytes(out)):
        raise Corrupt("incorrect data check")
    return bytes(out), blocks, np.array(src, np.int64)


def _chunks(data: bytes):
    i = 8
    while i + 12 <= len(data):
        n = struct.unpack(">I", data[i:i + 4])[0]
        yield data[i + 4:i + 8], data[i + 8:i + 8 + n]
        if data[i + 4:i + 8] == b"IEND":
            return
        i += 12 + n


def parse(data: bytes) -> dict:
    """IHDR, PLTE and the concatenated IDAT payloads of a well-formed file within the decoder's scope (the chunk-level checks of
    the host plan are pinned against PIL by the tests; this restates only what decoding needs)."""
    if data[:8] != SIGNATURE:
        raise Unsupported("not a PNG file")
    hdr, plte, idat = None, b"", bytearray()
    for t, s in _chunks(data):
        if t == b"IHDR":
            w, h, depth, ct, _, _, interlace = struct.unpack(">IIBBBBB", s)
            hdr = dict(w=w, h=h, depth=depth, color_type=ct, interlace=interlace)
        elif t == b"PLTE":
            plte = s
        elif t == b"IDAT":
            idat += s
        elif t in (b"acTL", b"fcTL", b"fdAT"):
            raise Unsupported("animated PNG")
    if hdr is None or not idat:
        raise Unsupported("malformed")
    if hdr["depth"] == 16:
        raise Unsupported("16-bit samples")
    if hdr["interlace"]:
        raise Unsupported("interlaced PNG")
    ch = CHANNELS[hdr["color_type"]]
    bits = ch * hdr["depth"]
    hdr.update(channels=ch, row_bytes=(hdr["w"] * bits + 7) // 8, filter_bpp=max(1, bits // 8), palette=plte, stream=bytes(idat))
    hdr["raw_bytes"] = hdr["h"] * (hdr["row_bytes"] + 1)
    return hdr


def unfilter(raw: bytes, h: int, row_bytes: int, bpp: int) -> np.ndarray:
    """The filtered rows (each with its filter-type byte) to uint8 [h, row_bytes]."""
    a = np.frombuffer(raw, np.uint8)[:h * (row_bytes + 1)].reshape(h, row_bytes + 1)
    out = np.zeros((h, row_bytes), np.uint8)
    prev = np.zeros(row_bytes, np.int32)
    for y in range(h):
        t, line = int(a[y, 0]), a[y, 1:].astype(np.int32)
        if t > 4:
            raise Corrupt("unrecognized filter type")
        if t == 2:
            cur = (line + prev) & 255
        elif t == 0:
            cur = line
        else:
            cur = line.copy()
            for j in range(row_bytes):
                left = cur[j - bpp] if j >= bpp else 0
                up, ul = prev[j], (prev[j - bpp] if j >= bpp else 0)
                if t == 1:
                    pred = left
                elif t == 3:
                    pred = (left + up) >> 1
                else:
                    p = left + up - ul
                    pa, pb, pc = abs(p - left), abs(p - up), abs(p - ul)
                    pred = left if pa <= pb and pa <= pc else (up if pb <= pc else ul)
                cur[j] = (line[j] + pred) & 255
        out[y] = cur
        prev = cur
    return out


def convert(rows: np.ndarray, hdr: dict) -> np.ndarray:
    """Unfiltered rows to PIL's convert('RGB'): uint8 [h, w, 3]."""
    h, w, d, ct = hdr["h"], hdr["w"], hdr["depth"], hdr["color_type"]
    if d < 8:
        bits = np.unpackbits(rows, axis=1).reshape(h, -1)[:, :w * d].reshape(h, w, d)
        v = (bits * (1 << np.arange(d - 1, -1, -1))).sum(axis=2).astype(np.int64)
    elif ct in (0, 3, 4):
        v = rows.reshape(h, w, CHANNELS[ct])[:, :, 0].astype(np.int64)
    else:
        return np.ascontiguousarray(rows.reshape(h, w, CHANNELS[ct])[:, :, :3])
    if ct == 3:
        pal = np.zeros((256, 3), np.uint8)
        p = np.frombuffer(hdr["palette"], np.uint8).reshape(-1, 3)
        pal[:len(p)] = p
        return pal[v]
    v = v * {1: 255, 2: 85, 4: 17, 8: 1}[d]
    return np.repeat(v.astype(np.uint8)[:, :, None], 3, axis=2)


def decode(data: bytes) -> np.ndarray:
    """The file as np.array(Image.open(f).convert('RGB')) gives it, for a file whose image data is exactly h rows."""
    hdr = parse(data)
    raw, _, _ = inflate(hdr["stream"], 1 << ((hdr["stream"][0] >> 4) + 8))
    if len(raw) != hdr["raw_bytes"]:
        raise Corrupt("image data of the wrong size")
    return convert(unfilter(raw, hdr["h"], hdr["row_bytes"], hdr["filter_bpp"]), hdr)
