"""The PNG fixture matrix the decoder's tests share: Pillow-written files in every supported mode at compress_level 0-9 and with
optimize, files compressed with each zlib strategy over rows that use every filter type, sizes from 1 x 1 to 1344 wide, and the
hand-written streams of png_writer (stored, fixed and dynamic blocks, matches at their limits, fixed blocks only, a false candidate).
Everything is generated from seeds."""
from __future__ import annotations

import io
import os
import sys
import zlib

import numpy as np
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import png_writer as pw  # noqa: E402
from oracle import png_oracle as po  # noqa: E402

SIZES = [(1, 1), (1, 7), (5, 1), (3, 13), (17, 9), (64, 97), (40, 1344)]


def pil_decode(data: bytes) -> np.ndarray:
    return np.array(Image.open(io.BytesIO(data)).convert("RGB"))


def image(h, w, kind, seed):
    """uint8 [h, w, 3]: 'doc' (text-like strokes on white), 'chart' (flat bars), 'photo' (smooth gradients and noise)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    if kind == "doc":
        a = np.full((h, w), 250, np.int32)
        a[(y % 12 < 2) & (rng.random((h, w)) < 0.6)] = 20
        a[(x % 9 == 0) & (y % 12 < 8)] = 40
        return np.repeat(a[:, :, None], 3, 2).astype(np.uint8)
    if kind == "chart":
        a = np.zeros((h, w, 3), np.int32) + 255
        for k in range(6):
            x0 = k * max(w // 6, 1)
            sel = (x >= x0) & (x < x0 + max(w // 8, 1)) & (y >= h - (k + 1) * h // 7)
            a[sel] = [(40 * k) % 256, (90 * k + 30) % 256, (200 - 25 * k) % 256]
        return a.astype(np.uint8)
    a = np.stack([(x * 255) // max(w, 1), (y * 255) // max(h, 1), ((x + y) * 127) // max(w + h, 1)], 2)
    return np.clip(a + rng.integers(-12, 13, a.shape), 0, 255).astype(np.uint8)


def save(a, mode, **kw):
    b = io.BytesIO()
    im = Image.fromarray(a)
    if mode == "P":
        im = im.convert("P", palette=Image.Palette.ADAPTIVE, colors=kw.pop("colors", 256))
    elif mode != "RGB":
        im = im.convert(mode)
    im.save(b, "PNG", **kw)
    return b.getvalue()


def filtered(rows: np.ndarray, bpp: int, types) -> bytes:
    """The PNG filter of each row (types[y % len(types)]), with its filter-type byte."""
    h, n = rows.shape
    out = bytearray()
    prev = np.zeros(n, np.int32)
    for y in range(h):
        t = types[y % len(types)]
        cur = rows[y].astype(np.int32)
        left = np.concatenate([np.zeros(bpp, np.int32), cur[:-bpp]]) if n > bpp else np.zeros(n, np.int32)
        ul = np.concatenate([np.zeros(bpp, np.int32), prev[:-bpp]]) if n > bpp else np.zeros(n, np.int32)
        if t == 0:
            f = cur
        elif t == 1:
            f = cur - left
        elif t == 2:
            f = cur - prev
        elif t == 3:
            f = cur - ((left + prev) >> 1)
        else:
            p = left + prev - ul
            pa, pb, pc = np.abs(p - left), np.abs(p - prev), np.abs(p - ul)
            f = cur - np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, prev, ul))
        out.append(t)
        out += (f & 255).astype(np.uint8).tobytes()
        prev = cur
    return bytes(out)


def gray_low_depth(h, w, depth, seed, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, types=(0, 1, 2, 3, 4)):
    """Gray at 1, 2 or 4 bits (2 and 4 Pillow does not write), rows packed high bits first."""
    rng = np.random.default_rng(seed)
    v = rng.integers(0, 1 << depth, (h, w)).astype(np.uint8)
    v[:, : w // 2] = (np.arange(w // 2) % (1 << depth)).astype(np.uint8)
    bits = np.unpackbits(v[:, :, None], axis=2)[:, :, 8 - depth:].reshape(h, -1)
    rows = np.packbits(bits, axis=1)
    c = zlib.compressobj(level, zlib.DEFLATED, 15, 8, strategy)
    return pw.png(w, h, depth, 0, c.compress(filtered(rows, 1, types)) + c.flush())


def strategy_file(h, w, ct, seed, strategy, level=6, types=(0, 1, 2, 3, 4)):
    """8-bit colour type ct compressed with zlib's strategy, every filter type in turn."""
    ch = {0: 1, 2: 3, 4: 2, 6: 4}[ct]
    a = image(h, w, "photo", seed)
    rows = np.concatenate([a, a[:, :, :1]], 2)[:, :, :ch].reshape(h, w * ch)
    c = zlib.compressobj(level, zlib.DEFLATED, 15, 8, strategy)
    return pw.png(w, h, 8, ct, c.compress(filtered(rows, ch, types)) + c.flush(), idat_sizes=[977, 1, 8192])


def limits_file():
    """Matches of length 258 at distance 32768 (the window's edge) and of length 3 and 258 at distance 1 (copies that overlap
    themselves), crossing row, block and IDAT boundaries: 8191-byte gray rows, so that a row repeated four rows down lies exactly
    32768 bytes back, with a 600-byte run in row 2."""
    w, h = 8191, 9
    r = np.random.default_rng(9).integers(0, 256, (h, w)).astype(np.uint8)
    r[2, 100:700] = r[2, 99]
    r[4:] = r[:h - 4]
    rows = filtered(r, 1, (0,))
    assert 4 * (w + 1) == 32768
    toks, i = [], 0
    while i < len(rows):
        if i >= 32768 and rows[i:i + 258] == rows[i - 32768:i - 32768 + 258]:
            toks.append((258, 32768))
            i += 258
        elif i >= 1 and rows[i:i + 258] == bytes([rows[i - 1]]) * 258:
            toks.append((258, 1))
            i += 258
        elif i >= 1 and rows[i:i + 3] == bytes([rows[i - 1]]) * 3:
            toks.append((3, 1))
            i += 3
        else:
            toks.append(rows[i])
            i += 1
    k = len(toks) // 2
    return pw.png(w, h, 8, 0, pw.zlib_stream([("dynamic", toks[:k], {}), ("fixed", toks[k:], {})], rows), idat_sizes=[4099, 1, 32768])


def hand_written():
    """(name, file) of the streams png_writer writes by hand."""
    out = []
    h, w = 7, 300
    a = image(h, w, "photo", 5)[:, :, 0]
    raw = filtered(a, 1, (0, 1, 2, 3, 4))
    n = len(raw)
    out.append(("stored-fixed-dynamic", pw.png(w, h, 8, 0, pw.zlib_stream([
        ("stored", raw[:400], {}), ("stored", b"", {}),
        ("fixed", pw.tokens_of(raw[400:900]), {}), ("dynamic", pw.tokens_of(raw[900:]), {})], raw))))
    out.append(("fixed-only", pw.png(w, h, 8, 0, pw.zlib_stream(
        [("fixed", pw.tokens_of(raw[k:k + 150]), {}) for k in range(0, n, 150)], raw))))
    out.append(("limits-across-boundaries", limits_file()))
    # a valid-looking dynamic header inside a stored block's data: a false candidate the chain must not take
    wdecoy = pw.BitWriter()
    pw.dynamic(wdecoy, pw.tokens_of(raw[:200]), 0)
    decoy = wdecoy.tobytes()
    body = (decoy * 8)[: n - 10]
    raw2 = bytes([0]) + body[: w] + raw[w + 1:]
    raw2 = raw2[:n]
    out.append(("false-candidate", pw.png(w, h, 8, 0, pw.zlib_stream([("stored", raw2[:1000], {}), ("dynamic", pw.tokens_of(raw2[1000:]), {})],
                                                                     raw2))))
    # chosen code lengths: a literal code of maximal 15-bit codes
    ll = pw.huffman_lengths([1 + (s < 256) * 1000 // (1 + s) for s in range(257)] + [0] * 29, 15)
    out.append(("chosen-lengths", pw.png(w, h, 8, 0, pw.zlib_stream([("dynamic", list(raw), {"lit_lengths": ll})], raw))))
    return out


def corrupt_set():
    """(file, status) of corrupt streams the GPU tests run once each: a bad Adler-32, a filter type of 7, a distance before the
    first byte, too little data, a stream cut in half, a block of type 3, and a distance one past a 256-byte window the zlib header
    declares.  tests/test_png_sanitized_host.py runs them first."""
    good = save(image(33, 250, "photo", 7), "RGB", compress_level=6)
    hdr = po.parse(good)
    s = hdr["stream"]
    raw = zlib.decompress(s)

    def wrap(stream, **kw):
        return pw.png(hdr["w"], hdr["h"], 8, 2, stream, **kw)
    bad_adler = s[:-1] + bytes([s[-1] ^ 1])
    bad_filter = bytearray(raw)
    bad_filter[hdr["row_bytes"] + 1] = 7
    far = pw.zlib_stream([("fixed", [1, 2, (3, 5)] + list(raw[5:]), {})], raw)
    short = zlib.compress(raw[:-50])
    btype3 = s[:2] + bytes([s[2] | 6]) + s[3:]
    small_window = pw.zlib_stream([("dynamic", list(raw[:300]) + [(3, 257)] + list(raw[303:]), {})], raw, cinfo=0)
    return [(wrap(bad_adler), 8), (wrap(zlib.compress(bytes(bad_filter))), 9), (wrap(far), 4), (wrap(short), 7),
            (wrap(s[:len(s) // 2]), 6), (wrap(btype3), 1), (wrap(small_window), 4)]


def matrix():
    """(name, file) of every fixture."""
    out = []
    for (h, w) in SIZES:
        seed = h * 131 + w
        for kind in ("doc", "chart", "photo"):
            a = image(h, w, kind, seed)
            for mode in ("RGB", "L", "LA", "RGBA", "1", "P"):
                if kind != "photo" and mode in ("LA", "RGBA"):
                    continue
                out.append((f"{h}x{w}-{kind}-{mode}", save(a, mode)))
        a = image(h, w, "chart", seed)
        for bits in (1, 2, 4):
            out.append((f"{h}x{w}-P{bits}", save(a, "P", colors=1 << bits, bits=bits)))
        for depth in (1, 2, 4):
            out.append((f"{h}x{w}-gray{depth}", gray_low_depth(h, w, depth, seed)))
    a = image(33, 250, "photo", 7)
    for level in range(10):
        out.append((f"level{level}", save(a, "RGB", compress_level=level)))
    out.append(("optimize", save(a, "RGB", optimize=True)))
    out.append(("optimize-P", save(a, "P", optimize=True)))
    for name, st in (("filtered", zlib.Z_FILTERED), ("huffman", zlib.Z_HUFFMAN_ONLY), ("rle", zlib.Z_RLE), ("fixed", zlib.Z_FIXED)):
        for ct in (0, 2, 4, 6):
            out.append((f"strategy-{name}-ct{ct}", strategy_file(29, 111, ct, 3 + ct, st)))
    out += hand_written()
    return out
