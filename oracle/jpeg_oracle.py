"""numpy restatement of the baseline JPEG decode that PIL runs (libjpeg-turbo with PIL's defaults: JDCT_ISLOW, fancy upsampling,
no merged upsampling), integer arithmetic throughout, so that it equals ``np.array(Image.open(f).convert('RGB'))`` bit for bit.

Scope as tokenpacker_b200.jpeg: SOF0 / SOF1, 8-bit, one scan with 1 component or 3 interleaved YCbCr components at 4:4:4, 4:2:2 or
4:2:0, Huffman coding, restart intervals.  The stages are exposed one by one for the GPU stage tests:
  parse(data)        -> header dict (frame, tables, scan byte range, MCU geometry)
  coefficients(hdr)  -> per component int16 [blocks_y, blocks_x, 64] in natural order, after DC prediction (before dequantisation)
  planes(hdr, coefs) -> per component uint8 [blocks_y * 8, blocks_x * 8]: dequantise + jpeg_idct_islow (16-bit, as PIL runs it)
  rgb(hdr, planes)   -> uint8 [h, w, 3]: h2v1 / h2v2 fancy upsampling + ycc_rgb_convert (grayscale replicated)
  decode(data)       -> rgb(parse(data), ...)
"""
from __future__ import annotations

import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
                   28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54,
                   47, 55, 62, 63], dtype=np.int64)       # ZIGZAG[k] = natural index of the k-th coefficient in the stream


class Unsupported(ValueError):
    pass


def _u16(d, i):
    return (d[i] << 8) | d[i + 1]


def parse(data: bytes) -> dict:
    d = bytes(data)
    if len(d) < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise Unsupported("not a JPEG file")
    i = 2
    q, dc, ac = {}, {}, {}
    hdr = {"restart": 0, "adobe": None, "jfif": False}
    while True:
        while i < len(d) and d[i] == 0xFF and i + 1 < len(d) and d[i + 1] == 0xFF:
            i += 1
        if i + 4 > len(d) or d[i] != 0xFF:
            raise Unsupported("truncated or malformed header")
        m = d[i + 1]
        if m == 0xD9:
            raise Unsupported("no scan")
        n = _u16(d, i + 2)
        seg = d[i + 4:i + 2 + n]
        if n < 2 or len(seg) != n - 2:
            raise Unsupported("truncated or malformed header")
        i += 2 + n
        if m in (0xC2, 0xC6, 0xCA):
            raise Unsupported("progressive")
        if m in (0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF):
            raise Unsupported("arithmetic coding")
        if m in (0xC3, 0xC5, 0xC7):
            raise Unsupported("lossless or hierarchical")
        if m == 0xCC:
            raise Unsupported("arithmetic coding")
        if m in (0xC0, 0xC1):
            if seg[0] != 8:
                raise Unsupported("not 8-bit")
            hdr["h"], hdr["w"], nc = _u16(seg, 1), _u16(seg, 3), seg[5]
            hdr["comps"] = [dict(id=seg[6 + 3 * c], hs=seg[7 + 3 * c] >> 4, vs=seg[7 + 3 * c] & 15, tq=seg[8 + 3 * c]) for c in range(nc)]
        elif m == 0xDB:
            j = 0
            while j < len(seg):
                pq, tq = seg[j] >> 4, seg[j] & 15
                if pq:
                    vals = [_u16(seg, j + 1 + 2 * k) for k in range(64)]
                    j += 129
                else:
                    vals = list(seg[j + 1:j + 65])
                    j += 65
                t = np.zeros(64, np.int64)
                t[ZIGZAG] = vals
                q[tq] = t
        elif m == 0xC4:
            j = 0
            while j < len(seg):
                tc, th = seg[j] >> 4, seg[j] & 15
                counts = list(seg[j + 1:j + 17])
                vals = list(seg[j + 17:j + 17 + sum(counts)])
                j += 17 + sum(counts)
                (ac if tc else dc)[th] = (counts, vals)     # checked and built only if the scan references it, as libjpeg does
        elif m == 0xDD:
            hdr["restart"] = _u16(seg, 0)
        elif m == 0xEE and seg[:5] == b"Adobe":
            hdr["adobe"] = seg[11]
        elif m == 0xE0 and seg[:5] == b"JFIF\0":
            hdr["jfif"] = True
        elif m == 0xDA:
            ns = seg[0]
            ids = [c["id"] for c in hdr["comps"]]
            hdr["scan"] = [(ids.index(seg[1 + 2 * k]), seg[2 + 2 * k] >> 4, seg[2 + 2 * k] & 15) for k in range(ns)]
            if [c for c, _, _ in hdr["scan"]] != list(range(ns)):
                raise Unsupported("scan components not in frame order")
            break
    nc = len(hdr["comps"])
    if nc == 3:
        if not hdr["jfif"] and hdr["adobe"] == 0:      # default_decompress_parms: JFIF first, then Adobe transform 0 = RGB
            raise Unsupported("RGB colour")
        if hdr["adobe"] is None and not hdr["jfif"] and [c["id"] for c in hdr["comps"]] == [82, 71, 66]:
            raise Unsupported("RGB colour")
        s = [(c["hs"], c["vs"]) for c in hdr["comps"]]
        if s[1] != (1, 1) or s[2] != (1, 1) or s[0] not in ((1, 1), (2, 1), (2, 2)):
            raise Unsupported("sampling factors")
    elif nc != 1:
        raise Unsupported("CMYK or YCCK colour")
    if len(hdr["scan"]) != nc:
        raise Unsupported("multi-scan")
    hdr["q"] = [q[c["tq"]] for c in hdr["comps"]]
    hdr["dc"] = [_huff(*dc[t], is_dc=True) for _, t, _ in hdr["scan"]]
    hdr["ac"] = [_huff(*ac[t], is_dc=False) for _, _, t in hdr["scan"]]
    # scan bytes: up to the first marker that is neither a stuffed 0xFF00 nor RSTn
    j = i
    while True:
        j = d.find(b"\xff", j)
        if j < 0 or j + 1 >= len(d):
            j = len(d)
            break
        nxt = d[j + 1]
        if nxt == 0 or 0xD0 <= nxt <= 0xD7 or nxt == 0xFF:
            j += 1 if nxt == 0xFF else 2
            continue
        break
    hdr["scan_bytes"] = d[i:j]
    if nc == 1:                                   # a single-component scan is non-interleaved: one block per MCU
        hmax = vmax = 1
        hdr["comps"][0]["hs"] = hdr["comps"][0]["vs"] = 1
    else:
        hmax, vmax = hdr["comps"][0]["hs"], hdr["comps"][0]["vs"]
    hdr["hmax"], hdr["vmax"] = hmax, vmax
    hdr["mcus_x"] = -(-hdr["w"] // (8 * hmax))
    hdr["mcus_y"] = -(-hdr["h"] // (8 * vmax))
    return hdr


def _huff(counts, vals, is_dc):
    """{(length, code): symbol}.  Refuses the tables libjpeg's jpeg_make_d_derived_tbl refuses: the codes of a length must fit in
    that many bits and the last of them must not be all ones, and a DC table lists no symbol above 15."""
    if is_dc and any(v > 15 for v in vals):
        raise Unsupported("DC Huffman table with a symbol above 15")
    table, code, k = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(counts[ln - 1]):
            table[(ln, code)] = vals[k]
            code += 1
            k += 1
        if counts[ln - 1] and code >= 1 << ln:
            raise Unsupported("Huffman table with an all-ones code or too many codes")
        code <<= 1
    return table


def unstuff(scan: bytes):
    """Entropy-coded bytes with stuffing removed, split at RSTn: a list of byte strings, one per restart interval.  Marker k (the
    one ending interval k) must be RST(k mod 8): libjpeg resynchronises on any other, which this decoder does not restate."""
    segs, cur, i = [], bytearray(), 0
    while i < len(scan):
        b = scan[i]
        if b == 0xFF and i + 1 < len(scan):
            n = scan[i + 1]
            if n == 0x00:
                cur.append(0xFF)
                i += 2
                continue
            if 0xD0 <= n <= 0xD7:
                if n - 0xD0 != len(segs) % 8:
                    raise ValueError("restart marker out of sequence")
                segs.append(bytes(cur))
                cur = bytearray()
                i += 2
                continue
            i += 1                                     # fill byte
            continue
        cur.append(b)
        i += 1
    segs.append(bytes(cur))
    return segs


def coefficients(hdr: dict):
    """Sequential Huffman decode + DC prediction: per component int16 [blocks_y, blocks_x, 64], natural order."""
    comps = hdr["comps"]
    mx, my = hdr["mcus_x"], hdr["mcus_y"]
    out = [np.zeros((my * c["vs"], mx * c["hs"], 64), np.int64) for c in comps]
    order = [(ci, v, h) for ci, c in enumerate(comps) for v in range(c["vs"]) for h in range(c["hs"])]
    ri = hdr["restart"] or mx * my
    segs = unstuff(hdr["scan_bytes"])
    n_mcu = mx * my
    if len(segs) < -(-n_mcu // ri):
        raise ValueError("missing restart intervals")
    for s in range(-(-n_mcu // ri)):
        bits = np.unpackbits(np.frombuffer(segs[s], np.uint8)).tolist()
        nb = len(bits)
        pos = 0

        def read(n):
            nonlocal pos
            v = 0
            for _ in range(n):
                v = (v << 1) | (bits[pos] if pos < nb else 0)
                pos += 1
            return v

        def sym(t):
            nonlocal pos
            code = 0
            for ln in range(1, 17):
                code = (code << 1) | (bits[pos] if pos < nb else 0)
                pos += 1
                v = t.get((ln, code))
                if v is not None:
                    return v
            raise ValueError("bad Huffman code")

        def extend(v, n):
            return v - (1 << n) + 1 if n and v < (1 << (n - 1)) else v

        pred = [0] * len(comps)
        for mcu in range(s * ri, min(n_mcu, (s + 1) * ri)):
            my_, mx_ = divmod(mcu, mx)
            for ci, v, h in order:
                blk = out[ci][my_ * comps[ci]["vs"] + v, mx_ * comps[ci]["hs"] + h]
                n = sym(hdr["dc"][ci])
                pred[ci] += extend(read(n), n)
                blk[0] = pred[ci]
                k = 1
                while k < 64:
                    rs = sym(hdr["ac"][ci])
                    r, n = rs >> 4, rs & 15
                    if n == 0:
                        if r != 15:
                            break
                        k += 16                        # a ZRL past 63 ends the block
                        continue
                    k += r                             # a run past 63 stores at 63 (libjpeg's padded jpeg_natural_order)
                    blk[ZIGZAG[min(k, 63)]] = extend(read(n), n)
                    k += 1
            if pos > nb:
                raise ValueError("truncated entropy-coded segment")
    return [o.astype(np.int16) for o in out]


CONST_BITS, PASS1_BITS = 13, 2
FIX = {n: int(v * (1 << CONST_BITS) + 0.5) for n, v in [
    ("0_298631336", 0.298631336), ("0_390180644", 0.390180644), ("0_541196100", 0.541196100), ("0_765366865", 0.765366865),
    ("0_899976223", 0.899976223), ("1_175875602", 1.175875602), ("1_501321110", 1.501321110), ("1_847759065", 1.847759065),
    ("1_961570560", 1.961570560), ("2_053119869", 2.053119869), ("2_562915447", 2.562915447), ("3_072711026", 3.072711026)]}


def _w16(x):
    """x wrapped to int16, as a 16-bit SIMD multiply or add leaves it."""
    return ((x + 32768) & 0xFFFF) - 32768


def _idct_1d(s, shift):
    """One islow pass over axis 1 of s [N, 8, ...] (int64 holding int16 values): the 8 outputs descaled by `shift` and saturated
    to int16.  The arithmetic of libjpeg-turbo's SIMD islow, which PIL runs on x86: the sums in0 + in4, in0 - in4, in7 + in3 and
    in5 + in1 are 16-bit (they wrap), every product pairs 16-bit operands into 32-bit sums, and each pass packs its outputs to int16
    with saturation.  It equals jidctint.c's jpeg_idct_islow whenever no value leaves 16 bits, which holds for every file with
    quantisers up to a few thousand; past that the SIMD and C builds of libjpeg-turbo differ, and this is the SIMD one."""
    z2, z3 = s[:, 2], s[:, 6]
    tmp3 = z2 * (FIX["0_541196100"] + FIX["0_765366865"]) + z3 * FIX["0_541196100"]
    tmp2 = z2 * FIX["0_541196100"] + z3 * (FIX["0_541196100"] - FIX["1_847759065"])
    tmp0 = _w16(s[:, 0] + s[:, 4]) << CONST_BITS
    tmp1 = _w16(s[:, 0] - s[:, 4]) << CONST_BITS
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    a0, a1, a2, a3 = s[:, 7], s[:, 5], s[:, 3], s[:, 1]
    z3, z4 = _w16(a0 + a2), _w16(a1 + a3)
    z3p = z3 * (FIX["1_175875602"] - FIX["1_961570560"]) + z4 * FIX["1_175875602"]
    z4p = z3 * FIX["1_175875602"] + z4 * (FIX["1_175875602"] - FIX["0_390180644"])
    b0 = a0 * (FIX["0_298631336"] - FIX["0_899976223"]) - a3 * FIX["0_899976223"] + z3p
    b3 = -a0 * FIX["0_899976223"] + a3 * (FIX["1_501321110"] - FIX["0_899976223"]) + z4p
    b1 = a1 * (FIX["2_053119869"] - FIX["2_562915447"]) - a2 * FIX["2_562915447"] + z4p
    b2 = -a1 * FIX["2_562915447"] + a2 * (FIX["3_072711026"] - FIX["2_562915447"]) + z3p
    o = [t10 + b3, t11 + b2, t12 + b1, t13 + b0, t13 - b0, t12 - b1, t11 - b2, t10 - b3]
    return np.stack([np.clip((x + (1 << (shift - 1))) >> shift, -32768, 32767) for x in o], axis=1)


def range_limit(v):
    """The IDCT's output: v saturated to -128 .. 127, plus 128 (a saturating pack to signed bytes, then the centre added)."""
    return (np.clip(v, -128, 127) + 128).astype(np.uint8)


def idct_islow(coef, q):
    """jpeg_idct_islow on int16 [N, 64] natural-order coefficients and their quantisation table: uint8 [N, 8, 8].  The products are
    16-bit (they wrap), as libjpeg-turbo's SIMD dequantisation leaves them."""
    x = _w16(coef.astype(np.int64).reshape(-1, 8, 8) * q.reshape(1, 8, 8))   # [N, row (v), col (u)]
    ws = _idct_1d(x, CONST_BITS - PASS1_BITS)                                  # columns: over rows (axis 1)
    # the SIMD pass 1 skips the column IDCT of a block whose coefficient rows 1 .. 7 are all zero: every output row is then
    # row 0 dequantised and shifted left by PASS1_BITS in 16 bits, which wraps where the full pass saturates
    flat = (coef.reshape(-1, 8, 8)[:, 1:, :] == 0).all(axis=(1, 2))
    ws[flat] = _w16(x[flat, :1, :] << PASS1_BITS)
    out = _idct_1d(ws.transpose(0, 2, 1), CONST_BITS + PASS1_BITS + 3)         # rows: over columns
    return range_limit(out.transpose(0, 2, 1))


def planes(hdr: dict, coefs):
    out = []
    for c, q in zip(coefs, hdr["q"]):
        by, bx = c.shape[:2]
        p = idct_islow(c.reshape(-1, 64), q).reshape(by, bx, 8, 8).transpose(0, 2, 1, 3).reshape(by * 8, bx * 8)
        out.append(p)
    return out


def _h2v1(p, cw):
    """h2v1_fancy_upsample over columns 0 .. cw - 1 (cw > 2) of the rows p (int64 [R, >= cw]): [R, 2 * cw]."""
    v = p[:, :cw]
    out = np.empty((p.shape[0], 2 * cw), np.int64)
    prev = np.concatenate([v[:, :1], v[:, :-1]], axis=1)
    nxt = np.concatenate([v[:, 1:], v[:, -1:]], axis=1)
    out[:, 0::2] = (v * 3 + prev + 1) >> 2
    out[:, 1::2] = (v * 3 + nxt + 2) >> 2
    out[:, 0], out[:, -1] = v[:, 0], v[:, -1]
    return out


def _h2v2(p, cw, ch):
    """h2v2_fancy_upsample of the ch x cw (cw > 2) component (context rows above the first and below the last replicate them): [2ch, 2cw]."""
    v = p[:ch, :cw]
    up = np.concatenate([v[:1], v[:-1]], axis=0)
    dn = np.concatenate([v[1:], v[-1:]], axis=0)
    out = np.empty((2 * ch, 2 * cw), np.int64)
    for r, near in ((0, up), (1, dn)):
        cs = v * 3 + near
        o = np.empty((ch, 2 * cw), np.int64)
        prev = np.concatenate([cs[:, :1], cs[:, :-1]], axis=1)
        nxt = np.concatenate([cs[:, 1:], cs[:, -1:]], axis=1)
        o[:, 0::2] = (cs * 3 + prev + 8) >> 4
        o[:, 1::2] = (cs * 3 + nxt + 7) >> 4
        o[:, 0] = (cs[:, 0] * 4 + 8) >> 4
        o[:, -1] = (cs[:, -1] * 4 + 7) >> 4
        out[r::2] = o
    return out


SCALEBITS = 16


def _fix(x):
    return int(x * (1 << SCALEBITS) + 0.5)


def ycc_tables():
    """ycc_rgb_convert's build_ycc_rgb_table: Cr->R, Cb->B (rounded), Cr->G, Cb->G (scaled, Cb_g carries ONE_HALF)."""
    x = np.arange(256, dtype=np.int64) - 128
    half = 1 << (SCALEBITS - 1)
    cr_r = (_fix(1.40200) * x + half) >> SCALEBITS
    cb_b = (_fix(1.77200) * x + half) >> SCALEBITS
    cr_g = -_fix(0.71414) * x
    cb_g = -_fix(0.34414) * x + half
    return cr_r, cb_b, cr_g, cb_g


def rgb(hdr: dict, pl):
    h, w = hdr["h"], hdr["w"]
    if len(pl) == 1:
        y = pl[0][:h, :w]
        return np.repeat(y[:, :, None], 3, axis=2)
    hs, vs = hdr["hmax"], hdr["vmax"]
    y = pl[0][:h, :w].astype(np.int64)
    cw, ch = -(-w // hs), -(-h // vs)                       # downsampled_width / _height of the chroma components
    up = []
    for p in pl[1:]:
        p = p.astype(np.int64)
        if (hs, vs) == (1, 1):
            u = p
        elif cw <= 2:                                        # jinit_upsampler: fancy only when downsampled_width > 2
            u = np.repeat(np.repeat(p[:ch, :cw], vs, axis=0), hs, axis=1)
        elif vs == 1:
            u = _h2v1(p[:ch], cw)
        else:
            u = _h2v2(p, cw, ch)
        up.append(u[:h, :w])
    cb, cr = up
    cr_r, cb_b, cr_g, cb_g = ycc_tables()
    r = y + cr_r[cr]
    g = y + ((cb_g[cb] + cr_g[cr]) >> SCALEBITS)
    b = y + cb_b[cb]
    return np.clip(np.stack([r, g, b], axis=2), 0, 255).astype(np.uint8)


def decode(data: bytes) -> np.ndarray:
    hdr = parse(data)
    return rgb(hdr, planes(hdr, coefficients(hdr)))
