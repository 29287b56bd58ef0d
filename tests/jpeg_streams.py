"""Crafted JPEG streams for the decoder's tests, written by tests/jpeg_writer.py from known coefficients: the table, slot, value,
subsequence-boundary and unstuffing edges that Pillow's encoder never writes, and streams that break the restart and run rules.
Every family is seeded.  valid_streams() and contract_streams() return (name, file, log); log is None where the stream is not a
plain encoding of its coefficients."""
from __future__ import annotations

import numpy as np

import jpeg_writer as jw

SUB_BITS = 1024                     # TP_JPEG_SUBSEQUENCE_BYTES * 8: the parallel Huffman decode's unit
CHUNK = 4096                        # bytes the unstuff kernel's CTA consumes per step (512 threads x 8 bytes)

def YCC(hs=1, vs=1):
    """Components 1, 2, 3: luma on slots 0, chroma on slots 1."""
    return [jw.Comp(1, hs, vs, 0, 0, 0), jw.Comp(2, 1, 1, 1, 1, 1), jw.Comp(3, 1, 1, 1, 1, 1)]

# tables: a DC table close to the common ones, an AC table with a 2-bit EOB and every other symbol at 8 or 9 bits, tables with
# codes of 16 bits only, 1-bit DC 0 and EOB codes, and a 256-symbol AC table
DC_STD = jw.table({0: 2, **{s: 3 for s in range(1, 6)}, **{s: s - 2 for s in range(6, 16)}})
AC_STD = jw.table({0x00: 2, **{s: 8 for s in jw.ALL_AC[1:129]}, **{s: 9 for s in jw.ALL_AC[129:]}})
DC_LONG = jw.uniform(range(16), 16)
AC_LONG = jw.uniform(jw.ALL_AC, 16)
DC_ONE = jw.table({0: 1, **{s: 5 for s in range(1, 16)}})
AC_ONE = jw.table({0x00: 1, **{s: 9 for s in jw.ALL_AC[1:]}})
AC_256 = jw.table({s: (8 if i < 128 else 9) for i, s in enumerate(np.random.default_rng(7).permutation(256).tolist())})
# one symbol at each length 1 .. 16: DC 15 and AC 0x0F take the codes 1111111111111110, so that their fields are almost all ones
DC_UNARY = jw.table({s: s + 1 for s in range(16)})
AC_UNARY = jw.table({**{s: i + 1 for i, s in enumerate([0x00, 0x01, 0x02, 0x03, 0x04, 0x05, 0x06, 0x07, 0x08, 0x09, 0x0A, 0x0B,
                                                           0x0C, 0x0D, 0xF0])}, 0x0F: 16})


def q(seed, lo=1, hi=40):
    return np.random.default_rng(seed).integers(lo, hi + 1, 64).tolist()


def coefs_for(h, w, comps, seed, density=0.15, ac_max=60, dc_max=400, cats=None):
    """Random coefficients: a DC per block within +-dc_max, AC nonzero with the given density; cats = (lo, hi) draws every nonzero
    value's category from that range instead (both signs)."""
    r = np.random.default_rng(seed)
    out = []
    for by, bx in jw.grid(h, w, comps):
        c = np.zeros((by, bx, 64), np.int64)
        c[..., 0] = r.integers(-dc_max, dc_max + 1, (by, bx))
        mask = r.random((by, bx, 63)) < density
        if cats is None:
            v = r.integers(1, ac_max + 1, (by, bx, 63))
        else:
            s = r.integers(cats[0], cats[1] + 1, (by, bx, 63))
            v = (1 << (s - 1)) + (r.integers(0, 1 << 30, (by, bx, 63)) & ((1 << (s - 1)) - 1))
        c[..., 1:] = np.where(mask, v * r.choice([-1, 1], (by, bx, 63)), 0)
        out.append(c)
    return out


def write(name, h, w, comps, coefs, *, dc=None, ac=None, qt=None, **kw):
    dc = dc if dc is not None else {0: DC_STD, 1: DC_STD}
    ac = ac if ac is not None else {0: AC_STD, 1: AC_STD}
    qt = qt if qt is not None else {0: q(1), 1: q(2)}
    f, log = jw.write_jpeg(h, w, comps, coefs, dc_tables=dc, ac_tables=ac, qtables=qt, **kw)
    return name, f, log


# ------------------------------------------------------------------------------------------------------------------------------
# tables and slots
# ------------------------------------------------------------------------------------------------------------------------------
def table_streams():
    out = []
    g = [jw.Comp(1)]
    out.append(write("long-codes-gray", 40, 56, g, coefs_for(40, 56, g, 1, density=0.3, cats=(1, 15)), dc={0: DC_LONG},
                     ac={0: AC_LONG}, qt={0: q(3)}))
    c = YCC(hs=2, vs=2)
    out.append(write("long-codes-chroma-420", 33, 47, c, coefs_for(33, 47, c, 2, density=0.2), dc={0: DC_STD, 1: DC_LONG},
                     ac={0: AC_STD, 1: AC_LONG}))
    z = [np.zeros(s + (64,), np.int64) for s in jw.grid(24, 24, YCC())]
    out.append(write("one-bit-codes-444-dri1", 24, 24, YCC(), z, dc={0: DC_ONE, 1: DC_ONE}, ac={0: AC_ONE, 1: AC_ONE}, restart=1))
    z = [np.zeros((4, 8, 64), np.int64)]
    out.append(write("one-bit-codes-gray-dri4", 32, 64, g, z, dc={0: DC_ONE}, ac={0: AC_ONE}, qt={0: q(4)}, restart=4))
    mixed = coefs_for(32, 64, g, 3, density=0.05, dc_max=3)
    for cf in mixed:
        cf[::2, ::3] = 0
    out.append(write("one-bit-codes-gray-mixed", 32, 64, g, mixed, dc={0: DC_ONE}, ac={0: AC_ONE}, qt={0: q(5)}, restart=3))
    c = YCC(hs=2, vs=1)
    out.append(write("ac-256-symbols-422", 30, 50, c, coefs_for(30, 50, c, 4, density=0.25), ac={0: AC_256, 1: AC_STD}))
    # every component on other slots, each slot's table and quantiser distinct, and tables defined in an unusual order
    c = [jw.Comp(1, 2, 2, tq=2, td=1, ta=3), jw.Comp(2, tq=0, td=3, ta=2), jw.Comp(3, tq=3, td=2, ta=1)]
    dcs = {0: DC_ONE, 1: DC_STD, 2: DC_LONG, 3: DC_UNARY}
    acs = {0: AC_ONE, 1: AC_LONG, 2: AC_256, 3: AC_STD}
    qts = {0: q(10, 1, 9), 1: q(11, 30, 90), 2: q(12, 2, 20), 3: q(13, 10, 50)}
    order = [("ac", 2), ("dc", 3), ("ac", 0), ("dc", 1), ("ac", 3), ("dc", 0), ("ac", 1), ("dc", 2)]
    out.append(write("swapped-slots-420", 41, 37, c, coefs_for(41, 37, c, 5, density=0.2), dc=dcs, ac=acs, qt=qts, dht_order=order))
    c = [jw.Comp(1, 1, 1, tq=1, td=1, ta=0), jw.Comp(2, tq=0, td=0, ta=1), jw.Comp(3, tq=0, td=0, ta=1)]
    out.append(write("swapped-slots-444-sof1", 19, 29, c, coefs_for(19, 29, c, 6), dc={0: DC_STD, 1: DC_LONG},
                     ac={0: AC_LONG, 1: AC_STD}, sof=0xC1))
    for ids in ([0, 1, 2], [7, 200, 33], [255, 0, 128]):
        c = [jw.Comp(ids[0], 2, 2), jw.Comp(ids[1], tq=1, td=1, ta=1), jw.Comp(ids[2], tq=1, td=1, ta=1)]
        out.append(write(f"ids-{ids[0]}-{ids[1]}-{ids[2]}", 25, 31, c, coefs_for(25, 31, c, 7 + ids[1])))
    c = YCC(hs=2, vs=1)
    segs = [(0xE1, b"Exif\x00\x00" + bytes(30)), (0xFE, b"a comment \xff\xd9 inside"), jw.adobe(1), (0xE2, bytes(5))]
    out.append(write("no-jfif-adobe1-appn-com", 21, 35, c, coefs_for(21, 35, c, 8), segments=segs))
    out.append(write("gray-sof1-no-jfif", 17, 9, g, coefs_for(17, 9, g, 9), dc={0: DC_STD}, ac={0: AC_STD}, qt={0: q(14)},
                     sof=0xC1, segments=()))
    return out


# ------------------------------------------------------------------------------------------------------------------------------
# values: DC categories 12 - 15, AC categories 11 - 15 at every zigzag position, DC sums past int16, 16-bit quantisers near 32767
# ------------------------------------------------------------------------------------------------------------------------------
def value_streams():
    out = []
    r = np.random.default_rng(20)
    g = [jw.Comp(1)]
    h, w = 8 * 9, 8 * 14                                              # 126 blocks: every zigzag position twice
    cf = np.zeros((9, 14, 64), np.int64)
    dc = np.cumsum(r.choice([-1, 1], 126) * r.integers(1 << 11, 1 << 15, 126)).reshape(9, 14)    # categories 12 .. 15
    cf[..., 0] = dc
    for b in range(126):
        k = 1 + b % 63
        s = 11 + b % 5
        cf[b // 14, b % 14, jw.ZIGZAG[k]] = r.choice([-1, 1]) * ((1 << (s - 1)) + int(r.integers(0, 1 << (s - 1))))
    assert np.abs(dc).max() > 32767                                   # the DC running sum leaves int16
    for qname, qt in [("q1", [1] * 64), ("q16-near-32767", r.integers(30000, 32768, 64).tolist()), ("q16-small", q(21, 1, 300))]:
        out.append(write(f"big-values-gray-{qname}", h, w, g, [cf], dc={0: DC_STD}, ac={0: AC_STD}, qt={0: qt}, q16=(0,)))
    c = YCC(hs=2, vs=2)
    cfs = coefs_for(48, 64, c, 22, density=0.1, cats=(11, 15))
    for x in cfs:
        x[..., 0] = r.integers(-(1 << 14), 1 << 14, x.shape[:2])     # differences up to category 15 in any coding order
    out.append(write("big-values-420-q16", 48, 64, c, cfs, qt={0: r.integers(32000, 32768, 64).tolist(), 1: q(23, 200, 4000)}))
    return out


# ------------------------------------------------------------------------------------------------------------------------------
# subsequence boundaries: gray, one block per restart interval, every code 16 bits, so that a block's fields are placed to the bit
# ------------------------------------------------------------------------------------------------------------------------------
def _block(fields):
    """One block's zigzag coefficients whose fields under DC_LONG / AC_LONG have the given lengths: fields[0] the DC field (16 + s),
    then one AC field (16 + s, s >= 1) per coefficient from zigzag 1 on; an EOB (16 bits) follows when fewer than 63."""
    zz = np.zeros(64, np.int64)
    zz[0] = (1 << (fields[0] - 17)) if fields[0] > 16 else 0
    for k, ln in enumerate(fields[1:], start=1):
        s = ln - 16
        assert 1 <= s <= 15
        zz[k] = -(1 << (s - 1))
    return zz


def _split(total, n, lo=17, hi=31):
    """n lengths in [lo, hi] summing to total."""
    assert lo * n <= total <= hi * n, (total, n)
    out = [lo] * n
    extra = total - lo * n
    for i in range(n):
        a = min(hi - lo, extra)
        out[i] += a
        extra -= a
    return out


def boundary_blocks():
    """(label, fields) per block: for every d in 1 .. 31, a code + value starting d bits before the first subsequence boundary; then
    interval lengths of 127, 128, 129 .. 132 bytes; and a 129-byte interval whose last code (an EOB from bit 1016) swallows the
    interval's 8-bit last subsequence."""
    out = []
    for d in range(1, 32):
        ln = max(d + 1, 17) if d < 31 else 31                        # it crosses the boundary (d = 31: it ends on it)
        prefix = SUB_BITS - d                                       # the DC field and m AC fields before it
        m = -(-(prefix - 31) // 31)
        dcl = max(16, prefix - 31 * m)
        out.append((f"d{d}", [dcl] + _split(prefix - dcl, m) + [ln]))
    for nbytes in (127, 128, 129, 130, 131, 132):
        total = 8 * nbytes                                          # no padding: the fields end on the interval's last bit
        body = total - 16                                           # EOB last
        n = -(-(body - 31) // 31)
        fields = [31] + _split(body - 31, n)
        out.append((f"len{nbytes}", fields))
    # the last field an EOB from bit 1016 to 1032: the 8-bit last subsequence [1024, 1032) has nothing left to decode
    body = 1016
    n = -(-(body - 31) // 31)
    out.append(("swallow", [31] + _split(body - 31, n)))
    return out


def boundary_stream():
    blocks = boundary_blocks()
    n = len(blocks)
    cf = np.zeros((1, n, 64), np.int64)
    for i, (_, fields) in enumerate(blocks):
        cf[0, i, jw.ZIGZAG] = _block(fields)
    return write("boundaries-gray-dri1", 8, 8 * n, [jw.Comp(1)], [cf], dc={0: DC_LONG}, ac={0: AC_LONG}, qt={0: q(30, 1, 20)},
                 restart=1)


def boundary_offsets(log):
    """The set of d (bits between a code + value's start and the next subsequence boundary that it reaches)."""
    start = log.code_pos
    end = start + log.code_len + log.val_len
    b = (start // SUB_BITS + 1) * SUB_BITS
    hit = end >= b
    return set((b - start)[hit].tolist())


# ------------------------------------------------------------------------------------------------------------------------------
# unstuffing: dense 0xFF00, a stuffed pair and an RSTn across the 4096-byte chunk and an 8-byte thread boundary, fill and garbage
# ------------------------------------------------------------------------------------------------------------------------------
def _dense(n_blocks, lead):
    """gray blocks whose fields are nearly all ones: DC and AC category 15 on the codes 1111111111111110; block 0 has `lead` such
    AC fields, which shifts everything after it."""
    cf = np.zeros((1, n_blocks, 64), np.int64)
    cf[0, :, 0] = 32767 * np.arange(1, n_blocks + 1)                 # DC differences of +32767: the sum wraps int16 many times
    cf[0, 1:, 1:] = 32767
    cf[0, 0, jw.ZIGZAG[1:1 + lead]] = 32767
    return cf


def dense_stream():
    for lead in range(64):
        name, f, log = write(f"dense-ff00-lead{lead}", 8, 8 * 24, [jw.Comp(1)], [_dense(24, lead)], dc={0: DC_UNARY},
                             ac={0: AC_UNARY}, qt={0: q(31)})
        rel = {p - log.scan_begin for p in log.stuffed}
        if CHUNK - 1 in rel and any(p % 8 == 7 and p % CHUNK != CHUNK - 1 for p in rel):
            return name, f, log
    raise AssertionError("no lead puts a stuffed pair across the chunk boundary")


def rst_stream():
    """4:2:0 with DRI = 2, garbage before one RSTn and 0xFF fill before others: one marker's 0xFF at scan byte 4095 (its Dn at
    4096, the next chunk), another's at a byte 8t + 7 inside a chunk, and fill before the EOI."""
    c = YCC(hs=2, vs=2)
    cf = coefs_for(64, 96, c, 40, density=0.35, ac_max=200)
    garbage = {3: b"\x12\x34\x00\x56\x00"}
    fills = {1: 3}

    def make():
        return write("rst-across-chunk-420", 64, 96, c, cf, restart=2, garbage_before_rst=lambda k: garbage.get(k, b""),
                     fill_before_rst=lambda k: fills.get(k, 0), fill_before_eoi=4)

    _, _, log = make()
    rel = [p - log.scan_begin for p in log.rst]
    k8 = 5
    fills[k8] = (7 - rel[k8]) % 8 + 8                                # marker k8's 0xFF at 8t + 7
    _, _, log = make()
    rel = [p - log.scan_begin for p in log.rst]
    k = max(i for i, p in enumerate(rel) if p <= CHUNK - 1 and i > k8)
    fills[k] = fills.get(k, 0) + CHUNK - 1 - rel[k]
    name, f, log = make()
    rel = [p - log.scan_begin for p in log.rst]
    assert CHUNK - 1 in rel and rel[k8] % 8 == 7 and rel[k8] % CHUNK != CHUNK - 1
    return name, f, log


# ------------------------------------------------------------------------------------------------------------------------------
# the contract: restart numbering, runs past 63, invalid codes
# ------------------------------------------------------------------------------------------------------------------------------
def _run_edit(kind):
    def edit(ci, by, bx, syms):
        if (ci, by, bx) != (0, 0, 1):
            return syms
        zrl = ("ac", 0xF0, 0, 0)
        if kind == "zrl":        # k 1 -> 50 by three ZRL, a value at 55, then a ZRL from 56 (past 63): the block ends
            return [syms[0], ("ac", 0x01, 1, 1), zrl, zrl, zrl, ("ac", 0x52, 2, 3), zrl]
        if kind == "zrl63":      # a ZRL from 63
            return [syms[0]] + [("ac", 0x01, 1, 1)] * 62 + [zrl]
        if kind == "run":        # a value at 59, then a run of 14 from 60: stored at 63
            return [syms[0], ("ac", 0x01, 1, 1), zrl, zrl, zrl, ("ac", 0x93, 3, 5), ("ac", 0xE2, 2, 1)]
        return [syms[0], ("ac", 0x01, 1, 1), zrl, zrl, zrl, ("ac", 0xFF, 15, 12345)]    # a run of 15 from 50 with 15 bits: at 63
    return edit


def _bad_code_edit(ci, by, bx, syms):
    if (ci, by, bx) == (0, 1, 2):
        return syms[:3] + [("raw", 16, 0xFFFF)] + syms[3:]          # AC_STD has no 16-bit code of all ones
    return syms


def contract_streams():
    """(name, file, log, expected) where expected is 'ok' (status 0, PIL's bytes), 'restart' or 'entropy' (that status)."""
    out = []
    c = YCC(hs=2, vs=2)
    cf = coefs_for(48, 80, c, 50, density=0.2)
    base = dict(restart=1)
    for label, numbering in [("rst-all-0", lambda k: 0), ("rst-one-skipped", lambda k: (k + (k >= 4)) % 8),
                             ("rst-one-repeated", lambda k: (k - (k >= 4)) % 8), ("rst-wrapped-correctly", lambda k: k % 8)]:
        expected = "ok" if label == "rst-wrapped-correctly" else "restart"
        out.append(write(label, 48, 80, c, cf, rst_number=numbering, **base) + (expected,))
    g = [jw.Comp(1)]
    cg = coefs_for(16, 24, g, 51, density=0.1)
    for kind in ("zrl", "zrl63", "run", "run15"):
        name, f, _ = write(f"ac-{kind}-past-63", 16, 24, g, cg, dc={0: DC_STD}, ac={0: AC_STD}, qt={0: q(52)}, edit=_run_edit(kind))
        out.append((name, f, None, "ok"))
    name, f, _ = write("bad-code-mid-interval", 48, 80, c, cf, restart=6, edit=_bad_code_edit)
    out.append((name, f, None, "entropy"))
    return out


def valid_streams():
    return table_streams() + value_streams() + [boundary_stream(), dense_stream(), rst_stream()]


# ------------------------------------------------------------------------------------------------------------------------------
# camera size
# ------------------------------------------------------------------------------------------------------------------------------
def camera_stream(sub: str):
    h, w = 3024, 4032
    c = YCC(hs=2, vs=2 if sub == "420" else 1)
    r = np.random.default_rng(60 if sub == "420" else 61)
    cfs = []
    for ci, (by, bx) in enumerate(jw.grid(h, w, c)):
        cf = np.zeros((by, bx, 64), np.int64)
        yy, xx = np.mgrid[0:by, 0:bx]
        cf[..., 0] = (200 * np.sin(yy / 37 + ci) * np.cos(xx / 53) + r.integers(-20, 21, (by, bx))).astype(np.int64)
        for k in (1, 2, 3, 8, 9):
            cf[..., jw.ZIGZAG[k]] = r.integers(-30, 31, (by, bx)) * (r.random((by, bx)) < 0.4)
        cfs.append(cf)
    mcus_x = -(-w // 16)
    return write(f"camera-4032x3024-{sub}", h, w, c, cfs, restart=mcus_x)
