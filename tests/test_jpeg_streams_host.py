"""The JPEG decoder's host side on streams Pillow never writes (tests/jpeg_streams.py, written by tests/jpeg_writer.py from known
coefficients), no GPU: the oracle's coefficients equal the writer's, its pixels equal PIL's, and jpeg_unsupported refuses a
Huffman table exactly where PIL raises."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jpeg_fixtures as jf  # noqa: E402
import jpeg_streams as js  # noqa: E402
import jpeg_writer as jw  # noqa: E402
from oracle import jpeg_oracle as jo  # noqa: E402


def _pil(data):
    """PIL's pixels, or None when PIL raises."""
    try:
        return jf.pil_decode(data)
    except (OSError, SyntaxError, ValueError):
        return None


@pytest.fixture(scope="module")
def valid():
    return js.valid_streams()


def test_writer_agrees_with_pil_on_its_own():
    """The writer's zigzag order, value coding and padding are T.81's: Pillow's own file, re-coded from the oracle's coefficients with
    Pillow's tables, decodes to the same pixels."""
    data = jf.encode(jf.image(40, 48, "noise", 3), "420", 90)
    hdr = jo.parse(data)
    coefs = [c.astype(np.int64) for c in jo.coefficients(hdr)]
    comps = [jw.Comp(1, 2, 2, 0, 0, 0), jw.Comp(2, 1, 1, 1, 1, 1), jw.Comp(3, 1, 1, 1, 1, 1)]
    qt = {0: hdr["q"][0], 1: hdr["q"][1]}
    f, log = jw.write_jpeg(40, 48, comps, coefs, dc_tables={0: js.DC_STD, 1: js.DC_STD}, ac_tables={0: js.AC_STD, 1: js.AC_STD},
                           qtables=qt)
    assert np.array_equal(jf.pil_decode(f), jf.pil_decode(data))
    assert all(np.array_equal(a, b) for a, b in zip(log.coefs, coefs))


def test_oracle_coefficients_equal_the_writer_and_pixels_equal_pil(valid):
    assert len(valid) >= 20
    for name, data, log in valid:
        hdr = jo.parse(data)
        coefs = jo.coefficients(hdr)
        for c, (got, want) in enumerate(zip(coefs, log.coefs)):
            assert np.array_equal(got, want), (name, c)
        assert np.array_equal(jo.rgb(hdr, jo.planes(hdr, coefs)), jf.pil_decode(data)), name


def test_valid_streams_are_supported(valid):
    from tokenpacker_b200 import jpeg_unsupported
    assert jpeg_unsupported([d for _, d, _ in valid]) == [None] * len(valid)


def test_the_families_reach_their_edges(valid):
    """What each family is for, read back from the writer's logs."""
    by = {n: (d, log) for n, d, log in valid}
    _, log = by["boundaries-gray-dri1"]
    assert js.boundary_offsets(log) >= set(range(1, 32))
    assert {n % 128 for n in log.intervals} >= {0, 1, 2, 3, 4, 127}
    # a code ending on the last bit of a 129-byte interval after starting before bit 1024: the 8-bit last subsequence is swallowed
    end = log.code_pos + log.code_len + log.val_len
    swallow = (end == 1032) & (log.code_pos < 1024) & (np.array(log.intervals)[log.interval] == 129)
    assert swallow.any()
    for name in ("dense-ff00-lead", "rst-across-chunk-420"):
        d, log = next(v for n, v in by.items() if n.startswith(name))
        rel = [p - log.scan_begin for p in (log.stuffed if name.startswith("dense") else log.rst)]
        assert js.CHUNK - 1 in rel, name                           # 0xFF the last byte of one 4096-byte chunk, its pair the next
        assert any(p % 8 == 7 and p % js.CHUNK != js.CHUNK - 1 for p in rel), name
    d, log = next(v for n, v in by.items() if n.startswith("dense-ff00-lead"))
    scan = d[log.scan_begin:]
    assert scan.count(b"\xff\x00") * 4 > len(scan)                  # over half the bytes are stuffed pairs
    d, log = by["big-values-gray-q1"]
    dc = log.coefs[0][..., 0].astype(np.int64)
    assert (np.abs(np.diff(dc.ravel())) >= 1 << 11).all()           # DC categories 12 .. 15 throughout
    assert d.count(b"\xff\xdb\x00\x83\x10") == 1                    # a 16-bit DQT


def _table_cases():
    """(name, dc counts / values, ac counts / values, referenced): tables at the edges of libjpeg's jpeg_make_d_derived_tbl.  The
    stream uses DC 0 and EOB only, which each of these tables can code."""
    def unary_all_ones(n_len, syms):                                # 0, 10, 110, ..: then two codes of n_len bits, the last all ones
        lengths = list(range(1, n_len)) + [n_len, n_len]
        counts = [lengths.count(l) for l in range(1, 17)]
        return counts, syms[:len(lengths)]
    dc_syms = list(range(16)) + [0]
    ac_syms = [0x00] + [s for s in jw.ALL_AC if s != 0x00]
    ok_dc, ok_ac = js.DC_STD, js.AC_STD
    cases = []
    for n in (1, 2, 5, 9, 10, 16):
        cases.append((f"dc-all-ones-{n}", unary_all_ones(n, dc_syms), ok_ac, True))
        cases.append((f"ac-all-ones-{n}", ok_dc, unary_all_ones(n, ac_syms), True))
    cases.append(("dc-last-code-one-below-all-ones", jw.table({0: 1, 1: 2, 2: 3}), ok_ac, True))
    cases.append(("dc-symbol-16", (ok_dc[0][:13] + [1] + ok_dc[0][14:], ok_dc[1] + [16]), ok_ac, True))
    cases.append(("dc-symbol-255", (ok_dc[0][:13] + [1] + ok_dc[0][14:], ok_dc[1] + [255]), ok_ac, True))
    cases.append(("oversubscribed-1-bit", ([3] + [0] * 15, [0, 1, 2]), ok_ac, True))
    cases.append(("oversubscribed-2-bit", ok_dc, ([0, 5] + [0] * 14, [0x00, 0x01, 0x02, 0x03, 0x04]), True))
    cases.append(("ac-256-symbols", ok_dc, js.AC_256, True))
    cases.append(("only-16-bit-codes", js.DC_LONG, js.AC_LONG, True))
    cases.append(("one-bit-dc-and-eob", js.DC_ONE, js.AC_ONE, True))
    cases.append(("unreferenced-dc-all-ones", unary_all_ones(4, dc_syms), ok_ac, False))
    cases.append(("unreferenced-dc-symbol-16", (ok_dc[0][:13] + [1] + ok_dc[0][14:], ok_dc[1] + [16]), ok_ac, False))
    cases.append(("unreferenced-ac-oversubscribed", ok_dc, ([0, 5] + [0] * 14, [0x00, 0x01, 0x02, 0x03, 0x04]), False))
    return cases


def _table_file(dc, ac, referenced, redefine=None):
    """Gray 16 x 24 of DC 0 and EOB blocks.  The table under test sits in slot 0 when referenced, else in slot 2 beside valid
    tables in slot 0; redefine = 'after' defines a valid table first and the one under test over it, 'before' the reverse."""
    z = [np.zeros((2, 3, 64), np.int64)]
    slot = 0 if referenced else 2
    dcs, acs = {0: js.DC_ONE}, {0: js.AC_ONE}
    dcs[slot], acs[slot] = dc, ac
    if redefine:
        # the same slot defined twice: the writer codes with the last definition it is given, so give it the valid one
        test_first = redefine == "before"
        f, _ = jw.write_jpeg(16, 24, [jw.Comp(1)], z, dc_tables={0: js.DC_ONE}, ac_tables={0: js.AC_ONE}, qtables={0: js.q(1)})
        dht_bad = b"\xff\xc4" + (2 + 17 + len(dc[1])).to_bytes(2, "big") + bytes([0] + list(dc[0]) + list(dc[1]))
        i = f.index(b"\xff\xc4")
        return f[:i] + dht_bad + f[i:] if test_first else f[:f.index(b"\xff\xda")] + dht_bad + f[f.index(b"\xff\xda"):]
    f, _ = jw.write_jpeg(16, 24, [jw.Comp(1)], z, dc_tables=dcs, ac_tables=acs, qtables={0: js.q(1)})
    return f


@pytest.mark.parametrize("case", _table_cases(), ids=lambda c: c[0])
def test_table_refusal_follows_pil(case):
    from tokenpacker_b200 import jpeg_unsupported
    name, dc, ac, referenced = case
    data = _table_file(dc, ac, referenced)
    pil = _pil(data)
    (reason,) = jpeg_unsupported([data])
    if pil is None:
        assert reason == "malformed or truncated header", name
        with pytest.raises(jo.Unsupported):
            jo.decode(data)
    else:
        assert reason is None, (name, reason)
        assert np.array_equal(jo.decode(data), pil), name
    if not referenced:
        assert pil is not None, name                                 # libjpeg checks only the tables a scan references


def test_table_refusal_expected_outcomes():
    """The cases above, pinned: PIL raises on every invalid referenced table and decodes everything else."""
    got = {name: _pil(_table_file(dc, ac, ref)) is None for name, dc, ac, ref in _table_cases()}
    raises = {n for n, r in got.items() if r}
    assert raises == {n for n, _, _, ref in _table_cases()
                      if ref and not n.startswith(("ac-256", "only-16", "one-bit", "dc-last-code-one-below"))}


@pytest.mark.parametrize("when", ["before", "after"])
def test_a_redefined_table_is_checked_as_the_scan_finds_it(when):
    """An invalid DC table in slot 0 that a valid one replaces before the scan is never used (PIL decodes); one that replaces the
    valid table is (PIL raises)."""
    from tokenpacker_b200 import jpeg_unsupported
    bad = ([1, 1, 2] + [0] * 13, [0, 1, 2, 3])                       # 0, 10, 110, 111: 111 is all ones
    data = _table_file(bad, js.AC_ONE, True, redefine=when)
    pil = _pil(data)
    assert (pil is None) == (when == "after")
    assert (jpeg_unsupported([data])[0] is not None) == (when == "after")
    if pil is not None:
        assert np.array_equal(jo.decode(data), pil)


def test_restart_markers_out_of_sequence_differ_in_pil_and_the_oracle_raises():
    streams = {n: (d, exp) for n, d, _, exp in js.contract_streams()}
    d, _ = streams["rst-wrapped-correctly"]
    ref = jf.pil_decode(d)
    assert np.array_equal(jo.decode(d), ref)
    for name in ("rst-all-0", "rst-one-skipped", "rst-one-repeated"):
        bad, exp = streams[name]
        assert exp == "restart"
        with pytest.raises(ValueError, match="out of sequence"):
            jo.decode(bad)
        pil = _pil(bad)
        assert pil is None or not np.array_equal(pil, ref), name     # libjpeg resynchronises: other pixels than the coded ones


def test_runs_past_63_decode_as_libjpeg_does():
    """A ZRL past coefficient 63 ends the block; a run past 63 stores its value at 63.  PIL, the oracle and the same coefficients
    written plainly agree."""
    streams = {n: d for n, d, _, _ in js.contract_streams()}
    for kind in ("zrl", "zrl63", "run", "run15"):
        d = streams[f"ac-{kind}-past-63"]
        pil = jf.pil_decode(d)
        assert np.array_equal(jo.decode(d), pil), kind
    g = [jw.Comp(1)]
    base = js.coefs_for(16, 24, g, 51, density=0.1)[0]
    plain = base.copy()
    plain[0, 1, 1:] = 0
    plain[0, 1, jw.ZIGZAG[1]] = 1
    plain[0, 1, jw.ZIGZAG[59]] = 5
    plain[0, 1, 63] = -2
    f, _ = jw.write_jpeg(16, 24, g, [plain], dc_tables={0: js.DC_STD}, ac_tables={0: js.AC_STD}, qtables={0: js.q(52)})
    assert np.array_equal(jf.pil_decode(f), jf.pil_decode(streams["ac-run-past-63"]))


def test_bad_code_mid_interval_is_a_warning_in_pil_and_an_error_in_the_oracle():
    """libjpeg decodes an invalid code as a zero and goes on, so PIL returns pixels; the decoder reports the file instead, which
    its contract allows (a status, never silently other pixels)."""
    d = {n: d for n, d, _, _ in js.contract_streams()}["bad-code-mid-interval"]
    with pytest.raises(ValueError):
        jo.decode(d)
    assert _pil(d) is not None


def test_the_zero_ac_rows_shortcut_of_the_simd_idct():
    """libjpeg-turbo's SIMD pass 1 takes a block whose coefficient rows 1 .. 7 are zero as row 0 shifted left by 2 in 16 bits, which
    wraps; the full pass would saturate.  A dequantised row-0 value past 8191 tells the two apart."""
    g = [jw.Comp(1)]
    cf = np.zeros((1, 4, 64), np.int64)
    cf[0, :, 0] = [9000, -9000, 3000, 12000]
    cf[0, 0, 3] = 700                                                 # row 0 only: the shortcut
    cf[0, 2, 8] = 1                                                   # a row-1 coefficient: the full pass
    cf[0, 3, 2] = -15000
    f, log = jw.write_jpeg(8, 32, g, [cf], dc_tables={0: js.DC_STD}, ac_tables={0: js.AC_STD}, qtables={0: [1] * 64})
    pil = jf.pil_decode(f)
    assert np.array_equal(jo.decode(f), pil)
    full = jo.range_limit(jo._idct_1d(jo._idct_1d(cf[0].reshape(-1, 8, 8), 11).transpose(0, 2, 1), 18).transpose(0, 2, 1))
    assert not np.array_equal(full[0], pil[:, 0:8, 0])               # the full pass alone would differ on the shortcut blocks
