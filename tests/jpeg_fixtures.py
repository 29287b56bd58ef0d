"""Seeded synthetic images and their JPEG encodings by Pillow, shared by the JPEG decoder's tests."""
from __future__ import annotations

import io
import itertools

import numpy as np
from PIL import Image

SIZES = [(1, 1), (7, 13), (8, 8), (16, 16), (17, 33), (333, 517), (1000, 1024), (1345, 224)]
SUBSAMPLING = {"444": 0, "422": 1, "420": 2, "gray": None}
QUALITIES = [5, 50, 75, 95, 100]
KINDS = ["grad", "noise", "edges", "sat"]


def image(h: int, w: int, kind: str, seed: int) -> np.ndarray:
    """uint8 [h, w, 3]: smooth gradients, noise, sharp edges or saturated colour blocks (every range-limit clamp fires)."""
    r = np.random.default_rng(seed)
    if kind == "noise":
        return r.integers(0, 256, (h, w, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    if kind == "grad":
        a = np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1), (xx + yy) * 255 // max(h + w - 2, 1)], 2)
        return a.astype(np.uint8)
    if kind == "edges":
        a = np.zeros((h, w, 3), np.uint8)
        a[(xx // 3 + yy // 5) % 2 == 1] = (255, 0, 255)
        a[(xx // 7) % 3 == 0, 1] = 255
        return a
    cols = np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255], [255, 255, 0], [0, 255, 255], [255, 0, 255], [0, 0, 0], [255, 255, 255]],
                    np.uint8)
    return cols[r.integers(0, 8, (h // 4 + 1, w // 4 + 1))].repeat(4, 0).repeat(4, 1)[:h, :w]


def encode(a: np.ndarray, sub: str, quality: int, **kw) -> bytes:
    b = io.BytesIO()
    if sub == "gray":
        Image.fromarray(a).convert("L").save(b, "JPEG", quality=quality, **kw)
    else:
        Image.fromarray(a).save(b, "JPEG", quality=quality, subsampling=SUBSAMPLING[sub], **kw)
    return b.getvalue()


def pil_decode(data: bytes) -> np.ndarray:
    return np.array(Image.open(io.BytesIO(data)).convert("RGB"))


def qtables16(top: int):
    """Two quantisation tables rising from 1 to top along the zigzag order: Pillow writes them as 16-bit DQT (Pq = 1) when top > 255."""
    ramp = [max(1, round(top * (k / 63) ** 2)) for k in range(64)]
    return [ramp, [min(top, 2 * v) for v in ramp]]


def with_adobe(data: bytes, transform: int) -> bytes:
    """data with an APP14 'Adobe' segment of the given colour transform inserted after its APP0 (JFIF) segment."""
    assert data[2:4] == b"\xff\xe0"
    end = 4 + ((data[4] << 8) | data[5])
    app14 = b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00" + bytes([transform])
    return data[:end] + app14 + data[end:]


def matrix(big: bool = True):
    """(name, bytes) over the fixture matrix: every size x subsampling x quality at one content and option set each, rotating the
    contents, optimize on / off and the restart options, so that each appears at every size.  big=False leaves out the two
    largest sizes."""
    out = []
    opts = [{}, {"optimize": True}, {"restart_marker_blocks": 3}, {"restart_marker_rows": 1}, {"optimize": True, "restart_marker_rows": 2}]
    for n, ((h, w), sub, q) in enumerate(itertools.product(SIZES, SUBSAMPLING, QUALITIES)):
        if not big and h * w > 400_000:
            continue
        kind = KINDS[n % len(KINDS)]
        kw = opts[(n // len(KINDS)) % len(opts)]
        a = image(h, w, kind, seed=n)
        out.append((f"{h}x{w}-{sub}-q{q}-{kind}-" + ",".join(f"{k}={v}" for k, v in kw.items()), encode(a, sub, q, **kw)))
    # 16-bit quantisation tables
    for n, ((h, w), sub, top) in enumerate(itertools.product([(17, 33), (333, 517)], ["444", "420", "gray"], [300, 2000, 30000])):
        kind = KINDS[n % len(KINDS)]
        b = io.BytesIO()
        im = Image.fromarray(image(h, w, kind, seed=500 + n))
        if sub == "gray":
            im.convert("L").save(b, "JPEG", qtables=qtables16(top)[:1])
        else:
            im.save(b, "JPEG", qtables=qtables16(top), subsampling=SUBSAMPLING[sub])
        out.append((f"{h}x{w}-{sub}-dqt16-top{top}-{kind}", b.getvalue()))
    return out
