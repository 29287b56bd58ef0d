"""Writes tests/golden/jpeg_fixtures.npz: small JPEG files encoded by Pillow from seeded synthetic images (tests/jpeg_fixtures.py),
one per subsampling, quality extreme and option, with the SHA-256 of PIL's decoded pixels.  Data only: the tests decode the files
with PIL, the oracle and the GPU and compare.

    python oracle/gen_golden_jpeg.py
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import jpeg_fixtures as jf  # noqa: E402

CASES = [((7, 13), "420", 5, "sat", {}), ((17, 33), "422", 100, "noise", {}), ((16, 16), "444", 75, "edges", {"optimize": True}),
         ((33, 65), "420", 95, "grad", {"restart_marker_blocks": 1}), ((40, 24), "gray", 50, "noise", {"restart_marker_rows": 1}),
         ((1, 1), "420", 75, "sat", {}), ((3, 5), "422", 90, "noise", {}), ((64, 48), "420", 100, "sat", {"optimize": True}),
         ((24, 40), "444", 5, "noise", {"restart_marker_rows": 2}), ((9, 4), "420", 50, "edges", {}),
         ((48, 80), "gray", 100, "edges", {"optimize": True, "restart_marker_blocks": 5}), ((30, 30), "422", 25, "grad", {})]


def main():
    out = {}
    names, shas = [], []
    for i, ((h, w), sub, q, kind, kw) in enumerate(CASES):
        data = jf.encode(jf.image(h, w, kind, seed=100 + i), sub, q, **kw)
        names.append(f"{h}x{w}-{sub}-q{q}-{kind}-" + ",".join(f"{k}={v}" for k, v in kw.items()))
        shas.append(hashlib.sha256(jf.pil_decode(data).tobytes()).hexdigest())
        out[f"file_{i}"] = np.frombuffer(data, np.uint8)
    path = os.path.join(ROOT, "tests", "golden", "jpeg_fixtures.npz")
    np.savez_compressed(path, names=np.array(names), sha256=np.array(shas), **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
