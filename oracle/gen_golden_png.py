"""Writes tests/golden/png_fixtures.npz: small Pillow-written PNG files of every supported mode (and a few written from the deflate
specification) with the SHA-256 of PIL's pixels, np.array(Image.open(f).convert('RGB')).  Run from the repository root:
python oracle/gen_golden_png.py"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import png_fixtures as pf  # noqa: E402
from oracle import png_oracle as po  # noqa: E402


def main():
    picked = [(n, d) for n, d in pf.matrix() if n.startswith(("17x9-", "3x13-")) or n in ("level0", "level9", "optimize-P",
                                                                                        "strategy-rle-ct4", "stored-fixed-dynamic",
                                                                                        "fixed-only", "false-candidate")]
    arrays = {"names": np.array([n for n, _ in picked]), "sha256": np.array([])}
    shas = []
    for i, (name, data) in enumerate(picked):
        pil = pf.pil_decode(data)
        assert np.array_equal(po.decode(data), pil), name
        arrays[f"file_{i}"] = np.frombuffer(data, np.uint8)
        shas.append(hashlib.sha256(pil.tobytes()).hexdigest())
    arrays["sha256"] = np.array(shas)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "png_fixtures.npz"), **arrays)
    print(f"{len(picked)} files")


if __name__ == "__main__":
    main()
