"""Writes tests/golden/clip_tower_l3.npz from transformers' CLIPVisionModel (full width, 3 layers, one crop, the oracle's seeded
weights): hidden_states[0..3] at a few sampled token rows, so that tests/test_clip_tower_host.py pins the oracle without transformers.

    python oracle/gen_golden_clip_tower.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import clip_tower_oracle as cto  # noqa: E402

WEIGHT_SEED, IMAGE_SEED = 4, 5
ROWS = [0, 1, 24, 288, 300, 575, 576]


def main():
    import transformers
    cfg = transformers.CLIPVisionConfig(hidden_size=1024, intermediate_size=4096, num_attention_heads=16, num_hidden_layers=3,
                                        image_size=336, patch_size=14, hidden_act="quick_gelu", layer_norm_eps=1e-5)
    model = transformers.CLIPVisionModel(cfg).eval()
    model.load_state_dict({"vision_model." + k: v for k, v in cto.make_weights(3, seed=WEIGHT_SEED).items()}, strict=False)
    with torch.no_grad():
        hs = model(pixel_values=cto.make_images(1, seed=IMAGE_SEED), output_hidden_states=True).hidden_states
    out = {"weight_seed": np.int64(WEIGHT_SEED), "image_seed": np.int64(IMAGE_SEED), "rows": np.array(ROWS, dtype=np.int64),
           "transformers_version": np.array(transformers.__version__)}
    for i in range(4):
        out[f"hs{i}"] = hs[i][0, ROWS].numpy().astype(np.float32)
    path = os.path.join(ROOT, "tests", "golden", "clip_tower_l3.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
