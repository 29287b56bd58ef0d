"""Generate tests/golden/reference_live.npz from the REFERENCE ITSELF: the randomised cases of tests/test_reference_live.py.

    python oracle/gen_golden_live.py REFERENCE_TREE

Like oracle/gen_golden.py, the reference modules are imported by file path (and two inline source ranges exec'd) where they
lie; nothing is copied.  Stored per case: the inputs the test cannot regenerate from a seed, and what the reference returned.
Outputs larger than a fixture should hold are stored as a seeded sample plus their global maximum magnitude (the tiling
crops: samples and per-crop-channel sums; the parameter gradients: samples and max |g|).
"""
from __future__ import annotations

import importlib
import importlib.util
import os
import sys
import textwrap
import types

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import hd_oracle as hdo            # noqa: E402
from oracle import tokenpacker_oracle as tpo  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "reference_live.npz")

PROJECTOR_CASES = [(2, 64, 901), (3, 96, 902), (4, 160, 903), (6, 32, 904), (12, 64, 905)]
GRADIENT_CASES = [(2, 64, 911), (3, 32, 912), (4, 96, 913), (8, 32, 914)]
GRAD_SAMPLES = 256
TILE_SAMPLES = 2048


def sample_index(n, k, seed):
    """The fixed sample of flat indices both the generator and the test use."""
    return np.sort(np.random.default_rng(seed).choice(n, size=min(n, k), replace=False))


def main(ref):
    def by_path(name, rel):
        spec = importlib.util.spec_from_file_location(name, os.path.join(ref, rel))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod

    builder = by_path("ref_builder_live", "llava/model/multimodal_projector/builder.py")
    patch_divide = by_path("ref_patch_divide_live", "llava/patch_divide.py")
    for name, sub in (("llava", "llava"), ("llava.model", "llava/model")):      # bypass the two __init__.py (transformers-4.31 imports)
        if name not in sys.modules:
            mod = types.ModuleType(name)
            mod.__path__ = [os.path.join(ref, sub)]
            sys.modules[name] = mod
    arch = importlib.import_module("llava.model.llava_arch")
    out = {}

    # projector forward: fresh weights, odd hidden sizes, N=2 (inputs regenerate from the seeds)
    for s, hidden, seed in PROJECTOR_CASES:
        params = tpo.make_params(hidden, seed=seed)
        x0, xm = tpo.make_inputs(2, seed=seed + 1000)
        m = builder.TokenPacker(hidden_size=hidden, scale_factor=s)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
        with torch.no_grad():
            out[f"proj_{s}_{hidden}_{seed}"] = m.eval()((torch.from_numpy(x0), torch.from_numpy(xm))).numpy()

    # grid selector: 600 sizes incl. extreme aspect ratios
    rng = np.random.default_rng(4242)
    for patch_num in (9, 16, 25):
        ip = patch_divide.Image_Patch(image_size=336, patch_num=patch_num)
        sizes = [tuple(int(v) for v in rng.integers(16, 3200, size=2)) for _ in range(170)]
        sizes += [(int(rng.integers(16, 200)), int(rng.integers(2000, 6000))) for _ in range(15)]
        sizes += [(int(rng.integers(2000, 6000)), int(rng.integers(16, 200))) for _ in range(15)]
        out[f"grid_{patch_num}_sizes"] = np.array(sizes, dtype=np.int64)
        out[f"grid_{patch_num}_want"] = np.array([[int(v) for v in ip.calculate(h, w)] for h, w in sizes], dtype=np.int64)

    # splice: random batches through prepare_inputs_labels_for_multimodal (both im_start_end branches, pad and slice modes)
    for start_end in (False, True):
        rng = np.random.default_rng(77 if start_end else 78)
        hdim, vocab, m = 8, 40, 3
        table = rng.standard_normal((vocab, hdim)).astype(np.float32)
        out[f"splice_{int(start_end)}_table"] = table
        for trial in range(40):
            B, L = int(rng.integers(1, 4)), int(rng.integers(6, 12))
            slice_mode = (not start_end) and trial % 2 == 1
            ids = rng.integers(7, vocab, size=(B, L))
            n_img = []
            for b in range(B):
                k = 1 if slice_mode else int(rng.integers(0, 3))
                if start_end:
                    # <im_start> IMAGE <im_end> triples (30 / 31 stand-ins), never at position 0 (upstream always has a BOS first)
                    pos = sorted(rng.choice(np.arange(2, L - 1, 3), size=min(k, (L - 3) // 3), replace=False).tolist())
                    for p in pos:
                        ids[b, p - 1], ids[b, p], ids[b, p + 1] = 30, -200, 31
                    n_img.append(len(pos))
                else:
                    pos = sorted(rng.choice(L, size=k, replace=False).tolist())
                    ids[b, pos] = -200
                    n_img.append(k)
            labels = ids.copy()
            mask = np.ones_like(ids, dtype=bool)
            if slice_mode:
                grids = [(int(rng.integers(1, 4)), int(rng.integers(1, 4))) for _ in range(B)]
                crops = sum(hdo.n_crops(a, b) for a, b in grids)
                feats = rng.standard_normal((crops, m, hdim)).astype(np.float32)
                hb, wb = [g[0] for g in grids], [g[1] for g in grids]
                mode = "slice"
            else:
                n_seq = sum(max(k, 1) for k in n_img)          # an image-free sample still consumes one (llava_arch.py:121-134)
                feats = rng.standard_normal((n_seq, m, hdim)).astype(np.float32)
                hb = wb = None
                mode = "pad"
            fake = _fake_model(arch, torch.from_numpy(table), torch.from_numpy(feats), start_end)
            _, ref_mask, _, ref_embeds, ref_labels = fake.prepare_inputs_labels_for_multimodal(
                torch.from_numpy(ids), torch.from_numpy(mask), None, torch.from_numpy(labels), object(), mode, hb, wb)
            key = f"splice_{int(start_end)}_{trial}"
            out[key + "_ids"] = ids
            out[key + "_feats"] = feats
            if slice_mode:
                out[key + "_grids"] = np.array(grids, dtype=np.int64)
            out[key + "_mask"] = ref_mask.numpy()
            out[key + "_embeds"] = ref_embeds.numpy()
            out[key + "_labels"] = ref_labels.numpy()

    # tiling block: eval/model_vqa.py:88-123 exec'd where it lies on fresh image sizes
    with open(os.path.join(ref, "llava/eval/model_vqa.py")) as f:
        src = textwrap.dedent("".join(f.readlines()[87:123]))
    assert src.lstrip().startswith("image = preprocess(image)")
    rng = np.random.default_rng(515)
    for trial in range(18):
        patch_num = (9, 16, 25)[trial % 3]
        h, w = (int(v) for v in rng.integers(40, 1500, size=2))
        img = rng.standard_normal((3, h, w)).astype(np.float32)
        ns = {"image": torch.from_numpy(img), "preprocess": (lambda t: t),
              "image_patch": patch_divide.Image_Patch(image_size=336, patch_num=patch_num), "F": F, "torch": torch}
        exec(src, ns)
        want = ns["image_tensor"].numpy()
        key = f"tile_{trial}"
        out[key + "_meta"] = np.array([h, w, patch_num, int(ns["h_block"]), int(ns["w_block"])] + list(want.shape), dtype=np.int64)
        out[key + "_sample"] = want.reshape(-1)[sample_index(want.size, TILE_SAMPLES, trial)]
        out[key + "_sums"] = want.astype(np.float64).sum(axis=(2, 3))
        out[key + "_absmax"] = np.array(np.abs(want).max(), dtype=np.float32)

    # parameter gradients through the reference module (fp32, CPU)
    for s, hidden, seed in GRADIENT_CASES:
        params = tpo.make_params(hidden, seed=seed)
        x0, xm = tpo.make_inputs(2, seed=seed + 1000)
        gw = torch.from_numpy(np.random.default_rng(seed).standard_normal((2, (24 // s) ** 2, hidden)).astype(np.float32))
        m = builder.TokenPacker(hidden_size=hidden, scale_factor=s)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
        (m((torch.from_numpy(x0), torch.from_numpy(xm))) * gw).sum().backward()
        for i, (name, p) in enumerate(m.named_parameters()):
            g = p.grad.numpy().reshape(-1)
            key = f"grad_{s}_{hidden}_{seed}_{name}"
            out[key + "_sample"] = g[sample_index(g.size, GRAD_SAMPLES, seed * 100 + i)]
            out[key + "_absmax"] = np.array(np.abs(g).max(), dtype=np.float32)

    # slice assembly: llava_arch.py:141-155 exec'd where it lies on random grids
    with open(os.path.join(ref, "llava/model/llava_arch.py")) as f:
        src = textwrap.dedent("".join(f.readlines()[140:155]))
    assert src.lstrip().startswith("image_feature_list = []")
    rng = np.random.default_rng(606)
    for trial in range(20):
        m, hdim = int(rng.integers(1, 6)), 4
        grids = [(int(rng.integers(1, 6)), int(rng.integers(1, 6))) for _ in range(int(rng.integers(1, 6)))]
        sep_row = rng.standard_normal(hdim).astype(np.float32)
        ret_row = rng.standard_normal(hdim).astype(np.float32)
        total = sum(hdo.n_crops(a, b) for a, b in grids)
        feats = rng.standard_normal((total, m, hdim)).astype(np.float32)

        class _Model:
            def embed_tokens(self, tok):
                return torch.from_numpy(sep_row if int(tok[0]) == 0 else ret_row)[None]

        class _Self:
            def get_model(self):
                return _Model()

        ns = {"image_features": torch.from_numpy(feats), "h_block": [g[0] for g in grids], "w_block": [g[1] for g in grids],
              "self": _Self(), "sep": torch.tensor([0]), "ret": torch.tensor([1]), "torch": torch, "cur_image_idx": 0}
        want = []
        for b in range(len(grids)):
            ns["batch_idx"] = b
            exec(src, ns)
            want.append(ns["cur_image_features"].numpy())
        key = f"assembly_{trial}"
        out[key + "_grids"] = np.array(grids, dtype=np.int64)
        out[key + "_rows"] = np.stack([sep_row, ret_row])
        out[key + "_feats"] = feats
        out[key + "_cu"] = np.concatenate([[0], np.cumsum([q.shape[0] for q in want])]).astype(np.int64)
        out[key + "_want"] = np.concatenate(want, axis=0)

    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out)} arrays, {os.path.getsize(OUT)} bytes")


def _fake_model(arch, table, feats, start_end):
    class _Model:
        def embed_tokens(self, ids):
            return table[ids]

    class _Tok:
        def convert_tokens_to_ids(self, toks):
            return [{",": 5, "\n": 6}[t] for t in toks]

    class _Fake(arch.LlavaMetaForCausalLM):
        def __init__(self):
            self._m, self.tokenizer = _Model(), _Tok()
            self.config = types.SimpleNamespace(tune_mm_mlp_adapter=start_end, mm_use_im_start_end=start_end)
            self.device = torch.device("cpu")

        def get_model(self):
            return self._m

        def get_vision_tower(self):
            return object()

        def encode_images(self, images):
            return feats

    return _Fake()


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
