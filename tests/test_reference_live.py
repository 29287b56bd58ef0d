"""Randomised comparison against what the REFERENCE ITSELF returned on cases beyond the fixed fixtures (tests/golden/
reference_live.npz, written by oracle/gen_golden_live.py from the reference tree).  Widens the pin of the oracle and of the
product's host logic: the seeds are fixed but different from the fixture seeds.  Inputs that regenerate from a seed are not
stored; the tiling crops and the parameter gradients are stored as seeded samples plus their global magnitudes."""
import os

import numpy as np
import pytest

from oracle.gen_golden_live import GRADIENT_CASES, GRAD_SAMPLES, PROJECTOR_CASES, TILE_SAMPLES, sample_index


@pytest.fixture(scope="module")
def live(golden_dir):
    with np.load(os.path.join(golden_dir, "reference_live.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("s,hidden,seed", PROJECTOR_CASES)
def test_oracle_vs_reference_module(live, s, hidden, seed):
    """Fresh weights (every 1-D parameter perturbed so LayerNorm / bias paths matter), odd hidden sizes, N=2."""
    import torch
    from oracle import tokenpacker_oracle as tpo
    from oracle import torch_port
    params = tpo.make_params(hidden, seed=seed)
    x0, xm = tpo.make_inputs(2, seed=seed + 1000)
    ref = live[f"proj_{s}_{hidden}_{seed}"]
    with torch.no_grad():
        port = torch_port.forward({k: torch.from_numpy(v) for k, v in params.items()}, torch.from_numpy(x0), torch.from_numpy(xm), s).numpy()
    out = tpo.tokenpacker_forward(params, x0, xm, s)
    assert out.shape == ref.shape and port.shape == ref.shape
    assert np.abs(out - ref).max() < 5e-6
    assert np.abs(port - ref).max() < 1e-6


def test_grid_selector_vs_reference_random(live):
    """Product (C ABI, host arithmetic) and oracle vs Image_Patch.calculate on 600 fresh sizes incl. extreme aspect ratios."""
    from oracle import hd_oracle as hdo
    from tokenpacker_b200 import hd_grid
    for patch_num in (9, 16, 25):
        sizes, wants = live[f"grid_{patch_num}_sizes"], live[f"grid_{patch_num}_want"]
        assert len(sizes) == 200
        for (h, w), want in zip(sizes.tolist(), wants.tolist()):
            want = tuple(want)
            assert hd_grid(h, w, patch_num) == want, (h, w, patch_num)
            assert tuple(hdo.hd_grid(h, w, patch_num)) == want, (h, w, patch_num)


@pytest.mark.parametrize("start_end", [False, True])
def test_splice_vs_reference_method_random(live, start_end):
    """Random batches through the reference's prepare_inputs_labels_for_multimodal vs the oracle AND the product's host planner
    (llava_arch.py:100-233, both mm_use_im_start_end branches, 'pad' and 'slice' modes, ragged and image-free samples)."""
    from oracle import hd_oracle as hdo
    from oracle import splice_oracle as spo
    from tokenpacker_b200 import splice_plan
    table = live[f"splice_{int(start_end)}_table"]
    hdim = table.shape[1]
    for trial in range(40):
        key = f"splice_{int(start_end)}_{trial}"
        ids, feats = live[key + "_ids"], live[key + "_feats"]
        ref_mask, ref_embeds, ref_labels = live[key + "_mask"], live[key + "_embeds"], live[key + "_labels"]
        B = ids.shape[0]
        labels = ids.copy()
        mask = np.ones_like(ids, dtype=bool)
        if key + "_grids" in live:
            grids = live[key + "_grids"].tolist()
            hb, wb = [g[0] for g in grids], [g[1] for g in grids]
            packed, cu = hdo.hd_assemble(feats, hb, wb, table[5], table[6])
            seqs = [packed[cu[i]:cu[i + 1]] for i in range(B)]
        else:
            seqs = [feats[i] for i in range(feats.shape[0])]
        o_mask, o_embeds, o_labels = spo.splice(ids, mask, labels, seqs, table, im_start_end=start_end)
        np.testing.assert_array_equal(o_embeds, ref_embeds)
        np.testing.assert_array_equal(o_labels, ref_labels)
        np.testing.assert_array_equal(o_mask, ref_mask)
        visual = np.concatenate(seqs, axis=0)
        cu_seq = np.concatenate([[0], np.cumsum([q.shape[0] for q in seqs])])
        plan = splice_plan(ids, cu_seq, labels, mask, im_start_end=start_end)
        rows = np.zeros((plan.src_index.shape[0], hdim), dtype=np.float32)
        src = plan.src_index
        rows[src >= 0] = table[src[src >= 0]]
        rows[src <= -2] = visual[-src[src <= -2] - 2]
        np.testing.assert_array_equal(rows.reshape(B, plan.lmax, hdim), ref_embeds)
        np.testing.assert_array_equal(plan.labels, ref_labels)
        np.testing.assert_array_equal(plan.attention_mask, ref_mask)


def test_tiling_block_vs_reference_source_random(live):
    """The resize -> pad -> split -> thumbnail block has no function boundary upstream (pasted inline 9 times); what the source
    range eval/model_vqa.py:88-123 returned on fresh image sizes vs the oracle restatement: grid, shape, a seeded sample of
    values, every crop-channel sum and the largest magnitude."""
    from oracle import hd_oracle as hdo
    rng = np.random.default_rng(515)
    for trial in range(18):
        patch_num = (9, 16, 25)[trial % 3]
        h, w = (int(v) for v in rng.integers(40, 1500, size=2))
        img = rng.standard_normal((3, h, w)).astype(np.float32)
        meta = live[f"tile_{trial}_meta"].tolist()
        assert meta[:3] == [h, w, patch_num]
        crops, hb, wb = hdo.hd_tile(img[None], patch_num)
        assert (hb, wb) == (meta[3], meta[4])
        assert list(crops.shape) == meta[5:], (crops.shape, meta[5:])
        got = crops.reshape(-1)[sample_index(crops.size, TILE_SAMPLES, trial)]
        assert np.abs(got - live[f"tile_{trial}_sample"]).max() <= 2e-6, (h, w, patch_num)
        sums = crops.astype(np.float64).sum(axis=(2, 3))
        assert np.abs(sums - live[f"tile_{trial}_sums"]).max() <= 2e-6 * crops.shape[2] * crops.shape[3], (h, w, patch_num)
        assert abs(float(np.abs(crops).max()) - float(live[f"tile_{trial}_absmax"])) <= 2e-6


@pytest.mark.parametrize("s,hidden,seed", GRADIENT_CASES)
def test_gradient_oracle_vs_reference_autograd(live, s, hidden, seed):
    """tests/test_backward_gpu.py uses autograd over oracle/torch_port.py as the gradient oracle: pin THAT to autograd through the
    reference module itself (fp32, CPU), every parameter (a seeded sample of each gradient and its largest magnitude)."""
    import torch
    from oracle import tokenpacker_oracle as tpo
    from oracle import torch_port
    params = tpo.make_params(hidden, seed=seed)
    x0, xm = tpo.make_inputs(2, seed=seed + 1000)
    x0, xm = torch.from_numpy(x0), torch.from_numpy(xm)
    gw = torch.from_numpy(np.random.default_rng(seed).standard_normal((2, (24 // s) ** 2, hidden)).astype(np.float32))
    p = {k: torch.from_numpy(v).clone().requires_grad_(True) for k, v in params.items()}
    (torch_port.forward(p, x0, xm, s) * gw).sum().backward()
    for i, name in enumerate(params):          # the reference module's named_parameters() order (its state_dict keys)
        g = p[name].grad.numpy().reshape(-1)
        key = f"grad_{s}_{hidden}_{seed}_{name}"
        scale = float(live[key + "_absmax"]) + 1e-12
        g_ref = live[key + "_sample"]
        err = float(np.abs(g[sample_index(g.size, GRAD_SAMPLES, seed * 100 + i)] - g_ref).max())
        assert err <= 2e-5 * scale + 1e-7, (name, err, scale)
        assert abs(float(np.abs(g).max()) - scale) <= 2e-5 * scale + 1e-7, (name, float(np.abs(g).max()), scale)


def test_slice_assembly_vs_reference_source_random(live):
    """What llava_arch.py:141-155 returned on random grids vs the oracle and the product's host plan (tp_hd_plan)."""
    from oracle import hd_oracle as hdo
    from tokenpacker_b200 import hd_plan
    for trial in range(20):
        key = f"assembly_{trial}"
        grids = live[key + "_grids"].tolist()
        sep_row, ret_row = live[key + "_rows"]
        feats, want, want_cu = live[key + "_feats"], live[key + "_want"], live[key + "_cu"]
        m = feats.shape[1]
        hb, wb = [g[0] for g in grids], [g[1] for g in grids]
        packed, cu = hdo.hd_assemble(feats, hb, wb, sep_row, ret_row)
        np.testing.assert_array_equal(packed, want)
        np.testing.assert_array_equal(cu, want_cu)
        plan = hd_plan(hb, wb, m)
        np.testing.assert_array_equal(plan.cu_seqlens.numpy(), want_cu)
        rebuilt = np.full_like(want, np.nan)
        for c, r0 in enumerate(plan.seg_row_offset.tolist()):
            rebuilt[r0:r0 + m] = feats[c]
        rebuilt[plan.sep_rows.numpy()] = sep_row
        rebuilt[plan.ret_rows.numpy()] = ret_row
        np.testing.assert_array_equal(rebuilt, want)
