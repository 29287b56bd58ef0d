"""Full-size parity: the CUDA path at BASELINE.json's own sizes (configs[1] N=64 s=2, configs[2] N=128 s in {2,3,4},
configs[3] 231 HD crops packed) against the oracle's torch port run IN FP32 ON THE GPU (TF32 off: the reference's op
sequence, builder.py:107-137, in full fp32 arithmetic — the port is pinned to reference-generated fixtures and to the live
reference by tests/test_oracle.py / tests/test_reference_live.py).  EVERY output row is compared.

Tolerances (bf16 storage + fp32 accumulation vs the fp32 oracle on identical bf16-rounded weights and inputs, output RMS ~0.1):
forward rel-RMS <= 4e-3 and max-abs <= 5e-3 at H=4096 (the error grows with the width of the last two linears — 2.0e-3 / 1.3e-3
at H=256, measured on an H100 — and the reference's own bf16 forward sits at
4.6e-3..5.3e-3 / up to 4.9e-3 on the same inputs); parameter gradients at H=4096, N=8: <= 1.5 % rel-RMS each.
"""
import numpy as np
import pytest
import torch

from oracle import hd_oracle as hdo
from oracle import torch_port

pytestmark = pytest.mark.gpu

REL_RMS_TOL = 4e-3
MAX_ABS_TOL = 5e-3


@pytest.fixture(autouse=True)
def _fp32_exact():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, torch.get_float32_matmul_precision())
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old[0], old[1]
    torch.set_float32_matmul_precision(old[2])
    torch.cuda.empty_cache()


def _module(hidden, s, seed=0):
    from tokenpacker_b200 import TokenPackerB200
    from tokenpacker_b200 import synthetic as syn
    sd = {k: torch.from_numpy(v).bfloat16() for k, v in syn.synthetic_state_dict(hidden, seed=seed).items()}
    m = TokenPackerB200(hidden_size=hidden, scale_factor=s)
    m.load_state_dict(sd)
    return m.to("cuda", torch.bfloat16).eval(), {k: v.float().cuda() for k, v in sd.items()}


def _inputs(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x0 = torch.randn(n, 576, 1024, device="cuda", generator=g).bfloat16()
    xm = torch.randn(n, 576, 4096, device="cuda", generator=g).bfloat16()
    return x0, xm


def _oracle_fp32(p32, x0, xm, s, chunk=32):
    """the fp32 port over the whole batch (chunked only to bound the fp32 intermediates; crops are independent)"""
    outs = []
    with torch.no_grad():
        for i in range(0, x0.shape[0], chunk):
            outs.append(torch_port.forward(p32, x0[i:i + chunk].float(), xm[i:i + chunk].float(), s))
    return torch.cat(outs)


def _check(out, ref):
    assert out.shape == ref.shape
    d = out.float() - ref
    rel = float(d.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())
    mx = float(d.abs().max())
    # per-row check as well: no single crop / token may hide behind the batch average
    row_rel = d.pow(2).mean(-1).sqrt() / ref.pow(2).mean(-1).sqrt().clamp_min(1e-6)
    assert rel <= REL_RMS_TOL and mx <= MAX_ABS_TOL and float(row_rel.max()) <= 3 * REL_RMS_TOL, (rel, mx, float(row_rel.max()))
    return rel, mx


def test_configs1_n64_s2_every_row():
    m, p32 = _module(4096, 2)
    x0, xm = _inputs(64, 1234)
    with torch.no_grad():
        out = m((x0, xm))
    assert out.shape == (64, 144, 4096) and out.is_contiguous()
    _check(out, _oracle_fp32(p32, x0, xm, 2))


@pytest.mark.parametrize("s", [2, 3, 4])
def test_configs2_n128_scale_sweep_every_row(s):
    m, p32 = _module(4096, s)
    x0, xm = _inputs(128, 77 + s)
    with torch.no_grad():
        out = m((x0, xm))
    assert out.shape == (128, (24 // s) ** 2, 4096)
    _check(out, _oracle_fp32(p32, x0, xm, s))


def test_configs3_hd_231_crops_packed_every_row():
    """patch_num=9, s=2, 32 seeded image sizes -> 231 crops: the packed output (TMA stores at crop stride M+1 + separator fill)
    against the fp32 port's crop blocks assembled by the oracle's restatement of llava_arch.py:139-155."""
    from tokenpacker_b200 import hd_grid
    g = torch.Generator().manual_seed(0)
    hs = torch.randint(224, 1345, (32,), generator=g).tolist()
    ws = torch.randint(224, 1345, (32,), generator=g).tolist()
    grids = [hd_grid(h, w, 9) for h, w in zip(hs, ws)]
    n = sum(hdo.n_crops(a, b) for a, b in grids)
    assert n == 231
    m, p32 = _module(4096, 2)
    x0, xm = _inputs(n, 5)
    gg = torch.Generator(device="cuda").manual_seed(6)
    sep = torch.randn(4096, device="cuda", generator=gg).bfloat16()
    ret = torch.randn(4096, device="cuda", generator=gg).bfloat16()
    hb, wb = [a for a, _ in grids], [b for _, b in grids]
    with torch.no_grad():
        packed, cu = m.forward_packed((x0, xm), hb, wb, sep, ret)
    feats = _oracle_fp32(p32, x0, xm, 2)
    ref, ref_cu = hdo.hd_assemble(feats.cpu().numpy(), hb, wb, sep.float().cpu().numpy(), ret.float().cpu().numpy())
    np.testing.assert_array_equal(cu.numpy(), ref_cu)
    _check(packed, torch.from_numpy(ref).cuda())
    # separator rows are pure copies: bit-exact
    plan_rows = torch.from_numpy(ref).cuda()
    is_sep = (plan_rows == sep.float()).all(-1) | (plan_rows == ret.float()).all(-1)
    assert int(is_sep.sum()) == n and torch.equal(packed[is_sep].float(), plan_rows[is_sep])


def test_gradients_h4096_n8():
    """Every parameter gradient at the real width (H=4096, N=8, s=2) against autograd over the fp32 port."""
    m, p32 = _module(4096, 2, seed=3)
    m.train()
    x0, xm = _inputs(8, 9)
    gen = torch.Generator(device="cuda").manual_seed(5)
    gw = torch.randn(8, 144, 4096, device="cuda", generator=gen).bfloat16()
    out = m((x0, xm))
    (out.float() * gw.float()).sum().backward()
    ref_p = {k: v.clone().requires_grad_(True) for k, v in p32.items()}
    ref_out = torch_port.forward(ref_p, x0.float(), xm.float(), 2)
    (ref_out * gw.float()).sum().backward()
    _check(out.detach(), ref_out.detach())
    worst = {}
    for name, p in m.named_parameters():
        gq, r = p.grad.float(), ref_p[name].grad
        assert gq.shape == r.shape and torch.isfinite(gq).all(), name
        worst[name] = (float((gq - r).pow(2).mean().sqrt()), float(r.pow(2).mean().sqrt()))
    # ln_k_1.bias and the k slice of in_proj_bias have analytically ZERO gradients (softmax is shift-invariant per window):
    # they are compared against rounding noise, bounded at 1 % of the k branch's own first-layer bias gradient
    floor = 1e-2 * worst["k_proj_1.0.bias"][1]
    bad = {k: (e, r) for k, (e, r) in worst.items() if e > 1.5e-2 * r + floor}
    assert not bad, (bad, worst)


@pytest.mark.parametrize("s,hidden", [(2, 512), (3, 256), (4, 512), (4, 4096)])
def test_packed_rows_pair_kernel_bit_exact(s, hidden, monkeypatch):
    """The 3-D clipped-box TMA stores of the packed layout (crop stride M+1) for M = 144 / 64 / 36, including a ragged last
    tile and grids of every shape: bit-identical to projecting densely and scattering afterwards.  TP_GEMM_MODE=2 forces the
    CTA-pair kernel (the one with TMA stores) even at these small sizes."""
    from tokenpacker_b200 import hd_assemble
    monkeypatch.setenv("TP_GEMM_MODE", "2")
    grids = [(1, 1), (2, 3), (3, 1), (1, 2), (2, 2)]
    n = sum(hdo.n_crops(a, b) for a, b in grids)
    m, _ = _module(hidden, s, seed=11)
    x0, xm = _inputs(n, 13)
    gg = torch.Generator(device="cuda").manual_seed(2)
    sep = torch.randn(hidden, device="cuda", generator=gg).bfloat16()
    ret = torch.randn(hidden, device="cuda", generator=gg).bfloat16()
    hb, wb = [a for a, _ in grids], [b for _, b in grids]
    with torch.no_grad():
        packed, cu = m.forward_packed((x0, xm), hb, wb, sep, ret)
        packed2, cu2 = hd_assemble(m((x0, xm)), hb, wb, sep, ret)
    assert torch.equal(cu, cu2)
    assert torch.equal(packed, packed2), int((packed != packed2).any(-1).sum())


def test_arbitrary_row_offsets_still_supported(monkeypatch):
    """tp_forward's seg_row_offset form (arbitrary destination rows, direct stores) is kept: scatter crops in REVERSE order.
    (That form runs the separate-kernel plan, so the dense reference is taken from the same plan: TP_FUSE_ATTN=0.)"""
    from tokenpacker_b200._lib import lib
    monkeypatch.setenv("TP_FUSE_ATTN", "0")
    m, _ = _module(512, 4, seed=4)
    x0, xm = _inputs(5, 3)
    with torch.no_grad():
        dense = m((x0, xm))
        seg = torch.tensor([(4 - i) * 40 for i in range(5)], dtype=torch.int64, device="cuda")
        out = torch.zeros(5 * 40, 512, dtype=torch.bfloat16, device="cuda")
        ws_bytes = lib.tp_workspace_bytes(5, 4, 512)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
        st = lib.tp_forward(m._packed_weights(x0.device).data_ptr(), x0.data_ptr(), xm.data_ptr(), 5, x0.stride(0), xm.stride(0), 4, 512,
                            out.data_ptr(), seg.data_ptr(), ws.data_ptr(), ws_bytes, torch.cuda.current_stream().cuda_stream)
        assert st == 0, lib.tp_strerror(st)
    for i in range(5):
        assert torch.equal(out[(4 - i) * 40:(4 - i) * 40 + 36], dense[i])


def test_data_alias_update_is_seen_in_training():
    """ZeRO-2 style updates write parameters through a ``.data`` alias: data_ptr and _version do not move.  A training forward
    must still use the new weights (it repacks every step), and so must the first eval forward after training."""
    m, _ = _module(256, 2, seed=8)
    x0, xm = _inputs(2, 21)
    m.train()
    out0 = m((x0, xm)).detach().clone()
    p = m.mlp[2].bias
    v0 = p._version
    p.data.add_(1.0)
    assert p._version == v0                      # the hazard this test is about
    out1 = m((x0, xm)).detach()
    assert float((out1.float() - out0.float()).mean()) > 0.9
    m.eval()
    with torch.no_grad():
        out2 = m((x0, xm))
    assert float((out2.float() - out0.float()).mean()) > 0.9
    # explicit invalidation covers .data writes outside of training
    p.data.sub_(1.0)
    m.invalidate_packed()
    with torch.no_grad():
        out3 = m((x0, xm))
    assert float((out3.float() - out0.float()).abs().mean()) < 2e-2


def test_forward_packed_is_differentiable():
    """HD training recipes (pretrain_hd.sh / finetune_hd.sh, mode='slice') run the slice assembly under autograd: the packed
    path must carry gradients to the projector AND to the separator embeddings."""
    from tokenpacker_b200 import hd_assemble
    m, _ = _module(256, 4, seed=2)
    m.train()
    grids = [(1, 2), (1, 1)]
    n = sum(hdo.n_crops(a, b) for a, b in grids)
    x0, xm = _inputs(n, 3)
    hb, wb = [a for a, _ in grids], [b for _, b in grids]
    sep = torch.randn(256, device="cuda").bfloat16().requires_grad_(True)
    ret = torch.randn(256, device="cuda").bfloat16().requires_grad_(True)
    packed, cu = m.forward_packed((x0, xm), hb, wb, sep, ret)
    assert packed.requires_grad
    w = torch.randn_like(packed.float())
    (packed.float() * w).sum().backward()
    g_packed = {k: p.grad.clone() for k, p in m.named_parameters()}
    g_sep, g_ret = sep.grad.clone(), ret.grad.clone()
    for p in m.parameters():
        p.grad = None
    sep.grad = ret.grad = None
    # the same through dense forward + differentiable hd_assemble
    packed2, _ = hd_assemble(m((x0, xm)), hb, wb, sep, ret)
    assert torch.equal(packed2.detach(), packed.detach())
    (packed2.float() * w).sum().backward()
    for k, p in m.named_parameters():
        assert torch.equal(p.grad, g_packed[k]), k
    assert torch.equal(sep.grad, g_sep) and torch.equal(ret.grad, g_ret)
    assert float(g_sep.float().abs().sum()) > 0 and float(g_packed["mlp.2.weight"].float().abs().sum()) > 0
    with pytest.raises(NotImplementedError):
        m.forward_layers([x0, x0, x0, x0])       # inference-only entry points refuse to run silently without gradients


def test_layernorm_statistics_survive_large_row_mean():
    """|row mean| >> std in the LayerNorm inputs (k/v_proj.2 biases shifted by +-30 against a std of a few tenths).  The kernels
    store those activations in bf16 (like a bf16 reference module does) and keep per-block (mean, M2) statistics of the stored
    values, combined Chan-style — no E[y^2] - mu^2 cancellation.  Oracle: the fp32 port with the same bf16 round trip applied
    to the LayerNorm inputs (at this offset bf16's ulp, 0.125..0.25, is the dominant error of ANY bf16 implementation, so the
    un-rounded fp32 result is not the right yardstick here)."""
    from tokenpacker_b200 import TokenPackerB200
    from tokenpacker_b200 import synthetic as syn
    sd = {k: torch.from_numpy(v) for k, v in syn.synthetic_state_dict(256, seed=1).items()}
    sd["k_proj_1.2.bias"] = sd["k_proj_1.2.bias"] + 30.0
    sd["v_proj_1.2.bias"] = sd["v_proj_1.2.bias"] - 30.0
    sd = {k: v.bfloat16() for k, v in sd.items()}
    m = TokenPackerB200(hidden_size=256, scale_factor=2)
    m.load_state_dict(sd)
    m = m.to("cuda", torch.bfloat16).eval()
    p32 = {k: v.float().cuda() for k, v in sd.items()}
    x0, xm = _inputs(2, 17)
    with torch.no_grad():
        out = m((x0, xm))
        ref = torch_port.forward(p32, x0.float(), xm.float(), 2, pre_ln=lambda t: t.bfloat16().float())
    d = out.float() - ref
    rel = float(d.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())
    assert torch.isfinite(out.float()).all() and rel < 3e-2, rel


def test_hd_tile_batch_matches_per_image_kernels_and_oracle():
    from tokenpacker_b200 import hd_tile, hd_tile_batch
    rng = np.random.default_rng(5)
    sizes = [(244, 1002), (500, 700), (336, 336), (1300, 900), (77, 1411), (1088, 1088), (300, 200)]
    for patch_num in (9, 25):
        imgs = [torch.from_numpy(rng.standard_normal((3, h, w)).astype(np.float32)).cuda() for h, w in sizes]
        crops, hb, wb = hd_tile_batch(imgs, patch_num)
        off = 0
        for im, a, b in zip(imgs, hb, wb):
            one, oa, ob = hd_tile(im[None], patch_num)
            assert (a, b) == (oa, ob)
            k = one.shape[0]
            assert torch.equal(crops[off:off + k], one)          # same arithmetic -> same bits as the two-pass kernels
            ref, _, _ = hdo.hd_tile(im.cpu().numpy()[None], patch_num)
            assert float((crops[off:off + k].cpu() - torch.from_numpy(ref)).abs().max()) < 3e-6
            off += k
        assert off == crops.shape[0]
