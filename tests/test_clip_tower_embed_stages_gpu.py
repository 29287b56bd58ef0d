"""The whole-tower training path's embedding stage, step by step against fp64 (tests/csrc/tp_clip_tower_embed_hooks.cu:
tpte_embed_backward runs run_clip_embed_backward up to a step from a caller-written fp32 carry), plus the GEMM engine's TN form with a
ragged M, a segmented B and split-K, which the patch weight gradient uses.

Each step is checked from the values the steps before it stored, within elementwise bounds derived from the fp32 operation order, or
bit for bit against a fixed-order fp32 emulation where the order is the kernel's own.  Every step writes only the regions it owns:
the rest of the workspace keeps a sentinel, and so do the gradients of later steps."""
import ctypes as C
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import clip_tower_embed_oracle as cte
from oracle import clip_tower_oracle as cto

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOOKS = os.path.join(ROOT, "tokenpacker_b200", "libtokenpacker_b200_clip_tower_embed_hooks.so")
ENGINE_HOOKS = os.path.join(ROOT, "tokenpacker_b200", "libtokenpacker_b200_testhooks.so")
U32 = 2.0 ** -24                   # fp32 unit roundoff
UBF = 2.0 ** -8                    # bf16 unit roundoff (round to nearest, 8 significand bits)
SENT = 0x7F                        # workspace sentinel byte (0x7F7F7F7F: an fp32 value no step computes here)
SENT16 = 0x7FA5                    # bf16 NaN bits: the gradients a step must not write


@pytest.fixture(scope="module")
def hooks():
    import tokenpacker_b200  # noqa: F401  (the product library is loaded next to this one)
    lib = C.CDLL(HOOKS)
    p, i64 = C.c_void_p, C.c_int64
    lib.tpte_offsets.restype, lib.tpte_offsets.argtypes = C.c_int, [i64, C.POINTER(i64)]
    lib.tpte_embed_backward.restype = C.c_int
    lib.tpte_embed_backward.argtypes = [p, p, i64, p, p, C.c_size_t, C.c_int, p]
    return lib


def _offsets(hooks, n):
    out = (C.c_int64 * 9)()
    assert hooks.tpte_offsets(n, out) == 0
    keys = ("patches", "rows", "embed_total", "carry32", "carry16", "ln_part", "splitk", "unused_grad", "total")
    return dict(zip(keys, list(out)))


def _weights(outlier):
    w = cto.round_bf16(cto.make_weights(23, seed=21, device=DEV))
    if outlier:                                 # a few huge channels in the pre-LN input: the LayerNorm backward's hard case
        pos = w["embeddings.position_embedding.weight"]
        pos[:, list(cto.OUTLIER_CHANNELS)] += torch.tensor([70.0, -60.0, 90.0, -50.0], device=DEV)
        w = cto.round_bf16(w)
    return w


def _forward(w, n, seed):
    """One whole-tower training forward (checkpointed: the smaller saved set); returns the autograd node, which holds the live weight
    struct and the embedding saved set, and the crops."""
    from tokenpacker_b200 import CLIPVisionTowerB200
    model = cto.FakeCLIPVisionModel({k: v.bfloat16() for k, v in w.items()}).to(DEV)
    for name, p in model.named_parameters():
        p.requires_grad_("encoder.layers." not in name)
    model.gradient_checkpointing = True
    t = CLIPVisionTowerB200(model, trainable_layers=23, train_embeddings=True)
    images = cto.make_images(n, seed=seed, device=DEV).bfloat16()
    outs = t.hidden_states(images)
    torch.cuda.synchronize()
    return outs[3].grad_fn, images, model


def _run(hooks, fn, n, g32, grads, step):
    """A fresh sentinel workspace with carry32 = g32, then steps 1 .. step; returns the workspace."""
    from tokenpacker_b200 import _lib
    off = _offsets(hooks, n)
    ws = torch.full((off["total"],), SENT, dtype=torch.uint8, device=DEV)
    ws[off["carry32"]:off["carry32"] + g32.numel() * 4].view(torch.float32).copy_(g32.reshape(-1))
    eg = _lib.TpClipTowerEmbedGrads(*[None if g is None else g.data_ptr() for g in grads])
    assert hooks.tpte_embed_backward(C.byref(fn.w), fn.embed_saved.data_ptr(), n, C.byref(eg), ws.data_ptr(), ws.numel(), step,
                                     torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    return ws


def _sent_grads(w):
    shapes = [w[k].shape for k in cte.EMBED_KEYS]
    return [torch.full(s, 0, dtype=torch.int16, device=DEV).fill_(SENT16).view(torch.bfloat16) for s in shapes]


def _untouched(t):
    return bool((t.view(torch.int16) == SENT16).all())


@pytest.mark.parametrize("n,outlier", [(1, False), (3, False), (3, True), (29, False), (29, True)],
                         ids=["N1", "N3", "N3-outlier", "N29-splitk", "N29-splitk-outlier"])
def test_embedding_stage_step_by_step(hooks, n, outlier):
    w = _weights(outlier)
    fn, images, _ = _forward(w, n, seed=30 + n)
    off = _offsets(hooks, n)
    M, R = n * 577, n * 576
    es = fn.embed_saved
    patches = es[off["patches"]:off["patches"] + R * 592 * 2].view(torch.bfloat16).view(R, 592)[:, :588]
    rows = es[off["rows"]:off["rows"] + M * 2048].view(torch.bfloat16).view(n, 577, 1024)
    # what the forward kept: the crops' patch rows in the conv weight's (c, ky, kx) order, and the patch GEMM's output rows
    assert torch.equal(patches, F.unfold(images, 14, stride=14).transpose(1, 2).reshape(R, 588))
    wp = w["embeddings.patch_embedding.weight"].reshape(1024, 588).double()
    ref_rows = patches.double() @ wp.T
    bound = UBF * ref_rows.abs() + 600 * U32 * (patches.double().abs() @ wp.abs().T)
    assert ((rows[:, 1:].reshape(R, 1024).double() - ref_rows).abs() <= bound).all()

    g = torch.Generator(device=DEV).manual_seed(7 + n)
    g32 = torch.randn(M, 1024, generator=g, device=DEV) * 1e-3        # not bf16-representable: the carry is fp32
    # ---- step 1: pre_layrnorm backward
    grads = _sent_grads(w)
    ws = _run(hooks, fn, n, g32, grads, 1)
    c32 = ws[off["carry32"]:off["carry32"] + M * 4096].view(torch.float32).view(M, 1024)
    c16 = ws[off["carry16"]:off["carry16"] + M * 2048].view(torch.bfloat16).view(M, 1024)
    assert torch.equal(c16, c32.bfloat16())
    src = rows.float().clone()
    src[:, 0] = w["embeddings.class_embedding"].float()
    e = (src + w["embeddings.position_embedding.weight"].float()).reshape(M, 1024).double()   # fl32(x + pos), as the forward forms it
    gam = w["pre_layrnorm.weight"].double()
    gd = g32.double()
    mu = e.mean(1, keepdim=True)
    dev = e - mu
    rstd = 1.0 / torch.sqrt((dev * dev).mean(1, keepdim=True) + 1e-5)
    xh = dev * rstd
    gg = gam * gd
    c1, c2 = gg.mean(1, keepdim=True), (gg * xh).mean(1, keepdim=True)
    de = rstd * (gg - c1 - xh * c2)
    # fp32 error terms: the row sums (32 sequential terms per lane, then 5 shuffle levels) carry <= 40 u of the sum of magnitudes;
    # mean -> deviations, variance -> rstd (<= 24 u with rsqrtf), x_hat; then c1, c2 and the final expression
    dmean = 40 * U32 * e.abs().mean(1, keepdim=True)
    rstd_rel = 24 * U32 + 2 * dmean * dev.abs().max(1, keepdim=True).values * rstd ** 2
    xh_err = rstd * (dmean + U32 * dev.abs()) + xh.abs() * rstd_rel
    c1_err = 40 * U32 * gg.abs().mean(1, keepdim=True)
    c2_err = 40 * U32 * (gg * xh).abs().mean(1, keepdim=True) + (gg.abs() * xh_err).mean(1, keepdim=True)
    terms = gg.abs() + c1.abs() + (xh * c2).abs()
    bound = 2 * (rstd * (4 * U32 * terms + c1_err + xh.abs() * c2_err + xh_err * c2.abs()) + de.abs() * rstd_rel)
    err = (c32.double() - de).abs()
    assert (err <= bound).all(), float((err / bound).max())
    # dgamma / dbeta: per-thread row sums, 8 warps, 296 CTAs in 16 lanes; one bf16 rounding
    sum_terms = M // 2368 + 1 + 8 + 19 + 16
    for got, ref, mag, extra in ((grads[3], (gd * xh).sum(0), (gd * xh).abs().sum(0), (gd.abs() * xh_err).sum(0)),
                                 (grads[4], gd.sum(0), gd.abs().sum(0), 0.0)):
        b = 2 * (UBF * ref.abs() + sum_terms * U32 * mag + extra)
        assert ((got.double() - ref).abs() <= b).all()
    assert _untouched(grads[0]) and _untouched(grads[1]) and _untouched(grads[2])
    owned = [(off["carry32"], M * 4096), (off["carry16"], M * 2048), (off["ln_part"], 296 * 3 * 4096)]
    rest = ws.clone()
    for o, size in owned:
        rest[o:o + size] = SENT
    assert bool((rest == SENT).all())
    state1 = ws.clone()

    # ---- step 2: class and position embeddings: bit-equal to the crop-order fp32 sum
    grads = _sent_grads(w)
    ws = _run(hooks, fn, n, g32, grads, 2)
    assert torch.equal(ws, state1)                                              # nothing of the workspace is step 2's
    de32 = c32.view(n, 577, 1024)
    s = torch.zeros(577, 1024, device=DEV)
    for k in range(n):
        s = s + de32[k]
    assert torch.equal(grads[2], s.bfloat16()) and torch.equal(grads[1], grads[2][0])
    assert _untouched(grads[0])

    # ---- step 3: the patch weight gradient, slice by slice, then the reduce and transpose
    grads = _sent_grads(w)
    ws = _run(hooks, fn, n, g32, grads, 3)
    splits = 4 if R >= 64 * 64 * 4 else 1
    part_bytes = splits * 588 * 1024 * 4
    rest = ws.clone()
    rest[off["splitk"]:off["splitk"] + part_bytes] = state1[off["splitk"]:off["splitk"] + part_bytes]
    assert torch.equal(rest, state1)
    part = ws[off["splitk"]:off["splitk"] + part_bytes].view(torch.float32).view(splits, 588, 1024)
    b16 = c16.view(n, 577, 1024)[:, 1:].reshape(R, 1024).double()
    a = patches.double()
    kb = (R + 63) // 64
    per = (kb + splits - 1) // splits
    for q in range(splits):
        r0, r1 = q * per * 64, min(R, (q + 1) * per * 64)
        ref = a[r0:r1].T @ b16[r0:r1]
        bound = 2 * ((r1 - r0) // 16 + 16) * 4 * U32 * (a[r0:r1].abs().T @ b16[r0:r1].abs())
        assert ((part[q].double() - ref).abs() <= bound).all(), q
    acc = torch.zeros(588, 1024, device=DEV)
    for q in range(splits):
        acc = acc + part[q]
    assert torch.equal(grads[0], acc.T.contiguous().bfloat16().view(1024, 3, 14, 14))
    assert torch.equal(grads[2], s.bfloat16()) and torch.equal(grads[1], grads[2][0])


class Desc(C.Structure):
    """mirror of tpt_gemm_desc (tests/csrc/tp_test_hooks.cu), field by field"""
    _fields_ = [("tn", C.c_int32), ("a_parts", C.c_int32), ("a", C.c_void_p), ("a_more", C.c_void_p * 3), ("lda", C.c_int64),
                ("a_seg_rows", C.c_int64), ("a_seg_stride", C.c_int64), ("b", C.c_void_p), ("b_more", C.c_void_p * 3),
                ("ldb", C.c_int64), ("b_parts", C.c_int32), ("pad0", C.c_int32), ("b_seg_rows", C.c_int64), ("b_seg_stride", C.c_int64),
                ("M", C.c_int64), ("N", C.c_int64), ("K", C.c_int64), ("c", C.c_void_p), ("ldc", C.c_int64), ("bias", C.c_void_p),
                ("col_a", C.c_void_p), ("stats_in", C.c_void_p), ("stats_out", C.c_void_p), ("seg_row_offset", C.c_void_p),
                ("stats_in_slots", C.c_int32), ("stats_out_slots", C.c_int32), ("ln_inv_dim", C.c_float), ("alpha", C.c_float),
                ("gelu", C.c_int32), ("dual", C.c_int32), ("c_pre", C.c_void_p), ("ld_pre", C.c_int64), ("out_f32", C.c_int32),
                ("k_splits", C.c_int32), ("seg_len", C.c_int32), ("seg_stride", C.c_int32), ("stage", C.c_int32), ("dep", C.c_int32)]


@pytest.mark.parametrize("m,segs,splits", [(588, 3, 1), (588, 3, 4), (588, 29, 4), (100, 5, 3), (588, 29, 1)])
def test_engine_tn_ragged_m_segmented_b_split_k(m, segs, splits):
    """C[s] = A[rows of slice s]^T B[rows of slice s] with A [K, m] (ld 592: m ragged, zero-filled by TMA) and B the token rows 1..576 of
    `segs` crops of [577, 1024] (b_seg_rows 576, 577 rows apart): every slice against fp64 over its own rows; nothing outside the
    slices written."""
    import tokenpacker_b200  # noqa: F401
    lib = C.CDLL(ENGINE_HOOKS)
    lib.tpt_gemm_group.restype = C.c_int
    lib.tpt_gemm_group.argtypes = [C.POINTER(Desc), C.c_int, C.c_int, C.c_void_p]
    lib.tpt_gemm_desc_size.restype = C.c_int
    assert lib.tpt_gemm_desc_size() == C.sizeof(Desc)
    g = torch.Generator(device=DEV).manual_seed(m + segs + splits)
    K = 576 * segs
    a = torch.randn(K, 592, generator=g, device=DEV).bfloat16()
    base = torch.randn(segs * 577, 1024, generator=g, device=DEV).bfloat16()
    out = torch.full(((splits + 1) * m * 1024,), 0, dtype=torch.int32, device=DEV).fill_(0x7FA5A5A5)
    d = Desc()
    d.tn, d.a, d.lda, d.b, d.ldb = 1, a.data_ptr(), 592, base[1:].data_ptr(), 1024
    d.b_seg_rows, d.b_seg_stride = 576, 577 * 1024
    d.M, d.N, d.K, d.c, d.ldc, d.alpha, d.out_f32, d.k_splits = m, 1024, K, out.data_ptr(), 1024, 1.0, 1, splits
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert lib.tpt_gemm_group(C.byref(d), 1, sms, torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    part = out[:splits * m * 1024].view(torch.float32).view(splits, m, 1024)
    assert bool((out[splits * m * 1024:] == 0x7FA5A5A5).all())
    A = a[:, :m].double()
    B = base.view(segs, 577, 1024)[:, 1:].reshape(K, 1024).double()
    per = (K // 64 + splits - 1) // splits
    for q in range(splits):
        r0, r1 = q * per * 64, min(K, (q + 1) * per * 64)
        ref = A[r0:r1].T @ B[r0:r1]
        bound = 2 * ((r1 - r0) // 16 + 16) * 4 * U32 * (A[r0:r1].abs().T @ B[r0:r1].abs())
        assert ((part[q].double() - ref).abs() <= bound).all(), q
