"""Training the whole CLIP tower, host side (no CUDA): include/tokenpacker_b200_clip_tower_embed.h, its exports and its ctypes binding
agree; a plain-C consumer links it; the size query and argument checks answer before any CUDA call; the constructor's train_embeddings
validation and the parameters the tower reads in place; the fp64 oracle of the embedding stage against transformers' CLIPVisionModel
and against finite differences."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

from oracle import clip_tower_embed_oracle as cte
from oracle import clip_tower_oracle as cto
from oracle import clip_tower_train_oracle as ctt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tokenpacker_b200_clip_tower_embed.h")
N_PAST_LIMIT = (1 << 31) // (577 * 4) + 1                  # the first crop count tp_clip_tower_workspace_bytes refuses


def _header_functions():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return {m.group(1): m.group(2) for m in re.finditer(r"TP_API\s+[\w\s\*]+?\b(tp_\w+)\s*\(([^)]*)\)", text)}


def test_header_binding_and_exports_agree():
    from tokenpacker_b200 import _lib
    fns = _header_functions()
    assert sorted(fns) == ["tp_clip_tower_backward_embed", "tp_clip_tower_embed_saved_bytes", "tp_clip_tower_forward_train_embed"]
    assert sorted(_lib.CLIP_TOWER_EMBED_SIGNATURES) == sorted(fns)
    for other in (_lib.SIGNATURES, _lib.HD_U8_SIGNATURES, _lib.CLIP_U8_SIGNATURES, _lib.INPUT_GRAD_SIGNATURES, _lib.LAYERS_SIGNATURES,
                  _lib.CLIP_TOWER_SIGNATURES, _lib.CLIP_TOWER_F16_SIGNATURES, _lib.CLIP_TOWER_TRAIN_SIGNATURES, _lib.CLIP_TOWER_CKPT_SIGNATURES):
        assert not set(fns) & set(other)
    for name, params in fns.items():
        assert len(params.split(",")) == len(_lib.CLIP_TOWER_EMBED_SIGNATURES[name][1]), name
    # the gradient struct has one destination per embedding-stage field of the weight struct, in its order
    text = open(HEADER).read()
    body = re.search(r"typedef struct tp_clip_tower_embed_grads \{(.*?)\}", text, flags=re.S).group(1)
    assert re.findall(r"void\*\s+(\w+);", body) == [f for f, _ in _lib.CLIP_TOWER_FIELDS]
    assert [f for f, _ in _lib.TpClipTowerEmbedGrads._fields_] == [f for f, _ in _lib.CLIP_TOWER_FIELDS]
    raw = C.CDLL(_lib.LIB_PATH)
    for n in fns:
        assert hasattr(raw, n), f"{n} declared in the header but not exported"


def test_plain_c_consumer_of_the_embed_header(tmp_path):
    from tokenpacker_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = str(tmp_path / "abi_check_clip_tower_embed")
    src = os.path.join(ROOT, "tests", "abi_c", "abi_check_clip_tower_embed.c")
    text = open(src).read()
    for name in _header_functions():
        assert name in text, f"{name} missing from abi_check_clip_tower_embed.c"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", libdir,
                    "-l:libtokenpacker_b200.so", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "abi clip tower embed ok" in r.stdout


def test_size_query():
    from tokenpacker_b200 import _lib
    q = _lib.lib.tp_clip_tower_embed_saved_bytes
    assert q(0) == 0 and q(-1) == 0 and q(N_PAST_LIMIT) == 0 and q(N_PAST_LIMIT - 1) > 0
    # per crop: the patch rows (576 x 592 bf16) and the patch GEMM's token rows (577 x 1024 bf16), each region 1 KiB aligned
    per_crop = 576 * 592 * 2 + 577 * 1024 * 2
    for n in (1, 3, 29, 231):
        assert n * per_crop <= q(n) <= n * per_crop + 2048
    assert q(64) - q(32) == 32 * per_crop


def _weights_struct(lib_mod):
    w = lib_mod.TpClipTowerWeights(*([4096] * 5))
    for i in range(23):
        w.layers[i] = lib_mod.TpClipTowerLayer(*([4096] * 16))
    return w


def test_abi_argument_validation():
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    bad, small = _lib.TP_ERR_INVALID_ARGUMENT, _lib.TP_ERR_WORKSPACE_TOO_SMALL
    w = _weights_struct(_lib)
    outs = (C.c_void_p * 4)(4096, 8192, 12288, 16384)
    cs = 3 * 336 * 336
    eb = lib.tp_clip_tower_embed_saved_bytes(1)
    sizes = {1: (lib.tp_clip_tower_ckpt_saved_bytes(1, 23), lib.tp_clip_tower_workspace_bytes(1), lib.tp_clip_tower_ckpt_backward_workspace_bytes(1, 23)),
             0: (lib.tp_clip_tower_train_saved_bytes(1, 23), lib.tp_clip_tower_train_workspace_bytes(1, 23),
                 lib.tp_clip_tower_backward_workspace_bytes(1, 23))}
    for ck, (sb, wsb, bwsb) in sizes.items():
        def fwd(packed=4096, w=w, crops=4096, n=1, outs=outs, saved=4096, sb=sb, es=4096, eb=eb, ws=4096, wsb=wsb):
            return lib.tp_clip_tower_forward_train_embed(packed, C.byref(w) if w is not None else None, crops, n, cs, ck, outs, saved, sb, es,
                                                         eb, ws, wsb, None)

        for kwargs in ({"packed": None}, {"w": None}, {"crops": None}, {"n": 0}, {"n": N_PAST_LIMIT}, {"outs": None}, {"saved": None},
                       {"saved": 4096 + 16}, {"es": None}, {"es": 4096 + 64}, {"ws": None},
                       {"outs": (C.c_void_p * 4)(4096, 4096, 12288, 16384)}):
            assert fwd(**kwargs) == bad, (ck, kwargs)
        assert fwd(sb=sb - 1) == small and fwd(eb=eb - 1) == small and fwd(wsb=wsb - 1) == small, ck
        d_outs = (C.c_void_p * 4)(None, None, None, 4096)
        grads = (_lib.TpClipTowerLayerGrads * 23)()
        eg = _lib.TpClipTowerEmbedGrads()

        def bwd(w=w, saved=4096, es=4096, n=1, d_outs=d_outs, grads=grads, eg=eg, ws=4096, wsb=bwsb):
            return lib.tp_clip_tower_backward_embed(C.byref(w) if w is not None else None, saved, es, n, ck, d_outs, grads,
                                                    C.byref(eg) if eg is not None else None, ws, wsb, None)

        for kwargs in ({"w": None}, {"saved": None}, {"saved": 4096 + 16}, {"es": None}, {"es": 4096 + 16}, {"n": 0}, {"d_outs": None},
                       {"grads": None}, {"eg": None}, {"ws": None}, {"ws": 4096 + 64},
                       {"d_outs": (C.c_void_p * 4)(None, 4096 + 2, None, 4096)}):
            assert bwd(**kwargs) == bad, (ck, kwargs)
        assert bwd(wsb=bwsb - 1) == small, ck
        for field, _ in _lib.CLIP_TOWER_FIELDS:
            odd = _lib.TpClipTowerEmbedGrads()
            setattr(odd, field, 4096 + 2)
            assert bwd(eg=odd) == bad, (ck, field)
        holey = _lib.TpClipTowerWeights.from_buffer_copy(w)
        holey.pos_emb = None
        assert bwd(w=holey) == bad and fwd(w=holey) == bad, ck
    # the checkpointed backward's workspace is the larger: the plain one's is refused in checkpoint mode
    d_outs = (C.c_void_p * 4)(None, None, None, 4096)
    assert lib.tp_clip_tower_backward_embed(C.byref(w), 4096, 4096, 1, 1, d_outs, (_lib.TpClipTowerLayerGrads * 23)(),
                                            C.byref(_lib.TpClipTowerEmbedGrads()), 4096, sizes[0][2], None) == small


def _fake_model():
    w = {k: v.bfloat16() for k, v in cto.make_weights(0, seed=0).items()}
    for i in range(23):                                               # tiny stand-ins: only names and config are looked at here
        for key in cto.layer_keys(i).values():
            w[key] = torch.zeros(1, dtype=torch.bfloat16)
    return cto.FakeCLIPVisionModel(w)


def test_constructor_validation():
    from tokenpacker_b200 import CLIPVisionTowerB200
    model = _fake_model()
    assert CLIPVisionTowerB200(model).train_embeddings is False
    assert CLIPVisionTowerB200(model, trainable_layers=23, train_embeddings=True).train_embeddings is True
    for k in (0, 1, 22):
        with pytest.raises(ValueError, match="trainable_layers=23"):
            CLIPVisionTowerB200(model, trainable_layers=k, train_embeddings=True)
    with pytest.raises(ValueError):
        CLIPVisionTowerB200(model, dtype=torch.float16, trainable_layers=23, train_embeddings=True)
    for v in (1, 0, "yes", None, 1.0):
        with pytest.raises(ValueError, match="train_embeddings"):
            CLIPVisionTowerB200(model, trainable_layers=23, train_embeddings=v)


def test_trainable_parameters_and_live_weights():
    """train_embeddings puts the five embedding-stage parameters first, in the weight struct's order, and the struct handed to the
    library points at them (read in place under the layers' rule)."""
    from tokenpacker_b200 import CLIPVisionTowerB200, _lib
    w = {k: v.bfloat16() for k, v in cto.make_weights(0, seed=0).items()}
    for i in range(23):
        for key in cto.layer_keys(i).values():
            w[key] = torch.zeros(8, dtype=torch.bfloat16)
    model = cto.FakeCLIPVisionModel(w)
    named = dict(model.named_parameters())
    plain = CLIPVisionTowerB200(model, trainable_layers=23)
    full = CLIPVisionTowerB200(model, trainable_layers=23, train_embeddings=True)
    tp = full._trainable_params()
    assert len(tp) == 5 + 23 * 16 and len(plain._trainable_params()) == 23 * 16
    assert all(a is b for a, b in zip(tp[5:], plain._trainable_params()))
    assert [id(p) for p in tp[:5]] == [id(named["vision_model." + key]) for _, key in _lib.CLIP_TOWER_FIELDS]
    base = _weights_struct(_lib)
    live = full._live_weights(base, tp, torch.device("cpu"))
    for (field, _), p in zip(_lib.CLIP_TOWER_FIELDS, tp[:5]):
        assert getattr(live, field) == p.data_ptr(), field
    assert live.layers[0].ln1_w == tp[5].data_ptr() and live.layers[22].fc2_b == tp[-1].data_ptr()
    assert plain._live_weights(base, plain._trainable_params(), torch.device("cpu")).patch_w == 4096   # untouched without the option
    named["vision_model.embeddings.class_embedding"].data = torch.zeros(1024)                          # fp32: not read in place
    with pytest.raises(ValueError, match="read in place"):
        full._live_weights(base, full._trainable_params(), torch.device("cpu"))


def _small_weights(n_layers, seed):
    return cto.round_bf16(cto.make_weights(n_layers, seed=seed))


def test_oracle_matches_transformers_clip_vision_model():
    transformers = pytest.importorskip("transformers")
    n_layers = 2
    w = _small_weights(n_layers, seed=3)
    cfg = transformers.CLIPVisionConfig(hidden_size=1024, intermediate_size=4096, num_attention_heads=16, num_hidden_layers=n_layers,
                                        image_size=336, patch_size=14, hidden_act="quick_gelu", layer_norm_eps=1e-5)
    model = transformers.CLIPVisionModel(cfg).double().train()
    model.load_state_dict({"vision_model." + k: v.double() for k, v in w.items()}, strict=False)
    model.requires_grad_(True)
    images = cto.make_images(1, seed=4).double()
    g = torch.Generator().manual_seed(5)
    d_outs = {j: torch.randn(1, 577, 1024, generator=g, dtype=torch.float64) for j in range(n_layers + 1)}
    hs = model(pixel_values=images, output_hidden_states=True).hidden_states
    sum((h * d_outs[j]).sum() for j, h in enumerate(hs)).backward()
    eg, lg, ours = cte.parameter_gradients(w, images, d_outs, n_layers=n_layers)
    for j in range(n_layers + 1):
        torch.testing.assert_close(ours[j], hs[j].detach(), rtol=1e-9, atol=1e-9)
    named = dict(model.named_parameters())
    for key in cte.EMBED_KEYS:
        ref = named["vision_model." + key].grad
        assert ref is not None, key
        torch.testing.assert_close(eg[key], ref, rtol=1e-8, atol=1e-10, msg=key)
    for key in ("self_attn.q_proj.weight", "layer_norm1.bias", "mlp.fc2.weight"):
        torch.testing.assert_close(lg[0][key], named[f"vision_model.encoder.layers.0.{key}"].grad, rtol=1e-8, atol=1e-10, msg=key)


def test_oracle_embedding_gradients_match_finite_differences():
    n_layers = 1
    w = _small_weights(n_layers, seed=6)
    images = cto.make_images(1, seed=7).double()
    g = torch.Generator().manual_seed(8)
    d_outs = {j: torch.randn(1, 577, 1024, generator=g, dtype=torch.float64) for j in (0, 1)}
    eg, _, _ = cte.parameter_gradients(w, images, d_outs, n_layers=n_layers)

    def value(wd):
        with torch.no_grad():
            x = cte.embedding_stage({k: wd[k] for k in cte.EMBED_KEYS}, images)
            total = (x * d_outs[0]).sum()
            x = ctt.layer(ctt.layer_params(wd, 0, torch.float64), x)
            return float(total + (x * d_outs[1]).sum())

    eps = 1e-4
    picks = {"embeddings.patch_embedding.weight": [(5, 1, 3, 7), (1000, 2, 13, 0)], "embeddings.class_embedding": [(3,), (611,)],
             "embeddings.position_embedding.weight": [(0, 9), (300, 1023)], "pre_layrnorm.weight": [(2,), (777,)],
             "pre_layrnorm.bias": [(4,), (1001,)]}
    wd = {k: v.double() for k, v in w.items()}
    for key, idxs in picks.items():
        for idx in idxs:
            plus, minus = dict(wd), dict(wd)
            plus[key], minus[key] = wd[key].clone(), wd[key].clone()
            plus[key][idx] += eps
            minus[key][idx] -= eps
            fd = (value(plus) - value(minus)) / (2 * eps)
            got = float(eg[key][idx])
            assert abs(fd - got) <= 1e-6 * max(1.0, abs(got)), (key, idx, fd, got)
