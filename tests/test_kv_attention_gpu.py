"""The fused plan's KV-attention tiles on their own: the window attention computed on the wgmma fragments of the K / V
in-projections, against a float64 reference, at s = 2 and 4.

Each forward runs on a poisoned, test-owned workspace (test_forward_stages_gpu._forward); the reference starts from the bf16 y_k,
y_v and q' the kernel itself stored, so only the KV-attention tiles are checked: the folded LayerNorm (row statistics from the
stored (mean, M2) slots), the scores against q', the softmax over the window's rows and the p-weighted sum of v'.  The bound is
the one of test_forward_stages_gpu's ctx check, whose operation counts (a 130-term score chain, log2(W) + 3 roundings in the
softmax, log2(W) + 2 in the context sum) cover the tiles' order: 32 products per lane, two shuffle adds, pairwise trees over the
window's rows.

Batch sizes: N = 1 (576 rows: the last tile of every head pair is partial, 64 of its 256 rows), N = 7 (4032 rows: a partial tile
of 192 rows) and N = 64 (the flagship batch, checked on a row sample holding the first and last query of every tile).  Weight
variants: plain; y_k / y_v rows with |mean| >> std (biases +-30); row variance at eps (rstd near 1000); 64 x the ln_k weight
(logits of several hundred: a saturated, one-hot softmax).  The context is also bit for bit the same for a crop whatever batch it
runs in, and from one run to the next.
"""
import pytest
import torch

import test_forward_stages_gpu as fs

pytestmark = pytest.mark.gpu

hk = fs.hk
_fp64_exact = fs._fp64_exact


def _ctx_check(record, hk, r, qs):
    w = fs._packed_views(hk, r)
    W = r.W
    st_k, st_v = fs._stats_ref(r.y_k), fs._stats_ref(r.y_v)
    kv_rows = (qs[:, None] * W + torch.arange(W, device="cuda")[None]).reshape(-1)
    kp, fk = fs._ln_fold_ref(r.y_k[kv_rows], {k: v[kv_rows] for k, v in st_k.items()}, w["w_ik"], w["c_k"])
    vp, fv = fs._ln_fold_ref(r.y_v[kv_rows], {k: v[kv_rows] for k, v in st_v.items()}, w["w_iv"], w["c_v"])
    lg = W.bit_length() - 1
    ref, floor, p = fs._attn_ref(r.q_p[qs], kp.view(-1, W, 1024), vp.view(-1, W, 1024), fk, fv, 130, 2, lg + 3, lg + 2)
    fs._check(record, "ctx", r.ctx[qs], ref, floor)
    return p, st_k


def _run(hk, s, n, H, kind, seed):
    m = fs._module(H, s, fs._state_dict(H, 80 + s, kind))
    x0, xm = fs._inputs(n, seed)
    r = fs._forward(hk, m, x0, xm)
    assert r.launches == 1
    fs._check_poison(r, fused=True)
    return m, x0, xm, r


@pytest.mark.parametrize("n,H", [(1, 256), (7, 256), (64, 4096)])
@pytest.mark.parametrize("s", [2, 4])
def test_kv_attention_batches(hk, record_property, monkeypatch, s, n, H):
    monkeypatch.delenv("TP_FUSE_ATTN", raising=False)
    m, x0, xm, r = _run(hk, s, n, H, "plain", 90 + n * s)
    assert r.R % 256 != 0 or n == 64
    qs = fs._sample(r.Q, r.Mq, 13, blocks=(256 // r.W,))
    _ctx_check(record_property, hk, r, qs)
    r2 = fs._forward(hk, m, x0, xm)                       # run to run: the same bits
    assert fs._bits_equal(r2.ctx, r.ctx)
    if n > 1:                                             # the first crop alone: the same bits as inside the batch
        r1 = fs._forward(hk, m, x0[:1].contiguous(), xm[:1].contiguous())
        assert fs._bits_equal(r1.ctx, r.ctx[:r.Mq])


@pytest.mark.parametrize("kind", ["bias30", "tinyvar", "gamma64"])
@pytest.mark.parametrize("s", [2, 4])
def test_kv_attention_adversarial(hk, record_property, monkeypatch, s, kind):
    monkeypatch.delenv("TP_FUSE_ATTN", raising=False)
    _, _, _, r = _run(hk, s, 7, 256, kind, 95 + s)
    p, st_k = _ctx_check(record_property, hk, r, torch.arange(r.Q, device="cuda"))
    if kind == "gamma64":
        assert float(p.amax(-1).median()) > 0.99
    if kind == "tinyvar":
        assert float(st_k["rstd"].min()) > 500
    if kind == "bias30":
        assert float((st_k["mu"].abs() * st_k["rstd"]).min()) > 10
