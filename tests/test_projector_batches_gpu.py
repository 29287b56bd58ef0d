"""The projector at every kernel plan its batch size selects, at the benchmarked batches and at batches past 32-bit offsets.

The tile engine picks each GEMM item's kernel (CTA-pair 256 x 256 tiles, one-CTA 128 x 256 or 128 x 128 tiles) by an estimated cost
that depends on M = 576 N for the k/v stages and Q = N (24 / s)^2 for the q and mlp stages, so the batch size changes what runs.
Every kernel gives the same bits, so a crop's output cannot depend on its batch:
- the plan table: for each (s, H), the smallest N in 1 .. 400 of every distinct combination of kernels the separate-plan forward and
  the training forward choose, read from the engine itself (``tpt_gemm_choice`` on items that mirror forward_impl's and
  forward_train_impl's), printed and recorded as the test property ``plans``; each such forward makes the launches the table predicts
  (the fused plan of s = 2 / 4 at H % 256 == 0 is exactly one);
- inference: every crop of a batch of N (every plan N, and the benchmarked 1, 64, 128, 231, 256) has the bits of that crop run alone,
  two of the batches passed as [:, 1:] views; forward_layers and forward_packed on the HD batch of the hd5 workload likewise;
- the forced plans (TP_GEMM_MODE = 1 / 2 / 3, TP_CHAIN = 0) give the default bits;
- training: at every training-plan N, crop i's output, every saved activation row, d_x0 and d_xm have the bits of crop i run alone,
  and the parameter gradients repeat bit for bit;
- batches of 912 and 1822 crops, whose buffers pass element or byte 2^31, against their crops run alone, and a training step of 912
  crops: picked crops against the crop run alone, the long weight gradients against fp64 on sampled rows;
- the host-buffer forward past its 64-event ring, and the transpose past 65535 x 32 rows.
"""
import ctypes as C
import time

import pytest
import torch

from test_forward_stages_gpu import _bits_equal, _module, _state_dict
from test_gemm_engine_gpu import Desc
from test_gemm_engine_gpu import Hooks as EngineHooks
from test_forward_stages_gpu import E, F64, _check
from test_train_kernels_gpu import Hooks as KernelHooks
from test_train_kernels_gpu import _reduce_emulated
from test_train_stages_gpu import SAVED, _train_forward

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
DEV = "cuda"
GiB = 1 << 30
BENCH_NS = (1, 64, 128, 231, 256)
PLAN_RANGE = range(1, 401)
POOL = 420                                    # distinct seeded crops; the batch of N takes N consecutive ones
STRIDED = (6, 64)                             # batches passed as [:, 1:] views of 577-row tensors
INFER = [(s, H) for s in (2, 3, 4) for H in (4096, 5120, 896)] + [(s, 4096) for s in (1, 6, 8, 12, 24)]
TRAIN = [(s, H) for s in (2, 3, 4) for H in (4096, 896)]
FAKE = 1 << 12                                # a pointer tpt_gemm_choice never dereferences


# ------------------------------------------------------------------------------------------------------------------------------
# the plan table, from the engine
# ------------------------------------------------------------------------------------------------------------------------------
def _desc(M, N, K, stats=False, dual=False):
    d = Desc()
    d.M, d.N, d.K, d.alpha, d.ln_inv_dim = M, N, K, 1.0, 1.0 / 1024
    d.a = d.b = d.c = FAKE
    d.lda, d.ldb, d.ldc = K, K, N
    if stats:
        d.stats_out, d.stats_out_slots = FAKE, N // 128
    if dual:
        d.dual, d.gelu, d.c_pre, d.ld_pre = 1, 1, FAKE, N
    return d


class Plans:
    """Kernel choices of forward_impl's separate plan and of forward_train_impl, as the engine makes them (0 pair, 1 one-CTA 128 x 256,
    2 one-CTA 128 x 128)."""

    def __init__(self):
        self.hk = EngineHooks()
        self.sms = self.hk.sms

    def _choose(self, d, count):
        c = self.hk.lib.tpt_gemm_choice(C.byref(d), count, self.sms)
        assert c in (0, 1, 2)
        return c

    def _chain_items(self, n, s, H):
        R, Q = 576 * n, n * (24 // s) ** 2
        a = [_desc(R, 2048, 4096)] + [_desc(M, 1024, 1024, stats=True) for M in (R, R, Q)] + [_desc(M, 1024, 1024) for M in (R, R, Q)]
        return a, [_desc(Q, H, 1024), _desc(Q, H, H)]

    def forward(self, n, s, H, separate=False):
        """('fused',) or (stage [1], stage [2] items, stage [3] items, ([4], [5]), chain A, chain B) as forward_impl launches them;
        separate: the separate plan also where the fused one runs (TP_FUSE_ATTN=0)"""
        if s in (2, 4) and H % 256 == 0 and not separate:
            return ("fused",)
        a, b = self._chain_items(n, s, H)
        # launch_chain: one persistent launch when the engine puts every item of the chain on the pair kernel (chain_feasible)
        chain_a = all(self._choose(d, 7) == 0 for d in a)
        chain_b = H % 256 == 0 and all(self._choose(d, 2) == 0 for d in b)
        return ((self._choose(a[0], 1),), tuple(self._choose(d, 3) for d in a[1:4]), tuple(self._choose(d, 3) for d in a[4:]),
                (self._choose(b[0], 1), self._choose(b[1], 1)), chain_a, chain_b)

    def chain_blockers(self, n, s, H):
        """the items that keep each chain off one launch, as chain_feasible costs them (a chain of 7 / 2 items): names of the items
        the engine puts on a one-CTA kernel"""
        a, b = self._chain_items(n, s, H)
        names_a = ["[1]", "[2]k", "[2]v", "[2]q", "[3]k", "[3]v", "[3]q"]
        block_a = [name for name, d in zip(names_a, a) if self._choose(d, 7) != 0]
        block_b = [name for name, d in zip(["[4]", "[5]"], b) if self._choose(d, 2) != 0] if H % 256 == 0 else ["H % 256"]
        return block_a, block_b

    def train(self, n, s, H):
        """forward_train_impl's items in launch order: [1] (dual), [2] x 3, [3] x 3, out_proj, mlp.0, mlp.2"""
        R, Q = 576 * n, n * (24 // s) ** 2
        return ((self._choose(_desc(R, 2048, 4096, dual=True), 1),) + tuple(self._choose(_desc(M, 1024, 1024, stats=True), 3) for M in (R, R, Q))
                + tuple(self._choose(_desc(M, 1024, 1024), 3) for M in (R, R, Q)) + (self._choose(_desc(Q, 1024, 1024), 1),
                self._choose(_desc(Q, H, 1024, dual=H % 256 == 0), 1), self._choose(_desc(Q, H, H), 1)))

    def first_ns(self, plan, s, H):
        """the smallest N of every distinct plan in PLAN_RANGE"""
        seen = {}
        for n in PLAN_RANGE:
            seen.setdefault(plan(n, s, H), n)
        return sorted(seen.values())


def _stage_launches(choices):
    """kernel launches of one launch_gemms call: one per one-CTA item, one for all pair items together"""
    return sum(1 for c in choices if c != 0) + (1 if 0 in choices else 0)


def predicted_launches(plan):
    if plan == ("fused",):
        return 1
    s1, s2, s3, _, chain_a, chain_b = plan
    a = 1 if chain_a else 1 + _stage_launches(s1) + _stage_launches(s2) + _stage_launches(s3)     # + the point-query kernel
    b = 1 if chain_b else 2
    return a + 1 + b                                                                            # + the attention kernel


@pytest.fixture(scope="module")
def plans():
    return Plans()


def infer_ns(plans, s, H):
    ns = set(plans.first_ns(plans.forward, s, H)) | set(BENCH_NS)
    if s in (2, 4) and H % 256 == 0:      # one plan at every N; its persistent schedule (tiles, waves, counters) still changes with N
        ns |= {2, 3, 5, 7, 11, 22, 33}
    return sorted(ns)


def train_ns(plans, s, H):
    return sorted(set(plans.first_ns(plans.train, s, H)) | {64})


def test_plan_table(plans, record_property):
    """The table of plans, and for each separate-plan N of it the items that keep chain A / chain B off one launch (recorded as
    ``chain_blockers``).  On an H100's 132 SMs the separate plan never runs either chain as one launch at any N up to 400: at every N
    some item of each chain goes to a one-CTA kernel (stage [1] at most N; at N = 2 and 3 the chain's 7-item cost puts [1] on the pair
    kernel and stage [3] blocks instead).  That is a property of the cost model at 132 SMs, which DESIGN.md and forward_impl's comment
    state; it is asserted at that SM count only."""
    table, blockers = {}, {}
    for s, H in INFER:
        table[f"fwd s={s} H={H}"] = {n: plans.forward(n, s, H) for n in plans.first_ns(plans.forward, s, H)}
        if not (s in (2, 4) and H % 256 == 0):
            blockers[f"fwd s={s} H={H}"] = {n: plans.chain_blockers(n, s, H) for n in plans.first_ns(plans.forward, s, H)}
    for s, H in TRAIN:
        table[f"train s={s} H={H}"] = {n: plans.train(n, s, H) for n in plans.first_ns(plans.train, s, H)}
    record_property("plans", {k: {n: str(p) for n, p in v.items()} for k, v in table.items()})
    record_property("chain_blockers", {k: {n: str(p) for n, p in v.items()} for k, v in blockers.items()})
    print(f"\nplans at {plans.sms} SMs (0 pair, 1 one-CTA 128x256, 2 one-CTA 128x128):")
    for k, v in table.items():
        print(f"  {k}: " + "; ".join(f"N={n} {p}" for n, p in v.items()))
    print("items that keep chain A / chain B off one launch:")
    for k, v in blockers.items():
        print(f"  {k}: " + "; ".join(f"N={n} {a} / {b}" for n, (a, b) in v.items()))
    if plans.sms != 132:
        return
    for s, H in INFER:
        if s in (2, 4) and H % 256 == 0:
            continue
        chained = [n for n in PLAN_RANGE if any(plans.forward(n, s, H)[4:])]
        assert not chained, ("the separate plan chains at 132 SMs, unlike DESIGN.md section 3 states", s, H, chained[:8])


# ------------------------------------------------------------------------------------------------------------------------------
# inference batch invariance at every plan
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pool():
    g = torch.Generator(device=DEV).manual_seed(301)
    return torch.randn((POOL, 576, 1024), device=DEV, generator=g).to(BF), torch.randn((POOL, 576, 4096), device=DEV, generator=g).to(BF)


def _offset(n):
    return (37 * n) % (POOL - n + 1)


def _view577(x):
    """x as the [:, 1:] view of a 577-row tensor whose class-token row is NaN"""
    big = torch.full((x.shape[0], 577, x.shape[2]), float("nan"), dtype=x.dtype, device=x.device)
    big[:, 1:] = x
    return big[:, 1:]


def _counted(m, x0, xm):
    from tokenpacker_b200 import _lib
    torch.cuda.synchronize()
    c0 = _lib.lib.tp_launch_count()
    with torch.no_grad():
        out = m((x0, xm))
    torch.cuda.synchronize()
    return out, _lib.lib.tp_launch_count() - c0


class Singles:
    """outputs of pool crops run alone, computed on first use"""

    def __init__(self, m, pool):
        self.m, self.pool = m, pool
        self.out = {}

    def __call__(self, lo, hi):
        for i in range(lo, hi):
            if i not in self.out:
                with torch.no_grad():
                    self.out[i] = self.m((self.pool[0][i:i + 1], self.pool[1][i:i + 1]))[0]
        return torch.stack([self.out[i] for i in range(lo, hi)])


def _assert_crops_equal(got, want, what, crops=None):
    assert got.shape == want.shape, what
    assert torch.isfinite(got).all(), what
    differ = (got.view(torch.int16) != want.view(torch.int16)).flatten(1).any(1).nonzero().flatten().tolist()
    assert not differ, (what, "crops", [i if crops is None else crops[i] for i in differ][:16])


@pytest.mark.parametrize("s,H", INFER)
def test_every_crop_has_the_bits_of_that_crop_alone(plans, pool, s, H, record_property):
    m = _module(H, s, _state_dict(H, 400 + s))
    singles = Singles(m, pool)
    singles(0, 1)                                   # packs the weights: the launches counted below are the forward's alone
    launches = {}
    for n in infer_ns(plans, s, H):
        off = _offset(n)
        x0, xm = pool[0][off:off + n], pool[1][off:off + n]
        if n in STRIDED:
            x0, xm = _view577(x0), _view577(xm)
        out, launches[n] = _counted(m, x0, xm)
        plan = plans.forward(n, s, H)
        assert launches[n] == predicted_launches(plan), (n, plan, launches[n])
        _assert_crops_equal(out, singles(off, off + n), f"s={s} H={H} N={n}")
    record_property("launches", launches)
    print(f"\ns={s} H={H}: launches per N {launches}")


@pytest.mark.parametrize("n_images", [1, 10], ids=["22-crops", "256-crops"])
def test_hd_batch_layers_and_packed_rows(n_images, record_property):
    """The hd5 workload's batch (s = 4, H = 4096; grids 9 x (5, 5) + (3, 7) = 256 crops; the (3, 7) image alone: 22 crops):
    forward_layers on the four hidden states ([N, 577, 1024] tensors, read in place) has the bits of each crop run alone through
    forward, and each image's rows of forward_packed have the bits of that image run alone through forward_packed."""
    from tokenpacker_b200.hd import n_crops
    s, H = 4, 4096
    grids = ([(5, 5)] * 9 + [(3, 7)])[-n_images:]
    n = sum(n_crops(a, b) for a, b in grids)
    m = _module(H, s, _state_dict(H, 420))
    g = torch.Generator(device=DEV).manual_seed(421)
    layers = [torch.randn((n, 577, 1024), device=DEV, generator=g).to(BF) for _ in range(4)]
    x0, xm = layers[3][:, 1:], torch.cat([t[:, 1:] for t in layers], dim=2)
    sep, ret = (torch.randn(H, device=DEV, generator=g).to(BF) for _ in range(2))
    with torch.no_grad():
        alone = torch.cat([m((x0[i:i + 1], xm[i:i + 1])) for i in range(n)])
        _assert_crops_equal(m.forward_layers(layers), alone, f"forward_layers N={n}")
        packed, cu = m.forward_packed((x0, xm), [a for a, _ in grids], [b for _, b in grids], sep, ret)
        c0 = 0
        for i, (a, b) in enumerate(grids):
            k = n_crops(a, b)
            one, one_cu = m.forward_packed((x0[c0:c0 + k], xm[c0:c0 + k]), [a], [b], sep, ret)
            assert int(cu[i + 1] - cu[i]) == int(one_cu[1]) == one.shape[0]
            assert _bits_equal(packed[int(cu[i]):int(cu[i + 1])], one), (i, a, b)
            c0 += k
    record_property("crops", n)


# ------------------------------------------------------------------------------------------------------------------------------
# forced plans
# ------------------------------------------------------------------------------------------------------------------------------
FORCED = {"one-CTA": {"TP_GEMM_MODE": "1"}, "pair": {"TP_GEMM_MODE": "2"}, "pair-ungrouped": {"TP_GEMM_MODE": "3"}, "unchained": {"TP_CHAIN": "0"}}


@pytest.mark.parametrize("s,n", [(3, 5), (3, 22), (3, 64), (2, 5), (2, 30), (2, 64)])
def test_forced_plans_give_the_default_bits(plans, pool, s, n, monkeypatch, record_property):
    """Every forced plan gives the default plan's bits at H = 4096.  At s = 2 the default is the separate plan (TP_FUSE_ATTN = 0):
    the fused plan rounds k' and v' differently by design.  N = 22 (s = 3) and N = 30 (s = 2, separate plan) mix kernels inside
    stage [3] (asserted from the engine's choices)."""
    H = 4096
    if (s, n) in ((3, 22), (2, 30)):
        stage3 = plans.forward(n, s, H, separate=True)[2]
        assert len(set(stage3)) > 1, (s, n, stage3)
    m = _module(H, s, _state_dict(H, 430 + s))
    x0, xm = pool[0][:n], pool[1][:n]
    for var in ("TP_GEMM_MODE", "TP_CHAIN", "TP_FUSE_ATTN"):
        monkeypatch.delenv(var, raising=False)
    if s in (2, 4):
        monkeypatch.setenv("TP_FUSE_ATTN", "0")
    _counted(m, x0[:1], xm[:1])                       # packs the weights
    default, launches = _counted(m, x0, xm)
    counts = {"default": launches}
    for name, env in FORCED.items():
        for var in ("TP_GEMM_MODE", "TP_CHAIN"):
            monkeypatch.delenv(var, raising=False)
        for var, value in env.items():
            monkeypatch.setenv(var, value)
        out, counts[name] = _counted(m, x0, xm)
        _assert_crops_equal(out, default, f"s={s} N={n} {name}")
    record_property("launches", counts)
    print(f"\ns={s} N={n}: launches {counts}")
    assert counts["pair"] == 3                              # chain A (point queries inside), attention, chain B
    assert counts["one-CTA"] == counts["pair-ungrouped"] == 1 + 1 + 3 + 3 + 1 + 2      # point queries, [1], [2] x 3, [3] x 3, attention, [4], [5]


# ------------------------------------------------------------------------------------------------------------------------------
# training batch invariance
# ------------------------------------------------------------------------------------------------------------------------------
R_REGIONS = ("z_kv", "h_kv", "y_k", "y_v", "k_p", "v_p")
Q_REGIONS = ("q", "y_q", "q_p", "ctx", "o", "z_m", "h_m")
assert set(R_REGIONS + Q_REGIONS + ("stats",)) == set(SAVED)


def _train_step(m, x0, xm, gout):
    """tp_forward_train + tp_backward_inputs on buffers owned here -> (step with saved views, grads, d_x0, d_xm); the backward
    workspace is kept as st.ws"""
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    st = _train_forward(m, x0, xm)
    n, s, H = st.n, st.s, st.H
    grads = [torch.full_like(t, float("nan")) for t in st.params]
    gs = _lib.TpWeights(*[t.data_ptr() for t in grads])
    ws = torch.empty(st.ws_total, dtype=torch.uint8, device=DEV)
    d_x0 = torch.full((n, 576, 1024), float("nan"), dtype=BF, device=DEV)
    d_xm = torch.full((n, 576, 4096), float("nan"), dtype=BF, device=DEV)
    _lib.check(lib.tp_backward_inputs(C.byref(st.w), st.packed.data_ptr(), xm.data_ptr(), 576 * 4096, n, s, H, gout.data_ptr(),
                                      st.saved.data_ptr(), C.byref(gs), d_x0.data_ptr(), d_xm.data_ptr(), ws.data_ptr(), st.ws_total,
                                      torch.cuda.current_stream().cuda_stream), "tp_backward_inputs")
    torch.cuda.synchronize()
    st.ws = ws
    return st, grads, d_x0, d_xm


def _crop_rows(st, i):
    """crop i's rows of the output and of every saved activation, d_x0 / d_xm excluded"""
    Mq, R = st.Mq, st.R
    rows = {"out": st.out[i * Mq:(i + 1) * Mq]}
    for k in R_REGIONS:
        rows[k] = st.sv[k][i * 576:(i + 1) * 576]
    for k in Q_REGIONS:
        rows[k] = st.sv[k][i * Mq:(i + 1) * Mq]
    stats = st.sv["stats"]
    rows["stats"] = torch.cat([stats[i * 576:(i + 1) * 576], stats[R + i * 576:R + (i + 1) * 576], stats[2 * R + i * Mq:2 * R + (i + 1) * Mq]])
    return rows


def _same(a, b):
    return torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


@pytest.mark.parametrize("s,H", TRAIN)
def test_training_crops_have_the_bits_of_the_crop_alone(plans, pool, s, H, record_property):
    m = _module(H, s, _state_dict(H, 440 + s))
    Mq = (24 // s) ** 2
    g = torch.Generator(device=DEV).manual_seed(441 + s)
    gpool = torch.randn((POOL * Mq, H), device=DEV, generator=g).to(BF)       # crop i's grad_out: rows i Mq .. (i + 1) Mq
    alone = {}

    def single(i):
        if i not in alone:
            st, _, d_x0, d_xm = _train_step(m, pool[0][i:i + 1], pool[1][i:i + 1], gpool[i * Mq:(i + 1) * Mq])
            alone[i] = {k: v.clone() for k, v in _crop_rows(st, 0).items()}
            alone[i]["d_x0"], alone[i]["d_xm"] = d_x0[0], d_xm[0]
        return alone[i]

    ns = train_ns(plans, s, H)
    for n in ns:
        off = _offset(n)
        x0, xm = pool[0][off:off + n], pool[1][off:off + n]
        gout = gpool[off * Mq:(off + n) * Mq]
        st, grads, d_x0, d_xm = _train_step(m, x0, xm, gout)
        fields = list(st.p)
        for i in range(n):
            want = single(off + i)
            got = _crop_rows(st, i)
            got["d_x0"], got["d_xm"] = d_x0[i], d_xm[i]
            differ = [k for k in want if not _same(got[k], want[k])]
            assert not differ, (f"s={s} H={H} N={n} crop {i}", differ)
        assert torch.isfinite(d_x0.float()).all() and torch.isfinite(d_xm.float()).all()
        _, grads2, _, _ = _train_step(m, x0, xm, gout)
        for f, a, b in zip(fields, grads, grads2):
            assert torch.isfinite(a.float()).all() and _bits_equal(a, b), (n, f)
        del st, grads, grads2, d_x0, d_xm
    record_property("ns", ns)
    print(f"\ntraining s={s} H={H}: N = {ns}")


# ------------------------------------------------------------------------------------------------------------------------------
# batches past 32-bit offsets
# ------------------------------------------------------------------------------------------------------------------------------
# 0-based crops: feat_multi [N, 576, 4096] passes element 2^31 in crop 910 and byte 2^31 in crop 455; at s = 1 (576 queries) the
# output [N, 576, 4096] and h_m likewise; h_kv [576 N, 2048] passes element 2^31 in crop 1820, and y_k, y_v, k', v' [576 N, 1024]
# pass byte 2^31 there
PICKS = [0, 454, 455, 456, 909, 910, 911]
BIG = [(912, 1), (912, 2), (1822, 2), (1822, 3)]


@pytest.mark.parametrize("n,s", BIG)
def test_batches_past_32_bit_offsets(n, s, record_property):
    from tokenpacker_b200 import _lib
    H = 4096
    assert 910 * 576 * 4096 < 2 ** 31 <= 911 * 576 * 4096 and 455 * 576 * 4096 * 2 < 2 ** 31 <= 456 * 576 * 4096 * 2
    assert 1820 * 576 * 2048 < 2 ** 31 <= 1821 * 576 * 2048 and 1820 * 576 * 1024 * 2 < 2 ** 31 <= 1821 * 576 * 1024 * 2
    picks = PICKS + ([1819, 1820, 1821] if n == 1822 else [])
    Mq = (24 // s) ** 2
    need = _lib.lib.tp_workspace_bytes(n, s, H) + n * 576 * 5120 * 2 + n * Mq * H * 2 + 2 * GiB       # + weights and the picks
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < need + 2 * GiB:
        pytest.skip(f"N={n} needs {need / GiB:.1f} GiB + a 2 GiB margin of device memory, {free / GiB:.1f} GiB free")
    m = _module(H, s, _state_dict(H, 450 + s))
    x0 = torch.empty((n, 576, 1024), dtype=BF, device=DEV)
    xm = torch.empty((n, 576, 4096), dtype=BF, device=DEV)
    for c0 in range(0, n, 128):
        g = torch.Generator(device=DEV).manual_seed(4500 + c0)
        k = min(128, n - c0)
        x0[c0:c0 + k] = torch.randn((k, 576, 1024), device=DEV, generator=g).to(BF)
        xm[c0:c0 + k] = torch.randn((k, 576, 4096), device=DEV, generator=g).to(BF)
    with torch.no_grad():
        alone = torch.cat([m((x0[i:i + 1], xm[i:i + 1])) for i in picks])
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    out, launches = _counted(m, x0, xm)
    wall = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() - base
    record_property("launches", launches)
    record_property("peak_bytes_above_inputs", peak)
    record_property("forward_seconds", round(wall, 3))
    print(f"\nN={n} s={s}: {launches} launches, peak {peak / GiB:.2f} GiB above the inputs, {wall:.2f} s")
    _assert_crops_equal(out[picks], alone, f"N={n} s={s}", picks)
    assert torch.isfinite(out).all()


TRAIN_BIG = 912             # s = 2, H = 4096: feat_multi and d_xm pass element 2^31 in crop 910, byte 2^31 in crop 455
WGRAD_ROWS = 64             # sampled output rows of each weight gradient checked against fp64
CHUNK = 32768               # rows of the fp64 references' contraction per step


def _wgrad_ref(dy, x, rows):
    """(dW[rows] = dY[:, rows]^T X in fp64, its fp32 floor (K + 1) E |dY[:, rows]|^T |X|), accumulated over CHUNK-row slices of
    the contraction"""
    ref = torch.zeros((len(rows), x.shape[1]), dtype=F64, device=DEV)
    mag = torch.zeros_like(ref)
    for r0 in range(0, dy.shape[0], CHUNK):
        d, xx = dy[r0:r0 + CHUNK][:, rows].to(F64), x[r0:r0 + CHUNK].to(F64)
        ref += d.t() @ xx
        mag += d.abs().t() @ xx.abs()
    return ref, (dy.shape[0] + 1) * E * mag


def test_training_past_32_bit_offsets(record_property):
    """A training step of 912 crops (s = 2, H = 4096; R = 525,312 rows): the picked crops' output, saved rows, d_x0 and d_xm have
    the bits of each crop run alone, and k/v_proj.0's weight gradients and the split-K 1024 x 1024 weight gradients of k/v_proj_1.2
    (bit for bit the fixed-order reduce of their fp32 slices, too) hold the bounds of test_train_stages_gpu.py against fp64 on
    WGRAD_ROWS seeded output rows."""
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    n, s, H = TRAIN_BIG, 2, 4096
    Mq = (24 // s) ** 2
    feats = n * 576 * 5120 * 2
    need = lib.tp_train_saved_bytes(n, s, H) + lib.tp_backward_workspace_bytes(n, s, H) + 2 * feats + 2 * n * Mq * H * 2 + 4 * GiB
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < need + 2 * GiB:
        pytest.skip(f"N={n} training needs {need / GiB:.1f} GiB + a 2 GiB margin of device memory, {free / GiB:.1f} GiB free")
    m = _module(H, s, _state_dict(H, 480))
    x0 = torch.empty((n, 576, 1024), dtype=BF, device=DEV)
    xm = torch.empty((n, 576, 4096), dtype=BF, device=DEV)
    for c0 in range(0, n, 128):
        g = torch.Generator(device=DEV).manual_seed(4800 + c0)
        k = min(128, n - c0)
        x0[c0:c0 + k] = torch.randn((k, 576, 1024), device=DEV, generator=g).to(BF)
        xm[c0:c0 + k] = torch.randn((k, 576, 4096), device=DEV, generator=g).to(BF)
    gout = torch.randn((n * Mq, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(481)).to(BF)
    alone = {}
    for i in PICKS:
        st1, _, a0, am = _train_step(m, x0[i:i + 1], xm[i:i + 1], gout[i * Mq:(i + 1) * Mq])
        alone[i] = {k: v.clone() for k, v in _crop_rows(st1, 0).items()}
        alone[i]["d_x0"], alone[i]["d_xm"] = a0[0], am[0]
    del st1, a0, am
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    st, grads, d_x0, d_xm = _train_step(m, x0, xm, gout)
    wall = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() - base
    record_property("peak_bytes_above_inputs", peak)
    record_property("step_seconds", round(wall, 3))
    print(f"\ntraining N={n}: peak {peak / GiB:.2f} GiB above the inputs, {wall:.2f} s for the step (buffers filled and synchronised)")
    for i in PICKS:
        got = _crop_rows(st, i)
        got["d_x0"], got["d_xm"] = d_x0[i], d_xm[i]
        differ = [k for k in alone[i] if not _same(got[k], alone[i][k])]
        assert not differ, (f"N={n} crop {i}", differ)
    assert torch.isfinite(d_x0.float()).all() and torch.isfinite(d_xm.float()).all() and torch.isfinite(st.out.float()).all()
    g = dict(zip(st.p, grads))
    for f, t in g.items():
        assert torch.isfinite(t.float()).all(), f
    hk = KernelHooks()
    assert st.R >= hk.split_min_rows
    R, off = st.R, st.BL
    region = lambda name, cols: st.ws[off[name][0]:off[name][0] + off[name][1]].view(BF).view(R, cols)    # noqa: E731
    dzkv, h_kv = region("dzkv", 2048), st.sv["h_kv"]
    splitk = st.ws[off["splitk"][0]:off["splitk"][0] + off["splitk"][1]].view(torch.float32).view(2, -1, 1024, 1024)
    rows = torch.randperm(1024, device=DEV, generator=torch.Generator(device=DEV).manual_seed(482))[:WGRAD_ROWS]
    xm2 = xm.reshape(R, 4096)
    for half, x in enumerate("kv"):
        ref, floor = _wgrad_ref(dzkv[:, half * 1024:(half + 1) * 1024], xm2, rows)
        _check(record_property, f"{x}_proj_0_w", g[f"{x}_proj_0_w"][rows], ref, floor)
        dy = region(f"dy{x}", 1024)
        ref, floor = _wgrad_ref(dy, h_kv[:, half * 1024:(half + 1) * 1024], rows)
        _check(record_property, f"{x}_proj_2_w", g[f"{x}_proj_2_w"][rows], ref, floor)
        assert _bits_equal(g[f"{x}_proj_2_w"], _reduce_emulated(splitk[half], 1.0)), x


# ------------------------------------------------------------------------------------------------------------------------------
# small related cases
# ------------------------------------------------------------------------------------------------------------------------------
def test_host_forward_past_its_event_ring(pool):
    """forward_host with one crop per chunk over 70 crops reuses its 64 (copy-in, compute) event pairs: the same bits as the
    device forward"""
    s, H, n = 2, 1024, 70
    m = _module(H, s, _state_dict(H, 460))
    x0, xm = pool[0][:n], pool[1][:n]
    with torch.no_grad():
        want = m((x0, xm))
    got = m.forward_host((x0.cpu().pin_memory(), xm.cpu().pin_memory()), chunk_crops=1)
    _assert_crops_equal(got.to(DEV), want, "forward_host")


def test_transpose_past_65535_row_tiles():
    """The transpose of the backward's H % 256 != 0 fallback at 2,097,153 rows (65,536 tiles of 32 rows) x 32 columns, bit for bit"""
    from test_train_stages_gpu import HOOKS
    import tokenpacker_b200  # noqa: F401
    fn = C.CDLL(HOOKS).tpt_transpose
    fn.restype, fn.argtypes = C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p]
    rows, cols = 65536 * 32 + 1, 32
    x = torch.randn((rows, cols), device=DEV, generator=torch.Generator(device=DEV).manual_seed(470)).to(BF)
    y = torch.full((cols, rows), float("nan"), dtype=BF, device=DEV)
    assert fn(x.data_ptr(), cols, y.data_ptr(), rows, rows, cols, torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    assert _bits_equal(y, x.t())
