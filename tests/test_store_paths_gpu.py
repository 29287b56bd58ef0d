"""The store side of the forward's last GEMM, on one GPU: the fused all-gather's multi-destination TMA stores, the packed-row
(crop stride M + 1) output at every scale factor, the emulated multi-rank HD all-gather and the forward plan cache.

These paths only move data, so the reference of every call is the dense [N, M, H] output of ``tp_forward`` for the same module,
inputs and plan (the per-stage float64 tests in test_forward_stages_gpu.py hold that output to fp64), and every check is bitwise:
each destination row equals the reference, and every other row of every buffer keeps its sentinel.  Buffers are filled with 0xFFFF
(a bf16 NaN) and framed by guard rows, so a store that spills one row into a separator gap, into a neighbouring rank's slot or past
either end of a buffer fails, as does a store that never happens.  Calls go through the C ABI (``tokenpacker_b200._lib``) on a
workspace the test owns.

The destinations of ``tp_forward_allgather`` are only global addresses: ordinary buffers on the current device exercise the same
maps, jobs and boxes as peer-mapped memory on other GPUs (what they do not exercise is NVLink and the cross-rank barrier).  With
eight destinations a packed slab at s = 4 needs 56 store jobs and at s = 12 needs 88, so the second and third job slot of the
store-warp lanes (jobs l + 32, l + 64) run here; the counts come from the host's worst-piece loop restated below (whose agreement
with the store warp's enumeration tests/test_store_plan_host.py checks on the CPU) and are recorded as test properties.  A store
warp that issued only each lane's first job fails exactly those two cases, with destination rows left unwritten.

The file runs in about 15 s on an H100 (80 GB HBM3, 700 W power limit).
"""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
SENT = -1                  # 0xFFFF as int16: a bf16 NaN nobody writes
GUARD = 3                  # sentinel rows before and after every buffer
SLAB, BOX_LEVELS, WHOLE_LEVELS, MAX_PEERS = 128, 4, 3, 8
H_SMALL = 256


@pytest.fixture(autouse=True)
def _default_plan(monkeypatch):
    for k in ("TP_GEMM_MODE", "TP_FUSE_ATTN", "TP_CHAIN"):
        monkeypatch.delenv(k, raising=False)


def _lib():
    from tokenpacker_b200 import _lib
    return _lib


# ------------------------------------------------------------------------------------------------------------------------------
# the host's store bookkeeping, restated
# ------------------------------------------------------------------------------------------------------------------------------
def _unit(m):
    """gcd(M, 128): the smallest store box of a packed output (seg_store_unit in tp_api.cu)"""
    u = SLAB
    while m % u:
        u >>= 1
    return u


def _worst_pieces(m, slabs=None):
    """launch_gemm_pair_group's worst-piece loop: the most store pieces a 128-row slab is cut into, over slabs (a0, end): a0 = 0 or
    minus the position of the slab's first row inside its segment, end = the slab's rows that exist.  Default: every a0 that is a
    multiple of unit with end = 128, as the host does."""
    unit, whole = _unit(m), m <= SLAB
    worst = 0
    for a0, end in (((a0, SLAB) for a0 in range(0, -m, -unit)) if slabs is None else slabs):
        pieces, a = 0, a0
        while a < end:
            if whole and a >= 0 and a + m <= SLAB:
                k = 1
                while k < WHOLE_LEVELS and a + (k + 1) * m <= end:
                    k += 1
                pieces += 1
                a += k * m
                continue
            length = min(a + m, SLAB) - max(a, 0)
            for lvl in range(BOX_LEVELS - 1, -1, -1):
                while length >= unit << lvl:
                    pieces += 1
                    length -= unit << lvl
            a += m
        worst = max(worst, pieces)
    return worst


def _call_worst_pieces(m, n):
    """the worst slab of an n-crop output: the same loop over the slabs this output has (the last one may end early)"""
    return _worst_pieces(m, [(-(r % m), min(SLAB, n * m - r)) for r in range(0, n * m, SLAB)])


def _pair_wins(rows, cols, k, sms, count):
    """choose_kernel's cost model (tp_api.cu): does the CTA-pair kernel win for a [rows, k] x [cols, k]^T GEMM of a ``count``-item
    launch?"""
    kb = -(-k // 64)

    def waves(t, u):
        return -(-t // u)
    t_pair = -(-rows // 256) * -(-cols // 256)
    t_256 = -(-rows // 128) * -(-cols // 256)
    t_128 = -(-rows // 128) * -(-cols // 128)
    l_pair = waves(t_pair, sms // 2) * kb * 1024 * 9 // 8 + 10000 // count
    l_256 = waves(t_256, sms) * kb * 1024 + 10000
    l_128 = waves(t_128, sms) * kb * 512 * 6 // 5 + 10000
    return l_pair <= l_256 and l_pair <= l_128


# ------------------------------------------------------------------------------------------------------------------------------
# module, inputs, calls on an owned workspace
# ------------------------------------------------------------------------------------------------------------------------------
_MODULES = {}
_INPUTS = {}


def _module(s, H):
    if (s, H) not in _MODULES:
        from tokenpacker_b200 import TokenPackerB200
        from tokenpacker_b200 import synthetic as syn
        m = TokenPackerB200(hidden_size=H, scale_factor=s)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in syn.synthetic_state_dict(H, seed=17 + s).items()})
        _MODULES[(s, H)] = m.to("cuda", BF).eval()
    return _MODULES[(s, H)]


def _inputs(n):
    if n not in _INPUTS:
        if len(_INPUTS) > 4:
            _INPUTS.clear()
        g = torch.Generator(device="cuda").manual_seed(1000 + n)
        _INPUTS[n] = (torch.randn(n, 576, 1024, device="cuda", generator=g).to(BF), torch.randn(n, 576, 4096, device="cuda", generator=g).to(BF))
    return _INPUTS[n]


class Forward:
    """one module and batch with a workspace of its own (0xFF-filled, 16-byte aligned)"""

    def __init__(self, m, x0, xm):
        self.lib = _lib().lib
        self.m, self.x0, self.xm = m, x0, xm
        self.n, self.s, self.H = x0.shape[0], m.scale_factor, m.hidden_size
        self.M = (24 // self.s) ** 2
        self.packed = m._packed_weights(x0.device)
        self.ws_bytes = self.lib.tp_workspace_bytes(self.n, self.s, self.H)
        self.ws = torch.full((self.ws_bytes,), 0xFF, dtype=torch.uint8, device="cuda")

    def _head(self):
        return (self.packed.data_ptr(), self.x0.data_ptr(), self.xm.data_ptr(), self.n, 576 * 1024, 576 * 4096, self.s, self.H)

    def _stream(self):
        return torch.cuda.current_stream().cuda_stream

    def dense_into(self, out_ptr):
        return self.lib.tp_forward(*self._head(), out_ptr, None, self.ws.data_ptr(), self.ws_bytes, self._stream())

    def packed_into(self, out_ptr, crop_rows):
        return self.lib.tp_forward_packed(*self._head(), out_ptr, crop_rows, self.ws.data_ptr(), self.ws_bytes, self._stream())

    def allgather(self, ptrs, crop_offset, crop_rows):
        arr = (C.c_void_p * len(ptrs))(*ptrs)
        return self.lib.tp_forward_allgather(*self._head(), arr, len(ptrs), crop_offset, crop_rows, self.ws.data_ptr(), self.ws_bytes,
                                             self._stream())

    def reference(self):
        """the dense [N, M, H] output in the current plan"""
        out = torch.empty((self.n, self.M, self.H), dtype=BF, device="cuda")
        st = self.dense_into(out.data_ptr())
        torch.cuda.synchronize()
        assert st == 0, self.lib.tp_strerror(st)
        return out


class Framed:
    """a [rows, H] bf16 destination filled with the sentinel, with GUARD sentinel rows before and after it"""

    def __init__(self, rows, H):
        self.rows, self.H = rows, H
        self.whole = torch.full((rows + 2 * GUARD, H), SENT, dtype=torch.int16, device="cuda")
        self.inner = self.whole[GUARD:GUARD + rows]

    @property
    def ptr(self):
        return self.inner.data_ptr()

    def reset(self):
        self.whole.fill_(SENT)

    def expected(self, placements):
        """sentinel everywhere except ``placements``: (first row, row stride, [n, M, H] blocks) -> crop i at first + i * stride"""
        e = torch.full_like(self.whole, SENT)
        for first, stride, block in placements:
            n, m = block.shape[:2]
            dst = e[GUARD + first:GUARD + first + n * stride].view(n, stride, self.H)
            dst[:, :m] = block.view(torch.int16)
        return e

    def check(self, placements, what):
        """bitwise against ``expected``; on a mismatch report rows that lost their sentinel and rows left unwritten"""
        e = self.expected(placements)
        if torch.equal(self.whole, e):
            return
        bad = (self.whole != e).any(-1)
        spilled = int((bad & (e == SENT).all(-1)).sum())
        unwritten = int((bad & (self.whole == SENT).all(-1)).sum())
        rows = torch.nonzero(bad).flatten()[:8].tolist()
        pytest.fail(f"{what}: {int(bad.sum())} rows differ ({spilled} sentinel rows written, {unwritten} destination rows left "
                    f"unwritten), first buffer rows (guard included) {rows}")


# ------------------------------------------------------------------------------------------------------------------------------
# 1. multi-destination stores
# ------------------------------------------------------------------------------------------------------------------------------
# N with a ragged last 256-row tile whose slabs start at every position inside a crop a 128-row slab can start at (so the
# host's worst slab occurs: at s = 4 that takes 32 crops)
_RAGGED_N = {1: 3, 2: 9, 3: 5, 4: 33, 6: 17, 8: 3, 12: 67, 24: 3}
_CACHE_REF = {}


def _ref(s, H, n):
    key = (s, H, n)
    if key not in _CACHE_REF:
        if len(_CACHE_REF) > 8:
            _CACHE_REF.clear()
        f = Forward(_module(s, H), *_inputs(n))
        _CACHE_REF[key] = (f, f.reference())
    return _CACHE_REF[key]


def _run_allgather(record, s, H, n, packed, n_peers, offsets):
    f, ref = _ref(s, H, n)
    M = f.M
    assert n * M % 256 != 0 or n == 1
    R = M + 1 if packed else M
    jobs = (_call_worst_pieces(M, n) if packed else 1) * n_peers
    record("worst_jobs_per_slab", jobs)
    assert jobs <= 96
    for off in offsets:
        total = off + n + 2                      # this rank's slot, with other ranks' crops before (off) and after (2) it
        bufs = [Framed(total * R, H) for _ in range(n_peers)]
        st = f.allgather([b.ptr for b in bufs], off, R if packed else 0)
        torch.cuda.synchronize()
        assert st == 0, f.lib.tp_strerror(st)
        for p, b in enumerate(bufs):
            b.check([(off * R, R, ref)], f"s={s} n={n} {'packed' if packed else 'dense'} destination {p}/{n_peers} crop_offset={off}")
    return jobs


@pytest.mark.parametrize("n_peers", [1, 2, 3, 8])
@pytest.mark.parametrize("packed", [False, True], ids=["dense", "packed"])
@pytest.mark.parametrize("ragged", [False, True], ids=["n1", "ragged"])
@pytest.mark.parametrize("s", [1, 2, 3, 4, 6, 12])
def test_allgather_destinations(record_property, s, ragged, packed, n_peers):
    """tp_forward_allgather into 1, 2, 3 or 8 destination buffers on this GPU, dense (out_crop_rows = 0) and packed (M + 1), at
    crop_offset 0 and 3, for one crop and for a batch with a ragged last tile.  Every destination holds the dense reference in rows
    (crop_offset + i) R .. + M - 1 and its sentinel everywhere else: the slots of the other ranks before and after, the separator
    gaps, the guard rows.  With eight destinations, s = 4 reaches 56 jobs per slab and s = 12 reaches 88."""
    n = _RAGGED_N[s] if ragged else 1
    jobs = _run_allgather(record_property, s, H_SMALL, n, packed, n_peers, (0, 3))
    if packed and ragged and n_peers == 8:
        if s == 4:
            assert jobs == 56 > 32
        if s == 12:
            assert jobs == 88 > 64


def test_allgather_destinations_h4096(record_property):
    """The same at the released width: s = 4, H = 4096 (64 column slabs per row block), packed, eight destinations, crop_offset 5,
    nine crops (324 rows: a ragged last tile)."""
    _run_allgather(record_property, 4, 4096, 9, True, 8, (5,))
    _CACHE_REF.clear()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("s", [8, 24])
def test_allgather_packed_needs_four_row_crops(s):
    """M = 9 and M = 1 (s = 8, 24) have no packed-row boxes on the pair kernel, the only kernel with peer stores: a packed all-gather
    is rejected with TP_ERR_INVALID_ARGUMENT before anything is launched, and its buffers stay untouched.  The dense all-gather of
    the same scale factors works."""
    lib = _lib()
    f, ref = _ref(s, H_SMALL, 3)
    bufs = [Framed(5 * (f.M + 1), H_SMALL) for _ in range(2)]
    torch.cuda.synchronize()
    c0 = f.lib.tp_launch_count()
    st = f.allgather([b.ptr for b in bufs], 1, f.M + 1)
    assert st == lib.TP_ERR_INVALID_ARGUMENT
    assert f.lib.tp_launch_count() == c0
    torch.cuda.synchronize()
    for b in bufs:
        b.check([], f"rejected s={s}")
    st = f.allgather([b.ptr for b in bufs], 1, 0)
    torch.cuda.synchronize()
    assert st == 0, f.lib.tp_strerror(st)
    for b in bufs:
        b.check([(f.M, f.M, ref)], f"dense s={s}")


# ------------------------------------------------------------------------------------------------------------------------------
# 2. packed rows at every scale factor, before any separator fill
# ------------------------------------------------------------------------------------------------------------------------------
_PLANS = {"default": {}, "one_cta": {"TP_GEMM_MODE": "1"}, "pair": {"TP_GEMM_MODE": "2"}, "unfused": {"TP_FUSE_ATTN": "0"}}


def _packed_case(record, monkeypatch, s, H, n, plan):
    for k, v in _PLANS[plan].items():
        monkeypatch.setenv(k, v)
    f = Forward(_module(s, H), *_inputs(n))
    ref = f.reference()
    R = f.M + 1
    out = Framed(n * R, H)
    c0 = f.lib.tp_launch_count()
    st = f.packed_into(out.ptr, R)
    torch.cuda.synchronize()
    assert st == 0, f"tp_forward_packed(s={s}, H={H}, n={n}, out_crop_rows={R}) under {plan}: status {st} ({f.lib.tp_strerror(st).decode()})"
    record("launches", int(f.lib.tp_launch_count() - c0))
    out.check([(0, R, ref)], f"packed s={s} n={n} plan={plan}")


@pytest.mark.parametrize("s,plan", [(s, p) for s in (1, 2, 3, 4, 6, 8, 12, 24) for p in ("default", "one_cta", "pair")]
                         + [(2, "unfused"), (4, "unfused")])
def test_packed_rows_every_scale(record_property, monkeypatch, s, plan):
    """tp_forward_packed (out_crop_rows = M + 1) into a sentinel buffer, read BEFORE any separator fill: crop rows equal the dense
    reference of the same plan bit for bit and every gap row keeps its sentinel.  Plans: the default, TP_GEMM_MODE=1 (one-CTA
    kernels' row stores), TP_GEMM_MODE=2 (pair kernel wherever it can store the rows: s = 8 and 24 fall back to the one-CTA
    kernels) and TP_FUSE_ATTN=0 for the fused scale factors."""
    _packed_case(record_property, monkeypatch, s, H_SMALL, _RAGGED_N[s], plan)


def test_packed_rows_s8_at_pair_kernel_size(record_property, monkeypatch):
    """s = 8 (M = 9), H = 1024 at the smallest batch for which choose_kernel's cost model sends stages [4] and [5] (Q = 9 N rows,
    1024 x 1024) to the CTA-pair kernel in a two-item chain on this GPU's SM count (228 crops on 132 SMs, 200 on 114).  The packed
    output there must leave through the one-CTA kernels' row stores, since the pair kernel has no boxes for 9-row crops (a kernel
    choice that did not know this returned TP_ERR_INVALID_ARGUMENT here, after the first stages had been launched)."""
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    n = next(n for n in range(1, 1024) if _pair_wins(9 * n, 1024, 1024, sms, 2))
    record_property("n_crops", n)
    _INPUTS.clear()
    try:
        _packed_case(record_property, monkeypatch, 8, 1024, n, "default")
    finally:
        _INPUTS.clear()
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------------
# 4. the fused HD all-gather of FusedGatherTokenPacker.forward_hd, with W ranks emulated in one process
# ------------------------------------------------------------------------------------------------------------------------------
_GRIDS = ((2, 2), (1, 1), (1, 3))          # tests/test_dist_gpu.py: 5 + 1 + 4 = 10 crops


@pytest.mark.parametrize("s,world,grids", [(4, 2, _GRIDS), (4, 3, _GRIDS), (4, 8, _GRIDS), (3, 3, _GRIDS),
                                           (4, 8, ((1, 1), (1, 2)))], ids=["s4-w2", "s4-w3", "s4-w8", "s3-w3", "s4-w8-idle"])
def test_emulated_fused_hd_allgather(s, world, grids):
    """What every rank of FusedGatherTokenPacker.forward_hd does, for W ranks in one process: fill the separator rows of its own
    buffer first, then rank r stores its crops x[lo:hi] (dist.shard_bounds) into all W buffers with forward_into_peers(crop_offset
    = lo, out_crop_rows = M + 1); a rank without crops skips the call (the last case has 4 crops on 8 ranks).  Shards are ragged and
    images straddle rank boundaries.  Every buffer must equal forward_packed bit for bit: a store that spilled into a gap would
    overwrite a separator filled before it.  The dense form (out_crop_rows = 0) must equal forward."""
    from tokenpacker_b200.dist import shard_bounds
    from tokenpacker_b200.hd import hd_plan_device, n_crops
    lib = _lib()
    m = _module(s, H_SMALL)
    M = m.num_queries
    hb, wb = [a for a, _ in grids], [b for _, b in grids]
    n = sum(n_crops(a, b) for a, b in grids)
    x0, xm = _inputs(n)
    g = torch.Generator(device="cuda").manual_seed(77)
    sep, ret = (torch.randn(H_SMALL, device="cuda", generator=g).to(BF) for _ in range(2))
    bounds = [shard_bounds(n, world, r) for r in range(world)]
    with torch.no_grad():
        ref, cu = m.forward_packed((x0, xm), hb, wb, sep, ret)
        dense = m((x0, xm))
    torch.cuda.synchronize()
    _, _, sep_rows, ret_rows = hd_plan_device(hb, wb, M, torch.device("cuda"))
    total = int(cu[-1])
    assert total == n * (M + 1)
    stream = torch.cuda.current_stream().cuda_stream
    for rows, out_rows, want in ((M + 1, total, ref.view(n, M + 1, H_SMALL)), (0, n * M, dense)):
        bufs = [Framed(out_rows, H_SMALL) for _ in range(world)]
        if rows:
            for b in bufs:
                lib.check(lib.lib.tp_hd_fill_separators(b.ptr, H_SMALL, sep_rows.data_ptr(), sep_rows.numel(), sep.data_ptr(),
                                                        ret_rows.data_ptr(), ret_rows.numel(), ret.data_ptr(), stream), "fill")
        with torch.no_grad():
            for lo, hi in bounds:
                if hi > lo:
                    m.forward_into_peers((x0[lo:hi], xm[lo:hi]), [b.ptr for b in bufs], crop_offset=lo, out_crop_rows=rows)
        torch.cuda.synchronize()
        stride = M + 1 if rows else M
        for r, b in enumerate(bufs):
            b.check([(0, stride, want)], f"rank {r}/{world} {'packed' if rows else 'dense'}")


# ------------------------------------------------------------------------------------------------------------------------------
# 5. the forward plan cache
# ------------------------------------------------------------------------------------------------------------------------------
def test_plan_cache_reuses_pointers():
    """forward_impl keeps the last four launch plans of the single-launch forward (s = 2, 4), keyed on every pointer and shape.
    Eight configurations share the module, inputs, workspace and three buffers A, B, C: A dense; A packed; A as the one destination
    of a dense all-gather; packed all-gathers into (A, B, C) at crop_offset 1, the same peers permuted (C, A, B), (A, B, C) at
    crop_offset 2, (A, B) only, and a dense all-gather into (A, B, C).  The cycle runs once (every plan built; slots evicted round
    robin), then the last four in reverse (cache hits, from every slot), then the whole cycle again (evicted plans rebuilt).  A
    plan replayed for the wrong call would store to the wrong place or through the wrong maps: every buffer is checked after
    every call."""
    s, n = 4, 3
    f, ref = _ref(s, H_SMALL, n)
    M, R = f.M, f.M + 1
    A, B, Cb = (Framed((n + 3) * R, H_SMALL) for _ in range(3))
    bufs = {"A": A, "B": B, "C": Cb}

    def gather(names, off, rows):
        return (lambda: f.allgather([bufs[k].ptr for k in names], off, rows)), {k: [(off * (rows or M), rows or M, ref)] for k in names}

    configs = [
        (lambda: f.dense_into(A.ptr), {"A": [(0, M, ref)]}),
        (lambda: f.packed_into(A.ptr, R), {"A": [(0, R, ref)]}),
        gather("A", 0, 0),
        gather("ABC", 1, R),
        gather("CAB", 1, R),
        gather("ABC", 2, R),
        gather("AB", 1, R),
        gather("ABC", 1, 0),
    ]
    order = list(range(8)) + [7, 6, 5, 4] + list(range(8))
    for step, i in enumerate(order):
        for b in bufs.values():
            b.reset()
        call, want = configs[i]
        st = call()
        torch.cuda.synchronize()
        assert st == 0, (step, i, f.lib.tp_strerror(st))
        for k, b in bufs.items():
            b.check(want.get(k, []), f"call {step} (configuration {i}), buffer {k}")
