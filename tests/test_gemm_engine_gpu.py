"""The GEMM tile engine on its own, through the test-hook library (tests/csrc/tp_test_hooks.cu: tpt_gemm_group / tpt_gemm_chain
hand arbitrary items to launch_gemms / launch_chain with a caller-chosen SM count): every operand form on every kernel that can run
it, the fused epilogues, the store paths, grouped and chained launches and the persistent schedule at any number of CTA pairs,
against float64 products of the same bf16 operands.

Tolerances are derived from the arithmetic, as in tests/test_train_kernels_gpu.py: |got - ref| <= U |ref| + (1 + U) floor
elementwise, with U = 2^-8 (the bf16 rounding of the stored result) and floor = (K + 1) E sum_k |a_ik| |b_kj| (the fp32
accumulation, E = 2^-24), plus one rounding per further fp32 step of the epilogue (bias, alpha), GELU's derivative bound 1.13 on
that error plus the 1e-6 |z| of its erf approximation, and for the LayerNorm fold the error bounds of ln_row_stats.  The worst
ratio error / bound of every check is recorded as a test property (``pytest -o junit_family=legacy --junitxml``).

Every output lives inside a larger buffer filled with a NaN sentinel: guard rows above and below, guard columns up to ldc > N, the
gap rows of segmented and scattered outputs, the unused split-K slice.  Every guard must keep its sentinel bits and every element
of C must be written.  Every test asserts, through tpt_gemm_choice, that the kernel it means to exercise is the one that ran:
kernel 0 = the CTA-pair kernel (tp_gemm2_kernel, 256 x 256 tiles), 1 / 2 = the one-CTA kernel with 128 x 256 / 128 x 128 tiles.
"""
import contextlib
import ctypes as C
import os
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOOKS = os.path.join(ROOT, "tokenpacker_b200", "libtokenpacker_b200_testhooks.so")
E = 2.0 ** -24            # fp32 unit roundoff
U = 2.0 ** -8             # bf16 unit roundoff
F64 = torch.float64
BF = torch.bfloat16
GELU_LIP = 1.13           # max |GELU'(z)| = 1.1289 (at z = sqrt 2)
GELU_APPROX = 1e-6        # |GELU error| / |z| of the Abramowitz & Stegun erf the epilogue evaluates in fp32
GUARD = 3                 # sentinel rows above and below every output
SENT16 = 0x7FA5           # bf16 NaN no kernel stores: the bits of every element the engine must not write
SENT32 = 0x7FA5A5A5       # the same for fp32 outputs (split-K slices, row statistics)
PAIR, ONE_256, ONE_128 = 0, 1, 2
INVALID = 1               # TP_ERR_INVALID_ARGUMENT
SMS_SWEEP = (2, 4, 10, 114)


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


class Hooks:
    def __init__(self):
        import tokenpacker_b200  # noqa: F401  (the product library is loaded next to this one, as in a real process)
        assert os.path.exists(HOOKS), f"{HOOKS} missing: build with `make -C tokenpacker_b200/csrc`"
        lib = C.CDLL(HOOKS)
        dp = C.POINTER(Desc)
        for name, res, args in (("tpt_launch_count", C.c_uint64, []), ("tpt_gemm_desc_size", C.c_int, []),
                                ("tpt_gemm_group", C.c_int, [dp, C.c_int, C.c_int, C.c_void_p]),
                                ("tpt_gemm_chain", C.c_int, [dp, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]),
                                ("tpt_gemm_choice", C.c_int, [dp, C.c_int, C.c_int])):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        self.lib = lib
        self.sms = torch.cuda.get_device_properties(0).multi_processor_count
        assert lib.tpt_gemm_desc_size() == C.sizeof(Desc), "tpt_gemm_desc layout drifted from its Python mirror"

    def launches(self):
        torch.cuda.synchronize()
        return self.lib.tpt_launch_count()

    def group(self, items, sms=None):
        arr = (Desc * len(items))(*[it.desc for it in items])
        return self.lib.tpt_gemm_group(arr, len(items), sms or self.sms, torch.cuda.current_stream().cuda_stream)

    def chain(self, items, flags, sms=None):
        arr = (Desc * len(items))(*[it.desc for it in items])
        return self.lib.tpt_gemm_chain(arr, len(items), flags.data_ptr(), flags.numel(), sms or self.sms,
                                       torch.cuda.current_stream().cuda_stream)

    def choice(self, item, count=1, sms=None):
        return self.lib.tpt_gemm_choice(C.byref(item.desc), count, sms or self.sms)


@pytest.fixture(scope="module")
def hk():
    return Hooks()


@pytest.fixture(autouse=True)
def _fp64_exact_and_default_engine():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    with _env(TP_GEMM_MODE=None, TP_CHAIN=None):
        yield
    torch.backends.cuda.matmul.allow_tf32 = old
    torch.cuda.empty_cache()


@contextlib.contextmanager
def _env(**kv):
    """TP_GEMM_MODE / TP_CHAIN for the calls inside (the engine reads them per call); None: unset"""
    old = {k: os.environ.get(k) for k in kv}

    def put(d):
        for k, v in d.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = str(v)
    put(kv)
    try:
        yield
    finally:
        put(old)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _r8(n):
    return (n + 7) // 8 * 8


def _sentinel(shape, dtype):
    t = torch.empty(shape, dtype=dtype, device="cuda")
    if dtype == BF:
        t.view(torch.int16).fill_(SENT16)
    else:
        t.view(torch.int32).fill_(SENT32)
    return t


def _bits(t):
    return t.view(torch.int16) if t.dtype == BF else t.view(torch.int32)


def _ratio(record, name, got, ref, floor, bf16=True):
    """bf16 result: |got - ref| <= U |ref| + (1 + U) floor; fp32 result: |got - ref| <= floor.  Records the worst ratio."""
    got = got.to(F64)
    assert torch.isfinite(got).all(), name
    bound = (U * ref.abs() + (1 + U) * floor) if bf16 else floor
    ratio = float(((got - ref).abs() / bound.clamp_min(1e-300)).max()) if got.numel() else 0.0
    record(name, f"{ratio:.3g}")
    assert ratio <= 1.0, (name, ratio)
    return ratio


def _store(mat, kind, seg_rows=576):
    """bf16 [rows, cols] into a NaN-padded buffer the way an operand of that kind lies in memory: 'plain' (ld = cols rounded to 8),
    'strided' (ld > cols) or 'crop' (segments of seg_rows rows, one NaN row between segments).  Returns (buffer, ld, seg_rows,
    seg_stride) in elements; the NaN padding is never inside the operand, so reading it would poison the result."""
    rows, cols = mat.shape
    if kind == "crop":
        assert rows % seg_rows == 0
        ld = _r8(cols)
        buf = torch.full((rows // seg_rows, seg_rows + 1, ld), float("nan"), dtype=BF, device="cuda")
        buf[:, :seg_rows, :cols] = mat.reshape(rows // seg_rows, seg_rows, cols)
        return buf, ld, seg_rows, (seg_rows + 1) * ld
    ld = _r8(cols) + (40 if kind == "strided" else 0)
    buf = torch.full((rows, ld), float("nan"), dtype=BF, device="cuda")
    buf[:, :cols] = mat
    return buf, ld, 0, 0


class Item:
    """One engine item: C = epilogue(A . B^T) in the operand form ``form`` (0: A [M, K], B [N, K];  1 (TN): A [K, M], B [K, N];
    2 (NN): A [M, K], B [K, N]), its bf16 operands laid out as ``a`` / ``b`` say, split into ``parts`` / ``b_parts`` tensors, and
    sentinel-filled outputs: ``out`` = 'plain', 'seg' (uniform-stride segments of seg = (len, stride) rows) or 'scatter' (segments
    at arbitrary row offsets); ``splits`` > 1: fp32 split-K slices."""

    def __init__(self, form, M, N, K, seed, a="plain", parts=1, b="plain", b_parts=1, bias=False, gelu=False, alpha=1.0, dual=False,
                 splits=1, out="plain", seg=(36, 37), ln=False, stats=False, a_src=None, ints=False):
        self.form, self.M, self.N, self.K, self.gelu, self.alpha, self.dual = form, M, N, K, gelu, alpha, dual
        self.splits, self.out, self.seg, self.ln, self.stats = splits, out, seg, ln, stats
        g = _gen(seed)
        if a_src is not None:                          # a chain consumer: A is the producer's stored C (a [M, K] view)
            at = a_src
        elif ln:                                       # rows of three kinds: ordinary, |mean| >> std, moderate offset
            kind = torch.arange(M, device="cuda") % 3
            mean = torch.where(kind == 1, 20.0, torch.where(kind == 2, -2.0, 0.0)) * torch.sign(torch.randn(M, device="cuda", generator=g))
            std = torch.where(kind == 1, 0.25, 1.0)
            at = (torch.randn(M, K, device="cuda", generator=g) * std[:, None] + mean[:, None]).to(BF)
        elif ints:                                     # integers in [-3, 3]: every fp32 partial sum is exact while 9 K < 2^24
            at = torch.randint(-3, 4, (M, K), device="cuda", generator=g).to(BF)
        else:
            at = torch.randn(M, K, device="cuda", generator=g).to(BF)
        if ints:
            bt = torch.randint(-3, 4, (N, K), device="cuda", generator=g).to(BF)
        else:
            bt = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(BF)
        self.at, self.bt = at, bt
        self.keep = []
        d = Desc()
        d.tn, d.M, d.N, d.K, d.alpha, d.gelu, d.dual, d.k_splits, d.dep = form, M, N, K, alpha, int(gelu), int(dual), splits, -1
        d.ln_inv_dim = 1.0 / 1024
        # A
        if a_src is not None:
            d.a, d.lda = a_src.data_ptr(), a_src.stride(0)
        else:
            a_log = at if form != 1 else at.t()
            if form == 1:
                assert parts == 1
            chunks = a_log.chunk(parts, dim=1) if parts > 1 else [a_log]
            ptrs = []
            for ch in chunks:
                buf, ld, sr, ss = _store(ch, a)
                self.keep.append(buf)
                ptrs.append(buf.data_ptr())
                d.lda, d.a_seg_rows, d.a_seg_stride = ld, sr, ss
            d.a, d.a_parts = ptrs[0], parts
            for i, p in enumerate(ptrs[1:]):
                d.a_more[i] = p
        # B
        b_log = bt if form == 0 else bt.t()
        bch = b_log.chunk(b_parts, dim=1) if b_parts > 1 else [b_log]
        ptrs = []
        for ch in bch:
            buf, ld, sr, ss = _store(ch.contiguous(), b)
            self.keep.append(buf)
            ptrs.append(buf.data_ptr())
            d.ldb, d.b_seg_rows, d.b_seg_stride = ld, sr, ss
        d.b, d.b_parts = ptrs[0], b_parts
        for i, p in enumerate(ptrs[1:]):
            d.b_more[i] = p
        # epilogue inputs
        self.bias = (torch.randn(N, device="cuda", generator=g) * 0.5) if bias else None
        d.bias = self.bias.data_ptr() if bias else None
        if ln:
            assert K % 128 == 0
            slots = K // 128
            ab = at.to(F64).view(M, slots, 128)
            mb = ab.mean(-1)
            self.stats_in = torch.stack([mb, ((ab - mb[..., None]) ** 2).sum(-1)], -1).to(torch.float32).contiguous()
            self.col_a = bt.to(F64).sum(1).to(torch.float32)        # row sums of the weight: the fold cancels the mean
            d.col_a, d.stats_in, d.stats_in_slots, d.ln_inv_dim = self.col_a.data_ptr(), self.stats_in.data_ptr(), slots, 1.0 / K
        # outputs
        self.ldc = N + 32
        if splits > 1:
            self.buf = _sentinel((2 * GUARD + (splits + 1) * M, self.ldc), torch.float32)
            d.out_f32 = 1
            self.rows = GUARD + torch.arange(M, device="cuda")
        elif out == "plain":
            self.buf = _sentinel((2 * GUARD + M, self.ldc), BF)
            self.rows = GUARD + torch.arange(M, device="cuda")
        else:
            L, S = seg
            assert M % L == 0
            n = M // L
            r = torch.arange(M, device="cuda")
            if out == "seg":
                d.seg_len, d.seg_stride = L, S
                dst = (r // L) * S + r % L
                total = n * S
            else:                                      # scattered: segments in a shuffled order, 3 gap rows between neighbours
                perm = torch.randperm(n, device="cuda", generator=g)
                self.offsets = (perm * (L + 3) + 1).to(torch.int64)
                d.seg_len, d.seg_row_offset = L, self.offsets.data_ptr()
                dst = self.offsets[r // L] + r % L
                total = n * (L + 3) + 1
            self.buf = _sentinel((2 * GUARD + total, self.ldc), BF)
            self.rows = GUARD + dst
        d.c, d.ldc = self.buf[GUARD].data_ptr(), self.ldc
        if dual:
            self.pre = _sentinel((2 * GUARD + M, self.ldc), BF)
            d.c_pre, d.ld_pre = self.pre[GUARD].data_ptr(), self.ldc
        if stats:
            self.st = _sentinel((2 * GUARD + M, N // 128, 2), torch.float32)
            d.stats_out, d.stats_out_slots = self.st[GUARD].data_ptr(), N // 128
        self.desc = d

    def outputs(self):
        return [t for t in (self.buf, getattr(self, "pre", None), getattr(self, "st", None)) if t is not None]

    def reset(self):
        for t in self.outputs():
            _bits(t).fill_(SENT16 if t.dtype == BF else SENT32)

    def snapshot(self):
        return [_bits(t).clone() for t in self.outputs()]

    def c(self, split=0):
        """the stored C (or split-K slice) as [M, N]"""
        return self.buf[self.rows + split * self.M, :self.N]

    def check_guards(self):
        """every element outside the outputs keeps the sentinel, every element inside was written"""
        for t, rows, cols in self._regions():
            inside = torch.zeros(t.shape[:2], dtype=torch.bool, device="cuda")
            inside[rows[:, None], torch.arange(cols, device="cuda")[None]] = True
            b = _bits(t)
            s = SENT16 if t.dtype == BF else SENT32
            b2 = b.reshape(b.shape[0], b.shape[1], -1)
            assert bool((b2[~inside] == s).all()), "a guard element was overwritten"
            assert bool((b2[inside] != s).all()), "an element of the output was not written"

    def _regions(self):
        r = [(self.buf, torch.cat([self.rows + s * self.M for s in range(self.splits)]), self.N)]
        if self.dual:
            r.append((self.pre, GUARD + torch.arange(self.M, device="cuda"), self.N))
        if self.stats:
            r.append((self.st, GUARD + torch.arange(self.M, device="cuda"), self.N // 128))
        return r

    # ---- fp64 references ----
    def _pre(self):
        """(z, floor): the fp64 pre-activation (after bias / LayerNorm fold) and the floor of the kernel's fp32 value of it"""
        a, b = self.at.to(F64), self.bt.to(F64)
        acc = a @ b.t()
        f_acc = (self.K + 1) * E * (a.abs() @ b.abs().t())
        bias = self.bias.to(F64) if self.bias is not None else torch.zeros(self.N, dtype=F64, device="cuda")
        if not self.ln:
            z = acc + bias
            return z, f_acc + E * z.abs()
        st = self._ln_stats()
        col_a = self.col_a.to(F64)
        pre = acc - st["mu"][:, None] * col_a
        rstd = st["rstd"][:, None]
        z = rstd * pre + bias
        f_inner = f_acc + st["dmu"][:, None] * col_a.abs() + E * pre.abs()
        return z, rstd * f_inner + st["rho"][:, None] * rstd * pre.abs() + E * z.abs()

    def _ln_stats(self):
        """ln_row_stats from the fp32 (mean, M2) slots, in fp64, with the error bounds of its fp32 sequence (slots adds for the mean,
        slots fmas for the between-block term, rsqrtf: 2 ulp); eps = 1e-6"""
        s = self.stats_in.to(F64)
        mb, m2 = s[..., 0], s[..., 1]
        slots = mb.shape[1]
        mu = mb.mean(-1)
        dmu = E * mb.abs().sum(-1) + 2 * E * mu.abs()
        dd = mb - mu[:, None]
        f_d = dmu[:, None] + E * dd.abs()
        between = (dd * dd).sum(-1)
        f_between = (2 * dd.abs() * f_d + f_d * f_d).sum(-1) + slots * E * between
        m2t = m2.sum(-1)
        var = (128 * between + m2t) / self.K
        f_var = (128 * f_between + slots * E * m2t) / self.K + 3 * E * var
        return {"mu": mu, "dmu": dmu, "rstd": 1 / torch.sqrt(var + 1e-6), "rho": 0.5 * (f_var + E * (var + 1e-6)) / (var + 1e-6) + 4 * E}

    def reference(self):
        """(ref, floor) of the stored C before its bf16 rounding"""
        z, f = self._pre()
        if self.gelu:
            v = torch.nn.functional.gelu(z)
            f = GELU_LIP * f + GELU_APPROX * z.abs() + 4 * E * v.abs() + 2.0 ** -133
        else:
            v = z
        if self.alpha != 1.0:
            v = self.alpha * v
            f = abs(self.alpha) * f + E * v.abs()
        return v, f

    def check(self, record, name):
        self.check_guards()
        worst = 0.0
        if self.splits > 1:
            a, b = self.at.to(F64), self.bt.to(F64)
            per = ((self.K + 63) // 64 + self.splits - 1) // self.splits * 64
            for s in range(self.splits):
                k0, k1 = s * per, min(self.K, (s + 1) * per)
                ref = self.alpha * (a[:, k0:k1] @ b[:, k0:k1].t())
                floor = abs(self.alpha) * (k1 - k0 + 1) * E * (a[:, k0:k1].abs() @ b[:, k0:k1].abs().t()) + E * ref.abs()
                worst = max(worst, _ratio(record, f"{name}_slice{s}", self.c(s), ref, floor, bf16=False))
            return worst
        ref, floor = self.reference()
        worst = _ratio(record, name, self.c(), ref, floor)
        if self.dual:
            z, fz = self._pre()
            worst = max(worst, _ratio(record, name + "_pre", self.pre[GUARD:GUARD + self.M, :self.N], z, fz))
        if self.stats:
            self._check_stats(record, name)
        return worst

    def _check_stats(self, record, name):
        """fp64 per-128-column (mean, M2) of the STORED bf16 row against the kernel's fp32 sequence (shift = the block's first value;
        s1 = 64 pair sums, s2 = 128 fmas; mean = shift + s1 / 128, M2 = max(s2 - s1 dm, 0))"""
        yd = self.c().to(F64).view(self.M, -1, 128)
        mean = yd.mean(-1)
        m2 = ((yd - mean[..., None]) ** 2).sum(-1)
        d = yd - yd[..., :1]
        S1, S2, A1 = d.sum(-1), (d * d).sum(-1), d.abs().sum(-1)
        f_s1, f_s2 = 66 * E * A1, 131 * E * S2
        dm = S1 / 128
        f_dm = f_s1 / 128 + E * dm.abs()
        got = self.st[GUARD:GUARD + self.M]
        _ratio(record, name + "_stats_mean", got[..., 0], mean, f_dm + E * mean.abs(), bf16=False)
        _ratio(record, name + "_stats_m2", got[..., 1], m2, f_s2 + f_s1 * dm.abs() + S1.abs() * f_dm + E * (S2 + f_s2), bf16=False)


def _run(hk, items, sms=None, mode=None, expect=None, launches=None):
    """one tpt_gemm_group call under TP_GEMM_MODE = mode; asserts the kernel choice of every item (expect: one id for all, or a
    list) and, if given, the number of kernels launched"""
    with _env(TP_GEMM_MODE=mode):
        if expect is not None:
            exp = expect if isinstance(expect, list) else [expect] * len(items)
            got = [hk.choice(it, len(items), sms) for it in items]
            assert got == exp, (got, exp)
        n0 = hk.launches()
        assert hk.group(items, sms) == 0
        n1 = hk.launches()
    if launches is not None:
        assert n1 - n0 == launches, (n1 - n0, launches)


def _one_cta(N):
    return ONE_256 if N % 256 == 0 else ONE_128


def _modes(N):
    """(TP_GEMM_MODE, kernel) of every forced choice the plain form allows at this N"""
    return [("1", _one_cta(N))] + ([("2", PAIR)] if N % 256 == 0 else [])


def _same_bits(x, y):
    return len(x) == len(y) and all(torch.equal(p, q) for p, q in zip(x, y))


# ------------------------------------------------------------------------------------------------------------------------------
# operand forms x kernels at the edges
# ------------------------------------------------------------------------------------------------------------------------------
_MS = [1, 64, 127, 129, 256, 257, 1000]
_NS = [32, 96, 160, 256, 512, 1280]
_KS = [1, 8, 48, 64, 72, 1000, 4104]
# every M, N and K at least once and 14 distinct (M, K) pairs (index rotations with steps coprime to the list lengths, K shifted by
# one on the second pass), then the largest of each together and a ragged M with a 40-column K tail on all three kernels
_ABT = [(_MS[i % 7], _NS[(5 * i) % 6], _KS[(3 * i + i // 7) % 7]) for i in range(14)] + [(1000, 1280, 4104), (257, 512, 1000)]


@pytest.mark.parametrize("m,n,k", _ABT)
def test_abt_every_kernel(hk, record_property, m, n, k):
    """C = A B^T on the one-CTA kernel (TP_GEMM_MODE=1), the pair kernel (=2, where N % 256 == 0) and the cost-based choice, A
    strided (lda > K, NaN between rows) in every other case: each against fp64, all guards intact, and all kernels bit for bit
    alike."""
    it = Item(0, m, n, k, seed=m * 31 + n * 7 + k, a="strided" if _ABT.index((m, n, k)) % 2 else "plain")
    results = {}
    for mode, kern in _modes(n):
        it.reset()
        _run(hk, [it], mode=mode, expect=kern)
        it.check(record_property, f"mode{mode}")
        results[kern] = it.snapshot()
    it.reset()
    kern = hk.choice(it)
    _run(hk, [it], expect=kern)
    it.check(record_property, "default")
    for other in results.values():
        assert _same_bits(it.snapshot(), other), "kernels disagree"


_TN = [(1, 256, 1), (100, 512, 63), (256, 256, 65), (300, 512, 576), (1, 512, 16704), (300, 256, 16704), (100, 256, 576),
       (256, 512, 1)]


@pytest.mark.parametrize("m,n,k", _TN)
def test_tn_form(hk, record_property, m, n, k):
    """C = A^T B (A [K, M], B [K, N] row-major; the weight-gradient form, contraction over K rows) on the pair kernel."""
    it = Item(1, m, n, k, seed=m + 3 * n + k)
    _run(hk, [it], expect=PAIR)
    it.check(record_property, "tn")


_NN = [(1, 256, 1), (129, 768, 32), (300, 256, 160), (1, 768, 1000), (129, 256, 1000), (300, 768, 1)]


@pytest.mark.parametrize("m,n,k", _NN)
def test_nn_form(hk, record_property, m, n, k):
    """C = A B (B [K, N] row-major: the input-gradient form with the weight as stored) on the pair kernel, alpha = 0.5."""
    it = Item(2, m, n, k, seed=m + 5 * n + k, alpha=0.5)
    _run(hk, [it], expect=PAIR)
    it.check(record_property, "nn")


@pytest.mark.parametrize("form,a,parts,mode,kern", [
    (0, "strided", 1, "1", ONE_256), (0, "strided", 1, "2", PAIR), (0, "crop", 1, "1", ONE_256), (0, "crop", 1, "2", PAIR),
    (0, "crop", 1, "1", ONE_128), (2, "crop", 1, None, PAIR), (2, "strided", 1, None, PAIR),
    (0, "plain", 2, None, PAIR), (0, "plain", 3, None, PAIR), (0, "strided", 4, None, PAIR), (0, "crop", 4, None, PAIR)])
def test_a_operand_layouts(hk, record_property, form, a, parts, mode, kern):
    """A as a strided view, as a crop-strided 3-D operand (576-row segments 577 rows apart: a [:, 1:] view of CLIP hidden states)
    and as 2 to 4 tensors side by side along K (the four CLIP layers); ragged M except where the crops fix it."""
    M = 1152 if a == "crop" else 300
    N = 160 if kern == ONE_128 else 512
    K = {1: 200, 2: 256, 3: 384, 4: 1024}[parts]
    it = Item(form, M, N, K, seed=17 + parts + M + N, a=a, parts=parts)
    _run(hk, [it], mode=mode, expect=kern)
    it.check(record_property, f"{a}{parts}")


@pytest.mark.parametrize("b,b_parts,n,k", [("plain", 2, 512, 300), ("plain", 3, 768, 65), ("plain", 4, 1024, 576),
                                           ("crop", 1, 256, 1152), ("crop", 4, 1024, 1152)])
def test_tn_b_operand_layouts(hk, record_property, b, b_parts, n, k):
    """TN form with B as 2 to 4 tensors side by side along N and / or with crop-strided K rows (576-row segments 577 rows apart)."""
    it = Item(1, 300, n, k, seed=23 + b_parts + k, b=b, b_parts=b_parts)
    _run(hk, [it], expect=PAIR)
    it.check(record_property, f"{b}{b_parts}")


@pytest.mark.parametrize("form,m,n,k,mode,kern", [(0, 257, 512, 4104, "1", ONE_256), (0, 257, 512, 4104, "2", PAIR),
                                                    (0, 129, 160, 4104, "1", ONE_128), (1, 300, 512, 16704, None, PAIR),
                                                    (1, 256, 256, 36864, None, PAIR), (2, 129, 768, 16704, None, PAIR)])
def test_exact_at_large_k(hk, form, m, n, k, mode, kern):
    """Integer operands in [-3, 3] at large K: every product and partial sum is exact in fp32 (9 K < 2^24), so C must be the bf16
    rounding of the exact product, bit for bit.  At these K the derived fp64 bound is loose (it grows like K, the actual error like
    sqrt K); here a single lost, repeated or misplaced k-block changes the result."""
    it = Item(form, m, n, k, seed=97 + k + n, ints=True)
    _run(hk, [it], mode=mode, expect=kern)
    it.check_guards()
    exact = (it.at.to(F64) @ it.bt.to(F64).t()).to(BF)
    assert torch.equal(_bits(it.c().contiguous()), _bits(exact))


# ------------------------------------------------------------------------------------------------------------------------------
# epilogues
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alpha", [1.0, 0.5, -3.0])
@pytest.mark.parametrize("gelu", [False, True])
@pytest.mark.parametrize("mode,kern,n", [("1", ONE_128, 160), ("1", ONE_256, 512), ("2", PAIR, 512)])
def test_epilogue_bias_gelu_alpha(hk, record_property, alpha, gelu, mode, kern, n):
    """v = alpha GELU(acc + bias) (or without GELU) at a ragged M and a K tail, on every kernel."""
    it = Item(0, 257, n, 200, seed=41 + n + int(gelu), bias=True, gelu=gelu, alpha=alpha)
    _run(hk, [it], mode=mode, expect=kern)
    it.check(record_property, "epilogue")


@pytest.mark.parametrize("m,alpha", [(100, 1.0), (257, -3.0)])
def test_epilogue_dual(hk, record_property, m, alpha):
    """dual: the pre-activation z = bf16(acc + bias) goes to c_pre and the activation bf16(alpha GELU(z_fp32)) to C, both against
    fp64 and both with every guard intact."""
    it = Item(0, m, 512, 200, seed=43 + m, bias=True, gelu=True, alpha=alpha, dual=True)
    _run(hk, [it], expect=PAIR)
    it.check(record_property, "dual")


@pytest.mark.parametrize("m,k", [(129, 1024), (257, 256), (1000, 1024)])
@pytest.mark.parametrize("mode,kern", [("1", ONE_256), ("2", PAIR)])
def test_epilogue_layernorm_fold(hk, record_property, m, k, mode, kern):
    """LayerNorm folded into the GEMM: v = rstd (acc - mu col_a) + col_b with (mu, rstd) combined from test-built per-128-column
    (mean, M2) slots; rows with |mean| >> std, where the fold cancels."""
    it = Item(0, m, 512, k, seed=47 + m + k, bias=True, ln=True)
    _run(hk, [it], mode=mode, expect=kern)
    it.check(record_property, "ln_fold")


@pytest.mark.parametrize("m,n", [(129, 256), (257, 1024), (1000, 256)])
@pytest.mark.parametrize("mode,kern", [("1", ONE_256), ("2", PAIR)])
def test_epilogue_stats_out(hk, record_property, m, n, mode, kern):
    """Per-128-column (mean, M2) of the stored bf16 row (the next LayerNorm's input), ragged M: rows >= M keep their sentinels."""
    it = Item(0, m, n, 300, seed=53 + m + n, bias=True, gelu=True, stats=True)
    _run(hk, [it], mode=mode, expect=kern)
    it.check(record_property, "stats")


@pytest.mark.parametrize("form,m,n,k,splits", [(1, 256, 256, 1000, 3), (1, 300, 512, 16704, 4), (0, 129, 256, 640, 2)])
def test_split_k_slices(hk, record_property, form, m, n, k, splits):
    """Split-K: fp32 slice s = the product over its own k-blocks, ragged M; rows >= M and the unused slice after the last keep
    their sentinels."""
    it = Item(form, m, n, k, seed=59 + k, splits=splits)
    _run(hk, [it], expect=PAIR)
    it.check(record_property, "splitk")


@pytest.mark.parametrize("out,seg", [("seg", (36, 37)), ("seg", (144, 145)), ("scatter", (36, 0)), ("scatter", (144, 0))])
@pytest.mark.parametrize("mode,kern", [("1", ONE_256), ("2", PAIR)])
def test_segmented_and_scattered_stores(hk, record_property, out, seg, mode, kern):
    """Rows in segments of seg_len: uniformly strided (the packed HD layout, one separator row after each crop) or at arbitrary
    offsets; gap rows keep their sentinels."""
    it = Item(0, seg[0] * 7, 512, 256, seed=61 + seg[0], bias=True, gelu=True, out=out, seg=seg)
    _run(hk, [it], mode=mode, expect=kern)
    it.check(record_property, out)


# ------------------------------------------------------------------------------------------------------------------------------
# bit identity: kernels, grouping, chaining, SM counts
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(m=257, k=72), dict(m=129, k=384, ln=True), dict(m=1000, k=4104, stats=True, gelu=True),
                                dict(m=1, k=8, bias=True, alpha=-3.0)])
def test_one_cta_and_pair_same_bits(hk, kw):
    """Wherever both can run (plain form, N % 256 == 0), the one-CTA and the pair kernel store the same bits: K tails, the LayerNorm
    fold, row statistics."""
    kw = dict(kw)
    m, k = kw.pop("m"), kw.pop("k")
    kw.setdefault("bias", True)
    it = Item(0, m, 512, k, seed=67 + m + k, **kw)
    _run(hk, [it], mode="1", expect=ONE_256)
    one = it.snapshot()
    it.reset()
    _run(hk, [it], mode="2", expect=PAIR)
    it.check_guards()
    assert _same_bits(it.snapshot(), one)


def _group_items(size):
    """8 heterogeneous items of one launch, ragged, in a seeded shuffled order: NT with bias + GELU, TN, NN, split-K, dual,
    segmented output, row statistics, LayerNorm fold.  'small': 15 pair tiles; 'large': 216, more than a full H100 SXM has CTA
    pairs (66), so that every SM count of the sweep walks its own tile sequence."""
    if size == "small":
        items = [Item(0, 257, 256, 72, 71, bias=True, gelu=True), Item(1, 300, 256, 65, 72), Item(2, 129, 256, 160, 73, alpha=0.5),
                 Item(1, 256, 256, 1000, 74, splits=3), Item(0, 100, 512, 128, 75, bias=True, gelu=True, alpha=-3.0, dual=True),
                 Item(0, 36 * 7, 256, 64, 76, out="seg", seg=(36, 37)), Item(0, 257, 256, 256, 77, stats=True),
                 Item(0, 129, 512, 256, 78, bias=True, ln=True)]
    else:
        items = [Item(0, 2049, 1024, 72, 171, bias=True, gelu=True), Item(1, 1300, 1024, 65, 172),
                 Item(2, 1025, 1280, 160, 173, alpha=0.5), Item(1, 512, 1024, 1000, 174, splits=3),
                 Item(0, 1000, 1536, 128, 175, bias=True, gelu=True, alpha=-3.0, dual=True),
                 Item(0, 36 * 57, 768, 64, 176, out="seg", seg=(36, 37)), Item(0, 2049, 1024, 256, 177, stats=True),
                 Item(0, 1025, 1024, 256, 178, bias=True, ln=True)]
    random.Random(5).shuffle(items)
    return items


def _pair_tiles(items):
    return sum(-(-it.M // 256) * -(-it.N // 256) * it.splits for it in items)


def _pairs(tiles, sms):
    """CTA pairs of a pair-kernel launch (launch_gemm_pair_group's grid): one per tile, at most sms / 2"""
    return min(tiles, sms // 2)


def _assert_sweep_reschedules(hk, tiles, large):
    """a large problem must run on fewer CTA pairs at every SM count of the sweep than on the whole device: each pair walks another
    tile sequence, instead of the full-device launch running again"""
    if large:
        assert tiles > hk.sms // 2, tiles
        for sms in SMS_SWEEP:
            if sms < hk.sms:
                assert _pairs(tiles, sms) < _pairs(tiles, hk.sms), (sms, tiles)


@pytest.mark.parametrize("size", ["small", "large"])
def test_group_same_bits_alone_ungrouped_and_any_sm_count(hk, record_property, size):
    """Each item of a grouped launch (TP_GEMM_MODE=2: every item on the pair kernel, one launch) against fp64, and bit for bit equal
    to the same item launched alone, to the ungrouped launches (TP_GEMM_MODE=3) and to the grouped launch at 2, 4, 10 and 114 SMs.
    The small group (15 tiles) runs on 1, 2, 5 and 15 pairs, the last the same grid as the full device; the large one (216 tiles)
    on 1, 2, 5 and 57 pairs against 66 on an H100 SXM: other tile sequences per pair, ring phases and slab numbers."""
    items = _group_items(size)
    _assert_sweep_reschedules(hk, _pair_tiles(items), size == "large")
    _run(hk, items, mode="2", expect=PAIR, launches=1)
    for i, it in enumerate(items):
        it.check(record_property, f"item{i}")
    ref = [it.snapshot() for it in items]
    for it, r in zip(items, ref):
        it.reset()
        _run(hk, [it], mode="2", expect=PAIR, launches=1)
        assert _same_bits(it.snapshot(), r), "alone"
    for it in items:
        it.reset()
    _run(hk, items, mode="3", expect=PAIR, launches=len(items))
    for it, r in zip(items, ref):
        assert _same_bits(it.snapshot(), r), "ungrouped"
    for sms in SMS_SWEEP:
        for it in items:
            it.reset()
        _run(hk, items, sms=sms, mode="2", expect=PAIR, launches=1)
        for i, (it, r) in enumerate(zip(items, ref)):
            it.check_guards()
            assert _same_bits(it.snapshot(), r), (sms, i)


def _chain(M, seed, widths):
    """3 stages: C0 = GELU(A B0^T + b0) [M, N0] (K = 256); C1 = C0 B1^T [M, N1] (A = the stored C0, ldc > N);
    C2 = -3 (C1 B2^T + b2) [M, N2]"""
    n0, n1, n2 = widths
    s0 = Item(0, M, n0, 256, seed, bias=True, gelu=True)
    s1 = Item(0, M, n1, n0, seed + 1, a_src=s0.buf[GUARD:GUARD + M, :n0])
    s2 = Item(0, M, n2, n1, seed + 2, bias=True, alpha=-3.0, a_src=s1.buf[GUARD:GUARD + M, :n1])
    for i, it in enumerate((s0, s1, s2)):
        it.desc.stage, it.desc.dep = i, i - 1
    return [s0, s1, s2]


@pytest.mark.parametrize("M,widths", [(100, (512, 256, 768)), (257, (512, 256, 768)), (1000, (512, 256, 768)),
                                      (3000, (1536, 1024, 1280))])
def test_chain_same_bits_unchained_and_any_sm_count(hk, record_property, M, widths):
    """A 3-stage GEMM chain in ONE persistent launch (tile counters order the stages): each stage against fp64 from the bf16 its
    producer stored, bit for bit equal to the stage-by-stage launches (TP_CHAIN=0) and to the chain at 2, 4, 10 and 114 SMs.  The
    M = 3000 chain has 180 tiles: 57 pairs at 114 SMs walk other tile sequences and counter interleavings than 66 on an H100 SXM."""
    items = _chain(M, 80 + M, widths)
    _assert_sweep_reschedules(hk, _pair_tiles(items), M == 3000)
    flags = torch.zeros(64, dtype=torch.int32, device="cuda")
    with _env(TP_GEMM_MODE="2"):
        assert [hk.choice(it, 3) for it in items] == [PAIR] * 3
        n0 = hk.launches()
        assert hk.chain(items, flags) == 0
        assert hk.launches() - n0 == 1, "not chained"
    for i, it in enumerate(items):
        it.check(record_property, f"stage{i}")          # a consumer's A (it.at) is a view of what its producer stored
    ref = [it.snapshot() for it in items]
    with _env(TP_GEMM_MODE="2", TP_CHAIN="0"):
        for it in items:
            it.reset()
        n0 = hk.launches()
        assert hk.chain(items, flags) == 0
        assert hk.launches() - n0 == 3
    for it, r in zip(items, ref):
        assert _same_bits(it.snapshot(), r), "unchained"
    for sms in SMS_SWEEP:
        for it in items:
            it.reset()
        flags.zero_()
        with _env(TP_GEMM_MODE="2"):
            n0 = hk.launches()
            assert hk.chain(items, flags, sms) == 0
            assert hk.launches() - n0 == 1
        for i, (it, r) in enumerate(zip(items, ref)):
            assert _same_bits(it.snapshot(), r), (sms, i)


# ------------------------------------------------------------------------------------------------------------------------------
# rejections
# ------------------------------------------------------------------------------------------------------------------------------
def _bad(case):
    if case == "n_not_32":
        return [Item(0, 129, 48, 64, 90)]
    if case == "c_misaligned":
        it = Item(0, 129, 256, 64, 91)
        it.desc.c += 2
        return [it]
    if case == "ldc_misaligned":
        it = Item(0, 129, 256, 64, 92)
        it.desc.ldc -= 4
        return [it]
    if case == "dual_without_gelu":
        it = Item(0, 129, 256, 64, 93, dual=True)
        return [it]
    if case == "dual_segmented":
        return [Item(0, 36 * 4, 256, 64, 94, gelu=True, dual=True, out="seg", seg=(36, 37))]
    if case == "splitk_bf16":
        it = Item(1, 256, 256, 1000, 95)
        it.desc.k_splits = 3
        return [it]
    if case == "b_parts_not_tn":
        it = Item(0, 129, 512, 64, 96)
        it.desc.b_parts, it.desc.b_more[0] = 2, it.desc.b
        return [it]
    if case == "a_parts_k":
        it = Item(0, 129, 256, 192, 97)
        it.desc.a_parts, it.desc.a_more[0] = 2, it.desc.a
        return [it]
    if case == "nine_items":
        return [Item(0, 64, 256, 64, 98 + i) for i in range(9)]
    if case == "pair_only_n":
        return [Item(1, 129, 160, 64, 99)]
    # a valid item that runs on a launch of its own first (a one-CTA kernel under TP_GEMM_MODE=1, an ungrouped pair launch under
    # =3), then an invalid one, refused by check_item, by the build of the pair group, by the build of an ungrouped pair launch
    if case == "one_cta_then_n_not_32":
        return [Item(0, 129, 256, 64, 100), Item(0, 129, 48, 64, 101)]
    if case == "one_cta_then_dual_without_gelu":
        return [Item(0, 129, 256, 64, 102), Item(0, 129, 256, 64, 103, dual=True)]
    if case == "ungrouped_then_a_parts_k":
        return [Item(1, 300, 256, 65, 104)] + _bad("a_parts_k")
    raise AssertionError(case)


@pytest.mark.parametrize("case,mode,first", [
    ("n_not_32", None, None), ("c_misaligned", None, None), ("ldc_misaligned", None, None), ("dual_without_gelu", None, None),
    ("dual_segmented", None, None), ("splitk_bf16", None, None), ("b_parts_not_tn", None, None), ("a_parts_k", None, None),
    ("nine_items", None, None), ("pair_only_n", None, None), ("one_cta_then_n_not_32", "1", ONE_256),
    ("one_cta_then_dual_without_gelu", "1", ONE_256), ("ungrouped_then_a_parts_k", "3", PAIR)])
def test_rejected_items_launch_nothing(hk, case, mode, first):
    """Invalid items: TP_ERR_INVALID_ARGUMENT, no kernel launched, no output byte written, also when a valid item that runs on a
    launch of its own comes first in the list."""
    items = _bad(case)
    before = [it.snapshot() for it in items]
    with _env(TP_GEMM_MODE=mode):
        if first is not None:
            assert hk.choice(items[0], len(items)) == first
        n0 = hk.launches()
        st = hk.group(items)
        assert st == INVALID, st
        assert hk.launches() == n0
    for it, b in zip(items, before):
        assert _same_bits(it.snapshot(), b)
