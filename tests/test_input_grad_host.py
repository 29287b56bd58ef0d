"""Gradients w.r.t. the CLIP features, host side (no CUDA): the companion header, its exports and its ctypes binding agree and stay
apart from tokenpacker_b200.h; a plain-C consumer links it; tp_backward_inputs refuses bad arguments with status codes before any
CUDA call; the module's switch is off by default, outside the constructor and the state_dict, and Python refuses bad input before
any device work.  Also pins the stencil transpose the GPU tests compare against to PyTorch's own bilinear backward."""
import ctypes as C
import inspect
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tokenpacker_b200_input_grad.h")


def _header_functions():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return {m.group(1): m.group(2) for m in re.finditer(r"TP_API\s+[\w\s\*]+?\b(tp_\w+)\s*\(([^)]*)\)", text)}


def test_header_binding_and_exports_agree():
    """include/tokenpacker_b200_input_grad.h only adds: its entry points are exported, bound by _lib.INPUT_GRAD_SIGNATURES with as many
    arguments as the header declares, and none of them is also declared by tokenpacker_b200.h or the 8-bit image header."""
    from tokenpacker_b200 import _lib
    fns = _header_functions()
    assert sorted(fns) == ["tp_backward_inputs"]
    assert sorted(_lib.INPUT_GRAD_SIGNATURES) == sorted(fns)
    assert not set(fns) & set(_lib.SIGNATURES)
    assert not set(fns) & set(_lib.HD_U8_SIGNATURES)
    for name, params in fns.items():
        assert len(params.split(",")) == len(_lib.INPUT_GRAD_SIGNATURES[name][1]), name
    raw = C.CDLL(_lib.LIB_PATH)
    for n in fns:
        assert hasattr(raw, n), f"{n} declared in the header but not exported"


def test_plain_c_consumer_of_the_input_grad_header(tmp_path):
    """The header is C99, its entry point links from plain C, and argument validation runs without a GPU
    (tests/abi_c/abi_check_input_grad.c)."""
    import shutil
    import subprocess
    from tokenpacker_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = str(tmp_path / "abi_check_input_grad")
    src = os.path.join(ROOT, "tests", "abi_c", "abi_check_input_grad.c")
    text = open(src).read()
    for name in _header_functions():
        assert f"&{name}" in text, f"{name} missing from abi_check_input_grad.c"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", libdir,
                    "-l:libtokenpacker_b200.so", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "abi input_grad ok" in r.stdout


def test_abi_argument_validation():
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    p = C.c_void_p(4096)             # never dereferenced: every call below is refused before any CUDA work
    w = _lib.TpWeights(*([4096] * len(_lib.WEIGHT_FIELDS)))
    g = _lib.TpWeights(*([4096] * len(_lib.WEIGHT_FIELDS)))
    bad = _lib.TP_ERR_INVALID_ARGUMENT
    xs = 576 * 4096

    def call(w=C.byref(w), packed=p, xm=p, xs=xs, n=1, s=2, h=4096, go=p, saved=p, g=C.byref(g), dx0=p, dxm=p, ws=p, wsb=1):
        return lib.tp_backward_inputs(w, packed, xm, xs, n, s, h, go, saved, g, dx0, dxm, ws, wsb, None)

    assert call(packed=None) == bad                       # d_xm reads [W_k0; W_v0] from the packed weights
    assert call(go=None) == bad
    assert call(saved=None) == bad
    assert call(xm=None) == bad
    assert call(ws=None) == bad
    assert call(w=None) == bad
    assert call(g=None) == bad
    assert call(n=0) == bad
    assert call(h=100) == bad                             # hidden must be a multiple of 32
    assert call(xs=xs + 8) == bad                         # the backward takes contiguous xm
    assert call(dx0=C.c_void_p(4096 + 2)) == bad          # 16-byte aligned outputs
    assert call(dxm=C.c_void_p(4096 + 8)) == bad
    for s in (0, 5, 7, 48):
        assert call(s=s) == _lib.TP_ERR_BAD_SCALE_FACTOR
    half = _lib.TpWeights(*([4096] * (len(_lib.WEIGHT_FIELDS) - 1) + [None]))
    assert call(g=C.byref(half)) == bad                   # every parameter gradient is written, as by tp_backward


def test_switch_is_off_by_default_and_outside_constructor_and_state_dict():
    from tokenpacker_b200 import TokenPackerB200
    assert "input_grad" not in inspect.signature(TokenPackerB200.__init__).parameters
    m = TokenPackerB200(hidden_size=256, scale_factor=2)
    assert m.input_grad is False
    keys = list(m.state_dict())
    m.input_grad = True
    assert list(m.state_dict()) == keys
    assert "input_grad" not in m.state_dict()
    m2 = TokenPackerB200(hidden_size=256, scale_factor=2)
    m2.load_state_dict(m.state_dict())
    assert m2.input_grad is False                         # loading a checkpoint does not switch it on


def test_python_refuses_bad_input_before_device_work():
    from tokenpacker_b200 import TokenPackerB200
    m = TokenPackerB200(hidden_size=256, scale_factor=2)
    m.input_grad = True
    x0 = torch.zeros(1, 576, 1024, requires_grad=True)
    xm = torch.zeros(1, 576, 4096, requires_grad=True)
    with pytest.raises(ValueError):
        m((x0[:, :100], xm))
    with pytest.raises(ValueError):
        m((x0, torch.zeros(2, 576, 4096, requires_grad=True)))
    with pytest.raises(TypeError):
        m(x0)
    with pytest.raises(NotImplementedError):
        m((x0, xm), attn_mask=torch.zeros(1))
    with pytest.raises(RuntimeError, match="no CPU path"):
        m((x0, xm))
    with pytest.raises(NotImplementedError):              # still an inference path, whatever the switch says
        m.forward_layers([torch.zeros(1, 577, 1024)] * 4)


# ------------------------------------------------------------------------------------------------------------------------------
# the transpose of the point-query stencil (builder.py:117-118), restated in numpy; tests/test_input_grad_gpu.py compares the
# kernel against it bit for bit
# ------------------------------------------------------------------------------------------------------------------------------
def stencil_t(dq: np.ndarray, s: int) -> np.ndarray:
    """dq [N, g*g, C] float32 (bf16 values) -> dx0 [N, 576, C] float32 before the bf16 rounding: odd s, dq at each window's centre
    token; even s, 0.25 dq on its centre 2x2; 0 elsewhere."""
    n, _, c = dq.shape
    g = 24 // s
    out = np.zeros((n, 24, 24, c), dtype=np.float32)
    q = dq.reshape(n, g, g, c)
    if s % 2:
        lo = (s - 1) // 2
        out[:, lo::s, lo::s] = q
    else:
        lo = s // 2 - 1
        for dr in (0, 1):
            for dc in (0, 1):
                out[:, lo + dr::s, lo + dc::s] = np.float32(0.25) * q
    return out.reshape(n, 576, c)


@pytest.mark.parametrize("s", [1, 2, 3, 4, 6, 8, 12, 24])
def test_stencil_transpose_matches_torch_bilinear_backward(s):
    """stencil_t, rounded to bf16, equals autograd through the reference's point-query ops (reshape, .float(), bilinear
    interpolate with align_corners=False, .to(bf16)) bit for bit, on dq values from every bf16 binade."""
    g = 24 // s
    rng = np.random.default_rng(s)
    e = rng.integers(-133, 128, size=(2, g * g, 64))
    dq = torch.from_numpy((rng.choice([-1.0, 1.0], size=e.shape) * rng.uniform(1, 1.99, size=e.shape) * np.exp2(e.astype(np.float64)))
                          .astype(np.float32)).to(torch.bfloat16)
    x0 = torch.zeros(2, 576, 64, dtype=torch.bfloat16, requires_grad=True)
    q = F.interpolate(x0.reshape(2, 24, 24, 64).float().permute(0, 3, 1, 2), size=(g, g), mode="bilinear")
    q = q.permute(0, 2, 3, 1).reshape(2, -1, 64).to(torch.bfloat16)
    q.backward(dq)
    ours = torch.from_numpy(stencil_t(dq.float().numpy(), s)).to(torch.bfloat16)
    assert torch.equal(ours.view(torch.int16), x0.grad.view(torch.int16))
