"""Training from the four CLIP hidden states, host side (no CUDA): include/tokenpacker_b200_layers.h, its exports and its ctypes
binding agree and stay apart from the other headers; a plain-C consumer links it; tp_forward_train_layers, tp_backward_layers and
tp_forward_layers_packed refuse bad arguments with status codes before any CUDA call; Python refuses bad input before any device
work."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tokenpacker_b200_layers.h")


def _header_functions():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return {m.group(1): m.group(2) for m in re.finditer(r"TP_API\s+[\w\s\*]+?\b(tp_\w+)\s*\(([^)]*)\)", text)}


def test_header_binding_and_exports_agree():
    """The header only adds: its entry points are exported, bound by _lib.LAYERS_SIGNATURES with as many arguments as it declares,
    and none of them is declared by another header."""
    from tokenpacker_b200 import _lib
    fns = _header_functions()
    assert sorted(fns) == ["tp_backward_layers", "tp_forward_layers_packed", "tp_forward_train_layers"]
    assert sorted(_lib.LAYERS_SIGNATURES) == sorted(fns)
    for other in (_lib.SIGNATURES, _lib.HD_U8_SIGNATURES, _lib.CLIP_U8_SIGNATURES, _lib.INPUT_GRAD_SIGNATURES):
        assert not set(fns) & set(other)
    for name, params in fns.items():
        assert len(params.split(",")) == len(_lib.LAYERS_SIGNATURES[name][1]), name
    raw = C.CDLL(_lib.LIB_PATH)
    for n in fns:
        assert hasattr(raw, n), f"{n} declared in the header but not exported"


def test_plain_c_consumer_of_the_layers_header(tmp_path):
    from tokenpacker_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = str(tmp_path / "abi_check_layers")
    src = os.path.join(ROOT, "tests", "abi_c", "abi_check_layers.c")
    text = open(src).read()
    for name in _header_functions():
        assert f"&{name}" in text, f"{name} missing from abi_check_layers.c"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", libdir,
                    "-l:libtokenpacker_b200.so", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "abi layers ok" in r.stdout


def _ptrs(*vals):
    return (C.c_void_p * 4)(*vals)


def test_abi_argument_validation():
    from tokenpacker_b200 import _lib
    lib = _lib.lib
    p = C.c_void_p(4096)             # never dereferenced: every call below is refused before any CUDA work
    w = _lib.TpWeights(*([4096] * len(_lib.WEIGHT_FIELDS)))
    g = _lib.TpWeights(*([4096] * len(_lib.WEIGHT_FIELDS)))
    bad, bad_s = _lib.TP_ERR_INVALID_ARGUMENT, _lib.TP_ERR_BAD_SCALE_FACTOR
    cs = 577 * 1024
    good = _ptrs(4096, 8192, 12288, 16384)

    def fwd(layers=good, cs=cs, n=1, s=2, h=4096, out=p, saved=p):
        return lib.tp_forward_train_layers(C.byref(w), p, layers, n, cs, s, h, out, saved, 1, None)

    def bwd(layers=good, cs=cs, packed=p, d=_ptrs(None, None, None, 4096), dcs=cs, s=2, h=4096, go=p):
        return lib.tp_backward_layers(C.byref(w), packed, layers, cs, 1, s, h, go, p, C.byref(g), d, dcs, p, 1, None)

    def pk(layers=good, cs=cs, s=2, rows=0, out=p):
        return lib.tp_forward_layers_packed(p, layers, 1, cs, s, 4096, out, rows, p, 1, None)

    for call in (fwd, bwd, pk):
        assert call(layers=None) == bad                              # no layer array
        assert call(layers=_ptrs(4096, None, 4096, 4096)) == bad     # a NULL layer
        assert call(layers=_ptrs(4096, 4096, 4096 + 2, 4096)) == bad  # an unaligned layer
        assert call(cs=575 * 1024) == bad                            # crops shorter than 576 rows
        assert call(cs=cs + 4) == bad                                # crop stride not a 16-byte multiple
        assert call(s=5) == bad_s
        assert call(s=0) == bad_s
    assert fwd(n=0) == bad
    assert fwd(out=None) == bad
    assert fwd(h=100) == bad
    assert bwd(packed=None) == bad                                    # layer gradients read [W_k0; W_v0] from the packed weights
    assert bwd(d=_ptrs(None, 4096 + 8, None, None)) == bad            # a misaligned gradient destination
    assert bwd(dcs=cs + 8) == bad                                     # not a whole number of 1024-channel rows
    assert bwd(dcs=575 * 1024) == bad
    assert bwd(go=None) == bad
    assert bwd(h=100) == bad
    assert pk(rows=100) == bad                                        # fewer rows per crop than queries (144 at s = 2)
    assert pk(out=C.c_void_p(4096 + 2)) == bad


def test_python_refuses_bad_input_before_device_work():
    from tokenpacker_b200 import TokenPackerB200
    m = TokenPackerB200(hidden_size=256, scale_factor=2)
    hs = [torch.zeros(1, 577, 1024) for _ in range(4)]
    with pytest.raises(ValueError):
        m.forward_hidden_states(hs[:3])
    with pytest.raises(ValueError):
        m.forward_hidden_states(hs[:3] + [torch.zeros(1, 575, 1024)])
    with pytest.raises(ValueError):
        m.forward_hidden_states(hs[:3] + [torch.zeros(2, 577, 1024)])
    with pytest.raises(ValueError):
        m.forward_hidden_states(hs[:3] + [torch.zeros(1, 577, 4096)])
    with pytest.raises(RuntimeError, match="no CPU path"):
        m.forward_hidden_states(hs)
    with pytest.raises(RuntimeError, match="no CPU path"):
        m.forward_hidden_states_packed(hs, [1], [1], torch.zeros(256), torch.zeros(256))
    # a layer that requires grad with input_grad off fails loudly, whatever else is wrong with it
    g = [t.clone().requires_grad_(True) for t in hs]
    with pytest.raises(NotImplementedError, match="input_grad"):
        m.forward_hidden_states(g)
    with pytest.raises(NotImplementedError, match="input_grad"):
        m.forward_hidden_states_packed(g, [1], [1], torch.zeros(256), torch.zeros(256))
    m.input_grad = True
    with pytest.raises(RuntimeError, match="no CPU path"):
        m.forward_hidden_states(g)
    with torch.no_grad():                                             # no gradient wanted: nothing to refuse but the device
        m.input_grad = False
        with pytest.raises(RuntimeError, match="no CPU path"):
            m.forward_hidden_states(g)


def test_forward_layers_refuses_bad_input_before_device_work():
    """forward_layers is inference only and checks its layers itself: training mode is refused first, then the layer count and
    each layer's shape and device, CPU tensors included, with ValueError; it has no input_grad refusal."""
    from tokenpacker_b200 import TokenPackerB200
    m = TokenPackerB200(hidden_size=256, scale_factor=2)
    hs = [torch.zeros(1, 577, 1024) for _ in range(4)]
    with pytest.raises(NotImplementedError, match="inference path"):
        m.forward_layers(hs[:3])                                      # trainable parameters under autograd, whatever the layers
    with torch.no_grad():
        with pytest.raises(ValueError, match="4 hidden states"):
            m.forward_layers(hs[:3])
        for bad in (torch.zeros(1, 575, 1024), torch.zeros(1, 577, 4096), torch.zeros(577, 1024)):
            with pytest.raises(ValueError, match="CUDA tensor"):
                m.forward_layers(hs[:3] + [bad])
        with pytest.raises(ValueError, match="CUDA tensor"):
            m.forward_layers(hs)                                      # CPU layers: ValueError here, not the RuntimeError of forward()
    m.requires_grad_(False)
    g = [t.clone().requires_grad_(True) for t in hs]
    with pytest.raises(ValueError, match="CUDA tensor"):
        m.forward_layers(g)                                           # layers that require grad are not refused for input_grad
