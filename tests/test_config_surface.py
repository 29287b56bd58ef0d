"""The library has one build and a fixed set of run-time switches: every environment variable it reads selects a reference path
that the GPU tests compare against bit for bit, and the only compile-time switch is the safety timeout of the bounded waits."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "tokenpacker_b200")

# TP_GEMM_MODE: force the one-CTA / pair kernels; TP_CHAIN=0: one launch per stage; TP_FUSE_ATTN=0: separate attention kernel
ENV_VARS = {"TP_GEMM_MODE", "TP_CHAIN", "TP_FUSE_ATTN"}
BUILD_SWITCHES = {"TP_SPIN_LIMIT_CYCLES"}


def native_sources():
    paths = sorted(p for p in glob.glob(os.path.join(PKG, "csrc", "*")) if os.path.isfile(p) and not p.endswith(".log"))
    assert any(p.endswith("tp_api.cu") for p in paths), paths
    return {p: open(p).read() for p in paths}


def python_sources():
    paths = sorted(glob.glob(os.path.join(PKG, "*.py")))
    assert any(p.endswith("_lib.py") for p in paths), paths
    return {p: open(p).read() for p in paths}


def test_environment_variables_read_by_the_library():
    found = set()
    for path, text in native_sources().items():
        names = re.findall(r'getenv\s*\(\s*"(\w+)"\s*\)', text)
        assert len(names) == len(re.findall(r"getenv\s*\(", text)), f"{path}: getenv with a non-literal name"
        found.update(names)
    for path, text in python_sources().items():
        names = re.findall(r"""os\.(?:environ\.get\(|environ\[|getenv\()\s*["'](\w+)["']""", text)
        assert len(names) == len(re.findall(r"\benviron\b|\bgetenv\b", text)), f"{path}: environment read with a non-literal name"
        found.update(names)
    assert found == ENV_VARS


def test_preprocessor_switches():
    found = set()
    for text in native_sources().values():
        found.update(re.findall(r"^\s*#\s*ifn?def\s+(TP_\w+)", text, flags=re.M))
        for line in re.findall(r"^\s*#\s*(?:el)?if\b.*$", text, flags=re.M):
            found.update(re.findall(r"\bdefined\s*\(?\s*(TP_\w+)", line))
    assert found == BUILD_SWITCHES
