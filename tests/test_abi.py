"""C-ABI surface: the library loads, and include/tzk.h <-> exported symbols <-> ctypes table agree."""
import os
import re
import subprocess
import sys

from torcheasyrec_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "tzk.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return set(re.findall(r"\b(tzk_[a-z0-9_]+)\s*\(", src))


def test_library_loads_and_reports_version():
    handle = _lib.lib()
    assert handle.tzk_abi_version() == 1
    assert handle.tzk_last_error() is not None


def test_every_declared_symbol_is_exported_and_bound():
    declared = _declared()
    assert len(declared) >= 20
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r" T (tzk_[a-z0-9_]+)", out))
    assert declared <= exported, f"declared but not exported: {sorted(declared - exported)}"
    assert exported <= declared, f"exported but not declared in tzk.h: {sorted(exported - declared)}"
    assert declared == set(_lib.SIGNATURES), sorted(declared ^ set(_lib.SIGNATURES))


def test_workspace_queries_need_no_gpu():
    handle = _lib.lib()
    assert handle.tzk_lengths_to_offsets_workspace_bytes(0) >= 8
    assert handle.tzk_lengths_to_offsets_workspace_bytes(1 << 20) >= (1 << 20) // 4096 * 8
    assert handle.tzk_fused_bwd_workspace_bytes(1000, 1 << 20, 16) > 1000 * 16
    assert handle.tzk_bucketize_rw_workspace_bytes(26, 512, 8, 26 * 512) > 0


def test_product_has_no_cpu_fallback():
    import pytest
    import torch

    from torcheasyrec_b200.kernels import CudaKernels, TzkError

    k = CudaKernels()
    with pytest.raises(TzkError):
        k.lengths_to_offsets(torch.ones(4, dtype=torch.int32))


def test_package_import_graph_never_reaches_the_oracle():
    """Import every module of the package in a FRESH interpreter and diff sys.modules: nothing under oracle/ (nor the
    tests' checker backend) may be pulled in, and no file of the package may mention them."""
    code = (
        "import sys, pkgutil, importlib\n"
        "before = set(sys.modules)\n"
        "import torcheasyrec_b200\n"
        "for m in pkgutil.walk_packages(torcheasyrec_b200.__path__, 'torcheasyrec_b200.'):\n"
        "    if '.csrc.' in m.name:\n"
        "        continue\n"
        "    importlib.import_module(m.name)\n"
        "new = set(sys.modules) - before\n"
        "bad = sorted(n for n in new if n == 'oracle' or n.startswith('oracle.') or n.startswith('tzk_oracle')"
        " or n.startswith('c_oracle') or n == 'oracle_backend')\n"
        "print('BAD=' + ','.join(bad))\n"
        "print('N=' + str(len([n for n in new if n.startswith('torcheasyrec_b200')])))\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, check=True)
    assert "BAD=\n" in r.stdout, r.stdout
    n = int(re.search(r"N=(\d+)", r.stdout).group(1))
    assert n >= 12, r.stdout                  # the walk really imported the package's modules
    pkg = os.path.join(ROOT, "torcheasyrec_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                src = open(os.path.join(dirpath, fn), errors="ignore").read()
                assert not re.search(r"^\s*(from|import)\s+(oracle|tzk_oracle|c_oracle|oracle_backend)\b", src, re.M), fn
                assert "libtzk_oracle" not in src, fn


def test_gemm3x_library_exports_its_header():
    """include/tzk_gemm3x.h <-> libtzk_gemm3x.so (the 3xTF32 GEMMs of the wide tower layer)."""
    src = open(os.path.join(ROOT, "include", "tzk_gemm3x.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    declared = set(re.findall(r"\b(tzk_[a-z0-9_]+)\s*\(", src))
    assert declared == {"tzk_gemm3x", "tzk_wgrad3x", "tzk_wgrad3x_partial_floats"}
    lib = os.path.join(ROOT, "torcheasyrec_b200", "csrc", "libtzk_gemm3x.so")
    out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    assert set(re.findall(r" T (tzk_[a-z0-9_]+)", out)) == declared
    import ctypes

    h = ctypes.CDLL(lib)
    h.tzk_wgrad3x_partial_floats.restype = ctypes.c_int64
    assert h.tzk_wgrad3x_partial_floats(784, 21) == 21 * 896 * 64
