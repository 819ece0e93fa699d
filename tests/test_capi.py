"""CPU: the C-ABI shared library loads and exports every symbol include/espresso_b200.h declares
(no compute calls -- there is no GPU here), and the product refuses to run without CUDA."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "espresso_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(esp_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from espresso_b200 import lib

    L = lib.load()
    names = _declared_symbols()
    assert len(names) >= 6
    for n in names:
        assert hasattr(L, n), "libespresso_b200.so does not export %s" % n
        assert n in lib.SIGNATURES, "ctypes signature table misses %s" % n
    assert set(lib.SIGNATURES) == set(names)
    assert L.esp_version() >= 100


def test_no_cpu_fallback():
    from espresso_b200 import lib, ops

    with pytest.raises(lib.EspressoB200Error):
        ops.linear(torch.zeros(4, 8, dtype=torch.bfloat16), torch.zeros(4, 8, dtype=torch.bfloat16))


def _csrc():
    d = os.path.join(ROOT, "espresso_b200", "csrc")
    return {f: open(os.path.join(d, f)).read() for f in sorted(os.listdir(d)) if f.endswith((".cu", ".cuh"))}


def test_kernels_launch_through_the_counted_launcher():
    """Every kernel goes through esp_launch* (common.cuh), which checks the launch and counts it for esp_launch_count();
    shared-memory limits are raised only by ESP_SMEM_OPTIN."""
    src = _csrc()
    assert "common.cuh" in src and "capi.cu" in src
    assert [f for f, s in src.items() if "<<<" in s] == []
    assert [f for f, s in src.items() if "esp_count_launch" in s] == ["capi.cu", "common.cuh"]
    assert [f for f, s in src.items() if "cudaFuncSetAttribute" in s] == ["common.cuh"]
    optin = re.search(r"#define ESP_SMEM_OPTIN\(kernel, bytes\)((?:.*\\\n)*.*\n)", src["common.cuh"]).group(1)
    assert src["common.cuh"].count("cudaFuncSetAttribute") == optin.count("cudaFuncSetAttribute") == 1


def test_product_never_imports_oracle():
    bad = []
    for d, _, files in os.walk(os.path.join(ROOT, "espresso_b200")):
        for f in files:
            if f.endswith(".py"):
                s = open(os.path.join(d, f)).read()
                if re.search(r"^\s*(from|import)\s+oracle\b", s, flags=re.M):
                    bad.append(os.path.join(d, f))
    assert not bad, bad
