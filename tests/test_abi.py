"""CPU suite: the C-ABI library loads and exports every symbol include/pydeseq2_b200.h declares;
the product fails loudly (no CPU fallback) when there is no device."""
import os
import re

import pytest

from pydeseq2_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "pydeseq2_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(pdq_[a-z0-9_]+)\s*\(", src)))


def test_header_and_binding_agree():
    assert header_symbols() == sorted(_lib.EXPORTED_SYMBOLS)


def test_library_exports_every_declared_symbol():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g

        g.build()
    lib = _lib.load()
    for name in header_symbols():
        assert hasattr(lib, name), name
    assert b"sm_90a" in lib.pdq_version()


def test_no_cpu_fallback_without_device():
    lib = _lib.load()
    if lib.pdq_device_count() > 0:
        pytest.skip("a CUDA device is visible")
    from pydeseq2_b200.inference import B200Inference

    with pytest.raises(_lib.B200Error):
        B200Inference()


def test_product_never_imports_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "pydeseq2_b200")):
        for f in files:
            if f.endswith(".py"):
                txt = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", txt, flags=re.M), f
