"""CPU tests of the drop-in boundary: the C-ABI library loads and exports every symbol
include/gtn_b200.h declares; without a GPU the product path fails loudly (no fallback)."""
import ctypes
import os
import re

import pytest

from gtn_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "gtn_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(gtnb_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(capi.LIB_PATH)
    names = header_symbols()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), "missing export: " + n
    assert sorted(s[0] for s in capi.SYMBOLS) == names
    assert capi.lib().gtnb_version() == 100


def _no_gpu():
    try:
        c = capi.Ctx(0)
        c.close()
        return False
    except capi.GtnbError:
        return True


@pytest.mark.skipif(not _no_gpu(), reason="a CUDA device is present")
def test_no_cpu_fallback():
    with pytest.raises(capi.GtnbError) as ei:
        capi.Ctx(0)
    assert "no CPU fallback" in str(ei.value) or "CUDA" in str(ei.value)


def test_product_library_contains_no_emulation_code():
    """tests/emu compiles kernel SOURCES with g++ (-DGTNB_HOST_EMU) for CPU-side logic tests; none of that
    may reach the product: the Makefile never defines the macro (gtnb_internal.h refuses it) and the
    library exports no emulator symbol."""
    import subprocess
    mk = open(os.path.join(ROOT, "gtn_b200", "csrc", "Makefile")).read()
    assert "GTNB_HOST_EMU" not in mk
    so = os.path.join(ROOT, "gtn_b200", "lib", "libgtn_b200.so")
    syms = subprocess.run(["nm", "-DC", "--defined-only", so], capture_output=True, text=True).stdout
    assert "emu::" not in syms and "simt" not in syms.lower()


def test_kernel_files_contain_no_inline_ptx():
    """Inline PTX lives in gtnb_ptx.h only, next to the emulated form tests/emu runs instead of it, so that one
    file shows every place where the emulated kernel sources differ from the compiled ones."""
    import glob
    import re
    files = sorted(glob.glob(os.path.join(ROOT, "gtn_b200", "csrc", "k_*.cu")))
    assert files
    offenders = [os.path.basename(f) for f in files if re.search(r"\basm\b", open(f).read())]
    assert offenders == []
