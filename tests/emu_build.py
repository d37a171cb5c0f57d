"""Builds the host-side kernel emulations of tests/emu (g++ -std=c++20, <barrier>) on demand."""
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
CSRC = os.path.join(HERE, "..", "gtn_b200", "csrc")


def build(name, kernels):
    """tests/emu/<name>_emu.cpp + the kernel sources it includes -> tests/emu/lib<name>_emu.so (path).
    Skips the calling test when the toolchain cannot build it (no C++20 <barrier>)."""
    so = os.path.join(EMU, "lib%s_emu.so" % name)
    # every kernel file includes gtnb_ptx.h, which includes gtnb_meta.h
    src = [os.path.join(EMU, "%s_emu.cpp" % name), os.path.join(EMU, "simt_emu.h")] + \
          [os.path.join(CSRC, k) for k in kernels + ["gtnb_ptx.h", "gtnb_meta.h"]]
    if os.path.exists(so) and all(os.path.getmtime(s) <= os.path.getmtime(so) for s in src):
        return so
    cmd = ["g++", "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-Wno-unknown-pragmas", "-I", EMU, "-I", CSRC,
           "-I", os.path.join(HERE, "..", "include"), src[0], "-o", so]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("cannot build the kernel emulation with this g++: " + r.stderr.strip().splitlines()[-1][:200])
    return so


def check(rc):
    """Return code of an emulation driver: 0 ok; 77 = the host refused to create the threads of a CTA
    (sandbox thread limit) -> skip, do not fail."""
    if rc == 77:
        pytest.skip("the host refused to create the emulator's threads (thread limit)")
    assert rc == 0, rc
