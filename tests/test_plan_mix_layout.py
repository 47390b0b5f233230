"""The ctypes mirror of ss_plan_mix (sonicsim_b200/_lib.py) against include/sonicsim_b200.h as gcc lays it out, and the
plan-mixture entry point's declaration (no GPU)."""
import ctypes
import os
import shutil
import subprocess

import pytest

from conftest import ROOT
from sonicsim_b200 import _lib


def test_ss_plan_mix_layout(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "sonicsim_b200.h"', 'int main(void) {',
             'printf("size %zu\\n", sizeof(ss_plan_mix));', 'printf("mono %u\\n", SS_MIX_MONO);']
    for fname, _ in _lib.SsPlanMix._fields_:
        lines.append('printf("%s %%zu\\n", offsetof(ss_plan_mix, %s));' % (fname, fname))
    lines += ['return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                    str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {l.split()[0]: int(l.split()[1]) for l in out if l.strip()}
    assert got["size"] == ctypes.sizeof(_lib.SsPlanMix)
    assert got["mono"] == _lib.SS_MIX_MONO
    for fname, _ in _lib.SsPlanMix._fields_:
        assert got[fname] == getattr(_lib.SsPlanMix, fname).offset, fname


def test_plan_create_mix_is_exported():
    lib = ctypes.CDLL(_lib.build())
    assert hasattr(lib, "ss_plan_create_mix") and "ss_plan_create_mix" in _lib.EXPORTS
    assert lib.ss_version() >= 105
