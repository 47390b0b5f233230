"""The ctypes mirror of ss_plan_target (sonicsim_b200/_lib.py) against include/sonicsim_b200.h as gcc lays it out, and
the dereverberation-target entry point's export and argument types (no GPU)."""
import ctypes
import os
import shutil
import subprocess

import pytest

from conftest import ROOT
from sonicsim_b200 import _lib


def _gcc(tmp_path, name, lines, link):
    src = tmp_path / (name + ".c")
    src.write_text("\n".join(lines))
    out = tmp_path / name
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                    str(out)] + ([] if link else ["-c"]), check=True)
    return out


def test_ss_plan_target_layout(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "sonicsim_b200.h"', 'int main(void) {',
             'printf("size %zu\\n", sizeof(ss_plan_target));', 'printf("mix_size %zu\\n", sizeof(ss_plan_mix));']
    for fname, _ in _lib.SsPlanTarget._fields_:
        lines.append('printf("%s %%zu\\n", offsetof(ss_plan_target, %s));' % (fname, fname))
    lines += ['return 0;', '}']
    exe = _gcc(tmp_path, "layout", lines, True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {l.split()[0]: int(l.split()[1]) for l in out if l.strip()}
    assert got["size"] == ctypes.sizeof(_lib.SsPlanTarget)
    for fname, _ in _lib.SsPlanTarget._fields_:
        assert got[fname] == getattr(_lib.SsPlanTarget, fname).offset, fname
    assert got["mix_size"] == ctypes.sizeof(_lib.SsPlanMix)        # ss_plan_mix keeps its layout
    # the declaration has the parameter list the ctypes argtypes state
    _gcc(tmp_path, "decl", ['#include "sonicsim_b200.h"',
                            'int (*f)(ss_ctx*, const ss_source*, int, const ss_plan_mix*, int, const ss_plan_draw*, int, '
                            'const ss_dry_pick*, const ss_pair_gains* const*, int, const ss_plan_target*, int, '
                            'ss_plan**) = ss_plan_create_target;'], False)
    assert len(_lib.load().ss_plan_create_target.argtypes) == 13


def test_plan_create_target_is_exported():
    lib = ctypes.CDLL(_lib.build())
    assert hasattr(lib, "ss_plan_create_target") and "ss_plan_create_target" in _lib.EXPORTS
    assert lib.ss_version() == 108


def test_mixture_direct_out_is_appended():
    """Mixture keeps every existing field at its position: positional calls stay valid, direct_out defaults to None."""
    from sonicsim_b200 import render
    f = render.Mixture._fields
    assert f[:9] == ("speakers", "noises", "sirs", "snr", "mix", "speakers_out", "rms_db", "mono", "noise_delay")
    assert f[9:] == ("direct_out",)
    m = render.Mixture([0], [1], None, 0, 0, None, None, True, 3)
    assert m.mono and m.noise_delay == 3 and m.direct_out is None
