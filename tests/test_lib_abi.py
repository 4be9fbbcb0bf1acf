"""CPU: the C-ABI library loads and exports every symbol include/fastmot_b200.h declares."""
import os
import re
import ctypes

from conftest import ROOT


def _declared():
    hdr = open(os.path.join(ROOT, "include", "fastmot_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(fm_[a-z0-9_]+)\s*\(", hdr)))


def test_header_symbols_exported():
    names = _declared()
    assert len(names) >= 10
    so = os.path.join(ROOT, "fastmot_b200", "libfastmot_b200.so")
    assert os.path.exists(so), "run python -m fastmot_b200.build"
    lib = ctypes.CDLL(so)
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing


def test_python_signatures_cover_header():
    from fastmot_b200 import _lib
    names = _declared()
    missing = [n for n in names if n not in _lib.SIGNATURES]
    assert not missing, missing
    _lib.load()
    assert _lib.load().fm_version() >= 100


def test_no_cpu_fallback_without_device():
    """Product classes must refuse to run without an H100 (no silent CPU path)."""
    import torch
    import pytest
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from fastmot_b200 import _lib, MultiTracker
    with pytest.raises(_lib.FastMOTLibError):
        MultiTracker((1920, 1080), 'cosine')


def test_device_code_is_sm90a_without_three_input_integer_minmax():
    """The library carries sm_90a machine code only, and no VIMNMX3: ptxas 12.9 fuses chained integer min / max into
    that three-input instruction for sm_90, and it returned wrong minima / maxima on the H100 (the FAST corner score
    in csrc/klt_feat.cu and the slice bounds in csrc/conv_tma.cu are written so that none is generated)."""
    import shutil
    import subprocess
    import pytest
    from fastmot_b200 import build
    so = os.path.join(ROOT, "fastmot_b200", "libfastmot_b200.so")
    assert os.path.exists(so), "run python -m fastmot_b200.build"
    tool = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    tool = tool if os.path.exists(tool) else shutil.which("cuobjdump")
    if tool is None:
        pytest.skip("no cuobjdump")
    elfs = subprocess.run([tool, "--list-elf", so], capture_output=True, text=True, check=True).stdout
    archs = set(re.findall(r"\.(sm_[0-9a-z]+)\.cubin", elfs))
    assert archs == {"sm_90a"}, archs
    sass = subprocess.run([tool, "-sass", so], capture_output=True, text=True, check=True).stdout
    assert "VIMNMX3" not in sass


def test_ctypes_struct_layouts_match_the_header(tmp_path):
    """Every struct the Python side mirrors (fastmot_b200/_lib.py) has the size and the field offsets the C compiler
    gives the declaration in include/fastmot_b200.h (plain C: the header must also compile without nvcc)."""
    import shutil
    import subprocess
    import pytest
    from fastmot_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    structs = [getattr(_lib, n) for n in dir(_lib)
               if n.startswith("Fm") and isinstance(getattr(_lib, n), type) and issubclass(getattr(_lib, n), ctypes.Structure)]
    assert len(structs) >= 9 and _lib.FmFrame in structs and _lib.FmFrameGeom in structs
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "fastmot_b200.h"', 'int main(void) {']
    for st in structs:
        lines.append(f'  printf("{st.__name__} %zu\\n", sizeof({st.__name__}));')
        for fname, _ in st._fields_:
            lines.append(f'  printf("{st.__name__}.{fname} %zu\\n", offsetof({st.__name__}, {fname}));')
    lines += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    r = subprocess.run([gcc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    c_layout = dict(zip(out[0::2], (int(v) for v in out[1::2])))
    for st in structs:
        assert c_layout[st.__name__] == ctypes.sizeof(st), st.__name__
        for fname, _ in st._fields_:
            assert c_layout[f"{st.__name__}.{fname}"] == getattr(st, fname).offset, f"{st.__name__}.{fname}"
