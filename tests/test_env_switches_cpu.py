"""CPU: the library reads exactly the FM_* environment switches that tests or bench.py set to select the second path
they compare the default against (INTEGRATION.md, "Environment switches").  Each switch is a code path the benchmark
does not run, so a new one has to be added here on purpose."""
import glob
import os
import re

from conftest import ROOT

PKG = os.path.join(ROOT, "fastmot_b200")

KEPT = {
    "FM_CONV_TMA",          # test_gpu_yolo_ops: every detector conv on conv_tc.cu
    "FM_CONV_TMA_SPLIT",    # test_gpu_nets: every cluster size of the TMA conv's split-K
    "FM_OSB_FUSED",         # test_gpu_osnet_fused, test_gpu_osnet_ops: OSNet one launch per layer
    "FM_FUSE_CASCADE",      # test_gpu_tracker_seq: per-stage and always-fused association
    "FM_SYNTH_OBJ_BIAS",    # bench.py and the GPU tests: synthetic detector heads
    "FM_SYNTH_HEAD_GAIN",
}

_C_READ = re.compile(r"""\bgetenv\s*\(\s*"(FM_\w+)"\s*\)""")
_PY_READ = re.compile(r"""\b(?:os\.environ(?:\.get|\.setdefault|\.pop)?\s*[(\[]|os\.getenv\s*\()\s*["'](FM_\w+)["']"""
                      r"""|["'](FM_\w+)["']\s+(?:not\s+)?in\s+os\.environ\b""")


def _read(path):
    with open(path, encoding="utf-8") as f:
        return f.read()


def _c_switches():
    found = {}
    for ext in ("cu", "cuh", "h", "cpp", "cc"):
        for p in glob.glob(os.path.join(PKG, "csrc", "**", f"*.{ext}"), recursive=True):
            for name in _C_READ.findall(_read(p)):
                found.setdefault(name, set()).add(os.path.relpath(p, ROOT))
    return found


def _py_switches():
    found = {}
    for p in glob.glob(os.path.join(PKG, "**", "*.py"), recursive=True):
        for m in _PY_READ.finditer(_read(p)):
            found.setdefault(m.group(1) or m.group(2), set()).add(os.path.relpath(p, ROOT))
    return found


def test_library_reads_only_the_kept_switches():
    c, py = _c_switches(), _py_switches()
    found = set(c) | set(py)
    extra = {n: sorted(c.get(n, set()) | py.get(n, set())) for n in found - KEPT}
    assert not extra, f"environment switches beyond the kept set: {extra}"
    assert found == KEPT, f"kept switches no longer read: {sorted(KEPT - found)}"
