"""The mode / distinct kernels of libtskv_gpu.so's sm_90a cubin (read with cuobjdump, demangled with cu++filt) are exactly
the instantiations tests/test_gpu_mode.py runs: k_scan_mode<EDGES> for the gathers of tumbling and edge scans,
k_merge_mode_rows for the merged rows of overlapping chunk files, and the helpers around the sorts."""
import re
import subprocess

import pytest

from cnosdb_b200 import cabi
from tests.test_kernel_list import cuda_tool

EXPECTED = {"k_scan_mode<false>", "k_scan_mode<true>", "k_merge_mode_rows", "k_mode_counts", "k_mode_heads", "k_mode_runs",
            "k_finalize_modes"}
PATTERN = re.compile(r"\b(k_scan_mode|k_merge_mode_rows|k_mode_counts|k_mode_heads|k_mode_runs|k_finalize_modes)(<[^>]*>)?\(")


def normalise(demangled):
    """'void tskv::k_scan_mode<(bool)1>(tskv::ScanParams, ...)' -> 'k_scan_mode<true>'."""
    m = PATTERN.search(demangled)
    if not m:
        return None
    if not m.group(2):
        return m.group(1)
    args = [{"(bool)0": "false", "(bool)1": "true"}.get(a.strip(), a.strip()) for a in m.group(2)[1:-1].split(",")]
    return "%s<%s>" % (m.group(1), ", ".join(args))


def test_normalise():
    assert normalise("void tskv::k_scan_mode<(bool)1>(tskv::ScanParams, const tskv::ModeGather *, tskv::ModeArgs)") == \
        "k_scan_mode<true>"
    assert normalise("tskv::k_mode_runs(tskv::ModeArgs, const unsigned int *)") == "k_mode_runs"
    assert normalise("void tskv::k_scan_median<(bool)0>(tskv::ScanParams, const tskv::MedianCol *, tskv::MedianArgs)") is None


def test_mode_kernels_match_the_library():
    cuobjdump, cufilt = cuda_tool("cuobjdump"), cuda_tool("cu++filt")
    if cuobjdump is None or cufilt is None:
        pytest.skip("cuobjdump / cu++filt (CUDA toolkit) not found: the kernel list cannot be read from the library")
    out = subprocess.run([cuobjdump, "-ltext", cabi.gpu_library_path()], check=True, capture_output=True, text=True).stdout
    mangled = [m for m in re.findall(r"SASS text section \d+ : \S*?-(_Z\w+)\.sm_90a\.", out) if "mode" in m.lower()]
    names = subprocess.run([cufilt], input="\n".join(mangled), check=True, capture_output=True, text=True).stdout.split("\n")
    found = [k for k in (normalise(n) for n in names) if k]
    assert len(found) == len(set(found)), found
    assert set(found) == EXPECTED, (sorted(set(found) - EXPECTED), sorted(EXPECTED - set(found)))
