"""The increase kernels of libtskv_gpu.so's sm_90a cubin (read with cuobjdump, demangled with cu++filt) are exactly the
instantiations tests/test_gpu_increase.py runs: k_scan_increase<EDGES> for the pages of tumbling and edge scans,
k_merge_increase for the merge groups of overlapping chunk files, and the helpers around the records' sorts."""
import re
import subprocess

import pytest

from cnosdb_b200 import cabi
from tests.test_kernel_list import cuda_tool

EXPECTED = {"k_scan_increase<false>", "k_scan_increase<true>", "k_merge_increase", "k_increase_init", "k_increase_gather",
            "k_increase_stitch", "k_finalize_increases"}
NAMES = r"k_scan_increase|k_merge_increase|k_increase_init|k_increase_gather|k_increase_stitch|k_finalize_increases"


def normalise(demangled):
    """'void tskv::k_scan_increase<(bool)1>(tskv::ScanParams, ...)' -> 'k_scan_increase<true>'."""
    m = re.search(r"\b(%s)(<[^>]*>)?\(" % NAMES, demangled)
    if not m:
        return None
    if not m.group(2):
        return m.group(1)
    args = [{"(bool)0": "false", "(bool)1": "true"}.get(a.strip(), a.strip()) for a in m.group(2)[1:-1].split(",")]
    return "%s<%s>" % (m.group(1), ", ".join(args))


def test_normalise():
    assert normalise("void tskv::k_scan_increase<(bool)1>(tskv::ScanParams, const tskv::IncreaseCol *, tskv::IncreaseArgs)") == \
        "k_scan_increase<true>"
    assert normalise("tskv::k_increase_gather(const unsigned long *, const unsigned int *, unsigned long, unsigned long *)") == \
        "k_increase_gather"
    assert normalise("void tskv::k_scan_median<(bool)0>(tskv::ScanParams, const tskv::MedianCol *, tskv::MedianArgs)") is None


def test_increase_kernels_match_the_library():
    cuobjdump, cufilt = cuda_tool("cuobjdump"), cuda_tool("cu++filt")
    if cuobjdump is None or cufilt is None:
        pytest.skip("cuobjdump / cu++filt (CUDA toolkit) not found: the kernel list cannot be read from the library")
    out = subprocess.run([cuobjdump, "-ltext", cabi.gpu_library_path()], check=True, capture_output=True, text=True).stdout
    mangled = [m for m in re.findall(r"SASS text section \d+ : \S*?-(_Z\w+)\.sm_90a\.", out) if "increase" in m.lower()]
    names = subprocess.run([cufilt], input="\n".join(mangled), check=True, capture_output=True, text=True).stdout.split("\n")
    found = [k for k in (normalise(n) for n in names) if k]
    assert len(found) == len(set(found)), found
    assert set(found) == EXPECTED, (sorted(set(found) - EXPECTED), sorted(EXPECTED - set(found)))
