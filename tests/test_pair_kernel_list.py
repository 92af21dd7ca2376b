"""The column-pair kernels of libtskv_gpu.so's sm_90a cubin (read with cuobjdump, demangled with cu++filt) are exactly the
instantiations tests/test_gpu_covariance.py runs: k_scan_pair<PASS2, EDGES> for both passes of tumbling and edge scans,
k_merge_pairs_rows<PASS2> for the merged rows of overlapping chunk files, and the three untemplated helpers."""
import re
import subprocess

import pytest

from cnosdb_b200 import cabi
from tests.test_kernel_list import cuda_tool

EXPECTED = {
    "k_scan_pair<false, false>", "k_scan_pair<false, true>", "k_scan_pair<true, false>", "k_scan_pair<true, true>",
    "k_merge_pairs_rows<false>", "k_merge_pairs_rows<true>", "k_pair_prep", "k_merge_pairs", "k_finalize_pairs",
}


def normalise(demangled):
    """'void tskv::k_scan_pair<(bool)0, (bool)1>(tskv::ScanParams, ...)' -> 'k_scan_pair<false, true>'."""
    m = re.search(r"\b(k_scan_pair|k_merge_pairs_rows|k_pair_prep|k_merge_pairs|k_finalize_pairs)(<[^>]*>)?\(", demangled)
    if not m:
        return None
    if not m.group(2):
        return m.group(1)
    args = [a.strip() for a in m.group(2)[1:-1].split(",")]
    args = [{"(bool)0": "false", "(bool)1": "true"}.get(a, a) for a in args]
    return "%s<%s>" % (m.group(1), ", ".join(args))


def test_normalise():
    assert normalise("void tskv::k_scan_pair<(bool)0, (bool)1>(tskv::ScanParams, const tskv::PairCol *, unsigned long)") == \
        "k_scan_pair<false, true>"
    assert normalise("tskv::k_merge_pairs(unsigned long *, const tskv::PairCol *)") == "k_merge_pairs"
    assert normalise("void tskv::k_merge_m2(unsigned long *)") is None


def test_pair_kernels_match_the_library():
    cuobjdump, cufilt = cuda_tool("cuobjdump"), cuda_tool("cu++filt")
    if cuobjdump is None or cufilt is None:
        pytest.skip("cuobjdump / cu++filt (CUDA toolkit) not found: the kernel list cannot be read from the library")
    out = subprocess.run([cuobjdump, "-ltext", cabi.gpu_library_path()], check=True, capture_output=True, text=True).stdout
    mangled = [m for m in re.findall(r"SASS text section \d+ : \S*?-(_Z\w+)\.sm_90a\.", out) if "pair" in m.lower()]
    names = subprocess.run([cufilt], input="\n".join(mangled), check=True, capture_output=True, text=True).stdout.split("\n")
    found = [k for k in (normalise(n) for n in names) if k]
    assert len(found) == len(set(found)), found
    assert set(found) == EXPECTED, (sorted(set(found) - EXPECTED), sorted(EXPECTED - set(found)))
