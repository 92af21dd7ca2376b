"""The gauge kernels of libtskv_gpu.so's sm_90a cubin (read with cuobjdump, demangled with cu++filt) are exactly the
instantiations tests/test_gpu_gauge.py runs: k_gauge_scan<EDGES> for tumbling / sliding and edge / label scans,
k_gauge_merge_rows for the merged rows of overlapping chunk files, the helpers around the sort and the reduce, and CUB's
DeviceCompactInitKernel over GaugeAcc. (The radix sort's kernels sort u64 keys and carry no gauge type; the section of
CUB's DeviceReduceByKeyKernel over GaugeAcc has a name too long for the ELF section listing, which shortens it, so only
its companion init kernel can be matched by name.)"""
import re
import subprocess

import pytest

from cnosdb_b200 import cabi
from tests.test_kernel_list import cuda_tool

EXPECTED = {"k_gauge_scan<false>", "k_gauge_scan<true>", "k_gauge_merge_rows", "k_gauge_gather", "k_gauge_scatter",
            "k_gauge_fold", "k_gauge_check", "k_merge_gauges", "k_finalize_gauges", "cub:DeviceCompactInitKernel"}
CUB = re.compile(r"\bcub::[\w:]*?(Device\w+Kernel)<")
PATTERN = re.compile(r"\b(k_gauge_scan|k_gauge_merge_rows|k_gauge_gather|k_gauge_scatter|k_gauge_fold|k_gauge_check|"
                     r"k_merge_gauges|k_finalize_gauges)(<[^>]*>)?\(")


def normalise(demangled):
    """'void tskv::k_gauge_scan<(bool)1>(tskv::ScanParams, ...)' -> 'k_gauge_scan<true>'."""
    m = PATTERN.search(demangled)
    if not m:
        c = CUB.search(demangled)
        return "cub:" + c.group(1) if c and "Gauge" in demangled else None
    if not m.group(2):
        return m.group(1)
    args = [{"(bool)0": "false", "(bool)1": "true"}.get(a.strip(), a.strip()) for a in m.group(2)[1:-1].split(",")]
    return "%s<%s>" % (m.group(1), ", ".join(args))


def test_normalise():
    assert normalise("void tskv::k_gauge_scan<(bool)1>(tskv::ScanParams, const tskv::GaugeCol *, tskv::GaugeArgs)") == \
        "k_gauge_scan<true>"
    assert normalise("tskv::k_merge_gauges(unsigned long *, unsigned long)") == "k_merge_gauges"
    assert normalise("void tskv::k_scan_mode<(bool)0>(tskv::ScanParams, const tskv::ModeGather *, tskv::ModeArgs)") is None
    assert normalise("void cub::CUB_200802_SM_900::DeviceCompactInitKernel<cub::CUB_200802_SM_900::ReduceByKeyScanTileState<"
                     "tskv::GaugeAcc, unsigned int, false>, int *>(T1, int, T2)") == "cub:DeviceCompactInitKernel"


def test_no_gauge_name_matches_another_family():
    for name in EXPECTED | {"GaugeCol", "GaugeAcc", "GaugeArgs", "GaugeJoin"}:
        assert not any(w in name.lower() for w in ("increase", "mode", "median", "pair")), name


def test_gauge_kernels_match_the_library():
    cuobjdump, cufilt = cuda_tool("cuobjdump"), cuda_tool("cu++filt")
    if cuobjdump is None or cufilt is None:
        pytest.skip("cuobjdump / cu++filt (CUDA toolkit) not found: the kernel list cannot be read from the library")
    out = subprocess.run([cuobjdump, "-ltext", cabi.gpu_library_path()], check=True, capture_output=True, text=True).stdout
    mangled = [m for m in re.findall(r"SASS text section \d+ : \S*?-(_Z\w+)\.sm_90a\.", out) if "gauge" in m.lower()]
    names = subprocess.run([cufilt], input="\n".join(mangled), check=True, capture_output=True, text=True).stdout.split("\n")
    found = [k for k in (normalise(n) for n in names) if k]
    assert len(found) == len(set(found)), found
    assert set(found) == EXPECTED, (sorted(set(found) - EXPECTED), sorted(EXPECTED - set(found)))
