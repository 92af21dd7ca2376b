"""The state agg kernels of libtskv_gpu.so's sm_90a cubin (read with cuobjdump, demangled with cu++filt) are exactly the
instantiations tests/test_gpu_state_agg.py runs: k_state_scan<EDGES> for tumbling and edge scans, k_state_merge_rows for
the merged rows of overlapping chunk files, the helpers around the sorts and the reduce, and CUB's
DeviceCompactInitKernel of the reduce by (segment, state key). (The radix sorts' and the scan's kernels carry no state agg
type; the section of CUB's DeviceReduceByKeyKernel over StateKey has a name too long for the ELF section listing, which
shortens it, so only its companion init kernel can be matched by name, by the init kernel's tile-state value type.)"""
import re
import subprocess

import pytest

from cnosdb_b200 import cabi
from tests.test_kernel_list import cuda_tool

EXPECTED = {"k_state_scan<false>", "k_state_scan<true>", "k_state_merge_rows", "k_state_init", "k_state_stitch",
            "k_state_gather", "k_state_order", "k_state_count", "k_state_check", "k_finalize_states"}
PATTERN = re.compile(r"\b(k_state_scan|k_state_merge_rows|k_state_init|k_state_stitch|k_state_gather|k_state_order|"
                     r"k_state_count|k_state_check|k_finalize_states)(<[^>]*>)?\(")


def normalise(demangled):
    """'void tskv::k_state_scan<(bool)1>(tskv::ScanParams, ...)' -> 'k_state_scan<true>'."""
    m = PATTERN.search(demangled)
    if not m:
        return None
    if not m.group(2):
        return m.group(1)
    args = [{"(bool)0": "false", "(bool)1": "true"}.get(a.strip(), a.strip()) for a in m.group(2)[1:-1].split(",")]
    return "%s<%s>" % (m.group(1), ", ".join(args))


def test_normalise():
    assert normalise("void tskv::k_state_scan<(bool)1>(tskv::ScanParams, const tskv::StateCol *, tskv::StateArgs)") == \
        "k_state_scan<true>"
    assert normalise("tskv::k_state_stitch(tskv::StateArgs)") == "k_state_stitch"
    assert normalise("void tskv::k_gauge_scan<(bool)0>(tskv::ScanParams, const tskv::GaugeCol *, tskv::GaugeArgs)") is None


def test_no_state_name_matches_another_family():
    for name in EXPECTED | {"StateCol", "StateArgs", "StateKey", "StateBound", "StateRun", "StateSum"}:
        assert not any(w in name.lower() for w in ("increase", "mode", "median", "pair", "gauge")), name


def test_state_kernels_match_the_library():
    cuobjdump, cufilt = cuda_tool("cuobjdump"), cuda_tool("cu++filt")
    if cuobjdump is None or cufilt is None:
        pytest.skip("cuobjdump / cu++filt (CUDA toolkit) not found: the kernel list cannot be read from the library")
    out = subprocess.run([cuobjdump, "-ltext", cabi.gpu_library_path()], check=True, capture_output=True, text=True).stdout
    mangled = re.findall(r"SASS text section \d+ : \S*?-(_Z\w+)\.sm_90a\.", out)
    names = subprocess.run([cufilt], input="\n".join(mangled), check=True, capture_output=True, text=True).stdout.split("\n")
    found = [k for k in (normalise(n) for n in names) if k]
    assert len(found) == len(set(found)), found
    assert set(found) == EXPECTED, (sorted(set(found) - EXPECTED), sorted(EXPECTED - set(found)))
    # the reduce by (segment, state key): its init kernel's tile state sums i64 durations
    assert any("DeviceCompactInitKernel" in n and "ReduceByKeyScanTileState<long, unsigned int" in n for n in names)
