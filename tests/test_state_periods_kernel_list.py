"""The state period kernels of libtskv_gpu.so's sm_90a cubin (read with cuobjdump, demangled with cu++filt) are exactly
the ones a query with TSKV_STATE_PERIODS adds to the state agg pass: k_period_keys, k_period_segs, k_period_mark and
k_period_write. (The pass's sorts, gather and exclusive sums reuse CUB's and the state aggs' kernels, which carry no
period type; tests/test_state_agg_kernel_list.py holds those.)"""
import re
import subprocess

import pytest

from cnosdb_b200 import cabi
from tests.test_kernel_list import cuda_tool
from tests.test_state_agg_kernel_list import PATTERN as STATE_PATTERN

EXPECTED = {"k_period_keys", "k_period_segs", "k_period_mark", "k_period_write"}
PATTERN = re.compile(r"\b(k_period_\w+)(<[^>]*>)?\(")


def normalise(demangled):
    m = PATTERN.search(demangled)
    if not m:
        return None
    return m.group(1) + (m.group(2) or "")


def test_normalise():
    assert normalise("tskv::k_period_mark(tskv::StateArgs, tskv::PeriodArgs)") == "k_period_mark"
    assert normalise("tskv::k_state_stitch(tskv::StateArgs)") is None


def test_no_period_kernel_matches_the_state_agg_list():
    for name in EXPECTED:
        assert not STATE_PATTERN.search(name + "("), name


def test_period_kernels_match_the_library():
    cuobjdump, cufilt = cuda_tool("cuobjdump"), cuda_tool("cu++filt")
    if cuobjdump is None or cufilt is None:
        pytest.skip("cuobjdump / cu++filt (CUDA toolkit) not found: the kernel list cannot be read from the library")
    out = subprocess.run([cuobjdump, "-ltext", cabi.gpu_library_path()], check=True, capture_output=True, text=True).stdout
    mangled = re.findall(r"SASS text section \d+ : \S*?-(_Z\w+)\.sm_90a\.", out)
    names = subprocess.run([cufilt], input="\n".join(mangled), check=True, capture_output=True, text=True).stdout.split("\n")
    found = [k for k in (normalise(n) for n in names) if k]
    assert len(found) == len(set(found)), found
    assert set(found) == EXPECTED, (sorted(set(found) - EXPECTED), sorted(EXPECTED - set(found)))
