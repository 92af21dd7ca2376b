"""The hand-written list of the fused scan's kernel instantiations (tests/sweep_reference.py: INSTANTIATIONS) equals the
k_scan_aggregate / k_scan_m2 entries of libtskv_gpu.so's sm_90a cubin, read with cuobjdump and demangled with cu++filt.
A change that adds or removes an instantiation must update the list, and with it the cases of
tests/test_gpu_kernel_sweep.py that aim at every entry."""
import os
import re
import shutil
import subprocess

import pytest

from cnosdb_b200 import cabi
from tests import sweep_reference as sw


def cuda_tool(name):
    """The CUDA toolkit's binary `name`: on PATH, else under CUDA_HOME / CUDA_PATH or /usr/local/cuda."""
    found = shutil.which(name)
    if found:
        return found
    for root in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if root and os.path.exists(os.path.join(root, "bin", name)):
            return os.path.join(root, "bin", name)
    return None


ENTRY = re.compile(r"\b(k_scan_aggregate|k_scan_m2)<([^>]*)>\(")


def parse_entry(demangled):
    """'void tskv::k_scan_aggregate<(int)2, (int)1, (bool)1, (int)0, (bool)0>(tskv::ScanParams, int)' -> the list key."""
    m = ENTRY.search(demangled)
    if not m:
        return None
    args = [re.sub(r"^\([a-z ]+\)", "", a.strip()) for a in m.group(2).split(",")]
    args = [{"false": 0, "true": 1}[a] if a in ("false", "true") else int(a) for a in args]
    if m.group(1) == sw.SCAN:
        tk, vk, sel, narrow, edges = args
        return (sw.SCAN, tk, vk, bool(sel), narrow, bool(edges))
    tk, vk, edges = args
    return (sw.M2, tk, vk, False, sw.NARROW_NONE, bool(edges))


def library_entries(cuobjdump, cufilt):
    """The demangled names of the scan kernels' SASS text sections for sm_90a."""
    out = subprocess.run([cuobjdump, "-ltext", cabi.gpu_library_path()], check=True, capture_output=True, text=True).stdout
    mangled = re.findall(r"SASS text section \d+ : \S*?-(_Z\w+)\.sm_90a\.", out)
    mangled = [m for m in mangled if "k_scan_aggregate" in m or "k_scan_m2" in m]
    assert mangled, "no scan kernel for sm_90a in %s" % cabi.gpu_library_path()
    names = subprocess.run([cufilt], input="\n".join(mangled), check=True, capture_output=True, text=True).stdout
    return names.strip().splitlines()


def test_parse_entry():
    assert parse_entry("void tskv::k_scan_aggregate<(int)2, (int)1, (bool)1, (int)0, (bool)0>(tskv::ScanParams, int)") == \
        (sw.SCAN, sw.TK_GEN, sw.VK_GOR, True, sw.NARROW_NONE, False)
    assert parse_entry("void tskv::k_scan_m2<(int)0, (int)2, (bool)1>(tskv::ScanParams, int)") == \
        (sw.M2, sw.TK_RLE, sw.VK_GEN, False, sw.NARROW_NONE, True)
    assert parse_entry("void tskv::k_scan_aggregate<0, 0, false, 1, true>(tskv::ScanParams, int)") == \
        (sw.SCAN, sw.TK_RLE, sw.VK_S8B, False, sw.NARROW_SOME, True)
    assert parse_entry("void tskv::k_merge_m2(unsigned long*)") is None


def test_list_has_no_duplicates_and_names_every_short_bin():
    assert len(set(sw.INSTANTIATIONS)) == len(sw.INSTANTIATIONS) == 62
    assert sorted(sw.SHORT_BINS) == list(range(sw.N_SERIAL_BINS, sw.N_BINS))
    assert {sw.serial_bin(b) for b in sw.SHORT_BINS} == {0, 1, 3, 4}


def test_instantiation_list_matches_the_library():
    cuobjdump, cufilt = cuda_tool("cuobjdump"), cuda_tool("cu++filt")
    if cuobjdump is None or cufilt is None:
        pytest.skip("cuobjdump / cu++filt (CUDA toolkit) not found: the kernel list cannot be read from the library")
    names = library_entries(cuobjdump, cufilt)
    keys = [parse_entry(n) for n in names]
    assert None not in keys, [n for n, k in zip(names, keys) if k is None]
    assert len(keys) == len(set(keys)), "a kernel listed twice in the cubin"
    missing = sorted(set(sw.INSTANTIATIONS) - set(keys), key=sw.key_name)
    extra = sorted(set(keys) - set(sw.INSTANTIATIONS), key=sw.key_name)
    assert not missing and not extra, "the library lacks %s; the list lacks %s" % (
        [sw.key_name(k) for k in missing], [sw.key_name(k) for k in extra])
