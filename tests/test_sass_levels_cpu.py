"""Resource budget of the level instances (DESIGN.md section 4.17) on sm_90a, read from the built libdpfhe.so (no GPU needed:
cuobjdump -res-usage).  Every level instance uses no local memory and no more registers than the instance it is a level form of:
ks_level_grouped_kernel<LOGN, .., MODE, RS> against ks_grouped_kernel<.., MODE> / ct_dot_grouped_kernel (RS = false) and
ks_rescale_grouped_kernel<.., MODE> (RS = true), ks_hybrid_level_kernel against ks_hybrid_kernel, rot_sum_grouped_level_kernel
against rot_sum_grouped_kernel, in both arithmetic variants and at N = 4096, 8192 and 16384."""
import os
import re
import shutil
import subprocess

import pytest

from deeppowers_b200 import _lib

KS_MUL_RELIN, KS_ROTATE, KS_DOT = 0, 2, 3


def _tool(name):
    for cand in (shutil.which(name), "/usr/local/cuda/bin/" + name):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def usage():
    """mangled kernel name -> (registers, stack bytes, local bytes)"""
    cuobjdump, so = _tool("cuobjdump"), _lib.so_path()
    if cuobjdump is None:
        pytest.skip("cuobjdump not found")
    assert os.path.exists(so), "libdpfhe.so is built by __graft_entry__.build()"
    out = subprocess.run([cuobjdump, "-res-usage", so], capture_output=True, text=True, check=True).stdout
    res, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", line)
        if m and cur:
            res[cur] = tuple(int(x) for x in m.groups())
            cur = None
    return res


def _one(usage, pat):
    names = [k for k in usage if re.search(pat, k)]
    assert len(names) == 1, (pat, names)
    return usage[names[0]]


def _pairs():
    """(level instance, sibling) name patterns"""
    for ns in ("3gen", "4fast"):
        pre = r"^_ZN5dpfhe%s" % ns
        for logn in (12, 13, 14):
            t = r"ILi%dELi256ELi3E" % logn
            for mode in (KS_MUL_RELIN, KS_ROTATE):
                yield (pre + r"23ks_level_grouped_kernel" + t + r"Li%dELb0EE" % mode, pre + r"17ks_grouped_kernel" + t + r"Li%dELb0EE" % mode)
                yield (pre + r"22ks_hybrid_level_kernel" + t + r"Li%dEEE" % mode, pre + r"16ks_hybrid_kernel" + t + r"Li%dEEE" % mode)
            yield (pre + r"23ks_level_grouped_kernel" + t + r"Li%dELb0EE" % KS_DOT, pre + r"21ct_dot_grouped_kernel" + t + r"EEv")
            for mode in (KS_MUL_RELIN, KS_DOT):
                yield (pre + r"23ks_level_grouped_kernel" + t + r"Li%dELb1EE" % mode, pre + r"25ks_rescale_grouped_kernel" + t + r"Li%dEEE" % mode)
            yield (pre + r"28rot_sum_grouped_level_kernel" + t + r"Li1EEE", pre + r"22rot_sum_grouped_kernel" + t + r"Li1EEE")


def test_every_level_instance_is_built(usage):
    level = [k for k in usage if re.search(r"(ks_level_grouped|ks_hybrid_level|rot_sum_grouped_level)_kernel", k)]
    assert len(level) == 2 * 3 * (5 + 2 + 1), sorted(level)
    assert len(level) == len(list(_pairs()))


@pytest.mark.parametrize("pair", list(_pairs()), ids=lambda p: re.sub(r"\\|\^_ZN5dpfhe", "", p[0]))
def test_no_local_memory_and_sibling_registers(usage, pair):
    lvl, sib = _one(usage, pair[0]), _one(usage, pair[1])
    assert lvl[2] == 0, ("local memory", lvl)
    assert lvl[0] <= sib[0], ("registers", lvl, sib)
