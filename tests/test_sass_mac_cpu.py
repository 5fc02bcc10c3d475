"""Instruction budget of the fused ct x ct kernel's multiply-accumulate with the key column on sm_90a (no GPU needed).

ks_blk_phase2's last loop (DESIGN.md §4.4) reads, in the fast variant, only the Shoup companions of the key row and rebuilds each
key word from its own (modarith.cuh shoup_w_from_companion: two IMAD.WIDE), so each product takes 6 IMAD.WIDE instead of 4 and
each chunk two 128-bit loads instead of four; the loop takes two chunks per iteration so that two chunks of companions are in
flight.  Pinned here for ks_fused_kernel<13,256,2,KS_MUL_RELIN> fast, with the register copies per chunk, together with the
registers and the absence of local memory of every fused instance at N <= 8192 in both variants."""
import collections
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import sass_loop  # noqa: E402

from deeppowers_b200 import build as dpbuild  # noqa: E402

FUSED = r"^_ZN5dpfhe4fast15ks_fused_kernelILi13ELi256ELi2ELi0ELb0ELb0EE"   # <13,256,2,KS_MUL_RELIN,PROF=false,FILTER=false>
FUSED_BLK = r"^_ZN5dpfhe%s15ks_fused_kernelILi1[23]ELi256ELi2E"            # every fused instance at N = 4096 and 8192
NS = {"fast": "4fast", "gen": "3gen"}
LDS_PER_CHUNK = 3          # the transform value u and the two accumulator half-rows
CANON_WIDE_PER_CHUNK = 4   # the last digit's canonicalisation: one word_reduce (one IMAD.WIDE) per value
PRODUCTS_PER_CHUNK = 4
WIDE_PER_PRODUCT = 6       # shoup_lazy (4) + the rebuild of the key word from its companion (2)
LOADS_PER_CHUNK = 2        # key.b and key.a companions
MOV_PER_CHUNK = 24         # IMAD.MOV.U32 register copies per chunk (the loop reading both rows had 27)
INSTR_PER_CHUNK = 216      # the loop reading both rows had 202


def _tool(name):
    for cand in (shutil.which(name), "/usr/local/cuda/bin/" + name):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """the main unit of kernels.cu (DPFHE_PART=1) of both variants, with build.py's flags: (SASS per kernel, ptxas -v log)"""
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if nvcc is None or cuobjdump is None:
        pytest.skip("nvcc / cuobjdump not found")
    d = tmp_path_factory.mktemp("sass_mac")
    procs = {}
    for v, fast in (("fast", 1), ("gen", 0)):
        cubin = str(d / ("kernels_%s.cubin" % v))
        cmd = [nvcc] + dpbuild.NVCC_FLAGS + ["-DDPFHE_FAST=%d" % fast, "-DDPFHE_PART=1", "-Xptxas", "-v", "-cubin", "-x", "cu",
                                os.path.join(dpbuild.CSRC, "kernels.cu"), "-o", cubin]
        procs[v] = (cubin, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    out = {}
    for v, (cubin, p) in procs.items():
        log, _ = p.communicate()
        assert p.returncode == 0, log[-4000:]
        out[v] = (sass_loop.kernels(cubin, cuobjdump), log)
    return out


def _innermost(ins):
    loops = sass_loop.loops(ins)
    inner = [(lo, hi) for lo, hi in loops if not any((a, b) != (lo, hi) and lo <= a and b <= hi for a, b in loops)]
    return [collections.Counter(sass_loop.opcode(t) for a, t in ins if lo <= a <= hi) for lo, hi in sorted(inner)]


def _mac_loop(kernels):
    names = [k for k in kernels if re.search(FUSED, k)]
    assert len(names) == 1, names
    loops = _innermost(kernels[names[0]])
    passes = [k for k, c in enumerate(loops) if c["IMAD.WIDE.U32"] == 128]
    assert len(passes) == 6, "three inverse and three forward register passes"
    # the first loop with products after the forward passes (a small index loop without any may come before it)
    return next(c for c in loops[passes[-1] + 1:] if c["IMAD.WIDE.U32"])


def test_mac_loop_reads_companions_only(compiled):
    kernels, _ = compiled["fast"]
    mac = _mac_loop(kernels)
    assert mac["IMAD.WIDE.U32"] != 128
    assert mac["LDS.128"] % LDS_PER_CHUNK == 0, mac
    chunks = mac["LDS.128"] // LDS_PER_CHUNK
    assert chunks == 2, ("two chunks per iteration", mac)
    loads = sum(v for k, v in mac.items() if k.startswith("LDG.E.128"))
    assert loads == LOADS_PER_CHUNK * chunks, ("128-bit key loads", loads, mac)
    wide = mac["IMAD.WIDE.U32"]
    assert wide == chunks * (PRODUCTS_PER_CHUNK * WIDE_PER_PRODUCT + CANON_WIDE_PER_CHUNK), ("IMAD.WIDE", wide)
    assert mac["IMAD.MOV.U32"] <= MOV_PER_CHUNK * chunks, ("register copies", mac["IMAD.MOV.U32"])
    assert sum(mac.values()) <= INSTR_PER_CHUNK * chunks, ("instructions", sum(mac.values()))


def _ptxas_props(log):
    """kernel -> (registers, stack frame bytes, spill store bytes, spill load bytes)"""
    res, cur, frame = {}, None, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur, frame = m.group(1), None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            frame = tuple(int(x) for x in m.groups())
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and cur and frame is not None:
            res[cur] = (int(m.group(1)),) + frame
            cur = None
    return res


def test_fused_block_instances_registers(compiled):
    for v in ("fast", "gen"):
        props = _ptxas_props(compiled[v][1])
        fused = [k for k in props if re.search(FUSED_BLK % NS[v], k)]
        assert len(fused) == 10, (v, fused)   # five modes / profiling instances at each of N = 4096, 8192
        for k in fused:
            regs, frame, st, ld = props[k]
            assert regs <= 128 and (frame, st, ld) == (0, 0, 0), (k, props[k])
