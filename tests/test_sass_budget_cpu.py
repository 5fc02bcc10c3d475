"""Instruction budget of the transform pass loops on sm_90a (no GPU needed: nvcc cross-compiles, cuobjdump disassembles).

The headline kernel, ks_fused_kernel<13,256,2,KS_MUL_RELIN> (DESIGN.md §4.4), is bound by the integer multiplier pipe (§4.1).
Its forward register passes used to carry a runtime loop per butterfly (the lazy-bound schedule evaluated at run time) and two
IMAD.MOV register copies per Shoup product; the inverse passes carry neither.  Both come back silently from edits to the
shared arithmetic in modarith.cuh / ntt_core.cuh, so the per-group counts of each pass loop (one loop iteration = one 16-point
group, 32 butterflies) are pinned here for the fast variant, together with the register counts and the absence of local
memory.  For the generic variant the ceilings are the counts of the same loops before the forward passes were reworked."""
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

FUSED = r"^_ZN5dpfhe%s15ks_fused_kernelILi13ELi256ELi2ELi0ELb0ELb0EE"   # <13,256,2,KS_MUL_RELIN,PROF=false,FILTER=false>
FUSED_ALL = r"^_ZN5dpfhe%s15ks_fused_kernelILi13ELi256ELi2E"           # every mode and profiling instance at N = 8192
NTT_FWD = r"^_ZN5dpfhe%s10ntt_kernelILi13ELi256ELi3ELb0EE"             # ntt_kernel<13,256,3,fwd>
NS = {"fast": "4fast", "gen": "3gen"}


def _tool(name):
    for cand in (shutil.which(name), "/usr/local/cuda/bin/" + name):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """the main unit of kernels.cu (DPFHE_PART=1) of both variants, with build.py's flags, as cubins + ptxas -v logs"""
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if nvcc is None or cuobjdump is None:
        pytest.skip("nvcc / cuobjdump not found")
    d = tmp_path_factory.mktemp("sass")
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
        out[v] = (sass_loop.kernels(cubin, cuobjdump), _ptxas_props(log))
    return out


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


def _one(kernels, pat):
    names = [k for k in kernels if re.search(pat, k)]
    assert len(names) == 1, (pat, names)
    return kernels[names[0]]


def _innermost_loops(ins):
    """opcode counters of the loops that contain no other loop, in code order"""
    loops = sass_loop.loops(ins)
    inner = [(lo, hi) for lo, hi in loops if not any((a, b) != (lo, hi) and lo <= a and b <= hi for a, b in loops)]
    return [collections.Counter(sass_loop.opcode(t) for a, t in ins if lo <= a <= hi) for lo, hi in sorted(inner)]


def _pass_loops(ins, wide):
    """the radix-16 register pass loops: `wide` IMAD.WIDE.U32 per group (32 butterflies)"""
    return [c for c in _innermost_loops(ins) if c["IMAD.WIDE.U32"] == wide]


def _n(c):
    return sum(c.values())


def test_fused_kernel_fast_pass_loops(compiled):
    kernels, _ = compiled["fast"]
    ins = _one(kernels, FUSED % NS["fast"])
    passes = _pass_loops(ins, 128)
    # code order: inverse passes C, B, A of the digit (phase 1), then forward passes A, B, C of a sibling digit (phase 2)
    assert len(passes) == 6, [_n(c) for c in passes]
    inv, fwd = passes[:3], passes[3:]
    for c, cap in zip(inv, (815, 748, 781)):
        assert _n(c) <= cap, ("inverse pass", _n(c), cap)
    for c in fwd:
        assert _n(c) <= 830, ("forward pass", _n(c))
        assert c["IMAD.MOV.U32"] <= 30, ("forward pass register copies", c["IMAD.MOV.U32"])
        assert c["BRA"] == 1, "the pass body is one basic block (no runtime loop inside)"


def test_fused_kernel_fast_tensor_loop(compiled):
    kernels, _ = compiled["fast"]
    ins = _one(kernels, FUSED % NS["fast"])
    loops = _innermost_loops(ins)
    first_pass = next(k for k, c in enumerate(loops) if c["IMAD.WIDE.U32"] == 128)
    # phase 1 (two coefficients per iteration: four 128-bit products, three Barrett and four Shoup reductions) precedes the passes
    tensor = max(loops[:first_pass], key=lambda c: c["IMAD.WIDE.U32"])
    assert 60 <= tensor["IMAD.WIDE.U32"] <= 68, tensor
    assert tensor["IMAD.MOV.U32"] <= 32, ("tensor loop register copies", tensor["IMAD.MOV.U32"])


def test_ntt_kernel_fast_forward_pass_loops(compiled):
    kernels, _ = compiled["fast"]
    passes = _pass_loops(_one(kernels, NTT_FWD % NS["fast"]), 128)
    assert len(passes) == 3, [_n(c) for c in passes]
    for c in passes:
        assert _n(c) <= 860, ("forward pass", _n(c))
        assert c["LDC.64"] <= 5, ("limb constants re-read from the constant bank", c["LDC.64"])


def test_registers_and_local_memory(compiled):
    for v in ("fast", "gen"):
        _, props = compiled[v]
        fused = [k for k in props if re.search(FUSED_ALL % NS[v], k)]
        assert len(fused) == 5, fused
        for k in fused:
            regs, frame, st, ld = props[k]
            assert regs <= 128 and (frame, st, ld) == (0, 0, 0), (k, props[k])
        regs, frame, st, ld = props[[k for k in props if re.search(NTT_FWD % NS[v], k)][0]]
        assert regs <= 80, (v, regs)
        if v == "fast":
            assert (frame, st, ld) == (0, 0, 0), (frame, st, ld)
        else:
            assert frame <= 8 and st <= 4 and ld <= 4, (frame, st, ld)   # as before the rework


def test_generic_variant_no_larger(compiled):
    """dpfhe::gen (5 IMAD.WIDE per butterfly): the same loops are no larger than before the forward passes were reworked"""
    kernels, _ = compiled["gen"]
    passes = _pass_loops(_one(kernels, FUSED % NS["gen"]), 160)
    assert len(passes) == 6, [_n(c) for c in passes]
    for c, cap in zip(passes, (817, 750, 783, 945, 929, 1043)):
        assert _n(c) <= cap, (_n(c), cap)
    ntt = _pass_loops(_one(kernels, NTT_FWD % NS["gen"]), 160)
    assert len(ntt) == 3
    for c, cap in zip(ntt, (996, 999, 1061)):
        assert _n(c) <= cap, (_n(c), cap)
