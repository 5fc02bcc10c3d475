"""Resource budget of the level layer's instances (DESIGN.md section 4.18) on sm_90a, read from the built libdpfhe.so (no GPU needed:
cuobjdump -res-usage), in both arithmetic variants and at N = 4096, 8192 and 16384:
- rot_apply_grouped_level_kernel (the hoisted multiply-accumulate at a level, one ciphertext per work item) fits the 80 registers of
  __launch_bounds__(256, 3) with no local memory and a stack frame of at most one 8-byte spill slot (none in the fast variant, 8 bytes
  in the generic one; with two ciphertexts per work item, the top-level kernel's split, it spilled 144 to 152 bytes);
- ks_level_horner_kernel (the fused Horner step at a level) uses no local memory and no more registers than the top-level Horner step,
  ks_grouped_kernel<.., KS_ROTATE, ADD = true>."""
import re

import pytest

from test_sass_levels_cpu import _one, usage  # noqa: F401  (usage is a fixture)

KS_ROTATE = 2


def _instances():
    """(level instance, sibling, the level instance's largest stack frame in bytes or None) name patterns"""
    for ns in ("3gen", "4fast"):
        pre = r"^_ZN5dpfhe%s" % ns
        for logn in (12, 13, 14):
            t = r"ILi%dELi256ELi3E" % logn
            yield (pre + r"30rot_apply_grouped_level_kernel" + t + r"Li1EEE", pre + r"24rot_apply_grouped_kernel" + t + r"Li2EEE",
                   0 if ns == "4fast" else 8)
            yield (pre + r"22ks_level_horner_kernel" + t + r"EEv", pre + r"17ks_grouped_kernel" + t + r"Li%dELb1EEE" % KS_ROTATE, None)


def test_every_instance_is_built(usage):  # noqa: F811
    built = [k for k in usage if re.search(r"(rot_apply_grouped_level|ks_level_horner)_kernel", k)]
    assert len(built) == 2 * 3 * 2, sorted(built)


@pytest.mark.parametrize("inst", list(_instances()), ids=lambda p: re.sub(r"\\|\^_ZN5dpfhe", "", p[0]))
def test_registers_and_spills(usage, inst):  # noqa: F811
    lvl, sib = _one(usage, inst[0]), _one(usage, inst[1])
    assert lvl[2] == 0, ("local memory", lvl)
    assert lvl[0] <= 80 and lvl[0] <= sib[0], ("registers", lvl, sib)
    if inst[2] is not None:
        assert lvl[1] <= inst[2], ("stack frame: spills", lvl)
