"""Counts SASS opcodes inside the innermost loops of a kernel (developer tool).
usage: sass_loop.py <cubin-or-so> <kernel-name-regex> [per]   (per = divide counts by this number)"""
import collections, re, subprocess, sys

def kernels(path, cuobjdump="cuobjdump"):
    out = subprocess.run([cuobjdump, "-sass", path], capture_output=True, text=True).stdout
    cur, res = None, {}
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1); res[cur] = []; continue
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
        if m and cur:
            res[cur].append((int(m.group(1), 16), m.group(2).strip()))
    return res

def loops(ins):
    out = []
    for addr, txt in ins:
        m = re.search(r"BRA(?:\.U)?\s+(?:\S+,\s*)?(0x[0-9a-f]+)", txt)
        if m and int(m.group(1), 16) < addr:
            out.append((int(m.group(1), 16), addr))
    return out

def opcode(txt):
    t = txt.split()
    return t[1] if t[0].startswith("@") else t[0]

if __name__ == "__main__":
    path, pat = sys.argv[1], sys.argv[2]
    per = float(sys.argv[3]) if len(sys.argv) > 3 else 1.0
    for name, ins in kernels(path).items():
        if not re.search(pat, name):
            continue
        print("==", name[:90], len(ins), "instructions")
        for lo, hi in loops(ins):
            body = [t for a, t in ins if lo <= a <= hi]
            c = collections.Counter(opcode(t) for t in body)
            cost = sum(v * (2.55 if k.startswith("IMAD.WIDE") else 5.8 if k.startswith("IMAD.HI") else 2.0 if k.startswith("IMAD") else 1.27) for k, v in c.items())
            print("  loop %#x-%#x: %d instr (%.2f per unit), est. cost %.1f clk/unit" % (lo, hi, len(body), len(body) / per, cost / per))
            print("   ", {k: round(v / per, 2) for k, v in c.most_common()})
