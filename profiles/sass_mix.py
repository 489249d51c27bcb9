"""Static SASS instruction mix of map_project_fast_kernel (the dominant kernel): `python profiles/sass_mix.py > sass_mix.md`.
Needs the built object lt_mapper_b200/csrc/project.o (cuobjdump works without a GPU).  The hot region is the branch-free "phase 1" of one
keyframe step (4 points: transform, azimuth, ranges, elevation, pixel + certainty, gather issue) plus the 4 decisions of "phase 2"; it is found
as the instruction window from the first FFMA after the per-keyframe constant loads up to the shared-memory queue test that follows the step."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "lt_mapper_b200", "csrc", "project.o")
LOG = OBJ + ".ptxas.log"

CLASSES = [("FP32 arithmetic (FFMA/FMUL/FADD)", r"^(FFMA|FMUL|FADD)\b"), ("FP32 compare / min / max / select", r"^(FSETP|FMNMX|FSEL)\b"),
           ("MUFU (rsq / rcp)", r"^MUFU"), ("integer / logic / convert", r"^(IMAD|IADD|IADD3|LOP3|SHF|LEA|VIMNMX|VIADDMNMX|VIADD|ISETP|SEL|MOV|I2F|F2I|PRMT|POPC|FLO|BREV|HFMA2|UMOV)\b"),
           ("global / constant loads", r"^(LDG|LDC|LDCU|ULDC)"), ("shared memory / atomics", r"^(LDS|STS|ATOMS|ATOMG|REDG|RED)"),
           ("control (BRA / BSSY / BSYNC / WARPSYNC / vote)", r"^(BRA|BSSY|BSYNC|WARPSYNC|VOTE|EXIT|CALL|RET|YIELD|NOP|S2R|S2UR|SHFL|BAR)"), ("uniform datapath", r"^U[A-Z]")]


def kernel_sass(pattern):
    txt = subprocess.run(["cuobjdump", "-sass", OBJ], capture_output=True, text=True, check=True).stdout
    out, on = [], False
    for line in txt.splitlines():
        if "Function :" in line:
            on = pattern in line
            continue
        if on:
            m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(.*?);", line)
            if m:
                ins = m.group(1).strip()
                ins = re.sub(r"^@!?U?P\d+\s+", "", ins)
                out.append(ins)
    return out


def classify(ins):
    op = ins.split()[0]
    for name, rx in CLASSES:
        if re.match(rx, op):
            return name
    return "other (" + op.split(".")[0] + ")"


def main():
    # default: the variant the HD / revert passes run (candidates only, short elevation path, not deferred, guard-padded test image)
    pat = sys.argv[1] if len(sys.argv) > 1 else "map_project_fast_kernelILb1ELb1ELb0ELb1"
    sass = kernel_sass(pat)
    # hot window = one keyframe step of the k loop: the densest cluster of 8 MUFU.RSQ (4 points x 2) marks phase 1; the window runs from
    # the first register-indexed constant load before it (the per-keyframe constants) to the shared-memory queue test after the step
    rsq = [i for i, s in enumerate(sass) if s.startswith("MUFU.RSQ")]
    best = None
    for a in range(len(rsq) - 7):
        span = rsq[a + 7] - rsq[a]
        if best is None or span < best[0]:
            best = (span, rsq[a], rsq[a + 7])
    lo, hi = best[1], best[2]
    first = lo
    for i in range(lo, max(lo - 120, 0), -1):
        if re.match(r"LDCU?(\.64)? .*c\[0x0\]\[U?R\d+\+", sass[i]):
            first = i
    last = next((i for i in range(hi, len(sass)) if sass[i].startswith("LDS")), len(sass))
    win = sass[first:last]
    # phase 1 = up to the last image gather issued before the first decision branch
    cnt = collections.Counter(classify(s) for s in win)
    n_mufu_rsq = sum(1 for s in win if s.startswith("MUFU.RSQ"))
    pts = max(1, n_mufu_rsq // 2)
    print(f"# SASS instruction mix of `{pat}` (static, sm_90a)\n")
    for line in open(LOG):
        if pat in line and "Compiling" in line:
            pass
    regs = [l.strip() for l in open(LOG)] if os.path.exists(LOG) else []
    for i, l in enumerate(regs):
        if pat in l and "Function properties" in l:
            print("`ptxas -v`:", regs[i + 1].strip(), "|", regs[i + 2].replace("ptxas info    :", "").strip(), "\n")
            break
    print(f"Kernel total: {len(sass)} SASS instructions.  One keyframe step of a warp (window of {len(win)} instructions, {pts} points per thread, "
          f"all branches of the rare paths included) by class:\n")
    print("| class | instructions | per point |\n|---|---|---|")
    for name, n in sorted(cnt.items(), key=lambda kv: -kv[1]):
        print(f"| {name} | {n} | {n / pts:.1f} |")
    print(f"| **all** | **{len(win)}** | **{len(win) / pts:.1f}** |")
    # common path: instructions before the first conditional branch of phase 2 + 3 per decision (the warp-uniform branch that sends a keyframe
    # without fast constants to the exact path precedes phase 1 and is part of the straight line)
    br = [i for i, s in enumerate(win) if (s.startswith("BRA") or " BRA " in s) and i > lo - first]
    common = br[0] if br else len(win)
    cc = collections.Counter(classify(s) for s in win[:common])
    print(f"\nStraight-line part before the first decision branch (the work EVERY pair pays): {common} instructions = {common / pts:.1f} per point:\n")
    print("| class | instructions | per point |\n|---|---|---|")
    for name, n in sorted(cc.items(), key=lambda kv: -kv[1]):
        print(f"| {name} | {n} | {n / pts:.1f} |")
    ops = collections.Counter(s.split()[0].split(".")[0] for s in win[:common])
    print("\nOpcodes of that part:", ", ".join(f"{k} {v}" for k, v in ops.most_common()))


if __name__ == "__main__":
    main()
