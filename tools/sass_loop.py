"""Static instruction count of the innermost loops of named kernels, from `cuobjdump -sass` of a built library (no GPU).

    python tools/sass_loop.py gaussian-splatting_b200/libgs_b200.so render_bwd_kernel [more name substrings ...]

For every kernel whose mangled name contains one of the substrings it finds the loops from their back-branches (a BRA
whose target is at or before the branch), merges the back-branches that share one loop head (a `continue` is a second
back-branch to the same head), and prints for each INNERMOST loop (one that contains no other loop head) the number of
instructions from the head to its last back-branch, without the NOP padding, and an opcode histogram.  One pass through
the body of the backward blend loop is one warp on one list entry, so this is the instruction count per (warp, entry)
that the blend kernels' design is judged by (DESIGN.md section 4).
"""
import argparse
import collections
import os
import re
import subprocess
import sys

CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
FUNC = re.compile(r"^\s*Function : (\S+)")
INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
BRA = re.compile(r"^(?:@!?U?P\w+\s+)?BRA(?:\.\w+)*\s+(?:`\(\.L_x_\d+\)|0x([0-9a-f]+))")


def parse(text):
    """{kernel: [(address, instruction text)]}"""
    out, cur = {}, None
    for line in text.splitlines():
        m = FUNC.match(line)
        if m:
            cur = out.setdefault(m.group(1), [])
            continue
        m = INSN.match(line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(2)))
    return out


def opcode(ins):
    s = re.sub(r"^@!?U?P\w+\s+", "", ins)
    return s.split()[0]


def innermost_loops(insns):
    """[(head, end)] address ranges of the innermost loops, end = address of the last back-branch"""
    ends = {}
    for addr, ins in insns:
        m = BRA.match(ins)
        if m and m.group(1):
            tgt = int(m.group(1), 16)
            if tgt < addr:      # (a branch to itself is the trap after the last EXIT, not a loop)
                ends[tgt] = max(ends.get(tgt, addr), addr)
    loops = sorted(ends.items())
    return [(h, e) for h, e in loops if not any(h < h2 <= e for h2, _ in loops if h2 != h)]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("binary", help="shared library or object file with sm_90a code")
    ap.add_argument("names", nargs="+", help="substrings of the mangled kernel names")
    ap.add_argument("--top", type=int, default=12, help="opcodes shown per histogram")
    args = ap.parse_args()
    text = subprocess.run([CUOBJDUMP, "-sass", args.binary], check=True, capture_output=True, text=True).stdout
    kernels = parse(text)
    found = False
    for name in sorted(kernels):
        if not any(s in name for s in args.names):
            continue
        found = True
        insns = kernels[name]
        print(f"{name}: {len(insns)} instructions")
        for head, end in innermost_loops(insns):
            body = [ins for a, ins in insns if head <= a <= end and opcode(ins) != "NOP"]
            hist = collections.Counter(opcode(ins).split(".")[0] for ins in body)
            top = " ".join(f"{op}:{n}" for op, n in hist.most_common(args.top))
            print(f"  loop {head:#06x}-{end:#06x}: {len(body):4d} instructions  {top}")
    if not found:
        sys.exit(f"no kernel matching {args.names} in {args.binary}")


if __name__ == "__main__":
    main()
