"""Static SASS of one LZ parse step of the speed-mode compressor (`zstd_enc_blocks_kernel`), on any CPU box.

    python scripts/parse_step_sass.py [--src DIR] [--parts SPEC] [--keep FILE] [--list]

Compiles `csrc/tsgpu.cu` to a cubin with the Makefile's flags (sm_90a, -O3, -lineinfo), disassembles it with
`nvdisasm -gi` and charges every instruction of the kernel's parse loop to the source line it comes from (the line in
`zstd_enc_blk.cuh` an inlined helper was called from).  The parts of the step are the `// step: NAME` markers inside the
parse loop of `zstd_enc_blk.cuh`: a part runs from its marker to the next one.  `walk` is executed once per taken match,
`long` only for matches that reach the end of the per-lane measurement; the other parts run once per step.  Prints the
static instruction count of each part, the per-step formula for the path without a long match, and the kernel's
registers, spills and stack frame from `ptxas -v`.

`--parts` replaces the markers by explicit line ranges (for a tree without them), e.g.
`--parts probe=293-331,select=346-355,walk=356-358+390-393,long=359-389,tail=394-409,literals=411-417`.
`--list` prints the step's SASS with the part of every instruction."""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = "tiered-storage-for-apache-kafka_b200"
KERNEL = "_ZN2ts22zstd_enc_blocks_kernelENS_11ZstdBlkArgsE"
BLK = "zstd_enc_blk.cuh"
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "--expt-relaxed-constexpr",
              "-Xptxas", "-v"]
PER_STEP = ("probe", "select", "tail", "literals")


def parts_from_markers(path):
    """{name: set(lines)} from the `// step: NAME` markers; the last marker (`end`) closes the last part."""
    marks = []
    with open(path) as f:
        for i, line in enumerate(f, 1):
            m = re.search(r"//\s*step:\s*(\w+)", line)
            if m:
                marks.append((i, m.group(1)))
    if not marks:
        raise SystemExit("%s has no `// step:` markers; pass --parts" % path)
    parts = {}
    for (a, name), (b, _) in zip(marks, marks[1:]):
        parts.setdefault(name, set()).update(range(a, b))
    return parts


def parts_from_spec(spec):
    parts = {}
    for item in spec.split(","):
        name, ranges = item.split("=")
        for r in ranges.split("+"):
            a, _, b = r.partition("-")
            parts.setdefault(name, set()).update(range(int(a), int(b or a) + 1))
    return parts


def kernel_sass(cubin):
    """[(address, source line in zstd_enc_blk.cuh or None, text)] of the kernel, in address order."""
    out = subprocess.run(["nvdisasm", "-gi", cubin], check=True, capture_output=True, text=True).stdout
    rows, inside, line = [], False, None
    for s in out.splitlines():
        if s.startswith(".text."):
            inside = s.strip() == ".text.%s:" % KERNEL
            continue
        if not inside:
            continue
        if "//##" in s:
            # the caller's line when the annotation is an inlined helper's, else the line itself
            hits = re.findall(r'File "([^"]+)", line (\d+)', s)
            blk = [int(n) for f, n in hits if f.endswith(BLK)]
            line = blk[-1] if blk else None
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", s)
        if m:
            rows.append((int(m.group(1), 16), line, m.group(2)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default=ROOT, help="tree to compile (default: this one)")
    ap.add_argument("--parts", default=None, help="name=a-b[+c-d],... instead of the source markers")
    ap.add_argument("--keep", default=None, help="also write the cubin here")
    ap.add_argument("--list", action="store_true")
    args = ap.parse_args()
    csrc = os.path.join(args.src, PKG, "csrc")
    parts = parts_from_spec(args.parts) if args.parts else parts_from_markers(os.path.join(csrc, BLK))
    owner = {ln: name for name, lines in parts.items() for ln in lines}

    with tempfile.TemporaryDirectory() as tmp:
        cubin = args.keep or os.path.join(tmp, "tsgpu.cubin")
        p = subprocess.run(["nvcc", *NVCC_FLAGS, "-cubin", "-o", cubin, os.path.join(csrc, "tsgpu.cu")],
                           capture_output=True, text=True)
        if p.returncode:
            sys.stderr.write(p.stderr)
            raise SystemExit("nvcc failed")
        rows = kernel_sass(cubin)
    ptx = p.stderr.split(KERNEL)
    regs = re.search(r"Used (\d+) registers", ptx[2] if len(ptx) > 2 else "")
    frame = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ptx[2] if len(ptx) > 2 else "")

    # the parse loop: from the first instruction of a part to the first one after it that belongs to a later line
    # (code the compiler moved out of line, e.g. the divergent-warp fallbacks at the kernel's end, is left out)
    last = max(owner)
    first = next(i for i, r in enumerate(rows) if r[1] in owner)
    end = next((i for i in range(first, len(rows)) if rows[i][1] is not None and rows[i][1] > last), len(rows))
    counts = {name: 0 for name in parts}
    other = 0
    for addr, ln, text in rows[first:end]:
        name = owner.get(ln)
        if name:
            counts[name] += 1
        else:
            other += 1
        if args.list:
            print("%6x %5s %-9s %s" % (addr, ln, name or "-", text))
    once = sum(counts.get(n, 0) for n in PER_STEP)
    walk = counts.get("walk", 0)
    print("part        SASS instructions (static)")
    for name in parts:
        print("%-10s  %4d%s" % (name, counts[name], "  per taken match" if name == "walk" else
                                  "  long matches only" if name == "long" else ""))
    print("%-10s  %4d  (lines outside the parts, e.g. the loop test; not in the total)" % ("other", other))
    print("one step, no long match: %d + %d*k  (k taken matches; %d at k = 3)" % (once, walk, once + 3 * walk))
    if regs and frame:
        print("zstd_enc_blocks_kernel: %s registers, %s-byte stack frame, spill stores %s, spill loads %s"
              % (regs.group(1), frame.group(1), frame.group(2), frame.group(3)))


if __name__ == "__main__":
    main()
