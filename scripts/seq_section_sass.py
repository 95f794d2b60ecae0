"""Static SASS of the speed-mode compressor's sequences section (`zb_encode_sequences` in `zstd_enc_blk.cuh`), and the
warp-instructions it issues for a block of given shape, on any CPU box.

    python scripts/seq_section_sass.py [--src DIR] [--nseq 776] [--list]

Compiles `csrc/tsgpu.cu` as `scripts/parse_step_sass.py` does and charges every instruction of `zstd_enc_blocks_kernel` to
the innermost source line in `zstd_enc_blk.cuh` it comes from.  The parts are the `// seq: NAME` markers of that file (a
part runs from its marker to the next one); the non-inlined `ze_build_kind` and `ze_write_ncount` are counted whole.
Trip counts per block: `fill`, `chain_sync` and `pack` run once per tile of 32 sequences, `chain` once per full tile (its
32 steps are unrolled), `chain_tail` once per sequence of the last partial tile (an upper bound: its loop is unrolled),
`ze_build_kind` three times and the rest once; `ze_write_ncount` runs once per block for all three descriptions, on three
lanes at once.  Loops inside `hist`, `desc` and the two functions are counted once, so for those parts the figure is the
static size, not what they issue; the full-tile chains, which hold most of the section's issue, have no hidden loop."""
import argparse
import os
import re
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parse_step_sass import NVCC_FLAGS, PKG, KERNEL, BLK, ROOT  # noqa: E402

FUNCS = {"ze_build_kind": "_ZN2ts13ze_build_kind", "ze_write_ncount": "_ZN2ts15ze_write_ncount"}


def seq_parts(path):
    marks = []
    with open(path) as f:
        for i, line in enumerate(f, 1):
            m = re.search(r"//\s*seq:\s*(\w+)", line)
            if m:
                marks.append((i, m.group(1)))
    if not marks:
        raise SystemExit("%s has no `// seq:` markers" % path)
    owner = {}
    for (a, name), (b, _) in zip(marks, marks[1:]):
        if name != "end":
            owner.update({ln: name for ln in range(a, b)})
    return owner, [n for _, n in marks if n != "end"]


def sections(cubin):
    """{section name: [(innermost-first [(file, line)], text)]}"""
    out = subprocess.run(["nvdisasm", "-gi", cubin], check=True, capture_output=True, text=True).stdout
    secs, cur, loc, stacked = {}, None, [], False
    for s in out.splitlines():
        if s.startswith(".text."):
            cur = s.strip()[6:-1]
            secs[cur] = []
            continue
        if cur is None:
            continue
        m = re.match(r"\$\w+\$(\w+):", s)                   # a non-inlined function placed inside the kernel's section
        if m:
            cur = m.group(1)
            secs[cur] = []
            continue
        if "//##" in s:                                  # an inlined call's lines come innermost first, one per line
            here = [(f, int(n)) for f, n in re.findall(r'"([^"]+)", line (\d+)', s)]
            loc = loc + here if stacked else here
            stacked = True
            continue
        stacked = False
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", s)
        if m:
            secs[cur].append((loc, m.group(2)))
    return secs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default=ROOT)
    ap.add_argument("--nseq", type=int, default=776)
    ap.add_argument("--list", action="store_true")
    args = ap.parse_args()
    csrc = os.path.join(args.src, PKG, "csrc")
    owner, order = seq_parts(os.path.join(csrc, BLK))
    with tempfile.TemporaryDirectory() as tmp:
        cubin = os.path.join(tmp, "tsgpu.cubin")
        p = subprocess.run(["nvcc", *NVCC_FLAGS, "-cubin", "-o", cubin, os.path.join(csrc, "tsgpu.cu")],
                           capture_output=True, text=True)
        if p.returncode:
            sys.stderr.write(p.stderr)
            raise SystemExit("nvcc failed")
        secs = sections(cubin)
    counts = {n: 0 for n in order}
    for loc, text in secs[KERNEL]:
        name = next((owner[ln] for f, ln in loc if f.endswith(BLK) and ln in owner), None)
        if name:
            counts[name] += 1
            if args.list:
                print("%-10s %s" % (name, text))
    for fn, mangled in FUNCS.items():
        counts[fn] = len(next((v for k, v in secs.items() if k.startswith(mangled)), []))
    n = args.nseq
    tiles, full = (n + 31) // 32, n // 32
    trips = {"fill": tiles, "chain": full, "chain_tail": n - 32 * full, "chain_sync": tiles, "pack": tiles,
             "ze_build_kind": 3}
    print("part             static  trips  dynamic (block of %d sequences, %d tiles)" % (n, tiles))
    total = 0
    for name, c in counts.items():
        t = trips.get(name, 1)
        total += c * t
        print("%-15s  %6d  %5d  %7d" % (name, c, t, c * t))
    print("%-15s  %6s  %5s  %7d" % ("total", "", "", total))


if __name__ == "__main__":
    main()
