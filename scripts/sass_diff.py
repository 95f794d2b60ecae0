"""Per-kernel SASS of two libtsgpu.so builds (cuobjdump -sass), compared with symbol names stripped: every kernel of the first
build against the same kernel of the second (the part-checksum kernels gained the CRC word as their first template argument, so
pcrc_tiles_kernel<false> of an older build is compared with pcrc_tiles_kernel<unsigned int, false>), then the kernels only the
second build has.  An optional regex limits the comparison to kernels whose demangled name matches.
Usage: python scripts/sass_diff.py OLD.so NEW.so [REGEX]"""
import re, subprocess, sys, collections
def kernels(so):
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    ks = collections.OrderedDict(); name = None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m: name = m.group(1); ks[name] = []; continue
        if name and re.search(r"/\*[0-9a-f]{4}\*/", line):
            ins = re.sub(r"/\*[0-9a-f]{4}\*/", "", line).split(";")[0].strip()
            ins = re.sub(r"_Z\w+", "SYM", ins)
            ks[name].append(ins)
    return ks
def demangle(n):
    return subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()
a, b = kernels(sys.argv[1]), kernels(sys.argv[2])
pat = sys.argv[3] if len(sys.argv) > 3 else ""
da = {demangle(k): v for k, v in a.items()}
db = {demangle(k): v for k, v in b.items()}
# map parent names to branch names: pcrc kernels gained the word type as first template argument
def to_branch(n):
    if "pcrc_" in n:
        n = re.sub(r"pcrc_(tiles|cuts)_kernel<(true|false)>", r"pcrc_\1_kernel<unsigned int, \2>", n)
        n = n.replace("ts::PcrcSlotsArgs,", "ts::PcrcSlotsArgs<unsigned int>,").replace("ts::PcrcArgs>", "ts::PcrcArgs<unsigned int> >")
    return n
same = diff = 0
for n, v in da.items():
    if pat and not re.search(pat, n): continue
    nb = to_branch(n)
    if nb not in db: print("MISSING in branch:", n); diff += 1; continue
    if db[nb] == v: same += 1
    else:
        diff += 1; print("DIFFERS:", n, len(v), len(db[nb]))
print("compared %d kernels: %d identical, %d differ" % (same + diff, same, diff))
new = [n for n in db if n not in {to_branch(x) for x in da}]
print("new in branch:", *new, sep="\n  ")
