#!/usr/bin/env python
"""Writes tests/golden/speed_frames.json: digests of the speed-mode frames (TSGPU_FLAG_ZSTD, independent 8 KiB blocks) that
the product's compressor writes under the test-only SIMT emulator.  On a GPU, which lane wins a hash slot varies from run to
run, so speed-mode frames are not a function of the input there; the emulator runs lanes in a fixed order, so there they are.
The digests pin the entropy stage's output: a change to it that alters a code length, a code or a table shows up.
Run from the repo root: `python tests/golden/make_speed_golden.py [--lib path/to/libtsgpu_simt.so]`."""
import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
HERE = os.path.dirname(os.path.abspath(__file__))

# (corpus, seed, segment bytes, chunk bytes): 1 to 4 chunks, whole and ragged last chunks and blocks, a chunk below the
# Huffman threshold, and the R corpus, whose byte values above 128 need FSE-compressed Huffman weights
SPEED_CASES = (("K", 31, 8192, 8192), ("K", 32, 2 * 65536, 65536), ("K", 33, 3 * 32768 + 4097, 32768),
               ("K", 34, 4 * 65536, 65536), ("K", 35, 100, 100), ("R", 36, 40000, 40000), ("R", 37, 3 * 16384 + 17, 16384),
               ("Z", 38, 70000, 32768), ("Z", 39, 4 * 16384, 16384))


def speed_digests(ctx):
    import tsgpu
    from tsgpu import corpus
    got = []
    for kind, seed, n, cs in SPEED_CASES:
        src = corpus.gen_segment(kind, seed, n, cs)
        out, sizes = ctx.transform(tsgpu.FLAG_ZSTD, src, cs)
        got.append({"kind": kind, "seed": seed, "n": n, "chunk_size": cs, "sizes": [int(x) for x in sizes],
                    "sha256": hashlib.sha256(out.tobytes()).hexdigest()})
    return got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so"))
    args = ap.parse_args()
    import tsgpu
    if args.lib == os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so"):
        subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so"])
    ctx = tsgpu.Context(max_chunk_bytes=1 << 17, max_batch=4, lib_path=args.lib)
    doc = {"generator": "the product's speed-mode compressor (TSGPU_FLAG_ZSTD) under the test-only SIMT emulator, "
                        "tests/golden/make_speed_golden.py", "cases": speed_digests(ctx)}
    ctx.close()
    with open(os.path.join(HERE, "speed_frames.json"), "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")
    print("wrote", len(doc["cases"]), "speed-frame digests")


if __name__ == "__main__":
    main()
