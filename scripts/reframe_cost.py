"""What TSGPU_FLAG_REFRAME costs in tsgpu_rewrite_object, and what sealed frames cost a reader: a 1 GiB Kafka segment with corpus-K
record payloads (tests/records_util.py) in 4 MiB chunks, pinned host buffers, 4 chunks per slot batch, 64 MiB upload parts.  Sources:
Zstd+AES objects written by this library in speed and in dense mode and by the oracle (libzstd level 3 + OpenSSL: what the Java
plugin wrote).  Each is rewritten to Zstd+AES under a new key with its frames kept, and with REFRAME|CHECKSUM (seal), REFRAME|DENSE
and REFRAME|DENSE|CHECKSUM, the four alternating in one process.  Prints one JSON line:
  e2e         GiB/s of original bytes per call: median, min, max over the repeats
  size_ratio  new object bytes / old object bytes
  kernel_ms   ms per GiB of original bytes of every kernel of one rewrite (per-kernel CUDA events of tsgpu_profile_report, in one
              separate profiled run)
  fetch_16mib ms per tsgpu_detransform of a 16 MiB fetch window (4 chunks) of the libzstd object rewritten with frames kept and
              sealed: median, min, max over the repeats, alternating
  gpu, power_limit_w   the card the numbers were taken on, read in the same call
Usage: python scripts/reframe_cost.py [--repeats 5] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import binding, corpus  # noqa: E402
from oracle import oracle as ora  # noqa: E402
import records_util as R  # noqa: E402
import rewrite_util as W  # noqa: E402

MIB = 1 << 20
CS = 4 * MIB
SEG = 1024 * MIB
PART = 64 * MIB
Z, A, D, CK, RF = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_ZSTD_CHECKSUM, tsgpu.FLAG_REFRAME
TARGETS = {"kept": Z | A, "seal": Z | A | CK | RF, "dense": Z | A | D | RF, "dense_seal": Z | A | D | CK | RF}


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return q[0], float(q[1])
    except Exception:                                    # noqa: BLE001 — the name still comes from torch
        return torch.cuda.get_device_name(0), None


def pinned(n):
    return torch.empty(n, dtype=torch.uint8).pin_memory().numpy()


def stats(x, nd=3):
    return {"median": round(statistics.median(x), nd), "min": round(min(x), nd), "max": round(max(x), nd)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("reframe_cost.py measures on a GPU; none is visible")
    C = binding.C
    lib = binding.load()
    ctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    seg = R.gen_segment(5, SEG - MIB, payload=corpus.gen_segment("K", 5, 64 * MIB, MIB), big=64 << 10)
    n = seg.size
    nch = (n + CS - 1) // CS
    key, aad, ivs = corpus.fixed_key_material(nch)
    nk, na, nivs = W.new_key_material(nch)
    k8, a8, nk8, na8, niv8 = (np.frombuffer(x, np.uint8) for x in (key, aad, nk, na, nivs))
    cap = nch * (int(lib.tsgpu_transform_bound(Z | A, CS, CS)) + 32) + 64
    new_dst = pinned(cap)
    nsz = np.zeros(nch + 1, np.uint32)
    crcs = np.zeros(cap // PART + 2, np.uint32)
    objects = {
        "speed": ctx.transform(Z | A, seg, CS, key, aad, ivs),
        "dense": ctx.transform(Z | D | A, seg, CS, key, aad, ivs),
        "libzstd": ora.transform_segment(Z | A, seg, CS, key, aad, ivs),
    }
    gib = n / (1 << 30)
    res = {"segment_bytes": n, "chunk_mib": CS // MIB, "part_mib": PART // MIB, "max_batch": 4,
           "corpus": "K payloads in Kafka record batches", "repeats": args.repeats, "target": "ZA, new key",
           "e2e": {}, "size_ratio": {}, "kernel_ms": {}}
    kept_windows = {}
    for mode, (obj_, sizes_) in objects.items():
        obj = pinned(obj_.size)
        obj[:] = obj_
        sizes = np.asarray(sizes_, np.uint32)
        rcur = np.zeros(binding.REWRITE_CURSOR_SIZE, np.uint8)
        w = [C.c_uint32(0) for _ in range(4)]

        def rewrite(tf):
            rcur[:] = 0
            rc = lib.tsgpu_rewrite_object(ctx.handle, Z | A, obj.ctypes.data, obj.size, sizes.ctypes.data, sizes.size, CS, n,
                                          k8.ctypes.data, a8.ctypes.data, a8.size, tf, nk8.ctypes.data, na8.ctypes.data, na8.size,
                                          niv8.ctypes.data, new_dst.ctypes.data, new_dst.size, nsz.ctypes.data, PART,
                                          crcs.ctypes.data, crcs.size, C.addressof(w[0]), rcur.ctypes.data, 1, C.addressof(w[1]),
                                          C.addressof(w[2]), C.addressof(w[3]))
            if rc:
                raise tsgpu.TsgpuError(rc, lib.tsgpu_last_error().decode())
            return int(nsz[:nch].sum(dtype=np.uint64))

        e2e = {k: [] for k in TARGETS}
        for rep in range(args.repeats + 2):
            for name, tf in TARGETS.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                rewrite(tf)
                dt = time.perf_counter() - t0
                if rep >= 2:
                    e2e[name].append(gib / dt)
        res["e2e"][mode] = {k: stats(v, 2) for k, v in e2e.items()}
        res["size_ratio"][mode], res["kernel_ms"][mode] = {}, {}
        for name, tf in TARGETS.items():
            new_len = rewrite(tf)
            res["size_ratio"][mode][name] = round(new_len / obj.size, 4)
            if mode == "libzstd" and name in ("kept", "seal"):
                w4 = int(nsz[:4].sum(dtype=np.uint64))
                kept_windows[name] = (new_dst[:w4].copy(), nsz[:4].copy())
            ctx.profile_enable(True)
            rewrite(tf)
            rep_ = ctx.profile_report()
            ctx.profile_enable(False)
            ks = {k: round(v["ms"] / gib, 3) for k, v in rep_.items()}
            ks["all_kernels"] = round(sum(v["ms"] for v in rep_.values()) / gib, 3)
            res["kernel_ms"][mode][name] = ks
    # a reader's 16 MiB fetch window (4 chunks) of the libzstd object, frames kept against sealed
    out = pinned(4 * CS + 64)
    osz = np.zeros(4, np.uint32)
    wins = {}
    for name, (b, s) in kept_windows.items():
        src = pinned(b.size)
        src[:] = b
        wins[name] = (src, s)
    fetch = {k: [] for k in wins}
    for rep in range(10 * args.repeats + 5):
        for name, (src, s) in wins.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rc = lib.tsgpu_detransform(ctx.handle, Z | A, src.ctypes.data, src.size, s.ctypes.data, 4, nk8.ctypes.data,
                                       na8.ctypes.data, na8.size, out.ctypes.data, out.size, osz.ctypes.data)
            if rc:
                raise tsgpu.TsgpuError(rc, lib.tsgpu_last_error().decode())
            if rep >= 5:
                fetch[name].append((time.perf_counter() - t0) * 1e3)
    res["fetch_16mib_ms"] = {k: stats(v) for k, v in fetch.items()}
    ctx.close()
    res["gpu"], res["power_limit_w"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
