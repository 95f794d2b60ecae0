"""What tsgpu_rewrite_object costs against the host route over the same stored object, tsgpu_detransform to a pinned host buffer
followed by tsgpu_transform_parts: a 1 GiB Kafka segment with corpus-K record payloads (tests/records_util.py) in 4 MiB chunks,
pinned host buffers, 4 chunks per slot batch, 64 MiB upload parts, the two routes alternating in one process.  Rewrites:
Zstd+AES to Zstd+AES under a new key, from objects written by this library in speed and in dense mode and by the oracle (libzstd
level 3 + OpenSSL: what the Java plugin wrote), whose frames the rewrite keeps; and a plain object to Zstd+AES (speed mode).
Prints one JSON line:
  e2e        GiB/s of original bytes per call: median, min, max over the repeats, for the rewrite and the host route, and the
             rewrite over the host route as a ratio of throughputs (> 1: the rewrite is faster)
  pcie_bytes_per_byte   bytes that cross PCIe per original byte, computed from the object sizes: the rewrite moves the old and
             the new object; the host route also moves the segment out and back in (a plain object is copied on the host)
  kernel_ms  ms per GiB of original bytes of every kernel of one rewrite (per-kernel CUDA events of tsgpu_profile_report, in one
             separate profiled run)
  gpu, power_limit_w    the card the numbers were taken on, read in the same call
Usage: python scripts/rewrite_cost.py [--repeats 5] [--out FILE]"""
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
Z, A, D = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE


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
        raise SystemExit("rewrite_cost.py measures on a GPU; none is visible")
    C = binding.C
    lib = binding.load()
    ctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    seg = R.gen_segment(5, SEG - MIB, payload=corpus.gen_segment("K", 5, 64 * MIB, MIB), big=64 << 10)
    n = seg.size
    nch = (n + CS - 1) // CS
    key, aad, ivs = corpus.fixed_key_material(nch)
    nk, na, nivs = W.new_key_material(nch)
    k8, a8, nk8, na8, niv8 = (np.frombuffer(x, np.uint8) for x in (key, aad, nk, na, nivs))
    cap = nch * (int(lib.tsgpu_transform_bound(Z | A, CS, CS)) + 28) + 64
    plain_mid, new_dst = pinned(n + 64), pinned(cap)
    osz = np.zeros(nch + 1, np.uint32)
    nsz = np.zeros(nch + 1, np.uint32)
    crcs = np.zeros(cap // PART + 2, np.uint32)
    objects = {
        "ZA_speed": (Z | A, ctx.transform(Z | A, seg, CS, key, aad, ivs)),
        "ZA_dense": (Z | A, ctx.transform(Z | D | A, seg, CS, key, aad, ivs)),
        "ZA_libzstd": (Z | A, ora.transform_segment(Z | A, seg, CS, key, aad, ivs)),
        "plain": (0, (seg, [min(CS, n - i * CS) for i in range(nch)])),
    }
    gib = n / (1 << 30)
    res = {"segment_bytes": n, "chunk_mib": CS // MIB, "part_mib": PART // MIB, "max_batch": 4,
           "corpus": "K payloads in Kafka record batches", "repeats": args.repeats, "target": "ZA speed, new key",
           "e2e": {}, "pcie_bytes_per_byte": {}, "kernel_ms": {}}
    for mode, (ff, (obj_, sizes_)) in objects.items():
        obj = pinned(obj_.size)
        obj[:] = obj_
        sizes = np.asarray(sizes_, np.uint32)
        rcur = np.zeros(binding.REWRITE_CURSOR_SIZE, np.uint8)
        pcur = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)
        w = [C.c_uint32(0) for _ in range(5)]

        def ok(rc):
            if rc:
                raise tsgpu.TsgpuError(rc, lib.tsgpu_last_error().decode())

        def rewrite():
            rcur[:] = 0
            ok(lib.tsgpu_rewrite_object(ctx.handle, ff, obj.ctypes.data, obj.size, sizes.ctypes.data, sizes.size, CS, n,
                                        k8.ctypes.data, a8.ctypes.data, a8.size, Z | A, nk8.ctypes.data, na8.ctypes.data, na8.size,
                                        niv8.ctypes.data, new_dst.ctypes.data, new_dst.size, nsz.ctypes.data, PART,
                                        crcs.ctypes.data, crcs.size, C.addressof(w[0]), rcur.ctypes.data, 1, C.addressof(w[1]),
                                        C.addressof(w[2]), C.addressof(w[3])))
            return int(nsz[:nch].sum(dtype=np.uint64))

        def host_route():
            ok(lib.tsgpu_detransform(ctx.handle, ff, obj.ctypes.data, obj.size, sizes.ctypes.data, sizes.size, k8.ctypes.data,
                                     a8.ctypes.data, a8.size, plain_mid.ctypes.data, plain_mid.size, osz.ctypes.data))
            pcur[:] = 0
            m = C.c_uint32(nch + 1)
            ok(lib.tsgpu_transform_parts(ctx.handle, Z | A, plain_mid.ctypes.data, n, CS, nk8.ctypes.data, na8.ctypes.data,
                                         na8.size, niv8.ctypes.data, new_dst.ctypes.data, new_dst.size, nsz.ctypes.data,
                                         C.addressof(m), None, 1, PART, pcur.ctypes.data, crcs.ctypes.data, crcs.size,
                                         C.addressof(w[0]), C.addressof(w[4])))

        runs = {"rewrite": rewrite, "host_route": host_route}
        e2e = {k: [] for k in runs}
        for rep in range(args.repeats + 2):
            for name, fn in runs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                if rep >= 2:
                    e2e[name].append(gib / dt)
        r = {k: stats(v, 2) for k, v in e2e.items()}
        r["rewrite_over_host_route"] = round(r["rewrite"]["median"] / r["host_route"]["median"], 3)
        res["e2e"][mode] = r
        new_len = rewrite()
        dev = (obj.size + new_len) / n
        host = ((obj.size + n) if ff else 0) / n + (n + new_len) / n
        res["pcie_bytes_per_byte"][mode] = {"rewrite": round(dev, 3), "host_route": round(host, 3)}
        ctx.profile_enable(True)
        rewrite()
        rep_ = ctx.profile_report()
        ctx.profile_enable(False)
        ks = {k: round(v["ms"] / gib, 3) for k, v in rep_.items()}
        ks["all_kernels"] = round(sum(v["ms"] for v in rep_.values()) / gib, 3)
        res["kernel_ms"][mode] = ks
    ctx.close()
    res["gpu"], res["power_limit_w"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
