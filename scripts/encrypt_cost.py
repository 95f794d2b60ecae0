"""What encrypting a stored unencrypted segment costs with tsgpu_encrypt_object against tsgpu_rewrite_object: a 1 GiB Kafka
segment with corpus-K record payloads (tests/records_util.py) in 4 MiB chunks, pinned host buffers, 4 chunks per slot batch, 64 MiB
upload parts.  Stored objects: Zstd-only written by this library in speed and in dense mode and by the oracle (libzstd level 3:
what the Java plugin wrote), and plain.  Each is encrypted by tsgpu_encrypt_object and by tsgpu_rewrite_object (to the same
compression with AES added, frames kept), the two alternating in one process.  Prints one JSON line:
  e2e_gib_s         GiB/s of original (segment) bytes per call: median, min, max over the repeats
  e2e_obj_gib_s     GiB/s of source object bytes per call, the same way
  pcie_bytes_per_object_byte   bytes the call copies over PCIe per object byte, from its copies: the object in and the new
                    object out (28 bytes more per chunk; descriptor blocks, sizes and checksum words are below 0.01 %)
  kernel_ms         ms per GiB of original bytes of every kernel of one call (per-kernel CUDA events of tsgpu_profile_report, in
                    one separate profiled run)
  gpu, power_limit_w   the card the numbers were taken on, read in the same call
Usage: python scripts/encrypt_cost.py [--repeats 5] [--out FILE]"""
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


def stats(x, nd=2):
    return {"median": round(statistics.median(x), nd), "min": round(min(x), nd), "max": round(max(x), nd)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("encrypt_cost.py measures on a GPU; none is visible")
    C = binding.C
    lib = binding.load()
    ctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    seg = R.gen_segment(5, SEG - MIB, payload=corpus.gen_segment("K", 5, 64 * MIB, MIB), big=64 << 10)
    n = seg.size
    nch = (n + CS - 1) // CS
    key, aad, ivs = corpus.fixed_key_material(nch)
    nk, na, nivs = W.new_key_material(nch)
    nk8, na8, niv8 = (np.frombuffer(x, np.uint8) for x in (nk, na, nivs))
    cap = nch * (int(lib.tsgpu_transform_bound(Z | A, CS, CS)) + 32) + 64
    new_dst = pinned(cap)
    nsz = np.zeros(nch + 1, np.uint32)
    crcs = np.zeros(cap // PART + 2, np.uint32)
    pcur = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)

    def own(flags):
        pcur[:] = 0
        obj, sizes, _, _ = ctx.transform_parts(flags, seg, CS, PART, pcur, True, np.zeros(binding.CURSOR_SIZE, np.uint8), key, aad, ivs)
        return obj, sizes

    objects = {
        "speed": (Z, own(Z)),
        "dense": (Z, own(Z | D)),
        "libzstd": (Z, ora.transform_segment(Z, seg, CS, key, aad, ivs)),
        "plain": (0, (seg, [min(CS, n - i) for i in range(0, n, CS)])),
    }
    gib = n / (1 << 30)
    res = {"segment_bytes": n, "chunk_mib": CS // MIB, "part_mib": PART // MIB, "max_batch": 4,
           "corpus": "K payloads in Kafka record batches", "repeats": args.repeats, "target": "same compression, encryption added",
           "object_bytes": {}, "e2e_gib_s": {}, "e2e_obj_gib_s": {}, "pcie_bytes_per_object_byte": {"encrypt": 2.0, "rewrite": 2.0},
           "kernel_ms": {}}
    for mode, (flags, (obj_, sizes_)) in objects.items():
        obj = pinned(obj_.size)
        obj[:] = obj_
        sizes = np.asarray(sizes_, np.uint32)
        ogib = obj.size / (1 << 30)
        res["object_bytes"][mode] = int(obj.size)
        ecur = np.zeros(binding.ENCRYPT_CURSOR_SIZE, np.uint8)
        rcur = np.zeros(binding.REWRITE_CURSOR_SIZE, np.uint8)
        w = [C.c_uint32(0) for _ in range(4)]

        def encrypt():
            ecur[:] = 0
            rc = lib.tsgpu_encrypt_object(ctx.handle, flags, obj.ctypes.data, obj.size, sizes.ctypes.data, sizes.size, CS, n,
                                          nk8.ctypes.data, na8.ctypes.data, na8.size, niv8.ctypes.data, new_dst.ctypes.data,
                                          new_dst.size, nsz.ctypes.data, PART, crcs.ctypes.data, crcs.size, C.addressof(w[0]),
                                          ecur.ctypes.data, 1, C.addressof(w[1]), C.addressof(w[2]))
            if rc:
                raise tsgpu.TsgpuError(rc, lib.tsgpu_last_error().decode())

        def rewrite():
            rcur[:] = 0
            rc = lib.tsgpu_rewrite_object(ctx.handle, flags, obj.ctypes.data, obj.size, sizes.ctypes.data, sizes.size, CS, n,
                                          None, None, 0, flags | A, nk8.ctypes.data, na8.ctypes.data, na8.size,
                                          niv8.ctypes.data, new_dst.ctypes.data, new_dst.size, nsz.ctypes.data, PART,
                                          crcs.ctypes.data, crcs.size, C.addressof(w[0]), rcur.ctypes.data, 1, C.addressof(w[1]),
                                          C.addressof(w[2]), C.addressof(w[3]))
            if rc:
                raise tsgpu.TsgpuError(rc, lib.tsgpu_last_error().decode())

        calls = {"encrypt": encrypt, "rewrite": rewrite}
        secs = {k: [] for k in calls}
        for rep in range(args.repeats + 2):
            for name, fn in calls.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                if rep >= 2:
                    secs[name].append(dt)
        res["e2e_gib_s"][mode] = {k: stats([gib / t for t in v]) for k, v in secs.items()}
        res["e2e_obj_gib_s"][mode] = {k: stats([ogib / t for t in v]) for k, v in secs.items()}
        res["kernel_ms"][mode] = {}
        for name, fn in calls.items():
            ctx.profile_enable(True)
            fn()
            rep_ = ctx.profile_report()
            ctx.profile_enable(False)
            ks = {k: round(v["ms"] / gib, 3) for k, v in rep_.items()}
            ks["all_kernels"] = round(sum(v["ms"] for v in rep_.values()) / gib, 3)
            res["kernel_ms"][mode][name] = ks
    ctx.close()
    res["gpu"], res["power_limit_w"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
