"""What CRC-64/NVME part and object checksums cost next to CRC-32C, alternating in one process on a 1 GiB corpus-K segment in
4 MiB chunks, host buffers (pinned):
  upload  tsgpu_transform_cursor (no checksum), tsgpu_transform_parts (CRC-32C) and tsgpu_transform_parts_crc64 (CRC-64/NVME),
          5 MiB parts, for Zstd+AES in speed and dense mode and AES alone
  check   tsgpu_check_object and tsgpu_check_object_crc64 on the Zstd+AES object
Prints one JSON line:
  e2e        GiB/s of original bytes per call: median, min, max over the repeats; for the uploads each checksum's throughput as
             a share of tsgpu_transform_cursor's, for the check CRC-64's as a share of CRC-32C's
  kernel_ms  ms per GiB of original bytes of each checksum kernel (pcrc_* / pcrc64_*) and of all kernels of the call (per-kernel
             CUDA events of tsgpu_profile_report, in one separate profiled run per call)
  gpu, power_limit_w  the card the numbers were taken on, read in the same call
Usage: python scripts/crc64_cost.py [--repeats 7] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import binding, corpus  # noqa: E402

C = binding.C
MIB = 1 << 20
CS = 4 * MIB
SEG = 1024 * MIB
PART = 5 * MIB
Z, A, D = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE
MODES = {"ZA_speed": Z | A, "ZA_dense": Z | D | A, "A": A}
UPLOADS = ("off", "crc32c", "crc64")


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


def upload(lib, ctx, kind, flags, src, key, aad, ivs, dst, sizes):
    """one whole-segment call; the pinned dst and the size array are allocated once"""
    n = C.c_uint32(sizes.size)
    rcur = np.zeros(binding.CURSOR_SIZE, np.uint8)
    args = [ctx.handle, flags, src.ctypes.data, src.size, CS, key.ctypes.data, aad.ctypes.data, aad.size, ivs.ctypes.data,
            dst.ctypes.data, dst.size, sizes.ctypes.data, C.addressof(n), rcur.ctypes.data, 1]
    pc = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)                # written by the call: kept alive across it
    if kind == "crc32c":
        crcs = np.zeros(dst.size // PART + 2, np.uint32)
        n_parts, obj = C.c_uint32(0), C.c_uint32(0)
        rc = lib.tsgpu_transform_parts(*args, PART, pc.ctypes.data, crcs.ctypes.data, crcs.size, C.addressof(n_parts),
                                       C.addressof(obj))
    elif kind == "crc64":
        crcs = np.zeros(dst.size // PART + 2, np.uint64)
        n_parts, obj = C.c_uint32(0), C.c_uint64(0)
        rc = lib.tsgpu_transform_parts_crc64(*args, PART, pc.ctypes.data, crcs.ctypes.data, crcs.size, C.addressof(n_parts),
                                             C.addressof(obj))
    else:
        rc = lib.tsgpu_transform_cursor(*args)
    if rc:
        raise tsgpu.TsgpuError(rc, lib.tsgpu_last_error().decode())
    return int(sizes[:n.value].sum(dtype=np.uint64))


def check(lib, ctx, kind, flags, obj, osizes, key, aad):
    word = C.c_uint64 if kind == "crc64" else C.c_uint32
    fn = lib.tsgpu_check_object_crc64 if kind == "crc64" else lib.tsgpu_check_object
    o, s = word(0), word(0)
    cursor = np.zeros(binding.CHECK_CURSOR_SIZE, np.uint8)          # written by the call: kept alive across it
    rc = fn(ctx.handle, flags, obj.ctypes.data, obj.size, osizes.ctypes.data, osizes.size, CS, SEG, key.ctypes.data,
            aad.ctypes.data, aad.size, cursor.ctypes.data, 1, C.addressof(o), C.addressof(s))
    if rc:
        raise tsgpu.TsgpuError(rc, lib.tsgpu_last_error().decode())


def profiled(ctx, fn, prefix):
    ctx.profile_enable(True)
    fn()
    rep = ctx.profile_report()
    ctx.profile_enable(False)
    gib = SEG / (1 << 30)
    ks = {k: round(v["ms"] / gib, 3) for k, v in rep.items() if k.startswith(prefix)}
    ks["all_kernels"] = round(sum(v["ms"] for v in rep.values()) / gib, 3)
    return ks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("crc64_cost.py measures on a GPU; none is visible")
    lib = binding.load()
    ctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    src = pinned(SEG)
    src[:] = corpus.gen_segment("K", 0, SEG, CS)
    nch = (src.size + CS - 1) // CS
    key, aad, ivs = (np.frombuffer(bytes(x), np.uint8) for x in corpus.fixed_key_material(nch))
    dst = pinned(int(lib.tsgpu_transform_bound(Z | A, src.size, CS)) + 64)
    sizes = np.zeros(nch + 1, np.uint32)
    res = {"segment_gib": SEG / (1 << 30), "chunk_mib": CS // MIB, "part_mib": PART // MIB, "corpus": "K", "repeats": args.repeats,
           "e2e": {}, "kernel_ms": {}}
    for mode, flags in MODES.items():
        e2e = {k: [] for k in UPLOADS}
        for rep in range(args.repeats + 2):
            for kind in UPLOADS:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                upload(lib, ctx, kind, flags, src, key, aad, ivs, dst, sizes)
                dt = time.perf_counter() - t0
                if rep >= 2:
                    e2e[kind].append(src.size / dt / (1 << 30))
        st = {k: stats(v, 2) for k, v in e2e.items()}
        res["e2e"][mode] = {"off_gib_s": st["off"], "crc32c_gib_s": st["crc32c"], "crc64_gib_s": st["crc64"],
                            "crc32c_over_off": round(st["crc32c"]["median"] / st["off"]["median"], 4),
                            "crc64_over_off": round(st["crc64"]["median"] / st["off"]["median"], 4)}
        res["kernel_ms"][mode] = {
            "crc32c": profiled(ctx, lambda: upload(lib, ctx, "crc32c", flags, src, key, aad, ivs, dst, sizes), "pcrc_"),
            "crc64": profiled(ctx, lambda: upload(lib, ctx, "crc64", flags, src, key, aad, ivs, dst, sizes), "pcrc64_")}
    # the check, on the Zstd+AES object
    n = upload(lib, ctx, "off", Z | A, src, key, aad, ivs, dst, sizes)
    obj = pinned(n)
    obj[:] = dst[:n]
    osizes = sizes[:nch].copy()
    e2e = {"crc32c": [], "crc64": []}
    for rep in range(args.repeats + 2):
        for kind in e2e:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            check(lib, ctx, kind, Z | A, obj, osizes, key, aad)
            dt = time.perf_counter() - t0
            if rep >= 2:
                e2e[kind].append(SEG / dt / (1 << 30))
    st = {k: stats(v, 2) for k, v in e2e.items()}
    res["e2e"]["check_ZA"] = {"crc32c_gib_s": st["crc32c"], "crc64_gib_s": st["crc64"],
                              "crc64_over_crc32c": round(st["crc64"]["median"] / st["crc32c"]["median"], 4)}
    res["kernel_ms"]["check_ZA"] = {"crc32c": profiled(ctx, lambda: check(lib, ctx, "crc32c", Z | A, obj, osizes, key, aad), "pcrc_"),
                                    "crc64": profiled(ctx, lambda: check(lib, ctx, "crc64", Z | A, obj, osizes, key, aad), "pcrc64_")}
    ctx.close()
    res["gpu"], res["power_limit_w"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
