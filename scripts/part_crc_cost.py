"""What the upload-part checksums of tsgpu_transform_parts cost, off (tsgpu_transform_cursor) and on (tsgpu_transform_parts, 5 MiB
parts) alternating in one process, on a 1 GiB corpus-K segment in 4 MiB chunks, host buffers (pinned), for Zstd+AES in speed and
dense mode and AES alone.  Prints one JSON line:
  e2e        GiB/s of the call: median, min, max over the repeats, and on/off as a ratio of throughputs (1.0 = free)
  kernel_ms  ms per GiB of original bytes of each part-checksum kernel, their total, and all kernels of the call (per-kernel
             CUDA events of tsgpu_profile_report, in one separate profiled run)
  hashed     bytes the kernels hash per original byte (the object's size over the segment's)
  gpu, power_limit_w  the card the numbers were taken on, read in the same call
Usage: python scripts/part_crc_cost.py [--repeats 7] [--out FILE]"""
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

MIB = 1 << 20
CS = 4 * MIB
SEG = 1024 * MIB
PART = 5 * MIB
Z, A, D = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE
MODES = {"ZA_speed": Z | A, "ZA_dense": Z | D | A, "A": A}


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


def call(lib, ctx, flags, src, key, aad, ivs, dst, sizes, on):
    """one whole-segment call; the pinned dst and the size / CRC arrays are allocated once"""
    n = binding.C.c_uint32(sizes.size)
    rcur = np.zeros(binding.CURSOR_SIZE, np.uint8)
    args = [ctx.handle, flags, src.ctypes.data, src.size, CS, key.ctypes.data, aad.ctypes.data, aad.size, ivs.ctypes.data,
            dst.ctypes.data, dst.size, sizes.ctypes.data, binding.C.addressof(n), rcur.ctypes.data, 1]
    if on:
        crcs = np.zeros(dst.size // PART + 2, np.uint32)
        n_parts, obj = binding.C.c_uint32(0), binding.C.c_uint32(0)
        rc = lib.tsgpu_transform_parts(*args, PART, np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8).ctypes.data, crcs.ctypes.data,
                                       crcs.size, binding.C.addressof(n_parts), binding.C.addressof(obj))
    else:
        rc = lib.tsgpu_transform_cursor(*args)
    if rc:
        raise tsgpu.TsgpuError(rc, lib.tsgpu_last_error().decode())
    return int(sizes[:n.value].sum(dtype=np.uint64))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("part_crc_cost.py measures on a GPU; none is visible")
    lib = binding.load()
    ctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    src = pinned(SEG)
    src[:] = corpus.gen_segment("K", 0, SEG, CS)
    nch = (src.size + CS - 1) // CS
    key, aad, ivs = (np.frombuffer(bytes(x), np.uint8) for x in corpus.fixed_key_material(nch))
    dst = pinned(int(lib.tsgpu_transform_bound(Z | A, src.size, CS)) + 64)
    sizes = np.zeros(nch + 1, np.uint32)
    res = {"segment_gib": SEG / (1 << 30), "chunk_mib": CS // MIB, "part_mib": PART // MIB, "corpus": "K", "repeats": args.repeats,
           "e2e": {}, "kernel_ms": {}, "hashed": {}}
    for mode, flags in MODES.items():
        e2e = {False: [], True: []}
        for rep in range(args.repeats + 2):
            for on in (False, True):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                obj = call(lib, ctx, flags, src, key, aad, ivs, dst, sizes, on)
                dt = time.perf_counter() - t0
                if rep >= 2:
                    e2e[on].append(src.size / dt / (1 << 30))
        off, on = stats(e2e[False], 2), stats(e2e[True], 2)
        res["e2e"][mode] = {"off_gib_s": off, "on_gib_s": on, "on_over_off": round(on["median"] / off["median"], 4)}
        res["hashed"][mode] = round(obj / src.size, 4)
        ctx.profile_enable(True)
        call(lib, ctx, flags, src, key, aad, ivs, dst, sizes, True)
        rep_ = ctx.profile_report()
        ctx.profile_enable(False)
        gib = src.size / (1 << 30)
        ks = {k: round(v["ms"] / gib, 3) for k, v in rep_.items() if k.startswith("pcrc_")}
        ks["total"] = round(sum(ks.values()), 3)
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
